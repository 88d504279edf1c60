"""Resident GFKB: ``failures.jsonl`` + a device index kept in sync (SURVEY.md section 8(f) ranks 1-2).

The reference's GFKB service re-reads and re-validates the whole JSONL on every request
(services/gfkb/app.py:49-51,81,106) and refits TF-IDF on it per query (similarity.py:17-18).  ``GfkbStore`` keeps
the records and their device index resident and reproduces the three handlers that touch the hot path:

* ``upsert``   -- services/gfkb/app.py:104-147: a (failure_type, signature_text) pair seen before appends a NEW
  version of the latest matching record (version+1, occurrences+1, app merged, fields evolve), otherwise a new
  ``F-%04d`` record; one JSON line is appended either way.
* ``match`` / ``match_batch`` -- services/gfkb/app.py:79-102: stable sort by score descending, first 5, THEN the
  failure_type filter, mapped to FailureMatch fields.
* ``warn_batch`` -- services/warning_policy/app.py:19-72: signature_text of the request, best match against the
  threshold, the reference's message strings.
* ``purge_apps`` -- services/dashboard/app.py:330-375 on failures.jsonl: the purged app ids leave every record's
  ``affected_apps``, records left with none are dropped, the file is rewritten.  The emptied records' device rows are
  deleted in place (``GfkbIndex.delete_rows`` + a statistics-only finalize) instead of rebuilding the index.

Index layout: a large MAIN segment (text-sorted scan layout, expensive to rebuild) plus a small TAIL segment that
receives upserts.  TF-IDF statistics are global (every append changes N and df of every row), so after an append
epoch both segments get the summed df / N -- the main segment through a statistics-only finalize
(``kv_index_last_finalize_kind`` == 2: idf tables, row norms and chunk minima recomputed on the device, nothing
re-sorted) -- and the tail is folded into the main segment once it grows past ``tail_limit`` rows.  Queries scan
both segments (K1b, float32 candidates); the candidates are re-scored in float64 (K6: summed in the row's own
feature order, so identical rows tie exactly in both segments) and ordered like Python's stable sort.
"""
from __future__ import annotations

import json
import shutil
import threading
from datetime import datetime, timezone
from pathlib import Path
from typing import Any, Callable, Dict, List, Mapping, Optional, Sequence, Tuple

import numpy as np

from .fingerprint import signature_text as _signature_text
from .gfkb import MATCH_LIMIT, _to_match
from . import sidecar as _sidecar
from .similarity import FeatureBatch, GfkbIndex, Vocabulary

CANDIDATES = 16  # float32 candidates per query and segment that get re-scored in float64 (>= MATCH_LIMIT)
MAX_LIMIT = 32   # the fused top-k of the scan holds at most 32 rows per query and segment
MAX_TF = 65535   # largest term frequency a row may hold (kv_index_append rejects more)
MAX_FEATURES = (1 << 26) - 2  # vocabulary capacity of the scan layout (kv_index_finalize rejects more)
PATTERN_NAME = "Citation hallucination without sources"  # services/pattern_detector/app.py:48
AMBIGUITY_RTOL = 4e-6  # float32 scores closer than this (relative) may order differently in float64
EXACT_SORT_MAX = 200_000  # up to this many rows the exact path orders with Python's own stable sort


def stable_top(scores: np.ndarray, limit: int) -> List[int]:
    """``sorted(range(n), key=lambda i: scores[i], reverse=True)[:limit]`` -- the reference's ordering
    (services/gfkb/app.py:88-89: stable, ties keep row order) -- in O(n) for large n."""
    n = len(scores)
    if n <= EXACT_SORT_MAX:
        vals = scores.tolist()
        return sorted(range(n), key=lambda i: vals[i], reverse=True)[:limit]
    if limit <= 0:
        return []
    v = np.partition(scores, n - limit)[n - limit]            # the limit-th largest score
    above = np.flatnonzero(scores > v)                         # fewer than `limit` rows, ascending
    ties = np.flatnonzero(scores == v)[: limit - len(above)]   # the lowest rows of the tie group fill the rest
    idx = np.concatenate([above, ties])
    return idx[np.lexsort((idx, -scores[idx]))].tolist()       # score descending, then row ascending


def ambiguous_candidates(s32: np.ndarray, rows: np.ndarray, limit: int) -> np.ndarray:
    """Per query: could a row that did NOT make a segment's float32 candidate list belong to the float64 top-``limit``?
    Only if the list is full and its last score is within float32 rounding of its ``limit``-th score.  Exact zeros are
    exact in both precisions (integer dot products), and equal float32 scores of identical rows are broken by row id
    exactly like the reference's stable sort -- but two DISTINCT texts whose scores collide in float32 cannot be told
    apart from the candidates alone (ADVICE round 1), so such queries take the exact path."""
    k = s32.shape[1]
    full = rows[:, k - 1] >= 0
    ref = s32[:, min(limit, k) - 1].astype(np.float64)
    last = s32[:, k - 1].astype(np.float64)
    return full & (last > 0.0) & (last >= ref - AMBIGUITY_RTOL * np.abs(ref))


def check_indexable(text: str, vocab_size: int = 0) -> Optional[str]:
    """None when ``text`` can be indexed, else the reason.  Called BEFORE a record is persisted: a row the index
    would reject (a 1- or 2-gram repeated more than 65535 times; a vocabulary past 2^26 features) must never reach
    failures.jsonl, or every later match/warn -- and every restart -- would fail on it (the reference has no such
    limits: these are capacity limits of the scan layout, reported to the caller instead of corrupting the store)."""
    n_tok_max = len(text) // 3 + 1                 # a token is >= 2 word characters + a separator
    if n_tok_max > MAX_TF:                          # only then can any feature repeat that often: count exactly
        import re
        from collections import Counter

        toks = re.findall(r"(?u)\b\w\w+\b", text.lower())
        grams = Counter(toks) + Counter(zip(toks, toks[1:]))
        if grams and max(grams.values()) > MAX_TF:
            return f"a feature of signature_text repeats more than {MAX_TF} times"
    if vocab_size + 2 * n_tok_max >= MAX_FEATURES:
        return f"the vocabulary would exceed its capacity of {MAX_FEATURES} features"
    return None


def _iso(dt: datetime) -> str:
    """pydantic's JSON form of an aware UTC datetime (model_dump(mode="json"), app.py:131,146)."""
    return dt.isoformat().replace("+00:00", "Z")


class GfkbStore:
    def __init__(self, path: Optional[Path] = None, device: int = 0, tail_limit: int = 65536,
                 now: Optional[Callable[[], datetime]] = None, sidecar: Optional[Path] = None):
        self.path = Path(path) if path is not None else None
        # optional binary sidecar (vocabulary + CSR of the rows, kakveda_b200/sidecar.py): a cold start then skips the
        # tokenisation of every stored signature_text; it is rewritten whenever the main segment is rebuilt
        self.sidecar_path = Path(sidecar) if sidecar is not None else None
        self.device = device
        self.tail_limit = int(tail_limit)
        self._now = now or (lambda: datetime.now(timezone.utc))  # app.py:34-35
        self._lock = threading.RLock()
        self._quarantine_set: set = set()
        self.records: List[Dict[str, Any]] = []
        self._latest: Dict[Tuple[str, str], int] = {}  # (failure_type, signature_text) -> index of the newest record
        self.vocab = Vocabulary()
        self._main: Optional[GfkbIndex] = None
        self._tail: Optional[GfkbIndex] = None
        self._n_main = 0          # device rows of the main segment (records[:_n_main] while no row is deleted)
        self._n_indexed = 0       # records[:_n_indexed] are on the device (main + tail)
        self._n_dev = 0           # device rows of main + tail, deleted ones included
        # Device row -> record index, -1 for a deleted row; None: the identity (no deletion since the last rebuild).
        # Deletion removes rows and appends go at the end, so device-row order is monotone in record order: the
        # (score desc, device row asc) order of a search is exactly the reference's stable order over the records.
        self._row2rec: Optional[np.ndarray] = None
        self._n_deleted = 0       # device rows deleted since the last rebuild (past tail_limit the next _sync compacts)
        self._sidecar_rows = 0    # the sidecar file holds the CSR of records[:_sidecar_rows]
        self._main_df: Optional[np.ndarray] = None
        self._dirty = False
        # failure_type -> row label of the device index, numbered in order of first appearance; label of each record
        self._type_ids: Dict[str, int] = {}
        self._labels: List[int] = []
        self.stats = {"full_rebuilds": 0, "stat_refreshes": 0, "compactions": 0, "quarantined": 0}
        self.quarantined: List[int] = []  # indices of loaded records that cannot be indexed (they keep their row, with no features)
        if self.path is not None and self.path.exists():
            self.load()

    # -- storage ---------------------------------------------------------------------------------------------
    def load(self) -> None:
        """Read the JSONL (app.py:38-46) and build the main segment from it."""
        with self._lock:
            rows = []
            if self.path is not None and self.path.exists():
                for line in self.path.read_text(encoding="utf-8").splitlines():
                    if line.strip():
                        rows.append(json.loads(line))
            self._reset(rows)

    def _index_text(self, i: int) -> str:
        """The text record i is indexed under: its signature_text, or '' (a row that matches nothing) when a record
        written by another program cannot be indexed -- the store stays usable and the record keeps its row id."""
        return "" if i in self._quarantine_set else self.records[i]["signature_text"]

    def _reset(self, rows: List[Dict[str, Any]]) -> None:
        self.records = list(rows)
        self.quarantined = [i for i, r in enumerate(self.records) if check_indexable(r["signature_text"]) is not None]
        self._quarantine_set = set(self.quarantined)
        self.stats["quarantined"] = len(self.quarantined)
        self._latest = {}
        for i, r in enumerate(self.records):
            self._latest[(r["failure_type"], r["signature_text"])] = i
        self._type_ids, self._labels = {}, []
        self._rebuild_main()

    def _row_labels(self, lo: int, hi: int) -> np.ndarray:
        """int32 row labels of records[lo:hi]: their failure types, numbered in order of first appearance."""
        for r in self.records[len(self._labels):hi]:
            self._labels.append(self._type_ids.setdefault(r["failure_type"], len(self._type_ids)))
        return np.asarray(self._labels[lo:hi], dtype=np.int32)

    def _rebuild_main(self) -> None:
        for ix in (self._main, self._tail):
            if ix is not None:
                ix.close()
        self._main = self._tail = None
        self._main_df = None
        n = len(self.records)
        if n:
            texts = [self._index_text(i) for i in range(n)]
            # the sidecar only serves a cold start (empty vocabulary); a compaction does not re-read and re-digest it
            cold = self.sidecar_path is not None and len(self.vocab) == 0
            cached = _sidecar.load(self.sidecar_path, texts) if cold else None
            if cached is not None:
                # cold start from the sidecar: the vocabulary and the first n0 rows come back as arrays
                self.vocab.close()
                self.vocab, head, n0 = cached
                self._main = GfkbIndex(device=self.device, row_base=0, vocab=self.vocab)
                self._main.add_features(head)
                self.stats["sidecar_rows"] = n0
                if n0 < n:
                    rest = self.vocab.featurize(texts[n0:], grow=True)
                    try:
                        self._main.add_features(rest)
                        if self.sidecar_path is not None:
                            both = _sidecar.ArrayBatch(np.concatenate([head.indptr, rest.indptr[1:] + head.indptr[-1]]),
                                                       np.concatenate([head.ids, rest.ids]), np.concatenate([head.tf, rest.tf]))
                            _sidecar.save(self.sidecar_path, self.vocab, both, texts)
                    finally:
                        rest.close()
            else:
                self._main = GfkbIndex(device=self.device, row_base=0, vocab=self.vocab)
                fb = self.vocab.featurize(texts, grow=True)
                try:
                    self._main.add_features(fb)
                    if self.sidecar_path is not None:
                        _sidecar.save(self.sidecar_path, self.vocab, fb, texts)
                finally:
                    fb.close()
            # persisted scan layout next to the sidecar: a cold start then skips the host sort + block build as well
            lay_path = Path(str(self.sidecar_path) + ".layout") if self.sidecar_path is not None else None
            restored = lay_path is not None and self._main.load_layout(lay_path)
            self._main.finalize()
            if restored and self._main.last_finalize_kind == 2:
                self.stats["layout_restored"] = self.stats.get("layout_restored", 0) + 1
            elif lay_path is not None:
                self._main.save_layout(lay_path)
            self._main.set_row_labels(self._row_labels(0, n))
            self.stats["full_rebuilds"] += 1
        self._n_main = self._n_indexed = self._n_dev = n
        self._sidecar_rows = n if self.sidecar_path is not None else 0  # the sidecar holds the CSR of records[:n]
        self._row2rec = None
        self._n_deleted = 0
        self._dirty = False

    def _dev_labels(self, n_dev: int) -> np.ndarray:
        """int32 failure-type label of the first ``n_dev`` device rows (main + tail), -1 for a deleted row."""
        if self._row2rec is None:
            return self._row_labels(0, n_dev)
        rec_labels = self._row_labels(0, self._n_indexed)
        out = np.full(n_dev, -1, dtype=np.int32)
        live = self._row2rec >= 0
        out[live] = rec_labels[self._row2rec[live]]
        return out

    def _to_records(self, rows: np.ndarray) -> np.ndarray:
        """Device rows -> record indices (-1 stays -1)."""
        if self._row2rec is None:
            return rows
        return np.where(rows >= 0, self._row2rec[np.clip(rows, 0, None)], -1)

    def _sync(self) -> None:
        """Bring the device index up to date with ``records`` (called lazily before a query)."""
        if not self._dirty and self._n_indexed == len(self.records):
            return
        pending = [self._index_text(i) for i in range(self._n_indexed, len(self.records))]
        n_tail = self._n_dev - self._n_main + len(pending)
        if self._main is None or n_tail > max(self.tail_limit, 0) or self._n_deleted > max(self.tail_limit, 0):
            self.stats["compactions"] += self._main is not None
            self._rebuild_main()
            return
        if self._tail is None and pending:  # a deletion alone needs no tail segment
            self._tail = GfkbIndex(device=self.device, row_base=self._n_main, vocab=self.vocab)
        if pending:
            self._tail.add_texts(pending)
            if self._row2rec is not None:
                self._row2rec = np.concatenate([self._row2rec, np.arange(self._n_indexed, len(self.records), dtype=np.int64)])
        self._n_dev += len(pending)
        self._n_indexed = len(self.records)
        segments = [ix for ix in (self._main, self._tail) if ix is not None]
        if self._tail is not None:
            tail_labels = self._dev_labels(self._n_dev)[self._n_main:]
            self._tail.set_row_labels(np.maximum(tail_labels, 0))  # an append dropped them; a deleted row's label is moot
        # global statistics = main + tail (the df all-reduce of a sharded GFKB, done in-process)
        v = len(self.vocab)
        if self._main_df is None:
            self._main_df = self._main.local_df().astype(np.int64)
        df = np.zeros(v, dtype=np.int64)
        df[: len(self._main_df)] = self._main_df
        if self._tail is not None:
            df += self._tail.local_df().astype(np.int64)
        df32 = df.astype(np.uint32)
        for ix in segments:
            ix.set_global_df(df32, len(self.records))
            ix.finalize()
        if self._main.last_finalize_kind == 2:
            self.stats["stat_refreshes"] += 1
        else:
            self.stats["full_rebuilds"] += 1
        self._dirty = False

    # -- upsert (services/gfkb/app.py:104-147) -----------------------------------------------------------------
    def upsert(self, req: Mapping[str, Any]) -> Dict[str, Any]:
        with self._lock:
            why = check_indexable(req["signature_text"], len(self.vocab))
            if why is not None:  # refuse BEFORE anything is persisted
                raise ValueError(f"upsert rejected: {why}")
            key = (req["failure_type"], req["signature_text"])
            idx = self._latest.get(key)  # == the reference's reversed() scan for the newest equal record (app.py:108-112)
            now = _iso(self._now())
            if idx is None:
                rec = {
                    "failure_id": f"F-{len(self.records) + 1:04d}",
                    "version": 1,
                    "created_at": now,
                    "updated_at": now,
                    "failure_type": req["failure_type"],
                    "root_cause": req.get("root_cause"),
                    "context_signature": req["context_signature"],
                    "impact_severity": getattr(req["impact_severity"], "value", req["impact_severity"]),
                    "resolution": req.get("resolution"),
                    "occurrences": 1,
                    "affected_apps": [req["app_id"]],
                    "signature_text": req["signature_text"],
                }
                created = True
            else:
                rec = json.loads(json.dumps(self.records[idx]))  # deep copy (app.py:134)
                rec["version"] += 1
                rec["updated_at"] = now
                rec["occurrences"] += 1
                if req["app_id"] not in rec["affected_apps"]:
                    rec["affected_apps"].append(req["app_id"])
                rec["root_cause"] = req.get("root_cause") or rec["root_cause"]
                rec["resolution"] = req.get("resolution") or rec["resolution"]
                rec["context_signature"] = req.get("context_signature") or rec["context_signature"]
                created = False
            if self.path is not None:
                with self.path.open("a", encoding="utf-8") as f:  # app.py:49-51
                    f.write(json.dumps(rec, ensure_ascii=False) + "\n")
            self.records.append(rec)
            self._latest[key] = len(self.records) - 1
            self._dirty = True
            return {"ok": True, "created": created, "failure": rec}

    # -- purge (services/dashboard/app.py:322-375, failures.jsonl only) -----------------------------------------
    def purge_apps(self, app_ids, backup: bool = True) -> Dict[str, int]:
        """Remove ``app_ids`` from every record's ``affected_apps`` and drop the records left with none, like the
        reference's ``_purge_jsonl_apps`` on failures.jsonl: a record counts as "updated" when its list changed and as
        "removed" when it became empty (both at once is possible), every other record as "kept".  The file is
        rewritten (after a ``failures.jsonl.bak-<UTC timestamp>`` copy when ``backup``).  The dropped records' device
        rows are deleted in place; the next query runs a statistics-only finalize, or compacts the main segment once
        more than ``tail_limit`` rows were deleted since the last rebuild."""
        purge = set(app_ids)
        with self._lock:
            kept = removed = updated = 0
            keep_idx: List[int] = []
            for i, rec in enumerate(self.records):
                apps = rec.get("affected_apps")
                if "affected_apps" in rec and isinstance(apps, list):
                    after = [a for a in apps if a not in purge]
                    if after != apps:
                        rec["affected_apps"] = after
                        updated += 1
                    if not after:
                        removed += 1
                        continue
                keep_idx.append(i)
                kept += 1
            if self.path is not None and self.path.exists():
                if backup:
                    stamp = self._now().astimezone(timezone.utc).strftime("%Y%m%dT%H%M%SZ")
                    shutil.copy2(self.path, self.path.with_name(f"{self.path.name}.bak-{stamp}"))
                lines = [json.dumps(self.records[i], ensure_ascii=False) for i in keep_idx]
                self.path.write_text("\n".join(lines) + ("\n" if lines else ""), encoding="utf-8")
            if removed:
                self._drop_records(keep_idx)
            return {"kept": kept, "removed": removed, "updated": updated}

    def _drop_records(self, keep_idx: List[int]) -> None:
        """records := records[keep_idx] (ascending); the dropped records' device rows are deleted."""
        n_old = len(self.records)
        keep = np.zeros(n_old, dtype=bool)
        keep[keep_idx] = True
        old_texts = [self._index_text(i) for i in range(n_old)] if self.sidecar_path is not None else None
        # device rows of the indexed records, in record order (monotone), and the new record index of every survivor
        live_rows = np.flatnonzero(self._row2rec >= 0) if self._row2rec is not None else np.arange(self._n_indexed)
        new_idx = np.cumsum(keep) - 1
        gone = live_rows[~keep[: self._n_indexed]]
        self.records = [self.records[i] for i in keep_idx]
        self._labels = [lab for i, lab in enumerate(self._labels) if keep[i]]
        self.quarantined = [int(new_idx[i]) for i in self.quarantined if keep[i]]
        self._quarantine_set = set(self.quarantined)
        self.stats["quarantined"] = len(self.quarantined)
        self._latest = {}
        for i, r in enumerate(self.records):  # the newest SURVIVING equal record (app.py:108-112)
            self._latest[(r["failure_type"], r["signature_text"])] = i
        n_idx_old = self._n_indexed
        self._n_indexed = int(keep[:n_idx_old].sum())
        if not self.records or self._main is None:
            self._rebuild_main()
        elif len(gone):
            row2rec = np.full(self._n_dev, -1, dtype=np.int64) if self._row2rec is None else self._row2rec.copy()
            row2rec[live_rows] = np.where(keep[:n_idx_old], new_idx[:n_idx_old], -1)
            self._row2rec = row2rec
            main_rows = gone[gone < self._n_main]
            if len(main_rows):
                self._main.delete_rows(main_rows)
                self._main_df = None  # the main segment's live df changed
            if self._tail is not None and len(gone) > len(main_rows):
                self._tail.delete_rows(gone[gone >= self._n_main] - self._n_main)
            self._n_deleted += len(gone)
            self._dirty = True
        if self.sidecar_path is not None:
            self._rewrite_sidecar(old_texts, keep_idx)

    def _rewrite_sidecar(self, old_texts: List[str], keep_idx: List[int]) -> None:
        """The sidecar of the surviving records (the vocabulary as it is, their CSR gathered from the old sidecar, the
        rows it did not hold featurised), so that a restart after a purge still skips the tokenisation; the persisted
        layout describes the old rows and is removed (the next cold start rebuilds it once).  The store wrote the old
        sidecar itself (records[:_sidecar_rows]), so it is read without checking its digest again; the cost is one read
        and one write of the file, a row gather and the digest of the surviving texts, under the store lock."""
        from .similarity import ArrayBatch, gather_rows

        lay_path = Path(str(self.sidecar_path) + ".layout")
        if lay_path.exists():
            lay_path.unlink()
        texts = [old_texts[i] for i in keep_idx]
        held = _sidecar.load_arrays(self.sidecar_path)
        n0 = held[1] if held is not None and held[1] == self._sidecar_rows else 0
        parts = []
        if n0:
            parts.append(gather_rows(held[0], np.asarray([i for i in keep_idx if i < n0], dtype=np.int64)))
        rest = [t for i, t in zip(keep_idx, texts) if i >= n0]
        if rest:
            fb = self.vocab.featurize(rest, grow=True)
            try:
                parts.append(ArrayBatch(np.array(fb.indptr), np.array(fb.ids), np.array(fb.tf)))
            finally:
                fb.close()
        indptr = [np.zeros(1, dtype=np.int64)]
        for p in parts:
            indptr.append(p.indptr[1:] + indptr[-1][-1])
        both = ArrayBatch(np.concatenate(indptr), np.concatenate([p.ids for p in parts] or [np.zeros(0, np.uint32)]),
                          np.concatenate([p.tf for p in parts] or [np.zeros(0, np.uint32)]))
        _sidecar.save(self.sidecar_path, self.vocab, both, texts)
        self._sidecar_rows = len(texts)

    # -- match (services/gfkb/app.py:79-102) -------------------------------------------------------------------
    def _candidates(self, fb: FeatureBatch, k: int, limit: int = MATCH_LIMIT,
                    labels: Optional[np.ndarray] = None) -> Tuple[np.ndarray, np.ndarray, np.ndarray]:
        """Per query: candidate rows from both segments with their float64 scores, ordered (score desc, row asc), and
        whether the candidate stage may have missed a top-``limit`` row (``ambiguous_candidates``).  ``labels``: per
        query the failure-type label its candidates must carry (-1: any)."""
        rows_all, f64_all = [], []
        amb = np.zeros(fb.n, dtype=bool)
        for ix in (self._main, self._tail):
            if ix is None or ix.n_rows == 0:
                continue
            kk = min(k, MAX_LIMIT)
            s32, rows = ix.topk_features(fb, kk) if labels is None else ix.topk_features(fb, kk, labels)
            amb |= ambiguous_candidates(s32, rows, limit)
            rows_all.append(rows)
            f64_all.append(ix.rescore(fb, rows))
        rows = np.concatenate(rows_all, axis=1)
        f64 = np.concatenate(f64_all, axis=1)
        big = np.where(rows < 0, np.iinfo(np.int64).max, rows)
        order = np.lexsort((big, -f64), axis=1)  # last key is primary: score descending, then row ascending
        return self._to_records(np.take_along_axis(rows, order, axis=1)), np.take_along_axis(f64, order, axis=1), amb

    def _exact_top(self, signature_text: str, limit: int, label: int = -1) -> Tuple[List[int], List[float]]:
        """Rows and float64 scores of the reference's ``sorted(..., reverse=True)[:limit]`` on the full score vector
        (K1a on both segments): no candidate stage at all.  ``label`` >= 0: over the rows of that failure-type label."""
        parts = [ix.score(signature_text) for ix in (self._main, self._tail) if ix is not None and ix.n_rows]
        scores = np.concatenate(parts)  # by device row; -inf for a deleted row
        if label >= 0:
            idx = np.flatnonzero(self._dev_labels(len(scores)) == label)  # ascending: the stable order is kept
            order = idx[stable_top(scores[idx], limit)]
        elif self._row2rec is not None:
            idx = np.flatnonzero(self._row2rec >= 0)
            order = idx[stable_top(scores[idx], limit)]
        else:
            order = np.asarray(stable_top(scores, limit), dtype=np.int64)
        return self._to_records(order).tolist(), [float(scores[i]) for i in order]

    def _match_filter_first(self, signature_texts: Sequence[str], failure_types: Sequence[Optional[str]],
                            limit: int) -> List[List[dict]]:
        """The best ``limit`` rows OF each query's failure type (all rows for a query without one)."""
        self._row_labels(0, len(self.records))  # number every stored type
        labels = np.array([-1 if not ft else self._type_ids.get(ft, -2) for ft in failure_types], dtype=np.int32)
        out: List[List[dict]] = [[] for _ in signature_texts]
        scan = np.flatnonzero(labels != -2)  # a type no stored row has: no match, and nothing to scan
        if len(scan) == 0:
            return out
        fb = self.vocab.featurize([signature_texts[i] for i in scan], grow=False)
        try:
            rows, f64, amb = self._candidates(fb, max(CANDIDATES, limit), limit, labels[scan])
        finally:
            fb.close()
        for j, i in enumerate(scan.tolist()):
            if amb[j]:
                top_r, top_s = self._exact_top(signature_texts[i], limit, int(labels[i]))
                self.stats["exact_fallbacks"] = self.stats.get("exact_fallbacks", 0) + 1
            else:
                top_r, top_s = rows[j, :limit].tolist(), f64[j, :limit].tolist()
            out[i] = [_to_match(self.records[r], s) for r, s in zip(top_r, top_s) if r >= 0]
        return out

    def match_batch(self, signature_texts: Sequence[str], failure_types: Optional[Sequence[Optional[str]]] = None,
                    limit: int = MATCH_LIMIT, filter_first: bool = False) -> List[List[dict]]:
        """``filter_first=False`` (default): the reference's handler -- the best ``limit`` rows, THEN the failure_type
        filter, so rows of other types can leave fewer than ``limit`` (or no) matches.  ``filter_first=True``: the best
        ``limit`` rows of the query's failure_type, searched on the device among that type's rows only."""
        if limit > MAX_LIMIT:
            raise ValueError(f"limit {limit} exceeds the {MAX_LIMIT} rows the fused top-k holds per query")
        with self._lock:
            if not self.records:
                return [[] for _ in signature_texts]  # app.py:82-83
            self._sync()
            if filter_first and failure_types is not None and any(failure_types):
                return self._match_filter_first(signature_texts, failure_types, limit)
            fb = self.vocab.featurize(list(signature_texts), grow=False)
            try:
                rows, f64, amb = self._candidates(fb, max(CANDIDATES, limit), limit)
            finally:
                fb.close()
            out = []
            for i in range(len(signature_texts)):
                ft = failure_types[i] if failure_types is not None else None
                matches = []
                if amb[i]:  # float32 candidates cannot decide this query's top rows: full float64 scan
                    top_r, top_s = self._exact_top(signature_texts[i], limit)
                    self.stats["exact_fallbacks"] = self.stats.get("exact_fallbacks", 0) + 1
                else:
                    top_r, top_s = rows[i, :limit].tolist(), f64[i, :limit].tolist()
                for r, s in zip(top_r, top_s):
                    if r < 0:
                        continue
                    rec = self.records[r]
                    if ft and rec["failure_type"] != ft:
                        continue
                    matches.append(_to_match(rec, s))
                out.append(matches)
            return out

    def match(self, signature_text: str, failure_type: Optional[str] = None, filter_first: bool = False) -> List[dict]:
        return self.match_batch([signature_text], [failure_type], filter_first=filter_first)[0]

    def match_exact(self, signature_text: str, failure_type: Optional[str] = None, limit: int = MATCH_LIMIT) -> List[dict]:
        """The handler on the full float64 score vector (K1a on both segments): no candidate stage at all."""
        with self._lock:
            if not self.records:
                return []
            self._sync()
            order, top = self._exact_top(signature_text, limit)
            out = []
            for i, sc in zip(order, top):
                rec = self.records[i]
                if failure_type and rec["failure_type"] != failure_type:
                    continue
                out.append(_to_match(rec, sc))
            return out

    # -- warn (services/warning_policy/app.py:19-72) ------------------------------------------------------------
    def warn_batch(self, requests: Sequence[Mapping[str, Any]], threshold: float = 0.8, default_action: str = "warn",
                   patterns: Optional[Sequence[Mapping[str, Any]]] = None) -> List[dict]:
        """One WarningResponse-shaped dict per request; all GFKB lookups go through ONE batched scan."""
        sigs = [_signature_text(r["prompt"], list(r.get("tools") or []), dict(r.get("env") or {})) for r in requests]
        all_matches = self.match_batch(sigs)
        out = []
        for matches in all_matches:
            best = matches[0] if matches else None
            score = float(best.get("score", 0.0)) if best else 0.0
            pattern_id = None
            if best and patterns:
                bt = best.get("failure_type")
                for p in reversed(list(patterns)):  # app.py:41-45
                    if p.get("name") == PATTERN_NAME and bt == "HALLUCINATION_CITATION":
                        pattern_id = p.get("pattern_id")
                        break
            if best and score >= threshold:
                msg = (
                    f"This execution matches past failure type {best.get('failure_type')} "
                    f"(failure_id={best.get('failure_id')}, similarity={score:.2f}). "
                    f"Suggested mitigation: {best.get('suggested_mitigation') or 'n/a'}"
                )
                out.append({"action": default_action, "confidence": score, "pattern_id": pattern_id,
                            "references": [best], "message": msg})
            else:
                out.append({"action": "silent" if default_action == "silent" else "warn", "confidence": score,
                            "pattern_id": pattern_id, "references": [],
                            "message": "No high-similarity match found in GFKB."})
        return out

    def close(self) -> None:
        with self._lock:
            for ix in (self._main, self._tail):
                if ix is not None:
                    ix.close()
            self._main = self._tail = None
