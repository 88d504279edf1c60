"""Resident GFKB: ``failures.jsonl`` + a device index kept in sync (SURVEY.md section 8(f) ranks 1-2).

The reference's GFKB service re-reads and re-validates the whole JSONL on every request
(services/gfkb/app.py:49-51,81,106) and refits TF-IDF on it per query (similarity.py:17-18).  ``GfkbStore`` keeps
the records and their device index resident and reproduces the three handlers that touch the hot path:

* ``upsert``   -- services/gfkb/app.py:104-147: a (failure_type, signature_text) pair seen before appends a NEW
  version of the latest matching record (version+1, occurrences+1, app merged, fields evolve), otherwise a new
  ``F-%04d`` record; one JSON line is appended either way.
* ``match`` / ``match_batch`` -- services/gfkb/app.py:79-102: stable sort by score descending, first 5, THEN the
  failure_type filter, mapped to FailureMatch fields.
* ``match_above`` / ``match_above_batch`` -- the same sort with a similarity threshold instead of the first 5: every
  record whose float64 score reaches it (the exact threshold search, ``GfkbIndex.range_exact``, on both segments).
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
from .similarity import FeatureBatch, GfkbIndex, Vocabulary, csr_rows

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


def _first_of_each_group(groups: np.ndarray) -> np.ndarray:
    """Ascending positions of the first entry of each group in ``groups``: a distinct result keeps its group's first
    row in the order given."""
    _, first = np.unique(groups, return_index=True)
    return np.sort(first)


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


class AppTags:
    """The records' affected_apps as interned row tags, kept as one CSR over the records in record order: app ids are
    numbered in order of first appearance, ``ip`` / ``vals`` hold each record's ids, ``count[id]`` how many list
    entries name the app.  New records are added incrementally; a purge filters the purged ids out in NumPy and a
    record drop keeps the surviving rows, so no call walks every record in Python again."""

    def __init__(self):
        self.ids: Dict[str, int] = {}
        self.ip = np.zeros(1, dtype=np.int64)
        self.vals = np.zeros(0, dtype=np.int32)
        self.count = np.zeros(0, dtype=np.int64)
        self._rec_of_val: Optional[np.ndarray] = None  # record of every entry (exact fallback), built on demand

    @property
    def n(self) -> int:
        return len(self.ip) - 1

    def extend(self, recs: Sequence[Mapping[str, Any]]) -> None:
        lens, flat = [], []
        for r in recs:
            apps = r.get("affected_apps")
            t = [self.ids.setdefault(a, len(self.ids)) for a in apps] if isinstance(apps, list) else []
            lens.append(len(t))
            flat.extend(t)
        if not lens:
            return
        self.ip = np.concatenate([self.ip, self.ip[-1] + np.cumsum(lens, dtype=np.int64)])
        self.vals = np.concatenate([self.vals, np.asarray(flat, dtype=np.int32)])
        grown = np.zeros(len(self.ids), dtype=np.int64)
        grown[:len(self.count)] = self.count
        self.count = grown + np.bincount(np.asarray(flat, dtype=np.int64), minlength=len(self.ids))
        self._rec_of_val = None

    def purge(self, apps) -> None:
        """Every list loses ``apps`` (as ``GfkbStore.purge_apps`` rewrites affected_apps)."""
        gone = [self.ids[a] for a in apps if a in self.ids]
        if not gone:
            return
        keep = ~np.isin(self.vals, gone)
        pos = np.zeros(len(keep) + 1, dtype=np.int64)
        np.cumsum(keep, out=pos[1:])
        self.ip = pos[self.ip]
        self.vals = self.vals[keep]
        self.count[gone] = 0
        self._rec_of_val = None

    def keep(self, keep_idx) -> None:
        """Only the records ``keep_idx`` (ascending) remain; dropped records list no app (a purge emptied them)."""
        self.ip, self.vals = csr_rows(self.ip, self.vals, np.asarray(keep_idx, dtype=np.int64))
        self._rec_of_val = None

    def listed(self, app: str) -> int:
        """The app's id when some record lists it, else -2."""
        i = self.ids.get(app, -1)
        return i if i >= 0 and self.count[i] > 0 else -2

    def rows(self, recs: np.ndarray) -> Tuple[np.ndarray, np.ndarray]:
        """CSR of the tags of records ``recs`` (-1: an empty set, e.g. a deleted device row)."""
        return csr_rows(self.ip, self.vals, recs)

    def records_with(self, tag: int) -> np.ndarray:
        """bool [n]: which records list app id ``tag``."""
        if self._rec_of_val is None:
            self._rec_of_val = np.repeat(np.arange(self.n, dtype=np.int64), np.diff(self.ip))
        out = np.zeros(self.n, dtype=bool)
        out[self._rec_of_val[self.vals == tag]] = True
        return out


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
        # (failure_type, signature_text) key -> row group of the device index (distinct match), numbered in order of
        # first appearance; group of each record.  Set on the segments only when a distinct match needs them.
        self._group_ids: Dict[Tuple[str, str], int] = {}
        self._groups: List[int] = []
        # affected_apps as row tags of the device index (app-scoped match), kept incrementally for records[:_apps.n].
        # A device row's tags are its record's apps; set on the segments only when an app-scoped match needs them
        # (_main_tags_ok / _tail_tag_rows: which segment's tags describe the records as they are).
        self._apps = AppTags()
        self._main_tags_ok = False
        self._tail_tag_rows = -1
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
        self._group_ids, self._groups = {}, []
        self._apps = AppTags()
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
            self._build_main([self._index_text(i) for i in range(n)])
            self._main.set_row_labels(self._row_labels(0, n))
            self.stats["full_rebuilds"] += 1
        self._n_main = self._n_indexed = self._n_dev = n
        self._main_tags_ok, self._tail_tag_rows = False, -1
        self._sidecar_rows = n if self.sidecar_path is not None else 0  # the sidecar holds the CSR of records[:n]
        self._row2rec = None
        self._n_deleted = 0
        self._dirty = False

    def _build_main(self, texts: List[str]) -> None:
        """The main segment over ``texts`` (one per record), finalized with the statistics of its own rows."""
        n = len(texts)
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

    def _dev_labels(self, n_dev: int) -> np.ndarray:
        """int32 failure-type label of the first ``n_dev`` device rows (main + tail), -1 for a deleted row."""
        if self._row2rec is None:
            return self._row_labels(0, n_dev)
        rec_labels = self._row_labels(0, self._n_indexed)
        out = np.full(n_dev, -1, dtype=np.int32)
        live = self._row2rec >= 0
        out[live] = rec_labels[self._row2rec[live]]
        return out

    def _rec_groups(self, hi: int) -> np.ndarray:
        """int32 group of records[:hi]: their (failure_type, signature_text) keys, numbered in order of first appearance.
        All rows of a group share their text, hence their score."""
        for r in self.records[len(self._groups):hi]:
            self._groups.append(self._group_ids.setdefault((r["failure_type"], r["signature_text"]), len(self._group_ids)))
        return np.asarray(self._groups[:hi], dtype=np.int32)

    def _dev_groups(self, n_dev: int) -> np.ndarray:
        """int32 group of the first ``n_dev`` device rows (main + tail); a deleted row's group (0) is never read."""
        rec_groups = self._rec_groups(self._n_indexed)
        if self._row2rec is None:
            return rec_groups[:n_dev]
        out = np.zeros(n_dev, dtype=np.int32)
        live = self._row2rec >= 0
        out[live] = rec_groups[self._row2rec[live]]
        return out

    def _ensure_groups(self) -> None:
        """Both segments carry the same group numbering (an append or a rebuild dropped it)."""
        groups = None
        for ix, lo in ((self._main, 0), (self._tail, self._n_main)):
            if ix is not None and ix.n_rows and not ix.has_row_groups:
                if groups is None:
                    groups = self._dev_groups(self._n_dev)
                ix.set_row_groups(groups[lo:lo + ix.n_rows])

    def _sync_apps(self) -> None:
        """Intern the apps of the records not seen yet (incremental, like ``_row_labels``)."""
        if self._apps.n < len(self.records):
            self._apps.extend(self.records[self._apps.n:])

    def _dev_recs(self, lo: int, hi: int) -> np.ndarray:
        """Record of device rows [lo, hi), -1 for a deleted row."""
        if self._row2rec is None:
            return np.arange(lo, hi, dtype=np.int64)
        return self._row2rec[lo:hi]

    def _ensure_tags(self) -> None:
        """The segments carry their rows' app tags: only a stale segment is uploaded (a rebuild or a purge makes the
        main segment stale, an append the tail).  Tags touch no statistics: no finalize follows."""
        tail = self._tail
        if not self._main_tags_ok and self._main is not None:
            self._main.set_row_tags(self._apps.rows(self._dev_recs(0, self._n_main)))
            self._main_tags_ok = True
        if tail is not None and tail.n_rows and self._tail_tag_rows != tail.n_rows:
            tail.set_row_tags(self._apps.rows(self._dev_recs(self._n_main, self._n_main + tail.n_rows)))
            self._tail_tag_rows = tail.n_rows

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
        if self._tail is not None:
            tail_labels = self._dev_labels(self._n_dev)[self._n_main:]
            self._tail.set_row_labels(np.maximum(tail_labels, 0))  # an append dropped them; a deleted row's label is moot
        self._refresh_statistics()
        self._dirty = False

    def _refresh_statistics(self) -> None:
        """Global statistics = main + tail (the df all-reduce of a sharded GFKB, done in-process) on both segments:
        a statistics-only finalize of the main segment, a finalize of the tail."""
        segments = [ix for ix in (self._main, self._tail) if ix is not None]
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

    @property
    def _writes_file(self) -> bool:
        """Whether this store writes ``path`` (upserts append to it, a purge rewrites it)."""
        return self.path is not None

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
            if self._writes_file:
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
            if self._writes_file and self.path.exists():
                if backup:
                    stamp = self._now().astimezone(timezone.utc).strftime("%Y%m%dT%H%M%SZ")
                    shutil.copy2(self.path, self.path.with_name(f"{self.path.name}.bak-{stamp}"))
                lines = [json.dumps(self.records[i], ensure_ascii=False) for i in keep_idx]
                self.path.write_text("\n".join(lines) + ("\n" if lines else ""), encoding="utf-8")
            if updated:  # the rewritten lists change their rows' app tags
                self._sync_apps()
                self._apps.purge(purge)
                self._main_tags_ok, self._tail_tag_rows = False, -1
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
        if self._apps.n:
            self._apps.keep(np.flatnonzero(keep[:self._apps.n]))
        self._groups = [g for i, g in enumerate(self._groups) if keep[i]]  # survivors keep their group ids
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
            self._dirty = self._delete_dev_rows(gone)
            self._n_deleted += len(gone)
        if self.sidecar_path is not None:
            self._rewrite_sidecar(old_texts, keep_idx)

    def _delete_dev_rows(self, gone: np.ndarray) -> bool:
        """Delete the device rows ``gone`` (ascending) from the segments that hold them; returns whether the statistics
        still need a refresh before the next search (here: yes, the next ``_sync`` runs it)."""
        main_rows = gone[gone < self._n_main]
        if len(main_rows):
            self._main.delete_rows(main_rows)
            self._main_df = None  # the main segment's live df changed
        if self._tail is not None and len(gone) > len(main_rows):
            self._tail.delete_rows(gone[gone >= self._n_main] - self._n_main)
        return True

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
    def _candidates(self, fb: FeatureBatch, k: int, limit: int = MATCH_LIMIT, labels: Optional[np.ndarray] = None,
                    distinct: bool = False, tags=None) -> Tuple[np.ndarray, np.ndarray, np.ndarray]:
        """Per query: candidate rows from both segments with their float64 scores, ordered (score desc, row asc), and
        whether the candidate stage may have missed a top-``limit`` row (``ambiguous_candidates``).  ``labels``: per
        query the failure-type label its candidates must carry (-1: any).  ``distinct``: each segment returns one row
        per (failure_type, signature_text) group, and the merge keeps the first row of each group.  ``tags``: per query
        the app tags one of which its candidates must carry (empty: any)."""
        kk = min(k, MAX_LIMIT)
        if fb.n == 0:
            return np.zeros((0, kk), np.int64), np.zeros((0, kk)), np.zeros(0, dtype=bool)
        if distinct:
            self._ensure_groups()
        rows_all, f64_all = [], []
        amb = np.zeros(fb.n, dtype=bool)
        for ix in (self._main, self._tail):
            if ix is None or ix.n_rows == 0:
                continue
            s32, rows, f64 = self._segment_candidates(ix, fb, kk, labels, distinct, tags)
            amb |= ambiguous_candidates(s32, rows, limit)
            rows_all.append(rows)
            f64_all.append(f64)
        return self._merge_candidates(rows_all, f64_all, distinct) + (amb,)

    def _segment_candidates(self, ix, fb: FeatureBatch, kk: int, labels: Optional[np.ndarray], distinct: bool,
                            tags) -> Tuple[np.ndarray, np.ndarray, np.ndarray]:
        """One segment's float32 candidates and their float64 (K6) scores: (scores, global rows, K6 scores), each
        [Q, kk].  ``ShardedGfkbStore`` replaces it for its sharded MAIN segment."""
        s32, rows = ix.topk_features(fb, kk, labels, distinct, tags)
        return s32, rows, ix.rescore(fb, rows)

    def _merge_candidates(self, rows_all: List[np.ndarray], f64_all: List[np.ndarray],
                          distinct: bool) -> Tuple[np.ndarray, np.ndarray]:
        """The segments' candidates with their float64 scores -> record indices and scores ordered (score desc, row
        asc); ``distinct``: the first record of each group."""
        rows = np.concatenate(rows_all, axis=1)
        f64 = np.concatenate(f64_all, axis=1)
        big = np.where(rows < 0, np.iinfo(np.int64).max, rows)
        order = np.lexsort((big, -f64), axis=1)  # last key is primary: score descending, then row ascending
        recs, f64 = self._to_records(np.take_along_axis(rows, order, axis=1)), np.take_along_axis(f64, order, axis=1)
        if distinct:
            recs, f64 = self._first_of_groups(recs, f64)
        return recs, f64

    def _first_of_groups(self, recs: np.ndarray, f64: np.ndarray) -> Tuple[np.ndarray, np.ndarray]:
        """Per query (rows ordered): the first record of each group, moved to the front; (-1, -inf) fill the rest."""
        groups = self._rec_groups(self._n_indexed)
        out_r = np.full_like(recs, -1)
        out_s = np.full_like(f64, -np.inf)
        for q in range(recs.shape[0]):
            live = np.flatnonzero(recs[q] >= 0)
            keep = live[_first_of_each_group(groups[recs[q, live]])]
            out_r[q, :len(keep)], out_s[q, :len(keep)] = recs[q, keep], f64[q, keep]
        return out_r, out_s

    def _distinct_match(self, rec: int, score: float) -> dict:
        """A distinct result: its key's NEWEST record (the one the next upsert would version) with the key's score."""
        r = self.records[rec]
        return _to_match(self.records[self._latest[(r["failure_type"], r["signature_text"])]], score)

    def _matches(self, recs: Sequence[int], scores: Sequence[float], distinct: bool,
                 failure_type: Optional[str] = None) -> List[dict]:
        """Records (-1: none) and scores -> FailureMatch dicts, after the reference's failure_type post-filter
        (app.py:91-93); ``distinct``: each reported with its key's newest record (``_distinct_match``)."""
        out = []
        for r, s in zip(recs, scores):
            if r < 0 or (failure_type and self.records[r]["failure_type"] != failure_type):
                continue
            out.append(self._distinct_match(r, s) if distinct else _to_match(self.records[r], s))
        return out

    def _exact_top(self, signature_text: str, limit: int, label: int = -1,
                   distinct: bool = False, app: int = -1) -> Tuple[List[int], List[float]]:
        """Rows and float64 scores of the reference's ``sorted(..., reverse=True)[:limit]`` on the full score vector
        (K1a on both segments): no candidate stage at all.  ``label`` >= 0: over the rows of that failure-type label.
        ``distinct``: over the first eligible row of each (failure_type, signature_text) group.  ``app`` >= 0: over
        the rows whose record lists that app (tag)."""
        parts = [ix.score(signature_text) for ix in (self._main, self._tail) if ix is not None and ix.n_rows]
        scores = np.concatenate(parts)  # by device row; -inf for a deleted row
        n = len(scores)
        if label < 0 and app < 0 and not distinct and self._row2rec is None:  # every row: no copy of the scores
            order = np.asarray(stable_top(scores, limit), dtype=np.int64)
        else:
            recs = self._dev_recs(0, n)
            elig = recs >= 0
            if label >= 0:
                elig &= self._dev_labels(n) == label
            if app >= 0:
                self._sync_apps()
                elig &= self._apps.records_with(app)[np.clip(recs, 0, None)]
            idx = np.flatnonzero(elig)  # ascending: the stable order is kept
            if distinct:
                idx = idx[_first_of_each_group(self._dev_groups(n)[idx])]
            order = idx[stable_top(scores[idx], limit)]
        return self._to_records(order).tolist(), [float(scores[i]) for i in order]

    def _resolve_filters(self, n: int, failure_types: Optional[Sequence[Optional[str]]],
                         app_ids: Optional[Sequence[Optional[str]]]) -> Tuple[np.ndarray, np.ndarray, np.ndarray]:
        """Per query of ``n``: the failure-type label (-1: any, -2: a type no record has), the app id (-1: any, -2: an
        app no record lists), and the queries to scan (neither -2: the others match nothing)."""
        labels = np.full(n, -1, dtype=np.int32)
        if failure_types is not None and any(failure_types):
            self._row_labels(0, len(self.records))  # number every stored type
            labels = np.array([-1 if not ft else self._type_ids.get(ft, -2) for ft in failure_types], dtype=np.int32)
        apps = np.full(n, -1, dtype=np.int64)
        if app_ids is not None and any(app_ids):
            self._sync_apps()                    # intern every listed app
            apps = np.array([-1 if not a else self._apps.listed(a) for a in app_ids], dtype=np.int64)
        return labels, apps, np.flatnonzero((labels != -2) & (apps != -2))

    def match_batch(self, signature_texts: Sequence[str], failure_types: Optional[Sequence[Optional[str]]] = None,
                    limit: int = MATCH_LIMIT, filter_first: bool = False, distinct: bool = False,
                    app_ids: Optional[Sequence[Optional[str]]] = None) -> List[List[dict]]:
        """``filter_first=False`` (default): the reference's handler -- the best ``limit`` rows, THEN the failure_type
        filter, so rows of other types can leave fewer than ``limit`` (or no) matches.  ``filter_first=True``: the best
        ``limit`` rows of the query's failure_type, searched on the device among that type's rows only.
        ``distinct=True``: the best ``limit`` distinct failures, one per (failure_type, signature_text) key instead of
        one per stored version, each reported with the fields of the key's newest record and the key's score.
        ``app_ids``: per query an app (None: any); the search is then limited, on the device, to the failures whose
        affected_apps list it, and an app no record lists matches nothing.  It combines with the other options."""
        if limit > MAX_LIMIT:
            raise ValueError(f"limit {limit} exceeds the {MAX_LIMIT} rows the fused top-k holds per query")
        if app_ids is not None and len(app_ids) != len(signature_texts):
            raise ValueError(f"app_ids: {len(app_ids)} apps for {len(signature_texts)} queries")
        out: List[List[dict]] = [[] for _ in signature_texts]
        with self._lock:
            if not self.records:
                return out  # app.py:82-83
            self._sync()
            labels, apps, scan = self._resolve_filters(len(signature_texts), failure_types if filter_first else None,
                                                       app_ids)
            if len(scan) == 0:
                return out
            tags = None
            if (apps[scan] >= 0).any():
                self._ensure_tags()
                tags = [[int(apps[i])] if apps[i] >= 0 else [] for i in scan.tolist()]
            fb = self.vocab.featurize([signature_texts[i] for i in scan], grow=False)
            try:
                rows, f64, amb = self._candidates(fb, max(CANDIDATES, limit), limit,
                                                  labels[scan] if (labels[scan] >= 0).any() else None, distinct, tags)
            finally:
                fb.close()
            for j, i in enumerate(scan.tolist()):
                if amb[j]:  # float32 candidates cannot decide this query's top rows: full float64 scan
                    top_r, top_s = self._exact_top(signature_texts[i], limit, int(labels[i]), distinct, int(apps[i]))
                    self.stats["exact_fallbacks"] = self.stats.get("exact_fallbacks", 0) + 1
                else:
                    top_r, top_s = rows[j, :limit].tolist(), f64[j, :limit].tolist()
                # under filter_first the rows already carry the type: the post-filter drops none of them
                out[i] = self._matches(top_r, top_s, distinct, failure_types[i] if failure_types is not None else None)
            return out

    def match(self, signature_text: str, failure_type: Optional[str] = None, filter_first: bool = False,
              distinct: bool = False, app_id: Optional[str] = None) -> List[dict]:
        return self.match_batch([signature_text], [failure_type], filter_first=filter_first, distinct=distinct,
                                app_ids=[app_id])[0]

    def match_exact(self, signature_text: str, failure_type: Optional[str] = None, limit: int = MATCH_LIMIT) -> List[dict]:
        """The handler on the full float64 score vector (K1a on both segments): no candidate stage at all."""
        with self._lock:
            if not self.records:
                return []
            self._sync()
            order, top = self._exact_top(signature_text, limit)
            return self._matches(order, top, False, failure_type)

    # -- match above a threshold (services/gfkb/app.py:88-89 without the first-5 cut) -----------------------------
    def _above(self, fb: FeatureBatch, threshold: float, labels: Optional[np.ndarray],
               tags) -> List[Tuple[np.ndarray, np.ndarray, np.ndarray]]:
        """The device step of ``match_above_batch``: the exact threshold search of every segment, each
        ``(indptr, global device rows, float64 scores)`` ordered per query by (score desc, row asc)."""
        return [ix.range_exact(fb, threshold, labels, tags) for ix in (self._main, self._tail)
                if ix is not None and ix.n_rows]

    def match_above_batch(self, signature_texts: Sequence[str], threshold: float,
                          failure_types: Optional[Sequence[Optional[str]]] = None,
                          app_ids: Optional[Sequence[Optional[str]]] = None, distinct: bool = False) -> List[List[dict]]:
        """Per query every stored failure whose similarity is >= ``threshold`` (0 < threshold <= 1), as FailureMatch
        dicts in the reference's stable order (score desc, record asc): the handler's ``sorted(..., reverse=True)``
        with a threshold instead of the first 5, and no result limit.  Scores are float64 and membership is decided on
        them (the exact threshold search), so a record whose score equals the threshold is returned.  With no cut,
        filtering before or after the sort gives the same list, so ``failure_types`` (per query a type, None: any) and
        ``app_ids`` (per query an app its failures' affected_apps must list, None: any) are searched on the device; a
        type or app no record has returns ``[]`` without a scan.  ``distinct``: one result per (failure_type,
        signature_text) key, its best row, reported with the fields of the key's newest record and the key's score.
        A threshold so low that the pairs do not fit in device memory raises ``MemoryError``."""
        if not (0.0 < threshold <= 1.0):
            raise ValueError(f"threshold {threshold} outside (0, 1]")
        n = len(signature_texts)
        for name, per_query in (("failure_types", failure_types), ("app_ids", app_ids)):
            if per_query is not None and len(per_query) != n:
                raise ValueError(f"{name}: {len(per_query)} entries for {n} queries")
        out: List[List[dict]] = [[] for _ in signature_texts]
        with self._lock:
            if not self.records:
                return out
            self._sync()
            labels, apps, scan = self._resolve_filters(n, failure_types, app_ids)
            if len(scan) == 0:
                return out
            tags = None
            if (apps[scan] >= 0).any():
                self._ensure_tags()
                tags = [[int(apps[i])] if apps[i] >= 0 else [] for i in scan.tolist()]
            fb = self.vocab.featurize([signature_texts[i] for i in scan], grow=False)
            try:
                parts = self._above(fb, threshold, labels[scan] if (labels[scan] >= 0).any() else None, tags)
            finally:
                fb.close()
            groups = self._rec_groups(self._n_indexed) if distinct else None
            for j, i in enumerate(scan.tolist()):
                rows = np.concatenate([p[1][p[0][j]:p[0][j + 1]] for p in parts] or [np.zeros(0, np.int64)])
                scores = np.concatenate([p[2][p[0][j]:p[0][j + 1]] for p in parts] or [np.zeros(0)])
                order = np.lexsort((rows, -scores))  # score desc, device row asc = the records' stable order
                recs, scores = self._to_records(rows[order]), scores[order]
                if distinct:
                    keep = _first_of_each_group(groups[recs])
                    recs, scores = recs[keep], scores[keep]
                out[i] = self._matches(recs.tolist(), scores.tolist(), distinct)
            return out

    def match_above(self, signature_text: str, threshold: float, failure_type: Optional[str] = None,
                    app_id: Optional[str] = None, distinct: bool = False) -> List[dict]:
        """``match_above_batch`` of one query."""
        return self.match_above_batch([signature_text], threshold, [failure_type], [app_id], distinct)[0]

    # -- warn (services/warning_policy/app.py:19-72) ------------------------------------------------------------
    def warn_batch(self, requests: Sequence[Mapping[str, Any]], threshold: float = 0.8, default_action: str = "warn",
                   patterns: Optional[Sequence[Mapping[str, Any]]] = None, app_scoped: bool = False) -> List[dict]:
        """One WarningResponse-shaped dict per request; all GFKB lookups go through ONE batched scan.  ``app_scoped``:
        each request is matched against the failures of its own ``app_id`` only (default: the reference's handler,
        which matches against every failure)."""
        sigs = [_signature_text(r["prompt"], list(r.get("tools") or []), dict(r.get("env") or {})) for r in requests]
        if app_scoped:
            all_matches = self.match_batch(sigs, app_ids=[r.get("app_id") for r in requests])
        else:
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
