"""Host-side mirror of the reference's similarity interface, backed by the CUDA library.

``SimilarityEngine`` keeps the reference's class name, constructor (no arguments) and method
signature -- ``score(self, query: str, corpus: List[str]) -> List[float]``
(services/shared/similarity.py:10-20) -- so ``services.gfkb.app.engine`` can be replaced by
assignment (services/gfkb/app.py:31,86).  ``GfkbIndex`` is the resident device index the
engine caches between calls, and the batched entry point (``topk``) the GFKB match handler's
sort/top-5 (services/gfkb/app.py:88-91) maps onto.

All arithmetic runs in libkakveda_b200.so (hand-written sm_90a kernels).  Nothing here falls
back to scikit-learn or NumPy math: without the library or without a GPU the calls raise.
"""
from __future__ import annotations

import ctypes as C
import re
import threading
from dataclasses import dataclass, field
from typing import List, Optional, Sequence, Tuple

import numpy as np

from . import _capi, _devout

_TOKEN = re.compile(r"(?u)\b\w\w+\b")  # sklearn text.py:1969; used only for non-ASCII documents


def _ptr(a: np.ndarray, ctype):
    return a.ctypes.data_as(C.POINTER(ctype))


def pack_texts(texts: Sequence[str]) -> Tuple[bytes, np.ndarray, int]:
    """Concatenate documents for kv_featurize.  Returns (bytes, offsets[int64 n+1], text mode).

    ASCII-only batches go through as raw text (tokenised in C++).  A batch containing any
    non-ASCII document is sent in KV_TEXT_MIXED mode: those documents are tokenised here with
    Python's own ``str.lower`` + ``re`` (exactly what sklearn's analyzer runs, so Unicode
    case-folding and ``\\w`` semantics cannot diverge) and passed as 0x1F-separated tokens.
    """
    n = len(texts)
    offsets = np.zeros(n + 1, dtype=np.int64)
    joined = "".join(texts)
    if joined.isascii() and "\x1f" not in joined:
        if n:
            np.cumsum(np.fromiter((len(t) for t in texts), dtype=np.int64, count=n), out=offsets[1:])
        return joined.encode("ascii"), offsets, _capi.KV_TEXT_RAW_ASCII
    parts: List[bytes] = []
    for i, t in enumerate(texts):
        if t.isascii() and not t.startswith("\x1f"):
            b = t.encode("ascii")
        else:
            b = b"\x1f" + "\x1f".join(_TOKEN.findall(t.lower())).encode("utf-8")
        parts.append(b)
        offsets[i + 1] = offsets[i] + len(b)
    return b"".join(parts), offsets, _capi.KV_TEXT_MIXED


class FeatureBatch:
    """CSR of a featurised batch; owns the native kv_csr and exposes zero-copy NumPy views."""

    def __init__(self, handle: C.c_void_p):
        lib = _capi.load()
        self._h = handle
        n = C.c_int64()
        indptr = _capi.c_i64p()
        ids = _capi.c_u32p()
        tf = _capi.c_u32p()
        oov = _capi.c_f64p()
        _capi.check(lib.kv_csr_view(handle, C.byref(n), C.byref(indptr), C.byref(ids), C.byref(tf), C.byref(oov)))
        self.n = n.value
        self.indptr = np.ctypeslib.as_array(indptr, shape=(self.n + 1,))
        nnz = int(self.indptr[-1])
        if nnz:
            self.ids = np.ctypeslib.as_array(ids, shape=(nnz,))
            self.tf = np.ctypeslib.as_array(tf, shape=(nnz,))
        else:
            self.ids = np.zeros(0, dtype=np.uint32)
            self.tf = np.zeros(0, dtype=np.uint32)
        self.oov = np.ctypeslib.as_array(oov, shape=(self.n,)) if self.n else np.zeros(0)

    def close(self) -> None:
        if self._h is not None:
            self.indptr = self.ids = self.tf = self.oov = None
            _capi.load().kv_csr_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class ArrayBatch:
    """A featurised batch held in plain NumPy arrays (same attributes as :class:`FeatureBatch`): what a sidecar
    file stores and what ``GfkbIndex.add_features`` / ``upload_queries`` accept."""

    def __init__(self, indptr: np.ndarray, ids: np.ndarray, tf: np.ndarray, oov: Optional[np.ndarray] = None):
        self.indptr = np.ascontiguousarray(indptr, dtype=np.int64)
        self.ids = np.ascontiguousarray(ids, dtype=np.uint32)
        self.tf = np.ascontiguousarray(tf, dtype=np.uint32)
        self.n = len(self.indptr) - 1
        self.oov = np.zeros(self.n, dtype=np.float64) if oov is None else np.ascontiguousarray(oov, dtype=np.float64)
        if self.n < 0 or self.indptr[0] != 0 or self.indptr[-1] != len(self.ids) or len(self.ids) != len(self.tf):
            raise ValueError("ArrayBatch: inconsistent CSR arrays")

    def close(self) -> None:
        pass


def text_order(batch, n_threads: int = 0) -> np.ndarray:
    """int32 [n]: the rows of a featurised batch in text order (feature-id sequence, equal rows by index) -- host only."""
    perm = np.empty(batch.n, dtype=np.int32)
    _capi.check(_capi.load().kv_text_order(_ptr(batch.indptr, C.c_int64), _ptr(batch.ids, C.c_uint32), batch.n,
                                           perm.ctypes.data_as(C.POINTER(C.c_int32)), n_threads))
    return perm


def gather_rows(batch, rows: np.ndarray, n_threads: int = 0) -> ArrayBatch:
    """The sub-batch made of ``rows`` (int64 indices into ``batch``), in that order -- host only."""
    rows = np.ascontiguousarray(rows, dtype=np.int64)
    if len(rows) and (rows.min() < 0 or rows.max() >= batch.n):
        raise ValueError("gather_rows: row index outside the batch")
    lengths = (batch.indptr[1:] - batch.indptr[:-1])[rows] if len(rows) else np.zeros(0, dtype=np.int64)
    indptr = np.zeros(len(rows) + 1, dtype=np.int64)
    np.cumsum(lengths, out=indptr[1:])
    ids = np.empty(int(indptr[-1]), dtype=np.uint32)
    tf = np.empty(int(indptr[-1]), dtype=np.uint32)
    _capi.check(_capi.load().kv_csr_gather_rows(_ptr(batch.indptr, C.c_int64), _ptr(batch.ids, C.c_uint32), _ptr(batch.tf, C.c_uint32),
                                                batch.n, _ptr(rows, C.c_int64), len(rows), _ptr(indptr, C.c_int64),
                                                _ptr(ids, C.c_uint32), _ptr(tf, C.c_uint32), n_threads))
    return ArrayBatch(indptr, ids, tf, np.asarray(batch.oov)[rows] if len(rows) else None)


class Vocabulary:
    """Word 1,2-gram vocabulary (feature -> uint32 id) shared by corpus rows and queries."""

    def __init__(self):
        lib = _capi.load()
        h = C.c_void_p()
        _capi.check(lib.kv_vocab_create(C.byref(h)))
        self._h = h

    def __len__(self) -> int:
        return int(_capi.load().kv_vocab_size(self._h))

    def export_keys(self) -> np.ndarray:
        """uint64 [V, 2]: the 128-bit key of every feature in id order (the whole state of the vocabulary)."""
        n = len(self)
        keys = np.zeros((n, 2), dtype=np.uint64)
        _capi.check(_capi.load().kv_vocab_export(self._h, _ptr(keys, C.c_uint64), n))
        return keys

    @classmethod
    def from_keys(cls, keys: np.ndarray) -> "Vocabulary":
        """Rebuild a vocabulary from ``export_keys`` output: every feature gets its old id back."""
        keys = np.ascontiguousarray(keys, dtype=np.uint64).reshape(-1, 2)
        v = cls()
        _capi.check(_capi.load().kv_vocab_import(v._h, _ptr(keys, C.c_uint64), keys.shape[0]))
        return v

    def featurize_packed(self, data, offsets: np.ndarray, mode: int, grow: bool, n_threads: int = 0) -> FeatureBatch:
        lib = _capi.load()
        offsets = np.ascontiguousarray(offsets, dtype=np.int64)
        out = C.c_void_p()
        bad = C.c_int64(-1)
        if isinstance(data, np.ndarray):
            buf = data.ctypes.data_as(C.c_char_p)
        else:
            buf = C.c_char_p(data)
        rc = lib.kv_featurize(self._h, buf, _ptr(offsets, C.c_int64), len(offsets) - 1, mode, 1 if grow else 0,
                              n_threads, C.byref(out), C.byref(bad))
        _capi.check(rc)
        return FeatureBatch(out)

    def featurize(self, texts: Sequence[str], grow: bool, n_threads: int = 0) -> FeatureBatch:
        data, offsets, mode = pack_texts(texts)
        return self.featurize_packed(data, offsets, mode, grow, n_threads)

    def close(self) -> None:
        if self._h is not None:
            _capi.load().kv_vocab_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class GfkbIndex:
    """Resident TF-IDF index of one row shard of the GFKB on one H100.

    ``row_base`` is the global index of the shard's first row; ``vocab`` may be shared between
    shards living in one process.  Usage: ``add_texts`` / ``add_features`` (append-only, like
    failures.jsonl), ``finalize`` (after every append epoch), then ``score`` / ``topk``.
    """

    def __init__(self, device: int = 0, row_base: int = 0, vocab: Optional[Vocabulary] = None):
        lib = _capi.load()
        self.vocab = vocab if vocab is not None else Vocabulary()
        h = C.c_void_p()
        _capi.check(lib.kv_index_create(device, row_base, C.byref(h)))
        self._h = h
        self.device = device
        self.row_base = row_base
        self._row_labels: Optional[np.ndarray] = None  # what set_row_labels gave, until the next append
        self._group_rows: Optional[int] = None  # rows set_row_groups described, until the next append

    # -- build ---------------------------------------------------------------------------
    def add_features(self, fb: FeatureBatch, lo: int = 0, hi: Optional[int] = None) -> None:
        hi = fb.n if hi is None else hi
        if hi <= lo:
            return
        ip = np.ascontiguousarray(fb.indptr[lo:hi + 1])
        _capi.check(_capi.load().kv_index_append(self._h, _ptr(ip, C.c_int64), _ptr(fb.ids, C.c_uint32),
                                                 _ptr(fb.tf, C.c_uint32), hi - lo))
        self._row_labels = None  # the library drops the labels (and the groups) on an append
        self._group_rows = None

    def set_row_labels(self, labels: Optional[np.ndarray]) -> None:
        """One label >= 0 per local row (e.g. a failure-type id), for the ``labels`` / ``same_label`` filters of the
        query methods; ``None`` clears.  Survives finalize; an append drops the labels (a filtered query then raises
        until they are set again)."""
        if labels is None:
            _capi.check(_capi.load().kv_index_set_row_labels(self._h, None, 0))
            self._row_labels = None
            return
        labels = np.ascontiguousarray(labels, dtype=np.int32)
        _capi.check(_capi.load().kv_index_set_row_labels(self._h, _ptr(labels, C.c_int32), len(labels)))
        self._row_labels = labels.copy()

    def set_row_groups(self, groups: Optional[np.ndarray]) -> None:
        """One group >= 0 per local row (e.g. one id per distinct text), for the ``distinct`` top-k of the query
        methods; ``None`` clears.  Survives finalize, a layout load and deletions; an append drops the groups (a
        distinct query then raises until they are set again).  Setting groups alone changes no result."""
        if groups is None:
            _capi.check(_capi.load().kv_index_set_row_groups(self._h, None, 0))
            self._group_rows = None
            return
        groups = np.ascontiguousarray(groups, dtype=np.int32)
        _capi.check(_capi.load().kv_index_set_row_groups(self._h, _ptr(groups, C.c_int32), len(groups)))
        self._group_rows = len(groups)

    @property
    def has_row_groups(self) -> bool:
        """Whether ``set_row_groups`` describes the current rows (an append drops the groups)."""
        return self._group_rows is not None and self._group_rows == self.n_rows

    def add_texts(self, texts: Sequence[str]) -> None:
        fb = self.vocab.featurize(texts, grow=True)
        try:
            self.add_features(fb)
        finally:
            fb.close()

    def local_df(self) -> np.ndarray:
        v = len(self.vocab)
        df = np.zeros(max(v, 1), dtype=np.uint32)
        _capi.check(_capi.load().kv_index_local_df(self._h, _ptr(df, C.c_uint32), v))
        return df[:v]

    def set_global_df(self, df: np.ndarray, n_rows_global: int) -> None:
        df = np.ascontiguousarray(df, dtype=np.uint32)
        _capi.check(_capi.load().kv_index_set_global_df(self._h, _ptr(df, C.c_uint32), len(df), n_rows_global))

    def set_mode(self, mode: int) -> None:
        """0 = the reference's refit-per-query TF-IDF cosine (default), 1 = token-set Jaccard, 2 = TF-IDF fitted on
        the corpus alone (symmetric; the measure of the all-pairs self-join).  Call before ``finalize``."""
        _capi.check(_capi.load().kv_index_set_mode(self._h, int(mode)))

    def finalize(self) -> None:
        _capi.check(_capi.load().kv_index_finalize(self._h, len(self.vocab)))

    @property
    def last_finalize_kind(self) -> int:
        """1 = full rebuild, 2 = statistics-only refresh (rows unchanged, only global N / df moved)."""
        return int(_capi.load().kv_index_last_finalize_kind(self._h))

    @property
    def n_rows(self) -> int:
        return int(_capi.load().kv_index_rows(self._h))

    def delete_rows(self, rows) -> None:
        """Delete local ``rows`` (any order; duplicates and rows deleted before are allowed).  A deleted row keeps its
        row id but no search returns it again and ``score`` gives it -inf; N and df count the live rows.  Like an
        append, the deletion takes effect at the next ``finalize`` (a statistics-only refresh when nothing was
        appended) and searches raise until then.  Not on a Jaccard index (mode 1)."""
        rows = np.ascontiguousarray(rows, dtype=np.int64).reshape(-1)
        _capi.check(_capi.load().kv_index_delete_rows(self._h, _ptr(rows, C.c_int64), len(rows)))

    def deleted_mask(self) -> np.ndarray:
        """bool [n_rows]: which local rows are deleted (the handle's own flags)."""
        n = self.n_rows
        out = np.zeros(n, dtype=np.uint8)
        _capi.check(_capi.load().kv_index_deleted_rows(self._h, _ptr(out, C.c_uint8), n))
        return out.astype(bool)

    @property
    def n_live_rows(self) -> int:
        """``n_rows`` minus the deleted rows."""
        return int(_capi.load().kv_index_live_rows(self._h))

    # -- query ---------------------------------------------------------------------------
    def score_features(self, ids: np.ndarray, tf: np.ndarray, oov_tf2: float) -> np.ndarray:
        out = np.empty(self.n_rows, dtype=np.float64)
        ids = np.ascontiguousarray(ids, dtype=np.uint32)
        tf = np.ascontiguousarray(tf, dtype=np.uint32)
        _capi.check(_capi.load().kv_score(self._h, _ptr(ids, C.c_uint32), _ptr(tf, C.c_uint32), len(ids),
                                          float(oov_tf2), _ptr(out, C.c_double)))
        return out

    def score(self, query: str) -> np.ndarray:
        """float64 cosine of ``query`` against every local row (K1a); -inf for a deleted row."""
        fb = self.vocab.featurize([query], grow=False)
        try:
            return self.score_features(fb.ids, fb.tf, float(fb.oov[0]))
        finally:
            fb.close()

    def topk_features(self, fb: FeatureBatch, k: int, labels: Optional[np.ndarray] = None,
                      distinct: bool = False) -> Tuple[np.ndarray, np.ndarray]:
        """``labels``: per query the row label its results must carry (-1: any row), see ``set_filter``.  ``distinct``:
        at most one row per group (``set_row_groups``), see ``set_distinct``."""
        if labels is not None or distinct:
            if fb.n == 0:
                return np.zeros((0, k), np.float32), np.zeros((0, k), np.int64)
            self.upload_queries(fb)
            if labels is not None:
                self.set_filter(labels)
            if distinct:
                self.set_distinct(True)
            return self.topk_resident_host(fb.n, k)
        scores = np.empty((fb.n, k), dtype=np.float32)
        rows = np.empty((fb.n, k), dtype=np.int64)
        _capi.check(_capi.load().kv_topk(self._h, _ptr(fb.indptr, C.c_int64), _ptr(fb.ids, C.c_uint32),
                                         _ptr(fb.tf, C.c_uint32), _ptr(fb.oov, C.c_double), fb.n, k,
                                         _ptr(scores, C.c_float), _ptr(rows, C.c_int64)))
        return scores, rows

    def topk_features_device(self, fb: FeatureBatch, k: int, d_scores_ptr: int, d_rows_ptr: int) -> None:
        """Results stay on the device: float32[n,k] / int64[n,k] buffers owned by the caller."""
        _capi.check(_capi.load().kv_topk_device(self._h, _ptr(fb.indptr, C.c_int64), _ptr(fb.ids, C.c_uint32),
                                                _ptr(fb.tf, C.c_uint32), _ptr(fb.oov, C.c_double), fb.n, k,
                                                C.c_void_p(d_scores_ptr), C.c_void_p(d_rows_ptr)))

    def upload_queries(self, fb: FeatureBatch) -> None:
        """Make a featurised batch resident on the device (host prep + H2D), for topk_resident."""
        _capi.check(_capi.load().kv_query_upload(self._h, _ptr(fb.indptr, C.c_int64), _ptr(fb.ids, C.c_uint32),
                                                 _ptr(fb.tf, C.c_uint32), _ptr(fb.oov, C.c_double), fb.n))

    def prepare_slice(self, fb, out=None):
        """A slice of a query batch re-stored in text order, as a run for ``upload_query_runs``: returns
        ``(indptr, ids, tf, oov, order, flags)`` where row p is the slice's p-th smallest query, ``order[p]`` its original
        index inside the slice and ``flags[p]`` its classification (a row-sharded GFKB prepares one slice per rank).
        ``out``: optional preallocated arrays of the same six kinds to write into (e.g. views of a pinned buffer)."""
        n = fb.n
        base, end = int(fb.indptr[0]), int(fb.indptr[n])
        nnz = end - base
        if out is None:
            out = (np.empty(n + 1, np.int64), np.empty(nnz, np.uint32), np.empty(nnz, np.uint32), np.empty(n, np.float64),
                   np.empty(n, np.int32), np.empty(n, np.uint8))
        ip, ids, tf, oov, order, flags = out
        _capi.check(_capi.load().kv_query_prepare_slice(self._h, _ptr(fb.indptr, C.c_int64), _ptr(fb.ids, C.c_uint32),
                                                        _ptr(fb.tf, C.c_uint32), _ptr(fb.oov, C.c_double), n,
                                                        _ptr(ip, C.c_int64), _ptr(ids, C.c_uint32), _ptr(tf, C.c_uint32),
                                                        _ptr(oov, C.c_double), _ptr(order, C.c_int32), _ptr(flags, C.c_uint8)))
        return out

    def upload_query_runs(self, runs) -> int:
        """``upload_queries`` of a batch given as consecutive slices: ``runs`` is a list of
        ``(indptr, ids, tf, oov, order, flags)`` NumPy arrays: either what ``prepare_slice`` returned for every
        slice, or plain CSR slices with ``order`` and ``flags`` None for all runs.  Returns the number of queries."""
        n = len(runs)
        arr = lambda: (C.c_void_p * n)()
        ip, ids, tf, oov, od, fl = arr(), arr(), arr(), arr(), arr(), arr()
        nq = np.empty(n, dtype=np.int64)
        with_prep = all(r[4] is not None and r[5] is not None for r in runs)
        keep = []
        for i, r in enumerate(runs):
            cols = [np.ascontiguousarray(r[0], dtype=np.int64), np.ascontiguousarray(r[1], dtype=np.uint32),
                    np.ascontiguousarray(r[2], dtype=np.uint32), np.ascontiguousarray(r[3], dtype=np.float64)]
            if with_prep:
                cols += [np.ascontiguousarray(r[4], dtype=np.int32), np.ascontiguousarray(r[5], dtype=np.uint8)]
            keep.append(cols)
            nq[i] = len(cols[0]) - 1
            for dst, c in zip((ip, ids, tf, oov, od, fl), cols):
                dst[i] = c.ctypes.data
        _capi.check(_capi.load().kv_query_upload_runs(self._h, n, ip, ids, tf, oov, od if with_prep else None,
                                                      fl if with_prep else None, _ptr(nq, C.c_int64)))
        return int(nq.sum())

    def last_prepare_ms(self) -> Tuple[float, float, float, float]:
        """Host-side split of the last upload: pinned staging, classification, text order, copies + table kernels."""
        ms = (C.c_float * 4)()
        _capi.check(_capi.load().kv_index_last_prepare_ms(self._h, ms))
        return tuple(ms)

    def set_exclusions(self, rows: Optional[np.ndarray]) -> None:
        """Query q of the resident batch must not match GLOBAL row ``rows[q]`` (-1 = none); ``None`` clears."""
        if rows is None:
            _capi.check(_capi.load().kv_query_set_exclusions(self._h, None, 0))
            return
        rows = np.ascontiguousarray(rows, dtype=np.int64)
        _capi.check(_capi.load().kv_query_set_exclusions(self._h, _ptr(rows, C.c_int64), len(rows)))

    def set_filter(self, labels: Optional[np.ndarray]) -> None:
        """Query q of the resident batch only matches rows labelled ``labels[q]`` (-1 = any row; ``set_row_labels``);
        ``None`` clears, and so does the next upload.  The index statistics are not changed: the scores are the
        unfiltered ones."""
        if labels is None:
            _capi.check(_capi.load().kv_query_set_filter(self._h, None, 0))
            return
        labels = np.ascontiguousarray(labels, dtype=np.int32)
        _capi.check(_capi.load().kv_query_set_filter(self._h, _ptr(labels, C.c_int32), len(labels)))

    def set_distinct(self, on: bool) -> None:
        """Distinct top-k for the resident batch (until the next upload): of the rows a query may match, the best row
        of each group (``set_row_groups``) in (score desc, row asc) order, the groups ranked by it, and the first k
        of them.  Scores are the non-distinct ones; threshold searches ignore the mode."""
        _capi.check(_capi.load().kv_query_set_distinct(self._h, 1 if on else 0))

    def topk_resident_host(self, n_q: int, k: int) -> Tuple[np.ndarray, np.ndarray]:
        """Scan + merge of the resident batch of ``n_q`` queries, results copied to the host."""
        scores = np.empty((n_q, k), dtype=np.float32)
        rows = np.empty((n_q, k), dtype=np.int64)
        _capi.check(_capi.load().kv_topk_resident_host(self._h, k, _ptr(scores, C.c_float), _ptr(rows, C.c_int64)))
        return scores, rows

    def _selfjoin_upload(self, lo: int, hi: int, same_label: bool) -> None:
        _capi.check(_capi.load().kv_selfjoin_upload(self._h, lo, hi))
        if same_label:
            if self._row_labels is None or len(self._row_labels) != self.n_rows:
                raise RuntimeError("same_label: the index has no row labels for its current rows (set_row_labels)")
            self.set_filter(self._row_labels[lo:hi])

    def selfjoin_topk(self, k: int, lo: int = 0, hi: Optional[int] = None,
                      same_label: bool = False, distinct: bool = False) -> Tuple[np.ndarray, np.ndarray]:
        """All-pairs: for local rows [lo, hi) the k best OTHER rows (the row itself is excluded).  ``same_label``:
        row i's list holds only rows with row i's label.  ``distinct``: at most one row per group (``set_row_groups``);
        row i's own group still counts, through its other rows."""
        hi = self.n_rows if hi is None else hi
        if hi <= lo:
            return np.zeros((0, k), np.float32), np.zeros((0, k), np.int64)
        self._selfjoin_upload(lo, hi, same_label)
        if distinct:
            self.set_distinct(True)
        return self.topk_resident_host(hi - lo, k)

    def _range_resident(self, n_q: int, threshold: float, device_out: bool = False):
        lib = _capi.load()
        n = C.c_int64(0)
        _capi.check(lib.kv_range_resident(self._h, np.float32(threshold), C.byref(n)))
        if device_out:
            out = _devout.range_arrays(self.device, n_q, n.value)
            _capi.check(lib.kv_range_fetch_device(self._h, *_devout.ptrs(out)))
            return out
        indptr = np.empty(n_q + 1, dtype=np.int64)
        rows = np.empty(n.value, dtype=np.int64)
        scores = np.empty(n.value, dtype=np.float32)
        _capi.check(lib.kv_range_fetch(self._h, _ptr(indptr, C.c_int64), _ptr(rows, C.c_int64), _ptr(scores, C.c_float)))
        return indptr, rows, scores

    def _empty_range(self, device_out: bool):
        if device_out:
            return _devout.empty_range(self.device)
        return np.zeros(1, np.int64), np.zeros(0, np.int64), np.zeros(0, np.float32)

    def range_features(self, fb: FeatureBatch, threshold: float, device_out: bool = False,
                       labels: Optional[np.ndarray] = None):
        """Threshold search: every (query, row) pair whose float32 score (the value ``topk`` reports) is >= ``threshold``,
        0 < threshold <= 1.  Returns ``(indptr int64[n_q+1], rows int64[P], scores float32[P])``: query q's pairs are
        ``[indptr[q], indptr[q+1])``, ordered by (score desc, row asc); rows are global.  ``device_out``: the same
        arrays as torch tensors on the index's device (nothing is copied to the host).  ``labels``: per query the row
        label its pairs must carry (-1: any row), see ``set_filter``."""
        if fb.n == 0:
            return self._empty_range(device_out)
        self.upload_queries(fb)
        if labels is not None:
            self.set_filter(labels)
        return self._range_resident(fb.n, threshold, device_out)

    def range(self, queries: Sequence[str], threshold: float, device_out: bool = False,
              labels: Optional[np.ndarray] = None):
        """``range_features`` of texts."""
        fb = self.vocab.featurize(queries, grow=False)
        try:
            return self.range_features(fb, threshold, device_out, labels)
        finally:
            fb.close()

    def selfjoin_range(self, threshold: float, lo: int = 0, hi: Optional[int] = None, device_out: bool = False,
                       same_label: bool = False):
        """All-pairs threshold search: for local rows [lo, hi) every OTHER row scoring >= ``threshold`` (CSR as in
        ``range_features``, query i = row lo + i).  ``same_label``: only rows with row i's label."""
        hi = self.n_rows if hi is None else hi
        if hi <= lo:
            return self._empty_range(device_out)
        self._selfjoin_upload(lo, hi, same_label)
        return self._range_resident(hi - lo, threshold, device_out)

    def rescore(self, fb: FeatureBatch, rows: np.ndarray) -> np.ndarray:
        """K6: float64 scores of the pairs (query q, GLOBAL row rows[q, j]); identical rows tie exactly on every shard."""
        rows = np.ascontiguousarray(rows, dtype=np.int64)
        k = rows.shape[1]
        out = np.empty((fb.n, k), dtype=np.float64)
        _capi.check(_capi.load().kv_rescore_pairs(self._h, _ptr(fb.indptr, C.c_int64), _ptr(fb.ids, C.c_uint32),
                                                  _ptr(fb.tf, C.c_uint32), _ptr(fb.oov, C.c_double), fb.n, k,
                                                  _ptr(rows, C.c_int64), _ptr(out, C.c_double)))
        return out

    def topk_resident(self, k: int, d_scores_ptr: int, d_rows_ptr: int) -> None:
        """Device-only scan + merge of the uploaded batch into caller-owned device buffers."""
        _capi.check(_capi.load().kv_topk_resident(self._h, k, C.c_void_p(d_scores_ptr), C.c_void_p(d_rows_ptr)))

    def topk_resident_seed(self, k: int, d_scores_ptr: int, d_rows_ptr: int) -> None:
        """Phase 1 of a sharded step: bound pass + seed scan; the buffers receive this shard's seed top-k."""
        _capi.check(_capi.load().kv_topk_resident_seed(self._h, k, C.c_void_p(d_scores_ptr), C.c_void_p(d_rows_ptr)))

    def raise_thresholds(self, d_kth_ptr: int, n_q: int) -> None:
        """Per query a lower bound of the GLOBAL k-th score (device float32[n_q]): raises the pruning thresholds."""
        _capi.check(_capi.load().kv_index_raise_thresholds(self._h, C.c_void_p(d_kth_ptr), n_q))

    def topk_resident_finish(self, k: int, d_scores_ptr: int, d_rows_ptr: int) -> None:
        """Phase 2 of a sharded step: candidate selection + scan + merge of the resident batch."""
        _capi.check(_capi.load().kv_topk_resident_finish(self._h, k, C.c_void_p(d_scores_ptr), C.c_void_p(d_rows_ptr)))

    def topk(self, queries: Sequence[str], k: int, labels: Optional[np.ndarray] = None,
             distinct: bool = False) -> Tuple[np.ndarray, np.ndarray]:
        """(scores float32 [Q,k], rows int64 [Q,k]) ordered by (score desc, row asc) (K1b+K5).  ``labels``: per query
        the row label its results must carry (-1: any row).  ``distinct``: at most one row per group (the best one;
        ``set_row_groups``)."""
        fb = self.vocab.featurize(queries, grow=False)
        try:
            return self.topk_features(fb, k, labels, distinct)
        finally:
            fb.close()

    def last_timing_ms(self) -> Tuple[float, float, float, float]:
        ms = (C.c_float * 4)()
        _capi.check(_capi.load().kv_index_last_timing(self._h, ms))
        return tuple(ms)

    def last_score_ms(self) -> float:
        ms = C.c_float()
        _capi.check(_capi.load().kv_index_last_score_ms(self._h, C.byref(ms)))
        return ms.value

    def last_kernel_ms(self) -> Tuple[float, float, float, float, float]:
        """CUDA-event ms of the last batch's kernels: bound pass 0 (seeds), seed scan, bound pass 1 (candidate lists),
        candidate scan, merge."""
        ms = (C.c_float * 5)()
        _capi.check(_capi.load().kv_index_last_kernel_ms(self._h, ms))
        return tuple(ms)

    def layout(self) -> dict:
        b = (C.c_int64 * 4)()
        c = (C.c_int64 * 18)()
        _capi.check(_capi.load().kv_index_layout(self._h, b, c))
        return {"block_bytes": b[0], "norm_bytes": b[1], "directory_bytes": b[2], "dense_bytes": b[3],
                "entries": c[0], "universal_features": c[1], "rows": c[2], "last_ctas": c[3], "last_tiles": c[4],
                "last_splits": c[5], "last_upload_bytes": c[6], "tf_overflow_entries": c[7], "chunks": c[8],
                "pairs_scored": c[9], "records_scanned": c[10], "pairs_passed_bound": c[11],
                "records_written": c[12], "kernel_launches": c[13], "rare_entries": c[14],
                "pool_pages_used": c[15], "pool_pages": c[16], "f2_outside_dictionary": c[17]}

    def save_layout(self, path) -> None:
        """Persist the built scan layout (row order, column blocks, bound structures) of a finalized index."""
        _capi.check(_capi.load().kv_index_layout_save(self._h, str(path).encode()))

    def load_layout(self, path) -> bool:
        """After appending the same rows and BEFORE finalize(): restore a persisted layout; False if the file is missing
        or was built for other rows (finalize then builds as usual)."""
        import os

        if not os.path.exists(str(path)):
            return False
        rc = _capi.load().kv_index_layout_load(self._h, str(path).encode())
        if rc in (_capi.KV_ERR_STATE, _capi.KV_ERR_INVALID):
            return False
        _capi.check(rc)
        return True

    def close(self) -> None:
        if self._h is not None:
            _capi.load().kv_index_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


@dataclass
class SimilarityEngine:
    """Drop-in for services.shared.similarity.SimilarityEngine (similarity.py:10-20).

    Same contract: ``score(query, corpus)`` returns ``len(corpus)`` Python floats (float64
    TF-IDF(1,2-gram) cosine, refit semantics included) in corpus order; ``[]`` for an empty
    corpus; ``ValueError`` when no document has a token.  The engine caches the device index of
    the last corpus it saw (GFKB re-reads failures.jsonl per request, app.py:81, but the rows
    only ever grow by appends, app.py:132,146): an unchanged corpus is reused, a corpus that
    extends the cached one is appended, anything else is rebuilt.  Thread-safe (match() runs on
    a worker pool).
    """

    device: int = 0
    _lock: threading.Lock = field(default_factory=threading.Lock, repr=False, compare=False)
    _index: Optional[GfkbIndex] = field(default=None, repr=False, compare=False)
    _rows: List[str] = field(default_factory=list, repr=False, compare=False)

    def _sync_index(self, corpus: Sequence[str]) -> GfkbIndex:
        # Identity of the cached corpus is decided by comparing the row strings themselves (a shallow copy of the last
        # corpus is kept) -- exact, no hash that could collide; the comparison is a C-level list compare.
        n, old_n = len(corpus), len(self._rows)
        if self._index is not None and n == old_n and (corpus is self._rows or list(corpus) == self._rows):
            return self._index
        if self._index is not None and 0 < old_n < n and list(corpus[:old_n]) == self._rows:
            self._index.add_texts(corpus[old_n:])
        else:
            if self._index is not None:
                self._index.close()
            self._index = GfkbIndex(device=self.device)
            self._index.add_texts(corpus)
        self._index.finalize()
        self._rows = list(corpus)
        return self._index

    def score(self, query: str, corpus: List[str]) -> List[float]:
        if not corpus:
            return []
        with self._lock:
            return self._sync_index(corpus).score(query).tolist()

    def topk(self, queries: Sequence[str], corpus: Sequence[str], k: int = 5) -> Tuple[np.ndarray, np.ndarray]:
        """Batched form: the k best rows per query, ties to the lower row (gfkb/app.py:89)."""
        if not corpus:
            return (np.zeros((len(queries), 0), np.float32), np.zeros((len(queries), 0), np.int64))
        with self._lock:
            return self._sync_index(corpus).topk(queries, min(k, 32))
