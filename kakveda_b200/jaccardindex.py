"""Token-set Jaccard index (K3, BASELINE configs[4]): rows and queries are sets of uint32 token ids.

Runs on the same device machinery as the TF-IDF scan (text-ordered stream, chunk summaries, block-max pruning,
fused top-k) with unit weights and the Jaccard epilogue; the exact (|∩|, |∪|) integers of the returned pairs come
back too, so ``inter / union`` in float64 is bit-identical to Python's set arithmetic.  The reference has no Jaccard
path: this is an extension with unpinned parity (oracle: ``oracle.tfidf_oracle.jaccard_sets``).

Besides top-k there is a threshold search (``range_csr`` / ``range_sets`` / ``selfjoin_range``, kernel K3-R): every
pair whose float32 score reaches the threshold, with the same exact counts; ``patterns.detect_patterns(k=None)``
clusters on it.
"""
from __future__ import annotations

import ctypes as C
from typing import Optional, Sequence, Tuple

import numpy as np

from . import _capi, _devout
from ._capi import no_distinct


def _csr(sets: Sequence[Sequence[int]]) -> Tuple[np.ndarray, np.ndarray]:
    indptr = np.zeros(len(sets) + 1, dtype=np.int64)
    uniq = [np.unique(np.asarray(s, dtype=np.uint32)) for s in sets]
    if uniq:
        np.cumsum([len(u) for u in uniq], out=indptr[1:])
    ids = np.concatenate(uniq).astype(np.uint32) if uniq and indptr[-1] else np.zeros(0, dtype=np.uint32)
    return indptr, ids


def _p(a: np.ndarray, t):
    return a.ctypes.data_as(C.POINTER(t))


class JaccardIndex:
    def __init__(self, vocab_size: int, device: int = 0, row_base: int = 0):
        h = C.c_void_p()
        _capi.check(_capi.load().kv_index_create(device, row_base, C.byref(h)))
        self._h, self.vocab_size, self.device = h, int(vocab_size), device
        # the appended rows, for the counts of self-join pairs (the query of a self-join is a stored row)
        self._parts = []
        _capi.check(_capi.load().kv_index_set_mode(h, 1))

    def add_csr(self, indptr: np.ndarray, ids: np.ndarray) -> None:
        indptr = np.ascontiguousarray(indptr, dtype=np.int64)
        ids = np.ascontiguousarray(ids, dtype=np.uint32)
        tf = np.ones(len(ids), dtype=np.uint32)
        _capi.check(_capi.load().kv_index_append(self._h, indptr.ctypes.data_as(C.POINTER(C.c_int64)),
                                                 ids.ctypes.data_as(C.POINTER(C.c_uint32)),
                                                 tf.ctypes.data_as(C.POINTER(C.c_uint32)), len(indptr) - 1))
        if len(indptr) > 1:
            self._parts.append((np.diff(indptr), ids[indptr[0]:indptr[-1]].copy()))

    def _rows_csr(self, lo: int, hi: int) -> Tuple[np.ndarray, np.ndarray]:
        """CSR of the local rows [lo, hi) as appended."""
        if len(self._parts) != 1:
            lens = np.concatenate([p[0] for p in self._parts]) if self._parts else np.zeros(0, np.int64)
            ids = np.concatenate([p[1] for p in self._parts]) if self._parts else np.zeros(0, np.uint32)
            self._parts = [(lens, ids)]
        lens, ids = self._parts[0]
        start = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
        return start[lo:hi + 1] - start[lo], ids[start[lo]:start[hi]]

    def _strip_oov(self, indptr: np.ndarray, ids: np.ndarray) -> Tuple[np.ndarray, np.ndarray, np.ndarray]:
        """(indptr, ids, oov): ids outside the index vocabulary cannot match any row, so they leave the CSR and only
        count towards |q| (oov[q] = how many query q had)."""
        indptr = np.ascontiguousarray(indptr, dtype=np.int64)
        ids = np.ascontiguousarray(ids, dtype=np.uint32)
        n = len(indptr) - 1
        inside = ids < self.vocab_size
        oov = np.zeros(n, dtype=np.float64)
        if not inside.all():
            seg = np.repeat(np.arange(n), np.diff(indptr))
            np.add.at(oov, seg[~inside], 1.0)
            keep = np.concatenate([[0], np.cumsum(inside)])
            indptr, ids = keep[indptr].astype(np.int64), ids[inside]
        return indptr, ids, oov

    def add_sets(self, sets: Sequence[Sequence[int]]) -> None:
        self.add_csr(*_csr(sets))

    def finalize(self) -> None:
        _capi.check(_capi.load().kv_index_finalize(self._h, self.vocab_size))

    @property
    def n_rows(self) -> int:
        return int(_capi.load().kv_index_rows(self._h))

    def topk_csr(self, indptr: np.ndarray, ids: np.ndarray, k: int = 16, distinct: bool = False):
        """(scores float32 [Q,k], rows int64 [Q,k], inter int32 [Q,k], union int32 [Q,k])."""
        no_distinct(distinct, "JaccardIndex.topk_csr")
        lib = _capi.load()
        indptr, ids, oov = self._strip_oov(indptr, ids)
        n = len(indptr) - 1
        tf = np.ones(len(ids), dtype=np.uint32)
        scores = np.empty((n, k), dtype=np.float32)
        rows = np.empty((n, k), dtype=np.int64)
        _capi.check(lib.kv_topk(self._h, _p(indptr, C.c_int64), _p(ids, C.c_uint32), _p(tf, C.c_uint32), _p(oov, C.c_double), n, k,
                                _p(scores, C.c_float), _p(rows, C.c_int64)))
        inter, union = self._counts(indptr, ids, oov, rows)
        return scores, rows, inter, union

    def _counts(self, indptr: np.ndarray, ids: np.ndarray, oov: np.ndarray, rows: np.ndarray):
        n, k = rows.shape
        inter = np.empty((n, k), dtype=np.int32)
        union = np.empty((n, k), dtype=np.int32)
        _capi.check(_capi.load().kv_jaccard_counts(self._h, _p(indptr, C.c_int64), _p(ids, C.c_uint32), _p(oov, C.c_double), n, k,
                                                   _p(rows, C.c_int64), _p(inter, C.c_int32), _p(union, C.c_int32)))
        return inter, union

    def counts_csr(self, indptr: np.ndarray, ids: np.ndarray, rows: np.ndarray):
        """Exact (|q ∩ row|, |q ∪ row|) of given (query, GLOBAL row) pairs; -1 for rows this shard does not hold."""
        indptr, ids, oov = self._strip_oov(indptr, ids)
        return self._counts(indptr, ids, oov, np.ascontiguousarray(rows, dtype=np.int64))

    def topk_sets(self, queries: Sequence[Sequence[int]], k: int = 16, distinct: bool = False):
        no_distinct(distinct, "JaccardIndex.topk_sets")
        return self.topk_csr(*_csr(queries), k=k)

    def _range_resident(self, n_q: int, threshold: float, device_out: bool = False):
        lib = _capi.load()
        n = C.c_int64(0)
        _capi.check(lib.kv_jaccard_range_resident(self._h, np.float32(threshold), C.byref(n)))
        if device_out:
            out = _devout.range_arrays(self.device, n_q, n.value, jaccard=True)
            _capi.check(lib.kv_jaccard_range_fetch_device(self._h, *_devout.ptrs(out)))
            return out
        indptr = np.empty(n_q + 1, dtype=np.int64)
        rows = np.empty(n.value, dtype=np.int64)
        scores = np.empty(n.value, dtype=np.float32)
        inter = np.empty(n.value, dtype=np.int32)
        union = np.empty(n.value, dtype=np.int32)
        _capi.check(lib.kv_jaccard_range_fetch(self._h, _p(indptr, C.c_int64), _p(rows, C.c_int64), _p(scores, C.c_float),
                                               _p(inter, C.c_int32), _p(union, C.c_int32)))
        return indptr, rows, scores, inter, union

    def _empty_range(self, device_out: bool = False):
        if device_out:
            return _devout.empty_range(self.device, jaccard=True)
        return (np.zeros(1, np.int64), np.zeros(0, np.int64), np.zeros(0, np.float32), np.zeros(0, np.int32),
                np.zeros(0, np.int32))

    def range_csr(self, indptr: np.ndarray, ids: np.ndarray, threshold: float, device_out: bool = False):
        """Threshold search: every (query, row) pair whose float32 score (the value ``topk_csr`` reports) is
        >= ``threshold``, 0 < threshold <= 1.  Returns ``(indptr int64[Q+1], rows int64[P], scores float32[P],
        inter int32[P], union int32[P])``: query q's pairs are ``[indptr[q], indptr[q+1])``, ordered by (score desc,
        row asc); rows are global; ``scores == float32(inter / union)`` with the exact counts.  ``device_out``: the
        same five arrays as torch tensors on the index's device."""
        indptr, ids, oov = self._strip_oov(indptr, ids)
        n = len(indptr) - 1
        if n == 0:
            return self._empty_range(device_out)
        tf = np.ones(len(ids), dtype=np.uint32)
        _capi.check(_capi.load().kv_query_upload(self._h, _p(indptr, C.c_int64), _p(ids, C.c_uint32), _p(tf, C.c_uint32),
                                                 _p(oov, C.c_double), n))
        return self._range_resident(n, threshold, device_out)

    def range_sets(self, queries: Sequence[Sequence[int]], threshold: float, device_out: bool = False):
        """``range_csr`` of token sets."""
        return self.range_csr(*_csr(queries), threshold, device_out)

    def selfjoin_topk(self, k: int, lo: int = 0, hi: Optional[int] = None, distinct: bool = False):
        """All-pairs: for local rows [lo, hi) the k best OTHER rows (the row itself is excluded), as ``topk_csr``:
        ``(scores float32[n,k], rows int64[n,k], inter int32[n,k], union int32[n,k])``."""
        no_distinct(distinct, "JaccardIndex.selfjoin_topk")
        hi = self.n_rows if hi is None else hi
        if hi <= lo:
            return (np.zeros((0, k), np.float32), np.zeros((0, k), np.int64), np.zeros((0, k), np.int32),
                    np.zeros((0, k), np.int32))
        lib = _capi.load()
        n = hi - lo
        _capi.check(lib.kv_selfjoin_upload(self._h, lo, hi))
        scores = np.empty((n, k), dtype=np.float32)
        rows = np.empty((n, k), dtype=np.int64)
        _capi.check(lib.kv_topk_resident_host(self._h, k, _p(scores, C.c_float), _p(rows, C.c_int64)))
        indptr, ids = self._rows_csr(lo, hi)
        inter, union = self._counts(indptr, ids, np.zeros(n, np.float64), rows)
        return scores, rows, inter, union

    def selfjoin_range(self, threshold: float, lo: int = 0, hi: Optional[int] = None, device_out: bool = False):
        """All-pairs threshold search: for local rows [lo, hi) every OTHER row scoring >= ``threshold`` (the five
        arrays of ``range_csr``, query i = row lo + i)."""
        hi = self.n_rows if hi is None else hi
        if hi <= lo:
            return self._empty_range(device_out)
        _capi.check(_capi.load().kv_selfjoin_upload(self._h, lo, hi))
        return self._range_resident(hi - lo, threshold, device_out)

    def last_timing_ms(self):
        ms = (C.c_float * 4)()
        _capi.check(_capi.load().kv_index_last_timing(self._h, ms))
        return tuple(ms)

    def close(self) -> None:
        if self._h is not None:
            _capi.load().kv_index_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
