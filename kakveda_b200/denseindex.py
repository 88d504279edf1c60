"""Dense-embedding cosine index (K2): bf16 GEMM on the Hopper tensor cores (wgmma) with a fused top-k.

Extension of the reference (which only has TF-IDF; embeddings are listed as a possible upgrade in
docs/failure-intelligence.md:43-46).  Rows and queries are float arrays rounded to bfloat16 on the way in;
the cosine is computed on those bf16 values (fp32 accumulation, fp32 norms).
"""
from __future__ import annotations

import ctypes as C
import threading
from typing import Optional, Tuple

import numpy as np

from . import _capi, _devout
from ._capi import no_distinct


def to_bf16_bits(x: np.ndarray) -> np.ndarray:
    """float32 -> bfloat16 bit patterns (uint16), round-to-nearest-even."""
    u = np.ascontiguousarray(x, dtype=np.float32).view(np.uint32).astype(np.uint64)
    return (((u + 0x7FFF + ((u >> 16) & 1)) >> 16) & 0xFFFF).astype(np.uint16)


def _ptr(a: np.ndarray, t):
    return a.ctypes.data_as(C.POINTER(t))


class DenseIndex:
    def __init__(self, dim: int, device: int = 0, row_base: int = 0):
        h = C.c_void_p()
        _capi.check(_capi.load().kv_dense_create(device, dim, row_base, C.byref(h)))
        self._h, self.dim, self.device = h, dim, device
        self._row_labels: Optional[np.ndarray] = None  # what set_row_labels gave, until the next append
        # a filtered search is two library calls (the query filter, then the search): threads sharing the index must
        # not interleave them
        self._lock = threading.Lock()

    def add(self, rows: np.ndarray) -> None:
        bits = rows if rows.dtype == np.uint16 else to_bf16_bits(rows)
        bits = np.ascontiguousarray(bits).reshape(-1, self.dim)
        with self._lock:
            _capi.check(_capi.load().kv_dense_append(self._h, bits.ctypes.data_as(C.POINTER(C.c_uint16)), bits.shape[0]))
            self._row_labels = None  # the library drops the labels on an append

    def add_device(self, rows) -> None:
        """Append rows that already live in HBM: a contiguous torch bfloat16 tensor [n, dim] on this device."""
        import torch

        assert rows.is_cuda and rows.is_contiguous() and rows.element_size() == 2 and rows.shape[-1] == self.dim
        torch.cuda.current_stream(rows.device).synchronize()  # the library copies on its own stream
        with self._lock:
            _capi.check(_capi.load().kv_dense_append_device(self._h, C.c_void_p(rows.data_ptr()), rows.shape[0]))
            self._row_labels = None

    def finalize(self) -> None:
        with self._lock:
            _capi.check(_capi.load().kv_dense_finalize(self._h))

    def set_row_labels(self, labels: Optional[np.ndarray]) -> None:
        """One label >= 0 per local row (e.g. a failure-type id), for the ``labels`` / ``same_label`` filters of the
        query methods; ``None`` clears.  Survives finalize and deletions; an append drops the labels (a filtered query
        then raises until they are set again)."""
        with self._lock:
            if labels is None:
                _capi.check(_capi.load().kv_dense_set_row_labels(self._h, None, 0))
                self._row_labels = None
                return
            labels = np.ascontiguousarray(labels, dtype=np.int32).reshape(-1)
            _capi.check(_capi.load().kv_dense_set_row_labels(self._h, _ptr(labels, C.c_int32), len(labels)))
            self._row_labels = labels.copy()

    def delete_rows(self, rows) -> None:
        """Delete local ``rows`` (any order; duplicates and rows deleted before are allowed).  A deleted row keeps its
        row id but no search returns it again, and a self-join query whose own row is deleted gets an empty list and
        no pairs.  Like an append, the deletion takes effect at the next ``finalize`` and searches raise until then."""
        rows = np.ascontiguousarray(rows, dtype=np.int64).reshape(-1)
        with self._lock:
            _capi.check(_capi.load().kv_dense_delete_rows(self._h, _ptr(rows, C.c_int64), len(rows)))

    def deleted_mask(self) -> np.ndarray:
        """bool [n_rows]: which local rows are deleted (the handle's own flags)."""
        with self._lock:
            n = self.n_rows
            out = np.zeros(n, dtype=np.uint8)
            _capi.check(_capi.load().kv_dense_deleted_rows(self._h, _ptr(out, C.c_uint8), n))
        return out.astype(bool)

    @property
    def n_live_rows(self) -> int:
        """``n_rows`` minus the deleted rows."""
        return int(_capi.load().kv_dense_live_rows(self._h))

    def _set_query_filter(self, labels: Optional[np.ndarray], n_q: int) -> None:
        """The query filter of the next search call (caller holds ``_lock``): query q only matches rows labelled
        ``labels[q]`` (-1: any row).  A count other than the search's ``n_q`` fails at the search (ValueError)."""
        if labels is None:
            return
        labels = np.ascontiguousarray(labels, dtype=np.int32).reshape(-1)
        _capi.check(_capi.load().kv_dense_set_query_filter(self._h, _ptr(labels, C.c_int32), len(labels)))

    def _same_label_filter(self, lo: int, hi: int) -> np.ndarray:
        if self._row_labels is None or len(self._row_labels) != self.n_rows:
            raise RuntimeError("same_label: the index has no row labels for its current rows (set_row_labels)")
        return self._row_labels[lo:hi]

    def last_skipped(self) -> Tuple[int, int]:
        """(items skipped, items) of the last search's kernel: (128-query tile, 256-row tile) pairs a filtered search
        did not compute because the row tile holds no live row of any label of the query tile."""
        sk, it = C.c_int64(), C.c_int64()
        _capi.check(_capi.load().kv_dense_last_skipped(self._h, C.byref(sk), C.byref(it)))
        return sk.value, it.value

    def topk_device(self, queries, k: int = 16, exclude_base: int = -1, distinct: bool = False,
                    labels: Optional[np.ndarray] = None):
        """Queries and results on the device (torch): queries bfloat16 [Q, dim]; returns (float32 [Q,k], int64 [Q,k]).
        ``exclude_base >= 0``: query q never matches GLOBAL row ``exclude_base + q`` (self-join).  ``labels``: per
        query the row label its results must carry (-1: any row; ``set_row_labels``)."""
        no_distinct(distinct, "DenseIndex.topk_device")
        import torch

        assert queries.is_cuda and queries.is_contiguous() and queries.element_size() == 2 and queries.shape[-1] == self.dim
        n = queries.shape[0]
        torch.cuda.current_stream(queries.device).synchronize()  # the library reads the queries on its own stream
        s = torch.empty((n, k), dtype=torch.float32, device=queries.device)
        r = torch.empty((n, k), dtype=torch.int64, device=queries.device)
        with self._lock:
            self._set_query_filter(labels, n)
            _capi.check(_capi.load().kv_dense_topk_device(self._h, C.c_void_p(queries.data_ptr()), n, k, exclude_base,
                                                          C.c_void_p(s.data_ptr()), C.c_void_p(r.data_ptr())))
        return s, r

    def selfjoin_topk(self, k: int = 32, lo: int = 0, hi: int | None = None, device_out: bool = False, distinct: bool = False,
                      same_label: bool = False):
        """All-pairs (BASELINE configs[3]): for local rows [lo, hi) the k nearest OTHER rows.  ``same_label``: row i's
        list holds only rows with row i's label."""
        no_distinct(distinct, "DenseIndex.selfjoin_topk")
        import torch

        hi = self.n_rows if hi is None else hi
        dev = torch.device("cuda", self.device)
        s = torch.empty((hi - lo, k), dtype=torch.float32, device=dev)
        r = torch.empty((hi - lo, k), dtype=torch.int64, device=dev)
        with self._lock:
            if same_label:
                self._set_query_filter(self._same_label_filter(lo, hi), hi - lo)
            _capi.check(_capi.load().kv_dense_selfjoin_device(self._h, lo, hi, k, C.c_void_p(s.data_ptr()),
                                                              C.c_void_p(r.data_ptr())))
        return (s, r) if device_out else (s.cpu().numpy(), r.cpu().numpy())

    @property
    def n_rows(self) -> int:
        return int(_capi.load().kv_dense_rows(self._h))

    def topk(self, queries: np.ndarray, k: int = 16, distinct: bool = False,
             labels: Optional[np.ndarray] = None) -> Tuple[np.ndarray, np.ndarray]:
        """(scores float32 [Q,k], rows int64 [Q,k]) ordered by (cosine desc, row asc); unused slots (-inf, -1).
        ``labels``: per query the row label its results must carry (-1: any row; ``set_row_labels``)."""
        no_distinct(distinct, "DenseIndex.topk")
        bits = queries if queries.dtype == np.uint16 else to_bf16_bits(queries)
        bits = np.ascontiguousarray(bits).reshape(-1, self.dim)
        n = bits.shape[0]
        scores = np.empty((n, k), dtype=np.float32)
        rows = np.empty((n, k), dtype=np.int64)
        with self._lock:
            self._set_query_filter(labels, n)
            _capi.check(_capi.load().kv_dense_topk(self._h, bits.ctypes.data_as(C.POINTER(C.c_uint16)), n, k,
                                                   scores.ctypes.data_as(C.POINTER(C.c_float)),
                                                   rows.ctypes.data_as(C.POINTER(C.c_int64))))
        return scores, rows

    def _range_fetch(self, n_q: int, n_pairs: int, device_out: bool = False):
        if device_out:
            out = _devout.range_arrays(self.device, n_q, n_pairs)
            _capi.check(_capi.load().kv_dense_range_fetch_device(self._h, *_devout.ptrs(out)))
            return out
        indptr = np.empty(n_q + 1, dtype=np.int64)
        rows = np.empty(n_pairs, dtype=np.int64)
        scores = np.empty(n_pairs, dtype=np.float32)
        _capi.check(_capi.load().kv_dense_range_fetch(self._h, indptr.ctypes.data_as(C.POINTER(C.c_int64)),
                                                      rows.ctypes.data_as(C.POINTER(C.c_int64)),
                                                      scores.ctypes.data_as(C.POINTER(C.c_float))))
        return indptr, rows, scores

    def range(self, queries: np.ndarray, threshold: float, device_out: bool = False, labels: Optional[np.ndarray] = None):
        """Threshold search: every (query, row) pair whose cosine (the float32 value ``topk`` reports, bit for bit) is
        >= ``threshold``, 0 < threshold <= 1.  ``queries``: float rows or bf16 bit patterns (uint16), host memory.
        Returns ``(indptr int64[n_q+1], rows int64[P], scores float32[P])``: query q's pairs are
        ``[indptr[q], indptr[q+1])``, ordered by (score desc, row asc); rows are global.  ``device_out``: the same
        arrays as torch tensors on the index's device.  ``labels``: per query the row label its pairs must carry (-1:
        any row; ``set_row_labels``)."""
        bits = queries if queries.dtype == np.uint16 else to_bf16_bits(queries)
        bits = np.ascontiguousarray(bits).reshape(-1, self.dim)
        n = C.c_int64(0)
        with self._lock:
            self._set_query_filter(labels, bits.shape[0])
            _capi.check(_capi.load().kv_dense_range(self._h, bits.ctypes.data_as(C.POINTER(C.c_uint16)), bits.shape[0],
                                                    np.float32(threshold), C.byref(n)))
            return self._range_fetch(bits.shape[0], n.value, device_out)

    def range_device(self, queries, threshold: float, exclude_base: int = -1, device_out: bool = False,
                     labels: Optional[np.ndarray] = None):
        """``range`` of queries on the device (a contiguous torch bfloat16 tensor [Q, dim]); results on the host, or
        with ``device_out`` as torch tensors on the index's device.
        ``exclude_base >= 0``: query q never matches GLOBAL row ``exclude_base + q``.  ``labels`` as in ``range``."""
        import torch

        assert queries.is_cuda and queries.is_contiguous() and queries.element_size() == 2 and queries.shape[-1] == self.dim
        n_q = queries.shape[0]
        torch.cuda.current_stream(queries.device).synchronize()  # the library reads the queries on its own stream
        n = C.c_int64(0)
        with self._lock:
            self._set_query_filter(labels, n_q)
            _capi.check(_capi.load().kv_dense_range_device(self._h, C.c_void_p(queries.data_ptr()), n_q,
                                                           np.float32(threshold), exclude_base, C.byref(n)))
            return self._range_fetch(n_q, n.value, device_out)

    def selfjoin_range(self, threshold: float, lo: int = 0, hi: int | None = None, device_out: bool = False,
                       same_label: bool = False):
        """All-pairs threshold search: for local rows [lo, hi) every OTHER row scoring >= ``threshold`` (CSR as in
        ``range``, query i = row lo + i).  ``same_label``: only rows with row i's label."""
        hi = self.n_rows if hi is None else hi
        n = C.c_int64(0)
        with self._lock:
            if same_label:
                self._set_query_filter(self._same_label_filter(lo, hi), hi - lo)
            _capi.check(_capi.load().kv_dense_selfjoin_range(self._h, lo, hi, np.float32(threshold), C.byref(n)))
            return self._range_fetch(hi - lo, n.value, device_out)

    def last_timing(self) -> Tuple[float, int]:
        ms, sp = C.c_float(), C.c_int64()
        _capi.check(_capi.load().kv_dense_last_timing(self._h, C.byref(ms), C.byref(sp)))
        return ms.value, sp.value

    def close(self) -> None:
        if self._h is not None:
            _capi.load().kv_dense_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
