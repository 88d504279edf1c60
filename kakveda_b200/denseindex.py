"""Dense-embedding cosine index (K2): bf16 GEMM on the Hopper tensor cores (wgmma) with a fused top-k.

Extension of the reference (which only has TF-IDF; embeddings are listed as a possible upgrade in
docs/failure-intelligence.md:43-46).  Rows and queries are float arrays rounded to bfloat16 on the way in;
the cosine is computed on those bf16 values (fp32 accumulation, fp32 norms).
"""
from __future__ import annotations

import ctypes as C
from typing import Tuple

import numpy as np

from . import _capi, _devout
from ._capi import no_distinct


def to_bf16_bits(x: np.ndarray) -> np.ndarray:
    """float32 -> bfloat16 bit patterns (uint16), round-to-nearest-even."""
    u = np.ascontiguousarray(x, dtype=np.float32).view(np.uint32).astype(np.uint64)
    return (((u + 0x7FFF + ((u >> 16) & 1)) >> 16) & 0xFFFF).astype(np.uint16)


class DenseIndex:
    def __init__(self, dim: int, device: int = 0, row_base: int = 0):
        h = C.c_void_p()
        _capi.check(_capi.load().kv_dense_create(device, dim, row_base, C.byref(h)))
        self._h, self.dim, self.device = h, dim, device

    def add(self, rows: np.ndarray) -> None:
        bits = rows if rows.dtype == np.uint16 else to_bf16_bits(rows)
        bits = np.ascontiguousarray(bits).reshape(-1, self.dim)
        _capi.check(_capi.load().kv_dense_append(self._h, bits.ctypes.data_as(C.POINTER(C.c_uint16)), bits.shape[0]))

    def add_device(self, rows) -> None:
        """Append rows that already live in HBM: a contiguous torch bfloat16 tensor [n, dim] on this device."""
        import torch

        assert rows.is_cuda and rows.is_contiguous() and rows.element_size() == 2 and rows.shape[-1] == self.dim
        torch.cuda.current_stream(rows.device).synchronize()  # the library copies on its own stream
        _capi.check(_capi.load().kv_dense_append_device(self._h, C.c_void_p(rows.data_ptr()), rows.shape[0]))

    def finalize(self) -> None:
        _capi.check(_capi.load().kv_dense_finalize(self._h))

    def topk_device(self, queries, k: int = 16, exclude_base: int = -1, distinct: bool = False):
        """Queries and results on the device (torch): queries bfloat16 [Q, dim]; returns (float32 [Q,k], int64 [Q,k]).
        ``exclude_base >= 0``: query q never matches GLOBAL row ``exclude_base + q`` (self-join)."""
        no_distinct(distinct, "DenseIndex.topk_device")
        import torch

        assert queries.is_cuda and queries.is_contiguous() and queries.element_size() == 2 and queries.shape[-1] == self.dim
        n = queries.shape[0]
        torch.cuda.current_stream(queries.device).synchronize()  # the library reads the queries on its own stream
        s = torch.empty((n, k), dtype=torch.float32, device=queries.device)
        r = torch.empty((n, k), dtype=torch.int64, device=queries.device)
        _capi.check(_capi.load().kv_dense_topk_device(self._h, C.c_void_p(queries.data_ptr()), n, k, exclude_base,
                                                      C.c_void_p(s.data_ptr()), C.c_void_p(r.data_ptr())))
        return s, r

    def selfjoin_topk(self, k: int = 32, lo: int = 0, hi: int | None = None, device_out: bool = False, distinct: bool = False):
        """All-pairs (BASELINE configs[3]): for local rows [lo, hi) the k nearest OTHER rows."""
        no_distinct(distinct, "DenseIndex.selfjoin_topk")
        import torch

        hi = self.n_rows if hi is None else hi
        dev = torch.device("cuda", self.device)
        s = torch.empty((hi - lo, k), dtype=torch.float32, device=dev)
        r = torch.empty((hi - lo, k), dtype=torch.int64, device=dev)
        _capi.check(_capi.load().kv_dense_selfjoin_device(self._h, lo, hi, k, C.c_void_p(s.data_ptr()), C.c_void_p(r.data_ptr())))
        return (s, r) if device_out else (s.cpu().numpy(), r.cpu().numpy())

    @property
    def n_rows(self) -> int:
        return int(_capi.load().kv_dense_rows(self._h))

    def topk(self, queries: np.ndarray, k: int = 16, distinct: bool = False) -> Tuple[np.ndarray, np.ndarray]:
        no_distinct(distinct, "DenseIndex.topk")
        bits = queries if queries.dtype == np.uint16 else to_bf16_bits(queries)
        bits = np.ascontiguousarray(bits).reshape(-1, self.dim)
        n = bits.shape[0]
        scores = np.empty((n, k), dtype=np.float32)
        rows = np.empty((n, k), dtype=np.int64)
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

    def range(self, queries: np.ndarray, threshold: float, device_out: bool = False):
        """Threshold search: every (query, row) pair whose cosine (the float32 value ``topk`` reports, bit for bit) is
        >= ``threshold``, 0 < threshold <= 1.  ``queries``: float rows or bf16 bit patterns (uint16), host memory.
        Returns ``(indptr int64[n_q+1], rows int64[P], scores float32[P])``: query q's pairs are
        ``[indptr[q], indptr[q+1])``, ordered by (score desc, row asc); rows are global.  ``device_out``: the same
        arrays as torch tensors on the index's device."""
        bits = queries if queries.dtype == np.uint16 else to_bf16_bits(queries)
        bits = np.ascontiguousarray(bits).reshape(-1, self.dim)
        n = C.c_int64(0)
        _capi.check(_capi.load().kv_dense_range(self._h, bits.ctypes.data_as(C.POINTER(C.c_uint16)), bits.shape[0],
                                                np.float32(threshold), C.byref(n)))
        return self._range_fetch(bits.shape[0], n.value, device_out)

    def range_device(self, queries, threshold: float, exclude_base: int = -1, device_out: bool = False):
        """``range`` of queries on the device (a contiguous torch bfloat16 tensor [Q, dim]); results on the host, or
        with ``device_out`` as torch tensors on the index's device.
        ``exclude_base >= 0``: query q never matches GLOBAL row ``exclude_base + q``."""
        import torch

        assert queries.is_cuda and queries.is_contiguous() and queries.element_size() == 2 and queries.shape[-1] == self.dim
        n_q = queries.shape[0]
        torch.cuda.current_stream(queries.device).synchronize()  # the library reads the queries on its own stream
        n = C.c_int64(0)
        _capi.check(_capi.load().kv_dense_range_device(self._h, C.c_void_p(queries.data_ptr()), n_q, np.float32(threshold),
                                                       exclude_base, C.byref(n)))
        return self._range_fetch(n_q, n.value, device_out)

    def selfjoin_range(self, threshold: float, lo: int = 0, hi: int | None = None, device_out: bool = False):
        """All-pairs threshold search: for local rows [lo, hi) every OTHER row scoring >= ``threshold`` (CSR as in
        ``range``, query i = row lo + i)."""
        hi = self.n_rows if hi is None else hi
        n = C.c_int64(0)
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
