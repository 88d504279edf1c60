"""64-bit fingerprint exact-match index (K4).

``fingerprint()`` of the reference (services/shared/fingerprint.py:69-71) is the first 16 hex digits of
sha256(signature_text); ``HashIndex`` stores those 64 bits per GFKB row on the device and answers "which
stored failures have exactly this fingerprint" for a batch of queries with one HBM-bound scan per 4096
queries.  The reference never queries its fingerprint, so this is an extension (oracle: integer equality).
"""
from __future__ import annotations

import ctypes as C
from typing import Iterable, Sequence, Tuple

import numpy as np

from . import _capi
from ._capi import no_distinct
from .fingerprint import fingerprint_u64


class HashIndex:
    def __init__(self, device: int = 0, row_base: int = 0):
        h = C.c_void_p()
        _capi.check(_capi.load().kv_hash_create(device, row_base, C.byref(h)))
        self._h = h

    def add_hashes(self, hashes: np.ndarray) -> None:
        hashes = np.ascontiguousarray(hashes, dtype=np.uint64)
        _capi.check(_capi.load().kv_hash_append(self._h, hashes.ctypes.data_as(C.POINTER(C.c_uint64)), len(hashes)))

    def add_signatures(self, signature_texts: Iterable[str]) -> None:
        self.add_hashes(np.fromiter((fingerprint_u64(s) for s in signature_texts), dtype=np.uint64))

    @property
    def n_rows(self) -> int:
        return int(_capi.load().kv_hash_rows(self._h))

    def match_hashes(self, hashes: np.ndarray, k: int = 16, distinct: bool = False) -> Tuple[np.ndarray, np.ndarray]:
        """(rows int64 [Q,k] ascending, -1 padded; counts int64 [Q])."""
        no_distinct(distinct, "HashIndex.match_hashes")
        hashes = np.ascontiguousarray(hashes, dtype=np.uint64)
        rows = np.empty((len(hashes), k), dtype=np.int64)
        counts = np.empty(len(hashes), dtype=np.int64)
        _capi.check(_capi.load().kv_hash_match(self._h, hashes.ctypes.data_as(C.POINTER(C.c_uint64)), len(hashes), k,
                                               rows.ctypes.data_as(C.POINTER(C.c_int64)),
                                               counts.ctypes.data_as(C.POINTER(C.c_int64))))
        return rows, counts

    def match_signatures(self, signature_texts: Sequence[str], k: int = 16, distinct: bool = False):
        no_distinct(distinct, "HashIndex.match_signatures")
        return self.match_hashes(np.fromiter((fingerprint_u64(s) for s in signature_texts), dtype=np.uint64), k)

    def last_timing(self) -> Tuple[float, int]:
        ms, passes = C.c_float(), C.c_int()
        _capi.check(_capi.load().kv_hash_last_timing(self._h, C.byref(ms), C.byref(passes)))
        return ms.value, passes.value

    def close(self) -> None:
        if self._h is not None:
            _capi.load().kv_hash_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
