"""Device outputs of the threshold searches (``device_out=True``): torch tensors on the index's device that the C ABI's
``*_range_fetch_device`` functions fill, with the dtypes and shapes of the host results."""
from __future__ import annotations

import ctypes as C


def range_arrays(device: int, n_q: int, n_pairs: int, jaccard: bool = False):
    """Uninitialised ``(indptr int64[n_q+1], rows int64[P], scores float32[P][, inter int32[P], union int32[P]])``."""
    import torch

    dev = torch.device("cuda", device)
    out = [torch.empty(n_q + 1, dtype=torch.int64, device=dev), torch.empty(n_pairs, dtype=torch.int64, device=dev),
           torch.empty(n_pairs, dtype=torch.float32, device=dev)]
    if jaccard:
        out += [torch.empty(n_pairs, dtype=torch.int32, device=dev), torch.empty(n_pairs, dtype=torch.int32, device=dev)]
    return tuple(out)


def empty_range(device: int, jaccard: bool = False):
    """The result of a search over no queries: indptr ``[0]`` and empty arrays."""
    out = range_arrays(device, 0, 0, jaccard)
    out[0].zero_()
    return out


def ptrs(tensors):
    return [C.c_void_p(t.data_ptr()) for t in tensors]
