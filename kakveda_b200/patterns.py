"""Pattern clustering on top of the all-pairs scan (SURVEY.md section 8(f) rank 3, BASELINE configs[3]).

The reference's pattern detector (services/pattern_detector/app.py:28-60) pulls every failure from the GFKB, keeps
those whose ``failure_type`` equals the event's, and upserts ONE named pattern when they span >= 2 apps.  This module
keeps that contract (``pattern_payload`` builds the same ``/patterns/upsert`` body: sorted unique failure_ids and
affected_apps, app.py:41-43,50-56) but can split a failure type into several patterns by similarity: every row's k
nearest other rows (or, with ``k=None``, every other row above the threshold) come from the device self-join, rows
whose similarity reaches the threshold are linked, connected components are the candidate patterns.  The grouping by similarity is an extension (the reference has none); its oracle
is a Python union-find over the float64 all-pairs matrix (tests).
"""
from __future__ import annotations

import ctypes as C
from typing import Any, Dict, List, Mapping, Optional, Sequence, Tuple

import numpy as np

from . import _capi


def cluster_topk(rows: np.ndarray, scores: np.ndarray, threshold: float) -> Tuple[np.ndarray, int]:
    """labels[i] = smallest row id of i's component in the graph {i ~ rows[i,j] : scores[i,j] >= threshold}."""
    rows = np.ascontiguousarray(rows, dtype=np.int64)
    scores = np.ascontiguousarray(scores, dtype=np.float32)
    n, k = rows.shape
    labels = np.empty(n, dtype=np.int64)
    count = C.c_int64(0)
    _capi.check(_capi.load().kv_cluster_topk(n, k, rows.ctypes.data_as(C.POINTER(C.c_int64)),
                                             scores.ctypes.data_as(C.POINTER(C.c_float)), float(threshold),
                                             labels.ctypes.data_as(C.POINTER(C.c_int64)), C.byref(count)))
    return labels, int(count.value)


def _cluster_csr_device(indptr, rows):
    import torch

    for name, t in (("indptr", indptr), ("rows", rows)):
        if not (isinstance(t, torch.Tensor) and t.is_cuda and t.dtype == torch.int64):
            raise ValueError(f"cluster_csr: {name} must be an int64 CUDA tensor when the other one is on the device")
    if indptr.device != rows.device or indptr.dim() != 1 or indptr.numel() < 1:
        raise ValueError("cluster_csr: indptr and rows must be on one device, indptr 1-D with n + 1 entries")
    indptr, rows = indptr.contiguous(), rows.contiguous()
    n = indptr.numel() - 1
    labels = torch.empty(n, dtype=torch.int64, device=indptr.device)
    count = C.c_int64(0)
    torch.cuda.current_stream(indptr.device).synchronize()  # the library reads the inputs on a stream of its own
    _capi.check(_capi.load().kv_cluster_csr_device(indptr.device.index, n, C.c_void_p(indptr.data_ptr()),
                                                   C.c_void_p(rows.data_ptr()), C.c_void_p(labels.data_ptr()),
                                                   C.byref(count)))
    return labels, int(count.value)


def cluster_csr(indptr, rows) -> Tuple[Any, int]:
    """labels[i] = smallest row id of i's component in the graph {i ~ rows[j] : indptr[i] <= j < indptr[i+1], rows[j] >= 0}.

    NumPy inputs are clustered on the host; int64 CUDA tensors (e.g. ``selfjoin_range(..., device_out=True)``) on
    their device, and the labels come back as a tensor there."""
    if getattr(indptr, "is_cuda", False) or getattr(rows, "is_cuda", False):
        return _cluster_csr_device(indptr, rows)
    indptr = np.ascontiguousarray(indptr, dtype=np.int64)
    rows = np.ascontiguousarray(rows, dtype=np.int64)
    n = len(indptr) - 1
    labels = np.empty(n, dtype=np.int64)
    count = C.c_int64(0)
    _capi.check(_capi.load().kv_cluster_csr(n, indptr.ctypes.data_as(C.POINTER(C.c_int64)),
                                            rows.ctypes.data_as(C.POINTER(C.c_int64)),
                                            labels.ctypes.data_as(C.POINTER(C.c_int64)), C.byref(count)))
    return labels, int(count.value)


def pattern_payload(name: str, records: Sequence[Mapping[str, Any]], description: Optional[str] = None) -> Dict[str, Any]:
    """The ``/patterns/upsert`` body the reference builds from a group of failures (app.py:41-43,50-56)."""
    affected = sorted(set(sum([list(r.get("affected_apps", [])) for r in records], [])))
    failure_ids = sorted(set(r.get("failure_id") for r in records if r.get("failure_id")))
    return {"name": name, "failure_ids": failure_ids, "affected_apps": affected, "description": description}


def detect_patterns(index, records: Sequence[Mapping[str, Any]], threshold: float = 0.8, k: Optional[int] = 32,
                    min_apps: int = 2, failure_type: Optional[str] = None,
                    filter_first: bool = False, distinct: bool = False) -> List[Dict[str, Any]]:
    """Similarity-split version of pattern_detector.on_failure.

    ``index``: a finalized ``GfkbIndex`` whose row i is ``records[i]['signature_text']`` (corpus-fit mode gives a
    symmetric measure; the default mode works too), a finalized ``DenseIndex`` whose row i is record i's embedding
    (cosine), or a finalized ``JaccardIndex`` whose row i is record i's token set.  Returns one payload per connected
    component that, restricted
    to ``failure_type`` (if given), spans at least ``min_apps`` apps (app.py:45-46) -- ordered by smallest row id.
    ``k``: rows are linked only through every row's k nearest other rows, so when a text is stored more than k times
    its copies fill the lists and pairs of similar texts are never seen.  ``k=None`` links on the exact threshold
    graph (``selfjoin_range``).
    ``filter_first`` (with ``failure_type``, ``GfkbIndex`` only): the index's row labels are set to the records' failure
    types and the self-join searches every row among the rows of its own type, so with an integer ``k`` other types
    cannot fill a row's list and hide its same-type neighbours.  With ``k=None`` the components are the default's.
    ``distinct`` (integer ``k``, ``GfkbIndex`` only): the index's row groups are set to text identity -- the records'
    (failure_type, signature_text) keys -- and every row's list holds at most one row per key, so copies link to
    their key's lowest other copy and the other k - 1 slots go to other texts: a text stored more than k times no
    longer hides its neighbours.  With ``k=None`` the components are the default's.
    """
    from .similarity import GfkbIndex

    # the index classes a mode is built for are checked before the index is touched
    if distinct and k is not None and not isinstance(index, GfkbIndex):
        raise NotImplementedError("detect_patterns(distinct=True) collapses copies on a GfkbIndex only")
    if filter_first and failure_type is not None and not isinstance(index, GfkbIndex):
        raise NotImplementedError("detect_patterns(filter_first=True) searches by label on a GfkbIndex only")
    n = len(records)
    keep = np.ones(n, dtype=bool)
    if failure_type is not None:
        keep = np.fromiter((r.get("failure_type") == failure_type for r in records), dtype=bool, count=n)
    if hasattr(index, "deleted_mask"):
        # deleted rows (GfkbIndex.delete_rows) join no pattern: the self-join never returns them and their own lists
        # are empty, so each is a singleton -- and a singleton record spanning two apps must not become a pattern
        dead = index.deleted_mask()[:n]
        keep[: len(dead)] &= ~dead
    if distinct and k is not None:
        keys: Dict[Any, int] = {}  # the (failure_type, signature_text) key an upsert versions: one text of one type
        index.set_row_groups(np.fromiter((keys.setdefault((r.get("failure_type"), r.get("signature_text")), len(keys))
                                          for r in records), dtype=np.int32, count=n))
    if filter_first and failure_type is not None:
        types: Dict[Any, int] = {}
        index.set_row_labels(np.fromiter((types.setdefault(r.get("failure_type"), len(types)) for r in records),
                                         dtype=np.int32, count=n))
        if k is None:
            indptr, rows = index.selfjoin_range(threshold, device_out=True, same_label=True)[:2]
            labels, _ = cluster_csr(indptr, rows)
            labels = labels.cpu().numpy()
        else:
            scores, rows = index.selfjoin_topk(k, same_label=True, distinct=distinct)
            labels, _ = cluster_topk(rows, scores, threshold)
    # a JaccardIndex returns the exact counts after these arrays: only the leading ones are used
    elif k is None:
        # the threshold graph stays on the device: only the n labels come back
        import torch

        indptr, rows = index.selfjoin_range(threshold, device_out=True)[:2]
        if failure_type is not None:  # rows of other failure types neither join nor bridge components
            m = indptr.numel() - 1
            if m > n or (rows.numel() and int(rows.max()) >= n):
                raise IndexError(f"detect_patterns: the index holds rows beyond the {n} records")
            keep_d = torch.from_numpy(keep).to(rows.device)
            src = torch.repeat_interleave(torch.arange(m, device=rows.device), torch.diff(indptr))
            rows = torch.where(keep_d[src] & keep_d[rows], rows, torch.full_like(rows, -1))
        labels, _ = cluster_csr(indptr, rows)
        labels = labels.cpu().numpy()
    else:
        scores, rows = index.selfjoin_topk(k, distinct=True)[:2] if distinct else index.selfjoin_topk(k)[:2]
        if failure_type is not None:
            # rows of other failure types neither join nor bridge components
            bad = ~keep[np.clip(rows, 0, n - 1)] | (rows < 0)
            scores = np.where(bad, -np.inf, scores).astype(np.float32)
            scores[~keep] = -np.inf
        labels, _ = cluster_topk(rows, scores, threshold)
    groups: Dict[int, List[int]] = {}
    for i, lab in enumerate(labels.tolist()):
        if keep[i]:
            groups.setdefault(lab, []).append(i)
    out = []
    for lab in sorted(groups):
        recs = [records[i] for i in groups[lab]]
        payload = pattern_payload(f"pattern-{lab:06d}", recs)
        if len(payload["affected_apps"]) >= min_apps:
            payload["rows"] = groups[lab]
            out.append(payload)
    return out
