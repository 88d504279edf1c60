"""Row-sharded GFKB over the GPUs of one box (SURVEY.md section 8e).

One process per GPU (``torch.distributed``, NCCL over NVLink/NVSwitch).  Corpus rows are split
contiguously (rank r owns rows [n*r/W, n*(r+1)/W)); every rank sees the same query batch.  The
only exchanges are

* once per append epoch: an all-reduce(sum) of the per-feature document-frequency vector, because
  TF-IDF's idf and row norms use GLOBAL df and N (``allreduce_df``);
* once per query batch: ONE all-gather of the per-shard partial top-k (scores float32, rows int64),
  followed by a local merge ordered by (score desc, row asc) -- identical on every rank
  (``gather_topk`` + ``kv_merge_topk_device``); a distinct batch merges with ``kv_merge_topk_distinct_device_on``,
  which keeps the first entry of each row group, and its seed exchange carries whole seed lists (scores and rows);
* once per deletion: an all-reduce of the live document frequencies and row count, then a statistics-only finalize
  of every shard (``ShardedGfkb.delete_rows``);
* once per threshold search: a 16-byte all-gather of the shards' pair counts, ONE all-gather of the per-shard CSR
  results packed in equal slots, and the W-way merge of the ordered runs on the device (``gather_range_packed`` +
  ``merge_range_on_device``, ``kv_merge_range_device_on``).  The threshold is fixed, so every shard searches alone.

Every rank featurises the whole corpus text so that feature ids agree without exchanging the
vocabulary (ids are deterministic, see csrc/featurizer.cpp); only its own rows go to its GPU.
The communication helpers take any torch tensors, so the world_size-2 ``gloo`` tests run them on
CPU; the compute stays in libkakveda_b200 (CUDA only).
"""
from __future__ import annotations

import ctypes as C
import os
import sys
from typing import Optional, Tuple

import numpy as np

from . import _capi, _devout
from ._capi import no_distinct
from .similarity import (MAX_QUERY_TAGS, FeatureBatch, GfkbIndex, Vocabulary, _featurize_on_device, csr_rows, gather_rows,
                         pack_texts, tag_csr, text_order)
from .store import GfkbStore


def shard_bounds(n_rows: int, world: int, rank: int) -> Tuple[int, int]:
    return n_rows * rank // world, n_rows * (rank + 1) // world


def shard_rows_by_text(batch, world: int, rank: int, n_threads: int = 0) -> np.ndarray:
    """int64, ascending: the global row ids of the ``rank``-th range of the corpus' text order (every rank computes
    the same order from the same featurised corpus, so the shards partition the rows without any exchange)."""
    perm = text_order(batch, n_threads)
    lo, hi = shard_bounds(batch.n, world, rank)
    return np.sort(perm[lo:hi].astype(np.int64))


def allreduce_df(local_df, group=None):
    """Sum per-feature document frequencies over ranks, in place; returns the tensor."""
    import torch.distributed as dist

    if dist.is_available() and dist.is_initialized() and dist.get_world_size(group) > 1:
        dist.all_reduce(local_df, op=dist.ReduceOp.SUM, group=group)
    return local_df


def gather_topk(scores, rows, group=None):
    """All-gather per-shard partial top-k: [Q,k] -> ([W,Q,k] scores, [W,Q,k] rows) on every rank."""
    import torch
    import torch.distributed as dist

    world = dist.get_world_size(group) if dist.is_available() and dist.is_initialized() else 1
    if world == 1:
        return scores.unsqueeze(0), rows.unsqueeze(0)
    q = scores.shape[0]
    gs = torch.empty((world * q,) + tuple(scores.shape[1:]), dtype=scores.dtype, device=scores.device)
    gr = torch.empty((world * q,) + tuple(rows.shape[1:]), dtype=rows.dtype, device=rows.device)
    dist.all_gather_into_tensor(gs, scores.contiguous(), group=group)  # rank-major concatenation
    dist.all_gather_into_tensor(gr, rows.contiguous(), group=group)
    return gs.view((world,) + tuple(scores.shape)), gr.view((world,) + tuple(rows.shape))


def merge_on_device(device: int, gs, gr):
    """K5 on the gathered lists: ([W,Q,k],[W,Q,k]) -> ([Q,k],[Q,k]).  Runs on torch's current stream (the one the
    all-gather was enqueued on), so no host synchronisation is needed between the collective and the merge."""
    import torch

    w, q, k = gs.shape
    out_s = torch.empty((q, k), dtype=torch.float32, device=gs.device)
    out_r = torch.empty((q, k), dtype=torch.int64, device=gs.device)
    stream = torch.cuda.current_stream(gs.device).cuda_stream
    _capi.check(_capi.load().kv_merge_topk_device_on(device, C.c_void_p(gs.data_ptr()), C.c_void_p(gr.data_ptr()), w, q, k,
                                                     q * k, q * k, C.c_void_p(out_s.data_ptr()), C.c_void_p(out_r.data_ptr()),
                                                     C.c_void_p(stream), 0))
    return out_s, out_r


def packed_layout(q: int, k: int) -> Tuple[int, int]:
    """(offset of the rows array, total bytes) of one rank's packed partial top-k: [q*k float32][pad to 8][q*k int64]."""
    off_r = (q * k * 4 + 7) // 8 * 8
    return off_r, off_r + q * k * 8


def packed_views(buf, q: int, k: int):
    """float32 [q,k] / int64 [q,k] views of a packed uint8 buffer (any torch device)."""
    import torch

    off_r, total = packed_layout(q, k)
    return (buf[: q * k * 4].view(torch.float32).view(q, k), buf[off_r:total].view(torch.int64).view(q, k))


def gather_packed(buf, group=None):
    """ONE all-gather of the packed per-shard partial top-k (scores and rows travel together): [total] uint8 ->
    [W, total] uint8 on every rank."""
    import torch
    import torch.distributed as dist

    world = dist.get_world_size(group) if dist.is_available() and dist.is_initialized() else 1
    if world == 1:
        return buf.unsqueeze(0)
    out = torch.empty((world, buf.numel()), dtype=torch.uint8, device=buf.device)
    dist.all_gather_into_tensor(out.view(-1), buf.contiguous(), group=group)
    return out


def merge_packed_on_device(device: int, gathered, q: int, k: int):
    """K5 directly on the packed all-gather buffer ([W, total] uint8), on torch's current stream, no host sync."""
    import torch

    w = gathered.shape[0]
    off_r, total = packed_layout(q, k)
    out_s = torch.empty((q, k), dtype=torch.float32, device=gathered.device)
    out_r = torch.empty((q, k), dtype=torch.int64, device=gathered.device)
    stream = torch.cuda.current_stream(gathered.device).cuda_stream
    _capi.check(_capi.load().kv_merge_topk_device_on(device, C.c_void_p(gathered.data_ptr()), C.c_void_p(gathered.data_ptr() + off_r),
                                                     w, q, k, total // 4, total // 8, C.c_void_p(out_s.data_ptr()),
                                                     C.c_void_p(out_r.data_ptr()), C.c_void_p(stream), 0))
    return out_s, out_r


def merge_packed_distinct_on_device(device: int, gathered, q: int, k: int, groups):
    """The K5 of a distinct batch (``kv_merge_topk_distinct_device_on``) directly on the packed all-gather buffer ([W,
    total] uint8): per query, in (score desc, row asc) order, the first entry of each group.  ``groups``: int32 device
    tensor, the group of every global row.  Runs on torch's current stream and waits for it: a row without a group
    raises ValueError."""
    import torch

    w = gathered.shape[0]
    off_r, total = packed_layout(q, k)
    out_s = torch.empty((q, k), dtype=torch.float32, device=gathered.device)
    out_r = torch.empty((q, k), dtype=torch.int64, device=gathered.device)
    stream = torch.cuda.current_stream(gathered.device).cuda_stream
    _capi.check(_capi.load().kv_merge_topk_distinct_device_on(device, C.c_void_p(gathered.data_ptr()),
                                                              C.c_void_p(gathered.data_ptr() + off_r), w, q, k, total // 4,
                                                              total // 8, C.c_void_p(groups.data_ptr()), groups.numel(),
                                                              C.c_void_p(out_s.data_ptr()), C.c_void_p(out_r.data_ptr()),
                                                              C.c_void_p(stream)))
    return out_s, out_r


# ---- threshold search: variable-sized results ------------------------------------------------------------------------

def range_layout(n_q: int, p_max: int, jaccard: bool = False) -> Tuple[Tuple[int, int, int, int, int], int]:
    """Byte offsets of one rank's packed threshold-search result and its slot size: indptr int64[n_q+1] | rows
    int64[p_max] | scores float32[p_max] (| inter int32[p_max] | union int32[p_max]), each 16-byte aligned."""
    al = lambda x: (x + 15) & ~15
    o_r = al(8 * (n_q + 1))
    o_s = al(o_r + 8 * p_max)
    o_i = al(o_s + 4 * p_max)
    o_u = al(o_i + 4 * p_max)
    return (0, o_r, o_s, o_i, o_u), (al(o_u + 4 * p_max) if jaccard else o_i)


def range_views(buf, n_q: int, n_pairs: int, p_max: int, jaccard: bool = False):
    """``(indptr, rows, scores[, inter, union])`` views of a packed slot (uint8 torch tensor) holding ``n_pairs`` pairs:
    what ``kv_range_fetch_device`` writes into."""
    import torch

    offs, _ = range_layout(n_q, p_max, jaccard)
    out = [buf[: 8 * (n_q + 1)].view(torch.int64), buf[offs[1]:offs[1] + 8 * n_pairs].view(torch.int64),
           buf[offs[2]:offs[2] + 4 * n_pairs].view(torch.float32)]
    if jaccard:
        out += [buf[offs[3]:offs[3] + 4 * n_pairs].view(torch.int32), buf[offs[4]:offs[4] + 4 * n_pairs].view(torch.int32)]
    return out


def gather_range_packed(device: int, n_q: int, n_pairs: int, fill, group=None, jaccard: bool = False):
    """The exchange of a sharded threshold search.  A 16-byte all-gather of (pairs, free device bytes) fixes the slot
    size from the largest shard's count; ``fill(views)`` then writes this rank's CSR result into ``range_views`` of its
    slot (no extra copy), and ONE all-gather carries every slot.  Returns ``([W, slot] uint8, pairs per rank)``.
    Every rank checks that the gathered slots plus the merged result fit the device with the least free memory, so
    they all raise the same ``MemoryError`` (with the pair counts) or none does."""
    import torch
    import torch.distributed as dist

    dev = torch.device("cuda", device)
    world = dist.get_world_size(group)
    free = torch.cuda.mem_get_info(dev)[0] + torch.cuda.memory_reserved(dev) - torch.cuda.memory_allocated(dev)
    sizes = torch.tensor([n_pairs, free], dtype=torch.int64).to(dev)
    all_sizes = torch.empty((world, 2), dtype=torch.int64, device=dev)
    dist.all_gather_into_tensor(all_sizes.view(-1), sizes, group=group)
    all_sizes = all_sizes.cpu().numpy()
    pairs = all_sizes[:, 0].astype(np.int64)
    p_max, total = int(pairs.max()), int(pairs.sum())
    _, slot = range_layout(n_q, p_max, jaccard)
    need = (world + 1) * slot + 8 * (n_q + 1) + total * (20 if jaccard else 12)
    if need > int(all_sizes[:, 1].min()):
        raise MemoryError(f"sharded threshold search: {pairs.tolist()} pairs per shard ({total} in all) need "
                          f"{need / 2**30:.2f} GiB for the exchange and the merged result, "
                          f"{int(all_sizes[:, 1].min()) / 2**30:.2f} GiB are free (raise the threshold or split the query batch)")
    buf = torch.empty(slot, dtype=torch.uint8, device=dev)
    fill(range_views(buf, n_q, n_pairs, p_max, jaccard))
    return gather_packed(buf, group), pairs


def merge_range_on_device(device: int, gathered, n_q: int, pairs, jaccard: bool = False):
    """``kv_merge_range_device_on`` directly on the gathered slots ([W, slot] uint8), on torch's current stream: the
    single CSR result ``(indptr, rows, scores[, inter, union])`` as torch tensors on the device."""
    import torch

    pairs = np.ascontiguousarray(pairs, dtype=np.int64)
    w = gathered.shape[0]
    offs, slot = range_layout(n_q, int(pairs.max()), jaccard)
    assert gathered.shape[1] == slot, (gathered.shape, slot)
    out = _devout.range_arrays(device, n_q, int(pairs.sum()), jaccard)
    base = gathered.data_ptr()
    vp = lambda o: C.c_void_p(base + o)
    stream = torch.cuda.current_stream(gathered.device).cuda_stream
    _capi.check(_capi.load().kv_merge_range_device_on(device, w, n_q, vp(0), slot // 8, vp(offs[1]), vp(offs[2]),
                                                      vp(offs[3]) if jaccard else None, vp(offs[4]) if jaccard else None,
                                                      slot, pairs.ctypes.data_as(C.POINTER(C.c_int64)),
                                                      *_devout.ptrs(out), *([None, None] if not jaccard else []),
                                                      C.c_void_p(stream)))
    return out


def _concat_ranges(parts):
    """Query blocks' CSR results (torch, on one device) -> one CSR over all the blocks."""
    import torch

    if len(parts) == 1:
        return parts[0]
    ips, off = [], 0
    for p in parts:
        ips.append(p[0][:-1] + off)
        off += int(p[0][-1])
    ips.append(torch.full((1,), off, dtype=torch.int64, device=parts[0][0].device))
    return (torch.cat(ips),) + tuple(torch.cat([p[j] for p in parts]) for j in range(1, len(parts[0])))


def _drop_queries(res, drop: np.ndarray):
    """A CSR result (torch, on one device) with no pairs for the queries where ``drop`` (bool per query) is set."""
    import torch

    if not drop.any():
        return res
    ip = res[0]
    d = torch.from_numpy(drop).to(ip.device)
    cnt = ip[1:] - ip[:-1]
    keep = torch.repeat_interleave(~d, cnt)
    out_ip = torch.zeros_like(ip)
    out_ip[1:] = torch.cumsum(torch.where(d, 0, cnt), 0)
    return (out_ip,) + tuple(t[keep] for t in res[1:])


def _host(out, device_out: bool):
    return out if device_out else tuple(t.cpu().numpy() for t in out)


def _join_blocks(n_rows: int, block: int, part, device_out: bool, empty):
    """A self-join of ``n_rows`` rows in query blocks of ``block`` rows: ``part(b0, b1)`` is the CSR result (torch, on
    the device) of the queries of rows [b0, b1); the blocks' results concatenated, or ``empty()`` without rows."""
    parts = [part(b0, min(n_rows, b0 + block)) for b0 in range(0, n_rows, block)]
    return _host(_concat_ranges(parts), device_out) if parts else empty()


def merge_exact_lists(rows: np.ndarray, scores: np.ndarray, k: int,
                      groups: Optional[np.ndarray] = None) -> Tuple[np.ndarray, np.ndarray]:
    """Per query, several ordered lists of (global row, float64 score) side by side ([Q, m] each, -1 rows unused) ->
    the first ``k`` in (score desc, row asc) order, (-1, -inf) past the last.  ``groups`` (by global row): keep only the
    first row of each group -- exact when each list is the distinct top-k of disjoint rows."""
    q = rows.shape[0]
    big = np.where(rows < 0, np.iinfo(np.int64).max, rows)
    order = np.lexsort((big, -scores), axis=1)   # last key is primary; a -1 row carries -inf
    rows, scores = np.take_along_axis(rows, order, axis=1), np.take_along_axis(scores, order, axis=1)
    out_r = np.full((q, k), -1, dtype=np.int64)
    out_s = np.full((q, k), -np.inf)
    if groups is None:
        m = min(k, rows.shape[1])
        out_r[:, :m], out_s[:, :m] = rows[:, :m], scores[:, :m]
        out_s[out_r < 0] = -np.inf
        return out_r, out_s
    for i in range(q):
        seen, j = set(), 0
        for r, sc in zip(rows[i].tolist(), scores[i].tolist()):
            if j == k:
                break
            if r < 0 or groups[r] in seen:
                continue
            seen.add(groups[r])
            out_r[i, j], out_s[i, j] = r, sc
            j += 1
    return out_r, out_s


class _ShardRows:
    """The global rows one ``ShardedGfkb`` shard holds, and the conversions between them and its index's row ids.

    Without ``row_map`` the shard holds the index range ``[lo, hi)`` and its index has ``row_base = lo``, so the index
    takes and reports global rows (every row in queries mode or on one GPU).  With ``row_map`` (a text-order shard,
    ``row_base = 0``) it holds the ascending global rows ``row_map`` lists, the ``[lo, hi)`` range of the text order,
    and its index numbers them 0, 1, ...; ``row_map_dev`` is the same array on ``device``."""

    def __init__(self, lo: int, hi: int, row_map: Optional[np.ndarray] = None, device=None):
        import torch

        self.lo, self.hi, self.row_map = lo, hi, row_map
        self.row_map_dev = None if row_map is None else torch.from_numpy(row_map).to(device)

    def part(self, per_row):
        """The entries of a per-global-row array for the local rows, in local order."""
        return per_row[self.lo:self.hi] if self.row_map is None else per_row[self.row_map]

    def local(self, rows: np.ndarray) -> np.ndarray:
        """Ascending global rows -> the local rows that hold them; the rows of other shards are dropped."""
        if self.row_map is None:
            return rows[(rows >= self.lo) & (rows < self.hi)] - self.lo
        pos = self.index_ids(rows)
        return pos[pos >= 0]

    def index_ids(self, rows: np.ndarray) -> np.ndarray:
        """Global rows -> the ids the index takes as global rows (``set_exclusions``); -1 for a row it does not hold."""
        m = self.row_map
        if m is None:
            return rows
        if not len(m):
            return np.full_like(rows, -1)
        pos = np.minimum(np.searchsorted(m, rows), len(m) - 1)
        return np.where(m[pos] == rows, pos, -1)

    def to_global(self, ids):
        """Row ids the index reports -> global rows, -1 stays -1 (ascending, so ordered lists stay ordered): a NumPy
        array is returned mapped, a torch tensor is mapped in place."""
        if self.row_map is None:
            return ids
        if isinstance(ids, np.ndarray):
            return np.where(ids >= 0, self.row_map[np.clip(ids, 0, None)], -1)
        import torch

        return ids.copy_(torch.where(ids >= 0, self.row_map_dev[ids.clamp(min=0)], ids))


class ShardedGfkb:
    """This rank's share of a GFKB job spread over ``world`` GPUs.

    ``mode="rows"`` (default, BASELINE configs[2]): the corpus rows are sharded, every rank scans its rows for
    ALL queries, one all-gather of partial top-k + merge.  ``mode="queries"``: every rank holds the WHOLE index
    (0.9 GB at 10M rows -- trivial next to 180 GB of HBM) and answers its contiguous slice of the query batch; the
    only exchange is the all-gather of the finished results.  Pruning thresholds are as tight as on one GPU, so
    this mode scales almost linearly; it is offered because the index is so small, not used for the headline.
    """

    def __init__(self, device: int, rank: int = 0, world: int = 1, group=None, mode: str = "rows", order: str = "index"):
        if mode not in ("rows", "queries"):
            raise ValueError("mode must be 'rows' or 'queries'")
        if order not in ("index", "text"):
            raise ValueError("order must be 'index' or 'text'")
        self.mode = mode
        # order="text" (rows mode): rank r owns the r-th RANGE OF THE GLOBAL TEXT ORDER instead of a range of row
        # indices.  Near-duplicate rows then sit in one shard and its 64-row chunks are as tight as the single
        # index's, which is what block-max pruning lives on; the rows keep their global ids (local results are
        # mapped through `row_map` before the all-gather; ties still order by global id because every shard keeps
        # its rows in ascending global order).  Host-only preparation, no kernel is involved.
        self.order = order
        self.row_map = None
        self._rows: Optional[_ShardRows] = None   # build_packed: the global rows this shard holds
        self.device, self.rank, self.world, self.group = device, rank, world, group
        self.vocab = Vocabulary()
        self.index: Optional[GfkbIndex] = None
        self.n_global = 0
        self._corpus = None   # (data, offsets, mode) of the corpus text: the queries of selfjoin_range
        self._has_labels = self._has_groups = False   # set_row_labels / set_row_groups
        self._has_tags = False                          # set_row_tags
        self._groups_dev = None   # rows mode on several GPUs: the group of every global row, for the distinct merges
        self._groups_host = None  # set_row_groups: the group of every global row, for the merge of exact_topk
        self._deleted = None      # delete_rows: bool per global row (every rank deletes the same rows)
        # (live df int64 by feature, live row count) of the whole sharded corpus, all-reduced by build_packed and
        # delete_rows in rows mode on several GPUs (None: not known, the shards' own statistics when W = 1)
        self._stats: Optional[Tuple[np.ndarray, int]] = None

    @property
    def n_rows(self) -> int:
        """Rows of the whole corpus, deleted ones included, as ``GfkbIndex.n_rows`` of one index holding them all."""
        return self.n_global

    def build_packed(self, data, offsets: np.ndarray, mode: int = 0, n_threads: int = 0) -> None:
        import torch

        self._corpus = (data, np.ascontiguousarray(offsets, dtype=np.int64), mode)
        fb = self.vocab.featurize_packed(data, offsets, mode, grow=True, n_threads=n_threads)
        self.n_global = fb.n
        lo, hi = shard_bounds(fb.n, self.world, self.rank) if self.mode == "rows" else (0, fb.n)
        if self.mode == "rows" and self.order == "text" and self.world > 1:
            sel = shard_rows_by_text(fb, self.world, self.rank, n_threads)
            self._rows = _ShardRows(lo, hi, sel, f"cuda:{self.device}")
            self.index = GfkbIndex(device=self.device, row_base=0, vocab=self.vocab)
            self.index.add_features(gather_rows(fb, sel, n_threads))
        else:
            self._rows = _ShardRows(lo, hi)
            self.index = GfkbIndex(device=self.device, row_base=lo, vocab=self.vocab)
            self.index.add_features(fb, lo, hi)
        self.row_map = self._rows.row_map_dev
        fb.close()
        self._stats = None
        if self.world > 1 and self.mode == "rows":
            df = torch.from_numpy(self.index.local_df().astype(np.int32)).to(f"cuda:{self.device}")
            allreduce_df(df, self.group)
            df = df.cpu().numpy()
            self._stats = (df.astype(np.int64), self.n_global)
            self.index.set_global_df(df.astype(np.uint32), self.n_global)
        self.index.finalize()

    def _exchange_thresholds(self, n_q: int) -> None:
        """Row-sharded mode: map every peer's pruning-threshold array into this rank's scan kernel (CUDA IPC over
        NVLink peer memory), so a k-th-score bound established on one GPU prunes on all of them while the kernels
        run.  Re-done only when a batch outgrows the exchanged capacity."""
        import os

        import torch.distributed as dist

        if self.world == 1 or self.mode != "rows" or os.environ.get("KAKVEDA_B200_NO_PEER_THR") == "1":
            return
        if n_q <= getattr(self, "_thr_cap", 0):
            return
        lib = _capi.load()
        cap = max(int(n_q), 1 << 20)
        _capi.check(lib.kv_index_thresholds_peers(self.index._h, None, 0, 0))       # unmap before re-exporting
        dist.barrier(group=self.group)                                             # nobody pushes into an array being replaced
        buf = C.create_string_buffer(64)
        mine = b""
        try:
            _capi.check(lib.kv_index_thresholds_export(self.index._h, cap, buf))
            mine = bytes(buf.raw)
        except RuntimeError as e:                                                  # no CUDA IPC here: scan with local bounds only
            print(f"[kakveda_b200] rank {self.rank}: thresholds not exported ({e})", file=sys.stderr)
        handles = [None] * self.world
        dist.all_gather_object(handles, mine, group=self.group)
        peers = [h for r, h in enumerate(handles) if r != self.rank and h]
        self.n_threshold_peers = 0
        if peers:
            try:
                _capi.check(lib.kv_index_thresholds_peers(self.index._h, b"".join(peers), len(peers), cap))
                self.n_threshold_peers = len(peers)
            except RuntimeError as e:
                print(f"[kakveda_b200] rank {self.rank}: peer thresholds not mapped ({e})", file=sys.stderr)
        dist.barrier(group=self.group)
        self._thr_cap = cap

    def set_resident(self, qfb: FeatureBatch) -> None:
        """Make a featurised batch the resident batch.  In queries mode on several GPUs this rank keeps only its slice
        of the queries, which is empty when the batch has fewer queries than there are ranks."""
        q = qfb.n
        lo, hi = shard_bounds(q, self.world, self.rank) if self.mode == "queries" and self.world > 1 else (0, q)
        if (lo, hi) == (0, q):
            self.index.upload_queries(qfb)
        elif hi > lo:   # this rank's slice of the batch: re-pack the CSR rows [lo, hi)
            self.index._upload(np.ascontiguousarray(qfb.indptr[lo:hi + 1]), qfb.ids, qfb.tf,
                               np.ascontiguousarray(qfb.oov[lo:hi]), hi - lo)
        self._resident_q, self._qslice = q, (lo, hi)
        self._exchange_thresholds(q)

    def _check_filters(self, q: int, labels: Optional[np.ndarray], tags, distinct: bool):
        """``labels=`` / ``tags=`` / ``distinct=`` of a batch of ``q`` queries, checked before anything is sent, so
        every rank raises the same error: ``(labels int32 or None, tags CSR or None)``."""
        if tags is not None:
            tags = tag_csr(tags, q, "tags")
            ip, t = tags
            if len(t) and t.min() < 0:
                raise ValueError("tags: a negative tag")
            if q and np.diff(ip).max() > MAX_QUERY_TAGS:
                raise ValueError(f"tags: a query with more than {MAX_QUERY_TAGS} tags")
            if not self._has_tags:
                raise ValueError("tags: the sharded index has no row tags (set_row_tags)")
        if labels is not None:
            labels = np.ascontiguousarray(labels, dtype=np.int32).reshape(-1)
            if len(labels) != q:
                raise ValueError(f"labels: {len(labels)} labels for a batch of {q} queries")
            if q and labels.min() < -1:
                raise ValueError("labels: a label below -1")
            if not self._has_labels:
                raise ValueError("labels: the sharded index has no row labels (set_row_labels)")
        if distinct and not self._has_groups:
            raise ValueError("distinct: the sharded index has no row groups (set_row_groups)")
        return labels, tags

    def _apply_filters(self, labels: Optional[np.ndarray], tags, distinct: bool) -> None:
        """Checked filters and distinct mode -> this rank's slice of the resident batch, the same on every rank (the
        threshold exchange relies on it).  A filter not given is cleared, so none carries over from an earlier search."""
        lo, hi = self._qslice
        if hi > lo:
            self.index.set_filter(None if labels is None else labels[lo:hi])
            self.index.set_tag_filter(None if tags is None else csr_rows(*tags, np.arange(lo, hi)))
            # rows mode on several GPUs runs the two-phase top-k, whose seed lists topk_resident merges group-aware
            self.index.set_distinct(distinct, merged_seeds=self.mode == "rows" and self.world > 1)

    def topk_resident(self, k: int, labels: Optional[np.ndarray] = None, distinct: bool = False, tags=None):
        """Device-only step on the uploaded batch: local scan+merge, all-gather, global merge.  ``labels``: per query
        the row label its results must carry (-1: any row; ``set_row_labels``).  ``distinct``: at most one row per group
        (``set_row_groups``), as ``GfkbIndex.topk_features``.  ``tags``: per query a tag set its results' rows must
        meet (``set_row_tags``; each shard filters its own rows, the exchanges are unchanged).  All combine."""
        import torch

        q = self._resident_q
        dev = f"cuda:{self.device}"
        labels, tags = self._check_filters(q, labels, tags, distinct)
        self._apply_filters(labels, tags, distinct)
        if self.mode == "queries" and self.world > 1:
            import torch.distributed as dist

            lo, hi = self._qslice
            per = (q + self.world - 1) // self.world  # equal-sized slots for the all-gather
            s = torch.full((per, k), float("-inf"), dtype=torch.float32, device=dev)
            r = torch.full((per, k), -1, dtype=torch.int64, device=dev)
            if hi > lo:
                self.index.topk_resident(k, s.data_ptr(), r.data_ptr())
            gs = torch.empty((self.world * per, k), dtype=torch.float32, device=dev)
            gr = torch.empty((self.world * per, k), dtype=torch.int64, device=dev)
            dist.all_gather_into_tensor(gs, s, group=self.group)
            dist.all_gather_into_tensor(gr, r, group=self.group)
            keep = torch.cat([torch.arange(w * per, w * per + (shard_bounds(q, self.world, w)[1] - shard_bounds(q, self.world, w)[0]),
                                           device=dev) for w in range(self.world)])
            return gs[keep], gr[keep]
        # rows mode: the local result lands in ONE packed buffer (scores + rows), which is what travels
        buf = torch.empty(packed_layout(q, k)[1], dtype=torch.uint8, device=dev)
        s, r = packed_views(buf, q, k)
        if self.world == 1:
            self.index.topk_resident(k, s.data_ptr(), r.data_ptr())
            self._rows.to_global(r)
            return s, r
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(5)]
        # phase 1: bounds + seed scan on every shard; the shards' seed lists are merged (small all-gather) and the GLOBAL
        # k-th seed score of every query becomes every shard's pruning threshold -- each shard then scans only what a
        # single index would scan of its rows
        import torch.distributed as dist

        if distinct:
            # One group can sit in several shards' seed lists, so the k-th of the W x k scores may count it twice: the
            # whole seed lists travel (12 bytes an entry, rows mapped to global ids first) and the k-th seed score is
            # slot k-1 of their distinct merge -- k distinct groups that good exist, a lower bound of the k-th group score.
            seed = torch.empty(packed_layout(q, k)[1], dtype=torch.uint8, device=dev)
            ss, sr = packed_views(seed, q, k)
            ss.fill_(float("-inf"))   # null and irregular queries get no seed list
            sr.fill_(-1)
            torch.cuda.current_stream().synchronize()   # the seed scan writes on the index's own stream
            self.index.topk_resident_seed(k, ss.data_ptr(), sr.data_ptr())
            ev[0].record()
            self._rows.to_global(sr)
            kth = merge_packed_distinct_on_device(self.device, gather_packed(seed, self.group), q, k,
                                                  self._groups_dev)[0][:, k - 1].contiguous()
        else:
            self.index.topk_resident_seed(k, s.data_ptr(), r.data_ptr())
            ev[0].record()
            # only the seed SCORES travel (6.4 MB per rank at 100k queries): the global k-th seed score of a query is the
            # k-th largest of the W x k gathered scores (the shards hold disjoint rows)
            gs = torch.empty((self.world, q, k), dtype=torch.float32, device=dev)
            dist.all_gather_into_tensor(gs.view(-1), s.contiguous().view(-1), group=self.group)
            kth = torch.topk(gs.permute(1, 0, 2).reshape(q, self.world * k), k, dim=1).values[:, k - 1].contiguous()
        ev[1].record()
        torch.cuda.current_stream().synchronize()
        self.index.raise_thresholds(kth.data_ptr(), q)
        # phase 2: candidate selection + scan, then the exchange of the partial top-k
        self.index.topk_resident_finish(k, s.data_ptr(), r.data_ptr())
        self._rows.to_global(r)
        ev[2].record()
        gathered = gather_packed(buf, self.group)          # the all-gather of the partial top-k
        ev[3].record()
        if distinct:
            out = merge_packed_distinct_on_device(self.device, gathered, q, k, self._groups_dev)
        else:
            out = merge_packed_on_device(self.device, gathered, q, k)
        ev[4].record()
        # The collective doubles as the barrier between batches for the cross-GPU threshold pushes: no rank may start
        # the next batch's scan (which resets and pushes thresholds) before every rank has finished this one's.
        torch.cuda.current_stream().synchronize()
        self.last_exchange_ms = (ev[2].elapsed_time(ev[3]), ev[3].elapsed_time(ev[4]), ev[0].elapsed_time(ev[1]))
        return out

    # ---- sharded preparation of a query batch (rows mode, world > 1) -------------------------------------------------
    @staticmethod
    def _slice_layout(nq_cap: int, nnz_cap: int):
        """Byte offsets of one rank's slot in the exchanged buffer: header int64[2] (queries, entries) | indptr
        int64[nq_cap+1] | oov float64[nq_cap] | order int32[nq_cap] | flags uint8[nq_cap] | ids uint32[nnz_cap] | tf."""
        al = lambda x: (x + 15) & ~15
        o_ip = 16
        o_oov = al(o_ip + 8 * (nq_cap + 1))
        o_ord = al(o_oov + 8 * nq_cap)
        o_fl = al(o_ord + 4 * nq_cap)
        o_ids = al(o_fl + nq_cap)
        o_tf = al(o_ids + 4 * nnz_cap)
        return o_ip, o_oov, o_ord, o_fl, o_ids, o_tf, al(o_tf + 4 * nnz_cap)

    def upload_text_sharded(self, data, offsets: np.ndarray, mode: int = 0) -> int:
        """Rows mode on several GPUs: every rank featurises, classifies and text-sorts only ITS slice of the query batch
        (1/world of the host work), the slices travel in one all-gather over NVLink (plus a 16-byte one for the sizes),
        and every rank uploads the assembled batch with the slice orders merged instead of re-sorted.  The resident
        batch is identical to ``upload(featurize(all queries))``.  Returns the number of queries."""
        import time

        import torch
        import torch.distributed as dist

        t0 = time.perf_counter()
        offsets = np.ascontiguousarray(offsets, dtype=np.int64)
        n_q = len(offsets) - 1
        dev = f"cuda:{self.device}"
        lo, hi = shard_bounds(n_q, self.world, self.rank)
        qfb = self.vocab.featurize_packed(data, offsets[lo:hi + 1], mode, grow=False)
        try:
            t1 = time.perf_counter()
            n_loc, nnz = qfb.n, int(qfb.indptr[qfb.n] - qfb.indptr[0])
            sizes = torch.tensor([n_loc, nnz], dtype=torch.int64).to(dev)
            all_sizes = torch.empty((self.world, 2), dtype=torch.int64, device=dev)
            dist.all_gather_into_tensor(all_sizes.view(-1), sizes, group=self.group)
            all_sizes = all_sizes.cpu().numpy()
            nq_cap, nnz_cap = int(all_sizes[:, 0].max()), int(all_sizes[:, 1].max())
            o_ip, o_oov, o_ord, o_fl, o_ids, o_tf, slot = self._slice_layout(nq_cap, nnz_cap)
            if getattr(self, "_xq_cap", 0) < slot:           # pinned staging + device buffers, grown geometrically
                cap = max(slot, 2 * getattr(self, "_xq_cap", 0))
                self._xq_send = torch.empty(cap, dtype=torch.uint8).pin_memory()
                self._xq_recv = torch.empty(cap * self.world, dtype=torch.uint8).pin_memory()
                self._xq_dsend = torch.empty(cap, dtype=torch.uint8, device=dev)
                self._xq_drecv = torch.empty(cap * self.world, dtype=torch.uint8, device=dev)
                self._xq_cap = cap
            send = self._xq_send.numpy()
            send[0:16].view(np.int64)[:] = (n_loc, nnz)
            # the slice goes out re-stored in text order, written straight into the pinned send buffer
            self.index.prepare_slice(qfb, out=(send[o_ip:o_ip + 8 * (n_loc + 1)].view(np.int64),
                                               send[o_ids:o_ids + 4 * nnz].view(np.uint32), send[o_tf:o_tf + 4 * nnz].view(np.uint32),
                                               send[o_oov:o_oov + 8 * n_loc].view(np.float64),
                                               send[o_ord:o_ord + 4 * n_loc].view(np.int32), send[o_fl:o_fl + n_loc]))
            self._xq_dsend[:slot].copy_(self._xq_send[:slot], non_blocking=True)
            dist.all_gather_into_tensor(self._xq_drecv[:slot * self.world], self._xq_dsend[:slot], group=self.group)
            self._xq_recv[:slot * self.world].copy_(self._xq_drecv[:slot * self.world], non_blocking=True)
            torch.cuda.current_stream().synchronize()
            t2 = time.perf_counter()
            recv = self._xq_recv.numpy()
            runs = []
            for w in range(self.world):
                b = recv[w * slot:(w + 1) * slot]
                nq_w, nnz_w = (int(x) for x in b[0:16].view(np.int64))
                if (nq_w, nnz_w) != (int(all_sizes[w, 0]), int(all_sizes[w, 1])):
                    raise RuntimeError("query-slice exchange: header does not match the announced sizes")
                runs.append((b[o_ip:o_ip + 8 * (nq_w + 1)].view(np.int64), b[o_ids:o_ids + 4 * nnz_w].view(np.uint32),
                             b[o_tf:o_tf + 4 * nnz_w].view(np.uint32), b[o_oov:o_oov + 8 * nq_w].view(np.float64),
                             b[o_ord:o_ord + 4 * nq_w].view(np.int32), b[o_fl:o_fl + nq_w]))
            got = self.index.upload_query_runs(runs)
            if got != n_q:
                raise RuntimeError(f"query-slice exchange: {got} queries assembled, {n_q} expected")
            self._exchange_thresholds(n_q)
            self._resident_q, self._qslice = n_q, (0, n_q)
            t3 = time.perf_counter()
            self.last_prepare_split_ms = {"featurize_slice": 1e3 * (t1 - t0), "slice_order_and_exchange": 1e3 * (t2 - t1),
                                          "assemble_and_upload": 1e3 * (t3 - t2),
                                          "slice_bytes": int(slot), "upload_host_ms": self.index.last_prepare_ms()}
            return n_q
        finally:
            qfb.close()

    def _read_back(self, s, r):
        """Device results -> NumPy through two alternating pinned host buffers (a pageable ``.cpu()`` copy of the 19 MB
        result costs 5 ms, a pinned one < 1 ms).  The returned arrays are views of those buffers: they stay valid until
        the second-next call; copy them to keep them longer."""
        import torch

        slot = getattr(self, "_rb_slot", 0) ^ 1
        self._rb_slot = slot
        bufs = getattr(self, "_rb_bufs", None)
        if bufs is None or bufs[0][0].shape != s.shape:   # both buffers at once: pinning memory is slow (cudaHostAlloc)
            bufs = self._rb_bufs = [(torch.empty(s.shape, dtype=s.dtype).pin_memory(), torch.empty(r.shape, dtype=r.dtype).pin_memory())
                                    for _ in range(2)]
        hs, hr = bufs[slot]
        hs.copy_(s, non_blocking=True)
        hr.copy_(r, non_blocking=True)
        torch.cuda.current_stream().synchronize()
        return hs.numpy(), hr.numpy()

    def topk_packed(self, data, offsets: np.ndarray, k: int, mode: int = 0, labels: Optional[np.ndarray] = None,
                    distinct: bool = False, tags=None):
        """End-to-end step from host text: featurise, upload, scan, exchange, merge, read back.  ``last_e2e_ms`` keeps
        the wall-clock split of the last call (featurise / upload incl. table kernels / device step / read-back).
        ``labels`` / ``distinct`` / ``tags`` as for ``topk_resident``."""
        import time

        import torch

        t0 = time.perf_counter()
        n_q = len(offsets) - 1
        sliced = self.world > 1 and self.mode == "rows" and os.environ.get("KAKVEDA_B200_NO_SLICED_PREP") != "1"
        qfb = None
        try:
            if sliced:
                self.upload_text_sharded(data, offsets, mode)
            elif self.world == 1 and n_q and _featurize_on_device(n_q):
                self.index.upload_text(data, offsets, mode)   # featurise, classify and order on the device
                self._resident_q, self._qslice = n_q, (0, n_q)
            else:
                qfb = self.vocab.featurize_packed(data, offsets, mode, grow=False)
                t1 = time.perf_counter()
                self.set_resident(qfb)
            t2 = time.perf_counter()
            s, r = self.topk_resident(k, labels, distinct, tags)
            torch.cuda.current_stream().synchronize()
            t3 = time.perf_counter()
            out = self._read_back(s, r)
            t4 = time.perf_counter()
        finally:
            if qfb is not None:
                qfb.close()
        step = {"device_step": 1e3 * (t3 - t2), "read_back": 1e3 * (t4 - t3)}
        if sliced:
            self.last_e2e_ms = {"prepare_sharded": 1e3 * (t2 - t0), **step, "prepare_split": self.last_prepare_split_ms}
        elif qfb is None:
            prep = self.index.last_prepare_ms()  # text upload + featurisation, classification, order, tables + copies
            self.last_e2e_ms = {"featurize": prep[0], "upload": 1e3 * (t2 - t0) - prep[0], **step, "upload_device_ms": prep}
        else:
            self.last_e2e_ms = {"featurize": 1e3 * (t1 - t0), "upload": 1e3 * (t2 - t1), **step,
                                "upload_host_ms": self.index.last_prepare_ms()}  # staging, classification, order, copies+tables
        return out

    # ---- threshold search ------------------------------------------------------------------------------------------
    def set_row_labels(self, global_labels: Optional[np.ndarray]) -> None:
        """One label >= 0 per GLOBAL row (e.g. a failure-type id): this shard keeps its rows' labels (by index range, or
        through ``row_map`` for a text-order shard), for ``labels=`` of the top-k and threshold searches.  ``None``
        clears."""
        if global_labels is None:
            self.index.set_row_labels(None)
            self._has_labels = False
            return
        lab = np.ascontiguousarray(global_labels, dtype=np.int32)
        if len(lab) != self.n_global:
            raise ValueError(f"set_row_labels: {len(lab)} labels for a corpus of {self.n_global} rows")
        self.index.set_row_labels(self._rows.part(lab))
        self._has_labels = True

    def set_row_tags(self, global_sets) -> None:
        """A tag set per GLOBAL row (a list of lists or an ``(indptr, tags)`` pair, as ``GfkbIndex.set_row_tags``): this
        shard keeps its rows' sets as ``set_row_labels`` keeps labels, for ``tags=`` of the top-k, exact top-k and
        threshold searches.  ``None`` clears."""
        if global_sets is None:
            self.index.set_row_tags(None)
            self._has_tags = False
            return
        ip, t = tag_csr(global_sets, self.n_global, "set_row_tags")
        self.index.set_row_tags(csr_rows(ip, t, self._rows.part(np.arange(self.n_global))))
        self._has_tags = True

    def set_row_groups(self, global_groups: Optional[np.ndarray]) -> None:
        """One group >= 0 per GLOBAL row (e.g. one id per distinct text), for ``distinct=True`` of the top-k: this shard
        keeps its rows' groups as ``set_row_labels`` keeps labels.  In rows mode on several GPUs the rank also keeps the
        whole table on its device (int32 per global row, 40 MB at 10M rows) for the distinct merges of the seed lists
        and of the partial top-k.  ``None`` clears."""
        import torch

        if global_groups is None:
            self.index.set_row_groups(None)
            self._has_groups, self._groups_dev, self._groups_host = False, None, None
            return
        grp = np.ascontiguousarray(global_groups, dtype=np.int32).reshape(-1)
        if len(grp) != self.n_global:
            raise ValueError(f"set_row_groups: {len(grp)} groups for a corpus of {self.n_global} rows")
        if len(grp) and grp.min() < 0:
            raise ValueError("set_row_groups: a negative group")
        self.index.set_row_groups(self._rows.part(grp))
        self._has_groups = True
        self._groups_host = grp
        self._groups_dev = torch.from_numpy(grp).to(f"cuda:{self.device}") if self.mode == "rows" and self.world > 1 else None

    # ---- global statistics -------------------------------------------------------------------------------------------
    def _reduce_stats(self) -> Tuple[np.ndarray, int]:
        """(live df int64, live row count) of the whole sharded corpus: ONE all-reduce in rows mode on several GPUs
        (cached until the next build or deletion), this shard's own statistics otherwise."""
        import torch

        if self.world > 1 and self.mode == "rows":
            if self._stats is None:
                cnt = torch.from_numpy(np.append(self.index.local_df().astype(np.int64), self.index.n_live_rows)).to(f"cuda:{self.device}")
                allreduce_df(cnt, self.group)
                cnt = cnt.cpu().numpy()
                self._stats = (cnt[:-1], int(cnt[-1]))
            return self._stats
        return self.index.local_df().astype(np.int64), self.index.n_live_rows

    @staticmethod
    def _check_extra(extra_df: Optional[np.ndarray], extra_rows: int) -> Optional[np.ndarray]:
        if extra_df is None:
            if extra_rows:
                raise ValueError("extra_rows without extra_df")
            return None
        extra = np.ascontiguousarray(extra_df, dtype=np.int64).reshape(-1)
        if extra_rows < 0 or (len(extra) and extra.min() < 0):
            raise ValueError("extra segment statistics: a negative count")
        return extra

    def _set_stats(self, extra: Optional[np.ndarray], extra_rows: int) -> Tuple[np.ndarray, int]:
        """The corpus' statistics plus an extra segment's (df, rows) -> every shard, by a statistics-only finalize."""
        df, n = self._reduce_stats()
        v = max(len(self.vocab), len(df), 0 if extra is None else len(extra))
        tot = np.zeros(v, dtype=np.int64)
        tot[:len(df)] += df
        if extra is not None:
            tot[:len(extra)] += extra
        n += extra_rows
        self.index.set_global_df(tot.astype(np.uint32), n)
        self.index.finalize()
        return tot, n

    def set_statistics(self, extra_df: Optional[np.ndarray] = None, extra_rows: int = 0) -> Tuple[np.ndarray, int]:
        """Global TF-IDF statistics for a corpus that is this sharded GFKB PLUS an extra segment held elsewhere (e.g.
        the replicated tail of ``ShardedGfkbStore``): df = the shards' live df + ``extra_df``, N = their live rows +
        ``extra_rows``; every shard then refreshes with a statistics-only finalize.  A collective (every rank passes the
        same arguments), but the shards' df are all-reduced only once per build or deletion and cached, so a refresh
        after an append to the extra segment exchanges nothing.  Returns ``(df int64 [vocabulary], N)``, which the extra
        segment needs too.  Bad arguments raise ValueError on every rank before anything is exchanged."""
        extra = self._check_extra(extra_df, extra_rows)
        return self._set_stats(extra, int(extra_rows))

    # ---- row deletion ------------------------------------------------------------------------------------------------
    def delete_rows(self, global_rows, extra_df: Optional[np.ndarray] = None,
                    extra_rows: int = 0) -> Optional[Tuple[np.ndarray, int]]:
        """Delete GLOBAL rows (any order, duplicates and rows deleted before allowed).  A collective: every rank calls it
        with the same rows.  Each shard deletes the rows it holds; in rows mode on several GPUs the live document
        frequencies and the live row count are then all-reduced, and every shard refreshes its statistics with a
        statistics-only finalize, so that every search afterwards equals a single index with the same deletions.  Rows
        outside the corpus raise ValueError on every rank before anything is deleted.  The resident batch is dropped.
        ``extra_df`` / ``extra_rows``: the statistics of an extra segment, as for ``set_statistics``, added in the same
        refresh (one all-reduce for the whole deletion); the call then returns what ``set_statistics`` returns."""
        rows = np.unique(np.ascontiguousarray(global_rows, dtype=np.int64).reshape(-1))
        if len(rows) and (rows[0] < 0 or rows[-1] >= self.n_global):
            bad = rows[0] if rows[0] < 0 else rows[-1]
            raise ValueError(f"delete_rows: row {bad} outside the corpus of {self.n_global} rows")
        extra = self._check_extra(extra_df, extra_rows)
        local = self._rows.local(rows)
        if len(local):
            self.index.delete_rows(local)
        self._stats = None
        out = None
        if extra is not None:
            out = self._set_stats(extra, int(extra_rows))
        else:
            if self.world > 1 and self.mode == "rows":
                df, n = self._reduce_stats()
                self.index.set_global_df(df.astype(np.uint32), n)
            self.index.finalize()
        if self._deleted is None:
            self._deleted = np.zeros(self.n_global, dtype=bool)
        self._deleted[rows] = True
        return out

    def deleted_mask(self) -> np.ndarray:
        """bool [n_global]: which global rows are deleted (the same on every rank)."""
        return np.zeros(self.n_global, dtype=bool) if self._deleted is None else self._deleted.copy()

    @property
    def n_live_rows(self) -> int:
        """The global row count minus the deleted rows."""
        return self.n_global - (0 if self._deleted is None else int(self._deleted.sum()))

    # ---- exact top-k -------------------------------------------------------------------------------------------------
    def exact_topk(self, qfb: FeatureBatch, k: int, labels: Optional[np.ndarray] = None,
                   distinct: bool = False, tags=None) -> Tuple[np.ndarray, np.ndarray]:
        """Every query's best ``k`` rows over the whole sharded corpus with no candidate stage: ``(rows int64 [Q,k],
        scores float64 [Q,k])``, global rows ordered by (score desc, row asc), (-1, -inf) past the last; identical on
        every rank.  Each shard runs ``GfkbIndex.exact_topk`` (K1a over its rows, selection on the device, K6 scores:
        only k rows per query leave the device); in rows mode on several GPUs ONE all-gather carries the shards' lists
        and every rank merges them.  ``labels`` / ``distinct`` / ``tags`` as for ``topk_resident``; a distinct merge keeps
        the first row of each group.  A collective; bad arguments raise ValueError on every rank before it starts."""
        import torch

        q = qfb.n
        if not 1 <= k <= 32:
            raise ValueError(f"exact_topk: k must be 1..32, not {k}")
        labels, tags = self._check_filters(q, labels, tags, distinct)
        rows, scores = self.index.exact_topk(qfb, k, labels, distinct, tags)
        rows = self._rows.to_global(rows)
        if self.world == 1 or self.mode != "rows":
            return rows, scores
        dev = f"cuda:{self.device}"
        buf = torch.empty(16 * q * k, dtype=torch.uint8)
        buf[:8 * q * k].view(torch.float64).copy_(torch.from_numpy(scores.reshape(-1)))
        buf[8 * q * k:].view(torch.int64).copy_(torch.from_numpy(rows.reshape(-1)))
        got = gather_packed(buf.to(dev), self.group).cpu()
        s_all = got[:, :8 * q * k].contiguous().view(torch.float64).numpy().reshape(self.world, q, k)
        r_all = got[:, 8 * q * k:].contiguous().view(torch.int64).numpy().reshape(self.world, q, k)
        s_all = s_all.transpose(1, 0, 2).reshape(q, self.world * k)
        r_all = r_all.transpose(1, 0, 2).reshape(q, self.world * k)
        return merge_exact_lists(r_all, s_all, k, self._groups_host if distinct else None)

    def close(self) -> None:
        """Release this shard's index (the vocabulary stays with its owner)."""
        if self.index is not None:
            self.index.close()
            self.index = None

    def range_resident(self, threshold: float, device_out: bool = False, labels: Optional[np.ndarray] = None, tags=None):
        """Threshold search of the resident batch over the whole sharded corpus: ``(indptr int64[n_q+1], rows int64[P],
        scores float32[P])`` as ``GfkbIndex.range`` returns them (global rows, each query's pairs by (score desc, row
        asc)), NumPy arrays or with ``device_out`` torch tensors on this rank's device; identical on every rank.
        ``labels``: per query the row label its pairs must carry (-1: any row; ``set_row_labels``).  ``tags``: per query
        a tag set its pairs' rows must meet (``set_row_tags``).  A search applies exactly the filters it is given: none
        carries over from an earlier search of the same batch.  Bad arguments raise ValueError on every rank before
        anything is exchanged.  Every shard searches its rows alone (the threshold is fixed); one all-gather of the
        results and the device merge follow.  In queries mode a rank whose slice of the batch is empty (a batch with
        fewer queries than ranks) contributes no pairs."""
        q = self._resident_q
        lo, hi = self._qslice
        labels, tags = self._check_filters(q, labels, tags, False)
        self._apply_filters(labels, tags, False)
        if self.world == 1:
            return self.index._range_resident(q, threshold, device_out)
        n = self.index._range_search(threshold) if hi > lo else 0

        def fill(views):
            ip = views[0]
            if hi == lo:
                ip.zero_()
                return
            # queries mode: this rank's run holds empty segments outside its slice [lo, hi)
            self.index._range_fetch_into([ip[lo:hi + 1]] + views[1:])
            ip[:lo] = 0
            ip[hi + 1:] = n
            self._rows.to_global(views[1])

        gathered, pairs = gather_range_packed(self.device, q, n, fill, self.group)
        return _host(merge_range_on_device(self.device, gathered, q, pairs), device_out)

    def _set_resident_text(self, data, offsets: np.ndarray, mode: int) -> None:
        """A batch of host text as the resident batch of a threshold search: ``upload_text_sharded`` in rows mode on
        several GPUs, host featurisation and ``set_resident`` otherwise."""
        if self.world > 1 and self.mode == "rows":
            self.upload_text_sharded(data, offsets, mode)
            return
        qfb = self.vocab.featurize_packed(data, offsets, mode, grow=False)
        try:
            self.set_resident(qfb)
        finally:
            qfb.close()

    def range_packed(self, data, offsets: np.ndarray, threshold: float, mode: int = 0, labels: Optional[np.ndarray] = None,
                     device_out: bool = False, tags=None):
        """``range_resident`` of a batch of host text (packed as for ``topk_packed``).  Rows mode on several GPUs
        prepares the batch with ``upload_text_sharded``."""
        offsets = np.ascontiguousarray(offsets, dtype=np.int64)
        if len(offsets) <= 1:
            return self.index._empty_range(device_out)
        self._set_resident_text(data, offsets, mode)
        return self.range_resident(threshold, device_out, labels, tags)

    def selfjoin_range(self, threshold: float, device_out: bool = False, block: int = 262144):
        """All-pairs threshold search over the whole sharded corpus: for every global row every OTHER row scoring
        >= ``threshold``, as ``GfkbIndex.selfjoin_range`` (query i = row i).  The queries are the corpus text that
        ``build_packed`` keeps a reference to, in blocks of ``block`` rows; each block's merged result is appended."""
        if self._corpus is None:
            raise ValueError("selfjoin_range: build_packed first")
        if self.world == 1:
            return self.index.selfjoin_range(threshold, device_out=device_out)
        data, off, mode = self._corpus

        def part(b0: int, b1: int):
            self._set_resident_text(data, off[b0:b1 + 1], mode)
            lo, hi = self._qslice
            if hi > lo:
                self.index.set_exclusions(self._rows.index_ids(np.arange(b0 + lo, b0 + hi, dtype=np.int64)))
            res = self.range_resident(threshold, device_out=True)
            if self._deleted is not None:   # a deleted row's query has no pairs, as in GfkbIndex.selfjoin_range
                res = _drop_queries(res, self._deleted[b0:b1])
            return res

        return _join_blocks(self.n_global, block, part, device_out, lambda: self.index._empty_range(device_out))


class ShardedDense:
    """Row-sharded dense-embedding GFKB (BASELINE configs[2] read as 768-d bf16 cosine, and configs[3] all-pairs).

    Rank r holds rows [n*r/W, n*(r+1)/W) as a ``DenseIndex`` (K2); queries are replicated; one all-gather of the
    per-shard partial top-k + K5 merge per batch -- the same exchange as the TF-IDF path, no df all-reduce needed.
    ``allpairs_topk`` makes every stored row a query: the row shards are all-gathered ONCE over NCCL (N x dim bf16,
    1.5 GB at 1M x 768) so that each rank can score all N rows against its shard, each query excluding itself.
    The label and tag filters need no exchange of their own: every rank keeps its rows' labels and tag sets and filters
    its own rows; the self-joins pass the global rows' labels and sets as the query filters of each block.
    """

    def __init__(self, dim: int, device: int, rank: int = 0, world: int = 1, group=None):
        from .denseindex import DenseIndex

        self.dim, self.device, self.rank, self.world, self.group = dim, device, rank, world, group
        self._mk = lambda base: DenseIndex(dim, device=device, row_base=base)
        self.index = None
        self.n_global = 0
        self._local = None
        self._labels: Optional[np.ndarray] = None                  # set_row_labels, by global row
        self._tags: Optional[Tuple[np.ndarray, np.ndarray]] = None  # set_row_tags, CSR by global row

    def build(self, rows_local, n_global: int) -> None:
        """``rows_local``: this rank's rows, a torch bfloat16 CUDA tensor [n_local, dim] (shard_bounds order)."""
        lo, hi = shard_bounds(n_global, self.world, self.rank)
        assert rows_local.shape[0] == hi - lo
        self.n_global = n_global
        self.index = self._mk(lo)
        self.index.add_device(rows_local.contiguous())
        self.index.finalize()
        self._local = rows_local
        self._labels = self._tags = None

    def set_row_labels(self, global_labels: Optional[np.ndarray]) -> None:
        """One label >= 0 per GLOBAL row (e.g. a failure-type id), for ``labels=`` / ``same_label=``: this rank keeps
        its rows' labels.  ``None`` clears.  Call it with the same labels on every rank."""
        if global_labels is None:
            self.index.set_row_labels(None)
            self._labels = None
            return
        lab = np.ascontiguousarray(global_labels, dtype=np.int32).reshape(-1)
        if len(lab) != self.n_global:
            raise ValueError(f"set_row_labels: {len(lab)} labels for a corpus of {self.n_global} rows")
        lo, hi = shard_bounds(self.n_global, self.world, self.rank)
        self.index.set_row_labels(lab[lo:hi])
        self._labels = lab.copy()

    def set_row_tags(self, global_sets) -> None:
        """A tag set per GLOBAL row (a list of lists or an ``(indptr, tags)`` pair, as ``DenseIndex.set_row_tags``),
        for ``tags=`` / ``same_tags=``: this rank keeps its rows' sets.  ``None`` clears.  Call it with the same sets on
        every rank."""
        if global_sets is None:
            self.index.set_row_tags(None)
            self._tags = None
            return
        ip, t = tag_csr(global_sets, self.n_global, "set_row_tags")
        lo, hi = shard_bounds(self.n_global, self.world, self.rank)
        self.index.set_row_tags(csr_rows(ip, t, np.arange(lo, hi)))
        self._tags = (ip.copy(), t.copy())

    def _block_filters(self, b0: int, b1: int, same_label: bool, same_tags: bool):
        """The query filters of self-join block [b0, b1) of global rows: the rows' own labels and tag sets."""
        from .denseindex import selfjoin_tags

        labels = tags = None
        if same_label:
            if self._labels is None:
                raise RuntimeError("same_label: the sharded index has no row labels (set_row_labels)")
            labels = self._labels[b0:b1]
        if same_tags:
            if self._tags is None:
                raise RuntimeError("same_tags: the sharded index has no row tags (set_row_tags)")
            tags = selfjoin_tags(*self._tags, b0, b1)
        return labels, tags

    def topk(self, queries, k: int = 16, exclude_base: int = -1, distinct: bool = False,
             labels: Optional[np.ndarray] = None, tags=None):
        """queries: torch bfloat16 CUDA [Q, dim], identical on every rank -> ([Q,k] float32, [Q,k] int64) on device.
        ``labels`` / ``tags``: per query the row label and the tag set its results' rows must carry / meet, as in
        ``DenseIndex.topk`` (identical on every rank)."""
        no_distinct(distinct, "ShardedDense.topk")
        s, r = self.index.topk_device(queries.contiguous(), k, exclude_base, labels=labels, tags=tags)
        if self.world == 1:
            return s, r
        gs, gr = gather_topk(s, r, self.group)
        return merge_on_device(self.device, gs, gr)

    def gather_rows(self):
        """All-gather the row shards into the full [N, dim] matrix (equal-sized slots, padding dropped)."""
        import torch
        import torch.distributed as dist

        if self.world == 1:
            return self._local
        per = (self.n_global + self.world - 1) // self.world + 1
        slot = torch.zeros((per, self.dim), dtype=self._local.dtype, device=self._local.device)
        slot[: self._local.shape[0]] = self._local
        full = torch.empty((self.world * per, self.dim), dtype=self._local.dtype, device=self._local.device)
        dist.all_gather_into_tensor(full, slot, group=self.group)
        parts = []
        for w in range(self.world):
            lo, hi = shard_bounds(self.n_global, self.world, w)
            parts.append(full[w * per: w * per + (hi - lo)])
        return torch.cat(parts).contiguous()

    def allpairs_topk(self, k: int = 32, block: int = 262144, same_label: bool = False, same_tags: bool = False):
        """Every row's k nearest OTHER rows over the whole sharded GFKB: ([N,k] float32, [N,k] int64), on every rank.
        ``same_label`` / ``same_tags``: row i's list holds only rows with its label / sharing one of its tags (a row
        with more than 16 tags raises ValueError), as ``DenseIndex.selfjoin_topk``."""
        import torch

        allrows = self.gather_rows()
        out_s, out_r = [], []
        for b0 in range(0, self.n_global, block):
            b1 = min(self.n_global, b0 + block)
            labels, tags = self._block_filters(b0, b1, same_label, same_tags)
            s, r = self.topk(allrows[b0:b1], k, exclude_base=b0, labels=labels, tags=tags)
            out_s.append(s)
            out_r.append(r)
        return torch.cat(out_s), torch.cat(out_r)

    def range(self, queries, threshold: float, device_out: bool = True, exclude_base: int = -1,
              labels: Optional[np.ndarray] = None, tags=None):
        """Threshold search over the whole sharded GFKB: queries torch bfloat16 CUDA [Q, dim], identical on every rank
        -> ``(indptr int64[Q+1], rows int64[P], scores float32[P])`` as ``DenseIndex.range_device`` returns them (torch
        tensors on the device, or NumPy arrays without ``device_out``); identical on every rank.  ``exclude_base >= 0``:
        query q never matches GLOBAL row ``exclude_base + q``.  ``labels`` / ``tags`` as in ``topk``."""
        idx = self.index
        queries = queries.contiguous()
        if self.world == 1:
            return idx.range_device(queries, threshold, exclude_base, device_out, labels=labels, tags=tags)
        n_q = queries.shape[0]
        with idx._lock:
            n = idx._range_search_device(queries, threshold, exclude_base, labels, tags)
            gathered, pairs = gather_range_packed(self.device, n_q, n, idx._range_fetch_into, self.group)
        return _host(merge_range_on_device(self.device, gathered, n_q, pairs), device_out)

    def selfjoin_range(self, threshold: float, block: int = 262144, device_out: bool = True, same_label: bool = False,
                       same_tags: bool = False):
        """Every row's OTHER rows scoring >= ``threshold`` over the whole sharded GFKB (query i = global row i): the row
        shards are all-gathered once (``gather_rows``), then blocks of ``block`` rows are searched as in ``range``.
        ``same_label`` / ``same_tags`` as in ``allpairs_topk``."""
        allrows = self.gather_rows()

        def part(b0: int, b1: int):
            labels, tags = self._block_filters(b0, b1, same_label, same_tags)
            return self.range(allrows[b0:b1], threshold, True, exclude_base=b0, labels=labels, tags=tags)

        return _join_blocks(self.n_global, block, part, device_out, lambda: _host(_devout.empty_range(self.device), device_out))


class ShardedJaccard:
    """Row-sharded token-set Jaccard GFKB (BASELINE configs[4]: 5M sets on 4 GPUs).  No global statistics exist for
    Jaccard (every token weighs 1), so the only exchanges are the all-gather of partial top-k and a max-reduce of the
    exact (|intersection|, |union|) integers, which each rank can only count for the rows it owns."""

    def __init__(self, vocab_size: int, device: int, rank: int = 0, world: int = 1, group=None):
        from .jaccardindex import JaccardIndex

        self.device, self.rank, self.world, self.group = device, rank, world, group
        self.vocab_size = vocab_size
        self._cls = JaccardIndex
        self.index = None
        self.n_global = 0
        self._csr = None   # the whole corpus (build_csr): the queries of selfjoin_range

    def build_csr(self, indptr: np.ndarray, ids: np.ndarray) -> None:
        """``indptr``/``ids``: the WHOLE corpus (every rank passes the same arrays); this rank keeps its row range."""
        n = len(indptr) - 1
        self.n_global = n
        self._csr = (np.ascontiguousarray(indptr, dtype=np.int64), np.ascontiguousarray(ids, dtype=np.uint32))
        lo, hi = shard_bounds(n, self.world, self.rank)
        self.index = self._cls(self.vocab_size, device=self.device, row_base=lo)
        ip = np.ascontiguousarray(indptr[lo:hi + 1], dtype=np.int64)
        self.index.add_csr(ip - ip[0], np.ascontiguousarray(ids[ip[0]:ip[-1]], dtype=np.uint32))
        self.index.finalize()

    def build_local_csr(self, indptr: np.ndarray, ids: np.ndarray, n_global: int) -> None:
        """``indptr``/``ids``: ONLY this rank's rows (global rows [n*r/W, n*(r+1)/W) of an n_global-row corpus)."""
        lo, hi = shard_bounds(n_global, self.world, self.rank)
        assert len(indptr) - 1 == hi - lo
        self.n_global = n_global
        self._csr = None
        self.index = self._cls(self.vocab_size, device=self.device, row_base=lo)
        self.index.add_csr(np.ascontiguousarray(indptr, dtype=np.int64), np.ascontiguousarray(ids, dtype=np.uint32))
        self.index.finalize()

    def topk_csr(self, indptr: np.ndarray, ids: np.ndarray, k: int = 16, distinct: bool = False):
        """(scores float32, rows int64, inter int32, union int32), each [Q,k], identical on every rank."""
        no_distinct(distinct, "ShardedJaccard.topk_csr")
        import torch
        import torch.distributed as dist

        s, r, inter, union = self.index.topk_csr(indptr, ids, k)
        if self.world == 1:
            return s, r, inter, union
        dev = f"cuda:{self.device}"
        gs, gr = gather_topk(torch.from_numpy(s).to(dev), torch.from_numpy(r).to(dev), self.group)
        ms, mr = merge_on_device(self.device, gs, gr)
        rows = mr.cpu().numpy()
        inter, union = self.index.counts_csr(indptr, ids, rows)      # -1 for rows of other shards
        cnt = torch.from_numpy(np.stack([inter, union])).to(dev)
        dist.all_reduce(cnt, op=dist.ReduceOp.MAX, group=self.group)
        cnt = cnt.cpu().numpy()
        return ms.cpu().numpy(), rows, cnt[0], cnt[1]

    def _range_csr(self, indptr: np.ndarray, ids: np.ndarray, threshold: float, exclude: Optional[np.ndarray], device_out: bool):
        idx = self.index
        ip, qids, oov = idx._strip_oov(indptr, ids)
        n_q = len(ip) - 1
        if n_q == 0:
            return idx._empty_range(device_out)
        idx._upload(ip, qids, np.ones(len(qids), dtype=np.uint32), oov, n_q)
        if exclude is not None:   # global rows; the shard maps them to its own rows
            idx.set_exclusions(exclude)
        gathered, pairs = gather_range_packed(self.device, n_q, idx._range_search(threshold),
                                              idx._range_fetch_into, self.group, jaccard=True)
        return _host(merge_range_on_device(self.device, gathered, n_q, pairs, jaccard=True), device_out)

    def range_csr(self, indptr: np.ndarray, ids: np.ndarray, threshold: float, device_out: bool = False):
        """Threshold search over the whole sharded GFKB, as ``JaccardIndex.range_csr``: ``(indptr, rows, scores, inter,
        union)``, identical on every rank.  The exact counts travel with the pairs (each shard counts its own rows)."""
        if self.world == 1:
            return self.index.range_csr(indptr, ids, threshold, device_out)
        return self._range_csr(indptr, ids, threshold, None, device_out)

    def selfjoin_range(self, threshold: float, device_out: bool = False, block: int = 262144):
        """Every row's OTHER rows scoring >= ``threshold`` over the whole sharded GFKB (query i = global row i), as
        ``JaccardIndex.selfjoin_range``; the queries are the corpus ``build_csr`` was given, in blocks of ``block`` rows.
        After ``build_local_csr`` a shard lacks the other shards' rows: ValueError."""
        if self._csr is None:
            raise ValueError("selfjoin_range: needs the whole corpus (build_csr); build_local_csr keeps only this shard's rows")
        if self.world == 1:
            return self.index.selfjoin_range(threshold, device_out=device_out)
        ip, ids = self._csr
        return _join_blocks(self.n_global, block,
                            lambda b0, b1: self._range_csr(ip[b0:b1 + 1] - ip[b0], ids[ip[b0]:ip[b1]], threshold,
                                                           np.arange(b0, b1, dtype=np.int64), True),
                            device_out, lambda: self.index._empty_range(device_out))


class ShardedGfkbStore(GfkbStore):
    """``GfkbStore`` on a row-sharded GFKB: the same upsert, match, warn and purge handlers, with the main segment
    spread over the GPUs of one box.  The record logic (versioning, quarantine, the purge's record rewriting, the match
    post-filters and the warning strings) is inherited unchanged; only the steps that touch the device index differ.

    SPMD, like ``ShardedGfkb``: every rank constructs the store with the same ``path`` and ``tail_limit`` and calls the
    same methods in the same order with the same arguments (and a ``now`` clock that gives every rank the same time, or
    the ranks' copies of a record differ in their timestamps).  Every rank holds all records and the same vocabulary;
    only rank 0 writes ``failures.jsonl`` and its purge backup, the others update their records in memory; the
    constructor and ``load`` end with a barrier, so no rank reads a file rank 0 has already changed.  Results
    are identical on every rank, and a rejected upsert or a bad argument raises the same exception on every rank
    before any collective starts.

    Segments: MAIN is a ``ShardedGfkb`` in rows mode (contiguous ranges of record rows per rank), built from the
    records' texts; TAIL holds the records appended since the last rebuild (at most ``tail_limit``) as a ``GfkbIndex``
    replicated on every rank (row_base = main rows, the store's vocabulary), so an upsert exchanges nothing.  The global
    statistics are the main shards' live df (all-reduced once per build or deletion and cached) plus the tail's,
    N = all records; the main shards and the tail get them through statistics-only finalizes.  Queries: the sharded
    top-k of MAIN, its candidates re-scored in float64 by every shard (K6: -inf for another shard's rows) and combined
    with one MAX all-reduce, the tail's candidates as in ``GfkbStore``, then the same host merge.  The exact fallback
    runs ``kv_exact_topk`` on every shard and on the tail and merges their ``limit`` rows per query (one all-gather):
    no score vector leaves a device.  A purge deletes the main rows and refreshes every statistic in one all-reduce.

    Not supported: the sidecar and the persisted layout, queries mode and text-order shards (ValueError), and
    ``match_above`` (NotImplementedError: the sharded threshold search merges float32 results)."""

    def __init__(self, path=None, device: int = 0, rank: int = 0, world: int = 1, group=None, tail_limit: int = 65536,
                 now=None, sidecar=None, mode: str = "rows", order: str = "index"):
        if sidecar is not None:
            raise ValueError("ShardedGfkbStore: the sidecar and the persisted layout are not supported on a sharded GFKB")
        if mode != "rows":
            raise ValueError("ShardedGfkbStore: only rows mode is supported (queries mode holds the whole index on every rank)")
        if order != "index":
            raise ValueError("ShardedGfkbStore: only index-order shards are supported (not text order)")
        self.rank, self.world, self.group = rank, world, group
        self._read_file = False
        super().__init__(path, device=device, tail_limit=tail_limit, now=now)
        if not self._read_file:
            self._barrier()

    def _barrier(self) -> None:
        """Rank 0 writes the file as soon as it returns from an upsert or a purge, and the ranks run without an exchange
        in between: every rank must have read (or found no) file before rank 0 may change it."""
        if self.world > 1:
            import torch.distributed as dist

            dist.barrier(group=self.group)

    def load(self) -> None:
        super().load()
        self._read_file = True
        self._barrier()

    @property
    def _writes_file(self) -> bool:
        return self.path is not None and self.rank == 0

    def _build_main(self, texts) -> None:
        main = ShardedGfkb(self.device, self.rank, self.world, self.group)
        main.vocab.close()
        main.vocab = self.vocab   # one vocabulary for both segments and every rebuild, as in GfkbStore
        self._main = main
        main.build_packed(*pack_texts(texts))

    def _global_statistics(self, main_rows: Optional[np.ndarray] = None) -> None:
        """The main shards' and the tail's live statistics -> every main shard and the tail, by statistics-only
        finalizes; ``main_rows``: main rows deleted in the same exchange."""
        tail = self._tail
        extra = (tail.local_df(), tail.n_live_rows) if tail is not None else (np.zeros(0, np.int64), 0)
        if main_rows is not None and len(main_rows):   # the deletion's all-reduce carries the refreshed statistics
            df, n = self._main.delete_rows(main_rows, *extra)
        else:                                           # the cached main statistics serve
            df, n = self._main.set_statistics(*extra)
        if tail is not None:
            tail.set_global_df(df.astype(np.uint32), n)
            tail.finalize()

    def _refresh_statistics(self) -> None:
        self._global_statistics()
        self.stats["stat_refreshes" if self._main.index.last_finalize_kind == 2 else "full_rebuilds"] += 1

    def _delete_dev_rows(self, gone: np.ndarray) -> bool:
        if self._n_deleted + len(gone) > max(self.tail_limit, 0):
            return True   # the next _sync compacts the main segment: nothing to delete or exchange now
        main_rows = gone[gone < self._n_main]
        tail = self._tail
        if tail is not None and len(gone) > len(main_rows):
            tail.delete_rows(gone[gone >= self._n_main] - self._n_main)
        self._global_statistics(main_rows)
        self.stats["stat_refreshes"] += 1
        return False

    def _ensure_groups(self) -> None:
        groups = None
        if not self._main._has_groups:
            groups = self._dev_groups(self._n_dev)
            self._main.set_row_groups(groups[:self._n_main])
        tail = self._tail
        if tail is not None and tail.n_rows and not tail.has_row_groups:
            groups = self._dev_groups(self._n_dev) if groups is None else groups
            tail.set_row_groups(groups[self._n_main:self._n_main + tail.n_rows])

    def _segment_candidates(self, ix, fb: FeatureBatch, kk: int, labels: Optional[np.ndarray], distinct: bool, tags):
        if ix is not self._main:
            return super()._segment_candidates(ix, fb, kk, labels, distinct, tags)
        ix.set_resident(fb)
        s, r = ix.topk_resident(kk, labels=labels, distinct=distinct, tags=tags)
        s32, rows = s.cpu().numpy(), r.cpu().numpy()
        f64 = ix.index.rescore(fb, rows)   # -inf for the rows of the other shards
        if self.world > 1:
            import torch
            import torch.distributed as dist

            t = torch.from_numpy(f64).to(f"cuda:{self.device}")
            dist.all_reduce(t, op=dist.ReduceOp.MAX, group=self.group)
            f64 = t.cpu().numpy()
        return s32, rows, f64

    def _above(self, fb: FeatureBatch, threshold: float, labels, tags):
        raise NotImplementedError("ShardedGfkbStore.match_above: the exact threshold search is not built for a "
                                  "sharded GFKB (its range merge is float32)")

    def _exact_top(self, signature_text: str, limit: int, label: int = -1, distinct: bool = False, app: int = -1):
        if distinct:
            self._ensure_groups()
        lab = None if label < 0 else np.array([label], dtype=np.int32)
        tags = None if app < 0 else [[app]]
        fb = self.vocab.featurize([signature_text], grow=False)
        try:
            parts = [self._main.exact_topk(fb, limit, lab, distinct, tags)]
            if self._tail is not None and self._tail.n_rows:
                parts.append(self._tail.exact_topk(fb, limit, lab, distinct, tags))
        finally:
            fb.close()
        groups = self._dev_groups(self._n_dev) if distinct else None
        rows, scores = merge_exact_lists(np.concatenate([p[0] for p in parts], axis=1),
                                         np.concatenate([p[1] for p in parts], axis=1), limit, groups)
        keep = rows[0] >= 0
        return self._to_records(rows[0][keep]).tolist(), scores[0][keep].tolist()
