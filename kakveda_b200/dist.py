"""Row-sharded GFKB over the GPUs of one box (SURVEY.md section 8e).

One process per GPU (``torch.distributed``, NCCL over NVLink/NVSwitch).  Corpus rows are split
contiguously (rank r owns rows [n*r/W, n*(r+1)/W)); every rank sees the same query batch.  The
only exchanges are

* once per append epoch: an all-reduce(sum) of the per-feature document-frequency vector, because
  TF-IDF's idf and row norms use GLOBAL df and N (``allreduce_df``);
* once per query batch: ONE all-gather of the per-shard partial top-k (scores float32, rows int64),
  followed by a local merge ordered by (score desc, row asc) -- identical on every rank
  (``gather_topk`` + ``kv_merge_topk_device``).

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

from . import _capi
from ._capi import no_distinct
from .similarity import FeatureBatch, GfkbIndex, Vocabulary, gather_rows, text_order


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
        self.device, self.rank, self.world, self.group = device, rank, world, group
        self.vocab = Vocabulary()
        self.index: Optional[GfkbIndex] = None
        self.n_global = 0

    def build_packed(self, data, offsets: np.ndarray, mode: int = 0, n_threads: int = 0) -> None:
        import torch

        fb = self.vocab.featurize_packed(data, offsets, mode, grow=True, n_threads=n_threads)
        self.n_global = fb.n
        lo, hi = shard_bounds(fb.n, self.world, self.rank) if self.mode == "rows" else (0, fb.n)
        if self.mode == "rows" and self.order == "text" and self.world > 1:
            sel = shard_rows_by_text(fb, self.world, self.rank, n_threads)
            self.index = GfkbIndex(device=self.device, row_base=0, vocab=self.vocab)
            self.index.add_features(gather_rows(fb, sel, n_threads))
            self.row_map = torch.from_numpy(sel).to(f"cuda:{self.device}")
        else:
            self.index = GfkbIndex(device=self.device, row_base=lo, vocab=self.vocab)
            self.index.add_features(fb, lo, hi)
        fb.close()
        if self.world > 1 and self.mode == "rows":
            df = torch.from_numpy(self.index.local_df().astype(np.int32)).to(f"cuda:{self.device}")
            allreduce_df(df, self.group)
            self.index.set_global_df(df.cpu().numpy().astype(np.uint32), self.n_global)
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

    def upload(self, qfb: FeatureBatch) -> None:
        if self.mode == "queries" and self.world > 1:
            # this rank's slice of the batch: re-pack the CSR rows [lo, hi)
            lo, hi = shard_bounds(qfb.n, self.world, self.rank)
            self._qslice = (lo, hi)
            ip = np.ascontiguousarray(qfb.indptr[lo:hi + 1])
            _capi.check(_capi.load().kv_query_upload(self.index._h, ip.ctypes.data_as(C.POINTER(C.c_int64)),
                                                     qfb.ids.ctypes.data_as(C.POINTER(C.c_uint32)),
                                                     qfb.tf.ctypes.data_as(C.POINTER(C.c_uint32)),
                                                     np.ascontiguousarray(qfb.oov[lo:hi]).ctypes.data_as(C.POINTER(C.c_double)),
                                                     hi - lo))
            return
        self.index.upload_queries(qfb)
        self._exchange_thresholds(qfb.n)

    def topk_resident(self, k: int, distinct: bool = False):
        """Device-only step on the uploaded batch: local scan+merge, all-gather, global merge."""
        no_distinct(distinct, "ShardedGfkb.topk_resident")
        import torch

        q = self._resident_q
        dev = f"cuda:{self.device}"
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
            if self.row_map is not None:
                r.copy_(torch.where(r >= 0, self.row_map[r.clamp(min=0)], r))
            return s, r
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(5)]
        # phase 1: bounds + seed scan on every shard; the shards' seed lists are merged (small all-gather) and the GLOBAL
        # k-th seed score of every query becomes every shard's pruning threshold -- each shard then scans only what a
        # single index would scan of its rows
        self.index.topk_resident_seed(k, s.data_ptr(), r.data_ptr())
        ev[0].record()
        # only the seed SCORES travel (6.4 MB per rank at 100k queries): the global k-th seed score of a query is the k-th
        # largest of the W x k gathered scores (the shards hold disjoint rows)
        import torch.distributed as dist

        gs = torch.empty((self.world, q, k), dtype=torch.float32, device=dev)
        dist.all_gather_into_tensor(gs.view(-1), s.contiguous().view(-1), group=self.group)
        kth = torch.topk(gs.permute(1, 0, 2).reshape(q, self.world * k), k, dim=1).values[:, k - 1].contiguous()
        ev[1].record()
        torch.cuda.current_stream().synchronize()
        self.index.raise_thresholds(kth.data_ptr(), q)
        # phase 2: candidate selection + scan, then the exchange of the partial top-k
        self.index.topk_resident_finish(k, s.data_ptr(), r.data_ptr())
        if self.row_map is not None:  # text-range shard: local row -> global row id (-1 stays -1)
            r.copy_(torch.where(r >= 0, self.row_map[r.clamp(min=0)], r))
        ev[2].record()
        gathered = gather_packed(buf, self.group)          # the all-gather of the partial top-k
        ev[3].record()
        out = merge_packed_on_device(self.device, gathered, q, k)
        ev[4].record()
        # The collective doubles as the barrier between batches for the cross-GPU threshold pushes: no rank may start
        # the next batch's scan (which resets and pushes thresholds) before every rank has finished this one's.
        torch.cuda.current_stream().synchronize()
        self.last_exchange_ms = (ev[2].elapsed_time(ev[3]), ev[3].elapsed_time(ev[4]), ev[0].elapsed_time(ev[1]))
        return out

    def set_resident(self, qfb: FeatureBatch) -> None:
        self.upload(qfb)
        self._resident_q = qfb.n

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
            self._resident_q = n_q
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

    def topk_packed(self, data, offsets: np.ndarray, k: int, mode: int = 0, distinct: bool = False):
        """End-to-end step from host text: featurise, upload, scan, exchange, merge, read back.  ``last_e2e_ms`` keeps
        the wall-clock split of the last call (featurise / upload incl. table kernels / device step / read-back)."""
        no_distinct(distinct, "ShardedGfkb.topk_packed")
        import time

        t0 = time.perf_counter()
        if self.world > 1 and self.mode == "rows" and os.environ.get("KAKVEDA_B200_NO_SLICED_PREP") != "1":
            import torch

            self.upload_text_sharded(data, offsets, mode)
            t2 = time.perf_counter()
            s, r = self.topk_resident(k)
            torch.cuda.current_stream().synchronize()
            t3 = time.perf_counter()
            out = self._read_back(s, r)
            t4 = time.perf_counter()
            self.last_e2e_ms = {"prepare_sharded": 1e3 * (t2 - t0), "device_step": 1e3 * (t3 - t2), "read_back": 1e3 * (t4 - t3),
                                "prepare_split": self.last_prepare_split_ms}
            return out
        qfb = self.vocab.featurize_packed(data, offsets, mode, grow=False)
        try:
            t1 = time.perf_counter()
            self.set_resident(qfb)
            t2 = time.perf_counter()
            s, r = self.topk_resident(k)
            import torch

            torch.cuda.current_stream().synchronize()
            t3 = time.perf_counter()
            out = self._read_back(s, r)
            t4 = time.perf_counter()
            self.last_e2e_ms = {"featurize": 1e3 * (t1 - t0), "upload": 1e3 * (t2 - t1), "device_step": 1e3 * (t3 - t2),
                                "read_back": 1e3 * (t4 - t3),
                                "upload_host_ms": self.index.last_prepare_ms()}  # staging, classification, order, copies+tables
            return out
        finally:
            qfb.close()


class ShardedDense:
    """Row-sharded dense-embedding GFKB (BASELINE configs[2] read as 768-d bf16 cosine, and configs[3] all-pairs).

    Rank r holds rows [n*r/W, n*(r+1)/W) as a ``DenseIndex`` (K2); queries are replicated; one all-gather of the
    per-shard partial top-k + K5 merge per batch -- the same exchange as the TF-IDF path, no df all-reduce needed.
    ``allpairs_topk`` makes every stored row a query: the row shards are all-gathered ONCE over NCCL (N x dim bf16,
    1.5 GB at 1M x 768) so that each rank can score all N rows against its shard, each query excluding itself.
    """

    def __init__(self, dim: int, device: int, rank: int = 0, world: int = 1, group=None):
        from .denseindex import DenseIndex

        self.dim, self.device, self.rank, self.world, self.group = dim, device, rank, world, group
        self._mk = lambda base: DenseIndex(dim, device=device, row_base=base)
        self.index = None
        self.n_global = 0
        self._local = None

    def build(self, rows_local, n_global: int) -> None:
        """``rows_local``: this rank's rows, a torch bfloat16 CUDA tensor [n_local, dim] (shard_bounds order)."""
        lo, hi = shard_bounds(n_global, self.world, self.rank)
        assert rows_local.shape[0] == hi - lo
        self.n_global = n_global
        self.index = self._mk(lo)
        self.index.add_device(rows_local.contiguous())
        self.index.finalize()
        self._local = rows_local

    def topk(self, queries, k: int = 16, exclude_base: int = -1, distinct: bool = False):
        """queries: torch bfloat16 CUDA [Q, dim], identical on every rank -> ([Q,k] float32, [Q,k] int64) on device."""
        no_distinct(distinct, "ShardedDense.topk")
        s, r = self.index.topk_device(queries.contiguous(), k, exclude_base)
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

    def allpairs_topk(self, k: int = 32, block: int = 262144):
        """Every row's k nearest OTHER rows over the whole sharded GFKB: ([N,k] float32, [N,k] int64), on every rank."""
        import torch

        allrows = self.gather_rows()
        out_s, out_r = [], []
        for b0 in range(0, self.n_global, block):
            b1 = min(self.n_global, b0 + block)
            s, r = self.topk(allrows[b0:b1], k, exclude_base=b0)
            out_s.append(s)
            out_r.append(r)
        return torch.cat(out_s), torch.cat(out_r)


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

    def build_csr(self, indptr: np.ndarray, ids: np.ndarray) -> None:
        """``indptr``/``ids``: the WHOLE corpus (every rank passes the same arrays); this rank keeps its row range."""
        n = len(indptr) - 1
        self.n_global = n
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
