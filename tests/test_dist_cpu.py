"""world_size-2 gloo tests (CPU) of the multi-GPU plumbing in kakveda_b200/dist.py: shard bounds,
the df all-reduce and the all-gather of per-shard partial top-k.  The device kernels cannot run
here, so each rank produces its shard's partial top-k with the oracle and the K5 merge is
restated in NumPy (test infrastructure); the assertion is that gather + merge over shards equals
the unsharded oracle top-k, ties included -- i.e. the exchange pattern of SURVEY section 8(e)."""
import os
import socket
import sys
from pathlib import Path

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

REPO = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(REPO))


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _merge_numpy(gs, gr, k):
    """Reference of kv_merge_topk_device: lists ordered by (score desc, row asc), -1 rows unused."""
    w, q, _ = gs.shape
    out_s = np.full((q, k), -np.inf, np.float32)
    out_r = np.full((q, k), -1, np.int64)
    for i in range(q):
        cand = [(-float(gs[l, i, j]), int(gr[l, i, j])) for l in range(w) for j in range(gs.shape[2]) if gr[l, i, j] >= 0]
        cand.sort()
        for j, (ns, r) in enumerate(cand[:k]):
            out_s[i, j], out_r[i, j] = -ns, r
    return out_s, out_r


def _worker(rank, world, port, n, q, k, tmp):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from kakveda_b200 import synth
        from kakveda_b200.dist import allreduce_df, gather_topk, shard_bounds
        from kakveda_b200.similarity import Vocabulary
        from oracle import tfidf_oracle as O

        corpus, queries = synth.corpus(n), synth.queries(q, n)
        lo, hi = shard_bounds(n, world, rank)
        assert shard_bounds(n, world, 0)[0] == 0 and shard_bounds(n, world, world - 1)[1] == n
        # every rank featurises the whole corpus: identical ids without exchanging the vocabulary
        vocab = Vocabulary()
        fb = vocab.featurize(corpus, grow=True, n_threads=1 + rank)  # thread count must not matter
        local_df = np.bincount(fb.ids[fb.indptr[lo]:fb.indptr[hi]], minlength=len(vocab)).astype(np.int32)
        total = allreduce_df(torch.from_numpy(local_df.copy())).numpy()
        want_df = np.bincount(fb.ids, minlength=len(vocab))
        np.testing.assert_array_equal(total, want_df)
        # partial top-k of this shard (oracle scores use the GLOBAL statistics), then the exchange
        full = O.score_matrix_closed_form(queries, corpus)
        idx, val = O.topk_rows(full[:, lo:hi], k)
        ps = torch.from_numpy(val.astype(np.float32))
        pr = torch.from_numpy((idx + lo).astype(np.int64))
        gs, gr = gather_topk(ps, pr)
        assert tuple(gs.shape) == (world, q, k) and tuple(gr.shape) == (world, q, k)
        ms, mr = _merge_numpy(gs.numpy(), gr.numpy(), k)
        widx, wval = O.topk_rows(full.astype(np.float32).astype(np.float64), k)
        np.testing.assert_array_equal(mr, widx)
        np.testing.assert_allclose(ms, wval, rtol=1e-7)
        Path(tmp, f"ok{rank}").write_text("ok")
    finally:
        dist.destroy_process_group()


def test_sharded_exchange_world2(built_lib, tmp_path):
    world, port = 2, _free_port()
    mp.spawn(_worker, args=(world, port, 1501, 24, 16, str(tmp_path)), nprocs=world, join=True)
    assert all((tmp_path / f"ok{r}").exists() for r in range(world))


def test_shard_bounds_cover_rows():
    from kakveda_b200.dist import shard_bounds

    for n in (0, 1, 7, 1000, 10_000_001):
        for w in (1, 2, 3, 8):
            spans = [shard_bounds(n, w, r) for r in range(w)]
            assert spans[0][0] == 0 and spans[-1][1] == n
            assert all(a[1] == b[0] for a, b in zip(spans, spans[1:]))
            assert max(b - a for a, b in spans) - min(b - a for a, b in spans) <= 1


def _gather_worker(rank, world, port, n, d, tmp):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from kakveda_b200.dist import ShardedDense, shard_bounds

        full = torch.arange(n * d, dtype=torch.float32).reshape(n, d).to(torch.bfloat16)
        lo, hi = shard_bounds(n, world, rank)
        sh = ShardedDense(d, device=0, rank=rank, world=world)   # no index is created: only the exchange is exercised
        sh._local, sh.n_global = full[lo:hi].contiguous(), n
        got = sh.gather_rows()                                    # the all-gather behind all-pairs (configs[3])
        assert got.shape == full.shape and torch.equal(got.view(torch.int16), full.view(torch.int16))
        # all-pairs exclusion bookkeeping: query block b0.. excludes GLOBAL rows b0.., whatever the shard
        assert [shard_bounds(n, world, w) for w in range(world)][rank] == (lo, hi)
        Path(tmp, f"g{rank}").write_text("ok")
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("world,n", [(2, 1001), (3, 10)])
def test_allpairs_row_gather(built_lib, tmp_path, world, n):
    mp.spawn(_gather_worker, args=(world, _free_port(), n, 64, str(tmp_path)), nprocs=world, join=True)
    assert all((tmp_path / f"g{r}").exists() for r in range(world))


def test_text_range_sharding_host_side(built_lib):
    """order="text" (dist.ShardedGfkb): the global text order and the row gather are host-only and must agree with a
    plain Python sort / slicing; the shards partition the rows, each in ascending global order."""
    from kakveda_b200 import synth
    from kakveda_b200.dist import shard_rows_by_text
    from kakveda_b200.similarity import Vocabulary, gather_rows, text_order

    v = Vocabulary()
    fb = v.featurize(synth.corpus(60001) + ["", "zz", synth.corpus(5)[3]], grow=True)
    for threads in (1, 8):
        perm = text_order(fb, threads)
        seqs = [tuple(fb.ids[fb.indptr[i]:fb.indptr[i + 1]].tolist()) for i in range(fb.n)]
        assert perm.tolist() == sorted(range(fb.n), key=lambda i: (seqs[i], i))
    parts = [shard_rows_by_text(fb, 4, r, 4) for r in range(4)]
    allr = np.concatenate(parts)
    assert len(allr) == fb.n == len(set(allr.tolist())) and all(np.all(np.diff(p) > 0) for p in parts)
    sub = gather_rows(fb, parts[2], 4)
    assert sub.n == len(parts[2])
    for j in range(0, sub.n, 997):
        i = parts[2][j]
        np.testing.assert_array_equal(sub.ids[sub.indptr[j]:sub.indptr[j + 1]], fb.ids[fb.indptr[i]:fb.indptr[i + 1]])
        np.testing.assert_array_equal(sub.tf[sub.indptr[j]:sub.indptr[j + 1]], fb.tf[fb.indptr[i]:fb.indptr[i + 1]])
    assert gather_rows(fb, np.zeros(0, dtype=np.int64)).n == 0
    with pytest.raises(ValueError):
        gather_rows(fb, np.array([fb.n], dtype=np.int64))


@pytest.mark.parametrize("layout", ["index", "text", "all"])
def test_shard_rows_conversions(built_lib, layout):
    """The rows a ``ShardedGfkb`` shard holds (dist._ShardRows) for each layout: an index range (rows mode), a range of
    the text order (``row_map``) and every row (queries mode).  ``part``, ``local``, ``index_ids`` and ``to_global``
    agree with each other and with ``shard_bounds`` / ``shard_rows_by_text``; the index-range and text-order shards
    partition the rows."""
    from kakveda_b200 import synth
    from kakveda_b200.dist import _ShardRows, shard_bounds, shard_rows_by_text
    from kakveda_b200.similarity import Vocabulary

    v = Vocabulary()
    for n_texts, world in ((997, 3), (40, 8)):
        texts = synth.corpus(n_texts)
        fb = v.featurize(texts + texts[:5], grow=True)   # duplicates: equal texts, consecutive in the text order
        n = fb.n
        rng = np.random.default_rng(n)
        per_row = rng.integers(0, 1000, n)
        probe = np.unique(rng.integers(0, n, n // 2))     # ascending global rows
        owner = np.full(n, -1)
        for rank in range(world):
            lo, hi = shard_bounds(n, world, rank)
            if layout == "index":
                rows, held, base = _ShardRows(lo, hi), np.arange(lo, hi), lo
            elif layout == "text":
                held = shard_rows_by_text(fb, world, rank)
                rows, base = _ShardRows(lo, hi, held, "cpu"), 0
            else:
                rows, held, base = _ShardRows(0, n), np.arange(n), 0
            assert len(held) == hi - lo or layout == "all"
            np.testing.assert_array_equal(rows.part(np.arange(n)), held)
            np.testing.assert_array_equal(rows.part(per_row), per_row[held])
            mine = probe[np.isin(probe, held)]
            pos = np.searchsorted(held, mine)
            np.testing.assert_array_equal(rows.local(probe), pos)
            ids = rows.index_ids(probe)
            if layout == "text":                          # local positions, -1 for rows of other shards
                np.testing.assert_array_equal(ids, np.where(np.isin(probe, held), np.searchsorted(held, probe), -1))
            else:                                         # the index takes global rows (row_base = lo)
                np.testing.assert_array_equal(ids, probe)
            # what the index reports for its rows (local row + row_base), and -1, back to global rows
            reported = np.concatenate([pos + base, [-1]]).astype(np.int64)
            want = np.concatenate([mine, [-1]])
            np.testing.assert_array_equal(rows.to_global(reported.copy()), want)
            t = torch.from_numpy(reported.copy())
            assert rows.to_global(t) is t and t.tolist() == want.tolist()
            np.testing.assert_array_equal(rows.to_global(ids[ids >= 0]), probe[ids >= 0])
            if layout != "all":
                assert (owner[held] == -1).all()
                owner[held] = rank
        assert layout == "all" or (owner >= 0).all()
        fb.close()


def test_query_slice_exchange_layout_is_aligned_and_disjoint():
    """Byte layout of one rank's slot in the query-slice all-gather (ShardedGfkb.upload_text_sharded): sections in
    order, 16-byte aligned, large enough for the capacities, nothing overlapping."""
    from kakveda_b200.dist import ShardedGfkb

    for nq, nnz in ((0, 0), (1, 0), (7, 33), (12500, 560001), (100000, 4500003)):
        o_ip, o_oov, o_ord, o_fl, o_ids, o_tf, slot = ShardedGfkb._slice_layout(nq, nnz)
        sections = [(16, 0), (o_ip, 8 * (nq + 1)), (o_oov, 8 * nq), (o_ord, 4 * nq), (o_fl, nq), (o_ids, 4 * nnz), (o_tf, 4 * nnz)]
        end = 0
        for i, (off, size) in enumerate(sections):
            if i:
                assert off % 16 == 0 and off >= end, (nq, nnz, i)
                end = off + size
            else:
                end = off
        assert slot >= end and slot % 16 == 0

