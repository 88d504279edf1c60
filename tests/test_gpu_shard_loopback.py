"""The row-sharded GFKB of ``kakveda_b200/dist.py`` on ONE GPU: W ranks as threads, each with its own real
``ShardedGfkb`` / ``ShardedDense`` / ``ShardedJaccard`` on device 0, talking through a thread-backed stand-in for the
``torch.distributed`` calls dist.py makes.  dist.py runs unmodified: the df all-reduce, the seed-threshold exchange
(seed scan -> global k-th of W x k seed scores -> raised thresholds -> finish scan), the packed all-gather and the K5
merge, the sliced query preparation of ``upload_text_sharded``, the ``row_map`` of text-order shards, queries mode and
the counts max-reduce of Jaccard.  ctypes releases the GIL, so the shards' kernels overlap as they do on W GPUs.

Every TF-IDF result is checked against the single index over the whole corpus (rows and float32 scores equal) and
against ``oracle/torch_oracle.SparseOracle`` over the whole corpus CSR (df and N of the whole corpus: the reference's
refit), with ``check_topk_device`` of test_gpu_scale_oracle.py; rows with identical text must carry identical float32
bits whichever shard returned them.  The peer threshold pushes are exercised through ``kv_debug_thresholds_link``,
which points a shard's peer array at the other shards' threshold arrays in this process.

Measured on an NVIDIA H100 80GB HBM3 (700 W limit): see DESIGN.md section 2 for the file's wall time.
"""
import ctypes as C
import math
import threading
import time

import numpy as np
import pytest

torch = pytest.importorskip("torch")
import torch.distributed as tdist  # noqa: E402

from oracle import tfidf_oracle as O  # noqa: E402
from oracle import torch_oracle as T  # noqa: E402
from test_gpu_scale_oracle import RTOL32, check_topk_device, corpus_common_unigrams, dense_rtol, q_arrays, q_block  # noqa: E402

gpu = pytest.mark.gpu
TIMEOUT = 180.0     # seconds a rank may wait in one collective before the run counts as failed
QBLOCK = 64


# ---------------------------------------------------------------------------------------------------------------------
# Thread-backed process group
# ---------------------------------------------------------------------------------------------------------------------

class _Shared:
    def __init__(self, world, timeout):
        self.world = world
        self.barrier = threading.Barrier(world, timeout=timeout)
        self.slots = [None] * world


class LoopbackGroup:
    """One rank's handle on a group of ``world`` threads.  Collectives are synchronous: every rank deposits a snapshot
    of its input and a signature of the call, waits for the others, checks that all of them made the same call, reads
    every snapshot and waits again before a slot may be reused.  CUDA inputs are synchronised before they are read."""

    def __init__(self, shared, rank):
        self.shared, self.rank, self.world = shared, rank, shared.world

    def _wait(self):
        self.shared.barrier.wait()

    def exchange(self, sig, payload):
        sh = self.shared
        sh.slots[self.rank] = (sig, payload)
        self._wait()
        sigs = [s[0] for s in sh.slots]
        if any(s != sig for s in sigs):
            raise RuntimeError(f"rank {self.rank}: ranks made different collective calls: {sigs}")
        got = [s[1] for s in sh.slots]
        return got

    def done(self):
        self._wait()


def _snapshot(t):
    if t.is_cuda:
        torch.cuda.synchronize(t.device)
    return t.detach().clone()


def _group(group):
    if not isinstance(group, LoopbackGroup):
        raise RuntimeError("the loopback collectives need the rank's LoopbackGroup (dist.py passes group=)")
    return group


def _lb_get_world_size(group=None):
    return _group(group).world


def _lb_barrier(group=None, **kw):
    g = _group(group)
    g.exchange(("barrier",), None)
    g.done()


def _lb_all_reduce(tensor, op=tdist.ReduceOp.SUM, group=None, async_op=False):
    g = _group(group)
    name = {tdist.ReduceOp.SUM: "sum", tdist.ReduceOp.MAX: "max"}.get(op)
    if name is None:
        raise RuntimeError(f"loopback all_reduce: unsupported op {op}")
    parts = g.exchange(("all_reduce", name, tuple(tensor.shape), tensor.dtype), _snapshot(tensor))
    acc = parts[0].to(tensor.device).clone()
    for p in parts[1:]:
        p = p.to(tensor.device)
        acc = acc + p if name == "sum" else torch.maximum(acc, p)
    g.done()
    tensor.copy_(acc)
    if tensor.is_cuda:
        torch.cuda.synchronize(tensor.device)


def _lb_all_gather_into_tensor(output, input, group=None, async_op=False):
    g = _group(group)
    parts = g.exchange(("all_gather_into_tensor", tuple(input.shape), input.dtype), _snapshot(input))
    if output.numel() != g.world * input.numel():
        raise RuntimeError(f"loopback all_gather_into_tensor: output of {output.numel()} elements for {g.world} x {input.numel()}")
    flat = torch.cat([p.reshape(-1).to(output.device) for p in parts])   # rank-major
    g.done()
    output.view(-1).copy_(flat)
    if output.is_cuda:
        torch.cuda.synchronize(output.device)


def _lb_all_gather_object(object_list, obj, group=None):
    g = _group(group)
    parts = g.exchange(("all_gather_object", len(object_list)), obj)
    g.done()
    object_list[:] = parts


@pytest.fixture
def loopback(monkeypatch):
    """Installs the loopback collectives in ``torch.distributed`` for the test."""
    monkeypatch.setattr(tdist, "is_available", lambda: True)
    monkeypatch.setattr(tdist, "is_initialized", lambda: True)
    monkeypatch.setattr(tdist, "get_world_size", _lb_get_world_size)
    monkeypatch.setattr(tdist, "barrier", _lb_barrier)
    monkeypatch.setattr(tdist, "all_reduce", _lb_all_reduce)
    monkeypatch.setattr(tdist, "all_gather_into_tensor", _lb_all_gather_into_tensor)
    monkeypatch.setattr(tdist, "all_gather_object", _lb_all_gather_object)
    return run_ranks


def run_ranks(world, fn, timeout=TIMEOUT):
    """Runs ``fn(rank, group)`` on ``world`` threads and returns their results by rank.  A rank that raises breaks the
    barrier, so the others fail at their next collective instead of waiting; every thread is joined; a barrier
    timeout or a thread still alive afterwards fails the test."""
    shared = _Shared(world, timeout)
    out, err = [None] * world, [None] * world

    def body(r):
        try:
            if torch.cuda.is_available():
                torch.cuda.set_device(0)
            out[r] = fn(r, LoopbackGroup(shared, r))
        except BaseException as e:   # noqa: BLE001 -- reported below
            err[r] = e
            shared.barrier.abort()

    threads = [threading.Thread(target=body, args=(r,), name=f"rank{r}", daemon=True) for r in range(world)]
    for t in threads:
        t.start()
    deadline = time.monotonic() + 2 * timeout + 60
    for t in threads:
        t.join(max(0.0, deadline - time.monotonic()))
    alive = [t.name for t in threads if t.is_alive()]
    if alive:
        shared.barrier.abort()
        for t in threads:
            t.join(60)
        raise AssertionError(f"ranks {alive} did not finish")
    first = [e for e in err if e is not None and not isinstance(e, threading.BrokenBarrierError)]
    if first:
        raise first[0]
    if any(e is not None for e in err):
        raise AssertionError(f"a collective timed out after {timeout} s: {err}")
    return out


# ---------------------------------------------------------------------------------------------------------------------
# The stand-in itself (CPU)
# ---------------------------------------------------------------------------------------------------------------------

def test_loopback_gather_is_rank_major(loopback):
    def fn(r, g):
        out = torch.empty(6, dtype=torch.int64)
        tdist.all_gather_into_tensor(out, torch.full((2,), r, dtype=torch.int64), group=g)
        objs = [None] * 3
        tdist.all_gather_object(objs, f"r{r}", group=g)
        return out.tolist(), objs, tdist.get_world_size(g)

    for got in loopback(3, fn, timeout=30):
        assert got == ([0, 0, 1, 1, 2, 2], ["r0", "r1", "r2"], 3)


def test_loopback_reduce_in_place(loopback):
    def fn(r, g):
        s = torch.tensor([r + 1, 10 * r], dtype=torch.int32)
        m = torch.tensor([r, -r], dtype=torch.float32)
        keep = s
        tdist.all_reduce(s, op=tdist.ReduceOp.SUM, group=g)
        tdist.all_reduce(m, op=tdist.ReduceOp.MAX, group=g)
        tdist.barrier(group=g)
        return keep is s, s.tolist(), m.tolist()

    for got in loopback(4, fn, timeout=30):
        assert got == (True, [10, 60], [3.0, 0.0])


def test_loopback_mismatched_calls_fail_fast(loopback):
    def fn(r, g):
        t = torch.zeros(2)
        if r == 0:
            tdist.all_reduce(t, group=g)
        else:
            tdist.all_gather_into_tensor(torch.empty(4), t, group=g)

    t0 = time.monotonic()
    with pytest.raises(RuntimeError, match="different collective calls"):
        loopback(2, fn, timeout=30)
    assert time.monotonic() - t0 < 10


def test_loopback_missing_call_is_a_failure_not_a_hang(loopback):
    def fn(r, g):
        if r == 0:
            tdist.barrier(group=g)

    t0 = time.monotonic()
    with pytest.raises(AssertionError, match="timed out"):
        loopback(2, fn, timeout=1.0)
    assert time.monotonic() - t0 < 30


# ---------------------------------------------------------------------------------------------------------------------
# TF-IDF corpus and checks
# ---------------------------------------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def lib(built_lib):
    from kakveda_b200 import _capi

    assert _capi.load().kv_device_count() > 0, "GPU tests need a CUDA device"
    return _capi.load()


class Corpus:
    """Texts, the single index over all of them and the float64 oracle over their CSR."""

    def __init__(self, texts, queries):
        from kakveda_b200 import GfkbIndex
        from kakveda_b200.similarity import pack_texts

        self.texts, self.queries = list(texts), list(queries)
        self.n = len(self.texts)
        self.data, self.off, self.mode = pack_texts(self.texts)
        self.qdata, self.qoff, self.qmode = pack_texts(self.queries)
        self.one = GfkbIndex()
        fb = self.one.vocab.featurize_packed(self.data, self.off, self.mode, grow=True)
        rows = (np.array(fb.indptr, np.int64), np.array(fb.ids, np.int64), np.array(fb.tf, np.float64))
        self.one.add_features(fb)
        fb.close()
        self.one.finalize()
        self.V = len(self.one.vocab)
        self.qfb = self.one.vocab.featurize(self.queries, grow=False)
        self.qa = q_arrays(self.qfb)
        self.single = {}
        _, self.text_id = np.unique(np.array(self.texts, dtype=object).astype(str), return_inverse=True)
        self.orc = T.SparseOracle(*rows, self.V, device="cuda")
        self.blocks = []
        for lo in range(0, len(self.queries), QBLOCK):
            hi = min(len(self.queries), lo + QBLOCK)
            self.blocks.append((lo, hi, self.orc.tfidf_scores(*q_block(self.qa, lo, hi))))

    def single_topk(self, k):
        if k not in self.single:
            self.single[k] = self.one.topk_features(self.qfb, k)
        return self.single[k]

    def check(self, name, s, r, k, exact=True):
        """``s`` / ``r``: a sharded top-k of every query.  Equal to the single index, inside the oracle's contract, and
        rows of identical text carry identical bits."""
        s, r = np.asarray(s), np.asarray(r)
        assert s.shape == (len(self.queries), k) and r.shape == s.shape, (name, s.shape, r.shape)
        for lo, hi, o in self.blocks:
            try:
                check_topk_device(s[lo:hi], r[lo:hi], o, k, RTOL32, first=lo)
            except AssertionError as e:
                raise AssertionError(f"{name}, k = {k}: {e}") from None
        tid = np.where(r >= 0, self.text_id[np.clip(r, 0, self.n - 1)], -1)
        for q in range(len(self.queries)):
            for t in np.unique(tid[q][tid[q] >= 0]):
                sc = s[q][tid[q] == t]
                assert np.all(sc.view(np.uint32) == sc[0].view(np.uint32)), \
                    f"{name}, k = {k}, query {q}: rows {r[q][tid[q] == t].tolist()} of one text scored {sc.tolist()}"
        if exact:
            s1, r1 = self.single_topk(k)
            bad = np.flatnonzero((r != r1).any(1) | (s.view(np.uint32) != s1.view(np.uint32)).any(1))
            assert len(bad) == 0, (f"{name}, k = {k}: {len(bad)} queries differ from the single index, first {bad[0]}: "
                                   f"sharded {r[bad[0]].tolist()} {s[bad[0]].tolist()} single {r1[bad[0]].tolist()} {s1[bad[0]].tolist()}")


def synth_texts(n, nq):
    """The synthetic corpus with stored duplicates across the corpus, a token held by 3 rows, and a batch of bench
    queries plus: null, all-OOV, universal-only, 65-feature, fewer-than-k-matches and stored-row queries."""
    from kakveda_b200 import synth

    texts = synth.corpus(n)
    rng = np.random.default_rng(5)
    for src in rng.choice(n, 40, replace=False):          # 40 texts stored 6 times each, anywhere in the corpus
        for dst in rng.choice(n, 5, replace=False):
            texts[dst] = texts[src]
    for i, dst in enumerate((7, n // 2 + 3, n - 2)):
        texts[dst] = texts[dst] + " qxrarezz"
    sample = [texts[i] for i in range(0, n, max(1, n // 2000))]
    univ = corpus_common_unigrams(sample)
    rare = sorted({w for t in sample[:400] for w in O.features(t) if " " not in w} - set(univ))
    queries = synth.queries(nq, n)
    queries += ["", "qqzzunseen xxyyq", " ".join(reversed(univ)), " ".join(rare[:65]), "qxrarezz",
                "qxrarezz qqzzunseen", texts[0], texts[n // 3], texts[n - 1]]
    return texts, queries


@pytest.fixture(scope="module")
def synth_corpus(lib):
    texts, queries = synth_texts(200_000, 502)
    c = Corpus(texts, queries)
    flags = np.empty(len(queries), np.uint8)
    c.one.upload_queries(c.qfb)
    qperm, fl = c.one.query_order(c.qfb.n)
    flags[qperm] = fl
    assert flags[-9] == 1 and flags[-8] == 1 and flags[-7] == 0 and flags[-6] == 2, flags[-9:]
    return c


def build_sharded(world, order, mode, c):
    """fn(rank, group) building rank's ShardedGfkb over corpus ``c``."""
    from kakveda_b200.dist import ShardedGfkb

    def build(r, g):
        sh = ShardedGfkb(device=0, rank=r, world=world, group=g, mode=mode, order=order)
        sh.build_packed(c.data, c.off, c.mode, n_threads=4)
        return sh
    return build


def _close(shards):
    for sh in shards:
        if sh is not None and getattr(sh, "index", None) is not None:
            sh.index.close()


def _copy(x):
    return np.array(x, copy=True)


# ---------------------------------------------------------------------------------------------------------------------
# Rows mode and queries mode
# ---------------------------------------------------------------------------------------------------------------------

ROW_CASES = [("index", 1), ("index", 2), ("index", 3), ("index", 8), ("text", 2), ("text", 3), ("text", 8)]


@gpu
@pytest.mark.parametrize("order,world", ROW_CASES, ids=[f"{o}-W{w}" for o, w in ROW_CASES])
def test_rows_mode_equals_single_index_and_oracle(synth_corpus, loopback, monkeypatch, order, world):
    """Rows mode through ``topk_packed`` (sliced preparation when W > 1), through ``set_resident`` + ``topk_resident``
    and once with ``KAKVEDA_B200_NO_SLICED_PREP=1``, at k = 1, 16, 32."""
    c = synth_corpus
    build = build_sharded(world, order, "rows", c)

    def fn(r, g):
        sh = build(r, g)
        try:
            res = {}
            for k in (1, 16, 32):
                s, rr = sh.topk_packed(c.qdata, c.qoff, k, c.qmode)
                res["topk_packed", k] = (_copy(s), _copy(rr))
                qfb = sh.vocab.featurize(c.queries, grow=False)
                try:
                    sh.set_resident(qfb)
                    s, rr = sh.topk_resident(k)
                    res["resident", k] = (s.cpu().numpy(), rr.cpu().numpy())
                finally:
                    qfb.close()
            univ = sh.index.layout()["universal_features"]
            return res, univ, getattr(sh, "n_threshold_peers", None)
        finally:
            _close([sh])

    out = loopback(world, fn)
    for r in range(1, world):
        for key, (s, rr) in out[0][0].items():
            np.testing.assert_array_equal(out[r][0][key][1], rr, err_msg=f"rank {r} {key}")
            np.testing.assert_array_equal(out[r][0][key][0], s, err_msg=f"rank {r} {key}")
    for (name, k), (s, rr) in out[0][0].items():
        c.check(f"{order} W={world} {name}", s, rr, k)
    print(f"\nuniversal features per shard {[o[1] for o in out]}, n_threshold_peers {[o[2] for o in out]}")

    if world > 1:
        monkeypatch.setenv("KAKVEDA_B200_NO_SLICED_PREP", "1")

        def fn2(r, g):
            sh = build(r, g)
            try:
                s, rr = sh.topk_packed(c.qdata, c.qoff, 16, c.qmode)
                return _copy(s), _copy(rr), "prepare_sharded" in sh.last_e2e_ms
            finally:
                _close([sh])

        out2 = loopback(world, fn2)
        assert not any(o[2] for o in out2)
        c.check(f"{order} W={world} unsliced", out2[0][0], out2[0][1], 16)


@gpu
@pytest.mark.parametrize("world", [2, 3])
def test_queries_mode_equals_single_index_and_oracle(synth_corpus, loopback, world):
    """Queries mode: every rank holds the whole index and answers its slice of a batch of 511 queries (not a multiple
    of W); the gathered results are the single index's."""
    c = synth_corpus
    assert len(c.queries) % world != 0
    build = build_sharded(world, "index", "queries", c)

    def fn(r, g):
        sh = build(r, g)
        try:
            res = {}
            for k in (1, 16, 32):
                s, rr = sh.topk_packed(c.qdata, c.qoff, k, c.qmode)
                res[k] = (_copy(s), _copy(rr))
            return res
        finally:
            _close([sh])

    out = loopback(world, fn)
    for k, (s, rr) in out[0].items():
        for r in range(1, world):
            np.testing.assert_array_equal(out[r][k][1], rr)
        c.check(f"queries W={world}", s, rr, k)


# ---------------------------------------------------------------------------------------------------------------------
# Ties across shard boundaries, with a word that only some shards fold
# ---------------------------------------------------------------------------------------------------------------------

def crafted_texts(n, world, order):
    """index order: 24 copies of one text straddle every shard boundary (12 on each side); every row of shard 0 holds
    the word ``zqmarker``, every other row of the other shards does.  text order: one text fills 70 % of the rows, so
    it covers the middle text range completely and straddles its boundaries; it holds ``zqmarker``, as does every other
    remaining row.  The queries are the copied texts with one extra word each and with words dropped."""
    from kakveda_b200 import synth

    base = synth.corpus(n, seed=synth.CORPUS_SEED + 17)
    rng = np.random.default_rng(world * 7 + (order == "text"))
    words = sorted({w for t in base[:300] for w in t.split()})
    texts = list(base)
    groups = []
    if order == "index":
        for r in range(world):
            lo, hi = n * r // world, n * (r + 1) // world
            for i in range(lo, hi):
                if r == 0 or i % 2 == 0:
                    texts[i] = texts[i] + " zqmarker"
        for r in range(1, world):
            b = n * r // world
            t = base[b] + " zqmarker"
            for i in range(b - 12, b + 12):
                texts[i] = t
            groups.append(t)
    else:
        t = base[1] + " zqmarker"
        for i in rng.choice(n, int(0.7 * n), replace=False):
            texts[i] = t
        for i in range(0, n, 2):
            if texts[i] != t:
                texts[i] = texts[i] + " zqmarker"
        groups.append(t)
    queries = []
    for t in groups:
        toks = t.split()
        queries.append(t)
        for _ in range(150):
            extra = " ".join(rng.choice(words, rng.integers(1, 4)))
            keep = [w for w in toks if rng.random() > 0.15] or toks[:1]
            queries.append(" ".join(keep + ["zqmarker"]) + " " + extra)
    queries += synth.signatures(synth.QUERY_SEED, 0, 40)
    return texts, queries


CRAFTED = [("index", 2), ("index", 3), ("text", 3)]


@gpu
@pytest.mark.parametrize("order,world", CRAFTED, ids=[f"{o}-W{w}" for o, w in CRAFTED])
def test_crafted_ties_across_shards(lib, loopback, order, world):
    """Duplicate groups straddle the shard boundaries with the k-th position inside the group, and the shards fold
    different sets of universal features (asserted through ``layout()``).  A row's float32 score must not depend on
    which features its shard folds: the merge then orders the copies by row id and no threshold from one shard drops
    an identical row of another."""
    c = Corpus(*crafted_texts(6000, world, order), )
    build = build_sharded(world, order, "rows", c)

    def fn(r, g):
        sh = build(r, g)
        try:
            res = {}
            for k in (1, 5, 16, 32):
                s, rr = sh.topk_packed(c.qdata, c.qoff, k, c.qmode)
                res[k] = (_copy(s), _copy(rr))
            return res, sh.index.layout()["universal_features"]
        finally:
            _close([sh])

    out = loopback(world, fn)
    univ = [o[1] for o in out]
    one = c.one.layout()["universal_features"]
    assert len(set(univ)) > 1 and max(univ) > one, f"the shards fold the same features: {univ}, single index {one}"
    for k, (s, rr) in out[0][0].items():
        c.check(f"crafted {order} W={world}", s, rr, k)


# ---------------------------------------------------------------------------------------------------------------------
# Peer threshold pushes
# ---------------------------------------------------------------------------------------------------------------------

def _link(lib, shards, rank, cap):
    peers = [sh.index._h for i, sh in enumerate(shards) if i != rank]
    arr = (C.c_void_p * max(1, len(peers)))(*[p.value for p in peers])
    from kakveda_b200 import _capi

    _capi.check(lib.kv_debug_thresholds_link(shards[rank].index._h, arr, len(peers), cap))


PEER_CASES = [("index", 3), ("index", 8), ("text", 8)]


@gpu
@pytest.mark.parametrize("order,world", PEER_CASES, ids=[f"{o}-W{w}" for o, w in PEER_CASES])
def test_peer_threshold_pushes(synth_corpus, lib, loopback, monkeypatch, order, world):
    """Rows mode with every shard pushing its thresholds into the other shards' arrays while the scans run: with the
    finish phases concurrent and one after another (later shards start from every earlier shard's pushes), for two
    different batches of the same size back to back.  The results are exact; the pushes never add scanned pairs."""
    from kakveda_b200 import _capi

    c = synth_corpus
    monkeypatch.setenv("KAKVEDA_B200_NO_PEER_THR", "1")   # dist.py's IPC exchange stays out; the links stand in for it
    build = build_sharded(world, order, "rows", c)
    half = len(c.queries) // 2
    batches = [c.queries[:half], c.queries[half:2 * half]]
    k = 16
    shards = [None] * world
    turn = threading.Condition()
    state = {"next": 0}

    def serial_finish(r, ix):
        inner = ix.topk_resident_finish

        def finish(*a):
            with turn:
                assert turn.wait_for(lambda: state["next"] == r, timeout=TIMEOUT), f"rank {r}: no turn to finish"
            try:
                inner(*a)
            finally:
                with turn:
                    state["next"] += 1
                    turn.notify_all()
        return finish

    def fn(r, g):
        sh = shards[r] = build(r, g)
        buf = C.create_string_buffer(64)
        _capi.check(lib.kv_index_thresholds_export(sh.index._h, len(c.queries), buf))
        tdist.barrier(group=g)
        res, pairs = {}, {}
        for linked in (False, True):
            _link(lib, shards, r, len(c.queries)) if linked else _capi.check(lib.kv_debug_thresholds_link(sh.index._h, None, 0, 0))
            for serial in ((False, True) if linked else (False,)):
                for b, qs in enumerate(batches):
                    qfb = sh.vocab.featurize(qs, grow=False)
                    try:
                        sh.set_resident(qfb)
                        if serial:
                            with turn:
                                if r == 0:
                                    state["next"] = 0
                            tdist.barrier(group=g)
                            sh.index.topk_resident_finish = serial_finish(r, sh.index)
                        try:
                            s, rr = sh.topk_resident(k)
                        finally:
                            sh.index.__dict__.pop("topk_resident_finish", None)
                        res[linked, serial, b] = (s.cpu().numpy(), rr.cpu().numpy())
                        pairs[linked, serial, b] = sh.index.layout()["pairs_scored"]
                    finally:
                        qfb.close()
        tdist.barrier(group=g)
        _capi.check(lib.kv_debug_thresholds_link(sh.index._h, None, 0, 0))
        tdist.barrier(group=g)
        return res, pairs

    try:
        out = loopback(world, fn)
    finally:
        _close(shards)
    for key in out[0][0]:
        linked, serial, b = key
        s, rr = out[0][0][key]
        lo = b * half
        full_s, full_r = np.full((len(c.queries), k), -np.inf, np.float32), np.full((len(c.queries), k), -1, np.int64)
        full_s[lo:lo + half], full_r[lo:lo + half] = s, rr
        for blo, bhi, o in c.blocks:
            if blo >= lo and bhi <= lo + half:
                check_topk_device(full_s[blo:bhi], full_r[blo:bhi], o, k, RTOL32, first=blo)
        s1, r1 = c.single_topk(k)
        np.testing.assert_array_equal(rr, r1[lo:lo + half], err_msg=f"linked {linked} serial {serial} batch {b}")
        np.testing.assert_array_equal(s, s1[lo:lo + half], err_msg=f"linked {linked} serial {serial} batch {b}")
    total = {key: sum(o[1][key] for o in out) for key in out[0][1]}
    print(f"\npairs scored over {world} shards: {total}")
    for b in (0, 1):
        assert total[True, False, b] <= total[False, False, b], total
        assert total[True, True, b] <= total[False, False, b], total


# ---------------------------------------------------------------------------------------------------------------------
# Fewer rows than shards
# ---------------------------------------------------------------------------------------------------------------------

@gpu
def test_empty_shards(lib, loopback):
    """5 rows on 8 shards, for the TF-IDF, dense and Jaccard classes: each either answers exactly or raises a clear
    error from dist.py."""
    from kakveda_b200 import synth
    from kakveda_b200.dist import ShardedDense, ShardedGfkb, ShardedJaccard

    world, k = 8, 4
    texts = synth.corpus(5)
    c = Corpus(texts, [texts[0], texts[3] + " extra", ""])

    def tfidf(r, g):
        sh = ShardedGfkb(device=0, rank=r, world=world, group=g)
        try:
            sh.build_packed(c.data, c.off, c.mode)
            s, rr = sh.topk_packed(c.qdata, c.qoff, k, c.qmode)
            return _copy(s), _copy(rr)
        finally:
            _close([sh])

    try:
        s, rr = loopback(world, tfidf)[0]
    except ValueError as e:
        assert "shard" in str(e), e
    else:
        c.check("5 rows on 8 shards", s, rr, k)

    rng = np.random.default_rng(3)
    dim = 64
    emb = torch.tensor(rng.standard_normal((5, dim)), dtype=torch.bfloat16, device="cuda")
    qe = torch.cat([emb[:2], torch.tensor(rng.standard_normal((3, dim)), dtype=torch.bfloat16, device="cuda")])

    def dense(r, g):
        from kakveda_b200.dist import shard_bounds

        lo, hi = shard_bounds(5, world, r)
        sh = ShardedDense(dim, device=0, rank=r, world=world, group=g)
        sh.build(emb[lo:hi].contiguous(), 5)
        s, rr = sh.topk(qe, k)
        return s.cpu().numpy(), rr.cpu().numpy()

    try:
        s, rr = loopback(world, dense)[0]
    except ValueError as e:
        assert "shard" in str(e), e
    else:
        check_topk_device(s, rr, T.dense_cosine(qe, emb), k, dense_rtol(dim), 1e-6)

    ip = np.array([0, 2, 5, 6, 8, 10], np.int64)
    ids = np.array([1, 2, 1, 3, 4, 5, 2, 3, 6, 7], np.int64)
    qip, qid = np.array([0, 2, 3], np.int64), np.array([1, 2, 7], np.int64)

    def jacc(r, g):
        sh = ShardedJaccard(16, device=0, rank=r, world=world, group=g)
        sh.build_csr(ip, ids)
        return sh.topk_csr(qip, qid.astype(np.uint32), k)

    try:
        s, rr, I, U = loopback(world, jacc)[0]
    except ValueError as e:
        assert "shard" in str(e), e
    else:
        _check_jaccard(ip, ids, qip, qid, 16, s, rr, I, U, k)


# ---------------------------------------------------------------------------------------------------------------------
# Dense and Jaccard
# ---------------------------------------------------------------------------------------------------------------------

def _ties_bit_identical(s, r, key):
    """Rows with the same ``key`` inside one query's result carry identical float32 bits."""
    for q in range(s.shape[0]):
        kq = np.where(r[q] >= 0, key[np.clip(r[q], 0, len(key) - 1)], -1)
        for t in np.unique(kq[kq >= 0]):
            sc = s[q][kq == t]
            assert np.all(sc.view(np.uint32) == sc[0].view(np.uint32)), (q, r[q][kq == t].tolist(), sc.tolist())


@gpu
@pytest.mark.parametrize("world", [2, 3, 8])
def test_sharded_dense(lib, loopback, world):
    """``topk`` and ``allpairs_topk`` of ``ShardedDense`` against the float64 cosine of the bf16 rows, with 20-row runs
    of one embedding straddling every shard boundary; identical rows tie bit for bit."""
    from kakveda_b200.dist import ShardedDense, shard_bounds

    n, dim, nq, k = 4000, 256, 300, 32
    g = torch.Generator(device="cpu").manual_seed(world)
    emb = torch.randn((n, dim), generator=g)
    key = np.arange(n)
    for r in range(1, world):
        b = shard_bounds(n, world, r)[0]
        emb[b - 10:b + 10] = emb[b - 10]
        key[b - 10:b + 10] = b - 10
    emb = emb.to(torch.bfloat16).cuda()
    qs = torch.cat([emb[[shard_bounds(n, world, r)[0] for r in range(1, world)]],
                    torch.randn((nq, dim), generator=g).to(torch.bfloat16).cuda()])

    def fn(r, grp):
        lo, hi = shard_bounds(n, world, r)
        sh = ShardedDense(dim, device=0, rank=r, world=world, group=grp)
        sh.build(emb[lo:hi].contiguous(), n)
        s, rr = sh.topk(qs, k)
        a_s, a_r = sh.allpairs_topk(k, block=1500)
        return s.cpu().numpy(), rr.cpu().numpy(), a_s.cpu().numpy(), a_r.cpu().numpy()

    out = loopback(world, fn)
    s, rr, a_s, a_r = out[0]
    for o in out[1:]:
        np.testing.assert_array_equal(o[1], rr)
        np.testing.assert_array_equal(o[3], a_r)
    rtol = dense_rtol(dim)
    check_topk_device(s, rr, T.dense_cosine(qs, emb), k, rtol, 1e-6)
    _ties_bit_identical(s, rr, key)
    for lo in range(0, n, 1000):
        o = T.dense_cosine(emb[lo:lo + 1000], emb)
        o[torch.arange(o.shape[0]), torch.arange(lo, lo + o.shape[0])] = -math.inf   # a row is not its own neighbour
        check_topk_device(a_s[lo:lo + 1000], a_r[lo:lo + 1000], o, k, rtol, 1e-6, first=lo)
    _ties_bit_identical(a_s, a_r, key)


def _check_jaccard(ip, ids, qip, qid, V, s, rr, I, U, k):
    orc = T.SparseOracle(ip, ids, np.ones(len(ids)), V, device="cuda")
    OI, OU = orc.jaccard_counts(qip, qid)
    ratio = torch.where(OU > 0, OI / OU.clamp(min=1), torch.zeros_like(OI))
    rt = torch.as_tensor(np.clip(rr, 0, len(ip) - 2), device="cuda")
    ok = torch.as_tensor(rr >= 0, device="cuda")
    assert torch.equal(torch.where(ok, torch.as_tensor(I, device="cuda").double(), 0), torch.where(ok, OI.gather(1, rt), 0))
    assert torch.equal(torch.where(ok, torch.as_tensor(U, device="cuda").double(), 0), torch.where(ok, OU.gather(1, rt), 0))
    exact = np.where(rr >= 0, I / np.maximum(U, 1), -np.inf)
    check_topk_device(exact, rr, ratio, k, 0.0)
    check_topk_device(s, rr, ratio, k, 1e-6, 1e-7)


@gpu
@pytest.mark.parametrize("world", [2, 3, 8])
def test_sharded_jaccard(lib, loopback, world):
    """``topk_csr`` of ``ShardedJaccard``: exact counts and the oracle's stable order, with copies of one set straddling
    every boundary and a query whose tokens only rows of shard 0 hold (the other shards' -1 counts go through the MAX
    reduce)."""
    from kakveda_b200.dist import ShardedJaccard, shard_bounds

    n, nq, V, k = 20000, 400, 5000, 16
    rng = np.random.default_rng(world)
    sets = [np.unique(rng.zipf(1.3, 20) % (V - 10)) for _ in range(n)]
    for r in range(1, world):
        b = shard_bounds(n, world, r)[0]
        for i in range(b - 20, b + 20):
            sets[i] = sets[b - 20]
    only0 = [V - 3, V - 2]
    for i in range(0, shard_bounds(n, world, 0)[1], 97):
        sets[i] = np.unique(np.r_[sets[i], only0])
    queries = [sets[shard_bounds(n, world, r)[0]] for r in range(1, world)] + [np.array(only0)]
    queries += [np.unique(rng.zipf(1.3, 12) % (V - 10)) for _ in range(nq)]
    ip = np.r_[0, np.cumsum([len(x) for x in sets])].astype(np.int64)
    ids = np.concatenate(sets).astype(np.int64)
    qip = np.r_[0, np.cumsum([len(x) for x in queries])].astype(np.int64)
    qid = np.concatenate(queries).astype(np.int64)

    def fn(r, g):
        sh = ShardedJaccard(V, device=0, rank=r, world=world, group=g)
        sh.build_csr(ip, ids)
        return sh.topk_csr(qip, qid.astype(np.uint32), k)

    out = loopback(world, fn)
    s, rr, I, U = out[0]
    for o in out[1:]:
        for a, b in zip(o, out[0]):
            np.testing.assert_array_equal(a, b)
    assert (rr[world - 1] >= 0).sum() > 0 and np.all(rr[world - 1][rr[world - 1] >= 0] < shard_bounds(n, world, 0)[1])
    _check_jaccard(ip, ids, qip, qid, V, s, rr, I, U, k)
    key = np.unique(np.array([",".join(map(str, x)) for x in sets]), return_inverse=True)[1]
    _ties_bit_identical(s, rr, key)


# ---------------------------------------------------------------------------------------------------------------------
# K5 directly
# ---------------------------------------------------------------------------------------------------------------------

def merge_numpy(gs, gr, k):
    """(score desc, row asc) merge of W sorted lists, rows -1 unused: [W,Q,k] -> [Q,k]."""
    w, q, _ = gs.shape
    out_s = np.full((q, k), -np.inf, np.float32)
    out_r = np.full((q, k), -1, np.int64)
    for i in range(q):
        cand = sorted((-float(gs[l, i, j]), int(gr[l, i, j])) for l in range(w) for j in range(gs.shape[2]) if gr[l, i, j] >= 0)
        for j, (ns, r) in enumerate(cand[:k]):
            out_s[i, j], out_r[i, j] = -ns, r
    return out_s, out_r


@gpu
@pytest.mark.parametrize("k", [1, 7, 16, 32])
def test_k5_merge_against_numpy(lib, k):
    """``merge_packed_on_device`` (packed strides of ``packed_layout``) and ``merge_on_device`` (contiguous lists)
    against a NumPy merge, for W = 1..8 lists of disjoint rows with heavy cross-list ties and (-inf, -1) padding."""
    from kakveda_b200.dist import merge_on_device, merge_packed_on_device, packed_layout, packed_views

    rng = np.random.default_rng(k)
    q = 67
    for w in range(1, 9):
        gs = np.full((w, q, k), -np.inf, np.float32)
        gr = np.full((w, q, k), -1, np.int64)
        levels = np.array([1.0, 0.75, 0.5, 0.5000001, 0.25, 0.0], np.float32)
        for i in range(q):
            rows = rng.permutation(50 * w * k + 10)[: w * k]
            for l in range(w):
                m = int(rng.integers(0, k + 1)) if i % 3 == 0 else k       # some lists hold fewer than k rows
                sc = levels[rng.integers(0, len(levels), m)]
                rw = rows[l * k:l * k + m]
                o = np.lexsort((rw, -sc))
                gs[l, i, :m], gr[l, i, :m] = sc[o], rw[o]
        es, er = merge_numpy(gs, gr, k)
        dev = "cuda"
        off_r, total = packed_layout(q, k)
        packed = torch.zeros((w, total), dtype=torch.uint8, device=dev)
        for l in range(w):
            s_v, r_v = packed_views(packed[l], q, k)
            s_v.copy_(torch.from_numpy(gs[l]))
            r_v.copy_(torch.from_numpy(gr[l]))
        ps, pr = merge_packed_on_device(0, packed, q, k)
        cs, cr = merge_on_device(0, torch.from_numpy(gs).to(dev), torch.from_numpy(gr).to(dev))
        torch.cuda.synchronize()
        for name, (s, r) in {"packed": (ps, pr), "contiguous": (cs, cr)}.items():
            np.testing.assert_array_equal(r.cpu().numpy(), er, err_msg=f"{name} W={w} k={k}")
            np.testing.assert_array_equal(s.cpu().numpy(), es, err_msg=f"{name} W={w} k={k}")
