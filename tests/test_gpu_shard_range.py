"""Row-sharded threshold search (dist.py) on ONE GPU, through the loopback collectives of test_gpu_shard_loopback.py.

* ``kv_merge_range_device_on`` (``merge_range_on_device``) against a NumPy merge: W = 1..8 crafted runs with empty
  runs, empty queries, every pair in one run, equal scores interleaved by row across runs, with and without the
  Jaccard counts; a million records; every invalid input it must refuse.
* ``ShardedGfkb.range_packed`` in rows mode (index and text order) and queries mode: identical on every rank, equal
  to ``GfkbIndex.range`` over the whole corpus bit for bit for the regular queries (irregular queries take K1a per
  shard, whose float32 may differ at a rounding boundary), and every query inside the float64 oracle's contract
  (``check_range_device``).  Crafted duplicates across shard boundaries, 5 rows on 8 shards, batches without pairs.
* ``set_row_labels`` + ``labels=``; ``selfjoin_range`` of the three sharded classes; ``detect_patterns(k=None)``.
* ``ShardedJaccard``: exact counts (``check_jaccard_range_device``); ``ShardedDense``: ``check_range_device`` with
  ``dense_rtol`` and identical rows tie bit for bit.
"""
import math

import numpy as np
import pytest

torch = pytest.importorskip("torch")

from oracle import torch_oracle as T  # noqa: E402
from test_gpu_scale_oracle import RTOL32, check_jaccard_range_device, check_range_device, dense_rtol  # noqa: E402
from test_gpu_shard_loopback import (Corpus, _close, build_sharded, crafted_texts, lib, loopback,  # noqa: E402,F401
                                     run_ranks, synth_corpus, synth_texts)

gpu = pytest.mark.gpu
THRESHOLDS = (0.3, 0.6, 0.9, 1.0)


# ---------------------------------------------------------------------------------------------------------------------
# The merge against NumPy
# ---------------------------------------------------------------------------------------------------------------------

def _pack_runs(runs, n_q, jaccard):
    """runs: per rank (indptr, rows, scores[, inter, union]) NumPy -> ([W, slot] uint8 CUDA buffer, pairs)."""
    from kakveda_b200.dist import range_layout, range_views

    pairs = np.array([len(r[1]) for r in runs], np.int64)
    p_max = int(pairs.max()) if len(pairs) else 0
    _, slot = range_layout(n_q, p_max, jaccard)
    buf = torch.zeros((len(runs), slot), dtype=torch.uint8, device="cuda")
    for w, run in enumerate(runs):
        for v, a in zip(range_views(buf[w], n_q, int(pairs[w]), p_max, jaccard), run):
            v.copy_(torch.from_numpy(np.ascontiguousarray(a)))
    return buf, pairs


def _merge_numpy(runs, n_q):
    ip = np.zeros(n_q + 1, np.int64)
    cols = [[] for _ in runs[0][1:]]
    for q in range(n_q):
        seg = [tuple(a[r[0][q]:r[0][q + 1]] for a in r[1:]) for r in runs]
        rows = np.concatenate([s[0] for s in seg])
        sc = np.concatenate([s[1] for s in seg])
        o = np.lexsort((rows, -sc.astype(np.float64)))
        for j in range(len(cols)):
            cols[j].append(np.concatenate([s[j] for s in seg])[o])
        ip[q + 1] = ip[q] + len(o)
    return (ip,) + tuple(np.concatenate(c) if c else np.zeros(0) for c in cols)


def _crafted_runs(rng, w, n_q, jaccard, max_per_q=12, all_in=None):
    levels = np.array([1.0, 0.75, 0.5, 0.5000001, 0.3, 0.25], np.float32)
    per = [[[] for _ in range(n_q)] for _ in range(w)]
    for q in range(n_q):
        m = 0 if q % 7 == 3 else int(rng.integers(0, max_per_q * w + 1))
        rows = rng.permutation(40 * w * max_per_q + 10)[:m]
        owner = np.full(m, all_in) if all_in is not None else rng.integers(0, w, m)
        if w > 2 and all_in is None:
            owner[owner == 1] = 0                                  # run 1 stays empty
        sc = levels[rng.integers(0, len(levels), m)]
        for r, s, o in zip(rows, sc, owner):
            per[o][q].append((s, r))
    runs = []
    for l in range(w):
        ip, rr, ss = [0], [], []
        for q in range(n_q):
            seg = sorted(per[l][q], key=lambda t: (-float(t[0]), int(t[1])))
            rr += [int(t[1]) for t in seg]
            ss += [t[0] for t in seg]
            ip.append(len(rr))
        run = [np.array(ip, np.int64), np.array(rr, np.int64), np.array(ss, np.float32)]
        if jaccard:
            run += [(np.array(rr, np.int64) * 3 % 1000).astype(np.int32), (np.array(rr, np.int64) * 7 % 1000 + 1).astype(np.int32)]
        runs.append(run)
    return runs


def _merge_and_compare(runs, n_q, jaccard, name):
    from kakveda_b200.dist import merge_range_on_device

    buf, pairs = _pack_runs(runs, n_q, jaccard)
    got = merge_range_on_device(0, buf, n_q, pairs, jaccard)
    want = _merge_numpy(runs, n_q)
    assert len(got) == len(want)
    for j, (g, e) in enumerate(zip(got, want)):
        g = g.cpu().numpy()
        assert g.dtype == np.asarray(runs[0][j]).dtype or j == 0, (name, j, g.dtype)
        np.testing.assert_array_equal(g, e.astype(g.dtype), err_msg=f"{name}: array {j}")


@gpu
@pytest.mark.parametrize("jaccard", [False, True], ids=["tfidf", "jaccard"])
def test_merge_against_numpy(lib, jaccard):
    rng = np.random.default_rng(11 + jaccard)
    n_q = 53
    for w in range(1, 9):
        _merge_and_compare(_crafted_runs(rng, w, n_q, jaccard), n_q, jaccard, f"W={w}")
        _merge_and_compare(_crafted_runs(rng, w, n_q, jaccard, all_in=w - 1), n_q, jaccard, f"W={w} all in the last run")
        _merge_and_compare(_crafted_runs(rng, w, n_q, jaccard, max_per_q=0), n_q, jaccard, f"W={w} no pairs")
    # no queries at all
    _merge_and_compare([[np.zeros(1, np.int64), np.zeros(0, np.int64), np.zeros(0, np.float32)]
                        + ([np.zeros(0, np.int32)] * 2 if jaccard else [])] * 3, 0, jaccard, "no queries")


@gpu
def test_merge_equal_scores_interleaved(lib):
    """Every pair of a query at one score, rows dealt round-robin to the runs: the merge interleaves them by row."""
    w, n_q, m = 5, 4, 97
    runs = []
    for l in range(w):
        rows = [np.arange(l, m, w, dtype=np.int64) + 1000 * q for q in range(n_q)]
        ip = np.r_[0, np.cumsum([len(r) for r in rows])].astype(np.int64)
        rr = np.concatenate(rows)
        runs.append([ip, rr, np.full(len(rr), 0.625, np.float32), rr.astype(np.int32) % 5, rr.astype(np.int32) % 5 + 8])
    _merge_and_compare(runs, n_q, True, "interleaved jaccard")
    _merge_and_compare([r[:3] for r in runs], n_q, False, "interleaved")


@gpu
def test_merge_million_records(lib):
    """About a million records over 4 runs and 3,000 queries: the grid-stride path of both kernels."""
    from kakveda_b200.dist import merge_range_on_device

    rng = np.random.default_rng(5)
    w, n_q = 4, 3000
    cnt = rng.integers(0, 160, (w, n_q))
    runs = []
    for l in range(w):
        c = cnt[l]
        ip = np.r_[0, np.cumsum(c)].astype(np.int64)
        q = np.repeat(np.arange(n_q), c)
        sc = (rng.integers(0, 64, len(q)) / 64.0).astype(np.float32)  # coarse scores: many ties across runs
        rows = rng.integers(0, 1 << 40, len(q)) * w + l                # disjoint rows per run
        o = np.lexsort((rows, -sc.astype(np.float64), q))
        runs.append([ip, rows[o], sc[o]])
    total = int(cnt.sum())
    assert total > 900_000
    buf, pairs = _pack_runs(runs, n_q, False)
    ip, rows, sc = (t.cpu().numpy() for t in merge_range_on_device(0, buf, n_q, pairs))
    np.testing.assert_array_equal(ip, np.r_[0, np.cumsum(cnt.sum(0))])
    q = np.repeat(np.arange(n_q), np.diff(ip))
    all_q = np.concatenate([np.repeat(np.arange(n_q), np.diff(r[0])) for r in runs])
    all_r, all_s = np.concatenate([r[1] for r in runs]), np.concatenate([r[2] for r in runs])
    o = np.lexsort((all_r, -all_s.astype(np.float64), all_q))
    np.testing.assert_array_equal(rows, all_r[o])
    np.testing.assert_array_equal(sc, all_s[o])
    np.testing.assert_array_equal(q, all_q[o])


@gpu
def test_merge_rejects_invalid_runs(lib):
    """A decreasing indptr, a count that does not match the announced pairs, a segment out of order and one (score,
    row) key in two runs are each ValueError."""
    from kakveda_b200.dist import merge_range_on_device, range_layout

    rng = np.random.default_rng(2)
    n_q = 9
    base = _crafted_runs(rng, 3, n_q, False, max_per_q=6)
    base[1] = _crafted_runs(rng, 1, n_q, False, max_per_q=6)[0]
    base[1][1] = base[1][1] + 10 ** 9                                        # disjoint from run 0
    assert all(len(r[1]) > 4 for r in base[:2])

    def bad(edit, what):
        runs = [[a.copy() for a in r] for r in base]
        pairs_override = edit(runs)
        buf, pairs = _pack_runs(runs, n_q, False)
        if pairs_override is not None:
            ip = buf[0, : 8 * (n_q + 1)].view(torch.int64)
            ip[n_q] = pairs_override
        with pytest.raises(ValueError, match=what):
            merge_range_on_device(0, buf, n_q, pairs)

    def decreasing(runs):
        ip = runs[0][0]
        q = int(np.flatnonzero(np.diff(ip) > 1)[0])
        ip[q + 1] = ip[q + 2] + 1 if q + 2 <= n_q else ip[q] - 1
    bad(decreasing, "indptr")
    bad(lambda runs: int(len(runs[0][1])) - 1, "indptr")                      # indptr[n_q] != announced count

    def unordered(runs):
        ip, rows, sc = runs[1][0], runs[1][1], runs[1][2]
        q = int(np.flatnonzero(np.diff(ip) > 1)[0])
        a = ip[q]
        rows[[a, a + 1]] = rows[[a + 1, a]]
        sc[[a, a + 1]] = sc[[a + 1, a]]
    bad(unordered, "not ordered")

    def duplicate(runs):
        ip0, ip1 = runs[0][0], runs[1][0]
        q = int(np.flatnonzero((np.diff(ip0) > 0) & (np.diff(ip1) > 0))[0])
        runs[1][1][ip1[q]] = runs[0][1][ip0[q]]
        runs[1][2][ip1[q]] = runs[0][2][ip0[q]]
        seg = slice(ip1[q], ip1[q + 1])
        o = np.lexsort((runs[1][1][seg], -runs[1][2][seg].astype(np.float64)))
        runs[1][1][seg], runs[1][2][seg] = runs[1][1][seg][o], runs[1][2][seg][o]
    bad(duplicate, "two runs")
    assert range_layout(n_q, 0)[1] % 16 == 0


# ---------------------------------------------------------------------------------------------------------------------
# ShardedGfkb
# ---------------------------------------------------------------------------------------------------------------------

def _flags(c):
    if not hasattr(c, "flags"):
        c.one.upload_queries(c.qfb)
        qperm, fl = c.one.query_order(c.qfb.n)
        c.flags = np.empty(c.qfb.n, np.uint8)
        c.flags[qperm] = fl
    return c.flags


def _np(res):
    return tuple(t.cpu().numpy() if torch.is_tensor(t) else np.array(t, copy=True) for t in res)


def _check_range(c, name, res, thr, single, exact=True, oracle_blocks=None):
    """res: a sharded (indptr, rows, scores) of every query of ``c``; single: the single index's."""
    ip, rows, sc = res[:3]
    assert len(ip) == len(c.queries) + 1 and ip[0] == 0 and ip[-1] == len(rows) == len(sc), name
    for lo, hi, o in (oracle_blocks or c.blocks):
        a, b = int(ip[lo]), int(ip[hi])
        try:
            check_range_device(ip[lo:hi + 1], rows[a:b], sc[a:b], o, thr, RTOL32, first=lo)
        except AssertionError as e:
            raise AssertionError(f"{name}, threshold {thr}: {e}") from None
    # rows of identical text carry identical float32 bits, whichever shard returned them
    q = np.repeat(np.arange(len(c.queries)), np.diff(ip))
    bad = _tie_breaks(q.astype(np.int64) * (c.n + 1) + c.text_id[rows], sc)
    assert len(bad) == 0, (name, thr, "rows of one text scored differently", int(q[bad[0]]), int(rows[bad[0]]))
    if exact:
        regular = _flags(c) != 2
        sip, srow, ssc = single[:3]
        for qq in np.flatnonzero(regular):
            a, b, e, f = ip[qq], ip[qq + 1], sip[qq], sip[qq + 1]
            if not (np.array_equal(rows[a:b], srow[e:f]) and np.array_equal(sc[a:b].view(np.uint32), ssc[e:f].view(np.uint32))):
                raise AssertionError(f"{name}, threshold {thr}, query {qq}: sharded {rows[a:b][:8].tolist()} "
                                     f"{sc[a:b][:8].tolist()} single {srow[e:f][:8].tolist()} {ssc[e:f][:8].tolist()}")


def _single_range(c, thr, labels=None):
    key = ("range", thr, None if labels is None else labels.tobytes())
    if key not in c.single:
        c.single[key] = _np(c.one.range_features(c.qfb, thr, labels=labels))
    return c.single[key]


def _run_range(c, world, order, mode, thresholds=THRESHOLDS):
    build = build_sharded(world, order, mode, c)

    def fn(r, g):
        sh = build(r, g)
        try:
            out = {}
            for thr in thresholds:
                for dev in (False, True):
                    out[thr, dev] = _np(sh.range_packed(c.qdata, c.qoff, thr, c.qmode, device_out=dev))
                    if dev:
                        assert out[thr, dev][0].dtype == np.int64
            return out
        finally:
            _close([sh])

    out = loopback_run(world, fn)
    for r in range(1, world):
        for key, res in out[0].items():
            for a, b in zip(out[r][key], res):
                np.testing.assert_array_equal(a, b, err_msg=f"rank {r} {key}")
    for (thr, dev), res in out[0].items():
        _check_range(c, f"{mode} {order} W={world} device_out={dev}", res, thr, _single_range(c, thr))
    return out[0]


def loopback_run(world, fn):
    return run_ranks(world, fn)


ROW_CASES = [("index", 1), ("index", 2), ("index", 3), ("index", 8), ("text", 2), ("text", 3), ("text", 8)]


@gpu
@pytest.mark.parametrize("order,world", ROW_CASES, ids=[f"{o}-W{w}" for o, w in ROW_CASES])
def test_rows_mode_range_equals_single_index_and_oracle(synth_corpus, loopback, order, world):
    out = _run_range(synth_corpus, world, order, "rows")
    print(f"\npairs per threshold: {[(k[0], len(v[1])) for k, v in out.items() if not k[1]]}")


@gpu
@pytest.mark.parametrize("world", [2, 3])
def test_queries_mode_range(synth_corpus, loopback, world):
    assert len(synth_corpus.queries) % world != 0
    _run_range(synth_corpus, world, "index", "queries", thresholds=(0.3, 0.9))


CRAFTED = [("index", 2), ("index", 3), ("text", 3)]


@gpu
@pytest.mark.parametrize("order,world", CRAFTED, ids=[f"{o}-W{w}" for o, w in CRAFTED])
def test_crafted_duplicates_across_shards(lib, loopback, order, world):
    """Duplicate texts straddle every shard boundary: their copies tie bit for bit and order by row."""
    c = Corpus(*crafted_texts(6000, world, order))
    _run_range(c, world, order, "rows", thresholds=(0.3, 0.6, 0.9))


@gpu
def test_no_pairs_and_empty_batch(synth_corpus, loopback):
    """A batch whose queries match nothing anywhere, and a batch of no queries."""
    from kakveda_b200.similarity import pack_texts

    c = synth_corpus
    data, off, mode = pack_texts(["qqzzunseen xxyyq", "", "zzqqnothing"])
    build = build_sharded(3, "index", "rows", c)

    def fn(r, g):
        sh = build(r, g)
        try:
            none = [_np(sh.range_packed(data, off, 0.3, mode, device_out=d)) for d in (False, True)]
            empty = [_np(sh.range_packed(data, np.zeros(1, np.int64), 0.3, mode, device_out=d)) for d in (False, True)]
            return none, empty
        finally:
            _close([sh])

    for none, empty in loopback_run(3, fn):
        for res in none:
            np.testing.assert_array_equal(res[0], np.zeros(4, np.int64))
            assert len(res[1]) == len(res[2]) == 0
        for res in empty:
            np.testing.assert_array_equal(res[0], np.zeros(1, np.int64))
            assert len(res[1]) == len(res[2]) == 0


@gpu
def test_five_rows_on_eight_shards(lib, loopback):
    from kakveda_b200 import synth
    from kakveda_b200.dist import ShardedGfkb

    world = 8
    texts = synth.corpus(5)
    c = Corpus(texts, [texts[0], texts[3] + " extra", ""])

    def fn(r, g):
        sh = ShardedGfkb(device=0, rank=r, world=world, group=g)
        try:
            sh.build_packed(c.data, c.off, c.mode)
            return [_np(sh.range_packed(c.qdata, c.qoff, thr, c.qmode)) for thr in (0.3, 1.0)]
        finally:
            _close([sh])

    try:
        out = loopback_run(world, fn)
    except ValueError as e:
        assert "shard" in str(e), e
    else:
        for res, thr in zip(out[0], (0.3, 1.0)):
            _check_range(c, "5 rows on 8 shards", res, thr, _single_range(c, thr))


@gpu
@pytest.mark.parametrize("order,world", [("index", 3), ("text", 3)])
def test_filtered_range(synth_corpus, loopback, order, world):
    """``set_row_labels`` (global labels) + ``labels=`` equal the single index's filtered threshold search."""
    c = synth_corpus
    rng = np.random.default_rng(world)
    row_labels = rng.integers(0, 4, c.n).astype(np.int32)
    qlab = rng.integers(-1, 4, len(c.queries)).astype(np.int32)
    build = build_sharded(world, order, "rows", c)

    def fn(r, g):
        sh = build(r, g)
        try:
            sh.set_row_labels(row_labels)
            return [_np(sh.range_packed(c.qdata, c.qoff, thr, c.qmode, labels=qlab, device_out=thr > 0.5)) for thr in (0.3, 0.6)]
        finally:
            _close([sh])

    out = loopback_run(world, fn)
    c.one.set_row_labels(row_labels)
    try:
        for res, thr in zip(out[0], (0.3, 0.6)):
            single = _np(c.one.range_features(c.qfb, thr, labels=qlab))
            blocks = [(lo, hi, torch.where(torch.as_tensor((qlab[lo:hi, None] < 0) | (qlab[lo:hi, None] == row_labels[None, :]),
                                                           device="cuda"), o, -math.inf)) for lo, hi, o in c.blocks]
            _check_range(c, f"filtered {order} W={world}", res, thr, single, oracle_blocks=blocks)
    finally:
        c.one.set_row_labels(None)


# ---------------------------------------------------------------------------------------------------------------------
# Self-joins and clustering
# ---------------------------------------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def join_corpus(lib):
    """20,000 synthetic rows with stored duplicates; the queries ARE the rows (the oracle excludes each row itself)."""
    texts, _ = synth_texts(20_000, 8)
    c = Corpus(texts, texts)
    blocks = []
    for lo, hi, o in c.blocks:
        o = o.clone()
        o[torch.arange(hi - lo), torch.arange(lo, hi)] = -math.inf
        blocks.append((lo, hi, o))
    c.blocks = blocks
    rng = np.random.default_rng(9)
    c.records = [{"failure_id": f"f{i:05d}", "signature_text": t, "failure_type": f"t{rng.integers(0, 3)}",
                  "affected_apps": [f"app{rng.integers(0, 5)}"]} for i, t in enumerate(texts)]
    return c


@gpu
@pytest.mark.parametrize("order,world", [("index", 3), ("text", 3), ("index", 8)])
def test_selfjoin_and_patterns_tfidf(join_corpus, loopback, order, world):
    from kakveda_b200.patterns import detect_patterns

    c = join_corpus
    thr = 0.8
    build = build_sharded(world, order, "rows", c)

    def fn(r, g):
        sh = build(r, g)
        try:
            res = _np(sh.selfjoin_range(thr, block=7000))
            pats = [detect_patterns(sh, c.records, threshold=thr, k=None, failure_type=ft) for ft in (None, "t1")]
            with pytest.raises(NotImplementedError):
                detect_patterns(sh, c.records, threshold=thr, k=8)
            return res, pats
        finally:
            _close([sh])

    out = loopback_run(world, fn)
    single = _np(c.one.selfjoin_range(thr))
    _check_range(c, f"selfjoin {order} W={world}", out[0][0], thr, single)
    want = [detect_patterns(c.one, c.records, threshold=thr, k=None, failure_type=ft) for ft in (None, "t1")]
    assert sum(len(p["rows"]) > 1 for p in want[0]) > 10
    for r in range(world):
        assert out[r][1] == want, f"rank {r}: patterns differ from the single index's"


def _jaccard_corpus(world, n=12000, nq=300, V=3000):
    from kakveda_b200.dist import shard_bounds

    rng = np.random.default_rng(40 + world)
    sets = [np.unique(rng.zipf(1.3, 15) % (V - 10)) for _ in range(n)]
    for r in range(1, world):
        b = shard_bounds(n, world, r)[0]
        for i in range(b - 20, b + 20):
            sets[i] = sets[b - 20]
    queries = [sets[shard_bounds(n, world, r)[0]] for r in range(1, world)]
    queries += [np.unique(rng.zipf(1.3, 10) % (V - 10)) for _ in range(nq)]
    csr = lambda ss: (np.r_[0, np.cumsum([len(x) for x in ss])].astype(np.int64), np.concatenate(ss).astype(np.int64))
    return (*csr(sets), *csr(queries), V)


@gpu
@pytest.mark.parametrize("world", [2, 3, 8])
def test_sharded_jaccard_range(lib, loopback, world):
    """Pairs and exact counts equal the oracle's for ``range_csr`` and ``selfjoin_range``; ``detect_patterns(k=None)``
    equals the single index's; ``build_local_csr`` cannot self-join."""
    from kakveda_b200 import JaccardIndex
    from kakveda_b200.dist import ShardedJaccard, shard_bounds
    from kakveda_b200.patterns import detect_patterns

    ip, ids, qip, qid, V = _jaccard_corpus(world)
    n = len(ip) - 1
    records = [{"failure_id": f"j{i}", "affected_apps": [f"a{i % 3}"], "failure_type": f"t{i % 2}"} for i in range(n)]

    def fn(r, g):
        sh = ShardedJaccard(V, device=0, rank=r, world=world, group=g)
        sh.build_csr(ip, ids)
        res = [_np(sh.range_csr(qip, qid.astype(np.uint32), thr, device_out=thr > 0.5)) for thr in (0.25, 0.6)]
        join = _np(sh.selfjoin_range(0.5, block=5000))
        pats = [detect_patterns(sh, records, threshold=0.5, k=None, failure_type=ft) for ft in (None, "t1")]
        lo, hi = shard_bounds(n, world, r)
        loc = ShardedJaccard(V, device=0, rank=r, world=world, group=g)
        loc.build_local_csr(ip[lo:hi + 1] - ip[lo], ids[ip[lo]:ip[hi]], n)
        with pytest.raises(ValueError):
            loc.selfjoin_range(0.5)
        return res, join, pats

    out = loopback_run(world, fn)
    for o in out[1:]:
        for a, b in zip(o[0] + [o[1]], out[0][0] + [out[0][1]]):
            for x, y in zip(a, b):
                np.testing.assert_array_equal(x, y)
    orc = T.SparseOracle(ip, ids, np.ones(len(ids)), V, device="cuda")
    I, U = orc.jaccard_counts(qip, qid)
    for res, thr in zip(out[0][0], (0.25, 0.6)):
        check_jaccard_range_device(*res, I, U, thr)
    I, U = orc.jaccard_counts(ip, ids)
    I[torch.arange(n), torch.arange(n)] = 0                                 # a row is not its own neighbour
    check_jaccard_range_device(*out[0][1], I, U, 0.5)
    one = JaccardIndex(V)
    one.add_csr(ip, ids.astype(np.uint32))
    one.finalize()
    try:
        for x, y in zip(out[0][1], _np(one.selfjoin_range(0.5))):
            np.testing.assert_array_equal(x, y)
        want = [detect_patterns(one, records, threshold=0.5, k=None, failure_type=ft) for ft in (None, "t1")]
    finally:
        one.close()
    for r in range(world):
        assert out[r][2] == want, f"rank {r}"


@gpu
@pytest.mark.parametrize("world", [2, 3, 8])
def test_sharded_dense_range(lib, loopback, world):
    """``range`` and ``selfjoin_range`` of ``ShardedDense`` against the float64 cosine of the bf16 rows, with 20-row
    runs of one embedding straddling every shard boundary; identical rows tie bit for bit."""
    from kakveda_b200.dist import ShardedDense, shard_bounds

    n, dim, nq, thr = 3000, 128, 200, 0.2
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
        return _np(sh.range(qs, thr)), _np(sh.range(qs, 0.9, device_out=False)), _np(sh.selfjoin_range(thr, block=1100))

    out = loopback_run(world, fn)
    for o in out[1:]:
        for a, b in zip(o, out[0]):
            for x, y in zip(a, b):
                np.testing.assert_array_equal(x, y)
    rtol = dense_rtol(dim)
    o = T.dense_cosine(qs, emb)
    for res, t in zip(out[0][:2], (thr, 0.9)):
        check_range_device(*res, o, t, rtol, 1e-6)
        _ties_bit_identical(res, key)
    ip, rows, sc = out[0][2]
    for lo in range(0, n, 1000):
        hi = min(n, lo + 1000)
        ob = T.dense_cosine(emb[lo:hi], emb)
        ob[torch.arange(hi - lo), torch.arange(lo, hi)] = -math.inf
        a, b = int(ip[lo]), int(ip[hi])
        check_range_device(ip[lo:hi + 1], rows[a:b], sc[a:b], ob, thr, rtol, 1e-6, first=lo)
    _ties_bit_identical(out[0][2], key)


def _ties_bit_identical(res, key):
    ip, rows, sc = res[:3]
    q = np.repeat(np.arange(len(ip) - 1), np.diff(ip))
    bad = _tie_breaks(q.astype(np.int64) * (len(key) + 1) + key[rows], sc)
    assert len(bad) == 0, ("identical rows scored differently", int(q[bad[0]]), int(rows[bad[0]]))


def _tie_breaks(key, sc):
    """Indices of pairs whose float32 bits differ from those of the first pair with the same key."""
    o = np.argsort(key, kind="stable")
    ks, bits = key[o], sc[o].view(np.uint32)
    first = np.r_[True, ks[1:] != ks[:-1]] if len(ks) else np.zeros(0, bool)
    lead = np.maximum.accumulate(np.where(first, np.arange(len(ks)), 0))
    return o[bits != bits[lead]]
