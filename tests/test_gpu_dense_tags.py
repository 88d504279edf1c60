"""Tag-filtered search on the dense index (kv_dense_set_row_tags / kv_dense_set_tag_filter; DenseIndex.set_row_tags,
tags=, same_tags=) and the label and tag filters of ShardedDense.

The oracle is the kernel itself on a smaller index, as in test_gpu_dense_filter.py: a pair's score is the same float32
expression wherever the pair sits in a tile, so a tag-filtered query over the full index must answer exactly like the
unfiltered query over an index holding only its eligible rows (in row order, rows mapped back).  Scores are also
checked against the float64 cosine of the same bf16 inputs (oracle.dense_cosine)."""
import numpy as np
import pytest

from oracle import tfidf_oracle as O
from test_gpu_dense_filter import BM, BN, RTOL, _assert_topk_equal, _data, _index, _lists, _sub_range, _sub_topk
from test_gpu_topk_edges import check_topk_strict

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def lib(built_lib):
    from kakveda_b200 import _capi

    assert _capi.load().kv_device_count() > 0, "GPU tests need a CUDA device"
    return _capi.load()


def _mask(ts):
    m = np.uint64(0)
    for t in ts:
        m |= np.uint64(1) << np.uint64(t & 63)
    return m


def _meets(row_set, q_set):
    return not q_set or bool(set(row_set) & set(q_set))


def _eligible(row_sets, q_set, dead=None, lab=None, qlab=-1):
    ok = np.array([_meets(s, q_set) for s in row_sets], bool)
    if dead is not None:
        ok &= ~dead
    if qlab >= 0:
        ok &= lab == qlab
    return np.nonzero(ok)[0]


def _predicted_skips(row_sets, dead, q_sets, n_rows, lab=None, qlab=None):
    """Host recomputation of the kernel's skip decision: queries stable-sorted by (label, smallest tag), per 256-row
    tile the OR of the live rows' tag masks (and, with labels, of 1 << (label & 63)), per 128-query tile the OR of the
    queries' masks (all ones for a query without tags or label); an item is skipped when either test finds no bit.  A
    query tile holding a query without tags takes no tag test: that query also matches rows without tags."""
    nq = len(q_sets)
    qlab = np.full(nq, -1) if qlab is None else np.asarray(qlab)
    order = sorted(range(nq), key=lambda q: (int(qlab[q]), min(q_sets[q]) if q_sets[q] else -1))
    full = np.uint64(0xFFFFFFFFFFFFFFFF)
    r_tiles = (n_rows + BN - 1) // BN
    tsig = np.zeros(r_tiles, np.uint64)
    lsig = np.zeros(r_tiles, np.uint64)
    for r in range(n_rows):
        if not dead[r]:
            tsig[r // BN] |= _mask(row_sets[r])
            if lab is not None:
                lsig[r // BN] |= np.uint64(1) << np.uint64(lab[r] & 63)
    q_tiles = (nq + BM - 1) // BM
    skipped = 0
    for qt in range(q_tiles):
        qs = order[qt * BM:(qt + 1) * BM]
        untagged = any(not q_sets[q] for q in qs)
        qm = np.uint64(0)
        ql = np.uint64(0)
        for q in qs:
            qm |= _mask(q_sets[q])
            ql |= full if qlab[q] < 0 else np.uint64(1) << np.uint64(qlab[q] & 63)
        for t in range(r_tiles):
            if (not untagged and (tsig[t] & qm) == 0) or (lab is not None and (qlab >= 0).any() and (lsig[t] & ql) == 0):
                skipped += 1
    return skipped, q_tiles * r_tiles


def _row_sets(n, exact, seed):
    """App-contiguous rows (blocks of sizes that are no multiple of 256), some with a second app, some with none.
    The inexact case uses tags >= 64, three of which (3, 67, 131) collide mod 64, and gives row 7 100 tags."""
    rng = np.random.default_rng(seed)
    pool = list(range(10)) if exact else [0, 1, 2, 3, 67, 131, 70, 1000, 5000, 9]
    cuts = np.sort(rng.choice(np.arange(1, n), len(pool) - 1, replace=False))
    block = np.searchsorted(cuts, np.arange(n), side="right")
    sets = []
    for r in range(n):
        s = {pool[block[r]]}
        u = rng.random()
        if u < 0.2:
            s.add(pool[rng.integers(0, len(pool))])
        elif u < 0.27:
            s = set()
        sets.append(sorted(s))
    if not exact:
        sets[7] = list(range(200, 300))
    return sets


def _query_sets(nq, exact, seed):
    """Query sets drawn from a few shapes: empty, one tag, two tags, 16 tags, a tag no row carries (63 or 195, which
    collides with 3 and 131 mod 64), and one of row 7's many tags."""
    rng = np.random.default_rng(seed)
    if exact:
        shapes = [[], [0], [4], [1, 5], list(range(10)) + [10, 11, 12, 13, 14, 15], [63], [9, 63]]
    else:
        shapes = [[], [3], [67], [131, 70], [0, 1, 2, 3, 67, 131, 70, 1000, 5000, 9, 11, 12, 13, 14, 15, 16], [195],
                  [250], [1000, 195]]
    return [list(shapes[i]) for i in rng.integers(0, len(shapes), nq)]


def _groups(q_sets, qlab=None):
    keys = {}
    for q, s in enumerate(q_sets):
        keys.setdefault((tuple(s), -1 if qlab is None else int(qlab[q])), []).append(q)
    return keys


@pytest.fixture(scope="module", params=[True, False], ids=["tags<64", "tags>=64"])
def tcase(request, lib):
    exact = request.param
    n, d, q = 3000, 128, 300
    C, Q = _data(n, d, q, seed=77 + exact)
    rsets = _row_sets(n, exact, seed=5 + exact)
    qsets = _query_sets(q, exact, seed=6 + exact)
    dx = _index(C)
    dx.set_row_tags(rsets)
    yield dx, C, Q, rsets, qsets
    dx.close()


@pytest.mark.parametrize("k", [1, 16, 32])
def test_tag_topk_equals_eligible_subindex(tcase, k):
    dx, C, Q, rsets, qsets = tcase
    s, r = dx.topk(Q, k, tags=qsets)
    assert dx.last_skipped() == _predicted_skips(rsets, np.zeros(len(C), bool), qsets, len(C))
    o = O.dense_cosine(Q, C)
    for (ts, _), qs in _groups(qsets).items():
        qs = np.asarray(qs)
        rows = _eligible(rsets, ts)
        _assert_topk_equal((s[qs], r[qs]), _sub_topk(C, rows, Q[qs], k))
        oo = np.full((len(qs), len(C)), -np.inf)
        oo[:, rows] = o[np.ix_(qs, rows)]
        check_topk_strict(s[qs], r[qs], oo, k, RTOL, atol=1e-6)
        if 1 in qs:  # the zero query: the lowest eligible rows with score 0
            m = min(k, len(rows))
            assert r[1][:m].tolist() == rows[:m].tolist() and np.all(s[1][:m] == 0)
    import torch

    from kakveda_b200.denseindex import to_bf16_bits

    qd = torch.from_numpy(to_bf16_bits(Q).view(np.int16)).view(torch.bfloat16).cuda()
    sd, rd = dx.topk_device(qd, k, tags=qsets)
    _assert_topk_equal((sd.cpu().numpy(), rd.cpu().numpy()), (s, r))


@pytest.mark.parametrize("thr", [0.3, 0.7])
def test_tag_range_equals_unfiltered_pairs(tcase, thr):
    dx, C, Q, rsets, qsets = tcase
    got = _lists(*dx.range(Q, thr, tags=qsets))
    un = _lists(*dx.range(Q, thr))
    o = O.dense_cosine(Q, C)
    for (ts, _), qs in _groups(qsets).items():
        sub = _sub_range(C, _eligible(rsets, ts), Q[qs], thr)
        for q, w in zip(qs, sub):
            assert got[q] == w, q
            keep = [i for i, row in enumerate(un[q][0]) if _meets(rsets[row], ts)]
            assert got[q] == ([un[q][0][i] for i in keep], [un[q][1][i] for i in keep])
            if got[q][0]:
                np.testing.assert_allclose(got[q][1], o[q, got[q][0]], rtol=RTOL, atol=1e-6)
    import torch

    from kakveda_b200.denseindex import to_bf16_bits

    qd = torch.from_numpy(to_bf16_bits(Q).view(np.int16)).view(torch.bfloat16).cuda()
    ip, r, s = dx.range_device(qd, thr, tags=qsets, device_out=True)
    assert _lists(ip.cpu().numpy(), r.cpu().numpy(), s.cpu().numpy()) == got


def test_labels_tags_and_deletions(tcase):
    """Labels and tags together on an index with deleted rows: per (label, tag set) the survivor sub-index's answer."""
    _, C, Q, rsets, qsets = tcase
    n = len(C)
    rng = np.random.default_rng(12)
    lab = (np.arange(n) // 900).astype(np.int32)
    dead = np.zeros(n, bool)
    dead[rng.choice(n, 150, replace=False)] = True
    dead[512:768] = True
    qlab = rng.integers(-1, lab.max() + 1, len(Q)).astype(np.int32)
    dx = _index(C)
    try:
        dx.set_row_tags(rsets)  # tags before labels and deletions: both keep them
        dx.set_row_labels(lab)
        dx.delete_rows(np.nonzero(dead)[0])
        dx.finalize()
        s, r = dx.topk(Q, 16, labels=qlab, tags=qsets)
        assert dx.last_skipped() == _predicted_skips(rsets, dead, qsets, n, lab, qlab)
        got = _lists(*dx.range(Q, 0.5, labels=qlab, tags=qsets))
        for (ts, L), qs in _groups(qsets, qlab).items():
            qs = np.asarray(qs)
            rows = _eligible(rsets, ts, dead, lab, L)
            _assert_topk_equal((s[qs], r[qs]), _sub_topk(C, rows, Q[qs], 16))
            for q, w in zip(qs, _sub_range(C, rows, Q[qs], 0.5)):
                assert got[q] == w, q
    finally:
        dx.close()


@pytest.mark.parametrize("exact", [True, False], ids=["tags<64", "tags>=64"])
def test_untagged_row_tiles_reach_untagged_queries(lib, exact):
    """Whole 256-row tiles of rows without tags (tile tag signature 0) next to tagged tiles, and a batch mixing queries
    without tags and tagged ones in the same query tiles: the untagged queries must still see the untagged tiles."""
    n, d, q = 2048, 128, 300
    C, Q = _data(n, d, q, seed=19)
    t5 = 5 if exact else 69
    rsets = [[] if (r // BN) % 2 == 0 else [t5] for r in range(n)]  # tiles 0, 2, 4, ... untagged
    rsets[BN + 3] = [t5, 7]
    qsets = [[] if i % 3 == 0 else [t5] for i in range(q)]
    qsets[4] = [7]
    dx = _index(C)
    try:
        dx.set_row_tags(rsets)
        s, r = dx.topk(Q, 16, tags=qsets)
        assert dx.last_skipped() == _predicted_skips(rsets, np.zeros(n, bool), qsets, n)
        got = _lists(*dx.range(Q, 0.3, tags=qsets))
        for (ts, _), qs in _groups(qsets).items():
            qs = np.asarray(qs)
            rows = _eligible(rsets, ts)
            _assert_topk_equal((s[qs], r[qs]), _sub_topk(C, rows, Q[qs], 16))
            for qq, w in zip(qs, _sub_range(C, rows, Q[qs], 0.3)):
                assert got[qq] == w, qq
        assert np.isin(r[::3], np.arange(BN)).any()  # the untagged queries do reach tile 0
        # a tagged-only batch skips the untagged tiles
        tagged = [i for i in range(q) if qsets[i]]
        dx.topk(Q[tagged], 16, tags=[qsets[i] for i in tagged])
        sk, items = dx.last_skipped()
        assert (sk, items) == _predicted_skips(rsets, np.zeros(n, bool), [qsets[i] for i in tagged], n) and sk > 0
    finally:
        dx.close()


def test_app_contiguous_rows_skip_most_items(lib):
    """One app per 2000-row block and one app per query: a query tile only needs the row tiles of its apps."""
    n, d, q = 40000, 64, 1000
    C, Q = _data(n, d, q, seed=3)
    rsets = [[r // 2000] for r in range(n)]
    qsets = [[int(a)] for a in np.random.default_rng(8).integers(0, n // 2000, q)]
    dx = _index(C)
    try:
        dx.set_row_tags(rsets)
        s, r = dx.topk(Q, 16, tags=qsets)
        sk, items = dx.last_skipped()
        assert (sk, items) == _predicted_skips(rsets, np.zeros(n, bool), qsets, n)
        assert sk > items // 2
        qa = np.array([t[0] for t in qsets])
        for a in np.unique(qa)[:4]:
            qs = np.nonzero(qa == a)[0]
            _assert_topk_equal((s[qs], r[qs]), _sub_topk(C, np.arange(a * 2000, (a + 1) * 2000), Q[qs], 16))
    finally:
        dx.close()


@pytest.mark.parametrize("same_label", [False, True])
def test_selfjoin_same_tags(lib, same_label):
    n, d = 2500, 128
    C, _ = _data(n, d, 1, seed=31)
    rng = np.random.default_rng(9)
    pool = [[], [1], [2], [1, 2], [70], [6, 134]]  # 6 and 134 collide mod 64, 70 and 6 too
    rsets = [list(pool[i]) for i in rng.integers(0, len(pool), n)]
    lab = rng.integers(0, 3, n).astype(np.int32)
    dead = np.zeros(n, bool)
    dead[rng.choice(n, 100, replace=False)] = True
    dx = _index(C)
    try:
        dx.set_row_tags(rsets)
        dx.set_row_labels(lab)
        dx.delete_rows(np.nonzero(dead)[0])
        dx.finalize()
        lo, hi = 50, 2400
        s, r = dx.selfjoin_topk(16, lo=lo, hi=hi, same_label=same_label, same_tags=True)
        got = _lists(*dx.selfjoin_range(0.4, lo=lo, hi=hi, same_label=same_label, same_tags=True))
        groups = {}
        for i in range(lo, hi):
            if not dead[i]:
                groups.setdefault((tuple(rsets[i]), int(lab[i]) if same_label else -1), []).append(i)
        for (ts, L), members in groups.items():
            keep = _eligible(rsets, ts, dead, lab, L)
            sub = _index(C[keep])
            try:
                ks, kr = sub.selfjoin_topk(16)
                kj = _lists(*sub.selfjoin_range(0.4))
            finally:
                sub.close()
            pos = np.searchsorted(keep, members)
            for row, j in zip(members, pos):
                i = row - lo
                np.testing.assert_array_equal(r[i], np.where(kr[j] >= 0, keep[np.maximum(kr[j], 0)], -1))
                np.testing.assert_array_equal(s[i].view(np.uint32), ks[j].view(np.uint32))
                assert got[i] == (keep[np.asarray(kj[j][0], np.int64)].tolist(), kj[j][1])
        for row in np.nonzero(dead[lo:hi])[0]:
            assert np.all(r[row] == -1) and got[row] == ([], [])
    finally:
        dx.close()


def test_errors_and_tag_lifetime(lib):
    n, d, q = 1000, 64, 50
    C, Q = _data(n, d, q, seed=41)
    rsets = [[r % 5] for r in range(n)]
    dx = _index(C)
    try:
        with pytest.raises(RuntimeError):
            dx.topk(Q, 4, tags=[[1]] * q)  # no row tags
        with pytest.raises(ValueError):
            dx.set_row_tags(rsets[:-1])  # wrong count
        with pytest.raises(ValueError):
            dx.set_row_tags(rsets[:-1] + [[-3]])  # negative row tag
        dx.set_row_tags(rsets)
        plain = dx.topk(Q, 8)
        with pytest.raises(ValueError):
            dx.topk(Q, 8, tags=[[1]] * (q + 1))  # count mismatch
        with pytest.raises(ValueError):
            dx.topk(Q, 8, tags=[list(range(17))] + [[1]] * (q - 1))  # 17 tags
        with pytest.raises(ValueError):
            dx.topk(Q, 8, labels=np.zeros(q, np.int32), tags=[[-1]] * q)  # negative query tag; the labels go too
        with pytest.raises(ValueError):
            dx.range(Q, 0.5, tags=[list(range(17))] * q)
        _assert_topk_equal(dx.topk(Q, 8), plain)  # nothing of the failed calls is left
        # the C filter is consumed by the next call, even one that fails
        ip = np.arange(q + 2, dtype=np.int64)
        t = np.ones(q + 1, np.int32)
        from kakveda_b200 import _capi
        from kakveda_b200.similarity import _ptr
        import ctypes as C_

        lib_ = _capi.load()
        _capi.check(lib_.kv_dense_set_tag_filter(dx._h, _ptr(ip, C_.c_int64), _ptr(t, C_.c_int32), q + 1))
        with pytest.raises(ValueError):
            dx.topk(Q, 8)
        _assert_topk_equal(dx.topk(Q, 8), plain)
        f = dx.topk(Q, 8, tags=[[2]] * q)
        assert np.all(np.array(rsets)[f[1], 0] == 2)
        _assert_topk_equal(dx.topk(Q, 8), plain)
        # empty query sets: the unfiltered call
        _assert_topk_equal(dx.topk(Q, 8, tags=[[]] * q), plain)
        assert dx.last_skipped()[0] == 0
        # tags survive deletion and finalize; an append drops them; set again, they need no finalize
        dx.delete_rows([2, 7])
        dx.finalize()
        f = dx.topk(Q, 8, tags=[[2]] * q)
        assert not np.isin(f[1], [2, 7]).any() and np.all(np.array(rsets)[f[1], 0] == 2)
        dx.add(C[:10])
        dx.finalize()
        with pytest.raises(RuntimeError):
            dx.topk(Q, 8, tags=[[2]] * q)
        with pytest.raises(RuntimeError):
            dx.selfjoin_topk(8, same_tags=True)
        rs2 = rsets + [[3]] * 10
        dx.set_row_tags(rs2)
        f = dx.topk(Q, 8, tags=[[3]] * q)
        assert np.all(np.array(rs2)[f[1], 0] == 3)
        # clearing
        dx.set_row_tags(None)
        with pytest.raises(RuntimeError):
            dx.range(Q, 0.5, tags=[[3]] * q)
        # a self-join row with more than 16 tags
        big = [list(s) for s in rs2]
        big[30] = list(range(40))
        dx.set_row_tags(big)
        with pytest.raises(ValueError, match="row 30"):
            dx.selfjoin_topk(8, same_tags=True)
        with pytest.raises(ValueError, match="row 30"):
            dx.selfjoin_range(0.5, same_tags=True)
        s, r = dx.selfjoin_topk(8, lo=31, hi=200, same_tags=True)  # rows outside [lo, hi) may have more
        for i, row in enumerate(range(31, 200)):
            assert all(_meets(big[x], big[row]) for x in r[i] if x >= 0)
    finally:
        dx.close()


# ---------------------------------------------------------------------------------------------------------------------
# ShardedDense through the loopback collectives
# ---------------------------------------------------------------------------------------------------------------------

from test_gpu_shard_loopback import loopback  # noqa: E402,F401  (the fixture)


@pytest.mark.parametrize("world", [1, 2, 3, 8])
def test_sharded_dense_filters_equal_single_index(lib, loopback, world):  # noqa: F811
    import torch

    from kakveda_b200.denseindex import to_bf16_bits
    from kakveda_b200.dist import ShardedDense, shard_bounds

    n, dim, nq, k, thr = 3000, 128, 200, 16, 0.45
    C, Q = _data(n, dim, nq, seed=100 + world)
    rsets = _row_sets(n, False, seed=world)
    rsets[7] = [3, 250]  # the self-joins take every row as a query: at most 16 tags each
    qsets = _query_sets(nq, False, seed=world + 1)
    lab = (np.arange(n) * 5 // n).astype(np.int32)
    qlab = np.random.default_rng(world).integers(-1, 5, nq).astype(np.int32)
    emb = torch.from_numpy(to_bf16_bits(C).view(np.int16)).view(torch.bfloat16).cuda()
    qe = torch.from_numpy(to_bf16_bits(Q).view(np.int16)).view(torch.bfloat16).cuda()

    def fn(r, grp):
        lo, hi = shard_bounds(n, world, r)
        sh = ShardedDense(dim, device=0, rank=r, world=world, group=grp)
        sh.build(emb[lo:hi].contiguous(), n)
        sh.set_row_labels(lab)
        sh.set_row_tags(rsets)
        s, rr = sh.topk(qe, k, labels=qlab, tags=qsets)
        ip, pr, ps = sh.range(qe, thr, device_out=False, labels=qlab, tags=qsets)
        a_s, a_r = sh.allpairs_topk(k, block=1100, same_label=True, same_tags=True)
        j_ip, j_r, j_s = sh.selfjoin_range(thr, block=1100, device_out=False, same_tags=True)
        out = (s.cpu().numpy(), rr.cpu().numpy(), _lists(ip, pr, ps), a_s.cpu().numpy(), a_r.cpu().numpy(),
               _lists(j_ip, j_r, j_s))
        sh.index.close()
        return out

    out = loopback(world, fn)
    for o in out[1:]:
        for a, b in zip(o, out[0]):
            if isinstance(a, np.ndarray):
                np.testing.assert_array_equal(a.view(np.uint32) if a.dtype == np.float32 else a,
                                              b.view(np.uint32) if b.dtype == np.float32 else b)
            else:
                assert a == b
    single = _index(C, lab)
    try:
        single.set_row_tags(rsets)
        s, rr, rng_, a_s, a_r, sj = out[0]
        _assert_topk_equal((s, rr), single.topk(Q, k, labels=qlab, tags=qsets))
        assert rng_ == _lists(*single.range(Q, thr, labels=qlab, tags=qsets))
        _assert_topk_equal((a_s, a_r), single.selfjoin_topk(k, same_label=True, same_tags=True))
        assert sj == _lists(*single.selfjoin_range(thr, same_tags=True))
        assert any(len(x[0]) for x in rng_) and any(len(x[0]) for x in sj)
    finally:
        single.close()
