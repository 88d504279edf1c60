"""Label-filtered search and row deletion on the dense index (kv_dense_set_row_labels / kv_dense_set_query_filter /
kv_dense_delete_rows; DenseIndex.set_row_labels, labels=, same_label=, delete_rows).

The oracle is the kernel itself on a smaller index: a pair's score is the same float32 expression wherever the pair sits
in a tile, so a filtered query over the full index must answer exactly like the unfiltered query over an index holding
only its label's rows (in row order, rows mapped back), and an index with deletions exactly like the index of its
survivors.  Scores are also checked against the float64 cosine of the same bf16 inputs (oracle.dense_cosine)."""
import numpy as np
import pytest

from oracle import tfidf_oracle as O
from test_gpu_topk_edges import check_topk_strict

pytestmark = pytest.mark.gpu

RTOL = 2e-5
BN, BM = 256, 128


@pytest.fixture(scope="module")
def lib(built_lib):
    from kakveda_b200 import _capi

    assert _capi.load().kv_device_count() > 0, "GPU tests need a CUDA device"
    return _capi.load()


def _data(n, d, q, seed):
    """Clustered rows (so that top-k lists and threshold pairs are not all noise), a zero row and duplicate rows; queries
    near the centroids, a zero query and copies of rows."""
    rng = np.random.default_rng(seed)
    cent = rng.standard_normal((max(4, n // 40), d))
    C = cent[rng.integers(0, len(cent), n)] + rng.uniform(0.2, 1.0, (n, 1)) * rng.standard_normal((n, d))
    Q = cent[rng.integers(0, len(cent), q)] + rng.uniform(0.1, 0.8, (q, 1)) * rng.standard_normal((q, d))
    C, Q = C.astype(np.float32), Q.astype(np.float32)
    if n > 301:
        C[5] = 0.0
        C[301] = C[300]
    if q > 2:
        Q[1] = 0.0
        Q[2] = C[min(300, n - 1)]
    return C, Q


def _index(C, labels=None):
    from kakveda_b200 import DenseIndex

    dx = DenseIndex(C.shape[1])
    if len(C):
        dx.add(C)
    dx.finalize()
    if labels is not None:
        dx.set_row_labels(labels)
    return dx


def _sub_topk(C, rows, Q, k):
    """Unfiltered top-k of Q over an index of C[rows] (rows ascending), rows mapped back to the full index."""
    if len(rows) == 0:
        return np.full((len(Q), k), -np.inf, np.float32), np.full((len(Q), k), -1, np.int64)
    sub = _index(C[rows])
    try:
        s, r = sub.topk(Q, k)
    finally:
        sub.close()
    return s, np.where(r >= 0, rows[np.maximum(r, 0)], -1)


def _sub_range(C, rows, Q, thr):
    """Unfiltered range result of Q over an index of C[rows] as per-query lists of (row, score), rows mapped back."""
    if len(rows) == 0:
        return [([], []) for _ in range(len(Q))]
    sub = _index(C[rows])
    try:
        ip, r, s = sub.range(Q, thr)
    finally:
        sub.close()
    return [(rows[r[ip[q]:ip[q + 1]]].tolist(), s[ip[q]:ip[q + 1]].tolist()) for q in range(len(Q))]


def _lists(ip, r, s):
    return [(r[ip[q]:ip[q + 1]].tolist(), s[ip[q]:ip[q + 1]].tolist()) for q in range(len(ip) - 1)]


def _assert_topk_equal(a, b):
    np.testing.assert_array_equal(a[1], b[1])
    np.testing.assert_array_equal(a[0].view(np.uint32), b[0].view(np.uint32))


def _predicted_skips(row_labels, dead, q_labels, n_rows):
    """Host recomputation of the kernel's skip decision: per 256-row tile the OR of 1 << (label & 63) over its live
    rows, per 128-query tile (queries stable-sorted by label) the same over its queries, all ones for a -1 query."""
    bits = np.where(dead, np.uint64(0), np.left_shift(np.uint64(1), (row_labels & 63).astype(np.uint64)))
    r_tiles = (n_rows + BN - 1) // BN
    tsig = np.zeros(r_tiles, np.uint64)
    for t in range(r_tiles):
        tsig[t] = np.bitwise_or.reduce(bits[t * BN:(t + 1) * BN])
    ql = np.sort(q_labels, kind="stable")
    q_tiles = (len(ql) + BM - 1) // BM
    skipped = 0
    for qt in range(q_tiles):
        lab = ql[qt * BM:(qt + 1) * BM]
        qs = np.uint64(0xFFFFFFFFFFFFFFFF) if (lab < 0).any() else \
            np.bitwise_or.reduce(np.left_shift(np.uint64(1), (lab & 63).astype(np.uint64)))
        skipped += int(np.count_nonzero((tsig & qs) == 0))
    return skipped, q_tiles * r_tiles


@pytest.fixture(scope="module", params=[(3000, 128, 300, 7), (9000, 256, 400, 80)], ids=["3000x128", "9000x256-80labels"])
def fcase(request, lib):
    """Rows with labels clustered in contiguous blocks of sizes that are no multiple of 256 (the second case with 80
    labels, so that signature bits collide), queries with random labels."""
    n, d, q, n_lab = request.param
    C, Q = _data(n, d, q, seed=n + d)
    rng = np.random.default_rng(n)
    cuts = np.sort(rng.choice(np.arange(1, n), n_lab - 1, replace=False))
    lab = np.zeros(n, np.int32)
    for i, c in enumerate(cuts):
        lab[c:] = i + 1
    qlab = rng.integers(0, n_lab, q).astype(np.int32)
    dx = _index(C, lab)
    yield dx, C, Q, lab, qlab
    dx.close()


@pytest.mark.parametrize("k", [1, 16, 32])
def test_filtered_topk_equals_label_subindex(fcase, k):
    dx, C, Q, lab, qlab = fcase
    s, r = dx.topk(Q, k, labels=qlab)
    o = O.dense_cosine(Q, C)
    for L in np.unique(qlab):
        qs = np.nonzero(qlab == L)[0]
        rows = np.nonzero(lab == L)[0]
        want = _sub_topk(C, rows, Q[qs], k)
        _assert_topk_equal((s[qs], r[qs]), want)
        oo = np.full((len(qs), len(C)), -np.inf)
        oo[:, rows] = o[np.ix_(qs, rows)]
        check_topk_strict(s[qs], r[qs], oo, k, RTOL, atol=1e-6)
    sk, items = dx.last_skipped()
    assert (sk, items) == _predicted_skips(lab, np.zeros(len(C), bool), qlab, len(C))
    assert sk > 0
    # the device form gives the same bits
    import torch

    from kakveda_b200.denseindex import to_bf16_bits

    qd = torch.from_numpy(to_bf16_bits(Q).view(np.int16)).view(torch.bfloat16).cuda()
    sd, rd = dx.topk_device(qd, k, labels=qlab)
    _assert_topk_equal((sd.cpu().numpy(), rd.cpu().numpy()), (s, r))


@pytest.mark.parametrize("thr", [0.3, 0.6, 0.9])
def test_filtered_range_equals_label_subindex(fcase, thr):
    dx, C, Q, lab, qlab = fcase
    got = _lists(*dx.range(Q, thr, labels=qlab))
    want = [None] * len(Q)
    for L in np.unique(qlab):
        qs = np.nonzero(qlab == L)[0]
        for q, w in zip(qs, _sub_range(C, np.nonzero(lab == L)[0], Q[qs], thr)):
            want[q] = w
    o = O.dense_cosine(Q, C)
    for q in range(len(Q)):
        assert got[q][0] == want[q][0], q
        assert np.array_equal(np.float32(got[q][1]).view(np.uint32), np.float32(want[q][1]).view(np.uint32)), q
        if got[q][0]:
            np.testing.assert_allclose(got[q][1], o[q, got[q][0]], rtol=RTOL, atol=1e-6)
            assert np.all(lab[got[q][0]] == qlab[q])
    assert dx.last_skipped()[0] > 0
    # device outputs and device queries: the same pairs, ordered like an unfiltered fetch
    import torch

    from kakveda_b200.denseindex import to_bf16_bits

    qd = torch.from_numpy(to_bf16_bits(Q).view(np.int16)).view(torch.bfloat16).cuda()
    ip, r, s = dx.range_device(qd, thr, labels=qlab, device_out=True)
    assert _lists(ip.cpu().numpy(), r.cpu().numpy(), s.cpu().numpy()) == got


def test_mixed_batch(fcase):
    """Labels, -1 queries and a label no row has, in shuffled order: per query the single-label answer; the -1 queries
    the unfiltered answer, bit for bit."""
    dx, C, Q, lab, qlab = fcase
    rng = np.random.default_rng(3)
    ql = qlab.copy()
    ql[rng.random(len(ql)) < 0.25] = -1
    ql[rng.random(len(ql)) < 0.1] = 10_000  # no row has it
    perm = rng.permutation(len(Q))
    Qs, ls = Q[perm], ql[perm]
    k = 16
    s, r = dx.topk(Qs, k, labels=ls)
    su, ru = dx.topk(Qs, k)
    for L in np.unique(ls):
        qs = np.nonzero(ls == L)[0]
        if L < 0:
            _assert_topk_equal((s[qs], r[qs]), (su[qs], ru[qs]))
        else:
            _assert_topk_equal((s[qs], r[qs]), dx.topk(Qs[qs], k, labels=np.full(len(qs), L, np.int32)))
            if L == 10_000:
                assert np.all(r[qs] == -1) and np.all(np.isneginf(s[qs]))
    got = _lists(*dx.range(Qs, 0.5, labels=ls))
    un = _lists(*dx.range(Qs, 0.5))
    for q in range(len(Qs)):
        if ls[q] < 0:
            assert got[q] == un[q]
        else:
            keep = [i for i, row in enumerate(un[q][0]) if lab[row] == ls[q]]
            assert got[q] == ([un[q][0][i] for i in keep], [un[q][1][i] for i in keep])


def test_one_unfiltered_query_per_tile_skips_nothing(fcase):
    """A query tile holding a -1 query needs every row tile.  The kernel sorts the queries by label, so the -1 queries
    come first: a one-tile batch with a single -1 query, and a batch whose -1 queries reach into its last tile."""
    dx, C, Q, lab, qlab = fcase
    r_tiles = (len(C) + BN - 1) // BN
    one = qlab[:100].copy()
    one[57] = -1
    s, r = dx.topk(Q[:100], 8, labels=one)
    assert dx.last_skipped() == (0, r_tiles)
    n3 = 2 * BM + 44
    many = np.full(n3, -1, np.int32)
    many[2 * BM + 1:] = qlab[:n3 - 2 * BM - 1]
    perm = np.random.default_rng(9).permutation(n3)
    dx.topk(Q[:n3][perm], 8, labels=many[perm])
    assert dx.last_skipped() == (0, 3 * r_tiles)
    assert _predicted_skips(lab, np.zeros(len(C), bool), many, len(C)) == (0, 3 * r_tiles)
    # the same queries with labels only do skip
    dx.topk(Q[:n3], 8, labels=qlab[:n3])
    assert dx.last_skipped()[0] > 0


def test_deletion_equals_survivor_index(lib):
    n, d, q = 2000, 128, 200
    C, Q = _data(n, d, q, seed=11)
    dead = np.zeros(n, bool)
    dead[[0, 255, 256, 257, n - 1, 300]] = True
    dead[512:768] = True  # one whole 256-row tile
    dead[np.random.default_rng(1).choice(n, 100, replace=False)] = True
    dx = _index(C)
    try:
        rows_del = np.nonzero(dead)[0]
        dx.delete_rows(np.concatenate([rows_del, rows_del[:5]]))  # duplicates allowed
        assert dx.n_live_rows == n - dead.sum()
        np.testing.assert_array_equal(dx.deleted_mask(), dead)
        with pytest.raises(RuntimeError):
            dx.topk(Q, 4)  # not finalized
        dx.finalize()
        live = np.nonzero(~dead)[0]
        o = O.dense_cosine(Q, C)
        o[:, dead] = -np.inf
        for k in (1, 16, 32):
            s, r = dx.topk(Q, k)
            _assert_topk_equal((s, r), _sub_topk(C, live, Q, k))
            check_topk_strict(s, r, o, k, RTOL, atol=1e-6)
            assert not np.isin(r, rows_del).any()
        for thr in (0.3, 0.8):
            assert _lists(*dx.range(Q, thr)) == _sub_range(C, live, Q, thr)
        # self-join: a deleted query row gets (-inf, -1) and no pairs; the live rows answer like the survivor index
        s, r = dx.selfjoin_topk(16)
        assert np.all(r[dead] == -1) and np.all(np.isneginf(s[dead]))
        sub = _index(C[live])
        try:
            ss, sr = sub.selfjoin_topk(16)
            _assert_topk_equal((s[live], r[live]), (ss, np.where(sr >= 0, live[np.maximum(sr, 0)], -1)))
            sj = _lists(*dx.selfjoin_range(0.5))
            subj = _lists(*sub.selfjoin_range(0.5))
            assert all(sj[i] == ([], []) for i in rows_del)
            assert [sj[i] for i in live] == [(live[np.asarray(rr, np.int64)].tolist(), sc) for rr, sc in subj]
        finally:
            sub.close()
        # deleting, then appending, then finalizing keeps the deletions; appended rows are live
        C2, _ = _data(300, d, 1, seed=12)
        dx.add(C2)
        dx.finalize()
        assert dx.n_live_rows == n + 300 - dead.sum()
        dead2 = np.concatenate([dead, np.zeros(300, bool)])
        np.testing.assert_array_equal(dx.deleted_mask(), dead2)
        Call = np.concatenate([C, C2])
        s, r = dx.topk(Q, 16)
        _assert_topk_equal((s, r), _sub_topk(Call, np.nonzero(~dead2)[0], Q, 16))
        with pytest.raises(ValueError):
            dx.delete_rows([n + 300])
        with pytest.raises(ValueError):
            dx.delete_rows([-1])
    finally:
        dx.close()


def test_skip_with_deletions_and_clustered_labels(lib):
    """An all-deleted tile has signature 0 and is skipped by every filtered query; results stay the survivor index's."""
    n, d, q = 5000, 128, 260
    C, Q = _data(n, d, q, seed=21)
    lab = (np.arange(n) // 700).astype(np.int32)  # blocks of 700 rows
    dead = np.zeros(n, bool)
    dead[1024:1280] = True
    dead[np.random.default_rng(2).choice(n, 200, replace=False)] = True
    dx = _index(C, lab)
    try:
        dx.delete_rows(np.nonzero(dead)[0])
        dx.finalize()  # labels survive the deletion
        qlab = np.random.default_rng(4).integers(0, lab.max() + 1, q).astype(np.int32)
        s, r = dx.topk(Q, 16, labels=qlab)
        for L in np.unique(qlab):
            qs = np.nonzero(qlab == L)[0]
            _assert_topk_equal((s[qs], r[qs]), _sub_topk(C, np.nonzero((lab == L) & ~dead)[0], Q[qs], 16))
        assert dx.last_skipped() == _predicted_skips(lab, dead, qlab, n)
        assert dx.last_skipped()[0] > 0
    finally:
        dx.close()


def test_selfjoin_same_label(lib):
    from kakveda_b200 import patterns

    n, d = 3000, 128
    C, _ = _data(n, d, 1, seed=31)
    rng = np.random.default_rng(5)
    lab = np.sort(rng.integers(0, 6, n)).astype(np.int32)  # label-sorted rows: the query order is the identity
    lab[rng.choice(n, 200, replace=False)] = 6  # and some out of order
    dead = np.zeros(n, bool)
    dead[rng.choice(n, 150, replace=False)] = True
    dead[[0, 255, 256]] = True
    dx = _index(C, lab)
    try:
        dx.delete_rows(np.nonzero(dead)[0])
        dx.finalize()
        lo, hi = 100, 2900
        s, r = dx.selfjoin_topk(16, lo=lo, hi=hi, same_label=True)
        ip, rr, ss = dx.selfjoin_range(0.5, lo=lo, hi=hi, same_label=True)
        got_range = _lists(ip, rr, ss)
        for L in np.unique(lab):
            keep = np.nonzero((lab == L) & ~dead)[0]
            sub = _index(C[keep])
            try:
                ks, kr = sub.selfjoin_topk(16)
                kj = _lists(*sub.selfjoin_range(0.5))
            finally:
                sub.close()
            for j, row in enumerate(keep):
                if lo <= row < hi:
                    i = row - lo
                    np.testing.assert_array_equal(r[i], np.where(kr[j] >= 0, keep[np.maximum(kr[j], 0)], -1))
                    np.testing.assert_array_equal(s[i].view(np.uint32), ks[j].view(np.uint32))
                    assert got_range[i] == (keep[np.asarray(kj[j][0], np.int64)].tolist(), kj[j][1])
        for row in np.nonzero(dead[lo:hi])[0]:
            assert np.all(r[row] == -1) and got_range[row] == ([], [])
        # patterns on the exact threshold graph leave the deleted rows out: the survivors' components
        recs = [{"failure_id": f"F-{i:04d}", "affected_apps": [f"app{i % 3}"], "failure_type": "t"} for i in range(n)]
        got = patterns.detect_patterns(dx, recs, threshold=0.7, k=None)
        live = np.nonzero(~dead)[0]
        sub = _index(C[live])
        try:
            want = patterns.detect_patterns(sub, [recs[i] for i in live], threshold=0.7, k=None)
        finally:
            sub.close()
        assert [p["failure_ids"] for p in got] == [p["failure_ids"] for p in want]
        assert all(not dead[int(f[2:])] for p in got for f in p["failure_ids"])
    finally:
        dx.close()


def test_errors_and_filter_lifetime(lib):
    n, d, q = 1000, 64, 50
    C, Q = _data(n, d, q, seed=41)
    lab = (np.arange(n) % 3).astype(np.int32)
    dx = _index(C)
    try:
        with pytest.raises(ValueError):
            dx.set_row_labels(lab[:-1])  # wrong length
        bad = lab.copy()
        bad[3] = -1
        with pytest.raises(ValueError):
            dx.set_row_labels(bad)  # row label < 0
        with pytest.raises(RuntimeError):
            dx.topk(Q, 4, labels=np.zeros(q, np.int32))  # no row labels
        dx.set_row_labels(lab)
        ql = np.zeros(q, np.int32)
        ql[0] = -2
        with pytest.raises(ValueError):
            dx.topk(Q, 4, labels=ql)  # query label < -1
        with pytest.raises(ValueError):
            dx.topk(Q, 4, labels=np.zeros(q + 1, np.int32))  # n_q mismatch
        plain = dx.topk(Q, 8)
        # the filter is consumed by one call, even one that fails
        _assert_topk_equal(dx.topk(Q, 8), plain)
        f = dx.topk(Q, 8, labels=np.ones(q, np.int32))
        assert np.all(lab[f[1]] == 1)
        _assert_topk_equal(dx.topk(Q, 8), plain)
        # a filtered range, then the fetch order of an unfiltered one (score desc, row asc)
        ip, r, s = dx.range(Q, 0.3, labels=np.ones(q, np.int32))
        for i in range(q):
            rr, sc = r[ip[i]:ip[i + 1]], s[ip[i]:ip[i + 1]]
            assert np.all((sc[:-1] > sc[1:]) | ((sc[:-1] == sc[1:]) & (rr[:-1] < rr[1:])))
            assert np.all(lab[rr] == 1)
        # labels survive finalize and deletion, an append drops them
        dx.delete_rows([1, 4])
        dx.finalize()
        f = dx.topk(Q, 8, labels=np.ones(q, np.int32))
        assert not np.isin(f[1], [1, 4]).any() and np.all(lab[f[1]] == 1)
        dx.add(C[:10])
        dx.finalize()
        with pytest.raises(RuntimeError):
            dx.topk(Q, 8, labels=np.ones(q, np.int32))
        with pytest.raises(RuntimeError):
            dx.selfjoin_topk(8, same_label=True)
        dx.set_row_labels(np.concatenate([lab, lab[:10]]))
        f = dx.topk(Q, 8, labels=np.ones(q, np.int32))
        assert np.all(np.concatenate([lab, lab[:10]])[f[1]] == 1)
        # all -1: the unfiltered call
        _assert_topk_equal(dx.topk(Q, 8, labels=np.full(q, -1, np.int32)), dx.topk(Q, 8))
        assert dx.last_skipped()[0] == 0
    finally:
        dx.close()
