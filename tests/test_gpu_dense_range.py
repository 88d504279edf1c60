"""Dense threshold search (kv_dense_range* / kv_dense_range_fetch, DenseIndex.range*) and pattern clustering of
embeddings on the exact threshold graph (detect_patterns(DenseIndex, k=None)).

Scores are the float32 values the dense top-k reports (rtol 2e-5 against the float64 cosine of the same bf16 inputs,
as for the dense top-k).  A pair is required when its float64 score clears the threshold by more than the band, and
may only be returned when it lies above the band's lower edge."""
import numpy as np
import pytest

from oracle import tfidf_oracle as O
from test_gpu_range import _components, _threshold_in_gap

RTOL = 2e-5
ATOL = 1e-6
BAND = 4e-5
THRESHOLDS = (0.3, 0.6, 0.8, 0.95)


@pytest.fixture(scope="module")
def lib(built_lib):
    from kakveda_b200 import _capi

    assert _capi.load().kv_device_count() > 0, "GPU tests need a CUDA device"
    return _capi.load()


def check_dense_range(indptr, rows, scores, oracle, thr, excl=None):
    """indptr/rows/scores: a range result; oracle: [Q, N] float64; excl[q]: the row query q must not return (or -1)."""
    Q, N = oracle.shape
    assert indptr.shape == (Q + 1,) and indptr[0] == 0 and np.all(np.diff(indptr) >= 0)
    assert indptr[-1] == len(rows) == len(scores)
    assert rows.dtype == np.int64 and scores.dtype == np.float32
    for q in range(Q):
        r, s = rows[indptr[q]:indptr[q + 1]], scores[indptr[q]:indptr[q + 1]]
        assert len(np.unique(r)) == len(r), "duplicate (query, row) pair"
        assert np.all((s[:-1] > s[1:]) | ((s[:-1] == s[1:]) & (r[:-1] < r[1:]))), "order is not (score desc, row asc)"
        assert np.all((r >= 0) & (r < N)) and np.all(s >= np.float32(thr))
        o = oracle[q]
        np.testing.assert_allclose(s, o[r], rtol=RTOL, atol=ATOL)
        assert np.all(o[r] >= thr * (1 - BAND) - ATOL), (q, o[r].min())
        want = np.nonzero(o >= thr * (1 + BAND) + ATOL)[0]
        if excl is not None and excl[q] >= 0:
            assert excl[q] not in r
            want = want[want != excl[q]]
        assert np.isin(want, r).all(), (q, np.setdiff1d(want, r)[:5])


def _clustered(n, d, q, seed):
    """Rows around n / 50 centroids with per-row noise levels (within-cluster cosines spread over ~0.4 .. 0.96), row 7
    zero, rows 101 = 100 and n-1 = n-2 duplicates; query 0 a scaled copy of a row (cosine 1), query 1 zero, query 2 a
    copy of row 100, up to 47 more scaled copies, the rest noisy centroids."""
    rng = np.random.default_rng(seed)
    cent = rng.standard_normal((max(4, n // 50), d))
    C = cent[rng.integers(0, len(cent), n)] + rng.uniform(0.2, 1.2, (n, 1)) * rng.standard_normal((n, d))
    Q = cent[rng.integers(0, len(cent), q)] + rng.uniform(0.1, 1.0, (q, 1)) * rng.standard_normal((q, d))
    C, Q = C.astype(np.float32), Q.astype(np.float32)
    C[7] = 0.0
    C[101] = C[100]
    C[n - 1] = C[n - 2]
    m = min(q, 50)
    Q[:m] = C[rng.integers(8, n, m)] * 1.5
    if q > 1:
        Q[1] = 0.0
    if q > 2:
        Q[2] = C[100]
    return C, Q


@pytest.fixture(scope="module", params=[(257, 64, 3), (3000, 128, 200), (20000, 768, 500)], ids=lambda p: "x".join(map(str, p)))
def case(request, lib):
    from kakveda_b200 import DenseIndex

    n, d, q = request.param
    C, Q = _clustered(n, d, q, seed=n + d)
    dx = DenseIndex(d)
    dx.add(C[: n // 2])
    dx.add(C[n // 2:])
    dx.finalize()
    yield dx, C, Q, O.dense_cosine(Q, C)
    dx.close()


@pytest.mark.gpu
@pytest.mark.parametrize("thr", THRESHOLDS)
def test_dense_range_vs_float64_oracle(case, thr):
    dx, C, Q, oracle = case
    indptr, rows, scores = dx.range(Q, thr)
    check_dense_range(indptr, rows, scores, oracle, thr)
    assert indptr[1] > indptr[0] and np.float32(scores[0]) >= np.float32(0.9999)  # a scaled copy of a row: cosine 1
    if len(Q) > 2:
        assert indptr[2] == indptr[1]                                              # the zero query: nothing
        seg = rows[indptr[2]:indptr[3]]
        assert seg[:2].tolist() == [100, 101]                                      # duplicates tie -> lower row first
    assert not np.any(rows == 7)                                                   # the zero row scores 0
    ms, splits = dx.last_timing()
    assert ms > 0 and splits >= 1


@pytest.mark.gpu
def test_dense_range_prefix_equals_topk_bit_for_bit(case):
    dx, C, Q, oracle = case
    k = 32

    def check(s_top, r_top, res):
        indptr, rows, scores = res
        for q in range(len(s_top)):
            m = int(np.sum((r_top[q] >= 0) & (s_top[q] >= np.float32(thr))))
            seg = slice(indptr[q], indptr[q + 1])
            assert indptr[q + 1] - indptr[q] >= m
            np.testing.assert_array_equal(rows[seg][:m], r_top[q, :m])
            np.testing.assert_array_equal(scores[seg][:m].view(np.int32), s_top[q, :m].view(np.int32))
            if m < k:
                assert indptr[q + 1] - indptr[q] == m, (thr, q)

    s_top, r_top = dx.topk(Q, k)
    ss_top, rs_top = dx.selfjoin_topk(k)
    for thr in THRESHOLDS:
        check(s_top, r_top, dx.range(Q, thr))
        check(ss_top, rs_top, dx.selfjoin_range(thr))


@pytest.mark.gpu
def test_dense_range_device_queries_shards_and_exclusion(lib):
    import torch
    from kakveda_b200 import DenseIndex

    n, d, q = 3000, 128, 200
    C, Q = _clustered(n, d, q, seed=11)
    dx = DenseIndex(d)
    dx.add(C)
    dx.finalize()
    dy = DenseIndex(d, row_base=1000)
    dy.add_device(torch.from_numpy(O.bf16_round(C)).to("cuda").to(torch.bfloat16).contiguous())
    dy.finalize()
    tq = torch.from_numpy(O.bf16_round(Q)).to("cuda").to(torch.bfloat16).contiguous()
    tc = torch.from_numpy(O.bf16_round(C[:q])).to("cuda").to(torch.bfloat16).contiguous()
    thr = 0.6
    host = dx.range(Q, thr)
    # device queries give the host queries' answer; a row_base=1000 shard gives the same pairs with global rows
    for a, b in zip(dx.range_device(tq, thr), host):
        np.testing.assert_array_equal(a, b)
    indptr, rows, scores = dy.range_device(tq, thr)
    np.testing.assert_array_equal(indptr, host[0])
    np.testing.assert_array_equal(rows, host[1] + 1000)
    np.testing.assert_array_equal(scores.view(np.int32), host[2].view(np.int32))
    # exclude_base: query i loses exactly the pair (i, 1000 + i)
    full = dy.range_device(tc, thr)
    excl = dy.range_device(tc, thr, exclude_base=1000)
    removed = 0
    for i in range(q):
        fr, fs = full[1][full[0][i]:full[0][i + 1]], full[2][full[0][i]:full[0][i + 1]]
        er, es = excl[1][excl[0][i]:excl[0][i + 1]], excl[2][excl[0][i]:excl[0][i + 1]]
        keep = fr != 1000 + i
        removed += int(np.sum(~keep))
        np.testing.assert_array_equal(er, fr[keep])
        np.testing.assert_array_equal(es, fs[keep])
    assert removed == q - 1  # every row but the zero row 7 reaches the threshold against itself
    # a self-join over part of the rows is the matching slice of the full self-join
    sj = dx.selfjoin_range(thr)
    check_dense_range(*sj, O.dense_cosine(C, C), thr, excl=np.arange(n))
    lo, hi = 500, 1700
    part = dx.selfjoin_range(thr, lo, hi)
    np.testing.assert_array_equal(part[0], sj[0][lo:hi + 1] - sj[0][lo])
    np.testing.assert_array_equal(part[1], sj[1][sj[0][lo]:sj[0][hi]])
    np.testing.assert_array_equal(part[2], sj[2][sj[0][lo]:sj[0][hi]])
    sy = dy.selfjoin_range(thr)
    np.testing.assert_array_equal(sy[0], sj[0])
    np.testing.assert_array_equal(sy[1], sj[1] + 1000)
    empty = dx.selfjoin_range(thr, 40, 40)
    assert empty[0].tolist() == [0] and len(empty[1]) == 0
    dx.close()
    dy.close()


@pytest.mark.gpu
def test_dense_range_pair_buffer_growth(lib):
    from kakveda_b200 import DenseIndex

    n, d = 3000, 128
    rng = np.random.default_rng(5)
    cent = rng.standard_normal((10, d))
    C = (cent[rng.integers(0, 10, n)] + 0.05 * rng.standard_normal((n, d))).astype(np.float32)
    dx = DenseIndex(d)
    dx.add(C)
    dx.finalize()
    thr = 0.9
    first = dx.selfjoin_range(thr)
    assert len(first[1]) > 65536  # more than the buffer's initial capacity: it grew and the kernel ran again
    check_dense_range(*first, O.dense_cosine(C, C), thr, excl=np.arange(n))
    second = dx.selfjoin_range(thr)
    for a, b in zip(first, second):
        np.testing.assert_array_equal(a, b)
    dx.close()


@pytest.mark.gpu
def test_dense_patterns_on_the_threshold_graph(lib):
    from kakveda_b200 import DenseIndex, patterns

    d, n0 = 64, 300
    rng = np.random.default_rng(9)
    a = rng.standard_normal(d)
    b = a + 0.45 * rng.standard_normal(d)  # cos(A, B) about 0.9
    emb = np.concatenate([rng.standard_normal((n0, d)), np.tile(a, (40, 1)), np.tile(b, (40, 1))]).astype(np.float32)
    n = len(emb)
    rows_a, rows_b = np.arange(n0, n0 + 40), np.arange(n0 + 40, n)
    records = [{"failure_id": f"F-{i + 1:04d}", "failure_type": "TOOL_TIMEOUT" if i % 3 else "OTHER",
                "affected_apps": [f"app-{i % 5}"]} for i in range(n)]
    for i in np.concatenate([rows_a, rows_b]):
        records[i]["failure_type"] = "TOOL_TIMEOUT"
    records[rows_b[0]]["failure_type"] = "OTHER"
    dx = DenseIndex(d)
    dx.add(emb)
    dx.finalize()
    S = O.dense_cosine(emb, emb)
    cos_ab = S[rows_a[0], rows_b[0]]
    assert 0.8 < cos_ab < 0.99
    off = ~np.eye(n, dtype=bool)
    thr = _threshold_in_gap(S[off], 0.75)
    assert thr < cos_ab
    # the exact threshold graph: A and B form one pattern even though each is stored 40 > k times
    want = _components((S >= thr) & off)
    groups = {}
    for i, lab in enumerate(want):
        groups.setdefault(lab, []).append(i)
    expect = [g for _, g in sorted(groups.items()) if len({records[i]["affected_apps"][0] for i in g}) >= 2]
    out = patterns.detect_patterns(dx, records, threshold=thr, k=None)
    assert [p["rows"] for p in out] == expect
    ab = [p for p in out if rows_a[0] in p["rows"]]
    assert len(ab) == 1 and set(rows_a) | set(rows_b) <= set(ab[0]["rows"])
    # the top-k linkage sees only copies of the same embedding in every list of A and B rows
    top = patterns.detect_patterns(dx, records, threshold=thr, k=32)
    pa = [p for p in top if rows_a[0] in p["rows"]]
    pb = [p for p in top if rows_b[1] in p["rows"]]
    assert len(pa) == 1 and len(pb) == 1 and pa[0]["rows"] != pb[0]["rows"]
    # failure_type: rows of other types neither join nor bridge
    keep = np.array([r["failure_type"] == "TOOL_TIMEOUT" for r in records])
    want = _components((S >= thr) & off & keep[:, None] & keep[None, :])
    groups = {}
    for i, lab in enumerate(want):
        if keep[i]:
            groups.setdefault(lab, []).append(i)
    expect = [g for _, g in sorted(groups.items()) if len({records[i]["affected_apps"][0] for i in g}) >= 2]
    out = patterns.detect_patterns(dx, records, threshold=thr, k=None, failure_type="TOOL_TIMEOUT")
    assert [p["rows"] for p in out] == expect
    ab = [p for p in out if rows_a[0] in p["rows"]]
    assert len(ab) == 1 and rows_b[0] not in ab[0]["rows"] and set(rows_b[1:]) <= set(ab[0]["rows"])
    dx.close()


@pytest.mark.gpu
def test_dense_range_state_and_errors(lib):
    import ctypes as C
    import torch
    from kakveda_b200 import DenseIndex

    n, d, q = 1000, 64, 40
    Cm, Q = _clustered(n, d, q, seed=4)
    dx = DenseIndex(d)
    dx.add(Cm)
    dx.finalize()
    # a range call leaves the top-k answer bit for bit as it was
    s1, r1 = dx.topk(Q, 16)
    dx.range(Q, 0.5)
    s2, r2 = dx.topk(Q, 16)
    np.testing.assert_array_equal(r1, r2)
    np.testing.assert_array_equal(s1.view(np.int32), s2.view(np.int32))
    tq = torch.from_numpy(O.bf16_round(Q)).to("cuda").to(torch.bfloat16).contiguous()
    for bad in (0.0, -0.5, 1.5, float("nan")):
        with pytest.raises(ValueError):
            dx.range(Q, bad)
        with pytest.raises(ValueError):
            dx.range_device(tq, bad)
        with pytest.raises(ValueError):
            dx.selfjoin_range(bad)
    # a result is fetched once; a top-k call drops an unfetched one
    with pytest.raises(RuntimeError):
        dx._range_fetch(q, 0)
    npairs = C.c_int64(0)
    assert lib.kv_dense_selfjoin_range(dx._h, 0, n, C.c_float(0.5), C.byref(npairs)) == 0 and npairs.value > 0
    dx.topk(Q, 4)
    with pytest.raises(RuntimeError):
        dx._range_fetch(n, npairs.value)
    # row ranges outside the index
    with pytest.raises(ValueError):
        dx.selfjoin_range(0.5, 0, n + 1)
    with pytest.raises(ValueError):
        dx.selfjoin_range(0.5, 5, 3)
    # an index that is not finalized (never, or appended to since)
    dx.add(Cm[:10])
    with pytest.raises(RuntimeError):
        dx.range(Q, 0.5)
    dz = DenseIndex(d)
    dz.add(Cm)
    with pytest.raises(RuntimeError):
        dz.selfjoin_range(0.5)
    dx.close()
    dz.close()
