"""Jaccard threshold search (kv_range_resident / kv_range_fetch on a Jaccard index, JaccardIndex.range_* and
selfjoin_*) and pattern clustering of token sets on the exact threshold graph (detect_patterns(JaccardIndex, k=None)).

The oracle is exact: (|q ∩ r|, |q ∪ r|) from ``oracle.tfidf_oracle.jaccard_sets`` (a scipy product of the binary
set matrices gives the same integers for all pairs at once), a pair is returned iff union > 0 and
float32(inter / union) >= float32(threshold), and its score is that float32 bit for bit.  For |∪| < 2^24 the float64
quotient rounded to float32 is the correctly rounded float32 quotient, so the device's __fdiv_rn, the float64 scan
of irregular queries and this oracle all agree."""
import ctypes as C

import numpy as np
import pytest

from oracle import tfidf_oracle as O
from test_gpu_range import _components

THRESHOLDS = (0.3, 0.6, 0.9)


@pytest.fixture(scope="module")
def lib(built_lib):
    from kakveda_b200 import _capi

    assert _capi.load().kv_device_count() > 0, "GPU tests need a CUDA device"
    return _capi.load()


def _binary(sets, width):
    from scipy.sparse import csr_matrix

    indptr = np.concatenate([[0], np.cumsum([len(s) for s in sets])]).astype(np.int64)
    ids = np.concatenate([np.asarray(s, np.int64) for s in sets]) if indptr[-1] else np.zeros(0, np.int64)
    return csr_matrix((np.ones(len(ids), np.int64), ids, indptr), shape=(len(sets), width))


def exact_counts(queries, rows):
    """(inter, union) int64 [Q, N] of every (query, row) pair: the integers jaccard_sets gives."""
    width = 1 + max([int(s.max()) for s in list(queries) + list(rows) if len(s)] + [0])
    inter = (_binary(queries, width) @ _binary(rows, width).T).toarray()
    nq = np.array([len(s) for s in queries], np.int64)
    nr = np.array([len(s) for s in rows], np.int64)
    return inter, nq[:, None] + nr[None, :] - inter


def score32(inter, union):
    return np.where(union > 0, inter / np.maximum(union, 1), 0.0).astype(np.float32)


def check_exact(res, queries, rows, inter_all, union_all, thr, excl=None, n_check=40):
    """res: (indptr, rows, scores, inter, union) of a range result against the exact counts."""
    indptr, rr, ss, ii, uu = res
    Q = len(queries)
    assert indptr.shape == (Q + 1,) and indptr[0] == 0 and np.all(np.diff(indptr) >= 0)
    assert indptr[-1] == len(rr) == len(ss) == len(ii) == len(uu)
    assert rr.dtype == np.int64 and ss.dtype == np.float32 and ii.dtype == np.int32 and uu.dtype == np.int32
    S = score32(inter_all, union_all)
    t = np.float32(thr)
    for q in range(Q):
        seg = slice(indptr[q], indptr[q + 1])
        r, s = rr[seg], ss[seg]
        want = np.nonzero((union_all[q] > 0) & (S[q] >= t))[0]
        if excl is not None and excl[q] >= 0:
            assert excl[q] not in r
            want = want[want != excl[q]]
        assert np.array_equal(np.sort(r), want), (q, np.setdiff1d(want, r)[:5], np.setdiff1d(r, want)[:5])
        np.testing.assert_array_equal(s.view(np.int32), S[q, r].view(np.int32))
        np.testing.assert_array_equal(ii[seg], inter_all[q, r])
        np.testing.assert_array_equal(uu[seg], union_all[q, r])
        assert np.all((s[:-1] > s[1:]) | ((s[:-1] == s[1:]) & (r[:-1] < r[1:]))), "order is not (score desc, row asc)"
    # the matrix above against the oracle itself, on the returned pairs of the first queries
    for q in range(min(Q, n_check)):
        for j in range(indptr[q], min(indptr[q + 1], indptr[q] + 8)):
            assert (int(ii[j]), int(uu[j])) == O.jaccard_sets(queries[q].tolist(), rows[int(rr[j])].tolist())


def _near(rng, base, V, swaps):
    """base with `swaps` tokens replaced by others (a planted near-duplicate)."""
    s = base.copy()
    if len(s):
        pos = rng.choice(len(s), size=min(swaps, len(s)), replace=False)
        s[pos] = rng.integers(0, V, size=len(pos), dtype=np.uint32)
    return np.unique(s)


def _sets(n, q, seed, V=1 << 14):
    """n Zipf(1.3) sets of ~40 draws with 5 % planted near-duplicates, rows 99 = 100 = 101 (ties), row 5 empty and row
    11 a 100-token set with near-duplicates in rows 12-14; queries: copies or near-copies of rows, an empty query (1),
    one with ids outside the vocabulary (2) and row 11 (3, more than 64 tokens: the float64 fallback)."""
    rng = np.random.default_rng(seed)
    zipf = lambda size: np.minimum(rng.zipf(1.3, size) - 1, V - 1).astype(np.uint32)
    rows = [np.unique(zipf(max(1, rng.poisson(40)))) for _ in range(n)]
    for i in rng.choice(np.arange(20, n), size=n // 20, replace=False):
        rows[i] = _near(rng, rows[rng.integers(0, n)], V, int(rng.integers(1, 4)))
    rows[5] = np.zeros(0, dtype=np.uint32)
    rows[100] = rows[99].copy()
    rows[101] = rows[99].copy()
    rows[11] = np.unique(rng.choice(V, size=100, replace=False).astype(np.uint32))
    for i in (12, 13, 14):
        rows[i] = _near(rng, rows[11], V, i - 11)
    queries = []
    for i in range(q):
        if i % 3 == 0:
            queries.append(np.unique(zipf(max(1, rng.poisson(40)))))
        else:
            queries.append(_near(rng, rows[rng.integers(0, n)], V, int(rng.integers(0, 5))))
    queries[0] = rows[99].copy()
    queries[1] = np.zeros(0, dtype=np.uint32)
    queries[2] = np.concatenate([rows[7], np.array([V + 5, V + 9], dtype=np.uint32)])
    queries[3] = rows[11].copy()
    return rows, queries, V


@pytest.fixture(scope="module")
def medium(lib):
    from kakveda_b200 import JaccardIndex

    rows, queries, V = _sets(6000, 160, seed=7)
    jx = JaccardIndex(V)
    jx.add_sets(rows[:3000])
    jx.add_sets(rows[3000:])
    jx.finalize()
    inter, union = exact_counts(queries, rows)
    yield jx, rows, queries, inter, union
    jx.close()


@pytest.mark.gpu
@pytest.mark.parametrize("thr", THRESHOLDS)
def test_jaccard_range_exact(medium, thr):
    jx, rows, queries, inter, union = medium
    res = jx.range_sets(queries, thr)
    check_exact(res, queries, rows, inter, union, thr)
    indptr, rr, ss, ii, uu = res
    assert indptr[1] - indptr[0] >= 3 and rr[indptr[0]:indptr[0] + 3].tolist() == [99, 100, 101]  # ties: row asc
    assert indptr[2] == indptr[1]                                   # the empty query matches nothing
    seg2 = rr[indptr[2]:indptr[3]].tolist()
    if 7 in seg2:                                                   # out-of-vocabulary ids count towards |q|
        j = indptr[2] + seg2.index(7)
        assert ii[j] == len(rows[7]) and uu[j] == len(rows[7]) + 2
    assert rr[indptr[3]] == 11 and ii[indptr[3]] == 100              # the irregular query finds itself
    if thr <= 0.9:
        assert 12 in rr[indptr[3]:indptr[4]]
    assert indptr[-1] >= 20


@pytest.mark.gpu
def test_jaccard_range_prefix_equals_topk(medium):
    jx, rows, queries, inter, union = medium
    k = 32
    s_top, r_top, i_top, u_top = jx.topk_sets(queries, k)
    for thr in THRESHOLDS:
        indptr, rr, ss, ii, uu = jx.range_sets(queries, thr)
        for q in range(len(queries)):
            m = int(np.sum((r_top[q] >= 0) & (s_top[q] >= np.float32(thr))))
            seg = slice(indptr[q], indptr[q + 1])
            assert indptr[q + 1] - indptr[q] >= m
            np.testing.assert_array_equal(rr[seg][:m], r_top[q, :m])
            np.testing.assert_array_equal(ss[seg][:m].view(np.int32), s_top[q, :m].view(np.int32))
            np.testing.assert_array_equal(ii[seg][:m], i_top[q, :m])
            np.testing.assert_array_equal(uu[seg][:m], u_top[q, :m])
            if m < k:
                assert indptr[q + 1] - indptr[q] == m, (thr, q)


@pytest.mark.gpu
def test_jaccard_selfjoin(lib):
    from kakveda_b200 import JaccardIndex

    rows, _, V = _sets(2000, 4, seed=11)
    n = len(rows)
    jx = JaccardIndex(V, row_base=0)
    jx.add_sets(rows)
    jx.finalize()
    inter, union = exact_counts(rows, rows)
    for thr in (0.3, 0.6):
        full = jx.selfjoin_range(thr)
        check_exact(full, rows, rows, inter, union, thr, excl=np.arange(n))
        indptr, rr = full[0], full[1]
        src = np.repeat(np.arange(n), np.diff(indptr))
        assert not np.any(rr == src)
        fwd = set(zip(src.tolist(), rr.tolist()))
        assert fwd == {(b, a) for a, b in fwd}                         # symmetric
        lo, hi = 700, 1300
        part = jx.selfjoin_range(thr, lo, hi)
        a, b = indptr[lo], indptr[hi]
        np.testing.assert_array_equal(part[0], indptr[lo:hi + 1] - a)
        for x, y in zip(part[1:], full[1:]):
            np.testing.assert_array_equal(x, y[a:b])
    # self-join top-k: the k best OTHER rows by (float32 score desc, row asc), with the exact counts
    k = 16
    s, r, i, u = jx.selfjoin_topk(k)
    S = score32(inter, union)
    np.fill_diagonal(S, -np.inf)
    for q in range(n):
        order = np.lexsort((np.arange(n), -S[q].astype(np.float64)))[:k]
        np.testing.assert_array_equal(r[q], order)
        np.testing.assert_array_equal(s[q].view(np.int32), S[q, order].view(np.int32))
        np.testing.assert_array_equal(i[q], inter[q, order])
        np.testing.assert_array_equal(u[q], union[q, order])
    s2, r2, i2, u2 = jx.selfjoin_topk(k, 100, 150)
    np.testing.assert_array_equal(r2, r[100:150])
    np.testing.assert_array_equal(i2, i[100:150])
    jx.close()


@pytest.mark.gpu
def test_jaccard_range_result_larger_than_initial_buffer(lib):
    from kakveda_b200 import JaccardIndex

    rng = np.random.default_rng(3)
    V = 1 << 14
    rows = [np.unique(np.minimum(rng.zipf(1.3, 40) - 1, 4095).astype(np.uint32)) for _ in range(3000)]
    target = np.arange(10000, 10030, dtype=np.uint32)  # tokens no other row holds
    copies = np.arange(300) * 10 + 3
    for c in copies:
        rows[c] = target
    jx = JaccardIndex(V)
    jx.add_sets(rows)
    jx.finalize()
    queries = [target] * 300
    first = jx.range_sets(queries, 0.9)
    indptr, rr, ss, ii, uu = first
    assert indptr[-1] == 300 * 300 > 65536
    for q in range(300):
        seg = slice(indptr[q], indptr[q + 1])
        np.testing.assert_array_equal(rr[seg], copies)
        assert np.all(ss[seg] == 1.0) and np.all(ii[seg] == 30) and np.all(uu[seg] == 30)
    again = jx.range_sets(queries, 0.9)
    for a, b in zip(first, again):
        np.testing.assert_array_equal(a, b)
    jx.close()


@pytest.mark.gpu
def test_jaccard_patterns_on_the_threshold_graph(lib):
    from kakveda_b200 import JaccardIndex, patterns

    rng = np.random.default_rng(21)
    V = 1 << 14
    a_set = np.arange(12000, 12030, dtype=np.uint32)
    b_set = np.concatenate([a_set[:-1], [12100]]).astype(np.uint32)    # J(A, B) = 29 / 31
    n0 = 600
    sets = [np.unique(np.minimum(rng.zipf(1.3, 40) - 1, 8191).astype(np.uint32)) for _ in range(n0)]
    sets += [a_set] * 40 + [b_set] * 40
    n = len(sets)
    rows_a, rows_b = np.arange(n0, n0 + 40), np.arange(n0 + 40, n)
    records = [{"failure_id": f"F-{i + 1:04d}", "failure_type": "HALLUCINATION_CITATION" if i % 3 else "OTHER",
                "affected_apps": [f"app-{i % 5}"]} for i in range(n)]
    for i in np.concatenate([rows_a, rows_b]):
        records[i]["failure_type"] = "HALLUCINATION_CITATION"
    jx = JaccardIndex(V)
    jx.add_sets(sets)
    jx.finalize()
    inter, union = exact_counts(sets, sets)
    S = score32(inter, union)
    thr = 0.9
    off = ~np.eye(n, dtype=bool)
    adj = (union > 0) & (S >= np.float32(thr)) & off
    assert adj[rows_a[0], rows_b[0]]
    want = _components(adj)
    groups = {}
    for i, lab in enumerate(want):
        groups.setdefault(lab, []).append(i)
    expect = [g for _, g in sorted(groups.items()) if len({records[i]["affected_apps"][0] for i in g}) >= 2]
    out = patterns.detect_patterns(jx, records, threshold=thr, k=None)
    assert [p["rows"] for p in out] == expect
    ab = [p for p in out if rows_a[0] in p["rows"]]
    assert len(ab) == 1 and set(rows_b) <= set(ab[0]["rows"]) and len(out) == 1
    # top-k linkage: every list of an A or B row holds only copies of the same set
    top = patterns.detect_patterns(jx, records, threshold=thr, k=32)
    pa = [p for p in top if rows_a[0] in p["rows"]]
    pb = [p for p in top if rows_b[0] in p["rows"]]
    assert len(top) == 2 and len(pa) == 1 and len(pb) == 1 and pa[0]["rows"] != pb[0]["rows"]
    # failure_type: rows of other types neither join nor bridge
    keep = np.array([r["failure_type"] == "HALLUCINATION_CITATION" for r in records])
    want = _components(adj & keep[:, None] & keep[None, :])
    groups = {}
    for i, lab in enumerate(want):
        if keep[i]:
            groups.setdefault(lab, []).append(i)
    expect = [g for _, g in sorted(groups.items()) if len({records[i]["affected_apps"][0] for i in g}) >= 2]
    out = patterns.detect_patterns(jx, records, threshold=thr, k=None, failure_type="HALLUCINATION_CITATION")
    assert [p["rows"] for p in out] == expect
    jx.close()


def _fetch(lib, h, n_q, n, counts=True):
    """kv_range_fetch with the count outputs of a Jaccard index, or (counts=False) with NULL ones as on a TF-IDF index."""
    from kakveda_b200 import _capi

    indptr = np.empty(n_q + 1, np.int64)
    rows, scores = np.empty(max(n, 1), np.int64), np.empty(max(n, 1), np.float32)
    inter, union = np.empty(max(n, 1), np.int32), np.empty(max(n, 1), np.int32)
    p = lambda a, t: a.ctypes.data_as(C.POINTER(t))
    _capi.check(lib.kv_range_fetch(h, p(indptr, C.c_int64), p(rows, C.c_int64), p(scores, C.c_float),
                                   p(inter, C.c_int32) if counts else None, p(union, C.c_int32) if counts else None))
    return indptr


@pytest.mark.gpu
def test_jaccard_range_fetch_counts_and_state(medium):
    from kakveda_b200 import GfkbIndex, JaccardIndex, _capi
    from kakveda_b200.jaccardindex import _csr

    jx, rows, queries, inter, union = medium
    lib = _capi.load()
    for bad in (0.0, -1.0, 1.5, float("nan")):
        with pytest.raises(ValueError):
            jx.range_sets(queries[:4], bad)
    # upload a batch without a search: no result to fetch
    ip, ids = _csr(queries[:8])
    tf = np.ones(len(ids), np.uint32)
    p = lambda a, t: a.ctypes.data_as(C.POINTER(t))
    upload = lambda: _capi.check(lib.kv_query_upload(jx._h, p(ip, C.c_int64), p(ids, C.c_uint32), p(tf, C.c_uint32), None, 8))
    upload()
    with pytest.raises(RuntimeError):
        _fetch(lib, jx._h, 8, 0)
    n = C.c_int64(0)
    _capi.check(lib.kv_range_resident(jx._h, C.c_float(0.5), C.byref(n)))
    assert n.value > 0
    with pytest.raises(ValueError):            # a Jaccard result is fetched with its counts
        _fetch(lib, jx._h, 8, n.value, counts=False)
    indptr = _fetch(lib, jx._h, 8, n.value)    # the rejected fetch left the result
    assert indptr[-1] == n.value
    _capi.check(lib.kv_range_resident(jx._h, C.c_float(0.5), C.byref(n)))
    upload()                                   # a new upload drops the result
    with pytest.raises(RuntimeError):
        _fetch(lib, jx._h, 8, n.value)
    _capi.check(lib.kv_range_resident(jx._h, C.c_float(0.5), C.byref(n)))
    indptr = _fetch(lib, jx._h, 8, n.value)
    assert indptr[-1] == n.value
    with pytest.raises(RuntimeError):          # fetched once
        _fetch(lib, jx._h, 8, n.value)
    # count outputs on a TF-IDF index
    tx = GfkbIndex()
    tx.add_texts(["alpha beta gamma", "beta gamma delta", "epsilon zeta"])
    tx.finalize()
    fb = tx.vocab.featurize(["alpha beta gamma"], grow=False)
    tx.upload_queries(fb)
    fb.close()
    with pytest.raises(ValueError):            # no result yet, and the outputs do not fit the mode
        _fetch(lib, tx._h, 1, 0)
    _capi.check(lib.kv_range_resident(tx._h, C.c_float(0.5), C.byref(n)))
    assert n.value > 0
    with pytest.raises(ValueError):
        _fetch(lib, tx._h, 1, n.value)
    indptr = _fetch(lib, tx._h, 1, n.value, counts=False)   # the rejected fetch left the result
    assert indptr[-1] == n.value
    tx.close()
    # an empty index: empty CSR arrays
    empty = JaccardIndex(16)
    empty.finalize()
    indptr, rr, ss, ii, uu = empty.range_sets([[1, 2], [3]], 0.5)
    assert indptr.tolist() == [0, 0, 0] and len(rr) == len(ss) == len(ii) == len(uu) == 0
    assert [len(a) for a in empty.selfjoin_range(0.5)] == [1, 0, 0, 0, 0]
    empty.close()
