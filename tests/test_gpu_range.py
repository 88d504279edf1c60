"""Threshold search (kv_range_resident / kv_range_fetch, GfkbIndex.range*) and clustering on the exact threshold graph
(kv_cluster_csr, detect_patterns(k=None)).

Scores are the float32 values the top-k path reports (rtol 1e-5 against the float64 oracle).  A pair is required when
its float64 score clears the threshold by more than that band, and may only be returned when it lies above the band's
lower edge."""
import numpy as np
import pytest

from oracle import tfidf_oracle as O

RTOL32 = 1e-5
BAND = 2e-5
THRESHOLDS = (0.3, 0.6, 0.8, 0.95)


@pytest.fixture(scope="module")
def lib(built_lib):
    from kakveda_b200 import _capi

    assert _capi.load().kv_device_count() > 0, "GPU tests need a CUDA device"
    return _capi.load()


def check_range(indptr, rows, scores, oracle, thr, excl=None):
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
        np.testing.assert_allclose(s, o[r], rtol=RTOL32, atol=1e-7)
        assert np.all(o[r] >= thr * (1 - BAND)), (q, o[r].min())
        want = np.nonzero(o >= thr * (1 + BAND))[0]
        if excl is not None and excl[q] >= 0:
            assert excl[q] not in r
            want = want[want != excl[q]]
        assert np.isin(want, r).all(), (q, np.setdiff1d(want, r)[:5])


@pytest.fixture(scope="module")
def medium(lib):
    """20k synthetic rows (pruned path), rows 17/18 with tf overflow, 300 queries plus a null, an all-unseen and an
    irregular (> 64 features) query."""
    from kakveda_b200 import GfkbIndex, synth

    n, q = 20000, 300
    corpus, queries = synth.corpus(n), synth.queries(q, n)
    corpus[17] = "tok " * 35 + "and and and include include citations"
    corpus[18] = corpus[17]
    queries[3] = "tok tok tok and and include citations citations"
    queries[4] = corpus[17]
    long_query = " ".join(f"w{i}x" for i in range(300)) + " " + corpus[5]
    corpus[11] = long_query
    queries += ["", "zz qq unseen", long_query]
    ix = GfkbIndex()
    ix.add_texts(corpus)
    ix.finalize()
    assert ix.layout()["chunks"] >= 512
    return ix, corpus, queries, O.score_matrix_closed_form(queries, corpus)


@pytest.mark.gpu
@pytest.mark.parametrize("thr", THRESHOLDS)
def test_range_vs_float64_oracle(medium, thr):
    ix, corpus, queries, oracle = medium
    indptr, rows, scores = ix.range(queries, thr)
    check_range(indptr, rows, scores, oracle, thr)
    q = len(queries) - 3
    assert indptr[q + 1] == indptr[q] and indptr[q + 2] == indptr[q + 1]  # null and all-unseen queries: nothing
    assert indptr[q + 3] > indptr[q + 2] and rows[indptr[q + 2]] == 11      # the irregular query finds itself
    lay = ix.layout()
    assert 0 < lay["pairs_passed_bound"] and lay["pairs_scored"] >= lay["pairs_passed_bound"]
    ms = ix.last_kernel_ms()
    assert ms[0] == 0 and ms[1] == 0 and ms[2] > 0 and ms[3] > 0 and ms[4] > 0


@pytest.mark.gpu
def test_range_prefix_equals_topk_bit_for_bit(medium):
    ix, corpus, queries, oracle = medium
    k = 32
    s_top, r_top = ix.topk(queries, k)
    for thr in THRESHOLDS:
        indptr, rows, scores = ix.range(queries, thr)
        for q in range(len(queries)):
            m = int(np.sum((r_top[q] >= 0) & (s_top[q] >= np.float32(thr))))
            seg = slice(indptr[q], indptr[q + 1])
            assert indptr[q + 1] - indptr[q] >= m
            np.testing.assert_array_equal(rows[seg][:m], r_top[q, :m])
            np.testing.assert_array_equal(scores[seg][:m].view(np.int32), s_top[q, :m].view(np.int32))
            if m < k:
                assert indptr[q + 1] - indptr[q] == m, (thr, q)


@pytest.mark.gpu
def test_range_pruned_equals_exhaustive(lib, monkeypatch):
    from kakveda_b200 import GfkbIndex, synth

    n, q = 300_000, 3000
    buf, off = synth.signatures_packed(synth.CORPUS_SEED, 0, n)
    ix = GfkbIndex()
    fb = ix.vocab.featurize_packed(buf, off, 0, grow=True)
    ix.add_features(fb)
    fb.close()
    ix.finalize()
    queries = synth.queries(q, n)
    for thr in (0.5, 0.8):
        pruned = ix.range(queries, thr)
        lay = ix.layout()
        assert 0 < lay["pairs_passed_bound"] < 0.2 * q * lay["chunks"], lay
        monkeypatch.setenv("KAKVEDA_B200_NO_PRUNE", "1")
        full = ix.range(queries, thr)
        assert ix.layout()["pairs_passed_bound"] == 0
        monkeypatch.delenv("KAKVEDA_B200_NO_PRUNE")
        for a, b in zip(pruned, full):
            assert a.tobytes() == b.tobytes()
        assert len(pruned[1]) > 0


@pytest.mark.gpu
def test_range_result_larger_than_initial_buffer(lib):
    from kakveda_b200 import GfkbIndex, synth

    text = "vendored parser crashed on malformed yaml manifest during nightly deploy"
    corpus = synth.corpus(20000)
    copies = np.arange(3000) * 6 + 5
    for r in copies:
        corpus[r] = text
    ix = GfkbIndex()
    ix.add_texts(corpus)
    ix.finalize()
    queries = [text] * 100
    first = ix.range(queries, 0.99)
    indptr, rows, scores = first
    assert indptr[-1] == 100 * 3000 > 65536
    for q in range(100):
        seg = slice(indptr[q], indptr[q + 1])
        np.testing.assert_array_equal(rows[seg], copies)
        assert len(np.unique(scores[seg])) == 1 and scores[indptr[q]] == pytest.approx(1.0, rel=1e-6)
    again = ix.range(queries, 0.99)
    for a, b in zip(first, again):
        np.testing.assert_array_equal(a, b)


def _threshold_in_gap(values, near):
    """A threshold between two consecutive distinct values, at least 1e-3 apart, close above `near`."""
    allv = np.unique(values)
    i = int(np.searchsorted(allv, near))
    while allv[i] - allv[i - 1] < 1e-3:
        i += 1
    return float((allv[i] + allv[i - 1]) / 2)


def _components(adj):
    """labels[i] = smallest member of i's component of the undirected graph adj (bool [n, n])."""
    from scipy.sparse import csr_matrix
    from scipy.sparse.csgraph import connected_components

    _, lab = connected_components(csr_matrix(adj), directed=False)
    smallest = {}
    for i, l in enumerate(lab):
        smallest.setdefault(l, i)
    return np.array([smallest[l] for l in lab])


@pytest.mark.gpu
def test_selfjoin_range_and_patterns_on_the_threshold_graph(lib):
    from kakveda_b200 import GfkbIndex, patterns, synth

    a_text = "checkout service timed out waiting for inventory lock after retry budget exhausted"
    b_text = a_text + " twice"
    n0 = 600
    corpus = synth.corpus(n0) + [a_text] * 40 + [b_text] * 40
    n = len(corpus)
    rows_a, rows_b = np.arange(n0, n0 + 40), np.arange(n0 + 40, n)
    records = [{"failure_id": f"F-{i + 1:04d}", "failure_type": "HALLUCINATION_CITATION" if i % 3 else "OTHER",
                "affected_apps": [f"app-{i % 5}"], "signature_text": t} for i, t in enumerate(corpus)]
    for i in np.concatenate([rows_a, rows_b]):
        records[i]["failure_type"] = "HALLUCINATION_CITATION"
    ix = GfkbIndex()
    ix.add_texts(corpus)
    ix.set_mode(2)
    ix.finalize()
    S = O.corpus_fit_scores(corpus, corpus)
    cos_ab = S[rows_a[0], rows_b[0]]
    assert 0.8 < cos_ab < 0.99
    off = ~np.eye(n, dtype=bool)
    thr = _threshold_in_gap(S[off], 0.75)
    assert thr < cos_ab
    indptr, rows, scores = ix.selfjoin_range(thr)
    src = np.repeat(np.arange(n), np.diff(indptr))
    assert not np.any(rows == src)                     # a row never matches itself
    check_range(indptr, rows, scores, S, thr, excl=np.arange(n))
    # the exact threshold graph: A and B (cos >= thr) form one pattern even though each text is stored 40 > k times
    want = _components((S >= thr) & off)
    out = patterns.detect_patterns(ix, records, threshold=thr, k=None)
    groups = {}
    for i, lab in enumerate(want):
        groups.setdefault(lab, []).append(i)
    expect = [g for _, g in sorted(groups.items()) if len({records[i]["affected_apps"][0] for i in g}) >= 2]
    assert [p["rows"] for p in out] == expect
    ab = [p for p in out if rows_a[0] in p["rows"]]
    assert len(ab) == 1 and set(rows_b) <= set(ab[0]["rows"])
    # the top-k linkage sees only copies of the same text in every list of A and B rows
    top = patterns.detect_patterns(ix, records, threshold=thr, k=32)
    pa = [p for p in top if rows_a[0] in p["rows"]]
    pb = [p for p in top if rows_b[0] in p["rows"]]
    assert len(pa) == 1 and len(pb) == 1 and pa[0]["rows"] != pb[0]["rows"]
    # failure_type: rows of other types neither join nor bridge
    keep = np.array([r["failure_type"] == "HALLUCINATION_CITATION" for r in records])
    want = _components((S >= thr) & off & keep[:, None] & keep[None, :])
    groups = {}
    for i, lab in enumerate(want):
        if keep[i]:
            groups.setdefault(lab, []).append(i)
    expect = [g for _, g in sorted(groups.items()) if len({records[i]["affected_apps"][0] for i in g}) >= 2]
    out = patterns.detect_patterns(ix, records, threshold=thr, k=None, failure_type="HALLUCINATION_CITATION")
    assert [p["rows"] for p in out] == expect


@pytest.mark.gpu
def test_range_leaves_the_batch_state_alone(medium):
    ix, corpus, queries, oracle = medium
    fb = ix.vocab.featurize(queries, grow=False)
    n_q = fb.n
    ix.upload_queries(fb)
    s1, r1 = ix.topk_resident_host(n_q, 16)
    g1 = ix._range_resident(n_q, 0.6)
    g2 = ix._range_resident(n_q, 0.6)
    s2, r2 = ix.topk_resident_host(n_q, 16)
    fb.close()
    np.testing.assert_array_equal(r1, r2)
    np.testing.assert_array_equal(s1.view(np.int32), s2.view(np.int32))
    for a, b in zip(g1, g2):
        np.testing.assert_array_equal(a, b)
    # exclusions are honoured: query q = corpus row q must not return row q
    fb = ix.vocab.featurize(corpus[:50], grow=False)
    ix.upload_queries(fb)
    ix.set_exclusions(np.arange(50))
    indptr, rows, scores = ix._range_resident(50, 0.6)
    plain = ix.range_features(fb, 0.6)
    fb.close()
    for q in range(50):
        got = rows[indptr[q]:indptr[q + 1]]
        want = plain[1][plain[0][q]:plain[0][q + 1]]
        assert q not in got
        np.testing.assert_array_equal(got, want[want != q])


@pytest.mark.gpu
def test_range_errors_and_fetch_outputs(medium):
    from kakveda_b200 import GfkbIndex, _capi

    ix, corpus, queries, oracle = medium
    for bad in (0.0, -1.0, 1.5, float("nan")):
        with pytest.raises(ValueError):
            ix.range(queries[:4], bad)
    fresh = GfkbIndex()
    fresh.add_texts(corpus[:100])
    fresh.finalize()
    with pytest.raises(RuntimeError):
        fresh._range_resident(1, 0.5)                     # no resident batch
    jac = GfkbIndex()
    jac.add_texts(["alpha beta gamma", "beta gamma delta", "epsilon zeta"])
    jac.set_mode(1)
    jac.finalize()
    with pytest.raises(ValueError):
        jac.range(["alpha beta"], 0.5)
    # the result belongs to the batch it was computed for
    import ctypes as C

    fb = ix.vocab.featurize(queries[:8], grow=False)
    ix.upload_queries(fb)
    n = C.c_int64(0)
    _capi.check(_capi.load().kv_range_resident(ix._h, C.c_float(0.5), C.byref(n)))
    ix.upload_queries(fb)
    fb.close()
    indptr = np.empty(9, np.int64)
    rows, scores = np.empty(max(n.value, 1), np.int64), np.empty(max(n.value, 1), np.float32)
    with pytest.raises(RuntimeError):
        _capi.check(_capi.load().kv_range_fetch(ix._h, indptr.ctypes.data_as(C.POINTER(C.c_int64)),
                                                rows.ctypes.data_as(C.POINTER(C.c_int64)),
                                                scores.ctypes.data_as(C.POINTER(C.c_float)), None, None))
    empty = GfkbIndex()
    empty.finalize()
    indptr, rows, scores = empty.range(["alpha beta", "gamma"], 0.5)
    assert indptr.tolist() == [0, 0, 0] and len(rows) == 0 and len(scores) == 0


def test_cluster_csr_matches_union_find(built_lib):
    from kakveda_b200 import patterns

    rng = np.random.default_rng(11)
    for n, deg in ((1, 0), (50, 1), (400, 3), (2000, 2)):
        lengths = rng.integers(0, 2 * deg + 1, n)
        indptr = np.zeros(n + 1, np.int64)
        np.cumsum(lengths, out=indptr[1:])
        rows = rng.integers(-3, n, int(indptr[-1])).astype(np.int64)   # rows < 0 are skipped
        labels, count = patterns.cluster_csr(indptr, rows)
        parent = list(range(n))

        def find(x):
            while parent[x] != x:
                x = parent[x]
            return x

        for i in range(n):
            for r in rows[indptr[i]:indptr[i + 1]]:
                if r >= 0:
                    a, b = find(i), find(int(r))
                    if a != b:
                        parent[max(a, b)] = min(a, b)
        want = [find(i) for i in range(n)]
        np.testing.assert_array_equal(labels, want)
        assert count == len(set(want))
    with pytest.raises(ValueError):
        patterns.cluster_csr(np.array([0, 1], np.int64), np.array([1], np.int64))   # row >= n
