"""Threshold-search results on the device: the device ordering of range records (kv_*range_fetch_device, the
``device_out=True`` forms, the kv_debug_range_order hook) and connected components on the device
(kv_cluster_csr_device, ``patterns.cluster_csr`` of CUDA tensors, ``detect_patterns(k=None)``).

The host fetch orders on the device too, and ``check_range`` in the other range tests checks its order independently of
the implementation; here the device outputs must equal the host outputs bit for bit, the hook must equal NumPy's
``lexsort`` on records a real search cannot cheaply produce, and device labels must equal the host union-find."""
import ctypes as C

import numpy as np
import pytest

RANGE_REC = np.dtype([("q", "<i4"), ("score", "<f4"), ("row", "<i8")])
JACC_REC = np.dtype([("q", "<i4"), ("row", "<i4"), ("inter", "<i4"), ("uni", "<i4")])


@pytest.fixture(scope="module")
def lib(built_lib):
    from kakveda_b200 import _capi

    assert _capi.load().kv_device_count() > 0, "GPU tests need a CUDA device"
    return _capi.load()


def assert_same(host, dev):
    """Device tensors equal host arrays: dtype, shape and bits."""
    assert len(host) == len(dev)
    for h, d in zip(host, dev):
        assert d.is_cuda
        d = d.cpu().numpy()
        assert d.dtype == h.dtype and d.shape == h.shape
        assert d.tobytes() == h.tobytes()


# ---- device fetch against host fetch, per index kind ----------------------------------------------------------------

@pytest.fixture(scope="module")
def tfidf(lib):
    """20k synthetic rows at row_base 2^40 (pruned path), duplicate rows 17/18 (tied scores), 300 queries plus a null,
    an all-unseen and an irregular (> 64 features) query."""
    from kakveda_b200 import GfkbIndex, synth

    n, q = 20000, 300
    corpus, queries = synth.corpus(n), synth.queries(q, n)
    corpus[17] = "tok " * 35 + "and and and include include citations"
    corpus[18] = corpus[17]
    queries[4] = corpus[17]
    long_query = " ".join(f"w{i}x" for i in range(300)) + " " + corpus[5]
    corpus[11] = long_query
    queries += ["", "zz qq unseen", long_query]
    ix = GfkbIndex(row_base=1 << 40)
    ix.add_texts(corpus)
    ix.finalize()
    yield ix, queries
    ix.close()


@pytest.mark.gpu
def test_tfidf_device_fetch_equals_host_fetch(tfidf):
    ix, queries = tfidf
    for thr in (0.3, 0.6, 0.95):
        host = ix.range(queries, thr)
        assert host[1].min() >= 1 << 40
        assert_same(host, ix.range(queries, thr, device_out=True))
        assert_same(host, ix.range(queries, thr, device_out=True))   # the same search repeated
    q = len(queries) - 3
    assert ix.range(queries, 0.3)[0][q + 3] > ix.range(queries, 0.3)[0][q + 2]   # the irregular query has pairs
    for thr in (0.5, 0.9):
        host = ix.selfjoin_range(thr, 0, 3000)
        assert_same(host, ix.selfjoin_range(thr, 0, 3000, device_out=True))
    # null and all-unseen queries only: no pairs at all
    host = ix.range(["", "zz qq unseen"], 0.5)
    assert host[0].tolist() == [0, 0, 0]
    assert_same(host, ix.range(["", "zz qq unseen"], 0.5, device_out=True))
    assert_same(ix.range([], 0.5), ix.range([], 0.5, device_out=True))
    assert_same(ix.selfjoin_range(0.5, 5, 5), ix.selfjoin_range(0.5, 5, 5, device_out=True))


def _embeddings(rng, n, dim, centers=50):
    c = rng.standard_normal((centers, dim)).astype(np.float32)
    return (c[rng.integers(0, centers, n)] + 0.3 * rng.standard_normal((n, dim))).astype(np.float32)


@pytest.mark.gpu
def test_dense_device_fetch_equals_host_fetch(lib):
    import torch

    from kakveda_b200 import DenseIndex
    from kakveda_b200.denseindex import to_bf16_bits

    rng = np.random.default_rng(5)
    X = _embeddings(rng, 20000, 64)
    X[100:140] = X[99]                                     # duplicate rows: tied scores, ordered by row
    Q = X[rng.integers(0, 20000, 300)] + 0.05 * rng.standard_normal((300, 64)).astype(np.float32)
    Q[7] = X[99]
    dx = DenseIndex(64, row_base=123)
    dx.add(X)
    dx.finalize()
    qd = torch.from_numpy(to_bf16_bits(Q).view(np.int16)).cuda().view(torch.bfloat16)
    for thr in (0.5, 0.8, 0.95):
        host = dx.range(Q, thr)
        assert_same(host, dx.range(Q, thr, device_out=True))
        assert_same(host, dx.range_device(qd, thr, device_out=True))
        for h, g in zip(host, dx.range_device(qd, thr)):          # device queries, host outputs
            assert h.tobytes() == g.tobytes()
    for thr in (0.7, 0.95):
        host = dx.selfjoin_range(thr, 0, 4000)
        assert_same(host, dx.selfjoin_range(thr, 0, 4000, device_out=True))
    host = dx.range(Q[:4], 1.0)                            # perhaps no pair reaches 1.0 exactly
    assert_same(host, dx.range(Q[:4], 1.0, device_out=True))
    dx.close()
    # one query holding more than 65,536 pairs
    big = np.concatenate([np.repeat(X[:1], 70000, axis=0), X[1:5001]])
    bx = DenseIndex(64)
    bx.add(big)
    bx.finalize()
    host = bx.range(big[:3], 0.99)
    assert host[0][1] - host[0][0] >= 70000
    assert_same(host, bx.range(big[:3], 0.99, device_out=True))
    bx.close()


def _jaccard_data(rng, n=6000, vocab=5000):
    bases = [rng.choice(2000, int(rng.integers(8, 30)), replace=False) for _ in range(200)]

    def perturb(s):
        s = list(s[rng.random(len(s)) > 0.1]) + list(rng.integers(0, vocab, int(rng.integers(0, 3))))
        return sorted(set(int(x) for x in s))

    sets = [perturb(bases[int(rng.integers(200))]) for _ in range(n)]
    for i in range(10, 50):
        sets[i] = sets[9]                                  # duplicate rows: tied scores
    queries = [perturb(np.array(sets[int(i)])) for i in rng.integers(0, n, 150)]
    queries += [[], [vocab + 7, vocab + 9], list(range(2000, 2100)) + sets[3], sets[9]]   # null, all-OOV, irregular
    return sets, queries


@pytest.mark.gpu
def test_jaccard_device_fetch_equals_host_fetch(lib):
    from kakveda_b200 import JaccardIndex

    rng = np.random.default_rng(9)
    sets, queries = _jaccard_data(rng)
    jx = JaccardIndex(5000, row_base=10 ** 9)
    jx.add_sets(sets)
    jx.finalize()
    for thr in (0.3, 0.6, 0.9):
        host = jx.range_sets(queries, thr)
        assert host[1].min() >= 10 ** 9
        assert_same(host, jx.range_sets(queries, thr, device_out=True))
        assert_same(host, jx.range_sets(queries, thr, device_out=True))
    for thr in (0.4, 0.8):
        host = jx.selfjoin_range(thr, 0, 3000)
        assert_same(host, jx.selfjoin_range(thr, 0, 3000, device_out=True))
    host = jx.range_sets([[], [5007]], 0.5)
    assert host[0].tolist() == [0, 0, 0]
    assert_same(host, jx.range_sets([[], [5007]], 0.5, device_out=True))
    assert_same(jx.range_sets([], 0.5), jx.range_sets([], 0.5, device_out=True))
    jx.close()
    # one query holding more than 65,536 pairs
    bx = JaccardIndex(5000)
    bx.add_sets([sets[0]] * 70000 + sets[1:1001])
    bx.finalize()
    host = bx.range_sets([sets[0], sets[1]], 0.95)
    assert host[0][1] >= 70000
    assert_same(host, bx.range_sets([sets[0], sets[1]], 0.95, device_out=True))
    bx.close()


# ---- the test hook against NumPy ------------------------------------------------------------------------------------

def _hook(lib, rec, n_q, row_base=0):
    from kakveda_b200 import _capi

    jac = rec.dtype == JACC_REC
    n = len(rec)
    rec = np.ascontiguousarray(rec)
    indptr = np.empty(n_q + 1, np.int64)
    rows, scores = np.empty(max(n, 1), np.int64), np.empty(max(n, 1), np.float32)
    inter, uni = np.empty(max(n, 1), np.int32), np.empty(max(n, 1), np.int32)
    p = lambda a, t: a.ctypes.data_as(C.POINTER(t))
    _capi.check(lib.kv_debug_range_order(0, int(jac), rec.ctypes.data, n, n_q, row_base, p(indptr, C.c_int64),
                                         p(rows, C.c_int64), p(scores, C.c_float), p(inter, C.c_int32), p(uni, C.c_int32)))
    out = (indptr, rows[:n], scores[:n])
    return out + ((inter[:n], uni[:n]) if jac else ())


def _expect(rec, n_q, row_base=0):
    jac = rec.dtype == JACC_REC
    q = rec["q"].astype(np.int64)
    if jac:
        scores = rec["inter"].astype(np.float32) / rec["uni"].astype(np.float32)
        rows = rec["row"].astype(np.int64) + row_base
    else:
        scores, rows = rec["score"], rec["row"]
    order = np.lexsort((rows, -scores, q))
    indptr = np.searchsorted(q[order], np.arange(n_q + 1), side="left").astype(np.int64)
    out = (indptr, rows[order], scores[order].astype(np.float32))
    return out + ((rec["inter"][order], rec["uni"][order]) if jac else ())


def _check_hook(lib, rec, n_q, row_base=0):
    got, want = _hook(lib, rec, n_q, row_base), _expect(rec, n_q, row_base)
    for g, w in zip(got, want):
        assert g.dtype == w.dtype and g.shape == w.shape
        assert g.tobytes() == w.tobytes()
    return got


def _range_records(rng, n, n_q, scores, rows):
    rec = np.empty(n, RANGE_REC)
    rec["q"] = rng.integers(0, n_q, n) if np.isscalar(n_q) else n_q
    rec["score"], rec["row"] = scores, rows
    return rec


@pytest.mark.gpu
def test_debug_range_order_matches_lexsort(lib):
    rng = np.random.default_rng(3)
    n = 300_000
    # all scores equal: the row decides
    _check_hook(lib, _range_records(rng, n, 1000, np.float32(0.7), rng.permutation(n)), 1000)
    # scores one ulp apart
    ulp = (np.float32(0.8).view(np.int32) + rng.integers(0, 4, n).astype(np.int32)).view(np.float32)
    _check_hook(lib, _range_records(rng, n, 500, ulp, rng.permutation(n) + (1 << 40)), 500)
    # one query holding 5M pairs
    m = 5_000_000
    rec = np.empty(m, RANGE_REC)
    rec["q"] = 1
    rec["score"] = (0.5 + 0.5 * rng.random(m)).astype(np.float32)
    rec["row"] = rng.permutation(m)
    indptr = _check_hook(lib, rec, 3)[0]
    assert indptr.tolist() == [0, 0, m, m]
    # 2^20 queries with 0-1 pairs
    nq = 1 << 20
    qs = rng.choice(nq, 600_000, replace=False)
    rec = _range_records(rng, len(qs), qs.astype(np.int32), rng.random(len(qs)).astype(np.float32) + 0.1,
                         rng.integers(0, 10 ** 7, len(qs)))
    _check_hook(lib, rec, nq)
    # rows spanning [0, 2^31 - 1), random scores
    rows = rng.integers(0, (1 << 31) - 1, n)
    rows[:2] = (0, (1 << 31) - 2)
    _check_hook(lib, _range_records(rng, n, 64, (0.3 + 0.7 * rng.random(n)).astype(np.float32), rows), 64)
    # tiny inputs: nothing, one record, one record out of many queries
    _check_hook(lib, np.empty(0, RANGE_REC), 5)
    _check_hook(lib, _range_records(rng, 1, 4, np.float32(0.9), 7), 4)
    _check_hook(lib, np.empty(0, RANGE_REC), 0)


@pytest.mark.gpu
def test_debug_range_order_jaccard_matches_lexsort(lib):
    rng = np.random.default_rng(4)
    n = 400_000
    rec = np.empty(n, JACC_REC)
    rec["q"] = rng.integers(0, 300, n)
    # large unions: many distinct quotients round to the same float32, and exact equal fractions (k / 3k)
    uni = rng.integers(10_000_000, 16_000_000, n)
    inter = (uni * (0.9 + 0.1 * rng.random(n))).astype(np.int64)
    k = rng.integers(1, 5_000_000, n // 4)
    uni[: n // 4], inter[: n // 4] = 3 * k, k
    rec["uni"], rec["inter"] = uni, np.minimum(inter, uni)
    rows = rng.integers(0, (1 << 31) - 1, n)
    rows[:2] = (0, (1 << 31) - 2)
    rec["row"] = rows
    scores = rec["inter"].astype(np.float32) / rec["uni"].astype(np.float32)
    assert len(np.unique(scores)) < len(np.unique(rec["inter"].astype(np.int64) * (1 << 25) + rec["uni"]))   # collisions
    _check_hook(lib, rec, 300, row_base=10 ** 9)
    # small counts: many exact ties
    rec["uni"] = rng.integers(1, 40, n)
    rec["inter"] = rng.integers(0, 40, n) % (rec["uni"] + 1)
    _check_hook(lib, rec, 300)


@pytest.mark.gpu
def test_debug_range_order_rejects_bad_records(lib):
    rec = np.zeros(3, RANGE_REC)
    rec["score"] = 0.5
    rec["q"] = (0, 1, 5)
    with pytest.raises(ValueError):
        _hook(lib, rec, 3)                                 # query outside 0..n_q-1
    j = np.zeros(2, JACC_REC)
    j["uni"] = (3, 0)
    with pytest.raises(ValueError):
        _hook(lib, j, 1)                                   # union 0


# ---- device clustering against host clustering ---------------------------------------------------------------------

def _both(indptr, rows, full_rows=None):
    """cluster_csr of NumPy arrays and of the same data as CUDA tensors: equal labels and counts."""
    import torch

    from kakveda_b200 import patterns

    want, wc = patterns.cluster_csr(indptr, rows if full_rows is None else full_rows)
    src = rows if full_rows is None else full_rows
    got, gc = patterns.cluster_csr(torch.from_numpy(indptr).cuda(), torch.from_numpy(np.ascontiguousarray(src)).cuda())
    assert got.is_cuda and got.dtype == torch.int64
    np.testing.assert_array_equal(got.cpu().numpy(), want)
    assert gc == wc
    return want


@pytest.mark.gpu
def test_cluster_csr_device_random_graphs(lib):
    rng = np.random.default_rng(11)
    for n, deg in ((1, 0), (50, 1), (400, 3), (2000, 2), (200_000, 3)):
        lengths = rng.integers(0, 2 * deg + 1, n)
        indptr = np.zeros(n + 1, np.int64)
        np.cumsum(lengths, out=indptr[1:])
        rows = rng.integers(-3, n, int(indptr[-1])).astype(np.int64)
        _both(indptr, rows)


@pytest.mark.gpu
def test_cluster_csr_device_deep_and_wide(lib):
    n = 1_000_000
    # a path listed forwards (i -> i+1) and backwards (i -> i-1): trees as deep as the graph
    indptr = np.concatenate([np.arange(n, dtype=np.int64), [n - 1]])
    labels = _both(indptr, np.arange(1, n, dtype=np.int64))
    assert labels.max() == 0
    indptr = np.concatenate([[0], np.arange(n, dtype=np.int64)])
    _both(indptr, np.arange(0, n - 1, dtype=np.int64))
    # a star: the last vertex lists every other one
    indptr = np.zeros(n + 1, np.int64)
    indptr[n] = n - 1
    labels = _both(indptr, np.arange(n - 1, dtype=np.int64)[::-1].copy())
    assert labels.max() == 0
    # two interleaved paths (even and odd vertices) listed backwards
    rows = np.arange(n, dtype=np.int64) - 2
    _both(np.arange(n + 1, dtype=np.int64), rows)


@pytest.mark.gpu
def test_cluster_csr_device_edge_cases(lib):
    import torch

    from kakveda_b200 import patterns

    # one-directional edges, self-loops and negative rows
    indptr = np.array([0, 2, 2, 4, 5, 5, 6], np.int64)
    rows = np.array([3, 0, -1, 2, 5, -7], np.int64)
    _both(indptr, rows)
    # indptr[0] > 0: rows are indexed absolutely; the rows before indptr[0] are never read (they would be invalid)
    full = np.array([10 ** 9, -5, 10 ** 9, 1, 4, 0, 3, 2], np.int64)
    indptr = np.array([3, 4, 5, 6, 8, 8], np.int64)
    _both(indptr, None, full_rows=full)
    # n = 0
    labels, count = patterns.cluster_csr(torch.zeros(1, dtype=torch.int64, device="cuda"),
                                         torch.zeros(0, dtype=torch.int64, device="cuda"))
    assert labels.numel() == 0 and count == 0
    labels, count = patterns.cluster_csr(torch.tensor([5], dtype=torch.int64, device="cuda"),
                                         torch.zeros(0, dtype=torch.int64, device="cuda"))
    assert count == 0
    # no edges at all
    _both(np.zeros(9, np.int64), np.zeros(0, np.int64))
    # row >= n and a non-monotone indptr: ValueError, as on the host
    cuda = lambda a: torch.tensor(a, dtype=torch.int64, device="cuda")
    with pytest.raises(ValueError):
        patterns.cluster_csr(cuda([0, 1]), cuda([1]))
    with pytest.raises(ValueError):
        patterns.cluster_csr(cuda([0, 2, 1, 3]), cuda([0, 1, 2]))
    with pytest.raises(ValueError):
        patterns.cluster_csr(cuda([0, 1, 1]).to(torch.int32), cuda([1]))            # wrong dtype
    with pytest.raises(ValueError):
        patterns.cluster_csr(cuda([0, 1, 1]), np.array([1], np.int64))               # one on the host


# ---- errors ---------------------------------------------------------------------------------------------------------

@pytest.mark.gpu
def test_device_entry_points_reject_bad_pointers(tfidf, lib):
    import torch

    from kakveda_b200 import DenseIndex, JaccardIndex, _capi

    ix, queries = tfidf
    fb = ix.vocab.featurize(queries[:20], grow=False)
    ix.upload_queries(fb)
    n = C.c_int64(0)
    _capi.check(lib.kv_range_resident(ix._h, C.c_float(0.3), C.byref(n)))
    assert n.value > 0
    host = [np.empty(21, np.int64), np.empty(n.value, np.int64), np.empty(n.value, np.float32)]
    dev = [torch.empty(21, dtype=torch.int64, device="cuda"), torch.empty(n.value, dtype=torch.int64, device="cuda"),
           torch.empty(n.value, dtype=torch.float32, device="cuda")]
    vp = lambda a: C.c_void_p(a.ctypes.data if isinstance(a, np.ndarray) else a.data_ptr())
    for i in range(3):                                     # a host array in any position
        args = [vp(d) for d in dev]
        args[i] = vp(host[i])
        with pytest.raises(ValueError):
            _capi.check(lib.kv_range_fetch_device(ix._h, *args))
    spare = torch.empty(n.value + 1, dtype=torch.int64, device="cuda")
    with pytest.raises(ValueError):                        # misaligned rows
        _capi.check(lib.kv_range_fetch_device(ix._h, vp(dev[0]), C.c_void_p(spare.data_ptr() + 4), vp(dev[2])))
    with pytest.raises(ValueError):                        # the Jaccard fetch on a TF-IDF index
        _capi.check(lib.kv_jaccard_range_fetch_device(ix._h, *[vp(d) for d in dev], vp(dev[2]), vp(dev[2])))
    # rejected calls leave the result: the fetch still works, once
    _capi.check(lib.kv_range_fetch_device(ix._h, *[vp(d) for d in dev]))
    assert int(dev[0][-1]) == n.value
    with pytest.raises(RuntimeError):
        _capi.check(lib.kv_range_fetch_device(ix._h, *[vp(d) for d in dev]))
    # a re-upload drops the result
    _capi.check(lib.kv_range_resident(ix._h, C.c_float(0.3), C.byref(n)))
    ix.upload_queries(fb)
    fb.close()
    with pytest.raises(RuntimeError):
        _capi.check(lib.kv_range_fetch_device(ix._h, *[vp(d) for d in dev]))

    # Jaccard: the TF-IDF fetch on a Jaccard index, host pointers, a re-upload
    jx = JaccardIndex(64)
    jx.add_sets([[1, 2, 3], [1, 2, 3, 4], [5, 6]])
    jx.finalize()
    jx.range_sets([[1, 2, 3]], 0.5)
    _capi.check(lib.kv_selfjoin_upload(jx._h, 0, 3))
    _capi.check(lib.kv_jaccard_range_resident(jx._h, C.c_float(0.5), C.byref(n)))
    assert n.value == 2
    jd = [torch.empty(4, dtype=torch.int64, device="cuda"), torch.empty(2, dtype=torch.int64, device="cuda"),
          torch.empty(2, dtype=torch.float32, device="cuda"), torch.empty(2, dtype=torch.int32, device="cuda"),
          torch.empty(2, dtype=torch.int32, device="cuda")]
    with pytest.raises(ValueError):
        _capi.check(lib.kv_range_fetch_device(jx._h, *[vp(d) for d in jd[:3]]))
    with pytest.raises(ValueError):
        _capi.check(lib.kv_jaccard_range_fetch_device(jx._h, *[vp(d) for d in jd[:4]], vp(np.empty(2, np.int32))))
    _capi.check(lib.kv_selfjoin_upload(jx._h, 0, 3))
    with pytest.raises(RuntimeError):
        _capi.check(lib.kv_jaccard_range_fetch_device(jx._h, *[vp(d) for d in jd]))
    jx.close()

    # dense: host pointers, and a top-k call drops the result
    dx = DenseIndex(64)
    X = _embeddings(np.random.default_rng(1), 500, 64)
    dx.add(X)
    dx.finalize()
    _capi.check(lib.kv_dense_selfjoin_range(dx._h, 0, 500, C.c_float(0.5), C.byref(n)))
    dd = [torch.empty(501, dtype=torch.int64, device="cuda"), torch.empty(n.value, dtype=torch.int64, device="cuda"),
          torch.empty(n.value, dtype=torch.float32, device="cuda")]
    with pytest.raises(ValueError):
        _capi.check(lib.kv_dense_range_fetch_device(dx._h, vp(np.empty(501, np.int64)), vp(dd[1]), vp(dd[2])))
    dx.topk(X[:2], 4)
    with pytest.raises(RuntimeError):
        _capi.check(lib.kv_dense_range_fetch_device(dx._h, *[vp(d) for d in dd]))
    dx.close()

    # clustering: host pointers and a misaligned labels buffer
    ip, rr = np.array([0, 1, 1], np.int64), np.array([1], np.int64)
    with pytest.raises(ValueError):
        _capi.check(lib.kv_cluster_csr_device(0, 2, vp(ip), vp(rr), vp(np.empty(2, np.int64)), None))
    ipd, rrd = torch.from_numpy(ip).cuda(), torch.from_numpy(rr).cuda()
    with pytest.raises(ValueError):
        _capi.check(lib.kv_cluster_csr_device(0, 2, vp(ipd), vp(rr), vp(torch.empty(2, dtype=torch.int64, device="cuda")),
                                              None))
    lab = torch.empty(3, dtype=torch.int64, device="cuda")
    with pytest.raises(ValueError):
        _capi.check(lib.kv_cluster_csr_device(0, 2, vp(ipd), vp(rrd), C.c_void_p(lab.data_ptr() + 4), None))
    _capi.check(lib.kv_cluster_csr_device(0, 2, vp(ipd), vp(rrd), vp(lab), None))
    assert lab[:2].tolist() == [0, 0]


# ---- end to end -----------------------------------------------------------------------------------------------------

def _patterns_on_host(index, records, thr, failure_type=None, min_apps=2):
    """detect_patterns(k=None) computed from the host-fetched CSR and the host union-find."""
    from kakveda_b200 import patterns

    n = len(records)
    keep = np.ones(n, bool)
    if failure_type is not None:
        keep = np.array([r.get("failure_type") == failure_type for r in records])
    indptr, rows = index.selfjoin_range(thr)[:2]
    if failure_type is not None:
        src = np.repeat(np.arange(n), np.diff(indptr))
        rows = np.where(keep[src] & keep[rows], rows, -1)
    labels, _ = patterns.cluster_csr(indptr, rows)
    groups = {}
    for i, lab in enumerate(labels.tolist()):
        if keep[i]:
            groups.setdefault(lab, []).append(i)
    out = []
    for lab in sorted(groups):
        p = patterns.pattern_payload(f"pattern-{lab:06d}", [records[i] for i in groups[lab]])
        if len(p["affected_apps"]) >= min_apps:
            p["rows"] = groups[lab]
            out.append(p)
    return out


@pytest.mark.gpu
def test_detect_patterns_on_the_device_equals_host(lib):
    from kakveda_b200 import DenseIndex, GfkbIndex, JaccardIndex, patterns, synth

    rng = np.random.default_rng(21)
    n = 1200
    records = [{"failure_id": f"F-{i:05d}", "failure_type": "A" if i % 3 else "B", "affected_apps": [f"app-{i % 7}"]}
               for i in range(n)]
    corpus = synth.corpus(n // 2) * 2
    tx = GfkbIndex()
    tx.add_texts(corpus)
    tx.set_mode(2)
    tx.finalize()
    dx = DenseIndex(64)
    dx.add(_embeddings(rng, n, 64, centers=30))
    dx.finalize()
    jx = JaccardIndex(5000)
    jx.add_sets(_jaccard_data(rng, n=n)[0])
    jx.finalize()
    for index, thr in ((tx, 0.6), (dx, 0.9), (jx, 0.5)):
        for ft in (None, "A"):
            want = _patterns_on_host(index, records, thr, ft)
            got = patterns.detect_patterns(index, records, threshold=thr, k=None, failure_type=ft)
            assert got == want
            assert len(want) > 1
    for index in (tx, dx, jx):
        index.close()
