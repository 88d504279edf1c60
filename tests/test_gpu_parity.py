"""Parity of the CUDA path (through the C ABI) against the oracle and the reference goldens.

Tolerances: the drop-in ``score`` path accumulates in float64 -> rtol 1e-9 against the
reference's float64 values (the contract in BASELINE.json is 1e-5 relative); the batched
top-k path accumulates in float32 -> rtol 1e-5 on scores, row sets equal up to ties that fall
inside that tolerance.
"""
import threading

import numpy as np
import pytest

from oracle import tfidf_oracle as O

pytestmark = pytest.mark.gpu

RTOL64 = 1e-9
RTOL32 = 1e-5


@pytest.fixture(scope="module")
def lib(built_lib):
    from kakveda_b200 import _capi

    assert _capi.load().kv_device_count() > 0, "GPU tests need a CUDA device"
    return _capi.load()


def check_topk(scores, rows, oracle_scores, k, rtol=RTOL32):
    """scores/rows: [Q,k] from the device; oracle_scores: [Q,N] float64."""
    oracle_scores = np.asarray(oracle_scores)
    Q, N = oracle_scores.shape
    kk = min(k, N)
    for q in range(Q):
        s, r = scores[q], rows[q]
        assert np.all(r[:kk] >= 0) and np.all(r[kk:] == -1)
        assert len(set(r[:kk].tolist())) == kk, "duplicate row in top-k"
        # ordering contract: score desc, ties -> lower row first
        for a in range(kk - 1):
            assert s[a] > s[a + 1] or (s[a] == s[a + 1] and r[a] < r[a + 1]), (q, a, s, r)
        want = oracle_scores[q, r[:kk]]
        np.testing.assert_allclose(s[:kk], want, rtol=rtol, atol=1e-7)
        # nothing outside the returned set may beat the k-th returned row by more than the tolerance
        if kk < N:
            rest = np.delete(oracle_scores[q], r[:kk])
            assert rest.max() <= want.min() * (1 + 2 * rtol) + 1e-7, (q, rest.max(), want.min())
        # exact ties in the float64 oracle (duplicate rows) must come back in ascending row order
        for a in range(kk - 1):
            if want[a] == want[a + 1] and s[a] == s[a + 1]:
                assert r[a] < r[a + 1]


def test_score_matches_reference_goldens(lib, golden):
    from kakveda_b200 import SimilarityEngine

    eng = SimilarityEngine()
    g = golden("ref_test_similarity.json")
    got = eng.score(g["query"], g["corpus"])
    assert isinstance(got, list) and isinstance(got[0], float) and len(got) == 2 and got[0] > got[1]
    np.testing.assert_allclose(got, g["scores"], rtol=RTOL64)

    g = golden("fixture54.json")
    corpus = [r["signature_text"] for r in g["records"]]
    for q, want in zip(g["queries"], g["scores"]):
        np.testing.assert_allclose(eng.score(q, corpus), want, rtol=RTOL64, atol=1e-15)

    g = golden("edge_cases.json")
    for q, want in zip(g["queries"], g["scores"]):
        np.testing.assert_allclose(eng.score(q, g["corpus"]), want, rtol=RTOL64, atol=1e-15)


def test_error_conventions(lib):
    from kakveda_b200 import SimilarityEngine

    eng = SimilarityEngine()
    assert eng.score("anything", []) == []                      # similarity.py:15-16
    with pytest.raises(ValueError, match="empty vocabulary"):   # sklearn's ValueError propagates
        eng.score("a", ["b", ""])
    assert eng.score("", ["alpha beta", ""]) == [0.0, 0.0]      # token-less query -> zeros
    assert eng.score("alpha beta", ["", "a"]) == [0.0, 0.0]     # token-less rows -> zeros


def test_gfkb_match_handler(lib, golden):
    from kakveda_b200 import SimilarityEngine, gfkb

    g = golden("fixture54.json")
    eng = SimilarityEngine()
    for case in g["match"]:
        got = gfkb.match_records(eng, case["signature_text"], g["records"], case["failure_type"])
        assert [m["failure_id"] for m in got] == [m["failure_id"] for m in case["matches"]]
        assert [m["version"] for m in got] == [m["version"] for m in case["matches"]]
        np.testing.assert_allclose([m["score"] for m in got], [m["score"] for m in case["matches"]], rtol=RTOL64)
    # batched handler form: device top-k (k=5) then the post-truncation filter
    corpus = [r["signature_text"] for r in g["records"]]
    qs = [c["signature_text"] for c in g["match"][::3]]
    scores, rows = eng.topk(qs, corpus, k=5)
    for i, case in enumerate(g["match"][::3]):
        got = gfkb.match_from_topk(g["records"], rows[i], scores[i], None)
        assert [(m["failure_id"], m["version"]) for m in got] == [(m["failure_id"], m["version"]) for m in case["matches"]]


def test_synthetic_small_full_scores(lib, golden):
    from kakveda_b200 import SimilarityEngine, synth

    g = golden("synthetic_small.json")
    corpus, queries = synth.corpus(g["n"]), synth.queries(g["q"], g["n"])
    eng = SimilarityEngine()
    for q, want in zip(queries, g["scores"]):
        np.testing.assert_allclose(eng.score(q, corpus), want, rtol=RTOL64, atol=1e-15)


@pytest.mark.parametrize("k", [5, 16, 32])
def test_cfg1_topk(lib, golden, k):
    """BASELINE configs[0]: 1k-entry GFKB, 128-query batch."""
    from kakveda_b200 import GfkbIndex, synth

    g = golden("synthetic_cfg1.json")
    corpus, queries = synth.corpus(g["n"]), synth.queries(g["q"], g["n"])
    ix = GfkbIndex()
    ix.add_texts(corpus)
    ix.finalize()
    scores, rows = ix.topk(queries, k)
    oracle = O.score_matrix_closed_form(queries, corpus)
    check_topk(scores, rows, oracle, k)
    if k == 16:
        np.testing.assert_allclose(scores, np.array(g["topk_scores"]), rtol=RTOL32)
        same = sum(int(a == b) for ra, rb in zip(rows.tolist(), g["topk_rows"]) for a, b in zip(ra, rb))
        assert same >= 0.98 * rows.size  # the rest are float32-vs-float64 near ties (checked by check_topk)
    # the float64 scan agrees with the reference's full vectors
    for i in range(4):
        np.testing.assert_allclose(ix.score(queries[i]), g["full_first8"][i], rtol=RTOL64, atol=1e-15)


def test_edge_topk_and_small_corpora(lib, golden):
    from kakveda_b200 import GfkbIndex

    g = golden("edge_cases.json")
    ix = GfkbIndex()
    ix.add_texts(g["corpus"])
    ix.finalize()
    for k in (1, 5, 16):
        scores, rows = ix.topk(g["queries"], k)
        check_topk(scores, rows, np.array(g["scores"]), k)
    # all-zero queries: the first k rows, in order (stable sort of equal keys, gfkb/app.py:89)
    s, r = ix.topk(["", "unseen words only"], 5)
    assert r.tolist() == [[0, 1, 2, 3, 4]] * 2 and np.all(s == 0)


def test_medium_vs_vectorised_oracle(lib):
    from kakveda_b200 import GfkbIndex, synth

    n, q, k = 20000, 300, 16
    corpus, queries = synth.corpus(n), synth.queries(q, n)
    # sprinkle rows/queries that exercise tf>1 on both sides and the overflow table
    corpus[17] = "tok " * 35 + "and and and include include citations"
    corpus[18] = corpus[17]
    queries[3] = "tok tok tok and and include citations citations"
    queries[4] = corpus[17]
    ix = GfkbIndex()
    ix.add_texts(corpus)
    ix.finalize()
    scores, rows = ix.topk(queries, k)
    oracle = O.score_matrix_closed_form(queries, corpus)
    check_topk(scores, rows, oracle, k)
    assert rows[4, 0] == 17 and rows[4, 1] == 18 and scores[4, 0] == pytest.approx(1.0, rel=1e-6)
    for i in (0, 3, 4, 77):
        np.testing.assert_allclose(ix.score(queries[i]), oracle[i], rtol=RTOL64, atol=1e-15)
    lay = ix.layout()
    assert lay["rows"] == n and lay["tf_overflow_entries"] >= 2   # "tok" x35 and "tok tok" x34 (rows 17, 18 share the block entries)
    clean = GfkbIndex()
    clean.add_texts(synth.corpus(5000))
    clean.finalize()
    assert clean.layout()["universal_features"] >= 4  # intent_tags, prompt_hint, tools, env_keys


def test_irregular_query_falls_back_to_full_scan(lib):
    from kakveda_b200 import GfkbIndex, synth

    n = 3000
    corpus = synth.corpus(n)
    long_query = " ".join(f"w{i}x" for i in range(1500)) + " " + corpus[5]
    corpus[11] = long_query
    queries = [corpus[7], long_query, corpus[9]]
    ix = GfkbIndex()
    ix.add_texts(corpus)
    ix.finalize()
    scores, rows = ix.topk(queries, 8)
    check_topk(scores, rows, O.score_matrix_closed_form(queries, corpus), 8)
    assert rows[1, 0] == 11


def test_append_then_finalize_equals_fresh_build(lib):
    from kakveda_b200 import SimilarityEngine, synth

    corpus = synth.corpus(4000)
    q = synth.queries(3, 4000)
    eng = SimilarityEngine()
    a1 = eng.score(q[0], corpus[:2500])
    a2 = eng.score(q[0], corpus)          # extends the cached index (append epoch, re-finalize)
    a3 = eng.score(q[1], corpus)          # cache hit
    fresh = SimilarityEngine()
    np.testing.assert_array_equal(a2, fresh.score(q[0], corpus))
    np.testing.assert_array_equal(a3, fresh.score(q[1], corpus))
    np.testing.assert_allclose(a1, O.score_matrix_closed_form([q[0]], corpus[:2500])[0], rtol=RTOL64, atol=1e-15)
    np.testing.assert_allclose(a2, O.score_matrix_closed_form([q[0]], corpus)[0], rtol=RTOL64, atol=1e-15)
    b = eng.score(q[2], corpus[:100])     # shrinking corpus -> rebuild
    np.testing.assert_allclose(b, O.score_matrix_closed_form([q[2]], corpus[:100])[0], rtol=RTOL64, atol=1e-15)


def test_sharded_resident_topk_equals_unsharded_on_one_gpu(lib):
    """Row shards with the global df + K5 merge reproduce the single-index result bit for bit."""
    import ctypes as C

    import torch

    from kakveda_b200 import GfkbIndex, Vocabulary, _capi, synth

    n, q, k, shards = 30000, 200, 16, 3
    corpus, queries = synth.corpus(n), synth.queries(q, n)
    one = GfkbIndex()
    one.add_texts(corpus)
    one.finalize()
    s1, r1 = one.topk(queries, k)

    vocab = Vocabulary()
    fb = vocab.featurize(corpus, grow=True)
    parts = []
    df = np.zeros(len(vocab), dtype=np.int64)
    for s in range(shards):
        lo, hi = n * s // shards, n * (s + 1) // shards
        ix = GfkbIndex(row_base=lo, vocab=vocab)
        ix.add_features(fb, lo, hi)
        df += ix.local_df()
        parts.append(ix)
    np.testing.assert_array_equal(df, one.local_df())
    qfb = vocab.featurize(queries, grow=False)
    ds = torch.empty((shards, q, k), dtype=torch.float32, device="cuda")
    dr = torch.empty((shards, q, k), dtype=torch.int64, device="cuda")
    for s, ix in enumerate(parts):
        ix.set_global_df(df.astype(np.uint32), n)
        ix.finalize()
        ix.upload_queries(qfb)
        ix.topk_resident(k, ds[s].data_ptr(), dr[s].data_ptr())
    out_s = torch.empty((q, k), dtype=torch.float32, device="cuda")
    out_r = torch.empty((q, k), dtype=torch.int64, device="cuda")
    _capi.check(_capi.load().kv_merge_topk_device(0, C.c_void_p(ds.data_ptr()), C.c_void_p(dr.data_ptr()), shards, q, k,
                                                  C.c_void_p(out_s.data_ptr()), C.c_void_p(out_r.data_ptr())))
    np.testing.assert_array_equal(out_r.cpu().numpy(), r1)
    np.testing.assert_array_equal(out_s.cpu().numpy(), s1)
    # float64 scores of a shard equal the matching slice of the unsharded scan
    full = one.score(queries[0])
    lo, hi = n // shards, 2 * n // shards
    np.testing.assert_allclose(parts[1].score(queries[0]), full[lo:hi], rtol=1e-12, atol=1e-15)


def test_pruned_scan_equals_exhaustive_scan(lib):
    """Block-max pruning is exact: same rows, same float32 scores as the exhaustive scan."""
    import os

    from kakveda_b200 import GfkbIndex, synth

    n, q, k = 300_000, 3000, 16
    buf, off = synth.signatures_packed(synth.CORPUS_SEED, 0, n)
    ix = GfkbIndex()
    fb = ix.vocab.featurize_packed(buf, off, 0, grow=True)
    ix.add_features(fb)
    fb.close()
    ix.finalize()
    queries = synth.queries(q, n) + ["", "zz qq unseen", "intent_tags prompt_hint tools env_keys"]
    s1, r1 = ix.topk(queries, k)
    lay = ix.layout()
    # the tensor-core bounds leave only a small share of the (query, chunk) pairs to the exact scan
    assert 0 < lay["pairs_passed_bound"] < 0.2 * len(queries) * lay["chunks"], lay
    assert lay["pairs_scored"] >= lay["pairs_passed_bound"] and lay["records_written"] > 0
    # without the stored bound codes, bound pass 1 recomputes the bounds to build the candidate lists: same results,
    # and no pair passes that the codes (bounds rounded up to 1/250) would have dropped
    os.environ["KAKVEDA_B200_BOUND_CODES"] = "0"
    try:
        s3, r3 = ix.topk(queries, k)
        lay3 = ix.layout()
    finally:
        del os.environ["KAKVEDA_B200_BOUND_CODES"]
    np.testing.assert_array_equal(r1, r3)
    np.testing.assert_array_equal(s1, s3)
    assert 0 < lay3["pairs_passed_bound"] <= lay["pairs_passed_bound"], (lay, lay3)
    os.environ["KAKVEDA_B200_NO_PRUNE"] = "1"
    try:
        s2, r2 = ix.topk(queries, k)
        lay2 = ix.layout()
        assert lay2["pairs_passed_bound"] == 0 and lay2["pairs_scored"] >= q * lay2["chunks"]  # exhaustive: no bound kernel
    finally:
        del os.environ["KAKVEDA_B200_NO_PRUNE"]
    np.testing.assert_array_equal(r1, r2)
    np.testing.assert_array_equal(s1, s2)
    # null queries: every score 0 -> the first k rows in order
    assert r1[q].tolist() == list(range(k)) and np.all(s1[q] == 0)
    assert r1[q + 1].tolist() == list(range(k)) and np.all(s1[q + 1] == 0)
    # and both agree with the float64 scan on a sample
    for i in (0, 1, 2, q + 2):
        full = ix.score(queries[i])
        order, vals = O.topk_stable(full.tolist(), k)
        np.testing.assert_allclose(s1[i], vals, rtol=RTOL32, atol=1e-7)
        for a, b in zip(order, r1[i].tolist()):
            assert a == b or full[a] == pytest.approx(full[b], rel=RTOL32)


@pytest.mark.parametrize("bound_codes", ["1", "0"])
def test_two_phase_batch_equals_one_phase_batch(lib, bound_codes):
    """kv_topk_resident_seed + kv_index_raise_thresholds with the index's own k-th seed score + kv_topk_resident_finish
    (the sharded step, on one index) returns bit for bit what kv_topk_resident does, with the bound codes kept and with
    the recomputing bound pass 1."""
    import os

    import torch

    from kakveda_b200 import GfkbIndex, synth

    n, q, k = 300_000, 3000, 16
    buf, off = synth.signatures_packed(synth.CORPUS_SEED, 0, n)
    ix = GfkbIndex()
    fb = ix.vocab.featurize_packed(buf, off, 0, grow=True)
    ix.add_features(fb)
    fb.close()
    ix.finalize()
    qfb = ix.vocab.featurize(synth.queries(q, n), grow=False)
    ix.upload_queries(qfb)
    qfb.close()
    s1 = torch.empty((q, k), dtype=torch.float32, device="cuda")
    r1 = torch.empty((q, k), dtype=torch.int64, device="cuda")
    s2, r2 = torch.empty_like(s1), torch.empty_like(r1)
    os.environ["KAKVEDA_B200_BOUND_CODES"] = bound_codes
    try:
        ix.topk_resident(k, s1.data_ptr(), r1.data_ptr())
        ix.topk_resident_seed(k, s2.data_ptr(), r2.data_ptr())
        kth = s2[:, k - 1].contiguous()
        torch.cuda.synchronize()  # the index runs on its own stream
        ix.raise_thresholds(kth.data_ptr(), q)
        ix.topk_resident_finish(k, s2.data_ptr(), r2.data_ptr())
    finally:
        del os.environ["KAKVEDA_B200_BOUND_CODES"]
    torch.cuda.synchronize()
    assert torch.isfinite(kth).any()
    np.testing.assert_array_equal(r1.cpu().numpy(), r2.cpu().numpy())
    np.testing.assert_array_equal(s1.cpu().numpy(), s2.cpu().numpy())


def test_query_batch_uploaded_as_slices_equals_whole_batch(lib):
    """kv_query_upload_runs (what a row-sharded GFKB's ranks exchange: slices featurised, classified and text-sorted
    separately, orders merged) leaves the same resident batch as kv_query_upload of the whole CSR: identical results
    and identical pruning work."""
    from kakveda_b200 import GfkbIndex, synth
    from kakveda_b200.similarity import pack_texts

    n, k = 120_000, 16
    buf, off = synth.signatures_packed(synth.CORPUS_SEED, 0, n)
    ix = GfkbIndex()
    fb = ix.vocab.featurize_packed(buf, off, 0, grow=True)
    ix.add_features(fb)
    fb.close()
    ix.finalize()
    queries = synth.queries(5000, n) + ["", "zz qq unseen", "intent_tags prompt_hint tools env_keys", " ".join(f"w{i}" for i in range(200))]
    nq = len(queries)
    s1, r1 = ix.topk(queries, k)
    lay1 = ix.layout()
    data, offsets, mode = pack_texts(queries)
    for cuts in ([0, nq], [0, 1700, 1700, 4100, nq], [0, 7, nq - 3, nq]):       # one run; an empty run; tiny runs
        for with_prep in (True, False):
            runs, keep = [], []
            for a, b in zip(cuts[:-1], cuts[1:]):
                qfb = ix.vocab.featurize_packed(data, offsets[a:b + 1], mode, grow=False)
                keep.append(qfb)
                if with_prep:
                    runs.append(ix.prepare_slice(qfb))          # rows re-stored in text order + order + flags
                else:
                    runs.append((qfb.indptr, qfb.ids, qfb.tf, qfb.oov, None, None))
            assert ix.upload_query_runs(runs) == nq
            s2, r2 = ix.topk_resident_host(nq, k)
            lay2 = ix.layout()
            for f in keep:
                f.close()
            np.testing.assert_array_equal(r1, r2)
            np.testing.assert_array_equal(s1, s2)
            assert lay2["pairs_passed_bound"] == lay1["pairs_passed_bound"], (cuts, with_prep)
    # a slice order that is not a permutation, or rows that are not stored in text order, are rejected
    qfb = ix.vocab.featurize_packed(data, offsets[0:11], mode, grow=False)
    run = ix.prepare_slice(qfb)
    bad = run[4].copy(); bad[0] = bad[1]
    with pytest.raises((ValueError, RuntimeError)):
        ix.upload_query_runs([run[:4] + (bad, run[5]), run])
    ident = np.arange(qfb.n, dtype=np.int32)
    with pytest.raises((ValueError, RuntimeError)):
        ix.upload_query_runs([(qfb.indptr, qfb.ids, qfb.tf, qfb.oov, ident, run[5]), run])   # unsorted rows claimed sorted
    qfb.close()


def test_concurrent_score_calls(lib):
    from kakveda_b200 import SimilarityEngine, synth

    corpus = synth.corpus(2000)
    qs = synth.queries(8, 2000)
    eng = SimilarityEngine()
    want = [eng.score(q, corpus) for q in qs]
    got = [None] * len(qs)

    def work(i):
        got[i] = eng.score(qs[i], corpus)

    th = [threading.Thread(target=work, args=(i,)) for i in range(len(qs))]
    [t.start() for t in th]
    [t.join() for t in th]
    assert got == want


def test_large_properties(lib):
    """Size-independent properties at 2M rows (the oracle cannot run here in seconds)."""
    from kakveda_b200 import GfkbIndex, synth

    n, q, k = 2_000_000, 2048, 16
    buf, off = synth.signatures_packed(synth.CORPUS_SEED, 0, n)
    ix = GfkbIndex()
    fb = ix.vocab.featurize_packed(buf, off, 0, grow=True)
    ix.add_features(fb)
    fb.close()
    ix.finalize()
    queries = synth.queries(q, n)
    s, r = ix.topk(queries, k)
    s2, r2 = ix.topk(queries, k)
    np.testing.assert_array_equal(r, r2)            # deterministic
    np.testing.assert_array_equal(s, s2)
    assert np.all(r >= 0) and np.all(r < n)
    assert np.all(np.diff(s, axis=1) <= 0)          # sorted by score
    ties = np.diff(s, axis=1) == 0
    assert np.all(np.diff(r, axis=1)[ties] > 0)     # equal scores -> ascending rows
    raw = buf.tobytes()
    text = lambda i: raw[off[i]:off[i + 1]].decode()
    exact = 0
    for i in range(0, q, 48):
        if abs(s[i, 0] - 1.0) < 1e-6:               # the query repeats a stored failure
            assert text(int(r[i, 0])) == queries[i]
            exact += 1
        # the float64 full scan agrees with the fused float32 top-k
        full = ix.score(queries[i])
        order, vals = O.topk_stable(full.tolist(), k)
        np.testing.assert_allclose(s[i], vals, rtol=RTOL32)
        for a, b in zip(order, r[i].tolist()):
            assert a == b or full[a] == pytest.approx(full[b], rel=RTOL32)
    assert exact > 10


def test_hash_fingerprint_match(lib):
    """K4 (parity unpinned: the reference never queries fingerprint()): integer equality, bit-exact."""
    from kakveda_b200 import HashIndex, synth
    from kakveda_b200.fingerprint import fingerprint_text

    n, q, k = 50_000, 9000, 4
    corpus, queries = synth.corpus(n), synth.queries(q, n) + ["never stored"]
    hx = HashIndex()
    hx.add_signatures(corpus)
    assert hx.n_rows == n
    rows, counts = hx.match_signatures(queries, k)
    where = {}
    for i, s in enumerate(corpus):
        where.setdefault(O.fingerprint64(s), []).append(i)
    for i, s in enumerate(queries):
        want = where.get(O.fingerprint64(s), [])
        assert counts[i] == len(want)
        assert rows[i].tolist() == (want[:k] + [-1] * k)[:k]
        assert O.fingerprint64(s) == int(fingerprint_text(s), 16)
    assert counts[-1] == 0 and 0.4 * q < np.count_nonzero(counts) < 0.6 * q + 1
    # large: 20M random hashes, 4096 planted queries (one pass) -- size-independent properties
    rng = np.random.default_rng(7)
    big = rng.integers(0, 2**63, size=20_000_000, dtype=np.uint64)
    hb = HashIndex(row_base=1000)
    hb.add_hashes(big)
    pick = rng.integers(0, len(big), size=4096)
    r, c = hb.match_hashes(big[pick], 2)
    assert np.all(c >= 1) and np.all(big[r[:, 0] - 1000] == big[pick]) and np.all(r[:, 0] - 1000 <= pick)
    ms, passes = hb.last_timing()
    assert passes == 1 and ms > 0


@pytest.mark.parametrize("n,d,q", [(3000, 128, 200), (20000, 768, 500), (257, 64, 3)])
def test_dense_cosine_topk(lib, n, d, q):
    """K2 (parity unpinned: no embedding path in the reference).  Tolerance from SURVEY 8(c): rtol 1e-5,
    atol 1e-6 on the returned scores against float64 cosine of the same bf16-rounded inputs."""
    from kakveda_b200 import DenseIndex

    rng = np.random.default_rng(n + d)
    C = rng.standard_normal((n, d)).astype(np.float32)
    Q = rng.standard_normal((q, d)).astype(np.float32)
    Q[: min(q, 50)] = C[rng.integers(0, n, size=min(q, 50))] * 1.5   # exact directional matches -> cosine 1
    C[7] = 0.0                                                        # zero vector scores 0
    if n > 1000:
        C[1001] = C[1000]                                             # duplicate rows tie -> lower row first
        Q[min(q, 50)] = C[1000]
    dx = DenseIndex(d)
    dx.add(C[: n // 2])
    dx.add(C[n // 2:])
    dx.finalize()
    k = 16
    s, r = dx.topk(Q, k)
    want = O.dense_cosine(Q, C)
    kk = min(k, n)
    for i in range(q):
        assert len(set(r[i, :kk].tolist())) == kk and np.all(r[i, :kk] >= 0)
        np.testing.assert_allclose(s[i, :kk], want[i, r[i, :kk]], rtol=1e-5, atol=1e-6)
        rest = np.delete(want[i], r[i, :kk])
        if rest.size:
            assert rest.max() <= want[i, r[i, :kk]].min() + 2e-6
        assert np.all(np.diff(s[i, :kk]) <= 0)
        ties = np.diff(s[i, :kk]) == 0
        assert np.all(np.diff(r[i, :kk])[ties] > 0)
    assert np.allclose(s[:min(q, 50), 0], 1.0, atol=1e-5)
    if n > 1000:
        assert r[min(q, 50), :2].tolist() == [1000, 1001]


def test_jaccard_token_sets(lib):
    """K3 (parity unpinned: no Jaccard in the reference).  Bit-exact: the device ranks by inter/union, the exact
    integers come back, and float64 inter/union equals Python's set arithmetic."""
    from kakveda_b200 import JaccardIndex

    rng = np.random.default_rng(5)
    V, n, q, k = 1 << 14, 6000, 160, 16
    zipf = lambda size: np.minimum(rng.zipf(1.3, size) - 1, V - 1).astype(np.uint32)
    rows = [np.unique(zipf(max(1, rng.poisson(40)))) for _ in range(n)]
    rows[5] = np.zeros(0, dtype=np.uint32)                 # empty set
    rows[100] = rows[99].copy()                            # duplicate rows tie -> lower row first
    queries = [np.unique(zipf(max(1, rng.poisson(40)))) for _ in range(q)]
    queries[0] = rows[99].copy()
    queries[1] = np.zeros(0, dtype=np.uint32)              # empty query: every score 0
    queries[2] = np.concatenate([rows[7], np.array([V + 5, V + 9], dtype=np.uint32)])  # ids outside the vocabulary
    jx = JaccardIndex(V)
    jx.add_sets(rows[: n // 2])
    jx.add_sets(rows[n // 2:])
    jx.finalize()
    s, r, inter, union = jx.topk_sets(queries, k)
    for i, qs in enumerate(queries):
        want = np.array([(lambda iu: iu[0] / iu[1] if iu[1] else 0.0)(O.jaccard_sets(qs.tolist(), c.tolist())) for c in rows])
        order, vals = O.topk_stable(want.tolist(), k)
        got64 = np.where(union[i] > 0, inter[i] / np.maximum(union[i], 1), 0.0)
        assert got64.tolist() == vals, (i, got64, vals)               # bit-exact float64 ratios
        assert r[i].tolist() == order, (i, r[i], order)               # same rows, ties -> lower row
        for j in range(k):
            assert (int(inter[i, j]), int(union[i, j])) == O.jaccard_sets(qs.tolist(), rows[int(r[i, j])].tolist())
        np.testing.assert_allclose(s[i], vals, rtol=1e-6, atol=1e-7)
    assert r[0, 0] == 99 and r[0, 1] == 100 and inter[0, 0] == union[0, 0]
    assert r[1].tolist() == list(range(k))


def test_bound_kernel_numerators_vs_numpy(lib):
    """K1b-B (wgmma GEMM over the frequent features + transposed bitmaps of the second class + rare-feature join): the
    dot-product upper bound of every (query, chunk) pair equals the exact union bound sum_{t in q and chunk}
    tf_q a(t) max_tf_chunk(t) computed with NumPy -- never below it (the pruning stays exact), and within 0.1 % of
    it for all but a sliver of the pairs (fp16 round-up of weights; a chunk holding tf >= 2 of a second-class
    feature is charged that feature's largest tf)."""
    import ctypes as C

    import scipy.sparse as sp

    from kakveda_b200 import GfkbIndex, _capi, synth

    n, q = 60_000, 256
    ix = GfkbIndex()
    buf, off = synth.signatures_packed(synth.CORPUS_SEED, 0, n)
    fb = ix.vocab.featurize_packed(buf, off, 0, grow=True)
    ip, ids, tf = fb.indptr.copy(), fb.ids.copy().astype(np.int64), fb.tf.copy().astype(np.float64)
    ix.add_features(fb)
    fb.close()
    ix.finalize()
    V = len(ix.vocab)
    qbuf, qoff = synth.signatures_packed(synth.QUERY_SEED, 0, q, dup_of_seed=synth.CORPUS_SEED, dup_rows=n)
    qfb = ix.vocab.featurize_packed(qbuf, qoff, 0, grow=False)
    qip, qids, qtf = qfb.indptr.copy(), qfb.ids.copy().astype(np.int64), qfb.tf.copy().astype(np.float64)
    ix.upload_queries(qfb)
    nch = (n + 31) // 32
    got = np.zeros((q, nch), dtype=np.float32)
    slot_query = np.zeros(q, dtype=np.int32)
    _capi.check(lib.kv_debug_bound_numerators(ix._h, 16, got.ctypes.data_as(C.POINTER(C.c_float)),
                                              slot_query.ctypes.data_as(C.POINTER(C.c_int32))))
    qfb.close()
    # NumPy: chunk unions (32 rows per chunk of the scan layout) with the max tf
    rowof = np.repeat(np.arange(n), np.diff(ip))
    df = np.bincount(ids, minlength=V).astype(np.float64)
    a = (np.log((n + 2) / (df + 2)) + 1) ** 2
    # the scan layout's row order, as the index built it (row_at_pos of kv_debug_bound_codes)
    row_at_pos = np.zeros(n, dtype=np.int32)
    _capi.check(lib.kv_debug_bound_codes(ix._h, 16, np.zeros((q, nch), dtype=np.uint8).ctypes.data_as(C.POINTER(C.c_uint8)),
                                         np.zeros(q, dtype=np.int32).ctypes.data_as(C.POINTER(C.c_int32)), None, None,
                                         None, row_at_pos.ctypes.data_as(C.POINTER(C.c_int32))))
    pos_of = np.empty(n, dtype=np.int64)
    pos_of[row_at_pos] = np.arange(n)
    key = (pos_of[rowof] // 32) * V + ids
    o = np.lexsort((tf, key))
    ks = key[o]
    last = np.r_[ks[1:] != ks[:-1], True]
    U = sp.csr_matrix((tf[o][last], (ks[last] // V, ks[last] % V)), shape=(nch, V))
    qrow = np.repeat(np.arange(q), np.diff(qip))
    known = qids < V
    W = sp.csc_matrix((qtf[known] * a[qids[known]], (qids[known], qrow[known])), shape=(V, q))
    want = np.asarray((U @ W).todense()).T[slot_query]
    ratio = (got + 1e-3) / (want + 1e-3)
    assert ratio.min() >= 1.0 - 1e-6, "a bound below the exact union bound: pruning would drop rows"
    assert np.quantile(ratio, 0.999) <= 1.002 and ratio.max() < 3.0, (np.quantile(ratio, [0.5, 0.999]), ratio.max())
