"""Every query of bench-scale TF-IDF, Jaccard and dense indexes against an independent float64 oracle, on the GPU.

The other large-index checks compare an index with itself (pruned against exhaustive scan, or against K1a, which reads
the same column blocks, df histogram, idf tables, row norms and fixed-point query weights as the path it checks).  Here
the oracle is ``oracle/torch_oracle.py``: float64 torch on the raw CSR the featuriser produced, never anything inside an
index.  It runs on the device beside the index, one block of queries at a time, and the checkers below evaluate the
strict top-k contract (``check_topk_strict`` of test_gpu_topk_edges.py) and the threshold-search contract on the device
too, so that every query is checked, not a sample.

Cases (each asserts which path ran through ``layout()`` / ``last_timing()`` / ``kernel_launches`` / the query flags):

* A: the bench corpus at 2M rows, 8,192 bench queries plus the query classes, k = 16 and 32 on the pruned path with
  the specialised and the generic bound kernel, with recomputed bounds, exhaustive, and through the device featuriser;
  K1a at rtol 1e-9 over all rows; threshold search (host and device results); deletion + label filters.
* B: one shard of the 8-GPU headline (rows [8.75M, 10M), global N = 10M and the df of all 10M rows).
* C: the largest idf values (global N up to 2^31 - 1, df = 1) on a small index with crafted tf up to 65535, queries on
  both sides of every ``classify_queries`` limit.
* D: Jaccard at the bench shape, 1M sets x 2,048 queries, bit-exact.
* E: dense at the bench shape, 1M x 768 bf16 rows x 2,048 queries, host and device; threshold search; self-join.

Measured on an NVIDIA H100 80GB HBM3 (700 W limit): the whole file runs in 177 s (pytest wall time, library build
excluded).  Per case: A 13 s index build + 65 s + 22 s (deletion), B 38 s (of which 25 s featurise the other 8.75M
rows on the host for the global df), C under 1 s per N, D 19 s, E 1.4 s.  The oracle's peak torch memory is
12.5 GiB (case A with deletions: [64, 2M] float64 blocks), 17.2 GiB in case E (the 1M x 768 rows in float64); the
device memory in use at the end of a case, index included, is at most 22 GiB.  ``device_memory_report`` prints these
figures for every GPU case.
"""
import math
import time

import numpy as np
import pytest

from oracle import tfidf_oracle as O
from oracle import torch_oracle as T

torch = pytest.importorskip("torch")

gpu = pytest.mark.gpu

RTOL32 = 1e-5                       # float32 top-k and threshold scores against the float64 closed form
RTOL64 = 1e-9                       # K1a (float64) against the float64 closed form
DENSE_RTOL, DENSE_ATOL = 1e-5, 1e-6


def dense_rtol(d):
    """As in test_gpu_topk_edges.py: the tensor cores' fp32 accumulation loses up to dim / 16 fp32 ulps."""
    return max(DENSE_RTOL, d / 16 * 2.0 ** -23)


# ---------------------------------------------------------------------------------------------------------------------
# Device checkers
# ---------------------------------------------------------------------------------------------------------------------

def _fail(bad, msg, detail):
    """Assert that no query of the block has ``bad`` set; name the first one that has."""
    if bool(bad.any()):
        q = int(torch.nonzero(bad)[0, 0])
        raise AssertionError(f"{msg}; {detail(q)}")


def check_topk_device(scores, rows, oracle64, k, rtol, atol=0.0, first=0):
    """The contract of ``check_topk_strict`` (test_gpu_topk_edges.py), evaluated on the oracle's device for a block of
    queries: scores [B,k] / rows [B,k] of a top-k (arrays or tensors), oracle64 float64 [B,N] (-inf: a row the query
    must not match).  ``first``: the batch index of the block's first query, for the messages."""
    o = oracle64
    dev = o.device
    s = torch.as_tensor(np.asarray(scores) if not torch.is_tensor(scores) else scores, device=dev).to(torch.float64)
    r = torch.as_tensor(np.asarray(rows) if not torch.is_tensor(rows) else rows, device=dev).to(torch.int64)
    nq, n = o.shape
    assert tuple(s.shape) == (nq, k) and tuple(r.shape) == (nq, k), (tuple(s.shape), tuple(r.shape), tuple(o.shape), k)
    detail = lambda q: f"query {first + q}: rows {r[q].tolist()} scores {s[q].tolist()}"
    kk = torch.clamp(torch.isfinite(o).sum(1), max=k)
    valid = torch.arange(k, device=dev)[None, :] < kk[:, None]
    _fail((~valid & ((r != -1) | (s != -math.inf))).any(1), "slots past min(k, N) must hold (-inf, -1)", detail)
    _fail((valid & ((r < 0) | (r >= n))).any(1), "row outside the index", detail)
    ov = torch.where(valid, o.gather(1, r.clamp(0, n - 1)), torch.full_like(s, math.nan))
    _fail((valid & ~torch.isfinite(ov)).any(1), "an excluded row was returned", detail)
    rs = torch.sort(torch.where(valid, r, -1 - torch.arange(k, device=dev)[None, :]), dim=1).values
    _fail((rs[:, 1:] == rs[:, :-1]).any(1), "duplicate row", detail)
    ordered = (s[:, :-1] > s[:, 1:]) | ((s[:, :-1] == s[:, 1:]) & (r[:, :-1] < r[:, 1:]))
    _fail((valid[:, 1:] & ~ordered).any(1), "order (score desc, row asc) broken", detail)
    _fail((valid & ((s - ov).abs() > atol + rtol * ov.abs())).any(1), "score outside tolerance", detail)
    has = kk > 0
    if not bool(has.any()):
        return
    top = torch.topk(o, int(kk.max()), dim=1).values
    kth = top.gather(1, (kk - 1).clamp(min=0)[:, None])[:, 0]
    kth = torch.where(has, kth, torch.full_like(kth, math.inf))
    tied = o == kth[:, None]
    # exact ties: when the k-th score's tie class has members past the k-th position, the returned members of the
    # class must be its lowest row ids (the zero-score fill makes the class the whole index)
    straddle = has & (tied.sum(1) > kk - (o > kth[:, None]).sum(1))
    mine_n = (valid & (ov == kth[:, None])).sum(1)
    idx = torch.nonzero(straddle)[:, 0]
    for c in range(0, len(idx), 16):
        qs = idx[c:c + 16]
        key = torch.where(tied[qs], torch.arange(n, device=dev)[None, :], n)
        lowest = torch.topk(key, k, dim=1, largest=False).values          # ascending
        mine = torch.sort(torch.where(valid[qs] & (ov[qs] == kth[qs, None]), r[qs], n + 1), dim=1).values
        wrong = (torch.arange(k, device=dev)[None, :] < mine_n[qs, None]) & (mine != lowest)
        bad = torch.zeros(nq, dtype=torch.bool, device=dev)
        bad[qs] = wrong.any(1)
        _fail(bad, "exact tie at the k-th score: returned members of its tie class are not its lowest row ids", detail)
    # near ties: a row above the k-th score by more than 2 rtol must be returned; a returned row may sit at most
    # 2 rtol below it
    tol = 2 * rtol * kth.abs() + 2 * atol
    above = o > (kth + tol)[:, None]
    got_above = (valid & (ov > (kth + tol)[:, None])).sum(1)
    _fail(has & (above.sum(1) != got_above), "rows missing from the top-k (oracle score above the k-th)", detail)
    _fail((valid & (ov < (kth - tol)[:, None])).any(1), "rows returned below the k-th score", detail)


def misordered(qrow, r, s):
    """Per pair of a range result: True where the next pair of the same query breaks (score desc, row asc)."""
    bad = torch.zeros_like(r, dtype=torch.bool)
    bad[:-1] = (qrow[1:] == qrow[:-1]) & ~((s[:-1] > s[1:]) | ((s[:-1] == s[1:]) & (r[:-1] < r[1:])))
    return bad


def check_range_device(indptr, rows, scores, oracle64, threshold, rtol, atol=0.0, first=0):
    """Threshold search of a block of queries: CSR (indptr [B+1] relative to the block, rows, scores) against
    oracle64 float64 [B,N].  The pair set must be {oracle >= threshold}, except pairs within 2 (rtol + atol) of the
    threshold; every score within rtol (+atol); (score desc, row asc) inside each query; no duplicate or excluded row."""
    o = oracle64
    dev = o.device
    nq, n = o.shape
    ip = torch.as_tensor(np.asarray(indptr) if not torch.is_tensor(indptr) else indptr, device=dev).to(torch.int64)
    r = torch.as_tensor(np.asarray(rows) if not torch.is_tensor(rows) else rows, device=dev).to(torch.int64)
    s = torch.as_tensor(np.asarray(scores) if not torch.is_tensor(scores) else scores, device=dev).to(torch.float64)
    ip = ip - ip[0]
    assert len(ip) == nq + 1 and int(ip[-1]) == len(r) == len(s), (len(ip), nq, len(r), len(s))
    qrow = torch.repeat_interleave(torch.arange(nq, device=dev), ip[1:] - ip[:-1])
    detail = lambda q: f"query {first + q}: rows {r[ip[q]:ip[q + 1]][:16].tolist()} scores {s[ip[q]:ip[q + 1]][:16].tolist()}"
    per_q = lambda bad_pairs: torch.zeros(nq, dtype=torch.bool, device=dev).index_fill_(0, qrow[bad_pairs], True)
    _fail(per_q((r < 0) | (r >= n)), "row outside the index", detail)
    ov = o[qrow, r.clamp(0, n - 1)]
    _fail(per_q(~torch.isfinite(ov)), "an excluded row was returned", detail)
    _fail(per_q(misordered(qrow, r, s)), "order (score desc, row asc) or a duplicate row", detail)
    _fail(per_q((s - ov).abs() > atol + rtol * ov.abs()), "score outside tolerance", detail)
    margin = 2 * (rtol * threshold + atol)
    _fail(per_q(ov < threshold - margin), "a pair below the threshold was returned", detail)
    must = (o >= threshold + margin).sum(1)
    got = torch.zeros(nq, dtype=torch.int64, device=dev).index_add_(0, qrow, (ov >= threshold + margin).to(torch.int64))
    _fail(must != got, "pairs above the threshold are missing", detail)


def check_jaccard_range_device(indptr, rows, scores, inter, union, I, U, threshold, first=0):
    """Jaccard threshold search, exact: the pair set is {float32(inter / union) >= threshold}, the counts are the
    oracle's, the scores are float32(inter / union) to 1e-6."""
    dev = I.device
    nq, n = I.shape
    conv = lambda a: torch.as_tensor(np.asarray(a) if not torch.is_tensor(a) else a, device=dev)
    ip, r, s, gi, gu = conv(indptr).to(torch.int64), conv(rows).to(torch.int64), conv(scores), conv(inter), conv(union)
    ip = ip - ip[0]
    ratio = torch.where(U > 0, I / U.clamp(min=1), torch.zeros_like(I))
    want = ratio.to(torch.float32) >= np.float32(threshold)
    qrow = torch.repeat_interleave(torch.arange(nq, device=dev), ip[1:] - ip[:-1])
    detail = lambda q: f"query {first + q}: rows {r[ip[q]:ip[q + 1]][:16].tolist()}"
    per_q = lambda bad_pairs: torch.zeros(nq, dtype=torch.bool, device=dev).index_fill_(0, qrow[bad_pairs], True)
    _fail(per_q((r < 0) | (r >= n)), "row outside the index", detail)
    rc = r.clamp(0, n - 1)
    _fail(per_q(~want[qrow, rc]), "a pair below the threshold was returned", detail)
    _fail(want.sum(1) != (ip[1:] - ip[:-1]), "pairs above the threshold are missing (or duplicated)", detail)
    _fail(per_q((gi.to(torch.float64) != I[qrow, rc]) | (gu.to(torch.float64) != U[qrow, rc])), "wrong (inter, union)", detail)
    _fail(per_q((s.to(torch.float64) - ratio[qrow, rc]).abs() > 1e-6 * ratio[qrow, rc] + 1e-7), "score outside tolerance", detail)
    _fail(per_q(misordered(qrow, r, s)), "order broken", detail)


# ---------------------------------------------------------------------------------------------------------------------
# Checker self-tests: the hand-made wrong answers of test_gpu_topk_edges.py, fed to the device checker (on CPU torch)
# ---------------------------------------------------------------------------------------------------------------------

def _chk(scores, rows, oracle, k, rtol, atol=0.0):
    check_topk_device(np.array([scores], np.float32), np.array([rows], np.int64), torch.tensor(oracle, dtype=torch.float64),
                      k, rtol, atol)


def test_device_checker_rejects_wrong_answers():
    ties = [[0.9, 0.5, 0.5, 0.5, 0.1]]
    _chk((0.9, 0.5), (0, 1), ties, 2, RTOL32)                                    # the right answer passes
    with pytest.raises(AssertionError, match="exact tie"):                      # tied row 1 replaced by tied row 2
        _chk((0.9, 0.5), (0, 2), ties, 2, RTOL32)
    with pytest.raises(AssertionError, match="exact tie"):
        _chk((0.9, 0.5, 0.5), (0, 1, 3), ties, 3, RTOL32)
    spread = [[0.9, 0.8, 0.7, 0.1]]
    with pytest.raises(AssertionError, match="returned|missing"):               # row 1 missing, far outside rtol
        _chk((0.9, 0.7), (0, 2), spread, 2, RTOL32)
    with pytest.raises(AssertionError, match="order"):                          # swapped pair
        _chk((0.8, 0.9), (1, 0), spread, 2, RTOL32)
    with pytest.raises(AssertionError, match="order"):                          # equal scores, rows descending
        _chk((0.9, 0.5, 0.5), (0, 2, 1), ties, 3, RTOL32)
    with pytest.raises(AssertionError, match="tolerance"):                      # right rows, score off by 1e-4
        _chk((0.9, 0.80008), (0, 1), spread, 2, RTOL32)
    with pytest.raises(AssertionError, match="duplicate"):
        _chk((0.9, 0.9), (0, 0), spread, 2, RTOL32)
    fill = [[0.5, 0.0, 0.0, 0.0, 0.0, 0.0]]                                     # one match, then the zero-score fill
    _chk((0.5, 0, 0, 0), (0, 1, 2, 3), fill, 4, RTOL32)
    with pytest.raises(AssertionError, match="order"):                          # fill not ascending
        _chk((0.5, 0, 0, 0), (0, 1, 3, 2), fill, 4, RTOL32)
    with pytest.raises(AssertionError, match="exact tie"):                      # fill skips row 3
        _chk((0.5, 0, 0, 0), (0, 1, 2, 4), fill, 4, RTOL32)
    with pytest.raises(AssertionError, match="exact tie"):                      # fill starts in a later split
        _chk((0.5, 0, 0, 0), (0, 3, 4, 5), fill, 4, RTOL32)
    full = ((0.5, 0, 0, 0, 0, 0, -np.inf, -np.inf), (0, 1, 2, 3, 4, 5, -1, -1))  # slots past N = 6 rows
    _chk(*full, fill, 8, RTOL32)
    with pytest.raises(AssertionError, match="slots past"):
        _chk((0.5, 0, 0, 0, 0, 0, 0, -np.inf), (0, 1, 2, 3, 4, 5, -1, -1), fill, 8, RTOL32)
    with pytest.raises(AssertionError, match="slots past"):
        _chk(full[0], (0, 1, 2, 3, 4, 5, 0, -1), fill, 8, RTOL32)
    excl = [[-np.inf, 0.7, 0.3]]                                                # an excluded row must never come back
    _chk((0.7,), (1,), excl, 1, RTOL32)
    with pytest.raises(AssertionError, match="excluded"):
        _chk((0.7, 0.0), (1, 0), excl, 2, RTOL32)
    # a block: only the wrong query is named
    o = torch.tensor([[0.9, 0.5, 0.5, 0.1], [0.9, 0.5, 0.5, 0.1]], dtype=torch.float64)
    with pytest.raises(AssertionError, match="query 8:"):
        check_topk_device(np.float32([[0.9, 0.5], [0.9, 0.5]]), np.int64([[0, 1], [0, 2]]), o, 2, RTOL32, first=7)


def test_device_checker_accepts_float32_near_tie_reordering():
    near = [[0.9, 0.7 + 6e-8, 0.7, 0.1]]
    _chk((0.9, 0.70000005, 0.7), (0, 2, 1), near, 3, RTOL32)
    _chk((0.9, 0.7), (0, 2), near, 2, RTOL32)
    _chk((0.9, 0.7, 0.7), (0, 1, 2), near, 3, RTOL32)                          # equal float32 scores, rows ascending
    _chk((3e-7, 0.0), (1, 0), [[0.0, 2e-7]], 2, DENSE_RTOL, DENSE_ATOL)


def test_range_checkers_reject_wrong_answers():
    o = torch.tensor([[0.9, 0.8, 0.5, 0.80000001, 0.1], [0.2, 0.95, 0.3, -math.inf, 0.85]], dtype=torch.float64)
    ok = ([0, 3, 5], [0, 1, 3, 1, 4], np.float32([0.9, 0.8, 0.8, 0.95, 0.85]))
    check_range_device(*ok, o, 0.8, RTOL32)
    check_range_device([0, 0, 0], [], np.float32([]), o, 0.99, RTOL32)                               # no pair at all
    check_range_device([0, 1, 2], [0, 1], np.float32([0.9, 0.95]), o, 0.85, RTOL32)                  # row 4 of query 1: at θ
    check_range_device([0, 2, 4], [0, 1, 1, 4], np.float32([0.9, 0.8, 0.95, 0.85]), o, 0.8, RTOL32)   # row 3: within rounding of θ
    with pytest.raises(AssertionError, match="missing"):
        check_range_device([0, 2, 3], [0, 3, 1], np.float32([0.9, 0.8, 0.95]), o, 0.8, RTOL32)       # row 4 of query 1 missing
    with pytest.raises(AssertionError, match="below"):
        check_range_device([0, 3, 5], [0, 1, 2, 1, 4], np.float32([0.9, 0.8, 0.5, 0.95, 0.85]), o, 0.8, RTOL32)
    with pytest.raises(AssertionError, match="order"):
        check_range_device([0, 3, 5], [1, 0, 3, 1, 4], np.float32([0.8, 0.9, 0.8, 0.95, 0.85]), o, 0.8, RTOL32)
    with pytest.raises(AssertionError, match="excluded"):
        check_range_device([0, 2, 5], [0, 1, 1, 4, 3], np.float32([0.9, 0.8, 0.95, 0.85, 0.85]), o, 0.8, RTOL32)
    with pytest.raises(AssertionError, match="tolerance"):
        check_range_device([0, 3, 5], [0, 1, 3, 1, 4], np.float32([0.9, 0.8001, 0.8, 0.95, 0.85]), o, 0.8, RTOL32)
    I = torch.tensor([[2.0, 1.0, 3.0]], dtype=torch.float64)
    U = torch.tensor([[2.0, 4.0, 4.0]], dtype=torch.float64)
    check_jaccard_range_device([0, 2], [0, 2], np.float32([1.0, 0.75]), [2, 3], [2, 4], I, U, 0.75)
    with pytest.raises(AssertionError, match="missing"):
        check_jaccard_range_device([0, 1], [0], np.float32([1.0]), [2], [2], I, U, 0.75)
    with pytest.raises(AssertionError, match="inter, union"):
        check_jaccard_range_device([0, 2], [0, 2], np.float32([1.0, 0.75]), [2, 3], [2, 5], I, U, 0.75)
    with pytest.raises(AssertionError, match="below"):
        check_jaccard_range_device([0, 3], [0, 2, 1], np.float32([1.0, 0.75, 0.25]), [2, 3, 1], [2, 4, 4], I, U, 0.75)


# ---------------------------------------------------------------------------------------------------------------------
# Oracle self-tests (CPU torch): the torch oracle against the NumPy / sklearn oracles and the goldens
# ---------------------------------------------------------------------------------------------------------------------

def text_csr(corpus, queries):
    """Raw CSR of rows and queries with a Python vocabulary (O.features), oov = tf² sum of unknown query features."""
    vocab, ip, ids, tf = {}, [0], [], []
    for c in corpus:
        for f, n in sorted(O.features(c).items()):
            ids.append(vocab.setdefault(f, len(vocab)))
            tf.append(n)
        ip.append(len(ids))
    qip, qids, qtf, oov = [0], [], [], []
    for q in queries:
        o = 0.0
        for f, n in O.features(q).items():
            if f in vocab:
                qids.append(vocab[f])
                qtf.append(n)
            else:
                o += float(n) ** 2
        qip.append(len(qids))
        oov.append(o)
    a = lambda x, t: np.asarray(x, dtype=t)
    return (a(ip, np.int64), a(ids, np.int64), a(tf, np.float64)), (a(qip, np.int64), a(qids, np.int64), a(qtf, np.float64), a(oov, np.float64)), len(vocab)


def closed_form_scores(corpus, queries, mode=0):
    (ip, ids, tf), qb, V = text_csr(corpus, queries)
    return T.SparseOracle(ip, ids, tf, V).tfidf_scores(*qb, mode=mode).numpy()


def test_torch_oracle_equals_closed_form(golden, built_lib):
    from kakveda_b200 import synth

    corpus, queries = synth.corpus(3000), synth.queries(48, 3000) + ["", "qqzz unseen", "intent_tags tools"]
    np.testing.assert_allclose(closed_form_scores(corpus, queries), O.score_matrix_closed_form(queries, corpus),
                               rtol=1e-12, atol=1e-15)
    g = golden("edge_cases.json")
    np.testing.assert_allclose(closed_form_scores(g["corpus"], g["queries"]), np.array(g["scores"]), rtol=1e-12, atol=1e-15)
    g = golden("synthetic_small.json")
    np.testing.assert_allclose(closed_form_scores(synth.corpus(g["n"]), synth.queries(g["q"], g["n"])), np.array(g["scores"]),
                               rtol=1e-12, atol=1e-15)
    g = golden("synthetic_cfg1.json")
    s = closed_form_scores(synth.corpus(g["n"]), synth.queries(g["q"], g["n"]))
    np.testing.assert_allclose(s[:8], np.array(g["full_first8"]), rtol=1e-12, atol=1e-15)
    np.testing.assert_allclose(s.sum(1), np.array(g["score_sums"]), rtol=1e-12)
    # mode 2 (fit on the corpus) against sklearn, with a query holding features no row has
    q2 = queries[:16] + ["qqzz unseen " + queries[3]]
    np.testing.assert_allclose(closed_form_scores(corpus[:500], q2, mode=2), O.corpus_fit_scores(q2, corpus[:500]),
                               rtol=1e-12, atol=1e-15)


def test_torch_oracle_jaccard_and_dense():
    rng = np.random.default_rng(3)
    rows = [np.unique(rng.integers(0, 50, rng.integers(0, 12))) for _ in range(300)]
    qs = [np.unique(rng.integers(0, 60, rng.integers(0, 12))) for _ in range(20)] + [rows[7].copy()]
    csr = lambda sets: (np.r_[0, np.cumsum([len(a) for a in sets])], np.concatenate(sets).astype(np.int64))
    I, U = T.SparseOracle(*csr(rows), np.ones(sum(len(a) for a in rows)), 50).jaccard_counts(*csr(qs))
    want = np.array([[O.jaccard_sets(q.tolist(), r.tolist()) for r in rows] for q in qs])
    assert np.array_equal(I.numpy(), want[..., 0]) and np.array_equal(U.numpy(), want[..., 1])
    Q, C = rng.standard_normal((9, 40)).astype(np.float32), rng.standard_normal((70, 40)).astype(np.float32)
    C[3] = 0
    np.testing.assert_allclose(T.dense_cosine(torch.from_numpy(Q), torch.from_numpy(C)).numpy(), O.dense_cosine(Q, C),
                               rtol=1e-13, atol=1e-15)


def test_torch_oracle_statistics_override_and_live_mask():
    """Global (df, N), a live mask and query labels, against the closed form written out by hand."""
    # rows over features 0..3; row 2 is deleted in the second part
    rows = [{0: 2, 1: 1}, {1: 3}, {0: 1, 2: 5}, {3: 1, 0: 1}]
    ip = np.r_[0, np.cumsum([len(r) for r in rows])]
    ids = np.array([f for r in rows for f in r], np.int64)
    tf = np.array([v for r in rows for v in r.values()], np.float64)
    q = {0: 1, 2: 2}
    qb = (np.array([0, 2]), np.array(list(q)), np.array(list(q.values()), np.float64), np.array([4.0]))   # oov tf² 4

    def hand(df, n, live):
        ib = lambda t: math.log((n + 2) / (df[t] + 1)) + 1
        iq = lambda t: math.log((n + 2) / (df[t] + 2)) + 1
        nq = sum((f * iq(t)) ** 2 for t, f in q.items()) + 4.0 * (math.log((n + 2) / 2) + 1) ** 2
        out = []
        for i, r in enumerate(rows):
            if not live[i]:
                out.append(-math.inf)
                continue
            dot = sum(q[t] * f * iq(t) ** 2 for t, f in r.items() if t in q)
            nc = sum((f * (iq(t) if t in q else ib(t))) ** 2 for t, f in r.items())
            out.append(dot / math.sqrt(nq * nc) if dot else 0.0)
        return out

    gdf, gn = np.array([7, 30, 1, 1000]), 5000
    got = T.SparseOracle(ip, ids, tf, 4, df=gdf, n_global=gn).tfidf_scores(*qb)
    np.testing.assert_allclose(got.numpy()[0], hand(gdf, gn, [1, 1, 1, 1]), rtol=1e-14)
    live = np.array([1, 1, 0, 1], bool)
    orc = T.SparseOracle(ip, ids, tf, 4, live=live, labels=np.array([0, 1, 0, 1]))
    np.testing.assert_allclose(orc.tfidf_scores(*qb).numpy()[0], hand([2, 2, 0, 1], 3, live), rtol=1e-14)
    lab = orc.tfidf_scores(*qb, query_labels=np.array([1])).numpy()[0]
    assert lab[0] == -math.inf and lab[2] == -math.inf and lab[1] == hand([2, 2, 0, 1], 3, live)[1]


def test_torch_oracle_duplicate_rows_bit_identical():
    """A row stored several times, with its CSR entries in different orders and at different offsets, scores the
    same bits in every mode; so does a Jaccard set."""
    rng = np.random.default_rng(11)
    V = 400
    base = [(int(t), float(rng.integers(1, 9))) for t in rng.choice(V, 13, replace=False)]
    rows = []
    for i in range(600):
        if i % 97 == 5:
            e = list(base)
            rng.shuffle(e)
            rows.append(e)
        else:
            rows.append([(int(t), float(rng.integers(1, 4))) for t in rng.choice(V, rng.integers(1, 30), replace=False)])
    ip = np.r_[0, np.cumsum([len(r) for r in rows])]
    ids = np.array([t for r in rows for t, _ in r], np.int64)
    tf = np.array([f for r in rows for _, f in r], np.float64)
    dup = [i for i in range(600) if i % 97 == 5]
    qs = [base[:7], base, [(t, 2.0) for t, _ in base[3:]]] + [rows[i][:9] for i in range(0, 60, 7)]
    qip = np.r_[0, np.cumsum([len(q) for q in qs])]
    qids = np.array([t for q in qs for t, _ in q], np.int64)
    qtf = np.array([f for q in qs for _, f in q], np.float64)
    orc = T.SparseOracle(ip, ids, tf, V)
    for mode in (0, 2):
        s = orc.tfidf_scores(qip, qids, qtf, np.zeros(len(qs)), mode=mode)[:, dup]
        assert torch.equal(s, s[:, :1].expand_as(s)), mode
        assert bool((s[:3] > 0).all())
    s = orc.jaccard_scores(qip, qids)[:, dup]
    assert torch.equal(s, s[:, :1].expand_as(s))
    assert len({tuple(t for t, _ in rows[i]) for i in dup}) > 1       # the copies' entry orders differ


# ---------------------------------------------------------------------------------------------------------------------
# GPU cases
# ---------------------------------------------------------------------------------------------------------------------

QBLOCK = 64                         # queries per oracle block (TF-IDF); [64, 2M] float64 = 1 GB per matrix


@pytest.fixture(scope="module")
def lib(built_lib):
    from kakveda_b200 import _capi

    assert _capi.load().kv_device_count() > 0, "GPU tests need a CUDA device"
    return _capi.load()


@pytest.fixture(autouse=True)
def device_memory_report(request):
    """Prints each GPU case's wall time, the oracle's peak torch memory and the device memory in use at its end, and
    hands the oracle's cached blocks back before the next case builds its index."""
    if request.node.get_closest_marker("gpu") is None:
        yield
        return
    torch.cuda.reset_peak_memory_stats()
    t0 = time.perf_counter()
    yield
    free, total = torch.cuda.mem_get_info()
    print(f"\n{request.node.name}: {time.perf_counter() - t0:.1f} s, oracle peak {torch.cuda.max_memory_allocated() / 2**30:.1f} GiB, "
          f"device in use at the end {(total - free) / 2**30:.1f} GiB")
    torch.cuda.empty_cache()


def csr_arrays(fb):
    return np.array(fb.indptr, np.int64), np.array(fb.ids, np.int64), np.array(fb.tf, np.float64)


def q_arrays(fb):
    return np.array(fb.indptr, np.int64), np.array(fb.ids, np.int64), np.array(fb.tf, np.float64), np.array(fb.oov, np.float64)


def q_block(qa, lo, hi):
    ip, ids, tf, oov = qa
    a, b = ip[lo], ip[hi]
    return ip[lo:hi + 1] - a, ids[a:b], tf[a:b], oov[lo:hi]


def range_block(res, lo, hi):
    ip = res[0]
    a, b = int(ip[lo]), int(ip[hi])
    return (ip[lo:hi + 1],) + tuple(x[a:b] for x in res[1:])


def set_env(monkeypatch, env):
    for k, v in env.items():
        monkeypatch.setenv(k, v)


def query_flags(ix, fb):
    """Per query of ``fb`` (original order) its class: 0 scanned, 1 null, 2 irregular (K1a + selection)."""
    ix.upload_queries(fb)
    qperm, flags = ix.query_order(fb.n)
    out = np.empty(fb.n, np.uint8)
    out[qperm] = flags
    return out


def corpus_common_unigrams(texts):
    common = None
    for t in texts:
        f = {w for w in O.features(t) if " " not in w}
        common = f if common is None else common & f
    return sorted(common)


class BenchCorpus:
    """Case A: rows [0, 2M) of the bench corpus stream, its index, and 8,192 bench queries plus the query classes."""

    N, NQ = 2_000_000, 8192

    def __init__(self):
        from kakveda_b200 import GfkbIndex, synth

        t0 = time.perf_counter()
        buf, off = synth.signatures_packed(synth.CORPUS_SEED, 0, self.N)
        self.ix = GfkbIndex()
        fb = self.ix.vocab.featurize_packed(buf, off, 0, grow=True)
        self.rows = csr_arrays(fb)
        self.ix.add_features(fb)
        fb.close()
        self.ix.finalize()
        self.V = len(self.ix.vocab)
        raw = buf.tobytes()
        text = lambda i: raw[off[i]:off[i + 1]].decode()
        sample = [text(i) for i in range(0, self.N, self.N // 2000)]
        univ = corpus_common_unigrams(sample)
        rare = sorted({w for t in sample[:400] for w in O.features(t) if " " not in w} - set(univ))
        self.queries = synth.signatures(synth.QUERY_SEED, 0, self.NQ, dup_of_seed=synth.CORPUS_SEED, dup_rows=self.N)
        self.extra = {"null": "", "oov": "qqzzunseen xxyyq", "universal": " ".join(reversed(univ)),
                      "wide65": " ".join(rare[:65]), "dup0": text(0), "dup_mid": text(self.N // 2 + 1), "dup_last": text(self.N - 1)}
        self.queries = self.queries + list(self.extra.values())
        self.fb = self.ix.vocab.featurize(self.queries, grow=False)
        self.qa = q_arrays(self.fb)
        self.build_s = time.perf_counter() - t0


@pytest.fixture(scope="module")
def bench_corpus(lib):
    return BenchCorpus()


TFIDF_PATHS = {   # name -> (environment, featuriser)
    "pruned_codes": ({}, "host"),
    "generic_bound": ({"KAKVEDA_B200_GENERIC_BOUND": "1"}, "host"),
    "recomputed_bounds": ({"KAKVEDA_B200_BOUND_CODES": "0"}, "host"),
    "exhaustive": ({"KAKVEDA_B200_NO_PRUNE": "1"}, "host"),
    "device_featuriser": ({"KAKVEDA_B200_FEATURIZE": "device"}, "device"),
}


@gpu
def test_bench_corpus_every_query_every_path(bench_corpus, monkeypatch):
    """Case A: k = 16 and 32 of every query on every path, K1a of 32 queries over all rows, threshold search at three
    thresholds (host and device results), all against one oracle pass per query block."""
    bc = bench_corpus
    ix, n, nq = bc.ix, bc.N, len(bc.queries)
    q = bc.queries
    flags = query_flags(ix, bc.fb)
    at = lambda name: q.index(bc.extra[name])
    assert flags[at("null")] == 1 and flags[at("oov")] == 1
    assert flags[at("universal")] == 0 and flags[at("wide65")] == 2, flags[[at("universal"), at("wide65")]]
    uq = q_block(bc.qa, at("universal"), at("universal") + 1)[1]
    assert len(uq) >= 4 and np.all(ix.local_df()[uq] == n), "the universal-only query holds a feature that is not in every row"
    assert ix.layout()["universal_features"] >= len(uq)
    n_skipped = int((flags != 0).sum())

    results, lays = {}, {}
    for k in (16, 32):
        for name, (env, feat) in TFIDF_PATHS.items():
            with monkeypatch.context() as m:
                set_env(m, env)
                results[name, k] = ix.topk(q, k) if feat == "device" else ix.topk_features(bc.fb, k)
                lays[name, k] = ix.layout()
        base = lays["pruned_codes", k]
        assert base["pairs_passed_bound"] > 0, base
        assert 0 < lays["recomputed_bounds", k]["pairs_passed_bound"] <= base["pairs_passed_bound"]
        assert lays["generic_bound", k]["pairs_passed_bound"] == base["pairs_passed_bound"]
        assert lays["exhaustive", k]["pairs_passed_bound"] == 0
        assert lays["exhaustive", k]["pairs_scored"] >= (nq - n_skipped) * base["chunks"]
        assert lays["device_featuriser", k]["pairs_passed_bound"] == base["pairs_passed_bound"]
    thetas = (0.5, 0.8, 0.95)
    ranges = {}
    for th in thetas:
        ranges[th, "host"] = ix.range_features(bc.fb, th)
        assert ix.layout()["pairs_passed_bound"] > 0
        ranges[th, "device"] = ix.range_features(bc.fb, th, device_out=True)
    k1a_q = list(range(0, bc.NQ, bc.NQ // 26))[:26] + [at(x) for x in ("null", "oov", "universal", "wide65", "dup0", "dup_mid")]
    k1a = {i: ix.score_features(*q_block(bc.qa, i, i + 1)[1:3], float(bc.qa[3][i])) for i in k1a_q}

    orc = T.SparseOracle(*bc.rows, bc.V, device="cuda")
    for lo in range(0, nq, QBLOCK):
        hi = min(nq, lo + QBLOCK)
        o = orc.tfidf_scores(*q_block(bc.qa, lo, hi))
        for (name, k), (s, r) in results.items():
            try:
                check_topk_device(s[lo:hi], r[lo:hi], o, k, RTOL32, first=lo)
            except AssertionError as e:
                raise AssertionError(f"path {name}, k = {k}: {e}") from None
        for (th, where), res in ranges.items():
            try:
                check_range_device(*range_block(res, lo, hi), o, th, RTOL32, first=lo)
            except AssertionError as e:
                raise AssertionError(f"range θ = {th} ({where} results): {e}") from None
        for i in range(lo, hi):
            if i in k1a:
                np.testing.assert_allclose(k1a[i], o[i - lo].cpu().numpy(), rtol=RTOL64, atol=1e-15, err_msg=f"K1a query {i}")
    s, r = results["pruned_codes", 32]
    for name in ("dup0", "dup_mid", "dup_last"):   # a stored row as the query: rank 1 at score 1
        assert abs(s[at(name), 0] - 1.0) < 1e-6, (name, s[at(name)])


@gpu
def test_bench_corpus_deletion_and_label_filters(bench_corpus):
    """Case A, deletion + filter variant: 1 % of the rows at random and a contiguous 5 % block deleted, a
    statistics-only finalize; unfiltered and label-filtered top-k and threshold search against the oracle with N and df
    counted over the live rows and the labels masked."""
    bc = bench_corpus
    ix, n = bc.ix, bc.N
    rng = np.random.default_rng(2024)
    dead = np.unique(np.r_[rng.choice(n, n // 100, replace=False), np.arange(700_000, 700_000 + n // 20)])
    ix.delete_rows(dead)
    ix.finalize()
    assert ix.last_finalize_kind == 2 and ix.n_live_rows == n - len(dead)
    labels = rng.integers(0, 8, n).astype(np.int32)
    ix.set_row_labels(labels)
    nq = 2048
    sub = bc.ix.vocab.featurize(bc.queries[:nq - 3] + [bc.extra["null"], bc.extra["dup0"], bc.extra["wide65"]], grow=False)
    qa = q_arrays(sub)
    qlab = rng.integers(-1, 8, nq).astype(np.int32)
    out = {}
    for k in (16, 32):
        out["all", k] = ix.topk_features(sub, k)
        assert ix.layout()["pairs_passed_bound"] > 0
        out["labels", k] = ix.topk_features(sub, k, labels=qlab)
        assert ix.layout()["pairs_passed_bound"] > 0
    rng_all = ix.range_features(sub, 0.8)
    rng_lab = ix.range_features(sub, 0.8, labels=qlab)
    live = ~ix.deleted_mask()
    assert np.array_equal(np.flatnonzero(~live), dead)
    orc = T.SparseOracle(*bc.rows, bc.V, device="cuda", live=live, labels=labels)
    for lo in range(0, nq, QBLOCK):
        hi = min(nq, lo + QBLOCK)
        blk = q_block(qa, lo, hi)
        o = orc.tfidf_scores(*blk)
        ol = orc.tfidf_scores(*blk, query_labels=qlab[lo:hi])
        for k in (16, 32):
            check_topk_device(*(x[lo:hi] for x in out["all", k]), o, k, RTOL32, first=lo)
            check_topk_device(*(x[lo:hi] for x in out["labels", k]), ol, k, RTOL32, first=lo)
        check_range_device(*range_block(rng_all, lo, hi), o, 0.8, RTOL32, first=lo)
        check_range_device(*range_block(rng_lab, lo, hi), ol, 0.8, RTOL32, first=lo)


@gpu
def test_headline_shard_with_global_statistics(lib):
    """Case B: the last of 8 row shards of the 10M-row headline, rows [8.75M, 10M) with row_base set, global N = 10M and
    the df of all 10M rows (the other rows featurised in slices with the same vocabulary)."""
    from kakveda_b200 import GfkbIndex, Vocabulary, synth

    N, lo_row, n = 10_000_000, 8_750_000, 1_250_000
    vocab = Vocabulary()
    buf, off = synth.signatures_packed(synth.CORPUS_SEED, lo_row, n)
    fb = vocab.featurize_packed(buf, off, 0, grow=True)
    rows = csr_arrays(fb)
    ix = GfkbIndex(row_base=lo_row, vocab=vocab)
    ix.add_features(fb)
    fb.close()
    df = np.bincount(rows[1], minlength=len(vocab)).astype(np.int64)
    t0 = time.perf_counter()
    for a in range(0, lo_row, n):
        b2, o2 = synth.signatures_packed(synth.CORPUS_SEED, a, min(n, lo_row - a))
        f2 = vocab.featurize_packed(b2, o2, 0, grow=True)
        ids = np.asarray(f2.ids)
        df = np.concatenate([df, np.zeros(len(vocab) - len(df), np.int64)])
        df += np.bincount(ids, minlength=len(vocab))
        f2.close()
    stats_s = time.perf_counter() - t0
    ix.set_global_df(df.astype(np.uint32), N)
    ix.finalize()
    V = len(vocab)
    nq, k = 2048, 32
    queries = synth.signatures(synth.QUERY_SEED, 0, nq - 2, dup_of_seed=synth.CORPUS_SEED, dup_rows=N) + \
        [synth.signatures(synth.CORPUS_SEED, lo_row + 5, 1)[0], ""]
    qfb = vocab.featurize(queries, grow=False)
    qa = q_arrays(qfb)
    res = {kk: ix.topk_features(qfb, kk) for kk in (16, k)}
    assert ix.layout()["pairs_passed_bound"] > 0
    rr = ix.range_features(qfb, 0.8)
    k1a = {i: ix.score_features(*q_block(qa, i, i + 1)[1:3], float(qa[3][i])) for i in (0, 1, 2, 100, nq - 2)}
    orc = T.SparseOracle(*rows, V, device="cuda", df=df, n_global=N)
    for lo in range(0, nq, QBLOCK):
        hi = min(nq, lo + QBLOCK)
        o = orc.tfidf_scores(*q_block(qa, lo, hi))
        for kk, (s, r) in res.items():
            g = np.where(r[lo:hi] >= 0, r[lo:hi] - lo_row, -1)   # global rows -> local
            check_topk_device(s[lo:hi], g, o, kk, RTOL32, first=lo)
        ip, r2, s2 = range_block(rr, lo, hi)
        check_range_device(ip, r2 - lo_row, s2, o, 0.8, RTOL32, first=lo)
        for i in range(lo, hi):
            if i in k1a:
                np.testing.assert_allclose(k1a[i], o[i - lo].cpu().numpy(), rtol=RTOL64, atol=1e-15, err_msg=f"K1a query {i}")
    assert res[k][1][nq - 2, 0] == lo_row + 5 or res[k][0][nq - 2, 0] == res[k][0][nq - 2, 1]
    print(f"case B: global statistics of {lo_row} other rows in {stats_s:.1f} s")


# -- case C ------------------------------------------------------------------------------------------------------------

def amax_of(n_total):
    """classify_queries' largest query weight a = (ln(N + 2) + 1)^2, same float64 operations."""
    return (math.log(float(n_total + 2)) + 1.0) ** 2


def classify(qfeats, tfmax, univ, amax):
    """classify_queries' regular (0) / irregular (2) decision for a query of known features [(id, tf)]."""
    feats, s_dot, s_corr, wmax = 0, 0.0, 0.0, 0.0
    for t, f in qfeats:
        if univ[t]:
            continue
        feats += 1
        tm = float(tfmax[t])
        s_dot += float(f) * tm
        s_corr += tm * tm
        wmax = max(wmax, float(f))
    return 2 if (feats > 64 or s_dot * amax >= 1073741824.0 or s_corr * 32.0 >= 1073741824.0 or wmax * amax > 60000.0) else 0


@gpu
@pytest.mark.parametrize("n_global", ["local", 100_000_000, 2**31 - 1])
def test_largest_idf_classify_limits(lib, n_global):
    """Case C: global N up to 2^31 - 1 with df = the local df, so a df = 1 feature gets the largest idf; crafted rows
    with tf up to 65535 on rare, mid-frequency and frequent features; queries just below and just above every
    classify_queries limit (64 / 65 features, s_dot amax against 2^30, wmax amax against 60000).  Asserts the class
    each query got, and both paths against the oracle."""
    from kakveda_b200 import GfkbIndex, synth
    from kakveda_b200.similarity import ArrayBatch

    n_syn = 20_000
    ix = GfkbIndex()
    names = [f"cxh{i}" for i in range(16)] + [f"cxp{i}" for i in range(65)] + ["cxw", "cxrare"]
    buf, off = synth.signatures_packed(synth.CORPUS_SEED, 0, n_syn)
    fb = ix.vocab.featurize_packed(buf, off, 0, grow=True)
    syn = csr_arrays(fb)
    ix.add_features(fb)
    fb.close()
    ix.vocab.featurize([" ".join(names)], grow=True).close()
    wfb = ix.vocab.featurize(names, grow=False)
    fid = {w: int(wfb.ids[wfb.indptr[i]]) for i, w in enumerate(names)}
    wfb.close()
    V = len(ix.vocab)
    df_syn = np.bincount(syn[1], minlength=V)
    mid = int(np.argmin(np.abs(df_syn - 100)))
    freq = int(np.argmin(np.abs(df_syn - n_syn // 3)))
    # universal features of the synthetic rows (every row, same tf): crafted rows hold them too, with that tf
    tfmin = np.full(V, np.inf)
    tfmax_s = np.zeros(V)
    np.minimum.at(tfmin, syn[1], syn[2])
    np.maximum.at(tfmax_s, syn[1], syn[2])
    univ_ids = np.flatnonzero((df_syn == n_syn) & (tfmin == tfmax_s))
    craft = [
        [(fid["cxrare"], 65535)],                                        # rare (df 1), tf 65535
        [(mid, 65535), (freq, 3)],                                       # mid-frequency feature, tf 65535
        [(freq, 65535)],                                                 # frequent feature, tf 65535
        [(fid["cxh%d" % i], 1400) for i in range(16)],                   # the s_dot set: tfmax 1400 each
        [(fid["cxh%d" % i], 1) for i in range(0, 16, 2)],
        [(fid["cxw"], 1)], [(fid["cxw"], 1), (fid["cxh0"], 2)],           # the wmax feature: tfmax 1
        [(fid["cxp%d" % i], 1) for i in range(65)],                      # the wide row
        [(fid["cxp%d" % i], 2) for i in range(0, 65, 5)],
    ]
    craft = [sorted(dict(r + [(int(u), int(tfmax_s[u])) for u in univ_ids]).items()) for r in craft]
    cip = np.r_[0, np.cumsum([len(r) for r in craft])].astype(np.int64)
    ix.add_features(ArrayBatch(cip, np.array([t for r in craft for t, _ in r]), np.array([f for r in craft for _, f in r])))
    n = n_syn + len(craft)
    ip = np.r_[syn[0], syn[0][-1] + cip[1:]]
    ids = np.r_[syn[1], [t for r in craft for t, _ in r]]
    tfs = np.r_[syn[2], [f for r in craft for _, f in r]]
    df = np.bincount(ids, minlength=V)
    N = n if n_global == "local" else n_global
    ix.set_global_df(df.astype(np.uint32), N)
    ix.finalize()
    lay = ix.layout()
    assert lay["universal_features"] > 0 and lay["rows"] == n and lay["chunks"] >= 512, lay   # 512 chunks: pruned
    tfmax = np.zeros(V)
    np.maximum.at(tfmax, ids, tfs)
    univ = np.zeros(V, bool)
    univ[univ_ids] = True
    amax = amax_of(N)

    # queries [(id, tf)], each with the class it must get
    def sdot_query(total):
        f = [total // 16 + (1 if i < total % 16 else 0) for i in range(16)]
        return [(fid["cxh%d" % i], f[i]) for i in range(16)]

    wlim = int(60000.0 // amax)
    while wlim * amax > 60000.0:
        wlim -= 1
    sdot_lim = next(s for s in range(1, 16 * wlim + 1) if classify(sdot_query(s), tfmax, univ, amax) == 2)
    assert classify(sdot_query(sdot_lim - 1), tfmax, univ, amax) == 0 and max(f for _, f in sdot_query(sdot_lim)) <= wlim
    qs = {
        "wide64": ([(fid["cxp%d" % i], 1) for i in range(64)], 0),
        "wide65": ([(fid["cxp%d" % i], 1) for i in range(65)], 2),
        "sdot_under": (sdot_query(sdot_lim - 1), 0),
        "sdot_over": (sdot_query(sdot_lim), 2),
        "wmax_under": ([(fid["cxw"], wlim)], 0),
        "wmax_over": ([(fid["cxw"], wlim + 1)], 2),
        "rare_tf65535": ([(fid["cxrare"], 1)], 2),
        "mid_freq": ([(mid, 2), (freq, 1)], 2),
        "rare_and_wide": ([(fid["cxrare"], 1)] + [(fid["cxp%d" % i], 1) for i in range(10)], 2),
    }
    syn_q = synth.queries(40, n_syn)
    sfb = ix.vocab.featurize(syn_q, grow=False)
    sqa = q_arrays(sfb)
    sfb.close()
    qlist = [sorted(v[0]) for v in qs.values()]
    for i in range(len(syn_q)):
        a, b = sqa[0][i], sqa[0][i + 1]
        qlist.append(list(zip(sqa[1][a:b].tolist(), sqa[2][a:b].astype(int).tolist())))
    want_cls = [v[1] for v in qs.values()] + [classify(x, tfmax, univ, amax) for x in qlist[len(qs):]]
    qip = np.r_[0, np.cumsum([len(x) for x in qlist])].astype(np.int64)
    qb = ArrayBatch(qip, np.array([t for x in qlist for t, _ in x]), np.array([f for x in qlist for _, f in x]),
                    np.r_[np.zeros(len(qs)), sqa[3]])
    got_cls = query_flags(ix, qb)
    assert got_cls.tolist() == want_cls, dict(zip(list(qs) + [f"syn{i}" for i in range(len(syn_q))], got_cls.tolist()))
    res = {k: ix.topk_features(qb, k) for k in (16, 32)}
    rr = ix.range_features(qb, 0.5)
    orc = T.SparseOracle(ip, ids, tfs, V, device="cuda", df=df, n_global=N)
    o = orc.tfidf_scores(qb.indptr, qb.ids.astype(np.int64), qb.tf.astype(np.float64), qb.oov)
    for k, (s, r) in res.items():
        check_topk_device(s, r, o, k, RTOL32)
    check_range_device(*rr, o, 0.5, RTOL32)
    for i, (name, _) in enumerate(qs.items()):   # the crafted row each crafted query targets ranks first
        assert res[32][0][i, 0] > 0, name
    for i in range(len(qlist)):
        a, b = qip[i], qip[i + 1]
        k1a = ix.score_features(qb.ids[a:b], qb.tf[a:b], float(qb.oov[i]))
        np.testing.assert_allclose(k1a, o[i].cpu().numpy(), rtol=RTOL64, atol=1e-15, err_msg=f"K1a query {i}")


# -- case D ------------------------------------------------------------------------------------------------------------

@gpu
def test_jaccard_bench_shape_exact(lib):
    """Case D: 1M Zipf token sets (64 draws over 2^20 tokens, as the benchmark) and 2,048 queries, a quarter of them
    stored sets and some stored sets repeated: top-16 / top-32 bit-exact in the oracle's stable order with exact
    (inter, union), and threshold search at 0.5 and 0.9 exactly the oracle's pair set and counts."""
    from kakveda_b200 import GfkbIndex, JaccardIndex

    n, nq, V = 1_000_000, 2048, 1 << 20
    rng = np.random.default_rng(77)
    draws = np.minimum(rng.zipf(1.2, size=(n + nq, 64)) - 1, V - 1).astype(np.int64)
    draws[n:n + nq // 4] = draws[rng.choice(n, nq // 4, replace=False)]      # stored sets as queries
    draws[rng.choice(n, 300, replace=False)] = draws[12345]                   # one set stored 301 times
    draws[n + nq // 4] = draws[12345]
    draws.sort(axis=1)
    keep = np.ones(draws.shape, dtype=bool)
    keep[:, 1:] = draws[:, 1:] != draws[:, :-1]
    ip = np.r_[0, np.cumsum(keep.sum(axis=1))].astype(np.int64)
    ids = draws[keep]
    del draws, keep
    jx = JaccardIndex(V)
    jx.add_csr(ip[:n + 1], ids[:ip[n]].astype(np.uint32))
    jx.finalize()
    qip, qid = ip[n:] - ip[n], ids[ip[n]:]
    assert np.diff(qip).max() <= 64          # every query fits a query table: K3, no fallback
    out = {}
    for k in (16, 32):
        out[k] = jx.topk_csr(qip, qid.astype(np.uint32), k)
        launches = GfkbIndex.layout(jx)["kernel_launches"]
        jx.topk_csr(qip[:33], qid[:qip[32]].astype(np.uint32), k)
        assert GfkbIndex.layout(jx)["kernel_launches"] == launches, "a query left K3 (K1a + selection add launches)"
    ranges = {th: jx.range_csr(qip, qid.astype(np.uint32), th) for th in (0.5, 0.9)}
    orc = T.SparseOracle(ip[:n + 1], ids[:ip[n]], np.ones(int(ip[n])), V, device="cuda")
    B = 128
    for lo in range(0, nq, B):
        hi = min(nq, lo + B)
        I, U = orc.jaccard_counts(*q_block((qip, qid, np.ones(len(qid)), np.zeros(nq)), lo, hi)[:2])
        ratio = torch.where(U > 0, I / U.clamp(min=1), torch.zeros_like(I))
        for k, (s, r, gi, gu) in out.items():
            rt = torch.as_tensor(r[lo:hi], device="cuda")
            assert torch.equal(torch.as_tensor(gi[lo:hi], device="cuda").double(), I.gather(1, rt)), (k, lo)
            assert torch.equal(torch.as_tensor(gu[lo:hi], device="cuda").double(), U.gather(1, rt)), (k, lo)
            exact = torch.as_tensor(gi[lo:hi] / np.maximum(gu[lo:hi], 1), device="cuda")
            check_topk_device(exact, r[lo:hi], ratio, k, 0.0, first=lo)        # rtol 0: the exact stable order
            check_topk_device(s[lo:hi], r[lo:hi], ratio, k, 1e-6, 1e-7, first=lo)
        for th, res in ranges.items():
            check_jaccard_range_device(*range_block(res, lo, hi), I, U, th, first=lo)
    dup = out[32][1][nq // 4]
    assert dup[0] == 12345 or np.all(out[32][0][nq // 4] == 1.0)


# -- case E ------------------------------------------------------------------------------------------------------------

@gpu
def test_dense_bench_shape(lib):
    """Case E: 1M x 768 bf16 rows, 2,048 queries (half of them a stored row plus noise), top-32 from host and device
    queries, threshold search at 0.8 (host and device), and a self-join top-32 of the first 4,096 rows."""
    from kakveda_b200 import DenseIndex

    n, d, nq, k = 1_000_000, 768, 2048, 32
    g = torch.Generator(device="cuda").manual_seed(5)
    C = torch.randn((n, d), generator=g, device="cuda").to(torch.bfloat16)
    Q = torch.randn((nq, d), generator=g, device="cuda")
    src = torch.randint(0, n, (nq // 2,), generator=g, device="cuda")
    Q[: nq // 2] = C[src].float() + 0.35 * torch.randn((nq // 2, d), generator=g, device="cuda")
    Q[nq // 2] = 0
    Qb = Q.to(torch.bfloat16).contiguous()
    dx = DenseIndex(d)
    dx.add_device(C)
    dx.finalize()
    host = dx.topk(Qb.float().cpu().numpy(), k)
    splits = dx.last_timing()[1]
    assert splits > 1, splits
    dev = dx.topk_device(Qb, k)
    r_host = dx.range(Qb.float().cpu().numpy(), 0.8)
    r_dev = dx.range_device(Qb, 0.8, device_out=True)
    sj = dx.selfjoin_topk(k, 0, 4096)
    rt = dense_rtol(d)
    C64 = T.bf16_round(C)
    C64n = torch.sqrt((C64 * C64).sum(1))
    B = 256

    def cosine(Qblk):
        q64 = T.bf16_round(Qblk)
        qn = torch.sqrt((q64 * q64).sum(1))
        den = qn[:, None] * C64n[None, :]
        return torch.where(den > 0, (q64 @ C64.T) / torch.where(den > 0, den, torch.ones_like(den)), torch.zeros_like(den))

    n_pairs = 0
    for lo in range(0, nq, B):
        hi = min(nq, lo + B)
        o = cosine(Qb[lo:hi])
        check_topk_device(host[0][lo:hi], host[1][lo:hi], o, k, rt, DENSE_ATOL, first=lo)
        check_topk_device(dev[0][lo:hi], dev[1][lo:hi], o, k, rt, DENSE_ATOL, first=lo)
        check_range_device(*range_block(r_host, lo, hi), o, 0.8, rt, DENSE_ATOL, first=lo)
        check_range_device(*range_block(r_dev, lo, hi), o, 0.8, rt, DENSE_ATOL, first=lo)
        n_pairs += int((o >= 0.8).sum())
    assert n_pairs >= nq // 4, n_pairs
    for lo in range(0, 4096, B):
        o = cosine(C[lo:lo + B])
        o[torch.arange(B, device="cuda"), torch.arange(lo, lo + B, device="cuda")] = -math.inf
        check_topk_device(sj[0][lo:lo + B], sj[1][lo:lo + B], o, k, rt, DENSE_ATOL, first=lo)
    np.testing.assert_allclose(T.dense_cosine(Qb[:4].cpu(), C[:1000].cpu()).numpy(), cosine(Qb[:4])[:, :1000].cpu().numpy(),
                               rtol=1e-12, atol=1e-15)
