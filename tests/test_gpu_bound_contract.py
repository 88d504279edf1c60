"""The bound contract of the pruned TF-IDF top-k (K1b), checked at every (query, chunk) pair.

The pruned path is exact only if, for every regular query q and every chunk c (scan positions 32c .. 32c + 31),

    the bound bound pass 0 stores as an 8-bit code, and the float bound bound pass 1 compares,
    never fall below s_max(q, c) = the best exact score of a LIVE row of c for q.

``kv_debug_bound_codes`` exports what bound pass 0 produced on the headline path (the specialised instantiation
``tfidf_bound_kernel<true>``, or the generic one under KAKVEDA_B200_GENERIC_BOUND=1): the codes, the threshold codes
the candidate scan compared them with, the query constants, the chunk minima and the scan layout's row order.  A
float64 oracle (scipy sparse products, DESIGN §3) gives s_max.  Per case:

1. codes: code >= min(255, ceil(250 s_max (1 - 1e-6))) at every regular slot and chunk; a chunk without a live row
   holding a feature has code 0;
2. float bounds: xs 1.0005 / sqrt(|q|^2 (minB + corrS)) >= s_max (1 + 1e-5) with xs from kv_debug_bound_numerators;
   and the query constants err outwards: dotS >= the exact dotU, corrS <= the exact corrU + corrS (a one-ulp error in
   the wrong direction hides under the 0.05 % slack in every score, so it is checked on the constants themselves);
3. the fused selection of the candidate scan: pairs_passed_bound / records_written equal the counts of
   code >= threshold code over the exported arrays;
4. the top-k of the run equals the exhaustive scan and the recomputed-bound path bit for bit, and the exhaustive
   top-k passes ``check_topk_strict`` against the oracle;
5. bound pass 1 at tight thresholds: a threshold search at exactly the float32 score of a query's 5th row returns the
   exhaustive search's bits and every top-k row that reaches the threshold.

Failures name the (slot, query, chunk) pair and the terms of its bound.  ``test_checker_rejects_faults`` shows on the
CPU that the checks reject hand-made faults of each kind.
"""
import ctypes as C

import numpy as np
import pytest

from oracle import tfidf_oracle as O
from test_gpu_topk_edges import RTOL32, check_topk_strict

gpu = pytest.mark.gpu

K = 16
UBQ_SCALE = 250.0
PRUNE_SLACK = 1.0005
NO_CANDIDATE = 256          # threshold code of a query that takes no candidate
GENERIC = {"KAKVEDA_B200_GENERIC_BOUND": "1"}
EXHAUSTIVE = {"KAKVEDA_B200_NO_PRUNE": "1"}
CODES_OFF = {"KAKVEDA_B200_BOUND_CODES": "0"}
SLAB = 1024                 # queries per oracle slab ([SLAB, N] float64 at a time)


# ---------------------------------------------------------------------------------------------------------------------
# float64 oracle
# ---------------------------------------------------------------------------------------------------------------------

class ExactScores:
    """Exact [Q, N] scores per DESIGN §3 for one index state.

    rows: (indptr, ids, tf) of the local rows (ids < V = len(df)); n_total, df: the statistics the index uses (global
    ones for a shard); mode 0 (refit per query) or 2 (fitted on the corpus: idf from N and df alone, features with
    df 0 and out-of-vocabulary ones ignored); live: bool [N] (deleted rows score -inf)."""

    def __init__(self, rows, n_total, df, mode, live=None):
        import scipy.sparse as sp

        ip, ids, tf = (np.asarray(a) for a in rows)
        self.n, self.V = len(ip) - 1, len(df)
        df = np.asarray(df, dtype=np.float64)
        if mode == 0:
            idf_b = np.log((n_total + 2.0) / (df + 1.0)) + 1.0
            idf_q = np.log((n_total + 2.0) / (df + 2.0)) + 1.0
            self.a, self.d = idf_q ** 2, idf_q ** 2 - idf_b ** 2
            self.idf0 = np.log((n_total + 2.0) / 2.0) + 1.0
        elif mode == 2:
            idf_b = np.log((n_total + 1.0) / (df + 1.0)) + 1.0
            self.a = np.where(df > 0, idf_b ** 2, 0.0)
            self.d = np.zeros_like(df)
            self.idf0 = 0.0
        else:
            raise ValueError(mode)
        self.C1 = sp.csr_matrix((np.asarray(tf, np.float64), np.asarray(ids, np.int64), np.asarray(ip, np.int64)),
                                shape=(self.n, max(self.V, 1)))
        self.C2 = self.C1.multiply(self.C1).tocsr()
        self.B = np.asarray(self.C2 @ np.resize(idf_b ** 2, max(self.V, 1))).ravel()
        self.live = np.ones(self.n, bool) if live is None else np.asarray(live, bool)
        self.featured = self.live & (np.diff(ip) > 0)     # live rows holding a feature
        # properties of the layout rows (deleted ones included): largest tf, and the universal features (in every row
        # with one tf), which the bound folds into dotS / corrS with that tf
        Vz = max(self.V, 1)
        ids, tf = np.asarray(ids, np.int64), np.asarray(tf, np.int64)
        self.tfmax = np.zeros(Vz, np.int64)
        np.maximum.at(self.tfmax, ids, tf)
        tfmin = np.full(Vz, np.iinfo(np.int64).max)
        np.minimum.at(tfmin, ids, tf)
        self.univ = (np.bincount(ids, minlength=Vz) == self.n) & (tfmin == self.tfmax) & (self.n > 0)

    def query_terms(self, queries, lo=0, hi=None):
        """Exact float64 (dotU, corrU + corrS) of queries lo .. hi - 1: the universal features' dot product, and every
        known feature's d(t) at its largest tf (a universal one at its tf)."""
        import scipy.sparse as sp

        qip, qids, qtf, _ = (np.asarray(a) for a in queries)
        hi = len(qip) - 1 if hi is None else hi
        a0, a1 = int(qip[lo]), int(qip[hi])
        ids, tf = qids[a0:a1].astype(np.int64), qtf[a0:a1].astype(np.float64)
        row = np.repeat(np.arange(hi - lo), np.diff(qip[lo:hi + 1]))
        known = ids < self.V
        Qm = sp.csr_matrix((tf[known], (row[known], ids[known])), shape=(hi - lo, max(self.V, 1)))
        a, d = np.resize(self.a, max(self.V, 1)), np.resize(self.d, max(self.V, 1))
        dotU = np.asarray(Qm @ np.where(self.univ, self.tfmax * a, 0.0)).ravel()
        corr = np.asarray((Qm > 0).astype(np.float64) @ (self.tfmax.astype(np.float64) ** 2 * d)).ravel()
        return dotU, corr

    def scores(self, queries, lo=0, hi=None):
        """float64 [hi - lo, N] of queries (indptr, ids, tf, oov_tf2) lo .. hi - 1; ids >= V count as out of vocabulary."""
        import scipy.sparse as sp

        qip, qids, qtf, qoov = (np.asarray(a) for a in queries)
        hi = len(qip) - 1 if hi is None else hi
        a0, a1 = int(qip[lo]), int(qip[hi])
        ids, tf = qids[a0:a1].astype(np.int64), qtf[a0:a1].astype(np.float64)
        ip = qip[lo:hi + 1] - a0
        known = ids < self.V
        row = np.repeat(np.arange(hi - lo), np.diff(ip))
        oov = np.asarray(qoov[lo:hi], np.float64) + np.bincount(row[~known], weights=tf[~known] ** 2, minlength=hi - lo)
        Qm = sp.csr_matrix((tf[known], (row[known], ids[known])), shape=(hi - lo, max(self.V, 1)))
        nq = np.asarray(Qm.multiply(Qm) @ np.resize(self.a, max(self.V, 1))).ravel() + oov * self.idf0 ** 2
        dot = (Qm @ sp.diags(np.resize(self.a, max(self.V, 1))) @ self.C1.T).toarray()
        member = (Qm > 0).astype(np.float64)
        corr = (member @ sp.diags(np.resize(self.d, max(self.V, 1))) @ self.C2.T).toarray()
        den = nq[:, None] * (self.B[None, :] + corr)
        ok = (den > 0) & (dot != 0)
        s = np.where(ok, dot / np.sqrt(np.where(ok, den, 1.0)), 0.0)
        s[:, ~self.live] = -np.inf
        return s


def chunk_max(S, row_at_pos, n_chunks):
    """s_max [Q, n_chunks]: the best score of a row at positions 32c .. 32c + 31 (-inf: no live row)."""
    q, n = S.shape
    P = np.full((q, n_chunks * 32), -np.inf)
    P[:, :n] = S[:, row_at_pos]
    return P.reshape(q, n_chunks, 32).max(axis=2)


def featured_chunks(featured_rows, row_at_pos, n_chunks):
    """bool [n_chunks]: the chunk holds a live row with at least one feature."""
    f = np.zeros(n_chunks * 32, bool)
    f[:len(row_at_pos)] = featured_rows[row_at_pos]
    return f.reshape(n_chunks, 32).any(axis=1)


# ---------------------------------------------------------------------------------------------------------------------
# the checks (pure functions: the CPU self-test feeds them hand-made faults)
# ---------------------------------------------------------------------------------------------------------------------

def need_codes(smax):
    return np.minimum(255.0, np.ceil(UBQ_SCALE * np.maximum(smax, 0.0) * (1.0 - 1e-6)))


def check_codes(codes, nq, smax, featured, slot_query):
    """Check 1.  codes uint8 [Q, n_chunks] by slot, nq float [Q] by slot, smax [Q, n_chunks] by slot."""
    reg = nq > 0
    need = need_codes(smax)
    low = reg[:, None] & (codes.astype(np.float64) < need)
    if low.any():
        s, c = np.argwhere(low)[np.argmax((need - codes)[low])]
        raise AssertionError(f"{int(low.sum())} bound codes below ceil(250 s_max); worst: slot {s} (query "
                             f"{slot_query[s]}) chunk {c}: code {codes[s, c]} < {int(need[s, c])} (s_max {smax[s, c]!r})")
    empty = reg[:, None] & ~featured[None, :] & (codes != 0)
    if empty.any():
        s, c = np.argwhere(empty)[0]
        raise AssertionError(f"{int(empty.sum())} non-zero codes on chunks without a live row holding a feature; first: "
                             f"slot {s} (query {slot_query[s]}) chunk {c}: code {codes[s, c]}")


def float_bounds(xs, q_terms, minB):
    """ub [Q, n_chunks] float64 of what bound pass 1 compares (inf where minB + corrS <= 0)."""
    nq, corrS = q_terms[:, 0].astype(np.float64), q_terms[:, 3].astype(np.float64)
    den = minB.astype(np.float64)[None, :] + corrS[:, None]
    with np.errstate(divide="ignore", invalid="ignore"):
        ub = xs.astype(np.float64) * PRUNE_SLACK / np.sqrt(nq[:, None] * den)
    return np.where(den > 0, ub, np.inf), den


def check_float_bounds(xs, q_terms, minB, smax, slot_query):
    """Check 2."""
    ub, den = float_bounds(xs, q_terms, minB)
    reg = q_terms[:, 0] > 0
    low = reg[:, None] & (den > 0) & (ub < smax * (1.0 + 1e-5))
    if low.any():
        ratio = np.where(low, ub / np.where(smax > 0, smax, 1.0), np.inf)
        s, c = np.unravel_index(np.argmin(ratio), ratio.shape)
        nq, dS, dX, cS = (float(v) for v in q_terms[s])
        raise AssertionError(f"{int(low.sum())} float bounds below s_max (1 + 1e-5); worst: slot {s} (query "
                             f"{slot_query[s]}) chunk {c}: ub {ub[s, c]!r} < s_max {smax[s, c]!r}; xs {float(xs[s, c])!r} "
                             f"(dotS {dS!r} + dotX {dX!r} + R), |q|^2 {nq!r}, minB {float(minB[c])!r}, corrS {cS!r}")


def check_query_terms(q_terms, dotU, corr, slot_query):
    """Check 2b: the query constants err outwards -- dotS >= the exact dotU (numerator), corrS <= the exact corrU +
    corrS (denominator).  The 1e-12 only absorbs the float64 summation order."""
    reg = q_terms[:, 0] > 0
    dS, cS = q_terms[:, 1].astype(np.float64), q_terms[:, 3].astype(np.float64)
    for bad, what in ((reg & (dS < dotU - 1e-12 * np.abs(dotU)), "dotS below the exact dotU"),
                      (reg & (cS > corr + 1e-12 * np.abs(corr)), "corrS above the exact corrU + corrS")):
        if bad.any():
            s = int(np.flatnonzero(bad)[0])
            raise AssertionError(f"{int(bad.sum())} queries with {what}; first: slot {s} (query {slot_query[s]}): dotS "
                                 f"{dS[s]!r} vs {dotU[s]!r}, corrS {cS[s]!r} vs {corr[s]!r}")


def selection_counts(codes, tcode):
    """(pairs, records) of the candidate scan's codes mode: pairs = #{(slot, chunk): code >= tcode < 256}, records =
    #{(32-slot group, chunk): some slot of the group passes}."""
    q, nch = codes.shape
    take = (tcode[:, None] < NO_CANDIDATE) & (codes.astype(np.int32) >= tcode[:, None])
    g = (q + 31) // 32
    pad = np.zeros((g * 32, nch), bool)
    pad[:q] = take
    return int(take.sum()), int(pad.reshape(g, 32, nch).any(axis=1).sum())


def check_selection(codes, tcode, lay):
    pairs, recs = selection_counts(codes, tcode)
    assert (lay["pairs_passed_bound"], lay["records_written"]) == (pairs, recs), \
        f"fused selection: the scan counted {lay['pairs_passed_bound']} pairs / {lay['records_written']} records, " \
        f"the exported codes and threshold codes give {pairs} / {recs}"


def tightness(codes, xs, q_terms, minB, smax):
    """Median and 99.9th percentile of ub / s_max and of code - ceil(250 s_max) over regular pairs with s_max > 0."""
    ub, _ = float_bounds(xs, q_terms, minB)
    m = (q_terms[:, 0] > 0)[:, None] & (smax > 0) & np.isfinite(ub)
    r = (ub / np.where(smax > 0, smax, 1.0))[m]
    d = (codes.astype(np.float64) - np.ceil(UBQ_SCALE * np.maximum(smax, 0.0)))[m]
    if not len(r):
        return {}
    return {"ub/s_max": np.quantile(r, [0.5, 0.999]).round(4).tolist(),
            "code-ceil": np.quantile(d, [0.5, 0.999]).round(2).tolist()}


# ---------------------------------------------------------------------------------------------------------------------
# CPU: the oracle against the closed forms, and the checks against hand-made faults
# ---------------------------------------------------------------------------------------------------------------------

def text_csr(texts, vocab, grow):
    ip, ids, tf, oov = [0], [], [], []
    for t in texts:
        o = 0.0
        for f, c in O.features(t).items():
            j = vocab.setdefault(f, len(vocab)) if grow else vocab.get(f)
            if j is None:
                o += float(c) ** 2
            else:
                ids.append(j)
                tf.append(c)
        ip.append(len(ids))
        oov.append(o)
    return np.array(ip, np.int64), np.array(ids, np.int64), np.array(tf, np.int64), np.array(oov)


def test_oracle_matches_closed_forms():
    """The array oracle against O.score_matrix_closed_form (mode 0) and sklearn's corpus fit (mode 2), on texts with
    empty rows, repeated words, duplicates of stored rows and out-of-vocabulary words."""
    from random import Random

    rnd = Random(3)
    words = [f"w{i}" for i in range(60)]
    corpus = [" ".join(rnd.choice(words) for _ in range(rnd.randint(0, 12))) for _ in range(300)]
    queries = corpus[:20] + ["w1 w2 unseenword", "nothing known here", "", corpus[5] + " w3 w3"]
    vocab = {}
    rows = text_csr(corpus, vocab, True)[:3]
    qs = text_csr(queries, vocab, False)
    df = np.bincount(rows[1], minlength=len(vocab))
    got0 = ExactScores(rows, len(corpus), df, 0).scores(qs)
    np.testing.assert_allclose(got0, O.score_matrix_closed_form(queries, corpus), rtol=0, atol=1e-12)
    got2 = ExactScores(rows, len(corpus), df, 2).scores(qs)
    np.testing.assert_allclose(got2, O.corpus_fit_scores(queries, corpus), rtol=0, atol=1e-12)


def _toy(seed=5, n=256, q=12, V=40):
    """A random index state with an honest bound pass: tight codes and float bounds."""
    rng = np.random.default_rng(seed)
    lens = rng.integers(0, 6, n)
    ip = np.r_[0, np.cumsum(lens)]
    ids = np.concatenate([np.sort(rng.choice(V, l, replace=False)) for l in lens])
    tf = rng.integers(1, 4, len(ids))
    qlens = rng.integers(1, 5, q)
    qip = np.r_[0, np.cumsum(qlens)]
    qids = np.concatenate([np.sort(rng.choice(V, l, replace=False)) for l in qlens])
    qtf = rng.integers(1, 3, len(qids))
    df = np.bincount(ids, minlength=V)
    ex = ExactScores((ip, ids, tf), n, df, 0)
    S = ex.scores((qip, qids, qtf, np.zeros(q)))
    perm = rng.permutation(n)
    nch = n // 32
    smax = chunk_max(S, perm, nch)
    featured = featured_chunks(ex.featured, perm, nch)
    codes = need_codes(smax).astype(np.uint8)
    q_terms = np.zeros((q, 4), np.float32)
    q_terms[:, 0] = rng.uniform(1, 4, q)
    q_terms[:, 3] = rng.uniform(0, 1, q)
    minB = rng.uniform(1, 4, nch).astype(np.float32)
    den = minB[None, :].astype(np.float64) + q_terms[:, 3:4]
    xs = np.maximum(smax, 0) * (1 + 3e-5) * np.sqrt(q_terms[:, :1].astype(np.float64) * den) / PRUNE_SLACK
    return S, perm, smax, featured, codes, q_terms, minB, xs, ex, nch


def test_checker_rejects_faults():
    S, perm, smax, featured, codes, q_terms, minB, xs, ex, nch = _toy()
    sq = np.arange(len(codes))
    check_codes(codes, q_terms[:, 0], smax, featured, sq)             # the honest bound pass passes
    check_float_bounds(xs, q_terms, minB, smax, sq)
    # one code decremented at the tightest pair (code == ceil(250 s_max) > 0)
    bad = codes.copy()
    s, c = np.unravel_index(np.argmax(np.where(codes > 0, smax, -1)), codes.shape)
    bad[s, c] -= 1
    with pytest.raises(AssertionError, match="codes below"):
        check_codes(bad, q_terms[:, 0], smax, featured, sq)
    # the checker reads a row order in which a chunk holds a row of the next chunk (a better one for some query)
    gain = smax[:, 1:] - smax[:, :-1]
    s, c = np.unravel_index(np.argmax(gain), gain.shape)
    assert gain[s, c] > 0.01
    wrong = perm.copy()
    p_best = 32 * (c + 1) + int(np.argmax(S[s, perm[32 * (c + 1):32 * (c + 2)]]))
    wrong[32 * c], wrong[p_best] = perm[p_best], perm[32 * c]
    with pytest.raises(AssertionError, match="codes below"):
        check_codes(codes, q_terms[:, 0], chunk_max(S, wrong, nch), featured_chunks(ex.featured, wrong, nch), sq)
    # a float bound lowered by 1e-4 on one pair
    ub, _ = float_bounds(xs, q_terms, minB)
    s, c = np.unravel_index(np.argmax(smax), smax.shape)
    low = xs.copy()
    low[s, c] *= 1 - 1e-4
    with pytest.raises(AssertionError, match="float bounds below"):
        check_float_bounds(low, q_terms, minB, smax, sq)
    # a non-zero code on a chunk without a live row holding a feature
    empty = codes.copy()
    nofeat = featured.copy()
    nofeat[c] = False
    with pytest.raises(AssertionError, match="non-zero codes"):
        check_codes(empty, q_terms[:, 0], smax, nofeat, sq)
    # query constants one float32 ulp on the wrong side of their exact values
    dotU, corr = ex.query_terms((np.r_[0, 1, 2], np.array([1, 4]), np.array([2, 1]), np.zeros(2)))
    dotU, corr = dotU + np.array([0.0, 3.25]), corr - np.array([0.7, 1.3])   # as if universal features were folded in
    qt = np.ones((2, 4), np.float32)
    qt[:, 1] = np.nextafter(dotU.astype(np.float32), np.float32(np.inf))
    qt[:, 3] = np.nextafter(corr.astype(np.float32), np.float32(-np.inf))
    check_query_terms(qt, dotU, corr, np.arange(2))
    for col, direction in ((1, -np.inf), (3, np.inf)):
        bad = qt.copy()
        bad[1, col] = np.nextafter(np.float32(dotU[1] if col == 1 else corr[1]), np.float32(direction))
        with pytest.raises(AssertionError, match="dotS below|corrS above"):
            check_query_terms(bad, dotU, corr, np.arange(2))
    # selection counts off by one
    tcode = np.full(len(codes), 100, np.int32)
    tcode[3] = NO_CANDIDATE
    pairs, recs = selection_counts(codes, tcode)
    assert pairs > 0 and recs > 0
    check_selection(codes, tcode, {"pairs_passed_bound": pairs, "records_written": recs})
    for lay in ({"pairs_passed_bound": pairs + 1, "records_written": recs},
                {"pairs_passed_bound": pairs - 1, "records_written": recs},
                {"pairs_passed_bound": pairs, "records_written": recs + 1}):
        with pytest.raises(AssertionError, match="fused selection"):
            check_selection(codes, tcode, lay)


# ---------------------------------------------------------------------------------------------------------------------
# GPU cases
# ---------------------------------------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def lib(built_lib):
    from kakveda_b200 import _capi

    assert _capi.load().kv_device_count() > 0, "GPU tests need a CUDA device"
    return _capi.load()


@pytest.fixture(scope="module")
def sm_count(lib):
    import torch

    return torch.cuda.get_device_properties(0).multi_processor_count


def _p(a, ct):
    return a.ctypes.data_as(C.POINTER(ct))


def bound_codes(ix, n_q, n_chunks, n_rows):
    from kakveda_b200 import _capi

    codes = np.zeros((n_q, n_chunks), np.uint8)
    sq = np.zeros(n_q, np.int32)
    tcode = np.zeros(n_q, np.int32)
    qt = np.zeros((n_q, 4), np.float32)
    minB = np.zeros(n_chunks, np.float32)
    rap = np.zeros(max(n_rows, 1), np.int32)
    _capi.check(_capi.load().kv_debug_bound_codes(ix._h, K, _p(codes, C.c_uint8), _p(sq, C.c_int32), _p(tcode, C.c_int32),
                                                  _p(qt, C.c_float), _p(minB, C.c_float), _p(rap, C.c_int32)))
    return codes, sq, tcode, qt, minB, rap[:n_rows]


def bound_numerators(ix, n_q, n_chunks):
    from kakveda_b200 import _capi

    xs = np.zeros((n_q, n_chunks), np.float32)
    sq = np.zeros(n_q, np.int32)
    _capi.check(_capi.load().kv_debug_bound_numerators(ix._h, K, _p(xs, C.c_float), _p(sq, C.c_int32)))
    return xs, sq


def csr_rows(ip, ids, tf, rows):
    """The CSR of ``rows`` of (ip, ids, tf)."""
    rows = np.asarray(rows, np.int64)
    lens = np.diff(ip)[rows]
    nip = np.r_[0, np.cumsum(lens)].astype(np.int64)
    take = np.concatenate([np.arange(ip[r], ip[r + 1]) for r in rows]) if len(rows) else np.zeros(0, np.int64)
    return nip, ids[take], tf[take]


def concat_csr(*parts):
    ip, ids, tf, oov = [np.zeros(1, np.int64)], [], [], []
    for p in parts:
        ip.append(p[0][1:] + ip[-1][-1])
        ids.append(np.asarray(p[1], np.int64))
        tf.append(np.asarray(p[2], np.int64))
        oov.append(np.asarray(p[3], np.float64) if len(p) > 3 else np.zeros(len(p[0]) - 1))
    return np.concatenate(ip), np.concatenate(ids), np.concatenate(tf), np.concatenate(oov)


def featurize(vocab, data, grow):
    """(indptr, ids, tf, oov) of texts, or of a packed (buffer, offsets) pair."""
    fb = vocab.featurize(data, grow=grow) if isinstance(data, list) else vocab.featurize_packed(data[0], data[1], 0, grow=grow)
    try:
        return (fb.indptr.copy().astype(np.int64), fb.ids.copy().astype(np.int64), fb.tf.copy().astype(np.int64),
                fb.oov.copy().astype(np.float64))
    finally:
        fb.close()


class Case:
    """An index state, a resident batch (query CSR or a self-join range) and the oracle of that pair.  qmap: the batch
    is distinct[qmap] (the oracle scores each distinct query once)."""

    def __init__(self, name, ix, rows, n_total, df, mode, queries=None, selfjoin=None, live=None, qmap=None):
        self.name, self.ix, self.rows = name, ix, rows
        self.selfjoin = selfjoin                              # (lo, hi): rows lo .. hi - 1 as queries, each excluding itself
        if selfjoin is not None:
            lo, hi = selfjoin
            nip, nids, ntf = csr_rows(*rows, np.arange(lo, hi))
            queries = (nip, nids, ntf, np.zeros(hi - lo))
        self.distinct = queries
        n_d = len(queries[0]) - 1
        self.qmap = np.arange(n_d) if qmap is None else np.asarray(qmap)
        self.queries = queries if qmap is None else csr_rows(*queries[:3], self.qmap) + (queries[3][self.qmap],)
        self.n_q = len(self.qmap)
        self.exact = ExactScores(rows, n_total, df, mode, live)
        self.smax_cache = None

    def upload(self, sub=None):
        from kakveda_b200.similarity import ArrayBatch

        if self.selfjoin is not None:
            lo, hi = self.selfjoin
            lo, hi = (lo, hi) if sub is None else (lo + sub, lo + sub + 1)
            self.ix._selfjoin_upload(lo, hi, False)
            return
        ip, ids, tf, oov = self.queries
        if sub is not None:
            nip, nids, ntf = csr_rows(ip, ids, tf, [sub])
            ip, ids, tf, oov = nip, nids, ntf, oov[[sub]]
        self.ix.upload_queries(ArrayBatch(ip, ids, tf, oov))

    def oracle(self, row_at_pos, n_chunks, exhaustive):
        """s_max [n_q, n_chunks] by original query (cached: the row order is a property of the index state), and the
        strict top-k check of the exhaustive result (first copy of each distinct query) against the oracle."""
        if self.smax_cache is not None:
            assert np.array_equal(self.smax_cache[0], row_at_pos), "the scan layout's row order changed between runs"
            return self.smax_cache[1]
        n_d = len(self.distinct[0]) - 1
        smax = np.zeros((n_d, n_chunks))
        terms = [t[self.qmap] for t in self.exact.query_terms(self.distinct)]
        _, first = np.unique(self.qmap, return_index=True)
        s, r = exhaustive[0][first], exhaustive[1][first]
        for lo in range(0, n_d, SLAB):
            hi = min(n_d, lo + SLAB)
            S = self.exact.scores(self.distinct, lo, hi)
            smax[lo:hi] = chunk_max(S, row_at_pos, n_chunks)  # a self-join row counts: the bound pass knows no exclusion
            if self.selfjoin is not None:
                S[np.arange(hi - lo), self.selfjoin[0] + np.arange(lo, hi)] = -np.inf
            check_topk_strict(s[lo:hi], r[lo:hi], S, K, RTOL32)
        smax = smax[self.qmap]
        self.smax_cache = (row_at_pos.copy(), smax, terms)
        return smax


def run_env(monkeypatch, env, fn):
    with monkeypatch.context() as m:
        for key, v in env.items():
            m.setenv(key, v)
        return fn()


REPORT = {}   # (case, variant) -> codes by slot, for the count of codes the two instantiations disagree on


def check_contract(case, monkeypatch, env):
    """Checks 1-5 on one case under one bound-kernel instantiation; returns the layout of the run."""
    ix = case.ix
    n_chunks, n_rows = ix.layout()["chunks"], ix.n_rows

    def hook():
        case.upload()
        return bound_codes(ix, case.n_q, n_chunks, n_rows) + (ix.layout(), ix.topk_resident_host(case.n_q, K))

    codes, sq, tcode, qt, minB, rap, lay, (s, r) = run_env(monkeypatch, env, hook)
    assert lay["pairs_passed_bound"] > 0 and lay["pool_pages_used"] == 0, ("codes mode did not run", lay)
    assert sorted(sq.tolist()) == list(range(case.n_q))
    # 4: the same batch, exhaustive and with recomputed bounds (pass 1 lists)
    ex = run_env(monkeypatch, EXHAUSTIVE, lambda: ix.topk_resident_host(case.n_q, K))
    assert ix.layout()["pairs_passed_bound"] == 0
    lists = run_env(monkeypatch, CODES_OFF, lambda: ix.topk_resident_host(case.n_q, K))
    assert ix.layout()["pool_pages_used"] > 0
    for name, other in (("exhaustive", ex), ("bound pass 1 lists", lists)):
        assert other[1].tobytes() == r.tobytes() and other[0].tobytes() == s.tobytes(), f"{case.name}: top-k != {name}"
    smax = case.oracle(rap, n_chunks, ex)[sq]
    featured = featured_chunks(case.exact.featured, rap, n_chunks)
    # 1, 3
    check_codes(codes, qt[:, 0], smax, featured, sq)
    check_selection(codes, tcode, lay)
    # 2: the numerators of the same batch (the hook runs the generic instantiation)
    xs, sq2 = bound_numerators(ix, case.n_q, n_chunks)
    assert np.array_equal(sq, sq2)
    check_float_bounds(xs, qt, minB, smax, sq)
    dotU, corr = case.smax_cache[2]
    check_query_terms(qt, dotU[sq], corr[sq], sq)
    # 5: bound pass 1 at the float32 score of the 5th row, one query at a time
    rng = np.random.default_rng(len(case.name))
    cand = np.flatnonzero(s[:, 4] > 0)
    for q in rng.choice(cand, size=min(6, len(cand)), replace=False):
        theta = float(s[q, 4])

        def search():
            case.upload(int(q))
            return ix._range_resident(1, theta)

        got = run_env(monkeypatch, env, search)
        want = run_env(monkeypatch, EXHAUSTIVE, search)
        for g, w in zip(got, want):
            assert g.tobytes() == w.tobytes(), f"{case.name}: range at {theta!r} of query {q} != exhaustive"
        top = s[q] >= np.float32(theta)
        have = dict(zip(got[1].tolist(), got[2].tolist()))
        for row, sc in zip(r[q][top].tolist(), s[q][top].tolist()):
            assert have.get(row) == sc, f"{case.name}: top-k row {row} ({sc!r}) missing from the range at {theta!r}"
    # the two instantiations may round differently; report how many codes differ
    variant = "generic" if env else "specialised"
    by_query = np.empty_like(codes)
    by_query[sq] = codes
    REPORT[case.name, variant] = by_query
    other = REPORT.get((case.name, "specialised" if env else "generic"))
    diff = None if other is None else int((other != by_query).sum())
    print(f"\n[{case.name} {variant}] chunks {n_chunks} queries {case.n_q} pairs {lay['pairs_passed_bound']} "
          f"codes differing between instantiations: {diff}; tightness {tightness(codes, xs, qt, minB, smax)}")
    return lay, codes, sq, minB


# ---- index states ----------------------------------------------------------------------------------------------------

N_A = 60_000          # 1875 chunks: the last 64-chunk block holds 19


@pytest.fixture(scope="module")
def corpus_a(lib):
    from kakveda_b200 import GfkbIndex, synth

    ix = GfkbIndex()
    rows = featurize(ix.vocab, synth.signatures_packed(synth.CORPUS_SEED, 0, N_A), True)
    from kakveda_b200.similarity import ArrayBatch

    ix.add_features(ArrayBatch(*rows[:3]))
    ix.finalize()
    return ix, rows[:3]


def df_of(rows, V, live=None):
    ip, ids, _ = rows
    if live is None:
        return np.bincount(ids, minlength=V)
    keep = np.repeat(live, np.diff(ip))
    return np.bincount(ids[keep], minlength=V)


def queries_a(ix, rows, n=300):
    """n queries: half synthetic, half exact copies of stored rows."""
    from kakveda_b200 import synth

    half = n // 2
    syn = featurize(ix.vocab, synth.signatures_packed(synth.QUERY_SEED, 0, n - half), False)
    dup_rows = np.random.default_rng(11).choice(len(rows[0]) - 1, half, replace=False)
    dup = csr_rows(*rows, dup_rows)
    return concat_csr(syn, dup), dup_rows


def build_case(name, sm_count, corpus_a):
    from kakveda_b200 import GfkbIndex, synth
    from kakveda_b200.similarity import ArrayBatch, Vocabulary

    ixA, rowsA = corpus_a
    V = len(ixA.vocab)
    if name == "A":
        q, dup_rows = queries_a(ixA, rowsA)
        return Case(name, ixA, rowsA, N_A, df_of(rowsA, V), 0, q)
    if name == "B":   # 513 chunks (a one-row last chunk) x 128 queries per SM: one row range per tile, as in the bench
        ix = GfkbIndex()
        rows = featurize(ix.vocab, synth.signatures_packed(synth.CORPUS_SEED, 0, 16_385), True)[:3]
        ix.add_features(ArrayBatch(*rows))
        ix.finalize()
        base, _ = queries_a(ix, rows, 600)
        return Case(name, ix, rows, 16_385, df_of(rows, len(ix.vocab)), 0, base, qmap=np.arange(128 * sm_count) % 600)
    if name == "C":
        return Case(name, ixA, rowsA, N_A, df_of(rowsA, V), 0, adversarial_queries(ixA, rowsA))
    if name in ("D", "D-universal"):
        ix = GfkbIndex()
        texts, qtexts = corpus_d(name == "D-universal")
        rows = featurize(ix.vocab, texts, True)[:3]
        ix.add_features(ArrayBatch(*rows))
        ix.finalize()
        q = featurize(ix.vocab, qtexts, False)
        return Case(name, ix, rows, len(texts), df_of(rows, len(ix.vocab)), 0, q)
    if name in ("E", "E-selfjoin"):
        vocab = Vocabulary.from_keys(ixA.vocab.export_keys())
        ghost = featurize(vocab, ["zzghost zzghostb zzghost"], True)   # vocabulary features no row holds (df 0)
        ix = GfkbIndex(vocab=vocab)
        ix.set_mode(2)
        ix.add_features(ArrayBatch(*rowsA))
        ix.finalize()
        Vg = len(vocab)
        assert Vg > V
        df = df_of(rowsA, Vg)
        if name == "E-selfjoin":
            return Case(name, ix, rowsA, N_A, df, 2, selfjoin=(1000, 1300))
        q, _ = queries_a(ixA, rowsA)
        # every fifth query also lists the df-0 features, one more an out-of-vocabulary feature: both ignored
        extra = [(np.array([0, len(ghost[1])]), ghost[1], ghost[2], np.array([3.0]))]
        parts = []
        for i in range(len(q[0]) - 1):
            a, b = q[0][i], q[0][i + 1]
            ids, tf = q[1][a:b], q[2][a:b]
            if i % 5 == 0:
                ids, tf = np.r_[ids, extra[0][1]], np.r_[tf, extra[0][2]]
                o = np.argsort(ids, kind="stable")
                ids, tf = ids[o], tf[o]
            parts.append((np.array([0, len(ids)]), ids, tf, np.array([q[3][i] + (2.0 if i % 7 == 0 else 0.0)])))
        return Case(name, ix, rowsA, N_A, df, 2, concat_csr(*parts))
    if name == "F":
        ix = GfkbIndex(vocab=ixA.vocab)
        ix.add_features(ArrayBatch(*rowsA))
        ix.finalize()
        q, _ = queries_a(ixA, rowsA)
        case = Case(name, ix, rowsA, N_A, df_of(rowsA, V), 0, q)
        case.upload()
        rap = bound_codes(ix, case.n_q, ix.layout()["chunks"], N_A)[5]
        rng = np.random.default_rng(23)
        gone = np.r_[rng.choice(N_A, N_A // 10, replace=False), rap[32 * 5:32 * 6], rap[32 * 700:32 * 702],
                     rap[32 * 1874:]]
        ix.delete_rows(gone)
        ix.finalize()
        assert ix.last_finalize_kind == 2
        live = ~ix.deleted_mask()
        assert (~live).sum() >= N_A // 10 and not live[rap[32 * 700:32 * 702]].any()
        return Case(name, ix, rowsA, int(live.sum()), df_of(rowsA, V, live), 0, q, live=live)
    if name in ("G", "G-grown"):
        lo, hi = 20_000, 40_000
        shard = csr_rows(*rowsA, np.arange(lo, hi))
        ix = GfkbIndex(vocab=ixA.vocab)
        ix.add_features(ArrayBatch(*shard))
        dfg, ng = df_of(rowsA, V), N_A
        ix.set_global_df(dfg, ng)
        ix.finalize()
        if name == "G-grown":   # rows upserted elsewhere: the global N and df grow, the shard's rows stay
            dfg, ng = dfg + df_of(csr_rows(*rowsA, np.arange(0, 15_000)), V), N_A + 15_000
            ix.set_global_df(dfg, ng)
            ix.finalize()
            assert ix.last_finalize_kind == 2
        q, _ = queries_a(ixA, rowsA)
        return Case(name, ix, shard, ng, dfg, 0, q)
    raise KeyError(name)


def adversarial_queries(ix, rows):
    """One batch through every way a term enters the bound's numerator (see the module docstring of the issue's case C):
    a 128-query tile listing several hundred second-class features (dictionary overflow), more than Q2CAP = 24
    second-class features, more than Q3CAP = 32 rare ones, exactly 64 known features, tf at the regular limit, out-of-
    vocabulary features and a query tf above every row's tf."""
    V = len(ix.vocab)
    n = len(rows[0]) - 1
    ip, ids, tf = rows
    df = np.bincount(ids, minlength=V)
    tfmax = np.zeros(V, np.int64)
    np.maximum.at(tfmax, ids, tf)
    ranked = np.argsort(-np.where(df == n, -1, df), kind="stable")
    ranked = ranked[df[ranked] > 0]
    f2, rare = ranked[300:1200], ranked[3000:]
    rng = np.random.default_rng(29)
    parts = []

    def add(i, t, oov=0.0):
        i = np.asarray(i, np.int64)
        o = np.argsort(i)
        parts.append((np.array([0, len(i)]), i[o], np.asarray(t, np.int64)[o], np.array([oov])))

    for _ in range(128):                                   # the f2 dictionary overflow tile
        add(rng.choice(f2, 20, replace=False), rng.integers(1, 3, 20))
    for _ in range(4):                                     # > Q2CAP second-class features
        add(rng.choice(f2, 30, replace=False), rng.integers(1, 4, 30))
    for _ in range(4):                                     # > Q3CAP rare features
        add(rng.choice(rare, 40, replace=False), rng.integers(1, 4, 40))
    for _ in range(4):                                     # exactly 64 known, non-universal features
        f = np.r_[rng.choice(ranked[:256], 16, replace=False), rng.choice(f2, 24, replace=False),
                  rng.choice(rare, 24, replace=False)]
        add(f, rng.integers(1, 3, 64))
    amax = (np.log(n + 2) + 1) ** 2
    for r in rng.choice(n, 6, replace=False):              # stored rows with tf just under the regular limit
        a, b = ip[r], ip[r + 1]
        mult = max(1, int(np.floor(59_000.0 / (amax * tf[a:b].max()))))
        add(ids[a:b], tf[a:b] * mult)
    for r in rng.choice(n, 4, replace=False):              # stored rows plus out-of-vocabulary features
        add(ids[ip[r]:ip[r + 1]], tf[ip[r]:ip[r + 1]], oov=7.0)
    for _ in range(4):                                     # query tf above every row's tf
        f = rng.choice(ranked[:2000], 12, replace=False)
        add(f, tfmax[f] + 3)
    return concat_csr(*parts)


def corpus_d(universal):
    """Rows with tf >= 31 (the 5-bit tf field's overflow table) on a rare, a mid-frequency and a frequent feature, a
    frequent feature with tf > 2048 in one row (kept out of the fp16 matrix), and 40 empty rows (they sort first: one
    chunk of only empty rows, chunk_minB = +inf).  universal: no empty rows, and a word every row holds once."""
    from kakveda_b200 import synth

    n = 20_000 if not universal else 16_385
    texts = synth.corpus(n)
    for i, r in enumerate(range(7, n, 997)):
        texts[r] += " rarebig" * (31 + i % 9)
    for i, r in enumerate(range(3, n, 41)):
        texts[r] += " midbig" * (35 if i % 25 == 0 else 1)
    for r in range(1, n, 3):
        texts[r] += " freqbig"
    texts[4] += " freqbig" * 2100
    if universal:
        texts = [t + " ustamp" for t in texts]
    else:
        for r in range(0, n, 500):
            texts[r] = ""
    qtexts = synth.queries(150, n) + [texts[r] for r in range(7, n, 997)][:10] + [texts[r] for r in range(3, n, 41 * 25)][:10]
    # ... and the row with tf 2100: irregular (the float64 fallback answers it; the bound pass switches it off)
    qtexts += ["rarebig " * 20, "midbig " * 40 + "freqbig", "freqbig " * 30, "rarebig midbig freqbig", texts[6], texts[4]]
    if universal:
        qtexts += ["ustamp", "ustamp " * 5 + texts[8]]
    return texts, qtexts


CASES = ["A", "B", "C", "D", "D-universal", "E", "E-selfjoin", "F", "G", "G-grown"]


@pytest.fixture(scope="module")
def cases(sm_count, corpus_a):
    cache = {}

    def get(name):
        if name not in cache:
            cache[name] = build_case(name, sm_count, corpus_a)
        return cache[name]

    return get


def assert_case_path(name, case, lay, minB, sm_count):
    n_blocks = (lay["chunks"] + 63) // 64
    if name == "A":
        assert lay["chunks"] == 1875 and lay["last_tiles"] == 3 and min(-(-sm_count // 3), n_blocks) > 1, lay
    elif name == "B":
        assert lay["chunks"] == 513 and lay["last_tiles"] >= sm_count, lay   # n_bsplits = 1
    elif name == "C":
        case.upload()
        assert case.ix.layout()["f2_outside_dictionary"] > 0
    elif name == "D":
        assert lay["tf_overflow_entries"] > 0 and np.isinf(minB).any(), (lay, np.isinf(minB).sum())
    elif name == "D-universal":
        assert lay["universal_features"] > 0 and lay["tf_overflow_entries"] > 0, lay
    elif name == "F":
        assert not case.exact.live.all()


@gpu
@pytest.mark.parametrize("variant", ["specialised", "generic"])
@pytest.mark.parametrize("name", CASES)
def test_bound_contract(cases, sm_count, monkeypatch, name, variant):
    case = cases(name)
    lay, codes, sq, minB = check_contract(case, monkeypatch, {} if variant == "specialised" else GENERIC)
    assert_case_path(name, case, lay, minB, sm_count)
    if name == "A":   # a stored row as the query: the bound of its chunk reaches 1
        q, dup_rows = queries_a(case.ix, case.rows)
        rap = case.smax_cache[0]
        pos = np.empty(len(rap), np.int64)
        pos[rap] = np.arange(len(rap))
        slot = np.empty(len(sq), np.int64)
        slot[sq] = np.arange(len(sq))
        half = case.n_q - len(dup_rows)
        got = codes[slot[half + np.arange(len(dup_rows))], pos[dup_rows] // 32]
        assert (got >= 250).all(), got.min()


@gpu
def test_bound_codes_after_layout_restore(cases, corpus_a, tmp_path):
    """H: an index restored from a persisted layout stores the same codes as the index that wrote it, bit for bit."""
    from kakveda_b200 import GfkbIndex
    from kakveda_b200.similarity import ArrayBatch

    a = cases("A")
    ixA, rowsA = corpus_a
    a.upload()
    n_chunks = ixA.layout()["chunks"]
    want = bound_codes(ixA, a.n_q, n_chunks, N_A)
    path = tmp_path / "a.layout"
    ixA.save_layout(path)
    ix = GfkbIndex(vocab=ixA.vocab)
    ix.add_features(ArrayBatch(*rowsA))
    assert ix.load_layout(path)
    ix.finalize()
    assert ix.last_finalize_kind == 2
    h = Case("H", ix, rowsA, N_A, df_of(rowsA, len(ixA.vocab)), 0, a.queries)
    h.upload()
    got = bound_codes(ix, h.n_q, n_chunks, N_A)
    for name, g, w in zip(("codes", "slot_query", "tcode", "q_terms", "chunk_minB", "row_at_pos"), got, want):
        assert g.tobytes() == w.tobytes(), name
