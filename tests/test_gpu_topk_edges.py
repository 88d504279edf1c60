"""Top-k boundary tests of the fused top-k kernels: TF-IDF (K1b), dense cosine (K2), token-set Jaccard (K3) and the
hash match (K4), at the k, tile, split and query-class edges, against float64 oracles of the same operation.

The contract is Python's stable sort (services/gfkb/app.py:89, ``O.topk_stable``): scores descending, and among equal
scores the lower row wins.  Exact ties are common in GFKB data -- stored duplicates, repeated failures, the zero-score
fill when a query matches fewer than k rows -- and the typical bug of a split/merge top-k (a tied row taken from the
wrong split or column half, or a tied row equal to the exchanged k-th score dropped) returns the right SCORES with the
wrong ROWS.  ``check_topk_strict`` therefore checks exact float64 ties by row id, not by score.

Every parametrised case names the path it pins (pruned / exhaustive, bound codes / recomputed bounds, specialised /
generic bound kernel, row splits, K3 / float64 fallback) and asserts that this path ran, through ``layout()`` or
``last_timing()``, so that a later sizing change cannot move a case onto another path unnoticed.
"""
import numpy as np
import pytest

from oracle import tfidf_oracle as O

gpu = pytest.mark.gpu

RTOL32 = 1e-5                       # float32 TF-IDF top-k against the float64 closed form
DENSE_RTOL, DENSE_ATOL = 1e-5, 1e-6  # K2 against float64 cosine of the same bf16 inputs


# ---------------------------------------------------------------------------------------------------------------------
# The strict checker
# ---------------------------------------------------------------------------------------------------------------------

def check_topk_strict(scores, rows, oracle64, k, rtol, atol=0.0):
    """scores float32 [Q,k] / rows int64 [Q,k] from a device top-k; oracle64 float64 [Q,N] (-inf: a row the query must
    not match, e.g. itself in a self-join).  Fails on:

    * a returned score outside ``atol + rtol |oracle|`` of the oracle value at that row;
    * a broken ordering contract: (score desc, row asc), a duplicate or excluded row, or anything but (-inf, -1) in the
      slots past min(k, N);
    * exact ties: for the float64 tie class of the k-th score, when it has members past the k-th position, the returned
      members of that class must be exactly its lowest row ids (scores compared with ==);
    * near ties: a row of the oracle's stable top-k that is missing, or a returned row that is not in it, is accepted
      only if its oracle score is within 2 rtol (+ 2 atol) of the oracle's k-th score.
    """
    scores = np.asarray(scores)
    rows = np.asarray(rows)
    o64 = np.asarray(oracle64, dtype=np.float64)
    n_q, n = o64.shape
    assert scores.shape == (n_q, k) and rows.shape == (n_q, k), (scores.shape, rows.shape, o64.shape, k)
    ref_all = np.argsort(-o64, axis=1, kind="stable")[:, :k]   # stable: equal scores keep ascending row ids
    n_ok = np.isfinite(o64).sum(axis=1)
    for q in range(n_q):
        o, s, r = o64[q], scores[q], rows[q]
        kk = min(k, int(n_ok[q]))
        where = f"query {q}: rows {r.tolist()} scores {s.tolist()}"
        assert np.all(r[kk:] == -1) and np.all(s[kk:] == -np.inf), "slots past min(k, N) must hold (-inf, -1); " + where
        if kk == 0:
            continue
        rr, ss = r[:kk], s[:kk]
        assert rr.min() >= 0 and rr.max() < n, "row outside the index; " + where
        assert np.isfinite(o[rr]).all(), "an excluded row was returned; " + where
        assert len(np.unique(rr)) == kk, "duplicate row; " + where
        ordered = (ss[:-1] > ss[1:]) | ((ss[:-1] == ss[1:]) & (rr[:-1] < rr[1:]))
        assert ordered.all(), f"order (score desc, row asc) broken at slot {int(np.argmin(ordered))}; " + where
        want = o[rr]
        bad = np.abs(ss.astype(np.float64) - want) > atol + rtol * np.abs(want)
        assert not bad.any(), f"score outside tolerance at slot {int(np.argmax(bad))} (oracle {want.tolist()}); " + where
        ref = ref_all[q, :kk]
        kth = o[ref[-1]]
        cls = np.flatnonzero(o == kth)                    # ascending row ids
        if len(cls) > np.count_nonzero(o[ref] == kth):    # the exact tie class straddles the k-th position
            mine = np.sort(rr[o[rr] == kth])
            assert np.array_equal(mine, cls[:len(mine)]), \
                f"exact tie at the k-th score {kth!r}: returned {mine.tolist()}, lowest ids {cls[:len(mine)].tolist()}; " + where
        tol = 2 * rtol * abs(kth) + 2 * atol
        missing, extra = np.setdiff1d(ref, rr), np.setdiff1d(rr, ref)
        assert np.all(o[missing] <= kth + tol), f"rows {missing.tolist()} missing (oracle {o[missing].tolist()}, k-th {kth!r}); " + where
        assert np.all(o[extra] >= kth - tol), f"rows {extra.tolist()} returned (oracle {o[extra].tolist()}, k-th {kth!r}); " + where


def _f32(*v):
    return np.array([v], dtype=np.float32)


def _rows(*v):
    return np.array([v], dtype=np.int64)


def test_checker_rejects_wrong_answers():
    """Hand-made wrong answers of the kinds a split/merge top-k produces; each one must be rejected."""
    ties = np.array([[0.9, 0.5, 0.5, 0.5, 0.1]])
    check_topk_strict(_f32(0.9, 0.5), _rows(0, 1), ties, 2, RTOL32)                 # the right answer passes
    with pytest.raises(AssertionError, match="exact tie"):                           # tied row 1 replaced by tied row 2
        check_topk_strict(_f32(0.9, 0.5), _rows(0, 2), ties, 2, RTOL32)
    with pytest.raises(AssertionError, match="exact tie"):
        check_topk_strict(_f32(0.9, 0.5, 0.5), _rows(0, 1, 3), ties, 3, RTOL32)

    spread = np.array([[0.9, 0.8, 0.7, 0.1]])
    with pytest.raises(AssertionError, match="returned|missing"):                    # row 1 missing, far outside rtol
        check_topk_strict(_f32(0.9, 0.7), _rows(0, 2), spread, 2, RTOL32)
    with pytest.raises(AssertionError, match="order"):                               # swapped pair
        check_topk_strict(_f32(0.8, 0.9), _rows(1, 0), spread, 2, RTOL32)
    with pytest.raises(AssertionError, match="order"):                               # equal scores, rows descending
        check_topk_strict(_f32(0.9, 0.5, 0.5), _rows(0, 2, 1), ties, 3, RTOL32)
    with pytest.raises(AssertionError, match="tolerance"):                           # right rows, score off by 1e-4
        check_topk_strict(_f32(0.9, 0.80008), _rows(0, 1), spread, 2, RTOL32)
    with pytest.raises(AssertionError, match="duplicate"):
        check_topk_strict(_f32(0.9, 0.9), _rows(0, 0), spread, 2, RTOL32)

    fill = np.array([[0.5, 0.0, 0.0, 0.0, 0.0, 0.0]])                               # one match, then the zero-score fill
    check_topk_strict(_f32(0.5, 0, 0, 0), _rows(0, 1, 2, 3), fill, 4, RTOL32)
    with pytest.raises(AssertionError, match="order"):                               # fill not ascending
        check_topk_strict(_f32(0.5, 0, 0, 0), _rows(0, 1, 3, 2), fill, 4, RTOL32)
    with pytest.raises(AssertionError, match="exact tie"):                           # fill skips row 3
        check_topk_strict(_f32(0.5, 0, 0, 0), _rows(0, 1, 2, 4), fill, 4, RTOL32)
    with pytest.raises(AssertionError, match="exact tie"):                           # fill starts in a later split
        check_topk_strict(_f32(0.5, 0, 0, 0), _rows(0, 3, 4, 5), fill, 4, RTOL32)

    # slots past N = 6 rows must be exactly (-inf, -1)
    full = (_f32(0.5, 0, 0, 0, 0, 0, -np.inf, -np.inf), _rows(0, 1, 2, 3, 4, 5, -1, -1))
    check_topk_strict(*full, fill, 8, RTOL32)
    with pytest.raises(AssertionError, match="slots past"):
        check_topk_strict(_f32(0.5, 0, 0, 0, 0, 0, 0, -np.inf), _rows(0, 1, 2, 3, 4, 5, -1, -1), fill, 8, RTOL32)
    with pytest.raises(AssertionError, match="slots past"):
        check_topk_strict(full[0], _rows(0, 1, 2, 3, 4, 5, 0, -1), fill, 8, RTOL32)
    # an excluded row (-inf in the oracle) must never come back
    excl = np.array([[-np.inf, 0.7, 0.3]])
    check_topk_strict(_f32(0.7), _rows(1), excl, 1, RTOL32)
    with pytest.raises(AssertionError, match="excluded"):
        check_topk_strict(_f32(0.7, 0.0), _rows(1, 0), excl, 2, RTOL32)


def test_checker_accepts_float32_near_tie_reordering():
    """Rows 1 and 2 differ by 6e-8 in float64; a float32 kernel may rank them either way, and at k = 2 keep either."""
    near = np.array([[0.9, 0.7 + 6e-8, 0.7, 0.1]])
    check_topk_strict(_f32(0.9, 0.70000005, 0.7), _rows(0, 2, 1), near, 3, RTOL32)
    check_topk_strict(_f32(0.9, 0.7), _rows(0, 2), near, 2, RTOL32)
    check_topk_strict(_f32(0.9, 0.7, 0.7), _rows(0, 1, 2), near, 3, RTOL32)        # equal float32 scores, rows ascending
    # and a dense-style absolute tolerance around zero
    check_topk_strict(_f32(3e-7, 0.0), _rows(1, 0), np.array([[0.0, 2e-7]]), 2, DENSE_RTOL, DENSE_ATOL)


# ---------------------------------------------------------------------------------------------------------------------
# Shared GPU fixtures
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


def index_layout(handle_owner) -> dict:
    """``GfkbIndex.layout`` of any object owning a kv_index handle (a ``JaccardIndex`` shares the TF-IDF index type)."""
    from kakveda_b200 import GfkbIndex

    return GfkbIndex.layout(handle_owner)


# ---------------------------------------------------------------------------------------------------------------------
# TF-IDF K1b: bound pass -> selection -> scan -> K5 merge, against O.score_matrix_closed_form
# ---------------------------------------------------------------------------------------------------------------------

PRUNE_MIN_CHUNKS = 512              # size_batch: fewer chunks -> the exhaustive scan
TIE_COPIES = {"a": 40, "b": 33, "e": 32, "c": 3, "d": 2}   # 40 = k + 8 at k = 32; 33, 32, 3, 2 = k + 1 at k = 32, 31, 2, 1
TOKEN = "zqxplant"                  # a word stored in exactly three rows
QFEATS = 64                         # features a query table holds; more -> the float64 fallback (K1a + selection)


def _wide_query(n_feats: int) -> str:
    # n_feats distinct known unigrams; in descending order none of its bigrams is stored, so they are out of vocabulary
    return " ".join(f"pw{i}" for i in reversed(range(n_feats)))


class TfidfCase:
    """A synthetic GFKB of n rows with planted ties and query classes, its index, a 129-query batch and its oracle."""

    def __init__(self, n: int):
        from kakveda_b200 import GfkbIndex, synth

        rng = np.random.default_rng(n)
        corpus = synth.corpus(n)
        self.token_rows = [5, n // 2 + 7, n - 3]
        wide_row = n // 3 + 1
        free = np.setdiff1d(np.arange(n), self.token_rows + [wide_row])
        pos = rng.choice(free, size=sum(TIE_COPIES.values()), replace=False)
        self.tie_text, self.tie_rows, o = {}, {}, 0
        for g, c in TIE_COPIES.items():
            text = corpus[1000 + len(self.tie_text)] + f" tiegrp{g} tiegrp{g}x"
            self.tie_rows[g] = np.sort(pos[o:o + c])
            self.tie_text[g] = text
            for r in self.tie_rows[g]:
                corpus[r] = text
            o += c
        for r in self.token_rows:
            corpus[r] = corpus[r] + " " + TOKEN
        corpus[wide_row] = " ".join(f"pw{i}" for i in range(70))
        # 129 queries the scan answers (batch prefixes hit the group and tile edges), then the other query classes:
        # null, out-of-vocabulary only, QFEATS and QFEATS + 1 known features
        planted = {0: self.tie_text["a"], 30: self.tie_text["b"], 31: self.tie_text["e"], 32: self.tie_text["c"],
                   33: self.tie_text["d"], 64: TOKEN, 127: _wide_query(QFEATS)}
        rest = iter(synth.queries(129 - len(planted), n))
        self.queries = [planted[i] if i in planted else next(rest) for i in range(129)]
        self.queries += ["", "qqzzunseen xxyyq", _wide_query(QFEATS + 1)]
        self.corpus, self.n = corpus, n
        self.ix = GfkbIndex()
        self.ix.add_texts(corpus)
        self.ix.finalize()
        self.oracle = O.score_matrix_closed_form(self.queries, corpus)
        lay = self.ix.layout()
        assert lay["rows"] == n and lay["chunks"] == (n + 31) // 32, lay
        self.pruned = lay["chunks"] >= PRUNE_MIN_CHUNKS

    def topk(self, queries, k):
        s, r = self.ix.topk(queries, k)
        return s, r, self.ix.layout()


@pytest.fixture(scope="module")
def tfidf_cases(lib):
    cache = {}

    def get(n):
        if n not in cache:
            cache[n] = TfidfCase(n)
        return cache[n]

    return get


def assert_tfidf_path(lay, pruned: bool):
    if pruned:
        assert lay["pairs_passed_bound"] > 0, ("the pruned path (bound kernel) did not run", lay)
    else:
        assert lay["pairs_passed_bound"] == 0 and lay["pairs_scored"] > 0, ("the exhaustive scan did not run", lay)


@gpu
@pytest.mark.parametrize("n,pruned", [(16352, False),    # 511 chunks: exhaustive, one below the pruning switch
                                      (16384, True),     # 512 chunks: pruned, 8 full 64-chunk blocks
                                      (16385, True),     # 513 chunks: pruned, a one-row last chunk in a ninth block
                                      (19999, True)])    # 625 chunks (625 % 64 = 49), a 31-row last chunk: pruned
def test_tfidf_corpus_sizes_planted_ties(tfidf_cases, n, pruned):
    case = tfidf_cases(n)
    assert case.pruned == pruned
    k = 32
    s, r, lay = case.topk(case.queries, k)
    assert_tfidf_path(lay, pruned)
    check_topk_strict(s, r, case.oracle, k, RTOL32)
    q = case.queries
    # one text stored k + 8 times: the k lowest copies, bit-identical scores (~1)
    assert r[q.index(case.tie_text["a"])].tolist() == case.tie_rows["a"][:k].tolist()
    # k + 1 copies: the tie sits on the k-th slot
    assert r[q.index(case.tie_text["b"])].tolist() == case.tie_rows["b"][:k].tolist()
    for g in "abe":
        assert np.all(s[q.index(case.tie_text[g]), :k] == s[q.index(case.tie_text[g]), 0])
    # the query's only known feature is in three rows: those three, then the zero-score fill in ascending row order
    t = q.index(TOKEN)
    fill = [i for i in range(k + 3) if i not in case.token_rows][:k - 3]
    assert sorted(r[t, :3].tolist()) == case.token_rows and np.all(s[t, :3] > 0)
    assert r[t, 3:].tolist() == fill and np.all(s[t, 3:] == 0)
    # null and out-of-vocabulary-only queries: the first k rows
    for null in ("", "qqzzunseen xxyyq"):
        assert r[q.index(null)].tolist() == list(range(k)) and np.all(s[q.index(null)] == 0)


@gpu
@pytest.mark.parametrize("k", [1, 2, 31, 32])
def test_tfidf_pruned_k_sweep_and_variants(tfidf_cases, monkeypatch, k):
    """Pruned path at 513 chunks.  Each variant must return the default's bits:
    exhaustive (KAKVEDA_B200_NO_PRUNE=1), recomputed bounds instead of the stored codes (KAKVEDA_B200_BOUND_CODES=0) and
    the generic bound instantiation instead of the specialised one (KAKVEDA_B200_GENERIC_BOUND=1)."""
    case = tfidf_cases(16385)
    s, r, lay = case.topk(case.queries, k)
    assert_tfidf_path(lay, True)
    check_topk_strict(s, r, case.oracle, k, RTOL32)
    for g, c in TIE_COPIES.items():   # k + 1 copies of "b", "e", "c", "d" at k = 32, 31, 2, 1
        assert r[case.queries.index(case.tie_text[g]), :min(k, c)].tolist() == case.tie_rows[g][:min(k, c)].tolist()
    for env, value in (("KAKVEDA_B200_NO_PRUNE", "1"), ("KAKVEDA_B200_BOUND_CODES", "0"), ("KAKVEDA_B200_GENERIC_BOUND", "1")):
        with monkeypatch.context() as m:
            m.setenv(env, value)
            s2, r2, lay2 = case.topk(case.queries, k)
        np.testing.assert_array_equal(r2, r, err_msg=env)
        np.testing.assert_array_equal(s2, s, err_msg=env)
        if env == "KAKVEDA_B200_NO_PRUNE":
            assert_tfidf_path(lay2, False)
            assert lay2["pairs_scored"] >= (len(case.queries) - 3) * lay2["chunks"], lay2   # every chunk of every scanned query
        elif env == "KAKVEDA_B200_BOUND_CODES":
            # recomputed bounds are exact; the codes round them up to 1/250: never more candidates than with the codes
            assert 0 < lay2["pairs_passed_bound"] <= lay["pairs_passed_bound"], (lay, lay2)
        else:
            # same bounds from both instantiations -> the same candidate pairs
            assert lay2["pairs_passed_bound"] == lay["pairs_passed_bound"], (lay, lay2)


@gpu
@pytest.mark.parametrize("batch", [1, 31, 32, 33, 127, 128, 129])
def test_tfidf_batch_sizes(tfidf_cases, batch):
    """32-query scan groups and 128-query bound tiles, full and partial, on the pruned path (513 chunks).  Every query
    of these batches is scanned (none is null or irregular), so the batch size is the scanned query count."""
    case = tfidf_cases(16385)
    assert "" not in case.queries[:batch] and _wide_query(QFEATS + 1) not in case.queries[:batch]
    for k in (1, 32):
        s, r, lay = case.topk(case.queries[:batch], k)
        assert_tfidf_path(lay, True)
        assert lay["last_tiles"] == (batch + 127) // 128, lay
        check_topk_strict(s, r, case.oracle[:batch], k, RTOL32)


@gpu
def test_tfidf_query_classes_in_one_batch(tfidf_cases):
    """Null, out-of-vocabulary-only, exactly QFEATS (64) and QFEATS + 1 non-universal known features, beside planted
    ties, in one pruned batch.  The 65-feature query alone takes the float64 fallback (two more launches: K1a and the
    selection); it must meet the same contract."""
    case = tfidf_cases(16385)
    q = case.queries
    base = [case.tie_text["a"], "", "qqzzunseen xxyyq", TOKEN, q[1], q[2]]
    wide64, wide65 = _wide_query(QFEATS), _wide_query(QFEATS + 1)
    launches = {}
    for name, batch in (("base", base), ("with64", base + [wide64]), ("with65", base + [wide64, wide65]),
                        ("first65", [wide65] + base)):
        want = case.oracle[[q.index(t) for t in batch]]
        for k in (1, 32):
            s, r, lay = case.topk(batch, k)
            assert_tfidf_path(lay, True)
            check_topk_strict(s, r, want, k, RTOL32)
            launches[name, k] = lay["kernel_launches"]
            # the wide row is the only match of both wide queries; then the zero-score fill from row 0
            for t in (wide64, wide65):
                if t in batch:
                    assert r[batch.index(t)].tolist() == [case.n // 3 + 1] + list(range(k - 1))
    for k in (1, 32):
        assert launches["with64", k] == launches["base", k], launches      # 64 features: the regular scan
        assert launches["with65", k] == launches["base", k] + 2, launches  # 65 features: K1a + selection
        assert launches["first65", k] == launches["base", k] + 2, launches


# ---------------------------------------------------------------------------------------------------------------------
# Dense K2 against O.dense_cosine (float64 cosine of the bf16-rounded inputs)
# ---------------------------------------------------------------------------------------------------------------------

def dense_planted(d, n, q, k, seed):
    """Random rows and queries with: k + 8 copies of one row (fewer when n is small) at rows of both column halves
    (column % 4 in {0, 1} and {2, 3}), a zero row, and the queries  copy * 1.5 (the copies tie at cosine 1),  zero,
    -copy  and  a stored row."""
    rng = np.random.default_rng(seed)
    C = rng.standard_normal((n, d)).astype(np.float32)
    Q = rng.standard_normal((q, d)).astype(np.float32)
    copies = np.zeros(0, dtype=np.int64)
    zero_row = None
    if n >= 4:
        c = min(k + 8, n // 3)
        copies = np.unique(np.linspace(1, n - 2, c).astype(np.int64))
        v = rng.standard_normal(d).astype(np.float32)
        C[copies] = v
        zero_row = int(np.setdiff1d(np.arange(n // 2, n), copies)[0])
        C[zero_row] = 0.0
        for i, row in enumerate([v * 1.5, np.zeros(d, np.float32), -v, C[n // 3]][:q]):
            Q[i] = row
    elif q >= 2:
        Q[1] = 0.0
    return C, Q, copies, zero_row


def dense_rtol(d):
    """The tensor cores' fp32 accumulation does not round to nearest: a dot product of same-sign terms (a row against
    a multiple of itself) can lose about one fp32 ulp per 16-element step, dim / 16 * 2^-23 relative.  Measured on an
    NVIDIA H100 80GB HBM3 (700 W limit): 4.1e-5 at dim 8192 (bound 6.1e-5); below dim 1344 the bound is under the
    general 1e-5."""
    return max(DENSE_RTOL, d / 16 * 2.0 ** -23)


DENSE_CASES = [  # (dim, rows, queries, k): one row split each
    (64, 513, 129, 32),
    (192, 257, 127, 31),    # 3 K slices: the 3-stage ring wraps exactly once per tile
    (256, 255, 128, 1),
    (8192, 257, 33, 32),    # the largest dim
    (128, 1, 129, 32),
    (128, 256, 1, 1),
    (128, 257, 128, 31),
    (64, 255, 129, 1),
    (192, 513, 1, 32),
]


@gpu
@pytest.mark.parametrize("d,n,q,k", DENSE_CASES)
def test_dense_shapes(lib, d, n, q, k):
    from kakveda_b200 import DenseIndex

    C, Q, copies, _ = dense_planted(d, n, q, k, seed=d * 7 + n * 3 + q + k)
    dx = DenseIndex(d)
    dx.add(C[: n // 2])
    dx.add(C[n // 2:])
    dx.finalize()
    s, r = dx.topk(Q, k)
    assert dx.last_timing()[1] == 1, "expected one row split"
    want = O.dense_cosine(Q, C)
    check_topk_strict(s, r, want, k, dense_rtol(d), DENSE_ATOL)
    kk = min(k, n)
    if len(copies):   # the copies tie bit for bit: the lowest ones, from both column halves
        m = min(kk, len(copies))
        assert r[0, :m].tolist() == copies[:m].tolist() and np.all(s[0, :m] == s[0, 0])
        assert {int(c) % 4 // 2 for c in copies} == {0, 1}
    if q >= 2:        # zero query: every score 0, rows 0 .. k-1
        assert r[1, :kk].tolist() == list(range(kk)) and np.all(s[1, :kk] == 0)


@gpu
@pytest.mark.parametrize("k", [1, 32])
def test_dense_row_splits_and_threshold_exchange(lib, k):
    """132 row splits of 8 tiles each (one 128-query tile): the CTAs exchange k-th-score lower bounds (gthr) while
    later splits are still scanning.  Planted so that a later split secures a k-th score of exactly 0 or a negative one
    while an earlier split still holds rows tying with it at lower ids:

    * Z = e0 scores negative against every row but the rows whose dim 0 is 0 (and the zero row), which score exactly 0:
      four of them in the last tile of split 0 (rows 1800..1803, both column halves), the zero row 1900, and 80 in the
      first tile of split 1.  The answer is 1800..1803, 1900, then split 1's rows -- never split 1's rows alone;
    * N (dim 0 = 0, the others negative) scores <= 0 against every row: the zero row first, then k + 8 copies of one row
      spread over splits and both column halves (negative keys in the exchange);
    * the copy itself: its k lowest copies;  the zero query: rows 0 .. k-1."""
    from kakveda_b200 import DenseIndex

    d, tiles_per_split = 64, 8
    n = 132 * tiles_per_split * 256
    rng = np.random.default_rng(20 + k)
    C = (np.abs(rng.standard_normal((n, d))) + 0.1).astype(np.float32)
    C[:, 0] = -C[:, 0]
    zero_dim0 = np.r_[1800:1804, 2048:2128]
    C[zero_dim0, 0] = 0.0
    C[1900] = 0.0
    v = np.full(d, 0.01, dtype=np.float32)
    v[0] = -1.0
    split_rows = tiles_per_split * 256
    copies = np.array([s * split_rows + 600 + 3 * s for s in range(0, 120, 3)], dtype=np.int64)   # k + 8 = 40 copies
    C[copies] = v
    Q = np.zeros((8, d), dtype=np.float32)
    Q[0, 0] = 1.0                                                 # Z
    Q[1, 1:] = -(np.abs(rng.standard_normal(d - 1)) + 0.1)        # N
    Q[2] = v                                                      # the copy
    # Q[3] = 0: the zero query
    Q[4:] = rng.standard_normal((4, d))
    dx = DenseIndex(d)
    dx.add(C)
    dx.finalize()
    s, r = dx.topk(Q, k)
    splits = dx.last_timing()[1]
    assert splits > 1 and (n // 256) // splits >= 4, f"expected many row splits of >= 4 tiles, got {splits}"
    want = O.dense_cosine(Q, C)
    assert np.all(want[1] <= 0)
    check_topk_strict(s, r, want, k, DENSE_RTOL, DENSE_ATOL)
    z = [1800, 1801, 1802, 1803, 1900] + list(range(2048, 2128))
    assert r[0].tolist() == z[:k] and np.all(s[0] == 0)
    assert r[1, 0] == 1900 and r[1, 1:].tolist() == copies[:k - 1].tolist()
    assert r[2].tolist() == copies[:k].tolist()
    assert r[3].tolist() == list(range(k)) and np.all(s[3] == 0)


@gpu
def test_dense_query_batch_over_one_wave(lib):
    """More than 132 x 128 queries against 250 rows: 133 query tiles, one row split."""
    from kakveda_b200 import DenseIndex

    d, n, q, k = 64, 250, 132 * 128 + 1, 32
    C, Q, copies, _ = dense_planted(d, n, q, k, seed=3)
    Q[q - 1] = Q[0]                     # the last (partial) query tile repeats the tie query
    dx = DenseIndex(d)
    dx.add(C)
    dx.finalize()
    s, r = dx.topk(Q, k)
    assert dx.last_timing()[1] == 1, "expected one row split"
    check_topk_strict(s, r, O.dense_cosine(Q, C), k, DENSE_RTOL, DENSE_ATOL)
    assert r[q - 1].tolist() == r[0].tolist() == copies[:k].tolist()


@gpu
@pytest.mark.parametrize("k", [1, 32])
def test_dense_selfjoin_keeps_tied_twins(lib, k):
    """Self-join top-k: every row's own entry is excluded, never its identical twin (which ties with it exactly)."""
    from kakveda_b200 import DenseIndex

    d, n = 128, 600
    rng = np.random.default_rng(41)
    C = rng.standard_normal((n, d)).astype(np.float32)
    groups = [[10, 11, 300], [50, 51], [2, 599], [256, 257, 258, 259]]   # twins within and across row tiles
    for g in groups:
        C[g[1:]] = C[g[0]]
    dx = DenseIndex(d)
    dx.add(C)
    dx.finalize()
    s, r = dx.selfjoin_topk(k)
    assert dx.last_timing()[1] == 1
    want = O.dense_cosine(C, C)
    np.fill_diagonal(want, -np.inf)
    check_topk_strict(s, r, want, k, DENSE_RTOL, DENSE_ATOL)
    for g in groups:
        for row in g:
            twins = [t for t in g if t != row]
            m = min(k, len(twins))
            assert r[row, :m].tolist() == twins[:m], (row, r[row, :m])


# ---------------------------------------------------------------------------------------------------------------------
# Jaccard K3: exact integers
# ---------------------------------------------------------------------------------------------------------------------

JV = 1 << 14


def jaccard_rows(n, rng):
    zipf = lambda size: np.minimum(rng.zipf(1.3, size) - 1, JV - 1)
    rows = [np.unique(np.concatenate([zipf(rng.poisson(15)), rng.integers(0, JV, rng.poisson(25))]).astype(np.uint32))
            for _ in range(n)]
    if n > 2:
        rows[2] = np.zeros(0, dtype=np.uint32)   # an empty row: no token is in every row
    return rows


def jaccard_matrix(queries, rows):
    """(inter, union) int64 [Q, N] over token sets: sparse products of exact 0/1 matrices."""
    import scipy.sparse as sp

    width = 1 + max([int(a.max()) for a in list(queries) + list(rows) if len(a)] + [0])

    def mat(sets):
        ip = np.zeros(len(sets) + 1, dtype=np.int64)
        np.cumsum([len(a) for a in sets], out=ip[1:])
        ids = np.concatenate([np.asarray(a, dtype=np.int64) for a in sets]) if ip[-1] else np.zeros(0, np.int64)
        return sp.csr_matrix((np.ones(len(ids)), ids, ip), shape=(len(sets), width))

    Qm, Rm = mat(queries), mat(rows)
    inter = np.rint((Qm @ Rm.T).toarray()).astype(np.int64)
    union = np.diff(Qm.indptr)[:, None] + np.diff(Rm.indptr)[None, :] - inter
    return inter, union


def jaccard_route(queries, rows, vocab):
    """True for queries the index answers with K3: at most QFEATS known tokens that are not in every row."""
    count = {}
    for a in rows:
        for t in a.tolist():
            count[t] = count.get(t, 0) + 1
    return [sum(1 for t in np.unique(a).tolist() if t < vocab and count.get(t, 0) < len(rows)) <= QFEATS for a in queries]


def check_jaccard(out, queries, rows, k):
    """Bit-exact: the rows of the stable top-k of the float64 ratios, and the exact counts of O.jaccard_sets."""
    s, r, inter, union = out
    I, U = jaccard_matrix(queries, rows)
    ratio = np.where(U > 0, I / np.maximum(U, 1), 0.0)
    order = np.argsort(-ratio, axis=1, kind="stable")
    kk = min(k, len(rows))
    for i, qs in enumerate(queries):
        assert r[i, :kk].tolist() == order[i, :kk].tolist(), (i, r[i], order[i, :kk])
        assert np.all(r[i, kk:] == -1) and np.all(s[i, kk:] == -np.inf)
        for j in range(kk):
            row = int(r[i, j])
            assert (int(inter[i, j]), int(union[i, j])) == O.jaccard_sets(qs.tolist(), rows[row].tolist()), (i, j, row)
        got64 = np.where(union[i, :kk] > 0, inter[i, :kk] / np.maximum(union[i, :kk], 1), 0.0)
        assert got64.tolist() == ratio[i, r[i, :kk]].tolist()
        np.testing.assert_allclose(s[i, :kk], got64, rtol=1e-6, atol=1e-7)


def jaccard_splits(chunks, n_q, sms, warps=8):
    """Partial lists of a K3 batch (run_jaccard): row splits x warps."""
    groups = (n_q + 31) // 32
    return max(1, min(min((4 * sms + groups - 1) // groups, 256), max(1, chunks // 64))) * warps


@gpu
@pytest.mark.parametrize("n", [1, 31, 33, 20000])   # 20,000 rows: 625 chunks, several row splits x 8 warps
def test_jaccard_row_counts_query_sizes_and_ties(lib, sm_count, n):
    from kakveda_b200 import JaccardIndex

    rng = np.random.default_rng(n + 1)
    rows = jaccard_rows(n, rng)
    dup = np.unique(rng.integers(0, JV, 30)).astype(np.uint32)
    n_dup = min(40, max(0, n - 3))                                         # k + 8 at k = 32
    dup_rows = np.sort(rng.choice(np.setdiff1d(np.arange(n), [2, n - 1]), size=n_dup, replace=False)) if n_dup else []
    for row in dup_rows:
        rows[row] = dup.copy()
    if n > 1:
        rows[n - 1] = np.array([0, 7, JV - 1], dtype=np.uint32)           # the last token id of the vocabulary

    def sized(m):   # m distinct tokens, half of them from a stored row
        own = rows[min(n - 1, 9)][: m // 2]
        extra = rng.permutation(np.setdiff1d(np.arange(JV), own))[: m - len(own)]
        return np.unique(np.concatenate([own, extra])).astype(np.uint32)

    queries = [dup.copy(), sized(63), sized(64), sized(65), np.array([0, 7, JV - 1, JV, JV + 3], dtype=np.uint32),
               np.zeros(0, dtype=np.uint32), np.array([JV + 1], dtype=np.uint32)]
    queries += [np.unique(np.minimum(rng.zipf(1.3, rng.poisson(30) + 1) - 1, JV - 1)).astype(np.uint32) for _ in range(25)]
    assert [len(a) for a in queries[1:4]] == [63, 64, 65]
    jx = JaccardIndex(JV)
    jx.add_sets(rows[: n // 2])
    jx.add_sets(rows[n // 2:])
    jx.finalize()
    k3 = jaccard_route(queries, rows, JV)
    if n > 2:
        assert k3[1] and k3[2] and not k3[3], "63 and 64 tokens stay on K3, 65 take the fallback"
    regular = [a for a, ok in zip(queries, k3) if ok]
    for k in (1, 32):
        out = jx.topk_sets(queries, k)
        lay = index_layout(jx)
        check_jaccard(out, queries, rows, k)
        if n_dup:
            assert out[1][0, :min(k, n_dup)].tolist() == list(dup_rows[:min(k, n_dup)])
        # path: every query outside K3 adds two launches (K1a and the selection)
        jx.topk_sets(regular, k)
        assert lay["kernel_launches"] == index_layout(jx)["kernel_launches"] + 2 * (len(queries) - len(regular)), lay
        if n == 20000:
            assert jaccard_splits(lay["chunks"], len(queries), sm_count) >= 16


@gpu
def test_jaccard_full_union_table(lib):
    """One scan group of 32 queries with 64 distinct tokens each, no token shared: 2,048 keys in the 4,096-slot union
    table (half full, long probe chains), all on K3."""
    from kakveda_b200 import JaccardIndex

    rng = np.random.default_rng(64)
    n = 20000
    rows = jaccard_rows(n, rng)
    toks = rng.permutation(JV)[: 32 * 64].reshape(32, 64)
    queries = [np.sort(t).astype(np.uint32) for t in toks]
    for i in range(0, 32, 4):   # some queries repeat a stored row exactly (tokens of their own, 64 of them)
        rows[100 + 600 * i] = queries[i].copy()
        rows[101 + 600 * i] = queries[i].copy()
    assert all(jaccard_route(queries, rows, JV))
    jx = JaccardIndex(JV)
    jx.add_sets(rows)
    jx.finalize()
    plain = [np.unique(rng.integers(0, JV, 20)).astype(np.uint32) for _ in range(32)]
    for k in (1, 32):
        jx.topk_sets(plain, k)
        base = index_layout(jx)["kernel_launches"]
        out = jx.topk_sets(queries, k)
        assert index_layout(jx)["kernel_launches"] == base, "a query left K3"
        check_jaccard(out, queries, rows, k)
        for i in range(0, 32, 4):
            assert out[1][i, :min(k, 2)].tolist() == [100 + 600 * i, 101 + 600 * i][:min(k, 2)]


# ---------------------------------------------------------------------------------------------------------------------
# Hash K4: integer equality
# ---------------------------------------------------------------------------------------------------------------------

def hash_oracle(stored, queries, k):
    where = {}
    for i, h in enumerate(stored.tolist()):
        where.setdefault(h, []).append(i)
    rows = np.array([(where.get(h, [])[:k] + [-1] * k)[:k] for h in queries.tolist()], dtype=np.int64).reshape(len(queries), k)
    counts = np.array([len(where.get(h, [])) for h in queries.tolist()], dtype=np.int64)
    return rows, counts


@gpu
def test_hash_edges(lib):
    from kakveda_b200 import HashIndex

    k = 16
    rng = np.random.default_rng(4)
    # 1-row appends: after every append the scan reads a row pair past the end, which must be padding
    hx = HashIndex()
    stored = np.zeros(0, dtype=np.uint64)
    seq = rng.integers(1, 2**63, size=41, dtype=np.uint64)
    seq[20] = 0                          # hash 0 is an ordinary value
    for i, h in enumerate(seq):
        hx.add_hashes(np.array([h], dtype=np.uint64))
        stored = np.append(stored, np.uint64(h))
        assert hx.n_rows == i + 1
        probe = np.concatenate([stored[-3:], seq[i + 1:i + 3], np.array([0], dtype=np.uint64)])
        rows, counts = hx.match_hashes(probe, k)
        want_r, want_c = hash_oracle(stored, probe, k)
        np.testing.assert_array_equal(counts, want_c, err_msg=f"after {i + 1} rows")
        np.testing.assert_array_equal(rows, want_r, err_msg=f"after {i + 1} rows")
    # 0xFFFF...FF is the padding value: rejected, and the index is unchanged
    with pytest.raises(Exception):
        hx.add_hashes(np.array([5, 0xFFFFFFFFFFFFFFFF], dtype=np.uint64))
    assert hx.n_rows == len(seq)

    # a hash stored 3k times among 100k rows: exact count, the first k rows ascending; a duplicate query on both sides
    # of the 4,096-query pass edge
    n = 100_001
    big = rng.integers(0, 2**63, size=n, dtype=np.uint64)
    rep = np.sort(rng.choice(np.setdiff1d(np.arange(n), [777]), size=3 * k, replace=False))
    big[rep] = np.uint64(0x1234567890ABCDEF)
    big[777] = 0
    hb = HashIndex(row_base=5)
    hb.add_hashes(big[:50_000])
    hb.add_hashes(big[50_000:])
    qh = big[rng.integers(0, n, size=4100)]
    qh[0] = qh[4095] = qh[4096] = np.uint64(0x1234567890ABCDEF)
    qh[1] = 0
    qh[2] = np.uint64(0xFFFFFFFFFFFFFFFF)        # never stored: no match
    qh[4097] = qh[4094]
    rows, counts = hb.match_hashes(qh, k)
    assert hb.last_timing()[1] == 2, "expected two query passes"
    want_r, want_c = hash_oracle(big, qh, k)
    np.testing.assert_array_equal(counts, want_c)
    np.testing.assert_array_equal(rows, np.where(want_r >= 0, want_r + 5, -1))
    assert counts[0] == 3 * k and rows[0].tolist() == (rep[:k] + 5).tolist()
    assert rows[4095].tolist() == rows[4096].tolist() == rows[0].tolist() and counts[4096] == 3 * k
    assert counts[1] == 1 and rows[1, 0] == 777 + 5 and counts[2] == 0 and np.all(rows[2] == -1)
