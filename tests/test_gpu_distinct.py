"""Distinct top-k (field collapsing): the k best rows with at most one row per group, against float64 oracles.

The distinct top-k of a query is defined on the rows it may match (live, not excluded, of its label when filtered):
the best row of each group is the first one in (score desc, row asc) order, the groups are ranked by their best rows
in that order, and the first k best rows are returned, (-inf, -1) past the last group.  So the oracle is the float64
score matrix with every row but its group's best masked to -inf, checked with the strict tie rules of
test_gpu_topk_edges.py; on top of that the returned groups must be distinct and each returned row must score within
rtol of its group's best (a float32 near tie inside a group may pick another row of it, an exact tie may not).
"""

import numpy as np
import pytest

from oracle import tfidf_oracle as O

gpu = pytest.mark.gpu

RTOL32 = 1e-5
N_ROWS = 60000          # 1875 chunks: the pruned path
KS = (1, 2, 5, 16, 31, 32)
QFEATS = 64
NO_PRUNE = ("KAKVEDA_B200_NO_PRUNE", "1")
ENVS = [None, ("KAKVEDA_B200_BOUND_CODES", "0"), NO_PRUNE]


# ---- the checker ----------------------------------------------------------------------------------------------------

def check_topk_strict(scores, rows, oracle64, k, rtol):
    """The checker of test_gpu_topk_edges.py: (score desc, row asc), (-inf, -1) past min(k, allowed rows), scores
    within rtol of the oracle, exact float64 ties straddling the k-th slot resolved to the lowest rows, and near-tie
    swaps only within 2 rtol of the k-th score.  oracle64 -inf: a row the query must not match."""
    o64 = np.asarray(oracle64, dtype=np.float64)
    n_q, n = o64.shape
    assert scores.shape == (n_q, k) and rows.shape == (n_q, k)
    ref_all = np.argsort(-o64, axis=1, kind="stable")[:, :k]
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
        assert np.isfinite(o[rr]).all(), "a masked row was returned; " + where
        assert len(np.unique(rr)) == kk, "duplicate row; " + where
        ordered = (ss[:-1] > ss[1:]) | ((ss[:-1] == ss[1:]) & (rr[:-1] < rr[1:]))
        assert ordered.all(), "order broken; " + where
        want = o[rr]
        bad = np.abs(ss.astype(np.float64) - want) > rtol * np.abs(want)
        assert not bad.any(), f"score outside tolerance (oracle {want.tolist()}); " + where
        ref = ref_all[q, :kk]
        kth = o[ref[-1]]
        cls = np.flatnonzero(o == kth)
        if len(cls) > np.count_nonzero(o[ref] == kth):
            mine = np.sort(rr[o[rr] == kth])
            assert np.array_equal(mine, cls[:len(mine)]), f"exact tie at {kth!r}: {mine.tolist()}; " + where
        tol = 2 * rtol * abs(kth)
        missing, extra = np.setdiff1d(ref, rr), np.setdiff1d(rr, ref)
        assert np.all(o[missing] <= kth + tol), f"rows {missing.tolist()} missing; " + where
        assert np.all(o[extra] >= kth - tol), f"rows {extra.tolist()} returned; " + where


def group_best(o64, groups):
    """Per query: the best row of every group -- first in (score desc, row asc) order among the finite rows -- as a
    [Q, N] matrix keeping only those rows (others -inf), and best[q, g] = that row (-1: no eligible row)."""
    o64 = np.asarray(o64, dtype=np.float64)
    n_q, n = o64.shape
    groups = np.asarray(groups)
    n_g = int(groups.max()) + 1 if n else 0
    out = np.full_like(o64, -np.inf)
    best = np.full((n_q, n_g), -1, dtype=np.int64)
    idx = np.arange(n)
    for q in range(n_q):
        o = o64[q]
        ok = np.isfinite(o)
        order = idx[ok][np.lexsort((idx[ok], -o[ok]))]
        _, first = np.unique(groups[order], return_index=True)
        b = order[first]
        out[q, b] = o[b]
        best[q, groups[b]] = b
    return out, best


def check_distinct(scores, rows, oracle64, groups, k, rtol=RTOL32, gb=None):
    """Distinct top-k check: distinct groups, each returned row within rtol of its group's best (the row itself when
    they tie exactly), and the strict top-k checker on the matrix that keeps only every group's best row.  ``gb``:
    group_best(oracle64, groups), when the caller has it already."""
    scores, rows, groups = np.asarray(scores), np.asarray(rows), np.asarray(groups)
    masked, best = gb if gb is not None else group_best(oracle64, groups)
    o64 = np.asarray(oracle64, dtype=np.float64)
    mapped = rows.copy()
    for q in range(rows.shape[0]):
        r = rows[q][rows[q] >= 0]
        where = f"query {q}: rows {rows[q].tolist()} scores {scores[q].tolist()}"
        g = groups[r]
        assert len(np.unique(g)) == len(g), "two rows of one group; " + where
        for j, (row, grp) in enumerate(zip(r.tolist(), g.tolist())):
            b = best[q, grp]
            assert b >= 0 and np.isfinite(o64[q, row]), "a row the query may not match; " + where
            ob = o64[q, b]
            if row != b:
                assert o64[q, row] != ob, f"row {row} ties its group's best row {b} exactly: the lower row wins; " + where
                assert abs(o64[q, row] - ob) <= rtol * abs(ob), f"row {row} is worse than its group's best {b}; " + where
                mapped[q, j] = b   # a near tie inside the group: judge the group by its best row
    check_topk_strict(scores, mapped, masked, k, rtol)


def test_checker_rejects_bad_answers():
    """CPU self-test of check_distinct on hand-made answers."""
    # rows 0..5; groups {0: rows 0, 3}, {1: rows 1, 4}, {2: row 2}, {3: row 5}
    groups = np.array([0, 1, 2, 0, 1, 3])
    o = np.array([[0.9, 0.5, 0.7, 0.9, 0.6, 0.1]])
    good_r = np.array([[0, 2, 4, 5]])
    good_s = o[0, good_r[0]].astype(np.float32)[None]
    check_distinct(good_s, good_r, o, groups, 4)
    k3_r, k3_s = good_r[:, :3], good_s[:, :3]
    check_distinct(k3_s, k3_r, o, groups, 3)
    with pytest.raises(AssertionError):   # two rows of one group
        check_distinct(np.float32([[0.9, 0.9, 0.7]]), np.array([[0, 3, 2]]), o, groups, 3)
    with pytest.raises(AssertionError):   # a clearly worse row of a group (row 1 instead of row 4)
        check_distinct(np.float32([[0.9, 0.7, 0.5]]), np.array([[0, 2, 1]]), o, groups, 3)
    with pytest.raises(AssertionError):   # a missing group (group 1 skipped for group 3)
        check_distinct(np.float32([[0.9, 0.7, 0.1]]), np.array([[0, 2, 5]]), o, groups, 3)
    with pytest.raises(AssertionError):   # the wrong row of an exact tie (row 3 instead of row 0)
        check_distinct(np.float32([[0.9, 0.7, 0.6]]), np.array([[3, 2, 4]]), o, groups, 3)
    with pytest.raises(AssertionError):   # (-inf, -1) missing past the last group
        check_distinct(np.float32([[0.9, 0.7, 0.6, 0.1, 0.0]]), np.array([[0, 2, 4, 5, 1]]), o, groups, 5)


# ---- the shared GPU case ---------------------------------------------------------------------------------------------

def text_groups(texts):
    _, inv = np.unique(np.asarray(texts, dtype=object).astype(str), return_inverse=True)
    return inv.astype(np.int32)


def wide(m):
    return " ".join(f"pw{i}" for i in reversed(range(m)))


def make_corpus(n, rng):
    """synth rows (30 % duplicates) plus: text A stored 40 (= k + 8) times and a similar text B stored 40 times, at
    scattered rows, and text C stored 2500 times -- a run of copies that spans more than one 64-chunk window and
    several row splits in text order."""
    from kakveda_b200 import synth

    corpus = synth.corpus(n)
    a = corpus[11]
    b = a + " variant"
    c = corpus[23] + " widely repeated"
    pos = rng.permutation(np.arange(100, n))
    for i in pos[:40]:
        corpus[i] = a
    for i in pos[40:80]:
        corpus[i] = b
    for i in pos[80:2580]:
        corpus[i] = c
    corpus[n // 3 + 1] = " ".join(f"pw{i}" for i in range(70))
    return corpus, (a, b, c)


def group_sets(corpus, rng):
    n = len(corpus)
    from kakveda_b200.similarity import Vocabulary, text_order

    v = Vocabulary()
    fb = v.featurize(corpus, grow=True)
    pos = np.empty(n, np.int64)
    pos[text_order(fb)] = np.arange(n)   # runs of 2100 rows in text order straddle 64-chunk windows and row splits
    fb.close()
    v.close()
    return {
        "text": text_groups(corpus),
        "random": rng.integers(0, 5000, size=n).astype(np.int32),
        "huge3": rng.integers(0, 3, size=n).astype(np.int32),
        "straddle": (pos // 2100).astype(np.int32),
    }


class Case:
    def __init__(self, n=N_ROWS, mode=0, seed=11):
        from kakveda_b200 import GfkbIndex, synth

        rng = np.random.default_rng(seed)
        self.corpus, (a, b, c) = make_corpus(n, rng)
        qs = synth.queries(150, n)
        # copies of A, B and C, a null query, an out-of-vocabulary one, a regular 64-feature and an irregular 65-feature
        self.queries = qs[:100] + [a, b, c, "", "qqzzunseen xxyyq", wide(QFEATS), wide(QFEATS + 1)] + qs[100:]
        self.ix = GfkbIndex()
        if mode:
            self.ix.set_mode(mode)
        self.ix.add_texts(self.corpus)
        self.ix.finalize()
        score = O.corpus_fit_scores if mode == 2 else O.score_matrix_closed_form
        self.oracle = score(self.queries, self.corpus)
        self.groups = group_sets(self.corpus, rng)
        self._best = {}

    def best(self, shape):
        if shape not in self._best:
            self._best[shape] = group_best(self.oracle, self.groups[shape])
        return self._best[shape]


@pytest.fixture(scope="module")
def lib(built_lib):
    from kakveda_b200 import _capi

    assert _capi.load().kv_device_count() > 0, "GPU tests need a CUDA device"
    return _capi.load()


@pytest.fixture(scope="module")
def case(lib):
    return Case()


@gpu
@pytest.mark.parametrize("shape", ["text", "random", "huge3", "straddle"])
@pytest.mark.parametrize("env", ENVS)
def test_distinct_topk_group_shapes(case, monkeypatch, shape, env):
    if env:
        monkeypatch.setenv(*env)
    g = case.groups[shape]
    case.ix.set_row_groups(g)
    gb = case.best(shape)
    for k in KS:
        s, r = case.ix.topk(case.queries, k, distinct=True)
        check_distinct(s, r, case.oracle, g, k, gb=gb)
        if shape == "huge3":
            assert np.all(r[:, 3:] == -1)   # three groups: the list is shorter than k


@gpu
def test_text_groups_collapse_copies(case):
    """Copies of one text are one result: a copy of A (stored 40 times) gets A first and B next; without distinct the
    40 copies fill the whole list."""
    ix = case.ix
    ix.set_row_groups(case.groups["text"])
    corpus = np.array(case.corpus, dtype=object)
    a, b = case.queries[100], case.queries[101]
    s0, r0 = ix.topk([a], 32)
    assert set(corpus[r0[0]].tolist()) == {a}   # 32 of the 41 copies of A
    s, r = ix.topk([a], 32, distinct=True)
    texts = corpus[r[0][r[0] >= 0]].tolist()
    assert texts[0] == a and b in texts and len(set(texts)) == len(texts) == 32
    assert r[0, 0] == np.flatnonzero(corpus == a)[0]   # the lowest copy


@gpu
@pytest.mark.parametrize("n_chunks", [511, 513, 1875])
def test_singleton_groups_give_non_distinct_bits(lib, case, monkeypatch, n_chunks):
    from kakveda_b200 import GfkbIndex

    if n_chunks == 1875:
        ix, qs = case.ix, case.queries
    else:
        rng = np.random.default_rng(n_chunks)
        corpus, _ = make_corpus(n_chunks * 32, rng)
        ix = GfkbIndex()
        ix.add_texts(corpus)
        ix.finalize()
        qs = case.queries
    ix.set_row_groups(np.arange(ix.n_rows, dtype=np.int32))
    for env in (None, NO_PRUNE):
        if env:
            monkeypatch.setenv(*env)
        for k in (1, 5, 16, 32):
            s0, r0 = ix.topk(qs, k)
            s1, r1 = ix.topk(qs, k, distinct=True)
            assert r1.tobytes() == r0.tobytes() and s1.tobytes() == s0.tobytes(), (n_chunks, env, k)


@gpu
def test_distinct_same_bits_on_every_path(case, monkeypatch):
    ix = case.ix
    ix.set_row_groups(case.groups["text"])
    for k in (5, 16, 32):
        s0, r0 = ix.topk(case.queries, k, distinct=True)
        check_distinct(s0, r0, case.oracle, case.groups["text"], k, gb=case.best("text"))
        runs = [("again", None)] + [(e, v) for e, v in (NO_PRUNE, ("KAKVEDA_B200_BOUND_CODES", "0"),
                                                          ("KAKVEDA_B200_GENERIC_BOUND", "1"))]
        runs += [("KAKVEDA_B200_CODE_SPLITS", str(c)) for c in (1, 2, 5)]
        for e, v in runs:
            with monkeypatch.context() as m:
                if v is not None:
                    m.setenv(e, v)
                s, r = ix.topk(case.queries, k, distinct=True)
            assert r.tobytes() == r0.tobytes() and s.tobytes() == s0.tobytes(), (e, v, k)


@gpu
@pytest.mark.parametrize("n_q", [1, 31, 33, 129])
def test_distinct_batch_sizes(case, n_q):
    ix = case.ix
    g = case.groups["random"]
    ix.set_row_groups(g)
    # the special queries (copies of A, B, C, null, out-of-vocabulary, 64 and 65 features) at the end of the batch
    others = [i for i in range(len(case.queries)) if not 100 <= i < 107]
    sel = [106] if n_q == 1 else others[:n_q - 7] + list(range(100, 107))
    assert len(sel) == n_q
    qs = [case.queries[i] for i in sel]
    masked, best = case.best("random")
    for k in (2, 31):
        s, r = ix.topk(qs, k, distinct=True)
        check_distinct(s, r, case.oracle[sel], g, k, gb=(masked[sel], best[sel]))


@gpu
def test_distinct_null_and_irregular_queries(case):
    ix = case.ix
    g = case.groups["text"]
    ix.set_row_groups(g)
    special = list(range(100, 107))
    qs = [case.queries[i] for i in special]
    for k in KS:
        s, r = ix.topk(qs, k, distinct=True)
        check_distinct(s, r, case.oracle[special], g, k)
    # the null query: the first row of each new group, in ascending row order
    s, r = ix.topk([""], 32, distinct=True)
    _, first = np.unique(g, return_index=True)
    assert r[0].tolist() == np.sort(first)[:32].tolist() and np.all(s[0] == 0)


@gpu
def test_distinct_corpus_fit_mode(lib):
    c = Case(n=20000, mode=2, seed=5)
    for shape in ("text", "random"):
        g = c.groups[shape]
        c.ix.set_row_groups(g)
        for k in KS:
            s, r = c.ix.topk(c.queries, k, distinct=True)
            check_distinct(s, r, c.oracle, g, k)


def masked(oracle, row_labels, q_labels):
    o = np.array(oracle, dtype=np.float64, copy=True)
    for q, lb in enumerate(q_labels):
        if lb >= 0:
            o[q, row_labels != lb] = -np.inf
    return o


@gpu
@pytest.mark.parametrize("nested", [True, False])
@pytest.mark.parametrize("env", [None, NO_PRUNE])
def test_distinct_with_label_filter(case, monkeypatch, nested, env):
    if env:
        monkeypatch.setenv(*env)
    rng = np.random.default_rng(3)
    g = case.groups["text"] if nested else case.groups["random"]
    labels = (g % 8).astype(np.int32) if nested else rng.integers(0, 8, size=N_ROWS).astype(np.int32)
    ql = rng.integers(-1, 8, size=len(case.queries)).astype(np.int32)
    ql[100:107] = [labels[np.flatnonzero(np.array(case.corpus, dtype=object) == case.queries[100])[0]], 3, -1, 2, 5, 1, 0]
    ix = case.ix
    ix.set_row_labels(labels)
    ix.set_row_groups(g)
    want = masked(case.oracle, labels, ql)
    gb = group_best(want, g)
    for k in (1, 5, 16, 32):
        s, r = ix.topk(case.queries, k, labels=ql, distinct=True)
        check_distinct(s, r, want, g, k, gb=gb)


@gpu
def test_distinct_selfjoin(case):
    ix = case.ix
    g = case.groups["text"]
    ix.set_row_groups(g)
    corpus = np.array(case.corpus, dtype=object)
    a_rows = np.flatnonzero(corpus == case.queries[100])   # row 11 and 40 scattered copies
    lo = max(0, int(a_rows[1]) - 40)
    hi = lo + 120
    o = O.score_matrix_closed_form(case.corpus[lo:hi], case.corpus)
    o[np.arange(hi - lo), np.arange(lo, hi)] = -np.inf   # the row itself is excluded
    for k in (1, 16, 32):
        s, r = ix.selfjoin_topk(k, lo, hi, distinct=True)
        check_distinct(s, r, o, g, k)
    # a copy of A: its own group still counts through its other copies -- the lowest other one comes first
    s, r = ix.selfjoin_topk(4, int(a_rows[1]), int(a_rows[1]) + 1, distinct=True)
    assert r[0, 0] == a_rows[0]
    s, r = ix.selfjoin_topk(4, int(a_rows[0]), int(a_rows[0]) + 1, distinct=True)
    assert r[0, 0] == a_rows[1]


@gpu
def test_distinct_with_deletions(lib, monkeypatch):
    from kakveda_b200 import GfkbIndex

    rng = np.random.default_rng(9)
    n = 20000
    corpus, (a, b, c) = make_corpus(n, rng)
    arr = np.array(corpus, dtype=object)
    g = text_groups(corpus)
    ix = GfkbIndex()
    ix.add_texts(corpus)
    ix.finalize()
    ix.set_row_groups(g)
    a_rows = np.flatnonzero(arr == a)
    rand = np.setdiff1d(rng.choice(n, 1500, replace=False), a_rows)
    dead = np.unique(np.concatenate([rand, a_rows[:3]]))  # A's three best rows among them
    ix.delete_rows(dead)
    ix.finalize()
    live = np.setdiff1d(np.arange(n), dead)
    from kakveda_b200 import synth

    qs = synth.queries(40, n) + [a, b, c, "", wide(QFEATS + 1)]
    o = np.full((len(qs), n), -np.inf)
    o[:, live] = O.score_matrix_closed_form(qs, [corpus[i] for i in live])
    gb = group_best(o, g)
    for env in (None, NO_PRUNE):
        if env:
            monkeypatch.setenv(*env)
        for k in (1, 16, 32):
            s, r = ix.topk(qs, k, distinct=True)
            check_distinct(s, r, o, g, k, gb=gb)
    s, r = ix.topk([a], 2, distinct=True)
    assert r[0, 0] == a_rows[3]   # the group's best live row


@gpu
def test_state_and_errors(lib, tmp_path):
    from kakveda_b200 import GfkbIndex, synth

    rng = np.random.default_rng(4)
    corpus, (a, b, c) = make_corpus(20000, rng)
    g = text_groups(corpus)
    ix = GfkbIndex()
    ix.add_texts(corpus)
    q = corpus[:20] + [a, b, c, "", "fresh text entirely unseen words"]
    fb = ix.vocab.featurize(q, grow=False)
    ix.set_row_groups(g)   # before finalize
    ix.finalize()
    assert ix.last_finalize_kind == 1
    s, r = ix.topk(q, 8, distinct=True)
    plain = ix.topk(q, 8)
    # setting groups changes nothing without distinct mode
    ix.set_row_groups(None)
    assert ix.topk(q, 8)[1].tobytes() == plain[1].tobytes()
    ix.set_row_groups(g)
    assert ix.topk(q, 8)[1].tobytes() == plain[1].tobytes()
    with pytest.raises(ValueError):
        ix.set_row_groups(g[:-1])
    with pytest.raises(ValueError):
        ix.set_row_groups(np.where(g == 0, -1, g))
    # kind-2 finalize and a layout reload keep the groups
    ix.set_global_df(ix.local_df(), 20000)
    ix.finalize()
    assert ix.last_finalize_kind == 2
    s2, r2 = ix.topk(q, 8, distinct=True)
    assert r2.tobytes() == r.tobytes() and s2.tobytes() == s.tobytes()
    path = tmp_path / "x.layout"
    ix.save_layout(path)
    b2 = GfkbIndex()
    b2.add_texts(corpus)
    b2.set_row_groups(g)
    assert b2.load_layout(path)
    b2.finalize()
    assert b2.last_finalize_kind == 2
    s3, r3 = b2.topk(q, 8, distinct=True)
    assert r3.tobytes() == r.tobytes() and s3.tobytes() == s.tobytes()
    # the two-phase top-k and the threshold exchange refuse distinct mode
    import torch

    ds = torch.empty((len(q), 8), dtype=torch.float32, device="cuda")
    dr = torch.empty((len(q), 8), dtype=torch.int64, device="cuda")
    ix.upload_queries(fb)
    ix.set_distinct(True)
    with pytest.raises(ValueError):
        ix.topk_resident_seed(8, ds.data_ptr(), dr.data_ptr())
    with pytest.raises(ValueError):
        ix.topk_resident_finish(8, ds.data_ptr(), dr.data_ptr())
    ix.topk_resident(8, ds.data_ptr(), dr.data_ptr())
    assert dr.cpu().numpy().tobytes() == r.tobytes()
    # the next upload switches distinct mode off
    ix.upload_queries(fb)
    assert ix.topk_resident_host(len(q), 8)[1].tobytes() == plain[1].tobytes()
    # threshold search ignores distinct mode
    ix.upload_queries(fb)
    ix.set_distinct(True)
    got = ix._range_resident(len(q), 0.5)
    want = ix.range(q, 0.5)
    assert all(np.array_equal(x, y) for x, y in zip(got, want))
    # an append makes the groups stale: distinct mode fails until they are set again
    ix.add_texts(["an appended row about citations"])
    ix.set_global_df(ix.local_df(), 20001)
    ix.finalize()
    assert not ix.has_row_groups
    with pytest.raises(RuntimeError):
        ix.topk(q, 8, distinct=True)
    with pytest.raises(RuntimeError):
        ix.selfjoin_topk(4, 0, 10, distinct=True)
    ix.set_row_groups(np.append(g, g.max() + 1).astype(np.int32))
    ix.topk(q, 8, distinct=True)
    # no groups at all
    ix.set_row_groups(None)
    ix.upload_queries(fb)
    with pytest.raises(RuntimeError):
        ix.set_distinct(True)
    fb.close()
    # Jaccard mode has no distinct top-k
    j = GfkbIndex()
    j.set_mode(1)
    j.add_texts([f"alpha{i} beta{i}" for i in range(500)])
    j.finalize()
    with pytest.raises(ValueError):
        j.set_row_groups(np.zeros(500, np.int32))
    with pytest.raises(ValueError):
        j.topk(["alpha1 beta1"], 4, distinct=True)
    from kakveda_b200 import DenseIndex, JaccardIndex, HashIndex

    with pytest.raises(NotImplementedError):
        DenseIndex.topk(object.__new__(DenseIndex), np.zeros((1, 8), np.float32), 4, distinct=True)
    with pytest.raises(NotImplementedError):
        JaccardIndex.topk_sets(object.__new__(JaccardIndex), [[1]], 4, distinct=True)
    with pytest.raises(NotImplementedError):
        HashIndex.match_signatures(object.__new__(HashIndex), ["x"], 4, distinct=True)


# ---- the store ---------------------------------------------------------------------------------------------------

def oracle_distinct_match(st, sig, limit, ft=None):
    """The newest version per (type, text) key, ranked by its float64 score and the key's first row."""
    texts = [r["signature_text"] for r in st.records]
    scores = O.score_sklearn(sig, texts)
    first = {}
    for i, r in enumerate(st.records):
        if ft and r["failure_type"] != ft:
            continue
        first.setdefault((r["failure_type"], r["signature_text"]), i)
    keys = sorted(first, key=lambda key: (-scores[first[key]], first[key]))[:limit]
    out = []
    for key in keys:
        rec = st.records[st._latest[key]]
        out.append((rec["failure_id"], rec["version"], scores[first[key]], rec["failure_type"]))
    return out


def check_store(st, sigs, limit=5, ft=None, filter_first=False):
    fts = [ft] * len(sigs)
    got = st.match_batch(sigs, fts, limit=limit, filter_first=filter_first, distinct=True)
    for sig, ms in zip(sigs, got):
        want = oracle_distinct_match(st, sig, limit, ft if filter_first else None)
        if ft and not filter_first:   # the reference's order: the best keys, then the filter
            want = [w for w in want if w[3] == ft]
        assert [(m["failure_id"], m["version"]) for m in ms] == [w[:2] for w in want], sig
        np.testing.assert_allclose([m["score"] for m in ms], [w[2] for w in want], rtol=1e-9)
        keys = [(m["failure_type"], m["failure_id"]) for m in ms]
        assert len(set(keys)) == len(keys)


@gpu
def test_store_distinct_fixture54(lib, golden):
    from kakveda_b200 import GfkbStore

    g = golden("fixture54.json")
    st = GfkbStore()
    st._reset([dict(r) for r in g["records"]])
    sigs = [c["signature_text"] for c in g["match"]] + [r["signature_text"] for r in g["records"][:12]]
    default = st.match_batch(sigs)
    check_store(st, sigs)
    check_store(st, sigs, limit=32)
    assert st.match_batch(sigs) == default   # the default still replays the reference


@gpu
def test_store_distinct_service_stream(lib, golden):
    from kakveda_b200 import GfkbStore

    g = golden("service_upsert.json")
    st = GfkbStore(tail_limit=30)
    sigs = []
    for i, step in enumerate(g["steps"]):
        st.upsert(step["upsert"])
        sigs.append(step["upsert"]["signature_text"])
        if i % 15 == 14:   # main and tail segments, and compactions
            check_store(st, sigs[-20:])
    assert st._tail is not None and st._tail.n_rows > 0
    types = sorted({r["failure_type"] for r in st.records})
    for ft in types[:3]:
        check_store(st, sigs[:30], ft=ft, filter_first=True)
        check_store(st, sigs[:30], ft=ft)


@gpu
def test_store_distinct_purge_replay(lib, golden):
    from kakveda_b200 import GfkbStore

    st = GfkbStore(tail_limit=1000)
    seen = []
    for step in golden("purge.json")["steps"]:
        if "upsert" in step:
            st.upsert(step["upsert"])
            seen.append(step["upsert"]["signature_text"])
        elif "purge" in step:
            st.purge_apps(step["purge"])
            check_store(st, seen[-25:])
            check_store(st, seen[-25:], limit=16)


@gpu
def test_store_distinct_main_and_tail(lib):
    from kakveda_b200 import GfkbStore, synth

    st = GfkbStore(tail_limit=5000)
    corpus = synth.corpus(3000)
    recs = [{"failure_id": f"F-{i + 1:04d}", "version": 1, "failure_type": ["X", "Y", "Z"][i % 3], "signature_text": t,
             "affected_apps": ["a"], "occurrences": 1, "root_cause": None, "resolution": None, "context_signature": {}}
            for i, t in enumerate(corpus)]
    st._reset(recs)
    for i in range(60):   # the tail: new versions of main keys, copies under other types, and new keys
        st.upsert({"failure_type": ["X", "W", "Y"][i % 3], "signature_text": corpus[(i // 3) * 3],
                   "context_signature": {}, "impact_severity": "low", "app_id": "b"})
    qs = corpus[:60:3] + synth.queries(10, 3000)
    check_store(st, qs)
    check_store(st, qs, limit=32)
    assert st._tail is not None and st._tail.n_rows == 60
    for ft in ("X", "W"):
        check_store(st, qs, ft=ft, filter_first=True)


def test_store_distinct_ambiguous_candidates_take_group_aware_exact_path(built_lib, monkeypatch):
    """Colliding float32 groups force the exact path, which must be group-aware: key B (rows 20..39) beats key A (rows
    0..19) in float64 only; rows 40..59 are distinct keys at 0.25.  Each key is reported with its newest record."""
    from kakveda_b200 import GfkbStore

    n = 60
    f64 = np.full(n, 0.25)
    f64[0:20] = 0.8
    f64[20:40] = 0.8 + 1e-9
    texts = ["a"] * 20 + ["b"] * 20 + [f"c{i}" for i in range(20)]

    class FakeIndex:
        n_rows = n
        has_row_groups = False

        def set_row_groups(self, groups):
            self.groups = np.asarray(groups)
            self.has_row_groups = True

        def topk_features(self, fb, k, labels=None, distinct=False, tags=None):
            assert distinct and self.has_row_groups
            s32 = f64.astype(np.float32)
            _, first = np.unique(self.groups, return_index=True)
            order = first[np.lexsort((first, -s32[first]))][:k]
            return np.tile(s32[order], (fb.n, 1)), np.tile(order.astype(np.int64), (fb.n, 1))

        def rescore(self, fb, rows):
            return f64[rows]

        def score(self, text):
            return f64.copy()

        def close(self):
            pass

    st = GfkbStore()
    st.records = [{"failure_id": f"F-{i:04d}", "version": 1, "failure_type": "T", "resolution": None,
                   "signature_text": texts[i]} for i in range(n)]
    st._latest = {("T", t): i for i, t in enumerate(texts)}
    st._n_main = st._n_indexed = st._n_dev = n
    monkeypatch.setattr(st, "_sync", lambda: None)

    class _B:
        n = 1

        def close(self):
            pass
    monkeypatch.setattr(st.vocab, "featurize", lambda texts, grow=False, n_threads=0: _B())
    st._main = FakeIndex()
    got = st.match("q", distinct=True)
    assert [m["failure_id"] for m in got] == ["F-0039", "F-0019", "F-0040", "F-0041", "F-0042"]
    assert st.stats["exact_fallbacks"] == 1
    st._main = None


def test_first_of_groups_merges_segments(built_lib):
    """The host merge keeps the first row of each group of the (score desc, row asc) candidates of both segments."""
    from kakveda_b200 import GfkbStore

    st = GfkbStore()
    st.records = [{"failure_type": "T", "signature_text": t} for t in ["a", "b", "a", "c", "b"]]
    st._n_indexed = 5
    recs = np.array([[0, 2, 1, 4, 3, -1], [4, 1, 3, 0, -1, -1]])
    f64 = np.array([[0.9, 0.9, 0.5, 0.5, 0.1, -np.inf], [0.7, 0.7, 0.3, 0.2, -np.inf, -np.inf]])
    r, s = st._first_of_groups(recs, f64)
    assert r.tolist() == [[0, 1, 3, -1, -1, -1], [4, 3, 0, -1, -1, -1]]
    assert s[0, :3].tolist() == [0.9, 0.5, 0.1] and s[1, :3].tolist() == [0.7, 0.3, 0.2]


@gpu
def test_detect_patterns_distinct(lib):
    from kakveda_b200 import GfkbIndex, synth
    from kakveda_b200.patterns import detect_patterns

    base = synth.corpus(400)
    a = base[7]
    b = a + " alpha"
    recs = [{"failure_id": f"F-{i:04d}", "failure_type": "OTHER", "signature_text": t, "affected_apps": ["z"]}
            for i, t in enumerate(base)]
    for i in range(40):   # A and a similar B, each stored 40 times, each from two apps
        recs.append({"failure_id": f"A-{i:04d}", "failure_type": "X", "signature_text": a, "affected_apps": [f"app{i % 2}"]})
        recs.append({"failure_id": f"B-{i:04d}", "failure_type": "X", "signature_text": b, "affected_apps": [f"app{2 + i % 2}"]})
    ix = GfkbIndex()
    ix.set_mode(2)
    ix.add_texts([r["signature_text"] for r in recs])
    ix.finalize()
    default = detect_patterns(ix, recs, threshold=0.5, k=32, failure_type="X")
    assert len(default) == 2   # the copies fill the lists: A and B stay apart
    got = detect_patterns(ix, recs, threshold=0.5, k=32, failure_type="X", distinct=True)
    assert [p["rows"] for p in got] == [list(range(400, 480))]   # row 7 (A, another type) is another group
    assert detect_patterns(ix, recs, threshold=0.5, k=32, failure_type="X") == default
