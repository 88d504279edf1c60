"""Tag-filtered search: top-k, exact top-k and threshold search restricted to the rows whose tag set meets the query's
(e.g. a failure's affected apps), on one index, across the shards of a ``ShardedGfkb`` and through ``GfkbStore``.

A query with tags matches the rows whose set shares one of its tags; the scores and statistics are the unfiltered
ones, so the oracle is the float64 ``O.score_matrix_closed_form`` of the whole corpus with the ineligible pairs set to
-inf, checked with the strict tie rules of test_gpu_filtered_search.py.  The pruning test reads the layout counters:
a query of a rare tag must score fewer (query, chunk) pairs than the unfiltered batch.
"""
import numpy as np
import pytest

from oracle import tfidf_oracle as O
from test_gpu_filtered_search import RTOL32, _csr_mask, check_topk_strict

torch = pytest.importorskip("torch")

from test_gpu_shard_loopback import loopback  # noqa: E402,F401

gpu = pytest.mark.gpu

N_ROWS = 60000
KS = (1, 5, 16, 32)
QFEATS = 64
WIDE_ROW = 777          # the row with 100 tags


def row_tag_sets(n, rng, kind):
    """0-4 tags per row from 8 tags, or from 1,000 Zipf-weighted tags; rows 10..20 alternate {5} / {69} (masks collide:
    69 & 63 == 5), WIDE_ROW carries 100 tags, every 97th row none."""
    if kind == "small8":
        pool, p = np.arange(8), None
    else:
        w = 1.0 / np.arange(1, 1001)
        pool, p = np.arange(1000), w / w.sum()
    sets = []
    for r in range(n):
        m = int(rng.integers(0, 5))
        sets.append(sorted(set(rng.choice(pool, size=m, p=p).tolist())) if m else [])
    for r in range(10, 20):
        sets[r] = [5] if r % 2 == 0 else [69]
    for r in range(0, n, 97):
        sets[r] = []
    sets[WIDE_ROW] = list(range(300, 400))
    return sets


def query_tag_sets(n_q, rng, kind):
    """Sizes 0 (unfiltered), 1, 4 and 16; the first queries hold {5}, {69}, {350} and a tag no row carries."""
    top = 8 if kind == "small8" else 1000
    out = []
    for q in range(n_q):
        m = (0, 1, 4, 16)[q % 4]
        out.append(sorted(set(rng.integers(0, top, size=m).tolist())))
    out[:4] = [[5], [69], [350], [5000]]
    return out


def tag_mask(row_sets, q_sets):
    """bool [Q, N]: whether query q may match row r (an empty query set: every row)."""
    n = len(row_sets)
    by_tag = {}
    for r, ts in enumerate(row_sets):
        for t in ts:
            by_tag.setdefault(t, []).append(r)
    out = np.ones((len(q_sets), n), dtype=bool)
    for q, qs in enumerate(q_sets):
        if qs:
            m = np.zeros(n, dtype=bool)
            for t in qs:
                m[by_tag.get(t, [])] = True
            out[q] = m
    return out


class Case:
    def __init__(self, mode=0):
        from kakveda_b200 import GfkbIndex, synth

        rng = np.random.default_rng(5)
        corpus = synth.corpus(N_ROWS)
        corpus[N_ROWS // 3 + 1] = " ".join(f"pw{i}" for i in range(70))
        qs = synth.queries(120, N_ROWS)   # stored copies and fresh texts
        wide = lambda m: " ".join(f"pw{i}" for i in reversed(range(m)))
        self.queries = qs[:4] + [corpus[11], corpus[12]] + qs[4:] + ["", "qqzzunseen xxyyq", wide(QFEATS), wide(QFEATS + 1)]
        self.corpus = corpus
        self.ix = GfkbIndex()
        if mode:
            self.ix.set_mode(mode)
        self.ix.add_texts(corpus)
        self.ix.finalize()
        self.oracle = O.corpus_fit_scores(self.queries, corpus) if mode == 2 else O.score_matrix_closed_form(self.queries, corpus)
        self.rows = {k: row_tag_sets(N_ROWS, rng, k) for k in ("small8", "zipf1000")}
        self.qtags = {k: query_tag_sets(len(self.queries), rng, k) for k in self.rows}
        self.masks = {k: tag_mask(self.rows[k], self.qtags[k]) for k in self.rows}


@pytest.fixture(scope="module")
def lib(built_lib):
    from kakveda_b200 import _capi

    assert _capi.load().kv_device_count() > 0, "GPU tests need a CUDA device"
    return _capi.load()


@pytest.fixture(scope="module")
def case(lib):
    return Case()


def masked(oracle, mask):
    return np.where(mask, oracle, -np.inf)


@gpu
@pytest.mark.parametrize("kind", ["small8", "zipf1000"])
@pytest.mark.parametrize("env", [None, ("KAKVEDA_B200_BOUND_CODES", "0"), ("KAKVEDA_B200_NO_PRUNE", "1")])
def test_tag_topk_equals_masked_oracle(case, monkeypatch, kind, env):
    if env:
        monkeypatch.setenv(*env)
    ix = case.ix
    ix.set_row_tags(case.rows[kind])
    want = masked(case.oracle, case.masks[kind])
    for k in KS:
        s, r = ix.topk(case.queries, k, tags=case.qtags[kind])
        check_topk_strict(s, r, want, k, RTOL32)
        # {5} and {69} share their mask bit: only the exact test keeps the neighbouring rows apart
        assert not np.isin(r[0], np.arange(11, 20, 2)).any() and not np.isin(r[1], np.arange(10, 20, 2)).any()
        if k >= 1:
            assert r[2, 0] == WIDE_ROW or case.masks[kind][2].sum() > 1
        assert np.all(r[3] == -1)   # a tag no row carries
        empty = np.array([len(t) == 0 for t in case.rows[kind]])
        filt = np.array([len(t) > 0 for t in case.qtags[kind]])
        assert not empty[np.clip(r[filt], 0, None)][r[filt] >= 0].any(), "a row with no tags matched a tag-filtered query"


@gpu
def test_tag_topk_corpus_fit_mode(lib):
    c = Case(mode=2)
    c.ix.set_row_tags(c.rows["zipf1000"])
    want = masked(c.oracle, c.masks["zipf1000"])
    for k in KS:
        s, r = c.ix.topk(c.queries, k, tags=c.qtags["zipf1000"])
        check_topk_strict(s, r, want, k, RTOL32)


@gpu
def test_unfiltered_queries_keep_their_bits(case):
    ix = case.ix
    q = case.queries
    s0, r0 = ix.topk(q, 16)
    ix.set_row_tags(case.rows["small8"])
    s1, r1 = ix.topk(q, 16, tags=[[] for _ in q])   # no query has tags: the unfiltered batch
    assert s1.tobytes() == s0.tobytes() and r1.tobytes() == r0.tobytes()
    qt = case.qtags["small8"]
    s2, r2 = ix.topk(q, 16, tags=qt)
    free = np.array([len(t) == 0 for t in qt])
    assert s2[free].tobytes() == s0[free].tobytes() and r2[free].tobytes() == r0[free].tobytes()


@gpu
@pytest.mark.parametrize("kind", ["small8", "zipf1000"])
def test_tag_range_equals_unfiltered_minus_ineligible(case, kind):
    ix = case.ix
    ix.set_row_tags(case.rows[kind])
    mask = case.masks[kind]
    q = case.queries
    for thr in (0.3, 0.8):
        ip, rows, sc = ix.range(q, thr)
        want = _csr_mask(ip, rows, sc, lambda i, rr: mask[i, rr])
        got = ix.range(q, thr, tags=case.qtags[kind])
        for a, b in zip(got, want):
            assert a.tobytes() == b.tobytes(), thr
        dev = ix.range(q, thr, device_out=True, tags=case.qtags[kind])
        for a, b in zip(dev, want):
            assert a.cpu().numpy().tobytes() == b.tobytes(), thr


@gpu
def test_tags_with_labels_and_distinct(case):
    ix = case.ix
    rows, qt = case.rows["zipf1000"], case.qtags["zipf1000"]
    rng = np.random.default_rng(3)
    rl = rng.integers(0, 4, N_ROWS).astype(np.int32)
    ql = rng.choice(np.array([-1, 0, 1, 2, 3], np.int32), len(case.queries)).astype(np.int32)
    ix.set_row_tags(rows)
    ix.set_row_labels(rl)
    lab_mask = (ql[:, None] < 0) | (rl[None, :] == ql[:, None])
    want = masked(case.oracle, case.masks["zipf1000"] & lab_mask)
    for k in (1, 16, 32):
        s, r = ix.topk(case.queries, k, labels=ql, tags=qt)
        check_topk_strict(s, r, want, k, RTOL32)
    # distinct: singleton groups give the non-distinct bits; text groups keep one row per group
    ix.set_row_groups(np.arange(N_ROWS, dtype=np.int32))
    s1, r1 = ix.topk(case.queries, 16, labels=ql, tags=qt)
    s2, r2 = ix.topk(case.queries, 16, labels=ql, distinct=True, tags=qt)
    assert s1.tobytes() == s2.tobytes() and r1.tobytes() == r2.tobytes()
    _, groups = np.unique(np.array(case.corpus), return_inverse=True)
    groups = groups.astype(np.int32)
    ix.set_row_groups(groups)
    elig = case.masks["zipf1000"] & lab_mask
    # the distinct oracle: per query only the best eligible row of each group stays (a group's rows share their text,
    # hence their score, so the best is its lowest eligible row)
    best = np.full_like(case.oracle, -np.inf)
    for q in range(len(case.queries)):
        rows_e = np.flatnonzero(elig[q])
        _, first = np.unique(groups[rows_e], return_index=True)
        keep = rows_e[first]
        best[q, keep] = case.oracle[q, keep]
    for k in (1, 16, 32):
        s3, r3 = ix.topk(case.queries, k, labels=ql, distinct=True, tags=qt)
        check_topk_strict(s3, r3, best, k, RTOL32)
        for q in range(len(case.queries)):
            rr = r3[q][r3[q] >= 0]
            assert len(np.unique(groups[rr])) == len(rr)
    ix.set_row_labels(None)
    ix.set_row_groups(None)


@gpu
def test_singleton_tag_equals_label_filter(case):
    ix = case.ix
    rng = np.random.default_rng(9)
    rl = rng.integers(0, 6, N_ROWS).astype(np.int32)
    ql = rng.integers(0, 6, len(case.queries)).astype(np.int32)
    ix.set_row_labels(rl)
    ix.set_row_tags([[int(x)] for x in rl])
    for k in (1, 32):
        s1, r1 = ix.topk(case.queries, k, labels=ql)
        s2, r2 = ix.topk(case.queries, k, tags=[[int(x)] for x in ql])
        assert s1.tobytes() == s2.tobytes() and r1.tobytes() == r2.tobytes()
    ix.set_row_labels(None)


@gpu
def test_exact_topk_tags(case):
    ix = case.ix
    ix.set_row_tags(case.rows["zipf1000"])
    q = case.queries[:24]
    qt = case.qtags["zipf1000"][:24]
    fb = ix.vocab.featurize(q, grow=False)
    try:
        rows, scores = ix.exact_topk(fb, 16, tags=qt)
        r0, s0 = ix.exact_topk(fb, 16)
    finally:
        fb.close()
    want = masked(case.oracle[:24], case.masks["zipf1000"][:24])
    for i in range(len(q)):
        o = want[i]
        order = np.argsort(-o, kind="stable")[:16]
        order = order[np.isfinite(o[order])]
        got = rows[i][rows[i] >= 0]
        assert len(got) == len(order)
        np.testing.assert_allclose(scores[i][:len(got)], o[order], rtol=1e-9)
        assert case.masks["zipf1000"][i, got].all()
        if not qt[i]:
            assert np.array_equal(rows[i], r0[i])


@gpu
def test_tags_after_deletion_and_layout_reload(lib, tmp_path):
    from kakveda_b200 import GfkbIndex, synth

    n = 20000
    corpus = synth.corpus(n)
    rng = np.random.default_rng(2)
    rows = row_tag_sets(n, rng, "small8")
    queries = synth.queries(40, n) + [""]
    qt = query_tag_sets(len(queries), rng, "small8")
    mask = tag_mask(rows, qt)
    oracle = O.score_matrix_closed_form(queries, corpus)
    ix = GfkbIndex()
    ix.add_texts(corpus)
    ix.finalize()
    ix.set_row_tags(rows)
    path = tmp_path / "lay.bin"
    ix.save_layout(path)
    gone = rng.choice(n, size=3000, replace=False)
    ix.delete_rows(gone)
    ix.finalize()
    assert ix.last_finalize_kind == 2
    live = np.setdiff1d(np.arange(n), gone)   # N and df now count the live rows
    o_live = np.full_like(oracle, -np.inf)
    o_live[:, live] = O.score_matrix_closed_form(queries, [corpus[i] for i in live])
    for k in (1, 32):
        s, r = ix.topk(queries, k, tags=qt)
        check_topk_strict(s, r, np.where(mask, o_live, -np.inf), k, RTOL32)
    # a fresh handle over the same rows: the persisted layout, tags set before the finalize that follows the load
    ix2 = GfkbIndex(vocab=ix.vocab)
    ix2.add_texts(corpus)
    assert ix2.load_layout(path)
    ix2.set_row_tags(rows)
    ix2.finalize()
    for k in (5, 16):
        s, r = ix2.topk(queries, k, tags=qt)
        check_topk_strict(s, r, np.where(mask, oracle, -np.inf), k, RTOL32)
    ix.close()
    ix2.close()


@gpu
@pytest.mark.parametrize("env", [None, ("KAKVEDA_B200_BOUND_CODES", "0"), ("KAKVEDA_B200_NO_PRUNE", "1")])
def test_rare_tag_prunes_chunks(case, monkeypatch, env):
    """A tag on 60 rows (6 texts stored 10 times, so they cluster into few chunks): its queries score fewer
    (query, chunk) pairs than the unfiltered batch, and only its rows come back."""
    from kakveda_b200 import GfkbIndex

    if env:
        monkeypatch.setenv(*env)
    rng = np.random.default_rng(11)
    corpus = list(case.corpus)
    src = [corpus[i] + f" raretag{i}" for i in range(6)]
    rare = rng.choice(np.arange(100, N_ROWS), size=60, replace=False)
    for j, r in enumerate(rare):
        corpus[r] = src[j // 10]
    ix = GfkbIndex()
    ix.add_texts(corpus)
    ix.finalize()
    sets = [[1, 2] for _ in range(N_ROWS)]
    for r in rare:
        sets[r] = [2, 700]
    ix.set_row_tags(sets)
    queries = src + case.queries[:100]
    ix.topk(queries, 16)
    unfiltered = ix.layout()["pairs_scored"]
    s, r = ix.topk(queries, 16, tags=[[700, 900]] * len(queries))
    filtered = ix.layout()["pairs_scored"]
    assert 0 < filtered <= 2 * len(queries) * 12 < unfiltered, (filtered, unfiltered)
    assert np.all(np.isin(r[r >= 0], rare))
    for j in range(6):
        assert sorted(r[j, :10].tolist()) == sorted(rare[j * 10:(j + 1) * 10].tolist())
    ix.close()


@gpu
def test_state_and_validation(lib):
    from kakveda_b200 import GfkbIndex, _capi, synth

    corpus = synth.corpus(5000)
    ix = GfkbIndex()
    ix.add_texts(corpus)
    with pytest.raises(ValueError):
        ix.set_row_tags([[0]] * 4999)                 # wrong length
    with pytest.raises(ValueError):
        ix.set_row_tags([[0]] * 4998 + [[-1], [1]])   # a negative tag
    sets = [[r % 70] for r in range(5000)]
    ix.set_row_tags(sets)                             # before finalize: uploaded by it
    ix.finalize()
    q = synth.queries(8, 5000)
    s, r = ix.topk(q, 4, tags=[[3]] * 8)
    assert np.all((r < 0) | (r % 70 == 3))
    with pytest.raises(ValueError):
        ix.topk(q, 4, tags=[list(range(17))] * 8)     # more than 16 tags
    with pytest.raises(ValueError):
        ix.topk(q, 4, tags=[[-2]] * 8)
    with pytest.raises(ValueError):
        ix.topk(q, 4, tags=[[1]] * 7)                 # wrong length
    # the filter goes with the next upload
    fb = ix.vocab.featurize(q, grow=False)
    ix.upload_queries(fb)
    ix.set_tag_filter([[3]] * 8)
    ix.upload_queries(fb)
    s1, r1 = ix.topk_resident_host(8, 4)
    s0, r0 = ix.topk(q, 4)
    assert r1.tobytes() == r0.tobytes()
    # tags reset on a finalized index need no finalize
    ix.set_row_tags([[(r + 1) % 70] for r in range(5000)])
    s, r = ix.topk(q, 4, tags=[[3]] * 8)
    assert np.all((r < 0) | ((r + 1) % 70 == 3))
    # an append makes the tags stale: a query with tags fails until they are set again, one without runs
    ix.add_texts(["fresh row text"])
    ix.finalize()
    with pytest.raises(RuntimeError):
        ix.topk(q, 4, tags=[[3]] * 8)
    ix.topk(q, 4, tags=[[]] * 8)
    with pytest.raises(RuntimeError):
        ix.exact_topk(fb, 4, tags=[[3]] * 8)
    ix.set_row_tags(sets + [[3]])
    ix.topk(q, 4, tags=[[3]] * 8)
    fb.close()
    # a Jaccard index has no tag filter
    j = GfkbIndex()
    j.set_mode(1)
    j.add_texts(["alpha1 beta1", "alpha2 beta2"])
    with pytest.raises(ValueError):
        j.set_row_tags([[0], [1]])
    j.finalize()
    with pytest.raises(ValueError, match="Jaccard"):
        j.topk(["alpha1 beta1", "alpha2"], 2, tags=[[0], [1]])      # kv_query_set_tag_filter
    jfb = j.vocab.featurize(["alpha1 beta1", "alpha2"], grow=False)
    try:
        with pytest.raises(ValueError, match="Jaccard"):
            j.exact_topk(jfb, 2, tags=[[0], [1]])                     # kv_exact_topk_tags
    finally:
        jfb.close()
    # a tuple of per-query lists is a sequence of sets, not a CSR pair
    s_t, r_t = ix.topk(q[:3], 4, tags=([3], [4], [5]))
    s_l, r_l = ix.topk(q[:3], 4, tags=[[3], [4], [5]])
    assert r_t.tobytes() == r_l.tobytes()
    ix.close()
    j.close()


# ---------------------------------------------------------------------------------------------------------------------
# ShardedGfkb: each shard filters its own rows; results equal the single index
# ---------------------------------------------------------------------------------------------------------------------

SHARD_CASES = [("rows", "index", 1), ("rows", "index", 2), ("rows", "index", 3), ("rows", "index", 8), ("rows", "text", 3),
               ("queries", "index", 2), ("queries", "index", 3)]


@gpu
@pytest.mark.parametrize("mode,order,world", SHARD_CASES, ids=[f"{m}-{o}-W{w}" for m, o, w in SHARD_CASES])
def test_sharded_tags_equal_single_index(lib, loopback, mode, order, world):
    from kakveda_b200 import GfkbIndex, synth
    from kakveda_b200.dist import ShardedGfkb
    from kakveda_b200.similarity import pack_texts
    from test_gpu_shard_loopback import run_ranks

    n = 30000
    corpus = synth.corpus(n)
    rng = np.random.default_rng(world)
    rows = row_tag_sets(n, rng, "zipf1000")
    queries = synth.queries(60, n) + ["", " ".join(f"w{i}" for i in range(80))]
    qt = query_tag_sets(len(queries), rng, "zipf1000")
    single = GfkbIndex()
    single.add_texts(corpus)
    single.finalize()
    single.set_row_tags(rows)
    fb = single.vocab.featurize(queries, grow=False)
    want_topk = {k: single.topk_features(fb, k, tags=qt) for k in (1, 16)}
    want_exact = single.exact_topk(fb, 8, tags=qt)
    fb.close()
    want_range = single.range(queries, 0.4, tags=qt)
    data, off, pmode = pack_texts(corpus)
    qdata, qoff, qmode = pack_texts(queries)

    def fn(rk, g):
        sh = ShardedGfkb(device=0, rank=rk, world=world, group=g, mode=mode, order=order)
        try:
            sh.build_packed(data, off, pmode)
            sh.set_row_tags(rows)
            out = {}
            for k in (1, 16):
                s, r = sh.topk_packed(qdata, qoff, k, qmode, tags=qt)
                out["topk", k] = (np.array(s), np.array(r))
            qfb = sh.vocab.featurize(queries, grow=False)
            try:
                out["exact"] = sh.exact_topk(qfb, 8, tags=qt)
                with pytest.raises(ValueError, match="tags"):
                    sh.exact_topk(qfb, 8, tags=qt[:3])
            finally:
                qfb.close()
            ip, rr, ss = sh.range_packed(qdata, qoff, 0.4, qmode, tags=qt)
            out["range"] = (np.asarray(ip), np.asarray(rr), np.asarray(ss))
            return out
        finally:
            sh.close()

    outs = run_ranks(world, fn)
    for out in outs:
        for k in (1, 16):
            s, r = out["topk", k]
            np.testing.assert_array_equal(r, want_topk[k][1])
            assert s.tobytes() == want_topk[k][0].tobytes()
        np.testing.assert_array_equal(out["exact"][0], want_exact[0])
        np.testing.assert_array_equal(out["exact"][1], want_exact[1])
        for a, b in zip(out["range"], want_range):
            assert a.tobytes() == b.tobytes()
    single.close()


# ---------------------------------------------------------------------------------------------------------------------
# GfkbStore: app-scoped match
# ---------------------------------------------------------------------------------------------------------------------

def _oracle_app_match(st, sig, app, limit, ft=None):
    """Brute-force float64 over the records listing ``app`` (and of type ``ft``), stable top ``limit``."""
    scores = O.score_sklearn(sig, [r["signature_text"] for r in st.records])
    cand = [(i, s) for i, s in enumerate(scores)
            if app in (st.records[i].get("affected_apps") or []) and (ft is None or st.records[i]["failure_type"] == ft)]
    return sorted(cand, key=lambda t: t[1], reverse=True)[:limit]


def _check_app_matches(st, sigs, apps, got, limit=5, ft=None):
    for sig, app, ms in zip(sigs, apps, got):
        want = _oracle_app_match(st, sig, app, limit, ft)
        assert [m["failure_id"] for m in ms] == [st.records[i]["failure_id"] for i, _ in want], (sig, app)
        np.testing.assert_allclose([m["score"] for m in ms], [s for _, s in want], rtol=1e-9)


def _fixture_records(golden):
    g = golden("fixture54.json")
    recs = [json_copy(r) for r in g["records"]]
    apps = ["app-a", "app-b", "app-c", "app-d"]
    types = ["TYPE_A", "TYPE_B", "TYPE_C"]
    for i, r in enumerate(recs):
        r["affected_apps"] = [apps[i % 4]] + ([apps[(i + 1) % 4]] if i % 3 == 0 else [])
        r["failure_type"] = types[(i * 7) % 3]
    sigs = [c["signature_text"] for c in g["match"]] + [r["signature_text"] for r in recs[:10]]
    return recs, sigs, apps, types


def json_copy(r):
    import json

    return json.loads(json.dumps(r))


@gpu
def test_store_app_match_fixture54(lib, golden):
    from kakveda_b200 import GfkbStore

    recs, sigs, apps, types = _fixture_records(golden)
    st = GfkbStore()
    st._reset(recs)
    before = st.match_batch(sigs)
    for app in apps:
        got = st.match_batch(sigs, app_ids=[app] * len(sigs))
        _check_app_matches(st, sigs, [app] * len(sigs), got)
        for ft in types:
            got = st.match_batch(sigs, [ft] * len(sigs), filter_first=True, app_ids=[app] * len(sigs))
            _check_app_matches(st, sigs, [app] * len(sigs), got, ft=ft)
            # without filter_first the reference's type post-filter follows the app-scoped top-k
            got = st.match_batch(sigs, [ft] * len(sigs), app_ids=[app] * len(sigs))
            for sig, ms in zip(sigs, got):
                want = [(i, s) for i, s in _oracle_app_match(st, sig, app, 5) if st.records[i]["failure_type"] == ft]
                assert [m["failure_id"] for m in ms] == [st.records[i]["failure_id"] for i, _ in want]
    assert st.match(sigs[0], app_id="no-such-app") == []
    assert st.match(sigs[0], app_id=None) == st.match(sigs[0])
    assert st.match_batch(sigs) == before
    # a purge rewrites affected_apps: the app tags follow
    st.purge_apps(["app-b"], backup=False)
    got = st.match_batch(sigs, app_ids=["app-c"] * len(sigs))
    _check_app_matches(st, sigs, ["app-c"] * len(sigs), got)
    scans = []
    orig = st._candidates
    st._candidates = lambda *a, **kw: scans.append(1) or orig(*a, **kw)
    assert st.match(sigs[0], app_id="app-b") == []   # no record lists it any more: no scan
    assert st.match(sigs[0], app_id="no-such-app") == [] and not scans
    assert st.match(sigs[0], app_id="app-c") and scans
    del st._candidates


def _synthetic_store(st, n, rng):
    """Records over synthetic texts; later versions of a failure add apps, so an app's rows are spread over main and
    tail segments."""
    from kakveda_b200 import synth

    texts = synth.corpus(n)
    recs = []
    for i, t in enumerate(texts):
        recs.append({"failure_id": f"F-{i + 1:04d}", "version": 1, "created_at": "2024-01-01T00:00:00Z",
                     "updated_at": "2024-01-01T00:00:00Z", "failure_type": f"T{i % 3}", "root_cause": None,
                     "context_signature": {}, "impact_severity": "low", "resolution": None, "occurrences": 1,
                     "affected_apps": [f"app{int(rng.integers(0, 20))}"], "signature_text": t})
    st._reset(recs)
    for j in range(300):   # upserts: new versions with an extra app land in the tail
        base = recs[int(rng.integers(0, n))]
        st.upsert({"failure_type": base["failure_type"], "signature_text": base["signature_text"],
                   "context_signature": {}, "impact_severity": "low", "app_id": f"app{int(rng.integers(0, 25))}"})
    return texts


@gpu
def test_store_app_match_main_tail_and_fallback(lib, monkeypatch):
    from kakveda_b200 import GfkbStore, synth
    from kakveda_b200 import store as store_mod

    rng = np.random.default_rng(4)
    st = GfkbStore(tail_limit=1000)
    texts = _synthetic_store(st, 3000, rng)
    sigs = [texts[i] for i in rng.choice(3000, 12, replace=False)] + synth.queries(8, 3000)
    apps = [f"app{int(a)}" for a in rng.integers(0, 25, len(sigs))]
    got = st.match_batch(sigs, app_ids=apps)
    assert st._tail is not None and st._tail.n_rows > 0
    _check_app_matches(st, sigs, apps, got)
    got = st.match_batch(sigs, ["T1"] * len(sigs), filter_first=True, app_ids=apps)
    for sig, app, ms in zip(sigs, apps, got):
        _check_app_matches(st, [sig], [app], [ms], ft="T1")
    # every query ambiguous: the exact fallback decides
    monkeypatch.setattr(store_mod, "ambiguous_candidates", lambda s32, rows, limit: np.ones(len(rows), dtype=bool))
    n0 = st.stats.get("exact_fallbacks", 0)
    got = st.match_batch(sigs, app_ids=apps)
    assert st.stats["exact_fallbacks"] == n0 + len(sigs)
    _check_app_matches(st, sigs, apps, got)
    monkeypatch.undo()
    # after a purge that deletes rows and rewrites lists
    st.purge_apps(["app3", "app7"], backup=False)
    got = st.match_batch(sigs, app_ids=apps)
    _check_app_matches(st, sigs, apps, got)


@gpu
def test_store_warn_app_scoped(lib, golden):
    from kakveda_b200 import GfkbStore
    from kakveda_b200 import store as store_mod

    recs, sigs, apps, _ = _fixture_records(golden)
    st = GfkbStore()
    st._reset(recs)
    reqs = [{"prompt": r["signature_text"], "app_id": apps[(i + 2) % 4], "tools": [], "env": {}}
            for i, r in enumerate(recs[:12])]
    plain = st.warn_batch(reqs)
    assert st.warn_batch(reqs, app_scoped=False) == plain
    scoped = st.warn_batch(reqs, app_scoped=True)
    sigs = [store_mod._signature_text(r["prompt"], [], {}) for r in reqs]
    matches = st.match_batch(sigs, app_ids=[r["app_id"] for r in reqs])
    _check_app_matches(st, sigs, [r["app_id"] for r in reqs], matches)
    for w, ms in zip(scoped, matches):
        assert w["references"] == (ms[:1] if ms and ms[0]["score"] >= 0.8 else [])
    assert scoped != plain


@gpu
@pytest.mark.parametrize("world", [1, 2, 3])
def test_sharded_store_app_match_equals_single(lib, loopback, golden, world):
    from kakveda_b200 import GfkbStore
    from kakveda_b200.dist import ShardedGfkbStore
    from test_gpu_shard_loopback import run_ranks

    recs, sigs, apps, types = _fixture_records(golden)
    st = GfkbStore()
    st._reset([json_copy(r) for r in recs])
    want = [st.match_batch(sigs, app_ids=[a] * len(sigs)) for a in apps]
    want_ff = st.match_batch(sigs, ["TYPE_B"] * len(sigs), filter_first=True, app_ids=["app-a"] * len(sigs))

    def fn(rank, group):
        sh = ShardedGfkbStore(device=0, rank=rank, world=world, group=group)
        try:
            sh._reset([json_copy(r) for r in recs])
            got = [sh.match_batch(sigs, app_ids=[a] * len(sigs)) for a in apps]
            ff = sh.match_batch(sigs, ["TYPE_B"] * len(sigs), filter_first=True, app_ids=["app-a"] * len(sigs))
            return got, ff
        finally:
            sh.close()

    for got, ff in run_ranks(world, fn):
        for a, b in zip(got, want):
            for x, y in zip(a, b):
                assert [m["failure_id"] for m in x] == [m["failure_id"] for m in y]
                np.testing.assert_allclose([m["score"] for m in x], [m["score"] for m in y], rtol=1e-12)
        for x, y in zip(ff, want_ff):
            assert [m["failure_id"] for m in x] == [m["failure_id"] for m in y]
