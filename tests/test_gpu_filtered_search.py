"""Label-filtered search: top-k and threshold search restricted to the rows of one label (a failure type), against
float64 oracles of the WHOLE index masked to the label, and bit for bit against the unfiltered path.

A filtered query's top-k is the stable top-k of the unfiltered float64 scores over the rows of its label (the index
statistics do not change), so the oracle is ``O.score_matrix_closed_form`` of the full corpus with the other rows set
to -inf, checked with the strict tie rules of test_gpu_topk_edges.py.  The pruning test asserts that filtered queries
only score chunks that hold their label: without it an implementation that never skips a chunk would pass the rest.
"""
import numpy as np
import pytest

from oracle import tfidf_oracle as O

gpu = pytest.mark.gpu

RTOL32 = 1e-5
N_ROWS = 60000          # 1875 chunks: the pruned path
SINGLE, NOBODY = 999, 1000   # a label carried by one row, a label carried by no row
KS = (1, 5, 16, 32)
QFEATS = 64


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
        assert np.isfinite(o[rr]).all(), "a row of another label (or excluded) was returned; " + where
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


def masked(oracle, row_labels, q_labels):
    """The oracle of a filtered batch: rows of other labels -inf for every query with a label >= 0."""
    o = np.array(oracle, dtype=np.float64, copy=True)
    for q, lb in enumerate(q_labels):
        if lb >= 0:
            o[q, row_labels != lb] = -np.inf
    return o


def label_sets(n, rng):
    """Three row labellings: one label, 8 Zipf-weighted labels, 200 labels (signatures collide); each with one row
    carrying SINGLE."""
    one = np.zeros(n, np.int32)
    w = 1.0 / np.arange(1, 9)
    zipf = rng.choice(8, size=n, p=w / w.sum()).astype(np.int32)
    many = rng.integers(0, 200, size=n).astype(np.int32)
    out = {}
    for name, lab in (("one", one), ("zipf8", zipf), ("many200", many)):
        lab = lab.copy()
        lab[n // 2 + 3] = SINGLE
        out[name] = lab
    return out


def query_labels(row_labels, n_q, rng):
    """A label per query: the labelling's own labels, -1 (unfiltered), SINGLE and NOBODY."""
    pool = np.concatenate([np.unique(row_labels[row_labels != SINGLE])[:16], [-1, SINGLE, NOBODY]])
    lab = rng.choice(pool, size=n_q).astype(np.int32)
    lab[:3] = [-1, SINGLE, NOBODY]
    return lab


class Case:
    def __init__(self, mode=0):
        from kakveda_b200 import GfkbIndex, synth

        rng = np.random.default_rng(7)
        corpus = synth.corpus(N_ROWS)
        self.wide_row = N_ROWS // 3 + 1
        corpus[self.wide_row] = " ".join(f"pw{i}" for i in range(70))
        qs = synth.queries(150, N_ROWS)   # half of them stored copies (score-1.0 ties across labels), half fresh
        wide = lambda m: " ".join(f"pw{i}" for i in reversed(range(m)))
        self.queries = qs + ["", "qqzzunseen xxyyq", wide(QFEATS), wide(QFEATS + 1)]  # null, null, regular, irregular
        self.corpus = corpus
        self.ix = GfkbIndex()
        if mode:
            self.ix.set_mode(mode)
        self.ix.add_texts(corpus)
        self.ix.finalize()
        self.oracle = O.corpus_fit_scores(self.queries, corpus) if mode == 2 else O.score_matrix_closed_form(self.queries, corpus)
        self.labels = label_sets(N_ROWS, rng)
        self.qlabels = {name: query_labels(lab, len(self.queries), rng) for name, lab in self.labels.items()}


@pytest.fixture(scope="module")
def lib(built_lib):
    from kakveda_b200 import _capi

    assert _capi.load().kv_device_count() > 0, "GPU tests need a CUDA device"
    return _capi.load()


@pytest.fixture(scope="module")
def case(lib):
    return Case()


@gpu
@pytest.mark.parametrize("dist", ["one", "zipf8", "many200"])
@pytest.mark.parametrize("env", [None, ("KAKVEDA_B200_BOUND_CODES", "0"), ("KAKVEDA_B200_NO_PRUNE", "1")])
def test_filtered_topk_equals_masked_oracle(case, monkeypatch, dist, env):
    if env:
        monkeypatch.setenv(*env)
    ix, rl, ql = case.ix, case.labels[dist], case.qlabels[dist]
    ix.set_row_labels(rl)
    want = masked(case.oracle, rl, ql)
    for k in KS:
        s, r = ix.topk(case.queries, k, labels=ql)
        lay = ix.layout()
        assert (lay["pairs_passed_bound"] > 0) == (env is None or env[0] != "KAKVEDA_B200_NO_PRUNE"), lay
        check_topk_strict(s, r, want, k, RTOL32)
        # the single-row label: that row, then (-inf, -1); the label no row carries: nothing
        assert r[1, 0] == N_ROWS // 2 + 3 and np.all(r[1, 1:] == -1)
        assert np.all(r[2] == -1) and np.all(s[2] == -np.inf)


@gpu
def test_filtered_topk_corpus_fit_mode(lib):
    c = Case(mode=2)
    rl, ql = c.labels["zipf8"], c.qlabels["zipf8"]
    c.ix.set_row_labels(rl)
    want = masked(c.oracle, rl, ql)
    for k in KS:
        s, r = c.ix.topk(c.queries, k, labels=ql)
        check_topk_strict(s, r, want, k, RTOL32)


@gpu
def test_unfiltered_bits_and_filtered_scores(case):
    ix = case.ix
    q = case.queries
    s0, r0 = ix.topk(q, 16)
    ix.set_row_labels(case.labels["zipf8"])
    # every query -1, or a label every row carries: the unfiltered bytes
    s1, r1 = ix.topk(q, 16, labels=np.full(len(q), -1, np.int32))
    assert r1.tobytes() == r0.tobytes() and s1.tobytes() == s0.tobytes()
    ix.set_row_labels(np.full(N_ROWS, 3, np.int32))
    s2, r2 = ix.topk(q, 16, labels=np.full(len(q), 3, np.int32))
    assert r2.tobytes() == r0.tobytes() and s2.tobytes() == s0.tobytes()
    # a filtered score is the unfiltered score of the same pair (the unfiltered threshold search at a low threshold)
    ix.set_row_labels(case.labels["many200"])
    sub = q[:40]
    ql = case.qlabels["many200"][:40]
    s3, r3 = ix.topk(sub, 32, labels=ql)
    ip, rows, sc = ix.range(sub, 1e-6)
    checked = 0
    for i in range(len(sub)):
        got = dict(zip(rows[ip[i]:ip[i + 1]].tolist(), sc[ip[i]:ip[i + 1]].tolist()))
        for rr, ss in zip(r3[i].tolist(), s3[i].tolist()):
            if rr >= 0 and ss > 0:
                assert np.float32(got[rr]).tobytes() == np.float32(ss).tobytes(), (i, rr)
                checked += 1
    assert checked > 100


def _csr_mask(ip, rows, sc, keep):
    """The CSR with only the pairs keep(q, row) holds."""
    out_ip, out_r, out_s = [0], [], []
    for q in range(len(ip) - 1):
        rr, ss = rows[ip[q]:ip[q + 1]], sc[ip[q]:ip[q + 1]]
        m = keep(q, rr)
        out_r.append(rr[m]); out_s.append(ss[m]); out_ip.append(out_ip[-1] + int(m.sum()))
    return np.array(out_ip, np.int64), np.concatenate(out_r), np.concatenate(out_s)


@gpu
def test_filtered_range_equals_unfiltered_minus_other_labels(case):
    ix = case.ix
    rl, ql = case.labels["zipf8"], case.qlabels["zipf8"]
    ix.set_row_labels(rl)
    q = case.queries
    keep = lambda i, rr: (ql[i] < 0) | (rl[rr] == ql[i])
    for thr in (0.3, 0.8):
        ip, rows, sc = ix.range(q, thr)
        want = _csr_mask(ip, rows, sc, keep)
        got = ix.range(q, thr, labels=ql)
        for a, b in zip(got, want):
            assert a.tobytes() == b.tobytes(), thr
        dev = ix.range(q, thr, device_out=True, labels=ql)
        for a, b in zip(dev, want):
            assert a.cpu().numpy().tobytes() == b.tobytes(), thr


@gpu
def test_selfjoin_same_label(case):
    ix = case.ix
    rl = case.labels["zipf8"]
    ix.set_row_labels(rl)
    lo, hi = 1000, 1300
    ip, rows, sc = ix.selfjoin_range(0.5, lo, hi)
    want = _csr_mask(ip, rows, sc, lambda i, rr: rl[rr] == rl[lo + i])
    got = ix.selfjoin_range(0.5, lo, hi, same_label=True)
    for a, b in zip(got, want):
        assert a.tobytes() == b.tobytes()
    assert not np.any(got[1] == np.repeat(np.arange(lo, hi), np.diff(got[0])))  # exclusions in effect
    # self-join top-k: the oracle of the rows as queries, the row itself and other labels masked out
    o = O.score_matrix_closed_form(case.corpus[lo:hi], case.corpus)
    o[np.arange(hi - lo), np.arange(lo, hi)] = -np.inf
    o = masked(o, rl, rl[lo:hi])
    for k in (1, 32):
        s, r = ix.selfjoin_topk(k, lo, hi, same_label=True)
        check_topk_strict(s, r, o, k, RTOL32)


@pytest.fixture(scope="module")
def rare_case(case):
    """A label on 60 rows (0.1 %): 6 texts stored 10 times each, so identical rows sit side by side in the scan order
    and the label occupies at most 12 chunks."""
    from kakveda_b200 import GfkbIndex

    rng = np.random.default_rng(11)
    corpus = list(case.corpus)
    src = [corpus[i] + f" rarelab{i}" for i in range(6)]
    rows = rng.choice(np.arange(100, N_ROWS), size=60, replace=False)
    for j, r in enumerate(rows):
        corpus[r] = src[j // 10]
    ix = GfkbIndex()
    ix.add_texts(corpus)
    ix.finalize()
    rl = np.zeros(N_ROWS, np.int32)
    rl[rows] = 1
    ix.set_row_labels(rl)
    return ix, src, rows


@gpu
@pytest.mark.parametrize("env", [None, ("KAKVEDA_B200_BOUND_CODES", "0"), ("KAKVEDA_B200_NO_PRUNE", "1")])
def test_rare_label_prunes_chunks(case, rare_case, monkeypatch, env):
    """Every scored (query, chunk) pair of a query filtered to the rare label -- seed scan and candidate scan, or the
    exhaustive scan -- must be one of the label's chunks."""
    if env:
        monkeypatch.setenv(*env)
    ix, src, rows = rare_case
    queries = src + case.queries[:100]
    n_scanned = len(queries)
    ix.topk(queries, 16)
    unfiltered = ix.layout()["pairs_scored"]
    s, r = ix.topk(queries, 16, labels=np.ones(n_scanned, np.int32))
    filtered = ix.layout()["pairs_scored"]
    label_chunks = 12
    assert 0 < filtered <= 2 * n_scanned * label_chunks < unfiltered, (filtered, unfiltered)
    assert np.all(np.isin(r[r >= 0], rows))
    for j in range(6):   # a stored text finds its 10 copies first
        assert sorted(r[j, :10].tolist()) == sorted(rows[j * 10:(j + 1) * 10].tolist())


@gpu
def test_state_and_validation(case, tmp_path):
    from kakveda_b200 import GfkbIndex, synth

    corpus = synth.corpus(20000)
    ix = GfkbIndex()
    ix.add_texts(corpus)
    rl = (np.arange(20000) % 5).astype(np.int32)
    ix.set_row_labels(rl)           # before finalize
    ix.finalize()
    assert ix.last_finalize_kind == 1
    q = corpus[:20] + ["fresh text entirely unseen words"]
    ql = np.full(len(q), 2, np.int32)
    s, r = ix.topk(q, 8, labels=ql)
    assert np.all(r[r >= 0] % 5 == 2)
    with pytest.raises(ValueError):
        ix.set_row_labels(rl[:-1])
    with pytest.raises(ValueError):
        ix.set_row_labels(np.where(rl == 0, -1, rl))
    ix.upload_queries(ix.vocab.featurize(q, grow=False))
    with pytest.raises(ValueError):
        ix.set_filter(ql[:-1])
    with pytest.raises(ValueError):
        ix.set_filter(np.full(len(q), -2, np.int32))
    # statistics-only finalize keeps the labels
    ix.set_global_df(ix.local_df(), 20000)
    ix.finalize()
    assert ix.last_finalize_kind == 2
    s2, r2 = ix.topk(q, 8, labels=ql)
    assert r2.tobytes() == r.tobytes() and s2.tobytes() == s.tobytes()
    # a persisted layout: labels set on the new index survive its statistics-only finalize
    path = tmp_path / "x.layout"
    ix.save_layout(path)
    b = GfkbIndex()
    b.add_texts(corpus)
    b.set_row_labels(rl)
    assert b.load_layout(path)
    b.finalize()
    assert b.last_finalize_kind == 2
    s3, r3 = b.topk(q, 8, labels=ql)
    assert r3.tobytes() == r.tobytes() and s3.tobytes() == s.tobytes()
    # an append drops the labels: a filtered query fails, it never uses stale labels
    ix.add_texts(["an appended row about citations"])
    ix.set_global_df(ix.local_df(), 20001)
    ix.finalize()
    with pytest.raises(RuntimeError):
        ix.topk(q, 8, labels=ql)
    with pytest.raises(RuntimeError):
        ix.selfjoin_topk(4, 0, 10, same_label=True)
    ix.topk(q, 8, labels=np.full(len(q), -1, np.int32))   # unfiltered still works
    rl2 = np.append(rl, 2).astype(np.int32)
    ix.set_row_labels(rl2)
    s4, r4 = ix.topk(q, 8, labels=ql)
    assert np.all(rl2[r4[r4 >= 0]] == 2)
    # Jaccard mode has no filter
    j = GfkbIndex()
    j.set_mode(1)
    j.add_texts([f"alpha{i} beta{i}" for i in range(500)])
    j.finalize()
    j.set_row_labels(np.zeros(500, np.int32))
    with pytest.raises(ValueError):
        j.topk(["alpha1 beta1", "alpha2", "beta3"], 4, labels=np.zeros(3, np.int32))


def _oracle_match(st, sig, ft, limit):
    scores = O.score_sklearn(sig, [r["signature_text"] for r in st.records])
    cand = sorted([(i, s) for i, s in enumerate(scores) if st.records[i]["failure_type"] == ft], key=lambda t: t[1], reverse=True)
    return cand[:limit]


@gpu
def test_store_filter_first_fixture54(lib, golden):
    from kakveda_b200 import GfkbStore

    g = golden("fixture54.json")
    recs = [dict(r) for r in g["records"]]
    types = ["TYPE_A", "TYPE_B", "TYPE_C"]
    for i, r in enumerate(recs):
        r["failure_type"] = types[(i * 7) % 3]
    st = GfkbStore()
    st._reset(recs)
    sigs = [c["signature_text"] for c in g["match"]] + [r["signature_text"] for r in recs[:10]]
    before = st.match_batch(sigs, ["TYPE_B"] * len(sigs))
    for ft in types:
        got = st.match_batch(sigs, [ft] * len(sigs), filter_first=True)
        for sig, ms in zip(sigs, got):
            want = _oracle_match(st, sig, ft, 5)
            assert [m["failure_id"] for m in ms] == [st.records[i]["failure_id"] for i, _ in want]
            np.testing.assert_allclose([m["score"] for m in ms], [s for _, s in want], rtol=1e-9)
    assert st.match_batch(sigs, ["TYPE_B"] * len(sigs), filter_first=False) == before
    assert st.match(sigs[0], "NO_SUCH_TYPE", filter_first=True) == []
    assert st.match(sigs[0], None, filter_first=True) == st.match(sigs[0])


@gpu
def test_store_filter_first_main_and_tail(lib):
    from kakveda_b200 import GfkbStore, synth

    st = GfkbStore(tail_limit=5000)
    corpus = synth.corpus(3000)
    recs = [{"failure_id": f"F-{i + 1:04d}", "version": 1, "failure_type": ["X", "Y", "Z"][i % 3], "signature_text": t,
             "affected_apps": ["a"], "occurrences": 1, "root_cause": None, "resolution": None, "context_signature": {}}
            for i, t in enumerate(corpus)]
    st._reset(recs)
    for i in range(40):   # the tail: copies of main rows under other types, and a new type
        st.upsert({"failure_type": ["Y", "W"][i % 2], "signature_text": corpus[i * 3], "context_signature": {},
                   "impact_severity": "low", "app_id": "b"})
    qs = corpus[:60:3] + synth.queries(10, 3000)
    for ft in ("X", "Y", "W"):
        got = st.match_batch(qs, [ft] * len(qs), filter_first=True)
        assert st._tail is not None and st._tail.n_rows == 40
        for sig, ms in zip(qs, got):
            want = _oracle_match(st, sig, ft, 5)
            assert [m["failure_id"] + str(m["version"]) for m in ms] == \
                   [st.records[i]["failure_id"] + str(st.records[i]["version"]) for i, _ in want], (ft, sig)
            np.testing.assert_allclose([m["score"] for m in ms], [s for _, s in want], rtol=1e-9)


def test_store_filter_first_ambiguous_candidates(built_lib, monkeypatch):
    """Colliding float32 groups of the filtered type force the exact path, which must be filter-aware: group B (rows
    20..39, type T) beats group A (rows 0..19, type T) in float64 only; rows 40..59 (type U) score higher than both."""
    from kakveda_b200 import GfkbStore

    n = 60
    f64 = np.full(n, 0.25)
    f64[0:20] = 0.8
    f64[20:40] = 0.8 + 1e-9
    f64[40:60] = 0.9
    types = ["T"] * 40 + ["U"] * 20
    allowed = np.array([t == "T" for t in types])

    class FakeIndex:
        n_rows = n

        def topk_features(self, fb, k, labels=None):
            s32 = np.where(allowed, f64, -np.inf).astype(np.float32) if labels is not None else f64.astype(np.float32)
            order = np.lexsort((np.arange(n), -s32))[:k]
            return np.tile(s32[order], (fb.n, 1)), np.tile(order.astype(np.int64), (fb.n, 1))

        def rescore(self, fb, rows):
            return f64[rows]

        def score(self, text):
            return f64.copy()

        def close(self):
            pass

    st = GfkbStore()
    st.records = [{"failure_id": f"F-{i:04d}", "version": 1, "failure_type": types[i], "suggested_mitigation": None,
                   "signature_text": "x"} for i in range(n)]
    monkeypatch.setattr(st, "_sync", lambda: None)

    class _B:
        n = 1

        def close(self):
            pass
    monkeypatch.setattr(st.vocab, "featurize", lambda texts, grow=False, n_threads=0: _B())
    st._main = FakeIndex()
    got = st.match("q", "T", filter_first=True)
    assert [m["failure_id"] for m in got] == [f"F-{i:04d}" for i in range(20, 25)]
    assert st.stats["exact_fallbacks"] == 1
    assert st.match("q", "T") == []   # the reference's order: five U rows first, then the filter
    st._main = None


@gpu
def test_detect_patterns_filter_first(lib):
    from kakveda_b200 import GfkbIndex, synth
    from kakveda_b200.patterns import detect_patterns

    base = synth.corpus(400)
    text = base[7]
    recs = []
    for i, t in enumerate(base):
        recs.append({"failure_id": f"F-{i:04d}", "failure_type": "OTHER", "signature_text": t, "affected_apps": ["z"]})
    for i in range(40):   # one text stored 40 times under another type
        recs.append({"failure_id": f"B-{i:04d}", "failure_type": "OTHER", "signature_text": text, "affected_apps": ["z"]})
    near = [text + " alpha", text + " beta", text + " gamma"]
    for i, t in enumerate(near):   # its near-duplicates of type X, from three apps
        recs.append({"failure_id": f"X-{i:04d}", "failure_type": "X", "signature_text": t, "affected_apps": [f"app{i}"]})
    ix = GfkbIndex()
    ix.set_mode(2)
    ix.add_texts([r["signature_text"] for r in recs])
    ix.finalize()
    x_rows = list(range(len(recs) - 3, len(recs)))
    default = detect_patterns(ix, recs, threshold=0.5, k=32, failure_type="X")
    assert not any(set(p["rows"]) == set(x_rows) for p in default)   # the 41 copies fill the lists
    got = detect_patterns(ix, recs, threshold=0.5, k=32, failure_type="X", filter_first=True)
    assert [p["rows"] for p in got] == [x_rows]
    full = detect_patterns(ix, recs, threshold=0.5, k=None, failure_type="X")
    assert [p["rows"] for p in full] == [x_rows]
    assert detect_patterns(ix, recs, threshold=0.5, k=None, failure_type="X", filter_first=True) == full
    from kakveda_b200 import DenseIndex
    with pytest.raises(NotImplementedError):
        detect_patterns(object.__new__(DenseIndex), recs, failure_type="X", filter_first=True)
