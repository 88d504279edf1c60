"""Exact threshold search (kv_range_resident_exact, kv_range_fetch_exact(_device), GfkbIndex.range_exact) and
GfkbStore.match_above.

The float64 decision is checked against K6 itself: ``GfkbIndex.rescore`` over every row gives the full K6 vector, and
a search at threshold t must return exactly the rows whose K6 score is >= t, with those bits, ordered by (score desc,
row asc).  Against sklearn (the reference's arithmetic) scores agree within 1e-12 relative, and membership outside a
1e-12 band around t."""
import ctypes as C

import numpy as np
import pytest

from oracle import tfidf_oracle as O

pytestmark = pytest.mark.gpu

THRESHOLDS = (0.3, 0.5, 0.8, 0.95, 1.0)
RTOL = 1e-12


@pytest.fixture(scope="module")
def lib(built_lib):
    from kakveda_b200 import _capi

    assert _capi.load().kv_device_count() > 0, "GPU tests need a CUDA device"
    return _capi.load()


def full_k6(ix, fb):
    """[Q, N] K6 scores of every (query, local row) pair; -inf for a deleted row."""
    rows = np.broadcast_to(np.arange(ix.row_base, ix.row_base + ix.n_rows, dtype=np.int64), (fb.n, ix.n_rows))
    return ix.rescore(fb, rows)


def check_exact(out, K, thr, elig=None, row_base=0):
    """out: an exact range result; K: the full K6 matrix; elig[q, r]: the filters let query q return row r."""
    ip, rows, sc = out
    Q, N = K.shape
    assert ip.shape == (Q + 1,) and ip[0] == 0 and ip[-1] == len(rows) == len(sc)
    assert rows.dtype == np.int64 and sc.dtype == np.float64
    for q in range(Q):
        k = K[q] if elig is None else np.where(elig[q], K[q], -np.inf)
        want = np.flatnonzero(k >= thr)
        want = want[np.lexsort((want, -k[want]))]
        np.testing.assert_array_equal(rows[ip[q]:ip[q + 1]] - row_base, want, err_msg=f"query {q} at {thr}")
        assert sc[ip[q]:ip[q + 1]].tobytes() == k[want].tobytes(), (q, thr)


class Corpus:
    """20k synthetic rows (the pruned path), two identical rows, an irregular row; queries with a null, an all-unseen,
    an irregular (> 64 features) and a large-tf one; 5 % of the rows deleted; a label and up to two tags (some >= 64)
    per row, and per query a label filter on odd queries and a tag filter on every third."""

    def __init__(self, mode):
        from kakveda_b200 import GfkbIndex, synth

        rng = np.random.default_rng(5 + mode)
        n = 20000
        corpus = synth.corpus(n)
        corpus[17] = "tok " * 35 + "and and and include include citations"
        corpus[18] = corpus[17]
        long_query = " ".join(f"w{i}x" for i in range(300)) + " " + corpus[5]
        corpus[11] = long_query
        self.queries = synth.queries(200, n) + [corpus[17], corpus[40], "", "zz qq unseen", long_query,
                                                "tok " * 400 + "citations include"]
        self.ix = ix = GfkbIndex()
        if mode:
            ix.set_mode(mode)
        ix.add_texts(corpus)
        ix.finalize()
        assert ix.layout()["chunks"] >= 512
        dead = rng.choice(n, size=n // 20, replace=False)
        dead = dead[(dead != 17) & (dead != 18) & (dead != 11)]
        ix.delete_rows(dead)
        ix.finalize()
        self.labels = rng.integers(0, 4, n).astype(np.int32)
        self.tags = [sorted(set(rng.integers(0, 70, rng.integers(0, 3)).tolist())) for _ in range(n)]
        ix.set_row_labels(self.labels)
        ix.set_row_tags(self.tags)
        Q = len(self.queries)
        self.qlab = np.where(np.arange(Q) % 2 == 1, rng.integers(0, 4, Q), -1).astype(np.int32)
        self.qtags = [[int(rng.integers(0, 70)), 66] if q % 3 == 0 else [] for q in range(Q)]
        self.fb = ix.vocab.featurize(self.queries, grow=False)
        self.K = full_k6(ix, self.fb)
        assert np.isneginf(self.K[:, dead]).all()
        lab_ok = (self.qlab[:, None] < 0) | (self.labels[None, :] == self.qlab[:, None])
        tag_ok = np.array([[not qt or bool(set(qt) & set(rt)) for rt in self.tags] for qt in self.qtags])
        self.elig = lab_ok & tag_ok


@pytest.fixture(scope="module", params=[0, 2], ids=["tfidf", "corpus_fit"])
def corpus(lib, request):
    return Corpus(request.param)


@pytest.mark.parametrize("thr", THRESHOLDS)
def test_exact_range_is_the_k6_decision(corpus, thr):
    """Membership is exactly K6 >= thr, scores are K6's bits, with deletions, labels and tags."""
    ix, fb, K = corpus.ix, corpus.fb, corpus.K
    out = ix.range_exact(fb, thr)
    check_exact(out, K, thr)
    assert ix.last_range_candidates >= len(out[1])
    Q = len(corpus.queries)
    assert out[0][Q - 4 + 1] == out[0][Q - 4] and out[0][Q - 3 + 1] == out[0][Q - 3]  # null and all-unseen queries
    if thr < 1.0:
        seg = out[1][out[0][Q - 6]:out[0][Q - 5]]  # the query equal to rows 17 and 18: both, tied exactly
        assert 17 in seg and 18 in seg
    check_exact(ix.range_exact(fb, thr, labels=corpus.qlab, tags=corpus.qtags), K, thr, corpus.elig)


def test_exact_range_boundary(corpus):
    """For pairs with score s (float32(s) != s among them): threshold s returns the pair, nextafter(s, 2) does not."""
    ix, K = corpus.ix, corpus.K
    picked = []
    for q in range(0, 200, 7):
        r = np.flatnonzero((K[q] > 0.05) & (K[q] < 1.0))
        if len(r):
            picked.append((q, int(r[np.argmax(K[q, r])])))
        if len(r) > 1:
            picked.append((q, int(r[len(r) // 2])))
    assert sum(np.float32(K[q, r]) != K[q, r] for q, r in picked) >= 10
    for q, r in picked:
        s = float(K[q, r])
        fb = ix.vocab.featurize([corpus.queries[q]], grow=False)
        try:
            ip, rows, sc = ix.range_exact(fb, s)
            assert r in rows and sc[rows == r][0] == s
            ip, rows, sc = ix.range_exact(fb, float(np.nextafter(s, 2.0)))
            assert r not in rows and np.all(sc > s)
        finally:
            fb.close()


def _golden_cases(golden):
    from kakveda_b200 import synth

    g = golden("ref_test_similarity.json")
    yield g["corpus"], [g["query"]], np.array([g["scores"]])
    g = golden("edge_cases.json")
    yield g["corpus"], g["queries"], np.array(g["scores"])
    g = golden("synthetic_small.json")
    yield synth.corpus(g["n"]), synth.queries(g["q"], g["n"]), np.array(g["scores"])


@pytest.mark.parametrize("thr", THRESHOLDS)
def test_exact_range_sklearn_goldens(lib, golden, thr):
    """On the reference's sklearn goldens: the K6 decision, scores within 1e-12 of sklearn, and sklearn's membership
    outside a 1e-12 band around the threshold."""
    from kakveda_b200 import GfkbIndex

    for corpus, queries, S in _golden_cases(golden):
        ix = GfkbIndex()
        ix.add_texts(corpus)
        ix.finalize()
        fb = ix.vocab.featurize(queries, grow=False)
        try:
            ip, rows, sc = ix.range_exact(fb, thr)
            check_exact((ip, rows, sc), full_k6(ix, fb), thr)
        finally:
            fb.close()
            ix.close()
        for q in range(len(queries)):
            r, s = rows[ip[q]:ip[q + 1]], sc[ip[q]:ip[q + 1]]
            np.testing.assert_allclose(s, S[q, r], rtol=RTOL, atol=0)
            assert np.all(S[q, r] >= thr * (1 - RTOL))
            assert np.isin(np.flatnonzero(S[q] >= thr * (1 + RTOL)), r).all()


def _exact_resident(lib, ix, fb, thr, n_q=None):
    from kakveda_b200.similarity import _ptr

    n, cand = C.c_int64(0), C.c_int64(0)
    rc = lib.kv_range_resident_exact(ix._h, _ptr(fb.indptr, C.c_int64), _ptr(fb.ids, C.c_uint32), _ptr(fb.tf, C.c_uint32),
                                     _ptr(fb.oov, C.c_double), fb.n if n_q is None else n_q, thr, C.byref(n), C.byref(cand))
    return rc, n.value


def _fetch_exact(lib, ix, n_q, n):
    from kakveda_b200.similarity import _ptr

    out = (np.empty(n_q + 1, np.int64), np.empty(n, np.int64), np.empty(n, np.float64))
    rc = lib.kv_range_fetch_exact(ix._h, _ptr(out[0], C.c_int64), _ptr(out[1], C.c_int64), _ptr(out[2], C.c_double))
    return rc, out


def test_exact_range_host_device_and_refusals(lib, corpus):
    from kakveda_b200 import JaccardIndex, _capi

    ix, fb = corpus.ix, corpus.fb
    for thr in (0.3, 0.8):  # 0.3: enough pairs that the host fetch orders on the device too
        host = ix.range_exact(fb, thr, labels=corpus.qlab)
        dev = ix.range_exact(fb, thr, labels=corpus.qlab, device_out=True)
        assert [d.dtype for d in (t.cpu().numpy() for t in dev)] == [np.int64, np.int64, np.float64]
        for a, b in zip(host, dev):
            assert a.tobytes() == b.cpu().numpy().tobytes()
    for bad in (float("nan"), 0.0, -0.5, 1.5):
        with pytest.raises(ValueError, match="threshold"):
            ix.range_exact(fb, bad)

    # the resident batch, its top-k thresholds and its exclusions are left as they were
    Q = fb.n
    ix.upload_queries(fb)
    ix.set_exclusions(np.arange(Q, dtype=np.int64))
    s0, r0 = ix.topk_resident_host(Q, 16)
    f32 = ix._range_resident(Q, 0.5)
    rc, n = _exact_resident(lib, ix, fb, 0.5)
    assert rc == _capi.KV_OK
    # a float32 fetch of an exact result, and the result stays
    with pytest.raises(RuntimeError, match="exact"):
        ix._range_fetch_into(ix._range_arrays(Q, n, False), device_out=False)
    with pytest.raises(RuntimeError, match="exact"):
        ix._range_fetch_into(ix._range_arrays(Q, n, True), device_out=True)
    rc, ex = _fetch_exact(lib, ix, Q, n)
    assert rc == _capi.KV_OK
    elig = np.ones_like(corpus.elig)
    elig[np.arange(Q), np.arange(Q)] = False  # the exclusions hold
    check_exact(ex, corpus.K, 0.5, elig)
    assert _fetch_exact(lib, ix, Q, n)[0] == _capi.KV_ERR_STATE  # consumed
    s1, r1 = ix.topk_resident_host(Q, 16)
    assert s1.tobytes() == s0.tobytes() and r1.tobytes() == r0.tobytes()
    # an exact fetch of a float32 result, and the result stays
    n32 = ix._range_search(0.5)
    assert _fetch_exact(lib, ix, Q, n32)[0] == _capi.KV_ERR_STATE
    again = ix._range_arrays(Q, n32, False)
    ix._range_fetch_into(again, device_out=False)
    for a, b in zip(f32, again):
        assert a.tobytes() == b.tobytes()

    assert _exact_resident(lib, ix, fb, 0.5, n_q=Q - 1)[0] == _capi.KV_ERR_INVALID  # not the batch's count
    ix._selfjoin_upload(0, 10)
    sub = ix.vocab.featurize(corpus.queries[:10], grow=False)
    try:
        assert _exact_resident(lib, ix, sub, 0.5)[0] == _capi.KV_ERR_INVALID  # a self-join batch
    finally:
        sub.close()

    jx = JaccardIndex(vocab_size=100)
    jx.add_csr(np.array([0, 2, 4], np.int64), np.array([1, 2, 2, 3], np.uint32))
    jx.finalize()
    assert _exact_resident(lib, jx, fb, 0.5)[0] == _capi.KV_ERR_INVALID
    jx.close()


# ---------------------------------------------------------------------------------------------------------------------
# GfkbStore.match_above
# ---------------------------------------------------------------------------------------------------------------------

def _oracle_above(st, sig, thr, ft=None, app=None, distinct=False):
    """The reference's stable sort over sklearn scores with the threshold and no cut, as entries (failure_id, version,
    score, near): ``near`` marks a score within 1e-12 of the threshold, which either decision may take.  ``distinct``:
    the best record of each key, reported as the key's newest record."""
    scores = O.score_sklearn(sig, [r["signature_text"] for r in st.records])
    out, seen = [], set()
    for i in sorted(range(len(scores)), key=lambda i: scores[i], reverse=True):
        r, s = st.records[i], scores[i]
        if s < thr * (1 - RTOL) or (ft and r["failure_type"] != ft) or (app and app not in (r.get("affected_apps") or [])):
            continue
        if distinct:
            key = (r["failure_type"], r["signature_text"])
            if key in seen:
                continue
            seen.add(key)
            r = st.records[st._latest[key]]
        out.append((r["failure_id"], r["version"], s, abs(s - thr) <= RTOL * thr))
    return out


def _check_above(got, want):
    """got: match_above's dicts; want: _oracle_above's entries."""
    sure = [(w[0], w[1]) for w in want if not w[3]]
    got_keys = [(m["failure_id"], m["version"]) for m in got]
    assert [k for k in got_keys if k in set(sure)] == sure
    allowed = {(w[0], w[1]): w[2] for w in want}
    assert all(k in allowed for k in got_keys), got_keys
    np.testing.assert_allclose([m["score"] for m in got], [allowed[k] for k in got_keys], rtol=RTOL)


@pytest.mark.parametrize("tail_limit", [40, 0])
def test_match_above_replays_reference_stream(lib, golden, tmp_path, tail_limit):
    from kakveda_b200 import GfkbStore

    g = golden("service_upsert.json")
    st = GfkbStore(path=tmp_path / f"above{tail_limit}.jsonl", tail_limit=tail_limit)
    n_checked = 0
    for step in g["steps"]:
        st.upsert(step["upsert"])
        app = step["upsert"].get("app_id")
        for m in step.get("matches", []):
            sig, ft = m["signature_text"], m["failure_type"]
            for thr in (0.2, 0.5, 0.8):
                got = st.match_above(sig, thr, ft)
                _check_above(got, _oracle_above(st, sig, thr, ft))
                _check_above(st.match_above(sig, thr, app_id=app), _oracle_above(st, sig, thr, app=app))
                _check_above(st.match_above(sig, thr, ft, distinct=True), _oracle_above(st, sig, thr, ft, distinct=True))
                # the first min(5, n) rows are match's rows at or above the threshold
                above = st.match_above(sig, thr)
                top = [x for x in st.match(sig) if x["score"] >= thr]
                head = above[:min(5, len(above))]
                assert [(x["failure_id"], x["version"]) for x in head] == [(x["failure_id"], x["version"]) for x in top]
                np.testing.assert_allclose([x["score"] for x in head], [x["score"] for x in top], rtol=RTOL)
                n_checked += 1
    assert n_checked > 0
    # a batch equals its single queries; unknown types and apps match nothing
    sigs = [r["signature_text"] for r in st.records[:6]] + ["unrelated text entirely"]
    batch = st.match_above_batch(sigs, 0.5)
    assert batch == [st.match_above(s, 0.5) for s in sigs]
    assert all(b for b in batch[:6])
    assert st.match_above(sigs[0], 0.5, "NO_SUCH_TYPE") == [] and st.match_above(sigs[0], 0.5, app_id="no-such-app") == []
    # after a purge: the purged app's records are gone, emptied records never match
    apps = sorted({a for r in st.records for a in (r.get("affected_apps") or [])})
    st.purge_apps(apps[:1])
    for sig in sigs:
        for thr in (0.2, 0.5, 0.8):
            _check_above(st.match_above(sig, thr), _oracle_above(st, sig, thr))
            _check_above(st.match_above(sig, thr, app_id=apps[-1]), _oracle_above(st, sig, thr, app=apps[-1]))
    with pytest.raises(ValueError, match="threshold"):
        st.match_above(sigs[0], 0.0)
    st.close()


def test_sharded_store_refuses_match_above(lib, golden):
    from kakveda_b200.dist import ShardedGfkbStore

    g = golden("service_upsert.json")
    st = ShardedGfkbStore(device=0)
    for step in g["steps"][:5]:
        st.upsert(step["upsert"])
    with pytest.raises(NotImplementedError, match="match_above"):
        st.match_above(g["steps"][0]["upsert"]["signature_text"], 0.5)
    st.close()
