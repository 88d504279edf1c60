"""CPU-side checks of the widened surface: the oracle's corpus-fit / all-pairs helpers against their sklearn goldens,
the union-find clustering (host C++ behind the C ABI) against the oracle, and the GFKB store's upsert bookkeeping
(services/gfkb/app.py:104-147) against the record stream the reference produced -- no device calls."""
import json

import numpy as np
import pytest

from oracle import tfidf_oracle as O


def test_oracle_corpus_fit_matches_golden(golden):
    from kakveda_b200 import synth

    g = golden("corpus_fit.json")
    corpus = synth.corpus(g["n"])
    S = O.corpus_fit_scores(corpus, corpus)
    np.testing.assert_allclose(S.sum(axis=1), g["row_sums"], rtol=1e-12)
    rows, vals = O.allpairs_topk(S, g["k"])
    np.testing.assert_array_equal(rows, np.array(g["allpairs_rows"]))
    np.testing.assert_allclose(vals, np.array(g["allpairs_scores"]), rtol=1e-12)
    assert np.allclose(S, S.T, rtol=0, atol=1e-15)  # the corpus-fit measure is symmetric


def test_cluster_topk_matches_oracle(built_lib):
    from kakveda_b200 import patterns

    rng = np.random.default_rng(5)
    n, k = 500, 6
    rows = rng.integers(-1, n, size=(n, k)).astype(np.int64)
    scores = rng.random((n, k)).astype(np.float32)
    scores[rng.random((n, k)) < 0.02] = np.nan  # NaN never links
    for thr in (0.0, 0.5, 0.9, 0.97, 2.0):
        labels, count = patterns.cluster_topk(rows, scores, thr)
        want = O.components(n, rows, np.nan_to_num(scores, nan=-1.0), thr)
        np.testing.assert_array_equal(labels, want)
        assert count == len(set(want))
        assert np.all(labels <= np.arange(n))  # label = smallest member
    with pytest.raises(ValueError):
        patterns.cluster_topk(np.array([[7]], dtype=np.int64), np.ones((1, 1), np.float32), 0.5)


def test_pattern_payload_matches_reference_shape():
    from kakveda_b200 import patterns

    recs = [{"failure_id": "F-0002", "affected_apps": ["b", "a"]}, {"failure_id": "F-0001", "affected_apps": ["a", "c"]},
            {"failure_id": None, "affected_apps": []}]
    p = patterns.pattern_payload("n", recs, "d")
    assert p == {"name": "n", "failure_ids": ["F-0001", "F-0002"], "affected_apps": ["a", "b", "c"], "description": "d"}


def test_store_upsert_bookkeeping_matches_reference(golden, built_lib, tmp_path):
    """Replays the reference's request stream; every returned record and the final JSONL must be identical
    (timestamps aside).  No query is issued, so no device is needed."""
    from kakveda_b200 import GfkbStore

    g = golden("service_upsert.json")
    path = tmp_path / "failures.jsonl"
    st = GfkbStore(path=path)
    for step in g["steps"]:
        out = st.upsert(step["upsert"])
        assert out["created"] == step["created"]
        got = {k: v for k, v in out["failure"].items() if k not in ("created_at", "updated_at")}
        assert got == step["failure"]
        assert out["failure"]["created_at"].endswith("Z") or "+" in out["failure"]["created_at"]
    lines = [json.loads(l) for l in path.read_text().splitlines()]
    assert [{k: v for k, v in r.items() if k not in ("created_at", "updated_at")} for r in lines] == g["final_records"]
    assert len(lines) == len(g["final_records"]) == len(st.records)
    # queries need the device: without one the store raises instead of falling back to a CPU path
    from kakveda_b200 import _capi
    if _capi.load().kv_device_count() == 0:
        with pytest.raises(RuntimeError, match="no CUDA device"):
            st.match("alpha beta gamma")


def test_vocabulary_export_import_round_trip(built_lib):
    """Sidecar support: a vocabulary rebuilt from its exported keys hands out the same ids, and keeps growing."""
    from kakveda_b200 import synth
    from kakveda_b200.similarity import Vocabulary

    corpus = synth.corpus(3000) + ["Ünïcödé naïve café", "tok " * 40 + "end"]
    a = Vocabulary()
    fa = a.featurize(corpus, grow=True)
    keys = a.export_keys()
    assert keys.shape == (len(a), 2) and len({(int(x), int(y)) for x, y in keys}) == len(a)
    b = Vocabulary.from_keys(keys)
    assert len(b) == len(a)
    fb = b.featurize(corpus, grow=False)
    np.testing.assert_array_equal(fa.indptr, fb.indptr)
    np.testing.assert_array_equal(fa.ids, fb.ids)
    np.testing.assert_array_equal(fa.tf, fb.tf)
    assert not fb.oov.any()
    # new text: both vocabularies assign the same NEW ids (numbering continues after the imported features)
    more = synth.queries(200, 3000) + ["completely new words zzzqqq yyyxxx"]
    ga, gb = a.featurize(more, grow=True), b.featurize(more, grow=True)
    np.testing.assert_array_equal(ga.ids, gb.ids)
    assert len(a) == len(b) > len(keys)
    # error conventions
    with pytest.raises(RuntimeError):
        b_keys = b.export_keys()
        from kakveda_b200 import _capi
        import ctypes as C
        _capi.check(_capi.load().kv_vocab_import(b._h, b_keys.ctypes.data_as(C.POINTER(C.c_uint64)), len(b_keys)))  # not empty
    with pytest.raises(ValueError):
        Vocabulary.from_keys(np.array([[1, 2], [1, 2]], dtype=np.uint64))                                     # duplicate key


def test_sidecar_save_load_and_staleness(built_lib, tmp_path):
    from kakveda_b200 import sidecar, synth
    from kakveda_b200.similarity import Vocabulary

    texts = synth.corpus(500)
    v = Vocabulary()
    fb = v.featurize(texts, grow=True)
    p = tmp_path / "failures.kvb.npz"
    sidecar.save(p, v, fb, texts)
    got = sidecar.load(p, texts)
    assert got is not None
    v2, batch, n0 = got
    assert n0 == 500 and len(v2) == len(v)
    np.testing.assert_array_equal(batch.indptr, fb.indptr)
    np.testing.assert_array_equal(batch.ids, fb.ids)
    np.testing.assert_array_equal(batch.tf, fb.tf)
    # an appended JSONL is a valid extension (GFKB is append-only): the sidecar covers its first 500 rows
    more = texts + synth.queries(20, 500)
    got = sidecar.load(p, more)
    assert got is not None and got[2] == 500
    rest = got[0].featurize(more[500:], grow=True)
    want = v.featurize(more[500:], grow=True)
    np.testing.assert_array_equal(rest.ids, want.ids)
    # anything else is stale: an edited row, a shorter file, a missing or corrupt sidecar
    edited = list(texts)
    edited[17] += " changed"
    assert sidecar.load(p, edited) is None
    assert sidecar.load(p, texts[:499]) is None
    assert sidecar.load(tmp_path / "absent.npz", texts) is None
    (tmp_path / "bad.npz").write_bytes(b"not an npz")
    assert sidecar.load(tmp_path / "bad.npz", texts) is None


def test_store_match_and_warn_host_logic_on_canned_candidate_stage(golden, built_lib, monkeypatch):
    """The host half of GfkbStore.match_batch / warn_batch (services/gfkb/app.py:88-100,
    services/warning_policy/app.py:30-72) on CPU: the device stage is replaced by candidates taken from the
    reference's recorded float64 scores, so the truncate-to-5-THEN-filter rule, the FailureMatch mapping and the
    warning texts are checked against the reference's recorded /failures/match responses without a GPU."""
    from kakveda_b200 import GfkbStore

    g = golden("fixture54.json")
    st = GfkbStore()
    st.records = [dict(r) for r in g["records"]]
    monkeypatch.setattr(st, "_sync", lambda: None)
    by_query = {q: np.array(s) for q, s in zip(g["queries"], g["scores"])}
    current = {}

    def fake_featurize(texts, grow=False, n_threads=0):
        current["texts"] = list(texts)

        class _B:
            n = len(texts)

            def close(self):
                pass
        return _B()

    def fake_candidates(fb, k, limit=5, labels=None, distinct=False, tags=None):
        rows, f64 = [], []
        for t in current["texts"]:
            s = by_query[t]
            order = sorted(range(len(s)), key=lambda i: s[i], reverse=True)[:k]   # stable: ties -> lower row
            rows.append(order)
            f64.append([s[i] for i in order])
        return np.array(rows, dtype=np.int64), np.array(f64), np.zeros(len(rows), dtype=bool)

    monkeypatch.setattr(st.vocab, "featurize", fake_featurize)
    monkeypatch.setattr(st, "_candidates", fake_candidates)
    cases = [c for c in g["match"] if c["signature_text"] in by_query]
    got = st.match_batch([c["signature_text"] for c in cases], [c["failure_type"] for c in cases])
    assert len(cases) >= 12
    for c, ms in zip(cases, got):
        assert ms == c["matches"]            # ids, versions, float64 scores, failure_type, suggested_mitigation
    # the filter runs AFTER the truncation: a foreign failure_type empties the list instead of digging deeper
    assert any(c["failure_type"] == "OTHER_TYPE" and c["matches"] == [] for c in cases)
    # warnings: threshold compare, reference message text, silent default
    monkeypatch.setattr("kakveda_b200.store._signature_text", lambda prompt, tools, env: prompt)
    q = cases[0]["signature_text"]
    w = st.warn_batch([{"app_id": "a", "prompt": q}], threshold=0.0, default_action="warn")[0]
    best = w["references"][0]
    assert w["confidence"] == best["score"] and w["message"].startswith("This execution matches past failure type ")
    assert f"similarity={best['score']:.2f}" in w["message"] and w["message"].endswith(str(best["suggested_mitigation"] or "n/a"))
    w = st.warn_batch([{"app_id": "a", "prompt": q}], threshold=2.0, default_action="silent")[0]
    assert w == {"action": "silent", "confidence": best["score"], "pattern_id": None, "references": [],
                 "message": "No high-similarity match found in GFKB."}


def test_stable_top_equals_python_stable_sort(monkeypatch):
    """store.stable_top == sorted(range(n), key=..., reverse=True)[:limit] (services/gfkb/app.py:88-89), on both of its
    branches, with heavy ties."""
    from kakveda_b200 import store

    rng = np.random.default_rng(5)
    for n, levels in ((1, 1), (7, 2), (300, 3), (5000, 40), (5000, 5000)):
        scores = rng.integers(0, levels, size=n).astype(np.float64) / max(levels, 1)
        vals = scores.tolist()
        for limit in (1, 5, 16, 32, n, n + 3):
            want = sorted(range(n), key=lambda i: vals[i], reverse=True)[:limit]
            assert store.stable_top(scores, limit) == want
            monkeypatch.setattr(store, "EXACT_SORT_MAX", 0)          # force the O(n) selection branch
            if limit <= n:
                assert store.stable_top(scores, limit) == want, (n, levels, limit)
            monkeypatch.undo()


def test_ambiguous_candidates_rule():
    from kakveda_b200.store import ambiguous_candidates

    k = 16
    rows = np.tile(np.arange(k, dtype=np.int64), (6, 1))
    s = np.tile(np.linspace(0.9, 0.1, k, dtype=np.float32), (6, 1))
    s[1, :] = 0.5                      # 16 equal scores: rows beyond the list may tie into the top 5
    s[2, 5:] = s[2, 4] * (1 - 1e-6)    # last score within float32 rounding of the 5th
    s[3, :] = 0.0                      # exact zeros are exact in float64 too
    rows[4, 10:] = -1; s[4, 10:] = -np.inf   # list not full: every row of the segment is a candidate
    s[5, 5:] = s[5, 4] * (1 - 1e-4)    # clearly below the 5th
    assert ambiguous_candidates(s, rows, 5).tolist() == [False, True, True, False, False, False]


def test_store_match_takes_exact_path_when_float32_scores_of_distinct_texts_collide(built_lib, monkeypatch):
    """ADVICE round 1: two distinct texts, each stored more than 16 times, whose float64 scores collide in float32.
    The float32 candidate list then holds only the group with the lower row ids; the reference's stable float64 top-5
    (services/gfkb/app.py:88-89) is the OTHER group.  The store must notice and take the exact path."""
    from kakveda_b200 import GfkbStore

    n = 60
    f64 = np.full(n, 0.25)
    f64[0:20] = 0.8                    # group A, rows 0..19
    f64[20:40] = 0.8 + 1e-9            # group B, rows 20..39: higher in float64, equal in float32
    assert np.float32(f64[0]) == np.float32(f64[20])
    want = sorted(range(n), key=lambda i: f64[i], reverse=True)[:5]
    assert want == [20, 21, 22, 23, 24]

    class FakeIndex:
        n_rows = n

        def topk_features(self, fb, k, labels=None, distinct=False, tags=None):
            s32 = f64.astype(np.float32)
            order = np.lexsort((np.arange(n), -s32))[:k]          # float32 score desc, row asc: what K1b returns
            return np.tile(s32[order], (fb.n, 1)), np.tile(order.astype(np.int64), (fb.n, 1))

        def rescore(self, fb, rows):
            return f64[rows]

        def score(self, text):
            return f64.copy()

        def close(self):
            pass

    st = GfkbStore()
    st.records = [{"failure_id": f"F-{i:04d}", "version": 1, "failure_type": "T", "suggested_mitigation": None,
                   "signature_text": "x"} for i in range(n)]
    monkeypatch.setattr(st, "_sync", lambda: None)

    class _B:
        n = 2

        def close(self):
            pass
    monkeypatch.setattr(st.vocab, "featurize", lambda texts, grow=False, n_threads=0: _B())
    st._main = FakeIndex()
    got = st.match_batch(["q0", "q1"])
    assert [[m["failure_id"] for m in ms] for ms in got] == [[f"F-{i:04d}" for i in want]] * 2
    assert [m["score"] for m in got[0]] == [f64[i] for i in want]
    assert st.stats["exact_fallbacks"] == 2
    assert [m["failure_id"] for m in st.match_exact("q0")] == [f"F-{i:04d}" for i in want]
    st._main = None


def test_store_exact_top_eligibility_matches_brute_force(built_lib):
    """The exact fallback (``GfkbStore._exact_top``) against Python's stable sort over the eligible records: live, of
    the label's failure type, listing the app, and under ``distinct`` only the first record of each (failure_type,
    signature_text) key.  Every combination of label, app and distinct, with and without deleted device rows, over two
    segments and a score vector with heavy ties (a deleted row scores above every live one, so it must be excluded)."""
    import itertools

    from kakveda_b200 import GfkbStore

    class Segment:
        def __init__(self, scores):
            self.scores, self.n_rows = scores, len(scores)

        def score(self, text):
            return self.scores.copy()

    rng = np.random.default_rng(11)
    n_rec, n_del = 240, 40
    records = [{"failure_type": "ABC"[rng.integers(0, 3)], "signature_text": f"t{rng.integers(0, 25)}",
                "affected_apps": sorted(set(rng.choice(list("wxyz"), size=rng.integers(1, 3)).tolist()))}
               for _ in range(n_rec)]
    for deleted in (False, True):
        n_dev = n_rec + (n_del if deleted else 0)
        scores = rng.integers(0, 4, size=n_dev) / 4
        live = np.arange(n_dev)
        st = GfkbStore()
        st.records = records
        st._n_indexed = n_rec
        if deleted:
            dead = rng.choice(n_dev, size=n_del, replace=False)
            scores[dead] = 1.0
            live = np.setdiff1d(live, dead)
            st._row2rec = np.full(n_dev, -1, dtype=np.int64)
            st._row2rec[live] = np.arange(n_rec)
        rec_score = scores[live].tolist()
        split = n_dev * 2 // 3
        st._main, st._tail = Segment(scores[:split]), Segment(scores[split:])
        st._row_labels(0, n_rec)
        st._sync_apps()
        app_name = {i: a for a, i in st._apps.ids.items()}
        for label, app, distinct, limit in itertools.product([-1] + sorted(st._type_ids.values()),
                                                             [-1] + sorted(app_name), (False, True), (1, 5, 32, 300)):
            elig = [r for r, rec in enumerate(records)
                    if (label < 0 or st._type_ids[rec["failure_type"]] == label)
                    and (app < 0 or app_name[app] in rec["affected_apps"])]
            if distinct:
                first = {}
                for r in elig:
                    first.setdefault((records[r]["failure_type"], records[r]["signature_text"]), r)
                elig = sorted(first.values())
            want = sorted(elig, key=lambda r: rec_score[r], reverse=True)[:limit]
            got = st._exact_top("q", limit, label, distinct, app)
            assert got == (want, [rec_score[r] for r in want]), (deleted, label, app, distinct, limit)
        st._main = st._tail = None


def test_store_rejects_unindexable_rows_before_persisting(tmp_path):
    """A record the scan layout cannot hold must never reach failures.jsonl (it would break every later request and
    every restart); loading a file that contains one quarantines it instead of failing."""
    from kakveda_b200 import store as S

    assert S.check_indexable("intent_tags: | prompt_hint:summarize this paper | tools: | env_keys:os") is None
    assert S.check_indexable("tok " * 70000) is not None               # 'tok' x 70000 > 65535
    assert S.check_indexable("ab cd", vocab_size=S.MAX_FEATURES) is not None
    assert S.check_indexable(" ".join(f"w{i}" for i in range(70000))) is None  # long, but no feature repeats
