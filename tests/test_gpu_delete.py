"""Row deletion: tombstoned rows of a finalized TF-IDF index, and the app purge of the resident store.

The oracle of a deletion is the float64 closed form (or sklearn's corpus fit) refitted on the SURVIVING rows and mapped
back to the original row ids, with the deleted rows set to -inf; it is checked with the strict tie rules of
test_gpu_topk_edges.py.  The deleted sets mix 10 % random rows, whole duplicate groups (identical rows sit side by side
in the scan order, so whole chunks die) and every row holding one feature f, which leaves f in the vocabulary with
df = 0.  The chunk-skipping test asserts that an all-deleted chunk is never scored: without it an implementation that
scans every chunk would pass the rest.
"""
import json
from datetime import datetime, timezone

import numpy as np
import pytest

from oracle import tfidf_oracle as O

gpu = pytest.mark.gpu

RTOL32 = 1e-5
RTOL64 = 1e-9
KS = (1, 5, 16, 32)
QFEATS = 64
THR = 0.3


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
        assert np.isfinite(o[rr]).all(), "a deleted (or excluded) row was returned; " + where
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


def survivors_oracle(queries, corpus, dead, mode):
    """[Q, N] float64 scores refitted on the live rows, -inf on the deleted ones."""
    live = np.flatnonzero(~dead)
    sub = [corpus[i] for i in live]
    s = O.corpus_fit_scores(queries, sub) if mode == 2 else O.score_matrix_closed_form(queries, sub)
    out = np.full((len(queries), len(corpus)), -np.inf)
    out[:, live] = s
    return out


def check_range(ip, rows, sc, oracle, dead, thr):
    """Every pair clearly above thr is there, every returned pair is near or above it, and no deleted row appears."""
    assert not dead[rows].any(), "a deleted row in a threshold result"
    for q in range(len(ip) - 1):
        rr, ss = rows[ip[q]:ip[q + 1]], sc[ip[q]:ip[q + 1]].astype(np.float64)
        o = oracle[q]
        assert np.all(np.abs(ss - o[rr]) <= RTOL32 * np.abs(o[rr])), q
        assert np.all(o[rr] >= thr * (1 - 2 * RTOL32)), q
        want = np.flatnonzero(o >= thr * (1 + 2 * RTOL32))
        assert np.isin(want, rr).all(), (q, np.setdiff1d(want, rr)[:10].tolist())


class Case:
    """n synthetic rows plus 24 texts stored 64 times each (whole duplicate groups) and a row of 70 features (queries
    with more than 64 of them take the float64 fallback); deleted: 10 % at random, 12 of the duplicate groups and
    every row holding the token f (planted in 25 rows)."""

    def __init__(self, n, mode):
        from kakveda_b200 import GfkbIndex, synth

        rng = np.random.default_rng(11 + n + mode)
        base = synth.corpus(n)
        groups = [f"dupgroup{g} alpha{g} beta{g} shared tokens of group {g}" for g in range(24)]
        corpus = list(base)
        slots = rng.choice(len(corpus) + 1, size=24 * 64, replace=True)
        for j, s in enumerate(sorted(slots, reverse=True)):
            corpus.insert(int(s), groups[j % 24])
        self.n = len(corpus)
        self.wide_row = self.n // 3 + 1
        corpus[self.wide_row] = " ".join(f"pw{i}" for i in range(70))
        self.f = "plantedfeature"
        self.f_rows = sorted(rng.choice(np.arange(self.n // 2, self.n), size=25, replace=False).tolist())
        for i in self.f_rows:
            corpus[i] = corpus[i] + " " + self.f
        self.corpus = corpus
        dead = np.zeros(self.n, dtype=bool)
        dead[rng.choice(self.n, size=self.n // 10, replace=False)] = True
        self.group_rows = [i for i, t in enumerate(corpus) if t in set(groups[:12])]
        dead[self.group_rows] = True
        dead[self.f_rows] = True
        dead[self.wide_row] = False
        self.dead = dead
        qs = synth.queries(120, n)
        wide = lambda m: " ".join(f"pw{i}" for i in reversed(range(m)))
        self.queries = (qs + [corpus[i] for i in np.flatnonzero(dead)[:20]] + groups[:2] + groups[12:14] +
                        [f"{self.f} {corpus[7]}", self.f, "", "qqzzunseen xxyyq", wide(QFEATS + 1) + " " + corpus[9]])
        self.mode = mode
        self.ix = GfkbIndex()
        if mode:
            self.ix.set_mode(mode)
        self.ix.add_texts(corpus)
        self.ix.finalize()
        self.oracle = survivors_oracle(self.queries, corpus, dead, mode)


@pytest.fixture(scope="module")
def lib(built_lib):
    from kakveda_b200 import _capi

    assert _capi.load().kv_device_count() > 0, "GPU tests need a CUDA device"
    return _capi.load()


@gpu
@pytest.mark.parametrize("n", [60000, 2000])   # the pruned path, the exhaustive scan
@pytest.mark.parametrize("mode", [0, 2])
def test_delete_topk_range_and_scores(lib, n, mode):
    c = Case(n, mode)
    ix = c.ix
    labels = (np.arange(c.n) % 7).astype(np.int32)
    ix.set_row_labels(labels)
    ix.delete_rows(np.flatnonzero(c.dead))
    with pytest.raises(RuntimeError):
        ix.topk(c.queries[:3], 4)          # a deletion needs finalize first
    ix.finalize()
    assert ix.last_finalize_kind == 2
    assert ix.n_live_rows == c.n - int(c.dead.sum()) and ix.n_rows == c.n
    np.testing.assert_array_equal(ix.deleted_mask(), c.dead)
    # live document frequencies: the survivors' own
    fb = ix.vocab.featurize([c.corpus[i] for i in np.flatnonzero(~c.dead)], grow=False)
    want_df = np.zeros(len(ix.vocab), np.int64)
    for q in range(fb.n):
        np.add.at(want_df, np.unique(fb.ids[fb.indptr[q]:fb.indptr[q + 1]]), 1)
    fb.close()
    np.testing.assert_array_equal(ix.local_df().astype(np.int64), want_df)
    f_id = ix.vocab.featurize([c.f], grow=False)
    assert len(f_id.ids) == 1 and want_df[int(f_id.ids[0])] == 0   # f stays in the vocabulary with df 0
    f_id.close()
    for k in KS:
        s, r = ix.topk(c.queries, k)
        check_topk_strict(s, r, c.oracle, k, RTOL32)
    assert (ix.layout()["pairs_passed_bound"] > 0) == (n == 60000)
    # null queries get the first k live rows
    live = np.flatnonzero(~c.dead)
    s, r = ix.topk(["", "qqzzunseen"], 32)
    assert r.tolist() == [live[:32].tolist()] * 2 and np.all(s == 0)
    # filtered: labels survive the deletion, a filtered null query gets the first live rows of its label
    ql = (np.arange(len(c.queries)) % 8 - 1).astype(np.int32)
    want = c.oracle.copy()
    for q, lb in enumerate(ql):
        if lb >= 0:
            want[q, labels != lb] = -np.inf
    for k in (5, 32):
        s, r = ix.topk(c.queries, k, labels=ql)
        check_topk_strict(s, r, want, k, RTOL32)
    s, r = ix.topk([""], 8, labels=np.array([3], np.int32))
    assert r[0].tolist() == live[labels[live] == 3][:8].tolist()
    # threshold search
    ip, rows, sc = ix.range(c.queries, THR)
    check_range(ip, rows, sc, c.oracle, c.dead, THR)
    # K1a and K6 against the survivors' float64 scores, -inf on deleted rows
    for qi in list(range(0, 120, 17)) + list(range(len(c.queries) - 5, len(c.queries))):
        got = ix.score(c.queries[qi])
        o = c.oracle[qi]
        assert np.all(np.isneginf(got[c.dead]))
        np.testing.assert_allclose(got[~c.dead], o[~c.dead], rtol=RTOL64, atol=1e-15)
    fb = ix.vocab.featurize(c.queries[:40], grow=False)
    s, r = ix.topk(c.queries[:40], 8)
    probe = np.concatenate([r, np.tile(np.flatnonzero(c.dead)[:4], (40, 1))], axis=1)
    got = ix.rescore(fb, probe)
    fb.close()
    want = np.take_along_axis(c.oracle[:40], np.where(probe < 0, 0, probe), axis=1)
    want[probe < 0] = -np.inf
    np.testing.assert_allclose(got, want, rtol=RTOL64, atol=1e-15)
    # self-joins: a deleted row's list is empty and no list holds a deleted row
    lo, hi = 0, 400
    qs = [c.corpus[i] for i in range(lo, hi)]
    so = survivors_oracle(qs, c.corpus, c.dead, mode)
    so[np.arange(hi - lo), np.arange(lo, hi)] = -np.inf
    so[c.dead[lo:hi]] = -np.inf
    for k in (1, 16):
        s, r = ix.selfjoin_topk(k, lo, hi)
        check_topk_strict(s, r, so, k, RTOL32)
    ip, rows, sc = ix.selfjoin_range(0.5, lo, hi)
    check_range(ip, rows, sc, so, c.dead, 0.5)
    assert np.all(np.diff(ip)[c.dead[lo:hi]] == 0)



@gpu
@pytest.mark.parametrize("n", [60000, 2000])
def test_exhaustive_scan_skips_deleted_chunks(lib, monkeypatch, n):
    """The exhaustive scan scores every (regular query, chunk) pair -- except the chunks whose rows are all deleted:
    each of the 12 deleted duplicate groups (64 identical rows, side by side in the scan order) covers a whole chunk."""
    monkeypatch.setenv("KAKVEDA_B200_NO_PRUNE", "1")
    c = Case(n, 0)
    ix = c.ix
    regular = len(c.queries) - 3   # the two null queries and the irregular one are answered elsewhere
    ix.topk(c.queries, 4)
    chunks = ix.layout()["chunks"]
    assert ix.layout()["pairs_scored"] == regular * chunks
    ix.delete_rows(np.flatnonzero(c.dead))
    ix.finalize()
    s, r = ix.topk(c.queries, 4)
    assert ix.layout()["pairs_scored"] <= regular * (chunks - 12)
    check_topk_strict(s, r, c.oracle, 4, RTOL32)


@gpu
def test_append_after_delete_and_errors(lib):
    from kakveda_b200 import GfkbIndex, synth

    corpus = synth.corpus(20000)
    ix = GfkbIndex()
    ix.add_texts(corpus)
    ix.finalize()
    dead = np.zeros(20000 + 300, dtype=bool)
    dead[np.arange(0, 20000, 9)] = True
    ix.delete_rows(np.flatnonzero(dead))
    ix.finalize()
    assert ix.last_finalize_kind == 2
    # a double delete is a no-op: no finalize needed
    ix.delete_rows(np.flatnonzero(dead)[:50])
    ix.delete_rows(np.array([5, 5, 5]) * 9)
    ix.topk(corpus[:3], 4)
    extra = synth.queries(300, 20000, seed=99)
    ix.add_texts(extra)
    ix.finalize()
    assert ix.last_finalize_kind == 1 and ix.n_live_rows == 20300 - int(dead.sum())
    full = corpus + extra
    qs = [corpus[i] for i in range(0, 900, 9)] + synth.queries(60, 20000)
    o = survivors_oracle(qs, full, dead, 0)
    for k in (1, 32):
        s, r = ix.topk(qs, k)
        check_topk_strict(s, r, o, k, RTOL32)
    with pytest.raises(ValueError):
        ix.delete_rows([20300])
    with pytest.raises(ValueError):
        ix.delete_rows([-1])
    j = GfkbIndex()
    j.add_texts([f"alpha{i} beta{i}" for i in range(100)])
    j.set_mode(1)
    j.finalize()
    with pytest.raises(ValueError):
        j.delete_rows([1])


@gpu
def test_detect_patterns_leaves_deleted_rows_out(lib):
    from kakveda_b200 import GfkbIndex, synth
    from kakveda_b200.patterns import detect_patterns

    base = synth.corpus(300)
    recs = [{"failure_id": f"F-{i:04d}", "failure_type": "T", "signature_text": t, "affected_apps": ["z"]}
            for i, t in enumerate(base)]
    recs.append({"failure_id": "S", "failure_type": "T", "signature_text": "lonely two app record", "affected_apps": ["a", "b"]})
    text = base[3]
    for i in range(3):
        recs.append({"failure_id": f"X-{i}", "failure_type": "T", "signature_text": text + f" tail{i}", "affected_apps": [f"app{i}"]})
    ix = GfkbIndex()
    ix.set_mode(2)
    ix.add_texts([r["signature_text"] for r in recs])
    ix.finalize()
    got = detect_patterns(ix, recs, threshold=0.6, k=8)
    assert any(p["rows"] == [300] for p in got)   # a singleton spanning two apps
    assert any({3, 301, 302, 303} <= set(p["rows"]) for p in got), got
    ix.delete_rows([300, 302])
    ix.finalize()
    for k in (8, None):
        got = detect_patterns(ix, recs, threshold=0.6, k=k)
        assert not any(300 in p["rows"] or 302 in p["rows"] for p in got), got
        assert any({3, 301, 303} <= set(p["rows"]) for p in got), got   # the surviving similar rows still group


# ---- store ----------------------------------------------------------------------------------------------------------

def _records(texts, rng):
    apps = ["a", "b", "c", "d"]
    out = []
    for i, t in enumerate(texts):
        aa = sorted(set(rng.choice(apps, size=int(rng.integers(1, 3))).tolist()))
        out.append({"failure_id": f"F-{i + 1:04d}", "version": 1, "created_at": "x", "updated_at": "x",
                    "failure_type": ["X", "Y", "Z"][i % 3], "root_cause": None, "context_signature": {},
                    "impact_severity": "low", "resolution": f"fix {i}", "occurrences": 1, "affected_apps": aa,
                    "signature_text": t})
    return out


def _expected_purge(records, purge):
    kept = removed = updated = 0
    lines = []
    for r in records:
        r = json.loads(json.dumps(r))
        if isinstance(r.get("affected_apps"), list):
            after = [a for a in r["affected_apps"] if a not in purge]
            if after != r["affected_apps"]:
                r["affected_apps"] = after
                updated += 1
            if not after:
                removed += 1
                continue
        lines.append(r)
        kept += 1
    return {"kept": kept, "removed": removed, "updated": updated}, lines


def _key(matches):
    return [[(m["failure_id"], m["version"], m.get("suggested_mitigation")) for m in ms] for ms in matches]


def _same_matches(a, b):
    assert _key(a) == _key(b)
    for x, y in zip(a, b):
        np.testing.assert_allclose([m["score"] for m in x], [m["score"] for m in y], rtol=RTOL64)


@gpu
@pytest.mark.parametrize("tail_limit", [5000, 40])   # main + tail segments; a forced compaction
def test_store_purge_matches_fresh_store(lib, tmp_path, tail_limit):
    from kakveda_b200 import GfkbStore, synth

    rng = np.random.default_rng(5)
    corpus = synth.corpus(3000)
    path = tmp_path / "failures.jsonl"
    path.write_text("".join(json.dumps(r) + "\n" for r in _records(corpus, rng)), encoding="utf-8")
    clock = lambda: datetime(2026, 1, 2, 3, 4, 5, tzinfo=timezone.utc)
    st = GfkbStore(path, tail_limit=tail_limit, now=clock)
    for i in range(30):   # tail rows: new versions and new records from purged and surviving apps
        st.upsert({"failure_type": ["X", "W"][i % 2], "signature_text": corpus[i * 7] if i % 2 == 0 else f"new tail text {i}",
                   "context_signature": {}, "impact_severity": "low", "app_id": ["a", "c"][i % 2], "resolution": f"r{i}"})
    qs = corpus[:90:3] + synth.queries(20, 3000) + ["new tail text 3", ""]
    st.match_batch(qs)   # the tail is on the device
    before = [json.loads(l) for l in path.read_text(encoding="utf-8").splitlines()]
    want_counts, want_lines = _expected_purge(before, {"a", "b"})
    got = st.purge_apps(["a", "b"])
    assert got == want_counts and got["removed"] > 0
    assert (tmp_path / "failures.jsonl.bak-20260102T030405Z").exists()
    assert [json.loads(l) for l in path.read_text(encoding="utf-8").splitlines()] == want_lines == st.records
    fresh_path = tmp_path / "fresh.jsonl"
    fresh_path.write_text(path.read_text(encoding="utf-8"), encoding="utf-8")
    fresh = GfkbStore(fresh_path)
    _same_matches(st.match_batch(qs), fresh.match_batch(qs))
    types = ["X", "Y", "W"] * (len(qs) // 3 + 1)
    _same_matches(st.match_batch(qs, types[:len(qs)], filter_first=True),
                  fresh.match_batch(qs, types[:len(qs)], filter_first=True))
    _same_matches([st.match_exact(q) for q in qs[:10]], [fresh.match_exact(q) for q in qs[:10]])
    if tail_limit == 5000:
        assert st._main.last_finalize_kind == 2 and st.stats["compactions"] == 0
    else:
        assert st.stats["compactions"] >= 1
    # upserts after the purge: new ids F-%04d of len(records) + 1 and the newest surviving version
    for s in (st, fresh):
        s._now = clock
    ups = [{"failure_type": "X", "signature_text": corpus[3], "context_signature": {}, "impact_severity": "low", "app_id": "q"},
           {"failure_type": "Q", "signature_text": "after purge", "context_signature": {}, "impact_severity": "low", "app_id": "q"}]
    for u in ups:
        assert st.upsert(u) == fresh.upsert(u)
    _same_matches(st.match_batch(qs), fresh.match_batch(qs))


@gpu
def test_store_purge_sidecar_restart(lib, tmp_path):
    from kakveda_b200 import GfkbStore, synth

    rng = np.random.default_rng(8)
    corpus = synth.corpus(2000)
    path, side = tmp_path / "failures.jsonl", tmp_path / "failures.side.npz"
    path.write_text("".join(json.dumps(r) + "\n" for r in _records(corpus, rng)), encoding="utf-8")
    st = GfkbStore(path, sidecar=side)
    st.upsert({"failure_type": "X", "signature_text": "tail row one", "context_signature": {}, "impact_severity": "low", "app_id": "a"})
    st.upsert({"failure_type": "X", "signature_text": "tail row two", "context_signature": {}, "impact_severity": "low", "app_id": "c"})
    qs = corpus[:40:2] + ["tail row two"]
    st.match_batch(qs)
    counts = st.purge_apps(["a"], backup=False)
    assert counts["removed"] > 0 and not list(tmp_path.glob("*.bak-*"))
    assert not (tmp_path / "failures.side.npz.layout").exists()
    again = GfkbStore(path, sidecar=side)
    assert again.stats.get("sidecar_rows") == len(st.records)
    _same_matches(st.match_batch(qs), again.match_batch(qs))
    _same_matches(again.match_batch(qs), GfkbStore(path).match_batch(qs))


# ---- the reference's own purge (tests/golden/purge.json, made by tests/golden/make_golden_purge.py) -------------------

def _strip(rec):
    return {k: v for k, v in rec.items() if k not in ("created_at", "updated_at")}


def _check_matches(st, step):
    for m in step["matches"]:
        got = st.match(m["signature_text"], m["failure_type"])
        want = m["matches"]
        assert [(x["failure_id"], x["version"], x["failure_type"], x["suggested_mitigation"]) for x in got] == \
               [(x["failure_id"], x["version"], x["failure_type"], x["suggested_mitigation"]) for x in want], m
        np.testing.assert_allclose([x["score"] for x in got], [x["score"] for x in want], rtol=RTOL64)


@gpu
@pytest.mark.parametrize("tail_limit", [1000, 10])   # deletions on main + tail segments; compactions
def test_store_replays_reference_purge(lib, golden, tmp_path, tail_limit):
    """Upserts, matches and two purges replayed through GfkbStore == what the reference's gfkb handlers and its
    dashboard's _purge_jsonl_apps produced: counts, surviving lines, new ids after a purge (F-%04d collisions), the
    newest surviving version on a repeat, and every match list."""
    from kakveda_b200 import GfkbStore

    g = golden("purge.json")
    clock = lambda: datetime(2026, 3, 4, 5, 6, 7, tzinfo=timezone.utc)
    path = tmp_path / "failures.jsonl"
    st = GfkbStore(path=path, tail_limit=tail_limit, now=clock)
    purges = 0
    for step in g["steps"]:
        if "upsert" in step:
            out = st.upsert(step["upsert"])
            assert out["created"] == step["created"] and _strip(out["failure"]) == step["failure"], step
        elif "matches" in step:
            _check_matches(st, step)
        else:
            assert [_strip(r) for r in st.records] == step["lines_before"]
            assert st.purge_apps(step["purge"]) == step["counts"]
            purges += 1
            assert [_strip(r) for r in st.records] == step["lines"]
            assert [_strip(json.loads(l)) for l in path.read_text(encoding="utf-8").splitlines()] == step["lines"]
            assert (tmp_path / "failures.jsonl.bak-20260304T050607Z").exists()
    assert purges == 2
    if tail_limit == 1000:
        assert st.stats["compactions"] == 0 and st._main.last_finalize_kind == 2
    else:
        assert st.stats["compactions"] > 0


@gpu
def test_store_purge_after_load_from_file(lib, golden, tmp_path):
    """The common case: a store opened on failures.jsonl and purged before any upsert (no tail segment).  Counts,
    lines and the reference's matches after the purge, and the same once records arrive in a tail afterwards."""
    from kakveda_b200 import GfkbStore

    steps = golden("purge.json")["steps"]
    for i, step in enumerate(steps):
        if "purge" not in step:
            continue
        path = tmp_path / f"failures{i}.jsonl"
        path.write_text("".join(json.dumps(r) + "\n" for r in step["lines_before"]), encoding="utf-8")
        st = GfkbStore(path=path)
        assert st._tail is None
        assert st.purge_apps(step["purge"], backup=False) == step["counts"]
        assert [_strip(r) for r in st.records] == step["lines"]
        _check_matches(st, steps[i + 1])
        assert st._tail is None and st._main.last_finalize_kind == 2
        st.upsert({"failure_type": "TIMEOUT", "signature_text": "a row for the tail after the purge",
                   "context_signature": {}, "impact_severity": "low", "app_id": "app-x"})
        fresh = GfkbStore(path=path)
        _same_matches(st.match_batch([m["signature_text"] for m in steps[i + 1]["matches"]]),
                      fresh.match_batch([m["signature_text"] for m in steps[i + 1]["matches"]]))
