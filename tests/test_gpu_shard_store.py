"""``ShardedGfkbStore`` (dist.py): the GFKB store on a row-sharded GFKB, run on ONE GPU through the loopback collectives
of test_gpu_shard_loopback.py at W = 1, 2, 3 and 8.  Every rank's results must be identical, and equal to the reference
goldens and to the single ``GfkbStore``:

* the reference's upsert/match stream (service_upsert.json) at tail_limit 40 and 0: the same responses, rows and order
  exactly, float64 scores within 1e-12, and a failures.jsonl byte-identical to the single store's (written by rank 0
  only);
* fixture54 matches, the reference's warnings and its purge (purge.json): a purge costs exactly one all-reduce and
  leaves every shard on a statistics-only finalize;
* the exact fallback (``kv_exact_topk`` on every shard and the tail, one all-gather) on duplicate groups straddling
  every shard boundary and on texts stored more than 16 times: filter_first, distinct and both, across a compaction;
* errors raise the same exception on every rank and leave the store usable.

``kv_exact_topk`` itself is checked on one index against the K1a score vector, and ``ShardedGfkb.exact_topk`` against
the single index bit for bit.
"""
import json
from datetime import datetime, timezone

import numpy as np
import pytest

torch = pytest.importorskip("torch")
import torch.distributed as tdist  # noqa: E402

from test_gpu_shard_loopback import lib, loopback, run_ranks  # noqa: E402,F401

gpu = pytest.mark.gpu
WORLDS = (1, 2, 3, 8)
RTOL = 1e-12
CLOCK = lambda: datetime(2026, 5, 6, 7, 8, 9, tzinfo=timezone.utc)  # noqa: E731


def _key(ms):
    return [(m["failure_id"], m["version"], m["failure_type"], m["suggested_mitigation"]) for m in ms]


def _same(a, b, rtol=RTOL):
    """Two match lists (or lists of them): equal fields, float64 scores within rtol."""
    if a and isinstance(a[0], list):
        assert len(a) == len(b)
        for x, y in zip(a, b):
            _same(x, y, rtol)
        return
    assert _key(a) == _key(b)
    np.testing.assert_allclose([m["score"] for m in a], [m["score"] for m in b], rtol=rtol)


def _identical_on_ranks(outs):
    for o in outs[1:]:
        assert o == outs[0]


def _sharded(rank, group, world, **kw):
    from kakveda_b200.dist import ShardedGfkbStore

    return ShardedGfkbStore(device=0, rank=rank, world=world, group=group, **kw)


class _CountAllReduce:
    """Counts each rank's all-reduce calls (installed on top of the loopback collectives)."""

    def __init__(self, monkeypatch):
        self.counts = {}
        inner = tdist.all_reduce

        def counted(tensor, op=tdist.ReduceOp.SUM, group=None, async_op=False):
            self.counts[group.rank] = self.counts.get(group.rank, 0) + 1
            return inner(tensor, op=op, group=group, async_op=async_op)

        monkeypatch.setattr(tdist, "all_reduce", counted)


# ---------------------------------------------------------------------------------------------------------------------
# Arguments refused before anything runs
# ---------------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("kw", [{"sidecar": "side.npz"}, {"mode": "queries"}, {"order": "text"}])
def test_sharded_store_refuses_unsupported_layouts(kw):
    from kakveda_b200.dist import ShardedGfkbStore

    with pytest.raises(ValueError, match="ShardedGfkbStore"):
        ShardedGfkbStore(device=0, **kw)


# ---------------------------------------------------------------------------------------------------------------------
# kv_exact_topk
# ---------------------------------------------------------------------------------------------------------------------

def _stable(scores, idx, k):
    """The first k of ``idx`` (ascending) in (score desc, row asc) order."""
    return idx[np.lexsort((idx, -scores[idx]))][:k]


@gpu
def test_exact_topk_matches_k1a_order(lib):
    from kakveda_b200 import GfkbIndex, synth

    n, k = 3000, 12
    corpus = synth.corpus(n)
    for i in range(0, n, 97):   # duplicates: exact ties broken by row
        corpus[i] = corpus[5]
    labels = (np.arange(n) % 4).astype(np.int32)
    _, groups = np.unique(np.array(corpus), return_inverse=True)
    ix = GfkbIndex(row_base=1000)
    ix.add_texts(corpus)
    ix.finalize()
    ix.delete_rows(np.arange(7, n, 211))
    ix.finalize()
    ix.set_row_labels(labels)
    ix.set_row_groups(groups.astype(np.int32))
    queries = [corpus[5], corpus[40], synth.queries(1, n)[0], ""]
    fb = ix.vocab.featurize(queries, grow=False)
    try:
        lab = np.array([-1, 2, 1, 3], dtype=np.int32)
        for distinct in (False, True):
            for labs in (None, lab):
                rows, sc = ix.exact_topk(fb, k, labs, distinct)
                for q, text in enumerate(queries):
                    full = ix.score(text)
                    live = np.flatnonzero(np.isfinite(full))
                    if labs is not None and labs[q] >= 0:
                        live = live[labels[live] == labs[q]]
                    if distinct:
                        _, first = np.unique(groups[live][np.lexsort((live, -full[live]))], return_index=True)
                        live = np.sort(live[np.lexsort((live, -full[live]))][first])
                    want = _stable(full, live, k)
                    got = rows[q][rows[q] >= 0] - 1000
                    assert got.tolist() == want.tolist(), (q, distinct, labs)
                    np.testing.assert_allclose(sc[q][: len(want)], full[want], rtol=1e-12)
                    assert np.all(np.isneginf(sc[q][len(want):]))
        with pytest.raises(ValueError, match="k must be 1..32"):
            ix.exact_topk(fb, 33)
    finally:
        fb.close()
    bare = GfkbIndex()
    bare.add_texts(corpus[:50])
    bare.finalize()
    fb = bare.vocab.featurize(corpus[:2], grow=False)
    with pytest.raises(RuntimeError, match="row groups"):
        bare.exact_topk(fb, 5, distinct=True)
    with pytest.raises(RuntimeError, match="row labels"):
        bare.exact_topk(fb, 5, np.array([0, -1], np.int32))
    fb.close()


@gpu
@pytest.mark.parametrize("world", (2, 3, 8))
def test_sharded_exact_topk_equals_single_index(lib, loopback, world):
    """K6 scores do not depend on the shard: the merged lists equal the single index's, bit for bit."""
    from kakveda_b200 import GfkbIndex, synth
    from kakveda_b200.dist import ShardedGfkb
    from kakveda_b200.similarity import pack_texts

    n, k = 2000, 16
    corpus = synth.corpus(n)
    for b in range(1, 8):   # copies of one text on every shard boundary
        for d in (-1, 0):
            corpus[n * b // 8 + d] = corpus[3]
    labels = (np.arange(n) % 3).astype(np.int32)
    _, groups = np.unique(np.array(corpus), return_inverse=True)
    groups = groups.astype(np.int32)
    queries = [corpus[3], corpus[100], synth.queries(1, n)[0]]
    lab = np.array([-1, 1, 0], dtype=np.int32)
    single = GfkbIndex()
    single.add_texts(corpus)
    single.finalize()
    single.set_row_labels(labels)
    single.set_row_groups(groups)
    fb = single.vocab.featurize(queries, grow=False)
    want = {(d, l is None): single.exact_topk(fb, k, l, d) for d in (False, True) for l in (None, lab)}
    fb.close()

    def fn(rank, group):
        sg = ShardedGfkb(0, rank, world, group)
        sg.build_packed(*pack_texts(corpus))
        sg.set_row_labels(labels)
        sg.set_row_groups(groups)
        qfb = sg.vocab.featurize(queries, grow=False)
        out = {(d, l is None): sg.exact_topk(qfb, k, l, d) for d in (False, True) for l in (None, lab)}
        with pytest.raises(ValueError, match="labels"):
            sg.exact_topk(qfb, k, lab[:2])
        qfb.close()
        sg.close()
        return out

    for out in loopback(world, fn):
        for key, (r, s) in want.items():
            np.testing.assert_array_equal(out[key][0], r)
            np.testing.assert_array_equal(out[key][1], s)


# ---------------------------------------------------------------------------------------------------------------------
# 1. The reference's upsert / match stream
# ---------------------------------------------------------------------------------------------------------------------

def _replay_upserts(st, g):
    created, matches = [], []
    for step in g["steps"]:
        out = st.upsert(step["upsert"])
        created.append((out["created"], out["failure"]))
        for m in step.get("matches", []):
            matches.append(st.match(m["signature_text"], m["failure_type"]))
    return created, matches


@gpu
@pytest.mark.parametrize("tail_limit", [40, 0])
@pytest.mark.parametrize("world", WORLDS)
def test_sharded_store_replays_reference_upserts(lib, loopback, golden, tmp_path, world, tail_limit):
    from kakveda_b200 import GfkbStore

    g = golden("service_upsert.json")
    want_matches = [m["matches"] for step in g["steps"] for m in step.get("matches", [])]
    single = GfkbStore(path=tmp_path / "single.jsonl", tail_limit=tail_limit, now=CLOCK)
    s_created, s_matches = _replay_upserts(single, g)
    path = tmp_path / "sharded.jsonl"

    def fn(rank, group):
        st = _sharded(rank, group, world, path=path, tail_limit=tail_limit, now=CLOCK)
        out = _replay_upserts(st, g)
        stats = dict(st.stats)
        st.close()
        return out, stats

    outs = loopback(world, fn)
    _identical_on_ranks([o[0] for o in outs])
    (created, matches), stats = outs[0]
    assert created == s_created
    assert [c[0] for c in created] == [step["created"] for step in g["steps"]]
    assert len(matches) == len(want_matches) > 0
    _same(matches, want_matches)
    _same(matches, s_matches)
    assert path.read_bytes() == single.path.read_bytes()
    if tail_limit:
        assert stats["stat_refreshes"] > 0 and stats["compactions"] > 0
    else:
        assert stats["stat_refreshes"] == 0
    single.close()


# ---------------------------------------------------------------------------------------------------------------------
# 2. fixture54 matches, the reference's warnings and purge
# ---------------------------------------------------------------------------------------------------------------------

def _strip(rec):
    return {k: v for k, v in rec.items() if k not in ("created_at", "updated_at")}


@gpu
@pytest.mark.parametrize("world", WORLDS)
def test_sharded_store_fixture_warn_and_purge(lib, loopback, golden, tmp_path, world, monkeypatch):
    from kakveda_b200 import GfkbStore

    fx, warn, purge = golden("fixture54.json"), golden("service_warn.json"), golden("purge.json")
    cases = fx["match"]
    sigs, fts = [c["signature_text"] for c in cases], [c["failure_type"] for c in cases]
    counter = _CountAllReduce(monkeypatch)
    path = tmp_path / "failures.jsonl"

    def fn(rank, group):
        out = {}
        st = _sharded(rank, group, world)
        st._reset([dict(r) for r in fx["records"]])
        out["fixture"] = st.match_batch(sigs, fts)
        st._reset([dict(r) for r in warn["failures"]])
        out["warn"] = [st.warn_batch(warn["requests"], threshold=p["threshold"], default_action=p["default_action"],
                                     patterns=[warn["pattern"]]) for p in warn["policies"]]
        st.close()
        st = _sharded(rank, group, world, path=path, tail_limit=1000, now=CLOCK)
        out["purge"], out["reduces"], out["kinds"] = [], [], []
        seen = []
        for step in purge["steps"]:
            if "upsert" in step:
                res = st.upsert(step["upsert"])
                out["purge"].append((res["created"], _strip(res["failure"])))
                seen.append(step["upsert"]["signature_text"])
            elif "matches" in step:
                out["purge"].append([st.match(m["signature_text"], m["failure_type"]) for m in step["matches"]])
            else:
                before = counter.counts.get(rank, 0)
                out["purge"].append(st.purge_apps(step["purge"]))
                out["reduces"].append(counter.counts.get(rank, 0) - before)
                out["kinds"].append((st._main.index.last_finalize_kind,
                                     None if st._tail is None else st._tail.last_finalize_kind))
                out["purge"].append([_strip(r) for r in st.records])
                out["purge"].append(st.match_batch(seen[-25:]))
                out["purge"].append(st.match_batch(seen[-25:], distinct=True))
        st.close()
        return out

    outs = loopback(world, fn)
    _identical_on_ranks(outs)
    out = outs[0]
    for c, ms in zip(cases, out["fixture"]):
        _same(ms, c["matches"])
    for pol, got in zip(warn["policies"], out["warn"]):
        assert len(got) == len(pol["responses"])
        for a, b in zip(got, pol["responses"]):
            assert (a["action"], a["pattern_id"]) == (b["action"], b["pattern_id"])
            if b["references"]:   # the text embeds the score with two decimals
                assert a["message"] == b["message"]
            else:
                assert a["message"] == b["message"] == "No high-similarity match found in GFKB."
            np.testing.assert_allclose(a["confidence"], b["confidence"], rtol=RTOL, atol=1e-15)
            _same(a["references"], b["references"])
    # the purge replay against the reference and against the single store
    single = GfkbStore(path=tmp_path / "single.jsonl", tail_limit=1000, now=CLOCK)
    got = iter(out["purge"])
    seen = []
    for step in purge["steps"]:
        if "upsert" in step:
            res = single.upsert(step["upsert"])
            assert next(got) == (step["created"], step["failure"]) == (res["created"], _strip(res["failure"]))
            seen.append(step["upsert"]["signature_text"])
        elif "matches" in step:
            ms = next(got)
            for m, x in zip(step["matches"], ms):
                _same(x, m["matches"])
        else:
            assert next(got) == step["counts"] == single.purge_apps(step["purge"])
            assert next(got) == step["lines"]
            _same(next(got), single.match_batch(seen[-25:]))
            _same(next(got), single.match_batch(seen[-25:], distinct=True))
    assert [json.loads(l) for l in path.read_text(encoding="utf-8").splitlines()] == single.records
    assert path.read_bytes() == single.path.read_bytes()
    assert (tmp_path / "failures.jsonl.bak-20260506T070809Z").exists()
    # a purge that deletes main rows is ONE all-reduce on every rank; one that only deletes tail rows reuses the cached
    # main statistics and exchanges nothing
    assert out["reduces"][0] == (1 if world > 1 else 0) and max(out["reduces"]) <= 1
    for main_kind, tail_kind in out["kinds"]:
        assert main_kind == 2 and tail_kind in (None, 2)
    single.close()


# ---------------------------------------------------------------------------------------------------------------------
# 3. The exact fallback: duplicate groups on every shard boundary, texts stored more than 16 times, a compaction
# ---------------------------------------------------------------------------------------------------------------------

def _synthetic_records(n):
    from kakveda_b200 import synth

    corpus = synth.corpus(n)
    a = corpus[11]
    b = a + " extra"           # close to a: both crowd the candidate lists of either query
    texts = list(corpus)
    for i in range(0, n, n // 24):
        texts[i] = a if (i // (n // 24)) % 2 else b
    for w in (2, 3, 8):        # a duplicate group on both sides of every shard boundary
        for r in range(1, w):
            lo = n * r // w
            texts[lo - 1] = texts[lo] = corpus[500 + w * 10 + r]
    types = ["X", "Y", "Z"]
    return [{"failure_id": f"F-{i + 1:04d}", "version": 1, "created_at": "2026-01-01T00:00:00Z",
             "updated_at": "2026-01-01T00:00:00Z", "failure_type": types[i % 3], "root_cause": None,
             "context_signature": {}, "impact_severity": "low", "resolution": f"r{i % 7}", "occurrences": 1,
             "affected_apps": [f"app-{i % 4}"], "signature_text": t} for i, t in enumerate(texts)], a, b, corpus


def _exact_stream(st, recs, a, b, corpus):
    """Matches in every mode, then upserts that fill the tail and force a compaction, with matches in between."""
    from kakveda_b200 import synth

    qs = [a, b, corpus[11], recs[-1]["signature_text"]] + [corpus[500 + w * 10 + r] for w in (2, 3, 8) for r in (1,)] + \
        synth.queries(6, len(recs))
    fts = ["X", "Y", "Z", None] * (len(qs) // 4 + 1)
    fts = fts[:len(qs)]
    out = []

    def probe():
        out.append(st.match_batch(qs, fts))
        out.append(st.match_batch(qs, fts, filter_first=True))
        out.append(st.match_batch(qs, fts, distinct=True))
        out.append(st.match_batch(qs, fts, filter_first=True, distinct=True))
        out.append(st.match_batch(qs[:6], limit=16, distinct=True))
        out.append(st.match_exact(a, "Y"))
        out.append(dict(st.stats))

    probe()
    for i in range(30):   # new versions of stored keys (a, b among them) and new keys, into the tail
        st.upsert({"failure_type": ["X", "Y", "W"][i % 3], "signature_text": [a, b, corpus[(i * 13) % len(recs)]][i % 3],
                   "context_signature": {}, "impact_severity": "low", "app_id": f"app-{i % 5}", "resolution": f"t{i}"})
        if i % 10 == 9:
            probe()
    st.purge_apps(["app-1"], backup=False)
    probe()
    return out


@gpu
@pytest.mark.parametrize("world", WORLDS)
def test_sharded_store_exact_fallback_filters_distinct_compaction(lib, loopback, world):
    from kakveda_b200 import GfkbStore

    n = 2400
    recs, a, b, corpus = _synthetic_records(n)
    single = GfkbStore(tail_limit=25, now=CLOCK)
    single._reset([dict(r) for r in recs])
    want = _exact_stream(single, recs, a, b, corpus)

    def fn(rank, group):
        st = _sharded(rank, group, world, tail_limit=25, now=CLOCK)
        st._reset([dict(r) for r in recs])
        out = _exact_stream(st, recs, a, b, corpus)
        st.close()
        return out

    outs = loopback(world, fn)
    _identical_on_ranks(outs)
    got = outs[0]
    assert len(got) == len(want)
    for x, y in zip(got, want):
        if isinstance(x, dict):
            assert x.get("exact_fallbacks", 0) == y.get("exact_fallbacks", 0)
            assert x["compactions"] == y["compactions"]
        else:
            _same(x, y)
    assert got[-1]["exact_fallbacks"] > 0 and got[-1]["compactions"] > 0


# ---------------------------------------------------------------------------------------------------------------------
# 4. Errors
# ---------------------------------------------------------------------------------------------------------------------

@gpu
@pytest.mark.parametrize("world", (2, 3))
def test_sharded_store_errors_on_every_rank(lib, loopback, golden, world):
    from kakveda_b200 import GfkbStore

    recs = golden("fixture54.json")["records"]
    sigs = [r["signature_text"] for r in recs[:10]]
    bad = {"failure_type": "X", "signature_text": "ab " * 70000, "context_signature": {}, "impact_severity": "low",
           "app_id": "a"}
    single = GfkbStore(now=CLOCK)
    single._reset([dict(r) for r in recs])

    def fn(rank, group):
        st = _sharded(rank, group, world, now=CLOCK)
        st._reset([dict(r) for r in recs])
        errs = []
        for call in (lambda: st.upsert(bad), lambda: st.match_batch(sigs, limit=33),
                     lambda: st.match_batch(sigs, limit=33, distinct=True)):
            with pytest.raises(ValueError) as e:
                call()
            errs.append(str(e.value))
        ok = st.match_batch(sigs)
        n = len(st.records)
        st.close()
        return errs, ok, n

    outs = loopback(world, fn)
    _identical_on_ranks(outs)
    errs, ok, n = outs[0]
    assert "upsert rejected" in errs[0] and "limit 33" in errs[1]
    assert n == len(recs)
    _same(ok, single.match_batch(sigs))
    single.close()
