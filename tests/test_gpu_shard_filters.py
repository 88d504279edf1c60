"""The query filters of a resident batch of the row-sharded GFKB (dist.py), on ONE GPU through the loopback collectives
of test_gpu_shard_loopback.py.

* A threshold search applies exactly the filters it is given: after a labelled or tagged top-k and threshold search of
  the same resident batch, an unfiltered threshold search equals the one of a fresh upload and the single index's, in
  rows mode (index and text order) and queries mode.
* Queries mode takes batches with fewer queries than ranks: ``topk_packed`` and ``range_packed`` of 1 and 2 queries on
  3 ranks equal the single index on every rank.
"""
import numpy as np
import pytest

torch = pytest.importorskip("torch")

from test_gpu_shard_loopback import Corpus, _close, _copy, build_sharded, lib, loopback, run_ranks, synth_texts  # noqa: E402,F401
from test_gpu_shard_range import _check_range, _np, _single_range  # noqa: E402

gpu = pytest.mark.gpu


@pytest.fixture(scope="module")
def corpus(lib):
    return Corpus(*synth_texts(30_000, 300))


def _row_and_query_filters(c, kind, rng):
    """Row labels and per-query labels (-1: any row), or row tag sets and per-query tag sets (empty: any row)."""
    nq = len(c.queries)
    if kind == "labels":
        return rng.integers(0, 4, c.n).astype(np.int32), rng.integers(-1, 4, nq).astype(np.int32)
    rows = [rng.choice(12, int(rng.integers(0, 3)), replace=False).tolist() for _ in range(c.n)]
    return rows, [rng.choice(12, int(rng.integers(0, 3)), replace=False).tolist() for _ in range(nq)]


CASES = [("rows", "index", 3), ("rows", "text", 3), ("queries", "index", 2)]


@gpu
@pytest.mark.parametrize("kind", ["labels", "tags"])
@pytest.mark.parametrize("mode,order,world", CASES, ids=[f"{m}-{o}-W{w}" for m, o, w in CASES])
def test_unfiltered_range_after_filtered_searches(corpus, loopback, mode, order, world, kind):
    c = corpus
    row_f, query_f = _row_and_query_filters(c, kind, np.random.default_rng(world))
    build = build_sharded(world, order, mode, c)
    k, thr = 16, 0.5

    def fn(r, g):
        sh = build(r, g)
        try:
            (sh.set_row_labels if kind == "labels" else sh.set_row_tags)(row_f)
            qfb = sh.vocab.featurize(c.queries, grow=False)
            try:
                sh.set_resident(qfb)
                sh.topk_resident(k, **{kind: query_f})
                filtered = _np(sh.range_resident(thr, **{kind: query_f}))
                after = _np(sh.range_resident(thr))
                sh.set_resident(qfb)
                fresh = _np(sh.range_resident(thr))
            finally:
                qfb.close()
            return filtered, after, fresh
        finally:
            _close([sh])

    out = run_ranks(world, fn)
    filtered, after, fresh = out[0]
    for rk, o in enumerate(out):
        for got, want in zip(o[1], after):
            np.testing.assert_array_equal(got, want, err_msg=f"rank {rk}")
    assert len(filtered[1]) < len(after[1]), "the filter removed no pair"
    for got, want in zip(after, fresh):
        assert got.tobytes() == want.tobytes()
    _check_range(c, f"{mode} {order} W={world} after {kind}", after, thr, _single_range(c, thr))


@gpu
@pytest.mark.parametrize("nq", [1, 2])
def test_queries_mode_batch_smaller_than_world(corpus, loopback, nq):
    from kakveda_b200.similarity import pack_texts

    c = corpus
    world, k, thr = 3, 16, 0.3
    queries = c.queries[:nq]
    qdata, qoff, qmode = pack_texts(queries)
    build = build_sharded(world, "index", "queries", c)

    def fn(r, g):
        sh = build(r, g)
        try:
            s, rr = sh.topk_packed(qdata, qoff, k, qmode)
            return _copy(s), _copy(rr), _np(sh.range_packed(qdata, qoff, thr, qmode))
        finally:
            _close([sh])

    out = run_ranks(world, fn)
    fb = c.one.vocab.featurize(queries, grow=False)
    try:
        want_s, want_r = c.one.topk_features(fb, k)
        want_range = _np(c.one.range_features(fb, thr))
    finally:
        fb.close()
    assert len(want_range[1]) > 0
    for rk, (s, rr, res) in enumerate(out):
        np.testing.assert_array_equal(rr, want_r, err_msg=f"rank {rk}")
        assert s.tobytes() == want_s.tobytes(), f"rank {rk}"
        for got, want in zip(res, want_range):
            assert got.tobytes() == want.tobytes(), f"rank {rk}"
