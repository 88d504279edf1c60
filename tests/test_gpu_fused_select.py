"""Candidate selection inside the candidate scan (codes mode of tfidf_scan_kernel): when bound pass 0 keeps its 8-bit
bound codes, the scan's warps turn their group's codes into {chunk, query mask} records themselves.  The results must be
the bits of the two independent paths -- the recomputing bound pass 1 with its paged lists (KAKVEDA_B200_BOUND_CODES=0)
and the exhaustive scan (KAKVEDA_B200_NO_PRUNE=1) -- and the selection must not depend on how many CTAs split a
group's chunks (KAKVEDA_B200_CODE_SPLITS) or on the run: the threshold codes are a snapshot taken before the scan.
"""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

KS = (1, 16, 32)
BATCHES = (1, 31, 33, 129)
CODES_OFF = {"KAKVEDA_B200_BOUND_CODES": "0"}
EXHAUSTIVE = {"KAKVEDA_B200_NO_PRUNE": "1"}
SPLITS = ("1", "2", "5")


@pytest.fixture(scope="module")
def lib(built_lib):
    from kakveda_b200 import _capi

    assert _capi.load().kv_device_count() > 0, "GPU tests need a CUDA device"
    return _capi.load()


def make_index(n, delete=None, labels=None):
    from kakveda_b200 import GfkbIndex, synth

    ix = GfkbIndex()
    ix.add_texts(synth.corpus(n))
    ix.finalize()
    if delete is not None:
        ix.delete_rows(delete)
        ix.finalize()
    if labels is not None:
        ix.set_row_labels(labels)
    return ix


@pytest.fixture(scope="module")
def indexes(lib):
    """513 chunks (8 windows of 64 and one chunk) and 1875 chunks (29 windows and 19 chunks)."""
    return {n: make_index(n) for n in (16385, 60000)}


def run(monkeypatch, env, fn):
    with monkeypatch.context() as m:
        for key, v in env.items():
            m.setenv(key, v)
        out = fn()
    return out


def topk_run(ix, queries, k, labels=None):
    s, r = ix.topk(queries, k, labels=labels)
    return s, r, ix.layout()


def assert_same(a, b):
    assert a[1].tobytes() == b[1].tobytes()
    assert a[0].tobytes() == b[0].tobytes()


def check_paths(monkeypatch, fn, filtered=False):
    """fn() -> (scores, rows, layout) on the fused path, then against the list path, the exhaustive scan and forced
    split counts; the split counts must select identical candidates.  filtered: bound pass 1 lists chunks without the
    label signature test (the scan drops them), so its pair count is not compared."""
    fused = fn()
    lay = fused[2]
    assert lay["pairs_passed_bound"] > 0 and lay["pool_pages_used"] == 0, lay  # the codes were selected in the scan
    assert lay["pairs_scored"] >= lay["pairs_passed_bound"], lay
    lists = run(monkeypatch, CODES_OFF, fn)
    assert lists[2]["pool_pages_used"] > 0, lists[2]
    assert_same(fused, lists)
    if not filtered:  # the codes (bounds rounded up to 1/250) pass at least the pairs the recomputed bounds pass
        assert 0 < lists[2]["pairs_passed_bound"] <= lay["pairs_passed_bound"], (lay, lists[2])
    assert_same(fused, run(monkeypatch, EXHAUSTIVE, fn))
    for sp in SPLITS:
        forced = run(monkeypatch, {"KAKVEDA_B200_CODE_SPLITS": sp}, fn)
        assert_same(fused, forced)
        for key in ("pairs_passed_bound", "records_written"):
            assert forced[2][key] == lay[key], (sp, key, lay, forced[2])
    return fused


@pytest.mark.parametrize("n", [16385, 60000])
@pytest.mark.parametrize("batch", BATCHES)
def test_fused_selection_equals_list_and_exhaustive_paths(indexes, monkeypatch, n, batch):
    from kakveda_b200 import synth

    ix = indexes[n]
    queries = synth.queries(batch, n)
    for k in KS:
        check_paths(monkeypatch, lambda: topk_run(ix, queries, k))


def test_fused_selection_is_deterministic(indexes):
    from kakveda_b200 import synth

    ix = indexes[60000]
    queries = synth.queries(129, 60000)
    a = topk_run(ix, queries, 16)
    b = topk_run(ix, queries, 16)
    assert_same(a, b)
    for key in ("pairs_passed_bound", "records_written", "pairs_scored"):
        assert a[2][key] == b[2][key], key


def test_fused_selection_label_filter(lib, monkeypatch):
    """Zipf-weighted labels plus a label on 40 rows: with fewer than k rows to find, the rare label's threshold stays
    at 0, every chunk whose signature holds it becomes a record, and a warp's windows fill up many times."""
    from kakveda_b200 import synth

    n = 60000
    rng = np.random.default_rng(5)
    w = 1.0 / np.arange(1, 9)
    labels = rng.choice(8, size=n, p=w / w.sum()).astype(np.int32)
    labels[rng.choice(n, size=40, replace=False)] = 77
    ix = make_index(n, labels=labels)
    queries = synth.queries(129, n)
    ql = rng.choice(np.array([-1, 0, 3, 77], np.int32), size=len(queries)).astype(np.int32)
    ql[:40] = 77
    for k in (1, 32):
        s, r, _ = check_paths(monkeypatch, lambda: topk_run(ix, queries, k, labels=ql), filtered=True)
        got = r[ql == 77]
        assert np.all(np.isin(got[got >= 0], np.flatnonzero(labels == 77)))


def test_fused_selection_deleted_rows(lib, monkeypatch):
    """1 % of the rows deleted at random and a run of 4096 row ids: deleted rows are never returned."""
    from kakveda_b200 import synth

    n = 60000
    rng = np.random.default_rng(9)
    dead = np.concatenate([rng.choice(n, size=n // 100, replace=False), np.arange(64 * 32 * 3, 64 * 32 * 5)])
    ix = make_index(n, delete=dead)
    queries = synth.queries(129, n)
    for k in (1, 16):
        s, r, _ = check_paths(monkeypatch, lambda: topk_run(ix, queries, k))
        assert not np.any(np.isin(r, dead))


def test_fused_selection_selfjoin(indexes, monkeypatch):
    ix = indexes[60000]
    lo, hi = 1000, 1129
    for k in (1, 32):
        def fn():
            s, r = ix.selfjoin_topk(k, lo, hi)
            return s, r, ix.layout()
        s, r, _ = check_paths(monkeypatch, fn)
        assert not np.any(r == np.arange(lo, hi)[:, None])


def test_fused_selection_two_phase(indexes, monkeypatch):
    """Seed phase, thresholds raised from the seed top-k, finish: the bits of the one-phase batch at every split count."""
    import torch

    from kakveda_b200 import synth

    ix = indexes[60000]
    q, k = 129, 16
    qfb = ix.vocab.featurize(synth.queries(q, 60000), grow=False)
    ix.upload_queries(qfb)
    qfb.close()
    s1 = torch.empty((q, k), dtype=torch.float32, device="cuda")
    r1 = torch.empty((q, k), dtype=torch.int64, device="cuda")
    ix.topk_resident(k, s1.data_ptr(), r1.data_ptr())
    torch.cuda.synchronize()
    pairs = set()
    for sp in SPLITS:
        with monkeypatch.context() as m:
            m.setenv("KAKVEDA_B200_CODE_SPLITS", sp)
            s2, r2 = torch.empty_like(s1), torch.empty_like(r1)
            ix.topk_resident_seed(k, s2.data_ptr(), r2.data_ptr())
            kth = s2[:, k - 1].contiguous()
            torch.cuda.synchronize()
            ix.raise_thresholds(kth.data_ptr(), q)
            ix.topk_resident_finish(k, s2.data_ptr(), r2.data_ptr())
            torch.cuda.synchronize()
        assert ix.layout()["pool_pages_used"] == 0
        assert r1.cpu().numpy().tobytes() == r2.cpu().numpy().tobytes(), sp
        assert s1.cpu().numpy().tobytes() == s2.cpu().numpy().tobytes(), sp
        pairs.add(ix.layout()["pairs_passed_bound"])
    assert len(pairs) == 1, pairs
