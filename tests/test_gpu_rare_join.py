"""The bound kernel's rare join on the two-choice rare tables (csrc/bound_kernel.cuh, csrc/block_builder.cuh).

1. A batch whose warps meet more than 32 bitmap hits in one 64-chunk block.  Each of N_HOST rows carries the words of
   PER_ROW crafted queries (32 words each, in this row only: rare), so those queries' rare lists all hit that row's
   block.  The crafted queries of one row are neighbours in the batch's text order, so a 32-query scan group holds at
   least PER_ROW / 2 of them and its warps meet at least 8 x PER_ROW / 2 = 64 hits in that block: two rounds or more.
   Bound codes, numerators, top-k and bound pass 1 are held to the float64 oracle and the exhaustive scan by
   test_gpu_bound_contract's checks, in both instantiations.
2. A persisted layout in the current format restores to identical results; a file of the previous format is refused.
"""
import numpy as np
import pytest

from test_gpu_bound_contract import (GENERIC, K, Case, bound_codes, check_contract, df_of, featurize)

gpu = pytest.mark.gpu

N_ROWS = 16_385
N_HOST = 12       # rows carrying crafted words
PER_ROW = 16      # crafted queries per such row
N_CRAFTED = N_HOST * PER_ROW


def crafted_corpus():
    from kakveda_b200 import synth

    texts = synth.corpus(N_ROWS)
    rng = np.random.default_rng(3)
    rows = rng.choice(N_ROWS, N_HOST, replace=False)
    words = [" ".join(f"zq{r:03d}x{s:02d}w{j:02d}" for j in range(32)) for r in range(N_HOST) for s in range(PER_ROW)]
    for i, r in enumerate(rows.tolist()):
        texts[r] += " " + " ".join(words[i * PER_ROW:(i + 1) * PER_ROW])
    # the crafted queries (their 32 unigrams and 31 bigrams are in one row only: rare), then ordinary ones
    qtexts = words + synth.queries(100, N_ROWS)
    return texts, qtexts


@pytest.fixture(scope="module")
def rare_case(built_lib):
    from kakveda_b200 import GfkbIndex, _capi
    from kakveda_b200.similarity import ArrayBatch

    assert _capi.load().kv_device_count() > 0, "GPU tests need a CUDA device"
    ix = GfkbIndex()
    texts, qtexts = crafted_corpus()
    rows = featurize(ix.vocab, texts, True)[:3]
    ix.add_features(ArrayBatch(*rows))
    ix.finalize()
    q = featurize(ix.vocab, qtexts, False)
    return Case("rare-rounds", ix, rows, N_ROWS, df_of(rows, len(ix.vocab)), 0, q), texts


@gpu
def test_crafted_queries_are_rare_and_co_located(rare_case):
    """The premise of the multi-round case: each crafted query's features are in one row, in neither dense class."""
    case, _ = rare_case
    ip, ids, _, _ = case.queries
    ix = case.ix
    rip, rids, _ = case.rows
    df = df_of(case.rows, len(ix.vocab))
    for i in range(0, N_CRAFTED, 17):
        f = ids[ip[i]:ip[i + 1]]
        assert len(f) >= 32 and (df[f] == 1).all()
        holders = {int(np.searchsorted(rip, p, side="right") - 1) for p in np.flatnonzero(np.isin(rids, f))}
        assert len(holders) == 1


@gpu
@pytest.mark.parametrize("variant", ["specialised", "generic"])
def test_rare_join_multiple_rounds(rare_case, monkeypatch, variant):
    case, _ = rare_case
    lay, _, sq, _ = check_contract(case, monkeypatch, {} if variant == "specialised" else GENERIC)
    assert lay["chunks"] == (N_ROWS + 31) // 32
    # sq[slot] = query: the crafted queries of a row share a 32-query scan group five or more at a time, so that
    # group's warps meet > 32 bitmap hits (8 per crafted query) in the row's block
    slot = np.empty(len(sq), np.int64)
    slot[sq] = np.arange(len(sq))
    for r in range(N_HOST):
        groups = slot[r * PER_ROW:(r + 1) * PER_ROW] // 32
        assert np.bincount(groups).max() >= 5, (r, groups)


@gpu
def test_layout_file_roundtrip_and_old_format_refused(rare_case, tmp_path):
    from kakveda_b200 import GfkbIndex
    from kakveda_b200.similarity import ArrayBatch

    case, _ = rare_case
    ix0 = case.ix
    case.upload()
    n_chunks = ix0.layout()["chunks"]
    want = bound_codes(ix0, case.n_q, n_chunks, N_ROWS)
    want_topk = ix0.topk_resident_host(case.n_q, K)
    path = tmp_path / "rare.layout"
    ix0.save_layout(path)
    assert path.read_bytes()[:8] == b"AKKVBLY3"

    ix = GfkbIndex(vocab=ix0.vocab)
    ix.add_features(ArrayBatch(*case.rows))
    assert ix.load_layout(path)
    ix.finalize()
    assert ix.last_finalize_kind == 2
    restored = Case("rare-restored", ix, case.rows, N_ROWS, df_of(case.rows, len(ix0.vocab)), 0, case.queries)
    restored.upload()
    got = bound_codes(ix, case.n_q, n_chunks, N_ROWS)
    for name, g, w in zip(("codes", "slot_query", "tcode", "q_terms", "chunk_minB", "row_at_pos"), got, want):
        assert g.tobytes() == w.tobytes(), name
    got_topk = ix.topk_resident_host(case.n_q, K)
    assert got_topk[0].tobytes() == want_topk[0].tobytes() and got_topk[1].tobytes() == want_topk[1].tobytes()

    old = tmp_path / "old.layout"
    old.write_bytes(b"AKKVBLY2" + path.read_bytes()[8:])
    ix2 = GfkbIndex(vocab=ix0.vocab)
    ix2.add_features(ArrayBatch(*case.rows))
    assert not ix2.load_layout(old)
    ix2.finalize()
    assert ix2.last_finalize_kind != 2
