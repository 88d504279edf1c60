"""The candidate scan's consumer loop (tfidf_scan_kernel): what the other GPU tests do not pin.

* records whose query masks hold 1, 2, 3 and 32 queries (batches of identical queries share every candidate chunk);
* a record where one query of the mask is null, or filtered out by its label, while its partners are scored;
* column blocks larger than a staging buffer (read in place) next to blocks that fit (staged by TMA), and entries held
  by every row of a chunk (summed once per warp) next to entries held by some rows (handed over by shuffle);
* one text stored 200 times across several chunks, k in {1, 16, 32}: every copy ties, the answer is the k lowest row
  ids, and a full list must turn the later copies away before the lock without turning away a row that belongs.
Every case is compared bit for bit with the exhaustive scan (KAKVEDA_B200_NO_PRUNE=1) under forced split counts
(KAKVEDA_B200_CODE_SPLITS), and with the float64 oracle (oracle/tfidf_oracle.py)."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

N_BASE = 20000          # 625 chunks: the pruned path runs
SPLITS = ("1", "3", "8")
COPIES = 200
DUP_TEXT = "intent_tags:task:triage | prompt_hint:restart the ingest worker after the quota error zuzu keke | tools:shell | env_keys:zone"
WORDS = ["".join(chr(97 + (i // 26 ** j) % 26) for j in range(3)) + "q" for i in range(4000)]


def long_text(rng, n_words):
    return "intent_tags: | prompt_hint:" + " ".join(rng.choice(WORDS, size=n_words, replace=False)) + " | tools:shell | env_keys:zone"


@pytest.fixture(scope="module")
def world(built_lib):
    """The synthetic corpus plus 200 copies of one text (scattered, so several chunks hold runs of them) and 96 long
    texts of distinct words (three chunks whose column blocks exceed a staging buffer)."""
    from kakveda_b200 import GfkbIndex, _capi, synth

    assert _capi.load().kv_device_count() > 0, "GPU tests need a CUDA device"
    rng = np.random.default_rng(11)
    corpus = list(synth.corpus(N_BASE))
    long_rows = [long_text(rng, 24) for _ in range(96)]  # 24 words: under the 64 features a scanned query may hold
    corpus += long_rows
    for pos in sorted(rng.choice(len(corpus), size=COPIES, replace=False).tolist()):
        corpus.insert(pos, DUP_TEXT)
    ix = GfkbIndex()
    ix.add_texts(corpus)
    ix.finalize()
    return ix, corpus, long_rows


def run_env(monkeypatch, env, fn):
    with monkeypatch.context() as m:
        for key, v in env.items():
            m.setenv(key, v)
        return fn()


def check(monkeypatch, ix, corpus, queries, k, labels=None, row_labels=None):
    """Pruned path under every forced split count == exhaustive scan, bit for bit; then the float64 oracle."""
    from oracle import tfidf_oracle as O

    fn = lambda: ix.topk(queries, k, labels=labels)
    want_s, want_r = run_env(monkeypatch, {"KAKVEDA_B200_NO_PRUNE": "1"}, fn)
    for sp in SPLITS:
        s, r = run_env(monkeypatch, {"KAKVEDA_B200_CODE_SPLITS": sp}, fn)
        assert ix.layout()["pairs_passed_bound"] > 0, "the pruned path did not run"
        assert r.tobytes() == want_r.tobytes(), sp
        assert s.tobytes() == want_s.tobytes(), sp
    exact = O.score_matrix_closed_form(queries, corpus)
    for i in range(len(queries)):
        ok = np.ones(len(corpus), bool) if labels is None or labels[i] < 0 else row_labels == labels[i]
        got = want_r[i][want_r[i] >= 0]
        assert len(got) == min(k, int(ok.sum())) and len(set(got.tolist())) == len(got) and np.all(ok[got]), i
        np.testing.assert_allclose(want_s[i][: len(got)], exact[i, got], rtol=1e-5, atol=1e-7)
        rest = ok.copy()
        rest[got] = False
        if rest.any() and len(got):
            assert exact[i, rest].max() <= exact[i, got].min() * (1 + 2e-5) + 1e-7, i
    return want_s, want_r


@pytest.mark.parametrize("k", [1, 16, 32])
def test_masks_of_1_2_3_and_32_queries(world, monkeypatch, k):
    from kakveda_b200 import synth

    ix, corpus, long_rows = world
    base = synth.queries(8, N_BASE)
    queries = [base[0]] * 32 + [base[1]] * 3 + [base[2]] * 2 + [base[3]] + [long_rows[5]] * 3 + [long_rows[40]]
    s, r = check(monkeypatch, ix, corpus, queries, k)
    for a, b in ((0, 32), (32, 35), (35, 37), (38, 41)):  # identical queries, identical answers
        assert all(r[i].tobytes() == r[a].tobytes() and s[i].tobytes() == s[a].tobytes() for i in range(a, b))


@pytest.mark.parametrize("k", [1, 16])
def test_null_or_filtered_partner_in_a_record(world, monkeypatch, k):
    """Identical queries share their records.  One of them is null (no known feature: answered outside the scan), one
    is filtered to a label that no row near the text carries, the others are scored."""
    from kakveda_b200 import synth

    ix, corpus, _ = world
    rng = np.random.default_rng(3)
    row_labels = rng.integers(0, 4, size=len(corpus)).astype(np.int32)
    near = np.flatnonzero(np.array([t == DUP_TEXT for t in corpus]))
    row_labels[near] = 1
    ix.set_row_labels(row_labels)
    base = synth.queries(4, N_BASE)
    queries = [DUP_TEXT, DUP_TEXT, "xqzzy", DUP_TEXT, base[0], base[0], base[0]]
    labels = np.array([1, 2, -1, -1, -1, 3, 0], np.int32)
    try:
        check(monkeypatch, ix, corpus, queries, k, labels=labels, row_labels=row_labels)
    finally:
        ix.set_row_labels(np.zeros(len(corpus), np.int32))


@pytest.mark.parametrize("k", [1, 16, 32])
def test_blocks_larger_than_a_staging_buffer(world, monkeypatch, k):
    """Queries built from the long rows: their candidates are the long rows' chunks (over 256 entries, read in place)
    and ordinary chunks sharing the frame words (staged)."""
    ix, corpus, long_rows = world
    rng = np.random.default_rng(7)
    queries = []
    for j in (0, 33, 70, 95):
        words = long_rows[j].split("prompt_hint:")[1].split(" | ")[0].split()
        queries.append("intent_tags: | prompt_hint:" + " ".join(words[:18] + rng.choice(WORDS, 4).tolist()) + " | tools:shell | env_keys:zone")
    queries.append(long_rows[12])
    check(monkeypatch, ix, corpus, queries, k)


@pytest.mark.parametrize("k", [1, 16, 32])
def test_200_copies_return_the_k_lowest_rows(world, monkeypatch, k):
    ix, corpus, _ = world
    copies = np.flatnonzero(np.array([t == DUP_TEXT for t in corpus]))
    assert len(copies) == COPIES and len(set((copies // 32).tolist())) > 8
    s, r = check(monkeypatch, ix, corpus, [DUP_TEXT, DUP_TEXT, DUP_TEXT + " zuzu"], k)
    for i in range(3):
        assert r[i].tolist() == copies[:k].tolist(), i
    assert np.all(s[:2] == s[0, 0]) and abs(float(s[0, 0]) - 1.0) < 1e-6
    # distinct mode: the copies are one group, so one of them (the lowest row) leads and other groups follow
    groups = np.arange(len(corpus), dtype=np.int32)
    groups[copies] = int(copies[0])
    ix.set_row_groups(groups)
    try:
        fn = lambda: ix.topk([DUP_TEXT, DUP_TEXT], k, distinct=True)
        want_s, want_r = run_env(monkeypatch, {"KAKVEDA_B200_NO_PRUNE": "1"}, fn)
        for sp in SPLITS:
            ds, dr = run_env(monkeypatch, {"KAKVEDA_B200_CODE_SPLITS": sp}, fn)
            assert dr.tobytes() == want_r.tobytes() and ds.tobytes() == want_s.tobytes(), sp
        assert want_r[0, 0] == copies[0] and not np.any(np.isin(want_r[:, 1:], copies))
    finally:
        ix.set_row_groups(np.arange(len(corpus), dtype=np.int32))
