"""Device featuriser (featurize_device.cu) and the text upload (kv_query_upload_text): the device CSR must equal the
host featuriser's bit for bit, and the resident batch built on the device must equal kv_query_upload's, so that every
result and pruning counter is unchanged."""
import ctypes as C
import json
import os
from contextlib import contextmanager
from pathlib import Path

import numpy as np
import pytest

from kakveda_b200 import GfkbIndex, _capi, synth
from kakveda_b200.similarity import DEVICE_FEATURIZE_MIN_QUERIES, Vocabulary, pack_texts

pytestmark = pytest.mark.gpu

GOLDEN = Path(__file__).resolve().parent / "golden"
COUNTERS = ("pairs_passed_bound", "records_written", "pairs_scored", "records_scanned", "f2_outside_dictionary")


@contextmanager
def featurize_path(which):
    old = os.environ.get("KAKVEDA_B200_FEATURIZE")
    os.environ["KAKVEDA_B200_FEATURIZE"] = which
    try:
        yield
    finally:
        if old is None:
            del os.environ["KAKVEDA_B200_FEATURIZE"]
        else:
            os.environ["KAKVEDA_B200_FEATURIZE"] = old


def _strings(x, out):
    if isinstance(x, str):
        out.append(x)
    elif isinstance(x, dict):
        for v in x.values():
            _strings(v, out)
    elif isinstance(x, list):
        for v in x:
            _strings(v, out)
    return out


def golden_texts():
    texts = []
    for name in ("fixture54.json", "edge_cases.json", "signature_text.json", "service_upsert.json", "service_warn.json",
                 "purge.json", "ref_test_similarity.json", "corpus_fit.json"):
        texts += _strings(json.loads((GOLDEN / name).read_text(encoding="utf-8")), [])
    for name in ("synthetic_small.json", "synthetic_cfg1.json"):
        g = json.loads((GOLDEN / name).read_text(encoding="utf-8"))
        texts += synth.corpus(g["n"]) + synth.queries(g["q"], g["n"])
    return texts


def assert_same_csr(dev, host):
    assert dev.n == host.n
    np.testing.assert_array_equal(dev.indptr, host.indptr)
    np.testing.assert_array_equal(dev.ids, host.ids)
    np.testing.assert_array_equal(dev.tf, host.tf)
    np.testing.assert_array_equal(np.asarray(dev.oov).view(np.uint64), np.asarray(host.oov).view(np.uint64))


def check_packed(vocab, data, offsets, mode):
    host = vocab.featurize_packed(data, offsets, mode, grow=False)
    dev = vocab.featurize_packed_device(data, offsets, mode)
    assert_same_csr(dev, host)
    return host


def check_texts(vocab, texts):
    return check_packed(vocab, *pack_texts(texts))


def test_csr_golden_texts(built_lib):
    texts = golden_texts()
    assert len(texts) > 1000
    v = Vocabulary()
    v.featurize(texts[::2], grow=True)  # half the texts: the other half brings out-of-vocabulary features
    check_texts(v, texts)
    v.featurize(texts, grow=True)
    check_texts(v, texts)
    v.close()


def test_csr_bench_queries(built_lib):
    v = Vocabulary()
    buf, off = synth.signatures_packed(synth.CORPUS_SEED, 0, 100_000)
    v.featurize_packed(buf, off, 0, grow=True)
    qbuf, qoff = synth.signatures_packed(synth.QUERY_SEED, 0, 200_000, dup_of_seed=synth.CORPUS_SEED, dup_rows=100_000)
    fb = check_packed(v, qbuf, qoff, _capi.KV_TEXT_RAW_ASCII)
    assert fb.oov.max() > 0 and len(fb.ids) > 200_000
    v.close()


def edge_texts():
    t = ["", "a", "a b c", "ab", "A", "AB ab Ab aB", "x1 1x __ _a a_ 12 1_2", "!!! ... ,,, ;;", "   ", "\t\n\r",
         "Hello, World! HELLO world", "a-b c.d e/f gh", "under_score UNDER_SCORE 0123456789"]
    for n in (7, 8, 9, 15, 16, 17, 31, 32, 33):  # Murmur blocks are 16 bytes, the tail splits at 8
        w = ("abcdefghij" * 4)[:n]
        t.append(f"{w} {w.upper()} {w[::-1]} {w}")
        t.append(f"xy {w} {w[:n - 1]}z")
    t.append("rep " * 70_000)  # one token repeated more than 65,536 times
    t.append(" ".join(f"w{i % 300}" for i in range(2000)))  # over 512 occurrences, repeats in a long document
    t.append(" ".join(f"tok{i}" for i in range(7000))[: 64 * 1024])  # 64 KiB
    return t


def test_csr_edge_cases(built_lib):
    texts = edge_texts()
    v = Vocabulary()
    v.featurize(texts[::3], grow=True)
    check_texts(v, texts)
    # pre-tokenised (0x1F) documents beside raw ones: UTF-8 tokens and empty tokens
    mixed = texts[:20] + ["Größe straße ÉCOLE école", "naïve café naïve", "éé aé", "日本語 テキスト 日本語"]
    data, offsets, mode = pack_texts(mixed)
    assert mode == _capi.KV_TEXT_MIXED
    v.featurize(mixed, grow=True)
    check_packed(v, data, offsets, mode)
    pre = b"\x1f" + b"\x1f".join([b"a", b"", b"bb", b"\xc3\xa9t\xc3\xa9", b"", b"", b"bb", b"a"]) + b"\x1f"
    raw = b"plain text here"
    for docs in ([pre], [pre, raw, pre, b"", b"\x1f", b"\x1f\x1f"]):
        data = b"".join(docs)
        offsets = np.cumsum([0] + [len(d) for d in docs]).astype(np.int64)
        check_packed(v, data, offsets, _capi.KV_TEXT_MIXED)
    check_packed(v, b"a\x1fbb\x1f\x1fccc", np.array([0, 10], np.int64), _capi.KV_TEXT_TOKENS)
    v.close()


@pytest.mark.parametrize("n_docs", [0, 1, 31, 33])
def test_csr_batch_sizes(built_lib, n_docs):
    texts = synth.queries(n_docs, 200) if n_docs else []
    v = Vocabulary()
    v.featurize(synth.corpus(200), grow=True)
    check_texts(v, texts)
    v.close()


def test_csr_all_oov_and_empty_vocab(built_lib):
    texts = synth.queries(40, 100)
    empty = Vocabulary()
    fb = check_texts(empty, texts)
    assert len(fb.ids) == 0 and fb.oov.min() > 0
    other = Vocabulary()
    other.featurize(["completely different words only"], grow=True)
    fb = check_texts(other, texts)
    assert len(fb.ids) == 0
    empty.close()
    other.close()


def _raw_bad_doc(fn, *args):
    bad = C.c_int64(-1)
    out = C.c_void_p()
    rc = fn(*args, C.byref(out), C.byref(bad))
    return rc, bad.value


def test_raw_mode_non_ascii(built_lib):
    lib = _capi.load()
    v = Vocabulary()
    v.featurize(["some words"], grow=True)
    docs = [b"ok text", b"fine", b"", b"bad \xc3\xa9 byte", b"ok", b"\xff also bad"]
    data = b"".join(docs)
    offsets = np.cumsum([0] + [len(d) for d in docs]).astype(np.int64)
    op = offsets.ctypes.data_as(C.POINTER(C.c_int64))
    rc_h, bad_h = _raw_bad_doc(lib.kv_featurize, v._h, data, op, len(docs), _capi.KV_TEXT_RAW_ASCII, 0, 0)
    rc_d, bad_d = _raw_bad_doc(lib.kv_featurize_device, v.mirror(0), v._h, data, op, len(docs), _capi.KV_TEXT_RAW_ASCII)
    assert rc_h == rc_d == _capi.KV_ERR_NONASCII and bad_h == bad_d == 3
    with pytest.raises(ValueError):
        v.featurize_packed_device(data, offsets, _capi.KV_TEXT_RAW_ASCII)
    # in mixed mode a raw document is checked too, a pre-tokenised one is not
    docs = [b"\x1f\xc3\xa9t\xc3\xa9", b"ok", b"caf\xc3\xa9"]
    data = b"".join(docs)
    offsets = np.cumsum([0] + [len(d) for d in docs]).astype(np.int64)
    op = offsets.ctypes.data_as(C.POINTER(C.c_int64))
    rc_h, bad_h = _raw_bad_doc(lib.kv_featurize, v._h, data, op, len(docs), _capi.KV_TEXT_MIXED, 0, 0)
    rc_d, bad_d = _raw_bad_doc(lib.kv_featurize_device, v.mirror(0), v._h, data, op, len(docs), _capi.KV_TEXT_MIXED)
    assert rc_h == rc_d == _capi.KV_ERR_NONASCII and bad_h == bad_d == 2
    with pytest.raises(ValueError):
        v.featurize_packed_device(b"abc", np.array([0, 3], np.int64), 7)
    v.close()


def test_mirror_sync(built_lib):
    v = Vocabulary()
    v.featurize(["alpha beta gamma"], grow=True)
    q = ["alpha beta delta epsilon", "zeta eta theta " * 3]
    fb = check_texts(v, q)
    n0 = len(fb.ids)
    for i in range(6):  # several growths of the device table (1024 slots at first)
        v.featurize([f"delta epsilon zeta eta theta {i}"] + synth.corpus(300 * (i + 1)), grow=True)
        fb = check_texts(v, q + synth.queries(50, 2000))
    assert len(fb.ids) > n0
    imported = Vocabulary.from_keys(v.export_keys())  # an import from a sidecar's keys
    check_texts(imported, q + synth.queries(50, 2000))
    v.close()
    imported.close()


# ---------------------------------------------------------------------------------------------------------------------
# resident batch identity
# ---------------------------------------------------------------------------------------------------------------------
N_ROWS = 40_000  # 625 chunks of 64 rows: the pruned path


def special_queries():
    base = synth.queries(1500, N_ROWS)
    irregular = [" ".join(base[10 * i:10 * i + 10]) for i in range(6)]  # > 64 features of the vocabulary
    huge_tf = [(base[i].split()[0] + " ") * 5000 + base[i] for i in range(4)]  # a huge tf
    null = ["qqqq zzzz unknown words", "", "!!!", "xyzzy " * 10]
    dup = [base[0], base[1], base[0], base[0]]
    words = base[2].split()
    prefixes = [" ".join(words[:n]) for n in range(1, len(words) + 1)]  # prefixes of one another, long shared prefixes
    shared = [" ".join(words) + f" tail{i}" for i in range(8)] + [" ".join(words[:-1]) + f" tail{i}" for i in range(8)]
    qs = base + irregular + huge_tf + null + dup + prefixes + shared
    rng = np.random.default_rng(7)
    return [qs[i] for i in rng.permutation(len(qs))]


def build_index(mode):
    ix = GfkbIndex()
    if mode:
        ix.set_mode(mode)
    buf, off = synth.signatures_packed(synth.CORPUS_SEED, 0, N_ROWS)
    fb = ix.vocab.featurize_packed(buf, off, 0, grow=True)
    ix.add_features(fb)
    fb.close()
    ix.finalize()
    assert ix.layout()["chunks"] >= 512
    return ix


@pytest.fixture(scope="module", params=[0, 2], ids=["default", "corpus_fit"])
def index(request, built_lib):
    ix = build_index(request.param)
    yield ix
    ix.close()


def upload_both(ix, texts):
    """(host, device) runner: each uploads the batch through its path and returns (qperm, flags)."""
    data, offsets, mode = pack_texts(texts)
    n = len(texts)

    def host():
        fb = ix.vocab.featurize_packed(data, offsets, mode, grow=False)
        ix.upload_queries(fb)
        fb.close()
        return ix.query_order(n)

    def device():
        ix.upload_text(data, offsets, mode)
        return ix.query_order(n)

    return host, device


def run_topk(ix, upload, n, k, labels=None, distinct=False, excl=None):
    order = upload()
    if labels is not None:
        ix.set_filter(labels)
    if excl is not None:
        ix.set_exclusions(excl)
    if distinct:
        ix.set_distinct(True)
    s, r = ix.topk_resident_host(n, k)
    lay = ix.layout()
    return order, s, r, {c: lay[c] for c in COUNTERS}


def assert_same_runs(a, b):
    (qa, fa), sa, ra, ca = a
    (qb, fb_), sb, rb, cb = b
    np.testing.assert_array_equal(qa, qb)
    np.testing.assert_array_equal(fa, fb_)
    np.testing.assert_array_equal(sa.view(np.uint32), sb.view(np.uint32))
    np.testing.assert_array_equal(ra, rb)
    assert ca == cb


def test_batch_identity(index):
    texts = special_queries()
    n = len(texts)
    host, device = upload_both(index, texts)
    flags = host()[1]
    assert (flags == 1).sum() >= 3 and (flags == 2).sum() >= 6  # null and irregular queries are present
    for k in (1, 16, 32):
        assert_same_runs(run_topk(index, host, n, k), run_topk(index, device, n, k))
    assert index.last_prepare_ms()[0] > 0


def test_batch_identity_filters(index):
    texts = special_queries()
    n = len(texts)
    host, device = upload_both(index, texts)
    rng = np.random.default_rng(3)
    index.set_row_labels(rng.integers(0, 5, index.n_rows).astype(np.int32))
    index.set_row_groups((np.arange(index.n_rows) // 3).astype(np.int32))
    labels = rng.integers(-1, 5, n).astype(np.int32)
    excl = rng.integers(-1, index.n_rows, n).astype(np.int64)
    for kw in (dict(labels=labels), dict(excl=excl), dict(distinct=True)):
        assert_same_runs(run_topk(index, host, n, 16, **kw), run_topk(index, device, n, 16, **kw))
    # threshold search, both fetches
    for dev_out in (False, True):
        got = []
        for up in (host, device):
            up()
            out = index._range_resident(n, 0.3, dev_out)
            got.append([np.asarray(x.cpu() if hasattr(x, "cpu") else x) for x in out])
        for x, y in zip(*got):
            np.testing.assert_array_equal(x.view(np.uint8), y.view(np.uint8))


def test_batch_identity_deleted_rows_and_new_ids(built_lib):
    ix = build_index(0)
    ix.delete_rows(np.arange(0, ix.n_rows, 7))
    ix.finalize()
    texts = special_queries()[:800]
    # features added to the vocabulary after finalize have ids >= the index's V
    ix.vocab.featurize(["brand new vocabulary words " + t for t in texts[:50]], grow=True)
    n = len(texts) + 1
    host, device = upload_both(ix, texts + ["brand new vocabulary words only"])
    for k in (1, 16):
        assert_same_runs(run_topk(ix, host, n, k), run_topk(ix, device, n, k))
    ix.close()


def test_entry_points_take_either_path(built_lib):
    ix = build_index(0)
    for n in (DEVICE_FEATURIZE_MIN_QUERIES - 1, DEVICE_FEATURIZE_MIN_QUERIES):
        texts = synth.queries(n, N_ROWS, seed=11)
        got = {}
        for path in ("host", "device"):
            with featurize_path(path):
                got[path] = (ix.topk(texts, 16), ix.range(texts, 0.4))
        (sh, rh), rg_h = got["host"]
        (sd, rd), rg_d = got["device"]
        np.testing.assert_array_equal(sh.view(np.uint32), sd.view(np.uint32))
        np.testing.assert_array_equal(rh, rd)
        for x, y in zip(rg_h, rg_d):
            np.testing.assert_array_equal(x, y)
    ix.close()


def test_sharded_topk_packed_world1(built_lib):
    from kakveda_b200.dist import ShardedGfkb

    sh = ShardedGfkb(device=0)
    buf, off = synth.signatures_packed(synth.CORPUS_SEED, 0, N_ROWS)
    sh.build_packed(buf, off, 0)
    for n in (100, DEVICE_FEATURIZE_MIN_QUERIES + 5):
        qbuf, qoff = synth.signatures_packed(synth.QUERY_SEED, 0, n, dup_of_seed=synth.CORPUS_SEED, dup_rows=N_ROWS)
        got = {}
        for path in ("host", "device"):
            with featurize_path(path):
                s, r = sh.topk_packed(qbuf, qoff, 16)
                got[path] = (s.copy(), r.copy(), dict(sh.last_e2e_ms))
        np.testing.assert_array_equal(got["host"][0].view(np.uint32), got["device"][0].view(np.uint32))
        np.testing.assert_array_equal(got["host"][1], got["device"][1])
        for key in ("featurize", "upload", "device_step", "read_back"):
            assert key in got["device"][2] and got["device"][2][key] >= 0
