"""The bound kernel evaluates a tile's second-class features through a dictionary of 256 GEMM columns.  A tile whose
queries list more distinct second-class features than that leaves the least listed ones to the epilogue, which adds
them per block from the bitmaps.  This checks such a tile: the numerators must never fall below the exact union bound,
and the layout counter of listings left out of the dictionary must be non-zero."""
import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def test_bound_numerators_with_dictionary_overflow(built_lib):
    import scipy.sparse as sp

    from kakveda_b200 import GfkbIndex, _capi, synth
    from kakveda_b200.similarity import ArrayBatch

    lib = _capi.load()
    assert lib.kv_device_count() > 0, "GPU tests need a CUDA device"
    n, q, per_q = 60_000, 128, 20
    ix = GfkbIndex()
    buf, off = synth.signatures_packed(synth.CORPUS_SEED, 0, n)
    fb = ix.vocab.featurize_packed(buf, off, 0, grow=True)
    ip, ids, tf = fb.indptr.copy(), fb.ids.copy().astype(np.int64), fb.tf.copy().astype(np.float64)
    ix.add_features(fb)
    fb.close()
    ix.finalize()
    V = len(ix.vocab)
    # one 128-query tile, each query 20 distinct features drawn from the document-frequency ranks just past the 256
    # frequent ones: the tile lists several hundred distinct second-class features
    df = np.bincount(ids, minlength=V)
    ranked = np.argsort(-np.where(df == n, -1, df), kind="stable")
    pool = ranked[300:1200]
    rng = np.random.default_rng(7)
    qids = np.concatenate([np.sort(rng.choice(pool, per_q, replace=False)) for _ in range(q)]).astype(np.int64)
    qip = np.arange(0, q * per_q + 1, per_q, dtype=np.int64)
    qtf = rng.integers(1, 3, size=len(qids)).astype(np.int64)
    ix.upload_queries(ArrayBatch(qip, qids, qtf))
    assert ix.layout()["f2_outside_dictionary"] > 0
    nch = (n + 31) // 32
    got = np.zeros((q, nch), dtype=np.float32)
    slot_query = np.zeros(q, dtype=np.int32)
    _capi.check(lib.kv_debug_bound_numerators(ix._h, 16, got.ctypes.data_as(C.POINTER(C.c_float)),
                                              slot_query.ctypes.data_as(C.POINTER(C.c_int32))))
    # NumPy union bound: chunk unions (32 rows per chunk of the scan layout) with the largest tf, times tf_q a(t)
    rowof = np.repeat(np.arange(n), np.diff(ip))
    a = (np.log((n + 2) / (df.astype(np.float64) + 2)) + 1) ** 2
    # the scan layout's row order, as the index built it (row_at_pos of kv_debug_bound_codes)
    row_at_pos = np.zeros(n, dtype=np.int32)
    _capi.check(lib.kv_debug_bound_codes(ix._h, 16, np.zeros((q, nch), dtype=np.uint8).ctypes.data_as(C.POINTER(C.c_uint8)),
                                         np.zeros(q, dtype=np.int32).ctypes.data_as(C.POINTER(C.c_int32)), None, None,
                                         None, row_at_pos.ctypes.data_as(C.POINTER(C.c_int32))))
    pos_of = np.empty(n, dtype=np.int64)
    pos_of[row_at_pos] = np.arange(n)
    key = (pos_of[rowof] // 32) * V + ids
    o = np.lexsort((tf, key))
    ks = key[o]
    last = np.r_[ks[1:] != ks[:-1], True]
    U = sp.csr_matrix((tf[o][last], (ks[last] // V, ks[last] % V)), shape=(nch, V))
    qrow = np.repeat(np.arange(q), np.diff(qip))
    W = sp.csc_matrix((qtf * a[qids], (qids, qrow)), shape=(V, q))
    want = np.asarray((U @ W).todense()).T[slot_query]
    assert want.max() > 0
    ratio = (got + 1e-3) / (want + 1e-3)
    assert ratio.min() >= 1.0 - 1e-6, "a bound below the exact union bound: pruning would drop rows"
