"""The bound kernel's R accumulator is fixed point per query (uint32 in units of 1 / s_q, s_q chosen from an upper bound
xmax_q of what R sums).  A wrapped or rounded-down sum would lower a bound and pruning would drop rows, so the
numerators are checked where xmax_q is largest: regular queries whose term frequencies sit at the top of the range
the regular path admits (largest weight tf_q a(t) just under the fp16 limit of classify_queries)."""
import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def test_bound_numerators_at_largest_query_tf(built_lib):
    import scipy.sparse as sp

    from kakveda_b200 import GfkbIndex, _capi, synth
    from kakveda_b200.similarity import ArrayBatch

    lib = _capi.load()
    assert lib.kv_device_count() > 0, "GPU tests need a CUDA device"
    n, q = 60_000, 256
    ix = GfkbIndex()
    buf, off = synth.signatures_packed(synth.CORPUS_SEED, 0, n)
    fb = ix.vocab.featurize_packed(buf, off, 0, grow=True)
    ip, ids, tf = fb.indptr.copy(), fb.ids.copy().astype(np.int64), fb.tf.copy().astype(np.float64)
    ix.add_features(fb)
    fb.close()
    ix.finalize()
    V = len(ix.vocab)
    qbuf, qoff = synth.signatures_packed(synth.QUERY_SEED, 0, q, dup_of_seed=synth.CORPUS_SEED, dup_rows=n)
    qfb = ix.vocab.featurize_packed(qbuf, qoff, 0, grow=False)
    qip, qids = qfb.indptr.copy(), qfb.ids.copy().astype(np.int64)
    qtf0 = qfb.tf.copy().astype(np.int64)
    qoov = qfb.oov.copy()
    qfb.close()
    # every query's tf scaled so that its largest weight tf_q a(t) lands just under the regular path's limit of 60000
    amax = (np.log(n + 2) + 1) ** 2
    qrow = np.repeat(np.arange(q), np.diff(qip))
    tfmax_q = np.maximum.reduceat(qtf0, qip[:-1]) if len(qtf0) else np.zeros(q, dtype=np.int64)
    mult = np.maximum(1, np.floor(59_000.0 / (amax * np.maximum(tfmax_q, 1)))).astype(np.int64)
    qtf = qtf0 * mult[qrow]
    assert (qtf.max() * amax > 50_000) and (np.maximum.reduceat(qtf, qip[:-1]) * amax <= 60_000).all()
    ix.upload_queries(ArrayBatch(qip, qids, qtf, qoov))
    nch = (n + 31) // 32
    got = np.zeros((q, nch), dtype=np.float32)
    slot_query = np.zeros(q, dtype=np.int32)
    _capi.check(lib.kv_debug_bound_numerators(ix._h, 16, got.ctypes.data_as(C.POINTER(C.c_float)),
                                              slot_query.ctypes.data_as(C.POINTER(C.c_int32))))
    # NumPy union bound: chunk unions (32 rows per chunk of the scan layout) with the largest tf, times tf_q a(t)
    rowof = np.repeat(np.arange(n), np.diff(ip))
    df = np.bincount(ids, minlength=V).astype(np.float64)
    a = (np.log((n + 2) / (df + 2)) + 1) ** 2
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
    known = qids < V
    W = sp.csc_matrix((qtf[known] * a[qids[known]], (qids[known], qrow[known])), shape=(V, q))
    want = np.asarray((U @ W).todense()).T[slot_query]
    assert want.max() > 4e4
    ratio = (got + 1e-3) / (want + 1e-3)
    assert ratio.min() >= 1.0 - 1e-6, "a bound below the exact union bound: pruning would drop rows"
    assert np.quantile(ratio, 0.999) <= 1.002 and ratio.max() < 3.0, (np.quantile(ratio, [0.5, 0.999]), ratio.max())
