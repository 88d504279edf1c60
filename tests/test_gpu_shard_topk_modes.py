"""Label-filtered and distinct top-k and row deletion on the row-sharded GFKB (dist.py), on ONE GPU through the loopback
collectives of test_gpu_shard_loopback.py.

* ``kv_merge_topk_distinct_device_on`` (``merge_packed_distinct_on_device``) against a NumPy merge: W = 1..8 and 64
  packed lists, groups spread over several lists, equal scores interleaved by row, short and empty lists; singleton
  groups give ``kv_merge_topk_device_on``'s bits; every invalid input is refused.
* ``topk_packed`` / ``topk_resident`` with ``labels=`` and ``distinct=True`` in rows mode (index and text order) and
  queries mode: identical on every rank and equal to ``GfkbIndex.topk_features`` over the whole corpus, bit for bit for
  the regular queries; filtered results inside the label-masked float64 oracle's contract (``check_topk_device``).
* The peer threshold pushes (``kv_debug_thresholds_link``) for filtered and distinct batches; on one index the
  two-phase top-k of a distinct batch runs only with ``KV_DISTINCT_MERGED_SEEDS``.
* ``delete_rows``: statistics-only refresh on every shard, and every search equals a single index with the same
  deletions.  Errors raise the same exception on every rank.
"""
import ctypes as C
import threading

import numpy as np
import pytest

torch = pytest.importorskip("torch")
import torch.distributed as tdist  # noqa: E402

from test_gpu_scale_oracle import RTOL32, check_topk_device  # noqa: E402
from test_gpu_shard_loopback import (TIMEOUT, Corpus, _close, _copy, _link, build_sharded, crafted_texts, lib,  # noqa: E402,F401
                                     loopback, merge_numpy, run_ranks, synth_corpus, synth_texts)
from test_gpu_shard_range import _check_range, _flags, _np, _single_range  # noqa: E402

gpu = pytest.mark.gpu


# ---------------------------------------------------------------------------------------------------------------------
# The distinct merge against NumPy
# ---------------------------------------------------------------------------------------------------------------------

def merge_distinct_numpy(gs, gr, groups, k):
    """(score desc, row asc) merge of W lists keeping the first entry of each group: [W,Q,k] -> [Q,k]."""
    w, q, kin = gs.shape
    out_s = np.full((q, k), -np.inf, np.float32)
    out_r = np.full((q, k), -1, np.int64)
    for i in range(q):
        cand = sorted((-float(gs[l, i, j]), int(gr[l, i, j])) for l in range(w) for j in range(kin) if gr[l, i, j] >= 0)
        taken, j = set(), 0
        for ns, r in cand:
            if j == k:
                break
            if groups[r] in taken:
                continue
            taken.add(groups[r])
            out_s[i, j], out_r[i, j] = -ns, r
            j += 1
    return out_s, out_r


def _packed(gs, gr):
    from kakveda_b200.dist import packed_layout, packed_views

    w, q, k = gs.shape
    buf = torch.zeros((w, packed_layout(q, k)[1]), dtype=torch.uint8, device="cuda")
    for l in range(w):
        s_v, r_v = packed_views(buf[l], q, k)
        s_v.copy_(torch.from_numpy(gs[l]))
        r_v.copy_(torch.from_numpy(gr[l]))
    return buf


def _lists(rng, w, q, k, groups, empty=False):
    """Per query W lists of disjoint rows, each of distinct groups, ordered (score desc, row asc); some short."""
    n = len(groups)
    gs = np.full((w, q, k), -np.inf, np.float32)
    gr = np.full((w, q, k), -1, np.int64)
    if empty:
        return gs, gr
    levels = np.array([1.0, 0.75, 0.5, 0.5000001, 0.25, 0.0], np.float32)
    for i in range(q):
        rows = rng.permutation(n)
        per = n // w
        for l in range(w):
            m = int(rng.integers(0, k + 1)) if i % 3 == 0 else k
            cand = rows[l * per:(l + 1) * per]
            _, first = np.unique(groups[cand], return_index=True)
            rw = cand[np.sort(first)][:m]
            sc = levels[rng.integers(0, len(levels), len(rw))]
            o = np.lexsort((rw, -sc))
            gs[l, i, :len(rw)], gr[l, i, :len(rw)] = sc[o], rw[o]
    return gs, gr


@gpu
@pytest.mark.parametrize("k", [1, 16, 32])
def test_distinct_merge_against_numpy(lib, k):
    from kakveda_b200.dist import merge_packed_distinct_on_device, merge_packed_on_device

    rng = np.random.default_rng(100 + k)
    q = 37
    for w in list(range(1, 9)) + [64]:
        n = 6 * w * k + 64
        groups = rng.integers(0, max(2, n // 5), n).astype(np.int32)   # ~5 rows a group, spread over the lists
        gdev = torch.from_numpy(groups).cuda()
        for empty in (True, False):
            gs, gr = _lists(rng, w, q, k, groups, empty)
            buf = _packed(gs, gr)
            s, r = merge_packed_distinct_on_device(0, buf, q, k, gdev)
            es, er = merge_distinct_numpy(gs, gr, groups, k)
            np.testing.assert_array_equal(r.cpu().numpy(), er, err_msg=f"W={w} k={k} empty={empty}")
            np.testing.assert_array_equal(s.cpu().numpy(), es, err_msg=f"W={w} k={k} empty={empty}")
        # singleton groups: exactly the plain K5
        single = torch.arange(n, dtype=torch.int32, device="cuda")
        s, r = merge_packed_distinct_on_device(0, buf, q, k, single)
        ps, pr = merge_packed_on_device(0, buf, q, k)
        torch.cuda.synchronize()
        np.testing.assert_array_equal(r.cpu().numpy(), pr.cpu().numpy())
        np.testing.assert_array_equal(s.cpu().numpy().view(np.uint32), ps.cpu().numpy().view(np.uint32))
    es, er = merge_numpy(gs, gr, k)
    np.testing.assert_array_equal(pr.cpu().numpy(), er)


@gpu
def test_distinct_merge_refuses_invalid_input(lib):
    from kakveda_b200 import _capi
    from kakveda_b200.dist import merge_packed_distinct_on_device, packed_layout

    rng = np.random.default_rng(7)
    w, q, k = 3, 20, 8
    n = 500
    groups = rng.integers(0, 80, n).astype(np.int32)
    gs, gr = _lists(rng, w, q, k, groups)
    gdev = torch.from_numpy(groups).cuda()
    buf = _packed(gs, gr)
    off_r, total = packed_layout(q, k)
    out_s = torch.empty((q, k), dtype=torch.float32, device="cuda")
    out_r = torch.empty((q, k), dtype=torch.int64, device="cuda")
    host = np.zeros(total * w, np.uint8)
    base = buf.data_ptr()
    P = C.c_void_p

    def call(si=base, ri=base + off_r, nl=w, nq=q, kk=k, ss=total // 4, sr=total // 8, g=gdev.data_ptr(), ng=n,
             so=out_s.data_ptr(), ro=out_r.data_ptr()):
        return _capi.load().kv_merge_topk_distinct_device_on(0, P(si), P(ri), nl, nq, kk, ss, sr, P(g), ng, P(so), P(ro), None)

    assert call() == _capi.KV_OK
    for kw in (dict(kk=0), dict(kk=33), dict(nl=0), dict(nl=2049), dict(ss=q * k - 1), dict(sr=q * k - 1), dict(ng=-1),
               dict(si=host.ctypes.data), dict(ri=host.ctypes.data), dict(g=host.ctypes.data), dict(so=0),
               dict(ri=base + off_r + 4), dict(si=base + 2), dict(ro=out_r.data_ptr() + 4), dict(g=gdev.data_ptr() + 2)):
        assert call(**kw) == _capi.KV_ERR_INVALID, kw
    # a row past the group table, and a table one row too short for the largest row: refused, nothing read past it
    for bad_rows in (n, n + 1_000_000_000):
        gr2 = gr.copy()
        gr2[1, 5, 0] = bad_rows
        with pytest.raises(ValueError, match="group table"):
            merge_packed_distinct_on_device(0, _packed(gs, gr2), q, k, gdev)
    with pytest.raises(ValueError, match="group table"):   # the head of a list is read at the first step
        merge_packed_distinct_on_device(0, buf, q, k, gdev[:int(gr[1, 5, 0])])
    s, r = merge_packed_distinct_on_device(0, buf, q, k, gdev[:int(gr.max()) + 1])   # the exact size is enough
    np.testing.assert_array_equal(r.cpu().numpy(), merge_distinct_numpy(gs, gr, groups, k)[1])
    assert call(nq=0) == _capi.KV_OK


# ---------------------------------------------------------------------------------------------------------------------
# Filtered and distinct top-k
# ---------------------------------------------------------------------------------------------------------------------

CASES = [("rows", "index", 1), ("rows", "index", 2), ("rows", "index", 3), ("rows", "index", 8), ("rows", "text", 2),
         ("rows", "text", 3), ("rows", "text", 8), ("queries", "index", 2), ("queries", "index", 3)]
IDS = [f"{m}-{o}-W{w}" for m, o, w in CASES]


def _modes(c, world, order, mode):
    """Row labels (4 labels, label 9 on rows of the last shard only), query labels (-1, a label no row has, 9 and the
    others) and row groups (neighbouring text classes)."""
    from kakveda_b200.dist import shard_bounds, shard_rows_by_text

    rng = np.random.default_rng(world * 11 + (order == "text"))
    row_labels = rng.integers(0, 4, c.n).astype(np.int32)
    if mode == "rows" and order == "text" and world > 1:
        fb = c.one.vocab.featurize_packed(c.data, c.off, c.mode, grow=False)
        try:
            last = shard_rows_by_text(fb, world, world - 1)
        finally:
            fb.close()
    else:
        lo, hi = shard_bounds(c.n, max(world, 2), max(world, 2) - 1)
        last = np.arange(lo, hi)
    row_labels[last[::7]] = 9
    qlab = rng.choice(np.array([-1, 0, 1, 2, 3, 9, 17], np.int32), len(c.queries)).astype(np.int32)
    groups = (c.text_id // 8).astype(np.int32)
    return row_labels, qlab, groups


def _masked_blocks(c, row_labels, qlab):
    lab = torch.as_tensor(row_labels, device="cuda")
    out = []
    for lo, hi, o in c.blocks:
        ql = torch.as_tensor(qlab[lo:hi], device="cuda")[:, None]
        out.append((lo, hi, torch.where((ql < 0) | (ql == lab[None, :]), o, -np.inf)))
    return out


def _single(c, k, labels=None, groups=None, distinct=False):
    c.one.set_row_labels(None if labels is None else c._row_labels)
    c.one.set_row_groups(groups)
    try:
        return c.one.topk_features(c.qfb, k, labels, distinct)
    finally:
        c.one.set_row_labels(None)
        c.one.set_row_groups(None)


def _same_as_single(c, name, s, r, single, regular):
    s1, r1 = single
    bad = np.flatnonzero(regular & ((r != r1).any(1) | (s.view(np.uint32) != s1.view(np.uint32)).any(1)))
    assert len(bad) == 0, (f"{name}: {len(bad)} regular queries differ from the single index, first {bad[0]}: sharded "
                           f"{r[bad[0]].tolist()} {s[bad[0]].tolist()} single {r1[bad[0]].tolist()} {s1[bad[0]].tolist()}")


def _distinct_ok(name, s, r, groups):
    for q in range(r.shape[0]):
        g = groups[r[q][r[q] >= 0]]
        assert len(np.unique(g)) == len(g), f"{name}, query {q}: two rows of one group {r[q].tolist()}"


def _check_modes(c, name, res, row_labels, qlab, groups, k):
    """res: {(path, what): (s, r)} of rank 0; what in filtered / distinct / both / singleton / plain."""
    regular = _flags(c) != 2
    c._row_labels = row_labels
    blocks = _masked_blocks(c, row_labels, qlab)
    want = {"filtered": _single(c, k, qlab), "distinct": _single(c, k, None, groups, True),
            "both": _single(c, k, qlab, groups, True)}
    for (path, what), (s, r) in res.items():
        label = f"{name} {path} {what}"
        if what == "singleton":
            ps, pr = res[path, "plain"]
            np.testing.assert_array_equal(r, pr, err_msg=label)
            np.testing.assert_array_equal(s.view(np.uint32), ps.view(np.uint32), err_msg=label)
            continue
        if what == "plain":
            c.check(label, s, r, k)
            continue
        _same_as_single(c, label, s, r, want[what], regular)
        if what in ("filtered", "both"):
            assert np.all(r[qlab == 17] == -1), label
            lab_ok = (r < 0) | (qlab[:, None] < 0) | (row_labels[np.clip(r, 0, c.n - 1)] == qlab[:, None])
            assert lab_ok.all(), f"{label}: a row of another label"
        if what == "filtered":
            for lo, hi, o in blocks:
                check_topk_device(s[lo:hi], r[lo:hi], o, k, RTOL32, first=lo)
        if what in ("distinct", "both"):
            _distinct_ok(label, s, r, groups)


def _run_modes(c, world, order, mode, k, row_labels, qlab, groups):
    build = build_sharded(world, order, mode, c)

    def fn(rk, g):
        sh = build(rk, g)
        try:
            res = {}
            sh.set_row_labels(row_labels)
            sh.set_row_groups(groups)
            for what, kw in (("plain", {}), ("filtered", dict(labels=qlab)), ("distinct", dict(distinct=True)),
                             ("both", dict(labels=qlab, distinct=True))):
                s, r = sh.topk_packed(c.qdata, c.qoff, k, c.qmode, **kw)
                res["packed", what] = (_copy(s), _copy(r))
                qfb = sh.vocab.featurize(c.queries, grow=False)
                try:
                    sh.set_resident(qfb)
                    s, r = sh.topk_resident(k, **kw)
                    res["resident", what] = (s.cpu().numpy(), r.cpu().numpy())
                finally:
                    qfb.close()
            sh.set_row_groups(np.arange(c.n, dtype=np.int32))
            s, r = sh.topk_packed(c.qdata, c.qoff, k, c.qmode, distinct=True)
            res["packed", "singleton"] = (_copy(s), _copy(r))
            return res
        finally:
            _close([sh])

    out = run_ranks(world, fn)
    for rk in range(1, world):
        for key, (s, r) in out[0].items():
            np.testing.assert_array_equal(out[rk][key][1], r, err_msg=f"rank {rk} {key}")
            np.testing.assert_array_equal(out[rk][key][0], s, err_msg=f"rank {rk} {key}")
    return out[0]


@gpu
@pytest.mark.parametrize("mode,order,world", CASES, ids=IDS)
def test_filtered_and_distinct_topk(synth_corpus, loopback, mode, order, world):
    """Filtered, distinct and filtered-distinct top-k through ``topk_packed`` (sliced preparation when W > 1) and
    ``set_resident`` + ``topk_resident``; singleton groups reproduce the non-distinct bits."""
    c = synth_corpus
    row_labels, qlab, groups = _modes(c, world, order, mode)
    for k in (16,) if world in (2, 3) else (1, 32):
        res = _run_modes(c, world, order, mode, k, row_labels, qlab, groups)
        _check_modes(c, f"{mode} {order} W={world} k={k}", res, row_labels, qlab, groups, k)


CRAFTED = [("index", 3), ("text", 3)]


@gpu
@pytest.mark.parametrize("order,world", CRAFTED, ids=[f"{o}-W{w}" for o, w in CRAFTED])
def test_distinct_groups_across_shard_boundaries(lib, loopback, order, world):
    """Groups are the text classes of the crafted corpus, whose copies straddle the shard boundaries (the k-th
    position inside a group), combined with labels."""
    c = Corpus(*crafted_texts(6000, world, order))
    rng = np.random.default_rng(3)
    row_labels = rng.integers(0, 3, c.n).astype(np.int32)
    qlab = rng.choice(np.array([-1, 0, 1, 2], np.int32), len(c.queries)).astype(np.int32)
    groups = c.text_id.astype(np.int32)
    for k in (1, 5, 16):
        res = _run_modes(c, world, order, "rows", k, row_labels, qlab, groups)
        _check_modes(c, f"crafted {order} W={world} k={k}", res, row_labels, qlab, groups, k)
        if k > 1:   # the copies across the boundaries collapse
            assert (res["packed", "distinct"][1] != res["packed", "plain"][1]).any()


# ---------------------------------------------------------------------------------------------------------------------
# Peer threshold pushes
# ---------------------------------------------------------------------------------------------------------------------

PEER_CASES = [("index", 3), ("text", 8)]


@gpu
@pytest.mark.parametrize("order,world", PEER_CASES, ids=[f"{o}-W{w}" for o, w in PEER_CASES])
def test_peer_pushes_filtered_and_distinct(synth_corpus, lib, loopback, monkeypatch, order, world):
    """Filtered and distinct batches with every shard pushing its thresholds into the others' arrays, with the finish
    phases concurrent and one after another: exact results, and the pushes never add scanned pairs."""
    from kakveda_b200 import _capi

    c = synth_corpus
    monkeypatch.setenv("KAKVEDA_B200_NO_PEER_THR", "1")
    row_labels, qlab, groups = _modes(c, world, order, "rows")
    build = build_sharded(world, order, "rows", c)
    k = 16
    shards = [None] * world
    turn = threading.Condition()
    state = {"next": 0}
    kinds = {"filtered": dict(labels=qlab), "distinct": dict(distinct=True)}

    def serial_finish(r, ix):
        inner = ix.topk_resident_finish

        def finish(*a):
            with turn:
                assert turn.wait_for(lambda: state["next"] == r, timeout=TIMEOUT), f"rank {r}: no turn to finish"
            try:
                inner(*a)
            finally:
                with turn:
                    state["next"] += 1
                    turn.notify_all()
        return finish

    def fn(r, g):
        sh = shards[r] = build(r, g)
        sh.set_row_labels(row_labels)
        sh.set_row_groups(groups)
        buf = C.create_string_buffer(64)
        _capi.check(lib.kv_index_thresholds_export(sh.index._h, len(c.queries), buf))
        tdist.barrier(group=g)
        res, pairs = {}, {}
        for linked in (False, True):
            _link(lib, shards, r, len(c.queries)) if linked else _capi.check(lib.kv_debug_thresholds_link(sh.index._h, None, 0, 0))
            for serial in ((False, True) if linked else (False,)):
                for kind, kw in kinds.items():
                    qfb = sh.vocab.featurize(c.queries, grow=False)
                    try:
                        sh.set_resident(qfb)
                        if serial:
                            with turn:
                                if r == 0:
                                    state["next"] = 0
                            tdist.barrier(group=g)
                            sh.index.topk_resident_finish = serial_finish(r, sh.index)
                        try:
                            s, rr = sh.topk_resident(k, **kw)
                        finally:
                            sh.index.__dict__.pop("topk_resident_finish", None)
                        res[linked, serial, kind] = (s.cpu().numpy(), rr.cpu().numpy())
                        pairs[linked, serial, kind] = sh.index.layout()["pairs_scored"]
                    finally:
                        qfb.close()
        tdist.barrier(group=g)
        _capi.check(lib.kv_debug_thresholds_link(sh.index._h, None, 0, 0))
        tdist.barrier(group=g)
        return res, pairs

    try:
        out = run_ranks(world, fn)
    finally:
        _close(shards)
    regular = _flags(c) != 2
    c._row_labels = row_labels
    want = {"filtered": _single(c, k, qlab), "distinct": _single(c, k, None, groups, True)}
    for (linked, serial, kind), (s, rr) in out[0][0].items():
        _same_as_single(c, f"{kind} linked {linked} serial {serial}", s, rr, want[kind], regular)
    total = {key: sum(o[1][key] for o in out) for key in out[0][1]}
    print(f"\npairs scored over {world} shards: {total}")
    for kind in kinds:
        assert total[True, False, kind] <= total[False, False, kind], total
        assert total[True, True, kind] <= total[False, False, kind], total


# ---------------------------------------------------------------------------------------------------------------------
# Deletion
# ---------------------------------------------------------------------------------------------------------------------

DELETE_CASES = [("rows", "index", 3), ("rows", "text", 3), ("rows", "index", 1), ("queries", "index", 2)]


@gpu
@pytest.mark.parametrize("mode,order,world", DELETE_CASES, ids=[f"{m}-{o}-W{w}" for m, o, w in DELETE_CASES])
def test_delete_rows_equals_single_index(lib, loopback, mode, order, world):
    """1 % of the rows at random, a range of the text order and every row of one shard are deleted on the sharded
    GFKB and on a single index: every shard refreshes its statistics only, and top-k (plain, filtered, distinct),
    threshold search and self-join equal the single index's; no deleted row comes back.  Rows out of range raise on
    every rank and change nothing."""
    from kakveda_b200.dist import shard_bounds, shard_rows_by_text

    texts, queries = synth_texts(30_000, 300)
    c = Corpus(texts, queries)
    n = c.n
    rng = np.random.default_rng(21)
    fb = c.one.vocab.featurize_packed(c.data, c.off, c.mode, grow=False)
    try:
        text_range = shard_rows_by_text(fb, 10, 4)
        whole = shard_rows_by_text(fb, world, world - 1) if order == "text" and world > 1 else None
    finally:
        fb.close()
    if whole is None:
        lo, hi = shard_bounds(n, max(world, 2), max(world, 2) - 1)
        whole = np.arange(lo, hi)
    dele = np.concatenate([rng.choice(n, n // 100, replace=False), text_range, whole])
    row_labels = rng.integers(0, 4, n).astype(np.int32)
    qlab = rng.choice(np.array([-1, 0, 1, 2, 3], np.int32), len(queries)).astype(np.int32)
    groups = (c.text_id // 8).astype(np.int32)
    k, thr = 16, 0.5
    build = build_sharded(world, order, mode, c)

    def fn(r, g):
        sh = build(r, g)
        try:
            sh.set_row_labels(row_labels)
            sh.set_row_groups(groups)
            errs = []
            for bad in ([n], [-1], [0, n + 5]):
                try:
                    sh.delete_rows(bad)
                except ValueError as e:
                    errs.append(str(e))
            assert sh.n_live_rows == n and not sh.deleted_mask().any()
            sh.delete_rows(dele)
            kind = sh.index.last_finalize_kind
            res = {}
            for what, kw in (("plain", {}), ("filtered", dict(labels=qlab)), ("distinct", dict(distinct=True))):
                s, rr = sh.topk_packed(c.qdata, c.qoff, k, c.qmode, **kw)
                res[what] = (_copy(s), _copy(rr))
            rng_res = _np(sh.range_packed(c.qdata, c.qoff, thr, c.qmode))
            join = _np(sh.selfjoin_range(0.8, block=12000))
            return errs, kind, res, rng_res, join, sh.n_live_rows, sh.deleted_mask()
        finally:
            _close([sh])

    out = run_ranks(world, fn)
    dead = np.zeros(n, bool)
    dead[dele] = True
    for rk, (errs, kind, res, rng_res, join, live, mask) in enumerate(out):
        assert len(errs) == 3 and all("outside the corpus" in e for e in errs), (rk, errs)
        assert kind == 2, f"rank {rk}: finalize kind {kind}"
        assert live == n - dead.sum() and np.array_equal(mask, dead), rk
        for what in res:
            np.testing.assert_array_equal(res[what][1], out[0][2][what][1], err_msg=f"rank {rk} {what}")
    c.one.delete_rows(np.flatnonzero(dead))
    c.one.finalize()
    regular = _flags(c) != 2
    c._row_labels = row_labels
    want = {"plain": _single(c, k), "filtered": _single(c, k, qlab), "distinct": _single(c, k, None, groups, True)}
    _, _, res, rng_res, join, _, _ = out[0]
    for what, (s, rr) in res.items():
        assert not dead[rr[rr >= 0]].any(), f"{what}: a deleted row came back"
        _same_as_single(c, f"deleted {what}", s, rr, want[what], regular)
    single = _np(c.one.range_features(c.qfb, thr))
    assert not dead[rng_res[1]].any()
    for q in np.flatnonzero(regular):
        a, b, e, f = rng_res[0][q], rng_res[0][q + 1], single[0][q], single[0][q + 1]
        np.testing.assert_array_equal(rng_res[1][a:b], single[1][e:f], err_msg=f"range query {q}")
        np.testing.assert_array_equal(rng_res[2][a:b].view(np.uint32), single[2][e:f].view(np.uint32))
    sj = _np(c.one.selfjoin_range(0.8))
    assert not dead[join[1]].any()
    np.testing.assert_array_equal(join[0], sj[0])
    np.testing.assert_array_equal(join[1], sj[1])
    np.testing.assert_array_equal(join[2].view(np.uint32), sj[2].view(np.uint32))


# ---------------------------------------------------------------------------------------------------------------------
# Errors
# ---------------------------------------------------------------------------------------------------------------------

@gpu
@pytest.mark.parametrize("mode,world", [("rows", 3), ("queries", 2)])
def test_mode_errors_raise_on_every_rank(synth_corpus, loopback, mode, world):
    """Distinct without ``set_row_groups``, labels of the wrong length or without ``set_row_labels``: the same
    ValueError on every rank, from the top-k and (labels) from the threshold search, and the sharded index still
    answers both afterwards."""
    c = synth_corpus
    build = build_sharded(world, "index", mode, c)
    nq, thr = len(c.queries), 0.6

    def fn(r, g):
        sh = build(r, g)
        topk = lambda **kw: sh.topk_packed(c.qdata, c.qoff, 8, c.qmode, **kw)
        search = lambda **kw: sh.range_packed(c.qdata, c.qoff, thr, c.qmode, **kw)
        try:
            msgs = []
            for call, kw in ((topk, dict(distinct=True)), (topk, dict(labels=np.full(nq, -1, np.int32))),
                             (search, dict(labels=np.full(nq, -1, np.int32)))):
                with pytest.raises(ValueError) as e:
                    call(**kw)
                msgs.append(str(e.value))
            sh.set_row_labels(np.zeros(c.n, np.int32))
            for lab in (np.zeros(nq - 1, np.int32), np.full(nq, -2, np.int32)):
                for call in (topk, search):
                    with pytest.raises(ValueError) as e:
                        call(labels=lab)
                    msgs.append(str(e.value))
            with pytest.raises(ValueError):
                sh.set_row_groups(np.zeros(c.n - 1, np.int32))
            s, rr = topk()
            return msgs, _copy(s), _copy(rr), _np(search())
        finally:
            _close([sh])

    out = run_ranks(world, fn)
    for o in out[1:]:
        assert o[0] == out[0][0]
    msgs = out[0][0]
    assert "set_row_groups" in msgs[0] and "set_row_labels" in msgs[1]
    assert msgs[1] == msgs[2] and msgs[3] == msgs[4] and msgs[5] == msgs[6], msgs
    c.check(f"{mode} W={world} after errors", out[0][1], out[0][2], 8)
    _check_range(c, f"{mode} W={world} after errors", out[0][3], thr, _single_range(c, thr))


# ---------------------------------------------------------------------------------------------------------------------
# The two-phase top-k of a distinct batch on one index
# ---------------------------------------------------------------------------------------------------------------------

@gpu
def test_two_phase_distinct_needs_merged_seeds(lib):
    """Plain distinct mode keeps refusing the two-phase top-k; with ``merged_seeds`` (KV_DISTINCT_MERGED_SEEDS) the seed
    list, raised to its own slot k-1 (the merge of one list), then the finish give the one-phase result bit for bit."""
    texts, queries = synth_texts(20_000, 60)
    c = Corpus(texts, queries)
    ix, k, nq = c.one, 8, len(queries)
    ix.set_row_groups((c.text_id // 8).astype(np.int32))
    try:
        want = ix.topk_features(c.qfb, k, distinct=True)
        ds = torch.full((nq, k), float("-inf"), dtype=torch.float32, device="cuda")
        dr = torch.full((nq, k), -1, dtype=torch.int64, device="cuda")
        torch.cuda.synchronize()
        ix.upload_queries(c.qfb)
        ix.set_distinct(True)
        with pytest.raises(ValueError, match="KV_DISTINCT_MERGED_SEEDS"):
            ix.topk_resident_seed(k, ds.data_ptr(), dr.data_ptr())
        with pytest.raises(ValueError, match="KV_DISTINCT_MERGED_SEEDS"):
            ix.topk_resident_finish(k, ds.data_ptr(), dr.data_ptr())
        ix.set_distinct(True, merged_seeds=True)
        ix.topk_resident_seed(k, ds.data_ptr(), dr.data_ptr())
        kth = ds[:, k - 1].contiguous()
        ix.raise_thresholds(kth.data_ptr(), nq)
        ix.topk_resident_finish(k, ds.data_ptr(), dr.data_ptr())
        assert dr.cpu().numpy().tobytes() == want[1].tobytes() and ds.cpu().numpy().tobytes() == want[0].tobytes()
        ix.upload_queries(c.qfb)   # the next upload switches both off
        ix.topk_resident(k, ds.data_ptr(), dr.data_ptr())
        assert dr.cpu().numpy().tobytes() == ix.topk_features(c.qfb, k)[1].tobytes()
    finally:
        ix.set_row_groups(None)
        ix.close()
