"""Sharded threshold search timing: `python profiles/run_shard_range.py [--merge] [--loopback ROWS]`.

--merge: kv_merge_range_device_on alone (``merge_range_on_device`` on a packed [W, slot] buffer built on the device),
W = 2, 4, 8 runs over 100k queries and 10M / 50M / 244M records (the 244M of the headline K1b-R search), coarse scores
so that runs tie often.  CUDA events around the call on torch's stream, one warm-up and three timed rounds, median
reported.  Bytes model: the records are read once and written once (12 B each: int64 row + float32 score), every
run's indptr is read twice and the output indptr written once; the binary-search probes are not counted.  For
comparison, the radix ordering of range_order.cu on 10M of the same records through kv_debug_range_order (host clock:
it includes the H2D copy of the 16-byte records and the D2H copy of the ordered arrays).

--loopback ROWS: ShardedGfkb.range_packed over a ROWS-row bench corpus, 8,192 bench queries, W = 1, 4, 8 ranks as
threads on this ONE GPU (the loopback collectives of tests/test_gpu_shard_loopback.py).  The ranks share the device,
so this is not a multi-GPU time: it shows the cost of the exchange and merge next to the searches, nothing more.

The card name and power limit are printed first, read in the same run."""
import ctypes as C
import subprocess
import sys
import time
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
from kakveda_b200 import _capi, synth  # noqa: E402
from kakveda_b200.dist import merge_range_on_device, range_layout, range_views  # noqa: E402

try:
    power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
except (OSError, subprocess.SubprocessError):
    power = "unknown"
print("card", torch.cuda.get_device_name(0), "power limit", power, flush=True)
HBM_TBS = 3.35


def packed_runs(w, n_q, total, seed=0):
    """[W, slot] uint8 buffer of W ordered runs of total / W records each (disjoint rows), built on the device."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    per = total // w
    _, slot = range_layout(n_q, per)
    buf = torch.empty((w, slot), dtype=torch.uint8, device="cuda")
    for l in range(w):
        q = torch.randint(0, n_q, (per,), device="cuda", generator=g)
        lev = torch.randint(0, 256, (per,), device="cuda", generator=g)
        loc = torch.randperm(per, device="cuda", generator=g)
        key = torch.sort((q << 36) | ((255 - lev) << 28) | loc).values       # (query, score desc, row asc)
        del q, lev, loc
        ip, rows, sc = range_views(buf[l], n_q, per, per)
        qs = key >> 36
        ip.copy_(torch.searchsorted(qs, torch.arange(n_q + 1, device="cuda")))
        rows.copy_((key & ((1 << 28) - 1)) * w + l)
        sc.copy_((255 - ((key >> 28) & 255)).to(torch.float32) / 256 + 0.25)
        del key, qs
    return buf, np.full(w, per, np.int64)


def merge_only():
    n_q = 100_000
    for total in (10_000_000, 50_000_000, 244_000_000):
        for w in (2, 4, 8):
            buf, pairs = packed_runs(w, n_q, total)
            p = int(pairs.sum())
            ms = []
            for it in range(4):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                out = merge_range_on_device(0, buf, n_q, pairs)
                e1.record()
                torch.cuda.synchronize()
                if it:
                    ms.append(e0.elapsed_time(e1))
                del out
            t = float(np.median(ms))
            bytes_ = 2 * 12 * p + (2 * w + 1) * 8 * (n_q + 1)
            gbs = bytes_ / t / 1e6
            print(f"merge W={w} queries={n_q} records={p}: {t:.2f} ms  model {bytes_ / 1e9:.2f} GB  {gbs:.0f} GB/s  "
                  f"{100 * gbs / 1000 / HBM_TBS:.1f} % of {HBM_TBS} TB/s", flush=True)
            del buf
            torch.cuda.empty_cache()
    # the radix ordering of the same kind of records (host clock, copies included)
    total = 10_000_000
    buf, pairs = packed_runs(2, n_q, total)
    ip, rows, sc = merge_range_on_device(0, buf, n_q, pairs)
    q = torch.repeat_interleave(torch.arange(n_q, device="cuda", dtype=torch.int32), torch.diff(ip))
    perm = torch.randperm(len(rows), device="cuda")
    rec = torch.empty((len(rows), 4), dtype=torch.int32, device="cuda")
    rec[:, 0] = q[perm]
    rec[:, 1] = sc[perm].view(torch.int32)
    rec[:, 2:4] = rows[perm].view(torch.int32).view(-1, 2)
    rec = rec.cpu().numpy()
    n = len(rows)
    h_ip, h_rows, h_sc = np.empty(n_q + 1, np.int64), np.empty(n, np.int64), np.empty(n, np.float32)
    lib = _capi.load()
    ts = []
    for it in range(3):
        t0 = time.perf_counter()
        _capi.check(lib.kv_debug_range_order(0, 0, rec.ctypes.data_as(C.c_void_p), n, n_q, 0,
                                             h_ip.ctypes.data_as(C.POINTER(C.c_int64)), h_rows.ctypes.data_as(C.POINTER(C.c_int64)),
                                             h_sc.ctypes.data_as(C.POINTER(C.c_float)), None, None))
        ts.append(1e3 * (time.perf_counter() - t0))
    assert np.array_equal(h_rows, rows.cpu().numpy()) and np.array_equal(h_ip, ip.cpu().numpy())
    print(f"radix ordering (kv_debug_range_order, copies included) records={n}: median {np.median(ts[1:]):.1f} ms", flush=True)


def loopback(n_rows):
    sys.path.insert(0, str(ROOT / "tests"))
    import torch.distributed as tdist
    import test_gpu_shard_loopback as L
    from kakveda_b200.dist import ShardedGfkb

    for name, fn in (("is_available", lambda: True), ("is_initialized", lambda: True), ("get_world_size", L._lb_get_world_size),
                     ("barrier", L._lb_barrier), ("all_reduce", L._lb_all_reduce),
                     ("all_gather_into_tensor", L._lb_all_gather_into_tensor), ("all_gather_object", L._lb_all_gather_object)):
        setattr(tdist, name, fn)
    data, off = synth.signatures_packed(synth.CORPUS_SEED, 0, n_rows)
    qdata, qoff = synth.signatures_packed(synth.QUERY_SEED, 0, 8192, dup_of_seed=synth.CORPUS_SEED, dup_rows=n_rows)
    for world in (1, 4, 8):
        def fn(r, g):
            sh = ShardedGfkb(device=0, rank=r, world=world, group=g)
            t0 = time.perf_counter()
            sh.build_packed(data, off, 0)
            if r == 0:
                print(f"loopback W={world}: shards built in {time.perf_counter() - t0:.1f} s", flush=True)
            res = {}
            for thr in (0.6, 0.9):
                sh.range_packed(qdata, qoff, thr, device_out=True)      # warm-up
                ts = []
                for _ in range(3):
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    out = sh.range_packed(qdata, qoff, thr, device_out=True)
                    torch.cuda.synchronize()
                    ts.append(1e3 * (time.perf_counter() - t0))
                res[thr] = (float(np.median(ts)), int(out[0][-1]))
            sh.index.close()
            return res

        for thr, (ms, pairs) in L.run_ranks(world, fn, timeout=1800)[0].items():
            print(f"loopback W={world} rows={n_rows} queries=8192 threshold={thr}: {ms:.1f} ms (rank 0 wall clock) "
                  f"pairs={pairs}", flush=True)


if "--merge" in sys.argv:
    merge_only()
if "--loopback" in sys.argv:
    loopback(int(sys.argv[sys.argv.index("--loopback") + 1]))
