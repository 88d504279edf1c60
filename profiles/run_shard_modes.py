"""Sharded top-k modes timing: `python profiles/run_shard_modes.py [--merge] [--w1 ROWS]`.

--merge: kv_merge_topk_distinct_device_on (``merge_packed_distinct_on_device``) next to kv_merge_topk_device_on
(``merge_packed_on_device``) on the same packed [W, total] all-gather buffer: 100k queries, W = 2, 4, 8 lists of k = 16,
disjoint rows, coarse scores so that lists tie often, groups of 4 consecutive row ids (each group spans the lists).
CUDA events around the call on torch's stream, one warm-up and five timed calls, median reported.  The distinct call
includes what it does to report a row without a group: a 4-byte memset and copy back, and the wait for the stream.

--w1 ROWS: ShardedGfkb at W = 1 against GfkbIndex over the same ROWS-row bench corpus and the same 16,384 bench
queries, filtered (4 row labels, query labels -1..3) and distinct (groups of 4 rows): the CUDA-event kernel times
(kv_index_last_kernel_ms, bound + scans + merge) of both, median of three runs.  Same kernels, so they should match.

Loopback runs at W > 1 share one GPU and are not multi-GPU times; this script does not report them.
The card name and power limit are printed first, read in the same run."""
import subprocess
import sys
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
from kakveda_b200 import synth  # noqa: E402
from kakveda_b200.dist import merge_packed_distinct_on_device, merge_packed_on_device, packed_layout, packed_views  # noqa: E402

try:
    power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
except (OSError, subprocess.SubprocessError):
    power = "unknown"
print("card", torch.cuda.get_device_name(0), "power limit", power, flush=True)


def packed_lists(w, q, k, seed=0):
    """[W, total] uint8: per query W lists of k disjoint rows ordered (score desc, row asc), built on the device."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    _, total = packed_layout(q, k)
    buf = torch.empty((w, total), dtype=torch.uint8, device="cuda")
    for l in range(w):
        s, r = packed_views(buf[l], q, k)
        lev = torch.randint(0, 64, (q, k), device="cuda", generator=g)
        row = (torch.randint(0, 1 << 20, (q, k), device="cuda", generator=g) * w + l)
        key = torch.sort(((63 - lev) << 40) | row, dim=1).values       # (score desc, row asc)
        s.copy_((63 - (key >> 40)).to(torch.float32) / 64)
        r.copy_(key & ((1 << 40) - 1))
    return buf


def timed(fn, reps=5):
    fn()
    ms = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        ms.append(e0.elapsed_time(e1))
    return float(np.median(ms))


def merge_only():
    q, k = 100_000, 16
    for w in (2, 4, 8):
        buf = packed_lists(w, q, k, seed=w)
        groups = (torch.arange((1 << 20) * w, device="cuda") // 4).to(torch.int32)
        t_plain = timed(lambda: merge_packed_on_device(0, buf, q, k))
        t_dist = timed(lambda: merge_packed_distinct_on_device(0, buf, q, k, groups))
        print(f"merge W={w} queries={q} k={k}: kv_merge_topk_device_on {t_plain:.3f} ms, "
              f"kv_merge_topk_distinct_device_on {t_dist:.3f} ms", flush=True)


def w1(n_rows):
    from kakveda_b200 import GfkbIndex
    from kakveda_b200.dist import ShardedGfkb

    data, off = synth.signatures_packed(synth.CORPUS_SEED, 0, n_rows)
    qdata, qoff = synth.signatures_packed(synth.QUERY_SEED, 0, 16384, dup_of_seed=synth.CORPUS_SEED, dup_rows=n_rows)
    rng = np.random.default_rng(0)
    row_labels = rng.integers(0, 4, n_rows).astype(np.int32)
    qlab = rng.integers(-1, 4, len(qoff) - 1).astype(np.int32)
    groups = (np.arange(n_rows) // 4).astype(np.int32)
    sh = ShardedGfkb(device=0)
    sh.build_packed(data, off, 0)
    sh.set_row_labels(row_labels)
    sh.set_row_groups(groups)
    one = GfkbIndex()
    fb = one.vocab.featurize_packed(data, off, 0, grow=True)
    one.add_features(fb)
    fb.close()
    one.finalize()
    one.set_row_labels(row_labels)
    one.set_row_groups(groups)
    qfb = one.vocab.featurize_packed(qdata, qoff, 0, grow=False)
    sqfb = sh.vocab.featurize_packed(qdata, qoff, 0, grow=False)
    k = 16
    for name, kw in (("plain", {}), ("filtered", dict(labels=qlab)), ("distinct", dict(distinct=True)),
                     ("filtered+distinct", dict(labels=qlab, distinct=True))):
        t_sh, t_one = [], []
        for it in range(4):
            sh.set_resident(sqfb)
            s, r = sh.topk_resident(k, **kw)
            torch.cuda.synchronize()
            if it:
                t_sh.append(sum(sh.index.last_kernel_ms()))
            s1, r1 = one.topk_features(qfb, k, kw.get("labels"), kw.get("distinct", False))
            if it:
                t_one.append(sum(one.last_kernel_ms()))
        same = np.array_equal(r.cpu().numpy(), r1) and np.array_equal(s.cpu().numpy().view(np.uint32), s1.view(np.uint32))
        print(f"W=1 {name} rows={n_rows} queries={len(qoff) - 1} k={k}: ShardedGfkb kernels {np.median(t_sh):.2f} ms, "
              f"GfkbIndex kernels {np.median(t_one):.2f} ms, identical results {same}", flush=True)
    qfb.close()
    sqfb.close()
    sh.index.close()
    one.close()


if "--merge" in sys.argv:
    merge_only()
if "--w1" in sys.argv:
    w1(int(sys.argv[sys.argv.index("--w1") + 1]))
