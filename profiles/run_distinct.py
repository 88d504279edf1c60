"""Distinct top-k timing: `python profiles/run_distinct.py [ROWS] [QUERIES] [ROUNDS]`.

Bench corpus (synth.CORPUS_SEED, default 10M rows, 30 % of them copies of other rows) and the bench query batch
(synth.QUERY_SEED, default 100k queries) resident.  Per round, in one process and alternating, top-16:
  * ``off``         -- distinct mode off (the bench path);
  * ``singleton``   -- distinct mode with one group per row (same result bits as ``off``);
  * ``duplicates``  -- distinct mode with one group per duplicate class (rows with an identical feature sequence,
                       i.e. synth's copies of one text).
Reports the CUDA-event kernel times (kv_index_last_kernel_ms: bound pass 0, seed scan, selection / bound pass 1, scan,
merge) and the (query, chunk) pairs scored, median over the rounds after one warm-up round, and checks that the
singleton run returns the bits of the ``off`` run."""
import subprocess
import sys
from pathlib import Path

import numpy as np
import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
from kakveda_b200 import GfkbIndex, synth

n = int(sys.argv[1]) if len(sys.argv) > 1 else 10_000_000
q = int(sys.argv[2]) if len(sys.argv) > 2 else 100_000
rounds = int(sys.argv[3]) if len(sys.argv) > 3 else 5
k = 16

try:
    power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
except (OSError, subprocess.SubprocessError):
    power = "unknown"
print("card", torch.cuda.get_device_name(0), "power limit", power, flush=True)


def duplicate_classes(fb, block: int = 1 << 20) -> np.ndarray:
    """int32 group per row: rows with the same (feature id, tf) sequence share one (a 64-bit hash of the sequence,
    computed in blocks of rows; a collision would only merge two classes)."""
    ip = np.asarray(fb.indptr, dtype=np.int64)
    n = len(ip) - 1
    row_h = np.zeros(n, dtype=np.uint64)
    with np.errstate(over="ignore"):
        for a in range(0, n, block):
            b = min(n, a + block)
            lo, hi = int(ip[a]), int(ip[b])
            lens = np.diff(ip[a:b + 1])
            ids = np.asarray(fb.ids[lo:hi], dtype=np.uint64)
            tf = np.asarray(fb.tf[lo:hi], dtype=np.uint64)
            pos = (np.arange(lo, hi, dtype=np.int64) - np.repeat(ip[a:b], lens)).astype(np.uint64)
            h = (ids * np.uint64(0x9E3779B97F4A7C15) + tf + np.uint64(1)) * (pos * np.uint64(0xBF58476D1CE4E5B9) + np.uint64(0x94D049BB133111EB))
            nz = lens > 0
            part = np.zeros(b - a, dtype=np.uint64)
            part[nz] = np.add.reduceat(h, (ip[a:b] - lo)[nz])
            row_h[a:b] = part ^ (lens.astype(np.uint64) * np.uint64(0xD6E8FEB86659FD93))
    _, inv = np.unique(row_h, return_inverse=True)
    return inv.astype(np.int32)


buf, off = synth.signatures_packed(synth.CORPUS_SEED, 0, n)
ix = GfkbIndex()
fb = ix.vocab.featurize_packed(buf, off, 0, grow=True)
ix.add_features(fb)
dup = duplicate_classes(fb)
fb.close()
ix.finalize()
qbuf, qoff = synth.signatures_packed(synth.QUERY_SEED, 0, q, dup_of_seed=synth.CORPUS_SEED, dup_rows=n)
qfb = ix.vocab.featurize_packed(qbuf, qoff, 0, grow=False)
single = np.arange(n, dtype=np.int32)
print("rows", n, "queries", q, "chunks", ix.layout()["chunks"], "duplicate classes", int(dup.max()) + 1, flush=True)

variants = [("off", None), ("singleton", single), ("duplicates", dup)]
results = {name: [] for name, _ in variants}
bits = {}
for r in range(rounds + 1):
    for name, groups in variants:
        ix.upload_queries(qfb)
        if groups is not None:
            ix.set_row_groups(groups)   # an upload of n int32 and one kernel, outside the timed kernels
            ix.set_distinct(True)
        s, rows = ix.topk_resident_host(q, k)
        results[name].append((ix.last_kernel_ms(), ix.layout()["pairs_scored"]))
        bits[name] = (s.tobytes(), rows.tobytes())
assert bits["singleton"] == bits["off"], "singleton groups must give the non-distinct result bits"

for name, runs in results.items():
    runs = runs[1:]
    ms = np.median(np.array([m for m, _ in runs]), axis=0)
    pairs = runs[-1][1]
    print(f"{name:12s} kernel ms [bound0 seed select/bound1 scan merge] {np.round(ms, 3).tolist()} "
          f"sum {ms.sum():.2f}  pairs_scored {pairs}", flush=True)
