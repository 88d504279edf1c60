"""Row deletion timing: `python profiles/run_delete.py [ROWS] [QUERIES] [ROUNDS]`.

Bench corpus (synth.CORPUS_SEED, default 10M rows) and the bench query batch (synth.QUERY_SEED, default 100k queries),
top-16.  Reports, in one process:
  * the first (full) finalize against delete + finalize of 1 % of the rows spread at random (a statistics-only
    refresh), and then of a further 10 % clustered in text order: a run of consecutive rows in text order, extended to
    whole duplicate groups;
  * per state (nothing deleted, 1 % random, 1 % + 10 % clustered): the CUDA-event kernel times
    (kv_index_last_kernel_ms: bound pass 0, seed scan, selection / bound pass 1, scan, merge) and the (query, chunk)
    pairs scored (kv_index_layout counter [9]), median over the rounds after one warm-up round.
"""
import subprocess
import sys
import time
from pathlib import Path

import numpy as np
import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
from kakveda_b200 import GfkbIndex, synth
from kakveda_b200.similarity import text_order

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

buf, off = synth.signatures_packed(synth.CORPUS_SEED, 0, n)
ix = GfkbIndex()
fb = ix.vocab.featurize_packed(buf, off, 0, grow=True)
ix.add_features(fb)
t0 = time.perf_counter()
ix.finalize()
t_full = time.perf_counter() - t0
print(f"full finalize {t_full:.3f} s (kind {ix.last_finalize_kind})", flush=True)

# 10 % clustered in text order, whole duplicate groups: a run of the text order, extended while the texts repeat
order = text_order(fb)
ip, ids = fb.indptr, fb.ids
row = lambda r: ids[ip[r]:ip[r + 1]].tobytes()
start = len(order) // 3
end = start + n // 10
while end < len(order) and row(order[end]) == row(order[end - 1]):
    end += 1
while start > 0 and row(order[start - 1]) == row(order[start]):
    start -= 1
clustered = np.sort(order[start:end].astype(np.int64))
fb.close()
rng = np.random.default_rng(2024)
spread = rng.choice(np.setdiff1d(np.arange(n), clustered), size=n // 100, replace=False)

qbuf, qoff = synth.signatures_packed(synth.QUERY_SEED, 0, q, dup_of_seed=synth.CORPUS_SEED, dup_rows=n)
qfb = ix.vocab.featurize_packed(qbuf, qoff, 0, grow=False)
print("rows", n, "queries", q, "chunks", ix.layout()["chunks"], flush=True)


def measure(name):
    ix.upload_queries(qfb)  # a deletion drops the resident batch
    runs = []
    for _ in range(rounds + 1):
        ix.topk_resident_host(q, k)
        runs.append((ix.last_kernel_ms(), ix.layout()["pairs_scored"]))
    ms = np.median(np.array([m for m, _ in runs[1:]]), axis=0)
    print(f"{name:22s} live {ix.n_live_rows:9d}  kernel ms [bound0 seed select/bound1 scan merge] "
          f"{np.round(ms, 3).tolist()} sum {ms.sum():.2f}  pairs_scored {runs[-1][1]}", flush=True)


measure("nothing deleted")
for name, rows in (("1% random", spread), ("+10% clustered", clustered)):
    t0 = time.perf_counter()
    ix.delete_rows(rows)
    ix.finalize()
    dt = time.perf_counter() - t0
    print(f"delete {len(rows)} rows ({name}) + finalize {dt:.3f} s (kind {ix.last_finalize_kind}) "
          f"against the full finalize {t_full:.3f} s", flush=True)
    measure(name)
