"""Label-filtered search timing: `python profiles/run_filtered.py [ROWS] [QUERIES] [ROUNDS]`.

Bench corpus (synth.CORPUS_SEED, default 10M rows) labelled with 16 Zipf-weighted failure types plus one type on 0.1 %
of the rows (seeded RNG); the bench query batch (synth.QUERY_SEED, default 100k queries) stays resident.  Per round, in
one process and alternating: unfiltered top-16, top-16 with every query filtered to the most common type, top-16 with
every query filtered to the rare type, and the rare-type threshold search at theta = 0.8.  Reports the CUDA-event
kernel times (kv_index_last_kernel_ms: bound pass 0, seed scan, selection / bound pass 1, scan, merge) and the
(query, chunk) pairs scored, median over the rounds after one warm-up round."""
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

buf, off = synth.signatures_packed(synth.CORPUS_SEED, 0, n)
ix = GfkbIndex()
fb = ix.vocab.featurize_packed(buf, off, 0, grow=True)
ix.add_features(fb)
fb.close()
ix.finalize()
rng = np.random.default_rng(2024)
w = 1.0 / np.arange(1, 17)
labels = rng.choice(16, size=n, p=w / w.sum()).astype(np.int32)
RARE = 16
labels[rng.choice(n, size=max(1, n // 1000), replace=False)] = RARE
ix.set_row_labels(labels)
qbuf, qoff = synth.signatures_packed(synth.QUERY_SEED, 0, q, dup_of_seed=synth.CORPUS_SEED, dup_rows=n)
qfb = ix.vocab.featurize_packed(qbuf, qoff, 0, grow=False)
ix.upload_queries(qfb)
print("rows", n, "queries", q, "chunks", ix.layout()["chunks"], "common type share", f"{np.mean(labels == 0):.3f}",
      "rare type rows", int(np.sum(labels == RARE)), flush=True)

variants = [("unfiltered", None), ("common", np.zeros(q, np.int32)), ("rare", np.full(q, RARE, np.int32))]
results = {name: [] for name, _ in variants}
results["range_rare_0.8"] = []
for r in range(rounds + 1):
    for name, filt in variants:
        ix.set_filter(filt)
        ix.topk_resident_host(q, k)
        results[name].append((ix.last_kernel_ms(), ix.layout()["pairs_scored"]))
    ix.set_filter(variants[2][1])
    ix._range_resident(q, 0.8)
    results["range_rare_0.8"].append((ix.last_kernel_ms(), ix.layout()["pairs_scored"]))
    ix.upload_queries(qfb)  # the fetch consumed the result; a fresh batch for the next round (no filter)

for name, runs in results.items():
    runs = runs[1:]
    ms = np.median(np.array([m for m, _ in runs]), axis=0)
    pairs = runs[-1][1]
    print(f"{name:16s} kernel ms [bound0 seed select/bound1 scan merge] {np.round(ms, 3).tolist()} "
          f"sum {ms.sum():.2f}  pairs_scored {pairs}", flush=True)
