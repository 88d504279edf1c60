"""Tag-filtered search timing: `python profiles/run_tags.py [ROWS] [QUERIES] [ROUNDS]`.

Bench corpus (synth.CORPUS_SEED, default 10M rows); every row carries one of 16 Zipf-weighted failure types (label) and
1-3 of 1,000 Zipf-weighted apps (tags), from a seeded RNG.  The bench query batch (synth.QUERY_SEED, default 100k
queries) stays resident.  Per round, in one process and alternating: unfiltered top-16; every query filtered to the
most common type; to one app (the tenth most common); to that app and the common type; to a set of 4 apps.  Reports
the CUDA-event kernel times (kv_index_last_kernel_ms: bound pass 0, seed scan, selection / bound pass 1, scan, merge)
and the (query, chunk) pairs scored, median over the rounds after one warm-up round, with the card and its power
limit."""
import subprocess
import sys
from pathlib import Path

import numpy as np
import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
from kakveda_b200 import GfkbIndex, synth

n = int(sys.argv[1]) if len(sys.argv) > 1 else 10_000_000
q = int(sys.argv[2]) if len(sys.argv) > 2 else 100_000
rounds = int(sys.argv[3]) if len(sys.argv) > 3 else 3
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
ix.set_row_labels(labels)
wa = 1.0 / np.arange(1, 1001)
counts = rng.integers(1, 4, size=n)
indptr = np.zeros(n + 1, np.int64)
np.cumsum(counts, out=indptr[1:])
tags = rng.choice(1000, size=int(indptr[-1]), p=wa / wa.sum()).astype(np.int32)
ix.set_row_tags((indptr, tags))
APP = 9
share = np.mean(np.add.reduceat(tags == APP, indptr[:-1]) > 0)
qbuf, qoff = synth.signatures_packed(synth.QUERY_SEED, 0, q, dup_of_seed=synth.CORPUS_SEED, dup_rows=n)
qfb = ix.vocab.featurize_packed(qbuf, qoff, 0, grow=False)
print("rows", n, "queries", q, "chunks", ix.layout()["chunks"], "common type share", f"{np.mean(labels == 0):.3f}",
      "app share", f"{share:.4f}", flush=True)

one_app = (np.arange(q + 1, dtype=np.int64), np.full(q, APP, np.int32))
four_apps = (np.arange(0, 4 * q + 1, 4, dtype=np.int64), np.tile(np.array([APP, 40, 200, 700], np.int32), q))
variants = [("unfiltered", None, None), ("label", np.zeros(q, np.int32), None), ("app", None, one_app),
            ("app+label", np.zeros(q, np.int32), one_app), ("4 apps", None, four_apps)]
results = {name: [] for name, _, _ in variants}
for r in range(rounds + 1):
    for name, filt, tg in variants:
        ix.upload_queries(qfb)
        ix.set_filter(filt)
        ix.set_tag_filter(tg)
        ix.topk_resident_host(q, k)
        results[name].append((ix.last_kernel_ms(), ix.layout()["pairs_scored"]))

for name, runs in results.items():
    runs = runs[1:]
    ms = np.median(np.array([m for m, _ in runs]), axis=0)
    pairs = runs[-1][1]
    print(f"{name:12s} kernel ms [bound0 seed select/bound1 scan merge] {np.round(ms, 3).tolist()} "
          f"sum {ms.sum():.2f}  pairs_scored {pairs}", flush=True)
