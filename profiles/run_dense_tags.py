"""Dense tag filter timing: `python profiles/run_dense_tags.py [ROWS] [QUERIES] [--reps R]`.

ROWS (1M) x 768 random bf16 rows (the bench's dense shape) and QUERIES (10k) queries, generated on the device, with 32
apps as row tag sets in three layouts: one random app per row; contiguous blocks of ROWS / 32 rows per app; and the same
blocks with app ids 100..131 (tags >= 64: the masks are not exact, so every mask hit that would enter a list is
confirmed on the row's tag list).  Every query gets one random app.  After one warm-up round, R (5) rounds alternate,
in one process:
  - unfiltered top-16;
  - every query tag-filtered, top-16, in each layout.
Each line gives the GEMM kernel's CUDA-event time (kv_dense_last_timing), its row splits and the (query tile, row tile)
items the kernel skipped out of all items (kv_dense_last_skipped); the medians over the rounds come last.  The card
and its power limit come first."""
import subprocess
import sys
from pathlib import Path

import numpy as np
import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
from kakveda_b200 import DenseIndex

args = [a for a in sys.argv[1:] if not a.startswith("--")]
n = int(args[0]) if args else 1_000_000
q = int(args[1]) if len(args) > 1 else 10_000
reps = int(sys.argv[sys.argv.index("--reps") + 1]) if "--reps" in sys.argv else 5
d, n_app = 768, 32

try:
    power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
except (OSError, subprocess.SubprocessError):
    power = "unknown"
print("card", torch.cuda.get_device_name(0), "power limit", power, flush=True)

dev = torch.device("cuda", 0)
g = torch.Generator(device=dev).manual_seed(7)
rows = torch.randn(n, d, generator=g, device=dev).to(torch.bfloat16)
queries = torch.randn(q, d, generator=g, device=dev).to(torch.bfloat16)
torch.cuda.synchronize()
rng = np.random.default_rng(7)


def csr(apps):
    return np.arange(len(apps) + 1, dtype=np.int64), np.ascontiguousarray(apps, dtype=np.int32)


blocks = (np.arange(n) * n_app // n).astype(np.int32)
q_app = rng.integers(0, n_app, q).astype(np.int32)
layouts = {  # name: (row tag sets, query tag sets)
    "random": (csr(rng.integers(0, n_app, n)), csr(q_app)),
    "contiguous": (csr(blocks), csr(q_app)),
    "contiguous_tags_ge_64": (csr(blocks + 100), csr(q_app + 100)),
}

dx = DenseIndex(d)
dx.add_device(rows)
dx.finalize()
print("rows", n, "dim", d, "queries", q, "apps", n_app, flush=True)
times = {}


def line(name):
    ms, splits = dx.last_timing()
    sk, items = dx.last_skipped()
    times.setdefault(name, []).append(ms)
    return f"{name} gemm_ms {ms:.2f} splits {splits} skipped {sk}/{items}"


def run_round(report):
    out = []
    dx.set_row_tags(None)
    dx.topk_device(queries, 16)
    out.append(line("unfiltered_topk16"))
    for name, (row_sets, q_sets) in layouts.items():
        dx.set_row_tags(row_sets)
        dx.topk_device(queries, 16, tags=q_sets)
        out.append(line(f"tag_topk16 {name}"))
    if report:
        print("\n".join(out), flush=True)
    else:
        times.clear()


run_round(report=False)
for rep in range(reps):
    print("round", rep, flush=True)
    run_round(report=True)
for name, ts in times.items():
    print(f"median {name} gemm_ms {float(np.median(ts)):.2f}", flush=True)
dx.close()
