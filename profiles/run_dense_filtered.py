"""Dense label filter and deletion timing: `python profiles/run_dense_filtered.py [ROWS] [QUERIES] [--reps R]`.

ROWS (1M) x 768 random bf16 rows (the bench's dense shape) and QUERIES (10k) queries, generated on the device, with 16
labels in two layouts: random per row, and contiguous blocks of ROWS / 16 rows.  Queries get random labels.  After one
warm-up round, R (3) rounds alternate, in one process:
  - unfiltered top-16;
  - every query filtered, top-16, in each layout;
  - the filtered threshold search at theta = 0.8 in each layout;
  - the same-label self-join top-32 of the first 200k rows in each layout;
  - unfiltered top-16 on copies of the index with 1 % of the rows deleted at random and with 10 % deleted in one
    contiguous block.
Each line gives the GEMM kernel's CUDA-event time (kv_dense_last_timing), its row splits and the (query tile, row tile)
items the kernel skipped out of all items (kv_dense_last_skipped).  The card and its power limit come first."""
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
reps = int(sys.argv[sys.argv.index("--reps") + 1]) if "--reps" in sys.argv else 3
d, n_lab = 768, 16
sj_rows = min(n, 200_000)

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
layouts = {
    "random": rng.integers(0, n_lab, n).astype(np.int32),
    "blocks": (np.arange(n) * n_lab // n).astype(np.int32),
}
q_labels = rng.integers(0, n_lab, q).astype(np.int32)


def index(deleted=None):
    dx = DenseIndex(d)
    dx.add_device(rows)
    if deleted is not None:
        dx.delete_rows(deleted)
    dx.finalize()
    return dx


dx = index()
del1 = index(rng.choice(n, n // 100, replace=False))
start = int(rng.integers(0, n - n // 10))
del10 = index(np.arange(start, start + n // 10))
print("rows", n, "dim", d, "queries", q, "labels", n_lab, "self-join rows", sj_rows, flush=True)


def line(name, ix):
    ms, splits = ix.last_timing()
    sk, items = ix.last_skipped()
    return f"{name} gemm_ms {ms:.2f} splits {splits} skipped {sk}/{items}"


def run_round(report):
    out = []
    s, r = dx.topk_device(queries, 16)
    out.append(line("unfiltered_topk16", dx))
    for name, lab in layouts.items():
        dx.set_row_labels(lab)
        s, r = dx.topk_device(queries, 16, labels=q_labels)
        out.append(line(f"filtered_topk16 {name}", dx))
        res = dx.range_device(queries, 0.8, labels=q_labels, device_out=True)
        out.append(line(f"filtered_range0.8 {name} pairs {len(res[1])}", dx))
        s, r = dx.selfjoin_topk(32, 0, sj_rows, device_out=True, same_label=True)
        out.append(line(f"selfjoin_same_label_topk32 {name}", dx))
    s, r = dx.selfjoin_topk(32, 0, sj_rows, device_out=True)
    out.append(line("selfjoin_topk32 unfiltered", dx))
    for name, ix in (("deleted_1pct_random", del1), ("deleted_10pct_block", del10)):
        s, r = ix.topk_device(queries, 16)
        out.append(line(f"unfiltered_topk16 {name}", ix))
    del s, r
    if report:
        print("\n".join(out), flush=True)


run_round(report=False)
for rep in range(reps):
    print("round", rep, flush=True)
    run_round(report=True)
for ix in (dx, del1, del10):
    ix.close()
