"""Dense threshold search timing: `python profiles/run_dense_range.py [ROWS] [QUERIES] [--reps R]`.

The bench's dense rows are random bf16, so almost no pair clears a useful threshold.  This script generates clustered
embeddings on the device instead: ROWS (1M) x 768 rows around ROWS / 1000 centroids of norm sqrt(768), each row the
centroid plus Gaussian noise of a per-row level s with ln(1 + s^2) = 0.64 v^(2/3), v uniform.  Two rows of a cluster
then have cosine about 1 / sqrt((1 + s_i^2)(1 + s_j^2)), so the self-join returns about 1e6 pairs at theta = 0.95,
1e7 at 0.9 and 1e8 at 0.8.  The last 10 % of the rows are exact copies of earlier rows.

Times, in one process and alternated per round: the self-join range (kv_dense_selfjoin_range) at each theta against
the self-join top-32 (kv_dense_selfjoin_device, the GEMM + top-k kernel) on the same rows, and a range of QUERIES
(10k) fresh rows of the same clusters against the index (kv_dense_range_device) against their top-32.  A warm-up round
grows the pair buffer first, so the timed rounds run each kernel once.  Kernel times are CUDA events
(kv_dense_last_timing); fetch + ordering is the host clock around kv_dense_range_fetch (copy back, counting sort by
query, (score desc, row asc) per query)."""
import math
import subprocess
import sys
import time
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
from kakveda_b200 import DenseIndex

args = [a for a in sys.argv[1:] if not a.startswith("--")]
n = int(args[0]) if args else 1_000_000
q = int(args[1]) if len(args) > 1 else 10_000
reps = int(sys.argv[sys.argv.index("--reps") + 1]) if "--reps" in sys.argv else 3
d = 768
thetas = (0.8, 0.9, 0.95)

try:
    power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
except (OSError, subprocess.SubprocessError):
    power = "unknown"
print("card", torch.cuda.get_device_name(0), "power limit", power, flush=True)

dev = torch.device("cuda", 0)
g = torch.Generator(device=dev).manual_seed(2024)
n_cent = max(1, n // 1000)
cent = torch.randn(n_cent, d, generator=g, device=dev)
cent *= math.sqrt(d) / cent.norm(dim=1, keepdim=True)


def clustered(m):
    out = torch.empty(m, d, dtype=torch.bfloat16, device=dev)
    for a in range(0, m, 1 << 17):
        b = min(m, a + (1 << 17))
        lab = torch.randint(0, n_cent, (b - a,), generator=g, device=dev)
        s = torch.sqrt(torch.expm1(0.64 * torch.rand(b - a, generator=g, device=dev) ** (2.0 / 3.0)))
        out[a:b] = (cent[lab] + s[:, None] * torch.randn(b - a, d, generator=g, device=dev)).to(torch.bfloat16)
    return out


rows = clustered(n)
n_dup = n // 10
rows[n - n_dup:] = rows[torch.randint(0, n - n_dup, (n_dup,), generator=g, device=dev)]
queries = clustered(q)
torch.cuda.synchronize()
dx = DenseIndex(d)
dx.add_device(rows)
dx.finalize()
print("rows", n, "dim", d, "clusters", n_cent, "duplicate rows", n_dup, "queries", q, flush=True)


def run_round(report):
    s, r = dx.selfjoin_topk(32, device_out=True)
    ms, splits = dx.last_timing()
    del s, r
    if report:
        print(f"selfjoin_topk32 kernel_ms {ms:.1f} splits {splits}", flush=True)
    for theta in thetas:
        t0 = time.perf_counter()
        indptr, rr, sc = dx.selfjoin_range(theta)
        t1 = time.perf_counter()
        ms, splits = dx.last_timing()
        t_fetch = dx.last_fetch_s
        if report:
            print(f"selfjoin_range theta {theta} pairs {len(rr)} kernel_ms {ms:.1f} splits {splits} "
                  f"fetch_order_ms {1e3 * t_fetch:.0f} call_ms {1e3 * (t1 - t0):.0f}", flush=True)
        del indptr, rr, sc
    s, r = dx.topk_device(queries, 32)
    ms, splits = dx.last_timing()
    del s, r
    if report:
        print(f"query_topk32 queries {q} kernel_ms {ms:.2f} splits {splits}", flush=True)
    for theta in thetas:
        t0 = time.perf_counter()
        indptr, rr, sc = dx.range_device(queries, theta)
        t1 = time.perf_counter()
        ms, splits = dx.last_timing()
        if report:
            print(f"query_range queries {q} theta {theta} pairs {len(rr)} kernel_ms {ms:.2f} splits {splits} "
                  f"fetch_order_ms {1e3 * dx.last_fetch_s:.1f} call_ms {1e3 * (t1 - t0):.1f}", flush=True)


# time kv_dense_range_fetch alone: wrap the index's fetch
_fetch = dx._range_fetch


def _timed_fetch(n_q, n_pairs):
    t0 = time.perf_counter()
    out = _fetch(n_q, n_pairs)
    dx.last_fetch_s = time.perf_counter() - t0
    return out


dx._range_fetch = _timed_fetch
dx.last_fetch_s = 0.0

run_round(report=False)  # warm-up: modules load, the pair buffer grows to the largest result
for rep in range(reps):
    print("round", rep, flush=True)
    run_round(report=True)
dx.close()
