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
(kv_dense_last_timing).  Every range runs twice in a row, once fetched to the host (kv_dense_range_fetch: ordering on
the device, ordered arrays copied back) and once to device memory (kv_dense_range_fetch_device); the fetch times are
the host clock around each call (both end in a stream synchronise).  The digest is that of the host arrays; the device
arrays must give the same one.  Last, the connected components of the self-join graph at theta = 0.8 (--cluster-theta):
kv_cluster_csr_device on the device arrays against kv_cluster_csr on the host arrays (host clock, alternated)."""
import ctypes as C
import hashlib
import math
import subprocess
import sys
import time
from pathlib import Path

import numpy as np
import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
from kakveda_b200 import DenseIndex, _capi

args = [a for a in sys.argv[1:] if not a.startswith("--")]
n = int(args[0]) if args else 1_000_000
q = int(args[1]) if len(args) > 1 else 10_000
reps = int(sys.argv[sys.argv.index("--reps") + 1]) if "--reps" in sys.argv else 3
cluster_theta = float(sys.argv[sys.argv.index("--cluster-theta") + 1]) if "--cluster-theta" in sys.argv else 0.8
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


def digest(arrays):
    arrays = [a.cpu().numpy() if torch.is_tensor(a) else a for a in arrays]
    return hashlib.sha256(b"".join(a.tobytes() for a in arrays)).hexdigest()[:16]


def both_fetches(label, search):
    """search(device_out) twice: host fetch, then device fetch; prints both fetch times and the digest."""
    t0 = time.perf_counter()
    host = search(False)
    t1 = time.perf_counter()
    ms, splits = dx.last_timing()
    t_host = dx.last_fetch_s
    dev = search(True)
    t_dev = dx.last_fetch_s
    dh, dd = digest(host), digest(dev)
    assert dh == dd, (label, dh, dd)
    del dev
    return (f"{label} pairs {len(host[1])} kernel_ms {ms:.2f} splits {splits} host_fetch_ms {1e3 * t_host:.1f} "
            f"device_fetch_ms {1e3 * t_dev:.1f} call_ms {1e3 * (t1 - t0):.1f} digest {dh}")


def run_round(report):
    s, r = dx.selfjoin_topk(32, device_out=True)
    ms, splits = dx.last_timing()
    del s, r
    if report:
        print(f"selfjoin_topk32 kernel_ms {ms:.1f} splits {splits}", flush=True)
    for theta in thetas:
        line = both_fetches(f"selfjoin_range theta {theta}", lambda dev: dx.selfjoin_range(theta, device_out=dev))
        if report:
            print(line, flush=True)
    s, r = dx.topk_device(queries, 32)
    ms, splits = dx.last_timing()
    del s, r
    if report:
        print(f"query_topk32 queries {q} kernel_ms {ms:.2f} splits {splits}", flush=True)
    for theta in thetas:
        line = both_fetches(f"query_range queries {q} theta {theta}",
                            lambda dev: dx.range_device(queries, theta, device_out=dev))
        if report:
            print(line, flush=True)


# time the fetch functions alone: wrap the index's fetch
_fetch = dx._range_fetch


def _timed_fetch(n_q, n_pairs, device_out=False):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = _fetch(n_q, n_pairs, device_out)
    dx.last_fetch_s = time.perf_counter() - t0
    return out


dx._range_fetch = _timed_fetch
dx.last_fetch_s = 0.0

run_round(report=False)  # warm-up: modules load, the pair buffer grows to the largest result
for rep in range(reps):
    print("round", rep, flush=True)
    run_round(report=True)

# connected components of the self-join graph: device union-find on the device CSR against the host union-find
lib = _capi.load()
indptr_h, rows_h = dx.selfjoin_range(cluster_theta)[:2]
indptr_d, rows_d = dx.selfjoin_range(cluster_theta, device_out=True)[:2]
labels_h = np.empty(n, np.int64)
labels_d = torch.empty(n, dtype=torch.int64, device=dev)
cnt_h, cnt_d = C.c_int64(0), C.c_int64(0)
p64 = lambda a: a.ctypes.data_as(C.POINTER(C.c_int64))
for rep in range(reps + 1):  # round 0 warms up
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    _capi.check(lib.kv_cluster_csr_device(0, n, C.c_void_p(indptr_d.data_ptr()), C.c_void_p(rows_d.data_ptr()),
                                          C.c_void_p(labels_d.data_ptr()), C.byref(cnt_d)))
    t1 = time.perf_counter()
    _capi.check(lib.kv_cluster_csr(n, p64(indptr_h), p64(rows_h), p64(labels_h), C.byref(cnt_h)))
    t2 = time.perf_counter()
    assert cnt_d.value == cnt_h.value and np.array_equal(labels_d.cpu().numpy(), labels_h)
    if rep:
        print(f"cluster_csr selfjoin theta {cluster_theta} edges {len(rows_h)} components {cnt_h.value} "
              f"device_ms {1e3 * (t1 - t0):.1f} host_ms {1e3 * (t2 - t1):.1f} labels_digest {digest([labels_h])}", flush=True)
dx.close()
