"""Jaccard threshold search timing: `python profiles/run_jaccard_range.py [ROWS] [QUERIES] [--selfjoin N] [--reps R]`.

The bench's K3 sets (64 Zipf(1.2) draws over 2^20, about 39 distinct tokens) almost never reach J = 0.5 with each
other, so this script plants near-duplicates: 5 % of the ROWS (1M) sets are copies of another set with one to three
tokens swapped.  QUERIES (2048): half fresh sets of the same generator, half near-copies of stored sets (one to three
swaps), so that theta in {0.5, 0.7, 0.9} returns a non-trivial number of pairs.

Times, in one process and alternated per round after a warm-up round (which also grows the pair buffer): K3 top-16
(`kv_topk_resident_host`, kernel = CUDA events around the scan) against K3-R (`kv_jaccard_range_resident`, kernel =
`kv_index_last_kernel_ms()[3]`, irregular-query fallbacks [4]) on the same uploaded batch, the host clock around
`kv_jaccard_range_fetch` (ordering on the device, arrays copied back) and, for the same search run again, around
`kv_jaccard_range_fetch_device` (arrays left in device memory; the digests must agree), and the self-join of the first
`--selfjoin` (200k) sets as an index of their own: self-join top-16 against the self-join range at each theta."""
import ctypes as C
import hashlib
import subprocess
import sys
import time
from pathlib import Path

import numpy as np
import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
from kakveda_b200 import JaccardIndex, _capi, _devout

args = [a for i, a in enumerate(sys.argv[1:]) if not a.startswith("--") and not sys.argv[i].startswith("--")]
n = int(args[0]) if args else 1_000_000
q = int(args[1]) if len(args) > 1 else 2048
n_self = int(sys.argv[sys.argv.index("--selfjoin") + 1]) if "--selfjoin" in sys.argv else 200_000
reps = int(sys.argv[sys.argv.index("--reps") + 1]) if "--reps" in sys.argv else 3
thetas = (0.5, 0.7, 0.9)
V = 1 << 20

try:
    power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
except (OSError, subprocess.SubprocessError):
    power = "unknown"
print("card", torch.cuda.get_device_name(0), "power limit", power, flush=True)

rng = np.random.default_rng(2024)


def zipf_sets(m):
    """The bench's K3 generator: 64 Zipf(1.2) draws over 2^20 per set, duplicates removed -> (lengths, ids)."""
    draws = np.minimum(rng.zipf(1.2, size=(m, 64)) - 1, V - 1).astype(np.uint32)
    draws.sort(axis=1)
    keep = np.ones(draws.shape, dtype=bool)
    keep[:, 1:] = draws[:, 1:] != draws[:, :-1]
    return [row[k] for row, k in zip(draws, keep)]


def near(s):
    s = s.copy()
    pos = rng.choice(len(s), size=min(len(s), int(rng.integers(1, 4))), replace=False)
    s[pos] = rng.integers(0, V, size=len(pos), dtype=np.uint32)
    return np.unique(s)


def csr(sets):
    indptr = np.concatenate([[0], np.cumsum([len(s) for s in sets])]).astype(np.int64)
    return indptr, np.concatenate(sets).astype(np.uint32)


rows = zipf_sets(n)
for i in rng.choice(n, size=n // 20, replace=False):
    rows[i] = near(rows[int(rng.integers(0, n))])
fresh = zipf_sets(q - q // 2)
queries = fresh + [near(rows[int(j)]) for j in rng.integers(0, n, size=q // 2)]
indptr, ids = csr(rows)
q_indptr, q_ids = csr(queries)
print("rows", n, "mean distinct tokens", round(len(ids) / n, 1), "near-duplicate rows", n // 20, "queries", q,
      "near-copy queries", q // 2, flush=True)

lib = _capi.load()
p = lambda a, t: a.ctypes.data_as(C.POINTER(t))


def kernel_ms(jx):
    ms = (C.c_float * 5)()
    _capi.check(lib.kv_index_last_kernel_ms(jx._h, ms))
    return list(ms)


def digest(arrays):
    return hashlib.sha256(b"".join(a.tobytes() for a in arrays)).hexdigest()[:16]


def range_timed(jx, n_q, theta):
    """(pairs, K3-R ms, fallback ms, call ms, host fetch ms, device fetch ms, digest): the search over the resident
    batch twice, fetched to host memory (ordering on the device, arrays copied back) and then to device memory."""
    cnt = C.c_int64(0)
    t0 = time.perf_counter()
    _capi.check(lib.kv_jaccard_range_resident(jx._h, C.c_float(theta), C.byref(cnt)))
    t1 = time.perf_counter()
    ms = kernel_ms(jx)
    m = cnt.value
    out = [np.empty(n_q + 1, np.int64), np.empty(max(m, 1), np.int64), np.empty(max(m, 1), np.float32),
           np.empty(max(m, 1), np.int32), np.empty(max(m, 1), np.int32)]
    t2 = time.perf_counter()
    _capi.check(lib.kv_jaccard_range_fetch(jx._h, p(out[0], C.c_int64), p(out[1], C.c_int64), p(out[2], C.c_float),
                                           p(out[3], C.c_int32), p(out[4], C.c_int32)))
    t3 = time.perf_counter()
    d_host = digest([out[0]] + [a[:m] for a in out[1:]])
    _capi.check(lib.kv_jaccard_range_resident(jx._h, C.c_float(theta), C.byref(cnt)))
    dout = _devout.range_arrays(0, n_q, cnt.value, jaccard=True)
    torch.cuda.synchronize()
    t4 = time.perf_counter()
    _capi.check(lib.kv_jaccard_range_fetch_device(jx._h, *_devout.ptrs(dout)))
    t5 = time.perf_counter()
    assert digest([a.cpu().numpy() for a in dout]) == d_host
    return m, ms[3], ms[4], 1e3 * (t1 - t0), 1e3 * (t3 - t2), 1e3 * (t5 - t4), d_host


def topk_timed(jx, n_q, k):
    s = np.empty((n_q, k), np.float32)
    r = np.empty((n_q, k), np.int64)
    _capi.check(lib.kv_topk_resident_host(jx._h, k, p(s, C.c_float), p(r, C.c_int64)))
    return jx.last_timing_ms()[1]


def run(jx, label, n_q, upload, report):
    upload()
    ms = topk_timed(jx, n_q, 16)
    if report:
        print(f"{label} K3_top16 kernel_ms {ms:.2f}", flush=True)
    for theta in thetas:  # the range leaves the uploaded batch as it was
        m, kms, fms, call, fetch, dfetch, dg = range_timed(jx, n_q, theta)
        if report:
            print(f"{label} K3R theta {theta} pairs {m} kernel_ms {kms:.2f} fallback_ms {fms:.2f} call_ms {call:.1f} "
                  f"host_fetch_ms {fetch:.1f} device_fetch_ms {dfetch:.1f} digest {dg}", flush=True)


jx = JaccardIndex(V)
jx.add_csr(indptr, ids)
jx.finalize()


def upload_queries():
    tf = np.ones(len(q_ids), np.uint32)
    _capi.check(lib.kv_query_upload(jx._h, p(q_indptr, C.c_int64), p(q_ids, C.c_uint32), p(tf, C.c_uint32), None, q))


sx = JaccardIndex(V)
sx.add_csr(indptr[:n_self + 1], ids[:indptr[n_self]])
sx.finalize()


def upload_self():
    _capi.check(lib.kv_selfjoin_upload(sx._h, 0, n_self))


for rep in range(reps + 1):
    report = rep > 0
    if report:
        print("round", rep - 1, flush=True)
    run(jx, f"{n}x{q}", q, upload_queries, report)
    run(sx, f"selfjoin{n_self}", n_self, upload_self, report)
jx.close()
sx.close()
