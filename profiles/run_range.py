"""Threshold search timing: `python profiles/run_range.py ROWS QUERIES THETA... [--selfjoin]`.

Bench corpus (synth.CORPUS_SEED) of ROWS rows; QUERIES bench queries (synth.QUERY_SEED, about half of them copies of
stored rows), or with --selfjoin the corpus-fit self-join of rows [0, QUERIES).  Per threshold one warm-up and three
timed rounds; a round runs kv_range_resident (device) twice, once followed by kv_range_fetch (ordering on the device,
ordered arrays copied to host memory) and once by kv_range_fetch_device (the same arrays left in device memory), so the
two fetches alternate in one process.  Fetch times are the host clock around the call (both end in a stream
synchronise).  The digest is that of the host arrays; the device arrays must give the same one."""
import ctypes as C
import hashlib
import subprocess
import sys
import time
from pathlib import Path

import numpy as np
import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
from kakveda_b200 import GfkbIndex, _capi, _devout, synth

args = [a for a in sys.argv[1:] if not a.startswith("--")]
selfjoin = "--selfjoin" in sys.argv
n = int(args[0]) if args else 1_000_000
q = int(args[1]) if len(args) > 1 else 16_384
thetas = [float(t) for t in args[2:]] or [0.8]

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
if selfjoin:
    ix.set_mode(2)  # corpus-fit TF-IDF: the measure of pattern clustering
ix.finalize()
lib = _capi.load()
if selfjoin:
    _capi.check(lib.kv_selfjoin_upload(ix._h, 0, q))
else:
    qbuf, qoff = synth.signatures_packed(synth.QUERY_SEED, 0, q, dup_of_seed=synth.CORPUS_SEED, dup_rows=n)
    ix.upload_queries(ix.vocab.featurize_packed(qbuf, qoff, 0, grow=False))
print("rows", n, "queries", q, "selfjoin" if selfjoin else "bench queries", "chunks", ix.layout()["chunks"], flush=True)


def digest(indptr, rows, scores):
    return hashlib.sha256(indptr.tobytes() + rows.tobytes() + scores.tobytes()).hexdigest()[:16]


def search(theta):
    n_pairs = C.c_int64(0)
    t0 = time.perf_counter()
    rc = lib.kv_range_resident(ix._h, C.c_float(theta), C.byref(n_pairs))
    t1 = time.perf_counter()
    if rc != _capi.KV_OK:
        raise RuntimeError(f"theta {theta} error {rc} {_capi.last_error()}")
    return n_pairs.value, t1 - t0


def fetch_host(m):
    indptr = np.empty(q + 1, np.int64)
    rows = np.empty(max(m, 1), np.int64)
    scores = np.empty(max(m, 1), np.float32)
    t0 = time.perf_counter()
    _capi.check(lib.kv_range_fetch(ix._h, indptr.ctypes.data_as(C.POINTER(C.c_int64)),
                                   rows.ctypes.data_as(C.POINTER(C.c_int64)), scores.ctypes.data_as(C.POINTER(C.c_float)),
                                   None, None))
    t1 = time.perf_counter()
    return digest(indptr, rows[:m], scores[:m]), t1 - t0


def fetch_device(m):
    out = _devout.range_arrays(0, q, m)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    _capi.check(lib.kv_range_fetch_device(ix._h, *_devout.ptrs(out), None, None))
    t1 = time.perf_counter()
    return digest(*(t.cpu().numpy() for t in out)), t1 - t0


for theta in thetas:
    for run in range(4):  # run 0 warms up (buffers grow to the result's size)
        m, t_call = search(theta)
        d_host, t_host = fetch_host(m)
        lay, kms = ix.layout(), ix.last_kernel_ms()
        m2, t_call2 = search(theta)
        d_dev, t_dev = fetch_device(m2)
        assert m2 == m and d_dev == d_host, (theta, m, m2, d_host, d_dev)
        if run == 0:
            continue
        print(f"theta {theta} pairs {m} pairs_passed_bound {lay['pairs_passed_bound']} "
              f"pairs_scored {lay['pairs_scored']} kernels_ms {[round(x, 2) for x in kms]} "
              f"range_call_ms {1e3 * t_call:.1f} {1e3 * t_call2:.1f} host_fetch_ms {1e3 * t_host:.1f} "
              f"device_fetch_ms {1e3 * t_dev:.1f} digest {d_host}", flush=True)
