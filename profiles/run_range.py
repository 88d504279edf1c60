"""Threshold search timing: `python profiles/run_range.py ROWS QUERIES THETA... [--selfjoin]`.

Bench corpus (synth.CORPUS_SEED) of ROWS rows; QUERIES bench queries (synth.QUERY_SEED, about half of them copies of
stored rows), or with --selfjoin the corpus-fit self-join of rows [0, QUERIES).  Per threshold one warm-up and three
timed runs of kv_range_resident (device) and kv_range_fetch (copy back + ordering on the host)."""
import ctypes as C
import hashlib
import subprocess
import sys
import time
from pathlib import Path

import numpy as np
import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
from kakveda_b200 import GfkbIndex, _capi, synth

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

for theta in thetas:
    for run in range(4):  # run 0 warms up (buffers grow to the result's size)
        n_pairs = C.c_int64(0)
        t0 = time.perf_counter()
        rc = lib.kv_range_resident(ix._h, C.c_float(theta), C.byref(n_pairs))
        t1 = time.perf_counter()
        if rc != _capi.KV_OK:
            print("theta", theta, "error", rc, _capi.last_error(), flush=True)
            break
        indptr = np.empty(q + 1, np.int64)
        rows = np.empty(max(n_pairs.value, 1), np.int64)
        scores = np.empty(max(n_pairs.value, 1), np.float32)
        t2 = time.perf_counter()
        _capi.check(lib.kv_range_fetch(ix._h, indptr.ctypes.data_as(C.POINTER(C.c_int64)),
                                       rows.ctypes.data_as(C.POINTER(C.c_int64)), scores.ctypes.data_as(C.POINTER(C.c_float))))
        t3 = time.perf_counter()
        if run == 0:
            continue
        lay = ix.layout()
        digest = hashlib.sha256(indptr.tobytes() + rows[:n_pairs.value].tobytes() + scores[:n_pairs.value].tobytes()).hexdigest()[:16]
        print(f"theta {theta} pairs {n_pairs.value} pairs_passed_bound {lay['pairs_passed_bound']} "
              f"pairs_scored {lay['pairs_scored']} kernels_ms {[round(x, 2) for x in ix.last_kernel_ms()]} "
              f"range_call_ms {1e3 * (t1 - t0):.1f} fetch_order_ms {1e3 * (t3 - t2):.1f} digest {digest}", flush=True)
