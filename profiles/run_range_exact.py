"""Exact threshold search timing: `python profiles/run_range_exact.py [--rows N] [--queries Q] [--store-rows M]
[--store-queries S]`.

Index part: the bench corpus (synth.CORPUS_SEED) of N rows (default 2,000,000) and Q bench queries (default 8,192;
synth.QUERY_SEED, generated as run_range.py does).  Per threshold in {0.5, 0.8, 0.95}, one warm-up and three timed
rounds; a round runs, alternating in one process:

* the float32 range: kv_range_resident + kv_range_fetch (host clock, both end in a stream synchronise);
* the exact range: kv_range_resident_exact + kv_range_fetch_exact, split into the float32 search (kernel events of
  the bound pass, scan and fallbacks), K6-R with its compaction (CUDA events, kv_index_last_kernel_ms()[0]), the rest
  of the call (query norms and the CSR upload for K6-R, read-backs) and the ordering (the fetch, host clock).

Candidates (float32 pairs at the lowered threshold) and kept pairs are printed with the float32 range's pair count.

Store part: a synthetic store of M records (default 1,000,000; synth.corpus texts, 8 failure types) and S bench
queries (default 2,000): ``match_above_batch`` at 0.8 against ``match_batch``, wall clock, median of three calls after
one warm-up, alternated.

The card name and power limit are printed first, read in the same run."""
import argparse
import ctypes as C
import statistics
import subprocess
import sys
import time
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
from kakveda_b200 import GfkbIndex, GfkbStore, _capi, synth  # noqa: E402
from kakveda_b200.similarity import _ptr  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--rows", type=int, default=2_000_000)
ap.add_argument("--queries", type=int, default=8192)
ap.add_argument("--store-rows", type=int, default=1_000_000)
ap.add_argument("--store-queries", type=int, default=2000)
args = ap.parse_args()

try:
    power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
except (OSError, subprocess.SubprocessError):
    power = "unknown"
print("card", torch.cuda.get_device_name(0), "power limit", power, flush=True)

lib = _capi.load()
n, q = args.rows, args.queries
buf, off = synth.signatures_packed(synth.CORPUS_SEED, 0, n)
ix = GfkbIndex()
fb = ix.vocab.featurize_packed(buf, off, 0, grow=True)
ix.add_features(fb)
fb.close()
ix.finalize()
qbuf, qoff = synth.signatures_packed(synth.QUERY_SEED, 0, q, dup_of_seed=synth.CORPUS_SEED, dup_rows=n)
qfb = ix.vocab.featurize_packed(qbuf, qoff, 0, grow=False)
ix.upload_queries(qfb)
print("rows", n, "queries", q, "chunks", ix.layout()["chunks"], flush=True)


def float32_range(theta):
    cnt = C.c_int64(0)
    t0 = time.perf_counter()
    _capi.check(lib.kv_range_resident(ix._h, C.c_float(theta), C.byref(cnt)))
    t1 = time.perf_counter()
    m = cnt.value
    out = (np.empty(q + 1, np.int64), np.empty(max(m, 1), np.int64), np.empty(max(m, 1), np.float32))
    _capi.check(lib.kv_range_fetch(ix._h, _ptr(out[0], C.c_int64), _ptr(out[1], C.c_int64), _ptr(out[2], C.c_float),
                                   None, None))
    t2 = time.perf_counter()
    return m, t1 - t0, t2 - t1


def exact_range(theta):
    cnt, cand = C.c_int64(0), C.c_int64(0)
    t0 = time.perf_counter()
    _capi.check(lib.kv_range_resident_exact(ix._h, _ptr(qfb.indptr, C.c_int64), _ptr(qfb.ids, C.c_uint32),
                                            _ptr(qfb.tf, C.c_uint32), _ptr(qfb.oov, C.c_double), q, theta,
                                            C.byref(cnt), C.byref(cand)))
    t1 = time.perf_counter()
    kms = ix.last_kernel_ms()
    m = cnt.value
    out = (np.empty(q + 1, np.int64), np.empty(max(m, 1), np.int64), np.empty(max(m, 1), np.float64))
    _capi.check(lib.kv_range_fetch_exact(ix._h, _ptr(out[0], C.c_int64), _ptr(out[1], C.c_int64), _ptr(out[2], C.c_double)))
    t2 = time.perf_counter()
    return m, cand.value, t1 - t0, t2 - t1, kms


for theta in (0.5, 0.8, 0.95):
    f32, ex = [], []
    for run in range(4):  # run 0 warms up (buffers grow to the result's size)
        a = float32_range(theta)
        b = exact_range(theta)
        if run:
            f32.append(a)
            ex.append(b)
    m32, m, cand = f32[0][0], ex[0][0], ex[0][1]
    med = lambda xs: 1e3 * statistics.median(xs)  # noqa: E731
    search_ms = statistics.median([sum(e[4][2:5]) for e in ex])
    k6r_ms = statistics.median([e[4][0] for e in ex])
    print(f"theta {theta} float32_pairs {m32} candidates {cand} kept {m} | float32 search_ms {med([a[1] for a in f32]):.1f} "
          f"fetch_ms {med([a[2] for a in f32]):.1f} total_ms {med([a[1] + a[2] for a in f32]):.1f} | exact call_ms "
          f"{med([e[2] for e in ex]):.1f} (search kernels {search_ms:.1f}, K6-R {k6r_ms:.2f}) order_fetch_ms "
          f"{med([e[3] for e in ex]):.1f} total_ms {med([e[2] + e[3] for e in ex]):.1f}", flush=True)
ix.close()

rng = np.random.default_rng(7)
types = [f"TYPE_{i}" for i in range(8)]
corpus = synth.corpus(args.store_rows)
records = [{"failure_id": f"F-{i + 1:04d}", "version": 1, "failure_type": types[i % 8], "root_cause": None,
            "context_signature": {}, "impact_severity": "low", "resolution": None, "occurrences": 1,
            "affected_apps": ["app0"], "signature_text": t} for i, t in enumerate(corpus)]
queries = synth.queries(args.store_queries, args.store_rows)
st = GfkbStore()
st._reset(records)
st.match_batch(queries)
st.match_above_batch(queries, 0.8)
t_match, t_above = [], []
for _ in range(3):
    t0 = time.perf_counter()
    st.match_batch(queries)
    t1 = time.perf_counter()
    res = st.match_above_batch(queries, 0.8)
    t2 = time.perf_counter()
    t_match.append(t1 - t0)
    t_above.append(t2 - t1)
print(f"store rows {args.store_rows} queries {len(queries)} match_batch_ms {1e3 * statistics.median(t_match):.1f} "
      f"match_above_batch_0.8_ms {1e3 * statistics.median(t_above):.1f} matches {sum(len(r) for r in res)}", flush=True)
st.close()
