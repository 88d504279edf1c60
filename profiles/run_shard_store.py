"""ShardedGfkbStore timing at W = 1: `python profiles/run_shard_store.py [--rows N] [--queries Q]`.

A synthetic store of N records (default 1,000,000; synth.corpus texts, 8 failure types) opened as a ``GfkbStore`` and
as a ``ShardedGfkbStore`` with one rank (no collective runs at W = 1).  Reported, wall clock, median of three calls
after one warm-up:

* ``match_batch`` of Q bench queries (default 2,000) and ``warn_batch`` of Q requests, on both stores;
* the exact fallback of one query (``_exact_top``, limit 5: plain, filtered to one type, distinct) before and after
  the device path: ``GfkbStore`` copies the K1a score vector of every row to the host (8 bytes per row) and orders it
  there; ``ShardedGfkbStore`` runs ``kv_exact_topk`` (K1a, selection and K6 on the device, 5 rows back) -- mean over
  20 queries.  Both must return the same records.

Loopback runs at W > 1 share one GPU and are not multi-GPU times, so this script does not report them; multi-GPU times
of the sharded store have not been measured.  The card name and power limit are printed first, read in the same run."""
import argparse
import statistics
import subprocess
import sys
import time
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
from kakveda_b200 import GfkbStore, synth  # noqa: E402
from kakveda_b200.dist import ShardedGfkbStore  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--rows", type=int, default=1_000_000)
ap.add_argument("--queries", type=int, default=2000)
args = ap.parse_args()

try:
    power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
except (OSError, subprocess.SubprocessError):
    power = "unknown"
print("card", torch.cuda.get_device_name(0), "power limit", power, flush=True)

types = [f"TYPE_{i}" for i in range(8)]
corpus = synth.corpus(args.rows)
records = [{"failure_id": f"F-{i + 1:04d}", "version": 1, "failure_type": types[i % 8], "root_cause": None,
            "context_signature": {}, "impact_severity": "low", "resolution": None, "occurrences": 1,
            "affected_apps": ["app"], "signature_text": t} for i, t in enumerate(corpus)]
queries = synth.queries(args.queries, args.rows)
requests = [{"app_id": "a", "prompt": q, "tools": [], "env": {}} for q in queries]


def timed(fn, reps=3):
    fn()
    ms = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        ms.append(1e3 * (time.perf_counter() - t0))
    return statistics.median(ms)


stores = {}
for name, cls in (("GfkbStore", GfkbStore), ("ShardedGfkbStore W=1", ShardedGfkbStore)):
    t0 = time.perf_counter()
    st = cls()
    st._reset([dict(r) for r in records])
    st.match_batch(queries[:1])
    stores[name] = st
    print(f"{name}: built {args.rows} records in {time.perf_counter() - t0:.1f} s", flush=True)

for name, st in stores.items():
    print(f"{name}: match_batch {args.queries} queries {timed(lambda: st.match_batch(queries)):.1f} ms, "
          f"warn_batch {args.queries} requests {timed(lambda: st.warn_batch(requests)):.1f} ms", flush=True)

exact_q = queries[:20]
for mode, kw in (("plain", {}), ("filtered", {"label": 3}), ("distinct", {"distinct": True})):
    res = {}
    for name, st in stores.items():
        st._exact_top(exact_q[0], 5, **kw)   # warm-up
        t0 = time.perf_counter()
        res[name] = [st._exact_top(q, 5, **kw) for q in exact_q]
        ms = 1e3 * (time.perf_counter() - t0) / len(exact_q)
        print(f"exact fallback ({mode}), {name}: {ms:.2f} ms per query", flush=True)
    a, b = res.values()
    assert [r for r, _ in a] == [r for r, _ in b], mode
for st in stores.values():
    st.close()
