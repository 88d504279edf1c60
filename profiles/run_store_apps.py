"""App-scoped store timing: `python profiles/run_store_apps.py [--rows N] [--queries Q]`.

The synthetic store of ``profiles/run_shard_store.py`` (N records, default 1,000,000; synth.corpus texts, 8 failure
types), each record listing 2 of 100 apps (seeded RNG), opened as a ``GfkbStore`` and as a ``ShardedGfkbStore`` with
one rank.  Reported, wall clock, median of three calls after one warm-up:

* ``match_batch`` of Q bench queries (default 2,000): unfiltered, and with ``app_ids`` (each query one app);
* ``warn_batch(app_scoped=True)`` and the reference's ``warn_batch`` of Q requests, each call right after one upsert
  (both then sync the tail and refresh the statistics; the app-scoped call also interns the new record and uploads
  the tail's tags again);
* the exact fallback of one app-scoped query (``_exact_top`` with ``app``), mean over 20 queries;
* the host tag work after an upsert (interning the new record, the tail's tag upload), and after a purge of one app
  (the purge itself, the deletion's finalize, the main segment's tag upload).

The card name and power limit are printed first, read in the same run."""
import argparse
import statistics
import subprocess
import sys
import time
from pathlib import Path

import numpy as np
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

rng = np.random.default_rng(7)
types = [f"TYPE_{i}" for i in range(8)]
corpus = synth.corpus(args.rows)
apps = rng.integers(0, 100, size=(args.rows, 2))
records = [{"failure_id": f"F-{i + 1:04d}", "version": 1, "failure_type": types[i % 8], "root_cause": None,
            "context_signature": {}, "impact_severity": "low", "resolution": None, "occurrences": 1,
            "affected_apps": sorted({f"app{a}" for a in apps[i]}), "signature_text": t} for i, t in enumerate(corpus)]
queries = synth.queries(args.queries, args.rows)
q_apps = [f"app{a}" for a in rng.integers(0, 100, size=len(queries))]
requests = [{"app_id": a, "prompt": q, "tools": [], "env": {}} for q, a in zip(queries, q_apps)]


def timed(fn, before=None, reps=3):
    if before:
        before()
    fn()
    ms = []
    for _ in range(reps):
        if before:
            before()
        t0 = time.perf_counter()
        fn()
        ms.append(1e3 * (time.perf_counter() - t0))
    return statistics.median(ms)


n_up = [0]


def upsert(st):
    def run():
        n_up[0] += 1
        st.upsert({"failure_type": "TYPE_0", "signature_text": f"fresh upsert text {n_up[0]} zz{n_up[0]}",
                   "context_signature": {}, "impact_severity": "low", "app_id": "app3"})
    return run


for name, cls in (("GfkbStore", GfkbStore), ("ShardedGfkbStore W=1", ShardedGfkbStore)):
    t0 = time.perf_counter()
    st = cls()
    st._reset([dict(r) for r in records])
    st.match_batch(queries[:1], app_ids=q_apps[:1])
    print(f"{name}: built {args.rows} records in {time.perf_counter() - t0:.1f} s", flush=True)
    print(f"{name}: match_batch {len(queries)} queries {timed(lambda: st.match_batch(queries)):.1f} ms, "
          f"with app_ids {timed(lambda: st.match_batch(queries, app_ids=q_apps)):.1f} ms", flush=True)
    print(f"{name}: warn_batch(app_scoped=True) {len(requests)} requests after an upsert "
          f"{timed(lambda: st.warn_batch(requests, app_scoped=True), before=upsert(st)):.1f} ms, "
          f"warn_batch (reference) after an upsert {timed(lambda: st.warn_batch(requests), before=upsert(st)):.1f} ms",
          flush=True)
    upsert(st)()
    st._sync()
    t0 = time.perf_counter()
    st._sync_apps()
    st._ensure_tags()
    print(f"{name}: host tag work after an upsert (intern the record, upload the tail's tags) "
          f"{1e3 * (time.perf_counter() - t0):.2f} ms", flush=True)
    exact_q = queries[:20]
    app = st._apps.listed("app5")
    st._exact_top(exact_q[0], 5, app=app)
    t0 = time.perf_counter()
    for q in exact_q:
        st._exact_top(q, 5, app=app)
    print(f"{name}: exact fallback (app) {1e3 * (time.perf_counter() - t0) / len(exact_q):.2f} ms per query", flush=True)
    t0 = time.perf_counter()
    st.purge_apps(["app99"], backup=False)
    t1 = time.perf_counter()
    st._sync()
    t2 = time.perf_counter()
    st._ensure_tags()
    t3 = time.perf_counter()
    print(f"{name}: purge of one app {1e3 * (t1 - t0):.1f} ms, the deletion's finalize {1e3 * (t2 - t1):.1f} ms, "
          f"the main segment's tags uploaded again {1e3 * (t3 - t2):.1f} ms", flush=True)
    st.close()
