"""Where the candidate scan's time goes: `python profiles/run_scan_split.py [ROWS] [QUERIES] [K]`.

Bench corpus (synth.CORPUS_SEED, default 10M rows) and bench query batch (synth.QUERY_SEED, default 100k queries),
top-K (default 16), once per library variant, each in a child process of its own that has finished before the next
one starts:
  * ``product``  -- kakveda_b200/lib/libkakveda_b200.so: the CUDA-event kernel times (kv_index_last_kernel_ms), median of
                    three steps after a warm-up step.  These are the only times this script reports.
  * ``clocks``   -- kakveda_b200/lib/libkakveda_b200_scanclocks.so (-DKV_SCAN_CLOCKS, `python -m kakveda_b200.build
                    --scan-clocks`): one step; every warp of the codes-mode scan splits its life into clock() spans and
                    counts what it meets (KV_SCAN_CLOCKS in csrc/tfidf_kernels.cuh).  Printed as cycles per (query,
                    chunk) pair and as shares of the warps' lives.  The instrumentation adds instructions and some
                    spills, so this build's time is never quoted.
Both libraries are used as they are when their stamps match the sources and are built otherwise."""
import ctypes
import hashlib
import os
import subprocess
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

SPANS = ["select+issue", "wait staged block", "record/pair set-up", "probe", "hit production", "hit accumulation",
         "reduce+epilogue", "lock wait", "insert under lock", "tail (warp done, CTA not)"]
COUNTERS = ["pairs", "trips", "hits", "hits_w_all", "lock_acquisitions", "lock_acquisitions_unchanged", "rows_passed_pretest",
            "blocks_read_in_place", "records", "warps", "ctas", "cta_pairs_max"]
N_HIST_Q, N_HIST_CTA = 33, 64
N_SLOTS = len(SPANS) + len(COUNTERS) + N_HIST_Q + N_HIST_CTA


def parse(argv):
    n = int(argv[0]) if len(argv) > 0 else 10_000_000
    q = int(argv[1]) if len(argv) > 1 else 100_000
    k = int(argv[2]) if len(argv) > 2 else 16
    if not (n > 0 and q > 0 and 1 <= k <= 32):
        raise SystemExit("usage: run_scan_split.py [ROWS] [QUERIES] [K]   (1 <= K <= 32)")
    return n, q, k


def child(variant: str, n: int, q: int, k: int) -> None:
    import numpy as np
    import torch

    from kakveda_b200 import GfkbIndex, _capi, synth

    if variant == "product":
        try:
            power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                                   capture_output=True, text=True, timeout=30).stdout.strip()
        except (OSError, subprocess.SubprocessError):
            power = "unknown"
        print("card", torch.cuda.get_device_name(0), "power limit, max SM clock:", power, flush=True)
    buf, off = synth.signatures_packed(synth.CORPUS_SEED, 0, n)
    ix = GfkbIndex()
    fb = ix.vocab.featurize_packed(buf, off, 0, grow=True)
    ix.add_features(fb)
    fb.close()
    ix.finalize()
    qbuf, qoff = synth.signatures_packed(synth.QUERY_SEED, 0, q, dup_of_seed=synth.CORPUS_SEED, dup_rows=n)
    qfb = ix.vocab.featurize_packed(qbuf, qoff, 0, grow=False)
    steps = 4 if variant == "product" else 1
    ms = []
    for _ in range(steps):
        ix.upload_queries(qfb)
        s, rows = ix.topk_resident_host(q, k)
        ms.append(ix.last_kernel_ms())
    lay = ix.layout()
    digest = hashlib.sha256(s.tobytes() + rows.tobytes()).hexdigest()[:16]
    print(f"[{variant}] rows {n} queries {q} k {k} chunks {lay['chunks']} pairs_scored {lay['pairs_scored']} "
          f"records_scanned {lay['records_scanned']} pairs_passed_bound {lay['pairs_passed_bound']} result digest {digest}", flush=True)
    if variant == "product":
        med = np.median(np.array(ms[1:]), axis=0)
        print(f"[product] last_kernel_ms [bound0 seed thresholds scan merge], median of {steps - 1} steps: {np.round(med, 3).tolist()}", flush=True)
        return
    prof = (ctypes.c_ulonglong * N_SLOTS)()
    fn = _capi.load().kv_debug_scan_profile
    fn.restype, fn.argtypes = ctypes.c_int, [ctypes.POINTER(ctypes.c_ulonglong), ctypes.c_int]
    if fn(prof, N_SLOTS) != 0:
        raise SystemExit("kv_debug_scan_profile failed: the library's profile layout is not this script's")
    v = np.array(list(prof), dtype=np.float64)
    spans, c = v[: len(SPANS)], dict(zip(COUNTERS, v[len(SPANS):len(SPANS) + len(COUNTERS)]))
    hq = v[len(SPANS) + len(COUNTERS):][:N_HIST_Q]
    hc = v[len(SPANS) + len(COUNTERS) + N_HIST_Q:]
    pairs = max(c["pairs"], 1.0)
    print("[clocks] warp cycles per (query, chunk) pair and share of the warps' lives (measuring build: a split, not a time)")
    for name, cyc in zip(SPANS, spans):
        print(f"  {name:28s} {cyc / pairs:9.1f}  {100 * cyc / spans.sum():5.1f} %")
    print(f"  {'total':28s} {spans.sum() / pairs:9.1f}")
    print("[clocks] counters:", {name: int(x) for name, x in c.items()})
    print(f"[clocks] per pair: trips {c['trips'] / pairs:.2f} hits {c['hits'] / pairs:.2f} of them W_ALL {c['hits_w_all'] / pairs:.2f}; "
          f"hits per trip {c['hits'] / max(c['trips'], 1):.2f}, not W_ALL {(c['hits'] - c['hits_w_all']) / max(c['trips'], 1):.2f}; "
          f"rows past the pre-test {c['rows_passed_pretest'] / pairs:.3f}; lock acquisitions {c['lock_acquisitions'] / pairs:.4f}, "
          f"unchanged {c['lock_acquisitions_unchanged'] / max(c['lock_acquisitions'], 1):.3f} of them; "
          f"blocks read in place {c['blocks_read_in_place'] / max(c['records'], 1):.4f} of the records")
    print("[clocks] records by queries in the mask (0..32):", hq.astype(np.int64).tolist())
    print(f"[clocks] CTAs by pairs scored, buckets of 512 (mean {pairs / max(c['ctas'], 1):.0f}, max {int(c['cta_pairs_max'])}):",
          hc.astype(np.int64).tolist(), flush=True)


def main() -> None:
    if len(sys.argv) > 1 and sys.argv[1] == "--child":
        child(sys.argv[2], *parse(sys.argv[3:]))
        return
    n, q, k = parse(sys.argv[1:])
    from kakveda_b200 import build as B

    libs = {"product": B.build(), "clocks": B.build(**B.SCAN_CLOCKS)}
    for variant, lib in libs.items():
        env = dict(os.environ, KAKVEDA_B200_LIB=str(lib))
        subprocess.run([sys.executable, __file__, "--child", variant, str(n), str(q), str(k)], env=env, check=True)


if __name__ == "__main__":
    main()
