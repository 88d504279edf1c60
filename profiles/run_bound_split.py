"""Where the bound pass's time goes: `python profiles/run_bound_split.py [ROWS] [QUERIES] [K]`.

Bench corpus (synth.CORPUS_SEED, default 10M rows) and bench query batch (synth.QUERY_SEED, default 100k queries),
top-K (default 16), once per library variant, each in a child process of its own that has finished before the next
one starts:
  * ``product``  -- kakveda_b200/lib/libkakveda_b200.so: the CUDA-event kernel times (kv_index_last_kernel_ms), median of
                    three steps after a warm-up step.  These are the only times this script reports.
  * ``clocks``   -- kakveda_b200/lib/libkakveda_b200_boundclocks.so (-DKV_BOUND_CLOCKS, `python -m kakveda_b200.build
                    --bound-clocks`): one step; every warp of bound pass 0 splits each 64-chunk block of its loop into
                    clock() spans, the rare join counts what it meets and every CTA notes its start and end
                    (KV_BOUND_CLOCKS in csrc/bound_kernel.cuh).  Printed as cycles per (warp, block), as counts per
                    (thread, block) and as the spread of the CTAs' durations.  The instrumentation adds instructions
                    and some spills, so this build's time is never quoted.
Both libraries are used as they are when their stamps match the sources and are built otherwise."""
import ctypes
import hashlib
import os
import subprocess
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

WORKER_SPANS = ["wait for the block's rare bitmap", "join: bit tests + ballots", "join: hit numbering + shuffles (per round)",
                "join: slot + weight loads (per round)", "join: fan-out into R (per round)", "wait for R complete (RFULL)", "R read-out",
                "second-class features left out of the dictionary", "bound, codes, seeds", "code store / list append",
                "RCLEAN arrive + WORKERS barrier"]
MMA_SPANS = ["chunk-slice waits + GEMM", "wait for R clean (RCLEAN)", "adds into R", "B2 build"]
COUNTERS = ["bit_hits", "rounds", "multi_round_warp_blocks", "table_hits", "mask_bits", "fan_iters", "join_slowest_warp_cycles", "mma_last_blocks", "mma_last_cycles", "workers_last_cycles", "worker_warp_blocks",
            "mma_warp_blocks", "cta_blocks", "ctas"]
MAX_CTAS = 4096
N_SLOTS = len(WORKER_SPANS) + len(MMA_SPANS) + len(COUNTERS) + 2 * MAX_CTAS
JOIN_SPANS = slice(1, 5)  # the worker spans between the bitmap wait and the RFULL wait


def parse(argv):
    n = int(argv[0]) if len(argv) > 0 else 10_000_000
    q = int(argv[1]) if len(argv) > 1 else 100_000
    k = int(argv[2]) if len(argv) > 2 else 16
    if not (n > 0 and q > 0 and 1 <= k <= 32):
        raise SystemExit("usage: run_bound_split.py [ROWS] [QUERIES] [K]   (1 <= K <= 32)")
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
          f"pairs_passed_bound {lay['pairs_passed_bound']} result digest {digest}", flush=True)
    if variant == "product":
        med = np.median(np.array(ms[1:]), axis=0)
        print(f"[product] last_kernel_ms [bound0 seed thresholds scan merge], median of {steps - 1} steps: {np.round(med, 3).tolist()}", flush=True)
        return
    prof = (ctypes.c_ulonglong * N_SLOTS)()
    fn = _capi.load().kv_debug_bound_profile
    fn.restype, fn.argtypes = ctypes.c_int, [ctypes.POINTER(ctypes.c_ulonglong), ctypes.c_int]
    if fn(prof, N_SLOTS) != 0:
        raise SystemExit("kv_debug_bound_profile failed: the library's profile layout is not this script's")
    v = np.array(list(prof), dtype=np.float64)
    nw, nm = len(WORKER_SPANS), len(MMA_SPANS)
    wspans, mspans = v[:nw], v[nw:nw + nm]
    c = dict(zip(COUNTERS, v[nw + nm:nw + nm + len(COUNTERS)]))
    n_ctas = int(c["ctas"])
    if n_ctas > MAX_CTAS:
        raise SystemExit(f"{n_ctas} CTAs: the profile keeps the times of {MAX_CTAS}")
    t0 = v[nw + nm + len(COUNTERS):][:n_ctas]
    t1 = v[nw + nm + len(COUNTERS) + MAX_CTAS:][:n_ctas]
    wb, mb, cb = max(c["worker_warp_blocks"], 1.0), max(c["mma_warp_blocks"], 1.0), max(c["cta_blocks"], 1.0)
    print("[clocks] bound pass 0, cycles per (warp, block) (measuring build: a split, not a time)")
    for name, cyc in zip(WORKER_SPANS, wspans):
        print(f"  workers: {name:50s} {cyc / wb:8.0f}  {100 * cyc / wspans.sum():5.1f} %")
    print(f"  workers: {'total':50s} {wspans.sum() / wb:8.0f}")
    join = wspans[JOIN_SPANS].sum() / wb
    print(f"  workers: rare join, mean {join:.0f}, slowest warp of a block {c['join_slowest_warp_cycles'] / cb:.0f} "
          f"({c['join_slowest_warp_cycles'] / cb / max(join, 1):.2f} x)")
    for name, cyc in zip(MMA_SPANS, mspans):
        print(f"  MMA warpgroup: {name:44s} {cyc / mb:8.0f}  {100 * cyc / mspans.sum():5.1f} %")
    print(f"  MMA warpgroup: {'total':44s} {mspans.sum() / mb:8.0f}")
    tb = wb * 32  # (worker thread, block)
    print(f"[clocks] rare join per (thread, block), 8 list entries each: bitmap hits {c['bit_hits'] / tb:.3f}, table hits "
          f"{c['table_hits'] / tb:.3f}, hit-mask bits (adds into R) {c['mask_bits'] / tb:.3f}")
    print(f"[clocks] per (warp, block): lookups {c['bit_hits'] / wb:.2f}, rounds {c['rounds'] / wb:.3f}, share needing a second "
          f"round {100 * c['multi_round_warp_blocks'] / wb:.2f} %, fan-out iterations {c['fan_iters'] / wb:.2f}")
    ml = c["mma_last_blocks"]
    print(f"[clocks] last at RFULL: the MMA warpgroup in {100 * ml / cb:.1f} % of the blocks (by {c['mma_last_cycles'] / max(ml, 1):.0f} "
          f"cycles), the slowest worker warp in the rest (by {c['workers_last_cycles'] / max(cb - ml, 1):.0f} cycles)")
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    dur = (t1 - t0) / 1e6
    span = (t1.max() - t0.min()) / 1e6
    print(f"[clocks] {n_ctas} CTAs on {sms} SMs ({n_ctas / sms:.2f} waves): CTA duration min {dur.min():.2f} median {np.median(dur):.2f} "
          f"max {dur.max():.2f} ms; first start to last end {span:.2f} ms; SM time without a CTA "
          f"{100 * (1 - dur.sum() / (sms * span)):.1f} % (ratios of the measuring build)", flush=True)


def main() -> None:
    if len(sys.argv) > 1 and sys.argv[1] == "--child":
        child(sys.argv[2], *parse(sys.argv[3:]))
        return
    n, q, k = parse(sys.argv[1:])
    from kakveda_b200 import build as B

    libs = {"product": B.build(), "clocks": B.build(**B.BOUND_CLOCKS)}
    for variant, lib in libs.items():
        env = dict(os.environ, KAKVEDA_B200_LIB=str(lib))
        subprocess.run([sys.executable, __file__, "--child", variant, str(n), str(q), str(k)], env=env, check=True)


if __name__ == "__main__":
    main()
