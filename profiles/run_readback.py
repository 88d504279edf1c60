"""Top-k read-back to host memory: `python profiles/run_readback.py [--reps R]`.

A top-k with host outputs ends by copying float32 scores[n_q*k] and int64 rows[n_q*k] from device memory into the
caller's arrays.  Two ways to do that on the handle's stream, timed here on device buffers of the result's size:

  direct  cudaMemcpyAsync of both arrays straight into the caller's (pageable) memory, then one stream synchronise
          (what kv_topk_resident_host does);
  staged  cudaMemcpyAsync of both into a pinned staging buffer kept by the handle, a stream synchronise, then two host
          memcpy into the caller's memory.

Shapes: 100,000 x 16 (the bench batch, 19.2 MB) and 2,048 x 16 (393 KB).  Each call gets freshly allocated NumPy outputs,
as GfkbIndex.topk_resident_host allocates them, so first-touch page faults count in both.  One warm-up round, then R
rounds alternating the two ways; times are the host clock around the whole read-back.  Prints the card and its power
limit and, per shape and way, the median and range in ms.
"""
import ctypes as C
import subprocess
import sys
import time

import numpy as np
import torch

reps = int(sys.argv[sys.argv.index("--reps") + 1]) if "--reps" in sys.argv else 30
D2H = 2  # cudaMemcpyDeviceToHost

try:
    power = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
except (OSError, subprocess.SubprocessError):
    power = "unknown"
print("card", torch.cuda.get_device_name(0), "| nvidia-smi name, power limit, max SM clock:", power, flush=True)

torch.cuda.init()
rt = C.CDLL("libcudart.so.12")  # the runtime torch loaded
rt.cudaMemcpyAsync.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_int, C.c_void_p]
rt.cudaStreamSynchronize.argtypes = [C.c_void_p]
stream = torch.cuda.Stream()
sp = C.c_void_p(stream.cuda_stream)


def check(rc):
    if rc != 0:
        raise RuntimeError(f"CUDA runtime error {rc}")


def direct(d_s, d_r, n):
    out_s, out_r = np.empty(n, np.float32), np.empty(n, np.int64)
    check(rt.cudaMemcpyAsync(out_s.ctypes.data, d_s.data_ptr(), n * 4, D2H, sp))
    check(rt.cudaMemcpyAsync(out_r.ctypes.data, d_r.data_ptr(), n * 8, D2H, sp))
    check(rt.cudaStreamSynchronize(sp))
    return out_s, out_r


def staged(d_s, d_r, n, h_s, h_r):
    out_s, out_r = np.empty(n, np.float32), np.empty(n, np.int64)
    check(rt.cudaMemcpyAsync(h_s.data_ptr(), d_s.data_ptr(), n * 4, D2H, sp))
    check(rt.cudaMemcpyAsync(h_r.data_ptr(), d_r.data_ptr(), n * 8, D2H, sp))
    check(rt.cudaStreamSynchronize(sp))
    np.copyto(out_s, h_s.numpy())
    np.copyto(out_r, h_r.numpy())
    return out_s, out_r


for n_q, k in ((100_000, 16), (2048, 16)):
    n = n_q * k
    d_s = torch.randn(n, device="cuda", dtype=torch.float32)
    d_r = torch.randint(0, 10_000_000, (n,), device="cuda", dtype=torch.int64)
    h_s, h_r = torch.empty(n, dtype=torch.float32, pin_memory=True), torch.empty(n, dtype=torch.int64, pin_memory=True)
    torch.cuda.synchronize()
    want = (d_s.cpu().numpy(), d_r.cpu().numpy())
    times = {"direct": [], "staged": []}
    ways = {"direct": lambda: direct(d_s, d_r, n), "staged": lambda: staged(d_s, d_r, n, h_s, h_r)}
    for rnd in range(reps + 1):
        for name, fn in ways.items():
            t0 = time.perf_counter()
            got = fn()
            dt = time.perf_counter() - t0
            assert all(np.array_equal(a, b) for a, b in zip(got, want)), name
            if rnd:
                times[name].append(dt * 1e3)
    mb = n * 12 / 1e6
    for name, ts in times.items():
        print(f"{n_q}x{k} ({mb:.2f} MB) {name}: median {np.median(ts):.3f} ms, range {min(ts):.3f}-{max(ts):.3f} ms, "
              f"{mb / 1e3 / (np.median(ts) / 1e3):.1f} GB/s", flush=True)
