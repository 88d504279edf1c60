"""Host against device preparation of a text query batch: `python profiles/run_featurize_device.py [ROWS] [ROUNDS]`.

Bench corpus (synth.CORPUS_SEED, default 10M rows) resident; query batches of the bench stream (synth.QUERY_SEED, half
of them copies of corpus rows) of 1 ... 100k texts.  Per batch size and round, in one process and alternating, top-16:
  * ``host``   -- kv_featurize on the host threads, kv_query_upload (staging, classification, text order, copies +
                  table kernels: kv_index_last_prepare_ms), then the resident top-k copied back;
  * ``device`` -- kv_query_upload_text (text upload + featurisation, classification, text order, tables + copies back),
                  then the same top-k.
Prints the card and its power limit, the medians over the rounds after one warm-up round, and checks that both paths
return the same bits.  The crossover sets DEVICE_FEATURIZE_MIN_QUERIES (kakveda_b200/similarity.py, DESIGN §6)."""
import os
import subprocess
import sys
import time
from pathlib import Path

import numpy as np
import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
from kakveda_b200 import GfkbIndex, synth

n = int(sys.argv[1]) if len(sys.argv) > 1 else 10_000_000
rounds = int(sys.argv[2]) if len(sys.argv) > 2 else 5
sizes = [1, 16, 128, 512, 1024, 2048, 8192, 32768, 100_000]
k = 16
threads = min(64, os.cpu_count() or 1)
os.environ.setdefault("KAKVEDA_B200_THREADS", str(threads))

try:
    power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
except (OSError, subprocess.SubprocessError):
    power = "unknown"
print("card", torch.cuda.get_device_name(0), "power limit", power, "host threads", threads, flush=True)

buf, off = synth.signatures_packed(synth.CORPUS_SEED, 0, n)
ix = GfkbIndex()
fb = ix.vocab.featurize_packed(buf, off, 0, grow=True, n_threads=threads)
ix.add_features(fb)
fb.close()
del buf, off
ix.finalize()
qbuf, qoff = synth.signatures_packed(synth.QUERY_SEED, 0, max(sizes), dup_of_seed=synth.CORPUS_SEED, dup_rows=n)


def host(q):
    t0 = time.perf_counter()
    qfb = ix.vocab.featurize_packed(qbuf, qoff[:q + 1], 0, grow=False, n_threads=threads)
    t1 = time.perf_counter()
    ix.upload_queries(qfb)
    t2 = time.perf_counter()
    s, r = ix.topk_resident_host(q, k)
    t3 = time.perf_counter()
    qfb.close()
    return s, r, {"featurize": 1e3 * (t1 - t0), "upload": 1e3 * (t2 - t1), "split": ix.last_prepare_ms(),
                  "e2e": 1e3 * (t3 - t0)}


def device(q):
    t0 = time.perf_counter()
    ix.upload_text(qbuf, qoff[:q + 1], 0)
    t1 = time.perf_counter()
    s, r = ix.topk_resident_host(q, k)
    t2 = time.perf_counter()
    return s, r, {"upload_text": 1e3 * (t1 - t0), "split": ix.last_prepare_ms(), "e2e": 1e3 * (t2 - t0)}


def med(rows, key, i=None):
    return float(np.median([x[key] if i is None else x[key][i] for x in rows]))


for q in sizes:
    h, d = [], []
    for rnd in range(rounds + 1):
        sh, rh, th = host(q)
        sd, rd, td = device(q)
        assert np.array_equal(sh.view(np.uint32), sd.view(np.uint32)) and np.array_equal(rh, rd), f"results differ at {q}"
        if rnd:
            h.append(th)
            d.append(td)
    print(f"q={q:>6}  host: featurize {med(h, 'featurize'):8.3f}  upload {med(h, 'upload'):8.3f} "
          f"(staging {med(h, 'split', 0):.3f} classify {med(h, 'split', 1):.3f} order {med(h, 'split', 2):.3f} "
          f"copies+tables {med(h, 'split', 3):.3f})  e2e {med(h, 'e2e'):8.3f} ms | "
          f"device: upload_text {med(d, 'upload_text'):8.3f} (featurize {med(d, 'split', 0):.3f} "
          f"classify {med(d, 'split', 1):.3f} order {med(d, 'split', 2):.3f} tables+copies {med(d, 'split', 3):.3f})  "
          f"e2e {med(d, 'e2e'):8.3f} ms", flush=True)
print("card", torch.cuda.get_device_name(0), "power limit", power, flush=True)
