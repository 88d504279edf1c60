"""The bound kernel's per-block rare tables at a given corpus size: `python profiles/run_rare_table.py [ROWS]`.

Builds the bench corpus (synth.CORPUS_SEED, default 10M rows) and finalizes it, then prints the finalize time, the rare
(chunk, feature) block entries, the tables' slots and bytes (16 per slot, plus the 8 KB presence bitmap per 64-chunk block),
slots per entry, and how many tables the cuckoo insertion had to enlarge past load 0.4 (kv_index_layout counters
[14], [18], [19])."""
import subprocess
import sys
import time
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))


def main() -> None:
    import torch

    from kakveda_b200 import GfkbIndex, synth

    n = int(sys.argv[1]) if len(sys.argv) > 1 else 10_000_000
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
    t = time.perf_counter()
    ix.finalize()
    t = time.perf_counter() - t
    lay = ix.layout()
    blocks = -(-lay["chunks"] // 128) * 2   # 64-chunk blocks of the padded chunk count
    slots, entries = lay["rare_table_slots"], lay["rare_entries"]
    print(f"rows {n}: finalize {t:.2f} s; rare (chunk, feature) entries {entries:,}; table slots {slots:,}; tables {slots * 16 / 1e9:.3f} GB "
          f"+ bitmaps {blocks * 8192 / 1e9:.3f} GB; tables enlarged {lay['rare_tables_enlarged']} of {blocks}", flush=True)


if __name__ == "__main__":
    main()
