"""Build libkakveda_b200.so in-tree with nvcc for sm_90a (H100; no torch types cross the C ABI).

    python -m kakveda_b200.build [--force] [--verbose] [--scan-clocks]

The shared object lands in ``kakveda_b200/lib/`` (git-ignored build product).  ``__graft_entry__.build()``
calls :func:`build`.  ``--scan-clocks`` builds the measuring variant of the candidate scan
(``-DKV_SCAN_CLOCKS``) into ``libkakveda_b200_scanclocks.so`` next to the product library, which it leaves alone;
``profiles/run_scan_split.py`` loads it through ``KAKVEDA_B200_LIB``.
"""
from __future__ import annotations

import hashlib
import os
import shutil
import subprocess
import sys
from pathlib import Path

PKG = Path(__file__).resolve().parent
CSRC = PKG / "csrc"
LIBDIR = PKG / "lib"
LIB = LIBDIR / "libkakveda_b200.so"
STAMP = LIBDIR / "libkakveda_b200.stamp"

GENCODE = ["-gencode", "arch=compute_90a,code=sm_90a"]
NVCC_FLAGS = ["-O3", "-std=c++17", "-lineinfo", "-Xcompiler", "-fPIC,-O3,-pthread", "--expt-relaxed-constexpr"]


def _nvcc() -> str:
    for cand in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and Path(cand).exists():
            return cand
    raise RuntimeError("nvcc not found: kakveda_b200 has no CPU fallback and cannot be built without the CUDA toolkit")


def sources() -> list[Path]:
    return sorted(list(CSRC.glob("*.cu")) + list(CSRC.glob("*.cpp")))


SCAN_CLOCKS = dict(defines=("KV_SCAN_CLOCKS",), name="libkakveda_b200_scanclocks")


def _digest(defines: tuple[str, ...] = ()) -> str:
    h = hashlib.sha256()
    for p in sources() + sorted(CSRC.glob("*.h")) + sorted(CSRC.glob("*.cuh")) + [PKG.parent / "include" / "kakveda_b200.h"]:
        h.update(p.name.encode())
        h.update(p.read_bytes())
    h.update(" ".join(GENCODE + NVCC_FLAGS + [f"-D{d}" for d in defines]).encode())
    return h.hexdigest()


def is_current(defines: tuple[str, ...] = (), name: str = LIB.stem) -> bool:
    """Whether the library of that name was built from the present sources with these flags."""
    lib, stamp = LIBDIR / f"{name}.so", LIBDIR / f"{name}.stamp"
    return lib.exists() and stamp.exists() and stamp.read_text().strip() == _digest(defines)


def build(force: bool = False, verbose: bool = False, defines: tuple[str, ...] = (), name: str = LIB.stem) -> Path:
    """Compile the sources with ``-D<define>`` for each of `defines` into ``lib/<name>.so`` (objects under
    ``lib/obj/<name>/``); a library whose stamp matches the sources and flags is kept."""
    LIBDIR.mkdir(exist_ok=True)
    LIB, STAMP = LIBDIR / f"{name}.so", LIBDIR / f"{name}.stamp"
    dig = _digest(defines)
    if not force and is_current(defines, name):
        return LIB
    nvcc = _nvcc()
    objs = []
    objdir = LIBDIR / "obj" / name
    objdir.mkdir(parents=True, exist_ok=True)
    procs = []
    for src in sources():
        obj = objdir / (src.stem + ".o")
        cmd = [nvcc, *GENCODE, *NVCC_FLAGS, *[f"-D{d}" for d in defines], "-x", "cu", "-c", str(src), "-o", str(obj)]
        if verbose:
            cmd.insert(1, "-Xptxas=-v")
            print(" ".join(cmd), flush=True)
        procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
        objs.append(str(obj))
    failed = False
    for src, p in procs:
        out, _ = p.communicate()
        if p.returncode != 0 or verbose:
            sys.stderr.write(f"--- {src.name}\n{out}\n")
        failed |= p.returncode != 0
    if failed:
        raise RuntimeError("nvcc failed (see output above)")
    cmd = [nvcc, *GENCODE, "-shared", "-o", str(LIB), *objs, "-lcudart_static", "-lpthread", "-ldl", "-lrt"]
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if r.returncode != 0:
        sys.stderr.write(r.stdout)
        raise RuntimeError("link failed")
    STAMP.write_text(dig)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="--verbose" in sys.argv, **(SCAN_CLOCKS if "--scan-clocks" in sys.argv else {})))
