"""CPU check of the bound kernel's per-block two-choice rare tables as build_blocks writes them
(tests/cpp/rare_table_check.cu; host code only, nvcc is just the compiler)."""
import shutil
import subprocess
from pathlib import Path

REPO = Path(__file__).resolve().parent.parent


def test_rare_tables(tmp_path):
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    exe = tmp_path / "rare_table_check"
    src = REPO / "tests" / "cpp" / "rare_table_check.cu"
    subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O2", "-std=c++17", "--expt-relaxed-constexpr",
                    "-Xcompiler", "-pthread", "-w", "-o", str(exe), str(src)],
                   check=True, stdout=subprocess.PIPE, stderr=subprocess.STDOUT)
    out = subprocess.run([str(exe)], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert out.returncode == 0, out.stdout
    assert "all rare-table cases passed" in out.stdout
