"""k_pf_finalize runs one CTA per frame with 256 threads.  At 64 registers or fewer four CTAs fit on an SM, so a 512-frame batch
is one wave on 132 SMs; a stack frame would put its per-lane arrays in local memory.  ptxas reports both without a GPU."""
import os
import re
import shutil
import subprocess

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(os.path.dirname(HERE), "pylinac_b200", "csrc")


def _nvcc():
    for cand in (shutil.which("nvcc"), os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "nvcc")):
        if cand and os.path.exists(cand):
            return cand
    return None


def test_finalize_kernel_fits_four_ctas_per_sm_without_stack(tmp_path):
    nvcc = _nvcc()
    if nvcc is None:
        pytest.skip("nvcc not found")
    out = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-fmad=false", "-std=c++17", "-Xptxas", "-v",
                          "-c", os.path.join(CSRC, "pf_finalize.cu"), "-o", str(tmp_path / "pf_finalize.o")],
                         capture_output=True, text=True)
    assert out.returncode == 0, out.stderr
    lines = out.stderr.splitlines()
    start = next(i for i, ln in enumerate(lines) if "Compiling entry function" in ln and "k_pf_finalize" in ln)
    block = "\n".join(lines[start:start + 4])
    frame = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", block)
    regs = re.search(r"Used (\d+) registers", block)
    assert frame and regs, block
    assert [int(x) for x in frame.groups()] == [0, 0, 0], block
    assert int(regs.group(1)) * 256 * 4 <= 65536, block
