"""The median networks of the PicketFence window kernels are Batcher sorting networks pruned to the wires that are read
(pf_win_common.cuh).  tests/pf_select_net_check.cu evaluates the compile-time comparator lists on the host, as the device applies
them, against sorted inputs: every 0/1 input up to 20 rows, random inputs with ties up to 32 rows, for the exact row counts
and for the symmetric padding of rank_keys."""
import os
import shutil
import subprocess

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))


def _nvcc():
    for cand in (shutil.which("nvcc"), os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "nvcc")):
        if cand and os.path.exists(cand):
            return cand
    return None


def test_pruned_median_networks_select_the_middles(tmp_path):
    nvcc = _nvcc()
    if nvcc is None:
        pytest.skip("nvcc not found")
    exe = str(tmp_path / "pf_select_net_check")
    subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O2", "-std=c++17", "-o", exe,
                    os.path.join(HERE, "pf_select_net_check.cu")], check=True, capture_output=True)
    out = subprocess.run([exe], capture_output=True, text=True)
    assert out.returncode == 0, out.stdout + out.stderr
    assert out.stdout.strip().endswith("ok")
    # the benchmark's 13-row leaves: 48 comparators of the sort, 27 full + 12 one-sided ones in the pruned network
    assert "N=13 sort 48 comparators, median 27 + 12 half" in out.stdout
