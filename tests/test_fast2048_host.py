"""The FFT stages of csrc/fast2048.cuh and csrc/fast1024.cuh are `__host__ __device__`, the mel packers (balanced 12-tap work items;
whole-filter rounds with their over-read clamp) are host code: this test compiles scripts/micro/f2k_host_check.cu (only its host side
is executed) and runs the 32 emulated lanes against a float64 DFT and the packers against a dense (K x M) mel product — the index
arithmetic of the kernels is checked without a GPU."""
import os
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _nvcc():
    return shutil.which("nvcc") or ("/usr/local/cuda/bin/nvcc" if os.path.exists("/usr/local/cuda/bin/nvcc") else None)


@pytest.mark.skipif(_nvcc() is None, reason="nvcc not found")
def test_fast2048_stages_on_the_host(tmp_path):
    exe = str(tmp_path / "f2k_host_check")
    src = os.path.join(ROOT, "scripts", "micro", "f2k_host_check.cu")
    res = subprocess.run([_nvcc(), "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-o", exe, src], capture_output=True, text=True)
    assert res.returncode == 0, res.stderr[-2000:]
    for args in ([], ["1200", "128"], ["1102", "40"], ["2047", "23"]):
        run = subprocess.run([exe, *args], capture_output=True, text=True)
        assert run.returncode == 0, run.stdout + run.stderr
        assert "0 bad" in run.stdout
