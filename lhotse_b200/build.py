"""In-tree build of the CUDA library (sm_90a only).  `python -m lhotse_b200.build`."""
from __future__ import annotations

import os
import shutil
import subprocess
import sys

PKG_DIR = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(PKG_DIR, "csrc")
LIB_PATH = os.path.join(PKG_DIR, "libb200feat.so")
SOURCES = ["b200feat.cu"]
HEADERS = ["common.cuh", "generic.cuh", "fast512.cuh", "tc512.cuh", "fast256.cuh", "fast2048.cuh", "fast1024.cuh", "fast400.cuh", "flac.cuh", "mix.cuh", "resample.cuh", "reverb.cuh", "specaug.cuh", "rirgen.cuh", "featmix.cuh", "backward.cuh", "collate.cuh", "wpe.cuh", os.path.join("..", "..", "include", "b200feat.h")]

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-O3", "-lineinfo", "-std=c++17",
    "-Xcompiler", "-fPIC", "-Xcompiler", "-mavx2", "-shared",
    "-Xptxas", "-v",
]


def _nvcc() -> str:
    for cand in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found: the b200feat CUDA library cannot be built")


def needs_build() -> bool:
    if not os.path.exists(LIB_PATH):
        return True
    t = os.path.getmtime(LIB_PATH)
    deps = [os.path.join(CSRC, s) for s in SOURCES + HEADERS]
    return any(os.path.getmtime(d) > t for d in deps if os.path.exists(d))


def build(force: bool = False, verbose: bool = False) -> str:
    if not force and not needs_build():
        return LIB_PATH
    cmd = [_nvcc(), *NVCC_FLAGS, "-o", LIB_PATH] + [os.path.join(CSRC, s) for s in SOURCES]
    res = subprocess.run(cmd, capture_output=True, text=True)
    if res.returncode != 0:
        raise RuntimeError("nvcc failed:\n" + res.stdout + res.stderr)
    log = res.stdout + res.stderr
    with open(os.path.join(PKG_DIR, "csrc", "ptxas.log"), "w") as f:
        f.write(log)
    if verbose:
        print(log)
    return LIB_PATH


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose=True))
