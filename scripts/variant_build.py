"""Developer tool: builds extra copies of libb200feat.so with -D overrides into build_variants/ (git-ignored, but it
travels with gpurun), so that one GPU call can time several kernel variants (scripts/variant_bench.py).

    python scripts/variant_build.py name1:-DF512_PREFETCH=2 name2:-DF512_MEL_UNROLL=4,-DF512_SUM2=1 ...
"""
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from lhotse_b200 import build as B  # noqa: E402

OUT = os.path.join(ROOT, "build_variants")


def one(spec):
    name, _, flags = spec.partition(":")
    flags = [f for f in flags.split(",") if f]
    path = os.path.join(OUT, f"libb200feat_{name}.so")
    cmd = [B._nvcc(), *B.NVCC_FLAGS, *flags, "-o", path] + [os.path.join(B.CSRC, s) for s in B.SOURCES]
    res = subprocess.run(cmd, capture_output=True, text=True)
    if res.returncode != 0:
        return name, "FAILED\n" + res.stderr[-2000:]
    log = res.stdout + res.stderr
    regs = [ln for ln in log.splitlines() if "fast512_kernelILi0ELi400ELi8ELi4" in ln or "Used" in ln]
    # registers / spills of the headline instantiation (F32, L = 400, variant 0, plain log-mel)
    info = ""
    lines = log.splitlines()
    for i, ln in enumerate(lines):
        if "Compiling entry function" in ln and "fast512_kernelILi0ELi400ELi8ELi4ELi0ELi2ELb1E" in ln:
            info = " | ".join(x.strip() for x in lines[i + 1:i + 4])
    return name, info


if __name__ == "__main__":
    os.makedirs(OUT, exist_ok=True)
    with ThreadPoolExecutor(max_workers=4) as ex:
        for name, info in ex.map(one, sys.argv[1:]):
            print(name, "->", info)
