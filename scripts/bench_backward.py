"""Forward plus backward of B200Fbank on the GPU, measured: fbank-80 at 16 kHz on one (B, n) batch of 10 s cuts, the input
requiring grad, `extract_batch` then `backward` of a weighted sum of the features, timed with CUDA events; alternated with
the oracle's float32 torch chain (tests/backward_cases.features_t: the same arithmetic as lhotse's modules) under autograd on
the same GPU, cut by cut.  Prints the card name and power limit and one JSON line, and writes it to --out when given
(profiles/h100_backward.json is one such run).

    python scripts/bench_backward.py [--batches 64,128,256] [--reps 10] [--out f.json]"""
import argparse
import json
import os
import statistics
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "scripts")]

from bench_flac import card  # noqa: E402

import backward_cases as BC  # noqa: E402


def timed(fn, reps):
    out = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        out.append(a.elapsed_time(b))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", default="64,128,256")
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_backward needs a GPU"
    import lhotse_b200 as lb

    name, limit = card()
    print(f"card: {name}, power limit {limit}")
    ext = lb.B200Fbank(lb.B200FbankConfig(device="cuda"))
    cfg = BC.cfg_of("fbank")
    n = 160000
    res = {"bench": "fbank-80 forward + backward, (B, 160000) float32 batch", "card": name, "power_limit": limit, "rows": []}
    for B in [int(b) for b in args.batches.split(",")]:
        rs = np.random.RandomState(B)
        X = torch.from_numpy((0.1 * rs.randn(B, n)).astype(np.float32)).cuda()
        W = None

        def b200():
            nonlocal W
            x = X.clone().requires_grad_(True)
            out = ext.extract_batch(x, 16000)
            if W is None:
                W = torch.randn(out.shape, device="cuda", generator=torch.Generator("cuda").manual_seed(0))
            (out * W).sum().backward()
            return x.grad

        def oracle():
            x = X.clone().requires_grad_(True)
            out = torch.stack([BC.features_t(x[i], cfg) for i in range(B)])
            (out * W).sum().backward()
            return x.grad

        g_b, g_o = b200(), oracle()
        rel = float((g_b - g_o).norm() / g_o.norm())
        for _ in range(2):
            b200(), oracle()
        tb, to = [], []
        for _ in range(args.reps):  # alternated
            tb += timed(b200, 1)
            to += timed(oracle, 1)
        row = {"B": B, "b200_ms": statistics.median(tb), "b200_ms_min": min(tb), "torch_fp32_autograd_ms": statistics.median(to),
               "speedup": statistics.median(to) / statistics.median(tb), "rel_diff_vs_torch_fp32": rel}
        res["rows"].append(row)
        print(json.dumps(row))
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
