"""Forward plus backward of B200WhisperFbank on the GPU, measured: whisper-fbank-80 on one (B, 480000) float32 batch of
30 s cuts (Whisper's window), the input requiring grad, `extract_batch` then `backward` of a weighted sum of the features,
timed with CUDA events, median of --reps; the backward alone is timed too (`torch.autograd.grad` on a graph built
beforehand).  Alternated with the float32 torch chain of lhotse's `log_mel_spectrogram` (tests/whisper_backward_cases
.features_t, the same ops) under autograd on the same GPU, cut by cut, which is what lhotse's WhisperFbank(device="cuda")
does.  Prints the card name and power limit and one JSON line, and writes it to --out when given
(profiles/h100_whisper_backward.json is one such run).

    python scripts/bench_whisper_backward.py [--batches 32,64,128] [--reps 5] [--out f.json]"""
import argparse
import json
import os
import statistics
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "scripts")]

from bench_backward import timed  # noqa: E402
from bench_flac import card  # noqa: E402

import whisper_backward_cases as WB  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", default="32,64,128")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_whisper_backward needs a GPU"
    import lhotse_b200 as lb

    name, limit = card()
    print(f"card: {name}, power limit {limit}")
    ext = lb.B200WhisperFbank(lb.B200WhisperFbankConfig(device="cuda"))
    n = 480000
    res = {"bench": "whisper-fbank-80 forward + backward, (B, 480000) float32 batch", "card": name, "power_limit": limit,
           "rows": []}
    for B in [int(b) for b in args.batches.split(",")]:
        rs = np.random.RandomState(B)
        X = torch.from_numpy((0.1 * rs.randn(B, n)).astype(np.float32)).cuda()
        W = torch.randn((B, 3000, 80), device="cuda", generator=torch.Generator("cuda").manual_seed(0))

        def b200():
            x = X.clone().requires_grad_(True)
            (ext.extract_batch(x, 16000) * W).sum().backward()
            return x.grad

        def oracle():
            x = X.clone().requires_grad_(True)
            out = torch.stack([WB.features_t(x[i]) for i in range(B)])
            (out * W).sum().backward()
            return x.grad

        x_bwd = X.clone().requires_grad_(True)
        loss = (ext.extract_batch(x_bwd, 16000) * W).sum()

        def b200_backward():
            return torch.autograd.grad(loss, x_bwd, retain_graph=True)

        g_b, g_o = b200(), oracle()
        rel = float((g_b - g_o).norm() / g_o.norm())
        for _ in range(2):
            b200(), oracle(), b200_backward()
        tb, to, tbb = [], [], []
        for _ in range(args.reps):  # alternated
            tb += timed(b200, 1)
            to += timed(oracle, 1)
            tbb += timed(b200_backward, 1)
        row = {"B": B, "b200_ms": statistics.median(tb), "b200_ms_min": min(tb), "b200_backward_ms": statistics.median(tbb),
               "torch_fp32_autograd_ms": statistics.median(to), "speedup": statistics.median(to) / statistics.median(tb),
               "rel_diff_vs_torch_fp32": rel}
        res["rows"].append(row)
        print(json.dumps(row))
        del loss, x_bwd
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
