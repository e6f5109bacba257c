"""Precomputed features with CutMix, measured: lhotse's PrecomputedFeatures (collate_features with its host FeatureMixer, then
`.to("cuda")` and a synchronise) against FusedPrecomputedFeatures (one H2D copy of the stored rows, the three feature-mix
kernels, a synchronise) on the same batches, alternated in one process after a warm-up of every batch, median of --reps; the
device times of the energy, gain and output kernels (torch.profiler, a separate pass), the H2D bytes, and the largest
difference of each route to the float64 truth (lhotse's own code with the stored rows read as float64).  Needs a GPU and the
lhotse package (tests/refshim.py).  Prints one JSON line (and writes it to --out when given).

    python scripts/bench_precomputed.py [--cuts 512] [--batches 2] [--reps 5] [--workers 8] [--out f.json]

Workload: 10-15 s cuts of seeded log-mel-like Fbank-80 rows at 100 frames/s and a 200-cut noise set of 2-20 s in one
b200_archive under a temporary directory (page-cached: written just before), CutMix(p=0.5, snr=(10, 20)) drawn once per
batch and shared by both routes."""
import argparse
import json
import os
import statistics
import sys
import tempfile
import time
from pathlib import Path

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "scripts")]

from bench_flac import card  # noqa: E402

import featmix_cases as FC  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cuts", type=int, default=512)
    ap.add_argument("--batches", type=int, default=2)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--workers", type=int, default=8)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_precomputed needs a GPU"
    import lhotse_env

    lhotse_env.setup_lhotse()
    from lhotse import CutSet
    from lhotse.dataset import CutMix
    from lhotse.dataset.input_strategies import PrecomputedFeatures

    import lhotse_b200 as lb
    from lhotse_b200.precomputed import FeatureStagingRing, precomputed_plan

    name, limit = card()
    tmp = Path(tempfile.mkdtemp(prefix="bench_precomputed_"))
    rs = np.random.RandomState(0)
    speech = FC.make_cuts(tmp / "feats", list(rs.randint(1000, 1501, size=args.cuts * args.batches)), seed=1)
    noise = FC.make_cuts(tmp / "feats", list(rs.randint(200, 2001, size=200)), seed=2, prefix="n", supervisions=False)
    cutmix = CutMix(noise, p=0.5, snr=(10, 20), seed=3)
    sp = list(speech)
    batches = [cutmix(CutSet.from_cuts(sp[b * args.cuts: (b + 1) * args.cuts])) for b in range(args.batches)]
    hours = [sum(c.duration for c in b) / 3600 for b in batches]
    ref = PrecomputedFeatures(num_workers=args.workers)
    ours = lb.FusedPrecomputedFeatures(num_workers=args.workers)
    dev = torch.device("cuda", torch.cuda.current_device())

    def run_ref(b):
        t = time.perf_counter()
        feats, _ = ref(b)
        feats = feats.to(dev)
        torch.cuda.synchronize()
        return time.perf_counter() - t, feats

    def run_ours(b):
        t = time.perf_counter()
        feats, _ = ours(b)
        torch.cuda.synchronize()
        return time.perf_counter() - t, feats

    worst = {"reference": 0.0, "archive": 0.0}
    for b in batches:  # warm-up of every shape, and the differences to the float64 truth
        _, r = run_ref(b)
        _, g = run_ours(b)
        assert ours.last_batch_route == "archive", ours.last_decline
        l32, _, truth = FC.lhotse_pair(b)
        truth = truth.numpy()
        FC.check_gate(g.cpu().numpy(), l32.numpy(), truth, "bench")
        worst["reference"] = max(worst["reference"], float(np.abs(r.cpu().numpy() - truth).max()))
        worst["archive"] = max(worst["archive"], float(np.abs(g.cpu().numpy() - truth).max()))
    t_ref, t_ours = [], []
    for _ in range(args.reps):
        a = b = 0.0
        for bt in batches:
            a += run_ref(bt)[0]
            b += run_ours(bt)[0]
        t_ref.append(a)
        t_ours.append(b)
    total_h = sum(hours)
    med_ref, med_ours = statistics.median(t_ref), statistics.median(t_ours)

    # kernel device times and H2D bytes of one batch, in a pass of their own
    from torch.profiler import ProfilerActivity, profile

    plan = precomputed_plan(batches[0])
    ring = FeatureStagingRing()
    staged, tracks = ring.stage(plan)
    h2d = int(staged.numel()) * 4
    src = staged.to(dev)
    out = torch.empty((len(plan.cuts), plan.T, plan.F), dtype=torch.float32, device=dev)
    for _ in range(3):
        lb.engine.feature_mix(src, tracks, plan.cuts, out, lb.LOG_EPSILON)
    torch.cuda.synchronize()
    n = 20
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(n):
            lb.engine.feature_mix(src, tracks, plan.cuts, out, lb.LOG_EPSILON)
        torch.cuda.synchronize()
    kern = {}
    for ev in prof.key_averages():
        for k in ("featmix_energy_kernel", "featmix_gain_kernel", "featmix_out_kernel"):
            if k in ev.key:
                kern[k] = round(ev.device_time_total / 1000.0 / n, 4)
    res = {
        "card": name, "power_limit": limit, "cuts_per_batch": args.cuts, "batches": args.batches, "reps": args.reps,
        "workers": args.workers, "hours_of_audio": round(total_h, 4),
        "mixed_cuts_first_batch": int((plan.cuts["mode"] == 1).sum()),
        "lhotse_s": round(med_ref, 4), "fused_s": round(med_ours, 4),
        "lhotse_hours_per_s": round(total_h / med_ref, 3), "fused_hours_per_s": round(total_h / med_ours, 3),
        "speedup": round(med_ref / med_ours, 2),
        "kernel_ms_per_batch": kern, "h2d_bytes_per_batch": h2d,
        "output_bytes_per_batch": int(out.numel()) * 4,
        "max_abs_diff_to_float64_truth": worst,
        "times_lhotse_s": [round(t, 4) for t in t_ref], "times_fused_s": [round(t, 4) for t in t_ours],
    }
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
