"""SpecAugment on the GPU, measured: device times of b200feat_specaug (warp-and-copy, mean, mask fill) on recipe-shaped
batches with the bytes the algorithm needs computed from the shapes and the planned rectangles; `B200SpecAugment.forward`
against lhotse's `SpecAugment.forward` on the same CUDA tensor (alternated, each call ending in a synchronise); and one epoch of
K2SpeechRecognitionDataset + FusedOnTheFlyFeatures with each of the two modules as the input transform.  Needs a GPU and the
lhotse package (tests/refshim.py).  Prints one JSON line (and writes it to --out when given).

    python scripts/bench_specaugment.py [--launches 50] [--reps 5] [--cuts 300] [--out f.json]

Batches are N(-8, 2^2) noise padded with log(eps) past each cut's length (lengths uniform in 40-100 % of T, one supervision per
cut); the epoch runs over N(0, 0.1^2) PCM16 WAV cuts of 2-30 s in a temporary directory, 600 s batches."""
import argparse
import json
import os
import re
import statistics
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "scripts")]

from bench_flac import card, event_ms  # noqa: E402

import specaug_cases as SC  # noqa: E402

HBM_TBS = 3.35  # H100 SXM data sheet, not a measurement
SHAPES = [(200, 3000, 80), (600, 1000, 80)]


def batch(B, T, F, seed):
    rs = np.random.RandomState(seed)
    lens = rs.randint(int(0.4 * T), T + 1, size=B)
    lens[0] = T
    x = torch.from_numpy((rs.randn(B, T, F) * 2.0 - 8.0).astype(np.float32))
    for b, n in enumerate(lens):
        x[b, n:] = SC.LOG_EPSILON
    return x.cuda(), SC.one_segment_per_cut(lens.tolist())


def kernels(args, sa):
    from torch.profiler import ProfilerActivity, profile

    from lhotse_b200.engine import specaug

    res = {}
    for B, T, F in SHAPES:
        x, segs = batch(B, T, F, 1)
        SC.seed_all(1)
        warps, masks = sa.spec_augment_plan(sa.B200SpecAugment(), B, T, F, sa.clipped_segments(segs, B, T))
        out = torch.empty_like(x)
        run = lambda: specaug(x, out, warps, masks)  # noqa: E731
        for _ in range(3):
            run()
        a = out.clone()
        run()
        identical = bool(torch.equal(a.view(torch.int32), out.view(torch.int32)))
        total_ms = event_ms(run, args.launches)
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(args.launches):
                run()
            torch.cuda.synchronize()
        per = {}
        for ev in prof.key_averages():  # "void specaug_warp_kernel<4>(...)", "specaug_fill_kernel(...)"
            m = re.search(r"specaug_[a-z]+_kernel", ev.key)
            if m:
                per[m.group(0) + "_ms"] = round(per.get(m.group(0) + "_ms", 0.0) + ev.device_time_total / 1000.0 / args.launches, 4)
        assert len(per) == 3, per
        filled = int(np.sum((masks["end"] - masks["start"]).astype(np.int64) * np.where(masks["axis"] == 0, F, T)))
        nbytes = 8 * B * T * F + 4 * filled  # one read and one write of the batch, the rectangles written once more
        kernel_ms = sum(per.values())
        res[f"{B}x{T}x{F}"] = {
            "warps": int(len(warps)), "masks": int(len(masks)), "masked_fraction_written": round(filled / (B * T * F), 3),
            "call_ms_events": round(total_ms, 4), **per, "kernels_ms": round(kernel_ms, 4), "algorithmic_gbytes": round(nbytes / 1e9, 4),
            "achieved_gb_per_s_kernels": round(nbytes / kernel_ms / 1e6, 1) if kernel_ms else None,
            "share_of_datasheet_hbm_3.35TBs_kernels": round(nbytes / kernel_ms / 1e6 / (HBM_TBS * 1e3), 3) if kernel_ms else None,
            "achieved_gb_per_s_call": round(nbytes / total_ms / 1e6, 1), "runs_identical": identical}
    return res


def forward(args, sa, SpecAugment):
    res = {}
    for B, T, F in SHAPES:
        x, segs = batch(B, T, F, 2)
        mods = {"fused": sa.B200SpecAugment(), "lhotse": SpecAugment()}
        for m in mods.values():  # warm-up
            SC.seed_all(0)
            m(x, supervision_segments=segs)
        torch.cuda.synchronize()
        times = {k: [] for k in mods}
        for r in range(args.reps):
            for k, m in mods.items():
                SC.seed_all(10 + r)
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                y = m(x, supervision_segments=segs)
                torch.cuda.synchronize()
                times[k].append((time.perf_counter() - t0) * 1e3)
                del y
        assert mods["fused"].last_route == "fused"
        med = {k: statistics.median(v) for k, v in times.items()}
        res[f"{B}x{T}x{F}"] = {"reps": args.reps, "fused_ms_median": round(med["fused"], 3), "lhotse_ms_median": round(med["lhotse"], 3),
                               "lhotse_over_fused": round(med["lhotse"] / med["fused"], 1),
                               "fused_ms_all": [round(v, 3) for v in times["fused"]], "lhotse_ms_all": [round(v, 3) for v in times["lhotse"]]}
    return res


def epoch(args, sa, SpecAugment, lb_ex, tmp):
    import lhotse_env
    from lhotse.dataset import DynamicBucketingSampler, K2SpeechRecognitionDataset

    from lhotse_b200.input_strategies import FusedOnTheFlyFeatures

    rs = np.random.RandomState(0)
    cuts = lhotse_env.make_cutset(tmp, np.round(rs.uniform(2.0, 30.0, size=args.cuts), 2).tolist(), seed=1)
    hours = sum(c.duration for c in cuts) / 3600
    ext = lb_ex.B200Fbank(lb_ex.B200FbankConfig(device="cuda:0"))
    mods = {"fused": sa.B200SpecAugment(), "lhotse": SpecAugment(), "none": None}

    def run(aug):
        sampler = DynamicBucketingSampler(cuts, max_duration=600.0, num_buckets=5, shuffle=True, seed=0)
        ds = K2SpeechRecognitionDataset(input_strategy=FusedOnTheFlyFeatures(ext), input_transforms=[aug] if aug is not None else None)
        SC.seed_all(0)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        n = 0
        for batch_cuts in sampler:
            ds[batch_cuts]["inputs"]
            n += 1
        torch.cuda.synchronize()
        return time.perf_counter() - t0, n

    for aug in mods.values():  # warm-up: page cache, staging rings, allocator
        run(aug)
    times = {k: [] for k in mods}
    for _ in range(args.reps):
        for k, aug in mods.items():
            s, batches = run(aug)
            times[k].append(s)
    assert mods["fused"].last_route == "fused"
    med = {k: statistics.median(v) for k, v in times.items()}
    return {"cuts": args.cuts, "hours": round(hours, 3), "batches": batches, "max_duration_s": 600.0, "reps": args.reps,
            **{f"epoch_s_{k}_median": round(v, 3) for k, v in med.items()},
            **{f"epoch_s_{k}_all": [round(x, 3) for x in v] for k, v in times.items()},
            "specaugment_s_per_epoch_fused": round(med["fused"] - med["none"], 3),
            "specaugment_s_per_epoch_lhotse": round(med["lhotse"] - med["none"], 3)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--launches", type=int, default=50)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--cuts", type=int, default=300)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_specaugment.py measures on a GPU; none is visible")
    import importlib
    import pathlib

    import lhotse_env

    lb_ex = lhotse_env.setup_lhotse()
    import lhotse_b200.spec_augment as sa

    if not sa.HAVE_LHOTSE:
        importlib.reload(sa)
    from lhotse.dataset.signal_transforms import SpecAugment

    name, limit = card()
    res = {"bench": "specaugment", "gpu": name, "power_limit": limit, "kernels": kernels(args, sa), "forward": forward(args, sa, SpecAugment)}
    with tempfile.TemporaryDirectory() as d:
        res["epoch"] = epoch(args, sa, SpecAugment, lb_ex, pathlib.Path(d))
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
