"""Reverberated cuts on the GPU (`reverb=True`), measured: per-kernel device times of b200feat_reverb (RIR spectra,
convolution, gain, output) against the fbank kernel on the same output, with the algorithmic FLOPs and bytes of the
convolution computed from the shapes; and FusedOnTheFlyFeatures(reverb=True) on the "transform" route against the float route
(alternated in one process), on reverb-only batches and on recipe batches (speed 0.9 / 1.0 / 1.1, CutMix p = 0.5, then the
reverb: the "mix" route with perturbed_tracks=True).  Prints one JSON line (and writes it to --out when given).

    python scripts/bench_reverb.py [--cuts 2048] [--otf-cuts 512] [--otf-reps 5] [--threads 8] [--out f.json]

Speech is N(0, 0.2^2) PCM16 WAV noise (eight 30 s files); cuts are 10-30 s slices; each cut is reverberated with p = 0.5
(lhotse's ReverbWithImpulseResponse cut transform) with one of 100 decaying-noise RIRs of 0.3-1 s.  Files live in a
temporary directory and are read from the page cache."""
import argparse
import json
import math
import os
import statistics
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "scripts")]

from bench_flac import card, event_ms  # noqa: E402

F, B = 4096, 2048  # csrc/reverb.cuh RV_F, RV_B


def recipe_batch(tmp, n, seed, recipe=False):
    import lhotse_env
    import reverb_cases as RC
    from lhotse import CutSet, Recording
    from lhotse.audio import AudioSource
    from lhotse.dataset.cut_transforms import CutMix, ReverbWithImpulseResponse

    rs = np.random.RandomState(seed)
    speech = lhotse_env.make_cutset(tmp, [30.0] * 8, seed=4, amp=0.2, prefix=f"s{seed}_")
    rirs = []
    for k in range(100):
        m = int(rs.uniform(0.3, 1.0) * 16000)
        p = tmp / f"rir{seed}_{k}.wav"
        RC.write_wav(p, RC.decaying_rir(m, seed=1000 * seed + k))
        rirs.append(Recording(id=f"rir{seed}_{k}", sources=[AudioSource(type="file", channels=[0], source=str(p))],
                              sampling_rate=16000, num_samples=m, duration=m / 16000))
    cuts = []
    for i in range(n):
        d = float(np.round(rs.uniform(10.0, 30.0), 3))
        a = float(np.round(rs.uniform(0.0, 30.0 - d), 3))
        c = speech[i % 8].truncate(offset=a, duration=d, preserve_id=False).with_id(f"c{seed}_{i}")
        if recipe:  # the LibriSpeech recipe's speed perturbation
            c = c.perturb_speed(0.9) if i % 3 == 0 else c.perturb_speed(1.1) if i % 3 == 1 else c
        cuts.append(c)
    cuts = CutSet.from_cuts(cuts)
    if recipe:
        noise = lhotse_env.make_cutset(tmp, [7.3, 12.1, 30.0, 4.4], seed=5, amp=0.05, supervisions=False, prefix=f"n{seed}_")
        cuts = CutSet.from_cuts(list(CutMix(noise, p=0.5, snr=(10, 20), seed=seed, pad_to_longest=True, preserve_id=True)(cuts)))
    return CutSet.from_cuts(list(ReverbWithImpulseResponse(rirs, p=0.5, randgen=__import__("random").Random(seed))(cuts)))


def kernels(args, lb_ex, tmp):
    from torch.profiler import ProfilerActivity, profile

    from lhotse_b200.engine import reverb
    from lhotse_b200.pcm_staging import TransformStagingRing, transform_requests_for_batch, transform_staged

    cuts = list(recipe_batch(tmp, args.cuts, 1))
    reqs = transform_requests_for_batch(cuts, reverb=True)
    assert reqs is not None
    ring = TransformStagingRing()
    t0 = time.perf_counter()
    batch, lens, offs, sr = ring.stage(reqs)
    stage_s = time.perf_counter() - t0
    dev = torch.device("cuda:0")
    ext = lb_ex.B200Fbank(lb_ex.B200FbankConfig(device="cuda:0"))
    eng = ext.engine
    out = transform_staged(batch, dev, handle=eng._h)[0]
    src0 = batch.pcm.to(dev)
    mid = torch.empty(batch.mid_elems, dtype=torch.float32, device=dev)
    from lhotse_b200.engine import resample

    resample(src0, None, mid, batch.stages, out)
    rirs, rcuts = batch.reverb_rirs.copy(), batch.reverb_cuts.copy()
    run = lambda: reverb(src0, None, mid, rirs, rcuts, out, eng._h)  # noqa: E731
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
    for ev in prof.key_averages():
        if ev.key.startswith("reverb_"):
            per[ev.key.split("(")[0] + "_ms"] = round(ev.device_time_total / 1000.0 / args.launches, 3)
    # the same cuts against one RIR at the 65536-sample cap (32 partitions): the convolution's worst case
    rs = np.random.RandomState(0)
    long_q = torch.from_numpy((rs.randn(65536) * np.exp(-np.arange(65536) / 9830.0) * 12000).astype(np.int16)).to(dev)
    long_rirs = rirs[:1].copy()
    long_rirs["source"], long_rirs["src_elem"], long_rirs["num_samples"] = 0, 0, 65536
    long_cuts = rcuts.copy()
    long_cuts["rir"] = 0
    long_ms = event_ms(lambda: reverb(long_q, None, mid, long_rirs, long_cuts, out, eng._h), max(2, args.launches // 5))
    eng.extract_device(out, lens, offsets=offs)
    fbank_ms = event_ms(lambda: eng.extract_device(out, lens, offsets=offs), args.launches)
    # algorithmic work of the convolution kernel, from the shapes: per CTA, one forward FFT per live partition, one inverse
    # FFT, and a complex multiply-accumulate (8 flops) per bin per live partition; a radix-2 FFT of F points is 5 F log2 F
    R = rirs["num_samples"][rcuts["rir"]]
    N = rcuts["in_len"]
    ctas = (N + 2 * B - 1) // (2 * B)
    P = (R + B - 1) // B
    fft = 5 * F * math.log2(F)
    conv_flops = float(np.sum(ctas * ((P + 1) * fft + P * 8 * F)))
    conv_bytes = float(np.sum(N) * 8 + np.sum(ctas * P) * F * 8)  # x in, y out, the spectra each CTA reads
    conv_ms = per.get("reverb_conv_kernel_ms", float("nan"))
    return {"cuts": len(cuts), "reverberated": int(len(rcuts)), "rirs": int(len(rirs)), "hours": round(sum(lens) / 16000 / 3600, 3),
            "reverb_hours": round(float(np.sum(N)) / 16000 / 3600, 3), "stage_s": round(stage_s, 3),
            "reverb_total_ms": round(total_ms, 3), **per, "reverb_total_ms_rir_65536": round(long_ms, 3), "fbank_ms": round(fbank_ms, 3),
            "conv_gflop": round(conv_flops / 1e9, 2), "conv_gbytes": round(conv_bytes / 1e9, 3),
            "conv_tflops_achieved": round(conv_flops / conv_ms / 1e9, 2) if conv_ms == conv_ms else None,
            "runs_identical": identical}


def on_the_fly(args, lb_ex, tmp, recipe=False):
    from lhotse_b200.input_strategies import FusedOnTheFlyFeatures

    ext = lb_ex.B200Fbank(lb_ex.B200FbankConfig(device="cuda:0"))
    batches = [recipe_batch(tmp, args.otf_cuts, 10 + k + 10 * recipe, recipe) for k in range(2)]
    hours = [sum(c.duration for c in b) / 3600 for b in batches]
    route = "mix" if recipe else "transform"
    fast = FusedOnTheFlyFeatures(ext, num_workers=args.threads, reverb=True, perturbed_tracks=recipe)
    slow = FusedOnTheFlyFeatures(ext, num_workers=args.threads, pcm16_fast_path=False)
    for b in batches:  # warm-up: page cache, rings, allocator
        fast(b), slow(b)
    rates = {route: [], "float": []}
    for r in range(args.otf_reps):
        for name, strat in ((route, fast), ("float", slow)):
            b = batches[r % 2]
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            strat(b)
            torch.cuda.synchronize()
            rates[name].append(hours[r % 2] / (time.perf_counter() - t0))
        assert fast.last_batch_route == route and slow.last_batch_route == "float"
    f1, l1 = fast(batches[0])
    f2, l2 = slow(batches[0])
    assert torch.equal(l1, l2)
    med = {k: statistics.median(v) for k, v in rates.items()}
    k = "recipe_" if recipe else ""
    return {f"{k}otf_cuts": args.otf_cuts, "threads": args.threads, "reps": args.otf_reps, f"{k}route": route,
            f"{k}staged_hours_per_s": round(med[route], 2), f"{k}float_hours_per_s": round(med["float"], 2),
            f"{k}staged_over_float": round(med[route] / med["float"], 2),
            f"{k}all_staged": [round(x, 2) for x in rates[route]], f"{k}all_float": [round(x, 2) for x in rates["float"]],
            f"{k}max_feature_diff": float((f1 - f2).abs().max())}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cuts", type=int, default=2048)
    ap.add_argument("--launches", type=int, default=10)
    ap.add_argument("--otf-cuts", type=int, default=512)
    ap.add_argument("--otf-reps", type=int, default=5)
    ap.add_argument("--threads", type=int, default=8)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import lhotse_env
    import transform_cases

    lb_ex = lhotse_env.setup_lhotse()
    name, limit = card()
    res = {"bench": "reverb", "gpu": name, "power_limit": limit}
    with tempfile.TemporaryDirectory() as d, transform_cases.torch_resampler():
        import pathlib

        tmp = pathlib.Path(d)
        res.update(kernels(args, lb_ex, tmp))
        res.update(on_the_fly(args, lb_ex, tmp))
        res.update(on_the_fly(args, lb_ex, tmp, recipe=True))
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
