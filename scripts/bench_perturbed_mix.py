"""MixedCuts with speed-perturbed tracks mixed on the GPU (`perturbed_tracks=True`), measured: the transform stages, the
energies and gains, the mix and the fbank kernel on the same recipe-shaped batch, and FusedOnTheFlyFeatures over such batches
on the "mix" route against the float route (alternated in one process, features compared).  Prints one JSON line (and
writes it to --out when given).

    python scripts/bench_perturbed_mix.py [--cuts 2048] [--launches 20] [--otf-cuts 512] [--otf-reps 5] [--threads 8] [--out f.json]

Speech is N(0, 0.2^2) PCM16 WAV noise (eight 30 s files), the noise four PCM16 WAV files; cuts are 10-30 s slices, a third
at speed 0.9, a third at 1.1, a third plain (the LibriSpeech recipe's `cuts + perturb_speed(0.9) + perturb_speed(1.1)`), with
CutMix(p=0.5, snr=(10, 20), pad_to_longest=True).  Files live in a temporary directory and are read from the page cache."""
import argparse
import json
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


def recipe_batch(tmp, n, seed):
    import lhotse_env
    from lhotse import CutSet
    from lhotse.dataset.cut_transforms import CutMix

    rs = np.random.RandomState(seed)
    speech = lhotse_env.make_cutset(tmp, [30.0] * 8, seed=4, amp=0.2, prefix=f"s{seed}_")
    noise = lhotse_env.make_cutset(tmp, [7.3, 12.1, 30.0, 4.4], seed=5, amp=0.05, supervisions=False, prefix=f"n{seed}_")
    cuts = []
    for i in range(n):
        d = float(np.round(rs.uniform(10.0, 30.0), 3))
        a = float(np.round(rs.uniform(0.0, 30.0 - d), 3))
        c = speech[i % 8].truncate(offset=a, duration=d, preserve_id=False).with_id(f"c{seed}_{i}")
        cuts.append(c.perturb_speed(0.9) if i % 3 == 0 else c.perturb_speed(1.1) if i % 3 == 1 else c)
    return CutSet.from_cuts(list(CutMix(noise, p=0.5, snr=(10, 20), seed=seed, pad_to_longest=True, preserve_id=True)(
        CutSet.from_cuts(cuts))))


def kernels(args, lb_ex, tmp):
    from lhotse_b200.engine import MIX_SRC_F32, mix
    from lhotse_b200.pcm_staging import MixStagingRing, mix_requests_for_batch, transform_staged

    cuts = list(recipe_batch(tmp, args.cuts, 1))
    reqs = mix_requests_for_batch(cuts, perturbed_tracks=True)
    assert reqs is not None
    ring = MixStagingRing()
    t0 = time.perf_counter()
    batch, lens, offs, sr = ring.stage(reqs)
    stage_s = time.perf_counter() - t0
    dev = torch.device("cuda:0")
    ext = lb_ex.B200Fbank(lb_ex.B200FbankConfig(device="cuda:0"))
    eng = ext.engine
    src0 = batch.pcm.to(dev)
    src2 = transform_staged(batch.transform, dev, handle=eng._h)[0]  # also uploads the rate pairs' tables once
    transform_ms = event_ms(lambda: transform_staged(batch.transform, dev, handle=eng._h), args.launches)
    out = torch.zeros(batch.out_elems, dtype=torch.float32, device=dev)
    tracks, cut_tab = batch.tracks.copy(), batch.cuts.copy()
    energy_only = cut_tab.copy()
    energy_only["target_len"] = 0  # the mix kernel then has nothing to write: the energy kernel alone
    both_ms = event_ms(lambda: mix(src0, None, tracks, cut_tab, out, src2=src2), args.launches)
    energy_ms = event_ms(lambda: mix(src0, None, tracks, energy_only, out, src2=src2), args.launches)
    eng.extract_device(out, lens, offsets=offs)
    fbank_ms = event_ms(lambda: eng.extract_device(out, lens, offsets=offs), args.launches)
    return {"cuts": len(cuts), "mixed_cuts": sum(getattr(c, "tracks", None) is not None for c in cuts),
            "tracks": int(len(tracks)), "float32_tracks": int((tracks["source"] == MIX_SRC_F32).sum()),
            "hours": round(sum(lens) / 16000 / 3600, 3), "stage_s": round(stage_s, 3),
            "transform_ms": round(transform_ms, 3), "energy_ms": round(energy_ms, 3), "mix_ms": round(both_ms - energy_ms, 3),
            "energy_plus_mix_ms": round(both_ms, 3), "fbank_ms": round(fbank_ms, 3)}


def on_the_fly(args, lb_ex, tmp):
    from lhotse_b200.input_strategies import FusedOnTheFlyFeatures

    ext = lb_ex.B200Fbank(lb_ex.B200FbankConfig(device="cuda:0"))
    batches = [recipe_batch(tmp, args.otf_cuts, 10 + k) for k in range(2)]
    hours = [sum(c.duration for c in b) / 3600 for b in batches]
    fast = FusedOnTheFlyFeatures(ext, num_workers=args.threads, perturbed_tracks=True)
    slow = FusedOnTheFlyFeatures(ext, num_workers=args.threads, pcm16_fast_path=False)
    for b in batches:  # warm-up: page cache, rings, resampler tables, allocator
        fast(b), slow(b)
    rates = {"mix": [], "float": []}
    for r in range(args.otf_reps):
        for name, strat in (("mix", fast), ("float", slow)):
            b = batches[r % 2]
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            feats, lens = strat(b)
            torch.cuda.synchronize()
            rates[name].append(hours[r % 2] / (time.perf_counter() - t0))
        assert fast.last_batch_route == "mix" and slow.last_batch_route == "float"
    f1, l1 = fast(batches[0])
    f2, l2 = slow(batches[0])
    equal = bool(torch.equal(f1, f2) and torch.equal(l1, l2))
    assert equal, "the perturbed mix route's features differ from the float route's"
    med = {k: statistics.median(v) for k, v in rates.items()}
    return {"otf_cuts": args.otf_cuts, "threads": args.threads, "reps": args.otf_reps,
            "mix_hours_per_s": round(med["mix"], 2), "float_hours_per_s": round(med["float"], 2),
            "mix_over_float": round(med["mix"] / med["float"], 2), "all_mix": [round(x, 2) for x in rates["mix"]],
            "all_float": [round(x, 2) for x in rates["float"]], "features_equal": equal}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cuts", type=int, default=2048)
    ap.add_argument("--launches", type=int, default=20)
    ap.add_argument("--otf-cuts", type=int, default=512)
    ap.add_argument("--otf-reps", type=int, default=5)
    ap.add_argument("--threads", type=int, default=8)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import lhotse_env
    import transform_cases

    lb_ex = lhotse_env.setup_lhotse()
    name, limit = card()
    res = {"bench": "perturbed_mix", "gpu": name, "power_limit": limit}
    with tempfile.TemporaryDirectory() as d, transform_cases.torch_resampler():
        import pathlib

        tmp = pathlib.Path(d)
        res.update(kernels(args, lb_ex, tmp))
        res.update(on_the_fly(args, lb_ex, tmp))
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
