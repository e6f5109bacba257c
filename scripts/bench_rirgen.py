"""The RIR generator on the GPU (`generated_rir=True`), measured: the host draws per RIR (rir_draws.draw, lhotse's NumPy
draws and the restated multinomial), the per-kernel device times of b200feat_rir_generate (entries, segmented sort, window,
biquad) and of the b200feat_resample stage that takes its output to sr, for batches of 256 and 1024 RIRs at 16 kHz with
lhotse's default generator (T60 ~ U(0.1, 0.8)), and lhotse's own generator on the host for comparison; then
FusedOnTheFlyFeatures(generated_rir=True) on the "transform" route against the float route with one torch thread (where
lhotse's comb keeps the last image at a shared position, as this route does), alternated in one process, median of --otf-reps,
on batches of --otf-cuts cuts of 5-15 s reverberated with p = 0.5 by lhotse's ReverbWithImpulseResponse cut transform with no
RIR corpus, and the largest log-mel difference between the two on one batch drawn from the same states.  Prints one JSON line
(and writes it to --out when given).

    python scripts/bench_rirgen.py [--launches 10] [--host-rirs 8] [--otf-cuts 512] [--otf-reps 5] [--out f.json]

Speech is N(0, 0.2^2) PCM16 WAV noise (eight 30 s files) in a temporary directory, read from the page cache; both routes read
the cuts in order on the calling thread (num_workers=0), the order in which lhotse's draws are deterministic."""
import argparse
import copy
import json
import os
import pathlib
import random
import statistics
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "scripts")]

from bench_flac import card, event_ms  # noqa: E402


def generators(n, seed):
    import rirgen_cases as RG

    return [RG.generator(16000, 0.8, seed + i, seed + 100000 + i) for i in range(n)]


def one_batch(n, launches):
    from torch.profiler import ProfilerActivity, profile

    from lhotse_b200.pcm_staging import GeneratedRirRequest, GeneratedRirs, _generate_rirs

    gen = GeneratedRirs([GeneratedRirRequest(g) for g in generators(n, 1000 * n)])
    t0 = time.perf_counter()
    gen.draw()
    draw_ms = (time.perf_counter() - t0) * 1000.0
    dev = torch.device("cuda:0")
    run = lambda: _generate_rirs(gen, dev)  # noqa: E731
    a = run()
    b = run()
    identical = bool(torch.equal(a.view(torch.int32), b.view(torch.int32)))
    total_ms = event_ms(run, launches)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(launches):
            run()
        torch.cuda.synchronize()
    per = {}
    for ev in prof.key_averages():
        k = ev.key.split("(")[0]
        if k.startswith(("rirgen_", "resample_stage_kernel")) or "RadixSort" in k:
            name = "segmented_sort" if "RadixSort" in k else k
            per[name + "_ms"] = round(per.get(name + "_ms", 0.0) + ev.device_time_total / 1000.0 / launches, 3)
    lens = gen.draws.lens
    return {"rirs": n, "host_draw_ms_per_rir": round(draw_ms / n, 3), "device_ms_with_upload": round(total_ms, 3),
            "kernels": per, "mean_rir_samples": round(float(np.mean(lens)), 1), "identical_run_to_run": identical}


def host_lhotse(n):
    ms = []
    for g in generators(n, 7):
        t0 = time.perf_counter()
        g(nsource=1)
        ms.append((time.perf_counter() - t0) * 1000.0)
    return {"rirs": n, "torch_threads": torch.get_num_threads(), "median_ms_per_rir": round(float(np.median(ms)), 2)}


def otf_batch(tmp, n, seed):
    import lhotse_env
    from lhotse import CutSet
    from lhotse.dataset.cut_transforms import ReverbWithImpulseResponse

    rs = np.random.RandomState(seed)
    speech = lhotse_env.make_cutset(tmp, [30.0] * 8, seed=4, amp=0.2, prefix=f"s{seed}_")
    cuts = []
    for i in range(n):
        d = float(np.round(rs.uniform(5.0, 15.0), 3))
        a = float(np.round(rs.uniform(0.0, 30.0 - d), 3))
        cuts.append(speech[i % 8].truncate(offset=a, duration=d, preserve_id=False).with_id(f"c{seed}_{i}"))
    return CutSet.from_cuts(list(ReverbWithImpulseResponse(p=0.5, randgen=random.Random(seed))(CutSet.from_cuts(cuts))))


def on_the_fly(args, lb_ex, tmp):
    from lhotse_b200.input_strategies import FusedOnTheFlyFeatures

    ext = lb_ex.B200Fbank(lb_ex.B200FbankConfig(device="cuda:0"))
    batches = [otf_batch(tmp, args.otf_cuts, 10 + k) for k in range(2)]
    hours = [sum(c.duration for c in b) / 3600 for b in batches]
    fast = FusedOnTheFlyFeatures(ext, generated_rir=True)
    slow = FusedOnTheFlyFeatures(ext, pcm16_fast_path=False)
    threads = torch.get_num_threads()
    warm = batches[0].subset(first=16)
    fast(warm), slow(warm)  # warm-up: rings, allocator, probes
    rates = {"transform": [], "float": []}
    for r in range(args.otf_reps):
        for name, strat in (("transform", fast), ("float", slow)):
            b = batches[r % 2]
            torch.set_num_threads(1 if name == "float" else threads)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            strat(b)
            torch.cuda.synchronize()
            rates[name].append(hours[r % 2] / (time.perf_counter() - t0))
        assert fast.last_batch_route == "transform" and slow.last_batch_route == "float"
    torch.set_num_threads(threads)
    torch.manual_seed(1)
    f1, l1 = fast(copy.deepcopy(batches[0]))
    torch.manual_seed(1)
    torch.set_num_threads(1)
    f2, l2 = slow(copy.deepcopy(batches[0]))
    torch.set_num_threads(threads)
    assert torch.equal(l1, l2)
    med = {k: statistics.median(v) for k, v in rates.items()}
    mask = torch.arange(f1.shape[1])[None, :] < l1[:, None]
    return {"otf_cuts": args.otf_cuts, "reps": args.otf_reps, "otf_hours_per_batch": [round(h, 3) for h in hours],
            "staged_hours_per_s": round(med["transform"], 3), "float_hours_per_s": round(med["float"], 3),
            "staged_over_float": round(med["transform"] / med["float"], 2),
            "all_staged": [round(x, 3) for x in rates["transform"]], "all_float": [round(x, 3) for x in rates["float"]],
            "max_logmel_diff": float((f1 - f2).abs()[mask.to(f1.device)].max())}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--launches", type=int, default=10)
    ap.add_argument("--host-rirs", type=int, default=8)
    ap.add_argument("--otf-cuts", type=int, default=512)
    ap.add_argument("--otf-reps", type=int, default=5)
    ap.add_argument("--out")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_rirgen needs a GPU"
    import lhotse_env

    lhotse_env.setup_lhotse()
    name, limit = card()
    res = {"bench": "rirgen", "gpu": name, "power_limit": limit,
           "batches": [one_batch(n, args.launches) for n in (256, 1024)],
           "lhotse_host": host_lhotse(args.host_rirs)}
    with tempfile.TemporaryDirectory() as tmp:
        res["on_the_fly"] = on_the_fly(args, lhotse_env.setup_lhotse(), pathlib.Path(tmp))
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
