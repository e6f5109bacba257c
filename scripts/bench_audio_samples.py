"""The padded waveform batch, measured: lhotse's AudioSamples (collate_audio: padding MixedCuts, per-cut decode / mix /
resample on the host, a float32 (B, T) tensor, then `.to("cuda")` and a synchronise) against FusedAudioSamples (the staged
route, the collation kernel, a synchronise) on the same batches, alternated in one process after a warm-up, median of --reps;
the collation kernel's device time (torch.profiler, a separate pass) and its achieved bytes/s against the algorithmic bytes
(each cut sample read once at 2 B (int16) or 4 B (float32), each output sample written once at 4 B), the H2D bytes of each
route (from the profiler's memcpy records), and torch.equal of the two outputs.  Needs a GPU and the lhotse package
(tests/refshim.py).  Prints one JSON line (and writes it to --out when given).

    python scripts/bench_audio_samples.py [--cuts 512] [--reps 5] [--workers 8] [--out f.json]

Workloads: 10-15 s slices of 16 kHz PCM16 WAV files under a temporary directory (page-cached: written just before), 512 cuts
per batch: "plain"; "cutmix", CutMix(p=0.5, snr=(10, 20)) over a noise set of 2-20 s, drawn once and shared by both routes;
"speed", every cut perturb_speed 0.9 or 1.1 (alternating)."""
import argparse
import glob
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

from bench_flac import card  # noqa: E402


def workloads(root, n_cuts):
    import lhotse_env
    from lhotse import CutSet
    from lhotse.dataset.cut_transforms import CutMix

    rs = np.random.RandomState(0)
    files = list(lhotse_env.make_cutset(root, [16.0] * 64, seed=1, amp=0.2, supervisions=False, prefix="s"))
    noise = CutSet.from_cuts(lhotse_env.make_cutset(root, np.round(rs.uniform(2.0, 20.0, 200), 3).tolist(), seed=2, amp=0.05,
                                                    supervisions=False, prefix="n"))
    cuts = []
    for i in range(n_cuts):
        d = float(np.round(rs.uniform(10.0, 15.0), 3))
        a = float(np.round(rs.uniform(0.0, 16.0 - d), 3))
        cuts.append(files[i % 64].truncate(offset=a, duration=d, preserve_id=False).with_id(f"c{i}"))
    plain = CutSet.from_cuts(cuts)
    mixed = CutSet.from_cuts(list(CutMix(cuts=noise, p=0.5, snr=(10, 20), seed=3)(plain)))
    speed = CutSet.from_cuts([c.perturb_speed(0.9 if i % 2 == 0 else 1.1) for i, c in enumerate(cuts)])
    return {"plain": plain, "cutmix": mixed, "speed": speed}


def h2d_bytes(fn, tmp):
    """Bytes of every host-to-device memcpy `fn` issues, from a torch.profiler trace."""
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:  # device records only: the host path's ops crowd them out
        out = fn()
        torch.cuda.synchronize()
    path = os.path.join(tmp, "trace.json")
    prof.export_chrome_trace(path)
    events = json.load(open(path)).get("traceEvents", [])
    os.remove(path)
    total = sum(int(e.get("args", {}).get("bytes", 0)) for e in events
                if e.get("cat") == "gpu_memcpy" and "HtoD" in e.get("name", ""))
    return total, out


def kernel_ms(fn):
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return sum(e.device_time_total for e in prof.key_averages() if "collate_audio_kernel" in e.key) / 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cuts", type=int, default=512)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--workers", type=int, default=8)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()

    import lhotse_env
    import refshim

    assert refshim.reference_available(), "needs the lhotse package (tests/refshim.py)"
    lhotse_env.setup_lhotse()
    from lhotse.dataset.input_strategies import AudioSamples

    from lhotse_b200 import FusedAudioSamples

    name, limit = card()
    res = {"card": name, "power_limit": limit, "cuts_per_batch": args.cuts, "reps": args.reps, "workers": args.workers,
           "workloads": {}}
    with tempfile.TemporaryDirectory() as tmp:
        from pathlib import Path

        loads = workloads(Path(tmp), args.cuts)
        for f in glob.glob(os.path.join(tmp, "*.wav")):  # page-cache every file
            open(f, "rb").read()
        ref = AudioSamples(num_workers=args.workers)
        fused = FusedAudioSamples(num_workers=args.workers)

        def run_ref(cuts):
            a, l = ref(cuts)
            a = a.to("cuda")
            torch.cuda.synchronize()
            return a, l

        def run_fused(cuts):
            a, l = fused(cuts)
            torch.cuda.synchronize()
            return a, l

        for wname, cuts in loads.items():
            a_ref, l_ref = run_ref(cuts)  # warm-up of both
            a_f, l_f = run_fused(cuts)
            route = fused.last_batch_route
            equal = bool(torch.equal(a_ref, a_f) and torch.equal(l_ref, l_f))
            t_ref, t_f = [], []
            for _ in range(args.reps):
                t0 = time.perf_counter()
                run_ref(cuts)
                t_ref.append(time.perf_counter() - t0)
                t0 = time.perf_counter()
                run_fused(cuts)
                t_f.append(time.perf_counter() - t0)
            hours = sum(c.duration for c in cuts) / 3600
            ms = kernel_ms(lambda: fused(cuts))
            B, T = a_f.shape
            esz = 2 if route in ("pcm16", "flac") else 4
            alg = int(l_f.sum()) * esz + B * T * 4
            h2d_ref, _ = h2d_bytes(lambda: ref(cuts)[0].to("cuda"), tmp)
            h2d_fused, _ = h2d_bytes(lambda: fused(cuts), tmp)
            res["workloads"][wname] = {
                "route": route, "mixed_cuts": sum(getattr(c, "tracks", None) is not None for c in cuts),
                "hours_of_audio": round(hours, 4), "B": B, "T": T, "torch_equal": equal,
                "lhotse_s": round(statistics.median(t_ref), 4), "fused_s": round(statistics.median(t_f), 4),
                "speedup": round(statistics.median(t_ref) / statistics.median(t_f), 2),
                "lhotse_hours_per_s": round(hours / statistics.median(t_ref), 3),
                "fused_hours_per_s": round(hours / statistics.median(t_f), 3),
                "collate_kernel_ms": round(ms, 4), "collate_source_bytes_per_sample": esz,
                "collate_algorithmic_bytes": alg, "collate_achieved_GB_per_s": round(alg / (ms * 1e-3) / 1e9, 1) if ms else None,
                "h2d_bytes_lhotse": h2d_ref, "h2d_bytes_fused": h2d_fused,
                "times_lhotse_s": [round(x, 4) for x in t_ref], "times_fused_s": [round(x, 4) for x in t_f],
            }
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
