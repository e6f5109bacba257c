"""WPE dereverberation on the GPU (`wpe=True`), measured: per-kernel device times of b200feat_wpe (STFT, per-bin filter,
iSTFT; `torch.profiler`) and the whole call (CUDA events) at 256 x 10 s and 64 x 30 s, with FLOPs and bytes computed from the
shapes and the bound each kernel would meet at the data-sheet peak; and FusedOnTheFlyFeatures(wpe=True) on the "transform"
route against the float route (alternated in one process, median of `--otf-reps`).  The float route runs lhotse's
DereverbWPE on a stand-in nara_wpe whose wpe_v8 is this project's numpy restatement (oracle/wpe_oracle.py), not nara_wpe
itself.  Prints one JSON line (and writes it to --out when given).

    python scripts/bench_wpe.py [--otf-cuts 64] [--otf-reps 5] [--threads 8] [--out f.json]

Signals are reverberant noise bursts (tests/wpe_cases.py); the end-to-end cuts are 10 s PCM16 WAV files in a temporary
directory, read from the page cache."""
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

FP64_PEAK, FP32_PEAK, HBM = 34e12, 67e12, 3.35e12  # H100 SXM data sheet: FP64 (non-tensor), FP32, HBM3 bytes/s
NAMES = {"wpe_stft_kernel": "stft", "wpe_bin_kernel": "bin", "wpe_istft_kernel": "istft"}


def shapes(B, L, taps=10, iterations=3):
    """FLOPs and bytes of one call from the shapes: FFTs at 5 N log2 N per 512-point complex transform (two frames each),
    the per-bin statistics at 10 float64 FLOPs per entry and frame, the filter at 8 per tap and frame."""
    T = 1 + L // 128
    E = taps * (taps + 1) // 2 + taps
    fft = B * (T / 2) * 5 * 512 * 9
    spec = B * 257 * T * 8
    return {
        "stft": {"flop": fft, "bytes": B * L * 4 + spec, "peak": "fp32"},
        "bin": {"flop": B * 257 * T * iterations * (E * 10 + taps * 8), "bytes": 2 * spec, "peak": "fp64"},
        "istft": {"flop": fft * (T + 3) / T, "bytes": spec + B * 128 * (L // 128) * 4, "peak": "fp32"},
    }


def kernel_times(B, L, reps=5):
    import wpe_cases as WC

    from lhotse_b200.engine import WPE_CUT_DTYPE, wpe

    xs = [WC.signal("reverb", L, seed=i) for i in range(B)]
    x = torch.from_numpy(np.concatenate(xs)).cuda()
    lz = 128 * (L // 128)
    ct = np.zeros(B, WPE_CUT_DTYPE)
    ct["struct_size"], ct["in_len"], ct["target_len"] = WPE_CUT_DTYPE.itemsize, L, lz
    ct["in_elem"], ct["out_elem"] = np.arange(B) * L, np.arange(B) * lz
    out = torch.empty(B * lz, device="cuda")
    call = lambda: wpe(x, ct, out)  # noqa: E731
    call()
    torch.cuda.synchronize()
    whole = event_ms(call, reps)
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            call()
        torch.cuda.synchronize()
    per = {v: 0.0 for v in NAMES.values()}
    for e in prof.key_averages():
        for k, v in NAMES.items():
            if k in e.key:
                per[v] += e.device_time_total / 1000.0 / reps
    res = {"cuts": B, "seconds": L / 16000, "call_ms": round(whole, 3), "audio_h_per_s": round(B * L / 16000 / 3600 / (whole / 1e3), 1)}
    for k, s in shapes(B, L).items():
        ms = per[k]
        bound_s = max(s["flop"] / (FP64_PEAK if s["peak"] == "fp64" else FP32_PEAK), s["bytes"] / HBM)
        which = "compute" if s["flop"] / (FP64_PEAK if s["peak"] == "fp64" else FP32_PEAK) > s["bytes"] / HBM else "hbm"
        res[k] = {"ms": round(ms, 3), "gflop": round(s["flop"] / 1e9, 2), "mb": round(s["bytes"] / 1e6, 1),
                  "tflop_s": round(s["flop"] / (ms / 1e3) / 1e12, 2) if ms else None, "bounded_by": f"{s['peak']} {which}",
                  "share_of_bound": round(bound_s / (ms / 1e3), 3) if ms else None}
    return res


def end_to_end(n, reps, threads):
    import lhotse_env
    import refshim
    import wpe_cases as WC

    refshim.import_reference()
    WC.install_nara_wpe_standin()
    lb_ex = lhotse_env.setup_lhotse()
    from lhotse_b200.input_strategies import FusedOnTheFlyFeatures

    tmp = tempfile.TemporaryDirectory()
    from pathlib import Path

    cuts = lhotse_env.make_cutset(Path(tmp.name), [10.0] * n, seed=3).dereverb_wpe()
    ext = lb_ex.B200Fbank(lb_ex.B200FbankConfig(device="cuda:0"))
    gpu = FusedOnTheFlyFeatures(ext, wpe=True, num_workers=threads)
    flt = FusedOnTheFlyFeatures(ext, pcm16_fast_path=False, num_workers=threads)
    times = {"transform": [], "float": []}
    fg, fl = None, None
    for r in range(reps + 1):
        for name, s in (("transform", gpu), ("float", flt)):
            torch.cuda.synchronize()
            t = time.perf_counter()
            f, _ = s(cuts)
            torch.cuda.synchronize()
            if r:
                times[name].append(time.perf_counter() - t)
            assert s.last_batch_route == name
            fg, fl = (f, fl) if name == "transform" else (fg, f)
    hours = n * 10.0 / 3600
    med = {k: statistics.median(v) for k, v in times.items()}
    tmp.cleanup()
    return {"cuts": n, "seconds": 10.0, "threads": threads, "reps": reps,
            "float_route": "lhotse DereverbWPE on the numpy restatement of wpe_v8 (stand-in, not nara_wpe)",
            "transform_s": round(med["transform"], 4), "float_s": round(med["float"], 4),
            "transform_h_per_s": round(hours / med["transform"], 2), "float_h_per_s": round(hours / med["float"], 3),
            "speedup": round(med["float"] / med["transform"], 1),
            "max_abs_fbank_diff": float((fg - fl).abs().max())}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--otf-cuts", type=int, default=64)
    ap.add_argument("--otf-reps", type=int, default=5)
    ap.add_argument("--threads", type=int, default=8)
    ap.add_argument("--out")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "bench_wpe needs a GPU"
    name, limit = card()
    line = {"bench": "wpe", "gpu": name, "power_limit": limit,
            "kernels": [kernel_times(256, 160000), kernel_times(64, 480000)],
            "end_to_end": end_to_end(a.otf_cuts, a.otf_reps, a.threads)}
    s = json.dumps(line)
    print(s)
    if a.out:
        with open(a.out, "w") as f:
            f.write(s + "\n")


if __name__ == "__main__":
    main()
