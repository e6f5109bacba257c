"""Speed-perturbed and resampled cuts on the GPU, measured: the resampling kernel per stage on 2048 cuts of 10 s (speed 0.9,
speed 1.1, 48 kHz -> 16 kHz) against the fbank kernel on the same output, and FusedOnTheFlyFeatures over speed-perturbed
batches on the "transform" route against the float route (alternated in one process, features compared).  Prints one JSON
line (and writes it to --out when given).

    python scripts/bench_transform.py [--cuts 2048] [--launches 20] [--otf-cuts 256] [--otf-reps 5] [--threads 8] [--out t.json]

Audio is N(0, 0.2^2) PCM16 WAV noise (eight 30 s files per rate) written to a temporary directory and read from the page
cache, through lhotse from the reference tree or archive (oracle/refimport.py) with a stdlib-`wave` audio backend.  lhotse
runs its Resample transform through its torch resampler only where torchaudio is installed; elsewhere the 48 kHz leg is
reported as not eligible."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile
import time
import wave

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    """(name, power limit) of the current GPU, read in the same run as the measurement."""
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i",
                              str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout.strip()
        name, limit = [s.strip() for s in out.split(",")]
        return name, limit
    except Exception:
        return torch.cuda.get_device_name(), "unknown"


def event_ms(fn, n):
    """Mean device time of fn() over n back-to-back calls, by CUDA events."""
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(n):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / n


def setup_lhotse():
    """Imports lhotse (before lhotse_b200, so its extractors bind to lhotse's base class) and reads WAV files with `wave`."""
    from oracle.refimport import import_reference

    import_reference()
    from lhotse.audio.backend import AudioBackend, LibsndfileCompatibleAudioInfo, set_current_audio_backend

    class WaveBackend(AudioBackend):
        def read_audio(self, path_or_fd, offset=0.0, duration=None, force_opus_sampling_rate=None):
            from lhotse.utils import compute_num_samples

            with wave.open(str(path_or_fd)) as w:
                sr = w.getframerate()
                w.setpos(compute_num_samples(offset, sr))
                n = w.getnframes() - w.tell() if duration is None else compute_num_samples(duration, sr)
                pcm = np.frombuffer(w.readframes(n), dtype="<i2")
            return (pcm.astype(np.float32) / 32768.0)[None, :], sr

        def is_applicable(self, path_or_fd):
            return True

        def supports_info(self):
            return True

        def info(self, path_or_fd, force_opus_sampling_rate=None, force_read_audio=False):
            with wave.open(str(path_or_fd)) as w:
                return LibsndfileCompatibleAudioInfo(channels=1, frames=w.getnframes(), samplerate=w.getframerate(),
                                                     duration=w.getnframes() / w.getframerate())

    set_current_audio_backend(WaveBackend())
    import lhotse_b200.extractors as lb_ex

    return lb_ex


def slices(tmp, n, sr, seed, dur=None):
    """n MonoCuts: slices of eight 30 s WAV files at `sr` (`dur` seconds long, else 5-15 s)."""
    from lhotse import MonoCut, Recording
    from lhotse.audio import AudioSource

    rs = np.random.RandomState(seed)
    recs = []
    for i in range(8):
        path = tmp / f"s{seed}_{sr}_{i}.wav"
        pcm = np.clip(rs.randn(30 * sr) * 0.2 * 32768, -32768, 32767).astype("<i2")
        with wave.open(str(path), "wb") as w:
            w.setnchannels(1); w.setsampwidth(2); w.setframerate(sr)
            w.writeframes(pcm.tobytes())
        recs.append(Recording(id=path.stem, sources=[AudioSource(type="file", channels=[0], source=str(path))], sampling_rate=sr,
                              num_samples=30 * sr, duration=30.0))
    out = []
    for i in range(n):
        d = dur if dur is not None else float(np.round(rs.uniform(5.0, 15.0), 3))
        a = float(np.round(rs.uniform(0.0, 30.0 - d), 3))
        out.append(MonoCut(id=f"c{seed}_{i}", start=a, duration=d, channel=0, recording=recs[i % 8]))
    return out


def kernels(args, lb_ex, tmp):
    from lhotse_b200.engine import resample, resample_table
    from lhotse_b200.pcm_staging import TransformStagingRing, resample_kernel, transform_requests_for_batch

    dev = torch.device("cuda:0")
    ext = lb_ex.B200Fbank(lb_ex.B200FbankConfig(device="cuda:0"))
    eng = ext.engine
    res = {"kernel_cuts": args.cuts}
    for name, sr, make in (("speed_0.9", 16000, lambda c: c.perturb_speed(0.9)), ("speed_1.1", 16000, lambda c: c.perturb_speed(1.1)),
                           ("resample_48000_16000", 48000, lambda c: c.resample(16000))):
        cuts = [make(c) for c in slices(tmp, args.cuts, sr, 1, dur=10.0)]
        reqs = transform_requests_for_batch(cuts)
        if reqs is None:
            res[name] = "not eligible on this host (see transform_request_for_cut)"
            continue
        batch, lens, offs, _ = TransformStagingRing().stage(reqs)
        ids = np.asarray([resample_table(a, b, *resample_kernel(a, b), dev, eng._h) for a, b in batch.pairs] + [-1], np.int32)
        st = batch.stages.copy()
        st["table"] = ids[batch.pair]
        src0 = batch.pcm.to(dev)
        out = torch.zeros(batch.out_elems, dtype=torch.float32, device=dev)
        resample(src0, None, None, st, out, eng._h)
        ms = event_ms(lambda: resample(src0, None, None, st, out, eng._h), args.launches)
        eng.extract_device(out, lens, offsets=offs)
        fb = event_ms(lambda: eng.extract_device(out, lens, offsets=offs), args.launches)
        n_in, n_out = int(st["in_len"].sum()), int(st["target_len"].sum())
        res[name] = {"pair": list(batch.pairs[0]), "in_samples": n_in, "out_samples": n_out, "resample_ms": round(ms, 3),
                     "fbank_ms": round(fb, 3), "hbm_gb_per_s": round((2 * n_in + 4 * n_out) / ms / 1e6, 1)}
    return res


def on_the_fly(args, lb_ex, tmp):
    from lhotse import CutSet

    from lhotse_b200.input_strategies import FusedOnTheFlyFeatures

    ext = lb_ex.B200Fbank(lb_ex.B200FbankConfig(device="cuda:0"))
    batches = []
    for k in range(2):
        cs = slices(tmp, args.otf_cuts, 16000, 10 + k)
        batches.append(CutSet.from_cuts([c.perturb_speed(0.9 if i % 2 else 1.1) for i, c in enumerate(cs)]))
    hours = [sum(c.duration for c in b) / 3600 for b in batches]
    fast = FusedOnTheFlyFeatures(ext, num_workers=args.threads)
    slow = FusedOnTheFlyFeatures(ext, num_workers=args.threads, pcm16_fast_path=False)
    for b in batches:  # warm-up: page cache, rings, allocator, probes
        fast(b), slow(b)
    rates = {"transform": [], "float": []}
    for r in range(args.otf_reps):
        for name, strat in (("transform", fast), ("float", slow)):
            b = batches[r % 2]
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            strat(b)
            torch.cuda.synchronize()
            rates[name].append(hours[r % 2] / (time.perf_counter() - t0))
        assert fast.last_batch_route == "transform" and slow.last_batch_route == "float"
    f1, l1 = fast(batches[0])
    f2, l2 = slow(batches[0])
    equal = bool(torch.equal(f1, f2) and torch.equal(l1, l2))
    med = {k: statistics.median(v) for k, v in rates.items()}
    return {"otf_cuts": args.otf_cuts, "threads": args.threads, "reps": args.otf_reps,
            "transform_hours_per_s": round(med["transform"], 2), "float_hours_per_s": round(med["float"], 2),
            "transform_over_float": round(med["transform"] / med["float"], 2),
            "all_transform": [round(x, 2) for x in rates["transform"]], "all_float": [round(x, 2) for x in rates["float"]],
            "features_equal": equal}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cuts", type=int, default=2048)
    ap.add_argument("--launches", type=int, default=20)
    ap.add_argument("--otf-cuts", type=int, default=256)
    ap.add_argument("--otf-reps", type=int, default=5)
    ap.add_argument("--threads", type=int, default=8)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    lb_ex = setup_lhotse()
    name, limit = card()
    res = {"bench": "transform", "gpu": name, "power_limit": limit}
    with tempfile.TemporaryDirectory() as d:
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
