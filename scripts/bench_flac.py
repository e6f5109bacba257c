"""FLAC on the GPU, measured: the decode kernel against the fbank kernel on the same batch, and FusedOnTheFlyFeatures over
FLAC cuts against the same audio as PCM16 WAV (alternated in one process, outputs compared).  Prints one JSON line (and
writes it to --out when given).

    python scripts/bench_flac.py [--cuts 2048] [--launches 20] [--otf-cuts 512] [--otf-reps 5] [--out flac.json]

Cuts are whole copies of the two LibriSpeech fixtures under tests/golden (16 kHz mono, about 11 s each, block size 4096), so
after the first read every file read is served by the page cache."""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time
import wave

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

import flac_oracle as F  # noqa: E402
import lhotse_b200 as lb  # noqa: E402
from lhotse_b200.engine import OUT_PADDED, Engine, flac_decode  # noqa: E402
from lhotse_b200.pcm_staging import FlacRequest, FlacStagingRing  # noqa: E402

GOLDEN = [os.path.join(ROOT, "tests", "golden", f"2412-153948-000{i}.flac") for i in (0, 1)]


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i",
                              str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout.strip()
        name, limit = [s.strip() for s in out.split(",")]
        return name, limit
    except Exception:
        return torch.cuda.get_device_name(), "unknown"


def event_ms(fn, n):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(n):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / n


def kernels(args, pcms):
    reqs = [FlacRequest(GOLDEN[i % 2], 0, pcms[i % 2].shape[0]) for i in range(args.cuts)]
    ring = FlacStagingRing()
    t0 = time.perf_counter()
    batch, lens, offs, sr = ring.stage(reqs)
    stage_s = time.perf_counter() - t0
    dev = torch.device("cuda:0")
    data, jobs = batch.data.to(dev), batch.jobs.to(dev)
    out = torch.zeros(batch.out_elems, dtype=torch.int16, device=dev)
    status = torch.empty(batch.njobs, dtype=torch.int32, device=dev)
    dec = lambda: flac_decode(data, jobs, batch.njobs, out, status, None)  # noqa: E731
    for _ in range(3):
        dec()
    torch.cuda.synchronize()
    assert int(torch.count_nonzero(status)) == 0
    host = out.cpu().numpy()
    exact = all(np.array_equal(host[o:o + n], pcms[i % 2][:, 0]) for i, (o, n) in enumerate(zip(offs, lens)))
    ext = lb.B200Fbank(lb.B200FbankConfig(device="cuda:0"))
    eng: Engine = ext.engine
    meta, tot = eng.plan_batch(lens, offs, out_mode=OUT_PADDED)
    meta_dev = torch.from_numpy(meta).to(dev)
    feats = torch.empty(int(tot.out_floats), dtype=torch.float32, device=dev)
    fb = lambda: eng.extract_device(out, lens, offs, out_mode=OUT_PADDED, out=feats, meta_dev=meta_dev, totals=tot)  # noqa: E731
    for _ in range(3):
        fb()
    dec_ms, fb_ms = [], []
    for _ in range(3):  # alternated
        dec_ms.append(event_ms(dec, args.launches))
        fb_ms.append(event_ms(fb, args.launches))
    hours = sum(lens) / sr / 3600
    d, f = float(np.median(dec_ms)), float(np.median(fb_ms))
    return {
        "cuts": args.cuts, "jobs": batch.njobs, "audio_hours": round(hours, 3), "compressed_bytes": int(batch.data.numel()),
        "pcm16_bytes": 2 * int(sum(lens)), "host_stage_s": round(stage_s, 4), "decode_bit_exact": bool(exact),
        "decode_ms": [round(x, 4) for x in dec_ms], "fbank_ms": [round(x, 4) for x in fb_ms],
        "decode_hours_per_s": round(hours / (d / 1e3), 1), "decode_compressed_GBps": round(batch.data.numel() / (d / 1e3) / 1e9, 2),
        "fbank_hours_per_s": round(hours / (f / 1e3), 1), "decode_over_fbank": round(d / f, 3),
    }


def on_the_fly(args, pcms):
    import refshim

    if not refshim.reference_available():
        return {"skipped": "no reference package (lhotse) available"}
    import lhotse_env

    lb_ex = lhotse_env.setup_lhotse()
    from lhotse import CutSet, MonoCut, Recording
    from lhotse.audio import AudioSource

    from lhotse_b200.input_strategies import FusedOnTheFlyFeatures

    tmp = tempfile.mkdtemp(prefix="bench_flac_")
    wavs = []
    for i, p in enumerate(pcms):
        w = os.path.join(tmp, f"twin{i}.wav")
        with wave.open(w, "wb") as fh:
            fh.setnchannels(1); fh.setsampwidth(2); fh.setframerate(16000)
            fh.writeframes(p[:, 0].astype("<i2").tobytes())
        wavs.append(w)

    def cutset(paths):
        cuts = []
        for i in range(args.otf_cuts):
            n = pcms[i % 2].shape[0]
            rec = Recording(id=f"r{i % 2}", sources=[AudioSource(type="file", channels=[0], source=paths[i % 2])],
                            sampling_rate=16000, num_samples=n, duration=n / 16000)
            cuts.append(MonoCut(id=f"c{i}", start=0.0, duration=n / 16000, channel=0, recording=rec))
        return CutSet.from_cuts(cuts)

    flac_cuts, wav_cuts = cutset(GOLDEN), cutset(wavs)
    ext = lb_ex.B200Fbank(lb_ex.B200FbankConfig(device="cuda:0"))
    strat = FusedOnTheFlyFeatures(ext, num_workers=8)
    hours = sum(c.duration for c in flac_cuts) / 3600
    res = {"flac": [], "pcm16": []}
    outs = {}
    for rep in range(args.otf_reps + 1):
        for route, cs in (("flac", flac_cuts), ("pcm16", wav_cuts)):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            feats, lens = strat(cs)
            torch.cuda.synchronize()
            dt = time.perf_counter() - t0
            assert strat.last_batch_route == route, (strat.last_batch_route, route)
            if rep == 0:
                outs[route] = (feats.clone(), lens.clone())
            else:
                res[route].append(round(hours / dt, 1))
    same = torch.equal(outs["flac"][0], outs["pcm16"][0]) and torch.equal(outs["flac"][1], outs["pcm16"][1])
    for w in wavs:
        os.remove(w)
    os.rmdir(tmp)
    return {"cuts": args.otf_cuts, "audio_hours": round(hours, 3), "num_workers": 8, "features_equal": bool(same),
            "flac_hours_per_s": res["flac"], "pcm16_hours_per_s": res["pcm16"],
            "flac_median": float(np.median(res["flac"])), "pcm16_median": float(np.median(res["pcm16"]))}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cuts", type=int, default=2048)
    ap.add_argument("--launches", type=int, default=20)
    ap.add_argument("--otf-cuts", type=int, default=512)
    ap.add_argument("--otf-reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_flac.py measures on a GPU; none is visible")
    pcms = [F.decode(open(p, "rb").read())[2] for p in GOLDEN]
    name, limit = card()
    res = {"gpu": name, "power_limit": limit, "kernels": kernels(args, pcms), "on_the_fly": on_the_fly(args, pcms)}
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
