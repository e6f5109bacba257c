"""Where the largest log-mel difference between the generated-RIR route and the float route comes from (DESIGN.md §3.1l),
on the CPU: rebuilds bench_rirgen.otf_batch(…, 10) (the generators seeded from counters, since lhotse seeds them from the
OS) and, for every reverberated cut in load order from torch.manual_seed(1), the two RIRs drawn from the same generator and
torch states: ours (the kernels' arithmetic in scripts/micro/rirgen_host_check.cu, then resample_reference to sr) and
lhotse's (its own generator with one torch thread).  Per cut it reports both shifts (first index of the maximum), both
maxima, how far below its own maximum each RIR's value at the other RIR's shift lies, and the largest log-mel difference
between lhotse's float32 reverb (reverb_cases.lhotse32) of the cut with either RIR through lhotse's CPU Fbank, with the
frame, the bin and the frame's energy.  Prints one JSON line per cut and a summary line.

    python scripts/rirgen_logmel_gap.py [--cuts 512] [--out f.jsonl]

Needs the reference (lhotse) and a host C++ compiler; no GPU."""
import argparse
import copy
import itertools
import json
import os
import pathlib
import shutil
import subprocess
import sys
import tempfile

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "scripts")]

NEAR_SILENT_DB = -40.0  # a frame whose energy is this far below the cut's loudest frame


def _harness(tmp):
    exe = os.path.join(tmp, "rirgen_host_check")
    src = os.path.join(ROOT, "scripts", "micro", "rirgen_host_check.cu")
    subprocess.run([shutil.which("g++") or "g++", "-x", "c++", "-std=c++17", "-O2", "-o", exe, src], check=True)
    return exe


def _seed_generators():
    """FastRandomRIRGenerator seeds from counters when none is given, so the batch is the same on every run."""
    from lhotse.augmentation.utils import FastRandomRIRGenerator

    orig = FastRandomRIRGenerator.__post_init__
    seeds = itertools.count(5000)

    def post_init(self):
        if self.room_seed is None:
            self.room_seed = next(seeds)
        if self.source_seed is None:
            self.source_seed = next(seeds)
        orig(self)

    FastRandomRIRGenerator.__post_init__ = post_init


def _pre_reverb(c):
    from lhotse.utils import fastcopy

    rec = fastcopy(c.recording, transforms=c.recording.transforms[:-1] or None)
    return np.asarray(fastcopy(c, recording=rec).load_audio(), np.float32)[0]


def _logmel(fbank, x, sr):
    return fbank.extract(x, sr)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cuts", type=int, default=512)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()

    import lhotse_env

    lhotse_env.setup_lhotse()
    _seed_generators()
    from lhotse import Fbank
    from lhotse.augmentation.rir import ReverbWithImpulseResponse

    import bench_rirgen
    import reverb_cases as RC
    import rirgen_cases as RG
    import test_rirgen
    from lhotse_b200 import rir_draws
    from lhotse_b200.pcm_staging import resample_reference

    fbank = Fbank()
    rows = []
    out = open(args.out, "w") if args.out else None
    with tempfile.TemporaryDirectory() as tmp:
        exe = _harness(tmp)
        batch = list(bench_rirgen.otf_batch(pathlib.Path(tmp), args.cuts, 10))
        torch.manual_seed(1)
        for k, c in enumerate(batch):
            tfs = getattr(c.recording, "transforms", None) or []
            t = tfs[-1] if tfs else None
            if not (isinstance(t, ReverbWithImpulseResponse) and t.rir is None):
                continue
            gen = t.rir_generator
            state = torch.get_rng_state()
            d = rir_draws.draw([copy.deepcopy(gen)])
            out8 = test_rirgen.run_harness(exe, pathlib.Path(tmp), d)[0][5]
            ours = resample_reference(out8, 8, 1)
            torch.set_rng_state(state)
            theirs, _, after = RG.lhotse_rir(gen)
            torch.set_rng_state(after)
            theirs = np.asarray(theirs, np.float32)
            s1, s2 = int(np.argmax(ours)), int(np.argmax(theirs))
            x = _pre_reverb(c)
            n = c.num_samples
            y1 = RC.lhotse32(x, ours * np.float32(32768), t.normalize_output, n)
            y2 = RC.lhotse32(x, theirs * np.float32(32768), t.normalize_output, n)
            f1, f2 = _logmel(fbank, y1, c.sampling_rate), _logmel(fbank, y2, c.sampling_rate)
            diff = np.abs(f1.astype(np.float64) - f2)
            fr, b = np.unravel_index(int(np.argmax(diff)), diff.shape)
            energy = 10 * np.log10(np.sum(np.exp(f2.astype(np.float64)), axis=1))
            row = {"cut": c.id, "shift_ours": s1, "shift_lhotse": s2, "max_ours": float(ours[s1]), "max_lhotse": float(theirs[s2]),
                   "ours_at_lhotse_shift_below_max": float(ours[s1] - ours[s2]),
                   "lhotse_at_our_shift_below_max": float(theirs[s2] - theirs[s1]),
                   "rir_max_abs_diff": float(np.max(np.abs(ours.astype(np.float64) - theirs))),
                   "max_logmel_diff": float(diff[fr, b]), "frame": int(fr), "bin": int(b),
                   "frame_db_below_loudest": float(energy.max() - energy[fr]),
                   "near_silent": bool(energy[fr] < energy.max() + NEAR_SILENT_DB)}
            rows.append(row)
            print(json.dumps(row), flush=True)
            if out:
                out.write(json.dumps(row) + "\n")
    worst = max(rows, key=lambda r: r["max_logmel_diff"])
    moved = [r for r in rows if r["shift_ours"] != r["shift_lhotse"]]
    summary = {"reverberated_cuts": len(rows), "shifts_differ": len(moved),
               "worst": worst, "worst_with_equal_shift": max((r["max_logmel_diff"] for r in rows if r not in moved), default=None),
               "worst_with_moved_shift": max((r["max_logmel_diff"] for r in moved), default=None),
               "cuts_over_0.1": sum(r["max_logmel_diff"] > 0.1 for r in rows),
               "cuts_over_0.1_near_silent": sum(r["max_logmel_diff"] > 0.1 and r["near_silent"] for r in rows),
               "worst_bin_counts": {str(b): sum(r["bin"] == b for r in rows) for b in sorted({r["bin"] for r in rows})}}
    print(json.dumps({"summary": summary}))
    if out:
        out.write(json.dumps({"summary": summary}) + "\n")
        out.close()


if __name__ == "__main__":
    main()
