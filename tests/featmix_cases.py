"""Test-only: archive-backed cut sets for the precomputed-features route, the float64 restatement of the feature-mix tables
(csrc/featmix.cuh, DESIGN.md §3.1m) and the checks shared by tests/test_precomputed.py and tests/test_gpu_precomputed.py."""
import math
import os
import subprocess

import numpy as np

EPSILON = 1e-10
DUMMY = -1000.0
LOG, LINEAR = 0, 1
COPY, MIX = 0, 1
MIXED, ENERGY = 1, 2


# the two laws as lhotse's statics state them, evaluated in float64
def law_mix(law, a, b, g):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return np.log(np.maximum(EPSILON, np.exp(a) + g * np.exp(b))) if law == LOG else a + g * b


def law_energy(law, x):
    x = np.asarray(x, np.float64)
    return float(np.sum(np.exp(x))) if law == LOG else float(np.sum(x))


def law_scale(law, x, g):
    x = np.asarray(x, np.float64)
    return x + np.log(g) if law == LOG else g * x


def track_rows(src, t, F):
    """The (num_rows, F) float64 rows of track record `t`."""
    n = int(t["num_rows"])
    if int(t["stored_rows"]) == 0:
        return np.full((n, F), np.float64(np.float32(t["value"])))
    st = int(t["stored_rows"])
    rows = np.asarray(src[int(t["src_elem"]): int(t["src_elem"]) + st * F], np.float64).reshape(st, F)
    return rows if n == st else np.concatenate([rows, rows[-1:]], axis=0)


def evaluate(src, tracks, cuts, F, T, pad_value):
    """The tables evaluated in float64 the way lhotse's FeatureMixer folds them: (B, T, F) float64.  The first track is scaled
    by _scale_features_for_snr's rejections (`<= 0` keeps it, so a NaN energy scales by NaN), later tracks by FeatureMixer's
    acceptance (`> 0` scales, so a NaN energy keeps gain 1)."""
    with np.errstate(all="ignore"):
        return _evaluate(src, tracks, cuts, F, T, pad_value)


def _evaluate(src, tracks, cuts, F, T, pad_value):
    out = np.full((len(cuts), T, F), np.float64(np.float32(pad_value)))
    for c, cu in enumerate(cuts):
        t0, nt, nr = int(cu["first_track"]), int(cu["num_tracks"]), int(cu["num_rows"])
        base = tracks[t0]
        brow = track_rows(src, base, F)
        if int(cu["mode"]) == COPY:
            res = np.full((nr, F), np.float64(np.float32(cu["pad_value"])))
            res[: len(brow)] = brow
            out[c, :nr] = res
            continue
        law = int(cu["law"])
        ref = t0 + int(cu["ref_track"])
        e_ref = law_energy(law, track_rows(src, tracks[ref], F))
        if int(cu["ref_track"]) != 0 and not math.isnan(base["snr_factor"]) and not e_ref <= 0:
            e0 = law_energy(law, brow)
            if not e0 <= 0:
                brow = law_scale(law, brow, e_ref * float(base["snr_factor"]) / e0)
        mix_rows = int(cu["mix_rows"])
        mix = np.full((mix_rows, F), DUMMY)
        mix[: len(brow)] = brow[:mix_rows]
        for k in range(1, nt):
            t = tracks[t0 + k]
            if not int(t["flags"]) & MIXED:
                continue
            rows = track_rows(src, t, F)
            g = 1.0
            if not math.isnan(t["snr_factor"]) and e_ref > 0:
                e = law_energy(law, rows)
                if e > 0:
                    g = e_ref * float(t["snr_factor"]) / e
            b = np.full((mix_rows, F), DUMMY)
            o = int(t["offset"])
            b[o: o + len(rows)] = rows
            mix = law_mix(law, mix, b, g)
        idx = np.minimum(np.arange(nr), mix_rows - 1)
        out[c, :nr] = mix[idx]
    return out


def ulp32(x):
    x = np.abs(np.asarray(x, np.float64)).astype(np.float32)
    return (np.nextafter(x, np.float32(np.inf)) - x).astype(np.float64)


def check_gate(ours, lhotse32, truth64, what=""):
    """Per cut: |ours - truth| <= 2 E_cut + ulp32(truth), E_cut = max |lhotse - truth| over the cut."""
    ours, lhotse32, truth64 = (np.asarray(a, np.float64) for a in (ours, lhotse32, truth64))
    assert ours.shape == truth64.shape == lhotse32.shape, (ours.shape, truth64.shape, lhotse32.shape)
    for c in range(ours.shape[0]):
        e_cut = float(np.max(np.abs(lhotse32[c] - truth64[c]))) if ours[c].size else 0.0
        err = np.abs(ours[c] - truth64[c])
        bad = err > 2 * e_cut + ulp32(truth64[c])
        assert not bad.any(), f"{what} cut {c}: {int(bad.sum())} elements over the gate, worst {float(err.max())} (E_cut {e_cut})"


# ---- archive-backed cut sets ----------------------------------------------------------------------------------------------

def write_features(writer, rs, frames, F, kind="log", cells=()):
    """Seeded log-mel-like rows (log law) or non-negative power-like rows (linear law), then the (row, col, value) `cells`."""
    x = rs.randn(frames, F).astype(np.float32)
    if kind == "log":
        x = (x * 2.0 - 6.0 + np.linspace(0, 3, F, dtype=np.float32)).astype(np.float32)
    else:
        x = np.abs(x * 3.0).astype(np.float32)
    for r, c, v in cells:
        x[r, c] = v
    return writer.write("k", x), x


def make_cuts(storage, frames_list, F=80, seed=0, prefix="c", ftype="b200-fbank", kind="log", frame_shift=0.01, sr=16000,
              supervisions=True, cells=None):
    """One feature-only MonoCut per entry of `frames_list`, its rows appended to the archive at `storage`; `cells[i]` are
    (row, col, value) cells written over cut i's rows."""
    from lhotse import CutSet, MonoCut, SupervisionSegment
    from lhotse.features.base import Features

    from lhotse_b200.storage import B200ArchiveWriter

    rs = np.random.RandomState(seed)
    cuts = []
    with B200ArchiveWriter(storage, mode="a") as w:
        for i, n in enumerate(frames_list):
            key, _ = write_features(w, rs, n, F, kind, (cells or {}).get(i, ()))
            dur = round(n * frame_shift, 6)
            fm = Features(type=ftype, num_frames=n, num_features=F, frame_shift=frame_shift, sampling_rate=sr, start=0.0,
                          duration=dur, storage_type="b200_archive", storage_path=str(w.storage_path), storage_key=key,
                          recording_id=f"{prefix}r{i}", channels=0)
            sups = [SupervisionSegment(id=f"{prefix}s{i}", recording_id=f"{prefix}r{i}", start=0.0, duration=dur, text="x")] \
                if supervisions else []
            cuts.append(MonoCut(id=f"{prefix}{i}", start=0.0, duration=dur, channel=0, features=fm, supervisions=sups))
    return CutSet.from_cuts(cuts)


def lhotse_pair(cuts):
    """(lhotse's collate_features, the float64 truth: the same lhotse code with every stored row read as float64)."""
    import torch
    from lhotse.dataset.collation import collate_features

    from lhotse_b200.storage import B200ArchiveReader

    feats, lens = collate_features(cuts)
    orig = B200ArchiveReader.read
    B200ArchiveReader.read = lambda self, *a, **k: orig(self, *a, **k).astype(np.float64)
    try:
        truth, _ = collate_features(cuts, features_dtype=torch.float64)
    finally:
        B200ArchiveReader.read = orig
    return feats, lens, truth


def host_evaluate(plan):
    """The plan's tables evaluated by `evaluate` over rows staged on the host (an unpinned ring)."""
    from lhotse_b200.plan import LOG_EPSILON
    from lhotse_b200.precomputed import FeatureStagingRing

    staged, tracks = FeatureStagingRing(pin_memory=False).stage(plan)
    return evaluate(staged.numpy(), tracks, plan.cuts, plan.F, plan.T, LOG_EPSILON)


def build_harness(tmp_dir):
    import shutil

    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    src = os.path.join(root, "scripts", "micro", "featmix_host_check.cu")
    gxx = shutil.which("g++") or shutil.which("c++")
    if gxx is None:
        return None
    exe = os.path.join(str(tmp_dir), "featmix_host_check")
    for flags in (["-fsanitize=address", "-fno-omit-frame-pointer"], []):
        res = subprocess.run([gxx, "-x", "c++", "-std=c++17", "-O1", "-g", *flags, "-o", exe, src], capture_output=True, text=True)
        if res.returncode == 0:
            return exe
    raise RuntimeError("featmix_host_check does not compile:\n" + res.stderr)


def run_harness(exe, tmp_path, src, tracks, cuts, F, T, pad_value):
    np.asarray(src, np.float32).tofile(tmp_path / "src.f32")
    np.ascontiguousarray(tracks).tofile(tmp_path / "tracks.bin")
    np.ascontiguousarray(cuts).tofile(tmp_path / "cuts.bin")
    subprocess.run([exe, str(tmp_path / "src.f32"), str(tmp_path / "tracks.bin"), str(tmp_path / "cuts.bin"), str(F), str(T),
                    repr(float(pad_value)), str(tmp_path / "out.f32")], check=True)
    return np.fromfile(tmp_path / "out.f32", dtype=np.float32).reshape(len(cuts), T, F)
