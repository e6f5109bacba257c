"""Test-only: the SpecAugment case matrix and the checks shared by tests/test_specaugment.py (plan + CPU harness) and
tests/test_gpu_specaugment.py (the kernels): seeded runs of lhotse's SpecAugment, the float64 warp it is compared with, and the
masks and warped regions a plan describes."""
import os
import random
import subprocess

import numpy as np
import torch

LOG_EPSILON = float(np.log(np.finfo(np.float32).eps))


def seed_all(seed):
    random.seed(seed)
    np.random.seed(seed)
    torch.manual_seed(seed)


def rng_states():
    s = np.random.get_state()
    return random.getstate(), (s[0], s[1].tolist(), s[2], s[3], s[4]), torch.get_rng_state().tolist()


def make_batch(B, T, F, lens=None, seed=0):
    """Log-mel-like features (mean about -8), the frames past each cut's length padded with LOG_EPSILON as collation does."""
    rs = np.random.RandomState(seed)
    x = (rs.randn(B, T, F) * 2.0 - 8.0).astype(np.float32)
    for b, n in enumerate(lens or []):
        x[b, n:] = LOG_EPSILON
    return torch.from_numpy(x)


def one_segment_per_cut(lens):
    return torch.tensor([[b, 0, n] for b, n in enumerate(lens)], dtype=torch.int32)


# name -> (SpecAugment kwargs, B, T, F, lens or None, supervision segments or None)
CASES = {
    "default_segments": ({}, 4, 600, 80, [600, 450, 300, 150], one_segment_per_cut([600, 450, 300, 150])),
    "default_no_segments": ({}, 3, 400, 80, None, None),
    "several_supervisions": ({"p": 1.0}, 3, 700, 80, [700, 520, 200],
                             torch.tensor([[0, 0, 250], [0, 250, 300], [1, 10, 200], [1, 300, 200], [0, 550, 150], [2, 0, 200]],
                                          dtype=torch.int32)),
    "segments_out_of_order": ({"p": 1.0, "time_warp_factor": 20}, 2, 500, 80, None,
                              torch.tensor([[1, 300, 200], [0, 250, 100], [1, 0, 300], [0, 0, 250]], dtype=torch.int32)),
    "clipped_by_T": ({"p": 1.0}, 3, 600, 80, None, torch.tensor([[0, 300, 400], [1, 0, 900], [2, 600, 50], [2, 599, 5]], dtype=torch.int32)),
    "too_short_to_warp": ({"p": 1.0}, 2, 400, 80, [161, 162], one_segment_per_cut([161, 162])),
    "warped_equals_center": ({"p": 1.0, "time_warp_factor": 1}, 6, 120, 80, None,
                             torch.tensor([[b, s, 20] for b in range(6) for s in range(0, 120, 20)], dtype=torch.int32)),
    "p0": ({"p": 0.0}, 3, 300, 80, None, one_segment_per_cut([300, 200, 100])),
    "p1_no_segments": ({"p": 1.0}, 3, 300, 80, [300, 250, 170], None),
    "no_warp_none": ({"time_warp_factor": None, "p": 1.0}, 2, 300, 80, None, one_segment_per_cut([300, 300])),
    "no_warp_zero": ({"time_warp_factor": 0, "p": 1.0}, 2, 300, 80, None, None),
    "no_feature_masks": ({"num_feature_masks": 0, "p": 1.0}, 2, 400, 80, None, one_segment_per_cut([400, 380])),
    "one_mask_per_axis": ({"num_feature_masks": 1, "num_frame_masks": 1, "p": 1.0}, 3, 400, 80, None, one_segment_per_cut([400, 380, 200])),
    "short_batch_one_frame_mask": ({"p": 1.0, "time_warp_factor": 10}, 3, 50, 80, None, one_segment_per_cut([50, 40, 30])),
    "many_masks": ({"num_feature_masks": 5, "features_mask_size": 10, "num_frame_masks": 20, "frames_mask_size": 30,
                    "max_frames_mask_fraction": 0.5, "p": 1.0}, 2, 500, 80, None, one_segment_per_cut([500, 480])),
    "F13_mask_wider_than_axis": ({"p": 1.0}, 3, 400, 13, [400, 300, 250], one_segment_per_cut([400, 300, 250])),
    "F81": ({"p": 1.0}, 2, 350, 81, [350, 200], one_segment_per_cut([350, 200])),
    "F257": ({"p": 1.0, "features_mask_size": 80}, 2, 330, 257, [330, 280], None),
    "padding_enters_mean": ({"p": 1.0, "time_warp_factor": 30}, 4, 900, 80, [900, 300, 120, 70], one_segment_per_cut([900, 300, 120, 70])),
}


def case_input(name, seed=0):
    kw, B, T, F, lens, segs = CASES[name]
    return kw, make_batch(B, T, F, lens, seed=seed + len(name)), segs


def regions(warps, masks, shape):
    """Boolean (B, T, F) arrays: inside a planned mask rectangle, inside a planned warped segment."""
    masked, warped = np.zeros(shape, bool), np.zeros(shape, bool)
    for m in masks:
        if m["axis"] == 0:
            masked[m["seq"], m["start"]:m["end"], :] = True
        else:
            masked[m["seq"], :, m["start"]:m["end"]] = True
    for w in warps:
        warped[w["seq"], w["start"]:w["start"] + w["len"], :] = True
    return masked, warped


def truth64(x, warps):
    """lhotse's time_warp arithmetic (signal_transforms.py:355-368) on the float64 input with the planned center / warped."""
    out = x.double().clone()
    F = x.shape[2]
    for w in warps:
        b, s, t, c, wd = (int(w[k]) for k in ("seq", "start", "len", "center", "warped"))
        seg = x[b, s:s + t].double().unsqueeze(0).unsqueeze(0)
        left = torch.nn.functional.interpolate(seg[:, :, :c, :], size=(wd, F), mode="bicubic", align_corners=False)
        right = torch.nn.functional.interpolate(seg[:, :, c:, :], size=(t - wd, F), mode="bicubic", align_corners=False)
        out[b, s:s + t] = torch.cat((left, right), dim=2)[0, 0]
    return out.numpy()


def check_against_lhotse(ours, mean_source, x, lhotse_out, warps, masks, what=""):
    """`ours` (numpy, what the kernels or the harness made of `x` under the plan) against lhotse's output on the same input
    under the same draws: the same masked set, bit-equal to the input outside masks and warped segments, the warped values
    within twice lhotse's own float32 error of the float64 warp, the mask value within 1 float32 ulp of the float64 mean of
    `mean_source` (the warped, unmasked batch)."""
    x, L = x.numpy(), lhotse_out.numpy()
    masked, warped = regions(warps, masks, x.shape)
    plain = ~masked & ~warped
    assert np.array_equal(ours[plain].view(np.int32), x[plain].view(np.int32)), what
    assert np.array_equal(L[plain].view(np.int32), x[plain].view(np.int32)), what
    t64 = truth64(torch.from_numpy(x), warps)
    w = warped & ~masked
    bound = np.maximum(2 * np.abs(L[w] - t64[w]), 1e-6 * np.abs(x).max())
    err = np.abs(ours[w] - t64[w])
    assert (err <= bound).all(), (what, float((err - bound).max()))
    for b in range(x.shape[0]):
        if not masked[b].any():
            continue
        v = L[b][masked[b]][0]
        assert np.array_equal(L[b] == v, masked[b]), (what, b)  # lhotse masked exactly the planned positions
        ours_v = ours[b][masked[b]]
        assert (ours_v == ours_v[0]).all(), (what, b)
        m64 = mean_source[b].astype(np.float64).mean()
        assert abs(float(ours_v[0]) - m64) <= np.spacing(np.float32(abs(m64))), (what, b, float(ours_v[0]), m64)


def build_harness(tmp_dir):
    import shutil

    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    src = os.path.join(root, "scripts", "micro", "specaug_host_check.cu")
    exe = str(tmp_dir / "specaug_host_check")
    gxx = shutil.which("g++")
    if gxx:
        for flags in (["-fsanitize=address", "-fno-omit-frame-pointer"], []):
            res = subprocess.run([gxx, "-x", "c++", "-std=c++17", "-O1", "-g", *flags, "-o", exe, src], capture_output=True, text=True)
            if res.returncode == 0:
                return exe
    return None


def run_harness(exe, tmp_path, x, warps, masks):
    """The CPU run of csrc/specaug.cuh on `x` (torch, (B, T, F)) under the tables -> (output, per-sequence mask values)."""
    B, T, F = x.shape
    x.numpy().tofile(tmp_path / "in.f32")
    warps.tofile(tmp_path / "warps.bin")
    masks.tofile(tmp_path / "masks.bin")
    env = dict(os.environ, ASAN_OPTIONS="detect_leaks=0:abort_on_error=0")
    files = [str(tmp_path / f) for f in ("in.f32", "warps.bin", "masks.bin", "out.f32", "means.f32")]
    r = subprocess.run([exe, *files[:3], str(B), str(T), str(F), *files[3:]], capture_output=True, text=True, env=env)
    assert r.returncode == 0 and "AddressSanitizer" not in r.stderr, r.stdout[-2000:] + r.stderr[-4000:]
    return np.fromfile(files[3], np.float32).reshape(B, T, F), np.fromfile(files[4], np.float32)
