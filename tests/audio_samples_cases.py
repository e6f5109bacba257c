"""Test-only: the batches `FusedAudioSamples` is checked on, the NumPy restatement of csrc/collate.cuh's row plan, and the host
harness that runs the header's index math under AddressSanitizer."""
import os
import shutil
import subprocess

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def setup_reference():
    """Imports lhotse and installs lhotse_env's stdlib-`wave` audio backend without re-binding lhotse_b200's base classes:
    lhotse_env.setup_lhotse reloads the extractor modules when they were imported without lhotse, which would change the
    classes that other test modules of the same session imported.  FusedAudioSamples needs lhotse's classes, not the rebinding."""
    import lhotse_env

    import lhotse_b200.base as lb_base

    had = lb_base.HAVE_LHOTSE
    lb_base.HAVE_LHOTSE = True  # setup_lhotse then only imports the reference and installs the backend
    try:
        lhotse_env.setup_lhotse()
    finally:
        lb_base.HAVE_LHOTSE = had


def plan(base_mod4, b, T):
    """The kernel's units of row b: [(first element, count, vector)] in unit order (head, float4 body, tail)."""
    h = min((4 - (base_mod4 + b * T) % 4) % 4, T)
    nv = (T - h) // 4
    return [(0, h, False)] + [(h + 4 * k, 4, True) for k in range(nv)] + [(h + 4 * nv, T - h - 4 * nv, False)]


def restate(src, offsets, lens, T, base_mod4=0):
    """(B, T) float32 that the kernel writes: row b's units filled from the source (int16 widened as q / 32768), zeros past
    the cut.  Each element is written once; an element left unwritten stays NaN."""
    src = np.asarray(src)
    x = src.astype(np.float32) * np.float32(1.0 / 32768.0) if src.dtype == np.int16 else src.astype(np.float32)
    out = np.full((len(lens), T), np.nan, np.float32)
    for b, (o, n) in enumerate(zip(offsets, lens)):
        for j, cnt, _ in plan(base_mod4, b, T):
            for e in range(j, j + cnt):
                assert np.isnan(out[b, e])
                out[b, e] = x[o + e] if e < n else np.float32(0.0)
    return out


def pack(rows, dtype, align=4):
    """Rows back to back on `align`-element boundaries, gaps zero: (buffer, offsets, lengths)."""
    lens = [len(r) for r in rows]
    offs, cur = [], 0
    for n in lens:
        cur = (cur + align - 1) // align * align
        offs.append(cur)
        cur += n
    buf = np.zeros(max(cur, 1), dtype)
    for r, o in zip(rows, offs):
        buf[o: o + len(r)] = r
    return buf, offs, lens


def load_f32(cut):
    return np.asarray(cut.load_audio(), np.float32)[0]


def lhotse_batches(root, noise):
    """name -> CutSet: plain, durations one sample short of the longest, speed / volume perturbed, resampled, CutMix,
    padding and concatenation.  `root`: a directory for the WAV files; `noise`: cuts CutMix draws from."""
    import lhotse_env
    from lhotse.dataset.cut_transforms import CutMix

    sr = 16000
    plain = list(lhotse_env.make_cutset(root, [1.0, 1.0 - 1 / sr, 0.7, 1.3 - 3 / sr, 0.25 + 1 / sr], seed=11, prefix="p"))
    out = {
        "plain": plain,
        "one_short": [plain[0], plain[1]],
        "speed": [c.perturb_speed(0.9) for c in plain[:3]] + [plain[3].perturb_speed(1.1), plain[4]],
        "volume": [plain[0].perturb_volume(1.3), plain[1].perturb_volume(0.5), plain[2]],
        "resample": [c.resample(8000) for c in plain],
        "padding_concat": [plain[0].pad(duration=1.5), plain[2].append(plain[4]), plain[1]],
    }
    from lhotse import CutSet

    out["cutmix"] = list(CutMix(cuts=CutSet.from_cuts(noise), p=1.0, snr=(10, 20), seed=3)(CutSet.from_cuts(plain)))
    return {k: CutSet.from_cuts(v) for k, v in out.items()}


def build_harness(tmp_dir):
    src = os.path.join(ROOT, "scripts", "micro", "collate_host_check.cu")
    gxx = shutil.which("g++") or shutil.which("c++")
    if gxx is None:
        return None
    exe = os.path.join(str(tmp_dir), "collate_host_check")
    for flags in (["-fsanitize=address", "-fno-omit-frame-pointer"], []):
        res = subprocess.run([gxx, "-x", "c++", "-std=c++17", "-O1", "-g", *flags, "-o", exe, src], capture_output=True, text=True)
        if res.returncode == 0:
            return exe
    raise RuntimeError("collate_host_check does not compile:\n" + res.stderr)


def run_harness(exe, tmp_path, src, offsets, lens, T, base_mod4):
    src = np.ascontiguousarray(src)
    src.tofile(tmp_path / "src.bin")
    np.concatenate([np.asarray(offsets, np.int64), np.asarray(lens, np.int64)]).tofile(tmp_path / "table.i64")
    dt = 1 if src.dtype == np.int16 else 0
    res = subprocess.run([exe, str(tmp_path / "src.bin"), str(dt), str(tmp_path / "table.i64"), str(T), str(base_mod4),
                          str(tmp_path / "out.f32")], capture_output=True, text=True)
    assert res.returncode == 0, res.stderr
    return np.fromfile(tmp_path / "out.f32", dtype=np.float32).reshape(len(lens), T)


def edge_table(rs, dtype):
    """A source and per-row (offset, length) over lengths = 0..3 mod 4, len 0, len == T, odd offsets, for T in a few sizes:
    [(T, src, offsets, lens)]."""
    out = []
    for T in (1, 2, 3, 4, 5, 7, 8, 13, 64, 257, 4099):
        lens = sorted({0, T, max(T - 1, 0), min(T, 1), T // 2, max(T - 2, 0), max(T - 3, 0), (T * 3) // 4})
        lens = (lens * 3)[: max(9, len(lens))]  # at least 9 rows: every row start alignment for odd T
        if dtype == np.int16:
            src = rs.randint(-32768, 32768, size=sum(lens) + 4 * len(lens) + 8).astype(np.int16)
        else:
            src = rs.randn(sum(lens) + 4 * len(lens) + 8).astype(np.float32)
        offs, cur = [], 0
        for i, n in enumerate(lens):
            cur += i % 4 if i % 5 == 3 else (-cur) % 4  # most rows on 4-sample boundaries, some not
            offs.append(cur)
            cur += n
        assert cur <= src.shape[0]
        out.append((T, src, offs, lens))
    return out
