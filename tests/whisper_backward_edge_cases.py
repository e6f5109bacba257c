"""Shared pieces of the whisper-fbank backward's edge tests (tests/test_whisper_backward_kernel_edges.py; csrc/backward.cuh,
DESIGN.md §3.1p): the table of cut lengths and filter counts, each with the columns its edges are read from; the forward
tile the fast400 kernel and its tiled normalise pass run, read from the header; the right-mirror reach of a length;
bwd_sample's per-sample fold of one frame's gradient, in float32 and in its order; and the forward's saved rows per cut."""
from __future__ import annotations

import os
import re
from dataclasses import dataclass

import numpy as np
import torch

import whisper_backward_cases as WB

HOP, N_FFT, PAD = WB.HOP, WB.N_FFT, WB.N_FFT // 2


def fast400_tile() -> int:
    """Rows of one fast400 tile (and of one CTA of the tiled normalise pass): 4 * F400_WARPS * F400_SLOTS, from the header."""
    src = open(os.path.join(WB.ROOT, "lhotse_b200", "csrc", "fast400.cuh")).read()
    warps = int(re.search(r"#define F400_WARPS (\d+)", src).group(1))
    slots = int(re.search(r"#define F400_SLOTS (\d+)", src).group(1))
    return 4 * warps * slots  # four quarter-warps per warp


def fast400_max_filters() -> int:
    """The largest M fast400_supported takes: F400_SLOTS * round4(M) <= 2 * F400_XBUF, from the header."""
    src = open(os.path.join(WB.ROOT, "lhotse_b200", "csrc", "fast400.cuh")).read()
    slots = int(re.search(r"#define F400_SLOTS (\d+)", src).group(1))
    xbuf = int(re.search(r"#define F400_XBUF (\d+)", src).group(1))
    return 2 * xbuf // slots // 4 * 4


def right_reach(n: int) -> int:
    """Padded positions past the cut's end that its last stft frame covers: the frame ends at sample 160 T + 39, so the
    right mirror is reached only when n mod 160 <= 39, by 40 - n mod 160 positions."""
    T = n // HOP
    return max(0, (T - 1) * HOP - PAD + N_FFT - n)


@dataclass(frozen=True)
class Row:
    """A row of the table: a cut of n samples, M filters, the kernel `auto` picks for M, and the derived columns: T stft
    frames, R output rows, the backward's tiles of 16 frames and T mod 16, the forward's tiles of 56 rows (fast400), and
    the right-mirror positions the last frame reaches."""
    n: int
    M: int
    kernel: str
    T: int
    R: int
    tiles: int
    t16: int
    ftiles: int
    reach: int

    @property
    def name(self):
        return f"n{self.n}-M{self.M}"


LENGTHS = (201, 319, 2438, 2520, 2560, 2721, 2800, 5160, 7719, 7760, 8880, 8960, 9040)
SUBSET = (201, 2438, 2800, 7719, 8960, 9040)  # the lengths run at the other filter counts
TABLE = [Row(*r) for r in [
    # n      M    kernel     T   R  tiles T%16 ftiles reach
    (201, 80, "fast", 1, 1, 1, 1, 1, 0),        # one frame, no zero row
    (319, 80, "fast", 1, 2, 1, 1, 1, 0),        # one frame and the zero row
    (2438, 80, "fast", 15, 15, 1, 15, 1, 2),    # T = 15: one partial tile; right mirror, 2 positions
    (2520, 80, "fast", 15, 16, 1, 15, 1, 0),    # T = 15 with the zero row
    (2560, 80, "fast", 16, 16, 1, 0, 1, 40),    # T = 16: one full tile; n mod 160 = 0, the whole mirror
    (2721, 80, "fast", 17, 17, 2, 1, 1, 39),    # T = 17: a one-frame second tile; n mod 160 = 1
    (2800, 80, "fast", 17, 18, 2, 1, 1, 0),     # T = 17 with the zero row
    (5160, 80, "fast", 32, 32, 2, 0, 1, 0),     # n mod 160 = 40: the last frame ends on the last sample
    (7719, 80, "fast", 48, 48, 3, 0, 1, 1),     # n mod 160 = 39: one mirrored position
    (7760, 80, "fast", 48, 49, 3, 0, 1, 0),     # T = 48 with the zero row
    (8880, 80, "fast", 55, 56, 4, 7, 1, 0),     # R = 56: one full forward tile, its last row the zero row
    (8960, 80, "fast", 56, 56, 4, 8, 1, 40),    # T = R = 56: one full forward tile
    (9040, 80, "fast", 56, 57, 4, 8, 2, 0),     # R = 57: the zero row alone in the second forward tile
]]
TABLE += [Row(r.n, 128, r.kernel, r.T, r.R, r.tiles, r.t16, r.ftiles, r.reach) for r in TABLE]
_BY_N = {r.n: r for r in TABLE if r.M == 80}
# M = 1: one value per row; 81: rows not float4-aligned (the normalise passes' scalar path); 264: the largest M of fast400's
# size rule (F400_SLOTS * round4(M) <= 2 * F400_XBUF), 49 of its filters empty (more filters than the 201 bins); 265: past
# that rule.  At M = 1 and 264 fast400_prepare declines the bank (its mel-round weights, one 200-bin filter or 17 rounds,
# do not fit the kernel's 113 KB shared-memory budget next to its frame buffers), so `auto` runs generic there too.
for M, kernel in ((1, "generic"), (81, "fast"), (264, "generic"), (265, "generic")):
    TABLE += [Row(n, M, kernel, *[getattr(_BY_N[n], c) for c in ("T", "R", "tiles", "t16", "ftiles", "reach")])
              for n in SUBSET]
MS = (1, 80, 81, 128, 264, 265)


def derived(n: int, R: int, ft: int, fwd_tile: int) -> tuple:
    """(T, R, tiles, T mod 16, forward tiles, reach) of a cut of n samples with R output rows, the backward's tile of ft
    frames and the forward's of fwd_tile rows."""
    T = n // HOP
    return T, R, -(-T // ft), T % ft, -(-R // fwd_tile), right_reach(n)


# ----------------------------------------------------------------------------- bwd_sample's fold of one frame
def expected_fold(Wp: np.ndarray, n: int) -> np.ndarray:
    """bwd_sample's per-sample sum (reflect = 1), in float32 and in its order, of the padded-position gradient Wp: own
    position, then the left mirror image (samples 1 .. 200), then the right one (samples n - 41 + n mod 160 .. n - 2);
    samples 0 and n - 1 have no image."""
    ext = Wp.shape[0]
    i = np.arange(n)
    acc = np.zeros(n, np.float32)
    own = i + PAD < ext
    acc[own] = acc[own] + Wp[(i + PAD)[own]]
    left = (i >= 1) & (i < PAD + 1)
    acc[left] = acc[left] + Wp[(PAD - i)[left]]
    qr = 2 * n - 2 - i + PAD
    right = (i < n - 1) & (qr < ext)
    acc[right] = acc[right] + Wp[qr[right]]
    return acc


# ----------------------------------------------------------------------------- the forward's saved rows
def pack(xs, dtype=torch.float32, align=8):
    """The cuts in one device buffer of `dtype` at `align`-element offsets: (buffer, lengths, offsets)."""
    lens = [int(np.asarray(x).shape[0]) for x in xs]
    offs, pos = [], 0
    for n in lens:
        offs.append(pos)
        pos += -(-n // align) * align
    buf = torch.zeros(max(pos, align), dtype=dtype)
    for x, o, n in zip(xs, offs, lens):
        buf[o:o + n] = torch.as_tensor(np.asarray(x)).to(dtype)
    return buf.cuda(), lens, offs


def keep_raw(ext, xs, dtype=torch.float32):
    """`extract_device_keep_raw` on the cuts packed as `pack` does: (features, [saved (R_i, M) rows], [maxima], row prefix),
    the rows and maxima as float32 NumPy."""
    buf, lens, offs = pack(xs, dtype)
    feats, raw, prefix = ext.engine.extract_device_keep_raw(buf, lens, offs)
    F = ext.engine.feature_dim
    R = int(prefix[-1])
    rows = raw[: R * F].view(R, F).cpu().numpy()
    maxima = raw[R * F:].cpu().numpy()
    return feats, [rows[prefix[i]:prefix[i + 1]] for i in range(len(xs))], [float(v) for v in maxima], prefix


def plain(ext, xs, dtype=torch.float32):
    """`extract_device` (the no-grad path) on the same packing."""
    buf, lens, offs = pack(xs, dtype)
    return ext.engine.extract_device(buf, lens, offs)[0]


def impulse_row(row: np.ndarray, saved: list, m: list) -> np.ndarray:
    """`row` zeroed wherever any of the given saved rows is at or below its cut's m - 8: every element left has weight 1 in
    each of those cuts, so the mass routed to the maximum is exactly 0 there, ties or not."""
    keep = np.ones(row.shape, bool)
    for xr, mm in zip(saved, m):
        keep &= xr > np.float32(mm) - np.float32(8.0)
    return np.where(keep, row, 0.0)
