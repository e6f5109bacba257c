"""The SpecAugment kernels (csrc/specaug.cuh, DESIGN.md §3.1k) at their edges: hand-built b200feat_specaug tables against a
NumPy restatement of the contract, written from §3.1k and not from the header.  The tables reach every rows-per-CTA count from
8192 down to 1 (F from 1 to 12000, rows wider than a CTA's tile, last tiles only partly filled), segments that start or end on
a tile boundary or one row either side of it, segments over whole tiles, adjacent segments, segments at row 0 and ending at T,
len 2 and every (center, warped) of len 3, scales of 1/3999 and 3999, thousands of segments in one tile, 300 sequences (three
mean-kernel blocks), rectangles that are empty, one element wide, whole axes, duplicated or overlapping, fill grids of 1, 2 and
64 rows (capped, with many passes), more than 65535 rectangles in one call, and a call with none.  The CPU tests hold the
tables to those edges and the host harness to the restatement bit for bit; the GPU tests require the device to equal the
restatement bit for bit on both unit widths (128-bit units on aligned tensors, scalar ones on a view 4 bytes off), to leave a
sentinel bit pattern around the output, and, independently of the restatement, the warp to stay within a derived bound of
torch's float64 bicubic and every mask value within half an ulp of the float64 mean."""
import math
import os
import re
from functools import lru_cache

import numpy as np
import pytest

import specaug_cases as SC
from test_augment_kernel_edges import GAP, SENTINEL, _assert_sentinel_outside, _bits_equal, _filled
from test_specaugment import harness as sa_harness  # noqa: F401  (fixtures)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
with open(os.path.join(ROOT, "lhotse_b200", "csrc", "specaug.cuh")) as _f:
    SA = {k: int(v) for k, v in re.findall(r"^#define (\w+) (\d+)\b", _f.read(), re.M)}
TILE, THREADS, FILL_THREADS = SA["SA_TILE_ELEMS"], SA["SA_THREADS"], SA["SA_FILL_THREADS"]
FILL_PER_THREAD, FILL_GY_CAP = 8, 64  # b200feat_specaug: gridDim.y = min(ceil(largest rectangle / (8 * 256)), 64)
MEAN_BLOCK = 128                      # specaug_mean_kernel: one thread per sequence, 128 per block
U32 = 2.0 ** -24                      # float32 unit roundoff
F32 = np.float32


def rows_per_cta(F):
    return 1 if F >= TILE else TILE // F


def fill_gy(largest):
    return min(max(-(-largest // (FILL_PER_THREAD * FILL_THREADS)), 1), FILL_GY_CAP)


def unit_width(F, aligned=True):
    return 4 if aligned and F % 4 == 0 else 1


# ---- the restatement --------------------------------------------------------------------------------------------------

A = F32(-0.75)  # Keys' cubic convolution parameter


def _keys_near(s):
    """|s| <= 1: (A + 2) s^3 - (A + 3) s^2 + 1, as fma(((A + 2) s - (A + 3)) s, s, 1)."""
    from lhotse_b200.pcm_staging import _fma32

    return _fma32(_fma32(F32(A + 2), s, F32(-(A + 3))) * s, s, F32(1))


def _keys_far(s):
    """1 < |s| < 2: A s^3 - 5 A s^2 + 8 A s - 4 A, by Horner in FMAs."""
    from lhotse_b200.pcm_staging import _fma32

    return _fma32(_fma32(_fma32(A, s, F32(-5 * A)), s, F32(8 * A)), s, F32(-4 * A))


def warp_rows(warps):
    """Every output row of every segment: (seq, segment start, row in the segment, first input row of its part, len_in,
    len_out, row in the part)."""
    seq, start, ln, c, w = (warps[k].astype(np.int64) for k in ("seq", "start", "len", "center", "warped"))
    idx = np.repeat(np.arange(len(warps)), ln)
    r = np.arange(int(ln.sum())) - np.repeat(np.cumsum(ln) - ln, ln)
    left = r < w[idx]
    len_in = np.where(left, c[idx], ln[idx] - c[idx])
    len_out = np.where(left, w[idx], ln[idx] - w[idx])
    return seq[idx], start[idx], r, np.where(left, 0, c[idx]), len_in, len_out, np.where(left, r, r - w[idx])


def restate_warp(x, warps):
    """out = in outside the segments; inside, F.interpolate(bicubic, align_corners=False) of each part along time in the
    contract's float32 operations, every row and feature at once."""
    from lhotse_b200.pcm_staging import _fma32

    out = x.copy()
    if len(warps) == 0:
        return out
    seq, start, r, base, len_in, len_out, j = warp_rows(warps)
    scale = len_in.astype(F32) / len_out.astype(F32)
    src = _fma32(scale, j.astype(F32) + F32(0.5), F32(-0.5))
    fl = np.floor(src)
    u = src - fl
    v = F32(1) - u
    w = [_keys_far(u + F32(1)), _keys_near(u), _keys_near(v), _keys_far(v + F32(1))]
    X = [x[seq, start + base + np.clip(fl.astype(np.int64) - 1 + k, 0, len_in - 1), :] for k in range(4)]
    col = [wk[:, None] for wk in w]
    y = _fma32(col[0], X[0], _fma32(col[1], X[1], _fma32(col[2], X[2], col[3] * X[3])))
    out[seq, start + r, :] = y
    return out


def restate_mean(out, V):
    """Per tile of R rows, thread t adds units t, t + 256, ... (V elements each, in element order) to +0.0 in float64; the 256
    accumulators go through the pairwise tree 128, 64, ..., 1; the tiles are added in order to +0.0, divided by T * F and
    rounded to float32 once.  Threads past the last unit add nothing, which is adding +0.0 (no accumulator is ever -0.0)."""
    B, T, F = out.shape
    R = rows_per_cta(F)
    tiles = -(-T // R)
    per_tile = R * F
    K = -(-(per_tile // V) // THREADS)
    a = np.zeros((B, tiles * per_tile), np.float64)
    a[:, :T * F] = out.reshape(B, T * F)
    pad = np.zeros((B, tiles, K * THREADS * V), np.float64)
    pad[:, :, :per_tile] = a.reshape(B, tiles, per_tile)
    pad = pad.reshape(B, tiles, K, THREADS, V)
    acc = np.zeros((B, tiles, THREADS), np.float64)
    for k in range(K):
        for i in range(V):
            acc = acc + pad[:, :, k, :, i]
    w = THREADS // 2
    while w:
        acc[:, :, :w] = acc[:, :, :w] + acc[:, :, w:2 * w]
        w //= 2
    s = np.zeros(B, np.float64)
    for t in range(tiles):
        s = s + acc[:, t, 0]
    return (s / float(T * F)).astype(F32)


def restate(x, warps, masks, V):
    """§3.1k on `x` (float32 (B, T, F)) under the tables with units of V elements -> (out, the B mask values, out before the
    masks)."""
    unmasked = restate_warp(x, warps)
    means = restate_mean(unmasked, V)
    out = unmasked.copy()
    for m in masks:  # the rectangles, in any order: they all write their sequence's mean
        if m["axis"] == 0:
            out[m["seq"], m["start"]:m["end"], :] = means[m["seq"]]
        else:
            out[m["seq"], :, m["start"]:m["end"]] = means[m["seq"]]
    return out, means, unmasked


# ---- the tables ---------------------------------------------------------------------------------------------------------


class SaTable:
    """One b200feat_specaug call: a (B, T, F) input whose rows differ and hand-placed segments and rectangles."""

    def __init__(self, B, T, F, seed):
        self.B, self.T, self.F, self.seed = B, T, F, seed
        self.rs = np.random.RandomState(seed)
        self.w, self.m = [], []

    def warp(self, seq, start, end, center=None, warped=None):
        n = end - start
        assert n >= 2 and 0 <= start and end <= self.T
        c = int(self.rs.randint(1, n)) if center is None else center
        wd = int(self.rs.randint(1, n)) if warped is None else warped
        self.w.append((seq, start, n, c, wd))

    def mask(self, seq, axis, start, end):
        self.m.append((seq, axis, start, end))

    def build(self):
        from lhotse_b200.engine import SPECAUG_MASK_DTYPE, SPECAUG_WARP_DTYPE

        self.warps = np.zeros(len(self.w), SPECAUG_WARP_DTYPE)
        self.warps["struct_size"] = SPECAUG_WARP_DTYPE.itemsize
        if self.w:
            (self.warps["seq"], self.warps["start"], self.warps["len"], self.warps["center"],
             self.warps["warped"]) = np.asarray(self.w, np.int64).T
        self.masks = np.zeros(len(self.m), SPECAUG_MASK_DTYPE)
        self.masks["struct_size"] = SPECAUG_MASK_DTYPE.itemsize
        if self.m:
            self.masks["seq"], self.masks["axis"], self.masks["start"], self.masks["end"] = np.asarray(self.m, np.int64).T
        self.x = SC.make_batch(self.B, self.T, self.F, seed=self.seed).numpy()
        return self

    def elems(self):
        """Element count of every rectangle."""
        return (self.masks["end"] - self.masks["start"]).astype(np.int64) * np.where(self.masks["axis"] == 0, self.F, self.T)


def _boundary(F):
    """Four sequences around the first tile boundaries (R rows per CTA): seq 0 adjacent segments from row 0 to T that break one
    row before and after the first boundary and on the second; seq 1 a segment ending on the first boundary, one starting on it
    and ending a row past the second; seq 2 one segment over two whole tiles; seq 3 none.  T leaves the last tile part full."""
    R = rows_per_cta(F)
    T = max(3 * R + max(R // 3, 1), 16)
    if R > 1 and T % R == 0:
        T += 1
    t = SaTable(4, T, F, seed=F)
    for seq, cuts in ((0, [(0, R - 1), (R - 1, R + 1), (R + 1, 2 * R), (2 * R, T)]),
                      (1, [(1, R), (R, 2 * R + 1), (2 * R + 3, T - 1)]),
                      (2, [(R - 1, 3 * R + 1)])):
        for a, e in cuts:
            if e - a >= 2 and a >= 0 and e <= T and not any(a < s + n and s < e for q, s, n, _, _ in t.w if q == seq):
                t.warp(seq, a, e)
    t.mask(0, 0, R - 1, R + 1)            # two rows over warped ones
    t.mask(1, 1, F - 1, F)                # the last column
    t.mask(3, 0, T - 1, T)                # the last row
    t.mask(3, 1, 0, min(2, F))
    return t.build()


def _scales():
    """len 4000 with (1, 3999) and (3999, 1): scales of 1/3999 and 3999, every tap clamped or src about 2000; then len 2 and
    every (center, warped) of len 3, adjacent, the last ending at T."""
    t = SaTable(2, 4100, 4, seed=41)
    t.warp(0, 0, 4000, 1, 3999)
    t.warp(0, 4000, 4002, 1, 1)
    for k, (c, w) in enumerate(((1, 1), (1, 2), (2, 1), (2, 2))):
        t.warp(0, 4002 + 3 * k, 4005 + 3 * k, c, w)
    t.warp(0, 4014, 4100)
    t.warp(1, 50, 4050, 3999, 1)
    t.warp(1, 4050, 4052, 1, 1)
    t.warp(1, 4097, 4100, 2, 1)
    t.mask(0, 0, 4050, 4060)
    t.mask(1, 0, 0, 10)
    return t.build()


def _packed():
    """F = 1: a tile of 8192 rows holds thousands of segments of len 2-5, adjacent in seq 0 (one across the tile boundary),
    with gaps of 0-2 rows in seq 1."""
    T = TILE + 600
    t = SaTable(2, T, 1, seed=7)
    for seq, gaps in ((0, False), (1, True)):
        a = 0
        while True:
            n = int(t.rs.randint(2, 6))
            if a + n > T:
                break
            t.warp(seq, a, a + n)
            a += n + (int(t.rs.randint(0, 3)) if gaps else 0)
    t.mask(0, 0, 100, 103)
    return t.build()


def _many_sequences():
    """B = 300: three blocks of the mean kernel.  Warps on every seventh sequence and on the last one (ending at T); masks on
    all but every fifth, so some have warps and no masks, most masks and no warps."""
    B, T, F = 300, 40, 80
    t = SaTable(B, T, F, seed=300)
    for b in range(B):
        if b % 7 == 3:
            a = int(t.rs.randint(0, T - 12))
            t.warp(b, a, a + int(t.rs.randint(2, 12)))
        if b % 5:
            axis = int(t.rs.randint(0, 2))
            n = T if axis == 0 else F
            a = int(t.rs.randint(0, n))
            t.mask(b, axis, a, min(n, a + int(t.rs.randint(1, 9))))
    t.warp(B - 1, T - 9, T)
    return t.build()


def _fill(B, T, F, seed, masks, warps):
    t = SaTable(B, T, F, seed)
    for w in warps:
        t.warp(*w)
    for m in masks:
        t.mask(*m)
    return t.build()


def _fill_2048():
    """The largest rectangle 2048 elements: one fill row per rectangle.  Empty rectangles on both axes (inside and at the
    end), one element wide on both axes, a duplicate, rectangles overlapping each other and the warped rows."""
    T, F = 256, 64
    return _fill(2, T, F, 2048, [(0, 0, 10, 42), (0, 0, 10, 42), (0, 0, 30, 50), (0, 0, 5, 5), (0, 1, 7, 7), (1, 0, T, T),
                                 (1, 1, F, F), (1, 1, 0, 0), (1, 0, T - 1, T), (1, 1, F - 1, F), (0, 1, 0, 1), (1, 1, 3, 8),
                                 (1, 1, 3, 8)],
                 [(0, 20, 60), (1, 0, 100), (1, 100, 256)])


def _fill_2049():
    """2049 elements (F = 3 columns of 683 rows, a whole axis either way): two fill rows."""
    return _fill(3, 683, 3, 2049, [(1, 1, 0, 3), (0, 0, 0, 683), (1, 1, 1, 2), (1, 1, 1, 2), (1, 0, 682, 683), (0, 1, 0, 0),
                                   (2, 1, 2, 2)],
                 [(0, 100, 200), (1, 0, 683), (2, 0, 300), (2, 300, 683)])


def _fill_131072():
    """131072 elements: 64 fill rows, the cap reached exactly."""
    return _fill(2, 1024, 128, 131072, [(0, 0, 0, 1024), (1, 1, 5, 6), (1, 0, 0, 1), (1, 1, 127, 128)],
                 [(1, 0, 500), (1, 600, 1024)])


def _fill_131073():
    """131073 elements (F = 1, T = 16 tiles and one row): the cap of 64 fill rows binds."""
    T = 16 * TILE + 1
    return _fill(2, T, 1, 131073, [(0, 1, 0, 1), (1, 0, 5, 9), (1, 0, T - 1, T)], [(0, TILE - 2, TILE + 3), (1, 1, T)])


def _fill_passes():
    """409600 elements (3.125 x 64 x 2048) on both axes: 25 passes of the capped fill grid."""
    return _fill(3, 1600, 256, 409600, [(0, 0, 0, 1600), (1, 1, 0, 256), (1, 0, 3, 4), (2, 0, 1599, 1600)],
                 [(0, 10, 40), (2, 0, 800), (2, 800, 1600)])


def _many_rectangles():
    """70000 rectangles of width 0-3 in one call (more than a grid's y or z dimension could hold); seq 3 has none."""
    B, T, F = 4, 200, 80
    t = SaTable(B, T, F, seed=70000)
    n = 70000
    seq, axis = t.rs.randint(0, 3, n), t.rs.randint(0, 2, n)
    size = np.where(axis == 0, T, F)
    start = (t.rs.rand(n) * (size + 1)).astype(np.int64)
    end = np.minimum(start + t.rs.randint(0, 4, n), size)
    t.m = list(zip(seq.tolist(), axis.tolist(), start.tolist(), end.tolist()))
    t.warp(0, 0, 200)
    t.warp(3, 10, 190)
    return t.build()


def _sum_order():
    """Cancellations that pin each level of the mean's float64 sum order (F = 4096: two rows per tile, V = 4 or 1).  With
    L = 2^53, L + 1 rounds to L but -L + 1 is exact, so (L + 1) - L = 0 while (-L + 1) + L = 1.  seq 0: L, 1, -L in tiles 0,
    1, 2 (tile order: 0, reversed 1).  seq 1: L, 1, -L in elements 0-2 (V = 4: one unit, element order, 0; V = 1: three
    threads, the tree, 1).  seq 2: L, -L, 1 in elements 0, 256 and 512 (V = 4: threads 0, 64, 128, the tree, 0; V = 1: one
    thread's units in order, 1).  Every sequence has one masked column."""
    t = _fill(3, 6, TILE // 2, 4096, [(b, 1, TILE // 2 - 1, TILE // 2) for b in range(3)], [])
    L = F32(2.0 ** 53)
    x = np.zeros_like(t.x)
    x[0, 0, 0], x[0, 2, 0], x[0, 4, 0] = L, 1, -L
    x[1, 0, :3] = L, 1, -L
    x[2, 0, 0], x[2, 0, 256], x[2, 0, 512] = L, -L, 1
    t.x = x
    return t


def _no_rectangles():
    """Warps and no rectangle: the mean and fill kernels are not launched."""
    return _fill(2, 300, 81, 81, [], [(0, 0, 150), (0, 150, 300), (1, 37, 38 + 200)])


BUILDERS = {
    **{f"F {F}": (lambda F=F: _boundary(F)) for F in (1, 2, 3, 4, 80, 81, 2049, 4096, 8192, 8193, 12000)},
    "scales": _scales, "packed": _packed, "300 sequences": _many_sequences, "fill 2048": _fill_2048, "fill 2049": _fill_2049,
    "fill 131072": _fill_131072, "fill 131073": _fill_131073, "fill passes": _fill_passes,
    "70000 rectangles": _many_rectangles, "no rectangles": _no_rectangles, "sum order": _sum_order,
}
LABELS = list(BUILDERS)


@lru_cache(maxsize=None)
def table(label):
    return BUILDERS[label]()


@lru_cache(maxsize=None)
def restated(label, V):
    t = table(label)
    return restate(t.x, t.warps, t.masks, V)


def _tile_segments(t):
    """The most segments that reach into one tile."""
    R = rows_per_cta(t.F)
    best = 0
    for b in range(t.B):
        w = t.warps[t.warps["seq"] == b]
        if len(w):
            first, last = w["start"] // R, (w["start"] + w["len"] - 1) // R
            best = max(best, int(np.bincount(np.concatenate([np.arange(a, e + 1) for a, e in zip(first, last)])).max()))
    return best


# ---- CPU: the tables reach their edges, the host harness is the restatement ----------------------------------------------


def test_specaug_tables_reach_their_edges():
    tabs = {k: table(k) for k in LABELS}
    # rows per CTA from 8192 down to 1, rows wider than a tile, the last tile part full
    Rs = {rows_per_cta(t.F) for t in tabs.values()}
    assert {TILE, TILE // 2, TILE // 4, 3, 2, 1} <= Rs
    assert any(t.F > TILE for t in tabs.values()) and any(t.F == TILE for t in tabs.values())
    assert any(rows_per_cta(t.F) * t.F < TILE for t in tabs.values())  # rows that do not fill a tile
    assert sum(rows_per_cta(t.F) > 1 and t.T % rows_per_cta(t.F) != 0 for t in tabs.values()) >= 6
    # both unit widths the host harness picks
    assert {unit_width(t.F) for t in tabs.values()} == {1, 4}
    # segments around tile boundaries, in every boundary table with R >= 3
    for F in (1, 2, 3, 4, 80, 81, 2049):
        t = tabs[f"F {F}"]
        R, T = rows_per_cta(F), t.T
        s, e = t.warps["start"].astype(np.int64), (t.warps["start"] + t.warps["len"]).astype(np.int64)
        assert R >= 3
        assert ((s % R == 0) & (s > 0)).any() and (s % R == 1).any() and (s % R == R - 1).any(), F
        assert ((e % R == 0) & (e < T)).any() and (e % R == 1).any() and (e % R == R - 1).any(), F
        assert (s == 0).any() and (e == T).any(), F
        assert ((-(-s // R) + 2) * R <= e).any(), F  # two whole tiles inside one segment
        same = t.warps["seq"][1:] == t.warps["seq"][:-1]
        assert (same & (e[:-1] == s[1:])).any(), F  # adjacent segments
    for F in (4096, 8192, 8193, 12000):
        t = tabs[f"F {F}"]
        assert (t.warps["len"] >= 3).any() and rows_per_cta(F) <= 2
    # short and extreme segments
    ws = {(int(w["len"]), int(w["center"]), int(w["warped"])) for t in tabs.values() for w in t.warps}
    assert (2, 1, 1) in ws and {(3, c, w) for c in (1, 2) for w in (1, 2)} <= ws
    assert (4000, 1, 3999) in ws and (4000, 3999, 1) in ws
    assert _tile_segments(tabs["packed"]) >= 2000 and tabs["packed"].F == 1
    # the mean kernel over three blocks, sequences with warps and no masks and the reverse, the last warp ending at T
    t = tabs["300 sequences"]
    assert -(-t.B // MEAN_BLOCK) >= 3
    warped, masked = set(t.warps["seq"].tolist()), set(t.masks["seq"].tolist())
    assert warped - masked and masked - warped and max(masked) == t.B - 1 and any(b >= 2 * MEAN_BLOCK for b in masked)
    last = t.warps[t.warps["seq"] == t.B - 1]
    assert (last["start"] + last["len"] == t.T).any()
    # rectangles: empty on both axes, whole axes, one element wide on both axes, duplicates, overlaps, over warped rows
    rects = [(lab, m, t) for lab, t in tabs.items() for m in t.masks if lab != "70000 rectangles"]
    assert any(m["start"] == m["end"] and m["axis"] == 0 for _, m, _ in rects)
    assert any(m["start"] == m["end"] and m["axis"] == 1 for _, m, _ in rects)
    assert any(m["start"] == m["end"] == t.T and m["axis"] == 0 for _, m, t in rects)
    for axis in (0, 1):
        assert any(m["axis"] == axis and m["start"] == 0 and m["end"] == (t.T if axis == 0 else t.F) for _, m, t in rects), axis
        assert any(m["axis"] == axis and m["end"] - m["start"] == 1 for _, m, _ in rects), axis
    assert any(len(t.masks) != len(np.unique(t.masks)) for t in tabs.values())
    masked_rows = [(lab, m) for lab, m, t in rects if m["axis"] == 0 and m["end"] > m["start"]]
    assert any(a is not b and la == lb and a["seq"] == b["seq"] and a["start"] < b["start"] < a["end"] < b["end"]
               for la, a in masked_rows for lb, b in masked_rows)
    over_warps = 0
    for t in tabs.values():
        masked, warped_ = SC.regions(t.warps, t.masks[:2000], (t.B, t.T, t.F))
        over_warps += int((masked & warped_).any())
    assert over_warps >= 5
    # fill grids: one row, two, exactly the cap, the cap with many passes; more than 65535 rectangles; none
    gys = {lab: fill_gy(int(t.elems().max())) if len(t.masks) else 0 for lab, t in tabs.items()}
    largest = {lab: int(t.elems().max()) if len(t.masks) else 0 for lab, t in tabs.items()}
    assert largest["fill 2048"] == 2048 and gys["fill 2048"] == 1
    assert largest["fill 2049"] == 2049 and gys["fill 2049"] == 2
    assert largest["fill 131072"] == FILL_GY_CAP * FILL_PER_THREAD * FILL_THREADS and gys["fill 131072"] == FILL_GY_CAP
    assert largest["fill 131073"] == 131073 and gys["fill 131073"] == FILL_GY_CAP
    assert largest["fill passes"] >= 3 * FILL_GY_CAP * FILL_PER_THREAD * FILL_THREADS
    assert len(tabs["70000 rectangles"].masks) > 65535 and len(tabs["no rectangles"].masks) == 0
    t = tabs["fill 131073"]
    assert t.T % TILE == 1  # a last tile of one row
    # the sum order: one mask value per order the cancellations distinguish
    t = tabs["sum order"]
    one = F32(1.0 / (t.T * t.F))
    assert rows_per_cta(t.F) == 2 and t.T == 3 * 2
    assert _bits_equal(restated("sum order", 4)[1], np.array([0, 0, 0], F32))
    assert _bits_equal(restated("sum order", 1)[1], np.array([0, one, one], F32))


@pytest.mark.parametrize("label", LABELS)
def test_host_harness_equals_restatement(sa_harness, tmp_path, label):
    import torch

    t = table(label)
    out, means, _ = restated(label, unit_width(t.F))
    got, got_means = SC.run_harness(sa_harness, tmp_path, torch.from_numpy(t.x), t.warps, t.masks)
    assert _bits_equal(got, out), label
    assert _bits_equal(got_means, means), label


def warp_bound(x, warps):
    """Per warped element, a bound on |ours - truth64| (torch's float64 bicubic of the same rows), derived a priori:

    position: scale = f32(len_in / len_out) and src = fma(scale, j + 0.5, -0.5) are each rounded once, so the float32 src is
      within ds = 2^-23 (scale (j + 0.5) + 1) rows of the exact one.  The interpolant is continuous in src (clamped taps
      repeat the edge row) with slope sum_k W_k'(u) x_k; the four weights sum to 1, so their derivatives sum to 0 and the
      slope is at most sum |W_k'| / 2 times the spread (max - min) of the rows near src.  |W'| <= 1.35 for |s| <= 1 and 0.75
      for 1 <= |s| <= 2, so sum |W_k'| <= 4.2, and the position term is 2.1 spread ds, the spread over the six rows
      floor(src) - 2 .. floor(src) + 3 (clamped) that either src's taps can reach.
    weights: u + 1 and 1 - u are rounded once (2^-24), then Horner in float32: the near polynomial's three roundings of values
      below 2.25 give at most 6 2^-24 and the argument 1.35 2^-24, the far polynomial's of values below 3.75 at most 12.25 2^-24
      and the argument 1.5 2^-24: sum |dw_k| <= 44 2^-24.
    chain: one product and three FMAs, each rounding a partial sum of at most sum |w_k| |x_k| <= 1.375 max|x| (Keys' weights at
      u = 1/2), so 5.5 2^-24 max|x|.
    So bound = 2.1 spread ds + 50 2^-24 max|x|, max|x| over the six rows; torch's own float64 error is below 2^-40 of that."""
    seq, start, r, base, len_in, len_out, j = warp_rows(warps)
    scale = len_in / len_out
    src = scale * (j + 0.5) - 0.5
    ds = 2.0 ** -23 * (scale * (j + 0.5) + 1.0)
    i0 = np.floor(src).astype(np.int64)
    near = np.stack([x[seq, start + base + np.clip(i0 + k, 0, len_in - 1), :] for k in range(-2, 4)]).astype(np.float64)
    spread = near.max(0) - near.min(0)
    big = np.abs(near).max(0)
    return (seq, start + r), 2.1 * spread * ds[:, None] + 50 * U32 * big


def check_against_float64(got, t, unmasked):
    """`got` (B, T, F): the warped, unmasked elements within warp_bound of SC.truth64, every other unmasked element the input
    bit for bit, every mask value within half an ulp of the float64 mean of `unmasked` plus the float64 sum's error."""
    import torch

    masked, warped = SC.regions(t.warps, t.masks, got.shape)
    plain = ~masked & ~warped
    assert _bits_equal(got[plain], t.x[plain])
    if len(t.warps):
        (seq, row), bound = warp_bound(t.x, t.warps)
        truth = SC.truth64(torch.from_numpy(t.x), t.warps)
        err = np.abs(got[seq, row, :].astype(np.float64) - truth[seq, row, :])
        seen = ~masked[seq, row, :]
        assert seen.any()
        worst = np.argmax(np.where(seen, err - bound, -np.inf))
        assert (err <= bound)[seen].all(), (float(err.flat[worst]), float(bound.flat[worst]))
        # far below the steps between neighbouring rows, so a wrong tap or clamp cannot hide in it
        assert float(np.median(bound[seen])) < 0.05 * float(np.median(np.abs(np.diff(t.x, axis=1))))
    for b in range(t.B):
        if not masked[b].any():
            continue
        v = got[b][masked[b]]
        assert (v.view(np.int32) == v[0].view(np.int32)).all(), b
        vals = unmasked[b].astype(np.float64).ravel()
        m64 = math.fsum(vals) / vals.size
        # the float64 sum: a chain of at most `depth` additions per element (units per thread, the tree, the tiles)
        R = rows_per_cta(t.F)
        depth = -(-R * t.F // THREADS) + int(math.log2(THREADS)) + -(-t.T // R)
        tol = 0.5 * float(np.spacing(F32(abs(m64)))) + 2.0 ** -53 * (depth * float(np.abs(vals).sum()) / vals.size + abs(m64))
        assert abs(float(v[0]) - m64) <= tol, (b, float(v[0]), m64)


@pytest.mark.parametrize("label", ["F 1", "F 81", "F 12000", "scales", "packed", "300 sequences", "fill 2048", "fill 2049"])
def test_restatement_against_float64(label):
    """The restatement itself against torch's float64 bicubic and an exact mean: what the GPU tests hold the device to is
    the operation, not only a copy of the header."""
    t = table(label)
    out, _, unmasked = restated(label, unit_width(t.F))
    check_against_float64(out, t, unmasked)


# ---- GPU: the device is the restatement on both unit widths -------------------------------------------------------------


def _device_run(t, aligned):
    """engine.specaug on `t` into a sentinel-filled buffer with sentinels on both sides of the output.  Aligned: the input
    and the output 16-byte aligned (128-bit units when F % 4 == 0); otherwise views 4 and 20 bytes into their allocations,
    which take the scalar kernel.  -> (the whole output buffer, the output's window, the input read back)."""
    import torch

    from lhotse_b200.engine import specaug

    dev = torch.device("cuda:0")
    n = t.x.size
    x_lead, o_lead = (0, 4) if aligned else (1, 5)
    xbuf = torch.zeros(n + x_lead, dtype=torch.float32, device=dev)
    x = xbuf[x_lead:].view(t.x.shape)
    x.copy_(torch.from_numpy(t.x))
    obuf = _filled(o_lead + n + GAP, dev)
    out = obuf[o_lead:o_lead + n].view(t.x.shape)
    assert (x.data_ptr() % 16 == 0 and out.data_ptr() % 16 == 0) == aligned
    specaug(x, out, t.warps, t.masks)
    torch.cuda.synchronize()
    return obuf.cpu().numpy(), (o_lead, n), x.cpu().numpy()


def _check_device(t, aligned, want, what):
    buf, (a, n), x_after = _device_run(t, aligned)
    _assert_sentinel_outside(buf, [(a, n)], what)
    got = buf[a:a + n]
    assert not (got.view(np.int32) == SENTINEL).any(), (what, "unwritten elements")
    assert _bits_equal(got.reshape(t.x.shape), want), what
    assert _bits_equal(x_after, t.x), (what, "the input changed")
    return got.reshape(t.x.shape)


@pytest.mark.gpu
@pytest.mark.parametrize("label", LABELS)
def test_gpu_aligned_equals_restatement(label):
    """128-bit units where F % 4 == 0, scalar ones otherwise: every element the restatement's bits, twice."""
    t = table(label)
    want, _, _ = restated(label, unit_width(t.F))
    first = _check_device(t, True, want, label)
    again = _check_device(t, True, want, label + " again")
    assert _bits_equal(first, again)


@pytest.mark.gpu
@pytest.mark.parametrize("label", LABELS)
def test_gpu_unaligned_equals_restatement_v1(label):
    """The same tables on views 4 bytes past 16-byte alignment: the scalar kernel, whose sum order the restatement with
    V = 1 pins, mask values included."""
    t = table(label)
    want, _, _ = restated(label, 1)
    _check_device(t, False, want, label)


@pytest.mark.gpu
@pytest.mark.parametrize("label", LABELS)
def test_gpu_against_float64(label):
    t = table(label)
    buf, (a, n), _ = _device_run(t, True)
    _, _, unmasked = restated(label, unit_width(t.F))
    check_against_float64(buf[a:a + n].reshape(t.x.shape), t, unmasked)


@pytest.mark.gpu
def test_gpu_loops_past_int_max():
    """B = 1, T = 1, F = 2^31 - 1 (odd: the scalar kernel): the warp kernel's one CTA walks 2^31 - 1 units and the fill
    kernel's 64 rows stride over a rectangle of 2^31 - 2 elements, both loop counters past 2^31 - 257.  Input 1 then zeros,
    the feature rectangle [1, F): out[0] stays 1, every other element is f32(1 / (2^31 - 1)).  Checked on the device."""
    import torch

    from lhotse_b200.engine import SPECAUG_FEATURE, SPECAUG_MASK_DTYPE, SPECAUG_WARP_DTYPE, specaug

    dev = torch.device("cuda:0")
    free, _ = torch.cuda.mem_get_info(dev)
    if free < 24 * 2 ** 30:
        pytest.skip(f"needs 24 GiB of free device memory, {free / 2 ** 30:.1f} GiB free")
    F = 2 ** 31 - 1
    masks = np.zeros(1, SPECAUG_MASK_DTYPE)
    masks["struct_size"], masks["seq"], masks["axis"], masks["start"], masks["end"] = SPECAUG_MASK_DTYPE.itemsize, 0, SPECAUG_FEATURE, 1, F
    x = torch.zeros((1, 1, F), dtype=torch.float32, device=dev)
    out = torch.zeros_like(x)
    try:
        x[0, 0, 0] = 1.0
        specaug(x, out, np.zeros(0, SPECAUG_WARP_DTYPE), masks)
        want = float(F32(1.0 / F))
        assert float(out[0, 0, 0]) == 1.0
        assert int((out[0, 0, 1:] != want).sum()) == 0
    finally:
        del x, out
        torch.cuda.empty_cache()
