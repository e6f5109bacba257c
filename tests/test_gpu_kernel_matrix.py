"""Every compiled kernel instantiation against the float64 oracle.

The fast kernels are templates: the host picks an instantiation per launch from the sample dtype, a compile-time frame
length (LCT), a launch shape and, for N = 512, the PLAIN flag (packed log-mel without energy, magnitude spectrum or output
affine).  CASES names the instantiation each row is meant to reach; `test_case_table_names_its_targets` (no GPU) checks
those labels against the plans and that every instantiation appears in some row.  The GPU tests then run every row in
both dtypes and both output layouts, the fused output affine on every kernel, unaligned cut starts, tile edges and
multi-chunk host staging.
"""
import zlib
from collections import namedtuple
from fractions import Fraction
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from helpers import gate
from lhotse_b200.engine import OUT_PACKED, OUT_PADDED, Engine
from lhotse_b200.plan import build_plan
from oracle import kaldi_oracle as O
from oracle import whisper_oracle as W

gpu = pytest.mark.gpu
PAD = -7.25  # not LOG_EPSILON: a pad row written with a default value would show

FAMILY_N = {"fast256": 256, "fast400": 400, "fast512": 512, "fast1024": 1024, "fast2048": 2048, "tc": 512}
SHAPE_ENV = {"fast512": "B200FEAT_FAST_VARIANT", "fast1024": "B200FEAT_FAST1024_VARIANT",
             "fast2048": "B200FEAT_FAST2048_VARIANT"}
SHAPES = {"fast512": (0, 2), "fast1024": (0, 1, 2, 3), "fast2048": (0, 1, 2, 3)}
CT_LENGTHS = {"fast512": (400,), "fast256": (200,), "fast1024": (600, 551), "fast2048": (1200, 1102)}


def compiled_length(family, L):
    """The LCT template argument the host dispatch picks for a frame length L (None: the family has no such argument)."""
    if family not in CT_LENGTHS:
        return None
    return L if L in CT_LENGTHS[family] else 0


# ------------------------------------------------------------------------------------------------ the case table
Case = namedtuple("Case", "family lct shape plain feature cfg")


def _cases():
    rows = []

    def add(family, lct, feature, cfg, shapes=(None,), plain=None):
        for s in shapes:
            rows.append(Case(family, lct, s, plain, feature, cfg))

    # fast512: LCT {400, 0} x shape {0, 2}; fbank without energy reaches PLAIN (packed) and general (padded)
    add("fast512", 400, "fbank", {}, (0, 2), plain=True)
    add("fast512", 0, "fbank", dict(frame_length=0.02), (0, 2), plain=True)                      # L = 320
    add("fast512", 400, "mfcc", dict(use_energy=True), (0,), plain=False)
    add("fast512", 0, "log-spectrogram", dict(frame_length=0.032, use_energy=True), (2,), plain=False)  # L = 512
    add("fast512", 0, "fbank", dict(frame_length=0.03, use_fft_mag=True, use_energy=True, htk_compat=True),
        (0,), plain=False)                                                                         # L = 480, energy last
    # fast256: LCT {200, 0}
    add("fast256", 200, "mfcc", dict(sampling_rate=8000, use_energy=True))
    add("fast256", 0, "fbank", dict(frame_length=0.016, frame_shift=0.008, use_energy=True, htk_compat=True))
    # fast400 (one instantiation per dtype)
    add("fast400", None, "fbank", dict(round_to_power_of_two=False, use_energy=True))
    # fast1024: LCT {600, 551, 0} x shape {0, 1, 2, 3}
    add("fast1024", 600, "fbank", dict(sampling_rate=24000, use_energy=True), (0, 1, 2, 3))
    add("fast1024", 551, "mfcc", dict(sampling_rate=22050, use_energy=True, htk_compat=True), (0, 1, 2, 3))
    add("fast1024", 0, "log-spectrogram", dict(sampling_rate=44100, frame_length=0.02), (0, 1, 2, 3))  # L = 882, S = 441
    # fast2048: LCT {1200, 1102, 0} x shape {0, 1, 2, 3}
    add("fast2048", 1200, "fbank", dict(sampling_rate=48000, use_energy=True, htk_compat=True), (0, 1, 2, 3))
    add("fast2048", 1102, "mfcc", dict(sampling_rate=44100, use_energy=True), (0, 1, 2, 3))              # S = 441
    add("fast2048", 0, "spectrogram", dict(sampling_rate=32000, frame_length=0.05, use_energy=True, raw_energy=False),
        (0, 1, 2, 3))                                                                              # L = 1600
    add("generic", None, "fbank", dict(use_energy=True, htk_compat=True))
    add("tc", None, "fbank", {})
    add("tc", None, "mfcc", dict(num_ceps=13, num_filters=23))
    return rows


CASES = _cases()


def case_id(c):
    extra = "-".join(f"{k}={v}" for k, v in sorted(c.cfg.items()))
    return f"{c.family}-L{c.lct}-s{c.shape}-{c.feature}" + (f"-{extra}" if extra else "")


def epilogue(c):
    """The epilogue branch a row's output takes: feature kind, energy column first or last, magnitude spectrum."""
    e = c.feature
    if c.cfg.get("use_energy"):
        e += "+energy-last" if c.cfg.get("htk_compat") else "+energy"
    return e + ("+mag" if c.cfg.get("use_fft_mag") else "")


def reached(c):
    """(family, LCT, PLAIN, shape, epilogue) instantiations a row launches over both output layouts."""
    if c.family == "fast512":
        plains = (False, True) if c.plain else (False,)
        return {(c.family, c.lct, pl, c.shape, epilogue(c)) for pl in plains}
    return {(c.family, c.lct, None, c.shape, epilogue(c))}


# None matches anything.  Beyond the template arguments, the general instantiations must run the epilogues that the
# PLAIN one compiles out (energy column first and last, MFCC, spectra, magnitude) and the tensor-core kernel both of its own.
REQUIRED = (
    [("fast512", lct, plain, s, None) for lct in (400, 0) for plain in (True, False) for s in SHAPES["fast512"]]
    + [("fast512", 400, False, 0, "mfcc+energy"), ("fast512", 0, False, 2, "log-spectrogram+energy"),
       ("fast512", 0, False, 0, "fbank+energy-last+mag")]
    + [("fast256", lct, None, None, None) for lct in (200, 0)]
    + [("fast400", None, None, None, None), ("generic", None, None, None, None),
       ("tc", None, None, None, "fbank"), ("tc", None, None, None, "mfcc")]
    + [(f, lct, None, s, None) for f in ("fast1024", "fast2048") for lct in CT_LENGTHS[f] + (0,) for s in SHAPES[f]]
)


def covers(req, inst):
    return all(r is None or r == i for r, i in zip(req, inst))


def plan_of(feature, cfg):
    return build_plan(feature, SimpleNamespace(**cfg))


def test_case_table_names_its_targets():
    """CPU only: every row's label matches its plan, no row repeats another, every instantiation has a row."""
    seen, got = set(), set()
    for c in CASES:
        key = (c.family, c.shape, c.feature, tuple(sorted(c.cfg.items())))
        assert key not in seen, f"duplicate row {case_id(c)}"
        seen.add(key)
        p = plan_of(c.feature, c.cfg)
        if c.family != "generic":
            assert p.N == FAMILY_N[c.family], (case_id(c), p.N)
        assert c.lct == compiled_length(c.family, p.L), (case_id(c), p.L)
        if c.family == "fast400":
            assert p.L == p.N == 400
        if c.family == "tc":
            assert c.feature in ("fbank", "mfcc") and not p.use_energy
        if c.family == "fast512":
            assert c.plain == (c.feature == "fbank" and not p.use_energy and not p.use_fft_mag), case_id(c)
        else:
            assert c.plain is None
        assert (c.shape is None) == (c.family not in SHAPES), case_id(c)
        assert p.energy_last == bool(c.cfg.get("htk_compat", False))
        got |= reached(c)
    missing = [r for r in REQUIRED if not any(covers(r, i) for i in got)]
    assert not missing, f"instantiations without a row: {missing}"


# ------------------------------------------------------------------------------------------------ helpers
def make_engine(family, feature, cfg, monkeypatch, shape=None):
    """An Engine on the kernel `family`; `shape` forces the launch shape (None: the one AUTO picks)."""
    if family in SHAPE_ENV:
        if shape is None:
            monkeypatch.delenv(SHAPE_ENV[family], raising=False)
        else:
            monkeypatch.setenv(SHAPE_ENV[family], str(shape))
    plan = plan_of(feature, cfg)
    kernel = family if family in ("generic", "tc") else "fast"
    eng = Engine(plan, 0, kernel=kernel)
    assert eng.kernel == kernel
    if family in FAMILY_N:
        assert plan.N == FAMILY_N[family]
    return eng


def oracle_cfg(feature, cfg, **over):
    c = {k: v for k, v in cfg.items() if k != "htk_compat"}
    c.update(over)
    return O.OracleConfig(feature=feature, **c)


def oracle(feature, cfg, x, dtype=torch.float32, **over):
    y = O.extract(x, oracle_cfg(feature, cfg, **over), dtype=dtype)
    if cfg.get("htk_compat"):  # energy (or C0's energy) in the last column
        y = np.roll(y, -1, axis=1)
    return y


def assert_gate(feature, cfg, x, got, **over):
    ref, truth = oracle(feature, cfg, x, **over), oracle(feature, cfg, x, torch.float64, **over)
    assert got.shape == ref.shape, (got.shape, ref.shape)
    ok, msg = gate(got, ref, truth, feature, cfg.get("use_energy", False), cfg.get("use_fft_mag", False))
    assert ok, msg


def signals(seed, lens):
    rs = np.random.RandomState(seed)
    xs = []
    for i, n in enumerate(lens):
        t = np.arange(n)
        x = 0.1 * rs.randn(n) + 0.05 * np.sin(2 * np.pi * (0.01 + 0.003 * i) * t)
        if i == 0:
            x += 0.02  # DC offset
        if i == 1:
            x[: n // 2] *= 1e-3  # a quiet stretch
        xs.append(x.astype(np.float32))
    return xs


def quantise(xs):
    return [np.clip(np.round(x * 32768.0), -32768, 32767).astype(np.int16) for x in xs]


def dequantise(qs):
    return [q.astype(np.float32) / np.float32(32768.0) for q in qs]


def aligned_offsets(lens, align, slack=0):
    offs, cur = [], 0
    for n in lens:
        cur = (cur + align - 1) // align * align
        offs.append(cur)
        cur += n + slack
    return offs


def run(eng, xs, out_mode=OUT_PACKED, offsets=None, pad=PAD):
    """All cuts in one device buffer (16-byte aligned starts unless `offsets`) -> (per-cut rows, per-cut pad rows)."""
    dt = xs[0].dtype
    lens = [len(x) for x in xs]
    if offsets is None:
        offsets = aligned_offsets(lens, 8 if dt == np.int16 else 4)
    buf = np.zeros(max(o + n for o, n in zip(offsets, lens)) + 16, dtype=dt)
    for o, x in zip(offsets, xs):
        buf[o: o + len(x)] = x
    out, prefix = eng.extract_device(torch.from_numpy(buf).cuda(), lens, offsets=list(offsets), out_mode=out_mode,
                                     pad_value=pad)
    out = out.cpu().numpy()
    Ts = np.diff(prefix)
    if out_mode == OUT_PACKED:
        assert out.shape[0] == prefix[-1]
        return [out[prefix[i]: prefix[i + 1]] for i in range(len(xs))], None
    return [out[i, :T] for i, T in enumerate(Ts)], [out[i, T:] for i, T in enumerate(Ts)]


def assert_same(a, b, what):
    assert len(a) == len(b)
    for i, (u, v) in enumerate(zip(a, b)):
        assert u.shape == v.shape and np.array_equal(u, v), f"{what}: cut {i} differs (max |d| {np.abs(u - v).max()})"


def assert_pad(tails, want):
    for t in tails:
        assert np.all(t == want[None, :] if np.ndim(want) else t == want)


def row_lengths(L, S):
    return [L, L + 1, 10 * S - 1, 10 * S + S // 2, 37 * S + 3, 90 * S + 7]


def seed_of(*parts):
    return zlib.crc32(repr(parts).encode()) & 0x7FFFFFFF


# ------------------------------------------------------------------------------------------------ 2. dtype x layout
@gpu
@pytest.mark.parametrize("c", CASES, ids=[case_id(c) for c in CASES])
def test_instantiation_vs_oracle(c, monkeypatch):
    """Each row in float32 and int16, packed and padded: every cut passes the gate against the float64 oracle; packed
    equals padded (on fast512: PLAIN equals general) and int16 equals float32 of q / 32768, bit for bit."""
    eng = make_engine(c.family, c.feature, c.cfg, monkeypatch, c.shape)
    L, S = eng.plan.L, eng.plan.S
    xs = signals(seed_of(c.feature, c.cfg), row_lengths(L, S))
    qs = quantise(xs)
    xq = dequantise(qs)
    packed, _ = run(eng, xs)
    for x, g in zip(xs, packed):
        assert_gate(c.feature, c.cfg, x, g)
    padded, tails = run(eng, xs, OUT_PADDED)
    assert_same(padded, packed, "float32 padded vs packed")
    assert_pad(tails, np.float32(PAD))
    fq, _ = run(eng, xq)
    for x, g in zip(xq, fq):
        assert_gate(c.feature, c.cfg, x, g)
    i16, _ = run(eng, qs)
    assert_same(i16, fq, "int16 vs float32(q / 32768), packed")
    i16p, tails = run(eng, qs, OUT_PADDED)
    assert_same(i16p, fq, "int16 padded vs float32 packed")
    assert_pad(tails, np.float32(PAD))


SHAPE_GROUPS = {}
for _c in CASES:
    if _c.family in SHAPES:
        SHAPE_GROUPS.setdefault((_c.family, _c.feature, tuple(sorted(_c.cfg.items()))), []).append(_c.shape)


@gpu
@pytest.mark.parametrize("family,feature,cfg_items", list(SHAPE_GROUPS),
                         ids=[f"{f}-{ft}-{dict(ci)}" for f, ft, ci in SHAPE_GROUPS])
def test_forced_launch_shapes_match_auto(family, feature, cfg_items, monkeypatch):
    """The shape AUTO picks and every forced shape of the same family give the same bits (both dtypes, both layouts)."""
    cfg = dict(cfg_items)
    auto = make_engine(family, feature, cfg, monkeypatch)
    L, S = auto.plan.L, auto.plan.S
    xs = signals(seed_of("shapes", feature, cfg), row_lengths(L, S))
    qs = quantise(xs)
    want = [run(auto, d, m)[0] for d in (xs, qs) for m in (OUT_PACKED, OUT_PADDED)]
    for shape in SHAPE_GROUPS[(family, feature, cfg_items)]:
        eng = make_engine(family, feature, cfg, monkeypatch, shape)
        got = [run(eng, d, m)[0] for d in (xs, qs) for m in (OUT_PACKED, OUT_PADDED)]
        for w, g, what in zip(want, got, ("f32 packed", "f32 padded", "i16 packed", "i16 padded")):
            assert_same(g, w, f"shape {shape} vs auto, {what}")


# ------------------------------------------------------------------------------------------------ 3. output affine
AFFINE_KERNELS = [("generic", None, {}), ("fast256", None, dict(sampling_rate=8000)),
                  ("fast400", None, dict(round_to_power_of_two=False)), ("fast512", 0, {}), ("fast512", 2, {}),
                  ("fast1024", None, dict(sampling_rate=24000)), ("fast2048", None, dict(sampling_rate=48000)),
                  ("tc", None, {})]
AFFINE_FEATURES = [("fbank", {}), ("fbank", dict(use_energy=True)), ("fbank", dict(use_energy=True, htk_compat=True)),
                   ("mfcc", {}), ("spectrogram", dict(use_energy=True)), ("log-spectrogram", {})]
AFFINE = [(fam, shape, feature, dict(geo, **fcfg)) for fam, shape, geo in AFFINE_KERNELS for feature, fcfg in AFFINE_FEATURES
          if fam != "tc" or (feature in ("fbank", "mfcc") and not fcfg)]


def ulps(a, b):
    """Distance in float32 units in the last place (finite values)."""
    def ordered(v):
        i = np.ascontiguousarray(v, dtype=np.float32).view(np.int32).astype(np.int64)
        return np.where(i < 0, -(i & 0x7FFFFFFF), i)
    return np.abs(ordered(a) - ordered(b))


def fma_near(v, scale, shift):
    """fmaf(v, scale[c], shift[c]) to within 1 ulp: the float64 product is exact, the sum is rounded twice."""
    return (v.astype(np.float64) * scale.astype(np.float64) + shift.astype(np.float64)).astype(np.float32)


def fma_exact(a, scale, shift):
    """fmaf(a, scale[c], shift[c]) per column, correctly rounded (round to nearest even)."""
    out = np.empty(scale.shape, dtype=np.float32)
    for c, (s, h) in enumerate(zip(scale, shift)):
        exact = Fraction(float(a)) * Fraction(float(s)) + Fraction(float(h))
        r = np.float32(float(exact))
        cands = (np.nextafter(r, np.float32(-np.inf)), r, np.nextafter(r, np.float32(np.inf)))
        out[c] = min(cands, key=lambda q: (abs(Fraction(float(q)) - exact), int(np.array(q).view(np.int32)) & 1))
    return out


def assert_affined(got, base, scale, shift, what):
    for i, (g, v) in enumerate(zip(got, base)):
        assert g.shape == v.shape and np.all(np.isfinite(g))
        d = ulps(g, fma_near(v, scale[None, :], shift[None, :]))
        assert d.max() <= 1, f"{what}: cut {i}, column {int(np.argmax(d.max(axis=0)))} is {int(d.max())} ulp off"


@gpu
@pytest.mark.parametrize("family,shape,feature,cfg", AFFINE,
                         ids=[f"{f}-s{s}-{ft}-{c}" for f, s, ft, c in AFFINE])
def test_output_affine_on_every_kernel(family, shape, feature, cfg, monkeypatch):
    """The fused per-column affine: fmaf(v, scale[c], shift[c]) of the kernel's own un-affined value, pad rows included;
    each special column (energy first / last, first and last mel or cepstral column, bin 0) gets its own scale and shift
    only; a new affine takes effect on the next call of a handle that has run; clearing it restores the bits."""
    eng = make_engine(family, feature, cfg, monkeypatch, shape)
    L, S, F = eng.plan.L, eng.plan.S, eng.feature_dim
    xs = signals(seed_of("affine", feature, cfg), [L + 1, 10 * S + S // 2, 57 * S + 3, 130 * S + 1])
    base, _ = run(eng, xs)                       # PLAIN on fast512 fbank
    base_pad, tails = run(eng, xs, OUT_PADDED)   # the general path
    assert_same(base, base_pad, "packed vs padded without affine")
    assert_pad(tails, np.float32(PAD))
    rs = np.random.RandomState(seed_of("affine-tables", family, feature, cfg))
    for rep in range(2):  # the second table replaces the first on a handle that has already run with one
        scale = rs.uniform(0.25, 4.0, F).astype(np.float32)
        shift = rs.uniform(-10.0, 10.0, F).astype(np.float32)
        eng.set_output_affine(scale, shift)
        got, _ = run(eng, xs)
        assert_affined(got, base_pad, scale, shift, f"packed, table {rep}")
        got, tails = run(eng, xs, OUT_PADDED)
        assert_affined(got, base_pad, scale, shift, f"padded, table {rep}")
        assert_pad(tails, fma_exact(PAD, scale, shift))
    for col in sorted({0, 1, F - 2, F - 1}):
        scale, shift = np.ones(F, dtype=np.float32), np.zeros(F, dtype=np.float32)
        scale[col], shift[col] = 2.5, 3.0 + col
        eng.set_output_affine(scale, shift)
        for mode in (OUT_PACKED, OUT_PADDED):
            got, tails = run(eng, xs, mode)
            for g, v in zip(got, base_pad):
                others = np.arange(F) != col
                assert np.array_equal(g[:, others], v[:, others]), f"column {col}'s affine reached another column"
                assert ulps(g[:, col], fma_near(v[:, col], scale[col], shift[col])).max() <= 1
            if tails is not None:
                assert_pad(tails, fma_exact(PAD, scale, shift))
    eng.set_output_affine(None, None)
    again, _ = run(eng, xs)
    assert_same(again, base, "packed after clearing the affine")
    again, tails = run(eng, xs, OUT_PADDED)
    assert_same(again, base_pad, "padded after clearing the affine")
    assert_pad(tails, np.float32(PAD))


# ------------------------------------------------------------------------------------------------ 4. alignment
ALIGN = [("generic", "fbank", {}), ("fast256", "fbank", dict(sampling_rate=8000)),
         ("fast400", "fbank", dict(round_to_power_of_two=False)), ("fast512", "fbank", {}),
         ("fast512", "mfcc", dict(use_energy=True)),
         ("fast1024", "fbank", dict(sampling_rate=24000)),                        # S = 240
         ("fast1024", "fbank", dict(sampling_rate=44100, frame_length=0.02)),     # S = 441
         ("fast2048", "fbank", dict(sampling_rate=48000)),                        # S = 480
         ("fast2048", "fbank", dict(sampling_rate=44100)),                        # S = 441
         ("tc", "fbank", {})]


@gpu
@pytest.mark.parametrize("family,feature,cfg", ALIGN, ids=[f"{f}-{ft}-{c}" for f, ft, c in ALIGN])
def test_unaligned_cut_starts(family, feature, cfg, monkeypatch):
    """The same odd-length cuts at every element offset modulo 16 bytes inside one device buffer, and back to back on the
    host path: the vector-load and the per-sample load paths give the aligned run's bits."""
    eng = make_engine(family, feature, cfg, monkeypatch)
    L, S = eng.plan.L, eng.plan.S
    lens = [n | 1 for n in (L + S, 7 * S + S // 2, 23 * S + 5, 61 * S + 2, L + 3)]
    xs = signals(seed_of("align", feature, cfg), lens)
    qs = quantise(xs)
    for data, lanes, truth_in in ((xs, 4, xs), (qs, 8, dequantise(qs))):
        ref, _ = run(eng, data)
        for x, g in zip(truth_in, ref):
            assert_gate(feature, cfg, x, g)
        slots = aligned_offsets(lens, 16, slack=8)
        for d in range(lanes):
            got, _ = run(eng, data, offsets=[o + d for o in slots])
            assert_same(got, ref, f"{data[0].dtype} cuts at element offset {d}")
        got, _ = run(eng, data, offsets=[o + (3 * i + 1) % lanes for i, o in enumerate(slots)])
        assert_same(got, ref, f"{data[0].dtype} cuts at mixed offsets")
        out, prefix = eng.extract_host(np.concatenate(data), lens)  # back to back: each cut starts where the last ended
        assert_same([out[prefix[i]: prefix[i + 1]] for i in range(len(lens))], ref, f"{data[0].dtype} back to back")


# ------------------------------------------------------------------------------------------------ 5. tile edges
TILES = [("generic", None, "fbank", {}), ("fast256", None, "fbank", dict(sampling_rate=8000)),
         ("fast400", None, "fbank", dict(round_to_power_of_two=False)), ("fast512", 0, "fbank", {}),
         ("fast512", 2, "fbank", dict(use_energy=True)), ("fast1024", None, "fbank", dict(sampling_rate=24000)),
         ("fast2048", None, "mfcc", dict(sampling_rate=48000)), ("tc", None, "fbank", {})]


def tile_frames(eng):
    """ft: the most frames one cut can have while it is still one work item of the kernel (from BatchTotals.total_tiles)."""
    L, S = eng.plan.L, eng.plan.S

    def tiles(T):  # one cut of T frames
        return int(eng.plan_batch([L + (T - 1) * S if eng.plan.snip_edges else T * S])[1].total_tiles)

    T = 16
    while tiles(T + 1) == tiles(T):
        T += 1
    ft = T // tiles(T)
    assert T % ft == 0 and tiles(ft) == 1 and tiles(ft + 1) == 2
    return ft


def edge_batch(eng, Ts, n_for):
    lens = []
    for T in sorted(set(t for t in Ts if t >= 1)):
        for n in n_for(T):
            try:
                if eng.num_frames(n) == T:
                    lens.append(n)
            except ValueError:  # too short to be framed
                pass
    return lens[::2] + lens[1::2][::-1]  # ragged order: short cuts next to long ones


def check_edges(eng, feature, cfg, lens, must_have, **over):
    xs = signals(seed_of("tiles", feature, cfg, over), lens)
    assert must_have <= {eng.num_frames(n) for n in lens}
    packed, _ = run(eng, xs)
    padded, tails = run(eng, xs, OUT_PADDED)
    assert_same(padded, packed, "padded vs packed")
    assert_pad(tails, np.float32(PAD))
    for x, g in zip(xs, packed):
        assert_gate(feature, cfg, x, g, **over)
        assert np.array_equal(run(eng, [x])[0][0], g), f"cut of {len(x)} samples alone differs from the batch"


@gpu
@pytest.mark.parametrize("family,shape,feature,cfg", TILES, ids=[f"{f}-s{s}-{ft}-{c}" for f, s, ft, c in TILES])
def test_tile_edges(family, shape, feature, cfg, monkeypatch):
    """Cuts of 1, ft - 1, ft, ft + 1 and 2 ft + 1 frames (ft: frames per work item) in one ragged batch, in both layouts,
    against the oracle and against the same cut alone; snip_edges cuts of L and L + S - 1 samples likewise."""
    eng = make_engine(family, feature, cfg, monkeypatch, shape)
    L, S = eng.plan.L, eng.plan.S
    ft = tile_frames(eng)
    Ts = (1, ft - 1, ft, ft + 1, 2 * ft + 1)
    lens = edge_batch(eng, Ts, lambda T: (T * S - S // 2, T * S + S - S // 2 - 1))  # shortest, longest cut of T frames
    check_edges(eng, feature, cfg, lens, {ft, ft + 1, 2 * ft + 1})
    snip = make_engine(family, feature, dict(cfg, snip_edges=True), monkeypatch, shape)
    assert tile_frames(snip) == ft
    lens = edge_batch(snip, Ts, lambda T: (L + (T - 1) * S, L + T * S - 1))
    assert L in lens and L + S - 1 in lens
    check_edges(snip, feature, cfg, lens, {1, ft, ft + 1, 2 * ft + 1}, snip_edges=True)


# ------------------------------------------------------------------------------------------------ 6. multi-chunk staging
CHUNK_ELEMS_F32 = (32 << 20) // 4  # the host entry points stage ~32 MB of samples per chunk
CHUNKS = [("fast512", "fbank", {}), ("fast1024", "fbank", dict(sampling_rate=24000, use_energy=True)),
          ("generic", "mfcc", {}), ("fast400", "whisper-fbank", {}), ("generic", "whisper-fbank", {})]


def host_chunks(lens, align, chunk_elems):
    """How the host entry points split a batch: whole cuts, a new chunk once the span exceeds chunk_elems."""
    offs = aligned_offsets(lens, align)
    n, b0 = 0, 0
    while b0 < len(lens):
        b1 = b0 + 1
        while b1 < len(lens) and offs[b1] + lens[b1] - offs[b0] <= chunk_elems:
            b1 += 1
        n, b0 = n + 1, b1
    return n


def whisper_check(x, got):
    """tests/test_whisper.py's gate: max|ours - truth64| <= max(2e-5, 3 max|ref32 - truth64|)."""
    ref, truth = W.extract(x), W.extract(x, dtype=torch.float64)
    assert got.shape == ref.shape
    err, noise = np.abs(got - truth).max(), np.abs(ref.astype(np.float64) - truth).max()
    assert err <= max(2e-5, 3.0 * noise), (err, noise)


def kaldi_windows(feature, cfg, x, got, S):
    """The oracle on windows of a long cut: interior frames depend only on their own samples."""
    T, n = got.shape[0], len(x)
    if T <= 300:
        return assert_gate(feature, cfg, x, got)
    for t0 in (0, T // 2, T - 100):
        t1 = min(t0 + 100, T)
        lo, hi = max(0, (t0 - 12) * S), min(n, (t1 + 12) * S)  # slice starts on a hop boundary
        ref, truth = oracle(feature, cfg, x[lo:hi]), oracle(feature, cfg, x[lo:hi], torch.float64)
        a0, a1, sh = t0 if lo == 0 else t0 + 2, t1 if hi == n else t1 - 2, lo // S
        ok, msg = gate(got[a0:a1], ref[a0 - sh: a1 - sh], truth[a0 - sh: a1 - sh], feature, cfg.get("use_energy", False))
        assert ok, f"frames {a0}..{a1}: {msg}"


@gpu
@pytest.mark.parametrize("family,feature,cfg", CHUNKS, ids=[f"{f}-{ft}-{c}" for f, ft, c in CHUNKS])
def test_multi_chunk_host_staging(family, feature, cfg, monkeypatch):
    """A batch of ~20 M float32 samples that extract_host and extract_host_list split into >= 3 chunks (each later
    chunk launches at a nonzero tile and cut index; whisper also offsets its per-cut maxima): every cut equals the
    same cut run alone through extract_device, bit for bit."""
    eng = make_engine(family, feature, cfg, monkeypatch)
    L, S = eng.plan.L, eng.plan.S
    rs = np.random.RandomState(seed_of("chunks", family, feature))
    lens = []
    for _ in range(9):
        lens += [int(rs.randint(L + S, 4 * S)) | 1, int(rs.randint(1_900_000, 2_500_000)), int(rs.randint(L + S, 20 * S))]
    assert host_chunks(lens, 1, CHUNK_ELEMS_F32) >= 3 and host_chunks(lens, 4, CHUNK_ELEMS_F32) >= 3
    xs = [(0.1 * rs.randn(n)).astype(np.float32) for n in lens]
    alone = [run(eng, [x])[0][0] for x in xs]
    per_chunk = 2 if feature == "whisper-fbank" else 1
    launches = eng.stats()["kernel_launches"]
    flat = np.concatenate(xs)
    out, prefix = eng.extract_host(flat, lens)
    assert eng.stats()["kernel_launches"] - launches >= 3 * per_chunk
    assert_same([out[prefix[i]: prefix[i + 1]] for i in range(len(xs))], alone, "extract_host packed")
    del out
    out, prefix = eng.extract_host(flat, lens, out_mode=OUT_PADDED, pad_value=PAD)
    Ts = np.diff(prefix)
    assert_same([out[i, :T] for i, T in enumerate(Ts)], alone, "extract_host padded")
    assert_pad([out[i, T:] for i, T in enumerate(Ts)], np.float32(PAD))
    del out, flat
    launches = eng.stats()["kernel_launches"]
    out, prefix = eng.extract_host_list(xs)
    assert eng.stats()["kernel_launches"] - launches >= 3 * per_chunk
    assert_same([out[prefix[i]: prefix[i + 1]] for i in range(len(xs))], alone, "extract_host_list")
    del out
    check = list(range(0, 6)) + [len(xs) - 3, len(xs) - 2, len(xs) - 1]  # short and long cuts, first and last chunk
    for i in check:
        if feature == "whisper-fbank":
            whisper_check(xs[i], alone[i])  # the whole cut: its maximum sets the clamp of every row
        else:
            kaldi_windows(feature, cfg, xs[i], alone[i], S)
