"""The RIR generator (csrc/rirgen.cuh) and the float32 RIR source of the reverb (csrc/reverb.cuh) at their edges: hand-built
b200feat_rir_gen records whose arithmetic needs no libm (R = 0: coef = 1, every value f32(1 / dist); R so large that
exp(-0.16 R / T60) underflows: coef = 0, every image +0 and the direct path f32(1 / d0)), so that a NumPy restatement is exact.
One call mixes every rate from 1 Hz to 192 kHz (3 to 384001 entries, sort segments and 256-entry blocks across RIR
boundaries), more than 32 RIRs (three biquad CTAs), out_len on either side of a window CTA and at the ABI's maximum, comb_len
1 (every entry at position 0), clamped tails, uniforms on the cdf's values, 0 and 1 - 2^-53, windows reaching below position 0
and entries on a window's first and last tap, a tiny d0 that drives the clamp to both ends, and d0 above 170 T60 (images
before the direct path).  The CPU tests hold the table to those edges and the host harness to the restatement; the GPU tests
require the device to equal both, RIRs drawn from lhotse's generators to be the same bits in one mixed batch as alone, a
record with d0 >= 340 T60 to be refused before any launch, and the reverb's float32 source to take the first maximum and
give the host harness's y bit for bit.  Every output buffer starts filled with a sentinel bit pattern."""
import math
import re
from functools import lru_cache

import numpy as np
import pytest

import refshim
import rirgen_cases as RG
import test_reverb
import test_rirgen
from test_augment_kernel_edges import GAP, RV, RV_B, SENTINEL, _assert_sentinel_outside, _bits_equal, _filled
from test_reverb import harness as rv_harness  # noqa: F401  (fixtures)
from test_rirgen import harness as rg_harness  # noqa: F401

RG_DEFS = {}
with open(test_reverb.os.path.join(test_reverb.ROOT, "lhotse_b200", "csrc", "rirgen.cuh")) as _f:
    RG_DEFS = {k: int(v) for k, v in re.findall(r"^#define (\w+) (\d+)\b", _f.read(), re.M)}
THREADS, O, WIDTH, TAPS = RG_DEFS["RG_THREADS"], RG_DEFS["RG_O"], RG_DEFS["RG_WIDTH"], RG_DEFS["RG_TAPS"]
RATES = (1, 8000, 11025, 16000, 22050, 44100, 48000, 192000)
T60_AT = {1: 0.5, 8000: 0.1, 11025: 0.05, 16000: 0.05, 22050: 0.03, 44100: 0.02, 48000: 0.02, 192000: 0.005}
U_LAST = 1.0 - 2.0 ** -53  # the largest double below 1


def _same_or_zeros(a, b):
    """Bit for bit, but for the sign of a zero where both are zero (the dense and the sparse chain differ only there)."""
    return a.shape == b.shape and bool(np.all((a.view(np.int32) == b.view(np.int32)) | ((a == 0) & (b == 0))))


@lru_cache(maxsize=None)
def _cdf(image):
    from lhotse_b200 import rir_draws

    return rir_draws.multinomial_cdf(0.25, image)


class RgTable:
    """b200feat_rir_gen records over hand-placed draws and distributions, each output window followed by GAP sentinels."""

    def __init__(self):
        self.cases = []  # (sr, t60, r, d0, u, comb_len, out_len, label)
        self.rs = np.random.RandomState(5)

    def add(self, sr, t60, d0, u=None, zero=False, comb_len=None, out_len=None, label=""):
        from lhotse_b200.pcm_staging import resampled_len

        image = 2 * sr
        if u is None:
            u = self.rs.uniform(0.0, 1.0, image)
        L = int(math.ceil(64 * sr * t60)) if comb_len is None else comb_len
        n8 = resampled_len(1, L, O) if out_len is None else out_len
        r = 1e5 * t60 if zero else 0.0
        assert (math.exp(-0.16 * r / t60) == 0.0) if zero else r == 0.0
        self.cases.append((sr, t60, r, d0, np.asarray(u, np.float64), L, n8, label))

    def build(self):
        from lhotse_b200 import rir_draws
        from lhotse_b200.engine import RIR_GEN_DTYPE

        n = len(self.cases)
        rec = np.zeros(n, RIR_GEN_DTYPE)
        rec["struct_size"] = RIR_GEN_DTYPE.itemsize
        draws, cdfs, cdf_at = [], [], {}
        at = cdf_len = out = 0
        self.windows = []
        for i, (sr, t60, r, d0, u, L, n8, _) in enumerate(self.cases):
            image = 2 * sr
            if image not in cdf_at:
                cdf_at[image] = cdf_len
                cdfs.append(_cdf(image))
                cdf_len += image
            draws += [u, self.rs.uniform(-2.0, 2.0, image)]
            rec[i]["sampling_rate"], rec[i]["t60"], rec[i]["r"], rec[i]["d0"], rec[i]["tau"] = sr, t60, r, d0, 0.2
            (rec[i]["b0"], rec[i]["b1"], rec[i]["b2"], rec[i]["a1"],
             rec[i]["a2"]) = rir_draws.biquad_coefficients(8 * sr)
            rec[i]["cdf_elem"], rec[i]["draw_elem"] = cdf_at[image], at
            rec[i]["comb_len"], rec[i]["out_len"], rec[i]["out_elem"] = L, n8, out
            self.windows.append((out, n8))
            at += 2 * image
            out += n8 + GAP
        self.records, self.draws, self.cdf, self.out_elems = rec, np.concatenate(draws), np.concatenate(cdfs), out
        return self

    def u(self, i):
        rec = self.records[i]
        return self.draws[rec["draw_elem"]: rec["draw_elem"] + 2 * rec["sampling_rate"]]

    def cdf_of(self, i):
        rec = self.records[i]
        return self.cdf[rec["cdf_elem"]: rec["cdf_elem"] + 2 * rec["sampling_rate"]]


def entries(rec, u, cdf):
    """Every entry of an exact record (0: the direct path): its comb position and value, in NumPy without libm."""
    from lhotse_b200 import rir_draws

    sr, t60, r, d0, L = int(rec["sampling_rate"]), float(rec["t60"]), float(rec["r"]), float(rec["d0"]), int(rec["comb_len"])
    lin_end = np.float32(340.0 * t60 / d0 - 1.0)
    ratio = rir_draws.linspace32(1.0, float(lin_end), 2 * sr)[rir_draws.multinomial_from_uniforms(cdf, u)]
    dist = np.concatenate(([d0], d0 * ratio.astype(np.float64)))
    pos = np.minimum(np.ceil(dist * (64.0 * sr) / 340.0), L - 1).astype(np.int64)  # float64 products: exact on both sides
    val = (1.0 / dist).astype(np.float32)
    if r != 0.0:  # coef = 0: pow(0, refl >= 1) = +0 for every image
        val[1:] = 0.0
    return pos, val


def kept(pos, val):
    """The last entry of every position, in position order (a stable argsort, then the end of each run)."""
    order = np.argsort(pos, kind="stable")
    sp, sv = pos[order], val[order]
    last = np.r_[sp[1:] != sp[:-1], True]
    return sp[last], sv[last]


def restate(T):
    """The exact records' outputs at 8 sr: the dense last-wins comb through resample_reference, then the biquad (one loop
    over samples, every RIR at once) and the clamp.  Returns (per RIR out8, per RIR (kept positions, kept values))."""
    from lhotse_b200.pcm_staging import _fma32, resample_reference

    x8, combs = [], []
    for i, rec in enumerate(T.records):
        kp, kv = kept(*entries(rec, T.u(i), T.cdf_of(i)))
        comb = np.zeros(int(rec["comb_len"]) + O, np.float32)  # O more zeros: resample_reference keeps every output then
        comb[kp] = kv
        x8.append(resample_reference(comb, O, 1)[: int(rec["out_len"])])
        combs.append((kp, kv))
    n = len(x8)
    width = max(len(x) for x in x8)
    X = np.zeros((n, width), np.float32)
    for i, x in enumerate(x8):
        X[i, :len(x)] = x
    b0, b1, b2, a1, a2 = (T.records[k].astype(np.float32) for k in ("b0", "b1", "b2", "a1", "a2"))
    Y = np.empty_like(X)
    zero = np.zeros(n, np.float32)
    x1 = x2 = y1 = y2 = zero
    for t in range(width):
        x0 = X[:, t]
        fir = _fma32(x2, b2, zero)
        fir = _fma32(x1, b1, fir)
        fir = _fma32(x0, b0, fir)
        y0 = (fir - y2 * a2) - y1 * a1
        Y[:, t] = np.clip(y0, np.float32(-1), np.float32(1))
        x2, x1, y2, y1 = x1, x0, y1, y0
    return [Y[i, :len(x)] for i, x in enumerate(x8)], combs


@lru_cache(maxsize=1)
def rg_table():
    from lhotse_b200.pcm_staging import resampled_len

    T = RgTable()
    rs = T.rs
    for sr in RATES:  # every rate, both families
        t60 = T60_AT[sr]
        for zero in (False, True):
            T.add(sr, t60, float(rs.uniform(0.2, min(12.0, 0.9 * 340 * t60))), zero=zero, label=f"rate {sr}")
    L = int(math.ceil(64 * 8000 * 0.1))
    for n8 in (1, 255, 256, 257, L // O + 1, resampled_len(1, L, O), 3000):  # out_len around a window CTA and the ABI's cap
        T.add(8000, 0.1, 1.3, out_len=n8, label=f"out_len {n8}")
    T.add(8000, 0.1, 1.3, comb_len=1, out_len=1, label="comb_len 1")
    T.add(8000, 0.1, 0.1, comb_len=300, label="clamped tail")
    cdf = _cdf(16000)
    T.add(8000, 0.05, 2.0, u=np.full(16000, 0.37), label="equal u")
    T.add(8000, 0.05, 2.0, u=np.where(rs.rand(16000) < 0.5, cdf[rs.randint(0, 16000, 16000)].astype(np.float64),
                                       rs.uniform(0, 1, 16000)), label="u on cdf values")
    u = rs.uniform(0, 1, 16000)
    u[[5, 9000]], u[[100, 15999]] = 0.0, U_LAST
    T.add(8000, 0.05, 2.0, u=u, label="u 0 and 1 - 2^-53")
    T.add(8000, 0.05, 2.0, u=u, zero=True, label="coef 0, an image on the direct path")
    T.add(8000, 0.05, 0.02, label="direct path below the first window")
    T.add(8000, 0.05, 1e-4, label="tiny d0")
    T.add(8000, 0.02, 5.0, label="0 < lin_end < 1")
    T.add(8000, 0.1, 0.53125, label="d0 S / 340 an integer")
    for k in range(50):  # more RIRs: three biquad CTAs, the last one partial
        sr = int(rs.randint(1, 400))
        t60 = float(rs.uniform(0.05, 0.8))
        T.add(sr, t60, float(rs.uniform(0.2, min(12.0, 0.9 * 340 * t60))), zero=k % 3 == 0, label=f"small {k}")
    return T.build()


@lru_cache(maxsize=1)
def rg_restated():
    return restate(rg_table())


def _index(label):
    return [c[7] for c in rg_table().cases].index(label)


def test_rirgen_table_reaches_its_edges():
    from lhotse_b200.pcm_staging import resampled_len

    T = rg_table()
    rec = T.records
    out8, combs = rg_restated()
    n = len(rec)
    assert n > 2 * 32 and n % 32 != 0  # three biquad CTAs, the last one partial
    srs = set(rec["sampling_rate"].tolist())
    assert set(RATES) <= srs
    ents = 2 * rec["sampling_rate"].astype(np.int64) + 1
    assert ents.min() == 3 and ents.max() == 384001
    starts = np.concatenate(([0], np.cumsum(ents)[:-1]))
    assert ((starts % THREADS) != 0).sum() >= n // 2  # 256-entry blocks straddle RIR boundaries
    n8, L = rec["out_len"], rec["comb_len"]
    assert {1, THREADS - 1, THREADS, THREADS + 1} <= set(n8.tolist())
    full = [resampled_len(1, int(c), O) for c in L]
    assert (n8 == L // O + 1).any() and (n8 > np.asarray(full)).any()
    assert (n8 == np.asarray(full)).any() and (n8 < np.asarray(full)).any()
    ctas = (n8 + THREADS - 1) // THREADS
    assert (ctas >= 3).any() and (ctas == 1).any()
    # comb_len 1: every entry at 0, the last image kept
    i = _index("comb_len 1")
    pos, val = entries(rec[i], T.u(i), T.cdf_of(i))
    assert (pos == 0).all() and len(combs[i][0]) == 1 and combs[i][1][0] == val[-1] != val[0]
    i = _index("clamped tail")
    pos, _ = entries(rec[i], T.u(i), T.cdf_of(i))
    assert (pos == L[i] - 1).mean() > 0.5
    # uniforms: all on one position; exactly on cdf values; 0 (the direct path's position) and 1 - 2^-53 (the last slot)
    i = _index("equal u")
    pos, _ = entries(rec[i], T.u(i), T.cdf_of(i))
    assert len(set(pos[1:].tolist())) == 1
    i = _index("u on cdf values")
    assert np.isin(T.u(i), T.cdf_of(i).astype(np.float64)).sum() > 5000
    i = _index("u 0 and 1 - 2^-53")
    u, cdf = T.u(i), T.cdf_of(i)
    from lhotse_b200 import rir_draws

    idx = rir_draws.multinomial_from_uniforms(cdf, u)
    assert (idx[u == 0] == 0).all() and (idx[u == U_LAST] == len(cdf) - 1).all()
    pos, val = entries(rec[i], u, cdf)
    assert (pos[1:][u == 0] == pos[0]).all()
    assert np.flatnonzero(pos == pos[0])[-1] > 0  # an image is the last entry at the direct path's position
    # coef = 0 with an image on the direct path: the whole RIR is zero
    i = _index("coef 0, an image on the direct path")
    assert (combs[i][1] == 0).all() and (out8[i] == 0).all()
    # windows: entries below the first window's reach (lo < 0), on a window's first tap (lo) and on its last (hi)
    i = _index("direct path below the first window")
    assert combs[i][0][0] < WIDTH
    lo_hit = hi_hit = 0
    for (kp, _), m in zip(combs, n8):
        lo_hit += int(((kp % O == O - 1) & ((kp + WIDTH) // O < m)).sum())
        hi_hit += int(((kp % O == 0) & (kp >= TAPS - 1 - WIDTH) & ((kp - (TAPS - 1 - WIDTH)) // O < m)).sum())
    assert lo_hit > 100 and hi_hit > 100
    # d0: a tiny one clamps at both ends; 170 T60 < d0 < 340 T60 puts images before the direct path; an exact position
    i = _index("tiny d0")
    assert (out8[i] == 1.0).any() and (out8[i] == -1.0).any()
    i = _index("0 < lin_end < 1")
    lin_end = np.float32(340 * rec[i]["t60"] / rec[i]["d0"] - 1)
    pos, _ = entries(rec[i], T.u(i), T.cdf_of(i))
    assert 0 < lin_end < 1 and (pos[1:] < pos[0]).mean() > 0.9
    i = _index("d0 S / 340 an integer")
    q = float(rec[i]["d0"]) * 64.0 * float(rec[i]["sampling_rate"]) / 340.0
    assert q == int(q)
    # both families at every rate
    for sr in RATES:
        mine = rec[rec["sampling_rate"] == sr]
        assert (mine["r"] == 0).any() and (mine["r"] > 0).any(), sr


def test_host_rirgen_edges_equal_restatement(rg_harness, tmp_path):
    T = rg_table()
    out8, combs = rg_restated()
    host = test_rirgen.run_harness(rg_harness, tmp_path, T)
    for i, (h, w, (kp, kv)) in enumerate(zip(host, out8, combs)):
        assert np.array_equal(h[0], kp) and _bits_equal(h[1], kv), T.cases[i][7]
        assert _same_or_zeros(h[5], w), T.cases[i][7]


def _generate(T, records, dev):
    import torch

    from lhotse_b200.engine import rir_generate
    from lhotse_b200.pcm_staging import resample_kernel

    out = _filled(int(records["out_elem"].max() + records["out_len"].max()) + GAP, dev)
    rir_generate(torch.from_numpy(T.draws).to(dev), torch.from_numpy(T.cdf).to(dev), resample_kernel(8, 1)[0][0], records, out)
    torch.cuda.synchronize()
    return out.cpu().numpy()


@pytest.mark.gpu
def test_gpu_rirgen_edges_bit_equal(rg_harness, tmp_path):
    import torch

    T = rg_table()
    out8, _ = rg_restated()
    dev = torch.device("cuda:0")
    got = _generate(T, T.records, dev)
    host = test_rirgen.run_harness(rg_harness, tmp_path, T)
    for (a, n), w, h, c in zip(T.windows, out8, host, T.cases):
        assert _bits_equal(got[a:a + n], h[5]), ("harness", c[7])
        assert _same_or_zeros(got[a:a + n], w), ("restatement", c[7])
    _assert_sentinel_outside(got, T.windows, "out")


def _bad_records():
    T = RgTable()
    T.add(16000, 0.1, 3.0)
    T.add(16000, 0.1, 3.0)
    T.add(8000, 0.02, 6.8)  # d0 = 340 T60: lin_end = 0
    T.add(8000, 0.02, 6.8 * (1 + 1e-12))
    T.add(8000, 0.02, 12.0)
    return T.build()


def test_work_bytes_refuse_d0_beyond_340_t60():
    """The work-bytes query treats a record with d0 >= 340 T60 as malformed (0), before it asks the sort for scratch."""
    from lhotse_b200.engine import load_library

    lib = load_library()
    T = _bad_records()
    for k in (2, 3, 4):
        recs = np.ascontiguousarray(T.records[[0, 1, k]])
        assert int(lib.b200feat_rir_generate_work_bytes(recs.ctypes.data, 3)) == 0
        assert float(np.float32(340 * T.records[k]["t60"] / T.records[k]["d0"] - 1)) <= 0


@pytest.mark.gpu
def test_gpu_rirgen_refuses_d0_beyond_340_t60():
    import torch

    from lhotse_b200.engine import B200FeatError, rir_generate
    from lhotse_b200.pcm_staging import resample_kernel

    T = _bad_records()
    dev = torch.device("cuda:0")
    draws, cdf = torch.from_numpy(T.draws).to(dev), torch.from_numpy(T.cdf).to(dev)
    for k in (2, 3, 4):
        recs = T.records[[0, 1, k]]
        out = _filled(T.out_elems, dev)
        with pytest.raises(B200FeatError, match=r"rir_generate: rir 2: d0 must be below 340 T60"):
            rir_generate(draws, cdf, resample_kernel(8, 1)[0][0], recs, out)
        torch.cuda.synchronize()
        assert (out.cpu().numpy().view(np.int32) == SENTINEL).all()
    good = _generate(T, T.records[:2], dev)  # the same buffers are taken once the record is gone
    assert np.isfinite(good[:T.windows[1][0] + T.windows[1][1]][:T.records[0]["out_len"]]).all()


# ---- realistic records: lhotse's generators, one mixed batch against each RIR alone ---------------------------------


@pytest.mark.gpu
@pytest.mark.skipif(not refshim.reference_available(), reason="no reference tree / oracle/_ref archive")
def test_gpu_rirgen_batch_equals_each_alone(rg_harness, tmp_path):
    """RG.CASES and 40 bench-like generators (16 kHz, T60 ~ U(0.1, 0.8)) in one call: every RIR the same bits as in a call
    of its own, within the §3.1l bound of the float64 truth of its draws, and counted against the host harness (libm's
    exp / log10 / pow may differ from libdevice's by an ulp, so that is reported, not required)."""
    import torch

    import lhotse_env
    from lhotse_b200 import rir_draws
    from lhotse_b200.pcm_staging import resample_reference

    lhotse_env.setup_lhotse()
    gens = [RG.generator(*c) for c in RG.CASES] + [RG.generator(16000, 0.8, 500 + k, 600 + k) for k in range(40)]
    refs = [RG.generator(*c) for c in RG.CASES] + [RG.generator(16000, 0.8, 500 + k, 600 + k) for k in range(40)]
    torch.manual_seed(77)
    state = torch.get_rng_state()
    d = rir_draws.draw(gens)

    class T:  # the batch's draws as RgTable's fields
        draws, cdf, records = d.draws, d.cdf, d.records.copy()

    off = 0
    for r in T.records:
        r["out_elem"] = off
        off += int(r["out_len"]) + GAP
    dev = torch.device("cuda:0")
    batch = _generate(T, T.records, dev)
    windows = [(int(r["out_elem"]), int(r["out_len"])) for r in T.records]
    _assert_sentinel_outside(batch, windows, "batch")
    host = test_rirgen.run_harness(rg_harness, tmp_path, T)
    same_as_host = 0
    torch.set_rng_state(state)
    for i, ((a, n), r) in enumerate(zip(windows, T.records)):
        one = r.copy().reshape(1)
        one["out_elem"] = 0
        alone = _generate(T, one, dev)
        assert _bits_equal(batch[a:a + n], alone[:n]), i
        same_as_host += _bits_equal(batch[a:a + n], host[i][5])
        image = 2 * int(r["sampling_rate"])
        u = d.draws[r["draw_elem"]: r["draw_elem"] + image]
        pert = d.draws[r["draw_elem"] + image: r["draw_elem"] + 2 * image]
        ref, _, _ = RG.lhotse_rir(refs[i])
        truth, _, _ = RG.truth64(r, u, pert, refs[i])
        err, bnd = RG.bound(resample_reference(batch[a:a + n], 8, 1), ref, truth)
        assert err <= bnd, (i, err, bnd)
    print(f"generated RIRs bit-equal to the host harness: {same_as_host} of {len(windows)}")


# ---- the reverb's float32 RIR source ----------------------------------------------------------------------------------


def _float_tie_rir(peaks, seed, n=3000, peak=0.75):
    h = np.random.RandomState(seed).uniform(-0.3, 0.3, n).astype(np.float32)
    h[list(peaks)] = np.float32(peak)
    return h


@lru_cache(maxsize=1)
def rv32_table():
    """(RIRs, cases): float32 RIRs at the argmax's edges and the generated RIRs of rg_table at their rate, each with a random
    input and an impulse (whose y is the RIR from its shift on)."""
    from lhotse_b200.pcm_staging import resample_reference

    rs = np.random.RandomState(21)
    rirs, labels = [], []
    T = RV["RV_THREADS"]
    for k, peaks in enumerate(([5, 9], [20, T + 3], [40, 300], [200, T + 88], [7, T + 7, 2 * T + 7], [31, 32],
                               [480, 481, 1000])):
        rirs.append(_float_tie_rir(peaks, 700 + k))
        labels.append(f"tie {peaks}")
    rirs.append(-rs.uniform(1e-3, 0.5, 2500).astype(np.float32))
    labels.append("all negative")
    z = np.zeros(1500, np.float32)
    z[rs.rand(1500) < 0.5] = -0.0
    z[0] = -0.0
    rirs.append(z)
    labels.append("+0 and -0")
    for R in (RV_B - 1, RV_B, RV_B + 1, RV["RV_MAX_RIR"]):
        h = rs.uniform(-0.5, 0.5, R).astype(np.float32)
        h[-1] = np.float32(0.9)
        rirs.append(h)
        labels.append(f"maximum last of {R}")
    h = (rs.randn(3000) * 1e-32).astype(np.float32)  # h 2^-27 subnormal: rounded, not exact
    h[1234] = np.float32(1e-31)
    rirs.append(h)
    labels.append("subnormal products")
    G = rg_table()
    out8, _ = rg_restated()
    for i, (x8, c) in enumerate(zip(out8, G.cases)):
        h = resample_reference(x8, 8, 1)
        if 1 <= len(h) <= RV["RV_MAX_RIR"] and i % 3 == 0:
            rirs.append(h)
            labels.append(f"generated: {c[7]}")
    cases = []
    for k, h in enumerate(rirs):
        n = int(rs.randint(len(h) // 2 + 1, 2 * len(h) + 2))
        cases.append(((rs.randn(n) * 0.1).astype(np.float32), k, n, labels[k]))
        imp = np.zeros(len(h), np.float32)
        imp[0] = 1.0
        cases.append((imp, k, len(h), labels[k] + " impulse"))
    return rirs, cases


def test_float_rir_table_reaches_its_edges():
    rirs, cases = rv32_table()
    T = RV["RV_THREADS"]
    firsts = [int(np.argmax(h)) for h in rirs]
    ties = [np.flatnonzero(h == h.max()) for h in rirs]
    many = [t for t in ties if len(t) > 1]
    assert any((t[1] - t[0]) % T == 0 for t in many)                     # one thread's strided steps
    assert any(t[0] // 32 != t[1] // 32 and t[0] % T // 32 != t[1] % T // 32 for t in many)  # two warps
    assert any(t[0] // 32 == t[1] // 32 for t in many)                     # two lanes of a warp
    assert any((h < 0).all() for h in rirs)
    assert any((h == 0).all() and np.signbit(h).any() and not np.signbit(h).all() for h in rirs)
    for R in (RV_B - 1, RV_B + 1, RV["RV_MAX_RIR"]):
        assert any(len(h) == R and f == R - 1 for h, f in zip(rirs, firsts)), R
    tiny = [h for h in rirs if 0 < np.abs(h).max() < 2.0 ** -99]
    assert tiny and any(np.any((h != 0) & (h * np.float32(2.0 ** -27) != h.astype(np.float64) * 2.0 ** -27)) for h in tiny)
    assert sum(c[3].startswith("generated") for c in cases) >= 10


@pytest.mark.gpu
def test_gpu_reverb_float_rirs_bit_equal(rv_harness, tmp_path):
    """normalize = 0: the device's y bit for bit as the host harness computes it (its shift the first maximum, as
    np.argmax); an impulse gives back the RIR from that shift on."""
    import torch

    from lhotse_b200.engine import REVERB_CUT_DTYPE, reverb

    rirs, cases = rv32_table()
    host = test_reverb.run_harness(rv_harness, tmp_path, rirs, [(c[0], c[1], False, c[2]) for c in cases])
    rt, _, s32 = test_reverb.rir_records(rirs)
    dev = torch.device("cuda:0")
    ct = np.zeros(len(cases), REVERB_CUT_DTYPE)
    ct["struct_size"] = REVERB_CUT_DTYPE.itemsize
    ct["rir"] = [c[1] for c in cases]
    ct["in_len"] = [len(c[0]) for c in cases]
    ct["target_len"] = [c[2] for c in cases]
    ct["in_elem"] = np.concatenate(([0], np.cumsum(ct["in_len"] + GAP)[:-1]))
    ct["out_elem"] = np.concatenate(([0], np.cumsum(ct["target_len"] + GAP)[:-1]))
    x = np.full(int(ct["in_elem"][-1] + ct["in_len"][-1] + GAP), SENTINEL, np.int32).view(np.float32)
    for a, c in zip(ct["in_elem"], cases):
        x[a:a + len(c[0])] = c[0]
    out = _filled(int(ct["out_elem"][-1] + ct["target_len"][-1] + GAP), dev)
    rir32 = _filled(len(s32) + GAP, dev)
    rir32[:len(s32)] = torch.from_numpy(s32).to(dev)
    reverb(None, None, torch.from_numpy(x).to(dev), rt, ct, out, rir32=rir32)
    torch.cuda.synchronize()
    buf = out.cpu().numpy()
    windows = list(zip(ct["out_elem"], ct["target_len"]))
    _assert_sentinel_outside(buf, windows, "out")
    for (a, n), c, h in zip(windows, cases, host):
        got = buf[a:a + n]
        assert _bits_equal(got, h), c[3]
        if c[3].endswith("impulse"):
            rir = rirs[c[1]]
            s = int(np.argmax(rir))
            want = rir[s:].astype(np.float64) * 2.0 ** -15
            scale = float(np.abs(rir).max()) * 2.0 ** -15
            if scale > 1e-20:  # the convolution's float32 error is relative to the RIR's largest sample
                assert np.abs(got[:len(want)] - want).max() <= 1e-4 * scale, c[3]
