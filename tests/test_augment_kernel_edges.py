"""The resample, reverb and mix-energy kernels at their edges: hand-built tables that reach the code only the device runs (the
chunk and window caps, both sides of the shared-memory table switch, reflect tails over several CTAs, thousands of ragged
stages or cuts behind one binary search, the reverb's argmax tree and gain loop, the warp's pairwise tree at every depth-5
shape).  The CPU tests hold the tables to the edges they name and the host harnesses to plain NumPy restatements; the GPU
tests require the device to equal both bit for bit (the reverb: y bit for bit, the gain within a derived bound, every sample
within the float64 bound), and every element outside the written windows to keep a sentinel bit pattern."""
import math
import os
import re
from functools import lru_cache

import numpy as np
import pytest

import reverb_cases as RC
import test_mix
import test_reverb
import test_transform
from test_mix import harness as mix_harness  # noqa: F401  (fixtures)
from test_reverb import harness as rv_harness  # noqa: F401
from test_transform import harness as rs_harness  # noqa: F401

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SENTINEL = 0x7FC0FFEE  # a quiet NaN whose payload none of these kernels writes
GAP = 3                # sentinel elements between written windows


def _defines(header):
    with open(os.path.join(ROOT, "lhotse_b200", "csrc", header)) as f:
        return {k: int(v) for k, v in re.findall(r"^#define (\w+) (\d+)\b", f.read(), re.M)}


RS, RV, MX = _defines("resample.cuh"), _defines("reverb.cuh"), _defines("mix.cuh")
RV_B = 1 << (RV["RV_LOG_F"] - 1)
U = 2.0 ** -24  # float32 unit roundoff


def _filled(n, dev):
    import torch

    return torch.full((max(n, 1),), SENTINEL, dtype=torch.int32, device=dev).view(torch.float32)


def _assert_sentinel_outside(buf, windows, what):
    keep = np.ones(buf.shape[0], bool)
    for a, n in windows:
        keep[a:a + n] = False
    bad = np.nonzero(keep & (buf.view(np.int32) != SENTINEL))[0]
    assert bad.size == 0, (what, "stray writes at", bad[:10])


def _bits_equal(a, b):
    return a.shape == b.shape and np.array_equal(a.view(np.int32), b.view(np.int32))


def _src_pos(p, n):  # mix_source_pos
    return np.where(p < n, p, 2 * (n - 1) - p)


# ---- resample ---------------------------------------------------------------------------------------------------------

RS_PAIRS = [(48000, 16000), (17600, 16000),  # small tables in shared memory
            (14800, 16000), (8640, 16000),   # N * K = 2040 and 2050: either side of RS_SMEM_TAB_FLOATS
            (44100, 16000),                  # a global table
            (1200, 1301),                    # chunk = N = 1301 > RS_CHUNK
            (30010, 1000)]                   # O = 3001, K = 3365: the window cap sets chunk = N = 100
RAGGED_PAIRS = [None, (48000, 16000), (17600, 16000), (14800, 16000), (8640, 16000)]
KINDS = ("trim1", "equal", "reflect1", "reflectmax")


def rs_chunk(N, O, K):
    """rs_chunk_outputs: a whole number of blocks, about RS_CHUNK outputs, a window of at most RS_WIN_FLOATS."""
    nb = max(RS["RS_CHUNK"] // N, 1)
    nb = min(nb, (RS["RS_WIN_FLOATS"] - K) // O)
    return max(nb, 1) * N


def _geometry(pair):
    from lhotse_b200.pcm_staging import _resample_geometry

    return _resample_geometry(*pair) if pair else (1, 1, 0, 1)  # (N, O, width, K)


def _out_len(pair, L):
    from lhotse_b200.pcm_staging import resampled_len

    N, O, _, _ = _geometry(pair)
    return resampled_len(N, L, O) if pair else L


def _len_for(pair, want):
    """The shortest input whose stage keeps at least `want` outputs."""
    N, O, _, _ = _geometry(pair)
    L = max(1, want * O // N - 2)
    while _out_len(pair, L) < want:
        L += 1
    return L


def _target(kind, n):
    return {"trim1": n - 1, "equal": n, "reflect1": n + 1, "reflectmax": 2 * n - 1}[kind]


class RsTable:
    """A b200feat_resample stage table over hand-placed inputs, with what each stage must write."""

    def __init__(self):
        self.src = [[], []]
        self.src_len = [0, 0]
        self.chains = []  # ((source, in_elem, input index), steps, target kind)
        self.inputs = []

    def input(self, source, q):
        self.src[source].append(q)
        elem = self.src_len[source]
        self.src_len[source] += len(q)
        self.inputs.append(q)
        return source, elem, len(self.inputs) - 1

    def chain(self, inp, steps, kind):
        self.chains.append((inp, tuple(steps), kind))

    def build(self):
        from lhotse_b200.engine import RESAMPLE_MID, RESAMPLE_STAGE_DTYPE, RESAMPLE_TO_MID, RESAMPLE_TO_OUT
        from lhotse_b200.pcm_staging import resample_reference

        self.pairs = list(dict.fromkeys(p for _, steps, _ in self.chains for _, p, _ in steps if p))
        refs = {}  # (input, steps) -> the chain's stage outputs, in NumPy (resample_reference and float32 scales)
        rows, want = [], []
        mid = out = 0
        self.mid_windows, self.out_windows = [], []
        for ci, ((source, elem, qi), steps, kind) in enumerate(self.chains):
            key = (qi, steps)
            if key not in refs:
                x, ys = self.inputs[qi].astype(np.float32) / np.float32(32768), []
                for s_in, pair, s_out in steps:
                    x = x * np.float32(s_in)
                    if pair:
                        x = resample_reference(x, *pair)
                    x = x * np.float32(s_out)
                    ys.append(x)
                refs[key] = ys
            L = len(self.inputs[qi])
            for d, (s_in, pair, s_out) in enumerate(steps):
                n = _out_len(pair, L)
                last = d == len(steps) - 1
                if last:
                    tl = min(_target(kind, n), 2 * n - 1)  # a single output cannot be reflect-padded
                    at, out = out, out + tl + GAP
                    self.out_windows.append((at, tl))
                    w = RC.length_fix(refs[key][d], tl)
                else:
                    tl = n
                    at, mid = mid, mid + n + GAP
                    self.mid_windows.append((at, n))
                    w = refs[key][d]
                rows.append(((d, ci), (d, self.pairs.index(pair) if pair else -1, source, elem, L,
                                       RESAMPLE_TO_OUT if last else RESAMPLE_TO_MID, at, n, tl, s_in, s_out)))
                want.append(w)
                source, elem, L = RESAMPLE_MID, at, n
        order = sorted(range(len(rows)), key=lambda i: rows[i][0])
        st = np.zeros(len(rows), RESAMPLE_STAGE_DTYPE)
        st["struct_size"] = RESAMPLE_STAGE_DTYPE.itemsize
        for j, i in enumerate(order):
            r = rows[i][1]
            for name, v in zip(("depth", "table", "source", "in_elem", "in_len", "target", "out_elem", "out_len", "target_len",
                                "scale_in", "scale_out"), r):
                st[j][name] = v
        self.stages, self.want = st, [want[i] for i in order]
        self.mid_elems, self.out_elems = mid, out
        self.src0 = np.concatenate(self.src[0]).astype(np.int16)
        self.src1 = np.concatenate(self.src[1]).astype(np.int16)
        return self


@lru_cache(maxsize=1)
def rs_table():
    rs = np.random.RandomState(1)
    T = RsTable()

    def q(n):
        return rs.randint(-32768, 32768, n).astype(np.int16)

    # per pair: 1, < O, < width, K, out_len at chunk - 1, chunk and just past it, and a length whose reflect-padded tail of
    # out_len - 1 spans at least 3 CTAs; each with every length fix.  Pairs round-robin, so depth 0 interleaves shared-table
    # and global-table stages.
    lens = {}
    for pair in RS_PAIRS:
        N, O, width, K = _geometry(pair)
        c = rs_chunk(N, O, K)
        lens[pair] = list(dict.fromkeys([1, max(1, O - 1), width - 1, K] + [_len_for(pair, m) for m in (c - 1, c, c + 1, 3 * c)]))
    scales = [(1.0, 1.0), (0.7, 1.0), (1.0, 1.3)]
    for i in range(max(map(len, lens.values()))):
        for pi, pair in enumerate(RS_PAIRS):
            if i < len(lens[pair]):
                inp = T.input((i + pi) % 2, q(lens[pair][i]))
                for k, kind in enumerate(KINDS):
                    s_in, s_out = scales[(i + k) % 3]
                    T.chain(inp, [(s_in, pair, s_out)], kind)
    # the scale-only stage around its chunk of RS_CHUNK, with a tail of 3 CTAs
    for L in (1, 2, 1023, 1024, 1025, 3075):
        inp = T.input(L % 2, q(L))
        for kind in KINDS:
            T.chain(inp, [(0.7, None, 1.3)], kind)
    # a long input on a cheap pair
    inp = T.input(0, q((1 << 21) + 5))
    for kind in ("equal", "reflectmax"):
        T.chain(inp, [(1.0, (48000, 16000), 1.0)], kind)
    # chains three deep: src -> mid -> mid -> out, with the volume before the first stage and after the last
    T.chain(T.input(0, q(30000)), [(0.7, (17600, 16000), 1.0), (1.0, (48000, 16000), 1.0), (1.0, (14800, 16000), 1.3)], "reflect1")
    T.chain(T.input(1, q(20000)), [(1.0, (44100, 16000), 0.9), (1.1, (8640, 16000), 1.0), (1.0, None, 1.2)], "trim1")
    # about 2000 ragged stages in the same depth, behind the CTA binary search
    for k in range(2000):
        pair = RAGGED_PAIRS[k % len(RAGGED_PAIRS)]
        L = int(rs.randint(1, 4000))
        T.chain(T.input(k % 2, q(L)), [(1.0, pair, 1.0)], KINDS[int(rs.randint(len(KINDS)))])
    return T.build()


def test_resample_table_reaches_its_edges():
    from lhotse_b200.engine import RESAMPLE_MID, RESAMPLE_SRC1, RESAMPLE_TO_OUT

    T = rs_table()
    st = T.stages
    assert (st["target_len"] <= 2 * st["out_len"] - 1).all() and (st["target_len"] >= 0).all()
    last = st["target"] == RESAMPLE_TO_OUT
    for pair in RS_PAIRS + [None]:
        N, O, width, K = _geometry(pair)
        c = rs_chunk(N, O, K)
        mine = st[st["table"] == (T.pairs.index(pair) if pair else -1)]
        first = mine[mine["source"] != RESAMPLE_MID]["in_len"]
        if pair:
            assert {1, K} <= set(first) and (first < O).any() and (first < width).any(), pair
        assert {c - 1, c, c + 1} <= set(np.minimum(mine["target_len"], mine["out_len"])), (pair, c)
        fin = mine[mine["target"] == RESAMPLE_TO_OUT]
        tl, n = fin["target_len"], fin["out_len"]
        for got in (tl == n - 1, tl == n, tl == n + 1, (tl == 2 * n - 1) & (n > 2)):
            assert got.any(), pair
        assert ((tl - n) > 2 * c).any(), pair  # a reflect tail of at least 3 CTAs
    geo = {p: _geometry(p) for p in RS_PAIRS}
    N, O, _, K = geo[(1200, 1301)]
    assert rs_chunk(N, O, K) == N > RS["RS_CHUNK"]
    N, O, _, K = geo[(30010, 1000)]
    assert (RS["RS_WIN_FLOATS"] - K) // O < RS["RS_CHUNK"] // N and rs_chunk(N, O, K) == N
    smem = {p: g[0] * g[3] <= RS["RS_SMEM_TAB_FLOATS"] for p, g in geo.items()}
    assert smem[(14800, 16000)] and not smem[(8640, 16000)] and not smem[(44100, 16000)]
    assert abs(geo[(14800, 16000)][0] * geo[(14800, 16000)][3] - RS["RS_SMEM_TAB_FLOATS"]) < 10
    assert abs(geo[(8640, 16000)][0] * geo[(8640, 16000)][3] - RS["RS_SMEM_TAB_FLOATS"]) < 10
    assert (st["in_len"] >= 1 << 21).any() and (st["target_len"] == 0).any()
    assert (st["source"] == RESAMPLE_SRC1).any() and st["depth"].max() == 2
    deep = [i for i in range(len(T.chains)) if len(T.chains[i][1]) == 3]
    assert any(T.chains[i][1][0][0] != 1.0 and T.chains[i][1][-1][2] != 1.0 for i in deep)
    d0 = st[(st["depth"] == 0) & (st["table"] >= 0)]
    kinds = np.asarray([smem[T.pairs[t]] for t in d0["table"]])
    assert (kinds[1:] != kinds[:-1]).sum() >= 100  # shared and global tables interleaved in one launch
    assert (st["depth"] == 0).sum() >= 2000
    assert last.sum() == len(T.out_windows)


def test_host_resample_edges_bit_equal_to_restatement(rs_harness, tmp_path):
    from lhotse_b200.engine import RESAMPLE_TO_OUT

    T = rs_table()
    out = test_transform.run_stages(rs_harness, tmp_path, T.src0, T.src1, T.pairs, T.stages, T.mid_elems, T.out_elems)
    for i, (r, w) in enumerate(zip(T.stages, T.want)):
        if r["target"] == RESAMPLE_TO_OUT:
            got = out[r["out_elem"]: r["out_elem"] + r["target_len"]]
            assert _bits_equal(got, w), (i, r)


@pytest.mark.gpu
def test_gpu_resample_edges_bit_equal(rs_harness, tmp_path):
    import torch

    from lhotse_b200.engine import RESAMPLE_TO_OUT, resample, resample_table
    from lhotse_b200.pcm_staging import resample_kernel

    T = rs_table()
    dev = torch.device("cuda:0")
    ids = np.asarray([resample_table(a, b, *resample_kernel(a, b), dev) for a, b in T.pairs] + [-1], np.int32)
    st = T.stages.copy()
    st["table"] = ids[T.stages["table"]]  # -1 picks the trailing -1
    mid, out = _filled(T.mid_elems, dev), _filled(T.out_elems, dev)
    resample(torch.from_numpy(T.src0).to(dev), torch.from_numpy(T.src1).to(dev), mid, st, out)
    torch.cuda.synchronize()
    mid, out = mid.cpu().numpy(), out.cpu().numpy()
    host = test_transform.run_stages(rs_harness, tmp_path, T.src0, T.src1, T.pairs, T.stages, T.mid_elems, T.out_elems)
    for i, (r, w) in enumerate(zip(T.stages, T.want)):
        a, n = r["out_elem"], r["target_len"]
        if r["target"] == RESAMPLE_TO_OUT:
            assert _bits_equal(out[a:a + n], w), ("restatement", i, r)
            assert _bits_equal(out[a:a + n], host[a:a + n]), ("harness", i, r)
        else:
            assert _bits_equal(mid[a:a + n], w), ("mid", i, r)
    _assert_sentinel_outside(out, T.out_windows, "out")
    _assert_sentinel_outside(mid, T.mid_windows, "mid")


# ---- mix energies -----------------------------------------------------------------------------------------------------

# 2175 / 2176: the longest tree whose depth-5 level misses a lane (31 present) and the shortest with all 32
MIX_LENS = sorted(set(list(range(1, 18)) + [63, 64, 65, 127, 128, 129, 130, 255, 256, 257, 1023, 1024, 1025, 2047, 2048, 2049,
                                             2175, 2176, 4095, 4096, 4097]
                      + [4096 * 2 ** k + d for k in range(8) for d in (-8, -1, 1, 8)] + [480001, (1 << 22) + 5]))
G_TARGET = 1.93  # g well inside [1, 2): f32(g)'s spacing is 2^-23, about 2^-24 of g, the finest relative spacing there is


def _present_lanes(n):
    """mix_top_node: how many of the 32 lanes hold a subtree at depth MIX_TOP_DEPTH of the pairwise tree of n samples."""
    leaf, depth = MX["MIX_LEAF"], MX["MIX_TOP_DEPTH"]

    def split(m):
        return m // 2 - (m // 2) % 8

    def count(m, k):
        if k == depth or m <= leaf:
            return 1
        n2 = split(m)
        return count(n2, k + 1) + count(m - n2, k + 1)

    return count(n, 0)


def _gain(e_ref, f, e_t):  # mix_gain in Python floats: the same double operations
    return math.sqrt(e_ref * f / e_t) if e_ref > 0 and e_t > 0 else 0.0


@lru_cache(maxsize=1)
def mix_table():
    """Two-track cuts at every length in MIX_LENS: int16 tracks (sources 0 and 1) and float32 tracks (source 2), each in
    MIX_F32 (reference first, the second track scaled) and MIX_SCALED_FIRST mode (the first track scaled against the second).
    The SNR factors put g near G_TARGET."""
    from lhotse_b200.engine import MIX_CUT_DTYPE, MIX_F32, MIX_ROLE_MIXED, MIX_SCALED_FIRST, MIX_SRC_F32, MIX_TRACK_DTYPE

    energy = test_mix._audio_energy()
    rs = np.random.RandomState(3)
    s0, s1, s2, xs = [], [], [], {}
    at = [0, 0, 0]
    for n in MIX_LENS:
        a = np.clip(rs.randn(n) * 4000, -32768, 32767).astype(np.int16)
        b = np.clip(rs.randn(n) * 9000, -32768, 32767).astype(np.int16)
        a[0], b[0] = 1234, -4321  # no silent track: every energy is positive
        c = (rs.randn(n) * 0.05).astype(np.float32)
        d = (rs.randn(n) * 0.3).astype(np.float32)
        xs[n] = {"int16": ((0, at[0]), (1, at[1]), a.astype(np.float32) / np.float32(32768), b.astype(np.float32) / np.float32(32768)),
                 "float32": ((MIX_SRC_F32, at[2]), (MIX_SRC_F32, at[2] + n), c, d)}
        s0.append(a); s1.append(b); s2 += [c, d]
        at[0] += n; at[1] += n; at[2] += 2 * n
    cuts, tracks, want, windows, meta = [], [], [], [], []
    out = 0
    for n in MIX_LENS:
        for src in ("int16", "float32"):
            (sa, ea), (sb, eb), x0, x1 = xs[n][src]
            e0, e1 = energy(x0[None, :]), energy(x1[None, :])
            for mode in (MIX_F32, MIX_SCALED_FIRST):
                jitter = 1 + rs.uniform(-0.003, 0.003)
                if mode == MIX_F32:  # track 1 scaled against track 0
                    f = G_TARGET ** 2 * e1 / e0 * jitter
                    g = _gain(e0, f, e1)
                    m = np.zeros(n, np.float32) + x0
                    w = m + x1 * np.float32(g)
                    snr, ref, e_ref, e_t = (math.nan, f), 0, e0, e1
                else:  # track 0 scaled against track 1: a float64 mix
                    f = G_TARGET ** 2 * e0 / e1 * jitter
                    g = _gain(e1, f, e0)
                    m = np.zeros(n, np.float64) + x0.astype(np.float64) * np.float64(g)
                    w = (m + x1).astype(np.float32)
                    snr, ref, e_ref, e_t = (f, math.nan), 1, e1, e0
                k = len(cuts)
                for (s, e), fac in zip(((sa, ea), (sb, eb)), snr):
                    tracks.append((MIX_TRACK_DTYPE.itemsize, s, e, n, 0, fac, k, MIX_ROLE_MIXED))
                cuts.append((MIX_CUT_DTYPE.itemsize, mode, out, n, n, 2 * k, 2, ref, 0))
                windows.append((out, n))
                want.append(w)
                meta.append((n, src, mode, e_ref, f, e_t))
                out += n + GAP
    return dict(src0=np.concatenate(s0), src1=np.concatenate(s1), src2=np.concatenate(s2),
                tracks=np.asarray(tracks, MIX_TRACK_DTYPE), cuts=np.asarray(cuts, MIX_CUT_DTYPE), out_elems=out,
                want=want, windows=windows, meta=meta)


def test_mix_lengths_reach_every_warp_tree_shape():
    present = {n: _present_lanes(n) for n in MIX_LENS}
    lanes = 1 << MX["MIX_TOP_DEPTH"]
    assert present[1] == present[MX["MIX_LEAF"]] == 1  # a single leaf: lane 0 alone
    assert present[2175] == lanes - 1 and present[2176] == lanes
    assert sum(1 < p < lanes for p in present.values()) >= 8  # depth-5 levels with absent lanes
    assert sum(p == lanes for p in present.values()) >= 30
    # f32(g) sees the energies: one float32 ulp on either energy moves it for most lengths (g sits where float32 is finest)
    T = mix_table()
    moved = total = 0
    for n, src, mode, e_ref, f, e_t in T["meta"]:
        if mode != 0:
            continue
        g32 = np.float32(_gain(e_ref, f, e_t))
        for which in (0, 1):
            e = np.float32((e_ref, e_t)[which])
            hit = False
            for d in (np.inf, -np.inf):
                ep = float(np.nextafter(e, np.float32(d)))
                g = _gain(ep, f, e_t) if which == 0 else _gain(e_ref, f, ep)
                hit |= np.float32(g) != g32
            moved += hit
            total += 1
    assert moved >= 0.9 * total, (moved, total)


def test_host_mix_energy_edges_bit_equal_to_numpy(mix_harness, tmp_path):
    T = mix_table()
    out = test_mix.run_mix(mix_harness, tmp_path, T["src0"], T["src1"], T["tracks"], T["cuts"], T["out_elems"], T["src2"])
    for (a, n), w, m in zip(T["windows"], T["want"], T["meta"]):
        assert _bits_equal(out[a:a + n], w), m[:3]


@pytest.mark.gpu
def test_gpu_mix_energy_edges_bit_equal(mix_harness, tmp_path):
    import torch

    from lhotse_b200.engine import mix

    T = mix_table()
    dev = torch.device("cuda:0")
    out = _filled(T["out_elems"], dev)
    mix(torch.from_numpy(T["src0"]).to(dev), torch.from_numpy(T["src1"]).to(dev), T["tracks"], T["cuts"], out,
        src2=torch.from_numpy(T["src2"]).to(dev))
    torch.cuda.synchronize()
    out = out.cpu().numpy()
    host = test_mix.run_mix(mix_harness, tmp_path, T["src0"], T["src1"], T["tracks"], T["cuts"], T["out_elems"], T["src2"])
    for (a, n), w, m in zip(T["windows"], T["want"], T["meta"]):
        assert _bits_equal(out[a:a + n], w), ("numpy", m[:3])
        assert _bits_equal(out[a:a + n], host[a:a + n]), ("harness", m[:3])
    _assert_sentinel_outside(out, T["windows"], "out")


# ---- reverb -----------------------------------------------------------------------------------------------------------


def _tie_rir(peaks, seed, n=1500):
    q = np.random.RandomState(seed).randint(-3000, 3000, n).astype(np.int16)
    q[list(peaks)] = 32767
    return q


@lru_cache(maxsize=1)
def rv_table():
    """(rirs, edge cases, ragged cases); a case is (x, rir index, target_len, label)."""
    rs = np.random.RandomState(11)
    rirs, edge = [], []

    def rir(q):
        rirs.append(np.asarray(q, np.int16))
        return len(rirs) - 1

    def x(n):
        return (rs.randn(n) * 0.1).astype(np.float32)

    for k, (R, N, peak, _) in enumerate(test_reverb._cases()):
        edge.append((x(N), rir(RC.decaying_rir(R, seed=k, peak_at=peak)), N, f"R={R} N={N} peak={peak}"))
    short1, short2 = rir(RC.decaying_rir(800, seed=100)), rir(RC.decaying_rir(RV_B + 900, seed=101))  # 1 and 2 partitions
    for k in (1, 2, 3):
        for d in (-1, 0, 1):
            N = 2 * RV_B * k + d
            edge.append((x(N), (short1, short2)[d % 2], N, f"N=2Bk{d:+d}"))
    # more than RV_GAIN_THREADS conv CTAs: gain threads sum several partials
    edge.append((x(600001), short2, 600001, "N=600001"))
    edge.append((x((1 << 20) + 1), short1, (1 << 20) + 1, "N=2^20+1"))
    edge.append((x(10000), rir(-rs.randint(1, 30000, 2500)), 10000, "all-negative RIR"))
    edge.append((x(5000), rir(np.zeros(1000)), 5000, "all-zero RIR"))
    edge.append((x(20000), rir(RC.decaying_rir(RV["RV_MAX_RIR"], seed=102, peak_at=RV["RV_MAX_RIR"] - 1)), 20000,
                 "32767 at the last of 65536"))
    # equal maxima: lanes of one warp (the later one in a lower lane too), warps (the earlier one in a later warp too), and
    # strided steps of one thread; the first index wins
    T = RV["RV_THREADS"]
    for k, peaks in enumerate(([5, 9], [20, T + 3], [40, 300], [200, T + 88], [7, T + 7, 2 * T + 7], [31, 32], [480, 481, 1000])):
        edge.append((x(3000), rir(_tie_rir(peaks, seed=300 + k)), 3000, f"tie {peaks}"))
    # length fixes
    x50 = x(50000)
    for t in (49999, 1, 50001, 99999, 0):
        edge.append((x50, short1, t, f"target {t} of 50000"))
    edge.append((x(3000), short2, 5999, "target 5999 of 3000"))
    # a ragged batch: 3000 cuts over 40 RIRs of 1 .. 10 partitions
    pool = [rir(RC.decaying_rir(int(rs.randint(1, 10 * RV_B)), seed=400 + k)) for k in range(40)]
    ragged = []
    for k in range(3000):
        N = int(rs.randint(1, 6000))
        t = N if rs.rand() < 0.7 else int(rs.randint(0, 2 * N))
        ragged.append((x(N), pool[int(rs.randint(40))], t, f"ragged {k}"))
    return rirs, edge, ragged


def test_reverb_table_reaches_its_edges():
    rirs, edge, ragged = rv_table()
    lens = [len(c[0]) for c in edge]
    assert max(lens) > 2 * RV_B * 128 and (1 << 20) + 1 in lens
    for k in (1, 2, 3):
        assert {2 * RV_B * k - 1, 2 * RV_B * k, 2 * RV_B * k + 1} <= set(lens)
    assert any((q < 0).all() for q in rirs) and any((q == 0).all() for q in rirs)
    assert any(len(q) == RV["RV_MAX_RIR"] and int(np.argmax(q)) == len(q) - 1 for q in rirs)
    targets = [(len(c[0]), c[2]) for c in edge + ragged]
    assert any(t == 0 for _, t in targets) and any(t == 2 * n - 1 for n, t in targets) and any(t < n for n, t in targets)
    parts = {(len(rirs[c[1]]) + RV_B - 1) // RV_B for c in ragged}
    assert len(ragged) >= 3000 and len({c[1] for c in ragged}) == 40 and len(parts) >= 8


def _run_reverb(rirs, cases, normalize, shared):
    """The device: every case with `normalize`, inputs and outputs in separate buffers or in one; returns the outputs, the
    whole output buffer and its written windows."""
    import torch

    from lhotse_b200.engine import REVERB_CUT_DTYPE, REVERB_RIR_DTYPE, reverb

    dev = torch.device("cuda:0")
    rt = np.zeros(len(rirs), REVERB_RIR_DTYPE)
    rt["struct_size"] = REVERB_RIR_DTYPE.itemsize
    rt["num_samples"] = [len(q) for q in rirs]
    rt["src_elem"] = np.concatenate(([0], np.cumsum([len(q) for q in rirs])[:-1]))
    ct = np.zeros(len(cases), REVERB_CUT_DTYPE)
    ct["struct_size"] = REVERB_CUT_DTYPE.itemsize
    ct["rir"] = [c[1] for c in cases]
    ct["normalize"] = normalize
    ct["in_len"] = [len(c[0]) for c in cases]
    ct["target_len"] = [c[2] for c in cases]
    ct["in_elem"] = np.concatenate(([0], np.cumsum(ct["in_len"] + GAP)[:-1]))
    in_elems = int(ct["in_elem"][-1] + ct["in_len"][-1] + GAP)
    ct["out_elem"] = np.concatenate(([0], np.cumsum(ct["target_len"] + GAP)[:-1])) + (in_elems if shared else 0)
    out_elems = int(ct["out_elem"][-1] + ct["target_len"][-1] + GAP)
    host_in = np.full(in_elems, SENTINEL, np.int32).view(np.float32)
    for (a, n), c in zip(zip(ct["in_elem"], ct["in_len"]), cases):
        host_in[a:a + n] = c[0]
    src0 = torch.from_numpy(np.concatenate(rirs)).to(dev)
    out = _filled(out_elems, dev)
    if shared:
        out[:in_elems] = torch.from_numpy(host_in).to(dev)
        x = out
    else:
        x = torch.from_numpy(host_in).to(dev)
    reverb(src0, None, x, rt, ct, out)
    torch.cuda.synchronize()
    buf = out.cpu().numpy()
    if shared:  # the inputs are left as they were
        assert _bits_equal(buf[:in_elems], host_in)
        buf = buf.copy()
        buf[:in_elems] = np.int32(SENTINEL).view(np.float32)
    windows = list(zip(ct["out_elem"], ct["target_len"]))
    return [buf[a:a + n] for a, n in windows], buf, windows


def _pairwise_roundings(n):
    """The most roundings on any term's path through NumPy's float32 pairwise sum of n terms (mix.cuh's tree)."""
    leaf = MX["MIX_LEAF"]

    @lru_cache(maxsize=None)
    def h(m):
        if m < 8:
            return max(m - 1, 0)
        if m <= leaf:  # 8 accumulators of m // 8 terms, a 3-level combine, then the tail one by one
            return m // 8 - 1 + 3 + m % 8
        n2 = m // 2 - (m // 2) % 8
        return 1 + max(h(n2), h(m - n2))

    return h(n)


def gain_bound(n):
    """|g - g64| / g64 for g = f32(sqrt(f32(pb / pa))) and g64 = sqrt(sum x^2 / sum y^2) in float64 over the same float32 x, y.
    With u = 2^-24 and nonnegative terms, a sum whose every term passes at most h roundings is within gamma_h = h u / (1 - h u)
    of its exact value:
      pb  f32(x^2) (1), NumPy's pairwise sum (_pairwise_roundings), / n (1);
      pa  per CTA: one thread's FMA chain over its 2 * RV_B / RV_THREADS squares (that many roundings: fma(v, v, 0) rounds
          too), the 5-level shuffle tree, the sequential pass over the other RV_THREADS / 32 - 1 warps; the float64 sum of
          the partials (at most `ctas` roundings of 2^-53); its float32 rounding (1), / n (1);
      g   the quotient (1), which the square root halves with the two sums, and the square root's own rounding (1)."""
    ctas = (n + 2 * RV_B - 1) // (2 * RV_B)
    h_b = 1 + _pairwise_roundings(n) + 1
    h_a = 2 * RV_B // RV["RV_THREADS"] + 5 + (RV["RV_THREADS"] // 32 - 1)

    def gamma(h):
        return h * U / (1 - h * U)

    e_b = gamma(h_b)
    e_a = (1 + gamma(h_a)) * (1 + ctas * 2.0 ** -53) * (1 + U) ** 2 - 1
    hi = math.sqrt((1 + e_b) * (1 + U) / (1 - e_a)) * (1 + U) - 1
    lo = 1 - math.sqrt((1 - e_b) * (1 - U) / (1 + e_a)) * (1 - U)
    return max(hi, lo)


def _check_gain(x, y, target, got, what):
    """The device gain from the outputs: exactly one float32 g (normally) reproduces every output as f32(y[src(p)] * g),
    within gain_bound of the float64 gain."""
    n = len(x)
    ys = y[_src_pos(np.arange(target), n)]
    sy = float(np.sum(y.astype(np.float64) ** 2))
    if sy == 0.0:  # pa = 0: no gain
        assert _bits_equal(got, ys), what
        return
    if target == 0:
        return
    i = int(np.argmax(np.abs(ys)))
    g0 = np.float32(got[i] / ys[i])
    cands = [g0, np.nextafter(g0, np.float32(np.inf)), np.nextafter(g0, np.float32(-np.inf))]
    ok = [g for g in cands if _bits_equal((ys * g).astype(np.float32), got)]
    assert ok and (len(ok) == 1 or target < 100), (what, ok)
    g64 = math.sqrt(float(np.sum(x.astype(np.float64) ** 2)) / sy)
    for g in ok:
        assert abs(float(g) - g64) <= gain_bound(n) * g64, (what, float(g), g64, abs(float(g) - g64) / g64, gain_bound(n))


@pytest.mark.gpu
def test_gpu_reverb_edges(rv_harness, tmp_path):
    """normalize = 0: y bit for bit as the harness computes it; normalize = 1: the gain within gain_bound; both within the
    float64 bound (the harness output standing in for lhotse's float32 reference)."""
    rirs, edge, ragged = rv_table()
    for cases, shared in ((edge, False), (ragged, True)):
        # the harness: y over the whole cut (normalize 0, no length fix), and each case with normalize 1 as it is
        full = [(c[0], c[1], False, len(c[0])) for c in cases]
        norm = [(c[0], c[1], True, c[2]) for c in cases]
        host = test_reverb.run_harness(rv_harness, tmp_path, rirs, full + norm)
        ys, h1 = host[:len(cases)], host[len(cases):]
        for normalize in (0, 1):
            got, buf, windows = _run_reverb(rirs, cases, normalize, shared)
            _assert_sentinel_outside(buf, windows, f"normalize={normalize}")
            for c, y, g, r1 in zip(cases, ys, got, h1):
                x, ri, target, what = c
                what = f"{what} normalize={normalize}"
                want = y[_src_pos(np.arange(target), len(x))]
                if normalize == 0:
                    assert _bits_equal(g, want), what
                    ref32 = want
                else:
                    _check_gain(x, y, target, g, what)
                    ref32 = r1
                RC.check(g, RC.truth64(x, rirs[ri], bool(normalize), target), ref32, what)
