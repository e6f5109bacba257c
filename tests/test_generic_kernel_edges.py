"""The generic kernel (csrc/generic.cuh) at its edges: every FFT factorization, launch shape and epilogue.

Without a GPU: the edge table names what each row reaches (generic_edge_cases.ROWS); a float64 restatement of the
Stockham passes and the packed-real split equals numpy's rfft for every N of the table; and the shared-memory layout the
header gives (compiled on the host) keeps every write of the kernel inside its own region, for the table and for every N
from 2 to 4096 under all four feature kinds.

On the H100: every row with kernel="generic" in float32 and int16, packed and padded, against the float64 oracles; bits
equal to the same cut alone and to a second run; pad rows and the memory around the output untouched; the creation-time
refusals; more than 65535 cuts, a grid that strides, a multi-chunk host-staged call; and both whisper normalise passes
at the row boundaries, with odd `num_filters` and a NaN sample.
"""
import numpy as np
import pytest
import torch

import generic_edge_cases as G
from test_gpu_kernel_matrix import (CHUNK_ELEMS_F32, PAD, assert_gate, assert_pad, assert_same, dequantise, host_chunks,
                                    kaldi_windows, quantise, run, seed_of, signals, whisper_check)
from test_librosa import librosa_gate
from lhotse_b200.engine import OUT_PACKED, OUT_PADDED, B200FeatError, Engine
from oracle import librosa_oracle as LO
from oracle import whisper_oracle as W

gpu = pytest.mark.gpu
SENTINEL = 0x7FC0FFEE  # a quiet NaN whose payload the kernels never write
EUNSUPPORTED = -2


# ------------------------------------------------------------------------------------------------ CPU: the table
def test_table_names_its_targets():
    """Each row's geometry, packing, radix list, launch shape and epilogue match its plan; every tag it names is reached
    by its plan; together the rows reach every branch in REQUIRED; the refused sizes are the first that do not fit."""
    names, reached = set(), set()
    for r in G.ROWS:
        assert r.name not in names, f"duplicate row {r.name}"
        names.add(r.name)
        p = G.check_row_geometry(r)
        Nc = p.N // 2 if p.N % 2 == 0 else p.N
        assert (r.packed, r.Nc) == (p.N % 2 == 0, Nc), r.name
        assert list(r.radix) == G.factorize(Nc), (r.name, G.factorize(Nc))
        w, smem, fits = G.launch_shape(r.feature, p.N, p.num_filters)
        assert fits and (r.warps, r.smem) == (w, smem), (r.name, w, smem)
        assert r.epilogue == G.epilogue_of(r.feature, r.cfg, p), r.name
        got = G.branches(r)
        assert r.targets <= got, (r.name, sorted(r.targets - got))
        reached |= got
    missing = [t for t in G.REQUIRED if t not in reached]
    assert not missing, f"branches without a row: {missing}"
    for name, feature, cfg, N in G.REFUSED:
        p = G.plan_of(feature, cfg)
        assert p.N == N, name
        assert not G.launch_shape(feature, N, 0)[2], name
    assert G.launch_shape("spectrogram", 16384, 0)[2] and not G.launch_shape("spectrogram", 32768, 0)[2]
    assert G.launch_shape("spectrogram", G.LARGEST_ODD, 0)[2] and not G.launch_shape("spectrogram", G.LARGEST_ODD + 2, 0)[2]


# ------------------------------------------------------------------------------------------------ CPU: the FFT
SMALL_N = list(range(2, 70)) + [96, 100, 121, 125, 128, 243, 256, 343]


@pytest.mark.parametrize("N", sorted({r.N for r in G.ROWS} | set(SMALL_N)))
def test_stockham_restatement_equals_rfft(N):
    """The kernel's passes (radix 4, radix 2, the prime radix's twiddle walk) and its packed-real split, in float64,
    equal numpy's rfft to 1e-12 of the largest line: the index and twiddle arithmetic is right for this N."""
    rs = np.random.RandomState(N)
    for y in (rs.randn(N), np.cos(2 * np.pi * 3.25 * np.arange(N) / N) + 0.5):
        got, want = G.generic_rfft(y), np.fft.rfft(y)
        assert got.shape == want.shape
        err = np.abs(got - want).max() / np.abs(want).max()
        assert err <= 1e-12, (N, err)


# ------------------------------------------------------------------------------------------------ CPU: the layout
@pytest.fixture(scope="module")
def header_layout(tmp_path_factory):
    q = G.layout_harness(tmp_path_factory.mktemp("glc"))
    if q is None:
        pytest.skip("nvcc not found")
    return q


SWEEP_M = {"fbank": (80,), "mfcc": (1, 13, 23, 33, 40, 64, 80, 128, 140, 200, 256), "spectrogram": (0,),
           "log-spectrogram": (0,)}


def _check_layouts(header_layout, plans, L_of):
    got = header_layout(plans)
    bad = []
    for (feature, N, M), h in zip(plans, got):
        want = G.layout(feature, N, M)
        w, smem, fits = G.launch_shape(feature, N, M)
        assert {k: h[k] for k in want} == want, (feature, N, M, h)
        assert (h["warps"], h["smem"], h["fits"]) == (w, smem, fits), (feature, N, M, h)
        assert h["fits"] and h["smem"] == 4 * h["floats"] * h["warps"] <= G.SMEM_OPTIN
        faults = G.region_faults(feature, N, L_of(N), M, h)
        if faults:
            bad.append((feature, N, M, faults))
    assert not bad, bad[:5]


def test_layout_keeps_every_write_in_its_region_table(header_layout):
    """For every row: the header's layout equals its restatement, and every write of a frame stays in its region."""
    plans, Ls = [], {}
    for r in G.ROWS:
        p = G.plan_of(r.feature, r.cfg)
        plans.append((r.feature if r.feature in G.SWEEP_FEATURES else "fbank", p.N, p.num_filters))
        Ls[p.N] = max(Ls.get(p.N, 0), p.L)
    _check_layouts(header_layout, plans, lambda N: Ls[N])


def test_layout_keeps_every_write_in_its_region_sweep(header_layout):
    """Every N from 2 to 4096, both parities, all four Kaldi feature kinds, M up to 256 (L = N: the longest frame)."""
    plans = [(f, N, M) for N in range(2, 4097) for f, Ms in SWEEP_M.items() for M in Ms]
    _check_layouts(header_layout, plans, lambda N: N)


def test_old_layout_overflowed_exactly_the_mfcc_plans():
    """The same write check on the layout from before the MFCC scratch had its own region (log-mels in the FFT buffer
    not holding the result, 2 Nc floats of room) flags exactly the table's M > 2 Nc MFCC rows, so it would have caught
    them."""
    flagged = set()
    for r in G.ROWS:
        p = G.plan_of(r.feature, r.cfg)
        feature = r.feature if r.feature in G.SWEEP_FEATURES else "fbank"
        if G.region_faults(feature, p.N, p.L, p.num_filters, G.head_layout(feature, p.N, p.num_filters)):
            flagged.add(r.name)
    assert flagged == {r.name for r in G.ROWS if "mfcc-M>2Nc" in G.branches(r)}, flagged
    assert flagged == {"mfcc-32-M40-16k", "mfcc-32-M40-8k", "mfcc-64-M80", "mfcc-128-M140"}


# ------------------------------------------------------------------------------------------------ GPU helpers
def make_engine(feature, cfg, kernel="generic"):
    eng = Engine(G.plan_of(feature, cfg), 0, kernel=kernel)
    assert eng.kernel == kernel
    return eng


def librosa_cfg(cfg):
    full = dict(sampling_rate=22050, fft_size=1024, hop_size=256, win_length=None, window="hann", num_mel_bins=80,
                fmin=80, fmax=7600)
    full.update(cfg)
    return full


def assert_oracle(r, x, got):
    kind = G.oracle_kind(r)
    if kind == "kaldi":
        assert_gate(r.feature, r.cfg, x, got)
    elif kind == "librosa":
        c = librosa_cfg(r.cfg)
        truth = LO.extract(x, float64=True, **c)
        assert got.shape == truth.shape
        ok, msg = librosa_gate(got, truth, c)
        assert ok, msg
    else:
        whisper_check(x, got)


def sentinel_buffer(n, margin=64):
    buf = torch.full((n + 2 * margin,), SENTINEL, dtype=torch.int32, device="cuda")
    return buf, buf.view(torch.float32)[margin: margin + n]


def run_into_sentinel(eng, xs, out_mode):
    """extract_device into a sentinel-filled buffer with margins: (rows per cut, pad tails, raw int32 buffer, rows)."""
    lens = [len(x) for x in xs]
    _, tot = eng.plan_batch(lens, out_mode=out_mode)
    buf, out = sentinel_buffer(int(tot.out_floats))
    dt = xs[0].dtype
    offs = np.cumsum([0] + [(n + 7) // 8 * 8 for n in lens[:-1]])
    flat = np.zeros(int(offs[-1]) + lens[-1] + 16, dtype=dt)
    for o, x in zip(offs, xs):
        flat[o: o + len(x)] = x
    res, prefix = eng.extract_device(torch.from_numpy(flat).cuda(), lens, offsets=[int(o) for o in offs],
                                     out_mode=out_mode, pad_value=PAD, out=out)
    torch.cuda.synchronize()
    return buf.cpu().numpy(), prefix, tot


# ------------------------------------------------------------------------------------------------ GPU: every row
@gpu
@pytest.mark.parametrize("r", G.ROWS, ids=G.row_id)
def test_row_vs_oracle(r):
    """float32 and int16, packed and padded: every cut within the gate of its float64 oracle; int16 equal to float32 of
    q / 32768 and padded equal to packed, bit for bit; each cut alone and a second run give the same bits; pad rows are
    pad_value; nothing outside the rows is written; the shortest framable cut runs and one sample fewer is refused."""
    eng = make_engine(r.feature, r.cfg)
    plan = eng.plan
    lens = G.cut_lengths(plan)
    n0 = G.shortest_framable(plan)
    assert n0 in lens and eng.num_frames(n0) >= 1
    with pytest.raises(ValueError):
        eng.num_frames(n0 - 1)
    with pytest.raises(ValueError):
        run(eng, signals(1, [n0 + 5, n0 - 1]))
    xs = signals(seed_of("generic-edges", r.name), lens)
    packed, _ = run(eng, xs)
    for x, g in zip(xs, packed):
        assert_oracle(r, x, g)
    assert_same(run(eng, xs)[0], packed, "second run")
    assert_same([run(eng, [x])[0][0] for x in xs], packed, "each cut alone")
    padded, tails = run(eng, xs, OUT_PADDED)
    assert_same(padded, packed, "padded vs packed")
    assert_pad(tails, np.float32(PAD))
    qs = quantise(xs)
    xq = dequantise(qs)
    fq, _ = run(eng, xq)
    for x, g in zip(xq, fq):
        assert_oracle(r, x, g)
    assert_same(run(eng, qs)[0], fq, "int16 vs float32(q / 32768)")
    i16p, tails = run(eng, qs, OUT_PADDED)
    assert_same(i16p, fq, "int16 padded vs float32 packed")
    assert_pad(tails, np.float32(PAD))
    F = eng.feature_dim
    rows = sum(p.shape[0] for p in packed)
    for data, want in ((xs, packed), (qs, fq)):
        for mode in (OUT_PACKED, OUT_PADDED):
            buf, prefix, tot = run_into_sentinel(eng, data, mode)
            m = 64
            body = buf[m: m + int(tot.out_floats)]
            assert np.all(buf[:m] == SENTINEL) and np.all(buf[m + int(tot.out_floats):] == SENTINEL), "write outside out"
            vals = body.view(np.float32)
            if mode == OUT_PACKED:
                got = vals[: rows * F].reshape(rows, F)
                assert_same([got[prefix[i]: prefix[i + 1]] for i in range(len(data))], want, "into sentinel, packed")
                if r.feature != "whisper-fbank":  # whisper keeps its per-cut maxima in the tail
                    assert np.all(body[rows * F:] == SENTINEL), "write past the packed rows"
            else:
                Tm = int(tot.max_frames)
                got = vals[: len(data) * Tm * F].reshape(len(data), Tm, F)
                Ts = np.diff(prefix)
                assert_same([got[i, :T] for i, T in enumerate(Ts)], want, "into sentinel, padded")
                assert_pad([got[i, T:] for i, T in enumerate(Ts)], np.float32(PAD))


@gpu
@pytest.mark.parametrize("name,feature,cfg,N", G.REFUSED, ids=[x[0] for x in G.REFUSED])
def test_refused_at_creation(name, feature, cfg, N):
    """One warp's region over the opt-in limit: creation fails with B200FEAT_EUNSUPPORTED, under generic and AUTO."""
    for kernel in ("generic", "auto"):
        with pytest.raises(B200FeatError) as e:
            Engine(G.plan_of(feature, cfg), 0, kernel=kernel)
        assert e.value.code == EUNSUPPORTED, (kernel, e.value)


@gpu
def test_largest_odd_size_is_accepted():
    cfg = dict(sampling_rate=G.LARGEST_ODD, frame_length=1.0, frame_shift=0.25, round_to_power_of_two=False)
    eng = make_engine("spectrogram", cfg)
    assert eng.plan.N == G.LARGEST_ODD
    xs = signals(seed_of("largest-odd"), [G.LARGEST_ODD + 3 * eng.plan.S + 7])
    got, _ = run(eng, xs)
    assert_gate("spectrogram", cfg, xs[0], got[0])


# ------------------------------------------------------------------------------------------------ GPU: batches
@gpu
def test_more_than_65535_cuts():
    """65540 short cuts in one call (cuts past 65535 are found by find_segment in packed mode, by the row index in padded
    mode): each cut equals the same cut alone, bit for bit, in both layouts."""
    eng = make_engine("mfcc", dict(num_filters=40, num_ceps=13))
    S = eng.plan.S
    protos = signals(seed_of("65540"), [S + S // 2, 2 * S + 1, 3 * S - 1, 5 * S + 3, 2 * S - 1, 4 * S])
    alone = [run(eng, [x])[0][0] for x in protos]
    for x, g in zip(protos, alone):
        assert_gate("mfcc", dict(num_filters=40, num_ceps=13), x, g)
    B = 65540
    pick = (np.arange(B) * 7919 + 3) % len(protos)
    xs = [protos[i] for i in pick]
    got, _ = run(eng, xs)
    for i in list(range(8)) + list(range(65530, B)):
        assert np.array_equal(got[i], alone[pick[i]]), f"cut {i}"
    cat = np.concatenate(got)
    want = np.concatenate([alone[i] for i in pick])
    assert np.array_equal(cat, want), "packed rows of 65540 cuts"
    padded, tails = run(eng, xs, OUT_PADDED)
    assert_same(padded[65530:], [alone[i] for i in pick[65530:]], "padded, last cuts")
    assert all(np.array_equal(p, alone[i]) for p, i in zip(padded, pick)), "padded rows of 65540 cuts"
    assert_pad(tails, np.float32(PAD))


@gpu
@pytest.mark.parametrize("name", ["n550", "pow2-16384"])
def test_long_cut_strides_the_grid(name):
    """A cut with more frames than the persistent grid has warps: the grid strides, and every frame still matches the
    oracle and the same cut in a batch."""
    r = next(x for x in G.ROWS if x.name == name)
    eng = make_engine(r.feature, r.cfg)
    S = eng.plan.S
    warps_in_grid = torch.cuda.get_device_properties(0).multi_processor_count * 8 * r.warps
    T = warps_in_grid + 300
    xs = signals(seed_of("stride", name), [T * S, eng.plan.L + 3 * S])
    assert eng.num_frames(len(xs[0])) > warps_in_grid
    got, _ = run(eng, xs)
    assert_same([run(eng, [x])[0][0] for x in xs], got, "alone vs batch")
    kaldi_windows(r.feature, r.cfg, xs[0], got[0], S)


@gpu
def test_multi_chunk_host_staging_odd_n():
    """extract_host splits ~20 M samples into >= 3 chunks, so later launches start at a nonzero tile and cut index: every
    cut equals the same cut alone (N = 210: radices 3, 5 and 7)."""
    r = next(x for x in G.ROWS if x.name == "n210")
    eng = make_engine(r.feature, r.cfg)
    L, S = eng.plan.L, eng.plan.S
    rs = np.random.RandomState(seed_of("chunks-generic"))
    lens = []
    for _ in range(8):
        lens += [int(rs.randint(L + S, 4 * S)) | 1, int(rs.randint(2_200_000, 2_600_000))]
    assert host_chunks(lens, 1, CHUNK_ELEMS_F32) >= 3
    xs = [(0.1 * rs.randn(n)).astype(np.float32) for n in lens]
    alone = [run(eng, [x])[0][0] for x in xs]
    launches = eng.stats()["kernel_launches"]
    out, prefix = eng.extract_host(np.concatenate(xs), lens)
    assert eng.stats()["kernel_launches"] - launches >= 3
    assert_same([out[prefix[i]: prefix[i + 1]] for i in range(len(xs))], alone, "extract_host packed")
    for i in (0, 1, len(xs) - 1):
        kaldi_windows(r.feature, r.cfg, xs[i], alone[i], S)


# ------------------------------------------------------------------------------------------------ GPU: whisper normalise
def whisper_lengths(S=160):
    return [k * S + d for k in (3, 10, 57) for d in (-1, 0, S // 2)]


@gpu
@pytest.mark.parametrize("kernel", ["generic", "fast"])
@pytest.mark.parametrize("M", [80, 81])
def test_whisper_normalize_passes(kernel, M):
    """b200feat_whisper_normalize_kernel (generic) and _tiled_kernel (fast400; F = 80 takes its float4 path, F = 81 its
    scalar one): cut lengths that move the boundary between stft rows and the zero row, packed and padded, and a cut
    with one NaN sample next to finite cuts."""
    eng = make_engine("whisper-fbank", dict(num_filters=M), kernel=kernel)
    lens = whisper_lengths()
    xs = signals(seed_of("whisper-norm", M), lens)
    for x, n in zip(xs, lens):
        assert eng.num_frames(n) == W.num_rows(n)
    packed, _ = run(eng, xs)
    for x, g in zip(xs, packed):
        _whisper_check_m(x, g, M)
        T = g.shape[0]
        if len(x) // 160 < T:
            assert np.all(g[-1] == 0.0), "the extra row is not zero"
    padded, tails = run(eng, xs, OUT_PADDED)
    assert_same(padded, packed, "padded vs packed")
    assert_pad(tails, np.float32(PAD))
    nan_xs = [x.copy() for x in xs[:4]]
    nan_xs[1][len(nan_xs[1]) // 3] = np.nan
    for mode in (OUT_PACKED, OUT_PADDED):
        got, _ = run(eng, nan_xs, mode)
        assert_whisper_nan_m(nan_xs[1], got[1], M)
        for i in (0, 2, 3):
            assert np.array_equal(got[i], packed[i]), f"cut {i} next to the NaN cut"


def _whisper_check_m(x, got, M):
    ref, truth = W.extract(x, num_filters=M), W.extract(x, num_filters=M, dtype=torch.float64)
    assert got.shape == ref.shape
    err, noise = np.abs(got - truth).max(), np.abs(ref.astype(np.float64) - truth).max()
    assert err <= max(2e-5, 3.0 * noise), (err, noise)


def assert_whisper_nan_m(x, got, M):
    ref = W.extract(x, num_filters=M)
    assert got.shape == ref.shape
    assert np.array_equal(np.isnan(got), np.isnan(ref)), "NaN positions differ"
    assert np.isnan(ref).any()
    fin = ~np.isnan(ref)
    assert np.array_equal(got[fin], ref[fin])
