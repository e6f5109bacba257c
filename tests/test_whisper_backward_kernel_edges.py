"""The whisper-fbank backward at its edges (csrc/backward.cuh, DESIGN.md §3.1p).

Without a GPU: every derived column of the edge table (stft frames, output rows, the backward's tiles and T mod 16, the
fast400 forward's tiles, the right-mirror reach) recomputed from the plan, the host harness's launch shape and fast400.cuh's
tile, and the table's coverage of the edges.  The restatement and the host harness run at the table's rows in
test_whisper_backward.py.

On the H100: accuracy at every row for both forwards, batched and alone bit for bit; the overlap-add and both centre mirrors
bit for bit from one frame's gradient; the reduction's cut stride, the frames kernel's tile stride at 30 s cuts, the combine
kernel's x and y strides; the saved maxima and the keep_raw features (float32 and int16); a NaN sample's cut beside clean
ones; the work-buffer size.  The accuracy gate is test_gpu_whisper_backward.py's: per cut,
||g - g64|| <= 8 ||g32 - g64|| + 1e-7 ||g64||."""
import re
import subprocess
import zlib

import numpy as np
import pytest
import torch

import whisper_backward_cases as WB
import whisper_backward_edge_cases as E
from oracle import whisper_oracle as W

HOP, N_FFT, PAD = E.HOP, E.N_FFT, E.PAD


def _rs(*key):
    return np.random.RandomState(zlib.crc32(repr(key).encode()))


def _case(n, kind, M, seed=0):
    """WB.case at the first seed from `seed` whose maximum is unique by 1e-3."""
    for s in range(seed, seed + 16):
        try:
            return WB.case(n, kind, M, s)
        except AssertionError:
            continue
    raise AssertionError((n, kind, M))


# ============================================================================= without a GPU
@pytest.fixture(scope="module")
def harness(tmp_path_factory):
    exe = WB.host_check_binary(tmp_path_factory.mktemp("wbwde"))
    if exe is None:
        pytest.skip("no host C++ compiler")
    return exe


def test_table_columns_follow_from_the_plan_and_the_headers(harness, tmp_path):
    """Each row's plan builds at its M and gives R rows; T, the backward's tiles (the header's launch shape, read from the
    host harness), T mod 16, the fast400 forward's tiles of 4 * F400_WARPS * F400_SLOTS rows and the reach are the row's."""
    import lhotse_b200 as lb

    fwd = E.fast400_tile()
    assert fwd == 56 and E.fast400_max_filters() == 264
    shape = {}
    for M in E.MS:
        x = WB.waveform(201, "noise").astype(np.float32).astype(np.float64)
        xr, m = WB.saved_rows(x, M)
        WB.host_check_input(str(tmp_path / "in.bin"), x, xr, m, np.zeros((1, M), np.float32), M)
        res = subprocess.run([harness, str(tmp_path / "in.bin"), str(tmp_path / "out.f32")], capture_output=True, text=True)
        assert res.returncode == 0, res.stderr
        got = re.search(r"tiles of (\d+) frames, (\d+) warps", res.stdout)
        shape[M] = (int(got.group(2)), int(got.group(1)))
    assert set(shape.values()) == {(4, 16)}, shape
    for r in E.TABLE:
        plan = lb.build_plan("whisper-fbank", lb.B200WhisperFbankConfig(num_filters=r.M))
        assert plan.mel_bank.shape == (201, r.M) and plan.feature_dim == r.M
        R = int(plan.num_frames(r.n))
        assert R == W.num_rows(r.n) == (r.n + 80) // 160
        assert (r.T, r.R, r.tiles, r.t16, r.ftiles, r.reach) == E.derived(r.n, R, shape[r.M][1], fwd), r.name
        assert r.M <= E.fast400_max_filters() or r.kernel == "generic", r.name  # past fast400's size rule: generic


def test_table_covers_the_edges():
    rows = E.TABLE
    for t16 in (0, 1, 15):  # each residue of the backward's tile, past the first tile, with and without the zero row
        assert {r.R - r.T for r in rows if r.t16 == t16 and r.T >= 15} == {0, 1}, t16
    assert {r.n % 160 for r in rows} >= {0, 1, 38, 39, 40}
    assert {r.n % 160: r.reach for r in rows if r.n % 160 in (0, 1, 38, 39, 40)} == {0: 40, 1: 39, 38: 2, 39: 1, 40: 0}
    assert {(r.n, r.T, r.R) for r in rows if r.T == 1} == {(201, 1, 1), (319, 1, 2)}
    assert {55, 56, 57} <= {r.R for r in rows} | {r.T for r in rows}
    assert any(r.R == 56 and r.T == 55 for r in rows) and any(r.R == r.T == 56 for r in rows) and any(r.R == 57 for r in rows)
    assert {r.M for r in rows} == set(E.MS) and {r.kernel for r in rows if r.M == 265} == {"generic"}
    assert {r.M for r in rows if r.kernel == "fast"} == {80, 81, 128}
    for M in E.MS:
        assert {r.n for r in rows if r.M == M} >= set(E.SUBSET)
    assert {r.n for r in rows if r.M in (80, 128)} == set(E.LENGTHS)
    assert len({r.name for r in rows}) == len(rows)


def test_fold_of_a_frame_by_hand():
    """expected_fold on a cut of 2560 samples: the first frame's padded positions 1 .. 200 fold onto samples 200 .. 1 (sample
    0 has no image), the last frame's 40 positions past the end onto samples 2558 .. 2519 (sample 2559 has none)."""
    n = 2560
    T = n // HOP
    ext = (T - 1) * HOP + N_FFT
    Wp = np.arange(1, ext + 1, dtype=np.float32)
    got = E.expected_fold(Wp, n)
    assert got[0] == Wp[PAD] and got[n - 1] == Wp[n - 1 + PAD]
    assert got[1] == Wp[1 + PAD] + Wp[PAD - 1] and got[200] == Wp[400] + Wp[0] and got[201] == Wp[401]
    assert got[n - 2] == Wp[n - 2 + PAD] + Wp[n + PAD] and got[n - 41] == Wp[n - 41 + PAD] + Wp[ext - 1]
    assert got[n - 42] == Wp[n - 42 + PAD]


# ============================================================================= on the H100
def _alone(ext, x, G):
    return WB.b200_grads(ext, [x], [G])[0]


@pytest.mark.gpu
def test_table_kernels_on_the_handle():
    """`auto` reaches fast400 at M = 80, 81 and 128 and generic at M = 1, 264 and 265; `generic` is generic at every M."""
    for M in E.MS:
        want = {r.kernel for r in E.TABLE if r.M == M}
        assert len(want) == 1
        assert WB.extractor("auto", M).engine.kernel == want.pop(), M
        assert WB.extractor("generic", M).engine.kernel == "generic", M


@pytest.mark.gpu
@pytest.mark.parametrize("M", E.MS)
@pytest.mark.parametrize("kernel", ["auto", "generic"])
def test_accuracy_at_every_row(kernel, M):
    """Noise and the burst at every length of the table for this M: each cut within the gate alone, then all of them in one
    launch, bit for bit."""
    ext = WB.extractor(kernel, M)
    cuts, worst = [], 0.0
    for r in [r for r in E.TABLE if r.M == M]:
        for kind in ("noise", "burst"):
            x, G = _case(r.n, kind, M)
            g = _alone(ext, x, G)
            err, bound, err32 = WB.gate(x, G, M, g.double().cpu().numpy())
            assert err <= bound, (kernel, r.name, kind, err, bound)
            worst = max(worst, err / max(err32, 1e-300))
            cuts.append((x, G, g))
    batched = WB.b200_grads(ext, [c[0] for c in cuts], [c[1] for c in cuts])
    for (x, _, g), b in zip(cuts, batched):
        assert torch.equal(g, b), (kernel, M, x.shape[0])
    print(f"whisper backward edges {kernel} M={M}: {len(cuts)} cuts, worst ratio to the float32 chain's error {worst:.2f}")


@pytest.mark.gpu
@pytest.mark.parametrize("n", [2560, 7719, 5160, 319], ids=["mod0", "mod39", "mod40", "one-frame"])
def test_overlap_add_and_centre_mirrors_bit_for_bit(n):
    """A hop-periodic waveform and one fixed random row at frame t, zero elsewhere and wherever a saved value is at or below
    its cut's m - 8 (the routed mass is then exactly 0, ties or not): the cut's gradient is that frame's
    gradient Gf at its samples and exactly 0 elsewhere, the same Gf for every interior frame, with the edge frames folded
    onto their sources in bwd_sample's order (own position, left image, right image).  An edge frame's Gf is taken from a
    probe cut whose interior frame 2 holds the edge frame's reflected samples."""
    ext = WB.extractor()
    T = n // HOP
    x = WB.waveform(n, "periodic").astype(np.float32).astype(np.float64)
    idx = WB.frame_index(n)
    interior = [t for t in range(T) if t * HOP - PAD >= 0 and t * HOP - PAD + N_FFT <= n]
    edges = [t for t in range(T) if t not in interior]
    assert edges and (T == 1 or interior)
    nP, tP = max(n, 960), 2
    wP = slice(tP * HOP - PAD, tP * HOP - PAD + N_FFT)
    probes = []
    for t in edges:
        y = WB.waveform(nP, "periodic").astype(np.float32).astype(np.float64)
        y[wP] = x[idx[t]]
        probes.append(y)
    _, saved, m, _ = E.keep_raw(ext, [x] + probes)
    row = E.impulse_row(_rs("oa", "row").randn(80), [saved[0][t] for t in range(T)] + [s[tP] for s in saved[1:]],
                        [m[0]] * T + m[1:])
    assert np.count_nonzero(row) >= 8, np.count_nonzero(row)
    X, Gs = [], []
    for t in range(T):
        G = np.zeros((W.num_rows(n), 80))
        G[t] = row
        X.append(x)
        Gs.append(G)
    for y in probes:
        G = np.zeros((W.num_rows(nP), 80))
        G[tP] = row
        X.append(y)
        Gs.append(G)
    grad = [g.cpu().numpy() for g in WB.b200_grads(ext, X, Gs)]
    gf = {t: grad[T + k][wP] for k, t in enumerate(edges)}
    if interior:
        t_ref = interior[0]
        win = slice(t_ref * HOP - PAD, t_ref * HOP - PAD + N_FFT)
        gf.update({t: grad[t_ref][win] for t in interior})
    assert all(np.abs(v).max() > 0 for v in gf.values())
    ext_len = (T - 1) * HOP + N_FFT
    for t in range(T):
        Wp = np.zeros(ext_len, np.float32)
        Wp[t * HOP: t * HOP + N_FFT] = gf[t]
        want = E.expected_fold(Wp, n)
        assert np.array_equal(grad[t], want), (n, t, t % 16, np.abs(grad[t] - want).max())
    extP = (nP // HOP - 1) * HOP + N_FFT
    for k, t in enumerate(edges):  # each probe's gradient is its Gf alone
        Wp = np.zeros(extP, np.float32)
        Wp[tP * HOP: tP * HOP + N_FFT] = gf[t]
        assert np.array_equal(grad[T + k], E.expected_fold(Wp, nP)), (n, t)
    if E.right_reach(n):  # the right image lands: the last frame's gradient at n - 2 is its own plus its image's
        last = grad[T - 1]
        assert last[n - 2] == np.float32(gf[T - 1][n - 2 - ((T - 1) * HOP - PAD)]) + np.float32(gf[T - 1][n - ((T - 1) * HOP - PAD)])


@pytest.mark.gpu
def test_reduction_kernel_cut_stride():
    """8 * multi_processor_count + 40 burst cuts of 0.1 to 2 s (the reduction's grid is min(B, 8 * SMs)): every cut of the
    second round bit for bit as itself alone, and a few of them against the restatement fed their saved rows and maximum."""
    ext = WB.extractor()
    grid = torch.cuda.get_device_properties(0).multi_processor_count * 8
    B = grid + 40
    rs = _rs("reduce")
    lens = [int(v) for v in rs.randint(1600, 32001, size=B)]
    xs = [WB.waveform(n, "burst", seed=i).astype(np.float32).astype(np.float64) for i, n in enumerate(lens)]
    Gs = [_rs("reduce", i).randn(W.num_rows(n), 80) for i, n in enumerate(lens)]
    batched = WB.b200_grads(ext, xs, Gs)
    for i in range(grid, B):
        assert torch.equal(batched[i], _alone(ext, xs[i], Gs[i])), i
    for i in (grid, grid + 17, B - 1):
        _, saved, m, _ = E.keep_raw(ext, [xs[i]])
        T = lens[i] // HOP
        xr = saved[0][:T].astype(np.float64)
        assert (xr < m[0] - 8.0).any()  # the clamp binds: mass is routed to the maximum
        want = WB.restated_grad(xs[i], Gs[i], 80, xr=xr, m=m[0])
        got = batched[i].double().cpu().numpy()
        assert WB.rel_err(got, want) < 2e-3, (i, WB.rel_err(got, want))


@pytest.mark.gpu
@pytest.mark.parametrize("M", [80, 128])
def test_frames_kernel_tile_stride_at_30_s(M):
    """(B, 480000) cuts, 188 tiles each, more tiles than the frames kernel's grid (64 * multi_processor_count): every cut bit
    for bit as itself alone; the first, a second-round and the last cut within the gate."""
    ext = WB.extractor("auto", M)
    n = 480000
    per_cut = -(-(n // HOP) // 16)
    assert per_cut == 188
    grid = torch.cuda.get_device_properties(0).multi_processor_count * 64
    B = grid // per_cut + 2
    second = -(-grid // per_cut)
    assert B * per_cut > grid and second < B
    gated = sorted({0, second, B - 1})
    xs, Gs = [], []
    for i in range(B):
        kind = ("burst", "noise")[i % 2]
        if i in gated:
            x, G = _case(n, kind, M, seed=i)
        else:
            x = WB.waveform(n, kind, seed=i).astype(np.float32).astype(np.float64)
            G = _rs("30s", M, i).randn(W.num_rows(n), M)
        xs.append(x)
        Gs.append(G)
    batched = WB.b200_grads(ext, xs, Gs)
    for i in range(B):
        assert torch.equal(batched[i], _alone(ext, xs[i], Gs[i])), (M, i)
    worst = 0.0
    for i in gated:
        err, bound, err32 = WB.gate(xs[i], Gs[i], M, batched[i].double().cpu().numpy())
        assert err <= bound, (M, i, err, bound, err / err32)
        worst = max(worst, err / err32)
    print(f"whisper backward 30 s M={M}: B={B}, worst ratio to the float32 chain's error {worst:.2f}")


@pytest.mark.gpu
def test_combine_kernel_strides_in_x():
    """A 70 s cut (more samples than 4096 blocks of 256 threads): within the gate, and an impulse row at a frame past sample
    1,048,576 is the same impulse at an early frame, shifted, bit for bit."""
    ext = WB.extractor()
    n = 70 * 16000
    assert n > 4096 * 256
    x, G = _case(n, "noise", 80)
    err, bound, err32 = WB.gate(x, G, 80, _alone(ext, x, G).double().cpu().numpy())
    assert err <= bound, (err, bound)
    xp = WB.waveform(n, "periodic").astype(np.float32).astype(np.float64)
    early, late = 3, (4096 * 256 + PAD) // HOP + 5
    _, saved, m, _ = E.keep_raw(ext, [xp])
    row = E.impulse_row(_rs("x-stride", "row").randn(80), [saved[0][early], saved[0][late]], m * 2)
    assert np.count_nonzero(row) >= 8
    Gs = []
    for t in (early, late):
        Gt = np.zeros((W.num_rows(n), 80))
        Gt[t] = row
        Gs.append(Gt)
    a, b = (g.cpu() for g in WB.b200_grads(ext, [xp, xp], Gs))
    wa = slice(early * HOP - PAD, early * HOP - PAD + N_FFT)
    wb = slice(late * HOP - PAD, late * HOP - PAD + N_FFT)
    assert late * HOP - PAD > 4096 * 256
    assert torch.equal(a[wa], b[wb]) and a[wa].abs().max() > 0
    a[wa] = 0
    b[wb] = 0
    assert not a.any() and not b.any()


@pytest.mark.gpu
def test_combine_kernel_strides_in_y():
    """65535 + 5 cuts of 201 to 800 samples as one (B, n) batch with lengths (the reduction strides 62 times over too): the
    last 12 cuts get a non-zero gradient, bit for bit what each gets alone, and exactly 0 past their lengths."""
    ext = WB.extractor()
    B, n = 65535 + 5, 800
    rs = _rs("y-stride")
    X = (0.1 * rs.randn(B, n)).astype(np.float32)
    lens = [int(v) for v in rs.randint(201, n + 1, size=B)]
    Gs = [_rs("y-stride", i).randn(W.num_rows(L), 80) if i >= B - 12 else np.ones((W.num_rows(L), 80))
          for i, L in enumerate(lens)]
    Xt = torch.tensor(X, device="cuda", requires_grad=True)
    outs = ext.extract_batch(Xt, 16000, lengths=lens)
    out = torch.cat(list(outs))
    G = torch.as_tensor(np.concatenate(Gs), dtype=torch.float32, device="cuda")
    (out * G).sum().backward()
    g = Xt.grad
    for i in range(B - 12, B):
        assert not g[i, lens[i]:].any(), i
        assert torch.equal(g[i, :lens[i]], _alone(ext, X[i, :lens[i]].astype(np.float64), Gs[i])), i
        assert g[i].abs().max() > 0, i


@pytest.mark.gpu
@pytest.mark.parametrize("M", E.MS)
@pytest.mark.parametrize("kernel", ["auto", "generic"])
def test_saved_maximum_and_keep_raw_features(kernel, M):
    """One batch of every length of the table for this M: each saved maximum is the maximum of the cut's T stft rows and
    one of them; the keep_raw features are torch.equal to the no-grad path's, for float32 and for int16 samples; the int16
    batch's saved rows and maxima are those of its float32 widening q / 32768."""
    ext = WB.extractor(kernel, M)
    ns = [r.n for r in E.TABLE if r.M == M]
    xs = [WB.waveform(n, ("burst", "noise")[i % 2], seed=i) for i, n in enumerate(ns)]
    qs = [np.clip(np.round(x * 8000.0), -32768, 32767).astype(np.int16) for x in xs]
    wide = [q.astype(np.float32) / np.float32(32768.0) for q in qs]
    for cuts, dt in ((xs, torch.float32), (qs, torch.int16)):
        feats, saved, m, prefix = E.keep_raw(ext, cuts, dt)
        assert torch.equal(feats, E.plain(ext, cuts, dt)), (kernel, M, dt)
        for n, xr, mm in zip(ns, saved, m):
            T = n // HOP
            assert mm == xr[:T].max() and (xr[:T] == mm).any(), (kernel, M, n, dt)
        if dt == torch.int16:
            _, saved_w, m_w, _ = E.keep_raw(ext, wide)
            assert m == m_w
            for n, a, b in zip(ns, saved, saved_w):
                assert np.array_equal(a[: n // HOP], b[: n // HOP]), (kernel, M, n)


@pytest.mark.gpu
def test_nan_sample_leaves_its_batch_mates_alone():
    """A NaN sample makes its cut's maximum NaN (atomic_max_float lets NaN win) and its tie count 0; the call completes and
    the cuts beside it get bit for bit their gradients alone."""
    ext = WB.extractor()
    xs = [WB.waveform(n, "noise", seed=i) for i, n in enumerate((16000, 16080, 12345))]
    xs[1] = xs[1].copy()
    xs[1][8000] = np.nan
    Gs = [_rs("nan", i).randn(W.num_rows(x.shape[0]), 80) for i, x in enumerate(xs)]
    g = WB.b200_grads(ext, xs, Gs)
    torch.cuda.synchronize()
    for i in (0, 2):
        assert torch.equal(g[i], _alone(ext, xs[i], Gs[i])) and g[i].abs().max() > 0, i
    _, _, m, _ = E.keep_raw(ext, xs)
    assert np.isnan(m[1]) and np.isfinite(m[0]) and np.isfinite(m[2])
    mid = g[1].cpu().numpy()
    nan = np.flatnonzero(np.isnan(mid))
    print(f"NaN cut: {nan.size} NaN samples ({nan.min() if nan.size else None} .. {nan.max() if nan.size else None}), "
          f"{int((mid == 0).sum())} zeros, {int(np.isfinite(mid).sum() - (mid == 0).sum())} other finite values")


@pytest.mark.gpu
def test_work_buffer_one_byte_short_is_refused():
    """b200feat_backward_work_bytes on a whisper handle is the int64 tables, the reduction's routed mass and tie count per
    cut (each block rounded to 256 bytes), then the tiles' spans; one byte less is refused with EINVAL, the exact size runs."""
    from lhotse_b200 import engine

    ext = WB.extractor()
    eng, lib = ext.engine, ext.engine.lib
    xs = [WB.waveform(n, "noise", seed=i) for i, n in enumerate((16000, 16080, 2721))]
    ns = np.asarray([x.shape[0] for x in xs], dtype=np.int64)
    B = len(xs)
    need = int(lib.b200feat_backward_work_bytes(eng._h, ns.ctypes.data, B))
    r256 = lambda v: (v + 255) // 256 * 256  # noqa: E731
    tiles = sum(-(-(int(n) // HOP) // 16) for n in ns)
    assert need == r256((4 * B + 2) * 8) + r256(8 * B) + tiles * (15 * HOP + N_FFT) * 4, need
    buf, lens, offs = E.pack(xs)
    _, raw, prefix = eng.extract_device_keep_raw(buf, lens, offs)
    R = int(prefix[-1])
    G = torch.as_tensor(_rs("work").randn(R, 80), dtype=torch.float32, device="cuda")
    off = np.asarray(offs, dtype=np.int64)
    rows = np.asarray(prefix, dtype=np.int64)
    work = torch.zeros(need, dtype=torch.uint8, device="cuda")
    out = torch.zeros_like(buf)

    def call(nbytes):
        return lib.b200feat_whisper_backward(eng._h, buf.data_ptr(), engine.DT_F32, ns.ctypes.data, off.ctypes.data, B,
                                             G.data_ptr(), raw.data_ptr(), raw.data_ptr() + 4 * R * 80, rows.ctypes.data,
                                             out.data_ptr(), work.data_ptr(), nbytes, None)

    assert call(need - 1) == -1 and "work buffer too small" in lib.b200feat_last_error(eng._h).decode()
    assert not out.any()
    assert call(need) == 0
    torch.cuda.synchronize()
    want = eng.whisper_backward_device(buf, lens, offs, G, raw, prefix)
    assert torch.equal(out, want) and out.abs().max() > 0
