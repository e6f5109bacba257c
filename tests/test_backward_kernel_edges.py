"""The backward of the Kaldi-family extractors at its edges (csrc/backward.cuh, DESIGN.md §3.1n).

Without a GPU: the launch shape of every row of the geometry table, read from the header's own `bwd_launch_shape` through
the host harness, and the frames it refuses; the float64 twin of the torchaudio and HTK conventions against torchaudio,
the restatement against the twin and the host harness (under AddressSanitizer) against the restatement, on a waveform where
the floors bind in part.

On the H100: accuracy at every launch shape and tile count, batched and alone bit for bit; the overlap-add and the mirror
fold bit for bit from one frame's gradient; the frame kernel's grid stride, the combine kernel's x and y strides; the
torchaudio and HTK conventions; the refused frames; an unaligned view and a list of mixed devices and dtypes.  The accuracy
gate is test_gpu_backward.py's: per cut, ||g - g64|| <= 8 ||g32 - g64|| + 1e-7 ||g64||."""
import re
import subprocess
import zlib

import numpy as np
import pytest
import torch

import backward_cases as BC
import backward_edge_cases as E

SR = E.SR


def _rs(*key):
    return np.random.RandomState(zlib.crc32(repr(key).encode()))


# ============================================================================= without a GPU
@pytest.fixture(scope="module")
def harness(tmp_path_factory):
    exe = BC.host_check_binary(tmp_path_factory.mktemp("bwde"))
    if exe is None:
        pytest.skip("no host C++ compiler")
    return exe


def _run_harness(harness, tmp_path, plan, x, G):
    inp, out = str(tmp_path / "in.bin"), str(tmp_path / "out.f32")
    BC.host_check_input(inp, plan, x, G)
    res = subprocess.run([harness, inp, out], capture_output=True, text=True)
    return res, out


@pytest.mark.parametrize("s", E.SHAPES, ids=[s.name for s in E.SHAPES])
def test_launch_shape_table_matches_the_header(s, harness, tmp_path):
    """Each row's plan builds for the forward, and the header's bwd_launch_shape gives the row's (warps, frames per tile), or
    refuses the frame; an accepted row's one-frame gradient on the host also matches the restatement."""
    plan = E.plan_of(s.feature, **E.shape_kw(s, snip_edges=True))
    assert plan.N == 1 << (plan.L - 1).bit_length() and plan.L == int(s.frame_length * SR)
    n = E.length_for(plan, 1)
    assert plan.num_frames(n) == 1
    x = E.waveform(n, "noise")
    G = _rs(s.name).randn(1, plan.feature_dim)
    res, out = _run_harness(harness, tmp_path, plan, x, G.astype(np.float32))
    if s.warps is None:
        assert res.returncode == 3 and "frame too long" in res.stdout, (res.returncode, res.stdout, res.stderr)
        m = re.search(r"(\d+) bytes of shared memory for one warp and one frame, limit (\d+)", res.stdout)
        assert int(m.group(1)) > int(m.group(2)) == 200 * 1024
        return
    assert res.returncode == 0, res.stderr
    m = re.search(r"tiles of (\d+) frames, (\d+) warps", res.stdout)
    assert (int(m.group(2)), int(m.group(1))) == (s.warps, s.ft), res.stdout
    got = np.fromfile(out, dtype=np.float32)
    want = BC.restated_grad_plan(x, plan, G.astype(np.float32).astype(np.float64))
    assert BC.rel_err(got, want) < 2e-4, BC.rel_err(got, want)


def test_the_table_covers_every_launch_shape():
    """One row per shape the header can choose at these N, and both kinds of refused frame."""
    assert [(s.warps, s.ft) for s in E.ACCEPTED] == [(4, 16), (4, 16), (4, 8), (4, 4), (2, 2), (1, 1)]
    assert {E.plan_of(s.feature, **E.shape_kw(s)).N for s in E.REFUSED} == {8192, 16384}


@pytest.mark.parametrize("s", E.ACCEPTED, ids=[s.name for s in E.ACCEPTED])
def test_lengths_give_their_frame_counts(s):
    for snip in (False, True):
        plan = E.plan_of(s.feature, **E.shape_kw(s, snip_edges=snip))
        counts = E.tile_counts(s.ft, 5 * s.ft + s.ft // 2 + 1)
        got = {T: E.length_for(plan, T) for T in counts}
        for T, n in got.items():
            if n is not None:
                assert plan.num_frames(n) == T and BC.O.frame_index_matrix(n, plan.L, plan.S, snip).shape[0] == T
        # snip_edges takes every count; reflect padding refuses the counts whose cut is shorter than the padding
        assert all((n is not None) == (snip or (T * plan.S + plan.S // 2 + plan.L) // 2 > plan.L) for T, n in got.items()) \
            if snip else True


def test_floors_waveform_binds_each_floor_in_part():
    """On one cut: frames where a floor binds everywhere, nowhere, and (mel, log-spectrogram) on some bins only."""
    x = E.waveform(16000, "floors")
    for feature, kw in (("fbank", {"use_energy": True}), ("log-spectrogram", {"use_energy": True})):
        plan = E.plan_of(feature, **E.compat_kw(kw))
        mel, spec, e = E.floor_values(x, plan)
        v, fl = (mel, plan.mel_floor) if mel is not None else (spec, -plan.log_spec_eps)
        below = (v < fl).mean(1)
        assert (below == 0).any() and (below == 1).any() and ((below > 0.05) & (below < 0.95)).sum() >= 3, below
        assert (e < BC.EPS32).any() and (e > 1.0).any() and ((e > BC.EPS32) & (e < 1.0)).any()


def test_plan_twin_is_the_oracle_chain_for_lhotse_configs():
    """The plan-driven twin with the oracle's float64 tables is the oracle's chain (forward and gradient)."""
    for name, cfg in BC.configs():
        n = 4001 if cfg.snip_edges else 3999
        x = BC.waveform(n)
        plan = BC.oracle_plan(cfg)
        a = torch.tensor(x)
        want = BC.features_t(a, cfg)
        got = BC.plan_features_t(a, plan)
        assert torch.allclose(got, want, rtol=1e-12, atol=1e-12), name
        G = np.random.RandomState(0).randn(*want.shape)
        assert BC.rel_err(BC.plan_autograd_grad(x, plan, G), BC.autograd_grad(x, cfg, G)) < 1e-12, name


COMPAT = E.COMPAT


def _compat_cut(name, kind, n=8000):
    return E.waveform(n, kind, seed=len(name))


@pytest.mark.parametrize("name,feature,kw", COMPAT, ids=[c[0] for c in COMPAT])
def test_compat_twin_matches_torchaudio(name, feature, kw):
    pytest.importorskip("torchaudio.compliance.kaldi")
    plan = E.plan_of(feature, **E.compat_kw(kw))
    for kind in ("noise", "floors"):
        x = _compat_cut(name, kind)
        xt = torch.tensor(x, requires_grad=True)
        ref = E.torchaudio_features(xt, feature, kw)
        tplan = E.with_torchaudio_tables(plan, kw)
        got = BC.plan_features_t(torch.tensor(x), tplan).detach()
        assert ref.shape == got.shape
        assert torch.allclose(got, ref.detach(), rtol=1e-10, atol=1e-10), (kind, float((got - ref.detach()).abs().max()))
        G = E.floor_conditioned(x, plan, _rs(name, kind).randn(*ref.shape))
        (ref * torch.as_tensor(G)).sum().backward()
        err = BC.rel_err(BC.plan_autograd_grad(x, tplan, G), xt.grad.numpy())
        assert err < 1e-10, (kind, err)


@pytest.mark.parametrize("name,feature,kw", COMPAT, ids=[c[0] for c in COMPAT])
def test_compat_restatement_and_host_harness(name, feature, kw, harness, tmp_path):
    """The compat-aware restatement against float64 autograd through the twin; the header's code on the host (the plan's
    energy style, energy column, mel shift and log-spectrogram floor in its header) against the restatement."""
    plan = E.plan_of(feature, **E.compat_kw(kw))
    for kind in ("noise", "floors"):
        x = _compat_cut(name, kind)
        T = plan.num_frames(x.shape[0])
        G = E.floor_conditioned(x, plan, _rs(name, kind).randn(T, plan.feature_dim))
        want = BC.plan_autograd_grad(x, plan, G)
        got = BC.restated_grad_plan(x, plan, G)
        assert BC.rel_err(got, want) < 1e-10, (kind, BC.rel_err(got, want))
        G32 = G.astype(np.float32)
        res, out = _run_harness(harness, tmp_path, plan, x, G32)
        assert res.returncode == 0, res.stderr
        h = np.fromfile(out, dtype=np.float32)
        err = BC.rel_err(h, BC.restated_grad_plan(x, plan, G32.astype(np.float64)))
        assert err < 2e-4, (kind, err)


# ============================================================================= on the H100
def _gate(x, plan, G, g):
    g64 = BC.plan_autograd_grad(x, plan, G)
    g32 = BC.plan_autograd_grad(x, plan, G, dtype=torch.float32, device="cuda")
    bound = 8 * np.linalg.norm(g32 - g64) + 1e-7 * np.linalg.norm(g64)
    return float(np.linalg.norm(g - g64)), float(bound)


def _G(x, plan, *key):
    T = plan.num_frames(x.shape[0])
    return E.floor_conditioned(x, plan, _rs(*key).randn(T, plan.feature_dim))


def _alone(ext, x, G):
    return E.b200_grads(ext, [x], [G])[0]


@pytest.mark.gpu
@pytest.mark.parametrize("s", E.ACCEPTED, ids=[s.name for s in E.ACCEPTED])
def test_accuracy_at_every_launch_shape_and_tile_count(s):
    """T = 1, ft +- 1, ft, 2 ft +- 1, 2 ft and a partial last tile, in both framings where the framing takes the length (the
    longest also on the floors waveform): each cut within the gate, then all of them in one launch, bit for bit."""
    long_T = 5 * s.ft + s.ft // 2 + 1 if s.ft > 1 else 23  # N = 8192 with reflect padding takes T >= 20 only
    ran = 0
    for snip in (False, True):
        ext = E.extractor(s.feature, **E.shape_kw(s, snip_edges=snip))
        plan = ext.plan
        cuts = []
        for T in E.tile_counts(s.ft, long_T):
            n = E.length_for(plan, T)
            if n is None:
                continue
            for kind in ("noise", "floors") if T == long_T else ("noise",):
                x = E.waveform(n, kind, seed=T)
                G = _G(x, plan, s.name, snip, T, kind)
                g = _alone(ext, x, G)
                err, bound = _gate(x, plan, G, g.double().cpu().numpy())
                assert err <= bound, (s.name, snip, T, n, kind, err, bound)
                cuts.append((x, G, g))
                ran += 1
        assert cuts, (s.name, snip)
        batched = E.b200_grads(ext, [c[0] for c in cuts], [c[1] for c in cuts])
        for (x, _, g), b in zip(cuts, batched):
            assert torch.equal(g, b), (s.name, snip, x.shape[0])
    assert ran >= len(E.tile_counts(s.ft, long_T)) + 1  # every count with snip_edges, and the long cut twice


def _expected_impulse(W, n, pad, snip):
    """bwd_sample's per-sample sum, in float32 and in its order, of the padded-position gradient W: own position, then the
    left mirror image, then the right one."""
    ext = W.shape[0]
    i = np.arange(n)
    acc = np.zeros(n, np.float32)
    own = i + pad < ext
    acc[own] = acc[own] + W[(i + pad)[own]]
    if not snip:
        left = i < pad
        acc[left] = acc[left] + W[(pad - 1 - i)[left]]
        qr = 2 * n - 1 - i + pad
        right = qr < ext
        acc[right] = acc[right] + W[qr[right]]
    return acc


OA = [s for s in E.ACCEPTED if s.ft in (16, 8, 1) and s.feature != "mfcc"]


@pytest.mark.gpu
@pytest.mark.parametrize("snip", [False, True], ids=["reflect", "snip"])
@pytest.mark.parametrize("s", OA, ids=[s.name for s in OA])
def test_overlap_add_and_mirror_fold_bit_for_bit(s, snip):
    """A waveform periodic with the hop and a row gradient that is one fixed random row at frame t and zero elsewhere: the
    cut's gradient is that frame's gradient Gf at its samples and exactly 0 elsewhere, the same Gf for every interior frame
    (every position in a tile, the first, middle and partial last tile), with edge frames folded onto their sources in
    bwd_sample's order (their Gf taken from a second cut whose interior frame holds the same reflected samples).  The sum of
    the impulse gradients is the full gradient to float32 round-off; with snip_edges the samples past the last frame are 0."""
    ext = E.extractor(s.feature, **E.shape_kw(s, snip_edges=snip))
    plan = ext.plan
    L, S, ft = plan.L, plan.S, s.ft
    pad = 0 if snip else (L - S) // 2
    m0 = -(-pad // S)  # first frame that needs no reflection
    T = max(3 * ft + max(ft // 2, 1), 2 * m0 + 2 * ft + 2)
    n = E.length_for(plan, T) if not snip else (T - 1) * S + L + S - 1
    assert plan.num_frames(n) == T
    x = E.periodic_waveform(n, S)
    idx = BC.O.frame_index_matrix(n, L, S, snip)
    interior = [t for t in range(T) if t * S - pad >= 0 and t * S - pad + L <= n]
    edges = [t for t in range(T) if t not in interior]
    t_probe = interior[0]
    row = _rs(s.name, "row").randn(plan.feature_dim)
    # one launch: an impulse cut for every frame, then a probe cut per edge frame (its reflected samples at frame t_probe)
    X, Gs = [], []
    for t in range(T):
        G = np.zeros((T, plan.feature_dim))
        G[t] = row
        X.append(x)
        Gs.append(G)
    for t in edges:
        y = x.copy()
        y[t_probe * S - pad: t_probe * S - pad + L] = x[idx[t]]
        G = np.zeros((T, plan.feature_dim))
        G[t_probe] = row
        X.append(y)
        Gs.append(G)
    grad = E.b200_rows_grad(ext, np.stack(X), Gs).cpu().numpy()
    win = slice(t_probe * S - pad, t_probe * S - pad + L)
    gf = {t: grad[t_probe][win] for t in interior}
    gf.update({t: grad[T + k][win] for k, t in enumerate(edges)})
    assert np.abs(gf[t_probe]).max() > 0
    ext_len = (T - 1) * S + L
    for t in range(T):
        W = np.zeros(ext_len, np.float32)
        W[t * S: t * S + L] = gf[t]
        want = _expected_impulse(W, n, pad, snip)
        assert np.array_equal(grad[t], want), (s.name, snip, t, t % ft, np.abs(grad[t] - want).max())
    assert all(np.array_equal(gf[t], gf[t_probe]) for t in interior)
    for k, t in enumerate(edges):  # each probe's gradient is its Gf alone
        W = np.zeros(ext_len, np.float32)
        W[t_probe * S: t_probe * S + L] = gf[t]
        assert np.array_equal(grad[T + k], _expected_impulse(W, n, pad, snip)), (s.name, t)
    # the full gradient against the sum of per-row impulses (summation order differs: a tolerance)
    Gfull = _rs(s.name, "full").randn(T, plan.feature_dim)
    rows = []
    for t in range(T):
        G = np.zeros_like(Gfull)
        G[t] = Gfull[t]
        rows.append(G)
    parts = E.b200_rows_grad(ext, np.stack([x] * T), rows).double().cpu().numpy()
    full = _alone(ext, x, Gfull).double().cpu().numpy()
    assert BC.rel_err(parts.sum(0), full) < 1e-5, BC.rel_err(parts.sum(0), full)
    if snip:
        assert not full[ext_len:].any() and ext_len < n and np.abs(full[:ext_len]).max() > 0


def _grid_stride_batch(s):
    ext = E.extractor(s.feature, **E.shape_kw(s))
    plan = ext.plan
    n = 10 * SR
    T = plan.num_frames(n)
    per_cut = -(-T // s.ft)
    grid = torch.cuda.get_device_properties(0).multi_processor_count * 64
    B = grid // per_cut + 2
    assert B * per_cut > grid
    second = -(-grid // per_cut)  # first cut whose tiles all come in the second stride round
    assert second < B
    return ext, plan, n, B, second


@pytest.mark.gpu
@pytest.mark.parametrize("s", [E.ACCEPTED[0], E.ACCEPTED[-1]], ids=["ft16", "ft1"])
def test_frames_kernel_grid_stride(s):
    """More tiles than the frames kernel's grid (multi_processor_count * 64): every cut bit for bit as itself alone, and
    the first, last and a second-round cut within the gate."""
    ext, plan, n, B, second = _grid_stride_batch(s)
    xs = [E.waveform(n, "noise", seed=i) for i in range(B)]
    Gs = [_rs(s.name, "stride", i).randn(plan.num_frames(n), plan.feature_dim) for i in range(B)]
    batched = E.b200_grads(ext, xs, Gs)
    for i in range(B):
        assert torch.equal(batched[i], _alone(ext, xs[i], Gs[i])), (s.name, i)
    for i in sorted({0, second, B - 1}):
        err, bound = _gate(xs[i], plan, Gs[i], batched[i].double().cpu().numpy())
        assert err <= bound, (s.name, i, err, bound)


@pytest.mark.gpu
def test_combine_kernel_strides_in_x():
    """A 70 s cut (more samples than 4096 blocks of 256 threads): within the gate, and an impulse at a frame past sample
    1,048,576 is the same impulse at an early frame, shifted, bit for bit."""
    s = E.ACCEPTED[0]
    ext = E.extractor(s.feature, **E.shape_kw(s))
    plan = ext.plan
    n = 70 * SR
    assert n > 4096 * 256
    x = E.waveform(n, "noise")
    G = _rs("x-stride").randn(plan.num_frames(n), plan.feature_dim)
    err, bound = _gate(x, plan, G, _alone(ext, x, G).double().cpu().numpy())
    assert err <= bound, (err, bound)
    L, S = plan.L, plan.S
    pad = (L - S) // 2
    T = plan.num_frames(n)
    xp = E.periodic_waveform(n, S)
    early, late = 3, (4096 * 256 + pad) // S + 5
    row = _rs("x-stride", "row").randn(plan.feature_dim)
    Gs = []
    for t in (early, late):
        Gt = np.zeros((T, plan.feature_dim))
        Gt[t] = row
        Gs.append(Gt)
    g = E.b200_rows_grad(ext, np.stack([xp, xp]), Gs).cpu()
    a, b = g[0], g[1]
    wa, wb = slice(early * S - pad, early * S - pad + L), slice(late * S - pad, late * S - pad + L)
    assert late * S - pad > 4096 * 256
    assert torch.equal(a[wa], b[wb]) and a[wa].abs().max() > 0
    a[wa] = 0
    b[wb] = 0
    assert not a.any() and not b.any()


@pytest.mark.gpu
def test_combine_kernel_strides_in_y():
    """65535 + 5 short cuts as one (B, n) batch with lengths: the cuts past index 65535 get a non-zero gradient, bit for bit
    what each gets alone, and nothing past its length."""
    ext = E.extractor("fbank")
    B, n = 65535 + 5, 800
    rs = np.random.RandomState(3)
    X = (0.1 * rs.randn(B, n)).astype(np.float32).astype(np.float64)
    lens = [int(v) for v in rs.randint(400, n + 1, size=B)]
    Gs = [_rs("y-stride", i).randn(ext.plan.num_frames(l), ext.plan.feature_dim) if i >= B - 12 else
          np.ones((ext.plan.num_frames(l), ext.plan.feature_dim)) for i, l in enumerate(lens)]
    g = E.b200_rows_grad(ext, X, Gs, lengths=lens)
    for i in range(B - 12, B):
        gi = g[i]
        assert not gi[lens[i]:].any()
        alone = _alone(ext, X[i, :lens[i]], Gs[i])
        assert torch.equal(gi[:lens[i]], alone), i
        if i >= 65535:
            assert gi.abs().max() > 0, i


@pytest.mark.gpu
@pytest.mark.parametrize("name,feature,kw", COMPAT, ids=[c[0] for c in COMPAT])
def test_compat_conventions_on_the_gpu(name, feature, kw):
    """The B200 forward against the twin's (float32 class), and the gradient within the gate against the twin, on noise and
    on the floors waveform, at a short and a multi-tile cut."""
    ext = E.extractor(feature, **E.compat_kw(kw))
    plan = ext.plan
    for n in (1000, 24000):
        for kind in ("noise", "floors"):
            x = E.waveform(n, kind, seed=len(name))
            with torch.no_grad():
                out = ext.extract(torch.tensor(x, dtype=torch.float32, device="cuda"), SR)
            out = out.double().cpu()
            f64 = BC.plan_features_t(torch.tensor(x), plan)
            G = _G(x, plan, name, kind, n)
            mask = torch.as_tensor(G != 0)
            if plan.feature in ("fbank", "mfcc"):
                mask = torch.ones_like(mask)
            d = (out - f64).abs()[mask]
            assert out.shape == f64.shape and bool((d <= 2e-3 + 1e-4 * f64.abs()[mask]).all()), (kind, n, float(d.max()))
            g = _alone(ext, x, G)
            err, bound = _gate(x, plan, G, g.double().cpu().numpy())
            assert err <= bound, (name, kind, n, err, bound)


@pytest.mark.gpu
@pytest.mark.parametrize("s", E.REFUSED, ids=[s.name for s in E.REFUSED])
def test_refused_frames(s):
    """The forward takes these frames; the backward refuses them with a RuntimeError that names the limit."""
    ext = E.extractor(s.feature, **E.shape_kw(s))
    n = 3 * ext.plan.L
    x = torch.tensor(E.waveform(n, "noise"), dtype=torch.float32, device="cuda", requires_grad=True)
    out = ext.extract(x, SR)
    assert out.requires_grad and out.shape == (ext.plan.num_frames(n), ext.plan.feature_dim)
    assert torch.isfinite(out).all()
    with pytest.raises(RuntimeError, match=r"frame too long .* over the backward's limit of 204800 bytes"):
        out.sum().backward()


@pytest.mark.gpu
def test_unaligned_view_input():
    """Features of leaf[1:] (4 bytes off a 16-byte boundary: the forward clones it) give leaf[1:] the gradient an aligned
    copy gets, bit for bit, and leaf[0] none."""
    ext = E.extractor("fbank", use_energy=True)
    x = E.waveform(16001, "noise")
    leaf = torch.tensor(x, dtype=torch.float32, device="cuda", requires_grad=True)
    view = leaf[1:]
    assert view.data_ptr() % 16
    out = ext.extract(view, SR)
    G = torch.as_tensor(_rs("unaligned").randn(*out.shape), dtype=torch.float32, device="cuda")
    (out * G).sum().backward()
    y = leaf.detach()[1:].clone().requires_grad_(True)
    (ext.extract(y, SR) * G).sum().backward()
    assert torch.equal(leaf.grad[1:], y.grad) and leaf.grad[0] == 0 and y.grad.abs().max() > 0


@pytest.mark.gpu
def test_list_of_mixed_devices_and_dtypes():
    """A CPU float64 item and a CUDA float32 item in one list: each gradient on its item's device and in its dtype, bit for
    bit what the item gets alone."""
    ext = E.extractor("mfcc", use_energy=True)
    a = torch.tensor(E.waveform(12345, "noise", seed=1), dtype=torch.float64, requires_grad=True)
    b = torch.tensor(E.waveform(16000, "noise", seed=2), dtype=torch.float32, device="cuda", requires_grad=True)
    outs = ext.extract_batch([a, b], SR)
    Ga = torch.as_tensor(_rs("mixed", 0).randn(*outs[0].shape), dtype=torch.float32, device="cuda")
    Gb = torch.as_tensor(_rs("mixed", 1).randn(*outs[1].shape), dtype=torch.float32, device="cuda")
    ((outs[0] * Ga).sum() + (outs[1] * Gb).sum()).backward()
    assert a.grad.device.type == "cpu" and a.grad.dtype == torch.float64
    assert b.grad.device.type == "cuda" and b.grad.dtype == torch.float32
    for leaf, G in ((a, Ga), (b, Gb)):
        y = leaf.detach().clone().requires_grad_(True)
        (ext.extract(y, SR) * G).sum().backward()
        assert torch.equal(leaf.grad, y.grad) and y.grad.abs().max() > 0
