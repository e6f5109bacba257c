"""The whisper-fbank backward on the H100 (csrc/backward.cuh, DESIGN.md §3.1p): accuracy per cut against float64 autograd
through the oracle's chain, gated at 8x the float32 torch chain's own error, for the fast400 and generic forwards at M = 80
and 128; exact properties (silence, clamped frames, the zero row, determinism, batch independence, lengths); every entry
point and container; the untouched no-grad path; the refusals; and a Conv1d ahead of the extractor as the caller."""
import numpy as np
import pytest
import torch

import refshim
import whisper_backward_cases as WB
from oracle import whisper_oracle as W

pytestmark = pytest.mark.gpu

LENS = (201, 16000, 16079, 16080, 48159)


@pytest.mark.parametrize("M", [80, 128])
@pytest.mark.parametrize("kernel", ["auto", "generic"])
def test_gpu_accuracy_per_cut(kernel, M):
    ext = WB.extractor(kernel, M)
    worst = 0.0
    for kind in ("noise", "burst"):
        for n in LENS:
            x, G = WB.case(n, kind, M)
            g = WB.b200_grad(ext, x, G)
            err, bound, err32 = WB.gate(x, G, M, g)
            assert err <= bound, (kernel, M, kind, n, err, bound)
            worst = max(worst, err / max(err32, 1e-300))
    print(f"whisper backward {kernel} M={M}: worst ratio to the float32 chain's error {worst:.2f}")


@pytest.mark.parametrize("kernel", ["auto", "generic"])
def test_gpu_tied_maximum_against_the_saved_rows(kernel):
    """A hop-periodic waveform ties its maximum across interior frames: the routed mass is split evenly over the ties the
    forward itself saw, so the reference is the restatement fed the forward's own rows and maximum."""
    ext = WB.extractor(kernel)
    for n in (16000, 16080, 32080):
        x = WB.waveform(n, "periodic").astype(np.float32).astype(np.float64)
        xt = torch.tensor(x, dtype=torch.float32, device="cuda")
        buf = xt.contiguous()
        _, raw, prefix = ext.engine.extract_device_keep_raw(buf, [n], [0])
        R = int(prefix[-1])
        xr = raw[: R * 80].view(R, 80)[: n // 160].double().cpu().numpy()
        m = float(raw[R * 80].item())
        assert (xr == m).sum() > 10 and (xr < m - 8.0).any()  # ties and a binding clamp
        G = np.random.RandomState(n).randn(R, 80)
        g = WB.b200_grad(ext, x, G)
        want = WB.restated_grad(x, G, 80, xr=xr, m=m)
        assert WB.rel_err(g, want) < 2e-3, (kernel, n, WB.rel_err(g, want))


def test_gpu_exact_properties():
    ext = WB.extractor()
    n = 48159
    G = np.random.RandomState(1).randn(W.num_rows(n), 80)
    assert not WB.b200_grad(ext, np.zeros(n), G).any()  # silence: every mel energy is clamped
    # a loud first second, then a tail 100 dB down whose log-mel values all sit below m - 8: the samples only the tail's
    # frames cover get exactly 0
    rs = np.random.RandomState(2)
    x = 1e-5 * rs.randn(n)
    x[:16000] = rs.randn(16000)
    g = WB.b200_grad(ext, x, G)
    assert g[:15000].any() and not g[160 * 101 + 200:].any()  # frame 101 is the last to reach a loud sample
    # the zero row's gradient does not matter, two runs agree, and so does a cut batched with others
    x = WB.waveform(16080, "burst")
    G = np.random.RandomState(3).randn(W.num_rows(16080), 80)
    g1 = WB.b200_grad(ext, x, G)
    G2 = G.copy()
    G2[-1] = 1e6
    assert np.array_equal(WB.b200_grad(ext, x, G2), g1)
    assert np.array_equal(WB.b200_grad(ext, x, G), g1)
    others = [WB.waveform(n, "noise", 5) for n in (4000, 16080, 31999)]
    items = [torch.tensor(a, dtype=torch.float32, device="cuda", requires_grad=True) for a in others[:1] + [x] + others[1:]]
    feats = ext.extract_batch(items, 16000)
    total = sum(WB.loss(f, np.random.RandomState(i).randn(*f.shape)) for i, f in enumerate(feats) if i != 1) + WB.loss(feats[1], G)
    total.backward()
    assert np.array_equal(items[1].grad.double().cpu().numpy(), g1)


def test_gpu_lengths_and_padded_rows():
    ext = WB.extractor()
    B, n = 3, 32000
    lengths = [32000, 16080, 20001]
    x = torch.tensor(np.stack([WB.waveform(n, "noise", i) for i in range(B)]), dtype=torch.float32, device="cuda",
                     requires_grad=True)
    feats = ext.extract_batch(x, 16000, lengths=lengths)
    Gs = [np.random.RandomState(i).randn(*f.shape) for i, f in enumerate(feats)]
    sum(WB.loss(f, g) for f, g in zip(feats, Gs)).backward()
    gx = x.grad.double().cpu().numpy()
    for i, L in enumerate(lengths):
        assert not gx[i, L:].any()
        alone = WB.b200_grad(ext, x.detach()[i, :L].double().cpu().numpy(), Gs[i])
        assert np.array_equal(gx[i, :L], alone), i


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
@pytest.mark.parametrize("device", ["cpu", "cuda"])
def test_gpu_containers(device, dtype):
    ext = WB.extractor()
    xs = [WB.waveform(n, "noise", 7) for n in (16000, 16080)]
    G = [np.random.RandomState(i).randn(W.num_rows(len(a)), 80) for i, a in enumerate(xs)]
    want = [WB.b200_grad(ext, a, g) for a, g in zip(xs, G)]
    # extract on one tensor
    t = torch.tensor(xs[0], dtype=dtype, device=device, requires_grad=True)
    WB.loss(ext.extract(t, 16000), G[0]).backward()
    assert t.grad.dtype == dtype and t.grad.device == t.device
    assert np.allclose(t.grad.double().cpu().numpy(), want[0], rtol=0, atol=1e-6 * np.abs(want[0]).max())
    # extract_batch on a list
    ts = [torch.tensor(a, dtype=dtype, device=device, requires_grad=True) for a in xs]
    out = ext.extract_batch(ts, 16000)
    sum(WB.loss(o, g) for o, g in zip(out, G)).backward()
    for tt, w in zip(ts, want):
        assert tt.grad.dtype == dtype and tt.grad.device == tt.device
        assert np.allclose(tt.grad.double().cpu().numpy(), w, rtol=0, atol=1e-6 * np.abs(w).max())
    # extract_batch on a (B, n) tensor without lengths
    b = torch.tensor(np.stack([xs[0], xs[0][::-1].copy()]), dtype=dtype, device=device, requires_grad=True)
    out = ext.extract_batch(b, 16000)
    assert out.shape == (2, 100, 80) and out.requires_grad
    WB.loss(out[0], G[0]).backward()
    assert b.grad.dtype == dtype and b.grad.device == b.device and not b.grad[1].any()
    assert np.allclose(b.grad[0].double().cpu().numpy(), want[0], rtol=0, atol=1e-6 * np.abs(want[0]).max())


def test_gpu_no_grad_path_untouched():
    ext = WB.extractor()
    x = torch.tensor(WB.waveform(48159, "burst"), dtype=torch.float32, device="cuda")
    before = ext.engine.stats()["kernel_launches"]
    ref = ext.extract(x, 16000)
    assert ext.engine.stats()["kernel_launches"] - before == 2 and not ref.requires_grad
    with torch.no_grad():
        assert torch.equal(ext.extract(x.clone().requires_grad_(), 16000), ref)
    assert np.array_equal(ref.cpu().numpy(), ext.extract(x.cpu().numpy(), 16000))
    xg = x.clone().requires_grad_()
    og = ext.extract(xg, 16000)
    assert og.requires_grad and torch.equal(og.detach(), ref)
    # the other detached classes stay detached
    import lhotse_b200 as lb

    assert not lb.B200LibrosaFbank().extract(x.clone().requires_grad_(), 22050).requires_grad


def test_gpu_failure_modes():
    ext = WB.extractor()
    xg = torch.tensor(WB.waveform(16000, "noise"), dtype=torch.float32, device="cuda", requires_grad=True)
    og = ext.extract(xg, 16000)
    with pytest.raises(RuntimeError):
        torch.autograd.grad(WB.loss(og, np.ones(og.shape)), xg, create_graph=True)
    with pytest.raises(ValueError):
        ext.extract(torch.zeros(200, device="cuda", requires_grad=True), 16000)
    with pytest.raises(NotImplementedError):
        ext.online_inference(torch.zeros(1, 16000))


def test_gpu_abi_refusals():
    from lhotse_b200 import engine

    eng = WB.extractor().engine
    lib = eng.lib
    x = torch.zeros(32000, device="cuda")
    g = torch.zeros(200 * 80, device="cuda")
    raw = torch.zeros(200 * 80 + 2, device="cuda")
    work = torch.zeros(1 << 24, dtype=torch.uint8, device="cuda")

    def call(ns, rows):
        ns = np.asarray(ns, dtype=np.int64)
        off = np.asarray([0, 16000][: len(ns)], dtype=np.int64)
        rows = np.asarray(rows, dtype=np.int64)
        return lib.b200feat_whisper_backward(eng._h, x.data_ptr(), engine.DT_F32, ns.ctypes.data, off.ctypes.data, len(ns),
                                             g.data_ptr(), raw.data_ptr(), raw.data_ptr() + 4 * 200 * 80, rows.ctypes.data,
                                             x.data_ptr(), work.data_ptr(), work.numel(), None)

    assert call([16000], [0, 100]) == 0
    assert call([16000], [0, 101]) == -1 and "row_off" in lib.b200feat_last_error(eng._h).decode()
    assert call([16000, 200], [0, 100, 101]) == -5
    ns = np.asarray([16000], dtype=np.int64)
    rc = lib.b200feat_backward(eng._h, x.data_ptr(), engine.DT_F32, ns.ctypes.data, ns.ctypes.data, 1, g.data_ptr(),
                               np.asarray([0, 100], dtype=np.int64).ctypes.data, x.data_ptr(), work.data_ptr(), work.numel(), None)
    assert rc == -1 and "b200feat_whisper_backward" in lib.b200feat_last_error(eng._h).decode()
    rc = lib.b200feat_whisper_backward(eng._h, x.data_ptr(), 1, ns.ctypes.data, ns.ctypes.data, 1, g.data_ptr(), raw.data_ptr(),
                                       raw.data_ptr(), np.asarray([0, 100], dtype=np.int64).ctypes.data, x.data_ptr(),
                                       work.data_ptr(), work.numel(), None)
    assert rc == -1 and "float32" in lib.b200feat_last_error(eng._h).decode()
    torch.cuda.synchronize()


@pytest.mark.reference
@pytest.mark.skipif(not refshim.reference_available(), reason="no reference tree / oracle/_ref archive")
def test_gpu_conv1d_ahead_of_the_extractor_matches_lhotse():
    pytest.importorskip("transformers")
    refshim.install_librosa_standin()
    refshim.import_reference()
    from lhotse.features.whisper_fbank import WhisperFbank, WhisperFbankConfig

    x = torch.tensor(WB.waveform(32000, "noise"), dtype=torch.float64)
    G = np.random.RandomState(0).randn(200, 80)

    def weight_grad(front, conv, dtype, device):
        conv = conv.to(device=device, dtype=dtype)
        y = conv(x.to(device=device, dtype=dtype).view(1, 1, -1)).view(-1)
        WB.loss(front(y), G).backward()
        return conv.weight.grad.double().cpu().numpy().ravel()

    torch.manual_seed(0)
    base = torch.nn.Conv1d(1, 1, 9, padding=4, bias=False)
    mk = lambda: torch.nn.Conv1d(1, 1, 9, padding=4, bias=False).requires_grad_(True)  # noqa: E731
    convs = []
    for _ in range(3):
        c = mk()
        c.load_state_dict(base.state_dict())
        convs.append(c)
    ref64 = WhisperFbank(WhisperFbankConfig())
    ref64.filters, ref64.window = ref64.filters.double(), ref64.window.double()
    ref32 = WhisperFbank(WhisperFbankConfig(device="cuda"))
    b200 = WB.extractor()
    w64 = weight_grad(lambda y: ref64.extract(y, 16000), convs[0], torch.float64, "cpu")
    w32 = weight_grad(lambda y: ref32.extract(y, 16000), convs[1], torch.float32, "cuda")
    wb = weight_grad(lambda y: b200.extract(y, 16000), convs[2], torch.float32, "cuda")
    err, err32 = np.linalg.norm(wb - w64), np.linalg.norm(w32 - w64)
    assert err <= 8.0 * err32 + 1e-7 * np.linalg.norm(w64), (err, err32)
