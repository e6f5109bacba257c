"""The backward of the Kaldi-family extractors on the H100 (csrc/backward.cuh, DESIGN.md §3.1n).  Accuracy is held to the
error class of torch's own float32 gradient: per cut, ||g_b200 - g64|| <= 8 ||g32 - g64|| + 1e-7 ||g64||, where g64 is autograd
through the oracle's chain in float64 and g32 the same chain in float32 on the GPU (8, not 2: the packed real FFT's split
cancels on the weak low bins that a pre-emphasised, DC-free frame has, see DESIGN.md §3.1n).  Then the containers, determinism,
dither, the untouched no-grad path, double backward, and lhotse's own modules as the caller."""
import numpy as np
import pytest
import torch

import backward_cases as BC
import refshim

pytestmark = pytest.mark.gpu

ACC = [c for c in BC.configs()]


def _gate(x, cfg, G, g):
    g64 = BC.autograd_grad(x, cfg, G)
    g32 = BC.autograd_grad(x.astype(np.float32).astype(np.float64), cfg, G, dtype=torch.float32, device="cuda")
    bound = 8 * np.linalg.norm(g32 - g64) + 1e-7 * np.linalg.norm(g64)
    return float(np.linalg.norm(g - g64)), float(bound)


def _b200_grad(ext, x, G):
    xt = torch.tensor(x, dtype=torch.float32, device="cuda", requires_grad=True)
    out = ext.extract(xt, 16000)
    (out.to("cuda") * torch.as_tensor(G, dtype=torch.float32, device="cuda")).sum().backward()
    return xt.grad.double().cpu().numpy()


@pytest.mark.parametrize("name,cfg", ACC, ids=[c[0] for c in ACC])
def test_gradient_within_float32_error_class(name, cfg):
    L, S, N = BC.O.layer_sizes(cfg)
    kernels = ["auto", "generic"]
    if N == 512 and cfg.feature in ("fbank", "mfcc") and not cfg.use_energy and not cfg.snip_edges:
        kernels.append("tc")
    for kernel in kernels:
        ext = BC.b200_extractor(cfg, kernel=kernel)
        for n in BC.lengths(cfg, long=name in ("fbank", "mfcc", "log-spectrogram-energy-raw")):
            for kind in ("noise", "full"):
                x = BC.waveform(n, kind).astype(np.float32).astype(np.float64)
                T = BC.features_t(torch.tensor(x), cfg).shape
                G = BC.conditioned(x, cfg, np.random.RandomState(n).randn(*T), rel=1e-4)
                g = _b200_grad(ext, x, G)
                err, bound = _gate(x, cfg, G, g)
                assert err <= bound, (name, kernel, ext.engine.kernel, n, kind, err, bound)


def test_silence_gives_zero_gradient():
    for feat in ("fbank", "mfcc"):
        ext = BC.b200_extractor(BC.cfg_of(feat, use_energy=True))
        g = _b200_grad(ext, np.zeros(16000), np.ones(BC.features_t(torch.zeros(16000, dtype=torch.float64), BC.cfg_of(feat, use_energy=True)).shape))
        assert not g.any()


def _loss(out):
    w = torch.arange(out.numel(), device=out.device, dtype=out.dtype).reshape(out.shape).sin()
    return (out * w).sum()


@pytest.mark.parametrize("device,dtype", [("cpu", torch.float32), ("cpu", torch.float64), ("cuda", torch.float32),
                                          ("cuda", torch.float64)])
def test_extract_grad_lands_on_the_input(device, dtype):
    import lhotse_b200 as lb

    x = torch.tensor(BC.waveform(16000), dtype=dtype, device=device, requires_grad=True)
    out = lb.B200Fbank(lb.B200FbankConfig()).extract(x, 16000)
    assert out.requires_grad
    _loss(out).backward()
    assert x.grad.device == x.device and x.grad.dtype == dtype and x.grad.abs().sum() > 0


def test_extract_batch_containers():
    import lhotse_b200 as lb

    ext = lb.B200Mfcc(lb.B200MfccConfig(use_energy=True))
    ns = [16000, 12345, 8000]
    xs = [torch.tensor(BC.waveform(n), dtype=torch.float32, device="cuda", requires_grad=True) for n in ns]
    outs = ext.extract_batch(xs, 16000)
    _loss(torch.cat(outs)).backward()
    ones = []
    for x in xs:  # each item alone gives the same gradient
        y = x.detach().clone().requires_grad_(True)
        o = ext.extract(y, 16000)
        ones.append((y, o))
    _loss(torch.cat([o for _, o in ones])).backward()
    for x, (y, _) in zip(xs, ones):
        assert torch.equal(x.grad, y.grad)
    # (B, n) with and without lengths: exact zeros past each length
    X = torch.tensor(np.stack([BC.waveform(16000, seed=s) for s in range(3)]), dtype=torch.float32, device="cuda", requires_grad=True)
    out = ext.extract_batch(X, 16000)
    _loss(out).backward()
    assert X.grad.shape == X.shape and X.grad.abs().sum() > 0
    X.grad = None
    lens = [16000, 9000, 4000]
    res = ext.extract_batch(X, 16000, lengths=lens)
    sum(_loss(r) for r in res).backward()
    for i, l in enumerate(lens):
        assert not X.grad[i, l:].any() and X.grad[i, :l].abs().sum() > 0
        y = X.detach()[i, :l].clone().requires_grad_(True)
        _loss(ext.extract(y, 16000)).backward()
        assert torch.equal(y.grad, X.grad[i, :l])


def test_spectrogram_cpu_outputs_keep_the_graph():
    import lhotse_b200 as lb

    for cls, ccls in ((lb.B200Spectrogram, lb.B200SpectrogramConfig), (lb.B200LogSpectrogram, lb.B200LogSpectrogramConfig)):
        x = torch.tensor(BC.waveform(8000), dtype=torch.float32, device="cuda", requires_grad=True)
        out = cls(ccls()).extract(x, 16000)
        assert out.device.type == "cpu" and out.requires_grad
        _loss(out).backward()
        assert x.grad.abs().sum() > 0
        xs = [torch.tensor(BC.waveform(n), dtype=torch.float32, device="cuda", requires_grad=True) for n in (8000, 8000)]
        out = cls(ccls()).extract_batch(xs, 16000)
        assert out.device.type == "cpu" and out.requires_grad
        _loss(out).backward()
        assert all(x.grad.abs().sum() > 0 for x in xs)


def test_backward_is_deterministic_and_batch_independent():
    import lhotse_b200 as lb

    ext = lb.B200Fbank(lb.B200FbankConfig(use_energy=True))
    rs = np.random.RandomState(1)
    ns = [int(n) for n in rs.randint(400, 160000, size=64)]
    xs = [torch.tensor(BC.waveform(n, seed=i), dtype=torch.float32, device="cuda") for i, n in enumerate(ns)]

    def grads(items):
        leaves = [x.clone().requires_grad_(True) for x in items]
        out = ext.extract_batch(leaves, 16000)
        (torch.cat(out) if isinstance(out, list) else out).sin().sum().backward()
        return [x.grad for x in leaves]

    a, b = grads(xs), grads(xs)
    assert all(torch.equal(u, v) for u, v in zip(a, b))
    alone = grads([xs[5]])[0]
    assert torch.equal(alone, a[5])


def test_dither_gradient_is_taken_at_the_noisy_waveform():
    import lhotse_b200 as lb

    x = torch.tensor(BC.waveform(16000), dtype=torch.float32, device="cuda", requires_grad=True)
    torch.manual_seed(7)
    out = lb.B200Fbank(lb.B200FbankConfig(dither=0.1)).extract(x, 16000)
    _loss(out).backward()
    torch.manual_seed(7)
    noisy = x.detach() + 0.1 * torch.randn(x.shape, device="cuda", dtype=torch.float32)
    y = noisy.clone().requires_grad_(True)
    _loss(lb.B200Fbank(lb.B200FbankConfig()).extract(y, 16000)).backward()
    assert torch.equal(x.grad, y.grad)


def test_no_grad_path_is_untouched():
    import lhotse_b200 as lb

    ext = lb.B200Fbank(lb.B200FbankConfig())
    x = torch.tensor(BC.waveform(16000), dtype=torch.float32, device="cuda")
    ref = ext.extract(x, 16000)
    before = ext.engine.stats()["kernel_launches"]
    xg = x.clone().requires_grad_(True)
    with torch.no_grad():
        out = ext.extract(xg, 16000)
    assert not out.requires_grad and torch.equal(out, ref)
    out = ext.extract(x, 16000)
    assert not out.requires_grad and torch.equal(out, ref)
    assert ext.engine.stats()["kernel_launches"] == before + 2
    og = ext.extract(xg, 16000)  # the graph path runs the same forward launch
    assert og.requires_grad and torch.equal(og.detach(), ref)
    with pytest.raises(RuntimeError):
        torch.autograd.grad(_loss(og), xg, create_graph=True)


@pytest.mark.reference
@pytest.mark.skipif(not refshim.reference_available(), reason="no reference tree / oracle/_ref archive")
def test_gradients_through_lhotse_modules():
    refshim.import_reference()
    from lhotse.features.kaldi.extractors import Fbank, FbankConfig, Mfcc, MfccConfig

    import lhotse_b200 as lb

    for ref_cls, ref_cfg, cls, ccls, ocfg in ((Fbank, FbankConfig, lb.B200Fbank, lb.B200FbankConfig, BC.cfg_of("fbank")),
                                              (Mfcc, MfccConfig, lb.B200Mfcc, lb.B200MfccConfig, BC.cfg_of("mfcc"))):
        x = BC.waveform(24000).astype(np.float32).astype(np.float64)
        module = ref_cls(ref_cfg(device="cpu")).extractor.double()
        xr = torch.tensor(x, requires_grad=True)
        out = module(xr.unsqueeze(0))[0]
        G = np.random.RandomState(0).randn(*out.shape)
        (out * torch.as_tensor(G)).sum().backward()
        g = _b200_grad(cls(ccls()), x, G)
        err_ref = float(np.linalg.norm(g - xr.grad.numpy()))
        _, bound = _gate(x, ocfg, G, g)
        assert err_ref <= bound + 1e-6 * np.linalg.norm(xr.grad.numpy()), (ref_cls.__name__, err_ref, bound)
