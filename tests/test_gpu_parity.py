"""Parity tests proper: CUDA kernels, called through the C ABI (lhotse_b200.engine.Engine ->
libb200feat.so), against (a) the committed golden vectors of the real reference, (b) the oracle
on seeded inputs, (c) size-independent properties at BASELINE sizes."""
import numpy as np
import pytest
import torch

from helpers import gate, load_golden, oracle_cfg
from lhotse_b200 import (B200Fbank, B200FbankConfig, B200LogSpectrogram, B200LogSpectrogramConfig, B200Mfcc,
                         B200MfccConfig, B200Spectrogram, B200SpectrogramConfig, LOG_EPSILON)
from lhotse_b200.engine import B200FeatError
from oracle import kaldi_oracle as O

pytestmark = pytest.mark.gpu

TYPES = {"fbank": (B200Fbank, B200FbankConfig), "mfcc": (B200Mfcc, B200MfccConfig),
         "spectrogram": (B200Spectrogram, B200SpectrogramConfig),
         "log-spectrogram": (B200LogSpectrogram, B200LogSpectrogramConfig)}
GOLD = load_golden()
IDS = [f"{i}-{c['feature']}-{c['kind']}-{c['n']}" for i, c, _, _ in GOLD]


def make(feature, cfg, kernel="auto"):
    cls, ccls = TYPES[feature]
    ext = cls(ccls(kernel=kernel, **cfg))
    try:
        ext.engine
    except B200FeatError as e:
        if e.code == -2 and kernel.startswith("fast"):
            pytest.skip("plan not supported by the fast kernel")
        raise
    return ext


def kernels_for(ext):
    """Every kernel that supports the plan is tested (generic always; fast when AUTO picks it)."""
    if ext.engine.kernel == "generic":
        return ["generic"]
    ks = ["generic", "fast"]
    if ext.plan.N == 512 and ext.plan.feature in ("fbank", "mfcc") and not ext.plan.use_energy:
        ks.append("tc")
    return ks


@pytest.mark.parametrize("i,c,x,y", GOLD, ids=IDS)
def test_golden_vectors(i, c, x, y):
    sr = c["cfg"].get("sampling_rate", 16000)
    truth = O.extract(x, oracle_cfg(c["feature"], c["cfg"]), dtype=torch.float64)
    for k in kernels_for(make(c["feature"], c["cfg"])):
        ext = make(c["feature"], c["cfg"], kernel=k)
        got = ext.extract(x, sr)
        assert got.dtype == np.float32 and got.shape == y.shape, (k, got.shape)  # frame counts: bit-exact
        ok, msg = gate(got, y, truth, c["feature"], c["cfg"].get("use_energy", False), c["cfg"].get("use_fft_mag", False))
        assert ok, f"kernel={k}: {msg}"


@pytest.mark.parametrize("kernel", ["generic", "fast", "tc"])
def test_ragged_batch_equals_per_cut(kernel):
    rs = np.random.RandomState(5)
    lens = [159, 160, 1599, 16000, 16001, 23456, 480, 100000, 16080]
    xs = [(0.1 * rs.randn(n)).astype(np.float32) for n in lens]
    ext = make("fbank", {}, kernel=kernel)
    batch = ext.extract_batch(xs, 16000)
    assert isinstance(batch, list) and len(batch) == len(xs)
    cfg = O.OracleConfig()
    for x, got in zip(xs, batch):
        ref = O.extract(x, cfg)
        truth = O.extract(x, cfg, dtype=torch.float64)
        assert got.shape == ref.shape
        ok, msg = gate(got, ref, truth, "fbank")
        assert ok, msg
        assert np.array_equal(got, ext.extract(x, 16000))  # batch item == single extract, bit for bit
    # torch inputs (device-resident path) give the same bits as the host path
    tb = ext.extract_batch([torch.from_numpy(x) for x in xs], 16000)
    for a, b in zip(batch, tb):
        assert b.is_cuda and np.array_equal(a, b.cpu().numpy())


@pytest.mark.parametrize("kernel", ["generic", "fast", "tc"])
def test_padded_mode_and_int16(kernel):
    rs = np.random.RandomState(6)
    pcm = [np.clip(rs.randn(n) * 3000, -32768, 32767).astype(np.int16) for n in (4000, 16000, 9999)]
    ext = make("fbank", {}, kernel=kernel)
    feats, lens = ext.extract_batch_padded([torch.from_numpy(p.astype(np.float32) / 32768.0) for p in pcm], 16000)
    assert feats.shape == (3, 100, 80) and lens.tolist() == [25, 100, 62]
    f = feats.cpu().numpy()
    assert np.all(f[0, 25:] == np.float32(LOG_EPSILON)) and np.all(f[2, 62:] == np.float32(LOG_EPSILON))
    cfg = O.OracleConfig()
    for i, p in enumerate(pcm):
        x = p.astype(np.float32) / 32768.0
        ok, msg = gate(f[i, : lens[i]], O.extract(x, cfg), O.extract(x, cfg, dtype=torch.float64), "fbank")
        assert ok, msg
    # int16 staging: same bits as float32 staging of x/32768
    i16 = ext.extract_batch(pcm, 16000)
    f32 = ext.extract_batch([p.astype(np.float32) / 32768.0 for p in pcm], 16000)
    for a, b in zip(i16, f32):
        assert np.array_equal(a, b)


def test_headline_size_properties():
    """BASELINE config 2 at full size (64 x 10 s): shapes, determinism, shift- and batch-invariance."""
    torch.manual_seed(0)
    B, n = 64, 160000
    x = (0.1 * torch.randn(B, n)).cuda()
    ext = make("fbank", {})
    y = ext.extract_batch(x, 16000)
    assert y.shape == (B, 1000, 80) and y.is_cuda and torch.isfinite(y).all()
    y2 = ext.extract_batch(x, 16000)
    assert torch.equal(y, y2)  # deterministic
    perm = torch.randperm(B)
    yp = ext.extract_batch(x[perm.cuda()], 16000)
    assert torch.equal(yp, y[perm.cuda()])  # cuts are independent
    # frames away from the edges depend only on their own 400 samples: shifting the cut by one hop
    # shifts the features by one frame, bit for bit
    ys = ext.extract_batch(x[:4, 160:], 16000)
    assert torch.equal(ys[:, 2:900], y[:4, 3:901])
    # a sample of cuts against the oracle
    cfg = O.OracleConfig()
    for b in (0, 31, 63):
        xb = x[b].cpu().numpy()
        ok, msg = gate(y[b].cpu().numpy(), O.extract(xb, cfg), O.extract(xb, cfg, dtype=torch.float64), "fbank")
        assert ok, msg
    # generic and fast kernels agree to fp32 noise
    if ext.engine.kernel == "fast":
        yg = make("fbank", {}, kernel="generic").extract_batch(x[:8], 16000)
        assert torch.allclose(yg, y[:8], rtol=1e-4, atol=2e-4)


def test_mfcc_config3_tolerance():
    """BASELINE config 3: Mfcc(num_ceps=13, num_mel_bins=23) at the reference's own tolerance (test/features/
    test_kaldi_features.py:122: rtol 1e-3, atol 1e-4), on every kernel."""
    torch.manual_seed(1)
    x = (0.1 * torch.randn(8, 160000)).numpy()
    cfg = O.OracleConfig(feature="mfcc", num_ceps=13, num_filters=23)
    refs = [O.extract(x[b], cfg) for b in range(8)]
    for k in ("generic", "fast", "tc"):
        ext = make("mfcc", dict(num_ceps=13, num_mel_bins=23), kernel=k)
        y = ext.extract_batch(x, 16000)
        assert y.shape == (8, 1000, 13)
        for b in range(8):
            np.testing.assert_allclose(y[b], refs[b], rtol=1e-3, atol=1e-4, err_msg=f"kernel={k}")


def test_device_tables_roundtrip():
    ext = make("mfcc", {})
    e = ext.engine
    assert np.array_equal(e.get_table(0), ext.plan.window)
    assert np.array_equal(e.get_table(1).reshape(ext.plan.mel_bank.shape), ext.plan.mel_bank)
    assert np.array_equal(e.get_table(2).reshape(ext.plan.dct.shape), ext.plan.dct)
    assert np.array_equal(e.get_table(3), ext.plan.lifter)
    tw = e.get_table(4).reshape(-1, 2)
    k = np.arange(tw.shape[0])
    assert np.allclose(tw[:, 0], np.cos(2 * np.pi * k / tw.shape[0]), atol=1e-7)
    st = e.stats()
    assert st["calls"] == 0


def test_errors_do_not_abort():
    ext = make("fbank", {})
    with pytest.raises(ValueError):
        ext.extract(np.zeros(100, dtype=np.float32), 16000)
    with pytest.raises(ValueError):
        ext.extract_batch([np.zeros(16000, dtype=np.float32), np.zeros(50, dtype=np.float32)], 16000)
    assert ext.extract(np.zeros(1600, dtype=np.float32), 16000).shape == (10, 80)  # still usable


def test_concurrent_streams():
    ext = make("fbank", {})
    torch.manual_seed(2)
    xs = [(0.1 * torch.randn(16, 32000)).cuda() for _ in range(4)]
    want = [ext.extract_batch(x, 16000) for x in xs]
    streams = [torch.cuda.Stream() for _ in xs]
    got = []
    for s, x in zip(streams, xs):
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            got.append(ext.extract_batch(x, 16000))
    torch.cuda.synchronize()
    for a, b in zip(want, got):
        assert torch.equal(a, b)


def test_long_recording_and_many_tiny_cuts():
    """Scale edges: one 30-minute recording (180 000 frames, SURVEY.md §5 'long input') and 5000 ragged
    0.2-1.2 s cuts in one call.  Interior frames depend only on their own 400 samples, so windows of the long
    cut are checked against the oracle run on the matching slice."""
    ext = make("fbank", {})
    rs = np.random.RandomState(11)
    n = 30 * 60 * 16000
    x = (0.1 * rs.randn(n)).astype(np.float32)
    y = ext.extract(x, 16000)
    assert y.shape == (180000, 80) and np.isfinite(y).all()
    cfg = O.OracleConfig()
    for t0 in (0, 1234, 99990, 179900):
        t1 = min(t0 + 100, 180000)
        lo, hi = max(0, (t0 - 12) * 160), min(n, (t1 + 12) * 160)  # slice starts on a hop boundary
        ref = O.extract(x[lo:hi], cfg)
        shift = lo // 160  # global index of the slice's frame 0
        # compare interior frames only (the slice reflects at its own ends)
        a0 = t0 if lo == 0 else t0 + 2
        a1 = t1 if hi == n else t1 - 2
        got = y[a0:a1]
        want = ref[a0 - shift:a1 - shift]
        assert got.shape == want.shape and got.shape[0] > 50
        np.testing.assert_allclose(got, want, rtol=1e-4, atol=1e-3)
    lens = rs.randint(3200, 19200, size=5000)
    xs = [(0.1 * rs.randn(m)).astype(np.float32) for m in lens]
    out = ext.extract_batch(xs, 16000)
    assert len(out) == 5000
    for i in rs.choice(5000, size=25, replace=False):
        ref = O.extract(xs[i], cfg)
        assert out[i].shape == ref.shape
        np.testing.assert_allclose(out[i], ref, rtol=1e-4, atol=1e-3)


def test_nan_inputs_stay_local():
    """A NaN sample poisons only the frames whose window covers it (as in the reference)."""
    ext = make("fbank", {})
    x = (0.1 * np.random.RandomState(3).randn(32000)).astype(np.float32)
    x[16000] = np.nan
    y = ext.extract(x, 16000)
    bad = np.where(~np.isfinite(y).all(axis=1))[0]
    assert bad.min() >= 98 and bad.max() <= 101 and len(bad) >= 2  # frames whose 400-sample window holds sample 16000
    assert np.isfinite(y[:98]).all() and np.isfinite(y[102:]).all()


def _torchaudio_golden():
    import json
    import os

    g = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "golden_torchaudio_v1.npz"))
    man = json.loads(bytes(g["manifest"]).decode())
    return [(i, c, g[f"x{i}"], g[f"y{i}"]) for i, c in enumerate(man)]


TA_GOLD = _torchaudio_golden()


@pytest.mark.parametrize("i,c,x,y", TA_GOLD, ids=[f"{i}-{c['feature']}" for i, c, _, _ in TA_GOLD])
@pytest.mark.parametrize("kernel", ["generic", "fast"])
def test_torchaudio_family_golden(kernel, i, c, x, y):
    """Second oracle: torchaudio.compliance.kaldi outputs (tests/golden/make_golden_torchaudio.py) for the
    TorchaudioFbank/TorchaudioMfcc config family — Kaldi log-energy convention, energy placement, blackman variant.
    Gate as in the reference's own comparison test (test/features/test_kaldi_features.py:116-122: rtol 1e-3, atol 1e-4),
    with the absolute part widened to the fp32 noise floor of log-mel values measured in helpers.py."""
    from types import SimpleNamespace

    from lhotse_b200 import from_reference_config

    cfg = SimpleNamespace(**c["cfg"])
    ext = from_reference_config(cfg, sampling_rate=16000)
    ext.config.kernel = kernel
    got = ext.extract(x, 16000)
    assert got.shape == y.shape and ext.engine.kernel == kernel
    np.testing.assert_allclose(got, y, rtol=1e-3, atol=5e-4)


def test_dither_is_waveform_noise_from_the_device_generator():
    """layers.py:190-193 semantics: features of (x + dither*randn) with randn from torch's CUDA generator."""
    x = (0.1 * np.random.RandomState(5).randn(16000)).astype(np.float32)
    ext = make("fbank", dict(dither=0.01))
    clean = make("fbank", {})
    torch.manual_seed(7)
    a = ext.extract(x, 16000)
    torch.manual_seed(7)
    noise = torch.randn(16000, device="cuda")
    want = clean.extract(torch.from_numpy(x).cuda() + 0.01 * noise, 16000).cpu().numpy()
    assert np.array_equal(a, want)
    torch.manual_seed(7)
    b = ext.extract_batch([x], 16000)[0]
    assert np.array_equal(a, b)
    assert not np.array_equal(a, clean.extract(x, 16000))
    # int16 input is scaled before the noise is added, exactly like float input
    pcm = (x * 32768).astype(np.int16)
    torch.manual_seed(7)
    c = ext.extract(pcm, 16000)
    torch.manual_seed(7)
    d = ext.extract(pcm.astype(np.float32) / 32768.0, 16000)
    assert np.array_equal(c, d)


@pytest.mark.parametrize("feature,cfg", [
    ("fbank", dict(sampling_rate=8000, num_filters=40)),
    ("fbank", dict(sampling_rate=8000, num_filters=23, use_energy=True)),
    ("fbank", dict(sampling_rate=8000, num_filters=40, use_fft_mag=True, window_type="hamming", preemph_coeff=0.0)),
    ("mfcc", dict(sampling_rate=8000)),
    ("mfcc", dict(sampling_rate=8000, use_energy=True, num_ceps=10)),
    ("spectrogram", dict(sampling_rate=8000)),
    ("log-spectrogram", dict(sampling_rate=8000, use_energy=True)),
    ("fbank", dict(sampling_rate=16000, frame_length=0.016, frame_shift=0.008, num_filters=40)),  # L = N = 256, S = 128
])
def test_fast256_kernel_vs_oracle(feature, cfg):
    """The N = 256 fast kernel (8 kHz geometry and every plan with 128 < L <= 256) against the oracle on ragged lengths
    that hit the frame-count edges, plus int16 staging and the padded output mode."""
    sr = cfg["sampling_rate"]
    ext = make(feature, cfg, kernel="fast")
    assert ext.engine.kernel == "fast" and ext.plan.N == 256
    gen = make(feature, cfg, kernel="generic")
    rs = np.random.RandomState(9)
    S, L = ext.plan.S, ext.plan.L
    lens = [L, L + 1, 10 * S - 1, 10 * S + S // 2, 10 * S + S // 2 - 1, 8000, 8003, 20000, 333 * S]
    xs = [(0.1 * rs.randn(m)).astype(np.float32) for m in lens]
    xs[3][: len(xs[3]) // 2] *= 1e-4
    got = ext.extract_batch(xs, sr)
    ocfg = oracle_cfg(feature, cfg)
    for x, g in zip(xs, got):
        ref = O.extract(x, ocfg)
        truth = O.extract(x, ocfg, dtype=torch.float64)
        assert g.shape == ref.shape
        ok, msg = gate(g, ref, truth, feature, cfg.get("use_energy", False), cfg.get("use_fft_mag", False))
        assert ok, msg
    for a, b_ in zip(got, gen.extract_batch(xs, sr)):
        np.testing.assert_allclose(a, b_, rtol=2e-4, atol=5e-4 if feature != "spectrogram" else 1e-3)
    if feature == "fbank" and not cfg.get("use_energy"):
        pcm = [np.clip(x * 32768, -32768, 32767).astype(np.int16) for x in xs]
        i16 = ext.extract_batch(pcm, sr)
        f32 = ext.extract_batch([q.astype(np.float32) / 32768.0 for q in pcm], sr)
        for a, b_ in zip(i16, f32):
            assert np.array_equal(a, b_)
        feats, flens = ext.extract_batch_padded([torch.from_numpy(x) for x in xs], sr)
        assert feats.shape[0] == len(xs) and flens.tolist() == [g.shape[0] for g in got]
        fcpu = feats.cpu().numpy()
        for i, g in enumerate(got):
            assert np.array_equal(fcpu[i, : g.shape[0]], g)
            assert np.all(fcpu[i, g.shape[0]:] == np.float32(LOG_EPSILON))


@pytest.mark.parametrize("variant", ["0", "1"])
@pytest.mark.parametrize("feature,cfg", [
    ("fbank", dict(sampling_rate=22050)),                                   # L = 551 (odd), S = 220
    ("fbank", dict(sampling_rate=24000, num_filters=128, use_energy=True)),  # L = 600, S = 240
    ("fbank", dict(sampling_rate=24000, use_fft_mag=True, window_type="hanning", preemph_coeff=0.0, snip_edges=True)),
    ("mfcc", dict(sampling_rate=24000, num_ceps=20, num_filters=40)),
    ("mfcc", dict(sampling_rate=22050, use_energy=True)),
    ("spectrogram", dict(sampling_rate=24000)),
    ("log-spectrogram", dict(sampling_rate=22050, use_energy=True)),
    ("fbank", dict(sampling_rate=16000, frame_length=0.064, frame_shift=0.016)),  # L = N = 1024, S = 256
    ("fbank", dict(sampling_rate=44100, frame_length=0.02, frame_shift=0.01)),    # L = 882
])
def test_fast1024_kernel_vs_oracle(feature, cfg, variant, monkeypatch):
    """The N = 1024 fast kernel (22.05 / 24 kHz geometry and every plan with 512 < L <= 1024), both launch shapes,
    against the oracle and the generic kernel on ragged lengths, plus int16 staging and the padded output mode."""
    monkeypatch.setenv("B200FEAT_FAST1024_VARIANT", variant)
    sr = cfg["sampling_rate"]
    ext = make(feature, cfg, kernel="fast")
    assert ext.engine.kernel == "fast" and ext.plan.N == 1024
    gen = make(feature, cfg, kernel="generic")
    rs = np.random.RandomState(10)
    S, L = ext.plan.S, ext.plan.L
    lens = [L, L + 1, 10 * S - 1, 10 * S + S // 2, 10 * S + S // 2 - 1, 22050, 24003, 60000, 333 * S]
    xs = [(0.1 * rs.randn(m)).astype(np.float32) for m in lens]
    xs[3][: len(xs[3]) // 2] *= 1e-4
    got = ext.extract_batch(xs, sr)
    ocfg = oracle_cfg(feature, cfg)
    for x, g in zip(xs, got):
        ref = O.extract(x, ocfg)
        truth = O.extract(x, ocfg, dtype=torch.float64)
        assert g.shape == ref.shape
        ok, msg = gate(g, ref, truth, feature, cfg.get("use_energy", False), cfg.get("use_fft_mag", False))
        assert ok, msg
    for a, b_ in zip(got, gen.extract_batch(xs, sr)):
        np.testing.assert_allclose(a, b_, rtol=2e-4, atol=5e-4 if feature != "spectrogram" else 2e-3)
    if feature == "fbank" and not cfg.get("use_energy"):
        pcm = [np.clip(x * 32768, -32768, 32767).astype(np.int16) for x in xs]
        i16 = ext.extract_batch(pcm, sr)
        f32 = ext.extract_batch([q.astype(np.float32) / 32768.0 for q in pcm], sr)
        for a, b_ in zip(i16, f32):
            assert np.array_equal(a, b_)
        feats, flens = ext.extract_batch_padded([torch.from_numpy(x) for x in xs], sr)
        assert feats.shape[0] == len(xs) and flens.tolist() == [g.shape[0] for g in got]
        fcpu = feats.cpu().numpy()
        for i, g in enumerate(got):
            assert np.array_equal(fcpu[i, : g.shape[0]], g)
            assert np.all(fcpu[i, g.shape[0]:] == np.float32(LOG_EPSILON))


@pytest.mark.parametrize("variant", ["0", "3"])  # {11 warps, 2 frames per warp} and {14, 1}
@pytest.mark.parametrize("feature,cfg", [
    ("fbank", dict(sampling_rate=24000, frame_length=0.05)),                 # L = 1200, S = 240 (test_cut_consistency.py:77-105)
    ("fbank", dict(sampling_rate=44100)),                                    # L = 1102, S = 441 (odd: every other frame unaligned)
    ("fbank", dict(sampling_rate=48000, num_filters=128, use_energy=True)),  # L = 1200, S = 480
    ("fbank", dict(sampling_rate=48000, use_fft_mag=True, window_type="hanning", preemph_coeff=0.0, snip_edges=True)),
    ("mfcc", dict(sampling_rate=44100, num_ceps=20, num_filters=40)),
    ("mfcc", dict(sampling_rate=48000, use_energy=True)),
    ("spectrogram", dict(sampling_rate=44100)),
    ("log-spectrogram", dict(sampling_rate=48000, use_energy=True)),
    ("fbank", dict(sampling_rate=16000, frame_length=0.128, frame_shift=0.032)),  # L = N = 2048, S = 512
    ("fbank", dict(sampling_rate=32000, frame_length=0.05, raw_energy=False, use_energy=True)),  # L = 1600 (run-time length)
])
def test_fast2048_kernel_vs_oracle(feature, cfg, variant, monkeypatch):
    """The N = 2048 fast kernel (44.1 / 48 kHz with 25 ms frames, 24 kHz with 50 ms frames, every plan with 1024 < L <= 2048),
    two launch shapes, against the oracle and the generic kernel on ragged lengths, plus int16 staging and the padded mode."""
    monkeypatch.setenv("B200FEAT_FAST2048_VARIANT", variant)
    sr = cfg["sampling_rate"]
    ext = make(feature, cfg, kernel="fast")
    assert ext.engine.kernel == "fast" and ext.plan.N == 2048
    gen = make(feature, cfg, kernel="generic")
    rs = np.random.RandomState(11)
    S, L = ext.plan.S, ext.plan.L
    lens = [L, L + 1, 10 * S - 1, 10 * S + S // 2, 10 * S + S // 2 - 1, 44100, 48003, 120000, 333 * S]
    xs = [(0.1 * rs.randn(m)).astype(np.float32) for m in lens]
    xs[3][: len(xs[3]) // 2] *= 1e-4
    got = ext.extract_batch(xs, sr)
    ocfg = oracle_cfg(feature, cfg)
    for x, g in zip(xs, got):
        ref = O.extract(x, ocfg)
        truth = O.extract(x, ocfg, dtype=torch.float64)
        assert g.shape == ref.shape
        ok, msg = gate(g, ref, truth, feature, cfg.get("use_energy", False), cfg.get("use_fft_mag", False))
        assert ok, msg
    for a, b_ in zip(got, gen.extract_batch(xs, sr)):
        np.testing.assert_allclose(a, b_, rtol=2e-4, atol=5e-4 if feature != "spectrogram" else 4e-3)
    if feature == "fbank" and not cfg.get("use_energy"):
        pcm = [np.clip(x * 32768, -32768, 32767).astype(np.int16) for x in xs]
        i16 = ext.extract_batch(pcm, sr)
        f32 = ext.extract_batch([q.astype(np.float32) / 32768.0 for q in pcm], sr)
        for a, b_ in zip(i16, f32):
            assert np.array_equal(a, b_)
        feats, flens = ext.extract_batch_padded([torch.from_numpy(x) for x in xs], sr)
        assert feats.shape[0] == len(xs) and flens.tolist() == [g.shape[0] for g in got]
        fcpu = feats.cpu().numpy()
        for i, g in enumerate(got):
            assert np.array_equal(fcpu[i, : g.shape[0]], g)
            assert np.all(fcpu[i, g.shape[0]:] == np.float32(LOG_EPSILON))


from helpers import load_golden_stream  # noqa: E402

STREAM = load_golden_stream()


@pytest.mark.parametrize("i,m,x,y,r", STREAM, ids=[f"{i}-{m['feature']}" for i, m, _, _, _ in STREAM])
def test_streaming_online_inference(i, m, x, y, r):
    """`online_inference` (layers.py:199-224, :326-333, :775-857) on the GPU: per-call frame counts and the carried
    remainder exactly as the reference's streaming run, values within the gate, and — the reference's own property
    (test_kaldi_layers.py:199-235) — streaming plus one flipped tail chunk reproduces the offline frames."""
    ext = make(m["feature"], m["cfg"])
    sr = m["cfg"].get("sampling_rate", 16000)
    ocfg = oracle_cfg(m["feature"], m["cfg"])
    xb = torch.from_numpy(np.stack([x, 0.5 * x, x]))
    rem, feats, counts = None, [], []
    for a, b in zip(m["bounds"][:-1], m["bounds"][1:]):
        f, rem = ext.online_inference(xb[:, a:b], context=rem)
        assert f.is_cuda and f.dim() == 3 and f.shape[0] == 3
        feats.append(f)
        counts.append(f.shape[1])
    assert counts == m["counts"]
    assert np.array_equal(rem[0].cpu().numpy(), r)
    got = torch.cat(feats, dim=1).cpu().numpy()
    assert np.array_equal(got[0], got[2])  # batch rows are independent
    assert got[0].shape == y.shape
    # truth: the float64 oracle on the same streaming schedule
    rem64, t64 = None, []
    for a, b in zip(m["bounds"][:-1], m["bounds"][1:]):
        f64, rem64 = O.online_inference(x[a:b], ocfg, context=rem64, dtype=torch.float64)
        t64.append(f64)
    ok, msg = gate(got[0], y, np.concatenate(t64, axis=0), m["feature"], m["cfg"].get("use_energy", False),
                   m["cfg"].get("use_fft_mag", False))
    assert ok, msg
    S = ext.plan.S
    if not m["cfg"].get("snip_edges", False) and m["n"] % S == 0:
        tail, _ = ext.online_inference(torch.flip(xb[:, -S:], (1,)), context=rem)
        online = torch.cat(feats + [tail], dim=1).cpu().numpy()
        offline = ext.extract_batch(xb, sr)
        offline = offline.cpu().numpy() if isinstance(offline, torch.Tensor) else np.asarray(offline)
        assert online.shape == offline.shape
        # same frames, same arithmetic: the only difference is which load path (interior / edge) fetched the samples
        assert np.array_equal(online, offline)


@pytest.mark.parametrize("feature,cfg", [
    ("fbank", dict(round_to_power_of_two=False)),                                    # the "n_fft = 400" geometry
    ("fbank", dict(round_to_power_of_two=False, num_filters=40, use_energy=True)),
    ("fbank", dict(round_to_power_of_two=False, use_fft_mag=True, window_type="hamming", preemph_coeff=0.0, snip_edges=True)),
    ("fbank", dict(round_to_power_of_two=False, raw_energy=False, use_energy=True, remove_dc_offset=False)),
    ("mfcc", dict(round_to_power_of_two=False)),
    ("mfcc", dict(round_to_power_of_two=False, use_energy=True, num_ceps=10)),
    ("spectrogram", dict(round_to_power_of_two=False)),
    ("log-spectrogram", dict(round_to_power_of_two=False, use_energy=True)),
])
def test_fast400_kernel_vs_oracle(feature, cfg):
    """The N = L = 400 prime-factor kernel (round_to_power_of_two=False at 16 kHz) against the oracle and the generic
    kernel on ragged lengths that hit the frame-count edges, plus int16 staging and the padded output mode."""
    sr = 16000
    ext = make(feature, cfg, kernel="fast")
    assert ext.engine.kernel == "fast" and ext.plan.N == 400 and ext.plan.L == 400
    gen = make(feature, cfg, kernel="generic")
    rs = np.random.RandomState(11)
    S, L = ext.plan.S, ext.plan.L
    lens = [L, L + 1, 10 * S - 1, 10 * S + S // 2, 10 * S + S // 2 - 1, 16000, 16003, 40000, 333 * S, 57 * 2 * S]
    xs = [(0.1 * rs.randn(m)).astype(np.float32) for m in lens]
    xs[3][: len(xs[3]) // 2] *= 1e-4
    xs[5] += 0.3  # DC offset
    got = ext.extract_batch(xs, sr)
    ocfg = oracle_cfg(feature, cfg)
    for x, g in zip(xs, got):
        ref = O.extract(x, ocfg)
        truth = O.extract(x, ocfg, dtype=torch.float64)
        assert g.shape == ref.shape
        ok, msg = gate(g, ref, truth, feature, cfg.get("use_energy", False), cfg.get("use_fft_mag", False))
        assert ok, msg
    for a, b_ in zip(got, gen.extract_batch(xs, sr)):
        np.testing.assert_allclose(a, b_, rtol=2e-4, atol=5e-4 if feature != "spectrogram" else 2e-3)
    again = ext.extract_batch(xs, sr)
    for a, b_ in zip(got, again):
        assert np.array_equal(a, b_)  # deterministic
    if feature == "fbank" and not cfg.get("use_energy"):
        pcm = [np.clip(x * 32768, -32768, 32767).astype(np.int16) for x in xs]
        i16 = ext.extract_batch(pcm, sr)
        f32 = ext.extract_batch([q.astype(np.float32) / 32768.0 for q in pcm], sr)
        for a, b_ in zip(i16, f32):
            assert np.array_equal(a, b_)
        feats, flens = ext.extract_batch_padded([torch.from_numpy(x) for x in xs], sr)
        assert feats.shape[0] == len(xs) and flens.tolist() == [g.shape[0] for g in got]
        fcpu = feats.cpu().numpy()
        for i, g in enumerate(got):
            assert np.array_equal(fcpu[i, : g.shape[0]], g)
            assert np.all(fcpu[i, g.shape[0]:] == np.float32(LOG_EPSILON))


def _fuzz_cases():
    rs = np.random.RandomState(2024)
    cases = []
    geoms = [(16000, 0.025, 0.01, True), (16000, 0.025, 0.01, False), (8000, 0.025, 0.01, True), (24000, 0.025, 0.01, True),
             (22050, 0.025, 0.01, True), (16000, 0.02, 0.01, True), (16000, 0.032, 0.016, True), (44100, 0.02, 0.01, True),
             (16000, 0.05, 0.0125, True), (8000, 0.032, 0.008, True)]
    for i in range(24):
        sr, fl, fs, pow2 = geoms[rs.randint(len(geoms))]
        feature = ["fbank", "fbank", "mfcc", "spectrogram", "log-spectrogram"][rs.randint(5)]
        cfg = dict(sampling_rate=sr, frame_length=fl, frame_shift=fs, round_to_power_of_two=pow2,
                   window_type=["povey", "hanning", "hamming", "rectangular", "blackman"][rs.randint(5)],
                   preemph_coeff=[0.97, 0.0, 0.5][rs.randint(3)], remove_dc_offset=bool(rs.randint(2)),
                   snip_edges=bool(rs.randint(4) == 0), use_energy=bool(rs.randint(3) == 0), raw_energy=bool(rs.randint(2)),
                   use_fft_mag=bool(rs.randint(4) == 0))
        if feature in ("fbank", "mfcc"):
            cfg.update(num_filters=int([4, 5, 23, 40, 80, 128][rs.randint(6)]), low_freq=float([20.0, 0.0, 100.0][rs.randint(3)]),
                       high_freq=float([-400.0, 0.0, -1000.0][rs.randint(3)]))
        if feature == "mfcc":
            cfg.update(num_ceps=int(min(cfg["num_filters"], [13, 20, 2][rs.randint(3)])), cepstral_lifter=int([22, 10][rs.randint(2)]))
        cases.append((i, feature, cfg))
    return cases


@pytest.mark.parametrize("i,feature,cfg", _fuzz_cases(), ids=[f"{i}-{f}" for i, f, _ in _fuzz_cases()])
def test_random_configs_auto_kernel_vs_oracle(i, feature, cfg):
    """Seeded random walk over the config space (geometry, window, flags, mel bank shape) through AUTO kernel selection —
    whichever kernel the plan lands on, and the generic kernel, must agree with the oracle and with each other."""
    sr = cfg["sampling_rate"]
    ext = make(feature, cfg)
    rs = np.random.RandomState(100 + i)
    S, L = ext.plan.S, ext.plan.L
    lens = [L + 3 * S, 17 * S + 5, 40 * S + S // 2, 123 * S]
    xs = [(0.1 * rs.randn(m)).astype(np.float32) for m in lens]
    xs[1] += 0.05
    ocfg = oracle_cfg(feature, cfg)
    outs = {}
    for kern in kernels_for(ext):
        e = make(feature, cfg, kernel=kern)
        got = e.extract_batch(xs, sr)
        outs[kern] = got
        for x, g in zip(xs, got):
            ref = O.extract(x, ocfg)
            truth = O.extract(x, ocfg, dtype=torch.float64)
            assert g.shape == ref.shape, (kern, g.shape, ref.shape)
            ok, msg = gate(g, ref, truth, feature, cfg["use_energy"], cfg["use_fft_mag"])
            assert ok, f"{kern}: {msg}"


def test_tensor_core_kernel_at_headline_size():
    """kernel="tc" (wgmma two-stage DFT, csrc/tc512.cuh) on BASELINE configs[1] inputs: against the register-FFT kernel
    (two independent CUDA implementations of layers.py:151-186, :32-42, :565-578) and against the oracle on a sample of cuts;
    deterministic, cuts independent, padded mode and MFCC epilogue included."""
    torch.manual_seed(0)
    B, n = 64, 160000
    x = (0.1 * torch.randn(B, n)).cuda()
    tc, fast = make("fbank", {}, kernel="tc"), make("fbank", {}, kernel="fast")
    assert tc.engine.kernel == "tc" and fast.engine.kernel == "fast"
    y = tc.extract_batch(x, 16000)
    assert y.shape == (B, 1000, 80) and torch.isfinite(y).all()
    assert torch.equal(y, tc.extract_batch(x, 16000))
    perm = torch.randperm(B).cuda()
    assert torch.equal(tc.extract_batch(x[perm], 16000), y[perm])
    yf = fast.extract_batch(x, 16000)
    assert torch.allclose(y, yf, rtol=1e-4, atol=5e-4), float((y - yf).abs().max())
    cfg = O.OracleConfig()
    for b in (0, 17, 63):
        xb = x[b].cpu().numpy()
        ok, msg = gate(y[b].cpu().numpy(), O.extract(xb, cfg), O.extract(xb, cfg, dtype=torch.float64), "fbank")
        assert ok, msg
    # ragged + padded collation in one launch
    lens = [16000, 159, 48000, 1599, 20001]
    xs = [x[i, :m].contiguous() for i, m in enumerate(lens)]
    feats, flens = tc.extract_batch_padded(xs, 16000)
    assert flens.tolist() == [(m + 80) // 160 for m in lens]
    ref, _ = fast.extract_batch_padded(xs, 16000)
    for i, T in enumerate(flens.tolist()):
        assert torch.allclose(feats[i, :T], ref[i, :T], rtol=1e-4, atol=5e-4)
        assert torch.all(feats[i, T:] == LOG_EPSILON)
    # MFCC epilogue
    m_tc, m_fast = make("mfcc", dict(num_ceps=13, num_mel_bins=23), kernel="tc"), make("mfcc", dict(num_ceps=13, num_mel_bins=23), kernel="fast")
    a, b_ = m_tc.extract_batch(x[:8], 16000), m_fast.extract_batch(x[:8], 16000)
    assert a.shape == (8, 1000, 13) and torch.allclose(a, b_, rtol=1e-3, atol=3e-4)


@pytest.mark.parametrize("kernel", ["generic", "fast", "tc"])
def test_views_with_a_storage_offset(kernel):
    """ADVICE r1: `wave[1:]` is contiguous, so its data pointer is misaligned for the vector loads; the engine must not fault."""
    rs = np.random.RandomState(9)
    full = torch.from_numpy((0.1 * rs.randn(32001)).astype(np.float32)).cuda()
    ext = make("fbank", {}, kernel=kernel)
    for off in (1, 2, 3):
        view = full[off:]
        got = ext.extract(view, 16000)
        want = ext.extract(view.clone(), 16000)
        assert torch.equal(got, want)
    pcm = (full * 20000).to(torch.int16)
    assert torch.equal(ext.extract(pcm[1:], 16000), ext.extract(pcm[1:].clone(), 16000))
