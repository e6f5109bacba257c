"""WPE dereverberation on the GPU (csrc/wpe.cuh): `engine.wpe` against the float64 restatement within the bound lhotse's own
float32 chain sets, at the edges (lengths, the frame cap, silence, zero and non-finite cuts, grid sizes, parameters);
run-to-run and batch independence; B200DereverbWPE; the "transform" route with `wpe=True` (samples and features, alone,
after speed perturbation and a reverb, inside K2SpeechRecognitionDataset) and the argument checks of b200feat_wpe."""
import numpy as np
import pytest
import torch

import refshim
import wpe_cases as WC

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ref():
    if not refshim.reference_available():
        pytest.skip("no reference tree / oracle/_ref archive")
    refshim.import_reference()
    WC.install_nara_wpe_standin()


def _check(xs, outs, targets=None, **p):
    for i, (x, o) in enumerate(zip(xs, outs)):
        t = None if targets is None else targets[i]
        ok, err, lim = WC.bound(o, WC.truth64(x, t, **p), WC.lhotse32(x, t, **p))
        assert ok, (i, len(x), err, lim)


def test_gpu_wpe_signals_and_lengths_within_bound(ref):
    """Noise, reverberant bursts, leading silence and full scale, at L mod 128 in {0, 1, 127}, the shortest cut (1536),
    trimmed and reflect-padded targets."""
    xs, targets = [], []
    for k, kind in enumerate(("noise", "reverb", "silence", "full")):
        for n in (16000 * 3, 16000 * 3 + 1, 16000 * 3 + 127, 1536):
            xs.append(WC.signal(kind, n, seed=k))
            lz = 128 * (n // 128)
            targets.append({0: lz, 1: lz - 37, 2: lz + 127, 3: lz + 1}[len(xs) % 4])
    outs, host = WC.run_wpe(xs, targets)
    _check(xs, outs, targets)
    assert np.all(np.isfinite(host))
    ends = np.cumsum([t + 3 for t in targets])
    for e in ends:  # the 3 samples after every window keep the sentinel
        assert np.all(host[e - 3: e] == np.float32(-7.25))


def test_gpu_wpe_parameters_within_bound(ref):
    xs = [WC.signal("reverb", 16000 * 2 + 55, seed=3), WC.signal("silence", 16000 * 2, seed=4)]
    for p in (dict(statistics_mode="valid"), dict(taps=1, delay=0), dict(taps=16, delay=5, iterations=1),
              dict(taps=4, delay=1, iterations=5), dict(iterations=0)):
        outs, _ = WC.run_wpe(xs, **p)
        _check(xs, outs, **p)


def test_gpu_wpe_zero_cut_nan_cut_and_batch_independence(ref):
    """An all-zero cut gives exact zeros; a NaN sample in one cut leaves the others bitwise as they are alone; two runs are
    bitwise equal."""
    base = [WC.signal("reverb", 16000 * 4 + 9, seed=5), WC.signal("noise", 40000, seed=6), WC.signal("zero", 20000)]
    bad = WC.signal("noise", 30000, seed=7)
    bad[12345] = np.nan
    a, _ = WC.run_wpe(base)
    b, _ = WC.run_wpe([base[0], bad, base[1], base[2]])
    c, _ = WC.run_wpe([base[0], bad, base[1], base[2]])
    assert np.array_equal(a[0].view(np.int32), b[0].view(np.int32)) and np.array_equal(a[1].view(np.int32), b[2].view(np.int32))
    assert np.array_equal(a[2], np.zeros_like(a[2])) and np.array_equal(b[3].view(np.int32), np.zeros(len(b[3]), np.int32))
    for u, v in zip(b, c):
        assert np.array_equal(u.view(np.int32), v.view(np.int32))
    for i, x in enumerate(base):
        alone, _ = WC.run_wpe([x])
        assert np.array_equal(alone[0].view(np.int32), a[i].view(np.int32))


def test_gpu_wpe_frame_cap_and_short_cuts(ref):
    """The cap: L = 128 * 8192 - 1 (8192 frames) is taken, one more sample is refused; L = 1535 (12 frames < taps + delay)
    and L = 256 are refused as too short."""
    from lhotse_b200.engine import B200FeatError, WPE_MAX_FRAMES

    n = 128 * WPE_MAX_FRAMES - 1
    x = WC.signal("reverb", n, seed=8)
    outs, _ = WC.run_wpe([x])
    _check([x], outs)
    for bad, code in ((n + 1, -1), (1535, -5), (256, -5)):
        with pytest.raises(B200FeatError) as e:
            WC.run_wpe([WC.signal("noise", bad)])
        assert e.value.code == code, (bad, e.value)


def test_gpu_wpe_grids_past_65535_ctas(ref):
    """300 cuts: 77100 per-bin CTAs; and one batch with more than 65535 STFT and iSTFT CTAs.  Cuts equal their solo runs bit
    for bit."""
    rs = np.random.RandomState(9)
    xs = [WC.signal("noise", int(n), seed=i) for i, n in enumerate(rs.randint(1536, 6000, size=300))]
    outs, _ = WC.run_wpe(xs)
    for i in (0, 137, 299):
        alone, _ = WC.run_wpe([xs[i]])
        assert np.array_equal(alone[0].view(np.int32), outs[i].view(np.int32))
    _check([xs[0], xs[299]], [outs[0], outs[299]])
    big = [WC.signal("noise", 128 * 8000, seed=100 + i) for i in range(264)]  # 264 * 250 STFT CTAs, 264 * 276 iSTFT CTAs
    outs, _ = WC.run_wpe(big)
    alone, _ = WC.run_wpe([big[-1]])
    assert np.array_equal(alone[0].view(np.int32), outs[-1].view(np.int32))


def test_gpu_wpe_argument_checks(ref):
    from lhotse_b200.engine import B200FeatError

    x = [WC.signal("noise", 4000)]
    for p, code in ((dict(n_fft=400), -2), (dict(hop_length=160), -2), (dict(taps=0), -1), (dict(taps=17), -1),
                    (dict(delay=-1), -1), (dict(iterations=65), -1)):
        with pytest.raises(B200FeatError) as e:
            WC.run_wpe(x, **p)
        assert e.value.code == code, (p, e.value)
    with pytest.raises(ValueError):
        WC.run_wpe(x, statistics_mode="other")
    with pytest.raises(B200FeatError):  # reflect padding longer than the signal
        WC.run_wpe(x, targets=[2 * 3968])
    # an output window over an input window
    from lhotse_b200.engine import WPE_CUT_DTYPE, wpe

    buf = torch.zeros(20000, device="cuda:0")
    ct = np.zeros(1, WPE_CUT_DTYPE)
    ct["struct_size"], ct["in_elem"], ct["in_len"], ct["out_elem"], ct["target_len"] = WPE_CUT_DTYPE.itemsize, 0, 8000, 7999, 7936
    with pytest.raises(B200FeatError, match="overlaps"):
        wpe(buf, ct, buf)
    ct["out_elem"] = 8000
    wpe(buf, ct, buf)


def test_gpu_b200_dereverb_wpe_module(ref):
    """B200DereverbWPE against the restatement row by row, padding included; lhotse's module on the same batch (wpe_v6 on
    the stand-in) sets the bound; 3-D input and inputs that require grad raise."""
    import importlib

    from lhotse.dataset.signal_transforms import DereverbWPE

    import lhotse_b200.dereverb as D

    B200DereverbWPE = importlib.reload(D).B200DereverbWPE  # bound to lhotse's class now that the reference is imported
    rows = [WC.signal("reverb", 30000, seed=11), WC.signal("silence", 30000, seed=12), WC.signal("noise", 30000, seed=13)]
    rows[2][20000:] = 0.0  # padding
    x = torch.from_numpy(np.stack(rows))
    mod = B200DereverbWPE()
    assert isinstance(mod, DereverbWPE)
    got = mod(x.cuda())
    assert got.shape == (3, 128 * (30000 // 128)) and got.device.type == "cuda"
    theirs = DereverbWPE()(x)
    for i in range(3):
        ok, err, lim = WC.bound(got[i].cpu().numpy(), WC.truth64(rows[i]), theirs[i].numpy())
        assert ok, (i, err, lim)
    assert mod(x).device.type == "cpu"
    with pytest.raises(NotImplementedError):
        mod(x[:, None, :])
    with pytest.raises(RuntimeError):
        mod(x.clone().requires_grad_(True))
    with torch.no_grad():
        mod(x.clone().requires_grad_(True))


@pytest.fixture(scope="module")
def env(tmp_path_factory, ref):
    import lhotse_env
    import test_reverb
    import transform_cases

    lb_ex = lhotse_env.setup_lhotse()
    root = tmp_path_factory.mktemp("gwpe")
    speech, rirs = test_reverb.make_sources(root)
    with transform_cases.torch_resampler():
        yield lb_ex, speech, rirs, root


def _pre_wpe(c) -> np.ndarray:
    """The float32 signal lhotse's DereverbWPE receives for a cut over a whole file: the file's samples through every
    transform of the chain but the last (lhotse's own transforms: the GPU's Speed / Volume / Resample are bit-identical to
    them)."""
    import wave

    from lhotse.augmentation.transform import AudioTransform

    rec = c.recording
    with wave.open(rec.sources[0].source) as w:
        x = (np.frombuffer(w.readframes(w.getnframes()), "<i2").astype(np.float32) / 32768.0)[None, :]
    for t in rec.transforms[:-1]:
        t = t if isinstance(t, AudioTransform) else AudioTransform.from_dict(t)
        x = t(x, rec.sampling_rate)
    return np.asarray(x, np.float32)[0]


def _truth(c) -> np.ndarray:
    return WC.truth64(_pre_wpe(c), c.num_samples)


def _frames(ext, cuts):
    return [int(ext.engine.plan.num_frames(np.asarray([c.num_samples]))[0]) for c in cuts]


def _gate(cuts, ours, float_route, frames):
    """Each cut's features (rows [0, T)) through helpers.gate against the float64 oracle on the float64 truth samples.  The
    gate's float32 reference is the float32 oracle on the truth samples rounded to float32: the float route's own features
    come from lhotse's complex64 WPE, 2-4 % of the peak off in samples, which the gate refuses as a reference (DESIGN.md
    §3.1q).  The float route's features only fix the frame counts here."""
    from helpers import gate
    from oracle import kaldi_oracle as O

    for i, c in enumerate(cuts):
        t = int(frames[i])
        x = _truth(c)
        truth = O.extract(x, O.OracleConfig(), dtype=torch.float64)
        ref32 = O.extract(x.astype(np.float32), O.OracleConfig())
        assert truth.shape[0] == t and float_route[i][:t].shape == ours[i][:t].shape, (c.id, truth.shape, t)
        ok, msg = gate(ours[i][:t].cpu().numpy(), ref32, truth, "fbank")
        assert ok, (c.id, msg)


def test_gpu_transform_cuts_wpe_within_bound(env):
    from lhotse_b200.pcm_staging import staged_route, transform_cuts

    _, speech, rirs, _ = env
    c0, c1, c2 = speech
    cuts = [c0.dereverb_wpe(), c1.perturb_speed(1.1).dereverb_wpe(), c2.perturb_volume(0.5).perturb_speed(0.9).dereverb_wpe(),
            c1]
    assert staged_route(cuts) is None and staged_route(cuts, wpe=True)[0] == "transform"
    out, lens, offs = transform_cuts(cuts, "cuda:0", wpe=True)
    host = out.cpu().numpy()
    for c, n, o in zip(cuts, lens, offs):
        got = host[o: o + n]
        assert n == c.num_samples
        if not c.recording.transforms:
            assert np.array_equal(got, np.asarray(c.load_audio(), np.float32)[0])
            continue
        x = _pre_wpe(c)
        ok, err, lim = WC.bound(got, WC.truth64(x, n), WC.lhotse32(x, n))
        assert ok, (c.id, err, lim)
        assert np.abs(got - np.asarray(c.load_audio(), np.float64)[0]).max() <= lim  # lhotse's own load_audio on the stand-in
    again, _, _ = transform_cuts(cuts, "cuda:0", wpe=True)
    assert torch.equal(out.view(torch.int32), again.view(torch.int32))


def test_gpu_fused_on_the_fly_and_audio_samples_wpe(env):
    from lhotse import CutSet

    from lhotse_b200.input_strategies import FusedAudioSamples, FusedOnTheFlyFeatures

    lb_ex, speech, rirs, _ = env
    ext = lb_ex.B200Fbank(lb_ex.B200FbankConfig(device="cuda:0"))
    c0, c1, c2 = speech
    batch = [c0.dereverb_wpe(), c1.perturb_speed(1.1).dereverb_wpe(), c2.reverb_rir(rirs["rir_short"]).dereverb_wpe()]
    cs = CutSet.from_cuts(batch)
    on, off, flt = (FusedOnTheFlyFeatures(ext, wpe=True, reverb=True), FusedOnTheFlyFeatures(ext, reverb=True),
                    FusedOnTheFlyFeatures(ext, pcm16_fast_path=False))
    f1, l1 = on(cs)
    f2, l2 = off(cs)
    f3, l3 = flt(cs)
    assert on.last_batch_route == "transform" and off.last_batch_route == "float" and flt.last_batch_route == "float"
    assert torch.equal(f2, f3) and torch.equal(l1, l3)  # wpe=False: exactly the float route
    _gate(batch[:2], f1[:2], f3[:2], l1[:2])
    _gate(batch[2:], f1[2:], f3[2:], l1[2:])  # the reverb ahead of WPE is held to its own tolerance (DESIGN.md §3.1j)
    a_on, a_off = FusedAudioSamples(wpe=True, reverb=True), FusedAudioSamples()
    x1, n1 = a_on(cs)
    x2, n2 = a_off(cs)
    assert a_on.last_batch_route == "transform" and a_off.last_batch_route == "reference" and torch.equal(n1.cpu(), n2.cpu())
    for i, c in enumerate(batch[:2]):
        x = _pre_wpe(c)
        ok, err, lim = WC.bound(x1[i, : n1[i]].cpu().numpy(), WC.truth64(x, c.num_samples), WC.lhotse32(x, c.num_samples))
        assert ok, (c.id, err, lim)


def test_gpu_wpe_in_k2_dataset_within_gate(env, tmp_path):
    """cuts.dereverb_wpe() alone and after perturb_speed and a recorded-RIR reverb, under DynamicBucketingSampler in
    K2SpeechRecognitionDataset: every batch stays on "transform"; the features pass the gate."""
    import lhotse_env
    from lhotse.dataset import DynamicBucketingSampler, K2SpeechRecognitionDataset
    from lhotse.dataset.input_strategies import OnTheFlyFeatures

    from lhotse_b200.input_strategies import FusedOnTheFlyFeatures

    lb_ex, _, rirs, _ = env
    rs = np.random.RandomState(0)
    base = lhotse_env.make_cutset(tmp_path, np.round(rs.uniform(2.0, 8.0, size=8), 2).tolist(), seed=3)
    sets = {"alone": base.dereverb_wpe(),
            "chain": (base.perturb_speed(1.1) + base).map(lambda c: c.reverb_rir(rirs["rir_long"])).dereverb_wpe()}
    ext = lb_ex.B200Fbank(lb_ex.B200FbankConfig(device="cuda:0"))
    for label, cuts in sets.items():
        got, routes = {}, []
        for name, strategy in (("reference", OnTheFlyFeatures(ext)), ("fused", FusedOnTheFlyFeatures(ext, reverb=True, wpe=True))):
            sampler = DynamicBucketingSampler(cuts, max_duration=20.0, num_buckets=2, shuffle=True, seed=0)
            ds = K2SpeechRecognitionDataset(input_strategy=strategy, return_cuts=True)
            out = []
            for batch_cuts in sampler:
                b = ds[batch_cuts]
                out.append((b["inputs"].cpu(), b["supervisions"]["num_frames"].clone(), list(b["supervisions"]["cut"])))
                if name == "fused":
                    routes.append(strategy.last_batch_route)
            got[name] = out
        assert routes and set(routes) == {"transform"}, (label, routes)
        for (x1, n1, c1), (x2, n2, c2) in zip(got["reference"], got["fused"]):
            assert [c.id for c in c1] == [c.id for c in c2] and torch.equal(n1, n2)
            _gate(c2, x2, x1, _frames(ext, c2))
