"""GPU reverb on the CPU: the partitioned FFT convolution, shift, gain and length fix of csrc/reverb.cuh run on the host
(scripts/micro/reverb_host_check.cu, under AddressSanitizer where the toolchain has it) against a float64 convolution, within
the bound lhotse's own float32 arithmetic sets; and which reverberated lhotse cuts the transform and mix routes take."""
import os
import shutil
import subprocess

import numpy as np
import pytest

import refshim
import reverb_cases as RC

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
needs_ref = pytest.mark.skipif(not refshim.reference_available(), reason="reference tree not present")
B = 2048  # csrc/reverb.cuh RV_B
CAP = 65536


@pytest.fixture(scope="module")
def harness(tmp_path_factory):
    d = tmp_path_factory.mktemp("rvh")
    src = os.path.join(ROOT, "scripts", "micro", "reverb_host_check.cu")
    exe = str(d / "reverb_host_check")
    gxx = shutil.which("g++")
    if gxx:
        for flags in (["-fsanitize=address", "-fno-omit-frame-pointer"], []):
            res = subprocess.run([gxx, "-x", "c++", "-std=c++17", "-O1", "-g", *flags, "-o", exe, src], capture_output=True, text=True)
            if res.returncode == 0:
                return exe
    pytest.skip("no host C++ compiler")


def run_harness(exe, tmp_path, rirs, cuts):
    """rirs: [int16 array]; cuts: [(float32 x, rir index, normalize, target_len)] -> [float32 output per cut]."""
    from lhotse_b200.engine import REVERB_CUT_DTYPE, REVERB_RIR_DTYPE

    rt = np.zeros(len(rirs), REVERB_RIR_DTYPE)
    rt["struct_size"] = REVERB_RIR_DTYPE.itemsize
    rt["num_samples"] = [len(q) for q in rirs]
    rt["src_elem"] = np.concatenate(([0], np.cumsum([len(q) for q in rirs])[:-1]))
    ct = np.zeros(len(cuts), REVERB_CUT_DTYPE)
    ct["struct_size"] = REVERB_CUT_DTYPE.itemsize
    ct["rir"] = [c[1] for c in cuts]
    ct["normalize"] = [int(c[2]) for c in cuts]
    ct["in_len"] = [len(c[0]) for c in cuts]
    ct["in_elem"] = np.concatenate(([0], np.cumsum([len(c[0]) for c in cuts])[:-1]))
    ct["target_len"] = [c[3] for c in cuts]
    np.concatenate(rirs).astype(np.int16).tofile(tmp_path / "s0.i16")
    rt.tofile(tmp_path / "rirs.bin")
    ct.tofile(tmp_path / "cuts.bin")
    np.concatenate([c[0] for c in cuts]).astype(np.float32).tofile(tmp_path / "in.f32")
    env = dict(os.environ, ASAN_OPTIONS="detect_leaks=0:abort_on_error=0")
    r = subprocess.run([exe, *(str(tmp_path / f) for f in ("s0.i16", "rirs.bin", "cuts.bin", "in.f32", "out.f32"))],
                       capture_output=True, text=True, env=env)
    assert r.returncode == 0 and "AddressSanitizer" not in r.stderr, r.stdout[-2000:] + r.stderr[-4000:]
    out = np.fromfile(tmp_path / "out.f32", np.float32)
    ends = np.cumsum([c[3] for c in cuts])
    return [out[e - c[3]: e] for e, c in zip(ends, cuts)]


def _cases():
    Rs = [1, 2, 800, B - 1, B, B + 1, 16000, CAP]
    cases = []
    for i, R in enumerate(Rs):
        for j, N in enumerate([1, max(1, R - 1), 160000, 160001]):
            peak = [0, R // 2, R - 1][(i + j) % 3]
            cases.append((R, N, peak, (i + j) % 2 == 0))
    return cases


@needs_ref
def test_host_reverb_within_float32_bound(harness, tmp_path):
    refshim.import_reference()
    rs = np.random.RandomState(7)
    rirs, cuts, meta = [], [], []
    for k, (R, N, peak, norm) in enumerate(_cases()):
        rirs.append(RC.decaying_rir(R, seed=k, peak_at=peak))
        x = (rs.randn(N) * 0.1).astype(np.float32)
        cuts.append((x, k, norm, N))
        meta.append(f"R={R} N={N} peak={peak} normalize={norm}")
    # length fixes: trimmed by 3, reflect-padded by 5 (what assert_and_maybe_fix_num_samples does after the reverb)
    x = (rs.randn(50000) * 0.1).astype(np.float32)
    cuts += [(x, 6, True, 49997), (x, 6, True, 50005), (x, 3, False, 50005)]
    meta += ["trim", "reflect", "reflect no-normalize"]
    # silence: exact zeros, no gain
    cuts.append((np.zeros(30000, np.float32), 6, True, 30000))
    got = run_harness(harness, tmp_path, rirs, cuts)
    for (x, r, norm, target), g, what in zip(cuts[:-1], got[:-1], meta[:-1]):
        q = rirs[r]
        RC.check(g, RC.truth64(x, q, norm, target), RC.lhotse32(x, q, norm, target), what)
    assert np.array_equal(got[-1].view(np.int32), np.zeros(30000, np.int32))


def test_host_reverb_shift_is_first_maximum(harness, tmp_path):
    """An impulse at 0 convolved with an RIR whose maximum appears twice: the output starts at the first one."""
    q = np.zeros(3000, np.int16)
    q[[0, 700, 2500]] = [100, 20000, 20000]
    x = np.zeros(6000, np.float32)
    x[0] = 1.0
    (y,) = run_harness(harness, tmp_path, [q], [(x, 0, False, 6000)])
    h = q.astype(np.float32) / np.float32(32768) * np.float32(0.5 ** 15)
    want = np.zeros(6000, np.float64)
    want[: 3000 - 700] = h[700:]
    assert np.abs(y - want).max() <= 1e-6 * np.abs(want).max()


# ---- eligibility on real lhotse cuts ------------------------------------------------------------------------------


@pytest.fixture(scope="module")
def lhotse_rvb(tmp_path_factory):
    if not refshim.reference_available():
        pytest.skip("reference tree not present")
    import lhotse_env

    lhotse_env.setup_lhotse()
    root = tmp_path_factory.mktemp("rvcuts")
    return root, make_sources(root)


def make_sources(root):
    """Speech cuts and RIR recordings (mono 0.3 s, mono 1 s, stereo 0.5 s, one longer than the cap) as 16-bit WAV files."""
    import lhotse_env
    from lhotse import Recording
    from lhotse.audio import AudioSource

    speech = lhotse_env.make_cutset(root, [3.0, 2.5, 4.0], seed=11)
    rirs = {}
    for name, n, ch, sr in (("rir_short", 4800, 1, 16000), ("rir_long", 16000, 1, 16000), ("rir_stereo", 8000, 2, 16000),
                            ("rir_huge", CAP + 1, 1, 16000), ("rir_8k", 2400, 1, 8000)):
        path = root / f"{name}.wav"
        RC.write_wav(path, RC.decaying_rir(n, seed=n, channels=ch), sr)
        rirs[name] = Recording(id=name, sources=[AudioSource(type="file", channels=list(range(ch)), source=str(path))],
                               sampling_rate=sr, num_samples=n, duration=n / sr)
    return list(speech), rirs


@needs_ref
def test_transform_route_takes_reverberated_cuts(lhotse_rvb):
    import transform_cases as T

    from lhotse_b200.pcm_staging import transform_request_for_cut, transform_requests_for_batch

    from lhotse.augmentation.rir import ReverbWithImpulseResponse
    from lhotse.utils import fastcopy

    _, (speech, rirs) = lhotse_rvb
    c = speech[0]
    with T.torch_resampler():
        r = transform_request_for_cut(c.reverb_rir(rirs["rir_short"]), reverb=True)
        assert r is not None and r.ops == () and r.reverb.normalize and r.reverb.rir.num_samples == 4800
        assert r.source.num_samples == r.num_samples == c.num_samples
        sp = transform_request_for_cut(c.perturb_speed(1.1).reverb_rir(rirs["rir_long"], normalize_output=False), reverb=True)
        assert sp is not None and sp.ops == (("resample", 17600, 16000),) and not sp.reverb.normalize
        early = transform_request_for_cut(c.reverb_rir(rirs["rir_long"], early_only=True), reverb=True)
        assert early.reverb.rir.num_samples == 800
        st = transform_request_for_cut(c.reverb_rir(rirs["rir_stereo"], rir_channels=[1]), reverb=True)
        assert st is not None and st.reverb.rir.channel == 1 and st.reverb.rir.num_samples == 8000
        # declines: lhotse's float route keeps them
        refused = {
            "generator": c.reverb_rir(),
            "too_long": c.reverb_rir(rirs["rir_huge"]),
            "reverb_not_last": c.reverb_rir(rirs["rir_short"]).perturb_speed(1.1),
            "two_reverbs": c.reverb_rir(rirs["rir_short"]).reverb_rir(rirs["rir_long"]),
            # lhotse's reverb_rir asserts equal rates; a manifest can still carry such a transform
            "rir_at_another_rate": fastcopy(c, recording=fastcopy(c.recording, transforms=[
                ReverbWithImpulseResponse(rir=rirs["rir_8k"]).to_dict()])),
            "rir_not_16bit_wav_or_flac": c.reverb_rir(fastcopy(rirs["rir_short"], sources=[
                fastcopy(rirs["rir_short"].sources[0], source=rirs["rir_short"].sources[0].source[:-4] + ".opus")])),
            "rir_with_transforms": c.reverb_rir(rirs["rir_short"].perturb_volume(2.0)),
        }
        for name, cut in refused.items():
            assert transform_request_for_cut(cut, reverb=True) is None, name
        # two RIR channels make a MultiCut: not a MonoCut the route takes
        assert transform_request_for_cut(c.reverb_rir(rirs["rir_stereo"], rir_channels=[0, 1]), reverb=True) is None
        # reverb=False (the default): exactly what the route returned before it knew about reverb
        for cut in (c.reverb_rir(rirs["rir_short"]), c.perturb_speed(1.1).reverb_rir(rirs["rir_long"])):
            assert transform_request_for_cut(cut) is None
            assert transform_requests_for_batch([speech[1], cut]) is None
        assert transform_requests_for_batch([speech[1], c.reverb_rir(rirs["rir_short"])], reverb=True) is not None
        # several sampling rates in one batch: the staged batch has no single rate, the callers keep the float route
        s8 = c.resample(8000).reverb_rir(rirs["rir_8k"])
        reqs = transform_requests_for_batch([c.reverb_rir(rirs["rir_short"]), s8], reverb=True)
        from lhotse_b200.pcm_staging import TransformStagingRing
        assert reqs is not None and TransformStagingRing(pin_memory=False).stage(reqs)[3] is None
        plain = transform_request_for_cut(c.perturb_speed(0.9))
        assert plain == transform_request_for_cut(c.perturb_speed(0.9), reverb=True) and plain.reverb is None


@needs_ref
def test_mix_route_takes_mixedcut_level_reverb(lhotse_rvb):
    from lhotse_b200.pcm_staging import mix_request_for_cut, mix_requests_for_batch

    _, (speech, rirs) = lhotse_rvb
    m = speech[0].mix(speech[1], snr=10, allow_padding=True)
    rv = m.reverb_rir(rirs["rir_short"])
    assert mix_request_for_cut(rv) is None  # the default keeps the float route
    r = mix_request_for_cut(rv, reverb=True)
    assert r is not None and r.reverb is not None and r.reverb.rir.num_samples == 4800
    base = mix_request_for_cut(m, reverb=True)
    assert repr(base) == repr(mix_request_for_cut(m)) and base.reverb is None  # repr: NaN SNR factors compare unequal
    assert repr(r.tracks) == repr(base.tracks) and r.num_samples == base.num_samples
    # per-track reverb (mix_first=False) stays refused, with or without perturbed tracks
    per_track = m.reverb_rir(rirs["rir_short"], mix_first=False)
    assert mix_request_for_cut(per_track, reverb=True) is None
    assert mix_request_for_cut(per_track, perturbed_tracks=True, reverb=True) is None
    # MixedCut-level transforms other than a single reverb
    assert mix_request_for_cut(rv.reverb_rir(rirs["rir_long"]), reverb=True) is None
    assert mix_request_for_cut(m.reverb_rir(), reverb=True) is None  # the RIR generator
    from lhotse.augmentation.rir import ReverbWithImpulseResponse
    from lhotse.utils import fastcopy

    other_rate = fastcopy(m, transforms=[ReverbWithImpulseResponse(rir=rirs["rir_8k"])])
    assert mix_request_for_cut(other_rate, reverb=True) is None
    # an SNR-scaled first track makes a float64 mix, which lhotse reverberates in float64
    from lhotse.cut import MixedCut, MixTrack

    scaled = MixedCut(id="scaled_first", tracks=[MixTrack(cut=speech[1], snr=7.0), MixTrack(cut=speech[0], offset=0.2)])
    assert mix_request_for_cut(scaled, reverb=True) is not None
    assert mix_request_for_cut(scaled.reverb_rir(rirs["rir_short"]), reverb=True) is None
    # a batch with reverberated plain slices beside the MixedCut
    batch = [rv, speech[2].reverb_rir(rirs["rir_long"]), speech[1]]
    assert mix_requests_for_batch(batch) is None
    reqs = mix_requests_for_batch(batch, reverb=True)
    assert reqs is not None and reqs[1].reverb is not None and reqs[2].reverb is None
    # a speed-perturbed, then reverberated MonoCut beside a MixedCut (the recipe's perturb_speed + CutMix + reverb): with
    # perturbed_tracks its chain, reverb included, runs on the transform route into the track buffer
    import transform_cases as T

    from lhotse_b200.pcm_staging import TransformRequest

    with T.torch_resampler():
        sp = speech[2].perturb_speed(1.1).reverb_rir(rirs["rir_long"])
        assert mix_requests_for_batch([rv, sp], reverb=True) is None
        assert mix_requests_for_batch([rv, sp], perturbed_tracks=True) is None
        reqs = mix_requests_for_batch([rv, sp], perturbed_tracks=True, reverb=True)
        assert reqs is not None and reqs[1].reverb is None
        src = reqs[1].tracks[0].source
        assert isinstance(src, TransformRequest) and src.reverb is not None and src.ops == (("resample", 17600, 16000),)
