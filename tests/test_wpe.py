"""GPU WPE on the CPU: the per-bin statistics, solve and filter and the per-sample overlap-add and length fix of csrc/wpe.cuh run
on the host (scripts/micro/wpe_host_check.cu, under AddressSanitizer where the toolchain has it, with a direct DFT for the
FFTs) against the float64 restatement of oracle/wpe_oracle.py; and which `dereverb_wpe()` cuts the "transform" route takes."""
import os
import shutil
import subprocess

import numpy as np
import pytest

import refshim
import wpe_cases as WC
from oracle import wpe_oracle as W

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
needs_ref = pytest.mark.skipif(not refshim.reference_available(), reason="reference tree not present")


@pytest.fixture(scope="module")
def harness(tmp_path_factory):
    d = tmp_path_factory.mktemp("wpeh")
    src = os.path.join(ROOT, "scripts", "micro", "wpe_host_check.cu")
    exe = str(d / "wpe_host_check")
    gxx = shutil.which("g++")
    if gxx:
        for flags in (["-fsanitize=address", "-fno-omit-frame-pointer"], []):
            res = subprocess.run([gxx, "-x", "c++", "-std=c++17", "-O1", "-g", *flags, "-o", exe, src], capture_output=True, text=True)
            if res.returncode == 0:
                return exe
    pytest.skip("no host C++ compiler")


def run_harness(exe, tmp_path, xs, targets=None, taps=10, delay=3, iterations=3, statistics_mode="full"):
    from lhotse_b200.engine import WPE_CUT_DTYPE

    targets = [128 * (len(x) // 128) for x in xs] if targets is None else targets
    ct = np.zeros(len(xs), WPE_CUT_DTYPE)
    ct["struct_size"] = WPE_CUT_DTYPE.itemsize
    ct["in_len"] = [len(x) for x in xs]
    ct["in_elem"] = np.concatenate(([0], np.cumsum([len(x) for x in xs])[:-1]))
    ct["target_len"] = targets
    ct.tofile(tmp_path / "cuts.bin")
    np.concatenate(xs).astype(np.float32).tofile(tmp_path / "in.f32")
    W.window().tofile(tmp_path / "win.f32")
    env = dict(os.environ, ASAN_OPTIONS="detect_leaks=0:abort_on_error=0")
    args = [str(tmp_path / f) for f in ("cuts.bin", "in.f32", "win.f32", "out.f32")]
    args += [str(taps), str(delay), str(iterations), str(int(statistics_mode == "valid"))]
    r = subprocess.run([exe, *args], capture_output=True, text=True, env=env)
    assert r.returncode == 0 and "AddressSanitizer" not in r.stderr, r.stdout[-2000:] + r.stderr[-4000:]
    out = np.fromfile(tmp_path / "out.f32", np.float32)
    ends = np.cumsum(targets)
    return [out[e - t: e] for e, t in zip(ends, targets)]


CASES = [
    ("noise", 16000 + 77, {}, 0), ("reverb", 24000, {}, 5), ("silence", 20000 + 127, {}, -40), ("full", 1536, {}, 0),
    ("reverb", 12000 + 1, dict(statistics_mode="valid"), 0), ("silence", 16000, dict(taps=3, delay=1, iterations=2), 100),
    ("reverb", 10000, dict(taps=16, delay=0, iterations=1), 0), ("noise", 9000, dict(taps=1, delay=7, iterations=4), 0),
]


@pytest.mark.parametrize("kind,n,p,pad", CASES)
def test_host_harness_within_bound_of_restatement(harness, tmp_path, kind, n, p, pad):
    """Per cut: max|harness - truth64| <= max(2 max|restated complex64 chain - truth64|, 1e-6 max|truth64|)."""
    x = WC.signal(kind, n, seed=n)
    target = 128 * (n // 128) + pad
    got = run_harness(harness, tmp_path, [x], [target], **p)[0]
    t64 = WC.truth64(x, target, **p)
    r32 = W.dereverb(x, target, np.float32, **{**WC.DEFAULT, **p})
    ok, err, lim = WC.bound(got, t64, r32)
    assert ok, (err, lim)


def test_host_harness_zero_cut_and_zero_bins(harness, tmp_path):
    """An all-zero cut gives exact zeros (R = 0 in every bin: G = 0); a pure tone leaves most bins exactly zero."""
    z, tone = WC.signal("zero", 5000), (0.5 * np.cos(2 * np.pi * 64 * np.arange(6000) / 512)).astype(np.float32)
    a, b = run_harness(harness, tmp_path, [z, tone])
    assert np.array_equal(a, np.zeros_like(a))
    assert np.all(np.isfinite(b))
    ok, err, lim = WC.bound(b, WC.truth64(tone), W.dereverb(tone, None, np.float32))
    assert ok or err < 1e-6, (err, lim)


def test_restatement_edges():
    """The oracle's own edge rules: eps = 0 gives unit weights (an all-zero bin filters to 0); the max is per bin (scaling
    one bin does not change another's result); the complex64 and complex128 restatements agree on a well-conditioned cut."""
    Y = np.zeros((2, 1, 40), np.complex128)
    rs = np.random.RandomState(0)
    Y[1, 0] = rs.randn(40) + 1j * rs.randn(40)
    X = W.wpe_v8(Y)
    assert np.array_equal(X[0], np.zeros_like(X[0]))
    Y2 = Y.copy()
    Y2[0, 0] = 1e6 * (rs.randn(40) + 1j * rs.randn(40))
    assert np.allclose(W.wpe_v8(Y2)[1], X[1], rtol=1e-12, atol=0)


# ---- routes ---------------------------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def lhotse_wpe(tmp_path_factory):
    if not refshim.reference_available():
        pytest.skip("reference tree not present")
    import lhotse_env
    import test_reverb

    lhotse_env.setup_lhotse()
    root = tmp_path_factory.mktemp("wpecuts")
    return root, test_reverb.make_sources(root)


def _cut(root, name, n, sr=16000):
    import lhotse_env
    from lhotse import MonoCut, Recording
    from lhotse.audio import AudioSource

    path = root / f"{name}.wav"
    lhotse_env.write_wav(path, (np.random.RandomState(n).randn(n) * 3000).astype("<i2"), sr)
    rec = Recording(id=name, sources=[AudioSource(type="file", channels=[0], source=str(path))], sampling_rate=sr,
                    num_samples=n, duration=n / sr)
    return MonoCut(id=name, start=0.0, duration=n / sr, channel=0, recording=rec)


@needs_ref
def test_transform_route_takes_wpe_last_chains(lhotse_wpe):
    import transform_cases as T

    from lhotse_b200.pcm_staging import WpeRequest, staged_route, transform_request_for_cut

    root, (speech, rirs) = lhotse_wpe
    c = speech[0]
    with T.torch_resampler():
        assert transform_request_for_cut(c.dereverb_wpe()) is None  # off by default
        assert staged_route([c.dereverb_wpe(), speech[1]]) is None
        r = transform_request_for_cut(c.dereverb_wpe(), wpe=True)
        assert r is not None and r.ops == () and r.wpe == WpeRequest() and r.reverb is None
        assert r.source.num_samples == c.num_samples and r.num_samples == c.num_samples
        sp = transform_request_for_cut(c.perturb_speed(1.1).dereverb_wpe(), wpe=True)
        assert sp.ops == (("resample", 17600, 16000),) and sp.wpe == WpeRequest()
        rv = transform_request_for_cut(c.perturb_speed(0.9).reverb_rir(rirs["rir_short"]).dereverb_wpe(), reverb=True, wpe=True)
        assert rv.reverb is not None and rv.wpe is not None
        assert transform_request_for_cut(c.reverb_rir(rirs["rir_short"]).dereverb_wpe(), wpe=True) is None  # reverb=False
        assert staged_route([c.dereverb_wpe(), speech[1]], wpe=True)[0] == "transform"
        # refused: WPE before another transform, two WPEs
        assert transform_request_for_cut(c.dereverb_wpe().perturb_volume(2.0), wpe=True) is None
        assert transform_request_for_cut(c.dereverb_wpe().perturb_speed(1.1), wpe=True) is None
        assert transform_request_for_cut(c.dereverb_wpe().dereverb_wpe(), wpe=True) is None
        # wpe=True changes nothing for cuts without DereverbWPE
        for cut in (c.perturb_speed(1.1), c.reverb_rir(rirs["rir_long"]), c.perturb_volume(0.5)):
            assert transform_request_for_cut(cut, reverb=True, wpe=True) == transform_request_for_cut(cut, reverb=True)


@needs_ref
def test_transform_route_wpe_lengths(lhotse_wpe):
    """The shortest cut (1536 samples: 13 frames = taps + delay) and the frame cap (8192 frames) are taken, one sample less
    and one more are refused; the duration tolerance is checked against DereverbWPE's length 128 (L // 128)."""
    from lhotse.audio.utils import get_audio_duration_mismatch_tolerance, set_audio_duration_mismatch_tolerance

    from lhotse_b200.engine import WPE_MAX_FRAMES
    from lhotse_b200.pcm_staging import WpeRequest, transform_request_for_cut, wpe_output_len

    root, _ = lhotse_wpe
    cap = 128 * WPE_MAX_FRAMES - 1
    for n, ok in ((1536, True), (1535, False), (cap, True), (cap + 1, False), (256, False)):
        r = transform_request_for_cut(_cut(root, f"len{n}", n).dereverb_wpe(), wpe=True)
        assert (r is not None) == ok, n
    assert wpe_output_len(1536, WpeRequest(taps=12, delay=2)) is None and wpe_output_len(1536, WpeRequest(taps=12, delay=1))
    saved = get_audio_duration_mismatch_tolerance()
    try:
        set_audio_duration_mismatch_tolerance(0.001)  # 16 samples at 16 kHz
        assert transform_request_for_cut(_cut(root, "m0", 16000).dereverb_wpe(), wpe=True) is not None  # 16000 = 125 * 128
        assert transform_request_for_cut(_cut(root, "m10", 16010).dereverb_wpe(), wpe=True) is not None  # 10 short
        assert transform_request_for_cut(_cut(root, "m100", 16100).dereverb_wpe(), wpe=True) is None  # 100 short
    finally:
        set_audio_duration_mismatch_tolerance(saved)


@needs_ref
def test_transform_staging_sends_wpe_input_to_mid(lhotse_wpe):
    """The stage table: a WPE cut's last stage (or its reverb) writes `mid` at its natural length; WPE reads it and writes the
    cut's window of the output."""
    import transform_cases as T

    from lhotse_b200.engine import RESAMPLE_TO_MID
    from lhotse_b200.pcm_staging import TransformStagingRing, staged_route

    root, (speech, rirs) = lhotse_wpe
    c0, c1, c2 = speech
    cuts = [c0.dereverb_wpe(), c1.perturb_speed(1.1), c2.perturb_speed(0.9).reverb_rir(rirs["rir_short"]).dereverb_wpe()]
    with T.torch_resampler():
        route, reqs = staged_route(cuts, reverb=True, wpe=True)
        batch, lens, offs, _ = TransformStagingRing(pin_memory=False).stage(reqs)
    assert route == "transform" and len(batch.wpe) == 1
    (w, table), = batch.wpe
    assert list(table["out_elem"]) == [offs[0], offs[2]] and list(table["target_len"]) == [lens[0], lens[2]]
    st = batch.stages
    first = st[(st["depth"] == 0) & (st["target"] == RESAMPLE_TO_MID)]
    assert first["out_elem"][0] == table["in_elem"][0] and first["target_len"][0] == first["out_len"][0] == c0.num_samples
    assert batch.reverb_cuts is None and len(batch.reverb_mid_cuts) == 1
    rm = batch.reverb_mid_cuts[0]
    assert rm["out_elem"] == table["in_elem"][1] and rm["target_len"] == rm["in_len"] == table["in_len"][1]
