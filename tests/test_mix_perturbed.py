"""Perturbed MixedCut tracks on the CPU: the "mix" route's requests with `perturbed_tracks=True` against lhotse (lengths,
offsets, factors, roles), the default still refusing every such cut, the cuts refused even with the flag, and the mixing
arithmetic of csrc/mix.cuh with float32 tracks (scripts/micro/mix_host_check.cu, under AddressSanitizer where the toolchain
has it) bit-equal to `MixedCut.load_audio()`, the float tracks taken from lhotse's own `track.cut.load_audio()`."""
import math
import os
import shutil
import subprocess

import numpy as np
import pytest

import refshim

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = [os.path.join(ROOT, "tests", "golden", f"2412-153948-000{i}.flac") for i in (0, 1)]


@pytest.fixture(scope="module")
def harness(tmp_path_factory):
    d = tmp_path_factory.mktemp("pmixh")
    src = os.path.join(ROOT, "scripts", "micro", "mix_host_check.cu")
    exe = str(d / "mix_host_check")
    gxx = shutil.which("g++")
    if gxx:
        for flags in (["-fsanitize=address", "-fno-omit-frame-pointer"], []):
            res = subprocess.run([gxx, "-x", "c++", "-std=c++17", "-O1", "-g", *flags, "-o", exe, src], capture_output=True, text=True)
            if res.returncode == 0:
                return exe
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("no host compiler")
    res = subprocess.run([nvcc, "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-o", exe, src], capture_output=True, text=True)
    assert res.returncode == 0, res.stderr[-2000:]
    return exe


@pytest.fixture(scope="module")
def env(tmp_path_factory):
    if not refshim.reference_available():
        pytest.skip("reference tree not present")
    import lhotse_env
    import perturbed_mix_cases as P
    import transform_cases

    lhotse_env.setup_lhotse()
    root = tmp_path_factory.mktemp("pmix")
    speech, noise, s48 = P.sources(root)
    with transform_cases.torch_resampler(), P.flac_backend():
        flac = P.flac_cuts(GOLDEN)
        yield root, speech, noise, P.cases(root, speech, noise, s48, flac)


def _run(exe, *args):
    env = dict(os.environ, ASAN_OPTIONS="detect_leaks=0:abort_on_error=0")
    r = subprocess.run([exe, *map(str, args)], capture_output=True, text=True, env=env)
    assert r.returncode == 0 and "AddressSanitizer" not in r.stderr, r.stdout[-2000:] + r.stderr[-4000:]


def test_default_refuses_and_flag_accepts_every_case(env):
    from lhotse_b200.pcm_staging import mix_request_for_cut, mix_requests_for_batch

    _, speech, _, cases = env
    assert sum(k.startswith("cutmix_") for k in cases) == 4 and "flac_speech_speed" in cases
    for name, cut in cases.items():
        assert mix_request_for_cut(cut) is None, name
        assert mix_request_for_cut(cut, perturbed_tracks=True) is not None, name
    cuts = list(cases.values()) + [speech[0], speech[1].perturb_speed(1.1)]
    assert mix_requests_for_batch(cuts) is None
    assert mix_requests_for_batch(cuts, perturbed_tracks=True) is not None
    # without a MixedCut the batch keeps the transform / pcm16 routes
    assert mix_requests_for_batch([speech[0], speech[1].perturb_speed(1.1)], perturbed_tracks=True) is None


def test_requests_follow_lhotse(env):
    import perturbed_mix_cases as P
    from lhotse.cut import PaddingCut
    from lhotse.utils import compute_num_samples

    from lhotse_b200.engine import MIX_ROLE_ENERGY, MIX_ROLE_MIXED, MIX_SCALED_FIRST
    from lhotse_b200.pcm_staging import TransformRequest, mix_request_for_cut, transform_request_for_cut

    _, _, _, cases = env
    for name, cut in cases.items():
        r = mix_request_for_cut(cut, perturbed_tracks=True)
        chosen = P.chosen_tracks(cut)
        assert len(r.tracks) == len(chosen), name
        for t, mt in zip(r.tracks, chosen):
            assert t.offset == compute_num_samples(mt.offset, 16000), name
            assert (math.isnan(t.snr_factor) if mt.snr is None else t.snr_factor == 10.0 ** (-mt.snr / 10)), name
            if isinstance(mt.cut, PaddingCut):
                assert t.source is None
            elif mt.cut.has_recording and mt.cut.recording.transforms:
                assert isinstance(t.source, TransformRequest) and t.source == transform_request_for_cut(mt.cut), name
                assert t.num_samples == t.source.num_samples == mt.cut.load_audio().shape[-1], name
            else:
                assert not isinstance(t.source, TransformRequest), name
    r = mix_request_for_cut(cases["muted_perturbed_reference"], perturbed_tracks=True)
    assert [t.role for t in r.tracks] == [MIX_ROLE_MIXED, MIX_ROLE_MIXED, MIX_ROLE_ENERGY] and r.ref == 2
    assert isinstance(r.tracks[2].source, TransformRequest)
    r = mix_request_for_cut(cases["scaled_perturbed_first"], perturbed_tracks=True)
    assert r.mode == MIX_SCALED_FIRST and isinstance(r.tracks[0].source, TransformRequest)
    # MixedCut.perturb_speed rescales the offsets and perturbs the padding
    m = cases["mixed_then_speed_0.9"]
    r = mix_request_for_cut(m, perturbed_tracks=True)
    assert any(t.source is None for t in r.tracks) and sum(isinstance(t.source, TransformRequest) for t in r.tracks) == 2
    noise = next(t for t in m.tracks if t.snr is not None)
    assert math.isclose(noise.offset, 0.3 / 0.9, abs_tol=1e-4)  # the mix offset, rescaled by the speed factor
    assert any(t.offset == compute_num_samples(noise.offset, 16000) > 0 for t in r.tracks)


def test_refused_even_with_the_flag(env, monkeypatch):
    import perturbed_mix_cases as P

    from lhotse_b200 import pcm_staging
    from lhotse_b200.pcm_staging import mix_request_for_cut

    root, speech, noise, cases = env
    for name, cut in P.refused_cases(root, speech, noise).items():
        assert mix_request_for_cut(cut, perturbed_tracks=True) is None, name
    ok = cases["speed_1.1_snr_0"]
    assert mix_request_for_cut(ok, perturbed_tracks=True) is not None
    # a host whose resampler does not match the kernel's arithmetic: the route declines
    monkeypatch.setattr(pcm_staging, "resample_probe", lambda a, b: False)
    assert mix_request_for_cut(ok, perturbed_tracks=True) is None
    assert mix_request_for_cut(cases["volume_track"], perturbed_tracks=True) is not None  # no resampling stage


def test_host_mix_with_float_tracks_is_bit_equal_to_load_audio(harness, env, tmp_path):
    import perturbed_mix_cases as P

    from lhotse_b200.engine import MIX_SCALED_FIRST, MIX_SRC_F32
    from lhotse_b200.pcm_staging import MixStagingRing, mix_requests_for_batch

    _, speech, _, cases = env
    names = sorted(k for k in cases if not k.startswith("flac_"))  # the harness reads int16 sources as WAV samples only
    cuts = [cases[k] for k in names] + [speech[0], speech[2].perturb_speed(0.9)]
    reqs = mix_requests_for_batch(cuts, perturbed_tracks=True)
    assert reqs is not None
    batch, lens, offs, sr = MixStagingRing(pin_memory=False).stage(reqs)
    assert sr == 16000 and batch.flac is None and batch.transform is not None
    # the float32 track buffer, filled from lhotse's own track.cut.load_audio() at the offsets the ring assigned
    src2 = np.zeros(max(batch.transform.out_elems, 1), np.float32)
    track_cuts = []
    for c in cuts:
        track_cuts += [t.cut for t in P.chosen_tracks(c)] if getattr(c, "tracks", None) is not None else [c]
    assert len(track_cuts) == len(batch.tracks)
    for row, tc in zip(batch.tracks, track_cuts):
        if row["source"] == MIX_SRC_F32:
            x = P.load_f32(tc)
            assert x.shape == (row["num_samples"],)
            src2[row["src_elem"]: row["src_elem"] + row["num_samples"]] = x
    assert (batch.tracks["source"] == MIX_SRC_F32).sum() >= len(names)
    batch.pcm.numpy().tofile(tmp_path / "s0.i16")
    np.zeros(0, np.int16).tofile(tmp_path / "s1.i16")
    src2.tofile(tmp_path / "s2.f32")
    batch.tracks.tofile(tmp_path / "t.bin")
    batch.cuts.tofile(tmp_path / "c.bin")
    _run(harness, "mix", tmp_path / "s0.i16", tmp_path / "s1.i16", tmp_path / "t.bin", tmp_path / "c.bin", batch.out_elems,
         tmp_path / "o.f32", tmp_path / "s2.f32")
    out = np.fromfile(tmp_path / "o.f32", dtype=np.float32)
    for name, c, o, n in zip(names + ["plain", "plain_speed"], cuts, offs, lens):
        want = P.load_f32(c)
        assert want.shape == (n,) and np.array_equal(out[o:o + n].view(np.int32), want.view(np.int32)), name
    # the arithmetic paths the table is meant to reach
    req = {k: r for k, r in zip(names, batch.cuts)}
    assert req["scaled_perturbed_first"]["mode"] == MIX_SCALED_FIRST
    assert cases["scaled_perturbed_first"].load_audio().dtype == np.float64
    assert req["reflect_pad"]["target_len"] == req["reflect_pad"]["mix_len"] + 1
    assert req["trim"]["target_len"] == req["trim"]["mix_len"] - 1


def test_host_mix_with_flac_speech_is_bit_equal_to_load_audio(harness, env, tmp_path):
    """FLAC speech under WAV noise: the FLAC tracks are perturbed, so they too reach the mix as float32 tracks."""
    import perturbed_mix_cases as P

    from lhotse_b200.engine import MIX_SRC_F32
    from lhotse_b200.pcm_staging import MixStagingRing, mix_requests_for_batch

    _, _, _, cases = env
    cuts = [cases["flac_speech_speed"], cases["flac_speech_volume"]]
    batch, lens, offs, _ = MixStagingRing(pin_memory=False).stage(mix_requests_for_batch(cuts, perturbed_tracks=True))
    assert batch.flac is None and batch.transform.flac is not None  # the FLAC slices go through the transform ring
    src2 = np.zeros(max(batch.transform.out_elems, 1), np.float32)
    track_cuts = [t.cut for c in cuts for t in P.chosen_tracks(c)]
    for row, tc in zip(batch.tracks, track_cuts):
        if row["source"] == MIX_SRC_F32:
            src2[row["src_elem"]: row["src_elem"] + row["num_samples"]] = P.load_f32(tc)
    batch.pcm.numpy().tofile(tmp_path / "s0.i16")
    np.zeros(0, np.int16).tofile(tmp_path / "s1.i16")
    src2.tofile(tmp_path / "s2.f32")
    batch.tracks.tofile(tmp_path / "t.bin")
    batch.cuts.tofile(tmp_path / "c.bin")
    _run(harness, "mix", tmp_path / "s0.i16", tmp_path / "s1.i16", tmp_path / "t.bin", tmp_path / "c.bin", batch.out_elems,
         tmp_path / "o.f32", tmp_path / "s2.f32")
    out = np.fromfile(tmp_path / "o.f32", dtype=np.float32)
    for c, o, n in zip(cuts, offs, lens):
        assert np.array_equal(out[o:o + n].view(np.int32), P.load_f32(c).view(np.int32)), c.id
