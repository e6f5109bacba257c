"""GPU mixing on the CPU: the exact energy tree and mixing arithmetic of csrc/mix.cuh run on the host
(scripts/micro/mix_host_check.cu, under AddressSanitizer where the toolchain has it) against lhotse's own `audio_energy` and
`MixedCut.load_audio()`, over the tables `MixStagingRing` builds; and `mix_request_for_cut`'s refusals."""
import math
import os
import shutil
import subprocess

import numpy as np
import pytest

import refshim

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
needs_ref = pytest.mark.skipif(not refshim.reference_available(), reason="reference tree not present")


@pytest.fixture(scope="module")
def harness(tmp_path_factory):
    d = tmp_path_factory.mktemp("mixh")
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


def _run(exe, *args):
    env = dict(os.environ, ASAN_OPTIONS="detect_leaks=0:abort_on_error=0")
    r = subprocess.run([exe, *map(str, args)], capture_output=True, text=True, env=env)
    assert r.returncode == 0 and "AddressSanitizer" not in r.stderr, r.stdout[-2000:] + r.stderr[-4000:]


def _audio_energy():
    if refshim.reference_available():
        refshim.import_reference()
        from lhotse.audio.mixer import audio_energy

        return audio_energy
    return lambda x: float(np.average(x ** 2))  # lhotse/audio/mixer.py audio_energy, verbatim


def test_energy_tree_is_bit_equal_to_audio_energy(harness, tmp_path):
    energy = _audio_energy()
    rs = np.random.RandomState(5)
    lens = list(range(1, 1101))
    lens += [8 * k + d for k in (16, 17, 31, 64, 125, 1000, 2001) for d in (-1, 1)] + [127, 128, 129]
    lens += [16000, 160000, 160001, 480007]
    segs = []
    for i, n in enumerate(lens):
        if i % 11 == 0:
            q = np.zeros(n, dtype=np.int16)
        elif i % 11 == 1:
            q = np.where(rs.rand(n) < 0.5, -32768, 32767).astype(np.int16)  # full scale
        else:
            q = np.clip(rs.randn(n) * rs.choice([30, 3000, 20000]), -32768, 32767).astype(np.int16)
        segs.append(q)
    segs += [np.full(1000, -32768, np.int16), np.zeros(480007, np.int16)]
    lens += [1000, 480007]
    np.concatenate(segs).tofile(tmp_path / "e.i16")
    np.asarray(lens, dtype=np.int64).tofile(tmp_path / "e.i64")
    _run(harness, "energy", tmp_path / "e.i16", tmp_path / "e.i64", tmp_path / "e.f64")
    got = np.fromfile(tmp_path / "e.f64", dtype=np.float64)
    want = np.asarray([energy((q.astype(np.float32) / 32768.0)[None, :]) for q in segs])
    bad = [lens[i] for i in np.nonzero(got != want)[0]]
    assert not bad, bad[:20]


@pytest.fixture(scope="module")
def lhotse_cuts(tmp_path_factory):
    if not refshim.reference_available():
        pytest.skip("reference tree not present")
    import lhotse_env
    import mix_cases

    lhotse_env.setup_lhotse()
    root = tmp_path_factory.mktemp("mixcuts")
    speech, noise = mix_cases.sources(root)
    return root, speech, noise, mix_cases.mixed_cases(root, speech, noise)


def _host_mix(harness, tmp_path, cuts):
    from lhotse_b200.pcm_staging import MixStagingRing, mix_requests_for_batch

    reqs = mix_requests_for_batch(cuts)
    assert reqs is not None
    batch, lens, offs, sr = MixStagingRing(pin_memory=False).stage(reqs)
    assert sr == 16000 and batch.flac is None and all(o % 4 == 0 for o in offs)
    out = run_mix(harness, tmp_path, batch.pcm.numpy(), np.zeros(0, np.int16), batch.tracks, batch.cuts, batch.out_elems)
    return [out[o:o + n] for o, n in zip(offs, lens)], batch


def run_mix(harness, tmp_path, src0, src1, tracks, cuts, out_elems, src2=None):
    """b200feat_mix_ex through the host harness: the int16 sources, the float32 track buffer `src2` (None: none) and the
    MIX_TRACK_DTYPE / MIX_CUT_DTYPE tables -> the float32 output buffer (zeros outside the cuts' windows)."""
    np.asarray(src0, np.int16).tofile(tmp_path / "s0.i16")
    np.asarray(src1, np.int16).tofile(tmp_path / "s1.i16")
    tracks.tofile(tmp_path / "t.bin")
    cuts.tofile(tmp_path / "c.bin")
    extra = []
    if src2 is not None:
        np.asarray(src2, np.float32).tofile(tmp_path / "s2.f32")
        extra = [tmp_path / "s2.f32"]
    _run(harness, "mix", tmp_path / "s0.i16", tmp_path / "s1.i16", tmp_path / "t.bin", tmp_path / "c.bin", out_elems,
         tmp_path / "o.f32", *extra)
    return np.fromfile(tmp_path / "o.f32", dtype=np.float32)


@needs_ref
def test_host_mix_is_bit_equal_to_load_audio(harness, lhotse_cuts, tmp_path):
    import mix_cases

    from lhotse_b200.engine import MIX_SCALED_FIRST

    _, speech, noise, cases = lhotse_cuts
    names = sorted(cases)
    assert {"mix_snr_None", "mix_snr_-5", "pad_left", "append_gap", "muted_reference", "scaled_first", "trim", "reflect_pad"} <= set(names)
    assert sum(n.startswith("cutmix_") for n in names) == 4
    cuts = [cases[k] for k in names] + [speech[0], noise[2]]  # plain slices ride along as one-track mixes
    got, batch = _host_mix(harness, tmp_path, cuts)
    for name, cut, g in zip(names + ["plain0", "plain1"], cuts, got):
        want = mix_cases.load_f32(cut)
        assert g.shape == want.shape and np.array_equal(g.view(np.int32), want.view(np.int32)), name
    # the arithmetic paths the table is meant to reach
    req = {k: r for k, r in zip(names, batch.cuts)}
    assert req["scaled_first"]["mode"] == MIX_SCALED_FIRST and req["mix_snr_0"]["mode"] == 0
    assert req["reflect_pad"]["target_len"] == req["reflect_pad"]["mix_len"] + 1
    assert req["trim"]["target_len"] == req["trim"]["mix_len"] - 1
    assert cases["scaled_first"].load_audio().dtype == np.float64
    assert any(len(cases[k].tracks) > 2 for k in names if k.startswith("cutmix_"))  # several noise pieces


@needs_ref
def test_mix_route_refuses_what_it_cannot_reproduce(lhotse_cuts, monkeypatch):
    import mix_cases
    from lhotse.audio.utils import get_audio_duration_mismatch_tolerance, set_audio_duration_mismatch_tolerance

    from lhotse_b200 import pcm_staging
    from lhotse_b200.pcm_staging import mix_request_for_cut, mix_requests_for_batch

    root, speech, noise, cases = lhotse_cuts
    for name, cut in mix_cases.refused_cases(root, speech, noise).items():
        assert mix_request_for_cut(cut) is None, name
    ok = cases["mix_snr_0"]
    assert mix_request_for_cut(ok) is not None
    # outside the duration-mismatch tolerance
    tol = get_audio_duration_mismatch_tolerance()
    set_audio_duration_mismatch_tolerance(1e-6)
    try:
        assert mix_request_for_cut(cases["trim"]) is None and mix_request_for_cut(cases["reflect_pad"]) is None
        assert mix_request_for_cut(ok) is not None
    finally:
        set_audio_duration_mismatch_tolerance(tol)
    assert mix_request_for_cut(cases["trim"]) is not None
    # NumPy 1.x promotes np.float64 * float32 arrays differently: the route declines
    monkeypatch.setattr(pcm_staging, "_numpy2", lambda: False)
    assert mix_request_for_cut(ok) is None
    monkeypatch.undo()
    # batches: plain slices alone keep their routes; one refused cut sends the whole batch to the float route
    assert mix_requests_for_batch([speech[0], speech[1]]) is None
    assert mix_requests_for_batch([speech[0], ok]) is not None
    assert mix_requests_for_batch([ok, mix_cases.refused_cases(root, speech, noise)["nested_mixed"]]) is None


@needs_ref
def test_mix_request_factors_and_offsets_follow_lhotse(lhotse_cuts):
    from lhotse.utils import compute_num_samples

    from lhotse_b200.engine import MIX_ROLE_ENERGY
    from lhotse_b200.pcm_staging import mix_request_for_cut

    _, _, _, cases = lhotse_cuts
    r = mix_request_for_cut(cases["muted_reference"])
    assert [t.role for t in r.tracks] == [0, 0, MIX_ROLE_ENERGY] and r.ref == 2
    assert r.tracks[1].offset == compute_num_samples(0.4, 16000)
    assert r.tracks[0].snr_factor == 10.0 ** (-10.0 / 10) and r.tracks[1].snr_factor == 10.0 ** (-3.0 / 10)
    assert math.isnan(mix_request_for_cut(cases["mix_snr_None"]).tracks[1].snr_factor)
