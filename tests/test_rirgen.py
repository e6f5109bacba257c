"""The host half of the RIR generator (lhotse_b200/rir_draws.py): the restated torch.multinomial against torch over many
generator states, torch.linspace against its float32 restatement, and the generator states a batch of draws leaves against
those lhotse's own generator leaves (DESIGN.md §3.1l).  No GPU needed."""
import copy

import numpy as np
import pytest
import torch

import refshim
import rirgen_cases as RG

from lhotse_b200 import rir_draws

needs_ref = pytest.mark.skipif(not refshim.reference_available(), reason="no reference tree / oracle/_ref archive")


@pytest.mark.parametrize("image", [16000, 32000, 96000])
def test_restated_multinomial_equals_torch(image):
    cdf = rir_draws.multinomial_cdf(0.25, image)
    probs = torch.linspace(0.25, 1.0, image).pow(2)
    probs = probs / probs.sum()
    # a fresh seed (left == 1), states on either side of a twist, and states deep in a block
    for seed, skip in [(0, 0), (1, 0), (2, 311), (3, 312), (4, 623), (5, 624), (6, 1000)] + [(100 + k, 37 * k) for k in range(33)]:
        g = torch.Generator().manual_seed(seed)
        torch.rand(skip, generator=g, dtype=torch.float64)
        got = rir_draws.torch_uniforms(g.get_state(), image)
        want = probs.multinomial(num_samples=image, replacement=True, generator=g)
        assert got is not None
        assert np.array_equal(rir_draws.multinomial_from_uniforms(cdf, got[0]), want.numpy())
        after = torch.Generator()
        after.set_state(got[1])
        assert torch.equal(torch.rand(7, generator=after), torch.rand(7, generator=g))


def test_restated_linspace_equals_torch():
    rs = np.random.RandomState(0)
    for steps in (16000, 32000, 96000, 1001):
        for end in rs.uniform(1.2, 3000.0, 8):
            want = torch.linspace(1.0, torch.tensor(float(end), dtype=torch.float64), steps).numpy()
            assert np.array_equal(rir_draws.linspace32(1.0, float(end), steps).view(np.int32), want.view(np.int32))


def test_state_layout_refused():
    assert rir_draws.torch_uniforms(torch.zeros(10, dtype=torch.uint8), 4) is None


@needs_ref
def test_draws_leave_lhotse_states():
    import lhotse_env

    lhotse_env.setup_lhotse()
    gens = [RG.generator(*c) for c in RG.CASES]
    refs = [copy.deepcopy(g) for g in gens]
    torch.manual_seed(11)
    d = rir_draws.draw(gens)
    after = torch.get_rng_state()
    torch.manual_seed(11)
    n = torch.get_num_threads()
    torch.set_num_threads(1)
    try:
        want = [g(nsource=1)[0] for g in refs]
    finally:
        torch.set_num_threads(n)
    assert torch.equal(torch.get_rng_state(), after)
    for g, r, w, L in zip(gens, refs, want, d.lens):
        assert g.room_rng.bit_generator.state == r.room_rng.bit_generator.state
        assert g.source_rng.bit_generator.state == r.source_rng.bit_generator.state
        assert w.shape == (L,)


@needs_ref
def test_truth_is_close_to_lhotse():
    """The float64 truth the GPU tests hold the RIRs to is lhotse's RIR up to float32 error."""
    import lhotse_env

    lhotse_env.setup_lhotse()
    for case in RG.CASES[:3]:
        gen = RG.generator(*case)
        torch.manual_seed(3)
        s = torch.get_rng_state()
        ref, _, _ = RG.lhotse_rir(gen)
        torch.set_rng_state(s)
        d = rir_draws.draw([gen])
        image = 2 * case[0]
        truth, _, _ = RG.truth64(d.records[0], d.draws[:image], d.draws[image: 2 * image], gen)
        assert truth.shape == ref.shape
        assert float(np.max(np.abs(ref - truth))) <= 1e-3 * float(np.max(np.abs(truth)))


@pytest.fixture(scope="module")
def harness(tmp_path_factory):
    import os
    import shutil
    import subprocess

    d = tmp_path_factory.mktemp("rgh")
    src = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "scripts", "micro", "rirgen_host_check.cu")
    exe = str(d / "rirgen_host_check")
    gxx = shutil.which("g++")
    if gxx:
        for flags in (["-fsanitize=address", "-fno-omit-frame-pointer"], []):
            res = subprocess.run([gxx, "-x", "c++", "-std=c++17", "-O1", "-g", *flags, "-o", exe, src],
                                 capture_output=True, text=True)
            if res.returncode == 0:
                return exe
    pytest.skip("no host C++ compiler")


def run_harness(exe, tmp_path, d):
    """The host harness over one batch of draws: per RIR (kept positions, kept values, direct position, entries there,
    direct value) and its samples at 8 sr after the biquad."""
    import os
    import subprocess

    from lhotse_b200.pcm_staging import resample_kernel

    d.records.tofile(tmp_path / "recs.bin")
    d.draws.tofile(tmp_path / "draws.f64")
    d.cdf.astype(np.float32).tofile(tmp_path / "cdf.f32")
    resample_kernel(8, 1)[0][0].astype(np.float32).tofile(tmp_path / "table.f32")
    files = [str(tmp_path / f) for f in ("recs.bin", "draws.f64", "cdf.f32", "table.f32", "entries.bin", "out8.f32")]
    env = dict(os.environ, ASAN_OPTIONS="detect_leaks=0:abort_on_error=0")
    r = subprocess.run([exe, *files], capture_output=True, text=True, env=env)
    assert r.returncode == 0 and "AddressSanitizer" not in r.stderr, r.stdout[-2000:] + r.stderr[-4000:]
    raw = open(files[4], "rb").read()
    out8 = np.fromfile(files[5], np.float32)
    res, at, o = [], 0, 0
    for rec in d.records:
        kept = int(np.frombuffer(raw, np.int64, 1, at)[0])
        dpos, ndir = np.frombuffer(raw, np.int32, 2, at + 8)
        dval = np.frombuffer(raw, np.float32, 1, at + 16)[0]
        kpos = np.frombuffer(raw, np.int32, kept, at + 20)
        kval = np.frombuffer(raw, np.float32, kept, at + 20 + 4 * kept)
        at += 20 + 8 * kept
        n8 = int(rec["out_len"])
        res.append((kpos, kval, int(dpos), int(ndir), dval, out8[o: o + n8]))
        o += n8
    return res


def lhotse_comb(gen):
    """lhotse's own comb (the first resampler's input row 0, float32) and RIR for a copy of `gen` from torch's current state,
    with one torch thread; torch's state is left where lhotse leaves it."""
    import lhotse.augmentation.torchaudio as lta

    seen = []
    orig = lta.get_or_create_resampler

    def spy(a, b):
        rs = orig(a, b)
        return (lambda x: seen.append(x[0].clone()) or rs(x)) if not seen else rs

    lta.get_or_create_resampler = spy
    try:
        rir, _, _ = RG.lhotse_rir(gen)
    finally:
        lta.get_or_create_resampler = orig
    return seen[0].numpy(), rir


def _ulps(a, b):
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    assert np.all(np.sign(a) == np.sign(b))
    return np.abs(a.view(np.int32).astype(np.int64) - b.view(np.int32).astype(np.int64))


@needs_ref
def test_host_harness_against_lhotse(harness, tmp_path):
    """The kernels' arithmetic on the CPU under AddressSanitizer: comb positions equal to lhotse's, values within 4 ulps
    (last wins where images share a position, the direct path's included), and each whole RIR within the float64 bound."""
    import lhotse_env

    from lhotse_b200.pcm_staging import resample_reference

    lhotse_env.setup_lhotse()
    collided = 0
    for k, case in enumerate(RG.CASES):
        gen = RG.generator(*case)
        torch.manual_seed(40 + k)
        s = torch.get_rng_state()
        comb, ref = lhotse_comb(gen)
        torch.set_rng_state(s)
        d = rir_draws.draw([gen])
        kpos, kval, dpos, ndir, dval, out8 = run_harness(harness, tmp_path, d)[0]
        nz = np.nonzero(comb)[0]
        assert np.array_equal(nz, kpos[kval != 0]), case
        assert int(_ulps(kval, comb[kpos]).max()) <= 4, case
        if ndir > 1:  # an image at the direct path's position: the last image's value is kept, not the direct path's
            collided += 1
            assert comb[dpos] == kval[np.searchsorted(kpos, dpos)]
        ours = resample_reference(out8, 8, 1)
        image = 2 * case[0]
        truth, _, _ = RG.truth64(d.records[0], d.draws[:image], d.draws[image: 2 * image], gen)
        err, bnd = RG.bound(ours, ref, truth)
        assert err <= bnd, (case, err, bnd)
    assert collided > 0
