"""GPU transforms on the CPU: the resampling table against lhotse's own, the exact chunking, window and FMA chain of
csrc/resample.cuh run on the host (scripts/micro/resample_host_check.cu, under AddressSanitizer where the toolchain has it)
against `cut.load_audio()` of real speed-perturbed, volume-perturbed and resampled lhotse cuts over the tables
`TransformStagingRing` builds; the oneDNN length boundary; and `transform_request_for_cut`'s refusals."""
import os
import shutil
import subprocess

import numpy as np
import pytest

import refshim

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
needs_ref = pytest.mark.skipif(not refshim.reference_available(), reason="reference tree not present")
PAIRS = [(14400, 16000), (17600, 16000), (15200, 16000), (16800, 16000), (48000, 16000), (44100, 16000), (22050, 16000),
         (16000, 22050), (16000, 8000), (8000, 16000)]


@pytest.fixture(scope="module")
def harness(tmp_path_factory):
    d = tmp_path_factory.mktemp("rsh")
    src = os.path.join(ROOT, "scripts", "micro", "resample_host_check.cu")
    exe = str(d / "resample_host_check")
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
def lhotse_cuts(tmp_path_factory):
    if not refshim.reference_available():
        pytest.skip("reference tree not present")
    import lhotse_env
    import transform_cases

    lhotse_env.setup_lhotse()
    root = tmp_path_factory.mktemp("tfcuts")
    return root, transform_cases.sources(root)


def host_transform(harness, tmp_path, cuts):
    """The cuts through TransformStagingRing and the host harness: ([samples per cut], batch)."""
    from lhotse_b200.pcm_staging import TransformStagingRing, resample_kernel, transform_requests_for_batch

    reqs = transform_requests_for_batch(cuts)
    assert reqs is not None
    batch, lens, offs, _ = TransformStagingRing(pin_memory=False).stage(reqs)
    assert batch.flac is None and all(o % 4 == 0 for o in offs)
    st = batch.stages.copy()
    st["table"] = batch.pair
    out = run_stages(harness, tmp_path, batch.pcm.numpy(), np.zeros(0, np.int16), batch.pairs, st, batch.mid_elems,
                     batch.out_elems)
    return [out[o:o + n] for o, n in zip(offs, lens)], batch


def run_stages(harness, tmp_path, src0, src1, pairs, stages, mid_elems, out_elems):
    """b200feat_resample through the host harness: the int16 sources, the rate pairs and RESAMPLE_STAGE_DTYPE records whose
    `table` indexes `pairs` (-1: no resampling) -> the float32 output buffer (zeros outside the stages' windows)."""
    from lhotse_b200.pcm_staging import resample_kernel

    np.asarray(src0, np.int16).tofile(tmp_path / "s0.i16")
    np.asarray(src1, np.int16).tofile(tmp_path / "s1.i16")
    with open(tmp_path / "tables.bin", "wb") as f:
        for a, b in pairs:
            table, width = resample_kernel(a, b)
            N, K = table.shape
            np.asarray([N, K - 2 * width, K, width], np.int32).tofile(f)
            table.tofile(f)
    stages.tofile(tmp_path / "st.bin")
    _run(harness, tmp_path / "s0.i16", tmp_path / "s1.i16", tmp_path / "tables.bin", tmp_path / "st.bin", mid_elems, out_elems,
         tmp_path / "o.f32")
    return np.fromfile(tmp_path / "o.f32", dtype=np.float32)


def _run(exe, *args):
    env = dict(os.environ, ASAN_OPTIONS="detect_leaks=0:abort_on_error=0")
    r = subprocess.run([exe, *map(str, args)], capture_output=True, text=True, env=env)
    assert r.returncode == 0 and "AddressSanitizer" not in r.stderr, r.stdout[-2000:] + r.stderr[-4000:]


@needs_ref
@pytest.mark.parametrize("pair", PAIRS, ids=[f"{a}_{b}" for a, b in PAIRS])
def test_table_is_bit_equal_to_lhotse(pair):
    refshim.import_reference()
    from lhotse.augmentation.resample import _get_sinc_resample_kernel

    from lhotse_b200.pcm_staging import _resample_geometry, resample_kernel

    a, b = pair
    import math

    want, wwidth = _get_sinc_resample_kernel(a, b, math.gcd(a, b))
    got, width = resample_kernel(a, b)
    assert width == wwidth and got.dtype == np.float32 and got.shape == tuple(want.shape[::2])
    assert np.array_equal(got.view(np.int32), want[:, 0, :].numpy().view(np.int32))
    N, O, w, K = _resample_geometry(a, b)
    assert (N, K, w) == (got.shape[0], got.shape[1], width) and K == 2 * w + O


@needs_ref
def test_host_transform_is_bit_equal_to_load_audio(harness, lhotse_cuts, tmp_path):
    import transform_cases as T

    root, src = lhotse_cuts
    with T.torch_resampler():
        cases = T.cases(src)
        trim, reflect = T.fix_cases(src)
        cases["trim"], cases["reflect_pad"] = trim, reflect
        names = sorted(cases)
        cuts = [cases[k] for k in names] + [src[16000][0], src[16000][1].truncate(offset=0.3, duration=1.1)]  # plain slices ride along
        got, batch = host_transform(harness, tmp_path, cuts)
        for name, cut, g in zip(names + ["plain0", "plain1"], cuts, got):
            want = T.load_f32(cut)
            assert g.shape == want.shape and np.array_equal(g.view(np.int32), want.view(np.int32)), name
    # what the table is meant to reach: every pair, two-stage chains, scale-only stages, both length fixes, a close-to-full read
    assert {(14400, 16000), (17600, 16000), (15200, 16000), (16800, 16000), (48000, 16000), (44100, 16000), (22050, 16000),
            (16000, 8000), (8000, 16000)} <= set(batch.pairs)
    assert batch.stages["depth"].max() >= 1 and batch.mid_elems > 0 and (batch.pair < 0).any()
    last = batch.stages[batch.stages["target"] == 1]
    assert (last["target_len"] > last["out_len"]).any() and (last["target_len"] < last["out_len"]).any()
    from lhotse_b200.pcm_staging import transform_request_for_cut

    whole = transform_request_for_cut(cases["speed_1.1"])
    assert whole.source.first_sample == 0 and whole.source.num_samples == src[16000][0].num_samples
    # a stage length where lhotse's float32 ceil drops a sample that a float64 ceil would keep
    import math

    from lhotse_b200.pcm_staging import resampled_len

    assert resampled_len(160, 180697, 441) == 65559 != math.ceil(160 * 180697 / 441)
    assert transform_request_for_cut(cases["resample_then_speed_f32_length"]).ops[0] == ("resample", 44100, 16000)


@needs_ref
def test_resampled_len_is_lhotse_output_length(lhotse_cuts):
    """`resampled_len` against the length lhotse's resampler returns, at lengths where the float32 quotient rounds across
    an integer and around them."""
    import math

    import torch
    from lhotse.augmentation.torchaudio import get_or_create_resampler

    from lhotse_b200.pcm_staging import _resample_geometry, resampled_len

    rs = np.random.RandomState(1)
    checked = crossing = 0
    for a, b in ((44100, 16000), (22050, 16000), (48000, 16000), (17600, 16000)):
        N, O, _, _ = _resample_geometry(a, b)
        lens = [L for L in range(180000, 400000) if resampled_len(N, L, O) != math.ceil(N * L / O)][:3]
        crossing += len(lens)
        for L in lens + [180697, 300001, 200000 + O]:
            y = get_or_create_resampler(a, b)(torch.from_numpy(rs.randn(L).astype(np.float32))[None])
            assert y.shape[-1] == resampled_len(N, L, O), (a, b, L)
            checked += 1
    assert crossing >= 6 and checked >= 12


@needs_ref
@pytest.mark.parametrize("pair", [(48000, 16000), (44100, 16000), (17600, 16000)], ids=lambda p: f"{p[0]}_{p[1]}")
def test_onednn_boundary(lhotse_cuts, pair):
    """A resampling stage's padded input L + 2 * width + O: 20480 elements is refused and torch does not run the conv
    through oneDNN; 20481 is taken, torch runs it through oneDNN, and lhotse's resampler equals the restatement bit for bit.
    48k -> 16k and 44.1k -> 16k are pairs whose outputs differ from the restatement on the im2col + sgemm side."""
    import torch
    import transform_cases
    from lhotse.augmentation.torchaudio import get_or_create_resampler

    from lhotse_b200.pcm_staging import _resample_geometry, resample_reference, transform_request_for_cut

    root, _ = lhotse_cuts
    a, b = pair
    N, O, w, K = _resample_geometry(a, b)
    resampler = get_or_create_resampler(a, b)
    speed = a == 17600  # Speed(1.1) on a 16 kHz file resamples 17600 -> 16000
    with transform_cases.torch_resampler():
        for n, taken in ((20480 - 2 * w - O, False), (20481 - 2 * w - O, True)):
            cut = transform_cases._cut(root, f"b{n}_{a}_{b}", n, 16000 if speed else a, seed=n)
            r = transform_request_for_cut(cut.perturb_speed(1.1) if speed else cut.resample(b))
            assert (r is not None) == taken, (a, b, n)
            x = np.asarray(cut.load_audio(), dtype=np.float32)[0]
            padded = torch.nn.functional.pad(torch.from_numpy(x)[None], (w, w + O))[:, None]
            backend = torch._C._select_conv_backend(padded, resampler.kernel, None, [O], [0], [1], False, [0], 1, None)
            assert (backend == torch._C._ConvBackend.Mkldnn) == taken, (a, b, n, backend)
            if taken:
                assert padded.shape[-1] == 20481
                with torch.no_grad():
                    y = resampler(torch.from_numpy(x)[None]).numpy()[0]
                assert np.array_equal(y.view(np.int32), resample_reference(x, a, b).view(np.int32))


@needs_ref
@pytest.mark.parametrize("pair", [(17600, 16000), (48000, 16000), (44100, 16000), (16000, 8000)], ids=lambda p: f"{p[0]}_{p[1]}")
def test_probe_passes_on_this_host(pair):
    refshim.import_reference()
    from lhotse_b200 import pcm_staging

    pcm_staging._PROBES.pop(pair, None)
    assert pcm_staging.resample_probe(*pair)


@needs_ref
def test_transform_route_refuses_what_it_cannot_reproduce(lhotse_cuts, monkeypatch):
    import torch
    import transform_cases as T
    from lhotse.audio.resampling_backend import set_current_resampling_backend
    from lhotse.augmentation import torchaudio as lta

    from lhotse_b200 import pcm_staging
    from lhotse_b200.pcm_staging import transform_request_for_cut, transform_requests_for_batch

    root, src = lhotse_cuts
    with T.torch_resampler():
        for name, cut in T.refused_cases(root, src).items():
            assert transform_request_for_cut(cut) is None, name
        ok_speed, ok_rs = src[16000][0].perturb_speed(1.1), src[48000].resample(16000)
        assert transform_request_for_cut(ok_speed) is not None and transform_request_for_cut(ok_rs) is not None
        # the sox backend: lhotse resamples with libsox
        set_current_resampling_backend("sox")
        try:
            assert transform_request_for_cut(ok_rs) is None
            assert transform_request_for_cut(ok_speed) is not None  # Speed always takes the torch resampler
        finally:
            set_current_resampling_backend("default")
        # a failing probe: this host's oneDNN would sum in another order
        monkeypatch.setattr(pcm_staging, "resample_probe", lambda a, b: False)
        assert transform_request_for_cut(ok_speed) is None
        monkeypatch.undo()
        # oneDNN off: the conv goes to another backend
        monkeypatch.setattr(torch.backends.mkldnn, "enabled", False)
        assert transform_request_for_cut(ok_speed) is None
        monkeypatch.undo()
    # no torchaudio: lhotse's Resample falls back to scipy in float64
    monkeypatch.setattr(lta, "is_torchaudio_available", lambda: False)
    assert transform_request_for_cut(ok_rs) is None
    monkeypatch.undo()
    # batches: plain slices alone keep their routes; a MixedCut or a refused cut sends the batch elsewhere
    with T.torch_resampler():
        assert transform_requests_for_batch([src[16000][0], src[16000][1]]) is None
        assert transform_requests_for_batch([src[16000][0], ok_speed]) is not None
        assert transform_requests_for_batch([ok_speed, src[16000][0].perturb_tempo(0.9)]) is None
        assert transform_requests_for_batch([ok_speed, src[16000][0].mix(src[16000][1], snr=10, allow_padding=True)]) is None


def test_chain_stages_keep_volume_where_it_sits():
    from lhotse_b200.pcm_staging import _chain_stages

    R, S = ("resample", 48000, 16000), ("resample", 17600, 16000)
    assert _chain_stages(()) == [(1.0, None, 1.0)]
    assert _chain_stages((("volume", 2.0), R)) == [(2.0, (48000, 16000), 1.0)]
    assert _chain_stages((R, ("volume", 2.0))) == [(1.0, (48000, 16000), 2.0)]
    assert _chain_stages((R, S)) == [(1.0, (48000, 16000), 1.0), (1.0, (17600, 16000), 1.0)]
    assert _chain_stages((("volume", 2.0), ("volume", 3.0), R)) == [(2.0, None, 3.0), (1.0, (48000, 16000), 1.0)]
    assert _chain_stages((R, ("volume", 2.0), ("volume", 3.0))) == [(1.0, (48000, 16000), 2.0), (3.0, None, 1.0)]


def test_fma_restatement_rounds_once():
    """_fma32 against an exact rational evaluation, on values whose float64 sum sits on a float32 midpoint."""
    from fractions import Fraction

    from lhotse_b200.pcm_staging import _fma32

    rs = np.random.RandomState(0)
    a = rs.randn(20000).astype(np.float32)
    b = rs.randn(20000).astype(np.float32)
    c = rs.randn(20000).astype(np.float32)
    # planted: a * b = +-2^-24 (1 - 2^-30), so that the float64 sum lands on the float32 midpoint next to c while the exact
    # value lies just inside, on the side whose float32 neighbour is odd (a second rounding of the float64 sum would tie
    # to the even one)
    a[:2] = np.float32(1 + 2.0 ** -15)
    b[:2] = np.asarray([2.0 ** -24 * (1 - 2.0 ** -15), -(2.0 ** -24) * (1 - 2.0 ** -15)], np.float32)
    c[:2] = np.asarray([1 + 2.0 ** -23, 1 + 3 * 2.0 ** -23], np.float32)
    got = _fma32(a, b, c)
    assert got[0] == np.float32(1 + 2.0 ** -23) and got[1] == np.float32(1 + 3 * 2.0 ** -23)
    for i in list(range(2)) + list(range(2, 20000, 97)):
        exact = Fraction(float(a[i])) * Fraction(float(b[i])) + Fraction(float(c[i]))
        lo = np.float32(float(exact))
        cands = [lo, np.nextafter(lo, np.float32(np.inf)), np.nextafter(lo, np.float32(-np.inf))]
        best = min(cands, key=lambda v: (abs(Fraction(float(v)) - exact), int(np.asarray(v).view(np.int32)) & 1))
        assert got[i] == best, (i, got[i], best)
