"""The whisper-fbank backward without a GPU (csrc/backward.cuh, DESIGN.md §3.1p): the float64 restatement of the kernels'
adjoint chain against autograd through a float64 twin of the oracle's chain (itself pinned bitwise to the oracle), the tie
rules on exact ties, lhotse's own code when it is present, the header's code run on the host under AddressSanitizer, and
the ABI's refusals."""
import numpy as np
import pytest
import torch

import refshim
import whisper_backward_cases as WB
import whisper_backward_edge_cases as E
from oracle import whisper_oracle as W

KINDS = ("noise", "burst", "periodic", "silence")


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
@pytest.mark.parametrize("n", [201, 4000, 16080, 31999])
def test_twin_is_the_oracle_bit_for_bit(n, dtype):
    x = WB.waveform(n, "burst").astype(np.float32)
    for M in (80, 128):
        want = W.extract(x, M, dtype=dtype)
        got = WB.features_t(torch.as_tensor(x).to(dtype), M).numpy()
        assert got.dtype == want.dtype and np.array_equal(got, want), (n, M, dtype)


def _with_edges(base, ident):
    """`base` cases (n, kind, M), then those of every row of the edge table (whisper_backward_edge_cases.TABLE) not among
    them, as pytest params with ids `ident(n, kind, M, is_edge_row)`.  The hop-periodic tone runs at M = 80 and 128 only:
    its interior frames hold whole periods, so the filters between its harmonics see rounding-level leakage, and at other
    filter counts some of it lands just above the 1e-10 floor, where the log's 1 / v turns rounding into gradient."""
    seen = set(base)
    cases = [pytest.param(*c, id=ident(*c, False)) for c in base]
    for r in E.TABLE:
        for kind in KINDS:
            if kind == "periodic" and r.M not in (80, 128):
                continue
            if (r.n, kind, r.M) not in seen:
                seen.add((r.n, kind, r.M))
                cases.append(pytest.param(r.n, kind, r.M, id=ident(r.n, kind, r.M, True)))
    return cases


@pytest.mark.parametrize("n,kind,M", _with_edges([(n, kind, M) for n in WB.LENGTHS for kind in KINDS for M in (80, 128)],
                                                 lambda n, kind, M, edge: f"{n}-{kind}-{M}"))
def test_restatement_matches_float64_autograd(n, kind, M):
    x = WB.waveform(n, kind)
    G = np.random.RandomState(n + M).randn(W.num_rows(n), M)
    want = WB.autograd_grad(x, G, M)
    got = WB.restated_grad(x, G, M)
    if kind == "silence":
        assert not got.any() and not want.any()  # every mel energy is clamped: no gradient at all
        return
    assert WB.rel_err(got, want) < 1e-11, (n, kind, WB.rel_err(got, want))


def test_cases_exercise_the_decisions():
    """The burst routes mass through the clamp; the hop-periodic tone ties its maximum across interior frames."""
    n = 160080
    xr = WB.logmel_t(torch.tensor(WB.waveform(n, "burst"))).numpy()
    assert (xr < xr.max() - 8.0).mean() > 0.2
    xr = WB.logmel_t(torch.tensor(WB.waveform(n, "periodic"))).numpy()
    assert (xr == xr.max()).sum() > 100


def _torch_rules(x, G):
    """Step 1 under torch autograd, exactly as lhotse writes it."""
    xt = torch.tensor(x, dtype=torch.float64, requires_grad=True)
    y = (torch.maximum(xt, xt.max() - 8.0) + 4.0) / 4.0
    (y * torch.as_tensor(G, dtype=torch.float64)).sum().backward()
    return xt.grad.numpy()


@pytest.mark.parametrize("x,G", [
    ([1.0, 3.0, 3.0, -6.0, -5.0, -5.5], [4.0, 8.0, 16.0, 32.0, 64.0, 128.0]),  # the issue's example, g / 4 = [1, 2, 4, ...]
    ([0.0, -8.0, -8.0, -9.0, 0.0, 0.0, -2.0, -8.5], [1.0, 2.0, 3.0, 4.0, 5.0, 6.0, 7.0, 8.0]),  # three maxima, ties at m - 8
    ([2.0, 2.0, 2.0, 2.0], [1.0, -1.0, 2.0, 0.5]),  # every element is the maximum
    ([5.0, -3.0, -3.0, -3.0], [0.0, 8.0, 4.0, 2.0]),  # everything else tied at m - 8
])
def test_tie_rules_equal_torch_autograd(x, G):
    x, G = np.asarray(x), np.asarray(G)
    want = _torch_rules(x, G)
    got = WB.row_grad(x, float(x.max()), G)
    assert np.array_equal(got, want), (got, want)
    if len(x) == 6:
        assert np.array_equal(got, [1.0, 26.0, 28.0, 0.0, 8.0, 0.0])


def test_log10_clamp_adjoint_matches_torch_autograd_at_the_floor():
    """The clamp's decision is exact (the tie passes, below it nothing); torch's float64 log10 backward rounds its division
    its own way, so the values agree to an ulp."""
    v = np.asarray([1e-10, 1e-10 * (1 - 2 ** -52), 0.0, 2.5e-3, 1e-10 * (1 + 2 ** -52), 1.0, 3.7e-7])
    gx = np.asarray([1.0, 2.0, 4.0, 0.5, 0.25, 8.0, -1.5])
    vt = torch.tensor(v, requires_grad=True)
    torch.clamp(vt, min=1e-10).log10().backward(torch.as_tensor(gx))
    want = vt.grad.numpy()
    got = WB.log10_adjoint(v, gx)
    assert np.array_equal(got == 0.0, want == 0.0) and list(np.flatnonzero(got == 0.0)) == [1, 2]
    assert np.allclose(got, want, rtol=4e-16, atol=0.0)


@pytest.mark.reference
@pytest.mark.skipif(not refshim.reference_available(), reason="no reference tree / oracle/_ref archive")
@pytest.mark.parametrize("kind", ("noise", "burst", "periodic"))
def test_restatement_matches_lhotse_whisper_fbank_in_float64(kind):
    pytest.importorskip("transformers")
    refshim.install_librosa_standin()
    refshim.import_reference()
    from lhotse.features.whisper_fbank import WhisperFbank, WhisperFbankConfig

    for M in (80, 128):
        ref = WhisperFbank(WhisperFbankConfig(num_filters=M))
        ref.filters, ref.window = ref.filters.double(), ref.window.double()
        for n in (201, 16080, 160079):
            x = WB.waveform(n, kind)
            xt = torch.tensor(x, requires_grad=True)
            out = ref.extract(xt, 16000)
            G = np.random.RandomState(n).randn(*out.shape)
            (out * torch.as_tensor(G)).sum().backward()
            got = WB.restated_grad(x, G, M)
            assert WB.rel_err(got, xt.grad.numpy()) < 1e-11, (kind, M, n)


@pytest.fixture(scope="module")
def harness(tmp_path_factory):
    exe = WB.host_check_binary(tmp_path_factory.mktemp("wbwdh"))
    if exe is None:
        pytest.skip("no host C++ compiler")
    return exe


@pytest.mark.parametrize("n,kind,M", _with_edges([(n, kind, 80) for n in (201, 16000, 16079, 16080, 16159) for kind in KINDS],
                                                 lambda n, kind, M, edge: f"{n}-{kind}" + (f"-M{M}" if edge else "")))
def test_host_harness_matches_restatement(n, kind, M, harness, tmp_path):
    """The header's per-cut, per-frame and per-sample code in float32 on the CPU, with every buffer at its exact size,
    against the restatement taking its decisions on the same saved rows."""
    x = WB.waveform(n, kind).astype(np.float32).astype(np.float64)
    xr, m = WB.saved_rows(x, M)
    G = np.random.RandomState(n).randn(W.num_rows(n), M).astype(np.float32)
    got = WB.run_host_check(harness, tmp_path, x, xr, m, G, M)
    want = WB.restated_grad(x, G.astype(np.float64), M, xr=xr.astype(np.float64), m=m)
    assert got.shape == want.shape
    if kind == "silence":
        assert not got.any()
        return
    assert WB.rel_err(got, want) < 2e-4, (n, kind, WB.rel_err(got, want))


def test_host_harness_folds_the_centre_mirror(harness, tmp_path):
    """Rows of gradient on the first and last frames only, at lengths whose last frame reaches 40, 39, 2, 1 and 0 positions
    past the cut (n mod 160 = 0, 1, 38, 39, 40): every sample those frames reach through torch's mirror gets its share,
    samples 0 and n - 1 no mirror image, nothing between the two frames, and the header's fold agrees with the
    restatement's sample by sample at both ends."""
    for n, reach in ((960, 40), (961, 39), (998, 2), (999, 1), (1000, 0)):
        T = n // 160
        assert E.right_reach(n) == reach
        raw = np.arange(T)[:, None] * 160 - 200 + np.arange(400)[None, :]
        idx = WB.frame_index(n)
        assert int((raw[-1] >= n).sum()) == reach and int((raw >= n).sum()) == reach
        assert sorted(idx[-1][raw[-1] >= n]) == list(range(n - 1 - reach, n - 1))  # n - 41 + n mod 160 .. n - 2
        for i in (0, n - 1):  # each appears where its own padded position does, and nowhere else
            assert np.array_equal(idx == i, raw == i), (n, i)
        x = WB.waveform(n, "noise").astype(np.float32).astype(np.float64)
        xr, m = WB.saved_rows(x)
        G = np.zeros((W.num_rows(n), 80), dtype=np.float32)
        G[0], G[T - 1] = 1.0, -1.0
        got = WB.run_host_check(harness, tmp_path, x, xr, m, G)
        want = WB.restated_grad(x, G.astype(np.float64), 80, xr=xr.astype(np.float64), m=m)
        assert WB.rel_err(got, want) < 2e-4, (n, WB.rel_err(got, want))
        ends = np.r_[0:202, (T - 1) * 160 - 200:n]
        assert np.allclose(got[ends], want[ends], rtol=1e-3, atol=1e-4 * np.abs(want).max()), n
        assert not got[201:(T - 1) * 160 - 200].any()  # frame 0 reaches 200 (its image of 200), the last starts at 160 (T - 1) - 200


def test_abi_whisper_entries_refuse_bad_calls_without_a_gpu():
    from lhotse_b200 import engine

    lib = engine.load_library()
    ns = np.asarray([16000], dtype=np.int64)
    off = np.asarray([0], dtype=np.int64)
    rows = np.asarray([0, 100], dtype=np.int64)
    rc = lib.b200feat_whisper_backward(None, 16, 0, ns.ctypes.data, off.ctypes.data, 1, 16, 16, 16, rows.ctypes.data, 16, 16,
                                       1 << 20, None)
    assert rc == -1 and "null handle" in lib.b200feat_global_error().decode()
    assert lib.b200feat_extract_keep_raw(None, 16, 0, 16, 1, None, 16, 16, None) == -1
    for name in ("b200feat_whisper_backward", "b200feat_extract_keep_raw"):
        assert name in engine.EXPORTS
    # the frame-count contract the backward checks row_off and short cuts against (b200feat_desc_num_frames, no GPU)
    plan = __import__("lhotse_b200").build_plan("whisper-fbank", __import__("lhotse_b200").B200WhisperFbankConfig())
    assert engine.desc_num_frames(plan, 200) == -5 and engine.desc_num_frames(plan, 201) == 1
    assert engine.desc_num_frames(plan, 16079) == 100 and engine.desc_num_frames(plan, 16080) == 101
