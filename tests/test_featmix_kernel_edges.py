"""The feature-mix kernels at their edges (csrc/featmix.cuh, DESIGN.md §3.1m), against lhotse's own mixer in float64.

Without a GPU: the edge table (tests/featmix_edge_cases.py) reaches every reference choice, every branch of the first track's
scaling, a mix that adds nothing, the EPSILON clamp binding on part of a cut, and NaN / +-inf in every kind of row, read from
the table's own data; `featmix_cases.evaluate` equals lhotse's `_scale_features_for_snr` + `FeatureMixer` on every row; the
host harness (the header's code, under AddressSanitizer) matches `evaluate` under the NaN-aware gate.

On the H100, through `engine.feature_mix`: every row against `evaluate` and lhotse's mixer, run to run, each cut alone, the
sentinels around the output, the host harness within 1 ulp32; 127 to 257 cuts around the gain kernel's blocks, 65535 and
65540 cuts (the output kernel's grid-y stride); and FusedPrecomputedFeatures over archive rows holding NaN and +-inf against
lhotse's collate_features.

The gate: NaN exactly where the truth is NaN, +-inf equal, finite elements within ulp32(truth) (hand tables) or
2 E_cut + ulp32(truth) (strategy batches, E_cut over the finite elements)."""
import numpy as np
import pytest
import torch

import featmix_cases as FC
import featmix_edge_cases as E
import refshim

needs_ref = pytest.mark.skipif(not refshim.reference_available(), reason="lhotse (oracle/_ref/lhotse_ref.zip) not present")

SENTINEL = np.float32(-7.75e30)
GUARD = 32


@pytest.fixture(scope="module")
def table():
    return E.build(E.edge_cuts())


@pytest.fixture(scope="module")
def evaluated(table):
    return E.evaluate(table)


# ============================================================================= without a GPU
@pytest.fixture(scope="module")
def harness(tmp_path_factory):
    exe = FC.build_harness(tmp_path_factory.mktemp("fme"))
    if exe is None:
        pytest.skip("no host C++ compiler")
    return exe


def _harness(harness, tmp_path, tab):
    return FC.run_harness(harness, tmp_path, tab.src, tab.tracks, tab.table, E.F, tab.T, E.PAD)


def test_table_reaches_every_branch(table, evaluated):
    reached = {}
    for c, cut in enumerate(table.cuts):
        reached.setdefault((cut.mode, cut.law), set()).update(E.branches(cut, evaluated[c]))
    for law in (E.LOG, E.LINEAR):
        assert E.REQUIRED_BOTH_LAWS <= reached[(E.MIX, law)], (law, E.REQUIRED_BOTH_LAWS - reached[(E.MIX, law)])
    assert E.REQUIRED_LOG <= reached[(E.MIX, E.LOG)], E.REQUIRED_LOG - reached[(E.MIX, E.LOG)]
    assert E.REQUIRED_COPY <= reached[(E.COPY, E.LOG)], E.REQUIRED_COPY - reached[(E.COPY, E.LOG)]
    # the non-finite rows do reach the output, and finite elements remain beside them
    assert np.isnan(evaluated).any() and np.isposinf(evaluated).any() and np.isneginf(evaluated).any()
    for c, cut in enumerate(table.cuts):
        assert np.isfinite(evaluated[c]).any(), cut.name


def test_batch_tables():
    for n in E.BATCH_SIZES[:5]:
        tab = E.build(E.batch_cuts(n))
        assert len(tab.table) == n and tab.T == 2 and (tab.table["num_rows"] == 1).all()
        assert set(tab.table["mode"]) == {E.COPY, E.MIX} and set(tab.table["law"]) == {E.LOG, E.LINEAR}


def test_offsets_are_exact_frames(table):
    """lhotse_mix gives add_to_mix offsets in seconds; compute_num_frames turns each back into the table's frame offset."""
    from lhotse_b200.precomputed import _compute_num_frames

    offsets = {t.offset for cut in table.cuts for t in cut.tracks}
    assert max(offsets) >= 6
    for o in offsets:
        assert _compute_num_frames(o * E.FRAME_SHIFT, E.FRAME_SHIFT, E.SR) == o


@needs_ref
def test_evaluate_equals_lhotse_mix(table, evaluated):
    truth = E.lhotse_mix(table)
    with np.errstate(invalid="ignore"):
        E.nan_gate(evaluated, truth, 1e-12 * np.abs(np.where(np.isfinite(truth), truth, 0.0)), "evaluate vs lhotse")


def test_host_harness_matches_evaluate(table, evaluated, harness, tmp_path):
    got = _harness(harness, tmp_path, table)
    for c, cut in enumerate(table.cuts):
        E.ulp_gate(got[c], evaluated[c], f"host harness {cut.name}")
    tab = E.build(E.batch_cuts(257))
    E.ulp_gate(_harness(harness, tmp_path, tab), E.evaluate(tab), "host harness, 257 cuts")


# ============================================================================= on the H100
def _run(tab):
    """engine.feature_mix on `tab` into an output with sentinels on both sides, which must survive."""
    from lhotse_b200 import engine as EN

    dev = torch.device("cuda", 0)
    n = len(tab.table) * tab.T * E.F
    buf = torch.full((n + 2 * GUARD,), float(SENTINEL), dtype=torch.float32, device=dev)
    out = buf[GUARD: GUARD + n].view(len(tab.table), tab.T, E.F)
    src = torch.from_numpy(tab.src).to(dev) if tab.src.size else None
    EN.feature_mix(src, tab.tracks, tab.table, out, E.PAD)
    torch.cuda.synchronize()
    host = buf.cpu().numpy()
    assert (host[:GUARD] == SENTINEL).all() and (host[GUARD + n:] == SENTINEL).all(), "write outside the output"
    return out.cpu().numpy()


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.int32)


def _alone(tab, c):
    return _run(E.build([tab.cuts[c]], T=tab.T))[0]


def _copy_want(cut, T):
    want = np.full((T, E.F), np.float32(E.PAD))
    rows = cut.tracks[0].rows64().astype(np.float32)
    want[: cut.num_rows()] = np.float32(cut.pad_value)
    want[: len(rows)] = rows
    return want


@pytest.mark.gpu
def test_every_row_on_the_gpu(table, evaluated):
    got = _run(table)
    truth = E.lhotse_mix(table) if refshim.reference_available() else None
    for c, cut in enumerate(table.cuts):
        E.ulp_gate(got[c], evaluated[c], f"{cut.name} vs evaluate")
        if truth is not None:
            E.ulp_gate(got[c], truth[c], f"{cut.name} vs lhotse")
        if cut.mode == E.COPY:
            assert E.copy_bits_equal(got[c], _copy_want(cut, table.T)), cut.name
    again = _run(table)
    assert np.array_equal(_bits(got), _bits(again)), "not identical from run to run"
    for c, cut in enumerate(table.cuts):
        assert np.array_equal(_bits(_alone(table, c)), _bits(got[c])), f"{cut.name}: not the same alone"


@pytest.mark.gpu
def test_gpu_and_host_harness_within_one_ulp(table, harness, tmp_path):
    """CUDA's and glibc's float64 exp and log may differ in the last bit; the float32 results then differ by at most one
    ulp, on a few elements."""
    got = _run(table)
    host = _harness(harness, tmp_path, table)
    E.ulp_gate(got, host, "gpu vs host harness")
    differ = int((np.isfinite(host) & (got != host)).sum())
    print(f"gpu vs host harness: {differ} of {host.size} elements differ (by at most one ulp32)")


@pytest.mark.gpu
@pytest.mark.parametrize("n", E.BATCH_SIZES)
def test_batch_shapes(n):
    tab = E.build(E.batch_cuts(n))
    got = _run(tab)
    E.ulp_gate(got, E.evaluate(tab), f"{n} cuts")
    for c in sorted({0, 126, 127, 128, n - 2, n - 1, 65534, 65535} & set(range(n))):
        assert np.array_equal(_bits(_alone(tab, c)), _bits(got[c])), f"{n} cuts: cut {c} not the same alone"


# ---- the public strategy over archive rows holding NaN and +-inf -----------------------------------------------------------
@pytest.fixture(scope="module")
def lhotse():
    if not refshim.reference_available():
        pytest.skip("lhotse (oracle/_ref/lhotse_ref.zip) not present")
    import lhotse_env

    lhotse_env.setup_lhotse()
    import lhotse

    return lhotse


def _nonfinite_batches(tmp_path):
    from lhotse import CutSet
    from lhotse.dataset import CutMix

    from test_precomputed import _mixed, _track

    nan, inf = np.float32(np.nan), np.float32(np.inf)
    sp = FC.make_cuts(tmp_path / "a", [120, 95, 150, 60], seed=11,
                      cells={0: [(3, 7, nan)], 1: [(10, 0, inf)], 2: [(20, 79, -inf), (21, 5, -inf)]})
    noise = FC.make_cuts(tmp_path / "a", [40, 260, 77], seed=12, prefix="n", supervisions=False,
                         cells={0: [(5, 5, nan)], 1: [(100, 30, inf), (101, 31, -inf)]})
    lin = FC.make_cuts(tmp_path / "a", [90, 70, 40], seed=13, prefix="l", ftype="b200-spectrogram", kind="linear",
                       cells={0: [(1, 2, nan)], 1: [(7, 3, -inf)], 2: [(0, 0, inf)]})
    lin_noise = FC.make_cuts(tmp_path / "a", [30, 120], seed=14, prefix="ln", ftype="b200-spectrogram", kind="linear",
                             supervisions=False, cells={1: [(50, 10, -inf), (60, 11, nan)]})
    clean = FC.make_cuts(tmp_path / "a", [100, 30], seed=15, prefix="k")
    s, n, k = list(sp), list(noise), list(clean)
    out = {
        "cutmix": CutMix(noise, p=1.0, snr=(10, 20), seed=3)(sp),
        "cutmix_linear": CutMix(lin_noise, p=1.0, snr=(0, 10), seed=4)(lin),
        "copy": CutSet.from_cuts(s),
    }
    # the reference after the first track: NaN in the reference's rows, NaN / +inf / -inf in the first track's
    for m in (_mixed([_track(k[0], snr=3), _track(s[0], 0.1, ref=True)], "rn"),
              _mixed([_track(s[0], snr=3), _track(k[0], 0.05, ref=True), _track(n[2], 0.2, snr=10)], "fn"),
              _mixed([_track(s[1], snr=5), _track(k[0], 0.0, mute=True, ref=True), _track(n[1], 0.3, snr=8)], "fi"),
              _mixed([_track(s[2], snr=-2), _track(n[0], 0.5, ref=True)], "fm")):
        out[f"tracks_{m.id}"] = CutSet.from_cuts([m, k[1]])
    return out


@pytest.mark.gpu
@needs_ref
def test_strategy_over_nonfinite_rows(lhotse, tmp_path):
    import lhotse_b200 as lb

    strategy = lb.FusedPrecomputedFeatures(num_workers=2)
    seen = set()
    for name, cuts in _nonfinite_batches(tmp_path).items():
        feats, lens = strategy(cuts)
        assert strategy.last_batch_route == "archive", (name, strategy.last_decline)
        l32, ref_lens, truth = FC.lhotse_pair(cuts)
        assert torch.equal(lens, ref_lens), name
        got = feats.cpu().numpy()
        if name == "copy":
            assert E.copy_bits_equal(got, l32.numpy()), name
        t = truth.numpy()
        E.cut_gate(got, l32.numpy(), t, name)
        assert np.isnan(t).any() and np.isfinite(t).any(), name  # every batch carries NaN into its output, beside finite values
        seen |= {"+inf"} if np.isposinf(t).any() else set()
        seen |= {"-inf"} if np.isneginf(t).any() else set()
    assert seen == {"+inf", "-inf"}
