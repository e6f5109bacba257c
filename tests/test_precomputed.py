"""Precomputed features on the CPU: the host plan of lhotse_b200/precomputed.py restates what lhotse's collate_features does
for archive-backed cuts (padding-only batches bit for bit, mixes within twice lhotse's own error of the float64 truth), it
declines what it cannot describe, the mix-law table matches each class's statics, the library refuses malformed tables, and
the arithmetic of csrc/featmix.cuh run on the host (scripts/micro/featmix_host_check.cu, under AddressSanitizer where the
toolchain has it) gives the float64 evaluation of the same tables."""
import ctypes as C
import math

import numpy as np
import pytest
import torch

import featmix_cases as FC
import refshim

needs_ref = pytest.mark.skipif(not refshim.reference_available(), reason="reference tree not present")


@pytest.fixture(scope="module")
def lhotse():
    if not refshim.reference_available():
        pytest.skip("reference tree not present")
    import lhotse_env

    lhotse_env.setup_lhotse()
    import lhotse

    return lhotse


@pytest.fixture(scope="module")
def harness(tmp_path_factory):
    exe = FC.build_harness(tmp_path_factory.mktemp("fmh"))
    if exe is None:
        pytest.skip("no host C++ compiler")
    return exe


def _mixed(tracks, cid="m"):
    from lhotse.cut import MixedCut

    return MixedCut(id=cid, tracks=tracks)


def _track(cut, offset=0.0, snr=None, mute=False, ref=False):
    from lhotse.cut import MixTrack

    return MixTrack(cut=cut, offset=offset, snr=snr, mute=mute, is_snr_reference=ref)


def _padding(n, F=80, value=-23.025850929940457):
    from lhotse.cut import PaddingCut

    return PaddingCut(id=f"pad{n}", duration=round(n * 0.01, 6), sampling_rate=16000, feat_value=value, num_frames=n,
                      num_features=F, frame_shift=0.01)


def batches(tmp_path):
    """name -> CutSet: every case the plan restates."""
    from lhotse import CutSet
    from lhotse.dataset import CutConcatenate, CutMix
    from lhotse.utils import fastcopy

    sp = FC.make_cuts(tmp_path / "a", [120, 95, 150, 60, 33, 1], seed=1)
    noise = FC.make_cuts(tmp_path / "a", [40, 260, 77, 1], seed=2, prefix="n", supervisions=False)
    lin = FC.make_cuts(tmp_path / "a", [90, 70, 40], seed=3, prefix="l", ftype="b200-spectrogram", kind="linear")
    lin_noise = FC.make_cuts(tmp_path / "a", [30, 120], seed=4, prefix="ln", ftype="b200-spectrogram", kind="linear",
                             supervisions=False)
    s = list(sp)
    out = {
        "plain": CutSet.from_cuts(s[:4]),
        "plain_one_frame": CutSet.from_cuts([s[5], s[4]]),
        "cutmix_p0": CutMix(noise, p=0.0, snr=(10, 20), seed=3)(sp),
        "cutmix_p05": CutMix(noise, p=0.5, snr=(10, 20), seed=4)(sp),
        "cutmix_p1_snr_none": CutMix(noise, p=1.0, snr=None, seed=5)(sp),
        "cutmix_p1_negative_snr": CutMix(noise, p=1.0, snr=(-10, 0), seed=6)(sp),
        "cutmix_linear": CutMix(lin_noise, p=1.0, snr=(0, 10), seed=7)(lin),
        "cutmix_linear_snr_none": CutMix(lin_noise, p=0.7, snr=None, seed=8)(lin),
        "append": CutSet.from_cuts([s[0].append(s[1]), s[2], s[3].append(s[4])]),
        "concatenate": CutConcatenate(gap=0.05)(CutSet.from_cuts(s[:5])),
        "pad": CutSet.from_cuts([s[0].pad(num_frames=140), s[1]]),
    }
    n = list(noise)
    # muted tracks, an explicit reference, a PaddingCut first, offsets on either side of a frame boundary.  Each mix is the
    # longest cut of its batch: lhotse pads a shorter MixedCut with muted tracks by nesting it in another MixedCut, which the
    # plan leaves to lhotse
    for m in (_mixed([_track(s[0]), _track(n[0], 0.125, snr=5, mute=True), _track(n[2], 0.135, snr=12)], "mu"),
              _mixed([_track(s[1], snr=3), _track(n[1], 0.004, ref=True), _track(n[0], 0.005, snr=8)], "rf"),
              _mixed([_track(s[2], snr=3), _track(n[2], 0.0, mute=True, ref=True), _track(n[0], 0.5, snr=8)], "rm"),
              _mixed([_track(_padding(20)), _track(s[3], 0.2), _track(n[0], 0.1, snr=10)], "pf"),
              _mixed([_track(s[4]), _track(n[3], 0.31, snr=4), _track(s[5], 0.1)], "of"),
              _mixed([_track(s[0], mute=True), _track(n[0], mute=True, snr=10)], "am")):
        out[f"tracks_{m.id}"] = CutSet.from_cuts([m, s[5]])
    # zero-row and one-frame tracks, partial reads, the +-1 adjustments of MonoCut and of the mix
    zero = s[2].truncate(offset=0.3, duration=0.004)
    part = s[2].truncate(offset=0.333, duration=0.5)
    long_by_one = fastcopy(s[3], duration=0.605)  # 60 stored rows, num_frames 61: the last row repeated
    out["edges"] = CutSet.from_cuts([
        _mixed([_track(part), _track(zero, 0.1, snr=10), _track(n[3], 0.2, snr=10)], "zr"),
        _mixed([_track(s[0].truncate(duration=1.125)), _track(s[1].truncate(duration=0.715), 1.125)], "tr"),
        _mixed([_track(s[0].truncate(duration=1.124)), _track(s[1].truncate(duration=0.714), 1.124)], "du"),
        _mixed([_track(long_by_one), _track(n[0], 0.2, snr=15)], "lb"),
        _mixed([_track(zero), _track(n[2], 0.0, snr=10)], "zb"),
        part,
        long_by_one,
    ])
    return out


@needs_ref
def test_plan_against_collate_features(lhotse, tmp_path):
    from lhotse_b200.precomputed import precomputed_plan

    seen_mix = seen_copy = 0
    for name, cuts in batches(tmp_path).items():
        plan = precomputed_plan(cuts)
        assert not isinstance(plan, str), (name, plan)
        l32, lens, truth = FC.lhotse_pair(cuts)
        assert lens.dtype == torch.int32 and torch.equal(lens, plan.lens), name
        ours = FC.host_evaluate(plan).astype(np.float32)
        mixes = int((plan.cuts["mode"] == FC.MIX).sum())
        seen_mix += mixes
        seen_copy += len(plan.cuts) - mixes
        if mixes == 0:
            assert torch.equal(torch.from_numpy(ours), l32), name
        else:
            FC.check_gate(ours, l32.numpy(), truth.numpy(), name)
        if name == "edges":  # a repeated last row and an energy-less zero-row track are really there
            assert ((plan.tracks["num_rows"] == plan.tracks["stored_rows"] + 1) & (plan.tracks["stored_rows"] > 0)).any()
        if name == "tracks_rm":  # the muted reference gives its energy only
            assert (plan.tracks["flags"] == FC.ENERGY).any()
    assert seen_mix > 20 and seen_copy > 10


@needs_ref
def test_plan_takes_lhotse_mix_length_adjustments(lhotse, tmp_path):
    """A concatenation one frame too long (trimmed) and one frame too short (last row repeated)."""
    from lhotse import CutSet

    from lhotse_b200.precomputed import precomputed_plan

    s = list(FC.make_cuts(tmp_path / "a", [120, 95], seed=1))
    cuts = CutSet.from_cuts([_mixed([_track(s[0].truncate(duration=1.125)), _track(s[1].truncate(duration=0.715), 1.125)], "tr"),
                             _mixed([_track(s[0].truncate(duration=1.124)), _track(s[1].truncate(duration=0.714), 1.124)], "du")])
    plan = precomputed_plan(cuts)
    assert not isinstance(plan, str)
    assert sorted((plan.cuts["mix_rows"] - plan.cuts["num_rows"]).tolist()) == [-1, 1]


@needs_ref
def test_declines_go_to_reference(lhotse, tmp_path):
    from lhotse import CutSet
    from lhotse.cut import MultiCut
    from lhotse.dataset import CutMix
    from lhotse.features.io import NumpyFilesWriter
    from lhotse.utils import fastcopy

    import lhotse_b200 as lb
    from lhotse_b200.precomputed import precomputed_plan

    sp = FC.make_cuts(tmp_path / "a", [50, 40, 30], seed=1)
    s = list(sp)
    # features in another backend
    with NumpyFilesWriter(tmp_path / "np") as w:
        x = np.random.RandomState(0).randn(40, 80).astype(np.float32)
        key = w.write("k", x)
        other = fastcopy(s[1], features=fastcopy(s[1].features, storage_type=w.name, storage_path=str(w.storage_path),
                                                    storage_key=key))
    cases = {
        "backend": CutSet.from_cuts([s[0], other]),
        "backend_in_a_track": CutSet.from_cuts([_mixed([_track(s[0]), _track(other, 0.0, snr=5)], "bt"), s[2]]),
        "multicut": CutSet.from_cuts([MultiCut(id="mc", start=0, duration=0.5, channel=[0, 1], features=s[0].features), s[1]]),
        "mix_law": CutMix(FC.make_cuts(tmp_path / "a", [20], seed=5, prefix="mf", ftype="b200-mfcc", supervisions=False), p=1.0,
                          snr=10, seed=1)(FC.make_cuts(tmp_path / "a", [30], seed=6, prefix="mm", ftype="b200-mfcc")),
        # stored rows two short of num_frames in a padded cut: the padding-only branch cannot fill it
        "short_rows": CutSet.from_cuts([fastcopy(s[1], duration=0.42), s[0]]),
    }
    for name, cuts in cases.items():
        why = precomputed_plan(cuts)
        assert isinstance(why, str), name
    assert isinstance(precomputed_plan(sp, pad_direction="left"), str)
    strategy = lb.FusedPrecomputedFeatures(features_on_device=False)
    from lhotse.dataset.collation import collate_features

    for cuts, pad in ((cases["backend"], "right"), (cases["backend_in_a_track"], "right"), (sp, "left"), (sp, "both")):
        feats, lens = strategy(cuts, pad_direction=pad)
        ref, ref_lens = collate_features(cuts, pad_direction=pad)
        assert strategy.last_batch_route == "reference" and strategy.last_decline
        assert torch.equal(feats, ref) and torch.equal(lens, ref_lens)
    with pytest.raises(Exception):  # lhotse raises on its own for the short rows
        strategy(cases["short_rows"])
    assert strategy.last_batch_route == "reference"


@needs_ref
def test_mix_law_table_matches_the_statics(lhotse):
    from lhotse_b200.precomputed import mix_laws

    rs = np.random.RandomState(0)
    a = (rs.randn(7, 5) - 3).astype(np.float32)
    b = (rs.randn(7, 5) - 2).astype(np.float32)
    laws = mix_laws()
    assert {FC.LOG, FC.LINEAR} == set(laws.values()) and len(laws) >= 10
    for cls, law in laws.items():
        for g in (0.25, 3.0):
            np.testing.assert_allclose(cls.mix(a, b, g), FC.law_mix(law, a, b, g), rtol=1e-6, atol=1e-6, err_msg=cls.__name__)
            np.testing.assert_allclose(cls.scale(a, g), FC.law_scale(law, a, g), rtol=1e-6, atol=1e-6, err_msg=cls.__name__)
        assert math.isclose(cls.compute_energy(a), FC.law_energy(law, a), rel_tol=1e-5, abs_tol=1e-6), cls.__name__


def _tables(n_cuts=1):
    from lhotse_b200.engine import FEATMIX_CUT_DTYPE, FEATMIX_TRACK_DTYPE

    tr = np.zeros(2 * n_cuts, dtype=FEATMIX_TRACK_DTYPE)
    cu = np.zeros(n_cuts, dtype=FEATMIX_CUT_DTYPE)
    tr["struct_size"], cu["struct_size"] = FEATMIX_TRACK_DTYPE.itemsize, FEATMIX_CUT_DTYPE.itemsize
    for c in range(n_cuts):
        tr[2 * c: 2 * c + 2]["cut"] = c
        tr[2 * c: 2 * c + 2]["flags"] = [FC.MIXED | FC.ENERGY, FC.MIXED | FC.ENERGY]
        tr[2 * c: 2 * c + 2]["stored_rows"] = tr[2 * c: 2 * c + 2]["num_rows"] = [10, 6]
        tr[2 * c + 1]["offset"] = 3
        tr[2 * c: 2 * c + 2]["src_elem"] = [0, 40]
        tr[2 * c: 2 * c + 2]["snr_factor"] = [math.nan, 0.1]
        cu[c] = (FEATMIX_CUT_DTYPE.itemsize, FC.MIX, FC.LOG, 10, 10, 2 * c, 2, 0, 0.0, 0)
    return tr, cu


def _call(tr, cu, F=4, T=10, src_elems=100, work=None):
    from lhotse_b200.engine import load_library

    lib = load_library()
    src = np.zeros(max(src_elems, 1), np.float32)
    out = np.zeros(len(cu) * T * F + 1, np.float32)
    wb = int(lib.b200feat_feature_mix_work_bytes(len(tr), len(cu))) if work is None else work
    scratch = np.zeros(max(wb, 1), np.uint8)
    rc = lib.b200feat_feature_mix(None, src.ctypes.data, src_elems, tr.ctypes.data, len(tr), cu.ctypes.data, len(cu), F,
                                  out.ctypes.data, T, C.c_float(0.0), scratch.ctypes.data, wb, None)
    return rc, lib.b200feat_global_error().decode()


@pytest.mark.parametrize("name", ["track_size", "cut_size", "cut_link", "flags", "rows", "stored_rows", "source", "mode", "law",
                                  "ref", "ref_energy", "snr_energy", "first_offset", "mix_rows", "adjust", "copy_tracks",
                                  "num_rows", "empty_further", "work", "cuts_limit"])
def test_abi_refuses_malformed_tables(name):
    tr, cu = _tables()
    kw = {}
    if name == "track_size":
        tr["struct_size"][1] = 8
    elif name == "cut_size":
        cu["struct_size"] = 4
    elif name == "cut_link":
        tr["cut"][1] = 1
    elif name == "flags":
        tr["flags"][1] = 4
    elif name == "rows":
        tr["offset"][1] = -1
    elif name == "stored_rows":
        tr["stored_rows"][1] = 3
    elif name == "source":
        tr["src_elem"][1] = 90
    elif name == "mode":
        cu["mode"] = 2
    elif name == "law":
        cu["law"] = 7
    elif name == "ref":
        cu["ref_track"] = 2
    elif name == "ref_energy":
        tr["flags"][0] = FC.MIXED
    elif name == "snr_energy":
        tr["flags"][1] = FC.MIXED
    elif name == "first_offset":
        tr["offset"][0] = 1
    elif name == "mix_rows":
        cu["mix_rows"] = 9
    elif name == "adjust":
        tr["num_rows"][1] = tr["stored_rows"][1] = 9
        cu["mix_rows"] = 12
    elif name == "copy_tracks":
        cu["mode"] = FC.COPY
    elif name == "num_rows":
        cu["num_rows"] = 11
    elif name == "empty_further":
        tr["num_rows"][1] = tr["stored_rows"][1] = 0
    elif name == "work":
        kw["work"] = 16
    elif name == "cuts_limit":
        tr, cu = _tables(65536)
        tr["src_elem"] = np.tile([0, 40], 65536)
    rc, msg = _call(tr, cu, **kw)
    assert rc == -1 and msg.startswith("feature_mix"), (name, rc, msg)


@needs_ref
def test_host_check_against_the_float64_tables(lhotse, harness, tmp_path):
    from lhotse_b200.plan import LOG_EPSILON
    from lhotse_b200.precomputed import FeatureStagingRing, precomputed_plan

    for name, cuts in batches(tmp_path).items():
        plan = precomputed_plan(cuts)
        staged, tracks = FeatureStagingRing(pin_memory=False).stage(plan)
        src = staged.numpy()
        truth = FC.evaluate(src, tracks, plan.cuts, plan.F, plan.T, LOG_EPSILON)
        got = FC.run_harness(harness, tmp_path, src, tracks, plan.cuts, plan.F, plan.T, LOG_EPSILON)
        err = np.abs(got.astype(np.float64) - truth)
        assert (err <= FC.ulp32(truth)).all(), (name, float(err.max()))
