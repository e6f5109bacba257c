"""SpecAugment on the CPU: the host plan (lhotse_b200/spec_augment.py) draws what lhotse's SpecAugment draws and leaves the
three generators where lhotse leaves them, and the arithmetic of csrc/specaug.cuh, run on the host
(scripts/micro/specaug_host_check.cu, under AddressSanitizer where the toolchain has it), gives lhotse's output: the same
masked positions, the input bit for bit outside masks and warped segments, the warp within lhotse's own float32 error."""
import importlib

import numpy as np
import pytest
import torch

import refshim
import specaug_cases as SC

needs_ref = pytest.mark.skipif(not refshim.reference_available(), reason="reference tree not present")


@pytest.fixture(scope="module")
def harness(tmp_path_factory):
    exe = SC.build_harness(tmp_path_factory.mktemp("sah"))
    if exe is None:
        pytest.skip("no host C++ compiler")
    return exe


@pytest.fixture(scope="module")
def modules():
    """(lhotse's SpecAugment, lhotse_b200.spec_augment bound to it)."""
    if not refshim.reference_available():
        pytest.skip("reference tree not present")
    refshim.import_reference()
    import lhotse_b200.spec_augment as sa

    if not sa.HAVE_LHOTSE:
        importlib.reload(sa)
    assert sa.HAVE_LHOTSE
    from lhotse.dataset.signal_transforms import SpecAugment

    assert issubclass(sa.B200SpecAugment, SpecAugment)
    return SpecAugment, sa


def plan_for(sa, kw, x, segs):
    B, T, F = x.shape
    clipped = None if segs is None else sa.clipped_segments(segs, B, T)
    assert not isinstance(clipped, str) and (clipped is None or not sa.segments_overlap(clipped))
    return sa.spec_augment_plan(sa.B200SpecAugment(**kw), B, T, F, clipped)


@needs_ref
@pytest.mark.parametrize("name", sorted(SC.CASES))
def test_plan_and_host_kernels_against_lhotse(modules, harness, tmp_path, name):
    SpecAugment, sa = modules
    for seed in (1, 2):
        kw, x, segs = SC.case_input(name, seed)
        SC.seed_all(seed)
        L = SpecAugment(**kw)(x, supervision_segments=segs)
        after_lhotse = SC.rng_states()
        SC.seed_all(seed)
        warps, masks = plan_for(sa, kw, x, segs)
        assert SC.rng_states() == after_lhotse, name
        got, means = SC.run_harness(harness, tmp_path, x, warps, masks)
        unmasked, _ = SC.run_harness(harness, tmp_path, x, warps, masks[:0])
        SC.check_against_lhotse(got, unmasked, x, L, warps, masks, f"{name} seed {seed}")
        masked, _ = SC.regions(warps, masks, tuple(x.shape))
        for b in range(x.shape[0]):
            assert (got[b][masked[b]] == means[b]).all()
        assert np.array_equal(got[~masked].view(np.int32), unmasked[~masked].view(np.int32))


@needs_ref
def test_the_matrix_covers_its_corners(modules):
    """The cases draw what their names say: warps that vanish, masks that wrap, segments that are clipped."""
    _, sa = modules

    def plan(name, seed=1):
        kw, x, segs = SC.case_input(name, seed)
        SC.seed_all(seed)
        return plan_for(sa, kw, x, segs), x

    (w, m), x = plan("too_short_to_warp")
    assert list(w["seq"]) == [1] and w["len"][0] == 162  # t - factor > factor + 1 first holds at t = 2 * 80 + 2
    (w, m), _ = plan("warped_equals_center")
    assert 0 < len(w) < 36  # 36 segments at p = 1, a third of them draw warped == center
    (w, m), _ = plan("p0")
    assert len(w) == 0 and len(m) == 0
    for name in ("no_warp_none", "no_warp_zero"):
        (w, m), _ = plan(name)
        assert len(w) == 0 and len(m) > 0
    (w, m), _ = plan("clipped_by_T")
    assert sorted(zip(w["seq"].tolist(), w["start"].tolist(), w["len"].tolist())) == [(0, 300, 300), (1, 0, 600)]
    (w, m), _ = plan("no_feature_masks")
    assert (m["axis"] == 0).all() and len(m) > 0
    (w, m), _ = plan("short_batch_one_frame_mask")
    assert (np.bincount(m["seq"][m["axis"] == 0], minlength=3) <= 1).all()  # ceil(0.15 * 50 / 100) = 1 frame mask
    (w, m), _ = plan("several_supervisions")
    assert np.bincount(w["seq"], minlength=3).max() >= 2


def test_plan_without_lhotse_needs_no_reference():
    """The plan is pure host code: the three generators are the only state, and the tables only depend on them."""
    import lhotse_b200 as lb
    from lhotse_b200.engine import SPECAUG_MASK_DTYPE, SPECAUG_WARP_DTYPE

    aug = lb.B200SpecAugment()
    SC.seed_all(5)
    w1, m1 = lb.spec_augment_plan(aug, 8, 1000, 80, [(b, 0, 1000 - 50 * b) for b in range(8)])
    SC.seed_all(5)
    w2, m2 = lb.spec_augment_plan(aug, 8, 1000, 80, [(b, 0, 1000 - 50 * b) for b in range(8)])
    assert w1.dtype == SPECAUG_WARP_DTYPE and m1.dtype == SPECAUG_MASK_DTYPE and w1.itemsize == 24 and m1.itemsize == 24
    assert np.array_equal(w1, w2) and np.array_equal(m1, m2) and len(w1) > 0 and len(m1) > 0
    assert ((w1["center"] > 0) & (w1["center"] < w1["len"]) & (w1["warped"] > 0) & (w1["warped"] < w1["len"])).all()
    assert (w1["start"] + w1["len"] <= 1000).all() and (np.abs(w1["center"] - w1["warped"]) <= 80).all()
    t = m1[m1["axis"] == 0]
    f = m1[m1["axis"] == 1]
    assert (t["end"] <= 1000).all() and (f["end"] <= 80).all() and (m1["start"] < m1["end"]).all()
    # ceil(0.15 * 1000 / 100) = 2 frame masks per sequence of fewer than 150 // 2 frames each
    assert (t["end"] - t["start"] < 75).all() and (f["end"] - f["start"] < 27).all() and np.bincount(t["seq"]).max() <= 2


def test_segment_eligibility():
    from lhotse_b200.spec_augment import clipped_segments, segments_overlap

    segs = clipped_segments(torch.tensor([[0, 0, 100], [0, 100, 500], [1, 700, 10]], dtype=torch.int32), 2, 400)
    assert segs == [(0, 0, 100), (0, 100, 300), (1, 700, 0)] and not segments_overlap(segs)
    assert segments_overlap(clipped_segments(torch.tensor([[0, 0, 101], [0, 100, 50]]), 1, 400))
    assert segments_overlap(clipped_segments(torch.tensor([[0, 100, 50], [1, 0, 10], [0, 0, 400]]), 2, 400))
    assert not segments_overlap(clipped_segments(torch.tensor([[0, 0, 400], [1, 0, 400]]), 2, 400))
    assert not segments_overlap(clipped_segments(torch.tensor([[0, 0, 400], [0, 500, 0]]), 1, 400))  # empty after clipping
    for bad in (torch.tensor([[2, 0, 10]]), torch.tensor([[-1, 0, 10]]), torch.tensor([[0, -5, 10]]), torch.tensor([[0, 5, -1]]),
                torch.tensor([0, 5, 1]), torch.tensor([[0.0, 5.0, 1.0]])):
        assert isinstance(clipped_segments(bad, 2, 400), str)


@needs_ref
def test_declined_inputs_take_lhotse_forward(modules):
    """CPU tensors (and anything else the kernels do not take) go to lhotse's own forward: the same output and the same
    generator states as lhotse's module under the same seeds."""
    SpecAugment, sa = modules
    kw, x, segs = SC.case_input("default_segments")
    overlapping = torch.tensor([[0, 0, 400], [0, 300, 300]], dtype=torch.int32)
    for s in (segs, None, overlapping):
        SC.seed_all(3)
        want = SpecAugment(**kw)(x, supervision_segments=s)
        states = SC.rng_states()
        SC.seed_all(3)
        aug = sa.B200SpecAugment(**kw)
        got = aug(x, supervision_segments=s)
        assert aug.last_route == "lhotse" and torch.equal(got, want) and SC.rng_states() == states
    aug = sa.B200SpecAugment()
    assert aug.decline_reason(x, None) == "features is not a CUDA tensor"


def test_mirror_raises_where_lhotse_would_have_taken_the_batch():
    import lhotse_b200.spec_augment as sa

    if sa.HAVE_LHOTSE:
        pytest.skip("lhotse is importable: declined inputs go to its forward")
    aug = sa.B200SpecAugment()
    with pytest.raises(ValueError, match="not a CUDA tensor"):
        aug(torch.zeros(2, 100, 80))
    assert aug.last_route == "lhotse"


def test_constructor_assertions_and_state_dict():
    import lhotse_b200 as lb

    for bad in ({"p": 1.5}, {"p": -0.1}, {"num_feature_masks": -1}, {"num_frame_masks": -1}, {"features_mask_size": 0},
                {"frames_mask_size": 0}):
        with pytest.raises(AssertionError):
            lb.B200SpecAugment(**bad)
    aug = lb.B200SpecAugment(time_warp_factor=None, num_feature_masks=3, features_mask_size=11, num_frame_masks=4,
                             frames_mask_size=50, max_frames_mask_fraction=0.3, p=0.5)
    sd = aug.state_dict()
    assert sd == dict(time_warp_factor=None, num_feature_masks=3, features_mask_size=11, num_frame_masks=4, frames_mask_size=50,
                      max_frames_mask_fraction=0.3, p=0.5)
    other = lb.B200SpecAugment()
    assert other.state_dict() == dict(time_warp_factor=80, num_feature_masks=2, features_mask_size=27, num_frame_masks=10,
                                      frames_mask_size=100, max_frames_mask_fraction=0.15, p=0.9)
    other.load_state_dict(sd)
    assert other.state_dict() == sd
    other.load_state_dict({"p": 0.25})
    assert other.p == 0.25 and other.num_feature_masks == 3
    assert isinstance(aug, torch.nn.Module) and aug.last_route is None


@needs_ref
def test_state_dict_round_trip_with_lhotse(modules):
    SpecAugment, sa = modules
    theirs = SpecAugment(time_warp_factor=40, num_feature_masks=1, features_mask_size=13, num_frame_masks=3, frames_mask_size=70,
                         max_frames_mask_fraction=0.2, p=0.7)
    ours = sa.B200SpecAugment()
    ours.load_state_dict(theirs.state_dict())
    assert ours.state_dict() == theirs.state_dict()
    back = SpecAugment()
    back.load_state_dict(ours.state_dict())
    assert back.state_dict() == theirs.state_dict()


@needs_ref
def test_parameter_errors_are_lhotse_errors(modules):
    """What lhotse raises for a parameter combination, the plan raises from the same expression."""
    SpecAugment, sa = modules
    x = SC.make_batch(2, 300, 80)
    for kw in ({"num_frame_masks": 0, "p": 1.0}, {"features_mask_size": 0.5, "p": 1.0}, {"frames_mask_size": 1000, "max_frames_mask_fraction": 0.001, "p": 1.0}):
        SC.seed_all(0)
        with pytest.raises(Exception) as theirs:
            SpecAugment(**kw)(x)
        SC.seed_all(0)
        with pytest.raises(type(theirs.value)) as ours:
            sa.spec_augment_plan(sa.B200SpecAugment(**kw), 2, 300, 80, None)
        assert str(ours.value) == str(theirs.value)
