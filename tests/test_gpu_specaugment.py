"""SpecAugment on the GPU (csrc/specaug.cuh through b200feat_specaug and lhotse_b200.B200SpecAugment): the device output is
the host harness's, bit for bit; the module gives lhotse's SpecAugment under the same seeds (same masks, the input outside
masks and warps, the warp within lhotse's own float32 error) and leaves the generators where lhotse leaves them; malformed
tables are refused by the host checks before anything is launched; and the real caller, K2SpeechRecognitionDataset with
FusedOnTheFlyFeatures and the module as its input transform."""
import importlib

import numpy as np
import pytest
import torch

import refshim
import specaug_cases as SC

pytestmark = pytest.mark.gpu
needs_ref = pytest.mark.skipif(not refshim.reference_available(), reason="no reference tree / oracle/_ref archive")
DEV = "cuda:0"


@pytest.fixture(scope="module")
def harness(tmp_path_factory):
    exe = SC.build_harness(tmp_path_factory.mktemp("sah"))
    if exe is None:
        pytest.skip("no host C++ compiler")
    return exe


@pytest.fixture(scope="module")
def modules():
    if not refshim.reference_available():
        pytest.skip("no reference tree / oracle/_ref archive")
    import lhotse_env

    lhotse_env.setup_lhotse()
    import lhotse_b200.spec_augment as sa

    if not sa.HAVE_LHOTSE:
        importlib.reload(sa)
    from lhotse.dataset.signal_transforms import SpecAugment

    assert issubclass(sa.B200SpecAugment, SpecAugment)
    return SpecAugment, sa


def device_run(x, warps, masks):
    from lhotse_b200.engine import specaug

    xd = x.to(DEV)
    out = torch.full_like(xd, float("nan"))
    specaug(xd, out, warps, masks)
    torch.cuda.synchronize()
    assert torch.equal(xd.cpu(), x)  # the input is read only
    return out.cpu()


def plan_for(kw, x, segs, seed):
    import lhotse_b200.spec_augment as sa

    B, T, F = x.shape
    SC.seed_all(seed)
    return sa.spec_augment_plan(sa.B200SpecAugment(**kw), B, T, F, None if segs is None else sa.clipped_segments(segs, B, T))


@pytest.mark.parametrize("name", sorted(SC.CASES))
def test_device_equals_host_harness(harness, tmp_path, name):
    kw, x, segs = SC.case_input(name, 1)
    warps, masks = plan_for(kw, x, segs, 1)
    want, _ = SC.run_harness(harness, tmp_path, x, warps, masks)
    got = device_run(x, warps, masks)
    assert torch.equal(got.view(torch.int32), torch.from_numpy(want).view(torch.int32)), name
    assert torch.equal(device_run(x, warps, masks).view(torch.int32), got.view(torch.int32))  # the same bits from run to run


def test_device_equals_host_harness_on_a_recipe_shaped_batch(harness, tmp_path):
    """Several CTAs per sequence and a tile boundary inside warped segments: 24 x 1500 x 80 with default parameters."""
    lens = [1500 - 37 * b for b in range(24)]
    x = SC.make_batch(24, 1500, 80, lens, seed=9)
    warps, masks = plan_for({}, x, SC.one_segment_per_cut(lens), 4)
    assert len(warps) > 12 and len(masks) > 100
    want, _ = SC.run_harness(harness, tmp_path, x, warps, masks)
    assert torch.equal(device_run(x, warps, masks).view(torch.int32), torch.from_numpy(want).view(torch.int32))


@needs_ref
@pytest.mark.parametrize("name", sorted(SC.CASES))
def test_module_against_lhotse(modules, name):
    from lhotse_b200.engine import specaug

    SpecAugment, sa = modules
    kw, x, segs = SC.case_input(name, 2)
    SC.seed_all(2)
    L = SpecAugment(**kw)(x, supervision_segments=segs)
    after_lhotse = SC.rng_states()
    aug = sa.B200SpecAugment(**kw)
    xd = x.to(DEV)
    SC.seed_all(2)
    got = aug(xd, supervision_segments=segs)
    assert aug.last_route == "fused" and SC.rng_states() == after_lhotse
    assert got.shape == xd.shape and got.data_ptr() != xd.data_ptr() and torch.equal(xd.cpu(), x)
    warps, masks = plan_for(kw, x, segs, 2)
    unmasked = torch.empty_like(xd)
    specaug(xd, unmasked, warps, masks[:0])
    SC.check_against_lhotse(got.cpu().numpy(), unmasked.cpu().numpy(), x, L, warps, masks, name)
    # the same seeds, the same bits; on a stream of the caller's choice too
    SC.seed_all(2)
    assert torch.equal(aug(xd, supervision_segments=segs), got)
    side = torch.cuda.Stream(DEV)
    side.wait_stream(torch.cuda.current_stream(DEV))
    with torch.cuda.stream(side):
        SC.seed_all(2)
        again = aug(xd, supervision_segments=segs)
    side.synchronize()
    assert torch.equal(again, got)


@needs_ref
def test_declined_inputs_take_lhotse_forward_on_the_device(modules):
    SpecAugment, sa = modules
    kw, x, _ = SC.case_input("default_segments")
    xd = x.to(DEV)
    overlapping = torch.tensor([[0, 0, 400], [0, 300, 300], [1, 0, 600]], dtype=torch.int32)
    declined = {
        "overlapping segments": (xd, overlapping),
        "float64": (xd.double(), None),
        "not contiguous": (xd.transpose(1, 2).contiguous().transpose(1, 2), None),
        "cpu": (x, None),
    }
    for what, (inp, segs) in declined.items():
        SC.seed_all(3)
        want = SpecAugment(**kw)(inp, supervision_segments=segs)
        states = SC.rng_states()
        SC.seed_all(3)
        aug = sa.B200SpecAugment(**kw)
        got = aug(inp, supervision_segments=segs)
        assert aug.last_route == "lhotse" and torch.equal(got, want) and SC.rng_states() == states, what
    aug = sa.B200SpecAugment(**kw)
    aug(xd, supervision_segments=overlapping[1:])
    assert aug.last_route == "fused"


def test_unaligned_tensor_takes_the_scalar_kernel():
    """A (B, T, F) view that starts 4 bytes into an allocation: F % 4 == 0 but no 16-byte alignment.  The same values outside
    the masks as the aligned run, the mask value within an ulp (the partial sums are taken in another order)."""
    from lhotse_b200.engine import specaug

    kw, x, segs = SC.case_input("default_segments")
    warps, masks = plan_for(kw, x, segs, 1)
    aligned = device_run(x, warps, masks)
    flat = torch.empty(x.numel() + 1, dtype=torch.float32, device=DEV)
    view = flat[1:].view(x.shape)
    view.copy_(x)
    assert view.data_ptr() % 16 == 4
    out_flat = torch.empty(x.numel() + 1, dtype=torch.float32, device=DEV)
    out = out_flat[1:].view(x.shape)
    specaug(view, out, warps, masks)
    masked, _ = SC.regions(warps, masks, tuple(x.shape))
    got = out.cpu().numpy()
    assert np.array_equal(got[~masked].view(np.int32), aligned.numpy()[~masked].view(np.int32))
    assert np.abs(got[masked] - aligned.numpy()[masked]).max() <= 1e-6


def test_malformed_tables_are_refused_before_any_launch():
    from lhotse_b200.engine import SPECAUG_MASK_DTYPE, SPECAUG_WARP_DTYPE, B200FeatError, load_library, specaug

    lib = load_library()
    B, T, F = 3, 400, 80
    x = SC.make_batch(B, T, F).to(DEV)

    def tables(warps, masks):
        w = np.zeros(len(warps), SPECAUG_WARP_DTYPE)
        m = np.zeros(len(masks), SPECAUG_MASK_DTYPE)
        w["struct_size"], m["struct_size"] = 24, 24
        for i, r in enumerate(warps):
            w["seq"][i], w["start"][i], w["len"][i], w["center"][i], w["warped"][i] = r
        for i, r in enumerate(masks):
            m["seq"][i], m["axis"][i], m["start"][i], m["end"][i] = r
        return w, m

    good_w, good_m = [(0, 0, 400, 200, 230), (1, 50, 100, 40, 30), (1, 150, 250, 100, 101)], [(0, 0, 10, 20), (2, 1, 70, 80), (1, 0, 5, 5)]
    w, m = tables(good_w, good_m)
    out = torch.empty_like(x)
    specaug(x, out, w, m)
    torch.cuda.synchronize()
    good = out.clone()

    def bad_struct(which):
        w, m = tables(good_w, good_m)
        (w if which == "warp" else m)["struct_size"][1] = 20
        return w, m

    bad = {
        "warp sequence index": tables([(3, 0, 400, 200, 230)], []),
        "negative warp sequence index": tables([(-1, 0, 400, 200, 230)], []),
        "segment past T": tables([(0, 10, 391, 200, 230)], []),
        "negative segment start": tables([(0, -1, 100, 50, 40)], []),
        "empty segment": tables([(0, 0, 0, 0, 0)], []),
        "center at 0": tables([(0, 0, 400, 0, 30)], []),
        "center at len": tables([(0, 0, 400, 400, 30)], []),
        "warped at 0": tables([(0, 0, 400, 200, 0)], []),
        "warped at len": tables([(0, 0, 400, 200, 400)], []),
        "overlapping segments": tables([(1, 100, 100, 50, 40), (0, 0, 50, 20, 30), (1, 0, 101, 50, 40)], []),
        "mask sequence index": tables([], [(3, 0, 0, 10)]),
        "bad axis": tables([], [(0, 2, 0, 10)]),
        "time mask past T": tables([], [(0, 0, 390, 401)]),
        "feature mask past F": tables([], [(0, 1, 70, 81)]),
        "negative mask start": tables([], [(0, 1, -1, 5)]),
        "start past end": tables([], [(0, 0, 20, 10)]),
        "warp struct size": bad_struct("warp"),
        "mask struct size": bad_struct("mask"),
    }
    for name, (bw, bm) in bad.items():
        out.fill_(7.0)
        with pytest.raises(B200FeatError) as ei:
            specaug(x, out, bw, bm)
        assert ei.value.code == -1 and lib.b200feat_global_error().decode().startswith("specaug:"), name
        torch.cuda.synchronize()
        assert bool((out == 7.0).all()), name  # nothing was launched

    def raw(inp, outp, work, work_bytes, shape=(B, T, F)):
        stream = torch.cuda.current_stream(x.device).cuda_stream
        return lib.b200feat_specaug(None, inp, outp, *shape, w.ctypes.data, len(w), m.ctypes.data, len(m), work.data_ptr(), work_bytes, stream)

    need = int(lib.b200feat_specaug_work_bytes(B, T, F, len(w), len(m)))
    work = torch.empty(need, dtype=torch.uint8, device=DEV)
    out.fill_(7.0)
    for name, rc in (("in place", raw(x.data_ptr(), x.data_ptr(), work, need)),
                     ("overlapping buffers", raw(x.data_ptr(), x.data_ptr() + 4 * T * F, work, need, (2, T, F))),
                     ("work buffer too small", raw(x.data_ptr(), out.data_ptr(), work, need - 1)),
                     ("null input", raw(None, out.data_ptr(), work, need)),
                     ("zero frames", raw(x.data_ptr(), out.data_ptr(), work, need, (B, 0, F)))):
        assert rc == -1 and lib.b200feat_global_error().decode().startswith("specaug:"), name
    assert lib.b200feat_specaug_work_bytes(B, 0, F, 1, 1) == 0 and lib.b200feat_specaug_work_bytes(B, T, F, -1, 1) == 0
    torch.cuda.synchronize()
    assert bool((out == 7.0).all())
    assert raw(x.data_ptr(), out.data_ptr(), work, need) == 0
    torch.cuda.synchronize()
    assert torch.equal(out, good)  # the same tables after the refusals: the same bits


@needs_ref
def test_k2_dataset_with_fused_features_and_fused_specaugment(modules, tmp_path):
    """The real caller: DynamicBucketingSampler -> K2SpeechRecognitionDataset(FusedOnTheFlyFeatures, input_transforms=[...])
    over 2-30 s cuts, with B200SpecAugment against lhotse's SpecAugment under the same seeds, batch by batch.  lhotse's module
    runs ATen's CUDA bicubic kernel there, so warped frames agree to float32 interpolation error, everything else exactly or
    (the mask value: a float32 mean against a float64 one) to a few ulps."""
    import lhotse_env
    from lhotse.dataset import DynamicBucketingSampler, K2SpeechRecognitionDataset

    from lhotse_b200.input_strategies import FusedOnTheFlyFeatures

    SpecAugment, sa = modules
    lb_ex = lhotse_env.setup_lhotse()
    rs = np.random.RandomState(0)
    cuts = lhotse_env.make_cutset(tmp_path, np.round(rs.uniform(2.0, 30.0, size=40), 2).tolist(), seed=1)
    ext = lb_ex.B200Fbank(lb_ex.B200FbankConfig(device=DEV))
    got = {}
    for name, aug in (("lhotse", SpecAugment()), ("fused", sa.B200SpecAugment())):
        sampler = DynamicBucketingSampler(cuts, max_duration=200.0, num_buckets=5, shuffle=True, seed=0)
        ds = K2SpeechRecognitionDataset(input_strategy=FusedOnTheFlyFeatures(ext), input_transforms=[aug], return_cuts=True)
        out = []
        for i, batch_cuts in enumerate(sampler):
            SC.seed_all(100 + i)
            b = ds[batch_cuts]
            assert b["inputs"].is_cuda
            if name == "fused":
                assert aug.last_route == "fused"
            out.append((b["inputs"].cpu(), [c.id for c in b["supervisions"]["cut"]], SC.rng_states()))
        got[name] = out
    assert len(got["fused"]) == len(got["lhotse"]) >= 3
    for (a, ids_a, st_a), (l, ids_l, st_l) in zip(got["fused"], got["lhotse"]):
        assert ids_a == ids_l and a.shape == l.shape and st_a == st_l
        assert torch.allclose(a, l, rtol=0, atol=5e-3 * float(l.abs().max())), float((a - l).abs().max())
