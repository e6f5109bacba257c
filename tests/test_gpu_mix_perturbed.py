"""MixedCuts with speed-, volume- and resample-perturbed tracks mixed on the GPU (`perturbed_tracks=True`): `mix_cuts`
bit-exact against float32(cut.load_audio()) on the perturbed case table and on a 2048-cut recipe-shaped batch; the real
callers (`FusedOnTheFlyFeatures` alone and inside K2SpeechRecognitionDataset over a speed-perturbed CutSet with CutMix,
`compute_and_store_features_fused`) against their float route; and the float32-source checks of `b200feat_mix_ex`."""
import os

import numpy as np
import pytest
import torch

import refshim

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = [os.path.join(ROOT, "tests", "golden", f"2412-153948-000{i}.flac") for i in (0, 1)]


@pytest.fixture(scope="module")
def env(tmp_path_factory):
    if not refshim.reference_available():
        pytest.skip("no reference tree / oracle/_ref archive")
    import lhotse_env
    import perturbed_mix_cases as P
    import transform_cases

    lb_ex = lhotse_env.setup_lhotse()
    root = tmp_path_factory.mktemp("gpmix")
    speech, noise, s48 = P.sources(root)
    with transform_cases.torch_resampler(), P.flac_backend():
        flac = P.flac_cuts(GOLDEN)
        yield lb_ex, root, speech, noise, P.cases(root, speech, noise, s48, flac)


def _check(cuts, ring=None):
    import perturbed_mix_cases as P

    from lhotse_b200 import mix_cuts

    buf, lens, offs = mix_cuts(cuts, "cuda:0", ring=ring, perturbed_tracks=True)
    assert buf.is_cuda and buf.dtype == torch.float32 and all(o % 4 == 0 for o in offs)
    host = buf.cpu().numpy()
    for c, o, n in zip(cuts, offs, lens):
        want = P.load_f32(c)
        assert want.shape == (n,) and np.array_equal(host[o:o + n].view(np.int32), want.view(np.int32)), c.id


def test_gpu_perturbed_mix_cuts_equal_load_audio(env):
    from lhotse_b200 import mix_cuts
    from lhotse_b200.pcm_staging import MixStagingRing

    _, _, speech, noise, cases = env
    cuts = [cases[k] for k in sorted(cases)] + [speech[0], speech[2].perturb_speed(0.9)]
    ring = MixStagingRing()
    _check(cuts, ring)
    _check(cuts[::-1], ring)  # the ring again, in another order
    with pytest.raises(ValueError):
        mix_cuts(cuts[:2], "cuda:0")  # the default refuses perturbed tracks


def test_gpu_perturbed_mix_cuts_2048_recipe_batch(env, tmp_path):
    """2048 cuts of 10-30 s at speed 0.9 / 1.0 / 1.1 under CutMix(p=0.5, snr 10-20): deep energy trees over float tracks."""
    import perturbed_mix_cases as P

    cuts = P.recipe_batch(tmp_path, 2048)
    assert 700 < sum(getattr(c, "tracks", None) is not None for c in cuts) < 1350
    _check(cuts)


def test_gpu_fused_on_the_fly_perturbed_mix_route_equals_float_route(env):
    from lhotse import CutSet
    from lhotse.dataset.signal_transforms import GlobalMVN

    from lhotse_b200.input_strategies import FusedOnTheFlyFeatures

    lb_ex, _, speech, noise, cases = env
    cuts = CutSet.from_cuts([cases[k] for k in sorted(cases) if k != "resampled_speech"] + [speech[0], speech[1].perturb_speed(1.1)])
    ext = lb_ex.B200Fbank(lb_ex.B200FbankConfig(device="cuda:0"))
    fast = FusedOnTheFlyFeatures(ext, perturbed_tracks=True)
    slow = FusedOnTheFlyFeatures(ext, pcm16_fast_path=False, perturbed_tracks=True)
    default = FusedOnTheFlyFeatures(ext)
    f1, l1 = fast(cuts)
    f2, l2 = slow(cuts)
    default(cuts)
    assert fast.last_batch_route == "mix" and slow.last_batch_route == "float" and default.last_batch_route == "float"
    assert torch.equal(l1, l2) and torch.equal(f1, f2)
    mvn = GlobalMVN(80)
    mvn.norm_means = torch.linspace(-3, 3, 80)
    mvn.norm_stds = torch.linspace(0.5, 2, 80)
    a = FusedOnTheFlyFeatures(ext, global_mvn=mvn, perturbed_tracks=True)
    g1, m1 = a(cuts)
    b = FusedOnTheFlyFeatures(ext, global_mvn=mvn, pcm16_fast_path=False)
    g2, m2 = b(cuts)
    assert a.last_batch_route == "mix" and b.last_batch_route == "float" and torch.equal(m1, m2) and torch.equal(g1, g2)
    ft = FusedOnTheFlyFeatures(ext, fault_tolerant=True, perturbed_tracks=True)
    h1, k1, kept = ft(cuts)
    assert ft.last_batch_route == "mix" and torch.equal(h1, f1) and len(kept) == len(cuts)
    # the resampled-speech case alone (its track starts from a 48 kHz file)
    one = CutSet.from_cuts([cases["resampled_speech"]])
    x1, _ = fast(one)
    x2, _ = slow(one)
    assert fast.last_batch_route == "mix" and torch.equal(x1, x2)
    # batches without MixedCuts keep their routes
    for batch, route in (([speech[0], speech[1]], "pcm16"), ([speech[0], speech[1].perturb_speed(1.1)], "transform")):
        s = FusedOnTheFlyFeatures(ext, perturbed_tracks=True)
        s(CutSet.from_cuts(batch))
        assert s.last_batch_route == route, route


def test_gpu_perturbed_cutmix_in_k2_dataset_equals_reference_strategy(env, tmp_path):
    import lhotse_env
    from lhotse.dataset import DynamicBucketingSampler, K2SpeechRecognitionDataset
    from lhotse.dataset.cut_transforms import CutMix
    from lhotse.dataset.input_strategies import OnTheFlyFeatures

    from lhotse_b200.input_strategies import FusedOnTheFlyFeatures

    lb_ex = env[0]
    rs = np.random.RandomState(0)
    cuts = lhotse_env.make_cutset(tmp_path, np.round(rs.uniform(2.0, 15.0, size=30), 2).tolist(), seed=1)
    cuts = cuts + cuts.perturb_speed(0.9) + cuts.perturb_speed(1.1)
    noise = lhotse_env.make_cutset(tmp_path, [1.5, 3.7, 8.2], seed=2, amp=0.05, supervisions=False, prefix="n")
    ext = lb_ex.B200Fbank(lb_ex.B200FbankConfig(device="cuda:0"))
    got = {}
    routes = set()
    for name, strategy in (("reference", OnTheFlyFeatures(ext)), ("fused", FusedOnTheFlyFeatures(ext, perturbed_tracks=True))):
        sampler = DynamicBucketingSampler(cuts, max_duration=60.0, num_buckets=3, shuffle=True, seed=0)
        ds = K2SpeechRecognitionDataset(input_strategy=strategy, return_cuts=True,
                                        cut_transforms=[CutMix(noise, p=0.5, snr=(10, 20), seed=5, preserve_id=True)])
        out = []
        for batch_cuts in sampler:
            b = ds[batch_cuts]
            out.append((b["inputs"].cpu(), b["supervisions"]["num_frames"].clone(), [c.id for c in b["supervisions"]["cut"]]))
            if name == "fused":
                routes.add(strategy.last_batch_route)
        got[name] = out
    assert "mix" in routes
    assert len(got["reference"]) == len(got["fused"])
    for (x1, n1, i1), (x2, n2, i2) in zip(got["reference"], got["fused"]):
        assert i1 == i2 and torch.equal(n1, n2) and torch.equal(x1, x2)


def test_gpu_store_route_over_perturbed_mixes_equals_the_reference_batch_store(env, tmp_path):
    from lhotse import CutSet
    from lhotse.features.io import NumpyFilesWriter

    from lhotse_b200.storage import compute_and_store_features_fused

    lb_ex, _, _, _, cases = env
    cuts = CutSet.from_cuts([cases[k].with_id(k) for k in sorted(cases)])
    ext = lb_ex.B200Fbank(lb_ex.B200FbankConfig(device="cuda:0"))
    want = cuts.compute_and_store_features_batch(ext, tmp_path / "ref", num_workers=0, batch_duration=20.0,
                                                 storage_type=NumpyFilesWriter, overwrite=True)
    calls = []
    orig = ext.extract_staged_packed
    ext.extract_staged_packed = lambda staged, *a, **k: calls.append(type(staged).__name__) or orig(staged, *a, **k)
    got = compute_and_store_features_fused(cuts, ext, tmp_path / "fused", manifest_path=tmp_path / "fused.jsonl.gz",
                                           batch_duration=20.0, num_workers=2, overwrite=True, perturbed_tracks=True)
    got = CutSet.from_cuts(list(got))
    assert calls and set(calls) == {"MixBatch"}
    assert [c.id for c in got] == [c.id for c in want]
    for g, w in zip(got, want):
        assert (g.num_frames, g.num_features) == (w.num_frames, w.num_features)
        assert np.array_equal(g.load_features(), w.load_features())


def test_gpu_mix_ex_argument_checks(env):
    import perturbed_mix_cases as P

    from lhotse_b200.engine import B200FeatError, MIX_SRC_F32, mix
    from lhotse_b200.pcm_staging import MixStagingRing, mix_requests_for_batch, transform_staged

    lb_ex, _, _, _, cases = env
    cuts = [cases["speed_1.1_snr_0"], cases["muted_perturbed_reference"], cases["mixed_then_speed_0.9"]]
    batch, lens, offs, _ = MixStagingRing(pin_memory=False).stage(mix_requests_for_batch(cuts, perturbed_tracks=True))
    ext = lb_ex.B200Fbank(lb_ex.B200FbankConfig(device="cuda:0"))
    h = ext.engine._h
    src0 = batch.pcm.cuda()
    src2 = transform_staged(batch.transform, "cuda:0", handle=h)[0]
    f32 = int(np.nonzero(batch.tracks["source"] == MIX_SRC_F32)[0][0])
    i16 = int(np.nonzero(batch.tracks["source"] == 0)[0][0])

    def run(tracks, cuts_t, s2=src2, out_elems=batch.out_elems):
        out = torch.zeros(max(out_elems, 1), dtype=torch.float32, device="cuda:0")
        mix(src0, None, tracks, cuts_t, out, h, src2=s2)
        torch.cuda.synchronize()
        return out.cpu()

    good = run(batch.tracks.copy(), batch.cuts.copy())
    for c, o, n in zip(cuts, offs, lens):
        assert torch.equal(good[o:o + n], torch.from_numpy(P.load_f32(c))), c.id

    def bad_tracks(field, value, i):
        t = batch.tracks.copy()
        t[field][i] = value
        return t, batch.cuts.copy()

    def bad_cuts(field, value, i=1):
        c = batch.cuts.copy()
        c[field][i] = value
        return batch.tracks.copy(), c

    def expect_einval(name, t, c, s2=src2):
        with pytest.raises(B200FeatError) as ei:
            run(t, c, s2)
        assert ei.value.code == -1 and ext.engine.lib.b200feat_last_error(h).decode().startswith("mix:"), name

    expect_einval("src2 missing", batch.tracks.copy(), batch.cuts.copy(), s2=None)
    expect_einval("track outside src2", *bad_tracks("src_elem", int(src2.numel()) - 10, f32))
    expect_einval("track past src2's end", *bad_tracks("num_samples", int(src2.numel()) + 1, f32))
    expect_einval("source index 3", *bad_tracks("source", 3, f32))
    # the bad tables of the int16 checks, through the new entry point
    for name, (t, c) in {
        "track outside its source": bad_tracks("src_elem", int(src0.numel()) - 10, i16),
        "negative source element": bad_tracks("src_elem", -1, f32),
        "source 1 missing": bad_tracks("source", 1, i16),
        "struct size": bad_tracks("struct_size", 40, f32),
        "bad role": bad_tracks("role", 7, f32),
        "track cut index": bad_tracks("cut", 9, f32),
        "cut outside its output": bad_cuts("out_elem", batch.out_elems - 5),
        "reference outside the cut's tracks": bad_cuts("ref_track", 5),
        "negative reference": bad_cuts("ref_track", -1),
        "tracks outside the table": bad_cuts("num_tracks", 99),
        "bad mode": bad_cuts("mode", 3),
        "mix_len": bad_cuts("mix_len", 5),
        "reflect longer than the mix": bad_cuts("target_len", 3 * int(batch.cuts["mix_len"][1])),
    }.items():
        expect_einval(name, t, c)
    with pytest.raises(B200FeatError):
        run(batch.tracks.copy(), batch.cuts.copy(), out_elems=batch.out_elems - 1)
    assert torch.equal(run(batch.tracks.copy(), batch.cuts.copy()), good)  # the same handle and stream, the same bits
