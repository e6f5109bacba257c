"""The RIR generator on the GPU (csrc/rirgen.cuh): each generated RIR against the float64 truth of the same draws within
twice lhotse's own float32 error; the generator states lhotse leaves; run-to-run identity; the "transform" and "mix" routes
within the §3.1j bound of a float64 reverb with the RIR they built; features through the gate in FusedOnTheFlyFeatures, the
recipe inside K2SpeechRecognitionDataset and the fused store; and the states put back when a staged batch falls back."""
import copy

import numpy as np
import pytest
import torch

import refshim
import reverb_cases as RC
import rirgen_cases as RG

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def env(tmp_path_factory):
    if not refshim.reference_available():
        pytest.skip("no reference tree / oracle/_ref archive")
    import lhotse_env
    import transform_cases

    lhotse_env.setup_lhotse()
    with transform_cases.torch_resampler():
        yield tmp_path_factory.mktemp("rirgen")


def _generate(gens):
    from lhotse_b200.pcm_staging import GeneratedRirRequest, GeneratedRirs, _generate_rirs

    g = GeneratedRirs([GeneratedRirRequest(x) for x in gens])
    g.draw()
    out = _generate_rirs(g, "cuda").cpu().numpy()
    return g, [out[e: e + n] for e, n in zip(g.elems, g.draws.lens)]


@pytest.mark.parametrize("case", RG.CASES)
def test_generated_rir_within_bound(env, case):
    gen = RG.generator(*case)
    torch.manual_seed(1234 + case[2])
    state = torch.get_rng_state()
    ref_rir, ref_gen, ref_state = RG.lhotse_rir(gen)
    torch.set_rng_state(state)
    g, (ours,) = _generate([gen])
    assert torch.equal(torch.get_rng_state(), ref_state)
    assert gen.room_rng.bit_generator.state == ref_gen.room_rng.bit_generator.state
    assert gen.source_rng.bit_generator.state == ref_gen.source_rng.bit_generator.state
    assert ours.shape == ref_rir.shape
    image = 2 * case[0]
    d = g.draws
    truth, _, _ = RG.truth64(d.records[0], d.draws[:image], d.draws[image: 2 * image], gen)
    err, bnd = RG.bound(ours, ref_rir, truth)
    assert err <= bnd, (err, bnd)


def test_generated_rirs_batch_identical_from_run_to_run(env):
    gens = [RG.generator(16000, 0.8, 100 + i, 200 + i) for i in range(40)]
    torch.manual_seed(5)
    a = _generate([copy.deepcopy(x) for x in gens])[1]
    torch.manual_seed(5)
    b = _generate([copy.deepcopy(x) for x in gens])[1]
    for x, y in zip(a, b):
        assert np.array_equal(x.view(np.int32), y.view(np.int32))


def _rirs_for(cuts, state, perturbed=True):
    """The generated RIRs a staged batch over `cuts` (copies no route has drawn from) builds from torch state `state`,
    keyed by id of their generator; torch's state is put back."""
    from lhotse_b200.pcm_staging import GeneratedRirs, _generate_rirs, _generated_in, staged_route

    reqs = staged_route(cuts, perturbed_tracks=perturbed, generated_rir=True)[1]
    keep = torch.get_rng_state()
    torch.set_rng_state(state)
    gen = GeneratedRirs(_generated_in(reqs))
    gen.draw()
    buf = _generate_rirs(gen, "cuda:0").cpu().numpy()
    torch.set_rng_state(keep)
    return {id(r.generator): buf[e: e + n] for r, e, n in zip(gen.reqs, gen.elems, gen.draws.lens)}


def _reverb_of(c):
    from lhotse.augmentation.rir import ReverbWithImpulseResponse

    tfs = c.transforms if getattr(c, "tracks", None) is not None else getattr(c.recording, "transforms", None)
    t = (tfs or [None])[-1]
    return t if isinstance(t, ReverbWithImpulseResponse) and t.rir is None else None


def _truth(c, rirs):
    """(float64 truth, lhotse's float32 arithmetic) of a cut's samples: a generated-RIR reverb of its pre-reverb samples
    (RC.truth64 / RC.lhotse32 with that RIR); a cut without one is what the float route reads."""
    import test_gpu_reverb as GR
    from lhotse.utils import fastcopy

    from lhotse_b200.pcm_staging import transform_request_for_cut

    t, n = _reverb_of(c), c.num_samples
    if t is None:
        x = np.asarray(c.load_audio(), np.float32)[0]
        return x.astype(np.float64), x
    if getattr(c, "tracks", None) is not None:
        x = np.asarray(fastcopy(c, transforms=None).load_audio(), np.float32)[0]
    else:
        x = GR._pre_reverb(transform_request_for_cut(c, generated_rir=True))
    q = rirs[id(t.rir_generator)] * np.float32(32768)  # the float32 RIR as the helpers' q / 32768, exactly
    return RC.truth64(x, q, t.normalize_output, n), RC.lhotse32(x, q, t.normalize_output, n)


def _route_within_bound(cuts, run, perturbed):
    """`run` on copies of the cuts, twice from one torch state: the §3.1j bound per cut against the float64 reverb with the
    RIR the route built, the same bits both times, and torch's state after equal to lhotse's load_audio() of the batch."""
    state = torch.get_rng_state()
    rirs_cuts = copy.deepcopy(cuts)
    rirs = _rirs_for(rirs_cuts, state, perturbed)
    outs = []
    for _ in range(2):
        torch.set_rng_state(state)
        out, lens, offs = run(copy.deepcopy(cuts))
        outs.append(out.cpu().numpy())
    after = torch.get_rng_state()
    torch.set_rng_state(state)
    for c in copy.deepcopy(cuts):
        c.load_audio()
    assert torch.equal(torch.get_rng_state(), after)
    assert np.array_equal(outs[0].view(np.int32), outs[1].view(np.int32))
    for c, o, n in zip(rirs_cuts, offs, lens):
        truth, ref32 = _truth(c, rirs)
        if _reverb_of(c) is None:
            assert np.array_equal(outs[0][o: o + n], ref32)
        else:
            RC.check(outs[0][o: o + n], truth, ref32, c.id)


def _speech(env):
    import test_reverb

    return test_reverb.make_sources(env)[0]


def test_transform_route_with_generated_rir(env):
    from lhotse_b200.pcm_staging import staged_route, transform_cuts

    c0, c1, c2 = _speech(env)
    cuts = [c0.reverb_rir(room_rng_seed=10, source_rng_seed=20), c1.perturb_speed(1.1).reverb_rir(room_rng_seed=11),
            c2.reverb_rir(normalize_output=False, room_rng_seed=12, source_rng_seed=22), c1]
    assert staged_route(cuts, generated_rir=False) is None
    assert staged_route(cuts, reverb=True) is None
    assert staged_route(cuts, generated_rir=True)[0] == "transform"
    torch.manual_seed(9)
    _route_within_bound(cuts, lambda cs: transform_cuts(cs, generated_rir=True), False)


def test_mix_route_with_generated_rir(env):
    from lhotse_b200.pcm_staging import mix_cuts, staged_route

    c0, c1, c2 = _speech(env)
    cuts = [c0.mix(c1, snr=10, allow_padding=True).reverb_rir(room_rng_seed=3, source_rng_seed=4),
            c2.reverb_rir(room_rng_seed=5, source_rng_seed=6),
            c1.perturb_speed(0.9).reverb_rir(normalize_output=False, room_rng_seed=7, source_rng_seed=8), c2]
    assert staged_route(cuts, perturbed_tracks=True) is None
    assert staged_route(cuts, perturbed_tracks=True, generated_rir=True)[0] == "mix"
    torch.manual_seed(9)
    _route_within_bound(cuts, lambda cs: mix_cuts(cs, perturbed_tracks=True, generated_rir=True), True)


@pytest.fixture
def one_thread():
    n = torch.get_num_threads()
    torch.set_num_threads(1)  # lhotse's comb keeps the last image at a shared position only with one thread
    yield
    torch.set_num_threads(n)


def _gate(cuts, rirs, ours, ext, frames):
    """Each cut's features through helpers.gate against the float64 oracle on the float64 truth samples, with the RIR the
    route built (the RIR itself is held to its own float64 bound above): the fp32 reference is the extractor on lhotse's
    float32 reverb arithmetic with that RIR (RC.lhotse32), as for a recorded RIR.  (lhotse's own generated RIR is within
    about 1e-4 of the truth of its draws, which moves log-mels by more than the gate's tolerance units; comparing with the
    float route's features would measure that, not this route.)"""
    from helpers import gate
    from oracle import kaldi_oracle as O

    for i, c in enumerate(cuts):
        t = int(frames[i])
        x64, x32 = _truth(c, rirs)
        truth = O.extract(x64, O.OracleConfig(), dtype=torch.float64)
        assert truth.shape[0] == t, (c.id, truth.shape, t)
        ref32 = ext.extract_batch_padded([torch.from_numpy(np.asarray(x32, np.float32))], c.sampling_rate)[0][0][:t]
        ok, msg = gate(ours[i][:t].cpu().numpy(), ref32.cpu().numpy(), truth, "fbank")
        assert ok, (c.id, msg)


def test_fused_on_the_fly_generated_rir_routes(env, one_thread):
    import lhotse_env
    from lhotse import CutSet

    from lhotse_b200.input_strategies import FusedOnTheFlyFeatures

    lb_ex = lhotse_env.setup_lhotse()
    ext = lb_ex.B200Fbank(lb_ex.B200FbankConfig(device="cuda:0"))
    c0, c1, c2 = _speech(env)
    batches = {
        "transform": [c0.reverb_rir(room_rng_seed=1), c1.perturb_speed(1.1).reverb_rir(room_rng_seed=2), c2],
        "mix": [c0.mix(c1, snr=10, allow_padding=True).reverb_rir(room_rng_seed=3), c2.reverb_rir(room_rng_seed=4), c1,
                c0.perturb_speed(0.9).reverb_rir(normalize_output=False, room_rng_seed=5)],
    }
    for route, batch in batches.items():
        torch.manual_seed(3)
        state = torch.get_rng_state()
        rirs_cuts = copy.deepcopy(batch)
        rirs = _rirs_for(rirs_cuts, state)
        res = {}
        for name, kw in (("on", dict(generated_rir=True, perturbed_tracks=True)), ("off", dict(perturbed_tracks=True)),
                         ("float", dict(pcm16_fast_path=False))):
            torch.set_rng_state(state)
            st = FusedOnTheFlyFeatures(ext, **kw)
            f, l = st(CutSet.from_cuts(copy.deepcopy(batch)))
            res[name] = (f, l, st.last_batch_route, torch.get_rng_state())
        assert res["on"][2] == route and res["off"][2] == "float" and res["float"][2] == "float"
        assert torch.equal(res["off"][0], res["float"][0])  # generated_rir=False: exactly the float route
        assert torch.equal(res["on"][3], res["float"][3]) and torch.equal(res["off"][3], res["float"][3])
        _gate(rirs_cuts, rirs, res["on"][0], ext, res["on"][1])
        # a staged batch that fails after its draws falls back with every state restored: the float route's features
        torch.set_rng_state(state)
        st = FusedOnTheFlyFeatures(ext, generated_rir=True, perturbed_tracks=True, fault_tolerant=True)
        st.extractor = _Failing(ext)
        f, l, _ = st(CutSet.from_cuts(copy.deepcopy(batch)))
        assert st.last_batch_route == "float" and torch.equal(f, res["float"][0])
        assert torch.equal(torch.get_rng_state(), res["float"][3])


class _Failing:
    """An extractor whose staged extraction raises (as a broken file would), the rest delegated."""

    def __init__(self, ext):
        self._ext = ext

    def extract_staged_padded(self, *a, **k):
        raise ValueError("staged extraction failed")

    def __getattr__(self, name):
        return getattr(self._ext, name)


@pytest.fixture
def seeded_lhotse(monkeypatch):
    """Unseeded RIR generators and MixedCut room seeds drawn from counters, so that two runs of a dataset build the same
    generators in the same order (lhotse seeds them from the OS and from uuid4 otherwise)."""
    import itertools
    import uuid

    import lhotse.cut.mixed as mixed
    from lhotse.augmentation.utils import FastRandomRIRGenerator

    orig = FastRandomRIRGenerator.__post_init__

    def reset():
        seeds, uids = itertools.count(1000), itertools.count(1)

        def post_init(self):
            if self.room_seed is None:
                self.room_seed = next(seeds)
            if self.source_seed is None:
                self.source_seed = next(seeds)
            orig(self)

        monkeypatch.setattr(FastRandomRIRGenerator, "__post_init__", post_init)
        monkeypatch.setattr(mixed, "uuid4", lambda: uuid.UUID(int=next(uids)))

    return reset


class _Recording:
    """A FusedOnTheFlyFeatures that keeps, per batch, copies of its cuts and torch's state from before it drew."""

    def __init__(self, inner):
        self.inner, self.seen = inner, []

    def __call__(self, cuts, *a, **k):
        self.seen.append((copy.deepcopy(list(cuts)), torch.get_rng_state()))
        return self.inner(cuts, *a, **k)

    def __getattr__(self, name):
        return getattr(self.inner, name)


def test_generated_rir_cutmix_in_k2_dataset(env, tmp_path, one_thread, seeded_lhotse):
    """The recipe with no RIR corpus: speed perturbation 0.9 / 1.0 / 1.1, CutMix(p=0.5), ReverbWithImpulseResponse(p=0.5),
    under DynamicBucketingSampler.  Every batch stays staged, torch's state after every batch is the float route's, the
    features pass the gate and are the same from run to run, and generated_rir=False gives the float route's outputs."""
    import random

    import lhotse_env
    from lhotse.dataset import DynamicBucketingSampler, K2SpeechRecognitionDataset
    from lhotse.dataset.cut_transforms import CutMix, ReverbWithImpulseResponse
    from lhotse.dataset.input_strategies import OnTheFlyFeatures

    from lhotse_b200.input_strategies import FusedOnTheFlyFeatures

    lb_ex = lhotse_env.setup_lhotse()
    rs = np.random.RandomState(0)
    cuts = lhotse_env.make_cutset(tmp_path, np.round(rs.uniform(2.0, 15.0, size=16), 2).tolist(), seed=1)
    cuts = cuts + cuts.perturb_speed(0.9) + cuts.perturb_speed(1.1)
    noise = lhotse_env.make_cutset(tmp_path, [1.5, 3.7, 8.2], seed=2, amp=0.05, supervisions=False, prefix="n")
    ext = lb_ex.B200Fbank(lb_ex.B200FbankConfig(device="cuda:0"))

    def run(strategy):
        seeded_lhotse()
        torch.manual_seed(17)
        sampler = DynamicBucketingSampler(cuts, max_duration=60.0, num_buckets=3, shuffle=True, seed=0)
        ds = K2SpeechRecognitionDataset(input_strategy=strategy, return_cuts=True, cut_transforms=[
            CutMix(noise, p=0.5, snr=(10, 20), seed=5, preserve_id=True),
            ReverbWithImpulseResponse(p=0.5, randgen=random.Random(7), preserve_id=True)])
        out, routes = [], []
        for batch_cuts in sampler:
            b = ds[batch_cuts]
            out.append((b["inputs"].cpu(), b["supervisions"]["num_frames"].clone(), torch.get_rng_state()))
            routes.append(getattr(strategy, "last_batch_route", None))
        return out, routes

    from lhotse import CutSet

    ref, _ = run(OnTheFlyFeatures(ext))
    rec = _Recording(FusedOnTheFlyFeatures(ext, perturbed_tracks=True, generated_rir=True))
    fused, routes = run(rec)
    assert "float" not in routes and len(ref) == len(fused) == len(rec.seen), routes
    again, off, flt = (FusedOnTheFlyFeatures(ext, perturbed_tracks=True, generated_rir=True),
                       FusedOnTheFlyFeatures(ext, perturbed_tracks=True), FusedOnTheFlyFeatures(ext, pcm16_fast_path=False))

    def rerun(strategy, bcuts, state):
        torch.set_rng_state(state)
        return strategy(CutSet.from_cuts(copy.deepcopy(bcuts)))[0].cpu()

    generated = 0
    for (_, n0, s0), (x1, n1, s1), (bcuts, state) in zip(ref, fused, rec.seen):
        assert torch.equal(s0, s1) and torch.equal(n0, n1)  # torch's state after every batch is the float route's
        has = any(_reverb_of(c) is not None for c in bcuts)
        x2, x3, x4 = rerun(again, bcuts, state), rerun(off, bcuts, state), rerun(flt, bcuts, state)
        assert torch.equal(x1, x2)  # the same batch from the same states: the same bits
        assert torch.equal(x3, x4) and off.last_batch_route == ("float" if has else rec.inner.last_batch_route)
        rirs = _rirs_for(bcuts, state) if has else {}
        generated += len(rirs)
        _gate(bcuts, rirs, x1, ext, [int(ext.engine.plan.num_frames(np.asarray([c.num_samples]))[0]) for c in bcuts])
    assert generated > 0


def test_store_route_over_generated_rir_cuts(env, tmp_path, one_thread):
    from lhotse import CutSet

    import lhotse_env
    from lhotse_b200.input_strategies import FusedOnTheFlyFeatures
    from lhotse_b200.storage import compute_and_store_features_fused

    lb_ex = lhotse_env.setup_lhotse()
    c0, c1, c2 = _speech(env)
    cuts = [c0.reverb_rir(room_rng_seed=1).with_id("a"), c1.perturb_speed(1.1).reverb_rir(room_rng_seed=2).with_id("b"),
            c0.mix(c2, snr=10, allow_padding=True).reverb_rir(room_rng_seed=3).with_id("c"), c2.with_id("d")]
    ext = lb_ex.B200Fbank(lb_ex.B200FbankConfig(device="cuda:0"))
    torch.manual_seed(21)
    state = torch.get_rng_state()
    # the on-the-fly "mix" route (gated against the float route above) and the float route's generator state, from the same
    # state: the store runs the same staging and kernels, so its features are those bits
    ref, ref_lens = FusedOnTheFlyFeatures(ext, perturbed_tracks=True, generated_rir=True)(CutSet.from_cuts(copy.deepcopy(cuts)))
    torch.set_rng_state(state)
    FusedOnTheFlyFeatures(ext, pcm16_fast_path=False)(CutSet.from_cuts(copy.deepcopy(cuts)))
    after = torch.get_rng_state()
    torch.set_rng_state(state)
    calls = []
    orig = ext.extract_staged_packed
    ext.extract_staged_packed = lambda staged, *a, **k: calls.append(type(staged).__name__) or orig(staged, *a, **k)
    got = compute_and_store_features_fused(CutSet.from_cuts(copy.deepcopy(cuts)), ext, tmp_path / "fused",
                                           manifest_path=tmp_path / "fused.jsonl.gz", batch_duration=200.0, num_workers=2,
                                           overwrite=True, generated_rir=True, perturbed_tracks=True)
    got = CutSet.from_cuts(list(got))
    assert calls == ["MixBatch"] and torch.equal(torch.get_rng_state(), after)
    assert [c.id for c in got] == [c.id for c in cuts]
    feats = [torch.from_numpy(g.load_features()) for g in got]
    assert [f.shape[0] for f in feats] == ref_lens.tolist()
    for f, r, n in zip(feats, ref.cpu(), ref_lens.tolist()):
        assert torch.equal(f, r[:n])


def test_fallback_after_drawing_restores_every_state(env):
    import test_reverb

    from lhotse_b200.pcm_staging import TransformStagingRing, staged_route, undo_draws

    speech, _ = test_reverb.make_sources(env)
    cuts = [c.reverb_rir(room_rng_seed=30 + i, source_rng_seed=40 + i) for i, c in enumerate(speech[:3])]
    gens = [c.recording.transforms[-1].rir_generator for c in cuts]
    torch.manual_seed(2)
    before = ([g.room_rng.bit_generator.state for g in gens], [g.source_rng.bit_generator.state for g in gens],
              torch.get_rng_state())
    staged, _, _, _ = TransformStagingRing().stage(staged_route(cuts, generated_rir=True)[1])
    assert not torch.equal(torch.get_rng_state(), before[2])
    undo_draws(staged)
    assert [g.room_rng.bit_generator.state for g in gens] == before[0]
    assert [g.source_rng.bit_generator.state for g in gens] == before[1]
    assert torch.equal(torch.get_rng_state(), before[2])
