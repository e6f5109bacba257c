"""The reverb route on the GPU: `transform_cuts(reverb=True)` and `mix_cuts(reverb=True)` against a float64 convolution of the
same pre-reverb samples, within the bound that lhotse's own float32 arithmetic (and `cut.load_audio()`) sets; run-to-run
identity; the routes FusedOnTheFlyFeatures picks; and the argument checks of b200feat_reverb."""
import os

import numpy as np
import pytest
import torch

import refshim
import reverb_cases as RC

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "2412-153948-0000.flac")


@pytest.fixture(scope="module")
def env(tmp_path_factory):
    if not refshim.reference_available():
        pytest.skip("no reference tree / oracle/_ref archive")
    import flac_oracle as F
    import lhotse_env
    import test_reverb
    import transform_cases

    lb_ex = lhotse_env.setup_lhotse()
    from lhotse import MonoCut, Recording
    from lhotse.audio import AudioSource
    from lhotse.audio.backend import AudioBackend, LibsndfileCompatibleAudioInfo, get_current_audio_backend, set_current_audio_backend

    wav_backend = get_current_audio_backend()

    class OracleFlacBackend(AudioBackend):
        """WAV through the test backend, FLAC through the oracle decoder (int16 / 32768, as libsndfile hands it to lhotse)."""

        def read_audio(self, path_or_fd, offset=0.0, duration=None, force_opus_sampling_rate=None):
            if not str(path_or_fd).endswith(".flac"):
                return wav_backend.read_audio(path_or_fd, offset, duration, force_opus_sampling_rate)
            si, _, pcm = F.decode(open(str(path_or_fd), "rb").read())
            a = int(round(offset * si.sample_rate))
            n = pcm.shape[0] - a if duration is None else int(round(duration * si.sample_rate))
            return (pcm[a:a + n].T.astype(np.float32) / 32768.0), si.sample_rate

        def is_applicable(self, path_or_fd):
            return True

        def supports_info(self):
            return True

        def info(self, path_or_fd, force_opus_sampling_rate=None, force_read_audio=False):
            si = F.read_streaminfo(open(str(path_or_fd), "rb").read())
            return LibsndfileCompatibleAudioInfo(channels=si.channels, frames=si.total_samples, samplerate=si.sample_rate,
                                                 duration=si.total_samples / si.sample_rate)

    set_current_audio_backend(OracleFlacBackend())
    root = tmp_path_factory.mktemp("grv")
    speech, rirs = test_reverb.make_sources(root)
    n = F.read_streaminfo(open(GOLDEN, "rb").read()).total_samples
    rec = Recording(id="fl0", sources=[AudioSource(type="file", channels=[0], source=GOLDEN)], sampling_rate=16000,
                    num_samples=n, duration=n / 16000)
    fl = [MonoCut(id="fl0", start=0.0, duration=n / 16000, channel=0, recording=rec)]
    with transform_cases.torch_resampler():
        yield lb_ex, speech, rirs, fl
    set_current_audio_backend(wav_backend)


def _read(req):
    """int16 samples of a PcmRequest / FlacRequest, read independently of the staging rings."""
    import flac_oracle as F

    from lhotse_b200.pcm_staging import PcmRequest, WavPcm16

    if isinstance(req, PcmRequest):
        out = np.empty(req.num_samples, np.int16)
        WavPcm16.open(req.path).read_into(out, req.first_sample, req.channel)
        return out
    _, _, pcm = F.decode(open(req.path, "rb").read())
    return pcm[req.first_sample: req.first_sample + req.num_samples, req.channel].astype(np.int16)


def _pre_reverb(req):
    """The chain's output before the reverb and before the length fix, as lhotse computes it (bit for bit)."""
    from lhotse_b200.pcm_staging import resample_reference

    x = _read(req.source).astype(np.float32) / np.float32(32768)
    for op in req.ops:
        x = (x * np.float32(op[1])).astype(np.float32) if op[0] == "volume" else resample_reference(x, op[1], op[2])
    return x


def _cases(speech, rirs, fl):
    c0, c1, c2 = speech
    return {
        "plain": c1,
        "speed_only": c2.perturb_speed(0.9),
        "speed_reverb": c0.perturb_speed(1.1).reverb_rir(rirs["rir_long"]),
        "reverb": c1.reverb_rir(rirs["rir_short"]),
        "early_only": c2.reverb_rir(rirs["rir_long"], early_only=True),
        "no_normalize": c0.reverb_rir(rirs["rir_short"], normalize_output=False),
        "flac_reverb": fl[0].truncate(offset=1.0, duration=6.0).reverb_rir(rirs["rir_long"]),
        "stereo_rir_ch1": c2.truncate(offset=0.5, duration=3.0).reverb_rir(rirs["rir_stereo"], rir_channels=[1]),
    }


def test_gpu_transform_cuts_reverb_within_bound(env):
    import transform_cases

    from lhotse_b200 import transform_cuts
    from lhotse_b200.pcm_staging import TransformStagingRing, transform_request_for_cut

    _, speech, rirs, fl = env
    cases = _cases(speech, rirs, fl)
    names = sorted(cases)
    cuts = [cases[k] for k in names]
    ring = TransformStagingRing()
    buf, lens, offs = transform_cuts(cuts, "cuda:0", ring=ring, reverb=True)
    again, _, _ = transform_cuts(cuts, "cuda:0", ring=ring, reverb=True)
    assert torch.equal(buf.view(torch.int32), again.view(torch.int32))  # identical from run to run
    host = buf.cpu().numpy()
    for name, c, o, n in zip(names, cuts, offs, lens):
        got = host[o:o + n]
        req = transform_request_for_cut(c, reverb=True)
        if req is None or req.reverb is None:  # a plain slice or a Speed chain: bit for bit as before
            assert np.array_equal(got.view(np.int32), transform_cases.load_f32(c).view(np.int32)), name
            continue
        x, q = _pre_reverb(req), _read(req.reverb.rir)
        truth = RC.truth64(x, q, req.reverb.normalize, n)
        RC.check(got, truth, RC.lhotse32(x, q, req.reverb.normalize, n), name)
        if name != "stereo_rir_ch1":  # the tests' WAV backend reads mono files only; the stereo RIR is read by _read above
            RC.check(got, truth, np.asarray(c.load_audio(), np.float32)[0], name + " vs load_audio")


def test_gpu_mix_cuts_reverb_within_bound(env):
    from lhotse.utils import fastcopy

    from lhotse_b200 import mix_cuts
    from lhotse_b200.pcm_staging import mix_request_for_cut, transform_request_for_cut

    _, speech, rirs, fl = env
    c0, c1, c2 = speech
    m = c0.mix(c1, snr=10, offset_other_by=0.4, allow_padding=True)
    mp = c0.perturb_speed(1.1).mix(c2, snr=5, allow_padding=True)
    cuts = [m.reverb_rir(rirs["rir_short"]), c2, c1.reverb_rir(rirs["rir_long"]), mp.reverb_rir(rirs["rir_long"]),
            c2.perturb_speed(0.9).reverb_rir(rirs["rir_short"])]  # the last two need perturbed_tracks
    for perturbed in (False, True):
        batch = cuts if perturbed else cuts[:3]
        buf, lens, offs = mix_cuts(batch, "cuda:0", perturbed_tracks=perturbed, reverb=True)
        host = buf.cpu().numpy()
        for i, (c, o, n) in enumerate(zip(batch, offs, lens)):
            got = host[o:o + n]
            if i == 1:
                assert np.array_equal(got, np.asarray(c.load_audio(), np.float32)[0])
                continue
            if getattr(c, "tracks", None) is not None:  # the mix without its reverb, as lhotse computes it
                x = np.asarray(fastcopy(c, transforms=None).load_audio(), np.float32)[0]
                rv = mix_request_for_cut(c, perturbed_tracks=perturbed, reverb=True).reverb
            else:  # a reverberated MonoCut: its chain's output before the reverb
                req = transform_request_for_cut(c, reverb=True)
                x, rv = _pre_reverb(req), req.reverb
            q = _read(rv.rir)
            truth = RC.truth64(x, q, rv.normalize, n)
            RC.check(got, truth, RC.lhotse32(x, q, rv.normalize, n), f"mix {i}")
            RC.check(got, truth, np.asarray(c.load_audio(), np.float32)[0], f"mix {i} vs load_audio")


def _truth_samples(c):
    """The float64 truth of a cut's samples: the reverb of its pre-reverb samples in float64 (RC.truth64); a cut without a
    reverb is what the float route reads (the staged routes are bit-exact there)."""
    from lhotse.utils import fastcopy

    from lhotse_b200.pcm_staging import mix_request_for_cut, transform_request_for_cut

    n = c.num_samples
    if getattr(c, "tracks", None) is not None and c.transforms:
        x = np.asarray(fastcopy(c, transforms=None).load_audio(), np.float32)[0]
        rv = mix_request_for_cut(c, perturbed_tracks=True, reverb=True).reverb
        return RC.truth64(x, _read(rv.rir), rv.normalize, n)
    req = transform_request_for_cut(c, reverb=True) if getattr(c, "tracks", None) is None else None
    if req is not None and req.reverb is not None:
        return RC.truth64(_pre_reverb(req), _read(req.reverb.rir), req.reverb.normalize, n)
    return np.asarray(c.load_audio(), np.float64)[0]


def _gate(cuts, ours, ref32, frames):
    """Each cut's features (rows [0, T)) through helpers.gate: ours and the float route's against the float64 oracle on the
    float64 truth samples."""
    from helpers import gate
    from oracle import kaldi_oracle as O

    for i, c in enumerate(cuts):
        t = int(frames[i])
        truth = O.extract(_truth_samples(c), O.OracleConfig(), dtype=torch.float64)
        assert truth.shape[0] == t, (c.id, truth.shape, t)
        ok, msg = gate(ours[i][:t].cpu().numpy(), ref32[i][:t].cpu().numpy(), truth, "fbank")
        assert ok, (c.id, msg)


def test_gpu_fused_on_the_fly_reverb_routes(env):
    from lhotse import CutSet

    from lhotse_b200.input_strategies import FusedOnTheFlyFeatures

    lb_ex, speech, rirs, fl = env
    ext = lb_ex.B200Fbank(lb_ex.B200FbankConfig(device="cuda:0"))
    c0, c1, c2 = speech
    batches = {
        "transform": [c0.reverb_rir(rirs["rir_short"]), c1.perturb_speed(1.1).reverb_rir(rirs["rir_long"]), c2],
        "mix": [c0.mix(c1, snr=10, allow_padding=True).reverb_rir(rirs["rir_long"]), c2.reverb_rir(rirs["rir_short"]), c1,
                c0.perturb_speed(0.9).reverb_rir(rirs["rir_short"], normalize_output=False)],
    }
    for route, batch in batches.items():
        cs = CutSet.from_cuts(batch)
        on, off, flt = (FusedOnTheFlyFeatures(ext, reverb=True, perturbed_tracks=True),
                        FusedOnTheFlyFeatures(ext, perturbed_tracks=True), FusedOnTheFlyFeatures(ext, pcm16_fast_path=False))
        f1, l1 = on(cs)
        f2, l2 = off(cs)
        f3, l3 = flt(cs)
        assert on.last_batch_route == route and off.last_batch_route == "float" and flt.last_batch_route == "float"
        assert torch.equal(f2, f3) and torch.equal(l1, l3)  # reverb=False: exactly the float route
        _gate(batch, f1, f3, l1)


def _recipe_sources(tmp_path, rirs):
    import lhotse_env

    rs = np.random.RandomState(0)
    cuts = lhotse_env.make_cutset(tmp_path, np.round(rs.uniform(2.0, 15.0, size=20), 2).tolist(), seed=1)
    cuts = cuts + cuts.perturb_speed(0.9) + cuts.perturb_speed(1.1)
    noise = lhotse_env.make_cutset(tmp_path, [1.5, 3.7, 8.2], seed=2, amp=0.05, supervisions=False, prefix="n")
    return cuts, noise, [rirs["rir_short"], rirs["rir_long"]]


def test_gpu_reverb_cutmix_in_k2_dataset_within_gate(env, tmp_path):
    """The standard recipe: speed perturbation 0.9 / 1.0 / 1.1, CutMix(p=0.5), lhotse's ReverbWithImpulseResponse(p=0.5),
    under DynamicBucketingSampler.  Every batch stays on a staged route; the features pass the gate."""
    import random

    from lhotse.dataset import DynamicBucketingSampler, K2SpeechRecognitionDataset
    from lhotse.dataset.cut_transforms import CutMix, ReverbWithImpulseResponse
    from lhotse.dataset.input_strategies import OnTheFlyFeatures

    from lhotse_b200.input_strategies import FusedOnTheFlyFeatures

    lb_ex, _, rirs, _ = env
    cuts, noise, pool = _recipe_sources(tmp_path, rirs)
    ext = lb_ex.B200Fbank(lb_ex.B200FbankConfig(device="cuda:0"))
    got, routes = {}, []
    for name, strategy in (("reference", OnTheFlyFeatures(ext)),
                           ("fused", FusedOnTheFlyFeatures(ext, perturbed_tracks=True, reverb=True))):
        sampler = DynamicBucketingSampler(cuts, max_duration=60.0, num_buckets=3, shuffle=True, seed=0)
        ds = K2SpeechRecognitionDataset(input_strategy=strategy, return_cuts=True, cut_transforms=[
            CutMix(noise, p=0.5, snr=(10, 20), seed=5, preserve_id=True),
            ReverbWithImpulseResponse(pool, p=0.5, randgen=random.Random(7), preserve_id=True)])
        out = []
        for batch_cuts in sampler:
            b = ds[batch_cuts]
            out.append((b["inputs"].cpu(), b["supervisions"]["num_frames"].clone(), list(b["supervisions"]["cut"])))
            if name == "fused":
                routes.append(strategy.last_batch_route)
        got[name] = out
    assert "mix" in routes and "float" not in routes, routes
    assert len(got["reference"]) == len(got["fused"])
    reverberated = 0
    for (x1, n1, c1), (x2, n2, c2) in zip(got["reference"], got["fused"]):
        assert [c.id for c in c1] == [c.id for c in c2] and torch.equal(n1, n2)
        _gate(c2, x2, x1, _frames(ext, c2))
        reverberated += sum(_has_reverb(c) for c in c2)
    assert reverberated > 0


def _has_reverb(c):
    from lhotse.augmentation.rir import ReverbWithImpulseResponse
    from lhotse.augmentation.transform import AudioTransform

    tfs = c.transforms if getattr(c, "tracks", None) is not None else c.recording.transforms
    return any(isinstance(t if isinstance(t, AudioTransform) else AudioTransform.from_dict(t), ReverbWithImpulseResponse)
               for t in tfs or [])


def _frames(ext, cuts):
    return [int(ext.engine.plan.num_frames(np.asarray([c.num_samples]))[0]) for c in cuts]


def test_gpu_store_route_over_reverberated_cuts_within_gate(env, tmp_path):
    from lhotse import CutSet
    from lhotse.features.io import NumpyFilesWriter

    from lhotse_b200.storage import compute_and_store_features_fused

    lb_ex, speech, rirs, _ = env
    c0, c1, c2 = speech
    cuts = CutSet.from_cuts([c0.reverb_rir(rirs["rir_short"]).with_id("a"),
                             c1.perturb_speed(1.1).reverb_rir(rirs["rir_long"]).with_id("b"),
                             c0.mix(c2, snr=10, allow_padding=True).reverb_rir(rirs["rir_long"]).with_id("c"), c2.with_id("d")])
    ext = lb_ex.B200Fbank(lb_ex.B200FbankConfig(device="cuda:0"))
    want = cuts.compute_and_store_features_batch(ext, tmp_path / "ref", num_workers=0, batch_duration=20.0,
                                                 storage_type=NumpyFilesWriter, overwrite=True)
    calls = []
    orig = ext.extract_staged_packed
    ext.extract_staged_packed = lambda staged, *a, **k: calls.append(type(staged).__name__) or orig(staged, *a, **k)
    got = compute_and_store_features_fused(cuts, ext, tmp_path / "fused", manifest_path=tmp_path / "fused.jsonl.gz",
                                           batch_duration=20.0, num_workers=2, overwrite=True, reverb=True,
                                           perturbed_tracks=True)
    got = CutSet.from_cuts(list(got))
    assert calls and set(calls) <= {"MixBatch", "TransformBatch"}
    assert [c.id for c in got] == [c.id for c in want]
    feats = [torch.from_numpy(g.load_features()) for g in got]
    refs = [torch.from_numpy(w.load_features()) for w in want]
    for g, w in zip(feats, refs):
        assert g.shape == w.shape
    _gate(list(cuts), feats, refs, [f.shape[0] for f in feats])


def test_gpu_transform_cuts_reverb_2048_cuts(env, tmp_path):
    """2048 cuts of 10-30 s, a third at speed 1.1, half of them reverberated with one of 40 RIRs: the bound per cut, and two
    runs bit-identical."""
    import random

    import lhotse_env
    from lhotse.dataset.cut_transforms import ReverbWithImpulseResponse

    from lhotse_b200 import transform_cuts
    from lhotse_b200.pcm_staging import transform_request_for_cut

    lb_ex, _, rirs, _ = env
    rs = np.random.RandomState(3)
    speech = lhotse_env.make_cutset(tmp_path, [30.0] * 8, seed=4, amp=0.2, prefix="ls")
    from lhotse import CutSet, Recording
    from lhotse.audio import AudioSource

    pool = []
    for k in range(40):
        m = int(rs.uniform(0.3, 1.0) * 16000)
        p = tmp_path / f"rir{k}.wav"
        RC.write_wav(p, RC.decaying_rir(m, seed=k))
        pool.append(Recording(id=f"rir{k}", sources=[AudioSource(type="file", channels=[0], source=str(p))],
                              sampling_rate=16000, num_samples=m, duration=m / 16000))
    cuts = []
    for i in range(2048):
        d = float(np.round(rs.uniform(10.0, 30.0), 3))
        a = float(np.round(rs.uniform(0.0, 30.0 - d), 3))
        c = speech[i % 8].truncate(offset=a, duration=d, preserve_id=False).with_id(f"l{i}")
        cuts.append(c.perturb_speed(1.1) if i % 3 == 0 else c)
    cuts = list(ReverbWithImpulseResponse(pool, p=0.5, randgen=random.Random(1))(CutSet.from_cuts(cuts)))
    buf, lens, offs = transform_cuts(cuts, "cuda:0", reverb=True)
    again, _, _ = transform_cuts(cuts, "cuda:0", reverb=True)
    assert torch.equal(buf.view(torch.int32), again.view(torch.int32))
    host = buf.cpu().numpy()
    checked = 0
    for i, (c, o, n) in enumerate(zip(cuts, offs, lens)):
        req = transform_request_for_cut(c, reverb=True)
        if req is None or req.reverb is None or i % 16:  # every 16th reverberated cut against float64 (time)
            continue
        x, q = _pre_reverb(req), _read(req.reverb.rir)
        RC.check(host[o:o + n], RC.truth64(x, q, True, n), RC.lhotse32(x, q, True, n), c.id)
        checked += 1
    assert checked > 30


def test_gpu_reverb_argument_checks(env):
    from lhotse_b200.engine import REVERB_CUT_DTYPE, REVERB_RIR_DTYPE, B200FeatError, reverb

    dev = torch.device("cuda:0")
    src0 = torch.zeros(1000, dtype=torch.int16, device=dev)
    x = torch.zeros(5000, dtype=torch.float32, device=dev)
    out = torch.zeros(5000, dtype=torch.float32, device=dev)

    def tables():
        rt = np.zeros(1, REVERB_RIR_DTYPE)
        rt["struct_size"], rt["source"], rt["src_elem"], rt["num_samples"] = REVERB_RIR_DTYPE.itemsize, 0, 0, 1000
        ct = np.zeros(1, REVERB_CUT_DTYPE)
        ct["struct_size"], ct["rir"], ct["normalize"] = REVERB_CUT_DTYPE.itemsize, 0, 1
        ct["in_elem"], ct["in_len"], ct["out_elem"], ct["target_len"] = 0, 4000, 0, 4000
        return rt, ct

    rt, ct = tables()
    reverb(src0, None, x, rt, ct, out)  # valid
    torch.cuda.synchronize()
    bad = [("rir", "struct_size", 8), ("rir", "source", 1), ("rir", "source", 2), ("rir", "src_elem", 1),
           ("rir", "num_samples", 0), ("rir", "num_samples", 65537), ("cut", "struct_size", 8), ("cut", "rir", 1),
           ("cut", "rir", -1), ("cut", "normalize", 2), ("cut", "in_len", 0), ("cut", "in_elem", 1001),
           ("cut", "out_elem", 1001), ("cut", "target_len", 8000), ("cut", "target_len", -1)]
    for table, field, value in bad:
        rt, ct = tables()
        (rt if table == "rir" else ct)[field] = value
        with pytest.raises(B200FeatError):
            reverb(src0, None, x, rt, ct, out)
    # one buffer for input and output: disjoint windows are taken, an output over an input window is refused
    both = torch.zeros(10000, dtype=torch.float32, device=dev)
    rt, ct = tables()
    ct["in_elem"] = 5000
    reverb(src0, None, both, rt, ct, both)
    torch.cuda.synchronize()
    for out_elem in (1001, 2000, 5000):
        ct["out_elem"] = out_elem
        with pytest.raises(B200FeatError):
            reverb(src0, None, both, rt, ct, both)
