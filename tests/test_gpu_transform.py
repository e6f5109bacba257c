"""Speed, Volume and Resample transforms run on the GPU (csrc/resample.cuh): `transform_cuts` bit-exact against
float32(cut.load_audio()) on WAV-only, FLAC-only and WAV + FLAC batches and on a 2048-cut batch of 10-30 s speed-perturbed
cuts; the real callers (`FusedOnTheFlyFeatures` alone and inside K2SpeechRecognitionDataset over a speed-perturbed CutSet,
`compute_and_store_features_fused`) against their float route; and the argument checks of `b200feat_resample`."""
import os

import numpy as np
import pytest
import torch

import flac_oracle as F
import refshim

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = [os.path.join(ROOT, "tests", "golden", f"2412-153948-000{i}.flac") for i in (0, 1)]


@pytest.fixture(scope="module")
def env(tmp_path_factory):
    if not refshim.reference_available():
        pytest.skip("no reference tree / oracle/_ref archive")
    import lhotse_env
    import transform_cases

    lb_ex = lhotse_env.setup_lhotse()
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
    root = tmp_path_factory.mktemp("gtf")
    src = transform_cases.sources(root)
    from lhotse import MonoCut, Recording
    from lhotse.audio import AudioSource

    fl = []
    for k, p in enumerate(GOLDEN):
        n = F.read_streaminfo(open(p, "rb").read()).total_samples
        rec = Recording(id=f"fl{k}", sources=[AudioSource(type="file", channels=[0], source=p)], sampling_rate=16000,
                        num_samples=n, duration=n / 16000)
        fl.append(MonoCut(id=f"fl{k}", start=0.0, duration=n / 16000, channel=0, recording=rec))
    with transform_cases.torch_resampler():
        yield lb_ex, root, src, fl
    set_current_audio_backend(wav_backend)


def _flac_cases(fl):
    f0, f1 = fl
    return {
        "flac_speed_0.9": f0.perturb_speed(0.9),
        "flac_speed_1.1_start": f1.truncate(offset=1.7, duration=4.2).perturb_speed(1.1),
        "flac_resample_8000": f0.truncate(offset=0.5, duration=5.0).resample(8000).resample(16000),
        "flac_volume_speed": f1.perturb_volume(0.6).perturb_speed(0.95),
        "flac_plain": f0.truncate(offset=2.0, duration=3.0),
    }


def _check(cuts, ring=None):
    import transform_cases

    from lhotse_b200 import transform_cuts

    buf, lens, offs = transform_cuts(cuts, "cuda:0", ring=ring)
    assert buf.is_cuda and buf.dtype == torch.float32 and all(o % 4 == 0 for o in offs)
    host = buf.cpu().numpy()
    for c, o, n in zip(cuts, offs, lens):
        want = transform_cases.load_f32(c)
        assert want.shape == (n,) and np.array_equal(host[o:o + n].view(np.int32), want.view(np.int32)), c.id


@pytest.mark.parametrize("kind", ["wav", "flac", "wav_flac"])
def test_gpu_transform_cuts_equal_load_audio(env, kind):
    import transform_cases

    from lhotse_b200.pcm_staging import TransformStagingRing

    _, root, src, fl = env
    cases = {}
    if kind != "flac":
        cases.update(transform_cases.cases(src))
        trim, reflect = transform_cases.fix_cases(src)
        cases["trim"], cases["reflect_pad"] = trim, reflect
    if kind != "wav":
        cases.update(_flac_cases(fl))
    cuts = [cases[k] for k in sorted(cases)]
    ring = TransformStagingRing()
    _check(cuts, ring)
    _check(cuts[::-1], ring)  # the ring again, in another order


def test_gpu_transform_cuts_2048_speed_perturbed_cuts(env, tmp_path):
    """2048 cuts of 10-30 s, a third at speed 0.9, a third at 1.1, a third plain."""
    import lhotse_env
    import transform_cases

    rs = np.random.RandomState(3)
    speech = lhotse_env.make_cutset(tmp_path, [30.0] * 8, seed=4, amp=0.2, prefix="ls")
    cuts = []
    for i in range(2048):
        d = float(np.round(rs.uniform(10.0, 30.0), 3))
        a = float(np.round(rs.uniform(0.0, 30.0 - d), 3))
        c = speech[i % 8].truncate(offset=a, duration=d, preserve_id=False).with_id(f"l{i}")
        cuts.append(c.perturb_speed(0.9) if i % 3 == 0 else c.perturb_speed(1.1) if i % 3 == 1 else c)
    from lhotse_b200 import transform_cuts

    buf, lens, offs = transform_cuts(cuts, "cuda:0")
    host = buf.cpu().numpy()
    for c, o, n in zip(cuts, offs, lens):
        assert np.array_equal(host[o:o + n].view(np.int32), transform_cases.load_f32(c).view(np.int32)), c.id


def test_gpu_fused_on_the_fly_transform_route_equals_float_route(env):
    import transform_cases
    from lhotse import CutSet
    from lhotse.dataset.signal_transforms import GlobalMVN

    from lhotse_b200.input_strategies import FusedOnTheFlyFeatures

    lb_ex, root, src, fl = env
    cases = {k: c for k, c in transform_cases.cases(src).items() if c.sampling_rate == 16000}  # one rate per batch
    cases.update(_flac_cases(fl))
    cuts = CutSet.from_cuts([cases[k] for k in sorted(cases)] + [src[16000][0]])
    ext = lb_ex.B200Fbank(lb_ex.B200FbankConfig(device="cuda:0"))
    fast, slow = FusedOnTheFlyFeatures(ext), FusedOnTheFlyFeatures(ext, pcm16_fast_path=False)
    f1, l1 = fast(cuts)
    f2, l2 = slow(cuts)
    assert fast.last_batch_route == "transform" and slow.last_batch_route == "float"
    assert torch.equal(l1, l2) and torch.equal(f1, f2)
    mvn = GlobalMVN(80)
    mvn.norm_means = torch.linspace(-3, 3, 80)
    mvn.norm_stds = torch.linspace(0.5, 2, 80)
    a = FusedOnTheFlyFeatures(ext, global_mvn=mvn)
    g1, m1 = a(cuts)
    b = FusedOnTheFlyFeatures(ext, global_mvn=mvn, pcm16_fast_path=False)
    g2, m2 = b(cuts)
    assert a.last_batch_route == "transform" and b.last_batch_route == "float" and torch.equal(m1, m2) and torch.equal(g1, g2)
    ft = FusedOnTheFlyFeatures(ext, fault_tolerant=True)
    h1, k1, kept = ft(cuts)
    assert ft.last_batch_route == "transform" and torch.equal(h1, f1) and len(kept) == len(cuts)
    # batches without transforms keep their routes; a refused cut sends the batch to the float route, and MixedCuts with
    # perturbed tracks stay refused by the mix route
    s, f = src[16000], fl
    for batch, route in (([s[0], s[1]], "pcm16"), ([f[0], f[1]], "flac"), ([s[0], f[0]], "float"),
                         ([s[0].perturb_speed(1.1), s[1].truncate(duration=0.5).perturb_speed(1.1)], "float"),
                         ([s[0].perturb_speed(1.1).mix(s[1], snr=10, allow_padding=True)], "float")):
        st = FusedOnTheFlyFeatures(ext)
        st(CutSet.from_cuts(batch))
        assert st.last_batch_route == route, route


def test_gpu_speed_perturbed_k2_dataset_equals_reference_strategy(env, tmp_path):
    import lhotse_env
    from lhotse.dataset import DynamicBucketingSampler, K2SpeechRecognitionDataset
    from lhotse.dataset.input_strategies import OnTheFlyFeatures

    from lhotse_b200.input_strategies import FusedOnTheFlyFeatures

    lb_ex = env[0]
    rs = np.random.RandomState(0)
    cuts = lhotse_env.make_cutset(tmp_path, np.round(rs.uniform(2.0, 15.0, size=30), 2).tolist(), seed=1)
    cuts = cuts + cuts.perturb_speed(0.9) + cuts.perturb_speed(1.1)
    ext = lb_ex.B200Fbank(lb_ex.B200FbankConfig(device="cuda:0"))
    got = {}
    routes = set()
    for name, strategy in (("reference", OnTheFlyFeatures(ext)), ("fused", FusedOnTheFlyFeatures(ext))):
        sampler = DynamicBucketingSampler(cuts, max_duration=60.0, num_buckets=3, shuffle=True, seed=0)
        ds = K2SpeechRecognitionDataset(input_strategy=strategy, return_cuts=True)
        out = []
        for batch_cuts in sampler:
            b = ds[batch_cuts]
            out.append((b["inputs"].cpu(), b["supervisions"]["num_frames"].clone(), [c.id for c in b["supervisions"]["cut"]]))
            if name == "fused":
                routes.add(strategy.last_batch_route)
        got[name] = out
    assert "transform" in routes
    assert len(got["reference"]) == len(got["fused"])
    for (x1, n1, i1), (x2, n2, i2) in zip(got["reference"], got["fused"]):
        assert i1 == i2 and torch.equal(n1, n2) and torch.equal(x1, x2)


def test_gpu_store_route_over_perturbed_cuts_equals_the_reference_batch_store(env, tmp_path):
    import transform_cases
    from lhotse import CutSet
    from lhotse.features.io import NumpyFilesWriter

    from lhotse_b200.storage import compute_and_store_features_fused

    lb_ex, root, src, fl = env
    cases = {k: c for k, c in transform_cases.cases(src).items() if c.sampling_rate == 16000}  # one rate per batch
    cases.update(_flac_cases(fl))
    cuts = CutSet.from_cuts([cases[k].with_id(k) for k in sorted(cases)])
    ext = lb_ex.B200Fbank(lb_ex.B200FbankConfig(device="cuda:0"))
    want = cuts.compute_and_store_features_batch(ext, tmp_path / "ref", num_workers=0, batch_duration=20.0,
                                                 storage_type=NumpyFilesWriter, overwrite=True)
    calls = []
    orig = ext.extract_staged_packed
    ext.extract_staged_packed = lambda staged, *a, **k: calls.append(type(staged).__name__) or orig(staged, *a, **k)
    got = compute_and_store_features_fused(cuts, ext, tmp_path / "fused", manifest_path=tmp_path / "fused.jsonl.gz",
                                           batch_duration=20.0, num_workers=2, overwrite=True)
    got = CutSet.from_cuts(list(got))
    assert calls and set(calls) == {"TransformBatch"}
    assert [c.id for c in got] == [c.id for c in want]
    for g, w in zip(got, want):
        assert (g.num_frames, g.num_features, g.features.recording_id, g.channel) == (w.num_frames, w.num_features,
                                                                                     w.features.recording_id, w.channel)
        assert np.array_equal(g.load_features(), w.load_features())


def test_gpu_resample_argument_checks(env):
    import transform_cases

    from lhotse_b200.engine import B200FeatError, resample, resample_table
    from lhotse_b200.pcm_staging import TransformStagingRing, resample_kernel, transform_requests_for_batch

    lb_ex, root, src, _ = env
    cases = transform_cases.cases(src)
    cuts = [cases["speed_1.1"], cases["resample_then_speed"], cases["volume_only"]]
    batch, lens, offs, _ = TransformStagingRing(pin_memory=False).stage(transform_requests_for_batch(cuts))
    src0 = batch.pcm.cuda()
    ext = lb_ex.B200Fbank(lb_ex.B200FbankConfig(device="cuda:0"))
    h = ext.engine._h
    ids = np.asarray([resample_table(a, b, *resample_kernel(a, b), "cuda:0", h) for a, b in batch.pairs] + [-1], np.int32)
    good_st = batch.stages.copy()
    good_st["table"] = ids[batch.pair]

    def run(st, out_elems=batch.out_elems, mid_elems=batch.mid_elems):
        out = torch.zeros(max(out_elems, 1), dtype=torch.float32, device="cuda:0")
        mid = torch.empty(max(mid_elems, 1), dtype=torch.float32, device="cuda:0")
        resample(src0, None, mid, st, out, h)
        torch.cuda.synchronize()
        return out.cpu()

    good = run(good_st.copy())
    for c, o, n in zip(cuts, offs, lens):
        assert torch.equal(good[o:o + n], torch.from_numpy(transform_cases.load_f32(c)))

    def bad(field, value, i=0):
        st = good_st.copy()
        st[field][i] = value
        return st

    assert (good_st["depth"] == 1).any()
    cases_bad = {
        "input outside its source": bad("in_elem", int(src0.numel()) - 10),
        "negative input element": bad("in_elem", -1),
        "empty input": bad("in_len", 0),
        "bad source": bad("source", 3),
        "source 1 missing": bad("source", 1),
        "struct size": bad("struct_size", 40),
        "unknown table": bad("table", 10 ** 6),
        "negative table": bad("table", -5),
        "out_len": bad("out_len", int(good_st["out_len"][0]) + 1),
        "output outside the buffer": bad("out_elem", batch.out_elems - 5),
        "reflect longer than the output": bad("target_len", 3 * int(good_st["out_len"][0])),
        "bad target": bad("target", 2),
        "intermediate length fix": bad("target_len", int(good_st["out_len"][0]) - 1, i=int(np.nonzero(good_st["target"] == 0)[0][0])),
        "depth order": bad("depth", 5, i=0),
    }
    for name, st in cases_bad.items():
        with pytest.raises(B200FeatError) as ei:
            run(st)
        assert ei.value.code == -1 and ext.engine.lib.b200feat_last_error(h).decode().startswith("resample"), name
    with pytest.raises(B200FeatError):
        run(good_st.copy(), out_elems=batch.out_elems - 1)
    with pytest.raises(B200FeatError):  # a table that is not N x (2 * width + O)
        resample_table(12345, 16000, np.zeros((3, 3), np.float32), 1, "cuda:0", h)
    assert torch.equal(run(good_st.copy()), good)  # the same handle and stream, the same bits
