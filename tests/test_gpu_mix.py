"""MixedCuts mixed on the GPU (csrc/mix.cuh): `mix_cuts` bit-exact against float32(cut.load_audio()) on WAV-only, FLAC-only
and FLAC-speech + WAV-noise batches and on a 2048-cut CutMix batch of 10-30 s cuts; the real callers (`FusedOnTheFlyFeatures`
alone and inside K2SpeechRecognitionDataset with CutMix, `compute_and_store_features_fused`) against their float route;
and every argument check of `b200feat_mix`."""
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
    import mix_cases

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
    root = tmp_path_factory.mktemp("gmix")
    wav_s, wav_n = mix_cases.sources(root)
    # FLAC: slices of the two LibriSpeech fixtures
    from lhotse import MonoCut, Recording
    from lhotse.audio import AudioSource

    fl = []
    for k, p in enumerate(GOLDEN):
        n = F.read_streaminfo(open(p, "rb").read()).total_samples
        fl.append(Recording(id=f"fl{k}", sources=[AudioSource(type="file", channels=[0], source=p)], sampling_rate=16000,
                            num_samples=n, duration=n / 16000))
    spans = [(0.0, 2.3), (2.4, 3.1), (5.6, 1.7), (0.3, 2.9), (3.0, 4.05), (7.1, 2.2), (1.0, 0.9), (2.0, 1.3), (4.0, 5.2), (9.5, 0.6)]
    flac = [MonoCut(id=f"f{i}", start=a, duration=d, channel=0, recording=fl[i % 2]) for i, (a, d) in enumerate(spans)]
    yield lb_ex, root, (wav_s, wav_n), (flac[:6], flac[6:])
    set_current_audio_backend(wav_backend)


def _check_mix(cuts, ring=None):
    import mix_cases

    from lhotse_b200 import mix_cuts

    buf, lens, offs = mix_cuts(cuts, "cuda:0", ring=ring)
    assert buf.is_cuda and buf.dtype == torch.float32 and all(o % 4 == 0 for o in offs)
    host = buf.cpu()
    for c, o, n in zip(cuts, offs, lens):
        want = torch.from_numpy(mix_cases.load_f32(c))
        assert torch.equal(host[o:o + n], want), c.id


@pytest.mark.parametrize("kind", ["wav", "flac", "flac_speech_wav_noise"])
def test_gpu_mix_cuts_equal_load_audio(env, kind):
    import mix_cases

    from lhotse_b200.pcm_staging import MixStagingRing

    _, root, (ws, wn), (fs, fn) = env
    speech, noise = {"wav": (ws, wn), "flac": (fs, fn), "flac_speech_wav_noise": (fs, wn)}[kind]
    cases = mix_cases.mixed_cases(root, speech, noise)
    cuts = [cases[k] for k in sorted(cases)] + [speech[0], noise[1]]
    ring = MixStagingRing()
    _check_mix(cuts, ring)
    _check_mix(cuts[::-1], ring)  # the ring again, in another order


def test_gpu_mix_cuts_2048_long_cutmix_cuts(env, tmp_path):
    """2048 cuts of 10-30 s with CutMix noise: deep energy trees (up to 480000 samples per track)."""
    import lhotse_env
    import mix_cases
    from lhotse import CutSet
    from lhotse.dataset.cut_transforms import CutMix

    rs = np.random.RandomState(3)
    speech = lhotse_env.make_cutset(tmp_path, [30.0] * 8, seed=4, amp=0.2, prefix="ls")
    noise = lhotse_env.make_cutset(tmp_path, [7.3, 12.1, 30.0, 4.4], seed=5, amp=0.05, prefix="ln")
    cuts = []
    for i in range(2048):
        src = speech[i % 8]
        d = float(np.round(rs.uniform(10.0, 30.0), 3))
        a = float(np.round(rs.uniform(0.0, 30.0 - d), 3))
        cuts.append(src.truncate(offset=a, duration=d, preserve_id=False).with_id(f"l{i}"))
    mixed = list(CutMix(noise, p=0.5, snr=(10, 20), seed=11, pad_to_longest=True, preserve_id=True)(CutSet.from_cuts(cuts)))
    assert 700 < sum(getattr(c, "tracks", None) is not None for c in mixed) < 1350
    from lhotse_b200 import mix_cuts

    buf, lens, offs = mix_cuts(mixed, "cuda:0")
    host = buf.cpu().numpy()
    for c, o, n in zip(mixed, offs, lens):
        assert np.array_equal(host[o:o + n].view(np.int32), mix_cases.load_f32(c).view(np.int32)), c.id


def test_gpu_fused_on_the_fly_mix_route_equals_float_route(env):
    import mix_cases
    from lhotse import CutSet
    from lhotse.dataset.signal_transforms import GlobalMVN

    from lhotse_b200.input_strategies import FusedOnTheFlyFeatures

    lb_ex, root, (ws, wn), (fs, fn) = env
    cases = mix_cases.mixed_cases(root, fs, wn)
    cuts = CutSet.from_cuts([cases[k] for k in sorted(cases)] + [ws[0], fs[1]])
    ext = lb_ex.B200Fbank(lb_ex.B200FbankConfig(device="cuda:0"))
    fast, slow = FusedOnTheFlyFeatures(ext), FusedOnTheFlyFeatures(ext, pcm16_fast_path=False)
    f1, l1 = fast(cuts)
    f2, l2 = slow(cuts)
    assert fast.last_batch_route == "mix" and slow.last_batch_route == "float"
    assert torch.equal(l1, l2) and torch.equal(f1, f2)
    mvn = GlobalMVN(80)
    mvn.norm_means = torch.linspace(-3, 3, 80)
    mvn.norm_stds = torch.linspace(0.5, 2, 80)
    a = FusedOnTheFlyFeatures(ext, global_mvn=mvn)
    g1, m1 = a(cuts)
    b = FusedOnTheFlyFeatures(ext, global_mvn=mvn, pcm16_fast_path=False)
    g2, m2 = b(cuts)
    assert a.last_batch_route == "mix" and b.last_batch_route == "float" and torch.equal(m1, m2) and torch.equal(g1, g2)
    ft = FusedOnTheFlyFeatures(ext, fault_tolerant=True)
    h1, k1, kept = ft(cuts)
    assert ft.last_batch_route == "mix" and torch.equal(h1, f1) and len(kept) == len(cuts)
    # plain batches keep their routes; a refused MixedCut sends the batch to the float route
    for batch, route in (([ws[0], ws[1]], "pcm16"), ([fs[0], fs[1]], "flac"), ([ws[0], fs[0]], "float"),
                         ([cases["mix_snr_0"], ws[0].perturb_volume(2.0).mix(wn[0], snr=10, allow_padding=True)], "float")):
        s = FusedOnTheFlyFeatures(ext)
        s(CutSet.from_cuts(batch))
        assert s.last_batch_route == route, route


def test_gpu_cutmix_in_k2_dataset_equals_reference_strategy(env, tmp_path):
    import lhotse_env
    from lhotse.dataset import DynamicBucketingSampler, K2SpeechRecognitionDataset
    from lhotse.dataset.cut_transforms import CutMix
    from lhotse.dataset.input_strategies import OnTheFlyFeatures

    from lhotse_b200.input_strategies import FusedOnTheFlyFeatures

    lb_ex = env[0]
    rs = np.random.RandomState(0)
    cuts = lhotse_env.make_cutset(tmp_path, np.round(rs.uniform(2.0, 15.0, size=40), 2).tolist(), seed=1)
    noise = lhotse_env.make_cutset(tmp_path, [1.5, 3.7, 8.2], seed=2, amp=0.05, supervisions=False, prefix="n")
    ext = lb_ex.B200Fbank(lb_ex.B200FbankConfig(device="cuda:0"))
    got = {}
    routes = set()
    for name, strategy in (("reference", OnTheFlyFeatures(ext)), ("fused", FusedOnTheFlyFeatures(ext))):
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


def test_gpu_store_route_over_mixed_cuts_equals_the_reference_batch_store(env, tmp_path):
    import mix_cases
    from lhotse import CutSet
    from lhotse.features.io import NumpyFilesWriter

    from lhotse_b200.storage import compute_and_store_features_fused

    lb_ex, root, (ws, wn), (fs, fn) = env
    cases = mix_cases.mixed_cases(root, ws, fn)
    cuts = CutSet.from_cuts([cases[k].with_id(k) for k in sorted(cases)])  # several cases keep their speech cut's id
    ext = lb_ex.B200Fbank(lb_ex.B200FbankConfig(device="cuda:0"))
    want = cuts.compute_and_store_features_batch(ext, tmp_path / "ref", num_workers=0, batch_duration=20.0,
                                                 storage_type=NumpyFilesWriter, overwrite=True)
    calls = []
    orig = ext.extract_staged_packed
    ext.extract_staged_packed = lambda staged, *a, **k: calls.append(type(staged).__name__) or orig(staged, *a, **k)
    got = compute_and_store_features_fused(cuts, ext, tmp_path / "fused", manifest_path=tmp_path / "fused.jsonl.gz",
                                           batch_duration=20.0, num_workers=2, overwrite=True)
    got = CutSet.from_cuts(list(got))
    assert calls and set(calls) == {"MixBatch"}
    assert [c.id for c in got] == [c.id for c in want]
    for g, w in zip(got, want):
        assert (g.num_frames, g.num_features, g.features.recording_id, g.channel) == (w.num_frames, w.num_features,
                                                                                     w.features.recording_id, w.channel)
        assert [s.id for s in g.supervisions] == [s.id for s in w.supervisions]
        assert np.array_equal(g.load_features(), w.load_features())


def test_gpu_mix_argument_checks(env):
    import mix_cases

    from lhotse_b200.engine import B200FeatError, mix
    from lhotse_b200.pcm_staging import MixStagingRing, mix_requests_for_batch

    lb_ex, root, (ws, wn), _ = env
    cases = mix_cases.mixed_cases(root, ws, wn)
    cuts = [cases["mix_snr_0"], cases["muted_reference"], cases["pad_both"]]
    batch, lens, offs, _ = MixStagingRing(pin_memory=False).stage(mix_requests_for_batch(cuts))
    src0 = batch.pcm.cuda()
    ext = lb_ex.B200Fbank(lb_ex.B200FbankConfig(device="cuda:0"))
    h = ext.engine._h

    def run(tracks, cuts_t, out_elems=batch.out_elems, s0=src0, s1=None):
        out = torch.zeros(max(out_elems, 1), dtype=torch.float32, device="cuda:0")
        mix(s0, s1, tracks, cuts_t, out, h)
        torch.cuda.synchronize()
        return out.cpu()

    good = run(batch.tracks.copy(), batch.cuts.copy())
    for c, o, n in zip(cuts, offs, lens):
        assert torch.equal(good[o:o + n], torch.from_numpy(mix_cases.load_f32(c)))

    def bad_tracks(field, value, i=1):
        t = batch.tracks.copy()
        t[field][i] = value
        return t, batch.cuts.copy()

    def bad_cuts(field, value, i=1):
        c = batch.cuts.copy()
        c[field][i] = value
        return batch.tracks.copy(), c

    cases_bad = {
        "track outside its source": bad_tracks("src_elem", int(src0.numel()) - 10),
        "negative source element": bad_tracks("src_elem", -1),
        "bad source index": bad_tracks("source", 2),
        "source 1 missing": bad_tracks("source", 1),
        "struct size": bad_tracks("struct_size", 40),
        "bad role": bad_tracks("role", 7),
        "track cut index": bad_tracks("cut", 9),
        "cut outside its output": bad_cuts("out_elem", batch.out_elems - 5),
        "reference outside the cut's tracks": bad_cuts("ref_track", 5),
        "negative reference": bad_cuts("ref_track", -1),
        "tracks outside the table": bad_cuts("num_tracks", 99),
        "bad mode": bad_cuts("mode", 3),
        "mix_len": bad_cuts("mix_len", 5),
        "reflect longer than the mix": bad_cuts("target_len", 3 * int(batch.cuts["mix_len"][1])),
    }
    for name, (t, c) in cases_bad.items():
        with pytest.raises(B200FeatError) as ei:
            run(t, c)
        assert ei.value.code == -1 and ext.engine.lib.b200feat_last_error(h).decode().startswith("mix:"), name
    with pytest.raises(B200FeatError):
        run(batch.tracks.copy(), batch.cuts.copy(), out_elems=batch.out_elems - 1)
    assert torch.equal(run(batch.tracks.copy(), batch.cuts.copy()), good)  # the same handle and stream, the same bits
