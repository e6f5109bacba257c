"""FLAC decoded on the GPU: `decode_flac` bit-exact against the oracle (whole files against their STREAMINFO MD5, trimmed
slices, channel selection, one batch mixing everything), a corrupted frame surfacing as ValueError, and the real callers
(`FusedOnTheFlyFeatures`, `compute_and_store_features_fused`) over FLAC cuts against their float route, which reads the
same files through a test audio backend built on the oracle decoder."""
import os

import numpy as np
import pytest
import torch

import flac_oracle as F
import flac_writer as W
import refshim

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = [os.path.join(ROOT, "tests", "golden", f"2412-153948-000{i}.flac") for i in (0, 1)]


@pytest.fixture(scope="module")
def files(tmp_path_factory):
    d = tmp_path_factory.mktemp("flac")
    out = {}
    for name, (data, _, pcm, sr) in W.streams().items():
        (d / f"{name}.flac").write_bytes(data)
        out[name] = (str(d / f"{name}.flac"), pcm)
    for p in GOLDEN:
        out[os.path.basename(p)] = (p, F.decode(open(p, "rb").read())[2])
    return out


def _run(reqs):
    from lhotse_b200 import decode_flac

    buf, lens, offs = decode_flac(reqs, "cuda:0")
    assert buf.is_cuda and buf.dtype == torch.int16 and all(o % 4 == 0 for o in offs)
    host = buf.cpu().numpy()
    return [host[o:o + n] for o, n in zip(offs, lens)]


def test_gpu_decode_whole_files_match_their_md5(files):
    from lhotse_b200 import FlacRequest

    for name, (path, pcm) in files.items():
        si = F.read_streaminfo(open(path, "rb").read())
        got = _run([FlacRequest(path, 0, pcm.shape[0], c) for c in range(pcm.shape[1])])
        assert F.md5_of(np.stack(got, axis=1)) == si.md5, name


def test_gpu_decode_slices_channels_and_a_mixed_batch(files):
    from lhotse_b200 import FlacRequest

    rs = np.random.RandomState(11)
    reqs, want = [], []
    for name, (path, pcm) in sorted(files.items()):
        for _ in range(3):
            n = int(rs.randint(1, pcm.shape[0]))
            a = int(rs.randint(0, pcm.shape[0] - n + 1))
            ch = int(rs.randint(pcm.shape[1]))
            reqs.append(FlacRequest(path, a, n, ch))
            want.append(pcm[a:a + n, ch])
    for r, w in zip(reqs, want):  # each alone
        assert np.array_equal(_run([r])[0], w), r
    order = rs.permutation(len(reqs))  # all together, shuffled: every subframe type, channel layout and blocking in one launch
    for i, g in zip(order, _run([reqs[i] for i in order])):
        assert np.array_equal(g, want[i]), reqs[i]


def test_gpu_corrupted_frame_raises_value_error(files, tmp_path):
    from lhotse_b200 import FlacRequest

    path, pcm = files["2412-153948-0000.flac"]
    raw = bytearray(open(path, "rb").read())
    from lhotse_b200.engine import flac_index

    _, frames = flac_index(bytes(raw))
    f = frames[10]
    raw[int(f["byte_offset"]) + int(f["byte_length"]) // 2] ^= 0x10
    bad = tmp_path / "bad.flac"
    bad.write_bytes(bytes(raw))
    a = int(f["first_sample"]) - 100
    with pytest.raises(ValueError, match="bad.flac.*CRC-16"):
        _run([FlacRequest(str(path), 0, 1000), FlacRequest(str(bad), a, 5000)])
    assert np.array_equal(_run([FlacRequest(str(bad), 0, a)])[0], pcm[:a, 0])  # the frames before it still decode


# ---- real callers ---------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def lhotse_flac(files):
    if not refshim.reference_available():
        pytest.skip("no reference tree / oracle/_ref archive")
    import lhotse_env

    lb_ex = lhotse_env.setup_lhotse()
    from lhotse.audio.backend import AudioBackend, LibsndfileCompatibleAudioInfo, get_current_audio_backend, set_current_audio_backend

    wav_backend = get_current_audio_backend()

    class OracleFlacBackend(AudioBackend):
        """The float route's decoder for these tests: the oracle, int16 / 32768 as libsndfile hands it to lhotse."""

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
    from lhotse import CutSet, MonoCut, Recording
    from lhotse.audio import AudioSource

    cuts = []
    for k, name in enumerate(["2412-153948-0000.flac", "2412-153948-0001.flac", "stereo", "variable_blocking"]):
        path, pcm = files[name]
        chans = list(range(pcm.shape[1]))
        rec = Recording(id=f"r{k}", sources=[AudioSource(type="file", channels=chans, source=path)], sampling_rate=16000,
                        num_samples=pcm.shape[0], duration=pcm.shape[0] / 16000)
        T = pcm.shape[0] / 16000
        for j, (s, d) in enumerate(((0.0, T), (0.1 * T, 0.5 * T), (0.37 * T, 0.41 * T))):
            cuts.append(MonoCut(id=f"c{k}_{j}", start=round(s, 4), duration=round(d, 4), channel=chans[-1] if j == 1 else 0,
                                recording=rec))
    yield lb_ex, CutSet.from_cuts(cuts)
    set_current_audio_backend(wav_backend)


def test_gpu_fused_on_the_fly_flac_route_equals_float_route(lhotse_flac, tmp_path):
    from lhotse.dataset.signal_transforms import GlobalMVN

    from lhotse_b200.input_strategies import FusedOnTheFlyFeatures

    lb_ex, cuts = lhotse_flac
    ext = lb_ex.B200Fbank(lb_ex.B200FbankConfig(device="cuda:0"))
    fast, slow = FusedOnTheFlyFeatures(ext), FusedOnTheFlyFeatures(ext, pcm16_fast_path=False)
    f1, l1 = fast(cuts)
    f2, l2 = slow(cuts)
    assert fast.last_batch_route == "flac" and slow.last_batch_route == "float"
    assert torch.equal(l1, l2) and f1.shape == f2.shape and torch.equal(f1, f2)
    mvn = GlobalMVN(80)
    mvn.norm_means = torch.linspace(-3, 3, 80)
    mvn.norm_stds = torch.linspace(0.5, 2, 80)
    g1, m1 = FusedOnTheFlyFeatures(ext, global_mvn=mvn)(cuts)
    s = FusedOnTheFlyFeatures(ext, global_mvn=mvn, pcm16_fast_path=False)
    g2, m2 = s(cuts)
    assert s.last_batch_route == "float" and torch.equal(m1, m2) and torch.equal(g1, g2)
    # a batch mixing a FLAC slice and a WAV cut takes the float route
    import lhotse_env

    from lhotse import CutSet

    wav = next(iter(lhotse_env.make_cutset(tmp_path, [0.5], prefix="w")))
    mixed = CutSet.from_cuts([cuts[1], wav])
    fm = FusedOnTheFlyFeatures(ext)
    fm(mixed)
    assert fm.last_batch_route == "float"


def test_gpu_store_route_over_flac_equals_the_reference_batch_store(lhotse_flac, tmp_path):
    from lhotse import CutSet
    from lhotse.features.io import NumpyFilesWriter

    from lhotse_b200.storage import compute_and_store_features_fused

    lb_ex, cuts = lhotse_flac
    ext = lb_ex.B200Fbank(lb_ex.B200FbankConfig(device="cuda:0"))
    want = cuts.compute_and_store_features_batch(ext, tmp_path / "ref", num_workers=0, batch_duration=20.0,
                                                 storage_type=NumpyFilesWriter, overwrite=True)
    calls = []
    orig = ext.extract_staged_packed
    ext.extract_staged_packed = lambda staged, *a, **k: calls.append(type(staged).__name__) or orig(staged, *a, **k)
    got = compute_and_store_features_fused(cuts, ext, tmp_path / "fused", manifest_path=tmp_path / "fused.jsonl.gz",
                                           batch_duration=20.0, num_workers=2, overwrite=True)
    got = CutSet.from_cuts(list(got))
    assert calls and set(calls) == {"FlacBatch"}
    assert [c.id for c in got] == [c.id for c in want]
    for g, w in zip(got, want):
        assert (g.num_frames, g.num_features, g.features.recording_id, g.channel) == (w.num_frames, w.num_features,
                                                                                     w.features.recording_id, w.channel)
        assert np.array_equal(g.load_features(), w.load_features())
