"""§8f-2: 16-bit PCM staging (lhotse_b200/pcm_staging.py) — the RIFF reader, the pinned int16 ring, the aligned host staging
of `extract_batch`, and the PCM fast path of FusedOnTheFlyFeatures through real lhotse cuts (build container only)."""
import struct
import wave

import numpy as np
import pytest
import torch

import refshim
from lhotse_b200.engine import stage_host
from lhotse_b200.pcm_staging import NotPcm16Wav, PcmRequest, PcmStagingRing, WavPcm16


def _write_wav(path, pcm, sr=16000):
    pcm = np.asarray(pcm, dtype="<i2")
    with wave.open(str(path), "wb") as w:
        w.setnchannels(1 if pcm.ndim == 1 else pcm.shape[1]); w.setsampwidth(2); w.setframerate(sr)
        w.writeframes(pcm.tobytes())


def test_wav_reader_mono_stereo_and_slices(tmp_path):
    rs = np.random.RandomState(0)
    mono = rs.randint(-32768, 32767, size=12345).astype(np.int16)
    _write_wav(tmp_path / "m.wav", mono, sr=8000)
    h = WavPcm16.open(str(tmp_path / "m.wav"))
    assert (h.sampling_rate, h.channels, h.num_samples) == (8000, 1, 12345)
    dst = np.empty(1000, dtype=np.int16)
    assert h.read_into(dst, first_sample=777) == 1000 and np.array_equal(dst, mono[777:1777])
    full = np.empty(12345, dtype=np.int16)
    h.read_into(full)
    assert np.array_equal(full, mono)
    with pytest.raises(ValueError):
        h.read_into(np.empty(10, dtype=np.int16), first_sample=12340)
    stereo = rs.randint(-32768, 32767, size=(5000, 2)).astype(np.int16)
    _write_wav(tmp_path / "s.wav", stereo)
    hs = WavPcm16.open(str(tmp_path / "s.wav"))
    assert (hs.channels, hs.num_samples) == (2, 5000)
    for ch in (0, 1):
        d = np.empty(300, dtype=np.int16)
        hs.read_into(d, first_sample=100, channel=ch)
        assert np.array_equal(d, stereo[100:400, ch])


def test_wav_reader_chunk_walk_extensible_and_rejections(tmp_path):
    pcm = np.arange(-50, 51, dtype="<i2")
    # a LIST chunk of odd size (padded) before "data", and a WAVE_FORMAT_EXTENSIBLE fmt chunk with the PCM sub-format GUID
    fmt = struct.pack("<HHIIHH", 0xFFFE, 1, 22050, 44100, 2, 16) + struct.pack("<HHI", 22, 16, 4) + bytes.fromhex(
        "0100000000001000800000aa00389b71")
    body = b"WAVE" + b"fmt " + struct.pack("<I", len(fmt)) + fmt + b"LIST" + struct.pack("<I", 5) + b"abcde\x00" + \
        b"data" + struct.pack("<I", pcm.nbytes) + pcm.tobytes()
    p = tmp_path / "ext.wav"
    p.write_bytes(b"RIFF" + struct.pack("<I", len(body)) + body)
    h = WavPcm16.open(str(p))
    assert (h.sampling_rate, h.channels, h.num_samples) == (22050, 1, 101)
    d = np.empty(101, dtype=np.int16)
    h.read_into(d)
    assert np.array_equal(d, pcm)
    # rejections: float WAV, 8-bit, not RIFF
    ffmt = struct.pack("<HHIIHH", 3, 1, 16000, 64000, 4, 32)
    fb = b"WAVE" + b"fmt " + struct.pack("<I", 16) + ffmt + b"data" + struct.pack("<I", 8) + b"\0" * 8
    (tmp_path / "f.wav").write_bytes(b"RIFF" + struct.pack("<I", len(fb)) + fb)
    with pytest.raises(NotPcm16Wav):
        WavPcm16.open(str(tmp_path / "f.wav"))
    with wave.open(str(tmp_path / "u8.wav"), "wb") as w:
        w.setnchannels(1); w.setsampwidth(1); w.setframerate(8000); w.writeframes(b"\x80" * 100)
    with pytest.raises(NotPcm16Wav):
        WavPcm16.open(str(tmp_path / "u8.wav"))
    (tmp_path / "x.wav").write_bytes(b"not a wave file at all")
    with pytest.raises(NotPcm16Wav):
        WavPcm16.open(str(tmp_path / "x.wav"))


def test_ring_stages_aligned_ragged_batches(tmp_path):
    rs = np.random.RandomState(1)
    files = []
    for i, n in enumerate((1001, 16000, 333, 4999)):
        pcm = rs.randint(-3000, 3000, size=n).astype(np.int16)
        _write_wav(tmp_path / f"{i}.wav", pcm)
        files.append(pcm)
    ring = PcmStagingRing(initial_samples=1024, pin_memory=False)  # forces a grow
    reqs = [PcmRequest(str(tmp_path / "0.wav"), 1, 1000), PcmRequest(str(tmp_path / "1.wav"), 0, 16000),
            PcmRequest(str(tmp_path / "2.wav"), 10, 301), PcmRequest(str(tmp_path / "3.wav"), 4000, 999)]
    buf, lens, offs, sr = ring.stage(reqs)
    assert sr == 16000 and lens == [1000, 16000, 301, 999] and all(o % 4 == 0 for o in offs)
    assert offs == [0, 1000, 17000, 17304] and buf.numel() == 17304 + 999 and buf.dtype == torch.int16
    b = buf.numpy()
    assert np.array_equal(b[0:1000], files[0][1:1001]) and np.array_equal(b[17000:17301], files[2][10:311])
    assert np.array_equal(b[17304:], files[3][4000:4999]) and np.all(b[17301:17304] == 0)
    from concurrent.futures import ThreadPoolExecutor

    with ThreadPoolExecutor(2) as ex:
        buf2, lens2, offs2, _ = ring.stage(reqs, executor=ex)
    assert np.array_equal(buf2.numpy(), b) and offs2 == offs
    _write_wav(tmp_path / "8k.wav", files[2], sr=8000)
    with pytest.raises(ValueError):
        ring.stage([reqs[0], PcmRequest(str(tmp_path / "8k.wav"), 0, 100)])


def test_stage_host_alignment():
    xs = [np.arange(n, dtype=np.float32) + 1 for n in (5, 8, 3, 1)]
    buf, lens, offs = stage_host(xs)
    assert lens == [5, 8, 3, 1] and offs == [0, 8, 16, 20] and buf.numel() == 21
    v = buf.numpy()
    assert np.array_equal(v[0:5], xs[0]) and np.all(v[5:8] == 0) and np.array_equal(v[16:19], xs[2]) and v[20] == 1
    bi, _, oi = stage_host([x.astype(np.int16) for x in xs], dtype=np.int16)
    assert bi.dtype == torch.int16 and oi == offs


@pytest.mark.reference
@pytest.mark.skipif(not refshim.reference_available(), reason="reference tree not present")
def test_fused_on_the_fly_pcm16_route_equals_float_route(tmp_path):
    """Real lhotse cuts (incl. a cut that starts inside its recording and a stereo recording's second channel):
    the PCM route must give exactly what the float route gives, and ineligible batches must fall back."""
    refshim.import_reference()
    import importlib

    import lhotse_b200.base as lb_base
    import lhotse_b200.extractors as lb_ex

    importlib.reload(lb_base)
    importlib.reload(lb_ex)
    from helpers import attach_oracle_engine
    from lhotse import CutSet, MonoCut, Recording
    from lhotse.audio import AudioSource
    from lhotse.audio.backend import AudioBackend, LibsndfileCompatibleAudioInfo, set_current_audio_backend
    from lhotse.cut import PaddingCut

    from lhotse_b200.input_strategies import FusedOnTheFlyFeatures
    from lhotse_b200.pcm_staging import pcm16_request_for_cut

    class WaveBackend(AudioBackend):
        def read_audio(self, path_or_fd, offset=0.0, duration=None, force_opus_sampling_rate=None):
            with wave.open(str(path_or_fd)) as w:
                sr, ch = w.getframerate(), w.getnchannels()
                w.setpos(int(round(offset * sr)))
                n = w.getnframes() - w.tell() if duration is None else int(round(duration * sr))
                pcm = np.frombuffer(w.readframes(n), dtype="<i2").reshape(-1, ch).T
            return pcm.astype(np.float32) / 32768.0, sr

        def is_applicable(self, path_or_fd):
            return True

    set_current_audio_backend(WaveBackend())
    rs = np.random.RandomState(4)
    cuts = []
    for i, (n, start, dur) in enumerate(((16000, 0.0, 1.0), (40000, 0.5, 1.25), (20001, 0.0, 20001 / 16000), (32000, 1.0, 0.7))):
        stereo = i == 3
        pcm = np.clip(rs.randn(n, 2 if stereo else 1) * 3000, -32768, 32767).astype(np.int16)
        path = tmp_path / f"r{i}.wav"
        _write_wav(path, pcm if stereo else pcm[:, 0])
        rec = Recording(id=f"r{i}", sources=[AudioSource(type="file", channels=[0, 1] if stereo else [0], source=str(path))],
                        sampling_rate=16000, num_samples=n, duration=n / 16000)
        cuts.append(MonoCut(id=f"c{i}", start=start, duration=dur, channel=1 if stereo else 0, recording=rec))
    cs = CutSet.from_cuts(cuts)
    reqs = [pcm16_request_for_cut(c) for c in cs]
    assert [(r.first_sample, r.num_samples, r.channel) for r in reqs] == [(0, 16000, 0), (8000, 20000, 0), (0, 20001, 0), (16000, 11200, 1)]

    ext = attach_oracle_engine(lb_ex.B200Fbank())
    fast = FusedOnTheFlyFeatures(ext)
    slow = FusedOnTheFlyFeatures(ext, pcm16_fast_path=False)
    f1, l1 = fast(cs)
    f2, l2 = slow(cs)
    assert fast.last_batch_route == "pcm16" and slow.last_batch_route == "float"
    assert torch.equal(l1, l2) and l1.tolist() == [100, 125, 125, 70]
    assert f1.shape == f2.shape and torch.equal(f1, f2)  # int16 / 32768 is exactly what the decoder hands out
    # anything that needs the float waveform (or is not a plain PCM slice) takes the float route
    assert FusedOnTheFlyFeatures(ext, return_audio=True)(cs)[0].shape == f1.shape
    withtf = FusedOnTheFlyFeatures(ext, wave_transforms=[lambda a: a * 0.5])
    withtf(cs)
    assert withtf.last_batch_route == "float"
    assert pcm16_request_for_cut(PaddingCut(id="p", duration=1.0, sampling_rate=16000, feat_value=0.0, num_samples=16000)) is None
    (tmp_path / "r0.flac").write_bytes(b"fLaC")
    rec = cuts[0].recording
    flac = MonoCut(id="f", start=0, duration=1.0, channel=0, recording=Recording(
        id="rf", sources=[AudioSource(type="file", channels=[0], source=str(tmp_path / "r0.flac"))],
        sampling_rate=16000, num_samples=16000, duration=1.0))
    assert pcm16_request_for_cut(flac) is None and rec is not None


# ------------------------------------------------------------------------------------------------ GPU tier
@pytest.mark.gpu
def test_gpu_staged_pcm16_equals_float_and_aligned_host_staging(tmp_path):
    import lhotse_b200 as lb

    rs = np.random.RandomState(9)
    lens = [15999, 16001, 4001, 23457, 801, 16000]  # mostly odd: back-to-back staging would leave cuts on odd offsets
    pcms = [np.clip(rs.randn(n) * 3000, -32768, 32767).astype(np.int16) for n in lens]
    for i, p in enumerate(pcms):
        _write_wav(tmp_path / f"{i}.wav", p)
    ring = PcmStagingRing()
    staged, slens, offs, sr = ring.stage([PcmRequest(str(tmp_path / f"{i}.wav"), 0, n) for i, n in enumerate(lens)])
    ext = lb.B200Fbank()
    feats, flens = ext.extract_staged_padded(staged, slens, offs, sr)
    floats = [p.astype(np.float32) / 32768.0 for p in pcms]
    want, wlens = ext.extract_batch_padded([torch.from_numpy(f) for f in floats], 16000)
    assert feats.is_cuda and torch.equal(flens, wlens) and torch.equal(feats, want)   # bit-identical to the float route
    # numpy list route (what compute_and_store_features_batch uses): aligned pinned staging + b200feat_extract_host_at
    per_cut = [ext.extract(f, 16000) for f in floats]
    batch = ext.extract_batch(floats, 16000)
    assert all(np.array_equal(a, b) for a, b in zip(batch, per_cut))
    # the C entry point with explicit offsets vs back to back: same bits (only the load path differs)
    eng = ext.engine
    buf, blens, boffs = stage_host(floats)
    a, _ = eng.extract_host(buf, blens, offsets=boffs)
    b, _ = eng.extract_host(np.concatenate(floats), blens)
    assert np.array_equal(a, b)
    with pytest.raises(lb.B200FeatError):
        eng.extract_host(buf, blens, offsets=[0, 10, 20, 30, 40, 50])  # overlapping


@pytest.mark.gpu
def test_gpu_packed_batch_to_archive_roundtrip(tmp_path):
    """§8f-3 on the device: one packed extraction, ONE device-to-host copy, ONE archive append; every cut reads back equal
    to its own `extract` (the archive backend itself needs no lhotse)."""
    import lhotse_b200 as lb
    from lhotse_b200.storage import B200ArchiveReader, B200ArchiveWriter

    rs = np.random.RandomState(12)
    xs = [(0.1 * rs.randn(n)).astype(np.float32) for n in (16000, 4001, 23457, 801, 48000)]
    for ext in (lb.B200Fbank(), lb.B200Mfcc(), lb.B200WhisperFbank()):
        packed, prefix = ext.extract_batch_packed(xs, 16000)
        assert packed.is_cuda and packed.shape == (int(prefix[-1]), ext.feature_dim(16000)) and prefix[0] == 0
        host = torch.empty(packed.shape, dtype=torch.float32, pin_memory=True)
        host.copy_(packed)
        with B200ArchiveWriter(tmp_path / ext.name) as w:
            keys = w.write_batch([f"c{i}" for i in range(len(xs))], host.numpy(), prefix)
        r = B200ArchiveReader(tmp_path / ext.name)
        for x, k in zip(xs, keys):
            want = ext.extract(x, 16000)
            assert np.array_equal(r.read(k), want)
            assert np.array_equal(r.read(k, 3, 9), want[3:9])
    pcm = [np.clip(x * 32768, -32768, 32767).astype(np.int16) for x in xs]
    buf, lens, offs = stage_host(pcm, dtype=np.int16)
    ext = lb.B200Fbank()
    a, pa = ext.extract_staged_packed(buf, lens, offs, 16000)
    b, pb = ext.extract_batch_packed([p.astype(np.float32) / 32768.0 for p in pcm], 16000)
    assert np.array_equal(pa, pb) and torch.equal(a, b)


@pytest.mark.gpu
def test_gpu_large_list_routes_take_the_staged_pipelines_and_match():
    """Lists and arrays big enough for the staged routes (the library's gather threads behind `extract_host_list`, the
    pageable (B, n) route, group-wise H2D in `pack_device`) give the same bits as the plain routes."""
    import lhotse_b200 as lb
    import lhotse_b200.engine as E

    rs = np.random.RandomState(17)
    B, n = 48, 160001                       # odd length: every cut needs its aligned offset
    arr = (0.1 * rs.randn(B, n)).astype(np.float32)
    ext = lb.B200Fbank()
    want = ext.extract_batch(torch.from_numpy(arr).pin_memory().numpy(), 16000)   # (B, n) pinned: direct C call
    lst = [arr[i].copy() for i in range(B)]
    out, prefix = ext.engine.extract_host_list(lst)                                 # 30 MB: gathered by the library
    assert np.array_equal(out.reshape(want.shape), want)
    assert np.array_equal(np.asarray(ext.extract_batch(lst, 16000)), want)
    assert np.array_equal(np.asarray(ext.extract_batch(arr, 16000)), want)          # pageable (B, n): staged route
    tens = [torch.from_numpy(a) for a in lst]                                       # 30 MB: group-wise H2D in pack_device
    got = ext.extract_batch(tens, 16000)
    assert got.is_cuda and np.array_equal(got.cpu().numpy(), want)
    keep = E.STAGING_THREADS
    try:
        E.STAGING_THREADS = 1                                                       # single-thread fallbacks
        assert np.array_equal(np.asarray(ext.extract_batch(lst, 16000)), want)
        assert np.array_equal(ext.extract_batch(tens, 16000).cpu().numpy(), want)
    finally:
        E.STAGING_THREADS = keep


def test_descriptor_cache_never_closes_a_descriptor_in_use(tmp_path, monkeypatch):
    """Many more files than cache slots, read concurrently: every read must return ITS file's samples (a descriptor closed under a
    concurrent reader could be re-issued by the OS for another file and silently deliver the wrong audio), replaced files are
    re-opened, and nothing leaks."""
    import threading

    import lhotse_b200.pcm_staging as ps

    monkeypatch.setattr(ps, "_FDS", ps._FdCache(capacity=3))
    n_files, n = 24, 4000
    paths = []
    for i in range(n_files):
        p = str(tmp_path / f"f{i}.wav")
        _write_wav(p, np.full(n, i + 1, dtype=np.int16), 16000)
        paths.append(p)
    headers = [WavPcm16.open_cached(p) for p in paths]
    errors = []

    def worker(seed):
        rs = np.random.RandomState(seed)
        buf = np.empty(512, dtype=np.int16)
        try:
            for _ in range(400):
                i = int(rs.randint(n_files))
                first = int(rs.randint(0, n - 512))
                headers[i].read_into(buf, first)
                if not np.all(buf == i + 1):
                    errors.append((i, int(buf[0])))
                    return
        except Exception as e:  # noqa: BLE001
            errors.append(repr(e))

    threads = [threading.Thread(target=worker, args=(s,)) for s in range(8)]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    assert not errors, errors[:3]
    assert len(ps._FDS) <= 3 + 8
    # a replaced file (new size / mtime) gets a fresh header and a fresh descriptor
    _write_wav(paths[0], np.full(n + 100, 77, dtype=np.int16), 16000)
    h = WavPcm16.open_cached(paths[0])
    assert h.num_samples == n + 100
    buf = np.empty(100, dtype=np.int16)
    h.read_into(buf, n)
    assert np.all(buf == 77)
    ps._FDS.clear()
    assert len(ps._FDS) == 0
