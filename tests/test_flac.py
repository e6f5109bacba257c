"""FLAC on the CPU: the oracle against the STREAMINFO MD5 of two real LibriSpeech files and against every stream of the
test writer; the library's host frame index (`b200feat_flac_index`) against the writer's frame log; the job table of
`FlacStagingRing` decoded frame by frame with the oracle; `flac_request_for_cut` against `pcm16_request_for_cut`; and the
exact per-frame decoder of csrc/flac.cuh run on the host (scripts/micro/flac_host_check.cu), under AddressSanitizer
where the toolchain has it, on whole streams and on truncated and bit-flipped frames."""
import os
import subprocess

import numpy as np
import pytest

import flac_cases as C
import flac_oracle as F
import flac_writer as W
import refshim

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = [os.path.join(ROOT, "tests", "golden", f"2412-153948-000{i}.flac") for i in (0, 1)]
GOLDEN_MD5 = ["5f641f92d4059f1cad5d601b35b4af38", "1302bf076abd37c69e4746e2952b74ab"]


@pytest.fixture(scope="module")
def streams():
    return W.streams()


@pytest.fixture(scope="module")
def stream_dir(streams, tmp_path_factory):
    d = tmp_path_factory.mktemp("flac")
    for name, (data, _, pcm, _) in streams.items():
        (d / f"{name}.flac").write_bytes(data)
        pcm.astype("<i2").tofile(str(d / f"{name}.pcm"))
    return d


def test_oracle_decodes_the_librispeech_fixtures_to_their_md5():
    for path, md5 in zip(GOLDEN, GOLDEN_MD5):
        si, frames, pcm = F.decode(open(path, "rb").read())
        assert si.md5.hex() == md5 and F.md5_of(pcm).hex() == md5
        assert pcm.shape == (si.total_samples, 1) and si.bits_per_sample == 16 and si.sample_rate == 16000
        assert {f.block_size for f in frames[:-1]} == {4096}
    assert [len(F.decode(open(p, "rb").read())[1]) for p in GOLDEN] == [46, 42]


def test_oracle_round_trips_every_writer_stream(streams):
    for name, (data, log, pcm, sr) in streams.items():
        si, frames, got = F.decode(data)
        assert np.array_equal(got, pcm), name
        assert F.md5_of(got) == si.md5 and si.sample_rate == sr, name
        assert [(f.byte_offset, f.first_sample, f.block_size) for f in frames] == log, name


def test_host_index_finds_exactly_the_written_frames(streams):
    from lhotse_b200.engine import flac_index

    assert {"channels8", "variable_blocking", "small_blocks", "false_sync", "stereo", "escapes", "wasted_bits"} <= set(streams)
    for name, (data, log, pcm, sr) in streams.items():
        info, frames = flac_index(data)
        got = [(int(f["byte_offset"]), int(f["first_sample"]), int(f["block_size"])) for f in frames]
        assert got == log, name
        ends = [o for o, _, _ in log[1:]] + [len(data)]
        assert [int(f["byte_offset"] + f["byte_length"]) for f in frames] == ends, name
        assert (info.sample_rate, info.channels, info.bits_per_sample, info.total_samples) == (sr, pcm.shape[1], 16, pcm.shape[0])
        assert bytes(info.md5) == F.md5_of(pcm)
        assert info.variable_blocking == (name == "variable_blocking")
    # the planted header: found by a sync search, refused for its frame number
    data = streams["false_sync"][0]
    fake = data.index(bytes([0xFF, 0xF8, 0xC0, 0x08, 0x05]))
    assert fake not in [o for o, _, _ in streams["false_sync"][1]] and F.crc8(data[fake:fake + 5]) == data[fake + 5]
    for path in GOLDEN:
        raw = open(path, "rb").read()
        info, frames = flac_index(raw)
        _, oframes, _ = F.decode(raw)
        assert [(int(f["byte_offset"]), int(f["byte_length"]), int(f["block_size"])) for f in frames] == \
            [(f.byte_offset, f.byte_length, f.block_size) for f in oframes]
    for bad in (b"", b"OggS" + bytes(60), b"fLaC" + bytes(10), data[:30]):
        with pytest.raises(ValueError):
            flac_index(bad)


def test_ring_job_table_decodes_to_the_requested_samples(streams, stream_dir):
    """The job table of random slices, each job decoded with the oracle and placed where the kernel would put it."""
    from lhotse_b200.engine import FLAC_JOB_DTYPE
    from lhotse_b200.pcm_staging import FlacRequest, FlacStagingRing

    rs = np.random.RandomState(3)
    names = ["subframe_types", "stereo", "channels5", "variable_blocking", "small_blocks"]
    reqs, want = [], []
    for name in names * 3:
        pcm = streams[name][2]
        n = int(rs.randint(1, min(pcm.shape[0], 9000)))
        a = int(rs.randint(0, pcm.shape[0] - n + 1))
        ch = int(rs.randint(pcm.shape[1]))
        reqs.append(FlacRequest(str(stream_dir / f"{name}.flac"), a, n, ch))
        want.append(pcm[a:a + n, ch])
    reqs.append(FlacRequest(str(stream_dir / "stereo.flac"), 0, streams["stereo"][2].shape[0], 1))  # a whole file
    want.append(streams["stereo"][2][:, 1])
    batch, lens, offs, sr = FlacStagingRing(pin_memory=False).stage(reqs)
    assert lens == [r.num_samples for r in reqs] and all(o % 4 == 0 for o in offs) and sr == 16000
    jobs = batch.jobs.numpy().view(FLAC_JOB_DTYPE)
    data = batch.data.numpy().tobytes()
    assert batch.njobs == len(jobs) and np.all(jobs["count"] >= 0) and np.all(jobs["skip"] + jobs["count"] <= jobs["block_size"])
    out = np.zeros(batch.out_elems, dtype=np.int16)
    si = F.read_streaminfo(open(reqs[0].path, "rb").read())
    si.max_frame = 0  # a frame on its own: the bit reader takes all its bytes
    for j in jobs:
        frame = data[j["src_byte"]: j["src_byte"] + j["byte_length"]]
        hdr = F._header(frame, 0)
        assert hdr["number"] == j["coded_number"] and hdr["block"] == j["block_size"]
        _, pcm, end = F.decode_frame(frame, 0, si)
        assert end == len(frame)
        out[j["dst_elem"]: j["dst_elem"] + j["count"]] = pcm[j["skip"]: j["skip"] + j["count"], j["want_channel"]]
    assert (jobs["scratch_elem"][jobs["channels"] > 1] >= 0).all() and (jobs["scratch_elem"][jobs["channels"] == 1] == -1).all()
    for w, o, n in zip(want, offs, lens):
        assert np.array_equal(out[o:o + n], w)


def test_kernel_frame_decoder_on_the_host(stream_dir, tmp_path):
    exe, asan = C.host_check_binary(tmp_path)
    env = dict(os.environ, ASAN_OPTIONS="detect_leaks=0:abort_on_error=0")
    files = sorted(str(p) for p in stream_dir.glob("*.flac")) + GOLDEN
    for path in files:
        raw = str(tmp_path / "out.raw")
        run = subprocess.run([exe, path, raw], capture_output=True, text=True, env=env)
        assert run.returncode == 0 and " 0 bad" in run.stdout, run.stdout[-2000:] + run.stderr[-4000:]
        got = np.fromfile(raw, dtype="<i2")
        if path in GOLDEN:
            assert F.md5_of(got).hex() == GOLDEN_MD5[GOLDEN.index(path)]
        else:
            assert np.array_equal(got, np.fromfile(path[:-5] + ".pcm", dtype="<i2")), path
        bad = subprocess.run([exe, path, "-", "corrupt", "4"], capture_output=True, text=True, env=env)
        assert bad.returncode == 0 and " 0 bad" in bad.stdout, bad.stdout[-2000:] + bad.stderr[-4000:]
        assert "AddressSanitizer" not in bad.stderr
    print("AddressSanitizer:", asan)


@pytest.mark.skipif(not refshim.reference_available(), reason="reference tree not present")
def test_flac_requests_match_wav_twins_and_refuse_ineligible_cuts(streams, tmp_path):
    refshim.import_reference()
    import wave

    from lhotse import MonoCut, Recording
    from lhotse.audio import AudioSource
    from lhotse.cut import PaddingCut

    from lhotse_b200.pcm_staging import flac_request_for_cut, pcm16_request_for_cut

    def rec(path, pcm, sr, channels):
        return Recording(id=os.path.basename(str(path)), sources=[AudioSource(type="file", channels=channels, source=str(path))],
                         sampling_rate=sr, num_samples=pcm.shape[0], duration=pcm.shape[0] / sr)

    checked = 0
    for name in ("stereo", "variable_blocking", "channels3", "subframe_types"):
        data, _, pcm, sr = streams[name]
        fp, wp = tmp_path / f"{name}.flac", tmp_path / f"{name}.wav"
        fp.write_bytes(data)
        with wave.open(str(wp), "wb") as w:
            w.setnchannels(pcm.shape[1]); w.setsampwidth(2); w.setframerate(sr)
            w.writeframes(pcm.astype("<i2").tobytes())
        chans = list(range(pcm.shape[1]))
        T = pcm.shape[0] / sr
        for start, dur, ch in ((0.0, T, 0), (0.0123 * T, 0.5 * T, chans[-1]), (0.3 * T, 0.3 * T - 1e-4, 0)):
            fc = MonoCut(id="f", start=start, duration=dur, channel=ch, recording=rec(fp, pcm, sr, chans))
            wc = MonoCut(id="w", start=start, duration=dur, channel=ch, recording=rec(wp, pcm, sr, chans))
            f, w = flac_request_for_cut(fc), pcm16_request_for_cut(wc)
            assert f is not None and w is not None
            assert (f.first_sample, f.num_samples, f.channel) == (w.first_sample, w.num_samples, w.channel)
            assert flac_request_for_cut(wc) is None and pcm16_request_for_cut(fc) is None
            checked += 1
    assert checked == 12
    data, _, pcm, sr = streams["stereo"]
    fp = tmp_path / "stereo.flac"
    ok = MonoCut(id="f", start=0, duration=0.1, channel=0, recording=rec(fp, pcm, sr, [0, 1]))
    assert flac_request_for_cut(ok) is not None
    # 24-bit STREAMINFO (bits 36-40 of the 144-bit block), an Ogg container, a source that is not a file, transforms,
    # a wrong sampling rate, a range past the end, padding and mixed cuts
    b24 = bytearray(data)
    b24[8 + 12] = (b24[8 + 12] & 0xFE) | 1
    b24[8 + 13] = (b24[8 + 13] & 0x0F) | (7 << 4)
    (tmp_path / "b24.flac").write_bytes(bytes(b24))
    (tmp_path / "ogg.flac").write_bytes(b"OggS" + data)
    bad = [
        MonoCut(id="a", start=0, duration=0.1, channel=0, recording=rec(tmp_path / "b24.flac", pcm, sr, [0, 1])),
        MonoCut(id="b", start=0, duration=0.1, channel=0, recording=rec(tmp_path / "ogg.flac", pcm, sr, [0, 1])),
        MonoCut(id="c", start=0, duration=0.1, channel=0, recording=Recording(
            id="u", sources=[AudioSource(type="url", channels=[0, 1], source="http://localhost/x.flac")], sampling_rate=sr,
            num_samples=pcm.shape[0], duration=pcm.shape[0] / sr)),
        MonoCut(id="d", start=0, duration=0.1, channel=0, recording=rec(fp, pcm, sr, [0, 1]).perturb_volume(0.5)),
        MonoCut(id="e", start=0, duration=0.1, channel=0, recording=rec(fp, pcm, 8000, [0, 1])),
        MonoCut(id="g", start=0.2, duration=0.2, channel=0, recording=rec(fp, pcm, sr, [0, 1])),
        PaddingCut(id="p", duration=1.0, sampling_rate=16000, feat_value=0.0, num_samples=16000),
        ok.mix(ok),
    ]
    for c in bad:
        assert flac_request_for_cut(c) is None, c.id
