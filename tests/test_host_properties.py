"""Property tests (hypothesis) of the host-side plumbing around the C ABI: staging layout, sub-batch grouping, the PCM reader
and the archive backend — integer / byte work whose bar is bit-exactness."""
import os
import wave

import numpy as np
import torch
from hypothesis import given, settings
from hypothesis import strategies as st

from lhotse_b200.engine import _aligned_offsets, _groups, pack_device, stage_host
from lhotse_b200.pcm_staging import PcmRequest, PcmStagingRing, WavPcm16
from lhotse_b200.storage import B200ArchiveReader, B200ArchiveWriter

lens_st = st.lists(st.integers(min_value=1, max_value=5000), min_size=1, max_size=40)


@given(lens=lens_st, align=st.sampled_from([1, 2, 4, 8]))
@settings(max_examples=60, deadline=None, derandomize=True)
def test_aligned_offsets_are_aligned_increasing_and_tight(lens, align):
    offs, total = _aligned_offsets(lens, align)
    assert all(o % align == 0 for o in offs) and offs[0] == 0 and total == offs[-1] + lens[-1]
    for (o0, n0), o1 in zip(zip(offs, lens), offs[1:]):
        assert o0 + n0 <= o1 < o0 + n0 + align  # no overlap, never more than align - 1 elements of gap


@given(lens=lens_st, target=st.integers(min_value=1, max_value=40000))
@settings(max_examples=60, deadline=None, derandomize=True)
def test_groups_partition_the_batch_in_order(lens, target):
    g = _groups(lens, target, 4)
    assert g[0][0] == 0 and g[-1][1] == len(lens) and all(a[1] == b[0] for a, b in zip(g, g[1:])) and all(b0 < b1 for b0, b1 in g)
    for b0, b1 in g[:-1]:  # every closed group reached its target; dropping its last cut would not
        assert 4 * sum(lens[b0:b1]) >= target > 4 * sum(lens[b0:b1 - 1])


@given(lens=lens_st, i16=st.booleans(), seed=st.integers(0, 2**31 - 1))
@settings(max_examples=40, deadline=None, derandomize=True)
def test_stage_host_and_pack_device_keep_every_sample(lens, i16, seed):
    rs = np.random.RandomState(seed)
    xs = [(rs.randint(-32768, 32767, size=n).astype(np.int16) if i16 else rs.randn(n).astype(np.float32)) for n in lens]
    buf, got_lens, offs = stage_host(xs, dtype=np.int16 if i16 else np.float32)
    v = buf.numpy()
    assert got_lens == lens and all(o % 4 == 0 for o in offs)
    covered = np.zeros(v.shape[0], dtype=bool)
    for x, o, n in zip(xs, offs, lens):
        assert np.array_equal(v[o:o + n], x)
        covered[o:o + n] = True
    assert np.all(v[~covered] == 0)  # alignment gaps carry defined bytes
    dev, l2, o2 = pack_device([torch.from_numpy(x) for x in xs], torch.device("cpu"), dtype=torch.int16 if i16 else torch.float32)
    assert l2 == lens and o2 == offs and np.array_equal(dev.numpy()[: v.shape[0]], v)


@given(shapes=st.lists(st.tuples(st.integers(0, 60), st.sampled_from([1, 13, 40, 80, 257])), min_size=1, max_size=8),
       seed=st.integers(0, 2**31 - 1))
@settings(max_examples=30, deadline=None, derandomize=True)
def test_archive_roundtrip_and_partial_reads(tmp_path_factory, shapes, seed):
    rs = np.random.RandomState(seed)
    path = tmp_path_factory.mktemp("arch") / "a"
    mats = [rs.randn(t, f).astype(np.float32) for t, f in shapes]
    with B200ArchiveWriter(path) as w:
        keys = [w.write(f"k{i}", m) for i, m in enumerate(mats)]
        same_f = [m for m in mats if m.shape[1] == mats[0].shape[1]]
        prefix = np.concatenate(([0], np.cumsum([m.shape[0] for m in same_f])))
        bkeys = w.write_batch([f"b{i}" for i in range(len(same_f))], np.concatenate(same_f, axis=0), prefix)
    assert os.path.getsize(str(path) + ".b200feat") == 4 * (sum(m.size for m in mats) + sum(m.size for m in same_f))
    r = B200ArchiveReader(path)
    for k, m in list(zip(keys, mats)) + list(zip(bkeys, same_f)):
        assert np.array_equal(r.read(k), m)
        lo, hi = sorted(rs.randint(0, m.shape[0] + 3, size=2))
        assert np.array_equal(r.read(k, int(lo), int(hi)), m[lo:hi])


@given(n=st.integers(1, 3000), ch=st.sampled_from([1, 2, 3]), sr=st.sampled_from([8000, 16000, 22050, 44100]),
       seed=st.integers(0, 2**31 - 1))
@settings(max_examples=30, deadline=None, derandomize=True)
def test_wav_reader_agrees_with_the_stdlib_wave_module(tmp_path_factory, n, ch, sr, seed):
    rs = np.random.RandomState(seed)
    pcm = rs.randint(-32768, 32767, size=(n, ch)).astype("<i2")
    path = str(tmp_path_factory.mktemp("wav") / "x.wav")
    with wave.open(path, "wb") as w:
        w.setnchannels(ch); w.setsampwidth(2); w.setframerate(sr)
        w.writeframes(pcm.tobytes())
    h = WavPcm16.open(path)
    assert (h.sampling_rate, h.channels, h.num_samples) == (sr, ch, n)
    first = int(rs.randint(0, n))
    cnt = int(rs.randint(1, n - first + 1))
    c = int(rs.randint(0, ch))
    dst = np.empty(cnt, dtype=np.int16)
    h.read_into(dst, first, c)
    assert np.array_equal(dst, pcm[first:first + cnt, c])
    buf, lens, offs, got_sr = PcmStagingRing(initial_samples=16, pin_memory=False).stage([PcmRequest(path, first, cnt, c)] * 2)
    assert got_sr == sr and lens == [cnt, cnt] and np.array_equal(buf.numpy()[offs[1]: offs[1] + cnt], pcm[first:first + cnt, c])
