"""The FLAC decoder (csrc/flac.cuh) at its edges, against the test writer's input PCM.

A named table of valid frames (tests/flac_cases.py) reaches what the writer's catalogue never does: unary codes longer than
one 64-bit refill (up to quotients near 96000), Rice parameters 0, 14 and 30, escape widths 17-31, partition orders 9-15
and an empty first partition, both sides of the 32-bit accumulation bound at its extreme values, full-scale stereo in every
channel assignment, 15 and 16 wasted bits, blocks of 1, 65535 and 65536 samples, and coded numbers of 4-7 bytes.  On the
CPU the oracle and the decoder's own code (the host check, under AddressSanitizer) must both give the PCM.  On the GPU the
whole table runs as one shuffled launch of full, partial and empty windows between sentinels, and each job alone.

A matrix of malformed frames whose CRC-8 and CRC-16 hold, and of jobs that disagree with their frame or their launch,
must give one named status each, on the host and (after the host run has passed) on the device, with the same bits in
the output and scratch buffers."""
import hashlib

import numpy as np
import pytest

import flac_cases as C
import flac_oracle as F
import flac_writer as W
from flac_writer import FrameSpec, Sub

# sha256 over (name, bytes) of W.streams(), sorted by name: the catalogue the other FLAC tests run stays what it was
STREAMS_SHA256 = "d8a2c7dd09fb226926b4069c47e092072f7515a427a31356b2835da95fd1eca6"


@pytest.fixture(scope="module")
def built():
    facts, cases = {}, []
    for e in C.edges():
        data, frames = C.build(e, facts)
        cases.append((e, data, frames))
    return facts, cases


@pytest.fixture(scope="module")
def valid(built):
    return C.valid_table([f for _, _, frames in built[1] for f in frames])


@pytest.fixture(scope="module")
def malformed():
    return C.malformed_table()


@pytest.fixture(scope="module")
def harness(tmp_path_factory):
    return C.host_check_binary(tmp_path_factory.mktemp("flac_edges"))


# ---- the writer ------------------------------------------------------------------------------------------------------
def test_writer_catalogue_is_byte_identical():
    h = hashlib.sha256()
    for name, (data, _, _, _) in sorted(W.streams().items()):
        h.update(name.encode())
        h.update(data)
    assert h.hexdigest() == STREAMS_SHA256


def test_writer_refuses_fields_that_do_not_fit():
    low = np.full((16, 1), -32768)
    lpc2 = dict(order=2, precision=15, shift=0, coefs=[-16384, -16384])
    bad = [
        (low, FrameSpec(16, subs=[Sub("lpc", escape=(0,), **lpc2)])),                          # escape width 32
        (low, FrameSpec(16, subs=[Sub("fixed", order=0, params=[15])])),                        # method 0's escape code
        (low, FrameSpec(16, subs=[Sub("fixed", order=0, method=1, params=[31])])),              # method 1's escape code
        (low, FrameSpec(16, subs=[Sub("lpc", order=4, precision=15, shift=0, coefs=[-16384] * 4)])),  # residual below -2^31
        (low, FrameSpec(16, subs=[Sub("verbatim", wasted=16)])),                               # wasted bits = width
        (low, FrameSpec(16, subs=[Sub("lpc", order=4, raw={"precision_code": 16})])),          # a raw field wider than 4 bits
        (low, FrameSpec(16, subs=[Sub("lpc", order=4, precision=16)])),                         # precision 16 (code 1111)
        (low, FrameSpec(16, subs=[Sub("fixed", order=2, porder=4)])),                           # psize 1 < order 2
        (low, FrameSpec(16, subs=[Sub("fixed", order=5)])),
        (low, FrameSpec(16, bs_code=6 + 2)),                                                    # code 8 is 256 samples
    ]
    for pcm, spec in bad:
        with pytest.raises(ValueError):
            W.frame(pcm, spec, 0)
    W.frame(low, FrameSpec(16, subs=[Sub("fixed", order=2, porder=3)]), 0)                   # psize 2 == order 2 is fine
    with pytest.raises(ValueError):
        W.frame(low, FrameSpec(16, subs=[Sub("fixed")]), 1 << 36)                              # coded number over 36 bits
    with pytest.raises(ValueError):
        W.encode(np.zeros((65536, 1), np.int16), 16000, [FrameSpec(65536, subs=[Sub("constant")])])  # STREAMINFO max block
    with pytest.raises(ValueError):
        W._streaminfo(4096, 4096, 100, 1 << 24, 16000, 1, 4096, bytes(16))                      # STREAMINFO max frame
    assert len(W._streaminfo(4096, 4096, 100, (1 << 24) - 1, 16000, 1, 4096, bytes(16))) == 34
    # the frame alone carries block 65536 (code 7, 0xFFFF); the decoder's own check takes it
    one = W.frame(np.zeros((65536, 1)), FrameSpec(65536, subs=[Sub("constant")]), 0)
    assert F._header(one, 0)["block"] == 65536


# ---- the edge table --------------------------------------------------------------------------------------------------
def test_edge_table_reaches_every_named_edge(built, valid):
    facts, cases = built
    q = facts["quotient"]
    assert max(q) > 65000 and sorted(q)[-2] > 64                                # past one 64-bit refill, in two partitions
    assert {(0, 0), (0, 14), (1, 30)} <= facts["rice"]
    assert set(range(17, 32)) <= facts["escape"]
    assert set(range(9, 16)) <= facts["porder"]
    assert {(1, 15), (16, 8), (4, 10)} <= facts["empty_first_partition"]          # psize == order
    assert {(32, True), (33, True)} <= facts["accumulation"]                      # both sides of the bound, extreme values
    assert {(a, True) for a in (-1, 8, 9, 10)} <= facts["assignment"]             # full scale in every assignment
    assert {(15, 16), (16, 17)} <= facts["wasted"]
    assert {1, 65535, 65536} <= facts["block"]
    assert {4, 5, 6, 7} <= facts["coded_number_bytes"]
    streams = {e.name for e, data, _ in cases if data is not None}
    assert {"block_sizes", "full_scale_stereo"} <= streams and "block_65536" not in streams
    # one launch: several CTAs, every channel, full / partial / empty windows, odd offsets, the last window at the end
    j = valid.jobs
    assert len(j) > 128                                                          # two CTAs or more
    assert (j["count"] == 0).sum() >= 50 and ((j["count"] > 0) & (j["count"] < j["block_size"])).sum() >= 50
    assert (j["count"] == j["block_size"]).sum() >= 50 and (j["dst_elem"] % 2 == 1).sum() >= 50
    assert int((j["dst_elem"] + j["count"]).max()) == valid.out_elems
    assert {(int(c), int(w)) for c, w in zip(j["channels"], j["want_channel"])} == {(1, 0), (2, 0), (2, 1)}
    assert (j["scratch_elem"][j["channels"] > 1] >= 0).all() and (j["scratch_elem"][j["channels"] == 1] == -1).all()
    assert int(j["block_size"].max()) == 65536 and int(j["coded_number"].max()) == (1 << 36) - 16


def test_oracle_decodes_every_edge_frame_to_the_writers_pcm(built):
    from lhotse_b200.engine import flac_index

    for e, data, frames in built[1]:
        if data is not None:  # the whole stream, and the library's frame index over it
            si, oframes, pcm = F.decode(data)
            assert np.array_equal(pcm, np.asarray(e.pcm, np.int16)) and F.md5_of(pcm) == si.md5, e.name
            info, idx = flac_index(data)
            assert [int(b) for b in idx["block_size"]] == [f.pcm.shape[0] for f in frames], e.name
        si = F.StreamInfo(0, 0, 0, 0, 16000, 0, 16, 0, b"", 0)  # max_frame 0: each frame's bit reader takes all its bytes
        for f in frames:
            fr, pcm, end = F.decode_frame(f.data, 0, si)
            assert end == len(f.data) and fr.number == f.number and np.array_equal(pcm, f.pcm), (e.name, f.number)


def test_host_decodes_the_edge_table_to_the_writers_pcm(harness, valid, tmp_path):
    exe, asan = harness
    st, out, scratch = C.run_host(exe, valid, tmp_path)
    bad = [valid.labels[i] for i, s in enumerate(st) if s]
    assert not bad, bad[:10]
    assert np.array_equal(out, valid.want_out) and np.array_equal(scratch, valid.want_scratch)
    print("AddressSanitizer:", asan)


def _check_malformed(t, st, out, scratch):
    got = {label: s for label, s in zip(t.labels, st)}
    want = dict(zip(t.labels, t.want_status))
    assert got == want, {k: (got[k], want[k]) for k in got if got[k] != want[k]}
    inside = C.windows_mask(t, t.out_elems, "dst_elem")
    assert (out[~inside] == C.OUT_FILL).all()
    sin = C.windows_mask(t, t.scratch_elems, "scratch_elem")
    assert (scratch[~sin] == C.SCRATCH_FILL).all()


def test_host_status_matrix(harness, malformed, tmp_path):
    # every malformed frame is well-formed at the CRC level: a status other than ECRC comes from the contents
    for j, label in zip(malformed.jobs, malformed.labels):
        b = malformed.data[int(j["src_byte"]) if j["src_byte"] >= 0 else 0:][:int(j["byte_length"])]
        if j["src_byte"] >= 0 and j["byte_length"] >= 8:
            assert F.crc16(b[:-2]) == int.from_bytes(b[-2:], "big"), label
    assert set(malformed.want_status) == set(range(11)) - {C.ECRC}
    exe, asan = harness
    st, out, scratch = C.run_host(exe, malformed, tmp_path)
    _check_malformed(malformed, st, out, scratch)
    print("AddressSanitizer:", asan)


# ---- the device ------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_gpu_edge_table_in_one_launch_and_each_job_alone(valid):
    st, out, scratch = C.run_device(valid)
    bad = [valid.labels[i] for i, s in enumerate(st) if s]
    assert not bad, bad[:10]
    assert np.array_equal(out, valid.want_out), np.flatnonzero(out != valid.want_out)[:10]
    assert np.array_equal(scratch, valid.want_scratch)
    for k in range(len(valid.jobs)):
        j = valid.jobs[k:k + 1]
        s1, o1, c1 = C.run_device(valid, j)
        a, n = int(j["dst_elem"][0]), int(j["count"][0])
        assert s1 == [0] and np.array_equal(o1[a:a + n], out[a:a + n]), valid.labels[k]
        assert (np.delete(o1, np.arange(a, a + n)) == C.OUT_FILL).all(), valid.labels[k]
        sa = int(j["scratch_elem"][0])
        if sa >= 0:
            assert np.array_equal(c1[sa:sa + n], scratch[sa:sa + n]), valid.labels[k]
            assert (np.delete(c1, np.arange(sa, sa + n)) == C.SCRATCH_FILL).all(), valid.labels[k]
        else:
            assert (c1 == C.SCRATCH_FILL).all()


@pytest.mark.gpu
def test_gpu_status_matrix_equals_the_host(harness, malformed, tmp_path):
    # the host run (AddressSanitizer where the toolchain has it) comes first; the device gets the table only once it passed
    exe, _ = harness
    hst, hout, hscratch = C.run_host(exe, malformed, tmp_path)
    _check_malformed(malformed, hst, hout, hscratch)
    st, out, scratch = C.run_device(malformed)
    assert st == hst, [(l, a, b) for l, a, b in zip(malformed.labels, st, hst) if a != b]
    assert np.array_equal(out, hout) and np.array_equal(scratch, hscratch)
