"""Shared by the FLAC decoder's edge tests: a named table of valid frames that reach the decoder's edges, a matrix of
malformed frames whose CRCs hold (each with the status it must give), both laid out as one b200feat_flac_job table, and
the two ways to run such a table: the host check's `jobs` mode (scripts/micro/flac_host_check.cu, the decoder's own
__host__ __device__ code, under AddressSanitizer where the toolchain has it) and the device (`engine.flac_decode`)."""
from __future__ import annotations

import os
import shutil
import subprocess
from dataclasses import dataclass, field
from typing import List, Optional

import numpy as np

import flac_writer as W
from flac_oracle import FlacError, _header
from flac_writer import FrameSpec, Sub

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT_FILL = -12345            # int16 sentinel of the output buffer
SCRATCH_FILL = 0x5A5A5A5A    # int32 sentinel of the scratch buffer

OK, EJOB, EHEADER, ECRC, ERESERVED, EPRECISION, ESHIFT, EPARTITION, ERANGE, ETRUNCATED, ELENGTH = range(11)


@dataclass
class Edge:
    """Valid frames: a stream written by `W.encode` (checked whole by the oracle and the host index too), or, with
    stream=False, bare frames for the direct ABI only (numbered from `first_number`)."""
    name: str
    pcm: np.ndarray
    specs: List[FrameSpec]
    variable: bool = False
    stream: bool = True
    first_number: int = 0


@dataclass
class Frame:
    edge: str
    data: bytes
    number: int
    variable: bool
    pcm: np.ndarray              # (block, channels) int16: the writer's input, the truth
    scratch: Optional[np.ndarray] = None  # a decorrelated pair's first coded channel (what the decoder leaves in scratch)


def _full_scale_stereo(rs, n):
    x = rs.randint(-32768, 32768, size=(n, 2))
    x[rs.rand(n, 2) < 0.5] = -32768
    x[rs.rand(n, 2) < 0.3] = 32767
    x[:4] = [[-32768, -32768], [-32768, 32767], [32767, -32768], [32767, 32767]]
    return x


def edges() -> List[Edge]:
    rs = np.random.RandomState(1234)
    out = []
    # Rice parameter 0: quotients just over one 64-bit refill and up to 65535 (full-scale samples through fixed order 0);
    # a spike through fixed order 4 gives quotients near 96000
    x = rs.randint(-40, 41, size=(512, 1))
    x[[3, 50, 100, 200, 254, 255], 0] = [-32768, 32767, -32768, 32767, 40, -41]
    x[256 + 128, 0] = 8000
    out.append(Edge("rice0_long_unary", x, [FrameSpec(256, subs=[Sub("fixed", order=0, params=[0])]),
                                            FrameSpec(256, subs=[Sub("fixed", order=4, params=[0])])]))
    # the largest Rice parameters: 14 (method 0) and 30 (method 1) on full-scale noise
    x = rs.randint(-32768, 32768, size=(2048, 1))
    out.append(Edge("rice_max_params", x, [FrameSpec(1024, subs=[Sub("fixed", order=0, params=[14])]),
                                           FrameSpec(1024, subs=[Sub("fixed", order=1, method=1, params=[30])])]))
    # 32-bit accumulation at its bound: precision 15 + 16 bits + lg(order 2) = 32, coefficients and samples at their most
    # negative (products 2^29), residuals near -2^30 Rice-coded with parameter 30; then full-scale noise of both signs
    x = np.full((128, 1), -32768)
    x[64:, 0] = _full_scale_stereo(rs, 64)[:, 0]
    lpc2 = dict(order=2, precision=15, shift=0, coefs=[-16384, -16384], method=1)
    out.append(Edge("accumulation_at_32", x, [FrameSpec(64, subs=[Sub("lpc", params=[30], **lpc2)]),
                                              FrameSpec(64, subs=[Sub("lpc", **lpc2)])]))
    # one past the bound (precision 15 + 16 + lg(order 4) = 33, 64-bit): four products of 2^29 sum to 2^31, which a 32-bit
    # accumulator would wrap; order 3 (3 * 2^29) as well
    x = np.full((128, 1), -32768)
    out.append(Edge("accumulation_at_33", x, [FrameSpec(64, subs=[Sub("lpc", order=4, precision=15, shift=15, coefs=[-16384] * 4)]),
                                              FrameSpec(64, subs=[Sub("lpc", order=3, precision=15, shift=14, coefs=[-16384] * 3)])]))
    # escape widths 31 down to 17: residuals -32768 - (2^30 >> shift)
    x = np.full((16 * 15, 1), -32768)
    out.append(Edge("escape_widths", x, [FrameSpec(16, subs=[Sub("lpc", order=2, precision=15, shift=s, coefs=[-16384, -16384],
                                                                  escape=(0,))]) for s in range(1, 16)]))
    # partition orders 9-15 at one sample per partition; order 15 with fixed order 1 leaves the first partition empty
    blocks = [1 << p for p in range(9, 16)]
    x = W._speech_like(rs, sum(blocks))
    out.append(Edge("partition_orders", x, [FrameSpec(b, subs=[Sub("fixed", order=int(b == 32768), porder=b.bit_length() - 1)])
                                            for b in blocks], variable=True))
    # psize == order: LPC order 16 at partition order 8 of 4096, fixed order 4 at partition order 10 of 4096
    x = W._speech_like(rs, 4096 + 4096)
    out.append(Edge("empty_first_partition", x, [FrameSpec(4096, subs=[Sub("lpc", order=16, porder=8)]),
                                                 FrameSpec(4096, subs=[Sub("fixed", order=4, porder=10)])]))
    # full-scale stereo in every channel assignment: the 17-bit side channel, mid/side's >> 1 on negative values
    x = _full_scale_stereo(rs, 1024 * 8)
    out.append(Edge("full_scale_stereo", x, [FrameSpec(1024, assignment=a, subs=s) for a in (-1, 8, 9, 10)
                                             for s in ([Sub("lpc", order=8, precision=15), Sub("fixed", order=2)], [Sub("verbatim")])]))
    # the most wasted bits: 15 of a 16-bit channel, 16 of a 17-bit side channel; constant subframes on a left/side pair
    m = rs.choice([-32768, 0], size=(256 * 3, 1))
    out.append(Edge("wasted_15", m, [FrameSpec(256, subs=[Sub("verbatim", wasted=15)]), FrameSpec(256, subs=[Sub("fixed", order=1, wasted=15)]),
                                     FrameSpec(256, subs=[Sub("fixed", order=2, wasted=15, porder=3)])]))
    m = rs.choice([-32768, 0], size=(256, 1))
    x = np.concatenate([np.concatenate([m, m], axis=1)] * 3 + [np.tile([[1234, 1000]], (256, 1))])
    out.append(Edge("wasted_16_side", x, [FrameSpec(256, assignment=8, subs=[Sub("verbatim", wasted=15), Sub("verbatim", wasted=16)]),
                                          FrameSpec(256, assignment=9, subs=[Sub("constant", wasted=16), Sub("fixed", order=1, wasted=15)]),
                                          FrameSpec(256, assignment=10, subs=[Sub("fixed", order=2, wasted=15), Sub("verbatim", wasted=16)]),
                                          FrameSpec(256, assignment=8, subs=[Sub("constant")])]))
    # block sizes 1 and 65535 (variable blocking, ending in a 1-sample frame); LPC order 1 on one sample
    blocks = [1, 65535, 1, 7, 1]
    x = W._speech_like(rs, sum(blocks))
    out.append(Edge("block_sizes", x, [FrameSpec(1, subs=[Sub("verbatim")]), FrameSpec(65535, subs=[Sub("fixed", order=2)]),
                                       FrameSpec(1, subs=[Sub("lpc", order=1, precision=4, shift=0, coefs=[1])]),
                                       FrameSpec(7, subs=[Sub("fixed", order=3)]), FrameSpec(1, subs=[Sub("constant")])],
                    variable=True))
    # direct ABI only: block 65536 (above STREAMINFO's 16-bit maximum), and coded numbers of 4 to 7 bytes
    x = W._speech_like(rs, 65536, 2)
    out.append(Edge("block_65536", x, [FrameSpec(65536, assignment=10, subs=[Sub("lpc", order=12), Sub("fixed", order=2, porder=4)])],
                    stream=False, first_number=3))
    for n, variable in ((1 << 16, False), ((1 << 21) + 5, False), ((1 << 26) + 9, False), ((1 << 31) - 1, False),
                        (1 << 31, True), ((1 << 36) - 16, True)):
        x = W._speech_like(rs, 16)
        out.append(Edge(f"coded_number_{n}", x, [FrameSpec(16, subs=[Sub("fixed", order=2)])], variable=variable, stream=False,
                        first_number=n))
    return out


def build(edge: Edge, facts: Optional[dict] = None):
    """(stream bytes or None, [Frame])."""
    pcm = np.asarray(edge.pcm, dtype=np.int64)
    frames, data = [], None
    if edge.stream:
        data, log = W.encode(pcm, 16000, edge.specs, edge.variable, facts)
        ends = [o for o, _, _ in log[1:]] + [len(data)]
        raw = [(data[o:e], f, b) for (o, f, b), e in zip(log, ends)]
    else:
        raw, first = [], 0
        for k, fs in enumerate(edge.specs):
            num = edge.first_number + (first if edge.variable else k)
            raw.append((W.frame(pcm[first:first + fs.block], fs, num, edge.variable, 16000, facts), first, fs.block))
            first += fs.block
    for (b, first, bs), fs in zip(raw, edge.specs):
        x = pcm[first:first + bs]
        num = (first if edge.variable else len(frames)) if edge.stream else \
            edge.first_number + (first if edge.variable else len(frames))
        scratch = None
        if fs.assignment == 8:
            scratch = x[:, 0]
        elif fs.assignment == 9:
            scratch = x[:, 0] - x[:, 1]
        elif fs.assignment == 10:
            scratch = (x[:, 0] + x[:, 1]) >> 1
        frames.append(Frame(edge.name, b, num, edge.variable, x.astype(np.int16), scratch))
    return data, frames


# ---- job tables ------------------------------------------------------------------------------------------------------
@dataclass
class Table:
    data: bytes
    jobs: np.ndarray             # FLAC_JOB_DTYPE
    out_elems: int
    scratch_elems: int
    want_out: np.ndarray         # int16, OUT_FILL outside the windows (valid tables only)
    want_scratch: np.ndarray     # int32
    labels: List[str] = field(default_factory=list)
    want_status: List[int] = field(default_factory=list)


def _job_dtype():
    from lhotse_b200.engine import FLAC_JOB_DTYPE

    return FLAC_JOB_DTYPE


def valid_table(frames: List[Frame], seed: int = 5) -> Table:
    """Every channel of every frame as a full window, a random partial window and an empty one (count 0), at odd and even
    offsets, gaps of sentinel between them, shuffled; the last window ends exactly at out_elems."""
    rs = np.random.RandomState(seed)
    data = bytearray()
    spec = []  # (frame, src, ch, skip, count)
    for f in frames:
        src = len(data)
        data += f.data
        data += bytes(int(rs.randint(0, 4)))
        bs, nch = f.pcm.shape
        for ch in range(nch):
            spec.append((f, src, ch, 0, bs))
            a = int(rs.randint(0, bs))
            spec.append((f, src, ch, a, int(rs.randint(0, bs - a + 1))))
            spec.append((f, src, ch, int(rs.randint(0, bs + 1)), 0))
    order = rs.permutation(len(spec))
    jobs = np.zeros(len(spec), dtype=_job_dtype())
    want_out, want_scratch, labels = [], [], []
    pos = spos = 0
    for j, i in enumerate(order):
        f, src, ch, skip, count = spec[i]
        pos += int(rs.randint(0, 3))
        bs, nch = f.pcm.shape
        jobs[j] = (src, pos, -1, f.number, len(f.data), bs, nch, ch, skip, count, int(f.variable), 0)
        want_out.append((pos, f.pcm[skip:skip + count, ch]))
        if nch > 1:
            spos += int(rs.randint(0, 3))
            jobs[j]["scratch_elem"] = spos
            if f.scratch is not None:
                want_scratch.append((spos, f.scratch[skip:skip + count]))
            spos += count
        pos += count
        labels.append(f"{f.edge}#{f.number} ch{ch} [{skip}, +{count})")
    out = np.full(pos, OUT_FILL, dtype=np.int16)
    for p, v in want_out:
        out[p:p + len(v)] = v
    scr = np.full(spos, SCRATCH_FILL, dtype=np.int32)
    for p, v in want_scratch:
        scr[p:p + len(v)] = v
    return Table(bytes(data), jobs, pos, spos, out, scr, labels, [OK] * len(jobs))


def _mono(n=64, seed=0):
    return W._speech_like(np.random.RandomState(seed), n)


def malformed() -> List[tuple]:
    """(label, frame bytes, job fields, status): frames whose CRC-8 and CRC-16 hold but whose contents are wrong, and jobs
    that disagree with their frame or their launch.  Job fields not given come from the frame (number 5, fixed blocking,
    the whole block of channel 0); `dst`, `scratch` and `src` place the job relative to its own window."""
    x = _mono()
    st = W._speech_like(np.random.RandomState(1), 64, 2)

    def fr(spec, pcm=x, number=5, variable=False):
        return W.frame(None if spec.chans is not None else pcm[:spec.block], spec, number, variable)

    good = fr(FrameSpec(64, subs=[Sub("fixed", order=2)]))
    pair = fr(FrameSpec(64, assignment=8, subs=[Sub("fixed", order=1)]), st)
    indep = fr(FrameSpec(64, subs=[Sub("fixed", order=1)]), st)
    rows = [
        ("reserved subframe type 2", fr(FrameSpec(64, subs=[Sub("verbatim", raw={"type": 2})])), {}, ERESERVED),
        ("reserved subframe type 13", fr(FrameSpec(64, subs=[Sub("verbatim", raw={"type": 13})])), {}, ERESERVED),
        ("reserved subframe type 31", fr(FrameSpec(64, subs=[Sub("verbatim", raw={"type": 31})])), {}, ERESERVED),
        ("subframe pad bit", fr(FrameSpec(64, subs=[Sub("fixed", order=2, raw={"pad": 1})])), {}, ERESERVED),
        ("second subframe's pad bit", fr(FrameSpec(64, assignment=8, subs=[Sub("fixed", order=1), Sub("verbatim", raw={"pad": 1})]), st),
         {"channels": 2}, ERESERVED),
        ("residual method 2", fr(FrameSpec(64, subs=[Sub("fixed", order=2, raw={"method": 2})])), {}, ERESERVED),
        ("residual method 3", fr(FrameSpec(64, subs=[Sub("lpc", order=4, raw={"method": 3})])), {}, ERESERVED),
        ("precision code 1111", fr(FrameSpec(64, subs=[Sub("lpc", order=4, raw={"precision_code": 15})])), {}, EPRECISION),
        ("shift -1", fr(FrameSpec(64, subs=[Sub("lpc", order=4, raw={"shift": -1})])), {}, ESHIFT),
        ("shift -16", fr(FrameSpec(64, subs=[Sub("lpc", order=4, raw={"shift": -16})])), {}, ESHIFT),
        ("fixed order 4 on a block of 2", fr(FrameSpec(2, subs=[Sub("verbatim", raw={"type": 12})])), {}, EPARTITION),
        ("LPC order 32 on a block of 16", fr(FrameSpec(16, subs=[Sub("verbatim", raw={"type": 63})])), {}, EPARTITION),
        ("partition order 3 of a block of 300", fr(FrameSpec(300, subs=[Sub("fixed", order=1, raw={"porder": 3})]), _mono(300)), {},
         EPARTITION),
        ("partition order 6 of 64 under order 2", fr(FrameSpec(64, subs=[Sub("fixed", order=2, raw={"porder": 6})])), {}, EPARTITION),
        ("partition order 4 of 64 under LPC order 8", fr(FrameSpec(64, subs=[Sub("lpc", order=8, raw={"porder": 4})])), {}, EPARTITION),
        ("partition order 15 of 64", fr(FrameSpec(64, subs=[Sub("fixed", order=0, raw={"porder": 15})])), {}, EPARTITION),
        ("16 wasted bits of 16", fr(FrameSpec(64, subs=[Sub("verbatim", raw={"wasted": 16})])), {}, ERANGE),
        ("17 wasted bits of a 17-bit side", fr(FrameSpec(64, assignment=8, subs=[Sub("verbatim"), Sub("verbatim", raw={"wasted": 17})]), st),
         {"channels": 2}, ERANGE),
        ("sample 32768 in a 16-bit subframe", fr(FrameSpec(16, chans=[[32767] + [32768] * 15], subs=[Sub("fixed", order=1)])), {}, ERANGE),
        ("sample -65537 in a 17-bit side", fr(FrameSpec(16, assignment=8, chans=[[0] * 16, [-65536] + [-65537] * 15],
                                                        subs=[Sub("verbatim"), Sub("fixed", order=1)])), {"channels": 2}, ERANGE),
        ("left/side right -32769", fr(FrameSpec(16, assignment=8, chans=[[-32768] * 16, [1] * 16], subs=[Sub("verbatim")])),
         {"channels": 2, "want_channel": 1}, ERANGE),
        ("left/side right -32769, left wanted", fr(FrameSpec(16, assignment=8, chans=[[-32768] * 16, [1] * 16], subs=[Sub("verbatim")])),
         {"channels": 2, "want_channel": 0}, OK),
        ("side/right left 32768", fr(FrameSpec(16, assignment=9, chans=[[1] * 16, [32767] * 16], subs=[Sub("verbatim")])),
         {"channels": 2, "want_channel": 0}, ERANGE),
        ("mid/side left 32768", fr(FrameSpec(16, assignment=10, chans=[[32767] * 16, [1] * 16], subs=[Sub("verbatim")])),
         {"channels": 2, "want_channel": 0}, ERANGE),
        ("mid/side right -32769 late in the window", fr(FrameSpec(16, assignment=10, chans=[[0] * 12 + [-32768] * 4, [0] * 12 + [2] * 4],
                                                                   subs=[Sub("verbatim")])), {"channels": 2, "want_channel": 1}, ERANGE),
        ("Rice quotient 4 over parameter 30's limit", fr(FrameSpec(16, subs=[Sub("fixed", order=0, method=1, raw={"tail": [(30, 5), (1, 5)]})])),
         {}, ERANGE),
        ("Rice quotient 2^18 over parameter 14's limit", fr(FrameSpec(16, subs=[Sub("fixed", order=0, raw={"tail": [(14, 4), (1, 262145)]})])),
         {}, ERANGE),
        ("subframes trimmed by 3 bytes", fr(FrameSpec(64, subs=[Sub("fixed", order=2)], raw={"trim": 3})), {}, ETRUNCATED),
        ("VERBATIM trimmed by 1 byte", fr(FrameSpec(64, subs=[Sub("verbatim")], raw={"trim": 1})), {}, ETRUNCATED),
        ("unary past the end", fr(FrameSpec(16, subs=[Sub("fixed", order=0, raw={"tail": [(0, 4), (0, 60)]})])), {}, ETRUNCATED),
        ("second channel missing", fr(FrameSpec(64, assignment=8, subs=[Sub("fixed", order=1)], raw={"trim": 40}), st),
         {"channels": 2, "want_channel": 1}, ETRUNCATED),
        ("1 spare byte", fr(FrameSpec(64, subs=[Sub("fixed", order=2)], raw={"pad": 1})), {}, ELENGTH),
        ("7 spare bytes after a pair", fr(FrameSpec(64, assignment=10, subs=[Sub("lpc", order=4)], raw={"pad": 7}), st),
         {"channels": 2}, ELENGTH),
        ("job block size + 1", good, {"block_size": 65}, EHEADER),
        ("job block size - 1", good, {"block_size": 63, "count": 63}, EHEADER),
        ("job channels 2", good, {"channels": 2}, EHEADER),
        ("job variable blocking", good, {"variable_blocking": 1}, EHEADER),
        ("job coded number 6", good, {"coded_number": 6}, EHEADER),
        ("sample-size code 1 (8 bits)", fr(FrameSpec(64, subs=[Sub("fixed", order=2)], raw={"ss_code": 1})), {}, EHEADER),
        ("sample-size code 5 (20 bits)", fr(FrameSpec(64, subs=[Sub("fixed", order=2)], raw={"ss_code": 5})), {}, EHEADER),
        ("sample-size code 3 (reserved)", fr(FrameSpec(64, subs=[Sub("fixed", order=2)], raw={"ss_code": 3})), {}, EHEADER),
        ("sample-size code 0 (from STREAMINFO)", fr(FrameSpec(64, subs=[Sub("fixed", order=2)], raw={"ss_code": 0})), {}, OK),
        ("channel code 11 (reserved)", fr(FrameSpec(64, subs=[Sub("fixed", order=2)], raw={"ch_code": 11})), {"channels": 2}, EHEADER),
        ("job block size 0", good, {"block_size": 0}, EJOB),
        ("job block size 65537", good, {"block_size": 65537}, EJOB),
        ("job byte length 7", good, {"byte_length": 7}, EJOB),
        ("job channels 0", good, {"channels": 0}, EJOB),
        ("job channels 9", good, {"channels": 9}, EJOB),
        ("job channel -1", good, {"want_channel": -1}, EJOB),
        ("job channel 1 of 1", good, {"want_channel": 1}, EJOB),
        ("job skip -1", good, {"skip": -1}, EJOB),
        ("job skip 1 + count 64 > 64", good, {"skip": 1}, EJOB),
        ("job skip 65 + count 0 > 64", good, {"skip": 65, "count": 0}, EJOB),
        ("job count -1", good, {"count": -1}, EJOB),
        ("job src_byte -1", good, {"src": -1}, EJOB),
        ("job dst_elem -1", good, {"dst": -1}, EJOB),
        ("job window one past out_elems", good, {"dst": "end+1"}, EJOB),
        ("job window ending at out_elems", good, {"dst": "end"}, OK),
        ("pair without scratch", pair, {"channels": 2, "scratch": -1}, EJOB),
        ("pair without scratch, count 0", pair, {"channels": 2, "scratch": -1, "count": 0}, OK),
        ("pair whose scratch ends past scratch_elems", pair, {"channels": 2, "scratch": "end+1"}, EJOB),
        ("pair whose scratch ends at scratch_elems", pair, {"channels": 2, "scratch": "end", "want_channel": 1}, OK),
        ("independent stereo without scratch", indep, {"channels": 2, "scratch": -1, "want_channel": 1}, OK),
    ]
    return rows


def malformed_table() -> Table:
    """The malformed rows as one launch: each job its own output and scratch window with sentinel gaps between them."""
    rows = malformed()
    data = bytearray()
    jobs = np.zeros(len(rows), dtype=_job_dtype())
    pos = spos = 1
    late_out, late_scr = [], []
    for j, (label, b, kw, _) in enumerate(rows):
        src = len(data)
        data += b + bytes(3)
        try:
            h = _header(b, 0)
        except FlacError:  # reserved header codes: the job describes the frame as written
            h = dict(ch=0, block=64, variable=0, number=5)
        nch = h["ch"] + 1 if h["ch"] < 8 else 2
        bs = h["block"]
        job = dict(byte_length=len(b), block_size=bs, channels=min(nch, 8), want_channel=0, skip=0, count=bs,
                   variable_blocking=h["variable"], coded_number=h["number"])
        job.update({k: v for k, v in kw.items() if k not in ("src", "dst", "scratch")})
        count = max(job["count"], 0)
        jobs[j]["src_byte"] = kw.get("src", src)
        dst = kw.get("dst", pos)
        if isinstance(dst, str):
            late_out.append((j, dst))
        else:
            jobs[j]["dst_elem"] = dst
            pos += count + 2
        scr = kw.get("scratch", spos if job["channels"] > 1 else -1)
        if isinstance(scr, str):
            late_scr.append((j, scr))
        else:
            jobs[j]["scratch_elem"] = scr
            if scr >= 0:
                spos += count + 2
        for k in ("byte_length", "block_size", "channels", "want_channel", "skip", "count", "variable_blocking", "coded_number"):
            jobs[j][k] = job[k]
    # the windows placed against the ends of the buffers (exactly at the end, and one element past it), in room of their
    # own so that no other job's window overlaps them
    for j, how in late_out:
        jobs[j]["dst_elem"] = pos
        pos += int(jobs[j]["count"])
    out_elems = pos
    for j, how in late_out:
        jobs[j]["dst_elem"] = out_elems - int(jobs[j]["count"]) + (1 if how == "end+1" else 0)
    for j, how in late_scr:
        jobs[j]["scratch_elem"] = spos
        spos += int(jobs[j]["count"])
    scratch_elems = spos
    for j, how in late_scr:
        jobs[j]["scratch_elem"] = scratch_elems - int(jobs[j]["count"]) + (1 if how == "end+1" else 0)
    return Table(bytes(data), jobs, out_elems, scratch_elems, None, None, [r[0] for r in rows], [r[3] for r in rows])


def windows_mask(t: Table, n: int, field_: str) -> np.ndarray:
    """True at every element some job's window [dst, dst + count) covers (field_ = dst_elem or scratch_elem)."""
    m = np.zeros(n, dtype=bool)
    for job in t.jobs:
        a, c = int(job[field_]), int(job["count"])
        if a >= 0 and c > 0:
            m[a:min(a + c, n)] = True
    return m


# ---- the two runners -------------------------------------------------------------------------------------------------
def host_check_binary(tmp_path):
    """scripts/micro/flac_host_check.cu compiled for the host: (path, built with AddressSanitizer)."""
    import pytest

    src = os.path.join(ROOT, "scripts", "micro", "flac_host_check.cu")
    exe = str(tmp_path / "flac_host_check")
    gxx = shutil.which("g++")
    if gxx:
        for flags in (["-fsanitize=address", "-fno-omit-frame-pointer"], []):
            res = subprocess.run([gxx, "-x", "c++", "-std=c++17", "-O1", "-g", *flags, "-o", exe, src], capture_output=True, text=True)
            if res.returncode == 0:
                return exe, bool(flags)
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("no host compiler")
    res = subprocess.run([nvcc, "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-o", exe, src], capture_output=True, text=True)
    assert res.returncode == 0, res.stderr[-2000:]
    return exe, False


def run_host(exe, t: Table, tmp_path):
    """The table through the host check's `jobs` mode: (statuses, out int16, scratch int32).  Fails on any
    AddressSanitizer report or a refused table."""
    d = tmp_path
    (d / "data.bin").write_bytes(t.data)
    (d / "jobs.bin").write_bytes(t.jobs.tobytes())
    env = dict(os.environ, ASAN_OPTIONS="detect_leaks=0:abort_on_error=0")
    run = subprocess.run([exe, "jobs", str(d / "data.bin"), str(d / "jobs.bin"), str(t.out_elems), str(t.scratch_elems),
                          str(OUT_FILL), str(SCRATCH_FILL), str(d / "out.bin"), str(d / "scratch.bin")],
                         capture_output=True, text=True, env=env)
    assert run.returncode == 0 and "AddressSanitizer" not in run.stderr, run.stdout[-2000:] + run.stderr[-4000:]
    line = run.stdout.strip().splitlines()[-1].split()
    assert line[0] == "statuses" and len(line) == 1 + len(t.jobs), run.stdout[-2000:]
    return ([int(v) for v in line[1:]], np.fromfile(str(d / "out.bin"), dtype=np.int16),
            np.fromfile(str(d / "scratch.bin"), dtype=np.int32))


def run_device(t: Table, jobs: Optional[np.ndarray] = None):
    """The table (or the given subset of its jobs) in one `b200feat_flac_decode` launch: (statuses, out, scratch), on
    buffers filled with the sentinels first."""
    import torch

    from lhotse_b200.engine import flac_decode

    jobs = t.jobs if jobs is None else jobs
    dev = torch.device("cuda:0")
    data = torch.frombuffer(bytearray(t.data), dtype=torch.uint8).to(dev)
    jd = torch.from_numpy(np.ascontiguousarray(jobs).view(np.uint8).copy()).to(dev)
    out = torch.full((t.out_elems,), OUT_FILL, dtype=torch.int16, device=dev)
    scratch = torch.full((t.scratch_elems,), SCRATCH_FILL, dtype=torch.int32, device=dev) if t.scratch_elems else None
    status = torch.full((len(jobs),), -1, dtype=torch.int32, device=dev)
    flac_decode(data, jd, len(jobs), out, status, scratch)
    torch.cuda.synchronize()
    return (status.cpu().numpy().tolist(), out.cpu().numpy(),
            scratch.cpu().numpy() if scratch is not None else np.zeros(0, np.int32))
