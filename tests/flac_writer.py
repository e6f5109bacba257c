"""Test-only FLAC encoder that emits exactly what it is told, frame by frame: subframe type, predictor order, coefficient
precision and shift, Rice method, partition order, escapes, wasted bits, channel assignment, block-size and sample-rate codes,
fixed or variable blocking.  CRCs and the STREAMINFO MD5 are computed here.  Its input PCM is the truth a decoder is checked
against, so round trips do not depend on any decoder.  `streams()` is the catalogue the tests run."""
from __future__ import annotations

import hashlib
from dataclasses import dataclass, field
from typing import Dict, List, Optional

import numpy as np

from flac_oracle import crc8, crc16

_RATE_CODES = {88200: 1, 176400: 2, 192000: 3, 8000: 4, 16000: 5, 22050: 6, 24000: 7, 32000: 8, 44100: 9, 48000: 10, 96000: 11}


class _BW:
    def __init__(self):
        self.acc, self.n = 0, 0

    def put(self, v: int, k: int):
        if k:
            self.acc = (self.acc << k) | (v & ((1 << k) - 1))
            self.n += k

    def unary(self, q: int):
        self.put(1, q + 1)

    def align(self):
        self.put(0, -self.n % 8)

    def bytes(self) -> bytes:
        assert self.n % 8 == 0
        return self.acc.to_bytes(self.n // 8, "big")


@dataclass
class Sub:
    """How to code one channel of one frame."""
    kind: str = "lpc"           # constant | verbatim | fixed | lpc
    order: int = 8
    precision: int = 12
    shift: Optional[int] = None  # None: chosen from the quantised coefficients
    coefs: Optional[List[int]] = None
    method: int = 0              # 0: 4-bit Rice parameters, 1: 5-bit
    porder: int = 0
    escape: tuple = ()           # partitions coded with the escape (raw width)
    params: Optional[List[int]] = None
    wasted: int = 0


@dataclass
class FrameSpec:
    block: int
    assignment: int = -1        # -1: independent channels; 8 left/side, 9 side/right, 10 mid/side
    subs: List[Sub] = field(default_factory=list)  # one per coded channel (the last one repeats)
    bs_code: Optional[int] = None
    sr_code: int = 0


def _bs_code(b: int) -> int:
    if b == 192:
        return 1
    for c in range(2, 6):
        if b == 576 << (c - 2):
            return c
    for c in range(8, 16):
        if b == 256 << (c - 8):
            return c
    return 6 if b <= 256 else 7


def _utf8(v: int) -> bytes:
    if v < 0x80:
        return bytes([v])
    for more in range(1, 7):  # `more` continuation bytes carry 6 bits each, the lead byte 6 - more
        if v < (1 << (6 * more + 6 - more)):
            lead = (0xFF << (7 - more)) & 0xFF
            out = [lead | (v >> (6 * more))]
            out += [0x80 | ((v >> (6 * k)) & 0x3F) for k in range(more - 1, -1, -1)]
            return bytes(out)
    raise ValueError(v)


def _residual(bw: _BW, res: List[int], bs: int, order: int, sub: Sub):
    bw.put(sub.method, 2)
    bw.put(sub.porder, 4)
    pbits = 5 if sub.method else 4
    esc, kmax = (1 << pbits) - 1, (1 << pbits) - 2
    psize = bs >> sub.porder
    i = 0
    for p in range(1 << sub.porder):
        n = psize - (order if p == 0 else 0)
        part = res[i:i + n]
        i += n
        if p in sub.escape:
            w = max((int(abs(r) if r >= 0 else abs(r) - 1).bit_length() + 1 for r in part), default=0)
            if all(r == 0 for r in part):
                w = 0
            bw.put(esc, pbits)
            bw.put(w, 5)
            for r in part:
                bw.put(r, w)
            continue
        us =[2 * r if r >= 0 else -2 * r - 1 for r in part]
        if sub.params is not None:
            k = sub.params[p % len(sub.params)]
        else:
            mean = (sum(us) / len(us)) if us else 0
            k = max(0, min(kmax, int(np.log2(mean)) if mean >= 1 else 0))
        bw.put(k, pbits)
        for u in us:
            bw.unary(u >> k)
            bw.put(u, k)


def _subframe(bw: _BW, s: List[int], sbps: int, sub: Sub):
    bs = len(s)
    if sub.wasted:
        assert all(v % (1 << sub.wasted) == 0 for v in s)
        s = [v >> sub.wasted for v in s]
        sbps -= sub.wasted
    typ = {"constant": 0, "verbatim": 1}.get(sub.kind)
    if sub.kind == "fixed":
        typ = 8 + sub.order
    elif sub.kind == "lpc":
        typ = 31 + sub.order
    bw.put(0, 1)
    bw.put(typ, 6)
    bw.put(1 if sub.wasted else 0, 1)
    if sub.wasted:
        bw.unary(sub.wasted - 1)
    if sub.kind == "constant":
        assert len(set(s)) == 1
        bw.put(s[0], sbps)
        return
    if sub.kind == "verbatim":
        for v in s:
            bw.put(v, sbps)
        return
    order = sub.order
    for v in s[:order]:
        bw.put(v, sbps)
    if sub.kind == "fixed":
        coefs, shift = [[], [1], [2, -1], [3, -3, 1], [4, -6, 4, -1]][order], 0
    else:
        coefs, shift = sub.coefs, sub.shift
        if coefs is None:  # least squares on the block, quantised to `precision` bits
            x = np.asarray(s, dtype=np.float64)
            A = np.stack([x[order - 1 - j: bs - 1 - j] for j in range(order)], axis=1) if bs > order else np.zeros((0, order))
            a = np.linalg.lstsq(A, x[order:], rcond=None)[0] if A.shape[0] >= order else np.zeros(order)
            cmax = (1 << (sub.precision - 1)) - 1
            top = max(float(np.abs(a).max()), 1e-9)
            if shift is None:
                shift = 0 if cmax == 0 else max(0, min(15, int(np.floor(np.log2(cmax / top)))))
            coefs = [int(np.clip(np.round(c * (1 << shift)), -cmax - 1, cmax)) for c in a]
        bw.put(sub.precision - 1, 4)
        bw.put(shift, 5)
        for c in coefs:
            bw.put(c, sub.precision)
    res = [s[i] - (sum(c * s[i - 1 - j] for j, c in enumerate(coefs)) >> shift) for i in range(order, bs)]
    _residual(bw, res, bs, order, sub)


def encode(pcm: np.ndarray, sample_rate: int, frames: List[FrameSpec], variable: bool = False):
    """pcm: (n, channels) int16.  Returns (file bytes, log) where log is [(byte offset, first sample, block size)]."""
    pcm = np.asarray(pcm, dtype=np.int64)
    n, nch = pcm.shape
    assert sum(f.block for f in frames) == n
    body, log, first = [], [], 0
    audio_offset = 4 + 4 + 34
    pos = audio_offset
    for fi, fs in enumerate(frames):
        bs = fs.block
        x = pcm[first:first + bs]
        bs_code = fs.bs_code if fs.bs_code is not None else _bs_code(bs)
        ch_code = nch - 1 if fs.assignment < 0 else fs.assignment
        hdr = bytearray([0xFF, 0xF8 | int(variable), bs_code << 4 | fs.sr_code, ch_code << 4 | 4 << 1])
        hdr += _utf8(first if variable else fi)
        if bs_code == 6:
            hdr += bytes([bs - 1])
        elif bs_code == 7:
            hdr += (bs - 1).to_bytes(2, "big")
        if fs.sr_code == 12:
            hdr += bytes([sample_rate // 1000])
        elif fs.sr_code == 13:
            hdr += sample_rate.to_bytes(2, "big")
        elif fs.sr_code == 14:
            hdr += (sample_rate // 10).to_bytes(2, "big")
        hdr.append(crc8(bytes(hdr)))
        if fs.assignment == 8:
            chans, side = [x[:, 0], x[:, 0] - x[:, 1]], [False, True]
        elif fs.assignment == 9:
            chans, side = [x[:, 0] - x[:, 1], x[:, 1]], [True, False]
        elif fs.assignment == 10:
            chans, side = [(x[:, 0] + x[:, 1]) >> 1, x[:, 0] - x[:, 1]], [False, True]
        else:
            chans, side = [x[:, c] for c in range(nch)], [False] * nch
        bw = _BW()
        for c, ch in enumerate(chans):
            sub = fs.subs[min(c, len(fs.subs) - 1)] if fs.subs else Sub()
            _subframe(bw, [int(v) for v in ch], 16 + side[c], sub)
        bw.align()
        frame = bytes(hdr) + bw.bytes()
        frame += crc16(frame).to_bytes(2, "big")
        log.append((pos, first, bs))
        body.append(frame)
        pos += len(frame)
        first += bs
    sizes = [len(b) for b in body]
    blocks = [f.block for f in frames]
    minb = min(blocks[:-1]) if len(blocks) > 1 and not variable else min(blocks)
    if not variable:
        minb = maxb = blocks[0]
    else:
        maxb = max(blocks)
    md5 = hashlib.md5(np.ascontiguousarray(pcm.astype("<i2")).tobytes()).digest()
    v = (minb << 128) | (maxb << 112) | (min(sizes) << 88) | (max(sizes) << 64) | (sample_rate << 44) | ((nch - 1) << 41) \
        | (15 << 36) | n
    info = v.to_bytes(18, "big") + md5
    head = b"fLaC" + bytes([0x80, 0, 0, 34]) + info
    return head + b"".join(body), log


# ---- the catalogue ------------------------------------------------------------------------------------------------
def _speech_like(rs, n, nch=1, amp=3000):
    """Smooth correlated noise (what LPC is for) with a little independent noise per channel."""
    base = np.convolve(rs.randn(n + 64), np.hanning(16), mode="same")[:n]
    out = np.stack([base * amp + rs.randn(n) * (amp / 20) * (c + 1) for c in range(nch)], axis=1)
    return np.clip(np.round(out), -32768, 32767).astype(np.int64)


def streams(seed: int = 0) -> Dict[str, tuple]:
    """name -> (file bytes, log, pcm (n, channels) int16, sample rate)."""
    rs = np.random.RandomState(seed)
    out = {}

    def add(name, pcm, frames, sr=16000, variable=False):
        data, log = encode(pcm, sr, frames, variable)
        out[name] = (data, log, np.asarray(pcm, dtype=np.int16), sr)

    # every subframe type, fixed orders 0-4 and LPC orders 1-32, both Rice methods, partition orders 0-8, escapes
    subs = [Sub("constant"), Sub("verbatim")] + [Sub("fixed", order=o, porder=o % 3) for o in range(5)]
    subs += [Sub("lpc", order=o, precision=1 + (o * 7) % 15, method=o % 2, porder=min(o % 9, int(np.log2(512 // o))),
                 escape=(0,) if o % 5 == 0 else ()) for o in range(1, 33)]
    bs = 512
    pcm = _speech_like(rs, bs * len(subs))
    pcm[0:bs] = 1234  # the CONSTANT frame
    add("subframe_types", pcm, [FrameSpec(bs, subs=[s]) for s in subs])
    # 64-bit accumulation: precision 15, order 32, 17-bit side channel; large coefficients with a large shift
    pcm = _speech_like(rs, 4096 * 3, 2, amp=12000)
    big = [Sub("lpc", order=32, precision=15, shift=14, coefs=[int(v) for v in rs.randint(-16384, 16384, 32)], method=1, porder=3),
           Sub("lpc", order=32, precision=15, method=1, porder=5)]
    add("wide_accumulation", pcm, [FrameSpec(4096, assignment=10, subs=big), FrameSpec(4096, assignment=8, subs=big[::-1]),
                                   FrameSpec(4096, assignment=-1, subs=big)])
    # escapes: raw widths 0 (an all-zero partition) and up to 16, partition order 8, fixed Rice parameters
    pcm = _speech_like(rs, 4096)
    pcm[0:512] = 0
    add("escapes", pcm, [FrameSpec(2048, subs=[Sub("lpc", order=4, porder=3, escape=(0, 1, 5))]),
                         FrameSpec(2048, subs=[Sub("fixed", order=2, porder=8, escape=tuple(range(0, 256, 3)), method=1)])])
    # wasted bits
    pcm = (_speech_like(rs, 4096 * 2) >> 3) << 3
    add("wasted_bits", pcm, [FrameSpec(4096, subs=[Sub("lpc", order=6, wasted=3)]), FrameSpec(4096, subs=[Sub("fixed", order=2, wasted=2)])])
    # the four stereo modes
    pcm = _speech_like(rs, 1152 * 4, 2)
    add("stereo", pcm, [FrameSpec(1152, assignment=a, subs=[Sub("lpc", order=8), Sub("fixed", order=2)]) for a in (-1, 8, 9, 10)])
    # 3-8 channels
    for nch in range(3, 9):
        pcm = _speech_like(rs, 1024 * 2, nch)
        add(f"channels{nch}", pcm, [FrameSpec(1024, subs=[Sub("lpc", order=nch), Sub("verbatim"), Sub("fixed", order=3)])] * 2)
    # variable blocking and every block-size code (1-15)
    blocks = [192, 576, 1152, 2304, 4608, 17, 256, 300, 512, 1024, 2048, 4096, 8192, 16384, 32768, 65535, 4000]
    pcm = _speech_like(rs, sum(blocks))
    add("variable_blocking", pcm, [FrameSpec(b, subs=[Sub("lpc", order=min(12, b - 1), porder=0 if b % 2 else 1)]) for b in blocks],
        variable=True)
    # every sample-rate code: 0 and 12-14 on a 16 kHz stream, 1-11 on one short stream each
    pcm = _speech_like(rs, 4 * 256)
    add("rate_codes_16k", pcm, [FrameSpec(256, sr_code=c, subs=[Sub("fixed", order=1)]) for c in (0, 12, 13, 14)])
    for sr, code in _RATE_CODES.items():
        pcm = _speech_like(rs, 256)
        add(f"rate_code_{code}", pcm, [FrameSpec(256, sr_code=code, subs=[Sub("fixed", order=1)])], sr=sr)
    # fixed block size 16 and 2100 frames: frame numbers from 2048 on take three UTF-8 bytes
    pcm = _speech_like(rs, 16 * 2100)
    add("small_blocks", pcm, [FrameSpec(16, subs=[Sub("fixed", order=2)])] * 2100)
    # a planted false sync: VERBATIM samples whose bytes are a valid header (CRC-8 included) with the wrong frame number
    pcm = _speech_like(rs, 4096 * 3)
    fake = bytearray([0xFF, 0xF8, 0xC0 | 0, 0x08, 0x05])  # block code 12 (4096), mono, 16 bit, frame number 5
    fake.append(crc8(bytes(fake)))
    vals = np.frombuffer(bytes(fake), dtype=">i2").astype(np.int64)
    pcm[4096 + 10: 4096 + 13, 0] = vals
    add("false_sync", pcm, [FrameSpec(4096, subs=[Sub("lpc", order=8)]), FrameSpec(4096, subs=[Sub("verbatim")]),
                            FrameSpec(4096, subs=[Sub("lpc", order=8)])])
    return out
