"""Test-only FLAC encoder that emits exactly what it is told, frame by frame: subframe type, predictor order, coefficient
precision and shift, Rice method, partition order, escapes, wasted bits, channel assignment, block-size and sample-rate codes,
fixed or variable blocking.  CRCs and the STREAMINFO MD5 are computed here.  Its input PCM is the truth a decoder is checked
against, so round trips do not depend on any decoder.  `streams()` is the catalogue the tests run.

Every field is checked against its width: a value that does not fit (a 32-bit escape, a Rice parameter above its method's
maximum, a residual outside int32, a block or frame too large for STREAMINFO) raises instead of being written wrapped.
`frame()` emits one frame with no stream around it.  `Sub.raw` and `FrameSpec.raw` write chosen header and subframe fields
as given (CRC-8 and CRC-16 are recomputed), so a malformed frame whose CRCs hold can be built.  `encode(..., facts=)` and
`frame(..., facts=)` record what the frames exercise (Rice parameters, quotients, escape widths, ...) into a dict of sets."""
from __future__ import annotations

import hashlib
from dataclasses import dataclass, field
from typing import Dict, List, Optional

import numpy as np

from flac_oracle import crc8, crc16

_RATE_CODES = {88200: 1, 176400: 2, 192000: 3, 8000: 4, 16000: 5, 22050: 6, 24000: 7, 32000: 8, 44100: 9, 48000: 10, 96000: 11}


def _need(ok: bool, what: str):
    if not ok:
        raise ValueError(what)


def _note(facts: Optional[dict], key: str, value):
    if facts is not None:
        facts.setdefault(key, set()).add(value)


class _BW:
    def __init__(self):
        self.acc, self.n = 0, 0

    def put(self, v: int, k: int):
        """`v` in `k` bits, as an unsigned or a two's complement value; anything wider raises."""
        _need(v == 0 if k == 0 else -(1 << (k - 1)) <= v < (1 << k), f"{v} does not fit in {k} bits")
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
    # fields written as given instead of the coded ones (the rest of the subframe is coded from the fields above):
    # pad, type, wasted (k, written as k - 1 in unary), precision_code, shift, method, porder, and tail: a list of
    # (value, bits) written in place of the residual's partitions
    raw: Dict[str, object] = field(default_factory=dict)


@dataclass
class FrameSpec:
    block: int
    assignment: int = -1        # -1: independent channels; 8 left/side, 9 side/right, 10 mid/side
    subs: List[Sub] = field(default_factory=list)  # one per coded channel (the last one repeats)
    bs_code: Optional[int] = None
    sr_code: int = 0
    # the coded channels (after decorrelation) as given, instead of being derived from the PCM: lets a subframe hold
    # samples no int16 PCM decorrelates to
    chans: Optional[List[List[int]]] = None
    # header fields written as given (ch_code, ss_code), and body edits before the CRC-16: trim (drop the last bytes of the
    # subframes) and pad (append zero bytes)
    raw: Dict[str, int] = field(default_factory=dict)


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
    _need(0 <= v < 1 << 36, f"coded number {v} does not fit in 36 bits")
    if v < 0x80:
        return bytes([v])
    for more in range(1, 7):  # `more` continuation bytes carry 6 bits each, the lead byte 6 - more
        if v < (1 << (6 * more + 6 - more)):
            lead = (0xFF << (7 - more)) & 0xFF
            out = [lead | (v >> (6 * more))]
            out += [0x80 | ((v >> (6 * k)) & 0x3F) for k in range(more - 1, -1, -1)]
            return bytes(out)
    raise ValueError(v)


def _residual(bw: _BW, res: List[int], bs: int, order: int, sub: Sub, facts: Optional[dict]):
    _need(sub.method in (0, 1), f"residual method {sub.method}")
    _need(0 <= sub.porder <= 15, f"partition order {sub.porder}")
    psize = bs >> sub.porder
    _need(bs % (1 << sub.porder) == 0 and psize >= order, f"partition order {sub.porder} does not fit block {bs}, order {order}")
    _need(all(-(1 << 31) <= r < (1 << 31) for r in res), "residual outside int32")
    bw.put(sub.raw.get("method", sub.method), 2)
    bw.put(sub.raw.get("porder", sub.porder), 4)
    if "tail" in sub.raw:
        for v, k in sub.raw["tail"]:
            bw.put(v, k)
        return
    pbits = 5 if sub.method else 4
    esc, kmax = (1 << pbits) - 1, (1 << pbits) - 2
    _note(facts, "porder", sub.porder)
    if psize == order:
        _note(facts, "empty_first_partition", (order, sub.porder))
    i = 0
    for p in range(1 << sub.porder):
        n = psize - (order if p == 0 else 0)
        part = res[i:i + n]
        i += n
        if p in sub.escape:
            w = max((int(abs(r) if r >= 0 else abs(r) - 1).bit_length() + 1 for r in part), default=0)
            if all(r == 0 for r in part):
                w = 0
            _need(w <= 31, f"escape width {w}")
            _note(facts, "escape", w)
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
        _need(0 <= k <= kmax, f"Rice parameter {k} with method {sub.method}")
        _note(facts, "rice", (sub.method, k))
        if us:
            _note(facts, "quotient", max(us) >> k)
        bw.put(k, pbits)
        for u in us:
            bw.unary(u >> k)
            bw.put(u & ((1 << k) - 1), k)


def _subframe(bw: _BW, s: List[int], sbps: int, sub: Sub, facts: Optional[dict]):
    bs = len(s)
    raw = sub.raw
    _need(0 <= sub.wasted < sbps, f"{sub.wasted} wasted bits of {sbps}")
    if sub.wasted:
        _need(all(v % (1 << sub.wasted) == 0 for v in s), "samples do not have the wasted bits")
        _note(facts, "wasted", (sub.wasted, sbps))
        s = [v >> sub.wasted for v in s]
        sbps -= sub.wasted
    typ = {"constant": 0, "verbatim": 1}.get(sub.kind)
    if sub.kind == "fixed":
        _need(0 <= sub.order <= 4, f"fixed order {sub.order}")
        typ = 8 + sub.order
    elif sub.kind == "lpc":
        _need(1 <= sub.order <= 32, f"LPC order {sub.order}")
        typ = 31 + sub.order
    _need(typ is not None, f"subframe kind {sub.kind}")
    bw.put(raw.get("pad", 0), 1)
    bw.put(raw.get("type", typ), 6)
    wasted = raw.get("wasted", sub.wasted)
    bw.put(1 if wasted else 0, 1)
    if wasted:
        bw.unary(wasted - 1)
    if sub.kind == "constant":
        _need(len(set(s)) == 1, "a CONSTANT subframe of different samples")
        bw.put(s[0], sbps)
        return
    if sub.kind == "verbatim":
        for v in s:
            bw.put(v, sbps)
        return
    order = sub.order
    _need(order <= bs, f"order {order} above block {bs}")
    for v in s[:order]:
        bw.put(v, sbps)
    if sub.kind == "fixed":
        coefs, shift = [[], [1], [2, -1], [3, -3, 1], [4, -6, 4, -1]][order], 0
    else:
        _need(1 <= sub.precision <= 15, f"coefficient precision {sub.precision}")
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
        _need(len(coefs) == order and 0 <= shift <= 15, f"{len(coefs)} coefficients for order {order}, shift {shift}")
        bw.put(raw.get("precision_code", sub.precision - 1), 4)
        bw.put(raw.get("shift", shift), 5)
        for c in coefs:
            bw.put(c, sub.precision)
        lg = max(0, (order - 1).bit_length())  # the decoder's ceil(log2(order))
        extreme = min(coefs) == -(1 << (sub.precision - 1)) and min(s) == -(1 << (sbps - 1))
        _note(facts, "accumulation", (sub.precision + sbps + lg, extreme))
    res = [s[i] - (sum(c * s[i - 1 - j] for j, c in enumerate(coefs)) >> shift) for i in range(order, bs)]
    _residual(bw, res, bs, order, sub, facts)


def frame(x: Optional[np.ndarray], fs: FrameSpec, number: int, variable: bool = False, sample_rate: int = 16000,
          facts: Optional[dict] = None) -> bytes:
    """One frame: x (fs.block, channels) int PCM (None when fs.chans gives the coded channels), `number` the frame number
    (fixed blocking) or first sample number (variable blocking).  Header, subframes, CRC-8 and CRC-16, nothing else."""
    bs = fs.block
    bs_code = fs.bs_code if fs.bs_code is not None else _bs_code(bs)
    _need(1 <= bs <= 65536, f"block size {bs}")
    fixed = {1: 192, 2: 576, 3: 1152, 4: 2304, 5: 4608, **{c: 256 << (c - 8) for c in range(8, 16)}}
    _need(bs <= 256 if bs_code == 6 else bs == fixed.get(bs_code) or bs_code == 7, f"block size {bs} with block-size code {bs_code}")
    if fs.chans is not None:
        chans = [np.asarray(c, dtype=np.int64) for c in fs.chans]
        nch = len(chans)
    else:
        x = np.asarray(x, dtype=np.int64)
        nch = x.shape[1]
        _need(x.shape[0] == bs, "PCM rows differ from the block size")
        if fs.assignment == 8:
            chans = [x[:, 0], x[:, 0] - x[:, 1]]
        elif fs.assignment == 9:
            chans = [x[:, 0] - x[:, 1], x[:, 1]]
        elif fs.assignment == 10:
            chans = [(x[:, 0] + x[:, 1]) >> 1, x[:, 0] - x[:, 1]]
        else:
            chans = [x[:, c] for c in range(nch)]
        _note(facts, "assignment", (fs.assignment, bool(all(x[:, c].min() == -32768 and x[:, c].max() == 32767 for c in range(nch)))))
    side = {8: [False, True], 9: [True, False], 10: [False, True]}.get(fs.assignment, [False] * nch)
    _need(1 <= nch <= 8 and (fs.assignment < 0 or nch == 2), f"{nch} channels with assignment {fs.assignment}")
    ch_code = nch - 1 if fs.assignment < 0 else fs.assignment
    hdr = bytearray([0xFF, 0xF8 | int(variable), bs_code << 4 | fs.sr_code,
                     fs.raw.get("ch_code", ch_code) << 4 | fs.raw.get("ss_code", 4) << 1])
    hdr += _utf8(number)
    _note(facts, "block", bs)
    _note(facts, "coded_number_bytes", len(_utf8(number)))
    if bs_code == 6:
        hdr += bytes([bs - 1])
    elif bs_code == 7:
        hdr += (bs - 1).to_bytes(2, "big")
    _need(fs.sr_code not in (12, 13, 14) or 0 <= {12: sample_rate // 1000, 13: sample_rate, 14: sample_rate // 10}[fs.sr_code]
          < (256 if fs.sr_code == 12 else 65536), f"sample rate {sample_rate} with code {fs.sr_code}")
    if fs.sr_code == 12:
        hdr += bytes([sample_rate // 1000])
    elif fs.sr_code == 13:
        hdr += sample_rate.to_bytes(2, "big")
    elif fs.sr_code == 14:
        hdr += (sample_rate // 10).to_bytes(2, "big")
    hdr.append(crc8(bytes(hdr)))
    bw = _BW()
    for c, ch in enumerate(chans):
        sub = fs.subs[min(c, len(fs.subs) - 1)] if fs.subs else Sub()
        _subframe(bw, [int(v) for v in ch], 16 + side[c], sub, facts)
    bw.align()
    body = bw.bytes()
    body = body[:len(body) - fs.raw.get("trim", 0)] + bytes(fs.raw.get("pad", 0))
    out = bytes(hdr) + body
    return out + crc16(out).to_bytes(2, "big")


def _streaminfo(minb: int, maxb: int, minf: int, maxf: int, sample_rate: int, nch: int, n: int, md5: bytes) -> bytes:
    _need(1 <= minb <= maxb < 1 << 16, f"block sizes {minb}..{maxb} do not fit STREAMINFO's 16-bit fields")
    _need(0 <= minf <= maxf < 1 << 24, f"frame sizes {minf}..{maxf} do not fit STREAMINFO's 24-bit fields")
    _need(0 < sample_rate < 1 << 20 and 1 <= nch <= 8 and 0 <= n < 1 << 36, "sample rate, channels or length")
    v = (minb << 128) | (maxb << 112) | (minf << 88) | (maxf << 64) | (sample_rate << 44) | ((nch - 1) << 41) | (15 << 36) | n
    return v.to_bytes(18, "big") + md5


def encode(pcm: np.ndarray, sample_rate: int, frames: List[FrameSpec], variable: bool = False, facts: Optional[dict] = None):
    """pcm: (n, channels) int16.  Returns (file bytes, log) where log is [(byte offset, first sample, block size)]."""
    pcm = np.asarray(pcm, dtype=np.int64)
    n, nch = pcm.shape
    assert sum(f.block for f in frames) == n
    _need(n == 0 or (pcm.min() >= -32768 and pcm.max() <= 32767), "PCM outside int16")
    body, log, first = [], [], 0
    audio_offset = 4 + 4 + 34
    pos = audio_offset
    for fi, fs in enumerate(frames):
        data = frame(pcm[first:first + fs.block], fs, first if variable else fi, variable, sample_rate, facts)
        log.append((pos, first, fs.block))
        body.append(data)
        pos += len(data)
        first += fs.block
    sizes = [len(b) for b in body]
    blocks = [f.block for f in frames]
    minb = min(blocks[:-1]) if len(blocks) > 1 and not variable else min(blocks)
    if not variable:
        minb = maxb = blocks[0]
    else:
        maxb = max(blocks)
    md5 = hashlib.md5(np.ascontiguousarray(pcm.astype("<i2")).tobytes()).digest()
    info = _streaminfo(minb, maxb, min(sizes), max(sizes), sample_rate, nch, n, md5)
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
