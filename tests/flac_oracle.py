"""Test / bench infrastructure: a plain Python + numpy FLAC decoder (RFC 9639) that restates the format, frame by frame,
with no sync search (each frame starts where the previous one's CRC-16 ended).  It checks what a decoder must check and
raises `FlacError` otherwise.  Never imported by lhotse_b200."""
from __future__ import annotations

import hashlib
from dataclasses import dataclass
from typing import List, Tuple

import numpy as np


class FlacError(ValueError):
    pass


@dataclass
class StreamInfo:
    min_block: int
    max_block: int
    min_frame: int
    max_frame: int
    sample_rate: int
    channels: int
    bits_per_sample: int
    total_samples: int
    md5: bytes
    audio_offset: int


@dataclass
class Frame:
    byte_offset: int
    byte_length: int
    first_sample: int
    block_size: int
    variable: bool
    number: int
    channel_assignment: int


def crc8(data: bytes) -> int:
    crc = 0
    for b in data:
        crc ^= b
        for _ in range(8):
            crc = ((crc << 1) ^ 0x07) & 0xFF if crc & 0x80 else (crc << 1) & 0xFF
    return crc


_CRC16 = []
for _t in range(256):
    _c = _t << 8
    for _ in range(8):
        _c = ((_c << 1) ^ 0x8005) if _c & 0x8000 else (_c << 1)
    _CRC16.append(_c & 0xFFFF)


def crc16(data: bytes) -> int:
    crc = 0
    for b in data:
        crc = ((crc << 8) ^ _CRC16[(crc >> 8) ^ b]) & 0xFFFF
    return crc


class _Bits:
    """MSB-first reader over a '0'/'1' string (str.index finds the end of a unary code at C speed)."""

    def __init__(self, data: bytes, pos_bytes: int, end_bytes: int):
        self.s = "".join(format(b, "08b") for b in data[pos_bytes:end_bytes])
        self.pos = 0

    def u(self, k: int) -> int:
        if k == 0:
            return 0
        if self.pos + k > len(self.s):
            raise FlacError("frame truncated")
        v = int(self.s[self.pos:self.pos + k], 2)
        self.pos += k
        return v

    def s_(self, k: int) -> int:
        v = self.u(k)
        return v - (1 << k) if v >> (k - 1) else v

    def unary(self) -> int:
        try:
            j = self.s.index("1", self.pos)
        except ValueError:
            raise FlacError("frame truncated") from None
        q = j - self.pos
        self.pos = j + 1
        return q


def read_streaminfo(data: bytes) -> StreamInfo:
    if data[:4] != b"fLaC":
        raise FlacError("not a native FLAC stream")
    pos, si, last = 4, None, False
    while not last:
        hdr = data[pos:pos + 4]
        if len(hdr) < 4:
            raise FlacError("metadata truncated")
        last, typ, ln = bool(hdr[0] & 0x80), hdr[0] & 0x7F, int.from_bytes(hdr[1:4], "big")
        body = data[pos + 4:pos + 4 + ln]
        if typ == 0:
            v = int.from_bytes(body[:18], "big")  # 144 bits
            si = dict(min_block=v >> 128, max_block=(v >> 112) & 0xFFFF, min_frame=(v >> 88) & 0xFFFFFF,
                      max_frame=(v >> 64) & 0xFFFFFF, sample_rate=(v >> 44) & 0xFFFFF, channels=((v >> 41) & 7) + 1,
                      bits_per_sample=((v >> 36) & 31) + 1, total_samples=v & ((1 << 36) - 1), md5=bytes(body[18:34]))
        pos += 4 + ln
    if si is None:
        raise FlacError("no STREAMINFO")
    return StreamInfo(audio_offset=pos, **si)


_SS_BITS = {1: 8, 2: 12, 4: 16, 5: 20, 6: 24, 7: 32}


def _header(data: bytes, pos: int):
    b = data[pos:pos + 16]
    if len(b) < 6 or b[0] != 0xFF or (b[1] & 0xFE) != 0xF8:
        raise FlacError(f"no frame sync at byte {pos}")
    variable = b[1] & 1
    bs, sr, ch, ss = b[2] >> 4, b[2] & 15, b[3] >> 4, (b[3] >> 1) & 7
    if bs == 0 or sr == 15 or ch > 10 or ss == 3 or b[3] & 1:
        raise FlacError("reserved header code")
    c0 = b[4]
    n_more = 0 if c0 < 0x80 else next((k for k, m in ((1, 0xE0), (2, 0xF0), (3, 0xF8), (4, 0xFC), (5, 0xFE), (6, 0xFF))
                                        if (c0 & m) == ((m << 1) & 0xFF)), None)
    if n_more is None:
        raise FlacError("bad coded number")
    number = c0 & (0x7F >> (n_more + 1)) if n_more else c0
    i = 5
    for _ in range(n_more):
        if (b[i] & 0xC0) != 0x80:
            raise FlacError("bad coded number")
        number = (number << 6) | (b[i] & 0x3F)
        i += 1
    if bs == 1:
        block = 192
    elif bs <= 5:
        block = 576 << (bs - 2)
    elif bs == 6:
        block = b[i] + 1; i += 1
    elif bs == 7:
        block = (b[i] << 8 | b[i + 1]) + 1; i += 2
    else:
        block = 256 << (bs - 8)
    i += {12: 1, 13: 2, 14: 2}.get(sr, 0)
    if crc8(b[:i]) != b[i]:
        raise FlacError("header CRC-8")
    return dict(variable=variable, block=block, ch=ch, ss=ss, number=number, length=i + 1)


def _residual(br: _Bits, bs: int, order: int) -> List[int]:
    method = br.u(2)
    if method > 1:
        raise FlacError("reserved residual method")
    pbits = 5 if method else 4
    esc = (1 << pbits) - 1
    porder = br.u(4)
    psize = bs >> porder
    if (porder and bs % (1 << porder)) or psize < order:
        raise FlacError("partition order does not fit the block")
    out = []
    for p in range(1 << porder):
        n = psize - (order if p == 0 else 0)
        k = br.u(pbits)
        if k == esc:
            w = br.u(5)
            out.extend(br.s_(w) if w else 0 for _ in range(n))
        else:
            for _ in range(n):
                u = (br.unary() << k) | br.u(k)
                out.append((u >> 1) ^ -(u & 1))
    return out


def _subframe(br: _Bits, bs: int, sbps: int) -> List[int]:
    if br.u(1):
        raise FlacError("subframe pad bit")
    typ = br.u(6)
    wasted = 0
    if br.u(1):
        wasted = br.unary() + 1
        if wasted >= sbps:
            raise FlacError("wasted bits")
        sbps -= wasted
    if typ == 0:
        s = [br.s_(sbps)] * bs
    elif typ == 1:
        s = [br.s_(sbps) for _ in range(bs)]
    elif 8 <= typ <= 12 or typ >= 32:
        order = typ - 8 if typ <= 12 else typ - 31
        if order > bs:
            raise FlacError("order above block size")
        s = [br.s_(sbps) for _ in range(order)]
        if typ >= 32:
            prec = br.u(4) + 1
            if prec == 16:
                raise FlacError("coefficient precision 1111")
            shift = br.s_(5)
            if shift < 0:
                raise FlacError("negative shift")
            coefs = [br.s_(prec) for _ in range(order)]
        else:
            coefs, shift = [[], [1], [2, -1], [3, -3, 1], [4, -6, 4, -1]][order], 0
        res = _residual(br, bs, order)
        rc = coefs[::-1]  # s[i] = r[i] + (sum_j c[j] s[i-1-j]) >> shift
        for r in res:
            s.append(r + (sum(c * x for c, x in zip(rc, s[-order:])) >> shift) if order else r)
        lo, hi = -(1 << (sbps - 1)), (1 << (sbps - 1)) - 1
        if any(v < lo or v > hi for v in s):
            raise FlacError("sample outside its subframe width")
    else:
        raise FlacError("reserved subframe type")
    return [v << wasted for v in s] if wasted else s


def decode_frame(data: bytes, pos: int, si: StreamInfo) -> Tuple[Frame, np.ndarray, int]:
    """(frame, samples (block, channels) int32, byte after the frame's CRC-16)."""
    h = _header(data, pos)
    if si.bits_per_sample != 16 or (h["ss"] not in (0, 4)):
        raise FlacError("only 16-bit streams")
    ch = h["ch"]
    nch = ch + 1 if ch < 8 else 2
    bs = h["block"]
    br = _Bits(data, pos + h["length"], pos + si.max_frame if si.max_frame else len(data))
    chans = []
    for c in range(nch):
        side = (ch == 8 and c == 1) or (ch == 9 and c == 0) or (ch == 10 and c == 1)
        chans.append(np.asarray(_subframe(br, bs, 16 + side), dtype=np.int64))
    if ch == 8:
        chans[1] = chans[0] - chans[1]
    elif ch == 9:
        chans[0] = chans[0] + chans[1]
    elif ch == 10:
        m = (chans[0] << 1) | (chans[1] & 1)
        chans = [(m + chans[1]) >> 1, (m - chans[1]) >> 1]
    end = pos + h["length"] + (br.pos + 7) // 8
    if end + 2 > len(data) or crc16(data[pos:end]) != int.from_bytes(data[end:end + 2], "big"):
        raise FlacError("frame CRC-16")
    pcm = np.stack(chans, axis=1)
    if pcm.min() < -32768 or pcm.max() > 32767:
        raise FlacError("sample outside int16")
    fr = Frame(byte_offset=pos, byte_length=end + 2 - pos, first_sample=-1, block_size=bs, variable=bool(h["variable"]),
               number=h["number"], channel_assignment=ch)
    return fr, pcm.astype(np.int32), end + 2


def decode(data: bytes) -> Tuple[StreamInfo, List[Frame], np.ndarray]:
    """The whole stream: (STREAMINFO, frames, samples (total, channels) int16)."""
    si = read_streaminfo(data)
    pos, first, frames, parts = si.audio_offset, 0, [], []
    while pos < len(data):
        fr, pcm, pos = decode_frame(data, pos, si)
        if pcm.shape[1] != si.channels:
            raise FlacError("channel count differs from STREAMINFO")
        want = first if fr.variable else len(frames)
        if fr.number != want:
            raise FlacError(f"frame {len(frames)} carries number {fr.number}, expected {want}")
        fr.first_sample = first
        first += fr.block_size
        frames.append(fr)
        parts.append(pcm)
    pcm = np.concatenate(parts).astype(np.int16) if parts else np.zeros((0, si.channels), np.int16)
    return si, frames, pcm


def md5_of(pcm: np.ndarray) -> bytes:
    return hashlib.md5(np.ascontiguousarray(pcm, dtype="<i2").tobytes()).digest()
