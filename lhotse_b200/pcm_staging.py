"""
"Next" row §8f-2 of the scope contract: the data format right BEFORE the hot path.

The reference feeds its extractors float32 waveforms decoded per cut (`AudioSource.load_audio`, lhotse/audio/source.py:70 ->
libsndfile -> float32 = int16 / 32768; `read_audio_from_cuts`, lhotse/dataset/collation.py:541-598).  For 16-bit PCM WAV —
what most speech corpora are stored as — that decode is a widening copy: every sample crosses the host memory bus twice
(int16 in, float32 out) and then PCIe as 4 bytes.  Here the PCM bytes go from the file straight into ONE pinned int16
ragged buffer (no float copy on the host), cross PCIe as 2 bytes per sample and are widened on load inside the kernel
(`B200FEAT_I16`: x / 32768, bit-identical to the float32 route; tests/test_gpu_parity.py).

  * `WavPcm16.open(path)`        minimal RIFF/WAVE reader (PCM or EXTENSIBLE/PCM, 16 bit, any channel count)
  * `PcmStagingRing`             grow-only pinned int16 buffer; `stage(requests)` fills it back to back
  * `pcm16_request_for_cut(cut)` the (path, first sample, sample count, channel) of a lhotse MonoCut when it is eligible
                                 (one "file" source, .wav, no augmentation transforms); None otherwise
Everything here is host-side I/O; the arithmetic stays in the CUDA kernels.
"""
from __future__ import annotations

import math
import os
import struct
import threading
from collections import OrderedDict
from dataclasses import dataclass
from typing import List, Optional, Sequence, Tuple

import numpy as np
import torch

from .engine import _aligned_offsets, _zero_gaps

_WAVE_FORMAT_PCM = 0x0001
_WAVE_FORMAT_EXTENSIBLE = 0xFFFE
_KSDATAFORMAT_SUBTYPE_PCM = bytes.fromhex("0100000000001000800000aa00389b71")


class NotPcm16Wav(ValueError):
    """The file is not a little-endian RIFF/WAVE file with 16-bit integer PCM samples."""


class _FdCache:
    """A few read-only descriptors kept open across cuts (a corpus job reads thousands of cuts out of the same recordings:
    one open + close per cut costs as much as the read itself).  Reads use `os.preadv`, which carries its own offset, so
    threads share a descriptor.  A descriptor is only ever closed when no read is using it: `acquire` / `release` count the
    readers, and an entry that is evicted (capacity) or superseded (the file's size / mtime changed) while in use is closed
    by its last reader — a closed descriptor number can be handed out again by the OS to ANOTHER file, so closing under a
    concurrent `preadv` would not fail loudly, it would read the wrong audio."""

    class _Entry:
        __slots__ = ("fd", "stamp", "users", "dead")

        def __init__(self, fd, stamp):
            self.fd, self.stamp, self.users, self.dead = fd, stamp, 0, False

    def __init__(self, capacity: int = 64):
        self._lock = threading.Lock()
        self._fds: "OrderedDict[str, _FdCache._Entry]" = OrderedDict()
        self._capacity = capacity

    def _retire(self, ent) -> None:  # lock held
        ent.dead = True
        if ent.users == 0:
            os.close(ent.fd)

    def acquire(self, path: str, stamp: Tuple[int, int]) -> "_FdCache._Entry":
        with self._lock:
            ent = self._fds.get(path)
            if ent is not None and ent.stamp != stamp:  # the file was replaced: a new descriptor, the old one goes when idle
                del self._fds[path]
                self._retire(ent)
                ent = None
            if ent is None:
                ent = self._fds[path] = _FdCache._Entry(os.open(path, os.O_RDONLY), stamp)
                if len(self._fds) > self._capacity:
                    for key in list(self._fds):
                        if len(self._fds) <= self._capacity:
                            break
                        old = self._fds[key]
                        if old is not ent and old.users == 0:  # entries in use stay; the cache may exceed its capacity for a while
                            del self._fds[key]
                            self._retire(old)
            else:
                self._fds.move_to_end(path)
            ent.users += 1
            return ent

    def release(self, ent) -> None:
        with self._lock:
            ent.users -= 1
            if ent.dead and ent.users == 0:
                os.close(ent.fd)

    def clear(self) -> None:
        with self._lock:
            for ent in self._fds.values():
                self._retire(ent)
            self._fds.clear()

    def __len__(self) -> int:
        with self._lock:
            return len(self._fds)


_FDS = _FdCache()
_HEADERS: "OrderedDict[str, Tuple[Tuple[int, int], object]]" = OrderedDict()  # path -> ((size, mtime_ns), WavPcm16 | exception)
_HEADERS_LOCK = threading.Lock()


def _stamp(path: str) -> Tuple[int, int]:
    st = os.stat(path)
    return (st.st_size, st.st_mtime_ns)


@dataclass(frozen=True)
class WavPcm16:
    path: str
    sampling_rate: int
    channels: int
    num_samples: int  # per channel
    data_offset: int  # byte offset of the first sample in the file
    stamp: Tuple[int, int] = (0, 0)  # (file size, mtime in ns) when the header was parsed

    @staticmethod
    def open_cached(path: str) -> "WavPcm16":
        """`open` with the parsed header remembered per path for as long as the file's size and mtime stay the same (one
        `stat` per call instead of open + parse + close); a file that is not 16-bit PCM is remembered too."""
        path = str(path)
        stamp = _stamp(path)
        with _HEADERS_LOCK:
            ent = _HEADERS.get(path)
            if ent is not None and ent[0] == stamp:
                _HEADERS.move_to_end(path)
                if isinstance(ent[1], Exception):
                    raise ent[1]
                return ent[1]
        try:
            h = WavPcm16.open(path)
        except NotPcm16Wav as e:
            h = e
        with _HEADERS_LOCK:
            _HEADERS[path] = (stamp, h)
            while len(_HEADERS) > 65536:
                _HEADERS.popitem(last=False)
        if isinstance(h, Exception):
            raise h
        return h

    @staticmethod
    def open(path: str) -> "WavPcm16":
        with open(path, "rb") as f:
            head = f.read(12)
            if len(head) < 12 or head[:4] != b"RIFF" or head[8:12] != b"WAVE":
                raise NotPcm16Wav(f"{path}: not a RIFF/WAVE file")
            fmt = None
            while True:
                hdr = f.read(8)
                if len(hdr) < 8:
                    raise NotPcm16Wav(f"{path}: no data chunk")
                cid, size = hdr[:4], struct.unpack("<I", hdr[4:])[0]
                if cid == b"fmt ":
                    body = f.read(size)
                    if len(body) < 16:
                        raise NotPcm16Wav(f"{path}: truncated fmt chunk")
                    tag, ch, sr, _, _, bits = struct.unpack("<HHIIHH", body[:16])
                    if tag == _WAVE_FORMAT_EXTENSIBLE and len(body) >= 40:
                        if body[24:40] != _KSDATAFORMAT_SUBTYPE_PCM:
                            raise NotPcm16Wav(f"{path}: extensible format is not integer PCM")
                        tag = _WAVE_FORMAT_PCM
                    fmt = (tag, ch, sr, bits)
                    if size & 1:
                        f.seek(1, os.SEEK_CUR)
                elif cid == b"data":
                    if fmt is None:
                        raise NotPcm16Wav(f"{path}: data chunk before fmt chunk")
                    tag, ch, sr, bits = fmt
                    if tag != _WAVE_FORMAT_PCM or bits != 16 or ch < 1:
                        raise NotPcm16Wav(f"{path}: format tag {tag}, {bits} bit — not 16-bit integer PCM")
                    off = f.tell()
                    avail = os.fstat(f.fileno()).st_size - off
                    if size == 0xFFFFFFFF or size > avail:  # streamed / truncated files: trust the file size
                        size = avail
                    st = os.fstat(f.fileno())
                    return WavPcm16(path=str(path), sampling_rate=sr, channels=ch, num_samples=size // (2 * ch), data_offset=off,
                                    stamp=(st.st_size, st.st_mtime_ns))
                else:
                    f.seek(size + (size & 1), os.SEEK_CUR)

    def read_into(self, dst: np.ndarray, first_sample: int = 0, channel: int = 0) -> int:
        """Fills the 1-D int16 array `dst` with samples [first_sample, first_sample + len(dst)) of `channel`.
        Mono files are read straight into `dst` (no intermediate copy).  Returns the number of samples read."""
        n = int(dst.shape[0])
        if first_sample < 0 or first_sample + n > self.num_samples:
            raise ValueError(f"{self.path}: samples [{first_sample}, {first_sample + n}) outside 0..{self.num_samples}")
        if not (0 <= channel < self.channels):
            raise ValueError(f"{self.path}: channel {channel} of {self.channels}")
        assert dst.dtype == np.int16 and dst.ndim == 1 and dst.flags.c_contiguous
        pos = self.data_offset + 2 * self.channels * first_sample
        if self.channels == 1:
            view = memoryview(dst).cast("B")
        else:
            raw = np.empty(self.channels * n, dtype="<i2")
            view = memoryview(raw).cast("B")
        ent = _FDS.acquire(self.path, self.stamp)  # shared descriptor, held for the duration of the read; preadv carries its own offset
        try:
            got = 0
            while got < len(view):
                k = os.preadv(ent.fd, [view[got:]], pos + got)
                if not k:
                    raise IOError(f"{self.path}: short read")
                got += k
        finally:
            _FDS.release(ent)
        if self.channels != 1:
            dst[:] = raw.reshape(n, self.channels)[:, channel]
        return n


@dataclass(frozen=True)
class PcmRequest:
    path: str
    first_sample: int
    num_samples: int
    channel: int = 0


class PcmStagingRing:
    """Grow-only pinned int16 buffer holding one ragged batch, every cut starting on a 4-sample boundary (the kernels'
    vector-load path; `b200feat_extract_host_at` / `b200feat_plan_batch` take the offsets).
    `stage` returns (buffer view, lengths, offsets, sampling rate)."""

    def __init__(self, initial_samples: int = 1 << 22, pin_memory: Optional[bool] = None):
        self._pin = torch.cuda.is_available() if pin_memory is None else pin_memory
        self._buf = torch.empty(int(initial_samples), dtype=torch.int16, pin_memory=self._pin)
        self._headers = {}
        self._in_flight = None  # CUDA event recorded after the last asynchronous H2D copy out of the ring

    def mark_in_flight(self, device=None) -> None:
        """Call right after an asynchronous (`non_blocking=True`) copy out of the ring: the next `stage()` waits for it before
        it overwrites the buffer (the dependency used to hold only because a later pageable copy happened to synchronise)."""
        if self._pin and torch.cuda.is_available():
            ev = torch.cuda.Event()
            ev.record(torch.cuda.current_stream(device))
            self._in_flight = ev

    def _header(self, path: str) -> WavPcm16:
        h = self._headers.get(path)
        if h is None:
            h = self._headers[path] = WavPcm16.open_cached(path)
            if len(self._headers) > 65536:
                self._headers.clear()
        return h

    ALIGN = 4

    def stage(self, requests: Sequence[PcmRequest], executor=None) -> Tuple[torch.Tensor, List[int], List[int], int]:
        if self._in_flight is not None:
            self._in_flight.synchronize()
            self._in_flight = None
        lens = [int(r.num_samples) for r in requests]
        offs, total = _aligned_offsets(lens, self.ALIGN)
        if total > self._buf.numel():
            self._buf = torch.empty(max(total, 2 * self._buf.numel()), dtype=torch.int16, pin_memory=self._pin)
        view = self._buf.numpy()
        _zero_gaps(view, lens, offs)
        srs = set()

        def one(i):
            r = requests[i]
            h = self._header(r.path)
            srs.add(h.sampling_rate)
            h.read_into(view[offs[i]: offs[i] + lens[i]], r.first_sample, r.channel)

        workers = getattr(executor, "_max_workers", 1) if executor is not None else 1
        if executor is None or workers <= 1 or len(requests) < 2 * workers:
            for i in range(len(requests)):
                one(i)
        else:  # one task per worker over a contiguous share of the batch (a task per cut costs more than the read it wraps)
            step = (len(requests) + workers - 1) // workers

            def share(a):
                for i in range(a, min(a + step, len(requests))):
                    one(i)

            list(executor.map(share, range(0, len(requests), step)))
        if len(srs) != 1:
            raise ValueError(f"one sampling rate per batch expected, got {sorted(srs)}")
        return self._buf[:total], lens, offs, srs.pop()


def pcm16_request_for_cut(cut) -> Optional[PcmRequest]:
    """The raw-PCM read that `cut.load_audio()` amounts to (cut/data.py + audio/recording.py:load_audio with
    offset = cut.start, duration = cut.duration), when it is nothing but a slice of one 16-bit PCM WAV file:
    a MonoCut over a single-source "file" recording with no augmentation transforms.  None when not eligible."""
    rec = getattr(cut, "recording", None)
    if rec is None or getattr(cut, "tracks", None) is not None or getattr(rec, "transforms", None):
        return None
    sources = getattr(rec, "sources", None) or []
    if len(sources) != 1 or sources[0].type != "file" or not str(sources[0].source).lower().endswith(".wav"):
        return None
    ch = cut.channel
    if not isinstance(ch, int) or ch not in sources[0].channels:
        return None
    try:
        h = WavPcm16.open_cached(str(sources[0].source))
    except (NotPcm16Wav, OSError):
        return None
    if h.sampling_rate != cut.sampling_rate or h.channels != len(sources[0].channels):
        return None
    # seconds -> samples as lhotse does (utils.py compute_num_samples: round half up after an 8-digit rounding)
    first = int(math.floor(round(cut.start * h.sampling_rate, 8) + 0.5))
    n = int(cut.num_samples)
    if first + n > h.num_samples:
        return None
    return PcmRequest(path=h.path, first_sample=first, num_samples=n, channel=sources[0].channels.index(ch))
