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
  * `slice_request_for_cut(cut)` the (path, first sample, sample count, channel) of a lhotse MonoCut when it is a plain
                                 slice (one "file" source, no augmentation transforms) of a 16-bit .wav (`PcmRequest`) or
                                 .flac (`FlacRequest`) file; None otherwise.  `pcm16_request_for_cut` / `flac_request_for_cut`
                                 take one of the two kinds
  * `FlacStream`, `FlacStagingRing`, `decode_flac`: 16-bit FLAC files, whose frames cross PCIe compressed and are decoded by
                                 the sm_90a kernel of csrc/flac.cuh
  * `mix_request_for_cut`, `MixStagingRing`, `mix_cuts`: MixedCuts of such slices, mixed by csrc/mix.cuh
  * `transform_request_for_cut`, `TransformStagingRing`, `transform_cuts`: speed / volume perturbed and resampled slices, the
                                 transforms run by csrc/resample.cuh
The mix and transform rings stage their int16 sources (WAV and FLAC slices, RIRs) through one `_SourceRing`.
`staged_route(cuts)` picks the route of a batch (one of `STAGED_ROUTES`) with its requests, `new_ring(route)` makes the ring
that stages them, and `staged_to_device` runs the device half of any staged batch; `collate_staged` turns it into lhotse's
padded (B, T) waveform batch (csrc/collate.cuh).
Everything here is host-side I/O; the arithmetic stays in the CUDA kernels.
"""
from __future__ import annotations

import math
import os
import struct
import threading
from collections import OrderedDict
from dataclasses import dataclass, field
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
_HEADERS: "OrderedDict[Tuple[str, str], Tuple[Tuple[int, int], object]]" = OrderedDict()  # (kind, path) -> ((size, mtime_ns), header | exception)
_HEADERS_LOCK = threading.Lock()


def _stamp(path: str) -> Tuple[int, int]:
    st = os.stat(path)
    return (st.st_size, st.st_mtime_ns)


def _open_cached(kind, path: str, refusal):
    """`kind.open(path)`, remembered in `_HEADERS` under (kind, path) while the file's size and mtime stay the same; a
    `refusal` (the file is not of this kind) is remembered and raised again."""
    path = str(path)
    stamp = _stamp(path)
    key = (kind.__name__, path)
    with _HEADERS_LOCK:
        ent = _HEADERS.get(key)
        if ent is not None and ent[0] == stamp:
            _HEADERS.move_to_end(key)
            if isinstance(ent[1], Exception):
                raise ent[1]
            return ent[1]
    try:
        h = kind.open(path)
    except refusal as e:
        h = e
    with _HEADERS_LOCK:
        _HEADERS[key] = (stamp, h)
        while len(_HEADERS) > 65536:
            _HEADERS.popitem(last=False)
    if isinstance(h, Exception):
        raise h
    return h


def _pread(path: str, stamp: Tuple[int, int], view: memoryview, pos: int) -> None:
    """Fills `view` with the file's bytes from `pos` on through the shared descriptor cache."""
    ent = _FDS.acquire(path, stamp)  # shared descriptor, held for the duration of the read; preadv carries its own offset
    try:
        got = 0
        while got < len(view):
            k = os.preadv(ent.fd, [view[got:]], pos + got)
            if not k:
                raise IOError(f"{path}: short read")
            got += k
    finally:
        _FDS.release(ent)


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
        return _open_cached(WavPcm16, path, NotPcm16Wav)

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
        _pread(self.path, self.stamp, view, pos)
        if self.channels != 1:
            dst[:] = raw.reshape(n, self.channels)[:, channel]
        return n


def _for_each(n: int, one, executor) -> None:
    """one(i) for i in [0, n), on `executor`'s threads when there is enough work: one task per worker over a contiguous share
    of the batch (a task per cut costs more than the read it wraps)."""
    workers = getattr(executor, "_max_workers", 1) if executor is not None else 1
    if executor is None or workers <= 1 or n < 2 * workers:
        for i in range(n):
            one(i)
        return
    step = (n + workers - 1) // workers

    def share(a):
        for i in range(a, min(a + step, n)):
            one(i)

    list(executor.map(share, range(0, n, step)))


@dataclass(frozen=True)
class _SliceRequest:
    path: str
    first_sample: int
    num_samples: int
    channel: int = 0


@dataclass(frozen=True)
class PcmRequest(_SliceRequest):
    """Samples [first_sample, first_sample + num_samples) of `channel` of a 16-bit PCM WAV file."""


def _samples(seconds: float, sr: int) -> int:
    return int(math.floor(round(seconds * sr, 8) + 0.5))  # lhotse's compute_num_samples


def _one_rate(srs) -> int:
    if len(srs) != 1:
        raise ValueError(f"one sampling rate per batch expected, got {sorted(srs)}")
    return next(iter(srs))


class _PinnedRing:
    """Grow-only pinned host buffers whose contents leave for the device with asynchronous copies: `mark_in_flight` after
    such a copy, and the next `_wait_idle` (before the buffers are refilled) waits for it."""

    def __init__(self, pin_memory: Optional[bool] = None):
        self._pin = torch.cuda.is_available() if pin_memory is None else pin_memory
        self._in_flight = None  # CUDA event recorded after the last asynchronous H2D copy out of the ring

    def mark_in_flight(self, device=None) -> None:
        """Call right after an asynchronous (`non_blocking=True`) copy out of the ring: the next `stage()` waits for it before
        it overwrites the buffer (the dependency used to hold only because a later pageable copy happened to synchronise)."""
        if self._pin and torch.cuda.is_available():
            ev = torch.cuda.Event()
            ev.record(torch.cuda.current_stream(device))
            self._in_flight = ev

    def _wait_idle(self) -> None:
        if self._in_flight is not None:
            self._in_flight.synchronize()
            self._in_flight = None

    def _grown(self, buf: torch.Tensor, n: int) -> torch.Tensor:
        return buf if n <= buf.numel() else torch.empty(max(n, 2 * buf.numel()), dtype=buf.dtype, pin_memory=self._pin)


class PcmStagingRing(_PinnedRing):
    """Grow-only pinned int16 buffer holding one ragged batch, every cut starting on a 4-sample boundary (the kernels'
    vector-load path; `b200feat_extract_host_at` / `b200feat_plan_batch` take the offsets).
    `stage` returns (buffer view, lengths, offsets, sampling rate)."""

    def __init__(self, initial_samples: int = 1 << 22, pin_memory: Optional[bool] = None):
        super().__init__(pin_memory)
        self._buf = torch.empty(int(initial_samples), dtype=torch.int16, pin_memory=self._pin)
        self._headers = {}

    def _header(self, path: str) -> WavPcm16:
        h = self._headers.get(path)
        if h is None:
            h = self._headers[path] = WavPcm16.open_cached(path)
            if len(self._headers) > 65536:
                self._headers.clear()
        return h

    ALIGN = 4

    def stage(self, requests: Sequence[PcmRequest], executor=None) -> Tuple[torch.Tensor, List[int], List[int], int]:
        buf, lens, offs, srs = self._fill(requests, executor)
        return buf, lens, offs, _one_rate(srs)

    def _fill(self, requests: Sequence[PcmRequest], executor=None) -> Tuple[torch.Tensor, List[int], List[int], set]:
        """`stage` without the one-rate check: (buffer view, lengths, offsets, the files' sampling rates)."""
        self._wait_idle()
        lens = [int(r.num_samples) for r in requests]
        offs, total = _aligned_offsets(lens, self.ALIGN)
        self._buf = self._grown(self._buf, total)
        view = self._buf.numpy()
        _zero_gaps(view, lens, offs)
        srs = set()

        def one(i):
            r = requests[i]
            h = self._header(r.path)
            srs.add(h.sampling_rate)
            h.read_into(view[offs[i]: offs[i] + lens[i]], r.first_sample, r.channel)

        _for_each(len(requests), one, executor)
        return self._buf[:total], lens, offs, srs


# ---- FLAC ----------------------------------------------------------------------------------------------------------
# The compressed frames go file -> pinned byte ring -> one H2D copy -> the sm_90a decode kernel (csrc/flac.cuh), which writes
# the int16 samples straight into the ragged device buffer the feature kernels take as B200FEAT_I16.  A FLAC batch crosses
# PCIe at about half the bytes of the same audio as PCM16.


class NotFlac16(ValueError):
    """The file is not a native FLAC stream of 16-bit samples that the frame index can walk."""


@dataclass(frozen=True, eq=False)
class FlacStream:
    path: str
    sampling_rate: int
    channels: int
    num_samples: int          # per channel (STREAMINFO total samples)
    variable_blocking: bool
    md5: bytes
    frames: np.ndarray        # engine.FLAC_FRAME_DTYPE: byte offset, first sample, block size, byte length
    stamp: Tuple[int, int] = (0, 0)

    @staticmethod
    def open_cached(path: str) -> "FlacStream":
        """`open`, remembered in the same per-path cache as the WAV headers (keyed on the file's size and mtime)."""
        return _open_cached(FlacStream, path, NotFlac16)

    @staticmethod
    def open(path: str) -> "FlacStream":
        from .engine import flac_index

        with open(path, "rb") as f:
            data = f.read()
            st = os.fstat(f.fileno())
        try:
            info, frames = flac_index(data)
        except ValueError as e:
            raise NotFlac16(f"{path}: {e}") from None
        if info.bits_per_sample != 16:
            raise NotFlac16(f"{path}: {info.bits_per_sample}-bit samples")
        total = int(frames["block_size"].sum())
        if not len(frames) or info.total_samples != total:
            raise NotFlac16(f"{path}: the frames hold {total} samples, STREAMINFO says {info.total_samples}")
        return FlacStream(path=str(path), sampling_rate=int(info.sample_rate), channels=int(info.channels), num_samples=total,
                          variable_blocking=bool(info.variable_blocking), md5=bytes(info.md5), frames=frames,
                          stamp=(st.st_size, st.st_mtime_ns))


@dataclass(frozen=True)
class FlacRequest(_SliceRequest):
    """Samples [first_sample, first_sample + num_samples) of `channel` of a 16-bit FLAC file."""


@dataclass
class FlacBatch:
    """One staged FLAC batch: the compressed frames in the ring's pinned bytes, the job table (engine.FLAC_JOB_DTYPE, one job
    per frame of each cut) and where every cut's samples go in the int16 output."""
    data: torch.Tensor        # pinned uint8 view, the frames of every cut back to back
    jobs: torch.Tensor        # pinned uint8 view of the job records
    njobs: int
    job_cut: np.ndarray       # cut index of every job
    lens: List[int]
    offsets: List[int]
    out_elems: int
    scratch_elems: int
    requests: Sequence[FlacRequest]


class FlacStagingRing(_PinnedRing):
    """Grow-only pinned byte buffers for one FLAC batch; `stage(requests)` reads each cut's frame range into it and builds the
    job table with vector operations over the cached frame tables.  Returns (FlacBatch, lengths, offsets, sampling rate), the
    rate None when the files have several."""

    ALIGN = 4

    def __init__(self, initial_bytes: int = 1 << 22, pin_memory: Optional[bool] = None):
        super().__init__(pin_memory)
        self._data = torch.empty(int(initial_bytes), dtype=torch.uint8, pin_memory=self._pin)
        self._jobs = torch.empty(1 << 16, dtype=torch.uint8, pin_memory=self._pin)

    def stage(self, requests: Sequence[FlacRequest], executor=None) -> Tuple[FlacBatch, List[int], List[int], int]:
        from .engine import FLAC_JOB_DTYPE

        self._wait_idle()
        B = len(requests)
        streams = [FlacStream.open_cached(r.path) for r in requests]
        srs = {s.sampling_rate for s in streams}
        lens = [int(r.num_samples) for r in requests]
        offs, out_elems = _aligned_offsets(lens, self.ALIGN)
        first = np.asarray([r.first_sample for r in requests], dtype=np.int64)
        # per cut: the frames [f0, f1) that hold samples [first, first + n)
        f0 = np.empty(B, dtype=np.int64)
        f1 = np.empty(B, dtype=np.int64)
        parts = []
        for i, (r, s) in enumerate(zip(requests, streams)):
            if r.first_sample < 0 or r.first_sample + r.num_samples > s.num_samples or not (0 <= r.channel < s.channels):
                raise ValueError(f"{r.path}: samples [{r.first_sample}, {r.first_sample + r.num_samples}) of channel {r.channel} "
                                 f"outside 0..{s.num_samples} x {s.channels}")
            fs = s.frames["first_sample"]
            f0[i] = np.searchsorted(fs, r.first_sample, "right") - 1
            f1[i] = max(int(f0[i]), int(np.searchsorted(fs, r.first_sample + r.num_samples, "left"))) if r.num_samples else f0[i]
            parts.append(s.frames[f0[i]: f1[i]])
        frames = np.concatenate(parts) if parts else np.empty(0, dtype=streams[0].frames.dtype)
        nfr = f1 - f0
        J = int(nfr.sum())
        cut = np.repeat(np.arange(B), nfr)
        start = np.concatenate(([0], np.cumsum(nfr)[:-1])).astype(np.int64)
        index = f0[cut] + (np.arange(J) - start[cut])  # frame number within its stream
        # the bytes of each cut's frames, back to back
        lo = np.asarray([p["byte_offset"][0] if len(p) else 0 for p in parts], dtype=np.int64)
        hi = np.asarray([p["byte_offset"][-1] + p["byte_length"][-1] if len(p) else 0 for p in parts], dtype=np.int64)
        base = np.concatenate(([0], np.cumsum(hi - lo)[:-1])).astype(np.int64)
        nbytes = int((hi - lo).sum())
        self._data = self._grown(self._data, max(nbytes, 1))
        data = self._data.numpy()

        def one(i):
            if hi[i] > lo[i]:
                s = streams[i]
                _pread(s.path, s.stamp, memoryview(data[base[i]: base[i] + hi[i] - lo[i]]), int(lo[i]))

        _for_each(B, one, executor)
        self._jobs = self._grown(self._jobs, max(J, 1) * FLAC_JOB_DTYPE.itemsize)
        jobs = self._jobs.numpy()[: J * FLAC_JOB_DTYPE.itemsize].view(FLAC_JOB_DTYPE)
        fsample = frames["first_sample"]
        block = frames["block_size"].astype(np.int64)
        a, n = first[cut], np.asarray(lens, dtype=np.int64)[cut]
        skip = np.maximum(0, a - fsample)
        count = np.minimum(block, a + n - fsample) - skip
        chans = np.asarray([s.channels for s in streams], dtype=np.int32)[cut]
        variable = np.asarray([s.variable_blocking for s in streams], dtype=np.int32)[cut]
        multi = chans > 1
        scr = np.cumsum(np.where(multi, count, 0))
        jobs["src_byte"] = base[cut] + frames["byte_offset"] - lo[cut]
        jobs["dst_elem"] = np.asarray(offs, dtype=np.int64)[cut] + fsample + skip - a
        jobs["scratch_elem"] = np.where(multi, scr - count, -1)
        jobs["coded_number"] = np.where(variable == 1, fsample, index)
        jobs["byte_length"] = frames["byte_length"]
        jobs["block_size"] = block
        jobs["channels"] = chans
        jobs["want_channel"] = np.asarray([r.channel for r in requests], dtype=np.int32)[cut]
        jobs["skip"] = skip
        jobs["count"] = count
        jobs["variable_blocking"] = variable
        jobs["reserved"] = 0
        batch = FlacBatch(data=self._data[:nbytes], jobs=self._jobs[: J * FLAC_JOB_DTYPE.itemsize], njobs=J, job_cut=cut,
                          lens=lens, offsets=offs, out_elems=out_elems, scratch_elems=int(scr[-1]) if J else 0,
                          requests=list(requests))
        return batch, lens, offs, (srs.pop() if len(srs) == 1 else None)  # None: several rates (decodable, not one extraction)


def decode_staged(batch: FlacBatch, device, ring: Optional[_PinnedRing] = None) -> Tuple[torch.Tensor, List[int], List[int]]:
    """The device half of the FLAC route on the current stream: H2D of the frames and the job table (then `ring`'s copy is
    marked in flight), the decode kernel, and one small D2H of the status words.  Returns (int16 samples on `device`, lengths,
    offsets); a frame that does not decode raises ValueError naming the file and the cut's sample range."""
    from .engine import FLAC_STATUS, flac_decode

    device = torch.device(device)
    out = torch.zeros(max(batch.out_elems, 1), dtype=torch.int16, device=device)
    if batch.njobs:
        data = batch.data.to(device, non_blocking=True)
        jobs = batch.jobs.to(device, non_blocking=True)
        if ring is not None:
            ring.mark_in_flight(device)
        status = torch.empty(batch.njobs, dtype=torch.int32, device=device)
        scratch = torch.empty(batch.scratch_elems, dtype=torch.int32, device=device) if batch.scratch_elems else None
        flac_decode(data, jobs, batch.njobs, out, status, scratch)
        bad = torch.nonzero(status).flatten().cpu().numpy()
        if bad.size:
            j = int(bad[0])
            st = int(status[j].item())
            r = batch.requests[int(batch.job_cut[j])]
            raise ValueError(f"{r.path}: samples [{r.first_sample}, {r.first_sample + r.num_samples}) of channel {r.channel}: "
                             f"FLAC decode failed ({FLAC_STATUS.get(st, st)}; {bad.size} bad frame(s) in the batch)")
    return out, batch.lens, batch.offsets


def decode_flac(requests: Sequence[FlacRequest], device="cuda", executor=None,
                ring: Optional[FlacStagingRing] = None) -> Tuple[torch.Tensor, List[int], List[int]]:
    """Decodes the sample ranges of 16-bit FLAC files on the GPU: (int16 device tensor holding every cut at its offset, on
    4-sample boundaries, lengths, offsets) — the ragged layout `Engine.extract_device` takes."""
    ring = ring or FlacStagingRing()
    batch, _, _, _ = ring.stage(requests, executor=executor)
    return decode_staged(batch, device, ring)


def _open_slice_file(path) -> Optional[Tuple[object, type]]:
    """The cached header of a 16-bit file chosen by its extension, with the request class that reads it: (WavPcm16,
    PcmRequest) for .wav, (FlacStream, FlacRequest) for .flac; None for another extension or a file the reader refuses."""
    path = str(path)
    try:
        if path.lower().endswith(".wav"):
            return WavPcm16.open_cached(path), PcmRequest
        if path.lower().endswith(".flac"):
            return FlacStream.open_cached(path), FlacRequest
    except (NotPcm16Wav, NotFlac16, OSError):
        pass
    return None


def slice_request_for_cut(cut) -> Optional[_SliceRequest]:
    """The raw read that `cut.load_audio()` amounts to (cut/data.py + audio/recording.py:load_audio with offset = cut.start,
    duration = cut.duration), when it is nothing but a slice of one 16-bit PCM WAV file (a PcmRequest) or one 16-bit FLAC
    file (a FlacRequest): a MonoCut over a single-source "file" recording with no augmentation transforms.  None when not
    eligible."""
    rec = getattr(cut, "recording", None)
    if rec is None or getattr(cut, "tracks", None) is not None or getattr(rec, "transforms", None):
        return None
    sources = getattr(rec, "sources", None) or []
    if len(sources) != 1 or sources[0].type != "file":
        return None
    ch = cut.channel
    if not isinstance(ch, int) or ch not in sources[0].channels:
        return None
    opened = _open_slice_file(sources[0].source)
    if opened is None:
        return None
    h, make = opened
    if h.sampling_rate != cut.sampling_rate or h.channels != len(sources[0].channels):
        return None
    first = _samples(cut.start, h.sampling_rate)
    n = int(cut.num_samples)
    if first + n > h.num_samples:
        return None
    return make(path=h.path, first_sample=first, num_samples=n, channel=sources[0].channels.index(ch))


def pcm16_request_for_cut(cut) -> Optional[PcmRequest]:
    """`slice_request_for_cut` for a slice of one 16-bit PCM WAV file; None otherwise."""
    r = slice_request_for_cut(cut)
    return r if isinstance(r, PcmRequest) else None


def flac_request_for_cut(cut) -> Optional[FlacRequest]:
    """`slice_request_for_cut` for a slice of one 16-bit FLAC file; None otherwise."""
    r = slice_request_for_cut(cut)
    return r if isinstance(r, FlacRequest) else None


class _SourceRing(_PinnedRing):
    """The int16 sources of a mix or transform batch: the WAV reads through a PcmStagingRing (files of any rate), the FLAC
    reads through a FlacStagingRing.  `stage(reads)` returns (pinned int16 view or None, FlacBatch or None, the source of
    each read: 0 WAV / 1 FLAC, the element offset of each read in its source, (the set of the WAV files' rates, the set of
    the FLAC batch's rate: None when the FLAC files have several))."""

    def __init__(self, pin_memory: Optional[bool] = None):
        super().__init__(pin_memory)
        self.pcm = PcmStagingRing(initial_samples=1 << 20, pin_memory=self._pin)
        self.flac = FlacStagingRing(initial_bytes=1 << 16, pin_memory=self._pin)

    def mark_in_flight(self, device=None) -> None:
        super().mark_in_flight(device)
        self.pcm.mark_in_flight(device)
        self.flac.mark_in_flight(device)

    def stage(self, reads: Sequence[_SliceRequest], executor=None):
        kind = np.asarray([0 if isinstance(r, PcmRequest) else 1 for r in reads], dtype=np.int32)
        elem = np.zeros(len(reads), dtype=np.int64)
        wav = [r for r, k in zip(reads, kind) if k == 0]
        flac = [r for r, k in zip(reads, kind) if k == 1]
        pcm_buf, flac_batch, wav_srs, flac_srs = None, None, set(), set()
        if wav:
            pcm_buf, _, offs, wav_srs = self.pcm._fill(wav, executor)
            elem[kind == 0] = offs
        if flac:
            flac_batch, _, offs, sr = self.flac.stage(flac, executor=executor)
            elem[kind == 1] = offs
            flac_srs = {sr}
        return pcm_buf, flac_batch, kind, elem, (wav_srs, flac_srs)


def _sources_to_device(batch, device) -> Tuple[Optional[torch.Tensor], Optional[torch.Tensor]]:
    """The device half of `_SourceRing.stage` for a batch with its `pcm` / `flac` fields: (the WAV reads' int16 H2D copy,
    the FLAC reads' decode), each None when the batch has no such read."""
    src0 = batch.pcm.to(device, non_blocking=True) if batch.pcm is not None else None
    src1 = decode_staged(batch.flac, device)[0] if batch.flac is not None else None
    return src0, src1


# ---- MixedCut ------------------------------------------------------------------------------------------------------
# A MixedCut's tracks are staged as int16 by the two rings above (WAV tracks through PcmStagingRing, FLAC tracks through
# FlacStagingRing), and the sm_90a kernels of csrc/mix.cuh compute the energies, the gains and the mix on the device, bit for
# bit what MixedCut.load_audio() returns under NumPy >= 2 (DESIGN.md §3.1h).  The mixes land as float32 in the ragged layout
# `Engine.extract_device` takes.


@dataclass(frozen=True)
class MixTrackRequest:
    source: Optional[object]  # PcmRequest | FlacRequest | TransformRequest (a perturbed track); None = a PaddingCut (zeros)
    num_samples: int
    offset: int               # first sample in the mix
    snr_factor: float         # 10 ** (-snr / 10) as Python evaluates it; NaN = no SNR
    role: int = 0             # engine.MIX_ROLE_MIXED | engine.MIX_ROLE_ENERGY (a muted SNR reference)


@dataclass(frozen=True)
class MixRequest:
    tracks: Tuple[MixTrackRequest, ...]  # the audible tracks in track order, then a muted SNR reference if there is one
    ref: int                             # index of the SNR reference in `tracks`
    mode: int                            # engine.MIX_F32 | engine.MIX_SCALED_FIRST
    mix_len: int                         # max(offset + length) over the mixed tracks
    num_samples: int                     # the cut's length: the mix is trimmed or reflect-padded to it
    reverb: Optional["ReverbRequest"] = None  # a cut-level ReverbWithImpulseResponse, run on the length-fixed mix


def _numpy2() -> bool:
    return int(np.__version__.split(".")[0]) >= 2


def mix_request_for_cut(cut, perturbed_tracks: bool = False, reverb: bool = False,
                        generated_rir: bool = False) -> Optional[MixRequest]:
    """What `MixedCut.load_audio()` (lhotse/cut/mixed.py) amounts to for a MixedCut of mono 16-bit WAV / FLAC slices and
    PaddingCuts: tracks, offsets, SNR factors, reference and length.  None when the cut is not eligible: not a MixedCut,
    cut-level transforms, a track that `pcm16_request_for_cut` / `flac_request_for_cut` refuse (MultiCut, nested MixedCut,
    recording transforms, other formats), a sampling rate other than the cut's, an empty track, a length outside lhotse's
    duration-mismatch tolerance, or NumPy 1.x (whose promotion of np.float64 * float32 arrays differs).

    `perturbed_tracks=True` also takes a MonoCut track whose recording carries a chain `transform_request_for_cut` accepts
    (Speed / Volume / Resample): its source is that TransformRequest and its length the request's, the resample kernel loads
    it into a float32 track buffer and the mix kernels read it there (DESIGN.md §3.1h).  The default is False so that
    existing callers keep exactly the routes they have; turning it on by default is a decision for when H100 measurements
    of the route exist.

    `reverb=True` also takes a MixedCut whose `transforms` are exactly one ReverbWithImpulseResponse that `reverb_request`
    accepts (what `MixedCut.reverb_rir(mix_first=True)` makes) over a float32 mix: the mix goes to a float32 buffer and the
    reverb kernel writes the cut, within a float32 tolerance of a float64 convolution (DESIGN.md §3.1j).  Tracks that carry a
    reverb of their own (mix_first=False) stay refused.  Off by default.  `generated_rir=True` takes such a reverb with an RIR
    that lhotse generates (see `reverb_request`), also off by default."""
    if not _numpy2():
        return None
    try:
        from lhotse.audio.utils import get_audio_duration_mismatch_tolerance
        from lhotse.augmentation.rir import ReverbWithImpulseResponse
        from lhotse.augmentation.transform import AudioTransform
        from lhotse.cut import MixedCut, MonoCut, PaddingCut
        from lhotse.utils import compute_num_samples
    except ImportError:
        return None
    from .engine import MIX_F32, MIX_ROLE_ENERGY, MIX_ROLE_MIXED, MIX_SCALED_FIRST

    if not isinstance(cut, MixedCut) or not cut.tracks:
        return None
    rv = None
    if getattr(cut, "transforms", None):
        tfs = [t if isinstance(t, AudioTransform) else AudioTransform.from_dict(t) for t in cut.transforms]
        if not (reverb or generated_rir) or len(tfs) != 1 or type(tfs[0]) is not ReverbWithImpulseResponse:
            return None
        rv = reverb_request(tfs[0], cut.sampling_rate, reverb, generated_rir)
        if rv is None:
            return None
    sr = cut.sampling_rate
    tracks = list(cut.tracks)
    if all(isinstance(t.cut, PaddingCut) for t in tracks):
        return None  # no recording: load_audio() returns None
    # _get_snr_reference_track / _get_audible_tracks
    ref = next((t for t in tracks if getattr(t, "is_snr_reference", False)), None)
    if ref is None:
        ref = next((t for t in tracks if not isinstance(t.cut, PaddingCut) and t.snr is None), None)
    if ref is None:
        return None  # lhotse raises its own error on the float route
    audible = [t for t in tracks if not t.mute] or tracks
    chosen = audible + ([ref] if all(t is not ref for t in audible) else [])

    def one(t, role):
        c = t.cut
        if c.sampling_rate != sr:
            return None
        if isinstance(c, PaddingCut):
            src, n = None, compute_num_samples(c.duration, sr)
        elif isinstance(c, MonoCut) and not isinstance(c, MixedCut):
            if perturbed_tracks and _has_transforms(c):
                src = transform_request_for_cut(c)  # num_samples: the chain's output after lhotse's length fix
            else:
                src = slice_request_for_cut(c)
            if src is None:
                return None
            n = src.num_samples
        else:
            return None
        if n <= 0:
            return None
        factor = float("nan") if t.snr is None else 10.0 ** (-t.snr / 10)
        return MixTrackRequest(source=src, num_samples=int(n), offset=int(compute_num_samples(t.offset, sr)),
                               snr_factor=factor, role=role)

    reqs = []
    for i, t in enumerate(chosen):
        r = one(t, MIX_ROLE_MIXED if i < len(audible) else MIX_ROLE_ENERGY)
        if r is None:
            return None
        reqs.append(r)
    mix_len = max(r.offset + r.num_samples for r in reqs[: len(audible)])
    target = int(cut.num_samples)
    tol = compute_num_samples(get_audio_duration_mismatch_tolerance(), sr)
    diff = mix_len - target
    if diff != 0 and not (-tol < diff < tol and -diff <= mix_len - 1):
        return None
    first = audible[0]
    mode = MIX_SCALED_FIRST if (ref is not first and first.snr is not None) else MIX_F32
    if rv is not None and mode != MIX_F32:
        return None  # a float64 mix would be reverberated in float64
    return MixRequest(tracks=tuple(reqs), ref=next(i for i, t in enumerate(chosen) if t is ref), mode=mode, mix_len=mix_len,
                      num_samples=target, reverb=rv)


def _plain_mix_request(cut, perturbed_tracks: bool = False, reverb: bool = False,
                       generated_rir: bool = False) -> Optional[MixRequest]:
    """A plain 16-bit WAV / FLAC slice as a mix of one track (the kernel writes x = q / 32768, what the float route reads);
    with `perturbed_tracks`, also a MonoCut with an eligible transform chain (the kernel copies the chain's float32 output);
    with `reverb`, also a plain slice whose only transform is an eligible reverb (a one-track mix, then the reverb), and with
    both, a chain that ends in such a reverb (the transform route reverberates it into the track buffer, the kernel copies
    that)."""
    from .engine import MIX_F32, MIX_ROLE_MIXED

    if getattr(cut, "tracks", None) is not None:
        return None
    if (reverb or generated_rir) and _has_transforms(cut):
        r = transform_request_for_cut(cut, reverb=reverb, generated_rir=generated_rir)
        if r is not None and r.reverb is not None and not r.ops and r.num_samples == r.source.num_samples > 0:
            n = int(r.num_samples)
            return MixRequest(tracks=(MixTrackRequest(r.source, n, 0, float("nan"), MIX_ROLE_MIXED),), ref=0, mode=MIX_F32,
                              mix_len=n, num_samples=n, reverb=r.reverb)
    if perturbed_tracks and _has_transforms(cut):
        src = transform_request_for_cut(cut, reverb=reverb, generated_rir=generated_rir)
    else:
        src = slice_request_for_cut(cut)
    if src is None or src.num_samples <= 0:
        return None
    return MixRequest(tracks=(MixTrackRequest(src, int(src.num_samples), 0, float("nan"), MIX_ROLE_MIXED),), ref=0,
                      mode=MIX_F32, mix_len=int(src.num_samples), num_samples=int(src.num_samples))


def _mix_or_plain_request(cut, perturbed_tracks: bool = False, reverb: bool = False,
                          generated_rir: bool = False) -> Optional[MixRequest]:
    if getattr(cut, "tracks", None) is not None:
        return mix_request_for_cut(cut, perturbed_tracks=perturbed_tracks, reverb=reverb, generated_rir=generated_rir)
    return _plain_mix_request(cut, perturbed_tracks=perturbed_tracks, reverb=reverb, generated_rir=generated_rir)


def mix_requests_for_batch(cuts, perturbed_tracks: bool = False, reverb: bool = False,
                           generated_rir: bool = False) -> Optional[List[MixRequest]]:
    """The "mix" route's requests for a batch: every cut a plain 16-bit WAV / FLAC slice or an eligible MixedCut, and at least
    one MixedCut (batches of plain slices keep the "pcm16" / "flac" / "float" routes).  None otherwise.  With
    `perturbed_tracks=True` (see `mix_request_for_cut`; off by default), MixedCut tracks and plain MonoCuts with an eligible
    Speed / Volume / Resample chain are taken too."""
    if not any(getattr(c, "tracks", None) is not None for c in cuts):
        return None
    reqs = []
    for c in cuts:
        r = _mix_or_plain_request(c, perturbed_tracks, reverb, generated_rir)
        if r is None:
            return None
        reqs.append(r)
    return reqs


@dataclass
class MixBatch:
    """One staged mix batch: the WAV tracks in the PCM ring's pinned int16 buffer, the FLAC tracks as a staged FlacBatch,
    and the b200feat_mix track / cut tables (pinned numpy views) that place every cut's float32 mix in the output; perturbed
    tracks (source 2) as a staged TransformBatch whose "cuts" are those tracks, run into the float32 track buffer first."""
    pcm: Optional[torch.Tensor]
    flac: Optional[FlacBatch]
    tracks: np.ndarray        # engine.MIX_TRACK_DTYPE
    cuts: np.ndarray          # engine.MIX_CUT_DTYPE
    lens: List[int]
    offsets: List[int]
    out_elems: int
    transform: Optional[TransformBatch] = None
    pre_elems: int = 0                        # the reverberated cuts' mixes, after the output in the same buffer
    reverb_rirs: Optional[np.ndarray] = None  # engine.REVERB_RIR_DTYPE
    reverb_cuts: Optional[np.ndarray] = None  # engine.REVERB_CUT_DTYPE, reading and writing that buffer
    generated: Optional["GeneratedRirs"] = None  # the generated RIRs of the batch and of its perturbed tracks


class MixStagingRing(_PinnedRing):
    """A _SourceRing for the int16 tracks, pinned table bytes for one mix batch, plus a TransformStagingRing for the
    perturbed tracks (made when a batch first has one); `stage(requests)` returns (MixBatch, lengths, offsets, sampling rate),
    the rate None when the tracks have several.  WAV tracks of several rates raise ValueError."""

    ALIGN = 4

    def __init__(self, pin_memory: Optional[bool] = None):
        super().__init__(pin_memory)
        self.sources = _SourceRing(pin_memory=self._pin)
        self.transform: Optional[TransformStagingRing] = None
        self._tables = torch.empty(1 << 16, dtype=torch.uint8, pin_memory=self._pin)

    def mark_in_flight(self, device=None) -> None:
        super().mark_in_flight(device)
        self.sources.mark_in_flight(device)
        if self.transform is not None:
            self.transform.mark_in_flight(device)

    def stage(self, requests: Sequence[MixRequest], executor=None) -> Tuple[MixBatch, List[int], List[int], Optional[int]]:
        from .engine import MIX_CUT_DTYPE, MIX_SRC_F32, MIX_TRACK_DTYPE

        self._wait_idle()
        flat = [t for r in requests for t in r.tracks]
        ints = [i for i, t in enumerate(flat) if isinstance(t.source, _SliceRequest)]
        perturbed = [t.source for t in flat if isinstance(t.source, TransformRequest)]
        # the RIRs are at the cut's rate (reverb_request), so one rate per WAV batch still holds
        rirs = _stage_rirs(requests)
        gen_reqs = _generated_in(requests)
        generated = GeneratedRirs(gen_reqs) if gen_reqs else None
        pcm_buf, flac_batch, read_kind, read_elem, (wav_srs, flac_srs) = self.sources.stage(
            [flat[i].source for i in ints] + rirs, executor=executor)
        if wav_srs:
            _one_rate(wav_srs)
        srs = wav_srs | flac_srs
        kind = np.asarray([-1 if t.source is None else MIX_SRC_F32 for t in flat], dtype=np.int32)
        src_elem = np.zeros(len(flat), dtype=np.int64)
        kind[ints] = read_kind[: len(ints)]
        src_elem[ints] = read_elem[: len(ints)]
        transform_batch = None
        if perturbed:
            if self.transform is None:
                self.transform = TransformStagingRing(pin_memory=self._pin)
            transform_batch, _, offs2, sr2 = self.transform.stage(perturbed, executor=executor, generated=generated)
            src_elem[kind == MIX_SRC_F32] = offs2
            srs.add(sr2)
        B, T = len(requests), len(flat)
        lens = [int(r.num_samples) for r in requests]
        offs, out_elems = _aligned_offsets(lens, self.ALIGN)
        tb, cb = T * MIX_TRACK_DTYPE.itemsize, B * MIX_CUT_DTYPE.itemsize
        self._tables = self._grown(self._tables, max(tb + cb, 1))
        raw = self._tables.numpy()
        tracks = raw[:tb].view(MIX_TRACK_DTYPE)
        cuts = raw[tb: tb + cb].view(MIX_CUT_DTYPE)
        ntr = np.asarray([len(r.tracks) for r in requests], dtype=np.int64)
        tracks["struct_size"] = MIX_TRACK_DTYPE.itemsize
        tracks["source"] = kind
        tracks["src_elem"] = src_elem
        tracks["num_samples"] = [t.num_samples for t in flat]
        tracks["mix_offset"] = [t.offset for t in flat]
        tracks["snr_factor"] = [t.snr_factor for t in flat]
        tracks["cut"] = np.repeat(np.arange(B), ntr)
        tracks["role"] = [t.role for t in flat]
        # a reverberated cut's mix goes to the pre-reverb region after the output, in the same buffer
        rv_ix = [i for i, r in enumerate(requests) if r.reverb is not None]
        pre_offs, pre_elems = _aligned_offsets([lens[i] for i in rv_ix], self.ALIGN)
        base = (out_elems + self.ALIGN - 1) // self.ALIGN * self.ALIGN
        mix_out = list(offs)
        for i, o in zip(rv_ix, pre_offs):
            mix_out[i] = base + o
        cuts["struct_size"] = MIX_CUT_DTYPE.itemsize
        cuts["mode"] = [r.mode for r in requests]
        cuts["out_elem"] = mix_out
        cuts["mix_len"] = [r.mix_len for r in requests]
        cuts["target_len"] = lens
        cuts["first_track"] = np.concatenate(([0], np.cumsum(ntr)[:-1])) if B else []
        cuts["num_tracks"] = ntr
        cuts["ref_track"] = [r.ref for r in requests]
        cuts["reserved"] = 0
        batch = MixBatch(pcm=pcm_buf, flac=flac_batch, tracks=tracks, cuts=cuts, lens=lens, offsets=offs, out_elems=out_elems,
                         transform=transform_batch)
        batch.generated = generated
        if rv_ix:
            batch.pre_elems = base - out_elems + pre_elems
            batch.reverb_rirs, batch.reverb_cuts = _reverb_tables(
                rirs, read_kind[len(ints):], read_elem[len(ints):],
                [(requests[i].reverb, mix_out[i], lens[i], offs[i], lens[i]) for i in rv_ix], generated)
        if generated is not None:
            generated.draw()  # after every read of the batch, its perturbed tracks' included
        return batch, lens, offs, (srs.pop() if len(srs) == 1 else None)


def mix_staged(batch: MixBatch, device, ring: Optional[_PinnedRing] = None, handle=None) -> Tuple[torch.Tensor, List[int], List[int]]:
    """The device half of the "mix" route on the current stream: H2D of the WAV tracks, the FLAC decode (if any), the
    perturbed tracks' transform stages into the float32 track buffer (if any), the table copies, the energy and mix kernels,
    the reverb of the reverberated cuts (if any); then `ring`'s copies are marked in flight.  Returns (float32 mixes on
    `device`, lengths, offsets)."""
    from .engine import mix

    device = torch.device(device)
    with torch.cuda.device(device):
        src0, src1 = _sources_to_device(batch, device)
        rir32 = _generate_rirs(batch.generated, device, handle) if batch.generated is not None else None
        src2 = (transform_staged(batch.transform, device, handle=handle, rir32=rir32)[0]
                if batch.transform is not None else None)
        out = torch.zeros(max(batch.out_elems + batch.pre_elems, 1), dtype=torch.float32, device=device)
        mix(src0, src1, batch.tracks, batch.cuts, out, handle, src2=src2)
        if batch.reverb_cuts is not None:
            _reverb_with(batch, src0, src1, out, out, handle, rir32)
            out = out[: max(batch.out_elems, 1)]
        if ring is not None:
            ring.mark_in_flight(device)
    return out, batch.lens, batch.offsets


def mix_cuts(cuts, device="cuda", executor=None, ring: Optional[MixStagingRing] = None,
             perturbed_tracks: bool = False, reverb: bool = False,
             generated_rir: bool = False) -> Tuple[torch.Tensor, List[int], List[int]]:
    """Mixes MixedCuts (and plain 16-bit WAV / FLAC slices) on the GPU: (float32 device tensor holding every cut's samples at
    its offset, on 4-sample boundaries, lengths, offsets), each cut bit-identical to float32(cut.load_audio()).  Raises
    ValueError naming the first cut the route cannot take.  `perturbed_tracks=True` also takes tracks (and plain cuts) with
    Speed / Volume / Resample chains, run on the GPU into a float32 track buffer first (see `mix_request_for_cut`; off by
    default, so that existing callers keep their behaviour until H100 measurements of the route exist).  `reverb=True` also
    takes MixedCut-level reverbs and plain slices whose only transform is a reverb, reverberated on the GPU within a float32
    tolerance of a float64 convolution (see `mix_request_for_cut`; off by default).  `generated_rir=True` takes those reverbs
    with RIRs that lhotse generates, drawn here from the cuts' generators (rir_draws.py; off by default)."""
    reqs = _requests_or_raise(cuts, lambda c: _mix_or_plain_request(c, perturbed_tracks, reverb, generated_rir),
                              "cannot be mixed on the GPU (see mix_request_for_cut)")
    ring = ring or MixStagingRing()
    batch, _, _, _ = ring.stage(reqs, executor=executor)
    return mix_staged(batch, device, ring)


def _requests_or_raise(cuts, request, refusal: str) -> list:
    """[request(cut) for cut in cuts]; ValueError naming the first cut for which `request` returns None."""
    reqs = []
    for c in cuts:
        r = request(c)
        if r is None:
            raise ValueError(f"cut {getattr(c, 'id', c)!r} {refusal}")
        reqs.append(r)
    return reqs


# ---- Speed / Volume / Resample transforms ---------------------------------------------------------------------------
# A MonoCut whose recording carries a chain of Speed, Volume and Resample transforms (CutSet.perturb_speed / perturb_volume /
# resample): its source slice is staged as int16 by the two rings above, and the sm_90a kernel of csrc/resample.cuh runs the
# chain on the device, bit for bit what cut.load_audio() returns where torch sends lhotse's resampling conv1d to oneDNN
# (DESIGN.md §3.1i).  The samples land as float32 in the ragged layout `Engine.extract_device` takes.

ONEDNN_MIN_INPUT = 20481     # ATen runs this conv1d through oneDNN only when the padded input has more than 20480 elements
_RESAMPLE_MAX_WINDOW = 8192  # K + O of a table the kernel takes (csrc/resample.cuh RS_WIN_FLOATS)
_RESAMPLE_MAX_TABLE = 1 << 22


def _resample_geometry(orig: int, new: int) -> Tuple[int, int, int, int]:
    """(N, O, width, K) of lhotse's resampler for orig -> new (lowpass filter width 6, rolloff 0.99)."""
    g = math.gcd(orig, new)
    O, N = orig // g, new // g
    width = math.ceil(6 * O / (min(O, N) * 0.99))
    return N, O, width, 2 * width + O


def resampled_len(N: int, L: int, O: int) -> int:
    """Samples lhotse's resampler keeps of an input of L samples: `torch.ceil(torch.as_tensor(N * L / O))`, where the Python
    float quotient becomes a float32 tensor (torch's default dtype; the route requires it), so a small fractional part is
    rounded away once the quotient reaches a few tens of thousands; never more than the N * (L // O + 1) outputs the conv
    produces."""
    return min(int(math.ceil(np.float32(N * L / O))), N * (L // O + 1))


_KERNELS: "dict[Tuple[int, int], Tuple[np.ndarray, int]]" = {}
_KERNELS_LOCK = threading.Lock()


def resample_kernel(orig: int, new: int) -> Tuple[np.ndarray, int]:
    """(float32 table [N][K], width) of lhotse's Hann-windowed sinc resampler for orig -> new.  Output phase p, tap k sits at
    time u = (-p / N + (k - width) / O) * min(O, N) * 0.99, clamped to +-6; its weight is sinc(pi u) * cos^2(pi u / 12) *
    min(O, N) * 0.99 / O.  The table is evaluated in float64 with the torch operations lhotse uses, in the same order (the
    phase offsets -p / N in torch's default float dtype), and rounded once."""
    key = (int(orig), int(new))
    with _KERNELS_LOCK:
        hit = _KERNELS.get(key)
    if hit is not None:
        return hit
    N, O, width, _ = _resample_geometry(*key)
    lpw, base = 6, min(O, N) * 0.99
    u = (torch.arange(0, -N, -1) / N)[:, None] + torch.arange(-width, width + O, dtype=torch.float64)[None, :] / O
    u *= base
    u = u.clamp_(-lpw, lpw)
    hann = torch.cos(u * math.pi / lpw / 2) ** 2
    u *= math.pi
    w = torch.where(u == 0, torch.tensor(1.0).to(u), u.sin() / u)
    w *= hann * (base / O)
    hit = (w.to(torch.float32).numpy().copy(), width)
    with _KERNELS_LOCK:
        _KERNELS[key] = hit
    return hit


def _fma32(a: np.ndarray, b: np.ndarray, c: np.ndarray) -> np.ndarray:
    """float32 fma(a, b, c), rounded once, for float32 arrays: a * b is exact in float64, the float64 sum's own rounding error
    comes from TwoSum, and a sum that sits exactly between two float32 values is rounded toward that error's side."""
    p = a.astype(np.float64) * b.astype(np.float64)
    c64 = c.astype(np.float64)
    s = p + c64
    z = s - p
    e = (p - (s - z)) + (c64 - z)  # p + c64 == s + e exactly
    r = s.astype(np.float32)
    d = s - r.astype(np.float64)
    cand = (e != 0) & (d != 0)
    if cand.any():
        other = np.nextafter(r, np.where(d > 0, np.float32(np.inf), np.float32(-np.inf)))
        tie = cand & ((r.astype(np.float64) + other.astype(np.float64)) * 0.5 == s)
        r = np.where(tie & ((e > 0) == (d > 0)), other, r)
    return r


def resample_reference(x: np.ndarray, orig: int, new: int) -> np.ndarray:
    """The resampling contract of DESIGN.md §3.1i in NumPy: the zero-padded segment, one float32 FMA chain per output over
    the K taps in tap order from +0, `resampled_len` outputs kept.  What the kernel computes, on the host."""
    table, width = resample_kernel(orig, new)
    N, K = table.shape
    O = K - 2 * width
    L = int(x.shape[0])
    xp = np.concatenate([np.zeros(width, np.float32), np.asarray(x, np.float32), np.zeros(width + O, np.float32)])
    at = np.arange((xp.shape[0] - K) // O + 1) * O
    acc = np.zeros((at.shape[0], N), np.float32)
    for t in range(K):
        acc = _fma32(xp[at + t][:, None], table[None, :, t], acc)
    return acc.reshape(-1)[: resampled_len(N, L, O)]


_PROBES: "dict[Tuple[int, int], bool]" = {}
_PROBES_LOCK = threading.Lock()


def resample_probe(orig: int, new: int) -> bool:
    """Whether lhotse's own resampler for orig -> new, run here by torch, equals `resample_reference` bit for bit on a
    seeded signal long enough for oneDNN (with a silent stretch, so signed zeros are compared too) and uses the same table.
    Run once per pair and process: on a host whose oneDNN sums in another order the route declines instead of diverging."""
    key = (int(orig), int(new))
    with _PROBES_LOCK:
        ok = _PROBES.get(key)
        if ok is not None:
            return ok
        from lhotse.augmentation.torchaudio import get_or_create_resampler

        rs = np.random.RandomState(key[0] * 7919 + key[1])
        q = rs.randint(-32768, 32768, ONEDNN_MIN_INPUT + 3000).astype(np.int16)
        q[4000:6000] = 0
        x = q.astype(np.float32) / np.float32(32768)
        resampler = get_or_create_resampler(*key)
        with torch.no_grad():
            got = resampler(torch.from_numpy(x)[None]).numpy()[0]
        want = resample_reference(x, *key)
        ok = bool(got.dtype == np.float32 and got.shape == want.shape and np.array_equal(got.view(np.int32), want.view(np.int32))
                  and np.array_equal(resampler.kernel[:, 0, :].numpy(), resample_kernel(*key)[0]))
        _PROBES[key] = ok
        return ok


@dataclass(frozen=True)
class ReverbRequest:
    rir: object                # PcmRequest | FlacRequest: the RIR's samples, what `rir.load_audio()` reads; or a GeneratedRirRequest
    normalize: bool            # lhotse's normalize_output


@dataclass(frozen=True, eq=False)
class GeneratedRirRequest:
    """An RIR that lhotse's FastRandomRIRGenerator `generator` makes when the cut is loaded (no recorded RIR): drawn on the host
    when the batch is staged (rir_draws.py) and built on the GPU (csrc/rirgen.cuh).  Every request is its own RIR."""
    generator: object


@dataclass(frozen=True)
class WpeRequest:
    """A DereverbWPE transform's parameters (its n_fft and hop are 512 and 128: `wpe_request` takes no others)."""
    taps: int = 10
    delay: int = 3
    iterations: int = 3
    statistics_mode: str = "full"


@dataclass(frozen=True)
class TransformRequest:
    source: object             # PcmRequest | FlacRequest: the slice of the file the chain starts from
    ops: Tuple[tuple, ...]     # in chain order: ("volume", float32 factor) | ("resample", orig, new)
    num_samples: int           # the cut's length: the chain's output is trimmed or reflect-padded to it
    sampling_rate: int         # the cut's (the recording's, after the chain)
    reverb: Optional[ReverbRequest] = None  # a last ReverbWithImpulseResponse, run on the chain's output before the length fix
    wpe: Optional[WpeRequest] = None  # a last DereverbWPE, run on the chain's (or the reverb's) output before the length fix


def wpe_request(t) -> Optional[WpeRequest]:
    """The parameters of a DereverbWPE transform the GPU takes (csrc/wpe.cuh): n_fft 512, hop_length 128, 1 <= taps <=
    WPE_MAX_TAPS, delay >= 0, 0 <= iterations <= 64, statistics_mode "full" or "valid", all plain ints.  None otherwise."""
    from .engine import WPE_MAX_TAPS

    ints = (t.n_fft, t.hop_length, t.taps, t.delay, t.iterations)
    if any(type(v) is not int for v in ints) or (t.n_fft, t.hop_length) != (512, 128):
        return None
    if not 1 <= t.taps <= WPE_MAX_TAPS or t.delay < 0 or not 0 <= t.iterations <= 64:
        return None
    if t.statistics_mode not in ("full", "valid"):
        return None
    return WpeRequest(taps=t.taps, delay=t.delay, iterations=t.iterations, statistics_mode=t.statistics_mode)


def wpe_output_len(L: int, w: WpeRequest) -> Optional[int]:
    """The length DereverbWPE gives a signal of L samples, 128 (L // 128); None when the GPU does not take it: L <= 256
    (torch.stft's reflect pad), fewer than taps + delay frames (R is singular in exact arithmetic), more than WPE_MAX_FRAMES
    frames (a bin no longer fits in shared memory)."""
    from .engine import WPE_MAX_FRAMES

    T = 1 + L // 128
    if L <= 256 or T < w.taps + w.delay or T > WPE_MAX_FRAMES:
        return None
    return 128 * (L // 128)


def reverb_request(t, sampling_rate: int, reverb: bool = True, generated_rir: bool = False) -> Optional[ReverbRequest]:
    """The RIR read of a ReverbWithImpulseResponse with a recorded mono RIR, as its __call__ loads it: `rir.to_cut()` for a
    Recording, `with_channels(rir_channels)`, `truncate(duration=0.05)` when early_only, then a cut that
    `pcm16_request_for_cut` / `flac_request_for_cut` accept, with no transforms of its own and 1 <= R <= REVERB_MAX_RIR
    samples, at `sampling_rate` (the cut's).  None otherwise: several RIR channels (a MultiCut), other formats, longer RIRs,
    an RIR at another rate (lhotse convolves it as it is stored; this route does not take it).  `reverb=False` refuses
    recorded RIRs.

    `generated_rir=True` also takes a ReverbWithImpulseResponse with no RIR whose generator `rir_draws.generator_eligible`
    accepts (exactly lhotse's FastRandomRIRGenerator, torchaudio present, float32 default dtype, a restatement of torch's
    multinomial that holds here), one RIR channel and RIRs of at most REVERB_MAX_RIR samples; lhotse ignores early_only
    for a generated RIR, and so does this route."""
    from lhotse import Recording
    from lhotse.cut import MonoCut

    from .engine import REVERB_MAX_RIR

    if len(t.rir_channels) != 1:
        return None
    if t.rir is None:
        from . import rir_draws

        gen = getattr(t, "rir_generator", None)
        if not generated_rir or not rir_draws.generator_eligible(gen) or rir_draws.max_rir_len(gen) > REVERB_MAX_RIR:
            return None
        return ReverbRequest(rir=GeneratedRirRequest(gen), normalize=bool(t.normalize_output))
    if not reverb:
        return None
    try:
        rir = t.rir.to_cut() if isinstance(t.rir, Recording) else t.rir
        rir = rir.with_channels(list(t.rir_channels))
        if t.early_only:
            rir = rir.truncate(duration=0.05)
    except Exception:  # lhotse would raise on the float route too
        return None
    if not isinstance(rir, MonoCut) or getattr(rir, "tracks", None) is not None or rir.sampling_rate != sampling_rate:
        return None
    src = slice_request_for_cut(rir)
    if src is None or not 1 <= src.num_samples <= REVERB_MAX_RIR:
        return None
    return ReverbRequest(rir=src, normalize=bool(t.normalize_output))


def transform_request_for_cut(cut, reverb: bool = False, generated_rir: bool = False,
                              wpe: bool = False) -> Optional[TransformRequest]:
    """What `cut.load_audio()` (audio/recording.py load_audio) amounts to for a MonoCut over a single-channel 16-bit WAV or
    FLAC file whose recording carries a non-empty chain of Speed, Volume and Resample transforms: the source slice (the
    transforms' own reverse_timestamps applied to the cut's range, a read to the end of the file when the cut's duration is
    within 1 ms of the recording's), the chain, and the cut's length.  None when not eligible: another kind of cut or
    transform, a Resample lhotse would not run through its torch resampler (sox backend, no torchaudio), a resampling stage
    whose padded input is too short for oneDNN, oneDNN off, a rate pair whose probe fails, or a length outside lhotse's
    duration-mismatch tolerance.

    `reverb=True` also takes a chain whose last transform is a ReverbWithImpulseResponse that `reverb_request` accepts (a
    reverb alone included): the stages before it write the pre-reverb signal, and the reverb kernel (csrc/reverb.cuh) writes
    the cut, within a float32 tolerance of a float64 convolution rather than bit for bit (DESIGN.md §3.1j).  Off by default
    so that existing callers keep exactly the routes and samples they have.  `generated_rir=True` takes such a last
    reverb with an RIR that lhotse generates (see `reverb_request`; DESIGN.md §3.1l), also off by default.

    `wpe=True` also takes a chain whose last transform is a DereverbWPE that `wpe_request` accepts, after Speed / Volume /
    Resample stages and an optional reverb (WPE alone on a plain slice included, what `cuts.dereverb_wpe()` makes): the
    signal before it goes to an intermediate buffer at its natural length and the WPE kernels (csrc/wpe.cuh) write the cut,
    within a float32 tolerance of a float64 restatement (DESIGN.md §3.1q).  The duration-mismatch check then applies to
    DereverbWPE's output length, 128 (L // 128).  Off by default."""
    try:
        from lhotse.augmentation.rir import ReverbWithImpulseResponse
        from lhotse.augmentation.wpe import DereverbWPE
        from lhotse.audio.resampling_backend import get_current_resampling_backend
        from lhotse.audio.utils import get_audio_duration_mismatch_tolerance
        from lhotse.augmentation import torchaudio as lta
        from lhotse.augmentation.transform import AudioTransform
        from lhotse.cut import MonoCut
    except ImportError:
        return None
    rec = getattr(cut, "recording", None)
    if not isinstance(cut, MonoCut) or getattr(cut, "tracks", None) is not None or rec is None or not rec.transforms:
        return None
    if getattr(rec, "has_video", False) or not (torch.backends.mkldnn.is_available() and torch.backends.mkldnn.enabled):
        return None
    if torch.get_default_dtype() != torch.float32:
        return None  # lhotse's table phases and output lengths are evaluated in the default dtype
    tfs = [t if isinstance(t, AudioTransform) else AudioTransform.from_dict(t) for t in rec.transforms]
    wr = None
    if wpe and type(tfs[-1]) is DereverbWPE:
        wr = wpe_request(tfs[-1])
        if wr is None:
            return None
        tfs = tfs[:-1]
    rv = None
    if (reverb or generated_rir) and tfs and type(tfs[-1]) is ReverbWithImpulseResponse:
        rv = reverb_request(tfs[-1], rec.sampling_rate, reverb, generated_rir)
        if rv is None:
            return None
        tfs = tfs[:-1]
    if any(type(t) not in (lta.Speed, lta.Volume, lta.Resample) for t in tfs):
        return None
    sources = rec.sources or []
    if len(sources) != 1 or sources[0].type != "file" or list(sources[0].channels) != [cut.channel]:
        return None
    opened = _open_slice_file(sources[0].source)
    if opened is None or opened[0].channels != 1:
        return None
    h, make = opened
    sr = rec.sampling_rate
    offset, duration = cut.start, cut.duration
    if math.isclose(duration, rec.duration, abs_tol=1e-3):
        duration = None  # load_audio reads to the end of the file
    for t in reversed(tfs):
        offset, duration = t.reverse_timestamps(offset=offset, duration=duration, sampling_rate=sr)
    first = _samples(offset, h.sampling_rate)
    n = h.num_samples - first if duration is None else _samples(duration, h.sampling_rate)
    if first < 0 or n <= 0 or first + n > h.num_samples:
        return None
    ops, L = [], n
    for t in tfs:
        if isinstance(t, lta.Volume):
            if type(t.factor) not in (int, float) or not math.isfinite(np.float32(t.factor)):
                return None  # a NumPy scalar factor would promote the samples to float64
            ops.append(("volume", float(np.float32(t.factor))))
            continue
        if isinstance(t, lta.Speed):
            a, b = round(sr * t.factor), sr
        else:
            if get_current_resampling_backend() != "default" or not lta.is_torchaudio_available():
                return None  # sox, or scipy's resample_poly in float64
            a, b = t.source_sampling_rate, t.target_sampling_rate
        if a == b:
            continue  # lhotse returns the samples unchanged
        N, O, width, K = _resample_geometry(a, b)
        if L + 2 * width + O < ONEDNN_MIN_INPUT or K + O > _RESAMPLE_MAX_WINDOW or N * K > _RESAMPLE_MAX_TABLE:
            return None
        if not resample_probe(a, b):
            return None
        ops.append(("resample", int(a), int(b)))
        L = resampled_len(N, L, O)
    if wr is not None:
        L = wpe_output_len(L, wr)
        if L is None:
            return None
    target = _samples(cut.duration, sr)
    diff = target - L
    if abs(diff) > int(math.ceil(get_audio_duration_mismatch_tolerance() * sr)) or diff > L - 1:
        return None
    return TransformRequest(source=make(path=h.path, first_sample=first, num_samples=n), ops=tuple(ops), num_samples=target,
                            sampling_rate=int(sr), reverb=rv, wpe=wr)


def _has_transforms(cut) -> bool:
    return bool(getattr(getattr(cut, "recording", None), "transforms", None))


def transform_requests_for_batch(cuts, reverb: bool = False, generated_rir: bool = False,
                                 wpe: bool = False) -> Optional[List[TransformRequest]]:
    """The "transform" route's requests for a batch: no MixedCut, every cut a plain 16-bit WAV / FLAC slice or an eligible
    transformed MonoCut, and at least one of the latter (batches of plain slices keep their routes).  None otherwise.
    `reverb=True`, `wpe=True`: see `transform_request_for_cut`."""
    if any(getattr(c, "tracks", None) is not None for c in cuts) or not any(_has_transforms(c) for c in cuts):
        return None
    reqs = [_transform_or_plain_request(c, reverb, generated_rir, wpe) for c in cuts]
    return None if any(r is None for r in reqs) else reqs


def _transform_or_plain_request(cut, reverb: bool = False, generated_rir: bool = False,
                                wpe: bool = False) -> Optional[TransformRequest]:
    """transform_request_for_cut, or a plain 16-bit WAV / FLAC slice as an empty chain (a copy of x = q / 32768)."""
    if _has_transforms(cut):
        r = transform_request_for_cut(cut, reverb=reverb, generated_rir=generated_rir, wpe=wpe)
    else:
        src = slice_request_for_cut(cut)
        r = (TransformRequest(source=src, ops=(), num_samples=int(src.num_samples), sampling_rate=int(cut.sampling_rate))
             if src is not None else None)
    return r if r is not None and r.num_samples > 0 else None


def _chain_stages(ops) -> List[Tuple[float, Optional[Tuple[int, int]], float]]:
    """The chain as kernel stages (load scale, rate pair or None, store scale): each Volume goes into the load scale of a stage
    that has not resampled yet, else into the store scale of a stage that has none yet, else it opens a new stage."""
    stages = [[1.0, None, 1.0, False]]  # load scale, pair, store scale, store scale taken
    for op in ops:
        s = stages[-1]
        if op[0] == "volume":
            if s[1] is None and s[0] == 1.0 and not s[3]:
                s[0] = op[1]
            elif not s[3]:
                s[2], s[3] = op[1], True
            else:
                stages.append([op[1], None, 1.0, False])
        elif s[1] is None and not s[3]:
            s[1] = (op[1], op[2])
        else:
            stages.append([1.0, (op[1], op[2]), 1.0, False])
    return [(a, p, b) for a, p, b, _ in stages]


@dataclass
class TransformBatch:
    """One staged transform batch: the WAV slices in the ring's pinned int16 buffer, the FLAC slices as a staged
    FlacBatch, and the b200feat_resample stage table (a pinned numpy view, sorted by depth) with the rate pair of each stage."""
    pcm: Optional[torch.Tensor]
    flac: Optional[FlacBatch]
    stages: np.ndarray        # engine.RESAMPLE_STAGE_DTYPE; `table` is filled per device by transform_staged
    pair: np.ndarray          # index into `pairs` of every stage, -1: no resampling
    pairs: List[Tuple[int, int]]
    mid_elems: int
    lens: List[int]
    offsets: List[int]
    out_elems: int
    reverb_rirs: Optional[np.ndarray] = None  # engine.REVERB_RIR_DTYPE: the batch's distinct RIRs in the two int16 sources
    reverb_cuts: Optional[np.ndarray] = None  # engine.REVERB_CUT_DTYPE: the reverberated cuts, reading `mid`
    generated: Optional["GeneratedRirs"] = None  # the generated RIRs, after the recorded ones in `reverb_rirs`
    reverb_mid_cuts: Optional[np.ndarray] = None  # engine.REVERB_CUT_DTYPE: the reverberated cuts that WPE follows, `mid` to `mid`
    wpe: List[Tuple[WpeRequest, np.ndarray]] = field(default_factory=list)  # engine.WPE_CUT_DTYPE per parameter set, `mid` to out


def _stage_rirs(reqs) -> List[_SliceRequest]:
    """The distinct RIR reads of `reqs` (objects with a `reverb` field) in order of first use, to be staged after the batch's
    own reads so that they cross with its samples."""
    rirs = {}
    for r in reqs:
        rv = getattr(r, "reverb", None)
        if rv is not None and not isinstance(rv.rir, GeneratedRirRequest):
            rirs.setdefault(rv.rir, None)
    return list(rirs)


class GeneratedRirs:
    """The generated RIRs of one staged batch, in batch order: each one's place in the float32 RIR buffer (room for the
    longest RIR its generator can give, so that the places are known before the draws), and once `draw` has run, the draws
    (rir_draws.RirDraws) and the generator states from before them."""

    ALIGN = 4

    def __init__(self, reqs: Sequence[GeneratedRirRequest]):
        from . import rir_draws

        self.reqs = list(reqs)
        self.index = {id(r): i for i, r in enumerate(self.reqs)}
        self.elems, self.elems_total = _aligned_offsets([rir_draws.max_rir_len(r.generator) for r in self.reqs], self.ALIGN)
        self.draws = None
        self.snapshot = None

    def draw(self) -> None:
        """Draws every RIR, after saving the state of every generator the draws touch (see `undo_draws`)."""
        from . import rir_draws

        gens = [r.generator for r in self.reqs]
        self.snapshot = rir_draws.snapshot(gens)
        try:
            self.draws = rir_draws.draw(gens)
        except BaseException:
            self.undo()
            raise

    def undo(self) -> None:
        from . import rir_draws

        rir_draws.restore(self.snapshot)
        self.snapshot, self.draws = None, None


def _generated_in(reqs) -> List[GeneratedRirRequest]:
    """The generated RIRs of `reqs` (TransformRequests, or MixRequests whose perturbed tracks may carry one), in batch order."""
    out = []
    for r in reqs:
        for t in getattr(r, "tracks", ()):
            rv = getattr(t.source, "reverb", None)
            if rv is not None and isinstance(rv.rir, GeneratedRirRequest):
                out.append(rv.rir)
        rv = getattr(r, "reverb", None)
        if rv is not None and isinstance(rv.rir, GeneratedRirRequest):
            out.append(rv.rir)
    return out


def undo_draws(staged) -> None:
    """Restores the generator states from before the draws of a staged batch that will not be used (the batch falls back
    to the float route, which then draws the same numbers); nothing for a batch without generated RIRs."""
    gen = getattr(staged, "generated", None)
    if gen is not None:
        gen.undo()


def _generate_rirs(gen: GeneratedRirs, device, handle=None) -> torch.Tensor:
    """The device half of the generated RIRs on the current stream: the draws' upload, b200feat_rir_generate at 8 x sr, then
    b200feat_resample with lhotse's 8 -> 1 table to sr.  Returns the float32 RIR buffer (RIR i at gen.elems[i])."""
    from .engine import RESAMPLE_MID, RESAMPLE_STAGE_DTYPE, RESAMPLE_TO_OUT, resample, resample_table, rir_generate

    d = gen.draws
    rec = d.records.copy()
    lens8 = [int(n) for n in rec["out_len"]]
    offs8, total8 = _aligned_offsets(lens8, GeneratedRirs.ALIGN)
    rec["out_elem"] = offs8
    table, width = resample_kernel(8, 1)
    draws = torch.from_numpy(d.draws).to(device)
    cdf = torch.from_numpy(d.cdf).to(device)
    mid = torch.empty(max(total8, 1), dtype=torch.float32, device=device)
    rir_generate(draws, cdf, table[0], rec, mid, handle)
    st = np.zeros(len(rec), dtype=RESAMPLE_STAGE_DTYPE)
    st["struct_size"] = RESAMPLE_STAGE_DTYPE.itemsize
    st["table"] = resample_table(8, 1, table, width, device, handle)
    st["source"], st["target"], st["scale_in"], st["scale_out"] = RESAMPLE_MID, RESAMPLE_TO_OUT, 1.0, 1.0
    st["in_elem"], st["in_len"] = offs8, lens8
    st["out_elem"], st["out_len"], st["target_len"] = gen.elems, d.lens, d.lens
    out = torch.zeros(max(gen.elems_total, 1), dtype=torch.float32, device=device)
    resample(None, None, mid, st, out, handle)
    return out


def _reverb_with(batch, src0, src1, x, out, handle, rir32, cuts: Optional[np.ndarray] = None) -> None:
    """b200feat_reverb_ex over a staged batch's reverb tables (`cuts`, or its reverb_cuts), the generated RIRs' lengths
    filled in from their draws."""
    from .engine import reverb

    rt = batch.reverb_rirs
    if batch.generated is not None:
        rt = rt.copy()
        rt["num_samples"][len(rt) - len(batch.generated.reqs):] = batch.generated.draws.lens
    reverb(src0, src1, x, rt, batch.reverb_cuts if cuts is None else cuts, out, handle, rir32=rir32)


def _reverb_tables(rirs, source, rir_elem, cuts, generated: Optional[GeneratedRirs] = None) -> Tuple[np.ndarray, np.ndarray]:
    """The b200feat_reverb_ex tables: RIR i in int16 source source[i] at rir_elem[i], then the generated RIRs of `generated`
    (their lengths filled in by `_reverb_with` once drawn); cuts = [(ReverbRequest, in_elem, in_len, out_elem,
    target_len)]."""
    from .engine import REVERB_CUT_DTYPE, REVERB_RIR_DTYPE, REVERB_RIR_F32

    ng = len(generated.reqs) if generated is not None else 0
    rt = np.zeros(len(rirs) + ng, dtype=REVERB_RIR_DTYPE)
    rt["struct_size"] = REVERB_RIR_DTYPE.itemsize
    rt["source"][: len(rirs)] = source
    rt["src_elem"][: len(rirs)] = rir_elem
    rt["num_samples"][: len(rirs)] = [r.num_samples for r in rirs]
    if ng:
        rt["source"][len(rirs):] = REVERB_RIR_F32
        rt["src_elem"][len(rirs):] = generated.elems
    ix = {r: i for i, r in enumerate(rirs)}
    if ng:
        ix.update({r: len(rirs) + i for i, r in enumerate(generated.reqs)})
    ct = np.zeros(len(cuts), dtype=REVERB_CUT_DTYPE)
    ct["struct_size"] = REVERB_CUT_DTYPE.itemsize
    ct["rir"] = [ix[rv.rir] for rv, *_ in cuts]
    ct["normalize"] = [int(rv.normalize) for rv, *_ in cuts]
    for name, col in zip(("in_elem", "in_len", "out_elem", "target_len"), range(1, 5)):
        ct[name] = [c[col] for c in cuts]
    return rt, ct


def _wpe_table(rows) -> np.ndarray:
    """The b200feat_wpe cut table of rows = [(in_elem, in_len, out_elem, target_len)]."""
    from .engine import WPE_CUT_DTYPE

    ct = np.zeros(len(rows), dtype=WPE_CUT_DTYPE)
    ct["struct_size"] = WPE_CUT_DTYPE.itemsize
    for name, col in zip(("in_elem", "in_len", "out_elem", "target_len"), range(4)):
        ct[name] = [r[col] for r in rows]
    return ct


class TransformStagingRing(_PinnedRing):
    """A _SourceRing for the source slices (files of several rates allowed: a Resample chain starts at its file's own rate)
    and pinned table bytes for one transform batch; `stage(requests)` returns (TransformBatch, lengths, offsets, the cuts'
    sampling rate), the rate None when the cuts have several."""

    ALIGN = 4

    def __init__(self, pin_memory: Optional[bool] = None):
        super().__init__(pin_memory)
        self.sources = _SourceRing(pin_memory=self._pin)
        self._tables = torch.empty(1 << 16, dtype=torch.uint8, pin_memory=self._pin)

    def mark_in_flight(self, device=None) -> None:
        super().mark_in_flight(device)
        self.sources.mark_in_flight(device)

    def stage(self, requests: Sequence[TransformRequest], executor=None,
              generated: Optional[GeneratedRirs] = None) -> Tuple[TransformBatch, List[int], List[int], Optional[int]]:
        """`generated`: the generated RIRs of an enclosing mix batch, which draws them; without it the generated RIRs of
        `requests` are drawn here, after the reads."""
        from .engine import RESAMPLE_MID, RESAMPLE_STAGE_DTYPE, RESAMPLE_TO_MID, RESAMPLE_TO_OUT

        self._wait_idle()
        B = len(requests)
        rirs = _stage_rirs(requests)
        gen_reqs = _generated_in(requests)
        own = generated is None and bool(gen_reqs)
        if own:
            generated = GeneratedRirs(gen_reqs)
        pcm_buf, flac_batch, kind, src_elem, _ = self.sources.stage([r.source for r in requests] + rirs, executor=executor)
        srs = {r.sampling_rate for r in requests}
        lens = [int(r.num_samples) for r in requests]
        offs, out_elems = _aligned_offsets(lens, self.ALIGN)
        pairs, pair_ix = [], {}
        rows = []  # (depth, cut, table pair, source, in_elem, in_len, target, out_elem, out_len, target_len, scale_in, scale_out)
        rv_cuts = []  # (ReverbRequest, in_elem, in_len, out_elem, target_len)
        rv_mid = []   # the same, for the reverbs that WPE follows: into `mid` at their natural length
        wpe_cuts = {}  # WpeRequest -> [(in_elem, in_len, out_elem, target_len)]
        mid = 0
        for i, r in enumerate(requests):
            chain = _chain_stages(r.ops)
            source, in_elem, L = int(kind[i]), int(src_elem[i]), int(r.source.num_samples)
            for d, (s_in, pair, s_out) in enumerate(chain):
                if pair is None:
                    pi, n_out = -1, L
                else:
                    pi = pair_ix.setdefault(pair, len(pairs))
                    if pi == len(pairs):
                        pairs.append(pair)
                    N, O, _, _ = _resample_geometry(*pair)
                    n_out = resampled_len(N, L, O)
                last = d == len(chain) - 1
                # a reverberated or dereverberated cut's last stage writes its signal into `mid` at its natural length
                to_out = last and r.reverb is None and r.wpe is None
                out_elem = offs[i] if to_out else mid
                rows.append((d, i, pi, source, in_elem, L, RESAMPLE_TO_OUT if to_out else RESAMPLE_TO_MID, out_elem, n_out,
                             lens[i] if to_out else n_out, s_in, s_out))
                if not to_out:
                    mid += n_out
                if last and r.reverb is not None and r.wpe is None:
                    rv_cuts.append((r.reverb, out_elem, n_out, offs[i], lens[i]))
                elif last and r.reverb is not None:
                    rv_mid.append((r.reverb, out_elem, n_out, mid, n_out))  # the reverb keeps the length: no length fix
                    out_elem = mid
                    mid += n_out
                if last and r.wpe is not None:
                    wpe_cuts.setdefault(r.wpe, []).append((out_elem, n_out, offs[i], lens[i]))
                source, in_elem, L = RESAMPLE_MID, out_elem, n_out
        rows.sort(key=lambda row: (row[0], row[1]))
        nb = len(rows) * RESAMPLE_STAGE_DTYPE.itemsize
        self._tables = self._grown(self._tables, max(nb, 1))
        st = self._tables.numpy()[:nb].view(RESAMPLE_STAGE_DTYPE)
        cols = list(zip(*rows)) if rows else [()] * 12
        st["struct_size"] = RESAMPLE_STAGE_DTYPE.itemsize
        st["table"] = -1
        st["depth"], st["source"], st["in_elem"], st["in_len"] = cols[0], cols[3], cols[4], cols[5]
        st["target"], st["out_elem"], st["out_len"], st["target_len"] = cols[6], cols[7], cols[8], cols[9]
        st["scale_in"], st["scale_out"] = cols[10], cols[11]
        st["reserved"] = 0
        batch = TransformBatch(pcm=pcm_buf, flac=flac_batch, stages=st, pair=np.asarray(cols[2], dtype=np.int64), pairs=pairs,
                               mid_elems=mid, lens=lens, offsets=offs, out_elems=out_elems)
        if rv_cuts or rv_mid:
            batch.generated = generated if gen_reqs else None
            batch.reverb_rirs, ct = _reverb_tables(rirs, kind[B:], src_elem[B:], rv_cuts + rv_mid, batch.generated)
            batch.reverb_cuts = ct[: len(rv_cuts)] if rv_cuts else None
            batch.reverb_mid_cuts = ct[len(rv_cuts):] if rv_mid else None
        for w, rows_w in wpe_cuts.items():
            batch.wpe.append((w, _wpe_table(rows_w)))
        if own:
            generated.draw()
        return batch, lens, offs, (srs.pop() if len(srs) == 1 else None)


def transform_staged(batch: TransformBatch, device, ring: Optional[_PinnedRing] = None, handle=None,
                     rir32: Optional[torch.Tensor] = None) -> Tuple[torch.Tensor, List[int], List[int]]:
    """The device half of the "transform" route on the current stream: the rate pairs' tables (built and uploaded once per
    device), H2D of the WAV slices, the FLAC decode (if any), the resampling stages, the reverb and WPE (if any); then `ring`'s copies
    are marked in flight.  Returns (float32 samples on `device`, lengths, offsets).  The generated RIRs are built first
    unless `rir32` holds them (an enclosing mix batch built them)."""
    from .engine import resample, resample_table, wpe

    device = torch.device(device)
    with torch.cuda.device(device):
        ids = np.asarray([resample_table(a, b, *resample_kernel(a, b), device, handle) for a, b in batch.pairs] + [-1],
                         dtype=np.int32)
        batch.stages["table"] = ids[batch.pair]  # pair -1 picks the trailing -1
        src0, src1 = _sources_to_device(batch, device)
        mid = torch.empty(batch.mid_elems, dtype=torch.float32, device=device) if batch.mid_elems else None
        out = torch.zeros(max(batch.out_elems, 1), dtype=torch.float32, device=device)
        resample(src0, src1, mid, batch.stages, out, handle)
        if batch.reverb_cuts is not None or batch.reverb_mid_cuts is not None:
            if batch.generated is not None and rir32 is None:
                rir32 = _generate_rirs(batch.generated, device, handle)
            if batch.reverb_cuts is not None:
                _reverb_with(batch, src0, src1, mid, out, handle, rir32)
            if batch.reverb_mid_cuts is not None:
                _reverb_with(batch, src0, src1, mid, mid, handle, rir32, batch.reverb_mid_cuts)
        for w, table in batch.wpe:
            wpe(mid, table, out, taps=w.taps, delay=w.delay, iterations=w.iterations, statistics_mode=w.statistics_mode,
                handle=handle)
        if ring is not None:
            ring.mark_in_flight(device)
    return out, batch.lens, batch.offsets


def transform_cuts(cuts, device="cuda", executor=None, ring: Optional[TransformStagingRing] = None,
                   reverb: bool = False, generated_rir: bool = False,
                   wpe: bool = False) -> Tuple[torch.Tensor, List[int], List[int]]:
    """Loads speed-perturbed, volume-perturbed and resampled cuts (and plain 16-bit WAV / FLAC slices) with the transforms run
    on the GPU: (float32 device tensor holding every cut's samples at its offset, on 4-sample boundaries, lengths, offsets),
    each cut bit-identical to float32(cut.load_audio()).  Raises ValueError naming the first cut the route cannot take.
    `reverb=True` also takes chains that end in a ReverbWithImpulseResponse with a recorded RIR, reverberated on the GPU
    within a float32 tolerance of a float64 convolution (see `transform_request_for_cut`; off by default).
    `generated_rir=True` takes such chains whose RIR lhotse generates, drawn here from the cuts' generators (rir_draws.py;
    off by default).  `wpe=True` takes chains that end in lhotse's DereverbWPE, dereverberated on the GPU within a float32
    tolerance of a float64 restatement (see `transform_request_for_cut`; off by default)."""
    reqs = _requests_or_raise(cuts, lambda c: _transform_or_plain_request(c, reverb, generated_rir, wpe),
                              "cannot be loaded on the GPU (see transform_request_for_cut)")
    ring = ring or TransformStagingRing()
    batch, _, _, _ = ring.stage(reqs, executor=executor)
    return transform_staged(batch, device, ring)


# ---- One entry point per step for the callers ----------------------------------------------------------------------

STAGED_ROUTES = ("pcm16", "flac", "mix", "transform")


def staged_route(cuts, perturbed_tracks: bool = False, reverb: bool = False,
                 generated_rir: bool = False, wpe: bool = False) -> Optional[Tuple[str, list]]:
    """(route, requests) of the staged route that takes the batch, the route one of STAGED_ROUTES; None when the cuts have
    more than one sampling rate or no staged route takes them.  A batch with a MixedCut can only go to "mix", else one with
    recording transforms only to "transform"; a batch of plain slices goes to "pcm16" when they are all WAV, to "flac" when
    they are all FLAC.  `perturbed_tracks`, `reverb` and `generated_rir`: see `mix_request_for_cut` and
    `transform_request_for_cut`; `wpe`: see `transform_request_for_cut` (the "transform" route only)."""
    if len({c.sampling_rate for c in cuts}) != 1:
        return None
    if any(getattr(c, "tracks", None) is not None for c in cuts):
        route, reqs = "mix", mix_requests_for_batch(cuts, perturbed_tracks=perturbed_tracks, reverb=reverb,
                                                    generated_rir=generated_rir)
    elif any(_has_transforms(c) for c in cuts):
        route, reqs = "transform", transform_requests_for_batch(cuts, reverb=reverb, generated_rir=generated_rir, wpe=wpe)
    else:
        reqs = [slice_request_for_cut(c) for c in cuts]
        route = {PcmRequest: "pcm16", FlacRequest: "flac"}.get(type(reqs[0]))
        if any(type(r) is not type(reqs[0]) for r in reqs):
            reqs = None
    return None if route is None or reqs is None else (route, reqs)


def new_ring(route: str, pin_memory: Optional[bool] = None) -> _PinnedRing:
    """A new ring that stages the requests of `route` (one of STAGED_ROUTES), with that ring's default sizes."""
    return {"pcm16": PcmStagingRing, "flac": FlacStagingRing, "mix": MixStagingRing,
            "transform": TransformStagingRing}[route](pin_memory=pin_memory)


def is_staged_batch(staged) -> bool:
    """Whether `staged` is a batch that `staged_to_device` runs through a device stage (FLAC decode, mix or transforms)
    rather than a raw int16 / float32 buffer that it only copies."""
    return isinstance(staged, (FlacBatch, MixBatch, TransformBatch))


def staged_to_device(staged, device, ring: Optional[_PinnedRing] = None,
                     handle=None) -> Tuple[torch.Tensor, Optional[List[int]], Optional[List[int]]]:
    """The device half of any staged route on the current stream, then `ring`'s copies are marked in flight: a raw int16 or
    float32 buffer is copied as it is, a FlacBatch / MixBatch / TransformBatch goes through `decode_staged` / `mix_staged` /
    `transform_staged`.  Returns (buffer on `device`, lengths, offsets); a raw buffer's lengths and offsets are None (the
    caller has them)."""
    if isinstance(staged, FlacBatch):
        return decode_staged(staged, device, ring)
    if isinstance(staged, MixBatch):
        return mix_staged(staged, device, ring, handle=handle)
    if isinstance(staged, TransformBatch):
        return transform_staged(staged, device, ring, handle=handle)
    buf = staged.to(device, non_blocking=True)
    if ring is not None:
        ring.mark_in_flight(device)
    return buf, None, None


def collate_staged(staged, lens: Sequence[int], offsets: Sequence[int], device, ring: Optional[_PinnedRing] = None,
                   handle=None) -> torch.Tensor:
    """`staged_to_device` and then the collation kernel (csrc/collate.cuh), on `device`'s current stream: the (B, T) float32
    batch whose row b is cut b's samples and then zeros, T the longest cut, what lhotse's `collate_audio` returns for the same
    cuts (DESIGN.md §3.1o).  `lens` / `offsets` are those the ring's `stage` returned (a raw int16 buffer's; a FLAC, mix or
    transform batch brings its own)."""
    from . import engine as E

    device = torch.device(device)
    with torch.cuda.device(device):
        buf, staged_lens, staged_offsets = staged_to_device(staged, device, ring, handle=handle)
        if staged_lens is not None:
            lens, offsets = staged_lens, staged_offsets
        if buf.data_ptr() % 16:  # a view with a storage offset: the kernel reads whole vectors from the buffer's start
            buf = buf.clone()
        lens, offsets = [int(n) for n in lens], [int(o) for o in offsets]
        out = torch.empty((len(lens), max(lens, default=0)), dtype=torch.float32, device=device)
        E.collate_audio(buf, offsets, lens, out, handle=handle)
    return out
