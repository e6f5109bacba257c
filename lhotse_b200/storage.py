"""
"Next" row §8f-3 of the scope contract: the caller right AFTER the hot path — feature storage fed from the device.

The reference's batch path (`CutSet.compute_and_store_features_batch`, lhotse/cut/set.py:2197-2408) hands the extractor one
ragged batch and then, per cut: `.cpu().numpy()` (a D2H copy each), `feats_writer.write(cut.id, feat_mat)` (a file or an
archive entry each), a `Features` manifest, `validate_features`.  With the extraction itself at thousands of hours per
second that per-cut tail is the whole cost.  Here the batch leaves the GPU as ONE packed `(sum T_i, F)` matrix (the layout
the kernels write), crosses PCIe once into pinned memory and is appended to ONE archive file with a single `write`;
the per-cut bookkeeping is reduced to building the manifests.

  * `B200ArchiveWriter` / `B200ArchiveReader` — storage backend "b200_archive": an append-only file of raw little-endian
    float32 rows; a storage key is "byte offset,rows,cols", so a reader slices frames without any index.  They implement
    lhotse's `FeaturesWriter` / `FeaturesReader` interfaces (features/io.py:26-176) and register in its backend registries
    (io.py:283-313) when lhotse is importable: `Features.load`, `cut.load_features()`, partial reads all work unchanged.
  * `compute_and_store_features_fused(cuts, extractor, storage_path, ...)` — the counterpart of
    `compute_and_store_features_batch` (same arguments where they apply, same resumable manifest writer, same `Features`
    fields, PaddingCut / MixedCut handling as set.py:2306-2362) on top of `extract_batch_packed`, the PCM16 ring of
    `pcm_staging` when the cuts allow it, and `write_batch`.
Not built: a lilcom-compatible quantiser (`LilcomChunkyWriter`, io.py:982): lilcom is an un-vendored optional dependency that
cannot be installed here, so its bit format could not be pinned; the archive is lossless float32 instead.
"""
from __future__ import annotations

import os
from concurrent.futures import ThreadPoolExecutor
from pathlib import Path
from typing import List, Optional, Sequence

import numpy as np
import torch

try:  # pragma: no cover - depends on the environment
    from lhotse.features.io import FeaturesReader, FeaturesWriter, register_reader, register_writer

    HAVE_LHOTSE_IO = True
except Exception:
    HAVE_LHOTSE_IO = False
    FeaturesReader = FeaturesWriter = object

    def register_reader(cls):
        return cls

    def register_writer(cls):
        return cls


ARCHIVE_SUFFIX = ".b200feat"


def _archive_path(storage_path) -> str:
    p = str(storage_path)
    return p if p.endswith(ARCHIVE_SUFFIX) else p + ARCHIVE_SUFFIX


@register_writer
class B200ArchiveWriter(FeaturesWriter):
    """Append-only archive of float32 feature matrices.  `mode="w"` truncates, `"a"` appends (keys stay valid: they are
    absolute byte offsets).  One `write_batch` = one `write` system call for the whole batch."""

    name = "b200_archive"

    def __init__(self, storage_path, mode: str = "w", *args, **kwargs):
        assert mode in ("w", "a"), mode
        self._path = _archive_path(storage_path)
        Path(self._path).parent.mkdir(parents=True, exist_ok=True)
        self._f = open(self._path, "wb" if mode == "w" else "ab")
        self._pos = self._f.seek(0, os.SEEK_END)

    @property
    def storage_path(self) -> str:
        return self._path

    def write(self, key: str, value: np.ndarray) -> str:
        value = np.ascontiguousarray(value, dtype="<f4")
        if value.ndim != 2:
            raise ValueError(f"b200_archive stores (frames, features) matrices, got shape {value.shape}")
        off = self._pos
        if value.size:  # (memoryview cannot cast an empty matrix)
            self._f.write(memoryview(value).cast("B"))
        self._pos += value.nbytes
        return f"{off},{value.shape[0]},{value.shape[1]}"

    def write_batch(self, keys: Sequence[str], packed: np.ndarray, row_prefix: Sequence[int]) -> List[str]:
        """`packed`: (sum T_i, F) float32 with cut i in rows row_prefix[i]:row_prefix[i+1] (what `extract_batch_packed`
        returns after ONE device-to-host copy).  Appends it with a single write and returns the per-cut storage keys."""
        packed = np.ascontiguousarray(packed, dtype="<f4")
        assert packed.ndim == 2 and len(row_prefix) == len(keys) + 1 and int(row_prefix[-1]) == packed.shape[0]
        base, F = self._pos, packed.shape[1]
        if packed.size:
            self._f.write(memoryview(packed).cast("B"))
        self._pos += packed.nbytes
        return [f"{base + int(row_prefix[i]) * F * 4},{int(row_prefix[i + 1]) - int(row_prefix[i])},{F}" for i in range(len(keys))]

    def flush(self):
        self._f.flush()

    def close(self):
        if not self._f.closed:
            self._f.close()

    def __enter__(self):
        return self

    def __exit__(self, *args, **kwargs):
        self.close()


@register_reader
class B200ArchiveReader(FeaturesReader):
    name = "b200_archive"

    def __init__(self, storage_path, *args, **kwargs):
        self._path = _archive_path(storage_path)
        self._fd = None

    def _file(self):
        if self._fd is None:
            self._fd = os.open(self._path, os.O_RDONLY)
        return self._fd

    def read(self, key: str, left_offset_frames: int = 0, right_offset_frames: Optional[int] = None) -> np.ndarray:
        off, rows, cols = (int(v) for v in key.split(","))
        hi = rows if right_offset_frames is None else min(rows, right_offset_frames)
        lo = max(0, left_offset_frames)
        n = max(0, hi - lo)
        out = np.empty((n, cols), dtype=np.float32)
        if n:
            view, got, pos = memoryview(out).cast("B"), 0, off + lo * cols * 4
            while got < len(view):
                k = os.preadv(self._file(), [view[got:]], pos + got)
                if k <= 0:
                    raise IOError(f"{self._path}: short read at {pos + got}")
                got += k
        return out

    def __del__(self):
        try:
            if self._fd is not None:
                os.close(self._fd)
        except Exception:
            pass


def register_with_lhotse() -> bool:
    """(Re-)registers the archive backend in lhotse's reader / writer registries (io.py:283-313).  Done at import when lhotse
    is importable; callable later for processes where lhotse only became importable after this module was loaded."""
    try:
        from lhotse.features.io import READER_BACKENDS, WRITER_BACKENDS
    except Exception:
        return False
    WRITER_BACKENDS[B200ArchiveWriter.name] = B200ArchiveWriter
    READER_BACKENDS[B200ArchiveReader.name] = B200ArchiveReader
    return True


def _features_dict(fm) -> dict:
    """`asdict_nonull(Features)` (lhotse/utils.py:166) without the generic dataclass recursion: same keys, same order."""
    d = {"type": fm.type, "num_frames": fm.num_frames, "num_features": fm.num_features, "frame_shift": fm.frame_shift,
         "sampling_rate": fm.sampling_rate, "start": fm.start, "duration": fm.duration, "storage_type": fm.storage_type,
         "storage_path": fm.storage_path, "storage_key": fm.storage_key, "recording_id": fm.recording_id, "channels": fm.channels}
    return {k: v for k, v in d.items() if v is not None}


def _plain_json(v) -> bool:
    """True for values `dataclasses.asdict` copies verbatim: str / int / float / bool / None and lists, tuples, str-keyed dicts of them."""
    t = type(v)
    if v is None or t in (str, int, float, bool):
        return True
    if t in (list, tuple):
        return all(_plain_json(x) for x in v)
    if t is dict:
        return all(type(k) is str and _plain_json(x) for k, x in v.items())
    return False


class _ManifestLines:
    """JSON lines for the cuts manifest.  A plain `MonoCut` over a one-source recording — what a corpus job writes by the
    million — is serialised field by field (the dict equals `cut.to_dict()`, lhotse/cut/data.py:90-98; tests/test_next_rows.py
    checks it), with the recording's dict built once per recording instead of twice per cut; everything else goes through the
    cut's own `to_dict()`."""

    def __init__(self):
        from lhotse.cut import MonoCut
        from lhotse.utils import asdict_nonull

        self._mono = MonoCut
        self._asdict = asdict_nonull
        self._recs = {}

    def _recording_dict(self, rec):
        src = rec.sources
        if rec.transforms is None and len(src) == 1 and isinstance(src[0].source, str):
            key = (rec.id, rec.sampling_rate, rec.num_samples, rec.duration, src[0].type, src[0].source, tuple(src[0].channels),
                   tuple(rec.channel_ids) if rec.channel_ids is not None else None)
            d = self._recs.get(key)
            if d is None:
                if len(self._recs) > 4096:
                    self._recs.clear()
                d = self._recs[key] = rec.to_dict()
            return d
        return rec.to_dict()

    def cut_dict(self, cut, fm) -> dict:
        """The manifest entry of `fastcopy(cut, features=fm)`."""
        # `custom` is usually None or the sampler's {"dataloading_info": {...}} (plain values, copied verbatim by asdict)
        if type(cut) is self._mono and cut.recording is not None and (cut.custom is None or _plain_json(cut.custom)):
            d = {"id": cut.id, "start": cut.start, "duration": cut.duration, "channel": cut.channel,
                 "supervisions": [self._asdict(s) for s in cut.supervisions], "features": _features_dict(fm),
                 "recording": self._recording_dict(cut.recording)}
            if cut.custom is not None:
                d["custom"] = cut.custom
            d["type"] = "MonoCut"
            return d
        from lhotse.utils import fastcopy

        return fastcopy(cut, features=fm).to_dict()


def compute_and_store_features_fused(
    cuts,
    extractor,
    storage_path,
    manifest_path=None,
    batch_duration: float = 600.0,
    num_workers: int = 4,
    overwrite: bool = False,
    pcm16_fast_path: bool = True,
    perturbed_tracks: bool = False,
    reverb: bool = False,
):
    """`CutSet.compute_and_store_features_batch(extractor, storage_path, manifest_path, batch_duration, num_workers,
    overwrite=...)` (lhotse/cut/set.py:2197-2408) with the batch kept whole from the GPU to the disk: one packed
    extraction, one D2H copy, one archive append per batch.  Returns the CutSet with `Features` attached (lazy when
    `manifest_path` is given, resumable exactly like the reference: cut ids already in the manifest are skipped).

    Three stages run concurrently, one batch apart: a reader thread samples the next batch and fills a pinned PCM ring
    (`num_workers` file readers), the calling thread moves it through the GPU, a writer thread appends the packed features
    to the archive and then writes the batch's manifest lines (in this order, so an entry never precedes its data).

    `perturbed_tracks=True` lets the "mix" stage also take MixedCuts whose tracks carry Speed / Volume / Resample chains
    (`pcm_staging.mix_request_for_cut`).  It is off by default so that existing calls keep exactly their routes, until H100
    measurements of it decide the default.  `reverb=True` lets the "transform" and "mix" stages also take cuts reverberated
    with a recorded RIR (`pcm_staging.transform_request_for_cut`, `mix_request_for_cut`); off by default because those
    samples match the float route within a float32 tolerance, not bit for bit (the float route's own convolution is not
    bit-reproducible), until H100 measurements of it decide the default."""
    import json
    import queue
    import threading

    from lhotse import CutSet
    from lhotse.cut import MixedCut, MonoCut, PaddingCut
    from lhotse.cut.data import DataCut
    from lhotse.dataset.collation import read_audio_from_cuts
    from lhotse.dataset.sampling import SimpleCutSampler
    from lhotse.features.base import Features
    from lhotse.qa import validate_features
    from lhotse.utils import fastcopy

    from .pcm_staging import STAGED_ROUTES, new_ring, staged_route

    register_with_lhotse()
    frame_shift = extractor.frame_shift
    cuts_writer = CutSet.open_writer(manifest_path, overwrite=overwrite)
    sampler = SimpleCutSampler(cuts, max_duration=batch_duration, world_size=1, rank=0)  # this rank's shard already: no second split under torch.distributed
    sampler.filter(lambda cut: cut.id not in cuts_writer.ignore_ids)
    use_ring = pcm16_fast_path and hasattr(extractor, "extract_staged_packed")
    pool = ThreadPoolExecutor(max_workers=num_workers) if num_workers > 0 else None
    lines = _ManifestLines()
    to_file = getattr(cuts_writer, "file", None) is not None or manifest_path is not None

    def _save(batch_cuts, feats: np.ndarray, prefix, keys):
        out = []
        for i, cut in enumerate(batch_cuts):
            rows = int(prefix[i + 1] - prefix[i])
            if isinstance(cut, PaddingCut):  # set.py:2307-2318: manifest fields only
                out.append(fastcopy(cut, num_frames=rows, num_features=feats.shape[1], frame_shift=frame_shift))
                continue
            fm = Features(
                start=cut.start, duration=cut.duration, type=extractor.name, num_frames=rows, num_features=feats.shape[1],
                frame_shift=frame_shift, sampling_rate=cut.sampling_rate, channels=cut.channel,
                storage_type=writer.name, storage_path=str(writer.storage_path), storage_key=keys[i],
            )
            validate_features(fm, feats_data=feats[prefix[i]: prefix[i + 1]])
            if isinstance(cut, MixedCut):  # set.py:2344-2361
                fm.recording_id = cut.id
                out.append(MonoCut(id=cut.id, start=0, duration=cut.duration, channel=0,
                                   supervisions=[fastcopy(s, recording_id=cut.id, channel=0) for s in cut.supervisions],
                                   features=fm, recording=None))
                continue
            if isinstance(cut, DataCut):
                fm.recording_id = cut.recording_id
            out.append(lines.cut_dict(cut, fm) if to_file else fastcopy(cut, features=fm))
        if to_file:
            # one write and one flush per BATCH (the reference prints and flushes per cut, set.py:2340: with a gzip manifest every
            # flush is a sync block); the archive was flushed before, so a manifest entry still never precedes its data
            cuts_writer._maybe_open()
            cuts_writer.file.write("".join(json.dumps(m if isinstance(m, dict) else m.to_dict(), ensure_ascii=False) + "\n" for m in out))
            cuts_writer.file.flush()
        else:
            for m in out:
                cuts_writer.write(m)

    failure = []  # first exception of a helper thread, re-raised by the caller
    # the free rings of each staged route: stage 1 takes one per batch, stage 2 hands it back once its H2D copy has completed
    free_rings = {route: queue.Queue() for route in STAGED_ROUTES}
    stop = threading.Event()
    cuda_index = None  # the GPU this call works on, resolved in the calling thread ("cuda" without an index = its current device)
    try:
        dev = torch.device(str(getattr(getattr(extractor, "config", None), "device", "cpu")))
        if dev.type == "cuda" and torch.cuda.is_available():
            cuda_index = dev.index if dev.index is not None else torch.cuda.current_device()
    except (RuntimeError, TypeError, ValueError):
        cuda_index = None

    def _bind_thread():  # a new thread starts on device 0: pinned allocations / event waits must use this rank's GPU
        if cuda_index is not None:
            torch.cuda.set_device(cuda_index)

    def _staged_batches():  # stage 1: sampler + PCM staging (or the reference's audio loading when the cuts are not plain PCM16 WAV)
        for batch in sampler:
            if stop.is_set():
                return
            batch_cuts = list(batch)
            if not batch_cuts:
                continue
            sr = batch_cuts[0].sampling_rate
            assert all(c.sampling_rate == sr for c in batch_cuts)
            item = None
            chosen = staged_route(batch_cuts, perturbed_tracks=perturbed_tracks, reverb=reverb) if use_ring else None
            if chosen is not None:
                kind, reqs = chosen
                free = free_rings[kind]
                ring = free.get()  # handed back by stage 2 once the batch's host-to-device copy has completed
                staged, lens, offs, fsr = ring.stage(reqs, executor=pool)
                if fsr == sr:
                    item = (kind, batch_cuts, sr, ring, staged, lens, offs)
                else:
                    free.put(ring)
            if item is None:
                audios, batch_cuts = read_audio_from_cuts(batch_cuts, executor=pool)
                if not batch_cuts:
                    continue
                item = ("audio", batch_cuts, sr, audios)
            yield item

    def _extract(item):  # stage 2: the GPU
        if item[0] in free_rings:
            _, batch_cuts, sr, ring, staged, lens, offs = item
            packed, prefix = extractor.extract_staged_packed(staged, lens, offs, sr, ring=ring)
        else:
            _, batch_cuts, sr, audios = item
            ring = None
            packed, prefix = extractor.extract_batch_packed(audios, sr)
        # ONE device-to-host copy of the batch, into pinned memory when there is a GPU
        if isinstance(packed, torch.Tensor):
            if packed.is_cuda:
                host = torch.empty(packed.shape, dtype=torch.float32, pin_memory=True)
                host.copy_(packed, non_blocking=False)
                packed = host
            packed = packed.numpy()
        if ring is not None:
            free_rings[item[0]].put(ring)  # the blocking copy above ordered the batch's H2D copy before this point
        return batch_cuts, packed, prefix

    def _store(batch_cuts, packed, prefix):  # stage 3: archive append, then the manifest
        keys = writer.write_batch([c.id for c in batch_cuts], packed, prefix)
        writer.flush()  # a manifest entry must never precede its data (resume after a crash skips what the manifest lists)
        _save(batch_cuts, packed, prefix, keys)

    pipelined = os.environ.get("B200FEAT_STORE_PIPELINE", "1") != "0"
    with cuts_writer, B200ArchiveWriter(storage_path, mode="w" if overwrite else "a") as writer:
        if use_ring:
            for _ in range(2 if pipelined else 1):
                for route in STAGED_ROUTES:
                    free_rings[route].put(new_ring(route))
        if not pipelined:  # stage 1 and 2 in the calling thread, stage 3 one batch behind in a saver thread
            with ThreadPoolExecutor(max_workers=1) as saver:
                futures = [saver.submit(_store, *_extract(item)) for item in _staged_batches()]
                for f in futures:
                    f.result()
        else:
            staged_q = queue.Queue(maxsize=1)
            store_q = queue.Queue(maxsize=2)

            def _reader():
                try:
                    _bind_thread()
                    for item in _staged_batches():
                        staged_q.put(item)
                except BaseException as e:  # noqa: BLE001 - handed to the caller
                    failure.append(e)
                finally:
                    staged_q.put(None)

            def _writer_loop():
                try:
                    _bind_thread()
                    while True:
                        item = store_q.get()
                        if item is None:
                            return
                        if not failure:
                            _store(*item)
                except BaseException as e:  # noqa: BLE001
                    failure.append(e)
                    while store_q.get() is not None:  # keep stage 2 from blocking on a full queue
                        pass

            t_read = threading.Thread(target=_reader, name="b200feat-reader", daemon=True)
            t_write = threading.Thread(target=_writer_loop, name="b200feat-writer", daemon=True)
            t_read.start()
            t_write.start()
            try:
                while True:
                    item = staged_q.get()
                    if item is None or failure:
                        break
                    store_q.put(_extract(item))
            except BaseException as e:  # noqa: BLE001
                failure.append(e)
            finally:
                stop.set()
                store_q.put(None)
                t_write.join()
                while t_read.is_alive():  # unblock a reader waiting for a ring or for room in the queue
                    try:
                        staged_q.get(timeout=0.05)
                    except queue.Empty:
                        pass
                    for route in STAGED_ROUTES:
                        if use_ring and free_rings[route].empty():
                            free_rings[route].put(new_ring(route, pin_memory=False))
                t_read.join()
    if pool is not None:
        pool.shutdown()
    if failure:
        raise failure[0]
    return cuts_writer.open_manifest()
