"""
Precomputed features collated and mixed on the GPU: a drop-in for lhotse's ``PrecomputedFeatures`` input strategy
(lhotse/dataset/input_strategies.py) over features stored in the ``b200_archive`` backend (storage.py).

lhotse's ``collate_features`` (dataset/collation.py) pads the batch with ``cuts.pad(...)`` and calls ``cut.load_features()``
once per cut: an archive read per track, NumPy exp / log over every frame of every CutMix track (``MixedCut.load_features``,
cut/mixed.py, and its ``FeatureMixer``, features/mixer.py), a CPU tensor at the end.  Here:

  * `precomputed_plan(cuts)` restates that as two tables: the row reads and mix steps ``load_features`` would perform, with
    lhotse's own ``cuts.pad`` making the padding tracks;
  * `FeatureStagingRing` reads every track's rows into one pinned float32 buffer (one ``preadv`` per track through the
    shared descriptor cache of pcm_staging), which crosses PCIe in one copy;
  * `b200feat_feature_mix` (csrc/featmix.cuh) computes the energies, the SNR gains, the mix and the padded (B, T_max, F)
    batch on the device;
  * `FusedPrecomputedFeatures` ties them together and hands a batch the tables cannot describe to lhotse's
    ``collate_features`` (route "reference").

The numeric contract is DESIGN.md §3.1m.
"""
from __future__ import annotations

import math
from concurrent.futures import ThreadPoolExecutor
from dataclasses import dataclass
from typing import List, Optional, Tuple, Type, Union

import numpy as np
import torch

from . import engine as E
from .engine import _aligned_offsets
from .pcm_staging import _for_each, _PinnedRing, _pread, _stamp
from .plan import LOG_EPSILON
from .storage import B200ArchiveReader, _archive_path


def mix_laws() -> dict:
    """The extractor classes whose ``mix`` / ``compute_energy`` / ``scale`` statics the kernels restate, with their law
    (engine.FEATMIX_LOG or engine.FEATMIX_LINEAR).  Looked up at call time: the classes are those the registry resolves now."""
    from . import extractors as ex
    from . import families as fam

    laws = {cls: E.FEATMIX_LOG for cls in (ex.B200Fbank, ex.B200WhisperFbank, ex.B200LibrosaFbank, fam.B200TorchaudioFbank,
                                           fam.B200TorchaudioSpectrogram, fam.B200KaldifeatFbank)}
    laws.update({cls: E.FEATMIX_LINEAR for cls in (ex.B200Spectrogram, ex.B200LogSpectrogram)})
    try:
        from lhotse.features.kaldi.extractors import Fbank, LogSpectrogram, Spectrogram
    except ImportError:
        return laws
    laws.update({Fbank: E.FEATMIX_LOG, Spectrogram: E.FEATMIX_LINEAR, LogSpectrogram: E.FEATMIX_LINEAR})
    return laws


def _compute_num_frames(duration: float, frame_shift: float, sampling_rate: int) -> int:
    """lhotse.utils.compute_num_frames."""
    num_samples = round(duration * sampling_rate)
    window_hop = round(frame_shift * sampling_rate)
    return int((num_samples + window_hop // 2) // window_hop)


@dataclass
class _Rows:
    """What ``cut.load_features()`` returns for a MonoCut or a PaddingCut: `stored` rows read from `path` at byte `pos`
    (0 for a constant), `num_rows` rows in all (stored or stored + 1, the last one repeated)."""
    path: Optional[str]
    pos: int
    stored: int
    num_rows: int
    cols: int
    value: float = 0.0


def _rows(cut) -> Union[_Rows, str]:
    from lhotse.cut import MonoCut, PaddingCut

    if isinstance(cut, PaddingCut):  # PaddingCut.load_features: float32 ones * feat_value
        return _Rows(None, 0, 0, int(cut.num_frames), int(cut.num_features), float(np.float32(cut.feat_value)))
    if type(cut) is not MonoCut:
        return f"{type(cut).__name__} track (multi-channel or nested cuts are lhotse's)"
    fm = cut.features
    if fm is None:
        return "a cut without features"
    if fm.storage_type != B200ArchiveReader.name:
        return f"features stored in {fm.storage_type!r}, not {B200ArchiveReader.name!r}"
    # Features.load(start=cut.start, duration=cut.duration) (features/base.py)
    if cut.start < fm.start - 1e-3:
        return "a cut starting before its features (lhotse raises)"
    left = 0
    if not math.isclose(cut.start, fm.start):
        left = _compute_num_frames(cut.start - fm.start, fm.frame_shift, fm.sampling_rate)
    right = left + _compute_num_frames(cut.duration, fm.frame_shift, fm.sampling_rate)
    off, rows, cols = (int(v) for v in fm.storage_key.split(","))
    lo, hi = max(0, left), min(rows, right)  # B200ArchiveReader.read's clamping
    n = max(0, hi - lo)
    # MonoCut.load_features: one row too many is dropped, one too few repeats the last one
    nf = cut.num_frames
    stored, num = n, n
    if n - nf == 1:
        stored = num = nf
    elif n - nf == -1 and n > 0:
        num = n + 1
    return _Rows(_archive_path(fm.storage_path), off + lo * cols * 4, stored, num, cols)


@dataclass
class PrecomputedPlan:
    """The batch as the kernels take it: `tracks` / `cuts` (engine.FEATMIX_TRACK_DTYPE / FEATMIX_CUT_DTYPE; a track's
    `src_elem` is set when it is staged), `reads[k] = (track, path, byte position, elements)`, the output's (T, F), and
    `lens`, the cuts' frame counts before padding (int32, as collate_features makes them)."""
    tracks: np.ndarray
    cuts: np.ndarray
    reads: List[Tuple[int, str, int, int]]
    T: int
    F: int
    lens: torch.Tensor


class _Tables:
    def __init__(self):
        self.tracks, self.cuts, self.reads = [], [], []

    def track(self, c: int, r: _Rows, flags: int, offset: int = 0, snr=None) -> None:
        t = len(self.tracks)
        self.tracks.append((np.dtype(E.FEATMIX_TRACK_DTYPE).itemsize, c, flags, r.stored, r.num_rows, offset, r.value, 0, 0,
                            math.nan if snr is None else 10.0 ** (-snr / 10)))
        if r.stored > 0:
            self.reads.append((t, r.path, r.pos, r.stored * r.cols))


def _plan_mixed(tab: _Tables, c: int, cut, F: int) -> Optional[str]:
    """Appends the tables of a MixedCut's ``load_features()`` (cut/mixed.py); a reason when they cannot describe it."""
    from lhotse.cut import PaddingCut
    from lhotse.cut.mixed import _get_audible_tracks, _get_snr_reference_track
    from lhotse.features.base import get_extractor_type

    tracks = _get_audible_tracks(cut)
    first = tracks[0]
    rows = [_rows(t.cut) for t in tracks]
    for r in rows:
        if isinstance(r, str):
            return r
        if r.cols != F:
            return "tracks of different feature dimensions (lhotse raises)"
    first_track = len(tab.tracks)
    if first.snr is None and tracks[1:] and all(isinstance(t.cut, PaddingCut) for t in tracks[1:]):
        # the padding-only branch: the first track's rows, then tracks[1]'s feat_value
        if rows[0].num_rows != first.cut.num_frames or cut.num_frames < rows[0].num_rows:
            return "a padding-only cut whose rows do not fill its first track (lhotse raises)"
        tab.track(c, rows[0], E.FEATMIX_MIXED)
        tab.cuts.append((np.dtype(E.FEATMIX_CUT_DTYPE).itemsize, E.FEATMIX_COPY, 0, cut.num_frames, 0, first_track, 1, 0,
                         float(np.float32(tracks[1].cut.feat_value)), 0))
        return None
    _, ref = _get_snr_reference_track(cut)
    cls = get_extractor_type(ref.cut.features_type)
    law = mix_laws().get(cls)
    if law is None:
        return f"no mix law for {cls.__name__}"
    ref_is_first = ref is first
    tab.track(c, rows[0], E.FEATMIX_MIXED | (E.FEATMIX_ENERGY if ref_is_first or first.snr is not None else 0), 0, first.snr)
    ref_k = 0 if ref_is_first else None
    mix_rows = rows[0].num_rows
    frame_shift = first.cut.frame_shift
    for t, r in zip(tracks[1:], rows[1:]):
        is_ref = t is ref
        if r.num_rows == 0:  # add_to_mix returns early; a reference still gives its (zero) energy
            if is_ref:
                ref_k = len(tab.tracks) - first_track
                tab.track(c, r, E.FEATMIX_ENERGY)
            continue
        if t.offset < 0:
            return "a negative track offset (lhotse asserts)"
        off = _compute_num_frames(t.offset, frame_shift, t.cut.sampling_rate) if t.offset > 0 else 0
        if is_ref:
            ref_k = len(tab.tracks) - first_track
        tab.track(c, r, E.FEATMIX_MIXED | (E.FEATMIX_ENERGY if is_ref or t.snr is not None else 0), off, t.snr)
        mix_rows = max(mix_rows, off + r.num_rows)
    if ref_k is None:  # a muted reference: its energy sets the gains, its rows are not mixed
        r = _rows(ref.cut)
        if isinstance(r, str):
            return r
        if r.cols != F:
            return "tracks of different feature dimensions (lhotse raises)"
        ref_k = len(tab.tracks) - first_track
        tab.track(c, r, E.FEATMIX_ENERGY)
    nf = cut.num_frames
    if abs(mix_rows - nf) > 1 or (nf > 0 and mix_rows == 0):
        return "a mix more than one frame away from its cut (lhotse asserts)"
    tab.cuts.append((np.dtype(E.FEATMIX_CUT_DTYPE).itemsize, E.FEATMIX_MIX, law, nf, mix_rows, first_track,
                     len(tab.tracks) - first_track, ref_k, 0.0, 0))
    return None


def precomputed_plan(cuts, pad_direction: str = "right") -> Union[PrecomputedPlan, str]:
    """The tables of ``collate_features(cuts, pad_direction)``, or the reason (a str) why the batch is left to it: features
    outside the b200_archive backend, multi-channel features or a MultiCut, a mix law outside `mix_laws()`, a pad direction
    other than "right", or a cut lhotse itself would refuse."""
    from lhotse.cut import MixedCut, MonoCut, PaddingCut

    if pad_direction != "right":
        return f"pad_direction={pad_direction!r}"
    cuts = list(cuts)
    if not cuts:
        return "an empty batch"
    if not all(c.has_features for c in cuts):
        return "a cut without features"
    for c in cuts:
        if not isinstance(c, (MonoCut, MixedCut, PaddingCut)):
            return f"{type(c).__name__} (multi-channel features are lhotse's)"
    from lhotse import CutSet

    lens = torch.tensor([c.num_frames for c in cuts], dtype=torch.int)
    padded = list(CutSet.from_cuts(cuts).pad(num_frames=int(lens.max()), direction="right"))
    T, F = int(padded[0].num_frames), int(padded[0].num_features)
    tab = _Tables()
    try:
        for c, cut in enumerate(padded):
            if cut.num_frames != T:
                return "cuts of different lengths after padding (lhotse raises)"
            if isinstance(cut, MixedCut):
                why = _plan_mixed(tab, c, cut, F)
                if why is not None:
                    return why
                continue
            r = _rows(cut)
            if isinstance(r, str):
                return r
            if r.cols != F or r.num_rows != T:
                return "a cut whose rows do not fill the batch (lhotse raises)"
            first_track = len(tab.tracks)
            tab.track(c, r, E.FEATMIX_MIXED)
            tab.cuts.append((np.dtype(E.FEATMIX_CUT_DTYPE).itemsize, E.FEATMIX_COPY, 0, T, 0, first_track, 1, 0, 0.0, 0))
    except (AttributeError, ValueError, AssertionError) as e:  # lhotse raises these for cuts it cannot load
        return f"lhotse refuses the cut: {e}"
    return PrecomputedPlan(np.array(tab.tracks, dtype=E.FEATMIX_TRACK_DTYPE), np.array(tab.cuts, dtype=E.FEATMIX_CUT_DTYPE),
                           tab.reads, T, F, lens)


class FeatureStagingRing(_PinnedRing):
    """Grow-only pinned float32 buffer holding a plan's stored rows, every track starting on a 16-byte boundary."""

    ALIGN = 4

    def __init__(self, initial_elems: int = 1 << 20, pin_memory: Optional[bool] = None):
        super().__init__(pin_memory)
        self._buf = torch.empty(int(initial_elems), dtype=torch.float32, pin_memory=self._pin)

    def stage(self, plan: PrecomputedPlan, executor=None) -> Tuple[torch.Tensor, np.ndarray]:
        """Reads every track's rows (one preadv each, on `executor`'s threads) -> (buffer view, the track table with each
        track's `src_elem`)."""
        self._wait_idle()
        offs, total = _aligned_offsets([n for _, _, _, n in plan.reads], self.ALIGN)
        self._buf = self._grown(self._buf, total)
        view = self._buf.numpy()
        stamps = {path: _stamp(path) for _, path, _, _ in plan.reads}
        tracks = plan.tracks.copy()
        for (t, _, _, _), o in zip(plan.reads, offs):
            tracks["src_elem"][t] = o

        def one(k):
            _, path, pos, n = plan.reads[k]
            _pread(path, stamps[path], memoryview(view[offs[k]: offs[k] + n]).cast("B"), pos)

        _for_each(len(plan.reads), one, executor)
        return self._buf[:total], tracks


def stage_and_mix(plan: PrecomputedPlan, ring: FeatureStagingRing, device, executor=None) -> torch.Tensor:
    """The device half of a plan: its rows staged by `ring`, one H2D copy, the kernels -> the (B, T, F) float32 batch on
    `device` (asynchronous on its current stream)."""
    staged, tracks = ring.stage(plan, executor)
    with torch.cuda.device(device):
        src = None
        if staged.numel():
            src = staged.to(device, non_blocking=True)
            ring.mark_in_flight(device)
        out = torch.empty((len(plan.cuts), plan.T, plan.F), dtype=torch.float32, device=device)
        E.feature_mix(src, tracks, plan.cuts, out, LOG_EPSILON)
    return out


class FusedPrecomputedFeatures:
    """lhotse's ``PrecomputedFeatures`` (same constructor and call) for features in the b200_archive backend: the batch's
    stored rows reach the GPU in one copy and are mixed, scaled and padded there (DESIGN.md §3.1m).  Returns
    ``(features, lens)``: (B, T_max, F) float32 on the current CUDA device (on the CPU with ``features_on_device=False``) and
    int32 lengths.  A batch `precomputed_plan` declines goes to lhotse's ``collate_features`` (``last_batch_route ==
    "reference"``, its reason in ``last_decline``); the others take ``"archive"``."""

    def __init__(self, num_workers: int = 0, executor_type: Type = ThreadPoolExecutor, features_on_device: bool = True) -> None:
        self.num_workers = num_workers
        self._executor_type = executor_type
        self._executor = None
        self.features_on_device = features_on_device
        self._ring = None
        self.last_batch_route = None  # "archive" | "reference"
        self.last_decline = None

    def _get_executor(self):
        if self.num_workers <= 0:
            return None
        if self._executor is None:
            self._executor = self._executor_type(max_workers=self.num_workers)
        return self._executor

    def __call__(self, cuts, pad_direction: Optional[str] = "right") -> Tuple[torch.Tensor, torch.Tensor]:
        plan = precomputed_plan(cuts, pad_direction)
        if isinstance(plan, str):
            from lhotse.dataset.collation import collate_features

            self.last_batch_route, self.last_decline = "reference", plan
            feats, lens = collate_features(cuts, pad_direction=pad_direction, executor=self._get_executor())
            return (feats.to(torch.device("cuda", torch.cuda.current_device())) if self.features_on_device else feats), lens
        self.last_batch_route, self.last_decline = "archive", None
        if self._ring is None:
            self._ring = FeatureStagingRing()
        feats = stage_and_mix(plan, self._ring, torch.device("cuda", torch.cuda.current_device()), self._get_executor())
        return (feats if self.features_on_device else feats.cpu()), plan.lens

    # lhotse's BatchIO protocol (input_strategies.py): used by K2SpeechRecognitionDataset for supervisions
    def supervision_intervals(self, cuts, pad_direction: Optional[str] = "right"):
        from lhotse.dataset.input_strategies import PrecomputedFeatures

        return PrecomputedFeatures.supervision_intervals(self, cuts, pad_direction)

    def supervision_masks(self, cuts, use_alignment_if_exists: Optional[str] = None, pad_direction: Optional[str] = "right"):
        from lhotse.dataset.input_strategies import PrecomputedFeatures

        return PrecomputedFeatures.supervision_masks(self, cuts, use_alignment_if_exists, pad_direction)
