"""
SpecAugment on the GPU as a drop-in for ``lhotse.dataset.signal_transforms.SpecAugment`` (signal_transforms.py:121-368).

lhotse draws every random number of SpecAugment on the host (Python ``random``, ``np.random`` and torch's CPU generator) and
then walks the batch one sequence at a time.  ``spec_augment_plan`` draws the same numbers in the same order and turns them
into two small tables (time warps, mask rectangles); ``b200feat_specaug`` (csrc/specaug.cuh) applies them to the whole batch
in three launches.  Same seeds, same warp points, same rectangles, same generator states afterwards.

When lhotse is importable ``B200SpecAugment`` subclasses its ``SpecAugment`` and hands it whatever the fused path declines;
otherwise a local mirror with the same constructor and ``state_dict`` is used, and a declined input raises.
"""
from __future__ import annotations

import math
import random
from typing import Any, Dict, Optional, Tuple

import numpy as np
import torch

from .engine import SPECAUG_FEATURE, SPECAUG_MASK_DTYPE, SPECAUG_TIME, SPECAUG_WARP_DTYPE, specaug

try:  # pragma: no cover - depends on the environment
    from lhotse.dataset.signal_transforms import SpecAugment as _SpecAugment

    HAVE_LHOTSE = True
except Exception:  # lhotse (or one of its hard deps) is not importable
    HAVE_LHOTSE = False

    class _SpecAugment(torch.nn.Module):  # mirrors lhotse/dataset/signal_transforms.py:121-290
        def __init__(self, time_warp_factor: Optional[int] = 80, num_feature_masks: int = 2, features_mask_size: int = 27,
                     num_frame_masks: int = 10, frames_mask_size: int = 100, max_frames_mask_fraction: float = 0.15, p=0.9):
            super().__init__()
            assert 0 <= p <= 1
            assert num_feature_masks >= 0
            assert num_frame_masks >= 0
            assert features_mask_size > 0
            assert frames_mask_size > 0
            self.time_warp_factor = time_warp_factor
            self.num_feature_masks = num_feature_masks
            self.features_mask_size = features_mask_size
            self.num_frame_masks = num_frame_masks
            self.frames_mask_size = frames_mask_size
            self.max_frames_mask_fraction = max_frames_mask_fraction
            self.p = p

        def state_dict(self, **kwargs) -> Dict[str, Any]:
            return dict(time_warp_factor=self.time_warp_factor, num_feature_masks=self.num_feature_masks,
                        features_mask_size=self.features_mask_size, num_frame_masks=self.num_frame_masks,
                        frames_mask_size=self.frames_mask_size, max_frames_mask_fraction=self.max_frames_mask_fraction, p=self.p)

        def load_state_dict(self, state_dict: Dict[str, Any]):
            for key in ("time_warp_factor", "num_feature_masks", "features_mask_size", "num_frame_masks", "frames_mask_size",
                        "max_frames_mask_fraction", "p"):
                setattr(self, key, state_dict.get(key, getattr(self, key)))


def clipped_segments(segments, B: int, T: int):
    """``supervision_segments`` as a list of (sequence, start, length clipped to T), or the reason (a string) why lhotse's
    slicing would not be a clip to [0, T): an index outside the batch, a negative start or length."""
    rows = torch.as_tensor(segments)
    if rows.dim() != 2 or rows.shape[1] != 3 or rows.is_floating_point():
        return "supervision_segments is not an (S, 3) integer tensor"
    out = []
    for b, start, num in rows.tolist():
        if not 0 <= b < B:
            return "a supervision segment names a sequence outside the batch"
        if start < 0 or num < 0:
            return "a supervision segment has a negative start or length"
        out.append((b, start, max(0, min(start + num, T) - start)))
    return out


def segments_overlap(segs) -> bool:
    """Whether two non-empty segments of one sequence share a frame (lhotse would then warp already warped frames)."""
    last: Dict[int, int] = {}
    for b, start, t in sorted(s for s in segs if s[2] > 0):
        if start < last.get(b, 0):
            return True
        last[b] = start + t
    return False


def _warp_draws(factor, t: int) -> Optional[Tuple[int, int]]:
    """time_warp's draws (signal_transforms.py:348-354) for a matrix of `t` frames: (center, warped), or None when lhotse
    returns the matrix as it is (both draws are consumed when warped == center)."""
    if t - factor <= factor + 1:
        return None
    center = np.random.randint(factor + 1, t - factor)
    warped = np.random.randint(center - factor, center + factor + 1)
    if warped == center:
        return None
    return int(center), int(warped)


def _mask_draws(mask_size, mask_times: int, extent: int):
    """mask_along_axis_optimized's draws (signal_transforms.py:316-319) with its own torch expressions, and the ranges its
    slice assignments then cover on an axis of `extent` (Python slice semantics: negative bounds wrap, empty ranges vanish)."""
    values = torch.randint(int(0), int(mask_size), (1, mask_times))
    min_values = torch.rand(1, mask_times) * (extent - values)
    starts = min_values.long().reshape(-1).tolist()
    ends = (min_values.long() + values.long()).reshape(-1).tolist()
    out = []
    for a, b in zip(starts, ends):
        a, b, _ = slice(a, b).indices(extent)
        if b > a:
            out.append((a, b))
    return out


def spec_augment_plan(params, B: int, T: int, F: int, segments=None) -> Tuple[np.ndarray, np.ndarray]:
    """The warps and mask rectangles lhotse's ``SpecAugment.forward`` would apply to a (B, T, F) batch, drawn from Python's
    ``random``, ``np.random`` and torch's CPU generator exactly as it draws them (so the three generators end in the state
    lhotse leaves them in).  `params` has SpecAugment's seven fields; `segments` is None or ``clipped_segments``' list.
    Returns (SPECAUG_WARP_DTYPE array, SPECAUG_MASK_DTYPE array) for ``engine.specaug``."""
    warps, masks = [], []

    def warp(b, start, t):
        if params.time_warp_factor is not None and params.time_warp_factor >= 1:
            cw = _warp_draws(params.time_warp_factor, t)
            if cw is not None:
                warps.append((b, start, t, cw[0], cw[1]))

    def mask(b):
        for a, e in _mask_draws(params.features_mask_size, params.num_feature_masks, F):
            masks.append((b, SPECAUG_FEATURE, a, e))
        max_tot_mask_frames = params.max_frames_mask_fraction * T
        num_frame_masks = min(params.num_frame_masks, math.ceil(max_tot_mask_frames / params.frames_mask_size))
        max_mask_frames = min(params.frames_mask_size, max_tot_mask_frames // num_frame_masks)
        for a, e in _mask_draws(max_mask_frames, num_frame_masks, T):
            masks.append((b, SPECAUG_TIME, a, e))

    if segments is None:
        for b in range(B):
            if random.random() > params.p:
                continue
            warp(b, 0, T)
            mask(b)
    else:
        for b, start, t in segments:
            if random.random() > params.p:
                continue
            warp(b, start, t)
        for b in range(B):
            if random.random() > params.p:
                continue
            mask(b)
    wt = np.zeros(len(warps), SPECAUG_WARP_DTYPE)
    wt["struct_size"] = SPECAUG_WARP_DTYPE.itemsize
    mt = np.zeros(len(masks), SPECAUG_MASK_DTYPE)
    mt["struct_size"] = SPECAUG_MASK_DTYPE.itemsize
    if warps:
        wt["seq"], wt["start"], wt["len"], wt["center"], wt["warped"] = np.asarray(warps, np.int64).T
    if masks:
        mt["seq"], mt["axis"], mt["start"], mt["end"] = np.asarray(masks, np.int64).T
    return wt, mt


class B200SpecAugment(_SpecAugment):
    """``lhotse.dataset.signal_transforms.SpecAugment`` with the batch warped and masked by the b200feat CUDA library.

    ``forward`` takes the fused path for a contiguous float32 CUDA tensor of rank 3 on an sm_90 device whose supervision
    segments (when given) do not overlap within a sequence: it returns a new tensor, enqueues its work on the current CUDA
    stream and does not synchronise.  Anything else goes to lhotse's own ``forward`` (a ``ValueError`` naming the reason where
    lhotse is not importable).  ``last_route`` is ``"fused"`` or ``"lhotse"`` after each call."""

    last_route: Optional[str] = None

    def decline_reason(self, features, segs) -> Optional[str]:
        if not isinstance(features, torch.Tensor) or features.dim() != 3:
            return "features is not a (B, T, F) tensor"
        if not features.is_cuda:
            return "features is not a CUDA tensor"
        if features.dtype != torch.float32:
            return "features is not float32"
        if not features.is_contiguous():
            return "features is not contiguous"
        if torch.cuda.get_device_capability(features.device) != (9, 0):
            return "the device is not sm_90"
        B, T, F = features.shape
        if features.numel() == 0 or T * F >= 2 ** 31:
            return "the batch is empty or too large for one call"
        if isinstance(segs, str):
            return segs
        if segs is not None and segments_overlap(segs):
            return "supervision segments of one sequence overlap"
        return None

    def forward(self, features: torch.Tensor, supervision_segments=None, *args, **kwargs) -> torch.Tensor:
        segs = None
        if supervision_segments is not None and isinstance(features, torch.Tensor) and features.dim() == 3:
            segs = clipped_segments(supervision_segments, features.shape[0], features.shape[1])
        reason = self.decline_reason(features, segs)
        if reason is not None:
            self.last_route = "lhotse"
            if not HAVE_LHOTSE:
                raise ValueError(f"B200SpecAugment: {reason}, and lhotse is not importable to take the batch")
            return super().forward(features, supervision_segments, *args, **kwargs)
        B, T, F = features.shape
        warps, masks = spec_augment_plan(self, B, T, F, segs)
        out = torch.empty_like(features)
        specaug(features, out, warps, masks)
        self.last_route = "fused"
        return out
