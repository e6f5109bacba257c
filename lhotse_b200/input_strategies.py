"""
"Next" row §8f-1 of the scope contract: the caller right after the hot path.

``FusedOnTheFlyFeatures`` is a drop-in for ``lhotse.dataset.input_strategies.OnTheFlyFeatures``
(input_strategies.py:351-476) for the B200 extractors: same constructor arguments, same return tuple
``(feats, feat_lens, [audios, audio_lens], [cuts])``, but the ragged batch is extracted AND collated
into the padded ``(B, T_max, F)`` tensor (pad value LOG_EPSILON, collation.py:506-533) by ONE kernel
launch (`B200FEAT_OUT_PADDED`), and the features stay on the GPU for the training step instead of
bouncing through the per-cut Python copy loop of ``collate_matrices``.

Needs lhotse for audio reading (``read_audio_from_cuts``, collation.py:541); everything numeric
happens in the extractor.
"""
from __future__ import annotations

from concurrent.futures import ThreadPoolExecutor
from typing import Callable, List, Optional, Type

import torch

from .plan import LOG_EPSILON


class FusedOnTheFlyFeatures:
    def __init__(
        self,
        extractor,
        wave_transforms: Optional[List[Callable[[torch.Tensor], torch.Tensor]]] = None,
        num_workers: int = 0,
        use_batch_extract: bool = True,
        fault_tolerant: bool = False,
        return_audio: bool = False,
        executor_type: Type = ThreadPoolExecutor,
        features_on_device: bool = True,
        pcm16_fast_path: bool = True,
        global_mvn=None,
        perturbed_tracks: bool = False,
        reverb: bool = False,
    ) -> None:
        if not hasattr(extractor, "extract_batch_padded"):
            raise TypeError("FusedOnTheFlyFeatures needs a lhotse_b200 extractor (extract_batch_padded)")
        self.extractor = extractor
        self.wave_transforms = list(wave_transforms or [])
        self.num_workers = num_workers
        # same position and meaning as the reference's argument (input_strategies.py:374, :391-394): True = one sampling rate
        # per batch (asserted); False = mixed sampling rates allowed — here one launch per sampling rate instead of one
        # `extract` call per cut
        self.use_batch_extract = use_batch_extract
        self.fault_tolerant = fault_tolerant
        self.return_audio = return_audio
        self.features_on_device = features_on_device
        # §8f-2: when every cut of the batch is a plain slice of a 16-bit PCM WAV file (and nothing has to see the float
        # waveform: no wave_transforms, no return_audio), the PCM bytes go file -> pinned int16 ring -> GPU, and are
        # widened inside the kernel (bit-identical to the float route).  When every cut is a slice of a 16-bit FLAC file, the
        # compressed frames go file -> pinned byte ring -> GPU and are decoded there into the same int16 buffer ("flac").
        # When the batch holds MixedCuts of such slices (CutMix noise, padding, concatenation) and every other cut is a plain
        # slice, the tracks are staged as int16 by those rings and mixed on the GPU, bit-identical to lhotse ("mix").
        # When the batch holds speed-perturbed, volume-perturbed or resampled cuts of such files (and no MixedCut), the
        # source slices are staged as int16 and the transforms run on the GPU, bit-identical to lhotse ("transform").
        # `perturbed_tracks=True` lets the "mix" route also take MixedCut tracks (and plain cuts beside them) with such
        # transforms: the resample kernel loads them into a float32 track buffer that the mix kernels read.  It is off by
        # default so that existing pipelines keep exactly their routes; whether to turn it on by default is decided once H100
        # measurements of it exist.  `reverb=True` lets the "transform" and "mix" routes also take cuts reverberated with a
        # recorded RIR (`cut.reverb_rir`, `MixedCut.reverb_rir` with mix_first, lhotse's ReverbWithImpulseResponse cut
        # transform): the RIR is staged beside the speech and convolved on the GPU.  The float route's own FFT convolution
        # is not bit-reproducible (its bits change with the CPU and the torch thread count), so this one is held to a float32
        # tolerance of a float64 convolution instead of bit equality; it is off by default so that existing pipelines keep
        # exactly their routes and features, and whether to turn it on by default is decided once H100 measurements of it
        # exist.  `pcm16_fast_path=False` turns all staged routes off.
        self.pcm16_fast_path = pcm16_fast_path and hasattr(extractor, "extract_staged_padded")
        self.perturbed_tracks = perturbed_tracks
        self.reverb = reverb
        self._rings = {}  # route -> its staging ring, made when a batch first takes the route
        self.last_batch_route = None  # "pcm16" | "flac" | "mix" | "transform" | "float" (introspection for tests / logs)
        self._executor_type = executor_type
        self._executor = None
        # §8f-1: GlobalMVN (lhotse/dataset/signal_transforms.py:16-58) fused into the kernels' epilogue.  `global_mvn` is a
        # lhotse GlobalMVN module, a dict with "norm_means" / "norm_stds", or a (means, stds) pair; the strategy then returns
        # (features - means) / stds — padding included, exactly what GlobalMVN()(collated batch) yields — with no second pass.
        self._mvn_engine = None
        if global_mvn is not None:
            import numpy as np

            if hasattr(global_mvn, "norm_means"):
                means, stds = global_mvn.norm_means, global_mvn.norm_stds
            elif isinstance(global_mvn, dict):
                means, stds = global_mvn["norm_means"], global_mvn["norm_stds"]
            else:
                means, stds = global_mvn
            means = np.asarray(torch.as_tensor(means).detach().cpu(), dtype=np.float64)
            stds = np.asarray(torch.as_tensor(stds).detach().cpu(), dtype=np.float64)
            if not hasattr(extractor, "affine_engine"):
                raise TypeError("global_mvn needs a lhotse_b200 extractor with one sampling rate (affine_engine)")
            self._mvn_engine = extractor.affine_engine((1.0 / stds).astype(np.float32), (-means / stds).astype(np.float32))

    def _get_executor(self):
        if self.num_workers <= 0:
            return None
        if self._executor is None:
            self._executor = self._executor_type(max_workers=self.num_workers)
        return self._executor

    def _try_staged(self, cuts, recording_field):
        """(route, (features, lengths)) of a staged route, or None: the float route takes the batch."""
        if not self.pcm16_fast_path or self.wave_transforms or self.return_audio or recording_field is not None:
            return None
        from .pcm_staging import new_ring, staged_route

        chosen = staged_route(cuts, perturbed_tracks=self.perturbed_tracks, reverb=self.reverb)
        if chosen is None:
            return None  # mixed sampling rates (grouped by the float route) or a cut no staged route takes
        route, reqs = chosen
        ring = self._rings.get(route)
        if ring is None:
            ring = self._rings[route] = new_ring(route)
        try:  # a FLAC frame that does not decode raises ValueError before any feature is handed back
            staged, lens, offs, sr = ring.stage(reqs, executor=self._get_executor())
            if sr != cuts[0].sampling_rate:
                return None
            out = self.extractor.extract_staged_padded(staged, lens, offs, sr, padding_value=LOG_EPSILON, ring=ring,
                                                       **({"engine": self._mvn_engine} if self._mvn_engine is not None else {}))
        except (OSError, ValueError):
            if self.fault_tolerant:
                return None  # the float route knows how to skip broken cuts
            raise
        return route, out

    def __call__(self, cuts, recording_field: Optional[str] = None):
        from lhotse.dataset.collation import collate_vectors, read_audio_from_cuts

        fast = self._try_staged(cuts, recording_field)
        if fast is not None:
            self.last_batch_route, (feats, feat_lens) = fast
            if not self.features_on_device:
                feats = feats.cpu()
            return (feats, feat_lens) + ((cuts,) if self.fault_tolerant else ())
        self.last_batch_route = "float"

        audios, cuts = read_audio_from_cuts(
            cuts, executor=self._get_executor(), suppress_errors=self.fault_tolerant, recording_field=recording_field
        )
        for tfnm in self.wave_transforms:
            for idx in range(len(audios)):
                audios[idx] = tfnm(audios[idx])
        sr = cuts[0].sampling_rate
        if all(c.sampling_rate == sr for c in cuts):
            kw = {"engine": self._mvn_engine} if self._mvn_engine is not None else {}
            feats, feat_lens = self.extractor.extract_batch_padded(audios, sr, padding_value=LOG_EPSILON, **kw)
        else:
            assert not self.use_batch_extract, "all cuts of a batch must share one sampling rate (or pass use_batch_extract=False)"
            assert self._mvn_engine is None, "global_mvn needs one sampling rate per batch"
            feats, feat_lens = self._extract_mixed_rates(audios, [c.sampling_rate for c in cuts])
        if not self.features_on_device:
            feats = feats.cpu()
        out = (feats, feat_lens)
        if self.return_audio:
            flat = [a.squeeze(0) if a.dim() > 1 else a for a in audios]
            audio_lens = torch.tensor([a.shape[0] for a in flat], dtype=torch.int64)
            out = out + (collate_vectors(flat, padding_value=0), audio_lens)
        if self.fault_tolerant:
            out = out + (cuts,)
        return out

    def _extract_mixed_rates(self, audios, rates):
        """One padded extraction per sampling rate (needs an extractor that accepts them, e.g. the torchaudio family),
        scattered back into one (B, T_max, F) tensor in the batch's order."""
        groups = {}
        for i, r in enumerate(rates):
            groups.setdefault(int(r), []).append(i)
        parts = {r: self.extractor.extract_batch_padded([audios[i] for i in idx], r, padding_value=LOG_EPSILON)
                 for r, idx in groups.items()}
        tmax = max(int(p[0].shape[1]) for p in parts.values())
        first = next(iter(parts.values()))[0]
        feats = torch.full((len(audios), tmax, first.shape[2]), LOG_EPSILON, dtype=first.dtype, device=first.device)
        feat_lens = torch.zeros(len(audios), dtype=torch.int64)
        for r, idx in groups.items():
            f, l = parts[r]
            sel = torch.tensor(idx, dtype=torch.int64)
            feats[sel.to(feats.device), : f.shape[1]] = f
            feat_lens[sel] = l
        return feats, feat_lens

    # lhotse's BatchIO protocol (input_strategies.py:52-110): used by K2SpeechRecognitionDataset for supervisions
    def supervision_intervals(self, cuts):
        from lhotse.dataset.input_strategies import OnTheFlyFeatures

        return OnTheFlyFeatures.supervision_intervals(self, cuts)

    def supervision_masks(self, cuts, use_alignment_if_exists: Optional[str] = None):
        from lhotse.dataset.input_strategies import OnTheFlyFeatures

        return OnTheFlyFeatures.supervision_masks(self, cuts, use_alignment_if_exists)
