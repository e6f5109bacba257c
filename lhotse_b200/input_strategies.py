"""
"Next" row §8f-1 of the scope contract: the caller right after the hot path.  ``FusedAudioSamples`` (below) is the same for
lhotse's ``AudioSamples``: the padded waveform batch of models that hold their front end, built on the GPU.

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
        generated_rir: bool = False,
        wpe: bool = False,
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
        # exist.  `generated_rir=True` does the same for cuts whose RIR lhotse generates (no RIR corpus): the generator's
        # random numbers are drawn on the host from the same generators in the same order, the RIRs are built on the GPU
        # (DESIGN.md §3.1l); it is a separate flag so that `reverb=True` pipelines keep exactly their routes.  `wpe=True`
        # lets the "transform" route also take cuts whose chain ends in lhotse's DereverbWPE (`cuts.dereverb_wpe()`, after
        # Speed / Volume / Resample and a reverb or not): the dereverberation runs on the GPU (DESIGN.md §3.1q) within a
        # float32 tolerance of a float64 restatement, not bit for bit, so it is off by default too.
        # `pcm16_fast_path=False` turns all staged routes off.
        self.pcm16_fast_path = pcm16_fast_path and hasattr(extractor, "extract_staged_padded")
        self.perturbed_tracks = perturbed_tracks
        self.reverb = reverb
        self.generated_rir = generated_rir
        self.wpe = wpe
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
        from .pcm_staging import new_ring, staged_route, undo_draws

        chosen = staged_route(cuts, perturbed_tracks=self.perturbed_tracks, reverb=self.reverb,
                              generated_rir=self.generated_rir, wpe=self.wpe)
        if chosen is None:
            return None  # mixed sampling rates (grouped by the float route) or a cut no staged route takes
        route, reqs = chosen
        ring = self._rings.get(route)
        if ring is None:
            ring = self._rings[route] = new_ring(route)
        staged = None
        try:  # a FLAC frame that does not decode raises ValueError before any feature is handed back
            staged, lens, offs, sr = ring.stage(reqs, executor=self._get_executor())
            if sr != cuts[0].sampling_rate:
                undo_draws(staged)  # the float route draws the generated RIRs again
                return None
            out = self.extractor.extract_staged_padded(staged, lens, offs, sr, padding_value=LOG_EPSILON, ring=ring,
                                                       **({"engine": self._mvn_engine} if self._mvn_engine is not None else {}))
        except (OSError, ValueError):
            undo_draws(staged)
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


class FusedAudioSamples:
    """lhotse's ``AudioSamples`` (same constructor and call) with the waveform batch built on the GPU.  A batch that a staged
    route takes (``pcm_staging.staged_route``: PCM16 WAV or FLAC slices, MixedCuts of them, speed / volume / resample
    transforms, reverb with ``reverb`` / ``generated_rir``) is staged without padding cuts, made on the device by that route
    and collated by one kernel (csrc/collate.cuh): ``(audio, audio_lens)`` equal to ``collate_audio``'s, audio (B, T) float32
    on the current CUDA device (``audio_on_device=False``: on the CPU), (B, 1, T) with ``mono_downmix=False``, audio_lens int32
    on the CPU (DESIGN.md §3.1o).  Other batches go to lhotse's ``collate_audio`` with the same arguments
    (``last_batch_route == "reference"``, the reason in ``last_decline``); the staged ones name their route in
    ``last_batch_route``."""

    def __init__(
        self,
        num_workers: int = 0,
        fault_tolerant: bool = False,
        executor_type: Type = ThreadPoolExecutor,
        use_batch_loader: bool = False,
        ais_force_individual: bool = False,
        mono_downmix: Optional[bool] = None,
        audio_on_device: bool = True,
        perturbed_tracks: bool = False,
        reverb: bool = False,
        generated_rir: bool = False,
        wpe: bool = False,
    ) -> None:
        self.num_workers = num_workers
        self.fault_tolerant = fault_tolerant
        self._executor_type = executor_type
        self._executor = None
        self.mono_downmix = mono_downmix
        self.use_batch_loader = use_batch_loader
        self.ais_batch_loader = None
        if use_batch_loader:  # as AudioSamples: AIStore fetches the whole batch, which then takes lhotse's collate_audio
            from lhotse.ais import AISBatchLoader

            self.ais_batch_loader = AISBatchLoader(force_individual=ais_force_individual, skip_failed_fetches=fault_tolerant)
        self.audio_on_device = audio_on_device
        # the staged routes' options, as in FusedOnTheFlyFeatures (off by default for the same reasons)
        self.perturbed_tracks = perturbed_tracks
        self.reverb = reverb
        self.generated_rir = generated_rir
        self.wpe = wpe
        self._rings = {}  # route -> its staging ring, made when a batch first takes the route
        self.last_batch_route = None  # one of pcm_staging.STAGED_ROUTES | "reference"
        self.last_decline = None

    def _get_executor(self):
        if self.num_workers <= 0:
            return None
        if self._executor is None:
            self._executor = self._executor_type(max_workers=self.num_workers)
        return self._executor

    def _decline_reason(self, cuts, recording_field) -> Optional[str]:
        if recording_field is not None:
            return "recording_field is set"
        if self.use_batch_loader:
            return "use_batch_loader is set"
        if any(type(c).__name__ == "MultiCut" or (getattr(c, "num_channels", 1) or 1) > 1 for c in cuts):
            return "a MultiCut or multi-channel cut"
        if len({c.sampling_rate for c in cuts}) > 1:
            return "more than one sampling rate"
        return None

    def _try_staged(self, cuts):
        """(route, (B, T) audio on the current CUDA device) of a staged route, or a str: why lhotse takes the batch."""
        from .pcm_staging import collate_staged, new_ring, staged_route, undo_draws

        chosen = staged_route(cuts, perturbed_tracks=self.perturbed_tracks, reverb=self.reverb,
                              generated_rir=self.generated_rir, wpe=self.wpe)
        if chosen is None:
            return "a cut that no staged route takes"
        route, reqs = chosen
        ring = self._rings.get(route)
        if ring is None:
            ring = self._rings[route] = new_ring(route)
        staged = None
        try:  # a read or a FLAC frame that fails raises before any audio is handed back
            staged, lens, offs, sr = ring.stage(reqs, executor=self._get_executor())
            if sr != cuts[0].sampling_rate:
                undo_draws(staged)  # lhotse draws the generated RIRs again
                return "the staged sampling rate is not the cuts'"
            audio = collate_staged(staged, lens, offs, torch.device("cuda", torch.cuda.current_device()), ring)
        except (OSError, ValueError) as e:
            undo_draws(staged)  # lhotse draws the generated RIRs again
            if self.fault_tolerant:
                return f"a staged read or decode failed: {e}"
            raise
        return route, audio

    def __call__(self, cuts, recording_field: Optional[str] = None):
        reason = self._decline_reason(cuts, recording_field)
        fast = reason or self._try_staged(cuts)
        if isinstance(fast, str):
            return self._reference(cuts, recording_field, fast)
        self.last_batch_route, audio = fast
        self.last_decline = None
        if self.mono_downmix is False:  # mono cuts in channel 0 of a (B, 1, T) batch, as collate_audio expands them
            audio = audio.unsqueeze(1)
        if not self.audio_on_device:
            audio = audio.cpu()
        audio_lens = torch.tensor([c.num_samples for c in cuts], dtype=torch.int32)
        if not self.fault_tolerant:
            return audio, audio_lens
        # collate_audio hands back the cuts it read: the batch padded to its longest duration
        from lhotse import CutSet

        padded = CutSet.from_cuts(cuts).pad(duration=max(c.duration for c in cuts), direction="right", preserve_id=True)
        return audio, audio_lens, padded

    def _reference(self, cuts, recording_field, reason: str):
        from lhotse.dataset.collation import collate_audio

        self.last_batch_route, self.last_decline = "reference", reason
        if self.use_batch_loader and self.ais_batch_loader is not None:
            cuts = self.ais_batch_loader(cuts)
        out = collate_audio(cuts, executor=self._get_executor(), fault_tolerant=self.fault_tolerant,
                            recording_field=recording_field, mono_downmix=self.mono_downmix)
        if self.audio_on_device:
            out = (out[0].to(torch.device("cuda", torch.cuda.current_device())),) + tuple(out[1:])
        return out

    # lhotse's BatchIO protocol (input_strategies.py): used by K2SpeechRecognitionDataset for supervisions
    def supervision_intervals(self, cuts):
        from lhotse.dataset.input_strategies import AudioSamples

        return AudioSamples.supervision_intervals(self, cuts)

    def supervision_masks(self, cuts, use_alignment_if_exists: Optional[str] = None):
        from lhotse.dataset.input_strategies import AudioSamples

        return AudioSamples.supervision_masks(self, cuts, use_alignment_if_exists)
