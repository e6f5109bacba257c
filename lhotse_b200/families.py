"""
Registry-level drop-ins for the two other config families of the same Kaldi arithmetic (SURVEY.md §8a row a2):

    reference class                                   registry name       here
    ------------------------------------------------------------------------------------------------
    TorchaudioFbank   lhotse/features/fbank.py:42      "fbank"             B200TorchaudioFbank   "b200-torchaudio-fbank"
    TorchaudioMfcc    lhotse/features/mfcc.py:42       "mfcc"              B200TorchaudioMfcc    "b200-torchaudio-mfcc"
    TorchaudioSpectrogram lhotse/features/spectrogram.py:35 "spectrogram"  B200TorchaudioSpectrogram "b200-torchaudio-spectrogram"
      (torchaudio's "spectrogram" is a LOG-power spectrum log(max(|X|^2, eps32)) whose bin 0 always carries the Kaldi
       log-energy: the log-spectrogram kernels with `log_spec_eps = -eps32` and `use_energy`)
    KaldifeatFbank    lhotse/features/kaldifeat.py:178 "kaldifeat-fbank"   B200KaldifeatFbank    "b200-kaldifeat-fbank"
    KaldifeatMfcc     lhotse/features/kaldifeat.py:249 "kaldifeat-mfcc"    B200KaldifeatMfcc     "b200-kaldifeat-mfcc"

The config dataclasses carry the reference's field names and defaults (plus `device` / `kernel`), so a YAML or a
`Features.type` written by the reference loads unchanged (`install_as_default()` re-points the registry names).  Each class
is a thin adapter over `B200Fbank` / `B200Mfcc` in `compat="torchaudio"` mode (Kaldi log-energy convention, energy
placement, 2*pi/(L-1) blackman — SURVEY.md §8a "semantic differences"); the arithmetic is the same CUDA kernels.

Family-specific behaviour kept from the reference:
  * torchaudio configs have no sampling rate — torchaudio receives it per call (base.py:408-424) — so the adapter keeps one
    inner extractor (one C-ABI handle) per sampling rate it has seen; `extract` returns numpy whatever the input type
    (base.py:421-424); `snip_edges` is always False (base.py:414).
  * kaldifeat's `extract` takes a single waveform OR a list / 2-D batch of waveforms and `extract_batch(..., lengths)`
    trims and forwards to it (kaldifeat.py:78-141); numpy in -> numpy out, tensors in -> tensors on the device.
`vtln_warp != 1` (torchaudio family) warps the mel filter edges exactly as torchaudio's `get_mel_banks` does (plan.py, bit-equal tables).
`htk_compat=True` (kaldifeat family) puts the log-energy / C0 column last (and scales C0 by sqrt(2) without `use_energy`), as Kaldi does;
pinned by tests/golden/golden_kaldi_htk_v1.npz (torchaudio's Kaldi-compatible functions with `htk_compat=True`).
Not supported (raise ValueError at construction / first use): `min_duration != 0`, `use_log_fbank=False`, `htk_mode=True`.
kaldifeat itself is an un-vendored, unpinned optional dependency (setup.py:188) that cannot be installed here: its parity
is anchored, as in the reference's own test (test/features/test_kaldifeat_features.py:103-116), on agreement with `Fbank` /
`Mfcc`; the torchaudio family is pinned by tests/golden/golden_torchaudio_v1.npz.
"""
from __future__ import annotations

from dataclasses import asdict, dataclass, field
from functools import partial
from typing import Any, Dict, Optional, Union

import numpy as np
import torch

from .base import FeatureExtractor, register_extractor
from .extractors import B200Fbank, B200LogSpectrogram, B200LogSpectrogramConfig, from_reference_config
from .plan import EPSILON, LOG_EPSILON

Seconds = float
ArrayLike = Union[np.ndarray, torch.Tensor]


# --------------------------------------------------------------------------------------------- configs
@dataclass
class B200TorchaudioFbankConfig:
    """Field-for-field TorchaudioFbankConfig (fbank.py:11-39) + device / kernel."""

    dither: float = 0.0
    window_type: str = "povey"
    frame_length: Seconds = 0.025
    frame_shift: Seconds = 0.01
    remove_dc_offset: bool = True
    round_to_power_of_two: bool = True
    energy_floor: float = EPSILON
    min_duration: float = 0.0
    preemphasis_coefficient: float = 0.97
    raw_energy: bool = True
    low_freq: float = 20.0
    high_freq: float = -400.0
    num_mel_bins: int = 80
    use_energy: bool = False
    vtln_low: float = 100.0
    vtln_high: float = -500.0
    vtln_warp: float = 1.0
    device: str = "cuda"
    kernel: str = "auto"

    def to_dict(self) -> Dict[str, Any]:
        return asdict(self)

    @classmethod
    def from_dict(cls, data: Dict[str, Any]):
        return cls(**data)


@dataclass
class B200TorchaudioMfccConfig(B200TorchaudioFbankConfig):
    """Field-for-field TorchaudioMfccConfig (mfcc.py:9-39) + device / kernel."""

    num_mel_bins: int = 23
    cepstral_lifter: float = 22.0
    num_ceps: int = 13


@dataclass
class B200TorchaudioSpectrogramConfig:
    """Field-for-field TorchaudioSpectrogramConfig (spectrogram.py:11-31) + device / kernel."""

    dither: float = 0.0
    window_type: str = "povey"
    frame_length: Seconds = 0.025
    frame_shift: Seconds = 0.01
    remove_dc_offset: bool = True
    round_to_power_of_two: bool = True
    energy_floor: float = EPSILON
    min_duration: float = 0.0
    preemphasis_coefficient: float = 0.97
    raw_energy: bool = True
    device: str = "cuda"
    kernel: str = "auto"

    def to_dict(self) -> Dict[str, Any]:
        return asdict(self)

    @classmethod
    def from_dict(cls, data: Dict[str, Any]):
        return cls(**data)


@dataclass
class B200KaldifeatFrameOptions:
    """KaldifeatFrameOptions (kaldifeat.py:14-42), including its ms / samp_freq dict spelling."""

    sampling_rate: int = 16000
    frame_shift: Seconds = 0.01
    frame_length: Seconds = 0.025
    dither: float = 0.0
    preemph_coeff: float = 0.97
    remove_dc_offset: bool = True
    window_type: str = "povey"
    round_to_power_of_two: bool = True
    blackman_coeff: float = 0.42
    snip_edges: bool = False

    def to_dict(self) -> Dict[str, Any]:
        d = asdict(self)
        d["samp_freq"] = float(d.pop("sampling_rate"))
        d["frame_shift_ms"] = d.pop("frame_shift") * 1000.0
        d["frame_length_ms"] = d.pop("frame_length") * 1000.0
        return d

    @classmethod
    def from_dict(cls, data: Dict[str, Any]):
        data = dict(data)
        if "samp_freq" in data:
            data["sampling_rate"] = int(data.pop("samp_freq"))
        for key in ("frame_shift_ms", "frame_length_ms"):
            if key in data:
                data[key[:-3]] = data.pop(key) / 1000
        return cls(**data)


@dataclass
class B200KaldifeatMelOptions:
    """KaldifeatMelOptions (kaldifeat.py:45-59)."""

    num_bins: int = 80
    low_freq: float = 20.0
    high_freq: float = -400.0
    vtln_low: float = 100.0
    vtln_high: float = -500.0
    debug_mel: bool = False
    htk_mode: bool = False

    def to_dict(self) -> Dict[str, Any]:
        return asdict(self)

    @classmethod
    def from_dict(cls, data: Dict[str, Any]):
        return cls(**data)


class _KaldifeatConfigMixin:
    def to_dict(self) -> Dict[str, Any]:
        d = asdict(self)
        d["frame_opts"] = self.frame_opts.to_dict()
        d["mel_opts"] = self.mel_opts.to_dict()
        return d

    @classmethod
    def from_dict(cls, data: Dict[str, Any]):
        data = dict(data)
        fo = B200KaldifeatFrameOptions.from_dict(data.pop("frame_opts", {}))
        mo = B200KaldifeatMelOptions.from_dict(data.pop("mel_opts", {}))
        return cls(frame_opts=fo, mel_opts=mo, **data)


@dataclass
class B200KaldifeatFbankConfig(_KaldifeatConfigMixin):
    """KaldifeatFbankConfig (kaldifeat.py:149-175); `chunk_size` is accepted and ignored (the fused kernel has no
    per-utterance intermediate to bound)."""

    frame_opts: B200KaldifeatFrameOptions = field(default_factory=B200KaldifeatFrameOptions)
    mel_opts: B200KaldifeatMelOptions = field(default_factory=B200KaldifeatMelOptions)
    use_energy: bool = False
    energy_floor: float = EPSILON
    raw_energy: bool = True
    htk_compat: bool = False
    use_log_fbank: bool = True
    use_power: bool = True
    device: str = "cuda"
    chunk_size: Optional[int] = 100 * 60 * 20
    kernel: str = "auto"


@dataclass
class B200KaldifeatMfccConfig(_KaldifeatConfigMixin):
    """KaldifeatMfccConfig (kaldifeat.py:218-246)."""

    frame_opts: B200KaldifeatFrameOptions = field(default_factory=B200KaldifeatFrameOptions)
    mel_opts: B200KaldifeatMelOptions = field(default_factory=partial(B200KaldifeatMelOptions, num_bins=23))
    num_ceps: int = 13
    use_energy: bool = False
    energy_floor: float = EPSILON
    raw_energy: bool = True
    cepstral_lifter: float = 22.0
    htk_compat: bool = False
    device: str = "cuda"
    chunk_size: Optional[int] = 1000
    kernel: str = "auto"


# --------------------------------------------------------------------------------------------- adapters
class _FamilyExtractor(FeatureExtractor):
    """Holds the family's config and one inner B200Fbank / B200Mfcc per sampling rate."""

    def __init__(self, config: Optional[Any] = None):
        super().__init__(config=config)
        self._inner_by_sr: Dict[int, Any] = {}
        self._validate()

    def _validate(self):
        raise NotImplementedError

    def _inner(self, sampling_rate: int):
        sr = int(sampling_rate)
        inner = self._inner_by_sr.get(sr)
        if inner is None:
            inner = from_reference_config(self.config, device=str(self.config.device), sampling_rate=sr)
            inner.config.kernel = self.config.kernel
            inner._grad = False  # the torchaudio and kaldifeat families return detached features
            self._inner_by_sr[sr] = inner
        return inner

    def __getstate__(self):  # picklable for ProcessPoolExecutor callers (set.py:2166): handles are re-created lazily
        return {"config": self.config}

    def __setstate__(self, state):
        self.config = state["config"]
        self._inner_by_sr = {}

    @property
    def device(self) -> Union[str, torch.device]:
        return self.config.device

    def to(self, device: str):
        self.config.device = str(device)
        for inner in self._inner_by_sr.values():
            inner.to(device)
        self._inner_by_sr = {}

    # the batch entry points of the fused callers (input_strategies.FusedOnTheFlyFeatures, storage.compute_and_store_features_fused)
    def extract_batch_padded(self, samples, sampling_rate: int, padding_value: float = LOG_EPSILON):
        return self._inner(sampling_rate).extract_batch_padded(samples, sampling_rate, padding_value=padding_value)

    def extract_batch_packed(self, samples, sampling_rate: int):
        return self._inner(sampling_rate).extract_batch_packed(samples, sampling_rate)

    def extract_staged_padded(self, staged, lens, offsets, sampling_rate: int, padding_value: float = LOG_EPSILON, ring=None):
        return self._inner(sampling_rate).extract_staged_padded(staged, lens, offsets, sampling_rate, padding_value=padding_value,
                                                                ring=ring)

    def extract_staged_packed(self, staged, lens, offsets, sampling_rate: int, ring=None):
        return self._inner(sampling_rate).extract_staged_packed(staged, lens, offsets, sampling_rate, ring=ring)

    # log-mel energies: same statics as the reference classes (fbank.py:57-76, kaldifeat.py:196-215)
    mix = staticmethod(B200Fbank.mix)
    compute_energy = staticmethod(B200Fbank.compute_energy)
    scale = staticmethod(B200Fbank.scale)


class _TorchaudioFamily(_FamilyExtractor):
    def _validate(self):
        if self.config.min_duration != 0.0:
            raise ValueError("min_duration != 0 is not supported")
        self._inner(16000).plan  # builds the tables once: raises on bad VTLN cut-offs, bad window names, ...
        self._inner_by_sr = {}

    @property
    def frame_shift(self) -> Seconds:
        return self.config.frame_shift

    def extract(self, samples: ArrayLike, sampling_rate: int) -> np.ndarray:
        """base.py:408-424: numpy out whatever came in; (C, n) input -> channel 0 (kaldi.py `channel` default)."""
        feats = self._inner(sampling_rate).extract(samples, sampling_rate)
        return feats.cpu().numpy() if isinstance(feats, torch.Tensor) else feats

    def extract_batch(self, samples, sampling_rate: int, lengths=None):
        """Ragged batch in one launch (the reference loops over `extract`, base.py:152-222); tensors in -> tensors on
        the device, numpy in -> numpy."""
        return self._inner(sampling_rate).extract_batch(samples, sampling_rate, lengths=lengths)


@register_extractor
class B200TorchaudioFbank(_TorchaudioFamily):
    name = "b200-torchaudio-fbank"
    config_type = B200TorchaudioFbankConfig

    def feature_dim(self, sampling_rate: int) -> int:
        return self.config.num_mel_bins


@register_extractor
class B200TorchaudioMfcc(_TorchaudioFamily):
    name = "b200-torchaudio-mfcc"
    config_type = B200TorchaudioMfccConfig

    def feature_dim(self, sampling_rate: int) -> int:
        return self.config.num_ceps

    mix = staticmethod(FeatureExtractor.mix)  # undefined for cepstra, as in the reference
    compute_energy = staticmethod(FeatureExtractor.compute_energy)
    scale = staticmethod(FeatureExtractor.scale)


@register_extractor
class B200TorchaudioSpectrogram(_TorchaudioFamily):
    name = "b200-torchaudio-spectrogram"
    config_type = B200TorchaudioSpectrogramConfig

    def _inner(self, sampling_rate: int):
        sr = int(sampling_rate)
        inner = self._inner_by_sr.get(sr)
        if inner is None:
            c = self.config
            inner = B200LogSpectrogram(B200LogSpectrogramConfig(
                sampling_rate=sr, frame_length=c.frame_length, frame_shift=c.frame_shift,
                round_to_power_of_two=c.round_to_power_of_two, remove_dc_offset=c.remove_dc_offset,
                preemph_coeff=c.preemphasis_coefficient, window_type=c.window_type, dither=c.dither,
                energy_floor=c.energy_floor, raw_energy=c.raw_energy, use_energy=True,  # kaldi.py: bin 0 <- log-energy, always
                device=str(c.device), kernel=c.kernel, compat="torchaudio"))
            inner._grad = False
            self._inner_by_sr[sr] = inner
        return inner

    def extract(self, samples: ArrayLike, sampling_rate: int) -> np.ndarray:
        feats = self._inner(sampling_rate).extract(samples, sampling_rate)
        return feats.cpu().numpy() if isinstance(feats, torch.Tensor) else feats

    def feature_dim(self, sampling_rate: int) -> int:
        return self._inner(sampling_rate).plan.K  # (the reference's non-power-of-two branch, spectrogram.py:52-57, returns L)

    # log-power spectra: logsumexp mixing, spectrogram.py:60-78 — the same formulas as the log-mel statics above


class _KaldifeatFamily(_FamilyExtractor):
    def _validate(self):
        if getattr(self.config.mel_opts, "htk_mode", False):
            raise ValueError("mel_opts.htk_mode=True is not supported")
        self._inner(self.config.frame_opts.sampling_rate).plan
        self._inner_by_sr = {}

    @property
    def frame_shift(self) -> Seconds:
        return self.config.frame_opts.frame_shift

    def extract(self, samples, sampling_rate: int):
        """kaldifeat.py:87-141: one waveform, a list of waveforms, or a 2-D batch (rows = utterances)."""
        expected_sr = self.config.frame_opts.sampling_rate
        assert sampling_rate == expected_sr, (
            f"Mismatched sampling rate: extractor expects {expected_sr}, " f"got {sampling_rate}"
        )
        inner = self._inner(sampling_rate)
        if isinstance(samples, (list, tuple)):
            return inner.extract_batch(list(samples), sampling_rate)
        return inner.extract_batch(samples, sampling_rate)

    def extract_batch(self, samples, sampling_rate: int, lengths=None):
        if lengths is not None:  # kaldifeat.py:84-86
            samples = [x[: int(l)] for x, l in zip(samples, lengths)]
        return self.extract(samples=samples, sampling_rate=sampling_rate)


@register_extractor
class B200KaldifeatFbank(_KaldifeatFamily):
    name = "b200-kaldifeat-fbank"
    config_type = B200KaldifeatFbankConfig

    def feature_dim(self, sampling_rate: int) -> int:
        return self.config.mel_opts.num_bins


@register_extractor
class B200KaldifeatMfcc(_KaldifeatFamily):
    name = "b200-kaldifeat-mfcc"
    config_type = B200KaldifeatMfccConfig

    def feature_dim(self, sampling_rate: int) -> int:
        return self.config.num_ceps

    mix = staticmethod(FeatureExtractor.mix)
    compute_energy = staticmethod(FeatureExtractor.compute_energy)
    scale = staticmethod(FeatureExtractor.scale)


FAMILY_ALIASES = {
    "fbank": B200TorchaudioFbank, "mfcc": B200TorchaudioMfcc, "spectrogram": B200TorchaudioSpectrogram,
    "kaldifeat-fbank": B200KaldifeatFbank, "kaldifeat-mfcc": B200KaldifeatMfcc,
}
