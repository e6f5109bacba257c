"""
H100-native counterparts of lhotse's Kaldi-family extractors, behind the unchanged
``FeatureExtractor`` API (lhotse/features/base.py:37-222):

    reference class (lhotse/features/kaldi/extractors.py)      here
    ---------------------------------------------------------------------------
    Fbank           :67   name "kaldi-fbank"                   B200Fbank           "b200-fbank"
    Mfcc            :201  name "kaldi-mfcc"                    B200Mfcc            "b200-mfcc"
    Spectrogram     :297  name "kaldi-spectrogram"             B200Spectrogram     "b200-spectrogram"
    LogSpectrogram  :407  name "kaldi-log-spectrogram"         B200LogSpectrogram  "b200-log-spectrogram"
    WhisperFbank (lhotse/features/whisper_fbank.py:103)  "whisper-fbank"    B200WhisperFbank    "b200-whisper-fbank"
    LibrosaFbank (lhotse/features/librosa_fbank.py:139)  "librosa-fbank"    B200LibrosaFbank    "b200-librosa-fbank"

Same config fields, same container rules for ``extract`` / ``extract_batch``
(extractors.py:92-132, :485-554), same ``mix`` / ``compute_energy`` / ``scale`` statics.
Deliberate differences, all documented in DESIGN.md:
  * ``extract_batch`` frames every cut on its own (ragged), so each item equals ``extract`` on that
    item; the reference zero-pads to the longest item and reflects at the *padded* end, which
    perturbs the last 1-2 frames of every shorter item (SURVEY.md §7).
  * ``dither != 0``: as in the reference (layers.py:190-193) ``dither * N(0,1)`` is added to the *waveform* before
    framing, drawn from torch's global generator — here the CUDA generator of the extractor's device, so the noise
    values differ from a CPU run (they also differ between any two reference runs that do not share a seed).
  * ``device`` must be a CUDA device; there is no CPU fallback.
  * A float tensor input that requires grad (with grad mode on) gives features with a graph back to it, as the reference's
    ``nn.Module`` chain does, for the Fbank / Mfcc / Spectrogram / LogSpectrogram classes through ``extract`` and
    ``extract_batch``: the gradient is the sm_90a backward kernel's (csrc/backward.cuh, DESIGN.md §3.1n).
"""
from __future__ import annotations

import dataclasses
import warnings
from dataclasses import asdict, dataclass
from typing import Any, Dict, List, Optional, Sequence, Tuple, Union

import numpy as np
import torch

from .base import FeatureExtractor, register_extractor
from .engine import OUT_PADDED, Engine, pack_device
from .pcm_staging import is_staged_batch, staged_to_device
from .plan import EPSILON, LOG_EPSILON, FeaturePlan, build_plan

Seconds = float
ArrayLike = Union[np.ndarray, torch.Tensor]


def _asdict_nonull(dclass) -> Dict[str, Any]:
    return {k: v for k, v in asdict(dclass).items() if v is not None}  # lhotse/utils.py asdict_nonull


class _ConfigMixin:
    def __post_init__(self):
        if getattr(self, "num_mel_bins", None) is not None:  # extractors.py:46-51
            self.num_filters = self.num_mel_bins
            self.num_mel_bins = None
        if self.snip_edges:
            warnings.warn(
                "`snip_edges` is set to True, which may cause issues in duration to num-frames conversion in Lhotse."
            )

    def to_dict(self) -> Dict[str, Any]:
        return _asdict_nonull(self)

    @classmethod
    def from_dict(cls, data: Dict[str, Any]):
        return cls(**data)


@dataclass
class B200FbankConfig(_ConfigMixin):
    """Field-for-field FbankConfig (extractors.py:24-44) with `device="cuda"` and a `kernel` knob."""

    sampling_rate: int = 16000
    frame_length: Seconds = 0.025
    frame_shift: Seconds = 0.01
    round_to_power_of_two: bool = True
    remove_dc_offset: bool = True
    preemph_coeff: float = 0.97
    window_type: str = "povey"
    dither: float = 0.0
    snip_edges: bool = False
    energy_floor: float = EPSILON
    raw_energy: bool = True
    use_energy: bool = False
    use_fft_mag: bool = False
    low_freq: float = 20.0
    high_freq: float = -400.0
    num_filters: int = 80
    num_mel_bins: Optional[int] = None  # do not use
    norm_filters: bool = False
    torchaudio_compatible_mel_scale: bool = True
    device: str = "cuda"
    kernel: str = "auto"  # auto | fast | tc | generic
    compat: str = "lhotse"  # "torchaudio": Kaldi log-energy convention + 2*pi/(L-1) blackman (TorchaudioFbank / KaldifeatFbank)
    blackman_coeff: float = 0.42  # window_type="blackman" only (kaldifeat frame_opts.blackman_coeff, kaldifeat.py:24)
    vtln_low: float = 100.0   # vtln_* : the torchaudio family's VTLN warp of the mel filter edges (fbank.py:30-32); 1.0 = off
    vtln_high: float = -500.0
    vtln_warp: float = 1.0
    htk_compat: bool = False  # kaldifeat family: energy / C0 column last (and C0 * sqrt(2) without use_energy), kaldifeat.py:158, :227


@dataclass
class B200MfccConfig(_ConfigMixin):
    """Field-for-field MfccConfig (extractors.py:156-178)."""

    sampling_rate: int = 16000
    frame_length: Seconds = 0.025
    frame_shift: Seconds = 0.01
    round_to_power_of_two: bool = True
    remove_dc_offset: bool = True
    preemph_coeff: float = 0.97
    window_type: str = "povey"
    dither: float = 0.0
    snip_edges: bool = False
    energy_floor: float = EPSILON
    raw_energy: bool = True
    use_energy: bool = False
    use_fft_mag: bool = False
    low_freq: float = 20.0
    high_freq: float = -400.0
    num_filters: int = 23
    torchaudio_compatible_mel_scale: bool = True
    num_mel_bins: Optional[int] = None  # do not use
    norm_filters: bool = False
    num_ceps: int = 13
    cepstral_lifter: int = 22
    device: str = "cuda"
    kernel: str = "auto"
    compat: str = "lhotse"  # "torchaudio": Kaldi log-energy convention, C0 <- energy (TorchaudioMfcc / KaldifeatMfcc)
    blackman_coeff: float = 0.42  # window_type="blackman" only
    vtln_low: float = 100.0   # vtln_* : the torchaudio family's VTLN warp of the mel filter edges (fbank.py:30-32); 1.0 = off
    vtln_high: float = -500.0
    vtln_warp: float = 1.0
    htk_compat: bool = False  # kaldifeat family: energy / C0 column last (and C0 * sqrt(2) without use_energy), kaldifeat.py:158, :227


@dataclass
class B200SpectrogramConfig(_ConfigMixin):
    """Field-for-field SpectrogramConfig (extractors.py:266-281)."""

    sampling_rate: int = 16000
    frame_length: Seconds = 0.025
    frame_shift: Seconds = 0.01
    round_to_power_of_two: bool = True
    remove_dc_offset: bool = True
    preemph_coeff: float = 0.97
    window_type: str = "povey"
    dither: float = 0.0
    snip_edges: bool = False
    energy_floor: float = EPSILON
    raw_energy: bool = True
    use_energy: bool = False
    use_fft_mag: bool = False
    device: str = "cuda"
    kernel: str = "auto"
    compat: str = "lhotse"  # "torchaudio" (log-spectrogram only): log(max(P, eps32)), Kaldi log-energy in bin 0 (TorchaudioSpectrogram)
    blackman_coeff: float = 0.42  # window_type="blackman" only


@dataclass
class B200LogSpectrogramConfig(B200SpectrogramConfig):
    """Field-for-field LogSpectrogramConfig (extractors.py:376-391)."""


def _first_channel_1d(x: ArrayLike) -> ArrayLike:
    """(n,) stays; (C, n) -> channel 0 (extractors.py:107-110 keeps `[0]` of the module output)."""
    if x.ndim == 1:
        return x
    if x.ndim == 2:
        return x[0]
    raise ValueError(f"expected a (n,) or (C, n) waveform, got shape {tuple(x.shape)}")


def _kernel_input(items: Sequence[ArrayLike]) -> Tuple[List[ArrayLike], bool]:
    """A batch as the kernels take it: every item (numpy array or tensor) flattened to 1-D, and `(items, pcm16)`.  An
    all-int16 batch stays int16 (the kernels widen it to x / 32768 on load); any other batch becomes float32, its int16
    items multiplied by 1/32768 here, so that an int16 item means the same waveform in either kind of batch."""
    flat = [x.reshape(-1) if isinstance(x, torch.Tensor) else np.asarray(x).reshape(-1) for x in items]
    if all(x.dtype in (torch.int16, np.int16) for x in flat):
        return flat, True
    return [_to_float32(x) for x in flat], False


def _to_float32(x: ArrayLike) -> ArrayLike:
    if isinstance(x, torch.Tensor):
        return x.to(torch.float32) * (1.0 / 32768.0) if x.dtype == torch.int16 else x.to(torch.float32)
    return x.astype(np.float32) * np.float32(1.0 / 32768.0) if x.dtype == np.int16 else x.astype(np.float32, copy=False)


_GRAD_KINDS = ("fbank", "mfcc", "spectrogram", "log-spectrogram")


class _KaldiFeatures(torch.autograd.Function):
    """Features of flat float32 waveforms with the backward kernel as their gradient.  `items` are the cuts' tensors (on
    the host or a device); one item may hold several cuts at `offs` (the rows of a (B, n) batch), several items are one cut
    each and are packed here.  The (dithered) packed device buffer is saved; the backward recomputes everything else."""

    @staticmethod
    def forward(ctx, ext, eng, lens, offs, info, *items):
        if len(items) == 1:
            buf = items[0].detach().reshape(-1).to(eng.device, non_blocking=True)
        else:
            buf, lens, offs = pack_device([x.detach().reshape(-1) for x in items], eng.device)
        buf = ext._dithered(buf).contiguous()
        if buf.data_ptr() % 16:
            buf = buf.clone()  # extract_device would copy an unaligned view; the backward must read the same buffer
        out, prefix = eng.extract_device(buf, list(lens), offsets=list(offs))
        info["prefix"] = prefix
        ctx.eng, ctx.lens, ctx.offs, ctx.prefix = eng, list(lens), list(offs), prefix
        ctx.items = [(x.shape, x.device, x.numel()) for x in items]
        ctx.save_for_backward(buf)
        return out

    @staticmethod
    def backward(ctx, grad_out):
        if torch.is_grad_enabled():
            raise RuntimeError("the b200 extractors' backward is not differentiable: double backward (create_graph=True) is "
                               "not supported")
        (buf,) = ctx.saved_tensors
        g = ctx.eng.backward_device(buf, ctx.lens, ctx.offs, grad_out, ctx.prefix)
        if len(ctx.items) == 1:
            shape, dev, numel = ctx.items[0]
            grads = [g[:numel].view(shape).to(dev)]
        else:
            grads = [g[o:o + numel].view(shape).to(dev) for o, (shape, dev, numel) in zip(ctx.offs, ctx.items)]
        return (None, None, None, None, None, *grads)


class _B200Extractor(FeatureExtractor):
    feature_kind: str = None
    _returns_cpu_tensor = False  # Spectrogram/LogSpectrogram `.cpu()` their tensor outputs (:343, :453)
    _grad = True  # the families' inner extractors keep detached outputs

    def __init__(self, config: Optional[Any] = None):
        super().__init__(config=config)
        self._engine: Optional[Engine] = None
        self._stream_eng: Optional[Engine] = None
        self._plan: Optional[FeaturePlan] = None
        self.plan  # validate the config eagerly (no CUDA needed)

    # -- lazy CUDA state (fork/spawn/pickle friendly: set.py:2166 pickles the extractor) ---------
    @property
    def plan(self) -> FeaturePlan:
        if self._plan is None:
            self._plan = build_plan(self.feature_kind, self.config)
        return self._plan

    def _new_engine(self, plan: FeaturePlan) -> Engine:
        return Engine(plan, device=self.config.device, kernel=getattr(self.config, "kernel", "auto"))

    @property
    def engine(self) -> Engine:
        if self._engine is None:
            self._engine = self._new_engine(self.plan)
        return self._engine

    def use_engine(self, engine: Engine) -> "_B200Extractor":
        """Adopts an existing handle (e.g. one created after an NCCL broadcast of the constant tables) instead of
        creating its own on first use."""
        self._plan, self._engine = engine.plan, engine
        return self

    def __getstate__(self):
        return {"config": self.config}

    def __setstate__(self, state):
        self.config = state["config"]
        self._engine = None
        self._plan = None
        self._stream_eng = None

    # -- FeatureExtractor protocol --------------------------------------------------------------
    @property
    def device(self) -> Union[str, torch.device]:
        return self.config.device

    def to(self, device: str):
        self.config.device = str(device)
        if self._engine is not None:
            self._engine.close()
            self._engine = None
        self._stream_eng = None

    @property
    def frame_shift(self) -> Seconds:
        return self.config.frame_shift

    def _check_sr(self, sampling_rate: int):
        assert sampling_rate == self.config.sampling_rate, (
            f"{type(self).__name__} was instantiated for sampling_rate "
            f"{self.config.sampling_rate}, but "
            f"sampling_rate={sampling_rate} was passed to extract(). "
            "Note you can use CutSet/RecordingSet.resample() to change the audio sampling rate."
        )

    def _dithered(self, buf: torch.Tensor) -> torch.Tensor:
        """layers.py:190-193: x + dither * randn(x.shape), on the device, from torch's global CUDA generator."""
        d = float(self.config.dither)
        if d == 0.0:
            return buf
        x = buf.to(torch.float32) * (1.0 / 32768.0) if buf.dtype == torch.int16 else buf
        return x + d * torch.randn(x.shape, device=x.device, dtype=torch.float32)

    def _wants_grad(self, items: Sequence[ArrayLike]) -> bool:
        """True when the features must carry a graph back to the float tensors `items` (the backward kernel's path)."""
        return (self._grad and self.feature_kind in _GRAD_KINDS and torch.is_grad_enabled()
                and any(isinstance(x, torch.Tensor) and x.requires_grad for x in items))

    def _extract_grad(self, items: Sequence[torch.Tensor], lens: Sequence[int], offsets: Sequence[int]):
        """`_extract_on_device` / `_extract_list_on_device` with a graph: (features, row prefix)."""
        info = {}
        out = _KaldiFeatures.apply(self, self.engine, list(lens), list(offsets), info, *items)
        return out, info["prefix"]

    def extract(self, samples: ArrayLike, sampling_rate: int) -> ArrayLike:
        self._check_sr(sampling_rate)
        (x,), _ = _kernel_input([_first_channel_1d(samples)])
        if isinstance(x, torch.Tensor):
            if self._wants_grad([x]):
                feats, _ = self._extract_grad([x], [x.numel()], [0])
                return feats.cpu() if self._returns_cpu_tensor else feats
            feats, _ = self._extract_on_device(x.contiguous(), [x.numel()], [0])
            return feats.cpu() if self._returns_cpu_tensor else feats
        if self.config.dither != 0.0:  # noise is generated on the device: take the tensor route
            feats, _ = self._extract_on_device(torch.from_numpy(np.ascontiguousarray(x)), [x.size], [0])
            return feats.cpu().numpy()
        feats, _ = self.engine.extract_host(x, [x.shape[0]])
        return feats

    def _extract_on_device(self, buf: torch.Tensor, lens: Sequence[int], offsets: Sequence[int],
                           engine: Optional[Engine] = None, ring=None, **kw):
        """Moves a staged 1-D batch to the engine's device (then marks `ring`'s copy in flight), adds the dither there and
        runs the kernels: (features, row prefix) of `Engine.extract_device`.  A staged FLAC, mix or transform batch of
        `pcm_staging` is decoded, mixed or resampled on the device into a ragged buffer first, on the same stream
        (`pcm_staging.staged_to_device`)."""
        eng = engine or self.engine
        # only the mix and transform stages use the library handle; an engine stand-in without one still takes raw buffers
        buf, staged_lens, staged_offsets = staged_to_device(buf, eng.device, ring, handle=getattr(eng, "_h", None))
        if staged_lens is not None:
            lens, offsets = staged_lens, staged_offsets
        return eng.extract_device(self._dithered(buf), list(lens), offsets=list(offsets), **kw)

    def _extract_list_on_device(self, samples: Sequence[ArrayLike], engine: Optional[Engine] = None, **kw):
        """A list of waveforms (numpy arrays or tensors, on the host or the device), packed into one device buffer."""
        eng = engine or self.engine
        flat, pcm16 = _kernel_input(samples)
        if engine is None and not kw and not pcm16 and self._wants_grad(flat):
            items = [torch.from_numpy(np.ascontiguousarray(x)) if isinstance(x, np.ndarray) else x for x in flat]
            return self._extract_grad(items, [int(x.numel()) for x in items], [0] * len(items))
        tensors = [torch.from_numpy(np.ascontiguousarray(x)) if isinstance(x, np.ndarray) else x for x in flat]
        buf, lens, offs = pack_device(tensors, eng.device, dtype=torch.int16 if pcm16 else torch.float32)
        return self._extract_on_device(buf, lens, offs, eng, **kw)

    def _extract_rows(self, samples: torch.Tensor, lengths: Optional[ArrayLike] = None):
        """A (B, n) tensor: its rows are the ragged buffer already (offset i * n; `lengths`: the samples of each row that
        belong to its cut), no packing.  Returns (features, per-row list of features)."""
        B, n = samples.shape
        lens = [n] * B
        if lengths is not None:
            lens = [int(l) for l in lengths]
            assert len(lens) == B and max(lens) <= n
        (buf,), _ = _kernel_input([samples])
        if self._wants_grad([buf]):
            out, prefix = self._extract_grad([buf], lens, [i * n for i in range(B)])
        else:
            out, prefix = self._extract_on_device(buf, lens, [i * n for i in range(B)])
        return out, [out[prefix[i]: prefix[i + 1]] for i in range(B)]

    def extract_batch(
        self,
        samples: Union[ArrayLike, Sequence[np.ndarray], Sequence[torch.Tensor]],
        sampling_rate: int,
        lengths: Optional[ArrayLike] = None,
    ) -> Union[ArrayLike, List[np.ndarray], List[torch.Tensor]]:
        """Container rules of `_extract_batch` (extractors.py:485-554)."""
        self._check_sr(sampling_rate)
        input_is_list = isinstance(samples, (list, tuple))
        input_is_torch = isinstance(samples, torch.Tensor)
        if lengths is not None:
            assert input_is_torch, "If `lengths` is provided, `samples` must be a batched and padded torch.Tensor."
            assert samples.dim() == 2
            out, result = self._extract_rows(samples, lengths)
        elif input_is_torch and samples.ndim == 2:
            out, result = self._extract_rows(samples)
        elif isinstance(samples, np.ndarray) and samples.ndim == 2 and self.config.dither == 0.0:
            # (B, n) array: handed to the C ABI host path as is (rows are back to back)
            B, nmax = samples.shape
            arr = np.ascontiguousarray(samples)
            if arr.dtype not in (np.float32, np.int16):
                arr = arr.astype(np.float32)
            if arr.nbytes >= (16 << 20) and not torch.from_numpy(arr).is_pinned():
                # pageable memory: the driver would bounce it through its own staging on ONE thread; the library's gather
                # threads copy the rows into its pinned staging instead, overlapped with the transfer
                out, prefix = self.engine.extract_host_list(list(arr), dtype=arr.dtype)
            else:
                out, prefix = self.engine.extract_host(arr.reshape(-1), [nmax] * B)
            result = [out[prefix[i]: prefix[i + 1]] for i in range(B)]
        else:
            items = list(samples) if input_is_list or samples.ndim > 1 else [samples]
            input_is_torch = any(isinstance(x, torch.Tensor) for x in items)
            if input_is_torch or self.config.dither != 0.0:  # numpy inputs with dither: device route (noise), numpy results
                out, prefix = self._extract_list_on_device(items)
                if not input_is_torch:
                    out = out.cpu().numpy()
            else:
                # the library gathers the cuts into pinned staging, every cut on a 16-byte boundary (vector-load path of
                # the kernels), overlapped with the H2D / kernel / D2H pipeline of the C call
                flat, pcm16 = _kernel_input(items)
                out, prefix = self.engine.extract_host_list(flat, dtype=np.int16 if pcm16 else np.float32)
            result = [out[prefix[i]: prefix[i + 1]] for i in range(len(items))]
        if self._returns_cpu_tensor and input_is_torch:
            result = [r.cpu() for r in result]

        # If all items are of the same shape, stack (a view of the packed buffer: no copy)
        if len(result) == 1:
            return result if input_is_list else result[0]
        if all(item.shape == result[0].shape for item in result[1:]):
            if self._returns_cpu_tensor and input_is_torch:
                return torch.stack(result, dim=0)
            return out.reshape(len(result), result[0].shape[0], result[0].shape[1])
        return result

    # -- streaming ("next", SURVEY.md §8f-4) ------------------------------------------------------
    @property
    def _stream_engine(self) -> Engine:
        """Inside a streaming buffer the frames sit at t*S with no padding, i.e. the snip_edges=True framing
        (layers.py:846-857), so streaming calls run the same kernels through a second handle built from the same
        config with snip_edges=True."""
        if getattr(self, "_stream_eng", None) is None:
            if self.plan.snip_edges:
                self._stream_eng = self.engine
            else:
                self._stream_eng = self._new_engine(build_plan(self.feature_kind, dataclasses.replace(self.config, snip_edges=True)))
        return self._stream_eng

    def online_inference(self, samples: torch.Tensor, context: Optional[torch.Tensor] = None):
        """Streaming twin of `extract_batch` for a `(B, n)` chunk: `Wav2*.online_inference` (layers.py:199-224,
        :326-333) over `_get_strided_batch_streaming` (layers.py:775-857).  `context` is the remainder returned by
        the previous call (None at the start of a recording: the left edge is reflected unless snip_edges).
        Returns `(features (B, T, F) on the device, remainder (B, r) on the device)`.  A buffer too short for one
        frame returns T = 0 and the whole buffer as remainder (the reference raises there)."""
        eng = self._stream_engine
        x = samples if isinstance(samples, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(samples))
        assert x.dim() == 2, "online_inference expects a (batch, samples) chunk"
        x = x.to(eng.device, non_blocking=True)
        if x.dtype == torch.int16:
            x = x.to(torch.float32) * (1.0 / 32768.0)
        x = self._dithered(x.to(torch.float32))  # layers.py:209-212: noise on the new chunk only
        L, S = self.plan.L, self.plan.S
        if context is None:
            if not self.plan.snip_edges:
                x = torch.cat((torch.flip(x[:, : (L - S) // 2], (1,)), x), dim=1)
        else:
            assert context.dim() == 2 and context.size(0) == x.size(0)
            x = torch.cat((context.to(eng.device, torch.float32), x), dim=1)
        B, n = x.shape
        if self.plan.snip_edges:
            T = 0 if n < L else 1 + (n - L) // S
        else:
            T = max(0, (n - (L - S)) // S)
        remainder = x[:, T * S:]
        if T == 0:
            return torch.empty((B, 0, eng.feature_dim), device=eng.device), remainder
        buf = x.contiguous().reshape(-1)
        out, prefix = eng.extract_device(buf, [n] * B, offsets=[i * n for i in range(B)])
        assert int(prefix[1]) == T
        return out.reshape(B, T, -1), remainder

    # -- extras used by the fused-collation ("next", SURVEY.md §8f-1) path -----------------------
    def affine_engine(self, scale, shift) -> Engine:
        """A second handle of the same plan whose kernels apply `v * scale[c] + shift[c]` in their epilogue (fused GlobalMVN,
        signal_transforms.py:16-58).  Pass it as `engine=` to the padded / packed batch entry points."""
        eng = self._new_engine(self.plan)
        eng.set_output_affine(scale, shift)
        return eng

    def extract_batch_padded(self, samples: Sequence[torch.Tensor], sampling_rate: int,
                             padding_value: float = LOG_EPSILON, engine: Optional[Engine] = None):
        """Ragged list -> ((B, T_max, F) padded with `padding_value`, int64 frame lengths), i.e.
        `extract_batch` + `collate_matrices(padding_value=LOG_EPSILON)` (collation.py:506-533,
        input_strategies.py:441-462) in one launch, staying on the device."""
        self._check_sr(sampling_rate)
        out, prefix = self._extract_list_on_device(samples, engine, out_mode=OUT_PADDED, pad_value=padding_value)
        return out, torch.from_numpy(np.diff(prefix)).to(torch.int64)

    def extract_batch_packed(self, samples: Sequence[ArrayLike], sampling_rate: int):
        """Ragged list -> (packed (sum T_i, F) tensor on the device, int64 row prefix [B + 1]): the kernels' native output
        layout, for callers that move the whole batch at once (lhotse_b200.storage, SURVEY.md §8f-3)."""
        self._check_sr(sampling_rate)
        out, prefix = self._extract_list_on_device(samples)
        return out, np.asarray(prefix, dtype=np.int64)

    def extract_staged_packed(self, staged: torch.Tensor, lens: Sequence[int], offsets: Sequence[int], sampling_rate: int,
                              ring=None):
        """`extract_batch_packed` for a batch already staged in ONE host buffer (the PCM16 ring, or a FLAC ring's batch; pass
        the ring as `ring` so that its next `stage()` waits for this asynchronous copy)."""
        self._check_sr(sampling_rate)
        out, prefix = self._extract_on_device(staged, lens, offsets, ring=ring)
        return out, np.asarray(prefix, dtype=np.int64)

    def extract_staged_padded(self, staged: torch.Tensor, lens: Sequence[int], offsets: Sequence[int], sampling_rate: int,
                              padding_value: float = LOG_EPSILON, ring=None, engine: Optional[Engine] = None):
        """`extract_batch_padded` for a batch that already sits in ONE (pinned) host buffer — e.g. the int16 PCM ring of
        `lhotse_b200.pcm_staging` (SURVEY.md §8f-2): one H2D copy of the raw bytes, one launch, features stay on the device."""
        self._check_sr(sampling_rate)
        assert is_staged_batch(staged) or (staged.dim() == 1 and staged.dtype in (torch.int16, torch.float32))
        out, prefix = self._extract_on_device(staged, lens, offsets, engine, ring, out_mode=OUT_PADDED, pad_value=padding_value)
        return out, torch.from_numpy(np.diff(prefix)).to(torch.int64)


@register_extractor
class B200Fbank(_B200Extractor):
    name = "b200-fbank"
    config_type = B200FbankConfig
    feature_kind = "fbank"

    def feature_dim(self, sampling_rate: int) -> int:
        return self.config.num_filters  # extractors.py:89-90 (ignores use_energy, as the reference does)

    @staticmethod
    def mix(features_a: np.ndarray, features_b: np.ndarray, energy_scaling_factor_b: float) -> np.ndarray:
        return np.log(np.maximum(EPSILON, np.exp(features_a) + energy_scaling_factor_b * np.exp(features_b)))

    @staticmethod
    def compute_energy(features: np.ndarray) -> float:
        return float(np.sum(np.exp(features)))

    @staticmethod
    def scale(features: np.ndarray, energy_scaling_factor: float) -> np.ndarray:
        return features + np.log(energy_scaling_factor)


@register_extractor
class B200Mfcc(_B200Extractor):
    name = "b200-mfcc"
    config_type = B200MfccConfig
    feature_kind = "mfcc"

    def feature_dim(self, sampling_rate: int) -> int:
        return self.config.num_ceps


@register_extractor
class B200Spectrogram(_B200Extractor):
    name = "b200-spectrogram"
    config_type = B200SpectrogramConfig
    feature_kind = "spectrogram"
    _returns_cpu_tensor = True

    def feature_dim(self, sampling_rate: int) -> int:
        return self.plan.N // 2 + 1

    @staticmethod
    def mix(features_a: np.ndarray, features_b: np.ndarray, energy_scaling_factor_b: float) -> np.ndarray:
        return features_a + energy_scaling_factor_b * features_b

    @staticmethod
    def compute_energy(features: np.ndarray) -> float:
        return float(np.sum(features))

    @staticmethod
    def scale(features: np.ndarray, energy_scaling_factor: float) -> np.ndarray:
        return energy_scaling_factor * features


@register_extractor
class B200LogSpectrogram(B200Spectrogram):
    name = "b200-log-spectrogram"
    config_type = B200LogSpectrogramConfig
    feature_kind = "log-spectrogram"


@dataclass
class B200WhisperFbankConfig:
    """WhisperFbankConfig (whisper_fbank.py:87-98: `num_filters`, `device`) plus the `kernel` knob.  The geometry is
    fixed by the reference's constructor (:107-111): 16 kHz, n_fft 400, hop 160 — class constants here, so that
    `to_dict()` stays loadable by the reference's config class once `kernel` is dropped."""

    num_filters: int = 80
    device: str = "cuda"
    kernel: str = "auto"  # auto | fast (N = 400 prime-factor kernel) | generic

    sampling_rate = 16000   # not dataclass fields: constants of the extractor
    frame_shift = 0.01
    frame_length = 0.025
    dither = 0.0
    snip_edges = False

    def to_dict(self) -> Dict[str, Any]:
        return _asdict_nonull(self)

    @classmethod
    def from_dict(cls, data: Dict[str, Any]):
        return cls(**data)


@register_extractor
class B200WhisperFbank(_B200Extractor):
    """`WhisperFbank` (whisper_fbank.py:103-184) on the fused N = 400 kernel: torch.stft(center=True) framing, periodic
    Hann window, |X|^2, librosa/Slaney mel filters, log10, clamp to the cut's maximum - 8, (x + 4) / 4, one zero row when
    `compute_num_frames_from_samples` asks for one more frame than the stft yields (:73-80).  The per-cut maximum makes it
    two launches per batch (fused kernel with an atomic per-cut max, then a 640 B/row normalise pass).
    In a batch every cut is normalised by its OWN maximum, i.e. `extract_batch(xs)[i] == extract(xs[i])` — what the
    reference's default `extract_batch` (base.py:152-222, a loop over `extract`) produces for unpadded inputs."""

    name = "b200-whisper-fbank"
    config_type = B200WhisperFbankConfig
    feature_kind = "whisper-fbank"

    def feature_dim(self, sampling_rate: int) -> int:
        return self.config.num_filters

    def extract(self, samples: ArrayLike, sampling_rate: int) -> ArrayLike:
        if samples.ndim == 2 and samples.shape[0] > 1:  # whisper_fbank.py:54-56
            raise ValueError("Whisper Fbank works only with single-channel recordings.")
        return super().extract(samples, sampling_rate)

    def online_inference(self, samples, context=None):
        raise NotImplementedError("WhisperFbank has no streaming mode (its normalisation needs the whole utterance)")

    # same statics as the reference class (whisper_fbank.py:167-184)
    mix = staticmethod(B200Fbank.mix)
    compute_energy = staticmethod(B200Fbank.compute_energy)
    scale = staticmethod(B200Fbank.scale)


@dataclass
class B200LibrosaFbankConfig:
    """Field-for-field LibrosaFbankConfig (librosa_fbank.py:16-38) + device / kernel."""

    sampling_rate: int = 22050
    fft_size: int = 1024
    hop_size: int = 256
    win_length: Optional[int] = None
    window: str = "hann"
    num_mel_bins: int = 80
    fmin: Optional[int] = 80
    fmax: Optional[int] = 7600
    device: str = "cuda"
    kernel: str = "auto"

    dither = 0.0        # not dataclass fields: the reference has no such knobs
    snip_edges = False

    def to_dict(self) -> Dict[str, Any]:
        return asdict(self)

    @classmethod
    def from_dict(cls, data: Dict[str, Any]):
        return cls(**data)


@register_extractor
class B200LibrosaFbank(_B200Extractor):
    """`LibrosaFbank` (librosa_fbank.py:139-184; the TTS-style log-mel of ParallelWaveGAN & co): centred STFT with a periodic
    window, magnitudes, Slaney mel filters between fmin and fmax, log10 — one launch of the fused kernel for the plan's
    fft_size (register-resident for 256 / 400 / 512 / 1024, generic otherwise).  librosa itself (an unpinned optional
    dependency of the reference, absent here) is restated; see oracle/librosa_oracle.py for how that is pinned."""

    name = "b200-librosa-fbank"
    config_type = B200LibrosaFbankConfig
    feature_kind = "librosa-fbank"

    @property
    def frame_shift(self) -> Seconds:
        return self.config.hop_size / self.config.sampling_rate  # librosa_fbank.py:149-151

    def feature_dim(self, sampling_rate: int) -> int:
        return self.config.num_mel_bins

    def extract(self, samples: ArrayLike, sampling_rate: int) -> ArrayLike:
        if samples.ndim == 2:  # librosa_fbank.py:101-105
            assert samples.shape[0] == 1, f"LibrosaFbank works only with single-channel recordings (shape: {samples.shape})"
        return super().extract(samples, sampling_rate)

    def online_inference(self, samples, context=None):
        raise NotImplementedError("LibrosaFbank has no streaming mode in the reference")

    mix = staticmethod(B200Fbank.mix)
    compute_energy = staticmethod(B200Fbank.compute_energy)
    scale = staticmethod(B200Fbank.scale)


_ALIASES = {
    "librosa-fbank": B200LibrosaFbank,
    "kaldi-fbank": B200Fbank, "kaldi-mfcc": B200Mfcc,
    "kaldi-spectrogram": B200Spectrogram, "kaldi-log-spectrogram": B200LogSpectrogram,
    "whisper-fbank": B200WhisperFbank,
}


def install_as_default() -> None:
    """Re-points lhotse's registry names ("kaldi-fbank", ...) at the B200 classes, so existing
    YAML configs and `Features.type` values in manifests (resolved by
    `create_default_feature_extractor`, base.py:381, used by MixedCut.load_features mixed.py:1252)
    pick the GPU implementation without editing them."""
    from .base import _REGISTRY
    from .families import FAMILY_ALIASES  # "fbank" / "mfcc" (torchaudio family), "kaldifeat-fbank" / "kaldifeat-mfcc"

    for name, cls in {**_ALIASES, **FAMILY_ALIASES}.items():
        _REGISTRY[name] = cls


def from_reference_config(cfg: Any, device: str = "cuda", sampling_rate: int = 16000):
    """Builds the matching B200 extractor from one of the reference's config objects:
      * FbankConfig / MfccConfig / SpectrogramConfig / LogSpectrogramConfig (kaldi/extractors.py) — field names identical;
      * TorchaudioFbankConfig / TorchaudioMfccConfig (fbank.py:11-39, mfcc.py:9-39) — these carry no sampling rate
        (torchaudio receives it per call), so pass `sampling_rate`;
      * KaldifeatFbankConfig / KaldifeatMfccConfig (kaldifeat.py:149-175, :218-246).
    The torchaudio / kaldifeat families map onto `compat="torchaudio"`."""
    kind = type(cfg).__name__
    table = {"FbankConfig": (B200Fbank, B200FbankConfig), "MfccConfig": (B200Mfcc, B200MfccConfig),
             "SpectrogramConfig": (B200Spectrogram, B200SpectrogramConfig),
             "LogSpectrogramConfig": (B200LogSpectrogram, B200LogSpectrogramConfig)}
    if kind in table:
        cls, ccls = table[kind]
        d = {k: v for k, v in cfg.to_dict().items() if k in ccls.__dataclass_fields__}
        d["device"] = device
        return cls(ccls(**d))
    is_mfcc = hasattr(cfg, "num_ceps")
    cls, ccls = (B200Mfcc, B200MfccConfig) if is_mfcc else (B200Fbank, B200FbankConfig)
    if hasattr(cfg, "preemphasis_coefficient"):  # torchaudio family
        d = dict(sampling_rate=sampling_rate, frame_length=cfg.frame_length, frame_shift=cfg.frame_shift,
                 round_to_power_of_two=cfg.round_to_power_of_two, remove_dc_offset=cfg.remove_dc_offset,
                 preemph_coeff=cfg.preemphasis_coefficient, window_type=cfg.window_type, dither=cfg.dither,
                 energy_floor=cfg.energy_floor, raw_energy=cfg.raw_energy, use_energy=cfg.use_energy,
                 low_freq=cfg.low_freq, high_freq=cfg.high_freq, num_filters=cfg.num_mel_bins,
                 vtln_low=getattr(cfg, "vtln_low", 100.0), vtln_high=getattr(cfg, "vtln_high", -500.0),
                 vtln_warp=getattr(cfg, "vtln_warp", 1.0))
    elif hasattr(cfg, "frame_opts"):  # kaldifeat family
        fo, mo = cfg.frame_opts, cfg.mel_opts
        if not getattr(cfg, "use_log_fbank", True):
            raise ValueError("use_log_fbank=False is not supported")
        d = dict(sampling_rate=fo.sampling_rate, frame_length=fo.frame_length, frame_shift=fo.frame_shift,
                 round_to_power_of_two=fo.round_to_power_of_two, remove_dc_offset=fo.remove_dc_offset,
                 preemph_coeff=fo.preemph_coeff, window_type=fo.window_type, dither=fo.dither, snip_edges=fo.snip_edges,
                 energy_floor=cfg.energy_floor, raw_energy=cfg.raw_energy, use_energy=cfg.use_energy,
                 low_freq=mo.low_freq, high_freq=mo.high_freq, num_filters=mo.num_bins,
                 use_fft_mag=not getattr(cfg, "use_power", True), blackman_coeff=float(getattr(fo, "blackman_coeff", 0.42)),
                 htk_compat=bool(getattr(cfg, "htk_compat", False)))
    else:
        raise ValueError(f"unsupported reference config type {kind}")
    if is_mfcc:
        d.update(num_ceps=cfg.num_ceps, cepstral_lifter=cfg.cepstral_lifter)
    d.update(device=device, compat="torchaudio")
    return cls(ccls(**d))
