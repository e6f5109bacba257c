"""
TEST INFRASTRUCTURE — NOT PRODUCT CODE.

CPU restatement (torch-CPU float32 ops, functional style) of the reference's Kaldi-style
feature-extraction hot path.  Only ``tests/``, ``__graft_entry__.smoke()`` and the
``cpu_baseline`` / ``--impl reference`` legs of ``bench.py`` may import this module; the
product (``lhotse_b200``) never does and fails loudly when its CUDA library is missing.

Why torch-CPU ops and not numpy/C: the reference path *is* a chain of ATen CPU ops
(pocketfft rfft, MKL matmul, vectorised mean/log); restating the chain with the same ops
makes the oracle bit-identical to the reference (pinned in ``tests/test_oracle_pin.py``
against the imported reference and against ``tests/golden/*.npz`` generated from it) and
makes its timing representative of the reference's CPU implementation.  A plain-C second
restatement lives in ``oracle/fbank_oracle.c``.

Reference citations (relative to the reference lhotse tree):
  frame count ............ lhotse/utils.py:424-434, lhotse/features/kaldi/layers.py:747-753
  reflect framing ........ lhotse/features/kaldi/layers.py:727-772
  DC / energy / preemph .. lhotse/features/kaldi/layers.py:151-186, :859-870
  windows ................ lhotse/features/kaldi/layers.py:921-940
  rfft / power / mag ..... lhotse/features/kaldi/layers.py:32-42
  spectrogram ............ lhotse/features/kaldi/layers.py:392-402
  log-spectrogram ........ lhotse/features/kaldi/layers.py:461-473
  mel bank (torchaudio) .. lhotse/features/kaldi/layers.py:960-1017
  mel bank (legacy) ...... lhotse/features/kaldi/layers.py:873-907
  fbank .................. lhotse/features/kaldi/layers.py:565-578
  mfcc (dct, lifter) ..... lhotse/features/kaldi/layers.py:681-724
"""
from __future__ import annotations

import math
from dataclasses import astuple, dataclass, replace
from functools import lru_cache
from typing import Optional, Tuple

import numpy as np
import torch

EPSILON = 1e-10  # lhotse/utils.py:50
LOG_EPSILON = math.log(EPSILON)  # lhotse/utils.py:51


@dataclass
class OracleConfig:
    """Union of FbankConfig / MfccConfig / SpectrogramConfig / LogSpectrogramConfig fields
    (lhotse/features/kaldi/extractors.py:24-63, :156-197, :266-293, :376-403)."""

    feature: str = "fbank"  # fbank | mfcc | spectrogram | log-spectrogram
    sampling_rate: int = 16000
    frame_length: float = 0.025
    frame_shift: float = 0.01
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
    num_filters: Optional[int] = None  # default: 80 (fbank, extractors.py:40) / 23 (mfcc, :172)
    norm_filters: bool = False
    torchaudio_compatible_mel_scale: bool = True
    num_ceps: int = 13
    cepstral_lifter: int = 22

    def __post_init__(self):
        if self.num_filters is None:
            self.num_filters = 23 if self.feature == "mfcc" else 80


# ----------------------------------------------------------------------------- integer contract
def hop_samples(frame_shift: float, sampling_rate: int) -> int:
    return round(frame_shift * sampling_rate)  # utils.py:432


def num_frames_api(num_samples: int, frame_shift: float, sampling_rate: int) -> int:
    """utils.py:424-434 — the manifest-level contract."""
    hop = hop_samples(frame_shift, sampling_rate)
    return int((num_samples + hop // 2) // hop)


def layer_sizes(cfg: OracleConfig) -> Tuple[int, int, int]:
    """(L, S, N): layers.py:114-116 (floor, not round) and :264-265."""
    L = int(math.floor(cfg.frame_length * cfg.sampling_rate))
    S = int(math.floor(cfg.frame_shift * cfg.sampling_rate))
    N = (1 if L == 0 else 2 ** (L - 1).bit_length()) if cfg.round_to_power_of_two else L
    return L, S, N


def num_frames_layer(n: int, L: int, S: int, snip_edges: bool) -> int:
    """layers.py:747-753."""
    if snip_edges:
        return 0 if n < L else 1 + (n - L) // S
    return (n + S // 2) // S


def frame_index_matrix(n: int, L: int, S: int, snip_edges: bool) -> np.ndarray:
    """Sample index feeding frame t, tap j — closed form of layers.py:753-772.

    snip_edges=False: i = t*S + j - (L-S)//2, reflected once about either end
    (i<0 -> -i-1 ; i>=n -> 2n-1-i).  Inputs too short for a single reflection are an
    error here, as they are in the reference (slice underflow / as_strided OOB).
    """
    T = num_frames_layer(n, L, S, snip_edges)
    if T <= 0:
        raise ValueError(f"input of {n} samples yields no frames")
    t = np.arange(T, dtype=np.int64)[:, None]
    j = np.arange(L, dtype=np.int64)[None, :]
    if snip_edges:
        return t * S + j
    left = (L - S) // 2
    right = (T - 1) * S + L - n - left
    if left > n or right > n:
        raise ValueError(f"input of {n} samples is too short for reflect padding ({left},{right})")
    i = t * S + j - left
    i = np.where(i < 0, -i - 1, i)
    i = np.where(i >= n, 2 * n - 1 - i, i)
    return i


# ----------------------------------------------------------------------------- tables
def make_window(L: int, window_type: str, dtype=torch.float32) -> torch.Tensor:
    """layers.py:921-940 (note: blackman uses 2*pi/L, unlike torchaudio)."""
    if window_type == "hanning":
        return torch.hann_window(L, periodic=False, dtype=dtype)
    if window_type == "hamming":
        return torch.hamming_window(L, periodic=False, alpha=0.54, beta=0.46, dtype=dtype)
    if window_type == "povey":
        return torch.hann_window(L, periodic=False, dtype=dtype).pow(0.85)
    if window_type == "rectangular":
        return torch.ones(L, dtype=dtype)
    if window_type == "blackman":
        a = 2 * math.pi / L
        k = torch.arange(L, dtype=dtype)
        return 0.42 - 0.5 * torch.cos(a * k) + (0.5 - 0.42) * torch.cos(2 * a * k)
    raise ValueError(f"Invalid window type: {window_type}")


def _lin2mel(x):
    return 1127.0 * np.log(1 + x / 700)  # layers.py:943 (np.log dispatches to torch.log for tensors)


def make_mel_bank(cfg: OracleConfig, N: int) -> torch.Tensor:
    """(K=N/2+1, M) float32 filterbank exactly as Wav2LogFilterBank builds ``_fb``
    (layers.py:541-563)."""
    M, sr = cfg.num_filters, cfg.sampling_rate
    if cfg.torchaudio_compatible_mel_scale:
        assert M > 3 and N % 2 == 0
        num_fft_bins = N / 2
        nyquist = 0.5 * sr
        hi = cfg.high_freq + nyquist if cfg.high_freq <= 0.0 else cfg.high_freq
        lo = cfg.low_freq
        assert 0.0 <= lo < nyquist and 0.0 < hi <= nyquist and lo < hi
        bin_width = sr / N
        mel_lo, mel_hi = _lin2mel(lo), _lin2mel(hi)
        delta = (mel_hi - mel_lo) / (M + 1)
        b = torch.arange(M).unsqueeze(1)
        left = mel_lo + b * delta
        center = mel_lo + (b + 1.0) * delta
        right = mel_lo + (b + 2.0) * delta
        mel = _lin2mel(bin_width * torch.arange(num_fft_bins)).unsqueeze(0)
        up = (mel - left) / (center - left)
        down = (right - mel) / (right - center)
        bank = torch.max(torch.zeros(1), torch.min(up, down))  # (M, N/2)
        return torch.nn.functional.pad(bank, (0, 1), mode="constant", value=0).T  # transposed *view*, as in the reference (affects the BLAS path for tiny T)
    # legacy scale, layers.py:873-907
    hi = cfg.high_freq
    if hi is None or hi == 0:
        hi = sr / 2
    if hi < 0:
        hi = sr / 2 + hi
    melfc = np.linspace(_lin2mel(cfg.low_freq), _lin2mel(hi), M + 2)
    mels = _lin2mel(np.linspace(0, sr, N))
    B = np.zeros((int(N / 2 + 1), M), dtype=np.float32)
    for k in range(M):
        l, c, r = melfc[k], melfc[k + 1], melfc[k + 2]
        for j in range(int(N / 2)):
            mj = mels[j]
            if l < mj < r:
                B[j, k] = (mj - l) / (c - l) if mj <= c else (r - mj) / (r - c)
    if cfg.norm_filters:
        B = B / np.sum(B, axis=0, keepdims=True)
    return torch.from_numpy(B)


def make_dct(num_ceps: int, num_filters: int) -> torch.Tensor:
    """layers.py:697-706."""
    n = torch.arange(float(num_filters)).unsqueeze(1)
    k = torch.arange(float(num_ceps))
    dct = torch.cos(math.pi / float(num_filters) * (n + 0.5) * k)
    dct[:, 0] *= 1.0 / math.sqrt(2.0)
    dct *= math.sqrt(2.0 / float(num_filters))
    return dct


def make_lifter(num_ceps: int, Q: int) -> Optional[torch.Tensor]:
    """layers.py:681-695."""
    if Q == 0:
        return None
    return 1 + 0.5 * Q * torch.sin(math.pi * torch.arange(num_ceps, dtype=torch.float32) / Q)


# ----------------------------------------------------------------------------- arithmetic
def _log_energy(frames: torch.Tensor, floor: float) -> torch.Tensor:
    """layers.py:859-870."""
    e = (frames.pow(2).sum(-1) + 1e-15).log()
    if floor > 0.0:
        e = torch.max(e, torch.tensor(math.log(floor), dtype=e.dtype))
    return e


def _frames_view(x: torch.Tensor, L: int, S: int, snip_edges: bool) -> torch.Tensor:
    """Overlapping-frame view of the (reflect-padded) waveform — the cheap formulation the reference
    uses (layers.py:753-772: flip/cat then a strided view); `frame_index_matrix` is its closed form
    and tests assert the two agree."""
    n = x.numel()
    T = num_frames_layer(n, L, S, snip_edges)
    if T <= 0:
        raise ValueError(f"input of {n} samples yields no frames")
    if not snip_edges:
        left = (L - S) // 2
        right = (T - 1) * S + L - n - left
        if left > n or right > n:
            raise ValueError(f"input of {n} samples is too short for reflect padding ({left},{right})")
        parts = [x[:left].flip(0), x]
        if right > 0:
            parts.append(x[n - right:].flip(0))
        x = torch.cat(parts)
    return x.unfold(0, L, S)[:T]


def windowed_frames(x: torch.Tensor, cfg: OracleConfig):
    """(n,) waveform -> ((T, N) zero-padded windowed frames, optional (T,) log-energy).
    layers.py:151-186 applied to the gather of layers.py:727-772."""
    assert cfg.dither == 0.0, "oracle is deterministic: dither must be 0"
    L, S, N = layer_sizes(cfg)
    f = _frames_view(x, L, S, cfg.snip_edges)  # (T, L) strided view, == x[frame_index_matrix(...)]
    if cfg.remove_dc_offset:
        f = f - torch.mean(f, dim=1, keepdim=True)
    log_e = None
    if cfg.use_energy and cfg.raw_energy:
        log_e = _log_energy(f, cfg.energy_floor)
    if cfg.preemph_coeff != 0.0:
        prev = torch.cat((f[:, :1], f[:, :-1]), dim=1)  # replicate-left
        f = f - cfg.preemph_coeff * prev
    f = f * _cached_tables(astuple(cfg), x.dtype)[0]
    if N != L:
        f = torch.nn.functional.pad(f, (0, N - L))
    if cfg.use_energy and not cfg.raw_energy:
        log_e = _log_energy(f, cfg.energy_floor)
    return f, log_e


@lru_cache(maxsize=64)
def _cached_tables(cfg_key, dtype):
    """The reference builds its tables once, in the module constructors (layers.py:117-119, :541-563,
    :673-680); cache them per config so that timing this oracle is representative."""
    cfg = OracleConfig(*cfg_key)
    L, S, N = layer_sizes(cfg)
    win = make_window(L, cfg.window_type, dtype=dtype)
    fb = dct = lifter = None
    if cfg.feature in ("fbank", "mfcc"):
        fb = make_mel_bank(cfg, N)  # keeps the reference's transposed-view layout
        fb = fb if fb.dtype == dtype else fb.to(dtype)
    if cfg.feature == "mfcc":
        dct = make_dct(cfg.num_ceps, cfg.num_filters).to(dtype)
        lifter = make_lifter(cfg.num_ceps, cfg.cepstral_lifter)
        lifter = None if lifter is None else lifter.to(dtype)
    return win, fb, dct, lifter


def extract(x, cfg: OracleConfig, dtype=torch.float32) -> np.ndarray:
    """One cut -> (T, F) features. ``dtype=torch.float64`` gives the high-precision truth."""
    x = torch.as_tensor(np.asarray(x)).reshape(-1).to(dtype)
    L, S, N = layer_sizes(cfg)
    frames, log_e = windowed_frames(x, cfg)
    X = torch.fft.rfft(frames, dim=-1)
    spec = X.abs() if cfg.use_fft_mag else X.abs() ** 2  # layers.py:38-42
    feat = cfg.feature
    if feat == "spectrogram":
        out = spec
        if log_e is not None:
            out[:, 0] = log_e
    elif feat == "log-spectrogram":
        out = (spec + 1e-15).log()
        if log_e is not None:
            out[:, 0] = log_e
    elif feat in ("fbank", "mfcc"):
        _, fb, dct_t, lifter_t = _cached_tables(astuple(cfg), dtype)
        eps = torch.tensor(torch.finfo(torch.float).eps, dtype=dtype)
        # the reference multiplies a (1, T, K) batch (layers.py:571); keep the leading dim so the
        # same BLAS path (and rounding) is taken for tiny T
        mel = torch.max(torch.matmul(spec.unsqueeze(0), fb), eps).log().squeeze(0)
        if feat == "fbank":
            out = mel if log_e is None else torch.cat((log_e.unsqueeze(-1), mel), dim=-1)
        else:
            out = torch.matmul(mel.unsqueeze(0), dct_t).squeeze(0)
            if lifter_t is not None:
                out = out * lifter_t
            if log_e is not None:
                # layers.py:722 writes `mfcc[:, 0] = log_e` on a 3-D tensor (broken upstream for
                # batched input); the intended Kaldi semantics — C0 <- log-energy — is restated here.
                out[:, 0] = log_e
    else:
        raise ValueError(feat)
    return out.numpy()


def stream_num_frames(num_samples: int, L: int, S: int, snip_edges: bool) -> int:
    """Frames that a streaming call emits from a buffer of `num_samples` (= carried remainder + new chunk, plus the
    reflected left pad on the very first call): layers.py:838-844."""
    if snip_edges:
        return 0 if num_samples < L else 1 + (num_samples - L) // S
    return max(0, (num_samples - (L - S)) // S)


def online_inference(chunk, cfg: OracleConfig, context=None, dtype=torch.float32):
    """Streaming twin of `extract` for one channel: `Wav2*.online_inference` (layers.py:199-224, :326-333) over
    `_get_strided_batch_streaming` (layers.py:775-857).  `context` is the remainder returned by the previous call
    (None at the start of a recording).  Returns ((T, F) features, remainder waveform)."""
    x = torch.as_tensor(np.asarray(chunk)).reshape(-1).to(dtype)
    L, S, _ = layer_sizes(cfg)
    if context is None:
        if not cfg.snip_edges:
            x = torch.cat((x[: (L - S) // 2].flip(0), x))  # layers.py:826-830
    else:
        x = torch.cat((torch.as_tensor(np.asarray(context)).reshape(-1).to(dtype), x))  # layers.py:834
    T = stream_num_frames(x.numel(), L, S, cfg.snip_edges)
    remainder = x[T * S:].numpy()
    if T == 0:
        F = extract(np.zeros(L, dtype=np.float32), replace(cfg, snip_edges=True)).shape[1]
        return np.zeros((0, F), dtype=remainder.dtype), remainder
    # inside the buffer the frames sit at t*S with no padding: exactly the snip_edges=True framing (layers.py:848-857)
    feats = extract(x[: (T - 1) * S + L], replace(cfg, snip_edges=True), dtype=dtype)
    return feats, remainder
