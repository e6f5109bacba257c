"""
TEST INFRASTRUCTURE — NOT PRODUCT CODE.

CPU restatement (torch-CPU ops) of the reference's Whisper log-mel path, `WhisperFbank.extract`
(lhotse/features/whisper_fbank.py:138-165) -> `log_mel_spectrogram` (:16-84).  Same rules as
``oracle/kaldi_oracle.py``: only ``tests/``, ``__graft_entry__.smoke()`` and the CPU legs of
``bench.py`` may import it.

Pinned: ``tests/test_whisper.py::test_whisper_oracle_bit_identical_to_live_reference`` runs the
imported reference class (build container) and ``test_whisper_oracle_matches_golden`` checks the
committed vectors ``tests/golden/golden_whisper_v1.npz`` (made by ``make_golden_whisper.py`` from
the real reference).  One third-party piece is NOT in the reference tree: the mel filter table comes
from ``librosa.filters.mel`` (whisper_fbank.py:117-120; librosa is an unpinned optional dependency,
absent from this image).  `slaney_mel_filters` restates its published algorithm; it is pinned
bit-for-bit against ``transformers.audio_utils.mel_filter_bank(norm="slaney", mel_scale="slaney")``
(present in this image; upstream tests that function against librosa), and the golden vectors were
generated with the reference's own code running on that transformers table.

Reference citations (relative to the reference lhotse tree):
  constants (16 kHz, n_fft 400, hop 160, periodic Hann) ... lhotse/features/whisper_fbank.py:107-123
  centred STFT, last frame dropped ....................... lhotse/features/whisper_fbank.py:62-63
  mel, log10, clamp to max - 8, (x + 4) / 4 ............... lhotse/features/whisper_fbank.py:65-69
  zero row up to compute_num_frames_from_samples ......... lhotse/features/whisper_fbank.py:71-80, lhotse/utils.py:424-434
"""
from __future__ import annotations

from functools import lru_cache

import numpy as np
import torch

SAMPLING_RATE, N_FFT, HOP = 16000, 400, 160


def _hz_to_mel(f):
    """Slaney (Auditory Toolbox) mel scale: linear below 1 kHz (200/3 Hz per mel), logarithmic above."""
    f = np.asarray(f, dtype=np.float64)
    lin = f / (200.0 / 3)
    return np.where(f >= 1000.0, 15.0 + np.log(np.maximum(f, 1e-30) / 1000.0) / (np.log(6.4) / 27.0), lin)


def _mel_to_hz(m):
    m = np.asarray(m, dtype=np.float64)
    return np.where(m >= 15.0, 1000.0 * np.exp((np.log(6.4) / 27.0) * (m - 15.0)), (200.0 / 3) * m)


@lru_cache(maxsize=8)
def slaney_mel_filters(n_mels: int, sr: int = SAMPLING_RATE, n_fft: int = N_FFT) -> np.ndarray:
    """(n_mels, n_fft//2 + 1) float32 == librosa.filters.mel(sr=sr, n_fft=n_fft, n_mels=n_mels): triangles in Hz whose
    corners are equally spaced on the Slaney mel scale between 0 and sr/2, each scaled to unit area (2 / width)."""
    bins = np.arange(n_fft // 2 + 1, dtype=np.float64) * (sr / n_fft)
    corners = _mel_to_hz(np.linspace(_hz_to_mel(0.0), _hz_to_mel(sr / 2), n_mels + 2))
    out = np.zeros((n_mels, bins.size), dtype=np.float64)
    for m in range(n_mels):
        lo, ce, hi = corners[m], corners[m + 1], corners[m + 2]
        rise = (bins - lo) / (ce - lo)
        fall = (hi - bins) / (hi - ce)
        out[m] = np.maximum(0.0, np.minimum(rise, fall)) * (2.0 / (hi - lo))
    return out.astype(np.float32)


def num_rows(n: int) -> int:
    return (n + HOP // 2) // HOP  # utils.py:424-434 with frame_shift = 160 / 16000


def extract(x, num_filters: int = 80, dtype=torch.float32) -> np.ndarray:
    """(n,) or (1, n) waveform -> (num_rows(n), num_filters).  dtype=float64 gives the tolerance gates their truth."""
    a = torch.as_tensor(np.asarray(x)).to(dtype).reshape(-1)
    n = a.numel()
    window = torch.hann_window(N_FFT).to(dtype)
    filters = torch.from_numpy(slaney_mel_filters(num_filters)).to(dtype)
    # torch.stft(center=True, pad_mode="reflect"): N_FFT/2 mirrored samples per side (edge not repeated),
    # frames every HOP samples, 1 + n // HOP of them; the reference drops the last one
    padded = torch.nn.functional.pad(a.view(1, 1, -1), (N_FFT // 2, N_FFT // 2), mode="reflect").view(-1)
    frames = padded.unfold(0, N_FFT, HOP)[:-1]
    spec = torch.fft.rfft(frames * window, dim=-1)  # (T, 201)
    power = spec.abs() ** 2
    mel = filters @ power.T  # (M, T), the reference's operand order
    v = torch.clamp(mel, min=1e-10).log10()
    v = torch.maximum(v, v.max() - 8.0)
    v = (v + 4.0) / 4.0
    rows = num_rows(n)
    if rows > v.shape[1]:
        v = torch.nn.functional.pad(v, (0, rows - v.shape[1]), mode="constant")
    return v.T.contiguous().to(torch.float32 if dtype == torch.float32 else dtype).numpy()
