"""Test-only helper: make the *reference* (lhotse) importable where `soundfile`, `intervaltree` and `cytoolz` are
absent (SURVEY.md §8c).  The reference is the tree named by LHOTSE_REFERENCE_ROOT or the archive
`oracle/_ref/lhotse_ref.zip` that `oracle/make_ref.py` packs from it during `build()` (see oracle/refimport.py); tests that
need lhotse itself skip where neither exists.  Never used by the product."""
import os
import sys
import types

_ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if _ROOT not in sys.path:
    sys.path.insert(0, _ROOT)
from oracle.refimport import (REFERENCE_ROOT, REFERENCE_ZIP, import_reference, reference_available,  # noqa: E402,F401
                              reference_kind)


def install_librosa_standin():
    """`WhisperFbank` takes its mel table from `librosa.filters.mel` (whisper_fbank.py:117-120) and refuses to construct
    without librosa (:112-115).  librosa is not in this image: register a stand-in whose `filters.mel` is the table of
    `transformers.audio_utils.mel_filter_bank(norm="slaney", mel_scale="slaney")` — an independent third-party
    implementation that upstream tests against librosa.  Raises ImportError when transformers is missing."""
    import importlib.machinery

    import numpy as np
    from transformers.audio_utils import mel_filter_bank

    if "librosa" in sys.modules and not getattr(sys.modules["librosa"], "_b200_standin", False):
        return  # the real thing
    def stft(y, n_fft=2048, hop_length=None, win_length=None, window="hann", center=True, pad_mode="constant"):
        """`librosa.stft` as LibrosaFbank calls it (librosa_fbank.py:108-115), on transformers' STFT: periodic window of
        win_length centred in an n_fft frame, centred (padded) framing, complex one-sided output (1 + n_fft/2, frames)."""
        from transformers.audio_utils import spectrogram, window_function

        wl = n_fft if win_length is None else win_length
        hop = wl // 4 if hop_length is None else hop_length
        win = window_function(wl, window, periodic=True, frame_length=n_fft, center=True)
        return spectrogram(np.asarray(y), win, frame_length=n_fft, hop_length=hop, fft_length=n_fft, power=None,
                           center=center, pad_mode=pad_mode, onesided=True)

    def mel(sr, n_fft, n_mels, fmin=0.0, fmax=None):
        fmax = sr / 2 if fmax is None else fmax
        return mel_filter_bank(1 + n_fft // 2, n_mels, float(fmin), float(fmax), sr, norm="slaney", mel_scale="slaney").T.astype(np.float32)

    lib = types.ModuleType("librosa")
    lib.__spec__ = importlib.machinery.ModuleSpec("librosa", None)
    lib._b200_standin = True
    lib.stft = stft
    lib.filters = types.ModuleType("librosa.filters")
    lib.filters.mel = mel
    sys.modules["librosa"] = lib
    sys.modules["librosa.filters"] = lib.filters
