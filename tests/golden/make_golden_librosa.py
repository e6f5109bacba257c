#!/usr/bin/env python
"""Generates tests/golden/golden_librosa_v1.npz by running the REAL reference class
`lhotse.features.librosa_fbank.LibrosaFbank` (imported from the reference lhotse tree, CPU) on seeded inputs.  Build container only:

    PYTHONDONTWRITEBYTECODE=1 python tests/golden/make_golden_librosa.py

librosa is not installed here: the reference's `import librosa` resolves to the stand-in of tests/refshim.py, whose `stft`
and `filters.mel` are transformers.audio_utils.spectrogram / mel_filter_bank.  Everything else that runs (magnitudes, the
mel product, log10 with its floor, pad_or_truncate_features) is the reference's own code."""
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
import refshim  # noqa: E402

CASES = [
    # (signal, n, seed, config overrides)
    ("noise", 22050, 0, {}), ("noise", 22050 + 127, 1, {}), ("noise", 22050 + 128, 2, {}), ("noise", 513, 3, {}),
    ("noise", 66150, 4, {}), ("sine", 30000, 0, {}), ("zeros", 8000, 0, {}), ("quiet", 22050, 5, {}),
    ("noise", 48000, 6, dict(sampling_rate=24000, fft_size=2048, hop_size=300, win_length=1200, fmin=80, fmax=7600)),
    ("noise", 32000, 7, dict(sampling_rate=16000, fft_size=512, hop_size=128, num_mel_bins=40, fmin=0, fmax=None)),
    ("noise", 16000, 8, dict(sampling_rate=16000, fft_size=400, hop_size=160, window="hamming", fmin=None, fmax=None)),
    ("noise", 24000, 9, dict(sampling_rate=8000, fft_size=256, hop_size=80, num_mel_bins=40, fmin=50, fmax=3800)),
    ("noise", 22050, 10, dict(win_length=800)),
]


def signal(kind, n, seed, sr):
    rs = np.random.RandomState(seed)
    if kind == "noise":
        return (0.1 * rs.randn(n)).astype(np.float32)
    if kind == "quiet":
        return (1e-4 * rs.randn(n)).astype(np.float32)
    if kind == "zeros":
        return np.zeros(n, dtype=np.float32)
    if kind == "sine":
        return (0.5 * np.sin(2 * np.pi * 440.0 * np.arange(n, dtype=np.float64) / sr)).astype(np.float32)
    raise ValueError(kind)


def main():
    refshim.install_librosa_standin()
    refshim.import_reference()
    from lhotse.features.librosa_fbank import LibrosaFbank, LibrosaFbankConfig

    out, man = {}, []
    for i, (kind, n, seed, over) in enumerate(CASES):
        cfg = LibrosaFbankConfig(**over)
        x = signal(kind, n, seed, cfg.sampling_rate)
        y = LibrosaFbank(cfg).extract(x, cfg.sampling_rate)
        assert y.shape == ((n + cfg.hop_size // 2) // cfg.hop_size, cfg.num_mel_bins), (y.shape, n)
        out[f"x{i}"], out[f"y{i}"] = x, y.astype(np.float32)
        man.append({"signal": kind, "n": n, "seed": seed, "cfg": cfg.to_dict()})
        print(i, kind, n, over, y.shape, y.dtype)
    out["manifest"] = np.frombuffer(json.dumps(man).encode(), dtype=np.uint8)
    path = os.path.join(HERE, "golden_librosa_v1.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
