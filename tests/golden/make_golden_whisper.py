#!/usr/bin/env python
"""Generates tests/golden/golden_whisper_v1.npz by running the REAL reference class
`lhotse.features.whisper_fbank.WhisperFbank` (imported from the reference lhotse tree, CPU, float32) on seeded inputs.
Build container only:

    PYTHONDONTWRITEBYTECODE=1 python tests/golden/make_golden_whisper.py

The reference takes its mel table from `librosa.filters.mel` (whisper_fbank.py:117-120); librosa is not installed in
this image, so a stand-in module is registered whose `filters.mel` returns the table computed by
`transformers.audio_utils.mel_filter_bank(norm="slaney", mel_scale="slaney")` — an independent third-party
implementation that upstream tests against librosa.  Everything else that runs is the reference's own code.
"""
import json
import os
import sys
import wave

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
import refshim  # noqa: E402


def signal(kind, n, seed):
    rs = np.random.RandomState(seed)
    if kind == "noise":
        return (0.1 * rs.randn(n)).astype(np.float32)
    if kind == "loud":
        return np.clip(0.6 * rs.randn(n), -1, 1).astype(np.float32)
    if kind == "quiet":
        return (1e-4 * rs.randn(n)).astype(np.float32)
    if kind == "zeros":
        return np.zeros(n, dtype=np.float32)
    if kind == "sine":
        t = np.arange(n, dtype=np.float64) / 16000
        return (0.5 * np.sin(2 * np.pi * 440.0 * t)).astype(np.float32)
    if kind == "burst":  # > 8 decades of dynamic range inside one cut: exercises the max - 8 clamp
        x = (1e-6 * rs.randn(n)).astype(np.float32)
        x[n // 2: n // 2 + 800] += (0.8 * rs.randn(800)).astype(np.float32)
        return x
    if kind == "speech":
        with wave.open(os.path.join(refshim.REFERENCE_ROOT, "test/fixtures/libri/libri-1088-134315-0000.wav")) as w:
            assert w.getframerate() == 16000 and w.getnchannels() == 1 and w.getsampwidth() == 2
            w.setpos(16000 * 2)
            pcm = np.frombuffer(w.readframes(n), dtype=np.int16)
        return (pcm.astype(np.float32) / 32768.0)[:n]
    raise ValueError(kind)


CASES = [
    # (signal, n, seed, num_filters)
    ("noise", 16000, 0, 80), ("noise", 16079, 1, 80), ("noise", 16080, 2, 80), ("noise", 16081, 3, 80),
    ("noise", 201, 4, 80), ("noise", 1000, 5, 80), ("noise", 15999, 6, 80), ("noise", 48000, 7, 128),
    ("speech", 48000, 0, 80), ("speech", 40000, 0, 128), ("sine", 24000, 0, 80), ("zeros", 8000, 0, 80),
    ("quiet", 16000, 8, 80), ("loud", 16000, 9, 80), ("burst", 32000, 10, 80), ("noise", 160000, 11, 80),
]


def main():
    refshim.install_librosa_standin()
    refshim.import_reference()
    from lhotse.features.whisper_fbank import WhisperFbank, WhisperFbankConfig

    out, man = {}, []
    ext = {}
    for i, (kind, n, seed, M) in enumerate(CASES):
        if M not in ext:
            ext[M] = WhisperFbank(WhisperFbankConfig(num_filters=M))
        x = signal(kind, n, seed)
        y = ext[M].extract(x, 16000)
        assert y.dtype == np.float32 and y.shape == ((n + 80) // 160, M), (y.shape, n)
        out[f"x{i}"], out[f"y{i}"] = x, y
        man.append({"signal": kind, "n": n, "seed": seed, "num_filters": M})
    out["manifest"] = np.frombuffer(json.dumps(man).encode(), dtype=np.uint8)
    path = os.path.join(HERE, "golden_whisper_v1.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, os.path.getsize(path), "bytes,", len(man), "cases")


if __name__ == "__main__":
    main()
