#!/usr/bin/env python
"""Generates tests/golden/golden_v1.npz by running the REAL reference (lhotse imported from
the reference lhotse tree, CPU, float32) on seeded inputs.  Run in the build container only:

    PYTHONDONTWRITEBYTECODE=1 python tests/golden/make_golden.py

Each case stores the input waveform, the reference output, and the config as JSON, so the
fixtures are self-contained on the GPU box (where the reference does not exist).
Reference entry points used: lhotse/features/kaldi/extractors.py:67 (Fbank), :201 (Mfcc),
:297 (Spectrogram), :407 (LogSpectrogram) — `.extract(samples, sampling_rate)`.
"""
import json
import os
import sys
import wave

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
import refshim  # noqa: E402

refshim.import_reference()
import torch  # noqa: E402
from lhotse.features.kaldi.extractors import (  # noqa: E402
    Fbank,
    FbankConfig,
    LogSpectrogram,
    LogSpectrogramConfig,
    Mfcc,
    MfccConfig,
    Spectrogram,
    SpectrogramConfig,
)

TYPES = {
    "fbank": (Fbank, FbankConfig),
    "mfcc": (Mfcc, MfccConfig),
    "spectrogram": (Spectrogram, SpectrogramConfig),
    "log-spectrogram": (LogSpectrogram, LogSpectrogramConfig),
}


def signal(kind, n, seed, sr):
    rs = np.random.RandomState(seed)
    if kind == "noise":
        return (0.1 * rs.randn(n)).astype(np.float32)
    if kind == "sine":
        t = np.arange(n, dtype=np.float64) / sr
        return (0.5 * np.sin(2 * np.pi * 1000.0 * t)).astype(np.float32)
    if kind == "zeros":
        return np.zeros(n, dtype=np.float32)
    if kind == "dc":
        return (0.3 + 0.01 * rs.randn(n)).astype(np.float32)
    if kind == "quiet":
        return (1e-4 * rs.randn(n)).astype(np.float32)
    if kind == "speech":
        with wave.open(os.path.join(refshim.REFERENCE_ROOT, "test/fixtures/libri/libri-1088-134315-0000.wav")) as w:
            assert w.getframerate() == 16000 and w.getnchannels() == 1 and w.getsampwidth() == 2
            w.setpos(16000 * 2)
            pcm = np.frombuffer(w.readframes(n), dtype="<i2")
        return (pcm.astype(np.float32) / 32768.0).astype(np.float32)
    raise ValueError(kind)


CASES = []


def add(feature, kind, n, seed=0, sr=16000, **cfg):
    CASES.append(dict(feature=feature, kind=kind, n=n, seed=seed, sr=sr, cfg=cfg))


# frame-count edges on the headline config (test/known_issues/test_cut_consistency.py:9-75)
for n in (159, 160, 240, 400, 15995, 16000, 16005, 16079, 16080):
    add("fbank", "noise", n, seed=n)
add("fbank", "noise", 100000, seed=7)  # 625 frames: several tiles
add("fbank", "speech", 32000)
add("fbank", "sine", 16000)
add("fbank", "zeros", 1600)
add("fbank", "dc", 8000, seed=3)
add("fbank", "quiet", 8000, seed=4)
add("mfcc", "noise", 16000, seed=11)
add("mfcc", "speech", 32000)
add("mfcc", "noise", 8000, seed=12, num_ceps=20, num_filters=40, cepstral_lifter=10)
add("spectrogram", "noise", 8000, seed=13)
add("spectrogram", "speech", 16000, use_energy=True)
add("log-spectrogram", "noise", 8000, seed=14)
add("log-spectrogram", "speech", 16000, use_fft_mag=True)
add("fbank", "noise", 8000, seed=20, use_energy=True)
add("fbank", "noise", 8000, seed=21, use_energy=True, raw_energy=False, energy_floor=0.0)
for w in ("hamming", "hanning", "rectangular", "blackman"):
    add("fbank", "noise", 4000, seed=22, window_type=w)
add("fbank", "speech", 8000, preemph_coeff=0.0)
add("fbank", "dc", 8000, seed=23, remove_dc_offset=False)
add("fbank", "noise", 8000, seed=24, use_fft_mag=True)
add("fbank", "noise", 8000, seed=25, round_to_power_of_two=False)  # N = 400 = 2^4 * 5^2
add("fbank", "speech", 16000, round_to_power_of_two=False, num_filters=40)
add("fbank", "noise", 8000, seed=26, torchaudio_compatible_mel_scale=False, norm_filters=True, num_filters=40)
add("fbank", "noise", 8000, seed=27, torchaudio_compatible_mel_scale=False, norm_filters=False, low_freq=0.0, high_freq=0.0)
add("fbank", "noise", 8000, seed=28, num_filters=23, low_freq=100.0, high_freq=7000.0)
add("fbank", "noise", 8000, seed=29, snip_edges=True)
add("fbank", "noise", 8000, seed=30, sr=8000, sampling_rate=8000, num_filters=40)  # L=200 S=80 N=256
add("mfcc", "noise", 8000, seed=31, sr=8000, sampling_rate=8000)
add("fbank", "noise", 24000, seed=32, sr=24000, sampling_rate=24000, frame_length=0.05)  # L=1200 N=2048
add("fbank", "noise", 22050, seed=33, sr=22050, sampling_rate=22050)  # L=551 S=220 N=1024
add("fbank", "noise", 22050, seed=34, sr=22050, sampling_rate=22050, round_to_power_of_two=False, num_filters=40, torchaudio_compatible_mel_scale=False)  # N=551=19*29 (odd: legacy mel only)
add("fbank", "noise", 44100, seed=35, sr=44100, sampling_rate=44100, num_filters=128)  # L=1102 N=2048
add("fbank", "noise", 8000, seed=36, frame_length=0.032, frame_shift=0.016)  # L=N=512 S=256
add("spectrogram", "noise", 4000, seed=37, round_to_power_of_two=False, use_fft_mag=True)
add("log-spectrogram", "noise", 11025, seed=38, sr=22050, sampling_rate=22050, round_to_power_of_two=False)  # N=551 odd


def main():
    torch.set_num_threads(1)
    out, manifest = {}, []
    import warnings

    warnings.simplefilter("ignore")
    for i, c in enumerate(CASES):
        x = signal(c["kind"], c["n"], c["seed"], c["sr"])
        cls, cfgcls = TYPES[c["feature"]]
        y = cls(cfgcls(**c["cfg"])).extract(x, c["cfg"].get("sampling_rate", 16000))
        assert y.dtype == np.float32
        out[f"x{i}"] = x
        out[f"y{i}"] = y
        manifest.append(dict(c, shape=list(y.shape)))
        print(i, c["feature"], c["kind"], c["n"], c["cfg"], y.shape)
    out["manifest"] = np.frombuffer(json.dumps(manifest).encode(), dtype=np.uint8)
    path = os.path.join(HERE, "golden_v1.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, os.path.getsize(path) / 1e6, "MB")


if __name__ == "__main__":
    main()
