"""Test-only: speed-perturbed, volume-perturbed and resampled MonoCuts built with real lhotse calls over PCM16 WAV files (or
given FLAC cuts), one per feature of the GPU transform route (DESIGN.md §3.1i), and the cuts it must refuse."""
import contextlib
import wave

import numpy as np

import lhotse_env


@contextlib.contextmanager
def torch_resampler():
    """lhotse's Resample transform runs its torch resampler only where torchaudio is installed (elsewhere scipy's
    resample_poly in float64): pretend it is, as a torchaudio install would make it."""
    from lhotse.augmentation import torchaudio as lta

    saved = lta.is_torchaudio_available
    lta.is_torchaudio_available = lambda: True
    try:
        yield
    finally:
        lta.is_torchaudio_available = saved


def _cut(root, name, n, sr, seed):
    from lhotse import MonoCut, Recording
    from lhotse.audio import AudioSource

    rs = np.random.RandomState(seed)
    t = np.arange(n) / sr
    x = 6000 * np.sin(2 * np.pi * (180 + 60 * rs.rand()) * t) + rs.randn(n) * 1500
    pcm = np.clip(x, -32768, 32767).astype("<i2")
    pcm[n // 3: n // 3 + sr // 10] = 0  # a silent stretch: signed zeros through the chain
    lhotse_env.write_wav(root / f"{name}.wav", pcm, sr=sr)
    rec = Recording(id=name, sources=[AudioSource(type="file", channels=[0], source=str(root / f"{name}.wav"))],
                    sampling_rate=sr, num_samples=n, duration=n / sr)
    return MonoCut(id=name, start=0.0, duration=n / sr, channel=0, recording=rec)


def sources(root):
    """rate -> a 3.1 s MonoCut over a WAV file of that rate (16 kHz: several)."""
    out = {sr: _cut(root, f"w{sr}", int(3.1 * sr), sr, seed=sr) for sr in (8000, 22050, 44100, 48000)}
    out[16000] = [_cut(root, f"w16k{i}", int(d * 16000), 16000, seed=i) for i, d in enumerate((3.1, 2.45, 4.0))]
    # 4.1 s at 44.1 kHz: 160 * 180697 / 441 = 65559.5283..., which lhotse's float32 ceil keeps as 65559 samples, not 65560
    out["44100_long"] = _cut(root, "w44k_long", 180697, 44100, seed=7)
    return out


def cases(src):
    """name -> cut, every one eligible for the transform route."""
    s16 = src[16000]
    c = {}
    for f in (0.9, 1.1, 0.95, 1.05):
        c[f"speed_{f}"] = s16[0].perturb_speed(f)
    for sr in (48000, 44100, 22050):
        c[f"resample_{sr}_16000"] = src[sr].resample(16000)
    c["resample_16000_8000"] = s16[1].resample(8000)
    c["resample_8000_16000"] = src[8000].resample(16000)
    c["resample_then_speed"] = src[48000].resample(16000).perturb_speed(1.1)
    c["resample_then_speed_f32_length"] = src["44100_long"].resample(16000).perturb_speed(1.1)
    c["volume_then_speed"] = s16[1].perturb_volume(0.7).perturb_speed(1.1)
    c["speed_then_volume"] = s16[1].perturb_speed(0.9).perturb_volume(1.37)
    c["volume_only"] = s16[2].perturb_volume(2.5)
    c["volume_volume_speed_volume"] = s16[2].perturb_volume(0.5).perturb_volume(3.0).perturb_speed(0.9).perturb_volume(0.8)
    c["start_speed"] = s16[2].truncate(offset=0.73, duration=2.2).perturb_speed(0.9)
    c["start_resample"] = src[44100].truncate(offset=0.41, duration=1.9).resample(16000)
    c["start_speed_volume"] = s16[2].truncate(offset=1.3, duration=1.61).perturb_speed(1.1).perturb_volume(0.9)
    return c


def fix_cases(src):
    """(trim cut, reflect cut): a speed-perturbed slice whose chain output is longer than the cut (found by scanning
    durations), and a speed-perturbed recording whose manifest declares 3 samples more than its file holds (the close-to-full
    read stops at the end of the file, and the output is reflect-padded)."""
    from lhotse.utils import fastcopy

    from lhotse_b200.pcm_staging import _resample_geometry, transform_request_for_cut

    def diff(cut):
        r = transform_request_for_cut(cut)
        L = r.source.num_samples
        for op in r.ops:
            if op[0] == "resample":
                N, O, _, _ = _resample_geometry(op[1], op[2])
                L = -(-N * L // O)
        return r.num_samples - L

    trim = next(c for c in (src[16000][2].truncate(offset=0.2, duration=1.6 + 0.00731 * k).perturb_speed(1.1) for k in range(400))
                if diff(c) < 0)
    s = src[16000][1]
    n = s.recording.num_samples + 3
    longer = fastcopy(s, duration=n / 16000, recording=fastcopy(s.recording, num_samples=n, duration=n / 16000))
    reflect = longer.perturb_speed(0.9)
    assert diff(reflect) > 0
    return trim, reflect


def refused_cases(root, src):
    """name -> cut the transform route must refuse (transform_request_for_cut returns None)."""
    from lhotse import MonoCut, Recording
    from lhotse.audio import AudioSource
    from lhotse.utils import fastcopy

    s = src[16000][0]
    pcm = np.zeros((48000, 2), dtype="<i2")
    with wave.open(str(root / "stereo.wav"), "wb") as w:
        w.setnchannels(2); w.setsampwidth(2); w.setframerate(16000)
        w.writeframes(pcm.tobytes())
    stereo = Recording(id="stereo", sources=[AudioSource(type="file", channels=[0, 1], source=str(root / "stereo.wav"))],
                       sampling_rate=16000, num_samples=48000, duration=3.0)
    short = s.truncate(duration=0.5)
    return {
        "plain": s,
        "tempo": s.perturb_tempo(0.9),
        "reverb": s.reverb_rir(),
        "multi_channel": MonoCut(id="st", start=0.0, duration=3.0, channel=0, recording=stereo).perturb_speed(1.1),
        "short_speed": short.perturb_speed(1.1),
        "short_resample": src[48000].truncate(duration=0.4).resample(16000),
        "mixed": s.perturb_speed(1.1).mix(src[16000][1], snr=10, allow_padding=True),
        "numpy_volume": fastcopy(s, recording=fastcopy(s.recording, transforms=[{"name": "Volume", "kwargs": {"factor": np.float64(2.0)}}])),
    }


def load_f32(cut):
    """float32(cut.load_audio()) as the float route feeds the kernels (1-D)."""
    return np.asarray(cut.load_audio()).reshape(-1).astype(np.float32)
