"""Test-only: MixedCuts built with real lhotse calls over PCM16 WAV (and optionally 16-bit FLAC) files, one per mixing
feature the GPU route reproduces (CutMix noise with several pieces and SNRs, padding on either side, append with gaps, a
muted SNR reference, silent tracks, an SNR-scaled first track, trim and reflect-pad), and a table of cuts it must refuse."""
import wave

import numpy as np

import lhotse_env


def _speechlike(rs, n, amp):
    t = np.arange(n) / 16000.0
    x = amp * np.sin(2 * np.pi * (150 + 40 * rs.rand()) * t) * (0.6 + 0.4 * np.sin(2 * np.pi * 3 * t)) + rs.randn(n) * amp * 0.2
    return np.clip(x, -32768, 32767).astype("<i2")


def _rec(path, n, sr=16000, channels=(0,)):
    from lhotse import Recording
    from lhotse.audio import AudioSource

    return Recording(id=str(path).rsplit("/", 1)[-1], sources=[AudioSource(type="file", channels=list(channels), source=str(path))],
                     sampling_rate=sr, num_samples=n, duration=n / sr)


def _mono(path, pcm, start=0.0, duration=None, sr=16000, cid=None):
    from lhotse import MonoCut

    n = pcm.shape[0]
    rec = _rec(path, n, sr)
    return MonoCut(id=cid or rec.id + f"_{start}", start=start, duration=(n / sr - start) if duration is None else duration,
                   channel=0, recording=rec)


def sources(root, seed=0, speech_flac=None, noise_flac=None):
    """(speech cuts, noise cuts): WAV files written under `root`, unless FLAC cuts are passed in."""
    rs = np.random.RandomState(seed)
    speech, noise = [], []
    for i, dur in enumerate((2.3, 3.1, 1.7, 2.9, 4.05, 2.2)):
        pcm = _speechlike(rs, int(dur * 16000), 6000)
        lhotse_env.write_wav(root / f"sp{i}.wav", pcm)
        speech.append(_mono(root / f"sp{i}.wav", pcm, cid=f"sp{i}"))
    for i, dur in enumerate((0.9, 1.3, 5.2, 0.6)):
        pcm = np.clip(rs.randn(int(dur * 16000)) * 2500, -32768, 32767).astype("<i2")
        lhotse_env.write_wav(root / f"nz{i}.wav", pcm)
        noise.append(_mono(root / f"nz{i}.wav", pcm, cid=f"nz{i}"))
    return (speech_flac or speech), (noise_flac or noise)


def mixed_cases(root, speech, noise):
    """name -> cut, every one eligible for the GPU mix route."""
    from lhotse import CutSet
    from lhotse.cut import MixedCut, MixTrack, PaddingCut
    from lhotse.dataset.cut_transforms import CutMix

    zeros = np.zeros(20000, dtype="<i2")
    lhotse_env.write_wav(root / "silent.wav", zeros)
    silent = _mono(root / "silent.wav", zeros, cid="silent")
    s, n = speech, noise
    cases = {}
    for k, snr in enumerate((None, 0, -5, 20)):
        cases[f"mix_snr_{snr}"] = s[k].mix(n[k], snr=snr, allow_padding=True, preserve_id="left")
    cases["mix_offset_gap"] = s[0].mix(n[1], offset_other_by=s[0].duration + 0.25, snr=10, allow_padding=True, preserve_id="left")
    cm = CutMix(CutSet.from_cuts(n), p=1.0, snr=(10, 20), seed=7, pad_to_longest=True, preserve_id=True)
    for c in cm(CutSet.from_cuts(s[:4])):
        cases[f"cutmix_{c.id}"] = c
    cases["pad_left"] = s[1].pad(duration=s[1].duration + 0.7, direction="left")
    cases["pad_right"] = s[2].pad(duration=s[2].duration + 0.5, direction="right")
    cases["pad_both"] = s[3].pad(duration=s[3].duration + 0.9, direction="both")
    cases["pad_left_then_noise"] = s[1].pad(duration=s[1].duration + 0.7, direction="left").mix(n[3], snr=5, preserve_id="left")
    cases["append"] = s[0].append(s[2])
    cases["append_gap"] = s[0].pad(duration=s[0].duration + 0.31).append(s[4])
    sr = 16000
    cases["muted_reference"] = MixedCut(id="muted_reference", tracks=[
        MixTrack(cut=s[5], is_snr_reference=True, mute=True),
        MixTrack(cut=n[0], snr=10.0),
        MixTrack(cut=n[1], offset=0.4, snr=3.0),
    ])
    cases["silent_noise"] = s[2].mix(silent, snr=10, allow_padding=True, preserve_id="left")
    cases["silent_reference"] = silent.mix(n[0], snr=10, allow_padding=True, preserve_id="left")
    cases["scaled_first"] = MixedCut(id="scaled_first", tracks=[
        MixTrack(cut=n[2], snr=7.0),
        MixTrack(cut=s[0], offset=0.2),
        MixTrack(cut=n[3], offset=0.5, snr=15.0),
    ])
    cases["scaled_first_padding"] = MixedCut(id="scaled_first_padding", tracks=[
        MixTrack(cut=PaddingCut(id="p0", duration=0.5, sampling_rate=sr, num_samples=8000, feat_value=-23.0), snr=4.0),
        MixTrack(cut=s[1], offset=0.1),
    ])
    # trim and reflect-pad: offsets and durations whose sample counts round apart from the mix's own duration
    from lhotse.utils import fastcopy

    base = lambda d, cid: fastcopy(s[4], id=cid, duration=d)  # noqa: E731  (off the sample grid on purpose)
    cases["reflect_pad"] = MixedCut(id="reflect_pad", tracks=[MixTrack(cut=base(1.0, "rp0")),
                                                             MixTrack(cut=base(1.00003, "rp1"), offset=0.00003, snr=5.0)])
    cases["trim"] = MixedCut(id="trim", tracks=[MixTrack(cut=base(1.0, "tr0")),
                                               MixTrack(cut=base(1.00004, "tr1"), offset=0.00004, snr=5.0)])
    return cases


def refused_cases(root, speech, noise):
    """name -> cut the GPU mix route must refuse (mix_request_for_cut returns None)."""
    from lhotse import MultiCut
    from lhotse.cut import MixedCut, MixTrack
    from lhotse.utils import fastcopy

    s, n = speech, noise
    ok = s[0].mix(n[0], snr=10, allow_padding=True, preserve_id="left")
    pcm = np.zeros((16000, 2), dtype="<i2")
    with wave.open(str(root / "stereo.wav"), "wb") as w:
        w.setnchannels(2); w.setsampwidth(2); w.setframerate(16000)
        w.writeframes(pcm.tobytes())
    multi = MultiCut(id="multi", start=0, duration=1.0, channel=[0, 1], recording=_rec(root / "stereo.wav", 16000, channels=(0, 1)))
    r8 = np.zeros(8000, dtype="<i2")
    lhotse_env.write_wav(root / "r8k.wav", r8, sr=8000)
    c8 = _mono(root / "r8k.wav", r8, sr=8000, cid="r8k")
    return {
        "plain_monocut": s[0],
        "cut_transforms": fastcopy(ok, transforms=[{"name": "Volume", "kwargs": {"factor": 0.5}}]),
        "volume_perturbed_track": s[0].perturb_volume(2.0).mix(n[0], snr=10, allow_padding=True),
        "speed_perturbed_track": s[0].perturb_speed(1.1).mix(n[0], snr=10, allow_padding=True),
        "other_sampling_rate": MixedCut(id="sr", tracks=[MixTrack(cut=s[0]), MixTrack(cut=c8, snr=10.0)]),
        "multicut_track": MixedCut(id="mc", tracks=[MixTrack(cut=s[0]), MixTrack(cut=multi, snr=10.0)]),
        "nested_mixed": MixedCut(id="nested", tracks=[MixTrack(cut=ok), MixTrack(cut=n[1], snr=10.0)]),
        "url_source": MixedCut(id="url", tracks=[MixTrack(cut=s[0]), MixTrack(cut=fastcopy(n[1], recording=fastcopy(
            n[1].recording, sources=[fastcopy(n[1].recording.sources[0], type="url", source="http://localhost/x.wav")])),
            snr=10.0)]),
    }


def load_f32(cut):
    """float32(cut.load_audio()) as the float route feeds the kernels (1-D)."""
    return np.asarray(cut.load_audio()).reshape(-1).astype(np.float32)
