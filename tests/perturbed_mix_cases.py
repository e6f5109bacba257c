"""Test-only: MixedCuts whose tracks carry Speed / Volume / Resample chains, built with real lhotse calls over the WAV (and
optionally FLAC) fixtures of mix_cases / transform_cases, one per feature of the "mix" route with `perturbed_tracks=True`
(CutMix over speed-perturbed speech, MixedCut.perturb_speed of a padded mix, a volume-perturbed track, resampled speech under
plain noise, a perturbed muted SNR reference, an SNR-scaled perturbed first track, trim and reflect-pad, FLAC speech under
WAV noise), the cuts the route must still refuse, and the recipe-shaped batches of the larger tests."""
import contextlib

import numpy as np

import flac_oracle as F
import lhotse_env
import mix_cases
import transform_cases


@contextlib.contextmanager
def flac_backend():
    """WAV through the current (test) backend, FLAC through the oracle decoder (int16 / 32768, as libsndfile hands it to
    lhotse); restores the backend afterwards."""
    from lhotse.audio.backend import AudioBackend, LibsndfileCompatibleAudioInfo, get_current_audio_backend, set_current_audio_backend

    wav_backend = get_current_audio_backend()

    class OracleFlacBackend(AudioBackend):
        def read_audio(self, path_or_fd, offset=0.0, duration=None, force_opus_sampling_rate=None):
            if not str(path_or_fd).endswith(".flac"):
                return wav_backend.read_audio(path_or_fd, offset, duration, force_opus_sampling_rate)
            si, _, pcm = F.decode(open(str(path_or_fd), "rb").read())
            a = int(round(offset * si.sample_rate))
            n = pcm.shape[0] - a if duration is None else int(round(duration * si.sample_rate))
            return (pcm[a:a + n].T.astype(np.float32) / 32768.0), si.sample_rate

        def is_applicable(self, path_or_fd):
            return True

        def supports_info(self):
            return True

        def info(self, path_or_fd, force_opus_sampling_rate=None, force_read_audio=False):
            si = F.read_streaminfo(open(str(path_or_fd), "rb").read())
            return LibsndfileCompatibleAudioInfo(channels=si.channels, frames=si.total_samples, samplerate=si.sample_rate,
                                                 duration=si.total_samples / si.sample_rate)

    set_current_audio_backend(OracleFlacBackend())
    try:
        yield
    finally:
        set_current_audio_backend(wav_backend)


def flac_cuts(paths):
    """Whole-file MonoCuts over the 16 kHz FLAC fixtures."""
    from lhotse import MonoCut, Recording
    from lhotse.audio import AudioSource

    out = []
    for k, p in enumerate(paths):
        n = F.read_streaminfo(open(p, "rb").read()).total_samples
        rec = Recording(id=f"pfl{k}", sources=[AudioSource(type="file", channels=[0], source=str(p))], sampling_rate=16000,
                        num_samples=n, duration=n / 16000)
        out.append(MonoCut(id=f"pfl{k}", start=0.0, duration=n / 16000, channel=0, recording=rec))
    return out


def sources(root):
    """(speech, noise, 48 kHz speech): the mix_cases WAV fixtures and one 3.1 s 48 kHz WAV cut."""
    speech, noise = mix_cases.sources(root)
    return speech, noise, transform_cases._cut(root, "pw48k", int(3.1 * 48000), 48000, seed=48)


def cases(root, speech, noise, s48, flac=None):
    """name -> cut, every one eligible for the mix route with perturbed_tracks=True (and refused without it).  Run inside
    transform_cases.torch_resampler() (Resample needs lhotse's torch resampler)."""
    from lhotse import CutSet
    from lhotse.cut import MixedCut, MixTrack
    from lhotse.dataset.cut_transforms import CutMix
    from lhotse.utils import fastcopy

    s, n = speech, noise
    c = {}
    # 1. CutMix over speed-perturbed speech, and explicit mixes at several SNRs
    cm = CutMix(CutSet.from_cuts(n), p=1.0, snr=(10, 20), seed=7, pad_to_longest=True, preserve_id=True)
    for cut in cm(CutSet.from_cuts([s[0].perturb_speed(0.9), s[1].perturb_speed(1.1), s[3].perturb_speed(0.9),
                                    s[4].perturb_speed(1.1)])):
        c[f"cutmix_{cut.id}"] = cut
    for k, (f, snr) in enumerate(((0.9, None), (1.1, 0), (0.9, -5), (1.1, 20))):
        c[f"speed_{f}_snr_{snr}"] = s[k].perturb_speed(f).mix(n[k], snr=snr, allow_padding=True, preserve_id="left")
    # 2. MixedCut.perturb_speed of a padded mix: every track perturbed (padding too), offsets rescaled
    padded = s[4].pad(duration=s[4].duration + 0.7, direction="left").mix(n[2].truncate(duration=3.0), snr=5, offset_other_by=0.3,
                                                                        preserve_id="left")
    c["mixed_then_speed_0.9"] = padded.perturb_speed(0.9)
    # 3. perturb_volume on one track
    c["volume_track"] = MixedCut(id="volume_track", tracks=[MixTrack(cut=s[0].perturb_volume(0.6)), MixTrack(cut=n[1], snr=10.0)])
    c["volume_noise"] = s[1].mix(n[2].perturb_volume(1.7), snr=8, allow_padding=True, preserve_id="left")
    # 4. 48 kHz speech resampled to 16 kHz under plain 16 kHz noise
    c["resampled_speech"] = s48.resample(16000).mix(n[2], snr=10, allow_padding=True, preserve_id="left")
    # 5. a perturbed muted SNR reference
    c["muted_perturbed_reference"] = MixedCut(id="muted_perturbed_reference", tracks=[
        MixTrack(cut=s[5].perturb_speed(1.1), is_snr_reference=True, mute=True),
        MixTrack(cut=n[0], snr=10.0),
        MixTrack(cut=n[1], offset=0.4, snr=3.0),
    ])
    # 6. an SNR-scaled perturbed first track: the mix is float64
    c["scaled_perturbed_first"] = MixedCut(id="scaled_perturbed_first", tracks=[
        MixTrack(cut=n[2].perturb_speed(1.1), snr=7.0),
        MixTrack(cut=s[0].perturb_speed(0.9), offset=0.2),
        MixTrack(cut=n[3], offset=0.5, snr=15.0),
    ])
    # 7. trim and reflect-pad: durations off the sample grid, so the mix is one sample longer / shorter than the cut
    sp = s[4].perturb_speed(1.1)
    c["reflect_pad"] = MixedCut(id="p_reflect_pad", tracks=[
        MixTrack(cut=fastcopy(s[4], id="prp0", duration=1.5)),
        MixTrack(cut=fastcopy(sp, id="prp1", duration=1.50003), offset=0.00003, snr=5.0)])
    c["trim"] = MixedCut(id="p_trim", tracks=[
        MixTrack(cut=fastcopy(s[4], id="ptr0", duration=1.5)),
        MixTrack(cut=fastcopy(sp, id="ptr1", duration=1.50004), offset=0.00004, snr=5.0)])
    # 8. FLAC speech under WAV noise
    if flac:
        c["flac_speech_speed"] = flac[0].truncate(offset=0.5, duration=4.0).perturb_speed(0.9).mix(
            n[2], snr=12, allow_padding=True, preserve_id="left")
        c["flac_speech_volume"] = flac[1].truncate(offset=1.0, duration=3.0).perturb_volume(0.8).perturb_speed(1.1).mix(
            n[0], snr=15, allow_padding=True, preserve_id="left")
    return c


def refused_cases(root, speech, noise):
    """name -> MixedCut the route must refuse even with perturbed_tracks=True."""
    from lhotse.cut import MixedCut, MixTrack
    from lhotse.utils import fastcopy

    s, n = speech, noise
    ok = s[0].perturb_speed(1.1).mix(n[0], snr=10, allow_padding=True, preserve_id="left")
    s8 = transform_cases._cut(root, "pw8k", int(3.1 * 8000), 8000, seed=8)
    return {
        "short_speed_track": s[0].truncate(duration=0.5).perturb_speed(1.1).mix(n[0], snr=10, allow_padding=True),
        "tempo_track": s[0].perturb_tempo(0.9).mix(n[0], snr=10, allow_padding=True),
        "cut_transforms": fastcopy(ok, transforms=[{"name": "Volume", "kwargs": {"factor": 0.5}}]),
        "other_rate_track": MixedCut(id="prate", tracks=[MixTrack(cut=s[0].perturb_speed(1.1)),
                                                         MixTrack(cut=s8.perturb_speed(1.1), snr=10.0)]),
    }


def chosen_tracks(cut):
    """The track cuts `mix_request_for_cut` lists, in its order: the audible tracks, then a muted SNR reference."""
    from lhotse.cut import PaddingCut

    tracks = list(cut.tracks)
    ref = next((t for t in tracks if getattr(t, "is_snr_reference", False)), None)
    if ref is None:
        ref = next((t for t in tracks if not isinstance(t.cut, PaddingCut) and t.snr is None), None)
    audible = [t for t in tracks if not t.mute] or tracks
    return audible + ([ref] if all(t is not ref for t in audible) else [])


def recipe_batch(tmp_path, n_cuts, seed=3):
    """`n_cuts` cuts of 10-30 s speech at speed 0.9 / 1.0 / 1.1 with CutMix(p=0.5, snr 10-20) noise: the LibriSpeech
    recipe's batch shape."""
    from lhotse import CutSet
    from lhotse.dataset.cut_transforms import CutMix

    rs = np.random.RandomState(seed)
    speech = lhotse_env.make_cutset(tmp_path, [30.0] * 8, seed=4, amp=0.2, prefix="ps")
    noise = lhotse_env.make_cutset(tmp_path, [7.3, 12.1, 30.0, 4.4], seed=5, amp=0.05, prefix="pn")
    cuts = []
    for i in range(n_cuts):
        d = float(np.round(rs.uniform(10.0, 30.0), 3))
        a = float(np.round(rs.uniform(0.0, 30.0 - d), 3))
        cut = speech[i % 8].truncate(offset=a, duration=d, preserve_id=False).with_id(f"p{i}")
        cuts.append(cut.perturb_speed(0.9) if i % 3 == 0 else cut.perturb_speed(1.1) if i % 3 == 1 else cut)
    return list(CutMix(noise, p=0.5, snr=(10, 20), seed=11, pad_to_longest=True, preserve_id=True)(CutSet.from_cuts(cuts)))


def load_f32(cut):
    """float32(cut.load_audio()) as the float route feeds the kernels (1-D)."""
    return np.asarray(cut.load_audio()).reshape(-1).astype(np.float32)
