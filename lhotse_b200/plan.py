"""
Config normalisation: any of the reference's Kaldi-family config dataclasses -> one
``FeaturePlan`` (integer sizes + flags + float32 constant tables) that the C ABI consumes.

The tables are built with the *same float32 torch op sequence* as the reference so they are
bit-identical to its ``_window`` / ``_fb`` / ``_dct`` / ``_lifter`` parameters
(lhotse/features/kaldi/layers.py:921-940, :960-1017, :873-907, :697-706, :681-695); tests assert
that.  Only table construction happens here (once per extractor, a few hundred KB): the
per-sample arithmetic lives exclusively in the CUDA kernels.
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field
from typing import Any, Optional, Union

import numpy as np
import torch

EPSILON = 1e-10  # lhotse/utils.py:50
LOG_EPSILON = math.log(EPSILON)  # lhotse/utils.py:51 — the collation pad value

FEATURE_KINDS = {"fbank": 0, "mfcc": 1, "spectrogram": 2, "log-spectrogram": 3, "whisper-fbank": 4, "librosa-fbank": 5}
ENERGY_LHOTSE, ENERGY_KALDI = 0, 1
PAD_KALDI, PAD_CENTER = 0, 1  # include/b200feat.h B200FEAT_PAD_*
WINDOWS = ("hamming", "hanning", "povey", "rectangular", "blackman")


def next_power_of_2(x: int) -> int:
    return 1 if x == 0 else 2 ** (x - 1).bit_length()  # layers.py:951


def make_window(L: int, window_type: str, blackman_coeff: float = 0.42, torchaudio_blackman: bool = False) -> np.ndarray:
    if window_type == "hanning":
        w = torch.hann_window(L, periodic=False)
    elif window_type == "hamming":
        w = torch.hamming_window(L, periodic=False, alpha=0.54, beta=0.46)
    elif window_type == "povey":
        w = torch.hann_window(L, periodic=False).pow(0.85)
    elif window_type == "rectangular":
        w = torch.ones(L, dtype=torch.float32)
    elif window_type == "blackman":
        # lhotse: 2*pi/L (layers.py:931); torchaudio/kaldi: 2*pi/(L-1) (kaldi.py:104)
        a = 2 * math.pi / (L - 1 if torchaudio_blackman else L)
        k = torch.arange(L, dtype=torch.float32)
        w = blackman_coeff - 0.5 * torch.cos(a * k) + (0.5 - blackman_coeff) * torch.cos(2 * a * k)
    else:
        raise ValueError(f"Invalid window type: {window_type}")
    return w.to(torch.float32).numpy().copy()


def _lin2mel(x):
    # np.log on a torch tensor evaluates in numpy and wraps back to a tensor — the reference does
    # exactly this (layers.py:943), and torch.log would differ in the last ulp of a few entries.
    return 1127.0 * np.log(1 + x / 700)


def _make_mel_bank_vtln(M, N, sr, low_freq, high_freq, vtln_low, vtln_high, warp) -> np.ndarray:
    """The Kaldi mel bank with VTLN warping, in float32 torch arithmetic ordered as torchaudio orders it (all-tensor mel scale,
    `1127 * log(1 + f / 700)` and its inverse) so that the weights come out bit-equal.  The warp F is continuous and piecewise
    linear on [low, high] with F(low) = low, F(high) = high and F(f) = f / warp between the knees
    l = vtln_low * max(1, warp) and h = vtln_high * min(1, warp)."""
    if M <= 3:
        raise ValueError("Must have at least 3 mel bins")
    if N % 2 != 0:
        raise ValueError("the Kaldi mel scale needs an even fft length")
    nyquist = 0.5 * sr
    hi = high_freq + nyquist if high_freq <= 0.0 else high_freq
    if not (0.0 <= low_freq < nyquist and 0.0 < hi <= nyquist and low_freq < hi):
        raise ValueError(f"Bad values in options: low-freq {low_freq} and high-freq {hi} vs. nyquist {nyquist}")
    vhi = vtln_high + nyquist if vtln_high < 0.0 else vtln_high
    if not (low_freq < vtln_low < hi and 0.0 < vhi < hi and vtln_low < vhi):
        raise ValueError(f"Bad values in options: vtln-low {vtln_low} and vtln-high {vhi}, versus low-freq {low_freq} and high-freq {hi}")
    knee_lo = vtln_low * max(1.0, warp)
    knee_hi = vhi * min(1.0, warp)
    if not (knee_lo > low_freq and knee_hi < hi):
        raise ValueError(f"vtln_warp {warp} moves the warp's knees outside ({low_freq}, {hi})")
    scale = 1.0 / warp
    slope_lo = (scale * knee_lo - low_freq) / (knee_lo - low_freq)
    slope_hi = (hi - scale * knee_hi) / (hi - knee_hi)

    def to_mel(f):
        return 1127.0 * (1.0 + f / 700.0).log()

    def warped(mel_edges):
        f = 700.0 * ((mel_edges / 1127.0).exp() - 1.0)
        out = hi + slope_hi * (f - hi)                                  # above the upper knee
        out = torch.where(f < knee_hi, scale * f, out)                   # between the knees
        out = torch.where(f < knee_lo, low_freq + slope_lo * (f - low_freq), out)
        out = torch.where((f < low_freq) | (f > hi), f, out)             # outside [low, high]: identity
        return to_mel(out)

    mel_lo = 1127.0 * math.log(1.0 + low_freq / 700.0)
    mel_hi = 1127.0 * math.log(1.0 + hi / 700.0)
    delta = (mel_hi - mel_lo) / (M + 1)
    b = torch.arange(M).unsqueeze(1)
    left, center, right = warped(mel_lo + b * delta), warped(mel_lo + (b + 1.0) * delta), warped(mel_lo + (b + 2.0) * delta)
    mel = to_mel((sr / N) * torch.arange(N / 2)).unsqueeze(0)
    up = (mel - left) / (center - left)
    down = (right - mel) / (right - center)
    bank = torch.zeros_like(up)
    rising = (mel > left) & (mel <= center)
    falling = (mel > center) & (mel < right)
    bank = torch.where(rising, up, bank)
    bank = torch.where(falling, down, bank)
    bank = torch.nn.functional.pad(bank, (0, 1), mode="constant", value=0).T
    return np.ascontiguousarray(bank.to(torch.float32).numpy())


def make_mel_bank(
    num_filters: int,
    fft_length: int,
    sampling_rate: int,
    low_freq: float,
    high_freq: float,
    torchaudio_compatible: bool = True,
    norm_filters: bool = False,
    vtln_low: float = 100.0,
    vtln_high: float = -500.0,
    vtln_warp: float = 1.0,
) -> np.ndarray:
    """Dense (K = N//2 + 1, M) float32 bank, equal to the reference's ``_fb``.  `vtln_warp != 1` (the torchaudio family only:
    `TorchaudioFbankConfig.vtln_*`, lhotse/features/fbank.py:30-32, handed to `torchaudio.compliance.kaldi.fbank`) moves the
    filter edges through Kaldi's piecewise-linear VTLN warp; the table is then bit-equal to torchaudio's `get_mel_banks`."""
    M, N, sr = num_filters, fft_length, sampling_rate
    if torchaudio_compatible and vtln_warp != 1.0:
        return _make_mel_bank_vtln(M, N, sr, low_freq, high_freq, vtln_low, vtln_high, vtln_warp)
    if torchaudio_compatible:
        if M <= 3:
            raise ValueError("Must have at least 3 mel bins")  # layers.py:976
        if N % 2 != 0:
            raise ValueError("torchaudio-compatible mel scale needs an even fft length")  # :977
        nyquist = 0.5 * sr
        hi = high_freq + nyquist if high_freq <= 0.0 else high_freq
        if not (0.0 <= low_freq < nyquist and 0.0 < hi <= nyquist and low_freq < hi):
            raise ValueError(f"Bad values in options: low-freq {low_freq} and high-freq {hi} vs. nyquist {nyquist}")
        mel_lo = _lin2mel(low_freq)
        mel_hi = _lin2mel(hi)
        delta = (mel_hi - mel_lo) / (M + 1)
        b = torch.arange(M).unsqueeze(1)
        left = mel_lo + b * delta
        center = mel_lo + (b + 1.0) * delta
        right = mel_lo + (b + 2.0) * delta
        mel = _lin2mel((sr / N) * torch.arange(N / 2)).unsqueeze(0)
        up = (mel - left) / (center - left)
        down = (right - mel) / (right - center)
        bank = torch.max(torch.zeros(1), torch.min(up, down))  # (M, N/2)
        bank = torch.nn.functional.pad(bank, (0, 1), mode="constant", value=0).T
        return np.ascontiguousarray(bank.to(torch.float32).numpy())
    # legacy numpy scale (layers.py:873-907)
    hi = high_freq
    if hi is None or hi == 0:
        hi = sr / 2
    if hi < 0:
        hi = sr / 2 + hi
    melfc = np.linspace(1127.0 * np.log(1 + low_freq / 700), 1127.0 * np.log(1 + hi / 700), M + 2)
    mels = 1127.0 * np.log(1 + np.linspace(0, sr, N) / 700)
    K = int(N / 2 + 1)
    B = np.zeros((K, M), dtype=np.float32)
    j = np.arange(int(N / 2))
    for k in range(M):
        l, c, r = melfc[k], melfc[k + 1], melfc[k + 2]
        mj = mels[: int(N / 2)]
        inside = (l < mj) & (mj < r)
        rising = inside & (mj <= c)
        falling = inside & (mj > c)
        B[j[rising], k] = (mj[rising] - l) / (c - l)
        B[j[falling], k] = (r - mj[falling]) / (r - c)
    if norm_filters:
        B = B / np.sum(B, axis=0, keepdims=True)
    return np.ascontiguousarray(B.astype(np.float32))


def _slaney_hz_to_mel(f):
    f = np.asanyarray(f, dtype=np.float64)
    f_sp = 200.0 / 3
    min_log_hz = 1000.0
    min_log_mel = min_log_hz / f_sp
    logstep = np.log(6.4) / 27.0
    return np.where(f >= min_log_hz, min_log_mel + np.log(np.maximum(f, 1e-30) / min_log_hz) / logstep, f / f_sp)


def _slaney_mel_to_hz(m):
    m = np.asanyarray(m, dtype=np.float64)
    f_sp = 200.0 / 3
    min_log_hz = 1000.0
    min_log_mel = min_log_hz / f_sp
    logstep = np.log(6.4) / 27.0
    return np.where(m >= min_log_mel, min_log_hz * np.exp(logstep * (m - min_log_mel)), f_sp * m)


def make_slaney_mel_bank(sampling_rate: int, n_fft: int, n_mels: int, fmin: float = 0.0,
                         fmax: Optional[float] = None) -> np.ndarray:
    """Dense (K = n_fft//2 + 1, M) float32 bank = ``librosa.filters.mel(sr, n_fft, n_mels).T`` — what WhisperFbank
    builds at whisper_fbank.py:117-120 (librosa defaults: Slaney mel scale, htk=False, norm="slaney", float32 output).
    librosa is a third-party dependency that is absent from the reference tree and from this image; this restates its
    published algorithm (librosa/filters.py ``mel``: triangles in Hz between Slaney-mel-spaced corner frequencies, each
    scaled by 2 / (f[m+2] - f[m]), evaluated in float64 and cast to float32).  tests/test_whisper.py pins it bit-for-bit
    to transformers.audio_utils.mel_filter_bank(norm="slaney", mel_scale="slaney"), which upstream tests against librosa."""
    fmax = sampling_rate / 2 if fmax is None else fmax
    fftfreqs = np.fft.rfftfreq(n=n_fft, d=1.0 / sampling_rate)
    mel_f = _slaney_mel_to_hz(np.linspace(_slaney_hz_to_mel(fmin), _slaney_hz_to_mel(fmax), n_mels + 2))
    fdiff = np.diff(mel_f)
    ramps = np.subtract.outer(mel_f, fftfreqs)
    w = np.zeros((n_mels, 1 + n_fft // 2), dtype=np.float64)
    for i in range(n_mels):
        lower = -ramps[i] / fdiff[i]
        upper = ramps[i + 2] / fdiff[i + 1]
        w[i] = np.maximum(0, np.minimum(lower, upper))
    enorm = 2.0 / (mel_f[2 : n_mels + 2] - mel_f[:n_mels])
    w *= enorm[:, np.newaxis]
    return np.ascontiguousarray(w.astype(np.float32).T)


def make_dct(num_ceps: int, num_filters: int) -> np.ndarray:
    n = torch.arange(float(num_filters)).unsqueeze(1)
    k = torch.arange(float(num_ceps))
    dct = torch.cos(math.pi / float(num_filters) * (n + 0.5) * k)
    dct[:, 0] *= 1.0 / math.sqrt(2.0)
    dct *= math.sqrt(2.0 / float(num_filters))
    return np.ascontiguousarray(dct.to(torch.float32).numpy())


def make_lifter(num_ceps: int, Q: float) -> Optional[np.ndarray]:
    if Q == 0:
        return None
    v = 1 + 0.5 * Q * torch.sin(math.pi * torch.arange(num_ceps, dtype=torch.float32) / Q)
    return np.ascontiguousarray(v.to(torch.float32).numpy())


@dataclass
class FeaturePlan:
    feature: str
    sampling_rate: int
    L: int
    S: int
    N: int
    num_filters: int = 0
    num_ceps: int = 0
    snip_edges: bool = False
    remove_dc_offset: bool = True
    use_energy: bool = False
    energy_last: bool = False  # htk_compat (kaldifeat family): the energy / C0 column is the last one instead of the first
    raw_energy: bool = True
    use_fft_mag: bool = False
    energy_style: int = ENERGY_LHOTSE
    preemph_coeff: float = 0.97
    energy_floor: float = EPSILON
    mel_floor: float = float(torch.finfo(torch.float).eps)  # layers.py:533-535
    log_spec_eps: float = 1e-15  # layers.py:467
    dither: float = 0.0
    pad_mode: int = PAD_KALDI
    window: np.ndarray = field(default=None, repr=False)
    mel_bank: Optional[np.ndarray] = field(default=None, repr=False)
    dct: Optional[np.ndarray] = field(default=None, repr=False)
    lifter: Optional[np.ndarray] = field(default=None, repr=False)

    @property
    def K(self) -> int:
        return self.N // 2 + 1

    @property
    def feature_dim(self) -> int:
        if self.feature == "fbank":
            return self.num_filters + (1 if self.use_energy else 0)
        if self.feature in ("whisper-fbank", "librosa-fbank"):
            return self.num_filters
        if self.feature == "mfcc":
            return self.num_ceps
        return self.K

    def num_frames(self, n: Union[int, np.ndarray]) -> Union[int, np.ndarray]:
        """layers.py:747-753 (the in-layer twin of utils.py:424-434); whisper-fbank: whisper_fbank.py:73-80.
        `n` is a sample count or an integer array of them (element-wise)."""
        if self.snip_edges and self.feature not in ("whisper-fbank", "librosa-fbank"):
            t = np.where(n < self.L, 0, 1 + (n - self.L) // self.S)
            return t if isinstance(n, np.ndarray) else int(t)
        return (n + self.S // 2) // self.S

    def tables_blob(self) -> np.ndarray:
        """All constant tables in one float32 vector (what rank 0 broadcasts over NCCL)."""
        parts = [self.window]
        for t in (self.mel_bank, self.dct, self.lifter):
            if t is not None:
                parts.append(t.reshape(-1))
        return np.concatenate(parts).astype(np.float32)

    def load_tables_blob(self, blob: np.ndarray) -> None:
        o = 0
        self.window = blob[o : o + self.L].copy(); o += self.L
        if self.mel_bank is not None:
            n = self.mel_bank.size
            self.mel_bank = blob[o : o + n].reshape(self.mel_bank.shape).copy(); o += n
        if self.dct is not None:
            n = self.dct.size
            self.dct = blob[o : o + n].reshape(self.dct.shape).copy(); o += n
        if self.lifter is not None:
            n = self.lifter.size
            self.lifter = blob[o : o + n].copy(); o += n
        assert o == blob.size


def _get(cfg: Any, *names, default=None):
    for n in names:
        if hasattr(cfg, n) and getattr(cfg, n) is not None:
            return getattr(cfg, n)
    return default


def build_plan(feature: str, cfg: Any) -> FeaturePlan:
    """Accepts our configs, lhotse's FbankConfig/MfccConfig/SpectrogramConfig/LogSpectrogramConfig
    (extractors.py:24-63, :156-197, :266-293, :376-403), TorchaudioFbankConfig/TorchaudioMfccConfig/
    TorchaudioSpectrogramConfig (fbank.py:11-39, mfcc.py:9-39, spectrogram.py:11-31) and
    KaldifeatFbankConfig/KaldifeatMfccConfig (kaldifeat.py:149-175, :218-246), duck-typed by field names."""
    if feature not in FEATURE_KINDS:
        raise ValueError(f"unknown feature kind {feature}")
    if feature == "whisper-fbank":
        return build_whisper_plan(cfg)
    if feature == "librosa-fbank":
        return build_librosa_plan(cfg)
    frame = _get(cfg, "frame_opts", default=cfg)  # kaldifeat nests the frame options
    melo = _get(cfg, "mel_opts", default=cfg)
    compat = getattr(cfg, "compat", "lhotse")  # our configs carry the family explicitly
    if compat not in ("lhotse", "torchaudio"):
        raise ValueError(f"compat must be 'lhotse' or 'torchaudio', got {compat!r}")
    is_torchaudio = hasattr(cfg, "preemphasis_coefficient") or compat == "torchaudio"
    is_kaldifeat = hasattr(cfg, "frame_opts")
    sr = int(_get(frame, "sampling_rate", default=16000))
    frame_length = float(_get(frame, "frame_length", default=0.025))
    frame_shift = float(_get(frame, "frame_shift", default=0.01))
    L = int(math.floor(frame_length * sr))  # layers.py:114
    S = int(math.floor(frame_shift * sr))  # layers.py:116
    if L < 2 or S < 1:
        raise ValueError(f"degenerate frame geometry L={L} S={S}")
    rpo2 = bool(_get(frame, "round_to_power_of_two", default=True))
    N = next_power_of_2(L) if rpo2 else L
    window_type = _get(frame, "window_type", default="povey")
    dither = float(_get(frame, "dither", default=0.0))
    if dither < 0.0:
        raise ValueError("dither must be >= 0")
    vtln = float(_get(melo, "vtln_warp", default=1.0))
    htk = bool(_get(cfg, "htk_compat", default=False))
    if htk and feature not in ("fbank", "mfcc"):
        raise ValueError("htk_compat=True applies to fbank / mfcc only")
    if not bool(_get(cfg, "use_log_fbank", default=True)):
        raise ValueError("use_log_fbank=False is not supported")
    use_fft_mag = bool(_get(cfg, "use_fft_mag", default=False))
    if hasattr(cfg, "use_power") and not cfg.use_power:
        use_fft_mag = True
    plan = FeaturePlan(
        feature=feature,
        sampling_rate=sr,
        L=L,
        S=S,
        N=N,
        snip_edges=bool(_get(frame, "snip_edges", default=False)),
        remove_dc_offset=bool(_get(frame, "remove_dc_offset", default=True)),
        use_energy=bool(_get(cfg, "use_energy", default=False)),
        raw_energy=bool(_get(cfg, "raw_energy", default=True)),
        use_fft_mag=use_fft_mag,
        energy_style=ENERGY_KALDI if (is_torchaudio or is_kaldifeat) else ENERGY_LHOTSE,
        preemph_coeff=float(_get(frame, "preemph_coeff", "preemphasis_coefficient", default=0.97)),
        energy_floor=float(_get(cfg, "energy_floor", default=EPSILON)),
        dither=dither,
    )
    if feature == "log-spectrogram" and is_torchaudio:
        # torchaudio.compliance.kaldi.spectrogram: log(max(|X|^2, eps32)) — a negative log_spec_eps selects the floor form
        plan.log_spec_eps = -float(torch.finfo(torch.float).eps)
    plan.window = make_window(
        L, window_type, blackman_coeff=float(_get(frame, "blackman_coeff", default=0.42)),
        torchaudio_blackman=is_torchaudio or is_kaldifeat,
    )
    if feature in ("fbank", "mfcc"):
        M = int(_get(melo, "num_filters", "num_mel_bins", "num_bins", default=80 if feature == "fbank" else 23))
        plan.num_filters = M
        plan.mel_bank = make_mel_bank(
            M, N, sr,
            float(_get(melo, "low_freq", default=20.0)),
            float(_get(melo, "high_freq", default=-400.0)),
            torchaudio_compatible=bool(_get(cfg, "torchaudio_compatible_mel_scale", default=True)),
            norm_filters=bool(_get(cfg, "norm_filters", default=False)),
            vtln_low=float(_get(melo, "vtln_low", default=100.0)),
            vtln_high=float(_get(melo, "vtln_high", default=-500.0)),
            vtln_warp=vtln,
        )
    if feature == "mfcc":
        C = int(_get(cfg, "num_ceps", default=13))
        if C > plan.num_filters:
            raise ValueError("num_ceps cannot exceed the number of mel filters")
        plan.num_ceps = C
        plan.dct = make_dct(C, plan.num_filters)
        plan.lifter = make_lifter(C, float(_get(cfg, "cepstral_lifter", default=22)))
        if htk:
            # Kaldi's htk_compat for cepstra (kaldifeat MfccOptions.htk_compat; torchaudio/compliance/kaldi.py mfcc: the same steps):
            # C0 — or the log-energy that replaces it — moves to the LAST column, and without use_energy it is multiplied by sqrt(2)
            # AFTER the lifter (whose first coefficient is 1).  Expressed as a column permutation of the DCT and the lifter tables,
            # the sqrt(2) riding on the lifter slot so that the arithmetic keeps the reference's order (matmul, then one multiply).
            perm = list(range(1, C)) + [0]
            plan.dct = np.ascontiguousarray(plan.dct[:, perm])
            lf = plan.lifter if plan.lifter is not None else np.ones(C, dtype=np.float32)
            lf = np.ascontiguousarray(lf[perm]).astype(np.float32)
            if not plan.use_energy:
                lf[-1] = np.float32(lf[-1] * np.float32(math.sqrt(2.0)))
            plan.lifter = lf
            plan.energy_last = True
    elif htk:
        plan.energy_last = plan.use_energy  # fbank: [mel bins..., log-energy] instead of [log-energy, mel bins...]
    return plan


def build_whisper_plan(cfg: Any) -> FeaturePlan:
    """WhisperFbankConfig (whisper_fbank.py:87-98: `num_filters`, `device`) -> plan.  Everything else is fixed by the
    reference's constructor (whisper_fbank.py:107-123): 16 kHz, n_fft = 400, hop 160, periodic Hann window, librosa
    (Slaney) mel filters over 0..8000 Hz; log_mel_spectrogram (:16-84): torch.stft(center=True) framing without DC
    removal or pre-emphasis, |X|^2, mel, log10(max(., 1e-10)), clamp to the utterance maximum - 8, (x + 4) / 4."""
    M = int(_get(cfg, "num_filters", default=80))
    if M < 1:
        raise ValueError("num_filters must be positive")
    sr, n_fft, hop = 16000, 400, 160
    plan = FeaturePlan(
        feature="whisper-fbank", sampling_rate=sr, L=n_fft, S=hop, N=n_fft, num_filters=M,
        snip_edges=False, remove_dc_offset=False, use_energy=False, raw_energy=True, use_fft_mag=False,
        preemph_coeff=0.0, mel_floor=1e-10, pad_mode=PAD_CENTER,
    )
    plan.window = torch.hann_window(n_fft).to(torch.float32).numpy().copy()  # whisper_fbank.py:116 (periodic)
    plan.mel_bank = make_slaney_mel_bank(sr, n_fft, M)
    return plan


def make_periodic_window(name: str, length: int) -> np.ndarray:
    """scipy.signal.get_window(name, length, fftbins=True) — what librosa.stft builds (float64) — for the cosine-sum
    windows, rounded once to float32."""
    k = np.arange(length, dtype=np.float64)
    a = 2.0 * np.pi * k / length
    if name in ("hann", "hanning"):
        w = 0.5 - 0.5 * np.cos(a)
    elif name == "hamming":
        w = 0.54 - 0.46 * np.cos(a)
    elif name == "blackman":
        w = 0.42 - 0.5 * np.cos(a) + 0.08 * np.cos(2 * a)
    elif name in ("boxcar", "rectangular", "ones"):
        w = np.ones(length)
    else:
        raise ValueError(f"unsupported librosa window {name!r} (hann, hamming, blackman, boxcar)")
    return w.astype(np.float32)


def build_librosa_plan(cfg: Any) -> FeaturePlan:
    """LibrosaFbankConfig (librosa_fbank.py:16-38: sampling_rate, fft_size, hop_size, win_length, window, num_mel_bins,
    fmin, fmax) -> plan for `logmelfilterbank` (:64-135): librosa.stft(n_fft, hop_length, win_length, window,
    pad_mode="reflect") = centred frames of n_fft samples under a periodic window of win_length centred in the frame;
    |X| (magnitudes, :117); librosa.filters.mel(sr, n_fft, n_mels, fmin, fmax) (Slaney); log10(max(1e-10, .)) (:126);
    rows = compute_num_frames(len / sr, hop / sr, sr) (:128-134: the stft's 1 + n // hop frames, minus the last one when
    n mod hop < hop / 2)."""
    sr = int(_get(cfg, "sampling_rate", default=22050))
    N = int(_get(cfg, "fft_size", default=1024))
    S = int(_get(cfg, "hop_size", default=256))
    wl = _get(cfg, "win_length", default=None)
    wl = N if wl is None else int(wl)
    M = int(_get(cfg, "num_mel_bins", default=80))
    if N < 2 or N % 2 or S < 1 or not (0 < wl <= N) or M < 1:
        raise ValueError(f"degenerate librosa geometry fft_size={N} hop_size={S} win_length={wl} num_mel_bins={M}")
    fmin = getattr(cfg, "fmin", 80)   # None is meaningful here (librosa_fbank.py:119-120): 0 Hz / Nyquist
    fmax = getattr(cfg, "fmax", 7600)
    fmin = 0.0 if fmin is None else float(fmin)
    fmax = sr / 2 if fmax is None else float(fmax)
    plan = FeaturePlan(
        feature="librosa-fbank", sampling_rate=sr, L=N, S=S, N=N, num_filters=M,
        snip_edges=False, remove_dc_offset=False, use_energy=False, raw_energy=True, use_fft_mag=True,
        preemph_coeff=0.0, mel_floor=EPSILON, pad_mode=PAD_CENTER,
    )
    win = np.zeros(N, dtype=np.float32)
    lo = (N - wl) // 2  # librosa.util.pad_center
    win[lo: lo + wl] = make_periodic_window(str(_get(cfg, "window", default="hann")), wl)
    plan.window = win
    plan.mel_bank = make_slaney_mel_bank(sr, N, M, fmin=fmin, fmax=fmax)
    return plan
