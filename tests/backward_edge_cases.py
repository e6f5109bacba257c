"""Shared pieces of the backward's edge tests (tests/test_backward_kernel_edges.py; csrc/backward.cuh, DESIGN.md §3.1n): the
table of frame geometries, one per launch shape of `bwd_launch_shape` plus the frames it refuses; a sample count for each
frame count; waveforms that are periodic with the hop, or on which the mel, energy and log-spectrogram floors bind in part;
the torchaudio and HTK configs; torchaudio's own functions for them; and the float32 gradient of the B200 classes."""
from __future__ import annotations

import math
from dataclasses import dataclass, field
from typing import Optional

import numpy as np
import torch

import backward_cases as BC
from lhotse_b200.plan import ENERGY_KALDI, FeaturePlan
from oracle import kaldi_oracle as O

SR = 16000


@dataclass(frozen=True)
class Shape:
    """A geometry of the table: the feature kind and frame length (seconds at 16 kHz, rounded up to a power of two) that give
    the launch shape (warps per CTA, frames per tile); `warps is None` for a frame the backward refuses."""
    name: str
    feature: str
    frame_length: float
    warps: Optional[int]
    ft: Optional[int]
    kw: dict = field(default_factory=dict, hash=False)


SHAPES = [
    Shape("N512-L400", "fbank", 0.025, 4, 16, {"use_energy": True}),
    Shape("N1024-L800", "mfcc", 0.05, 4, 16, {"use_energy": True, "raw_energy": False}),
    Shape("N2048-L1600", "log-spectrogram", 0.1, 4, 8, {}),
    Shape("N2048-L2048", "fbank", 0.128, 4, 4, {}),
    Shape("N4096-L4096", "spectrogram", 0.256, 2, 2, {"use_energy": True}),
    Shape("N8192-L6400", "fbank", 0.4, 1, 1, {"use_energy": True}),
    Shape("N8192-L8192-refused", "fbank", 0.512, None, None, {}),
    Shape("N16384-L9600-refused", "log-spectrogram", 0.6, None, None, {}),
]
ACCEPTED = [s for s in SHAPES if s.warps is not None]
REFUSED = [s for s in SHAPES if s.warps is None]


def config(feature: str, device="cuda", **kw):
    """The B200 config of a kind (16 kHz); unknown keys raise."""
    import warnings

    import lhotse_b200 as lb

    ccls = {"fbank": lb.B200FbankConfig, "mfcc": lb.B200MfccConfig, "spectrogram": lb.B200SpectrogramConfig,
            "log-spectrogram": lb.B200LogSpectrogramConfig}[feature]
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")  # snip_edges
        return ccls(device=device, **kw)


def extractor(feature: str, **kw):
    import lhotse_b200 as lb

    cls = {"fbank": lb.B200Fbank, "mfcc": lb.B200Mfcc, "spectrogram": lb.B200Spectrogram,
           "log-spectrogram": lb.B200LogSpectrogram}[feature]
    return cls(config(feature, **kw))


def shape_kw(s: Shape, **kw) -> dict:
    return {"frame_length": s.frame_length, **s.kw, **kw}


def plan_of(feature: str, **kw) -> FeaturePlan:
    from lhotse_b200.plan import build_plan

    return build_plan(feature, config(feature, **kw))


# ----------------------------------------------------------------------------- lengths
def length_for(plan: FeaturePlan, T: int) -> Optional[int]:
    """A sample count that the plan's framing turns into exactly T frames (its offset within the hop varies with T), or
    None where the framing refuses every such count (reflect padding longer than the cut)."""
    L, S = plan.L, plan.S
    if plan.snip_edges:
        cands = [L + (T - 1) * S + (7 * T) % S, L + (T - 1) * S]
    else:
        lo = T * S - S // 2
        cands = [lo + (7 * T) % S] + list(range(lo, lo + S))
    for n in cands:
        if n > 0 and O.num_frames_layer(n, L, S, plan.snip_edges) == T:
            try:
                O.frame_index_matrix(n, L, S, plan.snip_edges)
                return n
            except ValueError:
                pass
    return None


def tile_counts(ft: int, long: int) -> list:
    """T = 1, ft - 1, ft, ft + 1, 2 ft - 1, 2 ft, 2 ft + 1 and `long` (a partial last tile), without repeats or zeros."""
    return sorted(set(t for t in (1, ft - 1, ft, ft + 1, 2 * ft - 1, 2 * ft, 2 * ft + 1, long) if t >= 1))


# ----------------------------------------------------------------------------- waveforms
def floors_waveform(n: int, seed=0) -> np.ndarray:
    """Noise at 0.1, a run at 3e-5 (its weak bins fall under the log-spectrogram and mel floors, its strong ones do not), a
    run at 1e-6 (every floor binds, the energies under Kaldi's eps), a run of digital silence, then noise again: within one
    cut the floors bind on some bins and frames and not on others."""
    rs = np.random.RandomState(seed + n)
    x = rs.randn(n)
    amp = np.full(n, 0.1)
    q = n // 5
    amp[q:2 * q], amp[2 * q:3 * q], amp[3 * q:4 * q] = 3e-5, 1e-6, 0.0
    return amp * x


def periodic_waveform(n: int, period: int, seed=0) -> np.ndarray:
    """Noise repeating with `period` samples (float32-exact): every frame that starts a whole number of hops apart from
    another and needs no reflection holds the same samples."""
    p = (0.1 * np.random.RandomState(seed).randn(period)).astype(np.float32).astype(np.float64)
    return np.resize(p, n)


def waveform(n: int, kind: str, seed=0) -> np.ndarray:
    x = floors_waveform(n, seed) if kind == "floors" else BC.waveform(n, kind, seed)
    return x.astype(np.float32).astype(np.float64)


# ----------------------------------------------------------------------------- floors
def floor_values(x: np.ndarray, plan: FeaturePlan):
    """float64 values that meet a floor, per frame: (mel energies or None, spectrum values of a log-spectrogram or None,
    energies or None), with the floors (mel floor, log-spectrogram floor, Kaldi energy eps)."""
    idx = O.frame_index_matrix(x.shape[0], plan.L, plan.S, plan.snip_edges)
    f = x[idx]
    d = f - f.mean(1, keepdims=True) if plan.remove_dc_offset else f
    a = plan.preemph_coeff
    pre = d - a * np.concatenate((d[:, :1], d[:, :-1]), 1) if a != 0.0 else d
    y = pre * np.asarray(plan.window, dtype=np.float64)
    X = np.fft.rfft(y, n=plan.N)
    v = np.abs(X) if plan.use_fft_mag else np.abs(X) ** 2
    mel = v @ np.asarray(plan.mel_bank, dtype=np.float64) if plan.feature in ("fbank", "mfcc") else None
    spec = v if plan.feature == "log-spectrogram" else None
    e = ((d * d).sum(1) if plan.raw_energy else (y * y).sum(1)) if plan.use_energy else None
    return mel, spec, e


def floor_conditioned(x: np.ndarray, plan: FeaturePlan, G: np.ndarray, rel=1e-4, margin=1e-3) -> np.ndarray:
    """G without gradient where float32 cannot decide the chain: log-spectrogram bins below `rel` of their frame's largest
    (a log singularity, see BC.conditioned), and values within `margin` (relative) of the floor they meet, where float32
    and float64 may fall on different sides (an MFCC row loses its whole gradient then: each cepstrum reads every mel)."""
    mel, spec, e = floor_values(x, plan)
    G = G.copy()
    F = G.shape[1]
    ecol = BC.energy_col(plan, F)
    near = lambda v, fl: np.abs(v / fl - 1.0) < margin  # noqa: E731
    if spec is not None:
        fl = -plan.log_spec_eps if plan.log_spec_eps < 0 else None
        bad = spec < rel * spec.max(1, keepdims=True)
        if fl is not None:  # below the floor the gradient is exactly 0 in any precision: keep it
            bad = (bad & (spec > fl)) | near(spec, fl)
        if plan.use_energy:
            bad[:, 0] = False
        G[bad] = 0.0
    if mel is not None:
        bad = near(mel, plan.mel_floor)
        if plan.feature == "fbank":
            cols = [c for c in range(F) if not (plan.use_energy and c == ecol)]
            G[:, cols] = np.where(bad, 0.0, G[:, cols])
        else:
            G[bad.any(1)] = 0.0
    if e is not None:
        bad = np.zeros(e.shape, bool)
        if plan.energy_style == ENERGY_KALDI:
            bad |= near(e, BC.EPS32)
        if BC.energy_floor_binds(plan):
            lv = np.log(np.maximum(e, BC.EPS32)) if plan.energy_style == ENERGY_KALDI else np.log(e + 1e-15)
            bad |= np.abs(lv - math.log(plan.energy_floor)) < margin
        G[bad, ecol] = 0.0
    return G


# ----------------------------------------------------------------------------- the torchaudio and HTK conventions
COMPAT = [
    ("fbank-energy-raw", "fbank", {"use_energy": True, "energy_floor": 0.0}),
    ("fbank-energy-raw-floor", "fbank", {"use_energy": True, "energy_floor": 1.0}),
    ("fbank-htk-energy-win", "fbank", {"use_energy": True, "raw_energy": False, "htk_compat": True, "energy_floor": 0.0}),
    ("fbank-htk-blackman-floor", "fbank", {"use_energy": True, "htk_compat": True, "window_type": "blackman", "energy_floor": 0.5}),
    ("fbank-htk-noenergy", "fbank", {"htk_compat": True}),
    ("mfcc-energy-raw", "mfcc", {"use_energy": True, "energy_floor": 0.0}),
    ("mfcc-energy-win-floor", "mfcc", {"use_energy": True, "raw_energy": False, "energy_floor": 1.0}),
    ("mfcc-htk", "mfcc", {"htk_compat": True}),
    ("mfcc-htk-energy-nolifter", "mfcc", {"htk_compat": True, "use_energy": True, "cepstral_lifter": 0, "energy_floor": 0.0}),
    ("mfcc-htk-nolifter-snip", "mfcc", {"htk_compat": True, "cepstral_lifter": 0, "snip_edges": True}),
    ("log-spectrogram-energy", "log-spectrogram", {"use_energy": True, "energy_floor": 0.0}),
    ("log-spectrogram-energy-floor-snip", "log-spectrogram", {"use_energy": True, "energy_floor": 1.0, "snip_edges": True}),
]


def compat_kw(kw: dict) -> dict:
    return {"compat": "torchaudio", **kw}


def with_torchaudio_tables(plan: FeaturePlan, kw: dict) -> FeaturePlan:
    """The plan with torchaudio's own tables (kaldi.py: its float64 window, `get_mel_banks`, `_get_dct_matrix`,
    `_get_lifter_coeffs`) in place of the plan's, arranged as the plan arranges them (HTK: C0 last, sqrt(2) on it without
    energy).  The plan's mel bank is lhotse's and differs from torchaudio's in the float32 rounding of its weights, which
    the log of a weak low band amplifies to ~1e-5."""
    import dataclasses

    import torchaudio.compliance.kaldi as K

    c = config(plan.feature, **compat_kw(kw))
    w = K._feature_window_function(c.window_type, plan.L, c.blackman_coeff, torch.device("cpu"), torch.float64).numpy()
    out = dataclasses.replace(plan, window=w)
    if plan.feature in ("fbank", "mfcc"):
        fb, _ = K.get_mel_banks(plan.num_filters, plan.N, float(plan.sampling_rate), c.low_freq, c.high_freq, c.vtln_low,
                                c.vtln_high, c.vtln_warp)
        out.mel_bank = np.pad(fb.double().numpy(), ((0, 0), (0, 1))).T
    if plan.feature == "mfcc":
        C = plan.num_ceps
        dct = K._get_dct_matrix(C, plan.num_filters).double().numpy()
        lifter = K._get_lifter_coeffs(C, float(c.cepstral_lifter)).double().numpy() if c.cepstral_lifter else None
        if c.htk_compat:
            perm = list(range(1, C)) + [0]
            dct = dct[:, perm]
            lifter = np.ones(C) if lifter is None else lifter[perm]
            if not plan.use_energy:
                lifter[-1] *= math.sqrt(2.0)
        out.dct, out.lifter = dct, lifter
    return out


def torchaudio_features(x: torch.Tensor, feature: str, kw: dict) -> torch.Tensor:
    """torchaudio.compliance.kaldi's fbank / mfcc / spectrogram of a 1-D waveform with the settings of a compat config
    (defaults of the B200 configs for the rest).  The spectrogram stands for the log-spectrogram with use_energy: it always
    puts the log-energy in bin 0."""
    import torchaudio.compliance.kaldi as K

    c = config(feature, **compat_kw(kw))
    common = dict(sample_frequency=float(c.sampling_rate), frame_length=c.frame_length * 1000.0,
                  frame_shift=c.frame_shift * 1000.0, round_to_power_of_two=c.round_to_power_of_two,
                  remove_dc_offset=c.remove_dc_offset, preemphasis_coefficient=c.preemph_coeff, window_type=c.window_type,
                  blackman_coeff=c.blackman_coeff, dither=0.0, snip_edges=c.snip_edges, energy_floor=c.energy_floor,
                  raw_energy=c.raw_energy)
    w = x.reshape(1, -1)
    if feature == "log-spectrogram":
        assert c.use_energy
        return K.spectrogram(w, **common)
    mel = dict(num_mel_bins=c.num_filters, low_freq=c.low_freq, high_freq=c.high_freq, use_energy=c.use_energy,
               htk_compat=c.htk_compat)
    if feature == "fbank":
        return K.fbank(w, use_power=not c.use_fft_mag, **mel, **common)
    return K.mfcc(w, num_ceps=c.num_ceps, cepstral_lifter=float(c.cepstral_lifter), **mel, **common)


# ----------------------------------------------------------------------------- the B200 classes' gradient
def b200_grads(ext, xs, Gs):
    """float32 gradients (CUDA tensors) of sum_i <features(x_i), G_i> over one `extract_batch` call on the list `xs`."""
    leaves = [torch.tensor(x, dtype=torch.float32, device="cuda", requires_grad=True) for x in xs]
    outs = ext.extract_batch(leaves, SR)
    loss = sum((o.to("cuda") * torch.as_tensor(G, dtype=torch.float32, device="cuda")).sum() for o, G in zip(outs, Gs))
    loss.backward()
    return [x.grad for x in leaves]


def b200_rows_grad(ext, X: np.ndarray, Gs, lengths=None) -> torch.Tensor:
    """float32 gradient of a (B, n) batch (with `lengths`, or its full rows) whose cut i has row gradient Gs[i]."""
    Xt = torch.tensor(X, dtype=torch.float32, device="cuda", requires_grad=True)
    outs = ext.extract_batch(Xt, SR, lengths=lengths)
    if isinstance(outs, torch.Tensor):
        outs = [outs] if Xt.shape[0] == 1 else list(outs)
    out = torch.cat([o.to("cuda") for o in outs])
    G = torch.as_tensor(np.concatenate(Gs), dtype=torch.float32, device="cuda")
    (out * G).sum().backward()
    return Xt.grad
