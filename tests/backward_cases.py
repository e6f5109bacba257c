"""Shared pieces of the backward tests (csrc/backward.cuh, DESIGN.md §3.1n): the configs and lengths they sweep, the float64
autograd twin of the oracle's `extract` (a tensor out instead of a numpy array, so that autograd can run it), a twin driven
by a FeaturePlan that also follows the torchaudio and HTK conventions (common.cuh), a float64 NumPy restatement of the
adjoint chain written the way the kernel computes it, and the host harness (scripts/micro/backward_host_check.cu) with its
input file."""
from __future__ import annotations

import dataclasses
import math
import os
import shutil
import subprocess
from dataclasses import astuple

import numpy as np
import torch

from lhotse_b200.plan import ENERGY_KALDI, FeaturePlan
from oracle import kaldi_oracle as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EPS32 = float(torch.finfo(torch.float32).eps)

WINDOWS = ("povey", "hanning", "hamming", "rectangular", "blackman")
# frame_length / round_to_power_of_two giving each N at 16 kHz
GEOMETRIES = {256: (0.016, True), 400: (0.025, False), 512: (0.025, True), 1024: (0.05, True), 2048: (0.1, True),
              401: (0.0250625, False)}


def cfg_of(feature="fbank", N=512, **kw) -> O.OracleConfig:
    fl, pow2 = GEOMETRIES[N]
    return O.OracleConfig(feature=feature, frame_length=fl, round_to_power_of_two=pow2, **kw)


def configs():
    """(id, OracleConfig): every kind with energy off / raw / windowed, magnitudes, both framings, pre-emphasis on and off, DC
    removal on and off, every window, every N the tests cover (the odd one with the spectrum kinds: the torchaudio-compatible
    mel scale needs an even N)."""
    out = []
    for feat in ("fbank", "mfcc", "spectrogram", "log-spectrogram"):
        out.append((f"{feat}", cfg_of(feat)))
        out.append((f"{feat}-energy-raw", cfg_of(feat, use_energy=True)))
        out.append((f"{feat}-energy-win-snip", cfg_of(feat, use_energy=True, raw_energy=False, snip_edges=True)))
        out.append((f"{feat}-mag-nodc-nopre", cfg_of(feat, use_fft_mag=True, remove_dc_offset=False, preemph_coeff=0.0)))
    out.append(("mfcc-nolifter", cfg_of("mfcc", cepstral_lifter=0)))
    for w in WINDOWS:
        out.append((f"fbank-{w}", cfg_of("fbank", window_type=w, use_energy=True)))
    for N in (256, 400, 1024, 2048):
        out.append((f"fbank-N{N}", cfg_of("fbank", N=N)))
        out.append((f"log-spectrogram-N{N}-snip", cfg_of("log-spectrogram", N=N, snip_edges=True, use_energy=True)))
    out.append(("spectrogram-N401", cfg_of("spectrogram", N=401, use_energy=True, raw_energy=False)))
    out.append(("log-spectrogram-N401-mag", cfg_of("log-spectrogram", N=401, use_fft_mag=True)))
    return out


def framable(n, cfg) -> bool:
    L, S, _ = O.layer_sizes(cfg)
    try:
        O.frame_index_matrix(n, L, S, cfg.snip_edges)
        return True
    except ValueError:
        return False


def lengths(cfg, long=True):
    """The shortest cut the framing accepts and its neighbour, L - 1, L, L + 1, multiples of S +- 1, and 10 s."""
    L, S, _ = O.layer_sizes(cfg)
    n0 = next(n for n in range(1, 4 * L) if framable(n, cfg))
    ns = [n0, n0 + 1, L - 1, L, L + 1, 7 * S - 1, 7 * S, 7 * S + 1]
    if long:
        ns.append(10 * cfg.sampling_rate)
    return sorted(set(n for n in ns if framable(n, cfg)))


def waveform(n, kind="noise", seed=0):
    rs = np.random.RandomState(seed + n)
    if kind == "silence":
        return np.zeros(n)
    if kind == "full":
        return rs.uniform(-1.0, 1.0, n)
    return 0.1 * rs.randn(n)


# ----------------------------------------------------------------------------- float64 autograd twin of O.extract
def windowed_frames_t(x: torch.Tensor, cfg: O.OracleConfig):
    """O.windowed_frames with its window on the device of x."""
    L, S, N = O.layer_sizes(cfg)
    f = O._frames_view(x, L, S, cfg.snip_edges)
    if cfg.remove_dc_offset:
        f = f - torch.mean(f, dim=1, keepdim=True)
    log_e = None
    if cfg.use_energy and cfg.raw_energy:
        log_e = O._log_energy(f, cfg.energy_floor)
    if cfg.preemph_coeff != 0.0:
        f = f - cfg.preemph_coeff * torch.cat((f[:, :1], f[:, :-1]), dim=1)
    f = f * O._cached_tables(astuple(cfg), x.dtype)[0].to(x.device)
    if N != L:
        f = torch.nn.functional.pad(f, (0, N - L))
    if cfg.use_energy and not cfg.raw_energy:
        log_e = O._log_energy(f, cfg.energy_floor)
    return f, log_e


def features_t(x: torch.Tensor, cfg: O.OracleConfig) -> torch.Tensor:
    """O.extract's chain on a tensor, returning a tensor (in the dtype of x): autograd runs it."""
    dtype = x.dtype
    frames, log_e = windowed_frames_t(x.reshape(-1), cfg)
    X = torch.fft.rfft(frames, dim=-1)
    spec = X.abs() if cfg.use_fft_mag else X.abs() ** 2
    feat = cfg.feature
    if feat == "spectrogram":
        out = spec
    elif feat == "log-spectrogram":
        out = (spec + 1e-15).log()
    else:
        _, fb, dct_t, lifter_t = O._cached_tables(astuple(cfg), dtype)
        eps = torch.tensor(torch.finfo(torch.float).eps, dtype=dtype, device=x.device)
        mel = torch.max(torch.matmul(spec, fb.to(x.device)), eps).log()
        if feat == "fbank":
            return mel if log_e is None else torch.cat((log_e.unsqueeze(-1), mel), dim=-1)
        out = torch.matmul(mel, dct_t.to(x.device))
        if lifter_t is not None:
            out = out * lifter_t.to(x.device)
    if log_e is not None:  # C0 / bin 0 <- log-energy
        out = torch.cat((log_e.unsqueeze(-1), out[:, 1:]), dim=-1)
    return out


def autograd_grad(x: np.ndarray, cfg, G: np.ndarray, dtype=torch.float64, device="cpu") -> np.ndarray:
    """d sum(features * G) / dx through `features_t`."""
    xt = torch.tensor(x, dtype=dtype, device=device, requires_grad=True)
    if dtype != torch.float64:
        with torch.no_grad():
            xt.copy_(torch.as_tensor(x).to(dtype))
    out = features_t(xt, cfg)
    (out * torch.as_tensor(G, dtype=dtype, device=device)).sum().backward()
    return xt.grad.double().cpu().numpy()


# ----------------------------------------------------------------------------- the plan's conventions (common.cuh)
def oracle_plan(cfg: O.OracleConfig, dtype=torch.float64) -> FeaturePlan:
    """The oracle config as a FeaturePlan (lhotse's conventions) holding the oracle's tables in `dtype`, as float64 arrays."""
    L, S, N = O.layer_sizes(cfg)
    win, fb, dct, lifter = (None if t is None else t.numpy().astype(np.float64) for t in O._cached_tables(astuple(cfg), dtype))
    return FeaturePlan(feature=cfg.feature, sampling_rate=cfg.sampling_rate, L=L, S=S, N=N,
                       num_filters=0 if fb is None else fb.shape[1], num_ceps=0 if dct is None else dct.shape[1],
                       snip_edges=cfg.snip_edges, remove_dc_offset=cfg.remove_dc_offset, use_energy=cfg.use_energy,
                       raw_energy=cfg.raw_energy, use_fft_mag=cfg.use_fft_mag, preemph_coeff=cfg.preemph_coeff,
                       energy_floor=cfg.energy_floor, window=win, mel_bank=fb, dct=dct, lifter=lifter)


def energy_floor_binds(plan: FeaturePlan) -> bool:
    """Whether the log-energy is floored: Kaldi's rule is `energy_floor != 0`, lhotse's `energy_floor > 0` (b200feat.cu)."""
    return plan.energy_floor != 0.0 if plan.energy_style == ENERGY_KALDI else plan.energy_floor > 0.0


def energy_col(plan: FeaturePlan, F: int) -> int:
    """Column of the log-energy in a row of F features: last under htk_compat, else first."""
    return F - 1 if plan.energy_last else 0


def _log_energy_t(e: torch.Tensor, plan: FeaturePlan) -> torch.Tensor:
    """common.cuh log_energy_value: Kaldi log(max(e, eps32)) or lhotse log(e + 1e-15), then the floor."""
    if plan.energy_style == ENERGY_KALDI:
        le = torch.max(e, torch.tensor(EPS32, dtype=e.dtype, device=e.device)).log()
    else:
        le = (e + 1e-15).log()
    if energy_floor_binds(plan):
        le = torch.max(le, torch.tensor(math.log(plan.energy_floor), dtype=e.dtype, device=e.device))
    return le


def plan_features_t(x: torch.Tensor, plan: FeaturePlan) -> torch.Tensor:
    """The forward of `plan` on a tensor (in the dtype of x, on its device), with the plan's own tables and conventions:
    lhotse's or Kaldi's log-energy, the floor-form log-spectrogram, the energy column first or last, and the permuted HTK
    DCT and lifter.  autograd runs it."""
    dt, dev = x.dtype, x.device

    def tab(a):
        return torch.as_tensor(np.asarray(a, dtype=np.float64)).to(dtype=dt, device=dev)

    f = O._frames_view(x.reshape(-1), plan.L, plan.S, plan.snip_edges)
    if plan.remove_dc_offset:
        f = f - torch.mean(f, dim=1, keepdim=True)
    le = None
    if plan.use_energy and plan.raw_energy:
        le = _log_energy_t(f.pow(2).sum(1), plan)
    if plan.preemph_coeff != 0.0:
        f = f - plan.preemph_coeff * torch.cat((f[:, :1], f[:, :-1]), dim=1)
    f = f * tab(plan.window)
    if plan.use_energy and not plan.raw_energy:
        le = _log_energy_t(f.pow(2).sum(1), plan)
    X = torch.fft.rfft(f, n=plan.N, dim=-1)
    spec = X.abs() if plan.use_fft_mag else X.abs() ** 2
    if plan.feature == "spectrogram":
        out = spec
    elif plan.feature == "log-spectrogram":
        out = torch.max(spec, tab(-plan.log_spec_eps)).log() if plan.log_spec_eps < 0 else (spec + plan.log_spec_eps).log()
    else:
        mel = torch.max(torch.matmul(spec, tab(plan.mel_bank)), tab(plan.mel_floor)).log()
        if plan.feature == "fbank":
            if le is None:
                return mel
            return torch.cat((mel, le[:, None]), 1) if plan.energy_last else torch.cat((le[:, None], mel), 1)
        out = torch.matmul(mel, tab(plan.dct))
        if plan.lifter is not None:
            out = out * tab(plan.lifter)
        if le is not None:
            c = energy_col(plan, out.shape[1])
            out = torch.cat((out[:, :c], le[:, None], out[:, c + 1:]), 1)
        return out
    if le is not None:  # bin 0 <- log-energy
        out = torch.cat((le[:, None], out[:, 1:]), dim=1)
    return out


def plan_autograd_grad(x: np.ndarray, plan: FeaturePlan, G: np.ndarray, dtype=torch.float64, device="cpu") -> np.ndarray:
    """d sum(features * G) / dx through `plan_features_t`."""
    xt = torch.tensor(np.asarray(x, dtype=np.float64), dtype=dtype, device=device, requires_grad=True)
    out = plan_features_t(xt, plan)
    (out * torch.as_tensor(G, dtype=dtype, device=device)).sum().backward()
    return xt.grad.double().cpu().numpy()


# ----------------------------------------------------------------------------- float64 restatement of the adjoint chain
def _dlog_max(v, floor):
    return np.where(v > floor, 1.0 / np.where(v > 0, v, 1.0), np.where(v == floor, 0.5 / floor, 0.0))


def restated_grad(x: np.ndarray, cfg, G: np.ndarray) -> np.ndarray:
    """The kernel's adjoint chain in float64 for an oracle config, with the oracle's float64 tables."""
    return restated_grad_plan(x, oracle_plan(cfg), G)


def restated_grad_plan(x: np.ndarray, plan: FeaturePlan, G: np.ndarray) -> np.ndarray:
    """The kernel's adjoint chain in float64 with the plan's tables and conventions: recompute the frame, then log, mel /
    DCT, spectrum, frame preprocessing and overlap-add, in that order."""
    L, S, N = plan.L, plan.S, plan.N
    n = x.shape[0]
    idx = O.frame_index_matrix(n, L, S, plan.snip_edges)
    win, fb, dct, lifter = (None if t is None else np.asarray(t, dtype=np.float64)
                            for t in (plan.window, plan.mel_bank, plan.dct, plan.lifter))
    f = x[idx]
    mu = f.mean(1, keepdims=True) if plan.remove_dc_offset else 0.0
    d = f - mu
    a = plan.preemph_coeff
    pre = d - a * np.concatenate((d[:, :1], d[:, :-1]), 1) if a != 0.0 else d
    y = pre * win
    e = (d * d).sum(1) if plan.raw_energy else (y * y).sum(1)
    X = np.fft.rfft(y, n=N)
    P = X.real ** 2 + X.imag ** 2
    v = np.sqrt(P) if plan.use_fft_mag else P
    G = np.asarray(G, dtype=np.float64)
    ecol = energy_col(plan, G.shape[1])
    g_le = G[:, ecol] if plan.use_energy else np.zeros(G.shape[0])
    if plan.feature in ("fbank", "mfcc"):
        mel = v @ fb
        if plan.feature == "fbank":
            gml = np.delete(G, ecol, 1) if plan.use_energy else G
        else:
            gc = G.copy()
            if plan.use_energy:
                gc[:, ecol] = 0.0
            if lifter is not None:
                gc = gc * lifter
            gml = gc @ dct.T
        gv = (gml * _dlog_max(mel, plan.mel_floor)) @ fb.T
    else:
        gv = G.copy()
        if plan.feature == "log-spectrogram":
            gv = gv * (_dlog_max(v, -plan.log_spec_eps) if plan.log_spec_eps < 0 else 1.0 / (v + plan.log_spec_eps))
        if plan.use_energy:
            gv[:, 0] = 0.0
    if plan.energy_style == ENERGY_KALDI:
        lv = np.log(np.maximum(e, EPS32))
        ge = g_le * _dlog_max(e, EPS32)
    else:
        lv = np.log(e + 1e-15)
        ge = g_le / (e + 1e-15)
    if energy_floor_binds(plan):
        fl = math.log(plan.energy_floor)
        ge = ge * np.where(lv > fl, 1.0, np.where(lv == fl, 0.5, 0.0))
    if plan.use_fft_mag:
        A = v
        Z = np.where(A > 0, 0.5 * gv / np.where(A > 0, A, 1.0), 0.0) * X
    else:
        Z = gv * X
    H = Z.copy()
    H[:, 0] = 2.0 * Z[:, 0].real
    if N % 2 == 0:
        H[:, N // 2] = 2.0 * Z[:, N // 2].real
    gy = N * np.fft.irfft(H, n=N)[:, :L]
    if plan.use_energy and not plan.raw_energy:
        gy = gy + 2.0 * ge[:, None] * y
    gpre = gy * win
    gd = gpre.copy()
    if a != 0.0:
        gd[:, :-1] -= a * gpre[:, 1:]
        gd[:, 0] -= a * gpre[:, 0]
    if plan.use_energy and plan.raw_energy:
        gd = gd + 2.0 * ge[:, None] * d
    if plan.remove_dc_offset:
        gd = gd - gd.mean(1, keepdims=True)
    gx = np.zeros(n)
    np.add.at(gx, idx, gd)
    return gx


def conditioned(x: np.ndarray, cfg, G: np.ndarray, rel: float = 1e-6) -> np.ndarray:
    """G with the log-spectrogram bins at a log singularity (|X| or |X|^2 below `rel` times the frame's largest, e.g. the
    Nyquist bin of a mirror-symmetric edge frame, exactly 0 in exact arithmetic) left without gradient: there d log v / dv
    amplifies the last bit of v, and no two correct implementations agree."""
    if cfg.feature != "log-spectrogram":
        return G
    L, S, N = O.layer_sizes(cfg)
    win = O._cached_tables(astuple(cfg), torch.float64)[0].numpy()
    f = x[O.frame_index_matrix(x.shape[0], L, S, cfg.snip_edges)]
    if cfg.remove_dc_offset:
        f = f - f.mean(1, keepdims=True)
    if cfg.preemph_coeff != 0.0:
        f = f - cfg.preemph_coeff * np.concatenate((f[:, :1], f[:, :-1]), 1)
    v = np.abs(np.fft.rfft(f * win, n=N))
    if not cfg.use_fft_mag:
        v = v * v
    G = G.copy()
    G[v < rel * v.max(1, keepdims=True)] = 0.0
    return G


def rel_err(a, b) -> float:
    nb = float(np.linalg.norm(b))
    return float(np.linalg.norm(np.asarray(a) - np.asarray(b))) / (nb if nb > 0 else 1.0)


# ----------------------------------------------------------------------------- the B200 classes for an oracle config
def b200_extractor(cfg: O.OracleConfig, device="cuda", kernel="auto"):
    import lhotse_b200 as lb

    cls, ccls = {"fbank": (lb.B200Fbank, lb.B200FbankConfig), "mfcc": (lb.B200Mfcc, lb.B200MfccConfig),
                 "spectrogram": (lb.B200Spectrogram, lb.B200SpectrogramConfig),
                 "log-spectrogram": (lb.B200LogSpectrogram, lb.B200LogSpectrogramConfig)}[cfg.feature]
    d = {k: v for k, v in dataclasses.asdict(cfg).items() if k in ccls.__dataclass_fields__ and k != "num_mel_bins"}
    d.update(device=device, kernel=kernel)
    import warnings

    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        return cls(ccls(**d))


# ----------------------------------------------------------------------------- host harness
def host_check_binary(tmp_dir):
    """scripts/micro/backward_host_check.cu compiled for the host (with AddressSanitizer where the toolchain has it), or
    None without a C++ compiler."""
    src = os.path.join(ROOT, "scripts", "micro", "backward_host_check.cu")
    exe = os.path.join(str(tmp_dir), "backward_host_check")
    gxx = shutil.which("g++")
    if not gxx:
        return None
    for flags in (["-fsanitize=address", "-fno-omit-frame-pointer"], []):
        res = subprocess.run([gxx, "-x", "c++", "-std=c++17", "-O1", "-g", *flags, "-o", exe, src], capture_output=True, text=True)
        if res.returncode == 0:
            return exe
    raise RuntimeError("backward_host_check does not compile:\n" + res.stderr)


def host_check_input(path, cfg, x: np.ndarray, G: np.ndarray):
    """The harness's input file: int32 header, float32 scalars, then the float32 tables, the waveform and the row gradient.
    `cfg` is an oracle config (its float32 tables) or a FeaturePlan, whose energy style, energy column, mel shift and
    log-spectrogram floor the header then carries (b200feat.cu bwd_plan)."""
    plan = oracle_plan(cfg, torch.float32) if isinstance(cfg, O.OracleConfig) else cfg
    L, S, N = plan.L, plan.S, plan.N
    feat = {"fbank": 0, "mfcc": 1, "spectrogram": 2, "log-spectrogram": 3}[plan.feature]
    M = plan.num_filters if feat in (0, 1) else 0
    C = plan.num_ceps if feat == 1 else 0
    T, F = G.shape
    use_lifter = int(feat == 1 and plan.lifter is not None)
    ecol = energy_col(plan, F) if plan.use_energy else 0
    shift = 1 if (feat == 0 and plan.use_energy and not plan.energy_last) else 0
    hdr = np.asarray([feat, L, S, N, M, C, F, int(plan.snip_edges), int(plan.remove_dc_offset), int(plan.use_energy),
                      int(plan.raw_energy), int(plan.use_fft_mag), int(plan.energy_style), use_lifter, ecol, shift, x.shape[0], T,
                      (L - S) // 2, 0], dtype=np.int32)
    has_floor = energy_floor_binds(plan)
    floor_form = plan.log_spec_eps < 0
    sc = np.asarray([plan.preemph_coeff, math.log(plan.energy_floor) if has_floor else 0.0, 1.0 if has_floor else 0.0,
                     plan.mel_floor, 0.0 if floor_form else plan.log_spec_eps, -plan.log_spec_eps if floor_form else 0.0],
                    dtype=np.float32)
    parts = [hdr.tobytes(), sc.tobytes(), np.asarray(plan.window, dtype=np.float32).tobytes()]
    if M:
        parts.append(np.ascontiguousarray(plan.mel_bank, dtype=np.float32).tobytes())
    if C:
        parts.append(np.ascontiguousarray(plan.dct, dtype=np.float32).tobytes())
    if use_lifter:
        parts.append(np.asarray(plan.lifter, dtype=np.float32).tobytes())
    parts += [x.astype(np.float32).tobytes(), np.ascontiguousarray(G, dtype=np.float32).tobytes()]
    with open(path, "wb") as fh:
        fh.write(b"".join(parts))
