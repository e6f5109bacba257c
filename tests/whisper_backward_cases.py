"""Shared pieces of the whisper-fbank backward tests (csrc/backward.cuh, DESIGN.md §3.1p): the waveforms and lengths they
sweep, a float64 autograd twin of `oracle.whisper_oracle.extract` (a tensor out, so that autograd runs it), a float64 NumPy
restatement of the adjoint chain written the way the kernels compute it, and the host harness
(scripts/micro/whisper_backward_host_check.cu) with its input file."""
from __future__ import annotations

import functools
import math
import os
import shutil
import subprocess

import numpy as np
import torch

from oracle import whisper_oracle as W

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
N_FFT, HOP, FLOOR = W.N_FFT, W.HOP, 1e-10
LN10 = math.log(10.0)
LENGTHS = (201, 160000, 160079, 160080, 160159)  # shortest cut, 10 s, the zero-row boundary and its neighbours


def waveform(n, kind="noise", seed=0):
    """noise; burst: a loud first fifth then a tail 80 dB down, so that the clamp to m - 8 binds on part of the cut;
    periodic: a hop-periodic tone, so that the maximum ties across the interior frames; silence."""
    rs = np.random.RandomState(seed + n)
    if kind == "silence":
        return np.zeros(n)
    if kind == "burst":
        x = 1e-4 * rs.randn(n)
        x[: max(n // 5, 1)] *= 1e4
        return x
    if kind == "periodic":
        period = 0.3 * rs.randn(HOP // 4)
        return np.tile(period, n // period.size + 1)[:n]
    return 0.1 * rs.randn(n)


@functools.lru_cache(maxsize=16)
def tables(num_filters, dtype=torch.float64, device="cpu"):
    """The oracle's window and (M, K) filters in `dtype` on `device`: float32 tables cast, as WhisperFbank's are on a
    float64 run."""
    return (torch.hann_window(N_FFT).to(dtype=dtype, device=device),
            torch.from_numpy(W.slaney_mel_filters(num_filters)).to(dtype=dtype, device=device))


# ----------------------------------------------------------------------------- float64 autograd twin of W.extract
def logmel_t(a: torch.Tensor, num_filters=80):
    """The (T, M) log10 mel rows before the clamp, of W.extract's chain on a tensor (in the dtype of a)."""
    window, filters = tables(num_filters, a.dtype, str(a.device))
    a = a.reshape(-1)
    padded = torch.nn.functional.pad(a.view(1, 1, -1), (N_FFT // 2, N_FFT // 2), mode="reflect").view(-1)
    frames = padded.unfold(0, N_FFT, HOP)[:-1]
    power = torch.fft.rfft(frames * window, dim=-1).abs() ** 2
    return torch.clamp(filters @ power.T, min=FLOOR).log10().T


def features_t(a: torch.Tensor, num_filters=80) -> torch.Tensor:
    """W.extract's chain on a tensor, returning a tensor: autograd runs it."""
    n = a.numel()
    v = logmel_t(a, num_filters).T
    v = torch.maximum(v, v.max() - 8.0)
    v = (v + 4.0) / 4.0
    rows = W.num_rows(n)
    if rows > v.shape[1]:
        v = torch.nn.functional.pad(v, (0, rows - v.shape[1]), mode="constant")
    return v.T


def autograd_grad(x: np.ndarray, G: np.ndarray, num_filters=80, dtype=torch.float64, device="cpu") -> np.ndarray:
    """d sum(features * G) / dx through `features_t`."""
    xt = torch.tensor(np.asarray(x, dtype=np.float64), dtype=dtype, device=device, requires_grad=True)
    (features_t(xt, num_filters) * torch.as_tensor(G, dtype=dtype, device=device)).sum().backward()
    return xt.grad.double().cpu().numpy()


# ----------------------------------------------------------------------------- float64 restatement of the adjoint chain
def frame_index(n):
    """(T, N) sample index of every tap of the stft's n / S centred frames: torch's "reflect", the edge not repeated."""
    q = np.arange(n // HOP)[:, None] * HOP - N_FFT // 2 + np.arange(N_FFT)[None, :]
    q = np.where(q < 0, -q, q)
    return np.where(q >= n, 2 * n - 2 - q, q)


def row_grad(x: np.ndarray, m: float, G: np.ndarray) -> np.ndarray:
    """Rule 1: the gradient reaching the log-mel values x (cut maximum m) from the gradient G of (maximum(x, m - 8) + 4) / 4:
    g / 4 weighted 1, 1/2 or 0, plus the mass routed to m - 8 spread evenly over the elements equal to m."""
    thr = m - 8.0
    w = np.where(x > thr, 1.0, np.where(x == thr, 0.5, 0.0))
    q = G / 4.0
    routed = float((q * (1.0 - w)).sum())
    ties = int((x == m).sum())
    return q * w + np.where(x == m, routed / ties, 0.0)


def log10_adjoint(v: np.ndarray, gx: np.ndarray) -> np.ndarray:
    """Rule 2: log10(clamp(v, min=1e-10)) passes gx / (v ln 10) where v >= 1e-10, the tie included, and 0 below."""
    return np.where(v >= FLOOR, gx / (np.where(v > 0, v, 1.0) * LN10), 0.0)


def restated_grad(x: np.ndarray, G: np.ndarray, num_filters=80, xr: np.ndarray = None, m: float = None) -> np.ndarray:
    """The kernels' adjoint chain in float64 with the oracle's tables cast to float64.  `xr` and `m`: the log-mel rows and
    maximum the decisions of rule 1 are taken on (default: the chain's own float64 values)."""
    x = np.asarray(x, dtype=np.float64)
    n = x.shape[0]
    T = n // HOP
    window, filters = (t.numpy() for t in tables(num_filters))
    fb = filters.T  # (K, M)
    idx = frame_index(n)
    y = x[idx] * window
    X = np.fft.rfft(y, n=N_FFT)
    v = (X.real ** 2 + X.imag ** 2) @ fb
    if xr is None:
        xr = np.log10(np.maximum(v, FLOOR))
        m = float(xr.max())
    gv = log10_adjoint(v, row_grad(np.asarray(xr, dtype=np.float64)[:T], m, np.asarray(G, dtype=np.float64)[:T]))
    Z = (gv @ fb.T) * X
    H = Z.copy()
    H[:, 0] = 2.0 * Z[:, 0].real
    H[:, N_FFT // 2] = 2.0 * Z[:, N_FFT // 2].real
    gy = N_FFT * np.fft.irfft(H, n=N_FFT)
    gx = np.zeros(n)
    np.add.at(gx, idx, gy * window)
    return gx


def rel_err(a, b) -> float:
    nb = float(np.linalg.norm(b))
    return float(np.linalg.norm(np.asarray(a) - np.asarray(b))) / (nb if nb > 0 else 1.0)


def saved_rows(x: np.ndarray, num_filters=80):
    """The float32 log-mel rows and maximum of the float32 chain: what the forward keeps, up to its own rounding."""
    xr = logmel_t(torch.tensor(np.asarray(x, dtype=np.float32)), num_filters).numpy()
    return xr, float(xr.max())


# ----------------------------------------------------------------------------- the B200 class on the GPU
def extractor(kernel="auto", M=80):
    import lhotse_b200 as lb

    return lb.B200WhisperFbank(lb.B200WhisperFbankConfig(num_filters=M, kernel=kernel))


def loss(feats, G):
    return (feats * torch.as_tensor(G, dtype=feats.dtype, device=feats.device)).sum()


def b200_grad(ext, x, G, dtype=torch.float32, device="cuda"):
    """d sum(features * G) / dx of one cut through `extract`, as float64 NumPy."""
    xt = torch.tensor(np.asarray(x), dtype=dtype, device=device, requires_grad=True)
    loss(ext.extract(xt, 16000), G).backward()
    return xt.grad.double().cpu().numpy()


def b200_grads(ext, xs, Gs):
    """float32 gradients (CUDA tensors) of sum_i <features(x_i), G_i> over one `extract_batch` call on the list `xs`."""
    leaves = [torch.tensor(np.asarray(x), dtype=torch.float32, device="cuda", requires_grad=True) for x in xs]
    outs = ext.extract_batch(leaves, 16000)
    sum(loss(o, G) for o, G in zip(outs, Gs)).backward()
    return [t.grad for t in leaves]


def case(n, kind, M, seed=0):
    """A waveform and a row gradient whose decisions agree across precisions: G is 0 on values within 1e-3 of m - 8 or of
    the floor's log (-10), and the cut's maximum is unique by 1e-3 (asserted)."""
    x = waveform(n, kind, seed).astype(np.float32).astype(np.float64)
    xr = logmel_t(torch.tensor(x), M).numpy()
    m = xr.max()
    top = np.sort(xr.ravel())[-2:] if xr.size > 1 else np.asarray([-np.inf, m])
    assert top[1] - top[0] > 1e-3, (n, kind, M)
    G = np.random.RandomState(n + M + seed).randn(W.num_rows(n), M)
    near = (np.abs(xr - (m - 8.0)) < 1e-3) | (np.abs(xr + 10.0) < 1e-3)
    G[: xr.shape[0]][near] = 0.0
    return x, G


def gate(x, G, M, g):
    """(||g - g64||, the bound 8 ||g32 - g64|| + 1e-7 ||g64||, ||g32 - g64||): g64 float64 autograd through the oracle's
    chain, g32 the same chain in float32 on the GPU."""
    g64 = autograd_grad(x, G, M)
    g32 = autograd_grad(x, G, M, dtype=torch.float32, device="cuda")
    err, err32 = float(np.linalg.norm(g - g64)), float(np.linalg.norm(g32 - g64))
    return err, 8.0 * err32 + 1e-7 * float(np.linalg.norm(g64)), err32

# ----------------------------------------------------------------------------- host harness
def host_check_binary(tmp_dir):
    """scripts/micro/whisper_backward_host_check.cu compiled for the host (with AddressSanitizer where the toolchain has
    it), or None without a C++ compiler."""
    src = os.path.join(ROOT, "scripts", "micro", "whisper_backward_host_check.cu")
    exe = os.path.join(str(tmp_dir), "whisper_backward_host_check")
    gxx = shutil.which("g++")
    if not gxx:
        return None
    for flags in (["-fsanitize=address", "-fno-omit-frame-pointer"], []):
        res = subprocess.run([gxx, "-x", "c++", "-std=c++17", "-O1", "-g", *flags, "-o", exe, src], capture_output=True, text=True)
        if res.returncode == 0:
            return exe
    raise RuntimeError("whisper_backward_host_check does not compile:\n" + res.stderr)


def host_check_input(path, x: np.ndarray, xr: np.ndarray, m: float, G: np.ndarray, num_filters=80):
    """The harness's input file: int32 [M n R], float32 [m], then the float32 window [N], mel bank [K][M], samples [n],
    log-mel rows [R][M] and row gradient [R][M]."""
    n = x.shape[0]
    R = G.shape[0]
    window, filters = tables(num_filters, torch.float32)
    rows = np.zeros((R, num_filters), dtype=np.float32)
    rows[: xr.shape[0]] = xr
    parts = [np.asarray([num_filters, n, R], dtype=np.int32).tobytes(), np.asarray([m], dtype=np.float32).tobytes(),
             window.numpy().tobytes(), np.ascontiguousarray(filters.numpy().T).tobytes(), x.astype(np.float32).tobytes(),
             rows.tobytes(), np.ascontiguousarray(G, dtype=np.float32).tobytes()]
    with open(path, "wb") as fh:
        fh.write(b"".join(parts))


def run_host_check(exe, tmp_path, x, xr, m, G, num_filters=80) -> np.ndarray:
    inp, out = str(tmp_path / "in.bin"), str(tmp_path / "out.f32")
    host_check_input(inp, x, xr, m, G, num_filters)
    res = subprocess.run([exe, inp, out], capture_output=True, text=True)
    assert res.returncode == 0, res.stdout + res.stderr
    return np.fromfile(out, dtype=np.float32)
