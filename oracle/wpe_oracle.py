"""
TEST INFRASTRUCTURE — NOT PRODUCT CODE.

CPU restatement (numpy) of lhotse's `DereverbWPE` (lhotse/augmentation/wpe.py `dereverb_wpe_numpy`): torch.stft, nara_wpe's
`wpe_v8`, torch.istft, then `assert_and_maybe_fix_num_samples`.  Same rules as the other oracles: only ``tests/`` and the
CPU legs of the benchmarks may import it.

PARITY PIN — read this.  The dereverberation itself lives in a third-party dependency that is NOT in the reference tree:
**nara_wpe** (an optional extra of the reference, absent from this image).  `wpe` below restates its published `wpe_v8` /
`wpe_v7` / `get_power_inverse` / `get_filter_matrix_v7` / `_stable_solve` (and Drude et al., "NARA-WPE", ITG 2018) from
their description, as `oracle/librosa_oracle.py` restates librosa.  The tests register it as a stand-in `nara_wpe` module
(tests/wpe_cases.py) so that lhotse's own `DereverbWPE.__call__` and `signal_transforms.DereverbWPE` run end to end on it.
Two details decide edge cases and are stated here as restated:
  * get_power_inverse: power_t = mean over channels of |X_t|^2; eps = 1e-10 * max(power), the max over the frames of ONE
    frequency bin (wpe_v8 loops over the bins and calls wpe_v7 on each (D, T) slice, so np.max sees one bin); when eps == 0
    (an all-zero bin) every inverse power is 1 ("the scale of the power does not matter"), else 1 / max(power_t, eps).
    The inverse power is computed over every frame, also in "valid" mode, which only slices the statistics.
  * _stable_solve: G = np.linalg.solve(R, P); when that raises LinAlgError (an exactly singular R), np.linalg.lstsq(R, P),
    whose minimum-norm solution is G = 0 for R = 0.
Statistics, per bin, y~_t = [Y_{t-delay}, ..., Y_{t-delay-taps+1}] (channel-major within a lag, 0 before the first frame):
R = sum_{t in S} inv_t y~_t y~_t^H, P = sum_{t in S} inv_t y~_t Y_t^H, X_t = Y_t - G^H y~_t; S every frame ("full") or
t >= delay + taps - 1 ("valid").

torch.stft(x, 512, 128, window=torch.blackman_window(512), return_complex=True): centred (x reflect-padded by 256 on each
side), T = 1 + L // 128 frames, one-sided.  torch.istft(X, 512, 128, window=...): C2R inverse of every frame (imaginary parts
of bins 0 and n_fft/2 ignored), times the window, overlap-added, divided by the overlap-added squared window, 256 trimmed
from each end: 128 (T - 1) samples.  The window is torch's float32 window (element 0 is -2.98e-8), promoted exactly.
"""
from __future__ import annotations

import numpy as np


def window(n_fft: int = 512) -> np.ndarray:
    import torch

    return torch.blackman_window(n_fft).numpy().astype(np.float32)


def stft(x: np.ndarray, n_fft: int = 512, hop: int = 128, dtype=np.float64) -> np.ndarray:
    """(F, T) one-sided spectra of the 1-D signal x in `dtype` (float64: complex128; float32: complex64)."""
    x = np.asarray(x, dtype=dtype)
    xp = np.pad(x, n_fft // 2, mode="reflect")
    T = 1 + len(x) // hop
    idx = np.arange(T)[:, None] * hop + np.arange(n_fft)[None, :]
    frames = xp[idx] * window(n_fft).astype(dtype)
    Y = np.fft.rfft(frames, axis=-1)
    return Y.T.astype(np.complex128 if dtype == np.float64 else np.complex64)


def istft(X: np.ndarray, n_fft: int = 512, hop: int = 128) -> np.ndarray:
    """The 128 (T - 1) samples of torch.istft(center=True) of the (F, T) spectra, in X's precision."""
    real = np.float64 if X.dtype == np.complex128 else np.float32
    F, T = X.shape
    frames = np.fft.irfft(X.T, n=n_fft, axis=-1).astype(real) * window(n_fft).astype(real)
    n = n_fft + hop * (T - 1)
    y = np.zeros(n, real)
    env = np.zeros(n, real)
    w2 = window(n_fft).astype(real) ** 2
    for t in range(T):
        y[t * hop: t * hop + n_fft] += frames[t]
        env[t * hop: t * hop + n_fft] += w2
    return (y / env)[n_fft // 2: n - n_fft // 2]


def _stable_solve(R: np.ndarray, P: np.ndarray) -> np.ndarray:
    try:
        return np.linalg.solve(R, P)
    except np.linalg.LinAlgError:
        return np.linalg.lstsq(R, P, rcond=None)[0]


def wpe_bin(Y: np.ndarray, taps: int = 10, delay: int = 3, iterations: int = 3, statistics_mode: str = "full") -> np.ndarray:
    """wpe_v7 on one bin's (D, T) spectra, in Y's precision."""
    D, T = Y.shape
    Yt = np.zeros((taps, D, T), Y.dtype)  # y~_t, lag-major
    for k in range(taps):
        s = delay + k
        if s < T:
            Yt[k, :, s:] = Y[:, : T - s]
    Yt = Yt.reshape(taps * D, T)
    sl = slice(None) if statistics_mode == "full" else slice(delay + taps - 1, None)
    X = Y
    for _ in range(iterations):
        power = np.mean(np.abs(X) ** 2, axis=0)
        eps = 1e-10 * np.max(power)
        inv = np.ones_like(power) if eps == 0 else 1 / np.maximum(power, eps)
        Ytw = Yt[:, sl] * inv[sl]
        R = Ytw @ Yt[:, sl].conj().T
        P = Ytw @ Y[:, sl].conj().T
        G = _stable_solve(R, P)
        X = Y - G.conj().T @ Yt
    return X


def wpe_v8(Y: np.ndarray, taps: int = 10, delay: int = 3, iterations: int = 3, psd_context: int = 0,
           statistics_mode: str = "full") -> np.ndarray:
    """nara_wpe.wpe.wpe_v8 on (..., D, T) spectra: every leading index (the frequency bins) on its own."""
    if psd_context != 0:
        raise NotImplementedError("psd_context")
    Y = np.asarray(Y)
    out = np.empty_like(Y)
    for index in np.ndindex(Y.shape[:-2]):
        out[index] = wpe_bin(Y[index], taps, delay, iterations, statistics_mode)
    return out


def length_fix(z: np.ndarray, target_len: int) -> np.ndarray:
    """lhotse's assert_and_maybe_fix_num_samples: np.pad(mode="reflect") up to target_len, or trim."""
    if target_len > len(z):
        return np.pad(z, (0, target_len - len(z)), mode="reflect")
    return z[:target_len]


def dereverb(x: np.ndarray, target_len: int = None, dtype=np.float64, taps: int = 10, delay: int = 3, iterations: int = 3,
             statistics_mode: str = "full") -> np.ndarray:
    """The whole chain on the 1-D signal x in `dtype` (float64: the truth; float32: complex64 arithmetic throughout), then
    the length fix to `target_len` (None: none)."""
    Y = stft(x, dtype=dtype)
    X = wpe_v8(Y[:, None, :], taps=taps, delay=delay, iterations=iterations, statistics_mode=statistics_mode)[:, 0, :]
    z = istft(X)
    return z if target_len is None else length_fix(z, target_len)
