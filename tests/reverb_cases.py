"""Test-only: seeded RIR fixtures and the two references of the reverb route's tolerance contract (DESIGN.md §3.1j): the
float64 truth, and lhotse's own float32 ReverbWithImpulseResponse arithmetic, whose distance to the truth sets the bound."""
import wave

import numpy as np

NOISE_X = 2        # the bound is this many times the float32 reference's own error (tests/helpers.py uses the same factor)
FLOOR = 1e-6       # ... or this fraction of the truth's peak, whichever is larger


def decaying_rir(n, seed, peak_at=None, channels=1):
    """int16 [n] (or [n, channels]): exponentially decaying noise whose first maximum sits at `peak_at` (default: a few
    samples in, where a recorded RIR has its direct path)."""
    rs = np.random.RandomState(seed)
    t = np.arange(n)
    q = np.empty((n, channels), np.int16)
    for c in range(channels):
        env = np.exp(-t / max(1.0, 0.15 * n))
        q[:, c] = np.clip(rs.randn(n) * env * 12000, -30000, 30000).astype(np.int16)
        at = min(n - 1, 3 + 7 * c) if peak_at is None else peak_at
        q[at, c] = 32767
        if at + 5 < n:
            q[at + 5, c] = 32767  # a tie: the first index wins
    return q if channels > 1 else q[:, 0]


def write_wav(path, q, sr=16000):
    q = np.asarray(q, dtype="<i2")
    with wave.open(str(path), "wb") as w:
        w.setnchannels(1 if q.ndim == 1 else q.shape[1]); w.setsampwidth(2); w.setframerate(sr)
        w.writeframes(q.tobytes())


def length_fix(y, target):
    """lhotse's assert_and_maybe_fix_num_samples / MixedCut fix: trim, or np.pad(mode="reflect")."""
    n = y.shape[0]
    if target <= n:
        return y[:target]
    return np.pad(y, (0, target - n), mode="reflect")


def truth64(x, q, normalize=True, target=None):
    """The reverb of float32 x with the int16 RIR q in float64: scipy's float64 FFT convolution, the shift, the gain."""
    from scipy.signal import fftconvolve

    x64 = np.asarray(x, np.float64)
    h = q.astype(np.float64) / 32768.0 * 0.5 ** 15
    s = int(np.argmax(q))
    n = x64.shape[0]
    y = fftconvolve(x64, h)[s: s + n] if n else x64
    if normalize and n:
        pb, pa = np.sum(x64 ** 2) / n, np.sum(y ** 2) / n
        if pa > 0:
            y = y * np.sqrt(pb / pa)
    return length_fix(y, n if target is None else target)


def lhotse32(x, q, normalize=True, target=None):
    """ReverbWithImpulseResponse.__call__ for a mono input and RIR, step for step in float32, with lhotse's own convolve1d
    (needs the reference)."""
    import torch
    from lhotse.augmentation.utils import convolve1d

    samples = np.asarray(x, np.float32)[None]
    rir = (q.astype(np.float32) / np.float32(32768))[None] * 0.5 ** 15
    n = samples.shape[1]
    out = np.zeros_like(samples)
    pb = np.sum(np.abs(samples[0]) ** 2) / n
    aug = convolve1d(torch.from_numpy(samples[0]), torch.from_numpy(rir[0])).numpy()
    s = np.argmax(rir[0])
    out[0, :] = aug[s: s + n]
    if normalize:
        pa = np.sum(np.abs(out[0]) ** 2) / n
        if pa > 0:
            out[0] *= np.sqrt(pb / pa)
    return length_fix(out[0], n if target is None else target)


def bound(truth, ref32):
    return max(NOISE_X * float(np.abs(ref32.astype(np.float64) - truth).max(initial=0.0)),
               FLOOR * float(np.abs(truth).max(initial=0.0)))


def check(got, truth, ref32, what=""):
    assert got.shape == truth.shape, (what, got.shape, truth.shape)
    err = float(np.abs(got.astype(np.float64) - truth).max(initial=0.0))
    b = bound(truth, ref32)
    assert err <= b, (what, err, b)
    return err, b
