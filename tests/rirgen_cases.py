"""Shared by the RIR generator tests: seeded lhotse generators, lhotse's own RIR for the same generator state (float32, one
torch thread), and the float64 truth of the same draws (DESIGN.md §3.1l)."""
import copy
import math

import numpy as np
import torch

# (sr, max_T60, room_seed, source_seed): T60 near both ends of its range, the three rates, and seeds whose images collide
CASES = [
    (16000, 0.8, 1, 2),
    (16000, 0.1001, 3, 4),   # T60 in [0.1, 0.1001): the shortest RIRs
    (8000, 0.8, 5, 6),
    (48000, 0.8, 7, 8),
    (16000, 0.8, 11, 12),
    (16000, 0.3, 13, 14),
]


def generator(sr, max_t60, room_seed, source_seed):
    from lhotse.augmentation.utils import FastRandomRIRGenerator

    return FastRandomRIRGenerator(sr=sr, max_T60=max_t60, room_seed=room_seed, source_seed=source_seed)


def lhotse_rir(gen):
    """What lhotse's generator returns for a copy of `gen` from torch's current state, with one torch thread (the float
    route's last-wins comb; see DESIGN.md §3.1l).  Returns (rir, the copy, torch's state after)."""
    g = copy.deepcopy(gen)
    n = torch.get_num_threads()
    torch.set_num_threads(1)
    try:
        rir = g(nsource=1)[0]
    finally:
        torch.set_num_threads(n)
    return rir, g, torch.get_rng_state()


def _table64(orig_over_new=8):
    """lhotse's 8 -> 1 resampler table in float64, before its float32 rounding."""
    O, N = orig_over_new, 1
    width = math.ceil(6 * O / (min(O, N) * 0.99))
    base = min(O, N) * 0.99
    u = (torch.arange(0, -N, -1) / N)[:, None] + torch.arange(-width, width + O, dtype=torch.float64)[None, :] / O
    u = (u * base).clamp(-6, 6)
    hann = torch.cos(u * math.pi / 6 / 2) ** 2
    u = u * math.pi
    w = torch.where(u == 0, torch.tensor(1.0).to(u), u.sin() / u) * hann * (base / O)
    return w[0].numpy(), width


def _resample64(x, n_out):
    tab, width = _table64()
    K = tab.shape[0]
    xp = np.concatenate([np.zeros(width), x, np.zeros(width + 8 + K)])
    j = np.arange(n_out)
    out = np.zeros(n_out)
    for t in range(K):
        out += xp[8 * j + t] * tab[t]
    return out


def _sparse_resample64(pos, val, n_out):
    tab, width = _table64()
    out = np.zeros(n_out)
    for t in range(tab.shape[0]):
        # entry at comb position p feeds output j through tap t = p - 8 j + width
        num = pos + width - t
        ok = (num % 8 == 0)
        j = num[ok] // 8
        keep = (j >= 0) & (j < n_out)
        np.add.at(out, j[keep], val[ok][keep] * tab[t])
    return out


def truth64(rec, u, pert, gen):
    """The RIR of one draw record through a float64 comb (lhotse's positions, float64 decays, last wins), the float64
    resampler, scipy's lfilter with float64 coefficients, the clamp and the second resampler."""
    import scipy.signal

    from lhotse_b200 import rir_draws
    from lhotse_b200.pcm_staging import resampled_len

    sr = int(rec["sampling_rate"])
    image = 2 * sr
    S = 64 * sr
    t60, R, d0 = float(rec["t60"]), float(rec["r"]), float(rec["d0"])
    L = int(rec["comb_len"])
    cdf = rir_draws.multinomial_cdf(gen.alpha, image)
    idx = rir_draws.multinomial_from_uniforms(cdf, u)
    ratio = torch.linspace(1.0, torch.tensor(340.0 * t60 / d0 - 1, dtype=torch.float64), image).numpy()[idx].astype(np.float64)
    coef = math.sqrt(1 - (1 - math.exp(-0.16 * R / t60)) ** 2)
    rmax = (math.log10(340.0 * t60) - math.log10(d0) - 3) / math.log10(coef + 2.0 ** -10)
    dist = d0 * ratio
    refl = (dist / (340.0 * t60)) ** 2 * (rmax - 1) + 1
    refl = np.maximum(refl + pert * ratio.astype(np.float32).astype(np.float64) ** gen.tau, 1.0)
    dist = np.concatenate([[d0], dist])
    refl = np.concatenate([[0.0], refl])
    pos = np.minimum(np.ceil(dist * S / 340.0), L - 1).astype(np.int64)
    dec = coef ** refl / dist
    last = {}
    for p, v in zip(pos.tolist(), dec.tolist()):
        last[p] = v
    up = np.fromiter(last.keys(), np.int64)
    uv = np.fromiter(last.values(), np.float64)
    n8 = resampled_len(1, L, 8)
    x8 = _sparse_resample64(up, uv, n8)
    w0 = 2 * math.pi * 80.0 / (8 * sr)
    alpha = math.sin(w0) / 2.0 / 0.707
    b = np.array([(1 + math.cos(w0)) / 2, -1 - math.cos(w0), (1 + math.cos(w0)) / 2])
    a = np.array([1 + alpha, -2 * math.cos(w0), 1 - alpha])
    y = np.clip(scipy.signal.lfilter(b / a[0], a / a[0], x8), -1.0, 1.0)
    return _resample64(y, resampled_len(1, n8, 8)), pos, dec


def bound(ours, lhotse32, truth):
    """The §3.1j contract: max|ours - truth| <= max(2 max|lhotse32 - truth|, 1e-6 max|truth|).  Returns (ours' error, the
    bound)."""
    ref = 2 * float(np.max(np.abs(lhotse32.astype(np.float64) - truth)))
    return float(np.max(np.abs(ours.astype(np.float64) - truth))), max(ref, 1e-6 * float(np.max(np.abs(truth))))
