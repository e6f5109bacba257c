"""Test-only helpers for the WPE route (csrc/wpe.cuh): a stand-in `nara_wpe` module, test signals, the float64 truth, lhotse's
float32 chain, the per-cut bound, and a runner for `engine.wpe` on a list of signals."""
import importlib.machinery
import sys
import types

import numpy as np

import refshim  # noqa: F401  (puts the repository root on sys.path)
from oracle import wpe_oracle as W

DEFAULT = dict(taps=10, delay=3, iterations=3, statistics_mode="full")


def install_nara_wpe_standin():
    """lhotse's DereverbWPE needs nara_wpe (absent from this image): register a stand-in whose `wpe.wpe_v8` and
    `torch_wpe.wpe_v6` are the restatement of oracle/wpe_oracle.py, in the precision of their input (complex64 in lhotse's
    calls).  A `__spec__` makes lhotse's `is_module_available("nara_wpe")` see it.  The real package, when installed, is
    left alone."""
    if "nara_wpe" in sys.modules and not getattr(sys.modules["nara_wpe"], "_b200_standin", False):
        return

    def wpe_v6(Y, taps=10, delay=3, iterations=3, psd_context=0, statistics_mode="full"):
        import torch

        Z = W.wpe_v8(Y.detach().cpu().numpy(), taps=taps, delay=delay, iterations=iterations, psd_context=psd_context,
                     statistics_mode=statistics_mode)
        return torch.from_numpy(Z).to(Y.device)

    pkg = types.ModuleType("nara_wpe")
    pkg.__spec__ = importlib.machinery.ModuleSpec("nara_wpe", None, is_package=True)
    pkg.__path__ = []
    pkg._b200_standin = True
    pkg.wpe = types.ModuleType("nara_wpe.wpe")
    pkg.wpe.__spec__ = importlib.machinery.ModuleSpec("nara_wpe.wpe", None)
    pkg.wpe.wpe_v8 = W.wpe_v8
    pkg.torch_wpe = types.ModuleType("nara_wpe.torch_wpe")
    pkg.torch_wpe.__spec__ = importlib.machinery.ModuleSpec("nara_wpe.torch_wpe", None)
    pkg.torch_wpe.wpe_v6 = wpe_v6
    sys.modules["nara_wpe"] = pkg
    sys.modules["nara_wpe.wpe"] = pkg.wpe
    sys.modules["nara_wpe.torch_wpe"] = pkg.torch_wpe


def signal(kind: str, n: int, seed: int = 0) -> np.ndarray:
    """float32 test signals: "noise" (N(0, 0.1^2)), "reverb" (noise bursts convolved with a decaying RIR, so that the
    filter is far from 0), "silence" (leading digital silence, then a reverberant tail: the eps floor binds), "zero",
    "full" (full-scale int16 values)."""
    rs = np.random.RandomState(seed)
    if kind == "zero":
        return np.zeros(n, np.float32)
    if kind == "noise":
        return (0.1 * rs.randn(n)).astype(np.float32)
    if kind == "full":
        return (np.clip(np.round(rs.randn(n) * 30000), -32768, 32767) / 32768.0).astype(np.float32)
    bursts = np.zeros(n)
    for a in range(0, n, 4000):
        bursts[a: a + 800] = rs.randn(min(800, n - a))
    t = np.arange(4000) / 16000.0
    rir = rs.randn(4000) * np.exp(-t / 0.08)
    rir[0] = 3.0
    y = np.convolve(bursts, rir)[:n]
    y = 0.3 * y / max(np.abs(y).max(), 1e-9)
    if kind == "silence":
        y[: min(n // 3, 12000)] = 0.0
    return y.astype(np.float32)


def truth64(x: np.ndarray, target_len=None, **p) -> np.ndarray:
    """The float64 restatement on the float32 samples x."""
    return W.dereverb(np.asarray(x, np.float32).astype(np.float64), target_len, np.float64, **{**DEFAULT, **p})


def lhotse32(x: np.ndarray, target_len=None, **p) -> np.ndarray:
    """lhotse's own float32 chain (DereverbWPE.__call__ -> dereverb_wpe_numpy) on the stand-in, then the length fix.  Needs
    the reference imported (refshim.import_reference)."""
    from lhotse.augmentation.wpe import DereverbWPE

    install_nara_wpe_standin()
    z = DereverbWPE(**{**DEFAULT, **p})(np.asarray(x, np.float32)[None, :], 16000)[0]
    return z if target_len is None else W.length_fix(z, target_len)


def bound(ours, t64, l32):
    """(ok, err, limit): max|ours - truth64| <= max(2 max|lhotse32 - truth64|, 1e-6 max|truth64|) (DESIGN.md §3.1q)."""
    ours, t64, l32 = (np.asarray(a, np.float64) for a in (ours, t64, l32))
    assert ours.shape == t64.shape == l32.shape, (ours.shape, t64.shape, l32.shape)
    err = float(np.max(np.abs(ours - t64))) if ours.size else 0.0
    lim = max(2.0 * float(np.max(np.abs(l32 - t64))) if ours.size else 0.0, 1e-6 * float(np.max(np.abs(t64), initial=0.0)))
    return bool(err <= lim), err, lim


def run_wpe(xs, targets=None, device="cuda:0", sentinel=np.float32(-7.25), **p):
    """engine.wpe on the float32 signals xs (back to back in one input buffer), outputs back to back (gaps of 3 samples
    holding `sentinel`) with targets (default 128 (L // 128)).  Returns ([output per cut], output buffer as numpy)."""
    import torch

    from lhotse_b200.engine import WPE_CUT_DTYPE, wpe

    targets = [128 * (len(x) // 128) for x in xs] if targets is None else list(targets)
    ct = np.zeros(len(xs), WPE_CUT_DTYPE)
    ct["struct_size"] = WPE_CUT_DTYPE.itemsize
    ct["in_len"] = [len(x) for x in xs]
    ct["in_elem"] = np.concatenate(([0], np.cumsum([len(x) for x in xs])[:-1])).astype(np.int64)
    ct["target_len"] = targets
    ct["out_elem"] = np.concatenate(([0], np.cumsum([t + 3 for t in targets])[:-1])).astype(np.int64)
    x = torch.from_numpy(np.concatenate(xs).astype(np.float32)).to(device)
    out = torch.full((int(sum(targets)) + 3 * len(xs),), float(sentinel), dtype=torch.float32, device=device)
    wpe(x, ct, out, **{**DEFAULT, **p})
    host = out.cpu().numpy()
    return [host[o: o + t] for o, t in zip(ct["out_elem"], targets)], host
