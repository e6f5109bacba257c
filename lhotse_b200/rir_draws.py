"""The random draws of lhotse's FastRandomRIRGenerator (lhotse/augmentation/utils.py) for a batch of generated RIRs, made on
the host in lhotse's order and from lhotse's generator state, so that the GPU generator (csrc/rirgen.cuh) builds the RIRs
the float route would build and every generator ends where the float route leaves it (DESIGN.md §3.1l).

Per RIR, in batch order, `FastRandomRIRGenerator.__call__(nsource=1)` draws: room_rng.uniform for T60, room_rng.uniform for
R, source_rng.uniform for d0, `torch.multinomial` on torch's global CPU generator for the 2 sr image indices, then
source_rng.uniform for the 2 sr perturbations.  The NumPy draws are made from the generator object attached to the cut's
transform.  The multinomial is restated instead of called per RIR: its uniforms are torch's MT19937 words, taken for the
whole batch with one `numpy.random.MT19937.random_raw` call from torch's state, which is then written back advanced; the
binary search over the distribution runs on the GPU.  `restated_ok` checks the restatement against torch once per process
and (alpha, image count).

The result equals the float route when lhotse loads the batch's cuts one after another (`num_workers=0`, no reader thread
pool): with a pool, lhotse's own draw order across cuts is not deterministic."""
from __future__ import annotations

import functools
import math
import threading
from dataclasses import dataclass
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np
import torch

# torch's CPU generator state (CPUGeneratorImplStateLegacy at the front of torch.get_rng_state()): uint64 seed, int32 left,
# int32 seeded, uint64 next, then the 624 MT19937 words stored as uint64
_LEFT, _NEXT, _KEY, _MT_N = 8, 16, 24, 624
_STATE_MIN_BYTES = _KEY + 8 * _MT_N


@dataclass
class RirDraws:
    """The draws of a batch's generated RIRs: `records` (engine.RIR_GEN_DTYPE without the output fields), `draws` (float64:
    per RIR its 2 sr uniforms then its 2 sr perturbations), `cdf` (float32: the distributions the records point into) and
    `lens` (each RIR's length at sr)."""
    records: np.ndarray
    draws: np.ndarray
    cdf: np.ndarray
    lens: List[int]


def _state_words(state: torch.Tensor) -> Optional[Tuple[np.ndarray, int]]:
    """(the 624 words as uint32, NumPy's position) of torch's CPU generator state, None when it is not the layout above."""
    raw = state.numpy() if state.dtype == torch.uint8 else None
    if raw is None or raw.ndim != 1 or raw.shape[0] < _STATE_MIN_BYTES:
        return None
    left = int(raw[_LEFT:_LEFT + 4].view(np.int32)[0])
    nxt = int(raw[_NEXT:_NEXT + 8].view(np.uint64)[0])
    words = raw[_KEY:_KEY + 8 * _MT_N].view(np.uint64)
    if not 1 <= left <= _MT_N + 1 or nxt > _MT_N or (words >> np.uint64(32)).any():
        return None
    pos = _MT_N if left == 1 else nxt
    if left != 1 and left != _MT_N + 1 - nxt:
        return None
    return words.astype(np.uint32), pos


def torch_uniforms(state: torch.Tensor, n: int) -> Optional[Tuple[np.ndarray, torch.Tensor]]:
    """The n float64 uniforms torch's CPU generator in `state` gives `uniform_real_distribution<double>(0, 1)` (two words
    each, the first the high half, 53 bits kept) and the state after them; None when `state` is not the legacy layout."""
    parsed = _state_words(state)
    if parsed is None:
        return None
    key, pos = parsed
    bg = np.random.MT19937()
    bg.state = {"bit_generator": "MT19937", "state": {"key": key, "pos": pos}}
    w = bg.random_raw(2 * n).astype(np.uint64) if n else np.zeros(0, np.uint64)
    bits = ((w[0::2] << np.uint64(32)) | w[1::2]) & np.uint64((1 << 53) - 1)
    u = bits.astype(np.float64) * (1.0 / (1 << 53))
    st = bg.state["state"]
    out = state.clone()
    raw = out.numpy()
    raw[_KEY:_KEY + 8 * _MT_N].view(np.uint64)[:] = st["key"].astype(np.uint64)
    raw[_LEFT:_LEFT + 4].view(np.int32)[0] = _MT_N + 1 - int(st["pos"])
    raw[_NEXT:_NEXT + 8].view(np.uint64)[0] = int(st["pos"])
    return u, out


def multinomial_cdf(alpha: float, image: int) -> np.ndarray:
    """The float32 normalised cumulative distribution `torch.multinomial` searches for lhotse's
    `torch.linspace(alpha, 1.0, image).pow(2)` normalised by its sum: a sequential float32 sum, each entry divided by the
    total, the last set to 1."""
    p = torch.linspace(alpha, 1.0, image).pow(2)
    p = (p / p.sum()).numpy()
    c = np.cumsum(p, dtype=np.float32)
    c = (c / c[-1]).astype(np.float32)
    c[-1] = 1.0
    return c


def linspace32(start: float, end: float, steps: int) -> np.ndarray:
    """torch.linspace(start, end, steps) in float32 as csrc/rirgen.cuh rg_linspace computes it."""
    from .pcm_staging import _fma32

    s, e = np.float32(start), np.float32(end)
    step = np.float32(np.float32(e - s) / np.float32(steps - 1))
    i = np.arange(steps)
    a = _fma32(np.full(steps, step), i.astype(np.float32), np.full(steps, s))
    b = _fma32(np.full(steps, -step), (steps - i - 1).astype(np.float32), np.full(steps, e))
    return np.where(i < steps // 2, a, b)


def multinomial_from_uniforms(cdf: np.ndarray, u: np.ndarray) -> np.ndarray:
    """torch.multinomial's binary search: the first slot whose cumulative probability is not below u."""
    return np.searchsorted(cdf.astype(np.float64), u, side="left")


_PROBES: Dict[Tuple[float, int], bool] = {}
_PROBES_LOCK = threading.Lock()


def restated_ok(alpha: float, image: int) -> bool:
    """Whether torch here draws what the restatement draws for (alpha, image): `torch.multinomial` on two private generators
    (fresh from a seed, and advanced past a twist) against `torch_uniforms` + `multinomial_cdf`, the generator states after
    them, and torch.linspace against `linspace32` at a few ends.  Run once per process and (alpha, image); torch's global
    generator is not touched."""
    key = (float(alpha), int(image))
    with _PROBES_LOCK:
        ok = _PROBES.get(key)
        if ok is not None:
            return ok
        ok = True
        try:
            cdf = multinomial_cdf(alpha, image)
            probs = torch.linspace(alpha, 1.0, image).pow(2)
            probs = probs / probs.sum()
            for seed, skip in ((20251017, 0), (77, 401)):
                g = torch.Generator().manual_seed(seed)
                torch.rand(skip, generator=g, dtype=torch.float64)
                got = torch_uniforms(g.get_state(), image)
                want = probs.multinomial(num_samples=image, replacement=True, generator=g)
                if got is None or not np.array_equal(multinomial_from_uniforms(cdf, got[0]), want.numpy()):
                    ok = False
                    break
                if not torch.equal(got[1][:_STATE_MIN_BYTES], g.get_state()[:_STATE_MIN_BYTES]):
                    ok = False
                    break
            for end in (1.25, 37.7, 1234.5678):
                want = torch.linspace(1.0, torch.tensor(end, dtype=torch.float64), image).numpy()
                if not np.array_equal(linspace32(1.0, end, image).view(np.int32), want.view(np.int32)):
                    ok = False
        except Exception:
            ok = False
        _PROBES[key] = ok
        return ok


@functools.lru_cache(maxsize=None)
def biquad_coefficients(sample_rate: int) -> Tuple[float, float, float, float, float]:
    """(b0, b1, b2, a1, a2) of torchaudio's highpass_biquad(., sample_rate, 80.0) divided by a0, with torch's own float32
    operations, as lfilter takes them."""
    dtype = torch.float32
    cutoff = torch.as_tensor(80.0, dtype=dtype)
    Q = torch.as_tensor(0.707, dtype=dtype)
    w0 = 2 * math.pi * cutoff / sample_rate
    alpha = torch.sin(w0) / 2.0 / Q
    b0 = (1 + torch.cos(w0)) / 2
    b1 = -1 - torch.cos(w0)
    b2 = b0
    a0 = 1 + alpha
    a1 = -2 * torch.cos(w0)
    a2 = 1 - alpha
    a = torch.stack([a0, a1, a2]).view(1, 3)
    b = torch.stack([b0, b1, b2]).view(1, 3)
    bn, an = (b / a[:, 0:1])[0], (a / a[:, 0:1])[0]
    return float(bn[0]), float(bn[1]), float(bn[2]), float(an[1]), float(an[2])


def generator_eligible(gen) -> bool:
    """Whether the GPU generator takes `gen`: exactly lhotse's FastRandomRIRGenerator with its NumPy generators, torchaudio
    present (lhotse would raise without it), float32 as torch's default dtype, torch's CPU generator state in the layout
    `torch_uniforms` reads, and a restatement that holds here."""
    try:
        from lhotse.augmentation.torchaudio import is_torchaudio_available
        from lhotse.augmentation.utils import FastRandomRIRGenerator
    except ImportError:
        return False
    if type(gen) is not FastRandomRIRGenerator or not is_torchaudio_available():
        return False
    if torch.get_default_dtype() != torch.float32 or _state_words(torch.get_rng_state()) is None:
        return False
    if not all(isinstance(getattr(gen, n, None), np.random.Generator) for n in ("room_rng", "source_rng")):
        return False
    if not (isinstance(gen.sr, int) and 1 <= gen.sr <= 192000 and gen.max_T60 > 0.1):
        return False
    return restated_ok(gen.alpha, 2 * gen.sr)


def rir_len(comb_len: int) -> Tuple[int, int]:
    """(samples at 8 sr, samples at sr) lhotse's two resamplers keep of a comb of comb_len samples."""
    from .pcm_staging import resampled_len

    n8 = resampled_len(1, comb_len, 8)
    return n8, resampled_len(1, n8, 8)


def max_rir_len(gen) -> int:
    """The longest RIR `gen` can give: T60 < max_T60."""
    return rir_len(int(math.ceil(64 * gen.sr * gen.max_T60)))[1]


def snapshot(gens: Sequence) -> tuple:
    """Every generator state the draws of `gens` touch: each NumPy generator's and torch's CPU state."""
    seen, states = set(), []
    for g in gens:
        for rng in (g.room_rng, g.source_rng):
            if id(rng) not in seen:
                seen.add(id(rng))
                states.append((rng, rng.bit_generator.state))
    return states, torch.get_rng_state()


def restore(snap: Optional[tuple]) -> None:
    """Puts back the states `snapshot` saved, so that the float route draws what the staged route had drawn."""
    if snap is None:
        return
    states, t = snap
    for rng, st in states:
        rng.bit_generator.state = st
    torch.set_rng_state(t)


def draw(gens: Sequence) -> RirDraws:
    """The draws of one generated RIR per generator in `gens`, in order, as FastRandomRIRGenerator.__call__(nsource=1) makes
    them; torch's CPU generator is advanced past the batch's multinomials."""
    from .engine import RIR_GEN_DTYPE

    n = len(gens)
    rec = np.zeros(n, dtype=RIR_GEN_DTYPE)
    rec["struct_size"] = RIR_GEN_DTYPE.itemsize
    images = [2 * int(g.sr) for g in gens]
    total = sum(images)
    state = torch.get_rng_state()
    got = torch_uniforms(state, total)
    if got is None:
        raise ValueError("torch's CPU generator state is not the MT19937 layout the restatement reads")
    u, new_state = got
    draws = np.empty(2 * total, dtype=np.float64)
    cdfs: Dict[Tuple[float, int], int] = {}
    cdf_parts: List[np.ndarray] = []
    cdf_len, at, lens = 0, 0, []
    for i, g in enumerate(gens):
        image = images[i]
        t60 = float(g.room_rng.uniform(0.1, g.max_T60, size=(1,))[0])
        r = float(g.room_rng.uniform(0.1, 1.2, size=(1,))[0])
        d0 = float(g.source_rng.uniform(0.2, 12.0, size=(1,))[0])
        draws[at: at + image] = u[at // 2: at // 2 + image]
        draws[at + image: at + 2 * image] = g.source_rng.uniform(g.a, g.b, size=(1, image))[0]
        key = (float(g.alpha), image)
        if key not in cdfs:
            cdfs[key] = cdf_len
            cdf_parts.append(multinomial_cdf(*key))
            cdf_len += image
        comb = int(math.ceil(64 * int(g.sr) * t60))
        n8, n1 = rir_len(comb)
        b0, b1, b2, a1, a2 = biquad_coefficients(8 * int(g.sr))
        rec[i]["sampling_rate"] = g.sr
        rec[i]["t60"], rec[i]["r"], rec[i]["d0"], rec[i]["tau"] = t60, r, d0, float(g.tau)
        rec[i]["b0"], rec[i]["b1"], rec[i]["b2"], rec[i]["a1"], rec[i]["a2"] = b0, b1, b2, a1, a2
        rec[i]["cdf_elem"] = cdfs[key]
        rec[i]["draw_elem"] = at
        rec[i]["comb_len"] = comb
        rec[i]["out_len"] = n8
        lens.append(n1)
        at += 2 * image
    torch.set_rng_state(new_state)
    cdf = np.concatenate(cdf_parts) if cdf_parts else np.zeros(0, np.float32)
    return RirDraws(records=rec, draws=draws, cdf=cdf, lens=lens)
