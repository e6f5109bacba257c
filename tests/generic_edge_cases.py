"""The generic kernel's edge table and the float64 restatements its CPU tests check (csrc/generic.cuh, DESIGN.md §3.2).

ROWS names, per plan: the frame geometry (L, N, S), packed (even N, complex FFT of Nc = N / 2) or unpacked (odd N, Nc = N),
the radix list `factorize(Nc)` yields, the launch shape the host picks (warps per CTA, dynamic shared-memory bytes), the
epilogue and the branch tags the row is meant to reach.  `branches` derives the tags from the plan alone, so a label that
no longer matches its plan fails `test_table_names_its_targets`.

`stockham` restates the kernel's FFT pass by pass (output index, twiddle index and the prime radix's twiddle walk) and
`packed_split` its real split, in float64; `region_faults` restates where each phase of the kernel writes inside its
warp's region of shared memory, for a layout read from the header itself (scripts/micro/generic_layout_check.cu).
"""
import functools
import math
import os
import shutil
import subprocess
from collections import namedtuple
from types import SimpleNamespace

import numpy as np

from lhotse_b200.plan import build_plan

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FEATURE_CODE = {"fbank": 0, "mfcc": 1, "spectrogram": 2, "log-spectrogram": 3, "whisper-fbank": 4, "librosa-fbank": 5}
SMEM_OPTIN = 227 * 1024  # dynamic shared memory one CTA can opt in to on sm_90
SWEEP_FEATURES = ("fbank", "mfcc", "spectrogram", "log-spectrogram")  # the layout of the other kinds is fbank's


# ------------------------------------------------------------------------------------------------ plan arithmetic
def factorize(n):
    """b200feat.cu factorize: radix-4 passes, then radix 2, then odd primes in increasing order."""
    f = []
    while n % 4 == 0:
        f.append(4)
        n //= 4
    while n % 2 == 0:
        f.append(2)
        n //= 2
    p = 3
    while n > 1:
        while n % p == 0:
            f.append(p)
            n //= p
        p += 2
    return f


def layout(feature, N, M):
    """generic_layout: one warp's region in floats -> dict(bufA, bufB, mlog, floats)."""
    Nc = N // 2 if N % 2 == 0 else N
    bufA = (N + 3) & ~3
    scratch = (M + 3) & ~3 if feature == "mfcc" else 0
    return dict(bufA=bufA, bufB=bufA + 2 * Nc, mlog=bufA, floats=bufA + max(4 * Nc, scratch))


def launch_shape(feature, N, M):
    """generic_launch_shape: (warps per CTA, dynamic shared-memory bytes, fits the opt-in limit)."""
    per_warp = 4 * layout(feature, N, M)["floats"]
    w = min(8, max(1, (100 * 1024) // per_warp))
    return w, w * per_warp, w * per_warp <= SMEM_OPTIN


def head_layout(feature, N, M):
    """The layout before the MFCC scratch had a region of its own: log-mels in `dst`, the FFT buffer that does not hold
    the result (bufB after an even number of passes, bufA after an odd one), 2 Nc floats of room."""
    Nc = N // 2 if N % 2 == 0 else N
    bufA = (N + 3) & ~3
    even = len(factorize(Nc)) % 2 == 0
    mlog = bufA + 2 * Nc if even else bufA
    return dict(bufA=bufA, bufB=bufA + 2 * Nc, mlog=mlog, mlog_end=mlog + 2 * Nc, floats=bufA + 4 * Nc)


def region_faults(feature, N, L, M, lay):
    """Every write of one frame, phase by phase, against the region it belongs to.  Returns a list of faults (empty: all
    writes stay in their own region, the regions stay in the warp's, and mlog, written while the mel loop reads raw,
    does not overlap raw).  `lay` is a layout dict; `mlog_end` defaults to the end of the warp's region."""
    Nc = N // 2 if N % 2 == 0 else N
    packed = N % 2 == 0
    K = N // 2 + 1
    floats = lay["floats"]
    regions = {"raw": (0, lay["bufA"]), "bufA": (lay["bufA"], lay["bufA"] + 2 * Nc),
               "bufB": (lay["bufB"], lay["bufB"] + 2 * Nc), "mlog": (lay["mlog"], lay.get("mlog_end", floats))}
    faults = []
    for name, (a, b) in regions.items():
        if not (0 <= a <= b <= floats):
            faults.append(f"region {name} [{a}, {b}) outside the warp's [0, {floats})")
    writes = [("gather", "raw", 0, L), ("spectrum", "raw", 0, K),
              ("window", "bufA", 0, N if packed else 2 * N)]  # packed: N floats; unpacked: N complex
    for st, (lo, hi, once) in enumerate(pass_writes(Nc)):
        if not once:
            faults.append(f"pass {st} does not write each of its Nc outputs once")
        writes.append((f"pass {st}", "bufB" if st % 2 == 0 else "bufA", lo, hi))
    if feature == "mfcc":
        writes.append(("mfcc log-mels", "mlog", 0, M))
    for what, name, lo, hi in writes:
        a, b = regions[name]
        if a + hi > b:
            faults.append(f"{what}: writes [{a + lo}, {a + hi}) past {name}'s end {b}")
    if feature == "mfcc":
        a, b = lay["mlog"], lay["mlog"] + M
        if a < lay["bufA"] and b > 0:
            faults.append("mlog overlaps raw")
    return faults


# ------------------------------------------------------------------------------------------------ float64 Stockham
@functools.lru_cache(maxsize=None)
def pass_writes(Nc):
    """Per Stockham pass: the float range [lo, hi) it writes in its destination buffer and whether it writes each of the
    Nc complex outputs exactly once."""
    out, Ns = [], 1
    for R in factorize(Nc):
        o = pass_outputs(Nc, R, Ns)
        out.append((2 * int(o.min()), 2 * int(o.max()) + 2, bool(np.array_equal(np.sort(o), np.arange(Nc)))))
        Ns *= R
    return tuple(out)


def pass_outputs(Nc, R, Ns):
    """Output indices of one Stockham pass: o + q Ns for every butterfly j and every q, o = (j / Ns) Ns R + j % Ns."""
    j = np.arange(Nc // R)
    o = (j // Ns) * Ns * R + j % Ns
    return (o[:, None] + Ns * np.arange(R)[None, :]).ravel()


def stockham_pass(src, tw, Nc, R, Ns):
    """generic.cuh stockham_pass in float64, with the kernel's index and twiddle arithmetic."""
    nb = Nc // R
    tstep = Nc // (Ns * R)
    j = np.arange(nb)
    k = j % Ns
    o = (j // Ns) * Ns * R + k
    dst = np.full(Nc, np.nan + 0j)
    if R == 4:
        ti = k * tstep
        v0, v1, v2, v3 = src[j], src[j + nb] * tw[ti], src[j + 2 * nb] * tw[2 * ti], src[j + 3 * nb] * tw[3 * ti]
        a, b, c, d = v0 + v2, v0 - v2, v1 + v3, -1j * (v1 - v3)
        dst[o], dst[o + Ns], dst[o + 2 * Ns], dst[o + 3 * Ns] = a + c, b + d, a - c, b - d
    elif R == 2:
        v0, v1 = src[j], src[j + nb] * tw[k * tstep]
        dst[o], dst[o + Ns] = v0 + v1, v0 - v1
    else:
        qstep = Nc // R
        q = np.arange(R)[:, None]                         # every q at once: (R, nb)
        step = (k[None, :] * tstep + q * qstep) % Nc
        acc = np.broadcast_to(src[j], step.shape).astype(np.complex128)
        ti = np.zeros(step.shape, dtype=np.int64)
        for r in range(1, R):
            ti = ti + step
            ti = np.where(ti >= Nc, ti - Nc, ti)
            acc = acc + src[j + r * nb][None, :] * tw[ti]
        dst[o[None, :] + q * Ns] = acc
    return dst


def stockham(z):
    """The kernel's complex FFT of length Nc = len(z): every pass of factorize(Nc) over the table exp(-2 pi i k / Nc)."""
    Nc = len(z)
    tw = np.exp(-2j * np.pi * np.arange(Nc) / Nc)
    Ns = 1
    for R in factorize(Nc):
        z = stockham_pass(z, tw, Nc, R, Ns)
        Ns *= R
    return z


def packed_split(Z, N):
    """The spectrum loop's real split of the packed FFT Z (length Nc = N / 2) -> X[0..K), K = N / 2 + 1."""
    Nc, K = N // 2, N // 2 + 1
    k = np.arange(K)
    zk = Z[np.where(k == Nc, 0, k)]
    zc = Z[np.where(k == 0, 0, Nc - k)]
    er, ei = zk.real + zc.real, zk.imag - zc.imag
    orr, oi = zk.real - zc.real, zk.imag + zc.imag
    w = np.exp(-2j * np.pi * k / N)
    tr, ti = w.real * orr - w.imag * oi, w.real * oi + w.imag * orr
    return 0.5 * (er + ti) + 1j * 0.5 * (ei - tr)


def generic_rfft(y):
    """What the kernel computes for a windowed frame y of N reals: packed for even N, unpacked for odd N."""
    N = len(y)
    if N % 2 == 0:
        return packed_split(stockham(y[0::2] + 1j * y[1::2]), N)
    return stockham(y.astype(np.complex128))[: N // 2 + 1]


# ------------------------------------------------------------------------------------------------ the layout harness
def layout_harness(tmp_dir):
    """Compiles scripts/micro/generic_layout_check.cu (None: no nvcc) -> a function [(feature, N, M)] -> [dict]."""
    nvcc = shutil.which("nvcc") or ("/usr/local/cuda/bin/nvcc" if os.path.exists("/usr/local/cuda/bin/nvcc") else None)
    if nvcc is None:
        return None
    exe = os.path.join(str(tmp_dir), "generic_layout_check")
    src = os.path.join(ROOT, "scripts", "micro", "generic_layout_check.cu")
    res = subprocess.run([nvcc, "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-o", exe, src],
                         capture_output=True, text=True)
    assert res.returncode == 0, res.stderr[-2000:]

    def query(plans):
        inp = "".join(f"{FEATURE_CODE[f]} {N} {M}\n" for f, N, M in plans)
        r = subprocess.run([exe], input=inp, capture_output=True, text=True)
        assert r.returncode == 0, r.stderr
        out = []
        for line in r.stdout.split("\n")[: len(plans)]:
            N, Nc, bufA, bufB, mlog, floats, warps, smem, fits = map(int, line.split())
            out.append(dict(N=N, Nc=Nc, bufA=bufA, bufB=bufB, mlog=mlog, floats=floats, warps=warps, smem=smem,
                            fits=bool(fits)))
        assert len(out) == len(plans)
        return out

    return query


# ------------------------------------------------------------------------------------------------ the edge table
Row = namedtuple("Row", "name feature cfg L N S packed Nc radix warps smem epilogue targets")


def plan_of(feature, cfg):
    return build_plan(feature, SimpleNamespace(**cfg))


def epilogue_of(feature, cfg, plan):
    e = feature
    if plan.use_energy and feature != "mfcc":
        e += "+energy-last" if plan.energy_last else "+energy"
    if feature in ("spectrogram", "log-spectrogram") and plan.use_fft_mag:
        e += "+mag"
    if feature == "mfcc":
        e += f"-M{plan.num_filters}-C{plan.num_ceps}" + ("+lifter" if plan.lifter is not None else "")
    return e


def branches(row):
    """The branch tags a row's plan reaches, from the plan and the restated factorization and launch sizing."""
    p = plan_of(row.feature, row.cfg)
    Nc = p.N // 2 if p.N % 2 == 0 else p.N
    rad = factorize(Nc)
    w, smem, fits = launch_shape(row.feature, p.N, p.num_filters)
    tags = {f"radix{R}" for R in rad} | {f"warps{w}"}
    if all(R in (2, 4) for R in rad):
        tags.add("pow2-passes")
    if 3 in rad and rad.index(3) > 0 and all(R in (2, 4) for R in rad[: rad.index(3)]):
        tags.add("3-after-4s-and-2s")
    if len(rad) == 1 and rad[0] > 5:
        tags.add("prime-single-stage")  # R = Nc: nb = 1, lane 0 computes the whole DFT
    if len({R for R in rad if R % 2}) >= 2:
        tags.add("several-odd-primes")
    if any(R > 5 for R in rad):
        tags.add("prime-radix>5")
    tags.add("unpacked" if p.N % 2 else ("packed-pow2-Nc" if Nc & (Nc - 1) == 0 else "packed-odd-Nc" if Nc % 2 else "packed"))
    if smem > 100 * 1024:
        tags.add("smem>100KB")
    tags.add("L=N" if p.L == p.N else "L<N")
    if p.S > p.L:
        tags.add("S>L")
    if p.feature in ("whisper-fbank", "librosa-fbank"):
        tags.add("center")
    else:
        tags.add("snip" if p.snip_edges else "no-snip")
    ep = epilogue_of(row.feature, row.cfg, p)
    tags.add("epi:" + ep.split("-M")[0])
    if row.feature == "mfcc":
        if p.num_filters > 32 and p.num_ceps > 32 and p.lifter is not None:
            tags.add("mfcc-M>32-C>32+lifter")
        if p.num_filters > 2 * Nc:
            tags.add("mfcc-M>2Nc")
    return tags


def _rows():
    rows = []

    def add(name, feature, cfg, L, N, S, radix, warps, smem, targets):
        p = plan_of(feature, cfg)
        Nc = N // 2 if N % 2 == 0 else N
        rows.append(Row(name, feature, cfg, L, N, S, N % 2 == 0, Nc, tuple(radix), warps, smem,
                        epilogue_of(feature, cfg, p), frozenset(targets)))

    nope = dict(round_to_power_of_two=False)
    legacy = dict(torchaudio_compatible_mel_scale=False)  # the torchaudio mel scale needs an even N
    # radix passes, packed / unpacked, launch shapes
    add("pow2-4096", "fbank", dict(sampling_rate=48000, frame_length=0.085, use_energy=True),
        4080, 4096, 480, [4, 4, 4, 4, 4, 2], 2, 98304, {"pow2-passes", "warps2", "L<N", "epi:fbank+energy"})
    add("n1536", "spectrogram", dict(sampling_rate=16000, frame_length=0.096, use_energy=True, **nope),
        1536, 1536, 160, [4, 4, 4, 4, 3], 5, 92160, {"3-after-4s-and-2s", "warps5", "epi:spectrogram+energy"})
    add("n210", "log-spectrogram", dict(sampling_rate=8400, frame_length=0.025, use_energy=True, **nope),
        210, 210, 84, [3, 5, 7], 8, 20224, {"radix5", "radix7", "several-odd-primes", "epi:log-spectrogram+energy"})
    add("n1000-mfcc", "mfcc", dict(sampling_rate=40000, frame_length=0.025, num_filters=64, num_ceps=40, use_energy=True, **nope),
        1000, 1000, 400, [4, 5, 5, 5], 8, 96000, {"radix5", "mfcc-M>32-C>32+lifter", "warps8"})
    add("n401", "spectrogram", dict(sampling_rate=4010, frame_length=0.1, use_fft_mag=True, **nope),
        401, 401, 40, [401], 8, 64256, {"prime-single-stage", "unpacked", "epi:spectrogram+mag"})
    add("n1009", "fbank", dict(sampling_rate=10090, frame_length=0.1, use_energy=True, htk_compat=True, **nope, **legacy),
        1009, 1009, 100, [1009], 5, 100960, {"prime-single-stage", "unpacked", "epi:fbank+energy-last"})
    add("n1001-snip-S>L", "log-spectrogram", dict(sampling_rate=10010, frame_length=0.1, frame_shift=0.12, snip_edges=True, **nope),
        1001, 1001, 1201, [7, 11, 13], 5, 100160, {"several-odd-primes", "S>L", "snip", "epi:log-spectrogram"})
    add("n729-snip", "spectrogram", dict(sampling_rate=7290, frame_length=0.1, snip_edges=True, raw_energy=False, **nope),
        729, 729, 72, [3, 3, 3, 3, 3, 3], 7, 102144, {"radix3", "snip", "epi:spectrogram"})
    add("n551", "log-spectrogram", dict(sampling_rate=22050, frame_length=0.025, use_fft_mag=True, **nope),
        551, 551, 220, [19, 29], 8, 88192, {"radix19", "radix29", "epi:log-spectrogram+mag"})
    add("n550", "fbank", dict(sampling_rate=22000, frame_length=0.025, num_filters=40, **nope),
        550, 550, 220, [5, 5, 11], 8, 52864, {"packed-odd-Nc", "epi:fbank"})
    add("n802-snip", "spectrogram", dict(sampling_rate=8020, frame_length=0.1, snip_edges=True, use_energy=True,
                                        raw_energy=False, **nope),
        802, 802, 80, [401], 8, 77056, {"packed-odd-Nc", "prime-single-stage", "snip"})
    add("pow2-2048-L=N", "log-spectrogram", dict(sampling_rate=16000, frame_length=0.128, use_energy=True, use_fft_mag=True),
        2048, 2048, 160, [4, 4, 4, 4, 4], 4, 98304, {"warps4", "L=N", "epi:log-spectrogram+energy+mag"})
    add("n2400", "spectrogram", dict(sampling_rate=48000, frame_length=0.05, use_energy=True, raw_energy=False, **nope),
        2400, 2400, 480, [4, 4, 3, 5, 5], 3, 86400, {"warps3", "radix5"})
    add("pow2-8192", "spectrogram", dict(sampling_rate=16000, frame_length=0.512, frame_shift=0.02),
        8192, 8192, 320, [4, 4, 4, 4, 4, 4], 1, 98304, {"warps1"})
    add("pow2-16384", "log-spectrogram", dict(sampling_rate=32000, frame_length=0.512, frame_shift=0.02),
        16384, 16384, 640, [4, 4, 4, 4, 4, 4, 2], 1, 196608, {"warps1", "smem>100KB"})
    add("n11025", "spectrogram", dict(sampling_rate=44100, frame_length=0.25, frame_shift=0.02, **nope),
        11025, 11025, 882, [3, 3, 5, 5, 7, 7], 1, 220512, {"warps1", "smem>100KB", "unpacked", "radix7"})
    # the MFCC plans whose M log-mels did not fit the FFT buffer they were kept in
    add("mfcc-32-M40-16k", "mfcc", dict(sampling_rate=16000, frame_length=0.002, frame_shift=0.001, num_filters=40),
        32, 32, 16, [4, 4], 8, 3072, {"mfcc-M>2Nc", "L=N"})
    add("mfcc-32-M40-8k", "mfcc", dict(sampling_rate=8000, frame_length=0.004, frame_shift=0.002, num_filters=40),
        32, 32, 16, [4, 4], 8, 3072, {"mfcc-M>2Nc"})
    add("mfcc-64-M80", "mfcc", dict(sampling_rate=16000, frame_length=0.004, frame_shift=0.002, num_filters=80),
        64, 64, 32, [4, 4, 2], 8, 6144, {"mfcc-M>2Nc"})
    add("mfcc-128-M140", "mfcc", dict(sampling_rate=16000, frame_length=0.008, frame_shift=0.004, num_filters=140,
                                      use_energy=True),
        128, 128, 64, [4, 4, 4], 8, 12288, {"mfcc-M>2Nc"})
    # centred (librosa / whisper) framing
    add("librosa-800", "librosa-fbank", dict(sampling_rate=16000, fft_size=800, hop_size=200, num_mel_bins=80),
        800, 800, 200, [4, 4, 5, 5], 8, 76800, {"center", "epi:librosa-fbank"})
    add("librosa-4096", "librosa-fbank", dict(sampling_rate=44100, fft_size=4096, hop_size=512, win_length=2048,
                                             num_mel_bins=128, fmin=None, fmax=None),
        4096, 4096, 512, [4, 4, 4, 4, 4, 2], 2, 98304, {"center", "warps2"})
    add("whisper", "whisper-fbank", dict(num_filters=80),
        400, 400, 160, [4, 2, 5, 5], 8, 38400, {"center", "epi:whisper-fbank"})
    return rows


ROWS = _rows()

# branches the rows together must reach
REQUIRED = [
    "pow2-passes", "3-after-4s-and-2s", "radix5", "radix7", "prime-single-stage", "several-odd-primes", "radix19",
    "radix29", "packed-pow2-Nc", "packed-odd-Nc", "unpacked",
    "warps8", "warps5", "warps4", "warps3", "warps2", "warps1", "smem>100KB",
    "L=N", "L<N", "S>L", "snip", "no-snip", "center",
    "epi:spectrogram", "epi:spectrogram+energy", "epi:spectrogram+mag", "epi:log-spectrogram",
    "epi:log-spectrogram+energy", "epi:log-spectrogram+mag", "epi:fbank+energy", "epi:fbank+energy-last",
    "mfcc-M>32-C>32+lifter", "mfcc-M>2Nc", "epi:librosa-fbank", "epi:whisper-fbank",
]

# plans the kernel must refuse at creation: one warp's region is over the opt-in limit
REFUSED = [
    ("pow2-32768", "spectrogram", dict(sampling_rate=32000, frame_length=1.024, frame_shift=0.02), 32768),
    ("odd-11623", "spectrogram", dict(sampling_rate=11623, frame_length=1.0, frame_shift=0.02, round_to_power_of_two=False),
     11623),
]
LARGEST_ODD = 11621  # the largest odd N whose one-warp region fits


def row_id(r):
    return r.name


def oracle_kind(r):
    return {"librosa-fbank": "librosa", "whisper-fbank": "whisper"}.get(r.feature, "kaldi")


def kaldi_cfg(r):
    """The row's config for oracle/kaldi_oracle.OracleConfig (htk_compat is a column roll on the oracle's output)."""
    return {k: v for k, v in r.cfg.items() if k != "htk_compat"}


def shortest_framable(plan):
    """The fewest samples a cut may have and still be framed (b200feat.cu framable / frames_for)."""
    L, S, N = plan.L, plan.S, plan.N
    if plan.feature in ("whisper-fbank", "librosa-fbank"):
        return N // 2 + 1  # torch's reflect padding needs pad < n, and (n + S / 2) / S >= 1 holds from S / 2 on
    if plan.snip_edges:
        return L
    left = (L - S) // 2
    n = 1
    while True:
        T = (n + S // 2) // S
        if T >= 1 and left <= n and (T - 1) * S + L - n - left <= n:
            return n
        n += 1


def cut_lengths(plan):
    """Cuts for one row: the shortest framable one, one frame-count edge either side of it, and a few longer ones."""
    L, S = plan.L, plan.S
    n0 = shortest_framable(plan)
    lens = [n0, n0 + 1, max(n0, L) + S - 1, max(n0, L) + S, 7 * S + S // 2 + max(n0, L), 23 * S + 3 + max(n0, L)]
    return sorted(set(lens))


def check_row_geometry(r):
    """The frame geometry a row claims against floor(frame_length * sr) and the plan."""
    p = plan_of(r.feature, r.cfg)
    if r.feature not in ("whisper-fbank", "librosa-fbank"):
        sr = r.cfg.get("sampling_rate", 16000)
        assert math.floor(r.cfg.get("frame_length", 0.025) * sr) == r.L, r.name
        assert math.floor(r.cfg.get("frame_shift", 0.01) * sr) == r.S, r.name
    assert (p.L, p.N, p.S) == (r.L, r.N, r.S), (r.name, p.L, p.N, p.S)
    return p
