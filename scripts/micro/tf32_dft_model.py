"""Numerical model (numpy, CPU) of moving the 512-point real FFT of the headline path onto tensor cores as two
stages of small GEMMs (DESIGN.md §3.1e): what accuracy do plain TF32, the 3xTF32 split (A_hi*B_hi + A_lo*B_hi +
A_hi*B_lo) and a 2xBF16-style split give on the quantities the
parity gate looks at (power bins, log-mel)?  Operands are rounded exactly as `cvt.rna.tf32.f32` does (10 explicit mantissa
bits, round to nearest, ties away); products are exact (tensor cores multiply TF32 exactly), accumulation is float32.

Pipeline modelled (same algebra as csrc/fast512.cuh): z[n] = y[2n] + i*y[2n+1] (256 complex points) = 16 x 16;
stage A: DFT16 over n1 for every n2 as a (32 x 32 real) x (32 x 16) GEMM; twiddle W256^(n2*k1) on CUDA cores (fp32);
stage B: DFT16 over n2 as a second GEMM; real-FFT split, |X|^2, mel (80 filters), log — all fp32.
Run: python scripts/micro/tf32_dft_model.py  (prints the table)
"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
import numpy as np

import lhotse_b200 as lb


def tf32(x):
    """cvt.rna.tf32.f32: keep 10 explicit mantissa bits, round to nearest with ties away from zero."""
    b = np.asarray(x, dtype=np.float32).view(np.uint32)
    r = ((b + np.uint32(0x1000)) & np.uint32(0xFFFFE000)).astype(np.uint32)
    return r.view(np.float32)


def bf16(x):
    b = np.asarray(x, dtype=np.float32).view(np.uint32)
    r = ((b + np.uint32(0x8000)) & np.uint32(0xFFFF0000)).astype(np.uint32)
    return r.view(np.float32)


def mm(A, B, mode):
    """C = A @ B with tensor-core operand rounding; exact products, float32 accumulation (modelled with float64 products
    summed in float32 order-independent form: np.float32 of the float64 dot is within 1 ulp of any fp32 summation order)."""
    A = A.astype(np.float32)
    B = B.astype(np.float32)
    if mode == "fp32":
        return (A.astype(np.float64) @ B.astype(np.float64)).astype(np.float32)
    rnd = {"tf32": tf32, "3xtf32": tf32, "bf16x3": bf16}[mode]
    Ah, Bh = rnd(A), rnd(B)
    acc = Ah.astype(np.float64) @ Bh.astype(np.float64)
    if mode in ("3xtf32", "bf16x3"):
        Al, Bl = rnd(A - Ah), rnd(B - Bh)
        acc += Al.astype(np.float64) @ Bh.astype(np.float64) + Ah.astype(np.float64) @ Bl.astype(np.float64)
    return acc.astype(np.float32)


def dft16_real_matrix():
    k, n = np.meshgrid(np.arange(16), np.arange(16), indexing="ij")
    W = np.exp(-2j * np.pi * k * n / 16)
    return np.block([[W.real, -W.imag], [W.imag, W.real]]).astype(np.float32)  # acts on [Re; Im]


def fft512_two_stage(y, mode):
    """y: (T, 512) float32 windowed frames -> (T, 257) complex64 via the 16 x 16 two-stage factorisation."""
    T = y.shape[0]
    z = (y[:, 0::2] + 1j * y[:, 1::2]).astype(np.complex64)          # (T, 256), n = 16*n1 + n2
    Z = z.reshape(T, 16, 16)                                          # [t, n1, n2]
    F = dft16_real_matrix()
    # stage A: over n1 for each (t, n2): GEMM (32x32) x (32 x 16T)
    Bm = np.concatenate([Z.real, Z.imag], axis=1).transpose(1, 0, 2).reshape(32, T * 16)   # rows [Re n1; Im n1]
    Y = mm(F, Bm, mode).reshape(32, T, 16)
    Yc = (Y[:16] + 1j * Y[16:]).transpose(1, 0, 2)                     # [t, k1, n2]
    tw = np.exp(-2j * np.pi * np.outer(np.arange(16), np.arange(16)) / 256).astype(np.complex64)  # W256^(k1*n2)
    Yc = (Yc * tw[None]).astype(np.complex64)                          # fp32 complex multiply on CUDA cores
    # stage B: over n2 for each (t, k1)
    Bm = np.concatenate([Yc.real, Yc.imag], axis=2).transpose(2, 0, 1).reshape(32, T * 16)  # rows [Re n2; Im n2]
    X = mm(F, Bm, mode).reshape(32, T, 16)
    Xc = (X[:16] + 1j * X[16:]).transpose(1, 2, 0)                     # [t, k1, k2] -> Z[k1 + 16*k2]
    Zf = Xc.transpose(0, 2, 1).reshape(T, 256)                         # index k = k1 + 16*k2
    # real-FFT split (fp32)
    k = np.arange(257)
    Zk = Zf[:, k % 256]
    Zc = np.conj(Zf[:, (256 - k) % 256])
    E, O = Zk + Zc, Zk - Zc
    w = np.exp(-2j * np.pi * k / 512).astype(np.complex64)
    return (0.5 * (E - 1j * w * O)).astype(np.complex64)


def main():
    plan = lb.build_plan("fbank", lb.B200FbankConfig())
    rs = np.random.RandomState(0)
    sigs = {
        "white noise 0.1": 0.1 * rs.randn(64 * 160 + 400),
        "speech-like (1/f noise + harmonics)": np.cumsum(0.01 * rs.randn(64 * 160 + 400)) * 0.05
        + 0.2 * np.sin(2 * np.pi * 140 * np.arange(64 * 160 + 400) / 16000) * (1 + 0.5 * np.sin(2 * np.pi * 3 * np.arange(64 * 160 + 400) / 16000)),
        "sine 1 kHz 0.5": 0.5 * np.sin(2 * np.pi * 1000 * np.arange(64 * 160 + 400) / 16000),
    }
    lines = ["# TF32 / 3xTF32 / BF16x3 two-stage (16 x 16) DFT model vs float64 — see the docstring of scripts/micro/tf32_dft_model.py",
             "# columns: max relative error of the power bins (relative to the frame's largest bin), max |d log-mel| over 64 frames",
             "# parity gate for log-mel: 2e-4 + 1e-4*|x| (tests/helpers.py); the fp32 CUDA-core kernel sits at ~1e-6 / ~2e-6"]
    for name, x in sigs.items():
        x = x.astype(np.float32)
        frames = np.stack([x[t * 160: t * 160 + 400] for t in range(64)]).astype(np.float64)
        frames = frames - frames.mean(axis=1, keepdims=True)
        pre = np.concatenate([frames[:, :1], frames[:, :-1]], axis=1)
        y = ((frames - 0.97 * pre) * plan.window[None].astype(np.float64))
        y512 = np.zeros((64, 512)); y512[:, :400] = y
        X64 = np.fft.rfft(y512, axis=1)
        P64 = np.abs(X64) ** 2
        mel64 = np.log(np.maximum(P64 @ plan.mel_bank.astype(np.float64), 1.1920929e-07))
        lines.append(f"\n## {name}")
        for mode in ("fp32", "3xtf32", "bf16x3", "tf32"):
            X = fft512_two_stage(y512.astype(np.float32), mode)
            P = (np.abs(X.astype(np.complex128)) ** 2)
            rel = np.abs(P - P64).max(axis=1) / P64.max(axis=1)
            mel = np.log(np.maximum(P @ plan.mel_bank.astype(np.float64), 1.1920929e-07))
            lines.append(f"{mode:8s} power-bin err / frame peak: {rel.max():.2e}    max|d log-mel|: {np.abs(mel - mel64).max():.2e}")
    out = "\n".join(lines) + "\n"
    print(out)


if __name__ == "__main__":
    main()
