"""Informational GPU baseline: the reference's own CUDA path is the same torch op chain run on a
cuda tensor (`Fbank(FbankConfig(device="cuda"))`: cuFFT + cuBLAS + ATen elementwise, one HBM round
trip per op — SURVEY.md §2b).  The oracle restates that chain, so running it on device tensors gives
the GPU baseline to beat on the same GPU.  Asserts parity and that the fused kernel is faster."""
import json

import pytest
import torch

from lhotse_b200 import B200Fbank
from oracle import kaldi_oracle as O

pytestmark = pytest.mark.gpu


def torch_chain_fbank(x2d: torch.Tensor, cfg, tables):
    """(B, n) cuda -> (B, T, 80): the reference module's forward on a padded batch (layers.py:565-578)."""
    win, fb = tables
    L, S, N = O.layer_sizes(cfg)
    n = x2d.shape[1]
    T = O.num_frames_layer(n, L, S, False)
    left = (L - S) // 2
    right = (T - 1) * S + L - n - left
    xp = torch.cat((x2d[:, :left].flip(1), x2d, x2d[:, n - right:].flip(1)), dim=1)
    f = xp.unfold(1, L, S)[:, :T]
    f = f - f.mean(dim=2, keepdim=True)
    prev = torch.nn.functional.pad(f, (1, 0), mode="replicate")[:, :, :-1]
    f = f - cfg.preemph_coeff * prev
    f = torch.nn.functional.pad(f * win, (0, N - L))
    spec = torch.fft.rfft(f, dim=-1).abs() ** 2
    return torch.max(torch.matmul(spec, fb), torch.tensor(torch.finfo(torch.float).eps, device=x2d.device)).log()


def test_fused_kernel_beats_torch_cuda_chain():
    dev = torch.device("cuda")
    cfg = O.OracleConfig()
    win = O.make_window(400, "povey").to(dev)
    fb = O.make_mel_bank(cfg, 512).contiguous().to(dev)
    torch.manual_seed(0)
    B = 256
    x = 0.1 * torch.randn(B, 160000, device=dev)
    ext = B200Fbank()
    ours = ext.extract_batch(x, 16000)
    ref = torch_chain_fbank(x, cfg, (win, fb))
    assert ours.shape == ref.shape == (B, 1000, 80)
    assert torch.allclose(ours, ref, rtol=1e-4, atol=1e-3)

    def timeit(fn, reps=5):
        fn(); torch.cuda.synchronize()
        a, b_ = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(reps):
            fn()
        b_.record(); torch.cuda.synchronize()
        return a.elapsed_time(b_) / reps

    t_ours = timeit(lambda: ext.extract_batch(x, 16000))
    t_ref = timeit(lambda: torch_chain_fbank(x, cfg, (win, fb)))
    hours = B * 10 / 3600
    rec = {"cuts": B, "fused_ms": t_ours, "torch_cuda_chain_ms": t_ref, "fused_h_per_s": hours / (t_ours / 1e3),
           "torch_cuda_chain_h_per_s": hours / (t_ref / 1e3), "speedup": t_ref / t_ours, "kernel": ext.engine.kernel}
    print("\nGPU_BASELINE " + json.dumps(rec))
    assert t_ours < t_ref
