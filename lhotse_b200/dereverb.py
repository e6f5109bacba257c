"""
WPE dereverberation of a padded waveform batch on the GPU, as a drop-in for ``lhotse.dataset.signal_transforms.DereverbWPE``
with its defaults (n_fft 512, hop_length 128).  The kernels are csrc/wpe.cuh (DESIGN.md §3.1q); ``engine.wpe`` launches them.

When lhotse is importable ``B200DereverbWPE`` subclasses its ``DereverbWPE``; otherwise it is a ``torch.nn.Module`` with the
same constructor.
"""
from __future__ import annotations

import numpy as np
import torch

from .engine import WPE_CUT_DTYPE, WPE_MAX_FRAMES, wpe

try:  # pragma: no cover - depends on the environment
    from lhotse.dataset.signal_transforms import DereverbWPE as _DereverbWPE
except Exception:  # lhotse (or one of its hard deps) is not importable

    class _DereverbWPE(torch.nn.Module):  # mirrors lhotse/dataset/signal_transforms.py DereverbWPE.__init__
        def __init__(self, n_fft: int = 512, hop_length: int = 128):
            super().__init__()
            self.n_fft = n_fft
            self.hop_length = hop_length


class B200DereverbWPE(_DereverbWPE):
    """lhotse's ``DereverbWPE`` module for single-channel batches, on the GPU.

    A 2-D float32 tensor (B, L) is taken row by row, as lhotse does: each whole row, padding included, is dereverberated on
    its own and the result is (B, 128 * (L // 128)) on the input's device.  The arithmetic is nara_wpe's ``wpe_v8`` (taps 10,
    delay 3, 3 iterations, "full" statistics; the per-bin statistics and the solve in float64) between torch's STFT and
    iSTFT with the periodic Blackman window, within a float32 tolerance of a float64 restatement of that chain; lhotse's
    module calls nara_wpe's torch ``wpe_v6``, which computes the same filter in complex64.

    Raises NotImplementedError for 3-D (multi-channel) input and for n_fft / hop_length other than 512 / 128, TypeError for
    other dtypes, ValueError for rows of at most 256 samples or more than WPE_MAX_FRAMES frames, and RuntimeError for an
    input that requires grad under grad mode (there is no backward, and a detached output would be silently wrong)."""

    def __init__(self, n_fft: int = 512, hop_length: int = 128):
        super().__init__(n_fft=n_fft, hop_length=hop_length)
        if (n_fft, hop_length) != (512, 128):
            raise NotImplementedError("B200DereverbWPE supports n_fft=512 and hop_length=128 only")

    def forward(self, audio: torch.Tensor, *args, **kwargs) -> torch.Tensor:
        if audio.ndim == 3:
            raise NotImplementedError("B200DereverbWPE takes single-channel (B, T) batches only")
        if audio.ndim != 2:
            raise ValueError(f"expected a (B, T) batch, got shape {tuple(audio.shape)}")
        if audio.dtype != torch.float32:
            raise TypeError(f"B200DereverbWPE takes float32 audio, got {audio.dtype}")
        if audio.requires_grad and torch.is_grad_enabled():
            raise RuntimeError("B200DereverbWPE has no backward: call it on a tensor that does not require grad, or under "
                               "torch.no_grad()")
        B, L = audio.shape
        T = 1 + L // 128
        if L <= 256 or T < 13 or T > WPE_MAX_FRAMES:
            raise ValueError(f"rows of {L} samples: B200DereverbWPE takes 257 .. {128 * WPE_MAX_FRAMES - 1} samples")
        lz = 128 * (L // 128)
        device = audio.device if audio.is_cuda else torch.device("cuda", torch.cuda.current_device())
        x = audio.detach().to(device).contiguous()
        out = torch.empty((B, lz), dtype=torch.float32, device=device)
        if B:
            ct = np.zeros(B, dtype=WPE_CUT_DTYPE)
            ct["struct_size"] = WPE_CUT_DTYPE.itemsize
            ct["in_elem"] = np.arange(B, dtype=np.int64) * L
            ct["in_len"] = L
            ct["out_elem"] = np.arange(B, dtype=np.int64) * lz
            ct["target_len"] = lz
            with torch.cuda.device(device):
                wpe(x, ct, out)
        return out.to(audio.device)
