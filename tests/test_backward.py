"""The backward of the Kaldi-family extractors without a GPU (csrc/backward.cuh, DESIGN.md §3.1n): the float64 restatement
of the kernel's adjoint chain against autograd through the oracle's chain in float64, over every kind, energy form,
magnitude, framing, pre-emphasis, DC removal, window and N, at the framing's edge lengths; silence and full-scale input; the
header's own per-frame code run on the host (under AddressSanitizer) against the restatement; and the ABI's new entries."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

import backward_cases as BC

CASES = BC.configs()


@pytest.mark.parametrize("name,cfg", CASES, ids=[c[0] for c in CASES])
def test_restatement_matches_float64_autograd(name, cfg):
    for n in BC.lengths(cfg, long=name in ("fbank", "mfcc-nolifter", "log-spectrogram-energy-raw")):
        for kind in ("noise", "full", "silence"):
            x = BC.waveform(n, kind)
            T = BC.features_t(__import__("torch").tensor(x), cfg).shape
            G = BC.conditioned(x, cfg, np.random.RandomState(n).randn(*T))
            want = BC.autograd_grad(x, cfg, G)
            got = BC.restated_grad(x, cfg, G)
            assert BC.rel_err(got, want) < 1e-11, (name, n, kind, BC.rel_err(got, want))
            if kind == "silence" and cfg.feature in ("fbank", "mfcc") and not cfg.use_energy:
                assert not got.any()  # every floor binds: no gradient


def test_silence_with_energy_floor_has_no_gradient():
    cfg = BC.cfg_of("fbank", use_energy=True)
    x = np.zeros(4000)
    G = np.ones((25, 81))
    assert not BC.restated_grad(x, cfg, G).any()
    assert not BC.autograd_grad(x, cfg, G).any()


@pytest.fixture(scope="module")
def harness(tmp_path_factory):
    exe = BC.host_check_binary(tmp_path_factory.mktemp("bwdh"))
    if exe is None:
        pytest.skip("no host C++ compiler")
    return exe


HOST_CASES = [c for c in CASES if c[0] in ("fbank", "fbank-energy-raw", "mfcc-energy-win-snip", "mfcc-nolifter", "spectrogram-mag-nodc-nopre",
                                           "log-spectrogram-energy-raw", "fbank-blackman", "fbank-N400", "fbank-N2048",
                                           "log-spectrogram-N256-snip", "spectrogram-N401", "log-spectrogram-N401-mag")]


@pytest.mark.parametrize("name,cfg", HOST_CASES, ids=[c[0] for c in HOST_CASES])
def test_host_harness_matches_restatement(name, cfg, harness, tmp_path):
    """The header's per-frame and per-sample code in float32 on the CPU, with every buffer at its exact size."""
    import torch

    for n in BC.lengths(cfg, long=False) + [16000 + 37]:
        x = BC.waveform(n, "noise").astype(np.float32).astype(np.float64)
        T, F = BC.features_t(torch.tensor(x), cfg).shape
        G = BC.conditioned(x, cfg, np.random.RandomState(n).randn(T, F)).astype(np.float32)
        inp, out = str(tmp_path / "in.bin"), str(tmp_path / "out.f32")
        BC.host_check_input(inp, cfg, x, G)
        res = subprocess.run([harness, inp, out], capture_output=True, text=True)
        assert res.returncode == 0, res.stderr
        got = np.fromfile(out, dtype=np.float32)
        want = BC.restated_grad(x, cfg, G.astype(np.float64))
        assert got.shape == want.shape
        assert BC.rel_err(got, want) < 2e-4, (name, n, BC.rel_err(got, want))


def test_abi_backward_entries_refuse_bad_calls_without_a_gpu():
    from lhotse_b200 import engine

    lib = engine.load_library()
    ns = np.asarray([16000], dtype=np.int64)
    assert lib.b200feat_backward_work_bytes(None, ns.ctypes.data, 1) == -1
    rc = lib.b200feat_backward(None, None, 0, None, None, 1, None, None, None, None, 0, None)
    assert rc == -1
    assert "b200feat_backward" in engine.EXPORTS and "b200feat_backward_work_bytes" in engine.EXPORTS
