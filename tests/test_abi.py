"""The C-ABI shared library loads and exports every symbol include/b200feat.h declares
(no compute calls: there is no GPU in the CPU tier)."""
import ctypes
import os
import re

import pytest

from lhotse_b200 import engine

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def declared_symbols():
    src = open(os.path.join(ROOT, "include", "b200feat.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(b200feat_[a-z_]+)\s*\(", src)))


def test_header_symbols_are_exported():
    lib = ctypes.CDLL(engine.lib_path())
    syms = declared_symbols()
    assert len(syms) >= 15
    for s in syms:
        assert hasattr(lib, s), f"{s} declared in include/b200feat.h but not exported"
    assert sorted(engine.EXPORTS) == syms


def test_version_and_struct_layout():
    lib = engine.load_library()
    assert lib.b200feat_version() == 1
    assert ctypes.sizeof(engine.PlanDesc) == 16 * 4 + 4 * 4
    assert ctypes.sizeof(engine.BatchTotals) == 6 * 8
    assert lib.b200feat_meta_words(10) == 42


def test_library_is_sm90a_only():
    import shutil
    import subprocess

    cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(cuobjdump):
        pytest.skip("cuobjdump not available")
    out = subprocess.run([cuobjdump, "-lelf", engine.lib_path()], capture_output=True, text=True).stdout
    archs = set(re.findall(r"sm_\d+a?", out))
    assert archs == {"sm_90a"}, archs


def test_no_gpu_means_loud_failure():
    import torch

    if torch.cuda.is_available():
        pytest.skip("a GPU is visible")
    from lhotse_b200 import B200Fbank

    with pytest.raises(Exception) as ei:
        B200Fbank().extract(__import__("numpy").zeros(16000, dtype="float32"), 16000)
    assert "no CUDA device" in str(ei.value) or "CPU fallback" in str(ei.value)


def test_product_never_imports_oracle():
    pkg = os.path.join(ROOT, "lhotse_b200")
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h")):
                txt = open(os.path.join(dirpath, f)).read()
                assert not re.search(r"^\s*(from|import)\s+oracle", txt, flags=re.M), f
                assert "kaldi_oracle" not in txt, f


def test_frame_count_contract_through_the_c_abi_without_a_gpu():
    """`b200feat_desc_num_frames` is the C library's own integer contract (the same `frames_for` / `framable` the planner
    and the kernels use), callable without a device: bit-exact against the oracle's restatement of layers.py:747-753 /
    utils.py:424-434 for every feature kind, including which cuts are refused as too short."""
    import numpy as np

    import lhotse_b200 as lb
    from lhotse_b200.engine import desc_num_frames
    from oracle import kaldi_oracle as O
    from oracle import librosa_oracle as LO
    from oracle import whisper_oracle as W

    rs = np.random.RandomState(0)
    ns = sorted(set([1, 79, 80, 119, 120, 139, 140, 159, 160, 161, 239, 240, 399, 400, 401, 15995, 16000, 16079, 16080, 160000]
                    + [int(v) for v in rs.randint(1, 500000, size=200)]))
    cases = [
        (lb.B200FbankConfig(), False), (lb.B200FbankConfig(snip_edges=True), True),
        (lb.B200FbankConfig(sampling_rate=8000), False), (lb.B200FbankConfig(sampling_rate=24000, frame_length=0.05), False),
        (lb.B200FbankConfig(frame_length=0.032, frame_shift=0.016, snip_edges=True), True),
    ]
    import warnings
    for cfg, snip in cases:
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            plan = lb.build_plan("fbank", cfg)
        for n in ns:
            got = desc_num_frames(plan, n)
            try:
                want = O.frame_index_matrix(n, plan.L, plan.S, snip).shape[0]   # raises where the reference cannot frame
            except ValueError:
                want = -5
            assert got == want, (cfg, n, got, want)
            if got >= 0:
                assert got == plan.num_frames(n)
                if not snip:
                    assert got == O.num_frames_api(n, cfg.frame_shift, cfg.sampling_rate)
    wplan = lb.build_plan("whisper-fbank", lb.B200WhisperFbankConfig())
    lplan = lb.build_plan("librosa-fbank", lb.B200LibrosaFbankConfig())
    for n in ns:
        assert desc_num_frames(wplan, n) == (W.num_rows(n) if n > 200 else -5)      # torch reflect padding needs n > n_fft / 2
        assert desc_num_frames(lplan, n) == (LO.num_rows(n, 256) if n > 512 else -5)
    assert desc_num_frames(wplan, -1) == -1
