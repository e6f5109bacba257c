"""The drop-in boundary from plain C: tests/c_abi/abi_smoke.c is compiled with gcc against include/b200feat.h and linked
to the in-tree libb200feat.so — no Python, torch or C++ on the caller's side.  CPU tier: it builds, links, loads, and
`b200feat_create` refuses loudly without an sm_90 GPU (no CPU fallback).  GPU tier: its output equals the Python
extractor's, bit for bit."""
import os
import shutil
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIBDIR = os.path.join(ROOT, "lhotse_b200")


def _build(tmp_path):
    gcc = shutil.which("gcc") or shutil.which("cc")
    if gcc is None:
        pytest.skip("no C compiler on this box")
    exe = str(tmp_path / "abi_smoke")
    cmd = [gcc, "-std=c99", "-Wall", "-Werror", "-O1", "-I", os.path.join(ROOT, "include"),
           os.path.join(ROOT, "tests", "c_abi", "abi_smoke.c"), "-o", exe, "-L", LIBDIR, "-lb200feat", f"-Wl,-rpath,{LIBDIR}"]
    res = subprocess.run(cmd, capture_output=True, text=True)
    assert res.returncode == 0, res.stderr
    return exe


def _inputs(tmp_path):
    import lhotse_b200 as lb

    plan = lb.build_plan("fbank", lb.B200FbankConfig())
    rs = np.random.RandomState(21)
    lens = np.array([16000, 4001, 23457, 160, 48000], dtype=np.int64)
    xs = [(0.1 * rs.randn(int(n))).astype(np.float32) for n in lens]
    plan.window.astype("<f4").tofile(tmp_path / "window.f32")
    plan.mel_bank.astype("<f4").tofile(tmp_path / "bank.f32")
    np.concatenate(xs).astype("<f4").tofile(tmp_path / "samples.f32")
    lens.astype("<i8").tofile(tmp_path / "lens.i64")
    return xs, lens


def test_c_client_builds_links_and_refuses_without_a_gpu(tmp_path):
    import torch

    exe = _build(tmp_path)
    _inputs(tmp_path)
    res = subprocess.run([exe, str(tmp_path)], capture_output=True, text=True)
    if torch.cuda.is_available():
        assert res.returncode == 0, res.stderr
    else:
        assert res.returncode == 3 and "no CPU fallback" in res.stderr, (res.returncode, res.stderr)
        assert not (tmp_path / "out.f32").exists()


@pytest.mark.gpu
def test_gpu_c_client_matches_python_extractor(tmp_path):
    import lhotse_b200 as lb

    exe = _build(tmp_path)
    xs, lens = _inputs(tmp_path)
    res = subprocess.run([exe, str(tmp_path)], capture_output=True, text=True)
    assert res.returncode == 0, res.stderr
    rows = np.fromfile(tmp_path / "rows.i64", dtype="<i8")
    out = np.fromfile(tmp_path / "out.f32", dtype="<f4").reshape(-1, 80)
    ext = lb.B200Fbank()
    want = [ext.extract(x, 16000) for x in xs]
    assert rows.tolist() == [w.shape[0] for w in want] == [(int(n) + 80) // 160 for n in lens]
    assert np.array_equal(out, np.concatenate(want))
