"""Argument contract of the two host-staging entry points of the C ABI, b200feat_extract_host_at (one host buffer) and
b200feat_extract_host_ptrs (one pointer per cut):

- overlapping or decreasing sample offsets, a null cut pointer with samples behind it, and a bad sample dtype are
  B200FEAT_EINVAL;
- a cut too short to be framed in the middle of a batch is B200FEAT_ESHORT, and the handle's last error names that cut;
- after any of these refusals the same handle still takes a valid batch and returns the same bits as a fresh handle
  (the staging lock is released and the staging buffers stay usable).

Both entry points are called through ctypes on the library engine.load_library() loads, with the plain fbank plan on
the fast kernel (tiled plans: the short cut is found while sizing the tile table) and on the generic kernel."""
import ctypes as C

import numpy as np
import pytest

import lhotse_b200 as lb
from lhotse_b200.engine import DT_F32, DT_I16, OUT_PACKED, Engine
from lhotse_b200.plan import build_plan

pytestmark = pytest.mark.gpu

EINVAL, ESHORT = -1, -5
BAD_DTYPE = DT_I16 + 1  # neither B200FEAT_F32 nor B200FEAT_I16
SHORT = 100  # samples: fewer than one 400-sample frame can be framed from
LENS = [16000, 4001, 23457, 8000]


def signals(lens, seed=5):
    rs = np.random.RandomState(seed)
    return [(0.1 * rs.randn(n)).astype(np.float32) for n in lens]


def packed_rows(eng, lens):
    return sum(int(eng.lib.b200feat_num_frames(eng._h, n)) for n in lens)


def host_at(eng, xs, offsets=None, dt=DT_F32):
    """b200feat_extract_host_at over the cuts laid out back to back (or at `offsets`) in one buffer; returns (rc, out)."""
    lens = np.asarray([len(x) for x in xs], dtype=np.int64)
    buf = np.concatenate(xs)
    off = None if offsets is None else np.asarray(offsets, dtype=np.int64)
    out = np.zeros((packed_rows(eng, [n for n in lens if n >= 400]) + 8, eng.feature_dim), dtype=np.float32)
    rc = eng.lib.b200feat_extract_host_at(eng._h, buf.ctypes.data, dt, lens.ctypes.data,
                                          None if off is None else off.ctypes.data, len(lens), out.ctypes.data, OUT_PACKED, 0.0)
    return rc, out


def host_ptrs(eng, xs, dt=DT_F32, null_at=None):
    """b200feat_extract_host_ptrs over one pointer per cut (cut `null_at` passed as a null pointer); returns (rc, out)."""
    lens = np.asarray([len(x) for x in xs], dtype=np.int64)
    ptrs = (C.c_void_p * len(xs))(*[None if i == null_at else x.ctypes.data for i, x in enumerate(xs)])
    out = np.zeros((packed_rows(eng, [n for n in lens if n >= 400]) + 8, eng.feature_dim), dtype=np.float32)
    rc = eng.lib.b200feat_extract_host_ptrs(eng._h, ptrs, dt, lens.ctypes.data, len(xs), out.ctypes.data, OUT_PACKED, 0.0)
    return rc, out


def last_error(eng):
    return eng.lib.b200feat_last_error(eng._h).decode()


def refusals(xs):
    """(name, call on an engine, expected code, substring of the handle's last error)"""
    n0 = len(xs[0])
    short = [xs[0], xs[1], np.zeros(SHORT, np.float32), xs[2]]
    return [
        ("at-overlapping-offsets", lambda e: host_at(e, xs, offsets=[0, n0 - 1, 2 * n0, 3 * n0]), EINVAL, "offsets"),
        ("at-decreasing-offsets", lambda e: host_at(e, xs, offsets=[3 * n0, 2 * n0, n0, 0]), EINVAL, "offsets"),
        ("at-bad-dtype", lambda e: host_at(e, xs, dt=BAD_DTYPE), EINVAL, "dtype"),
        ("at-short-cut", lambda e: host_at(e, short), ESHORT, f"cut 2 with {SHORT} samples"),
        ("ptrs-null-cut", lambda e: host_ptrs(e, xs, null_at=1), EINVAL, "null cut pointer"),
        ("ptrs-bad-dtype", lambda e: host_ptrs(e, xs, dt=BAD_DTYPE), EINVAL, "dtype"),
        ("ptrs-short-cut", lambda e: host_ptrs(e, short), ESHORT, f"cut 2 with {SHORT} samples"),
    ]


NAMES = [r[0] for r in refusals(signals([1] * 4))]


@pytest.fixture(scope="module")
def plan():
    return build_plan("fbank", lb.B200FbankConfig())


@pytest.fixture(scope="module")
def fresh(plan):
    """What a fresh handle computes for the valid batch, through each entry point, per kernel."""
    xs = signals(LENS)
    got = {}
    for kernel in ("fast", "generic"):
        eng = Engine(plan, 0, kernel=kernel)
        rc_at, out_at = host_at(eng, xs)
        rc_ptrs, out_ptrs = host_ptrs(eng, xs)
        assert rc_at == 0 and rc_ptrs == 0, last_error(eng)
        assert np.array_equal(out_at.view(np.uint32), out_ptrs.view(np.uint32))
        got[kernel] = out_at
        eng.close()
    return got


@pytest.mark.parametrize("kernel", ["fast", "generic"])
@pytest.mark.parametrize("name", NAMES)
def test_refusal_leaves_the_handle_usable(plan, fresh, kernel, name):
    xs = signals(LENS)
    eng = Engine(plan, 0, kernel=kernel)
    try:
        assert eng.lib.b200feat_num_frames(eng._h, SHORT) == ESHORT
        rc, _ = host_at(eng, xs)  # the staging buffers exist before the refusal
        assert rc == 0, last_error(eng)
        call, code, msg = next((c, k, m) for n, c, k, m in refusals(xs) if n == name)
        rc, _ = call(eng)
        assert rc == code, (rc, last_error(eng))
        assert msg in last_error(eng), last_error(eng)
        for entry in (host_at, host_ptrs):
            rc, out = entry(eng, xs)
            assert rc == 0, last_error(eng)
            assert np.array_equal(out.view(np.uint32), fresh[kernel].view(np.uint32)), entry.__name__
    finally:
        eng.close()
