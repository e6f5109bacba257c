"""Which engine call each container of the batch API reaches, with which dtype, lengths and offsets, and what comes back;
on the CPU, through a recording wrapper around the oracle-backed engine (tests/helpers.py::OracleEngine).

Every input below means the same waveform x = q / 32768 whatever its dtype (int16 q, float32 or float64 x), so every row
also checks that each entry point gives int16 `q` the features of float32 `q / 32768`, bit for bit."""
import numpy as np
import pytest
import torch

from helpers import attach_oracle_engine
from lhotse_b200 import LOG_EPSILON, B200Fbank
from lhotse_b200.engine import stage_host
from oracle import kaldi_oracle as O

SR, F = 16000, 80
DTYPES = ("int16", "float32", "float64")
UNEVEN = (4000, 6003, 4000)          # 25, 38, 25 frames; 6003 is odd, so the cut after it needs an aligned offset
ALIGNED = [0, 4000, 10004]           # their offsets in a packed device buffer (4-element boundaries)
BIG = 4_200_000                      # (2, BIG) rows hold >= 16 MB in every kernel dtype: the pageable-array route


def frames(n):
    return (n + 80) // 160


def kernel_dtype(dtype):
    return "int16" if dtype == "int16" else "float32"


def _pcm(n, seed):
    return np.clip(np.random.RandomState(seed).randn(n) * 3000, -32768, 32767).astype(np.int16)


def wave(n, dtype, seed):
    """Cut `seed` of `n` samples as `dtype`: int16 q, or x = q / 32768 (exact in float32 and float64)."""
    q = _pcm(n, seed)
    return q if dtype == "int16" else (q.astype(np.float64) / 32768.0).astype(dtype)


_EXPECTED = {}


def expected(n, seed):
    """Oracle features of x = q / 32768 for cut `seed`."""
    if (n, seed) not in _EXPECTED:
        _EXPECTED[n, seed] = O.extract(_pcm(n, seed).astype(np.float32) / 32768.0, O.OracleConfig())
    return _EXPECTED[n, seed]


def _dtype_name(x):
    return str(x.dtype).replace("torch.", "")


class RecordingEngine:
    """Delegates to the oracle engine; records (method, dtype, lengths, offsets) of every extraction call."""

    def __init__(self, inner):
        self.inner, self.calls = inner, []

    def __getattr__(self, name):
        return getattr(self.inner, name)

    def extract_host(self, samples, num_samples, **kw):
        offs = kw.get("offsets")
        self.calls.append(("extract_host", _dtype_name(samples), list(num_samples), None if offs is None else list(offs)))
        return self.inner.extract_host(samples, num_samples, **kw)

    def extract_host_list(self, arrays, dtype=np.float32):
        self.calls.append(("extract_host_list", np.dtype(dtype).name, [int(np.asarray(a).size) for a in arrays], None))
        return self.inner.extract_host_list([np.asarray(a, dtype=dtype) for a in arrays], dtype)  # the C call casts so

    def extract_device(self, samples, num_samples, offsets=None, **kw):
        self.calls.append(("extract_device", _dtype_name(samples), list(num_samples), list(offsets)))
        return self.inner.extract_device(samples, num_samples, offsets=offsets, **kw)


def extractor(dither=0.0):
    ext = attach_oracle_engine(B200Fbank())
    ext._engine = RecordingEngine(ext._engine)
    ext.config.dither = dither  # the extractor adds the noise before the engine call; the oracle itself refuses dither
    return ext


def uneven(dtype):
    return [wave(n, dtype, i) for i, n in enumerate(UNEVEN)]


def mixed(dtype):  # an int16 cut next to a cut of `dtype`
    return [wave(UNEVEN[0], "int16", 0), wave(UNEVEN[1], dtype, 1)]


def tensors(arrays):
    return [torch.from_numpy(a) for a in arrays]


def padded_rows(dtype):  # a (2, 6003) tensor whose first row holds a 4000-sample cut
    x = torch.zeros((2, UNEVEN[1]), dtype=getattr(torch, dtype))
    x[0, : UNEVEN[0]] = torch.from_numpy(wave(UNEVEN[0], dtype, 0))
    x[1] = torch.from_numpy(wave(UNEVEN[1], dtype, 1))
    return x


def staged(dtype):
    return stage_host(uneven(dtype), dtype=np.dtype(kernel_dtype(dtype)))


# (row id, call, engine method, dtype it receives ("kernel": int16 stays, anything else float32), lengths, offsets,
#  return container, cut seeds of the result)
ROWS = [
    ("extract/array-1d", lambda e, d: e.extract(wave(4000, d, 0), SR),
     "extract_host", "kernel", [4000], None, "array", [(4000, 0)]),
    ("extract/tensor-1d", lambda e, d: e.extract(torch.from_numpy(wave(4000, d, 0)), SR),
     "extract_device", "kernel", [4000], [0], "tensor", [(4000, 0)]),
    ("batch/array-1d", lambda e, d: e.extract_batch(wave(4000, d, 0), SR),
     "extract_host_list", "kernel", [4000], None, "array", [(4000, 0)]),
    ("batch/array-2d", lambda e, d: e.extract_batch(np.stack([wave(4000, d, 0), wave(4000, d, 2)]), SR),
     "extract_host", "kernel", [4000, 4000], None, "stacked-array", [(4000, 0), (4000, 2)]),
    ("batch/array-2d-pageable-16MB", lambda e, d: e.extract_batch(np.stack([wave(BIG, d, 0), wave(BIG, d, 1)]), SR),
     "extract_host_list", "kernel", [BIG, BIG], None, "stacked-array", [(BIG, 0), (BIG, 1)]),
    ("batch/list-equal", lambda e, d: e.extract_batch([wave(4000, d, 0), wave(4000, d, 2)], SR),
     "extract_host_list", "kernel", [4000, 4000], None, "stacked-array", [(4000, 0), (4000, 2)]),
    ("batch/list-one", lambda e, d: e.extract_batch([wave(4000, d, 0)], SR),
     "extract_host_list", "kernel", [4000], None, "array-list", [(4000, 0)]),
    ("batch/list-uneven", lambda e, d: e.extract_batch(uneven(d), SR),
     "extract_host_list", "kernel", list(UNEVEN), None, "array-list", list(zip(UNEVEN, range(3)))),
    ("batch/list-mixed-int16", lambda e, d: e.extract_batch(mixed(d), SR),
     "extract_host_list", "kernel", list(UNEVEN[:2]), None, "array-list", list(zip(UNEVEN[:2], range(2)))),
    ("batch/tensor-list", lambda e, d: e.extract_batch(tensors(uneven(d)), SR),
     "extract_device", "kernel", list(UNEVEN), ALIGNED, "tensor-list", list(zip(UNEVEN, range(3)))),
    ("batch/tensor-list-mixed-int16", lambda e, d: e.extract_batch(tensors(mixed(d)), SR),
     "extract_device", "kernel", list(UNEVEN[:2]), ALIGNED[:2], "tensor-list", list(zip(UNEVEN[:2], range(2)))),
    ("batch/tensor-2d", lambda e, d: e.extract_batch(torch.from_numpy(np.stack([wave(4000, d, 0), wave(4000, d, 2)])), SR),
     "extract_device", "kernel", [4000, 4000], [0, 4000], "stacked-tensor", [(4000, 0), (4000, 2)]),
    ("batch/tensor-2d-lengths", lambda e, d: e.extract_batch(padded_rows(d), SR, lengths=[UNEVEN[0], UNEVEN[1]]),
     "extract_device", "kernel", list(UNEVEN[:2]), [0, UNEVEN[1]], "tensor-list", list(zip(UNEVEN[:2], range(2)))),
    ("padded/list-uneven", lambda e, d: e.extract_batch_padded(uneven(d), SR),
     "extract_device", "kernel", list(UNEVEN), ALIGNED, "padded", list(zip(UNEVEN, range(3)))),
    ("padded/tensor-list", lambda e, d: e.extract_batch_padded(tensors(uneven(d)), SR),
     "extract_device", "kernel", list(UNEVEN), ALIGNED, "padded", list(zip(UNEVEN, range(3)))),
    ("padded/tensor-list-mixed-int16", lambda e, d: e.extract_batch_padded(tensors(mixed(d)), SR),
     "extract_device", "kernel", list(UNEVEN[:2]), ALIGNED[:2], "padded", list(zip(UNEVEN[:2], range(2)))),
    ("packed/list-uneven", lambda e, d: e.extract_batch_packed(uneven(d), SR),
     "extract_device", "kernel", list(UNEVEN), ALIGNED, "packed", list(zip(UNEVEN, range(3)))),
    ("packed/tensor-list", lambda e, d: e.extract_batch_packed(tensors(uneven(d)), SR),
     "extract_device", "kernel", list(UNEVEN), ALIGNED, "packed", list(zip(UNEVEN, range(3)))),
    ("packed/tensor-list-mixed-int16", lambda e, d: e.extract_batch_packed(tensors(mixed(d)), SR),
     "extract_device", "kernel", list(UNEVEN[:2]), ALIGNED[:2], "packed", list(zip(UNEVEN[:2], range(2)))),
    ("staged-padded", lambda e, d: e.extract_staged_padded(*staged(d), SR),
     "extract_device", "kernel", list(UNEVEN), ALIGNED, "padded", list(zip(UNEVEN, range(3)))),
    ("staged-packed", lambda e, d: e.extract_staged_packed(*staged(d), SR),
     "extract_device", "kernel", list(UNEVEN), ALIGNED, "packed", list(zip(UNEVEN, range(3)))),
]


def check_result(got, container, cuts):
    """The return container of `container`, holding exactly the oracle features of each cut's x = q / 32768."""
    want = [expected(n, s) for n, s in cuts]
    if container == "array":
        assert isinstance(got, np.ndarray) and got.dtype == np.float32 and got.shape == want[0].shape
        per_cut = [got]
    elif container == "tensor":
        assert isinstance(got, torch.Tensor) and got.dtype == torch.float32 and tuple(got.shape) == want[0].shape
        per_cut = [got.numpy()]
    elif container in ("stacked-array", "stacked-tensor"):
        kind = np.ndarray if container == "stacked-array" else torch.Tensor
        assert isinstance(got, kind) and tuple(got.shape) == (len(want),) + want[0].shape
        per_cut = [np.asarray(g) for g in got]
    elif container in ("array-list", "tensor-list"):
        kind = np.ndarray if container == "array-list" else torch.Tensor
        assert isinstance(got, list) and all(isinstance(g, kind) for g in got)
        per_cut = [np.asarray(g) for g in got]
    elif container == "padded":
        feats, lens = got
        assert isinstance(feats, torch.Tensor) and tuple(feats.shape) == (len(want), max(w.shape[0] for w in want), F)
        assert lens.dtype == torch.int64 and lens.tolist() == [w.shape[0] for w in want]
        for i, w in enumerate(want):
            assert torch.all(feats[i, w.shape[0]:] == np.float32(LOG_EPSILON))
        per_cut = [feats[i, : w.shape[0]].numpy() for i, w in enumerate(want)]
    else:
        assert container == "packed"
        feats, prefix = got
        assert isinstance(feats, torch.Tensor) and isinstance(prefix, np.ndarray) and prefix.dtype == np.int64
        assert prefix.tolist() == np.concatenate(([0], np.cumsum([w.shape[0] for w in want]))).tolist()
        per_cut = [feats[prefix[i]: prefix[i + 1]].numpy() for i in range(len(want))]
    assert len(per_cut) == len(want)
    for g, w in zip(per_cut, want):
        assert g.dtype == np.float32 and np.array_equal(g, w)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("row", ROWS, ids=[r[0] for r in ROWS])
def test_container_reaches_its_engine_call_in_the_kernel_dtype(row, dtype):
    _, call, method, sent, lens, offs, container, cuts = row
    ext = extractor()
    got = call(ext, dtype)
    assert ext._engine.calls == [(method, kernel_dtype(dtype) if sent == "kernel" else sent, lens, offs)]
    check_result(got, container, cuts)


@pytest.mark.parametrize("dtype", DTYPES)
def test_numpy_list_with_dither_takes_the_device_route_and_returns_numpy(dtype):
    ext = extractor(dither=0.1)
    got = ext.extract_batch(uneven(dtype), SR)
    assert ext._engine.calls == [("extract_device", "float32", list(UNEVEN), ALIGNED)]  # the noise makes every batch float
    assert isinstance(got, list) and all(isinstance(g, np.ndarray) and g.dtype == np.float32 for g in got)
    assert [g.shape for g in got] == [(frames(n), F) for n in UNEVEN]

