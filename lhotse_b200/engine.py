"""
ctypes binding of ``libb200feat.so`` (include/b200feat.h) + the host-side staging of ragged
batches.  torch is used here for device memory, pinned memory and streams only.

There is NO CPU fallback: if the library is missing, or no sm_90 GPU is visible, creating an
``Engine`` raises.  (The CPU oracle under ``oracle/`` is test infrastructure and is never
imported from this package.)
"""
from __future__ import annotations

import ctypes as C
import os
import threading
from concurrent.futures import ThreadPoolExecutor
from typing import List, Optional, Sequence, Tuple, Union

import numpy as np
import torch

from .plan import FEATURE_KINDS, FeaturePlan

LIB_NAME = "libb200feat.so"
_LIB = None
_LIB_LOCK = threading.Lock()

OUT_PACKED, OUT_PADDED = 0, 1
DT_F32, DT_I16 = 0, 1
KERNELS = {"auto": 0, "generic": 1, "fast": 2, "tc": 3}
KERNEL_NAMES = {1: "generic", 2: "fast", 3: "tc"}


class B200FeatError(RuntimeError):
    def __init__(self, code: int, msg: str):
        super().__init__(f"b200feat error {code}: {msg}")
        self.code = code


class PlanDesc(C.Structure):
    _fields_ = [
        ("struct_size", C.c_int32), ("feature", C.c_int32), ("frame_length", C.c_int32),
        ("frame_shift", C.c_int32), ("fft_length", C.c_int32), ("num_filters", C.c_int32),
        ("num_ceps", C.c_int32), ("snip_edges", C.c_int32), ("remove_dc_offset", C.c_int32),
        ("use_energy", C.c_int32), ("raw_energy", C.c_int32), ("use_fft_mag", C.c_int32),
        ("energy_style", C.c_int32), ("use_lifter", C.c_int32), ("kernel", C.c_int32),
        ("pad_mode", C.c_int32), ("preemph_coeff", C.c_float), ("energy_floor", C.c_float),
        ("mel_floor", C.c_float), ("log_spec_eps", C.c_float),
    ]


class BatchTotals(C.Structure):
    _fields_ = [("total_rows", C.c_int64), ("max_frames", C.c_int64), ("total_tiles", C.c_int64),
                ("span_samples", C.c_int64), ("out_floats", C.c_int64), ("meta_words", C.c_int64)]


class Stats(C.Structure):
    _fields_ = [("calls", C.c_int64), ("cuts", C.c_int64), ("frames", C.c_int64),
                ("samples", C.c_int64), ("kernel_launches", C.c_int64)]


EXPORTS = [
    "b200feat_version", "b200feat_global_error", "b200feat_create", "b200feat_destroy",
    "b200feat_last_error", "b200feat_num_frames", "b200feat_feature_dim", "b200feat_kernel_kind",
    "b200feat_meta_words", "b200feat_plan_words", "b200feat_plan_batch", "b200feat_extract", "b200feat_extract_host",
    "b200feat_extract_host_at", "b200feat_desc_num_frames",
    "b200feat_get_table", "b200feat_get_stats", "b200feat_set_output_affine", "b200feat_extract_host_ptrs",
]


def lib_path() -> str:
    """The in-tree library; `B200FEAT_LIBRARY` points a developer run at another build of the same sources
    (scripts/variant_build.py) — same ABI, same version check."""
    return os.environ.get("B200FEAT_LIBRARY") or os.path.join(os.path.dirname(os.path.abspath(__file__)), LIB_NAME)


def load_library():
    """Loads the in-tree CUDA library; raises (never falls back) when it is absent."""
    global _LIB
    with _LIB_LOCK:
        if _LIB is not None:
            return _LIB
        path = lib_path()
        if not os.path.exists(path):
            raise ImportError(
                f"{path} is missing: build it with `python -m lhotse_b200.build` (needs nvcc). "
                "lhotse_b200 has no CPU fallback."
            )
        lib = C.CDLL(path)
        vp, i32, i64 = C.c_void_p, C.c_int32, C.c_int64
        lib.b200feat_version.restype = C.c_int
        lib.b200feat_global_error.restype = C.c_char_p
        lib.b200feat_create.restype = C.c_int
        lib.b200feat_create.argtypes = [C.POINTER(PlanDesc), vp, vp, vp, vp, C.c_int, C.POINTER(vp)]
        lib.b200feat_destroy.restype = None
        lib.b200feat_destroy.argtypes = [vp]
        lib.b200feat_last_error.restype = C.c_char_p
        lib.b200feat_last_error.argtypes = [vp]
        lib.b200feat_num_frames.restype = i64
        lib.b200feat_num_frames.argtypes = [vp, i64]
        lib.b200feat_feature_dim.restype = i32
        lib.b200feat_feature_dim.argtypes = [vp]
        lib.b200feat_kernel_kind.restype = i32
        lib.b200feat_kernel_kind.argtypes = [vp]
        lib.b200feat_meta_words.restype = i64
        lib.b200feat_meta_words.argtypes = [i32]
        lib.b200feat_plan_words.restype = i64
        lib.b200feat_plan_words.argtypes = [vp, vp, i32, i32]
        lib.b200feat_plan_batch.restype = C.c_int
        lib.b200feat_plan_batch.argtypes = [vp, vp, vp, i32, i32, i32, vp, i64, C.POINTER(BatchTotals)]
        lib.b200feat_extract.restype = C.c_int
        lib.b200feat_extract.argtypes = [vp, vp, i32, vp, i32, C.POINTER(BatchTotals), vp, i32, C.c_float, vp]
        lib.b200feat_extract_host.restype = C.c_int
        lib.b200feat_extract_host.argtypes = [vp, vp, i32, vp, i32, vp, i32, C.c_float]
        lib.b200feat_extract_host_at.restype = C.c_int
        lib.b200feat_extract_host_at.argtypes = [vp, vp, i32, vp, vp, i32, vp, i32, C.c_float]
        lib.b200feat_desc_num_frames.restype = i64
        lib.b200feat_desc_num_frames.argtypes = [C.POINTER(PlanDesc), i64]
        lib.b200feat_get_table.restype = i64
        lib.b200feat_get_table.argtypes = [vp, i32, vp, i64]
        lib.b200feat_get_stats.restype = C.c_int
        lib.b200feat_get_stats.argtypes = [vp, C.POINTER(Stats)]
        lib.b200feat_extract_host_ptrs.restype = C.c_int
        lib.b200feat_extract_host_ptrs.argtypes = [vp, vp, i32, vp, i32, vp, i32, C.c_float]
        lib.b200feat_set_output_affine.restype = C.c_int
        lib.b200feat_set_output_affine.argtypes = [vp, vp, vp]
        if lib.b200feat_version() != 1:
            raise ImportError("libb200feat.so ABI version mismatch")
        _LIB = lib
        return lib


def plan_desc(plan: FeaturePlan, kernel: str = "auto") -> PlanDesc:
    """FeaturePlan -> b200feat_plan_desc (include/b200feat.h)."""
    d = PlanDesc()
    d.struct_size = C.sizeof(PlanDesc)
    d.feature = FEATURE_KINDS[plan.feature]
    d.frame_length, d.frame_shift, d.fft_length = plan.L, plan.S, plan.N
    d.num_filters, d.num_ceps = plan.num_filters, plan.num_ceps
    d.snip_edges, d.remove_dc_offset = int(plan.snip_edges), int(plan.remove_dc_offset)
    d.use_energy = (2 if getattr(plan, "energy_last", False) else 1) if plan.use_energy else 0  # 2: energy column last (htk_compat)
    d.raw_energy, d.use_fft_mag = int(plan.raw_energy), int(plan.use_fft_mag)
    d.energy_style = plan.energy_style
    d.use_lifter = int(plan.lifter is not None)
    d.kernel = KERNELS[kernel]
    d.pad_mode = int(getattr(plan, "pad_mode", 0))
    d.preemph_coeff, d.energy_floor = plan.preemph_coeff, plan.energy_floor
    d.mel_floor, d.log_spec_eps = plan.mel_floor, plan.log_spec_eps
    return d


def desc_num_frames(plan: FeaturePlan, num_samples: int) -> int:
    """Rows the kernels produce for a cut of `num_samples` under `plan` — the C library's own integer contract, callable
    without a GPU (negative: B200FEAT_ESHORT -5 when the cut cannot be framed)."""
    return int(load_library().b200feat_desc_num_frames(C.byref(plan_desc(plan)), int(num_samples)))


def _ptr(a: Optional[np.ndarray]):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


class Engine:
    """One handle = one (plan, device).  Thread-safe for `extract_device` on distinct streams."""

    def __init__(self, plan: FeaturePlan, device: Union[int, str, torch.device] = 0, kernel: str = "auto"):
        self.lib = load_library()
        self.plan = plan
        dev = torch.device(device) if not isinstance(device, int) else torch.device("cuda", device)
        if dev.type != "cuda":
            raise ValueError(f"lhotse_b200 extractors run on CUDA devices only, got {dev}")
        self.device_index = dev.index if dev.index is not None else (
            torch.cuda.current_device() if torch.cuda.is_available() else 0)
        self.device = torch.device("cuda", self.device_index)
        d = plan_desc(plan, kernel)
        tabs = [None if t is None else np.ascontiguousarray(t, dtype=np.float32)
                for t in (plan.window, plan.mel_bank, plan.dct, plan.lifter)]
        h = C.c_void_p()
        rc = self.lib.b200feat_create(C.byref(d), _ptr(tabs[0]), _ptr(tabs[1]), _ptr(tabs[2]), _ptr(tabs[3]),
                                      self.device_index, C.byref(h))
        if rc != 0:
            raise B200FeatError(rc, self.lib.b200feat_global_error().decode())
        self._h = h
        self.feature_dim = int(self.lib.b200feat_feature_dim(h))
        self.kernel = KERNEL_NAMES[int(self.lib.b200feat_kernel_kind(h))]

    def close(self):
        if getattr(self, "_h", None):
            self.lib.b200feat_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _check(self, rc: int):
        if rc != 0:
            raise B200FeatError(rc, self.lib.b200feat_last_error(self._h).decode())

    # ------------------------------------------------------------------ integer contract
    def num_frames(self, num_samples: int) -> int:
        t = int(self.lib.b200feat_num_frames(self._h, int(num_samples)))
        if t < 0:
            raise ValueError(
                f"a cut of {num_samples} samples cannot be framed with L={self.plan.L}, S={self.plan.S} "
                "(too short for reflect padding) — the reference raises on such inputs as well")
        return t

    def plan_batch(self, num_samples: Sequence[int], offsets: Optional[Sequence[int]] = None,
                   align: int = 4, out_mode: int = OUT_PACKED) -> Tuple[np.ndarray, BatchTotals]:
        B = len(num_samples)
        ns = np.ascontiguousarray(num_samples, dtype=np.int64)
        off = None if offsets is None else np.ascontiguousarray(offsets, dtype=np.int64)
        words = int(self.lib.b200feat_plan_words(self._h, _ptr(ns), B, out_mode))
        if words == -5:
            raise ValueError(self.lib.b200feat_last_error(self._h).decode())
        if words < 0:
            self._check(words)
        meta = np.empty(words, dtype=np.int64)
        tot = BatchTotals()
        rc = self.lib.b200feat_plan_batch(self._h, _ptr(ns), _ptr(off), B, align, out_mode, _ptr(meta), words, C.byref(tot))
        if rc == -5:
            raise ValueError(self.lib.b200feat_last_error(self._h).decode())
        self._check(rc)
        return meta[: tot.meta_words], tot

    # ------------------------------------------------------------------ device-resident path
    def extract_device(self, samples: torch.Tensor, num_samples: Sequence[int],
                       offsets: Optional[Sequence[int]] = None, out_mode: int = OUT_PACKED,
                       pad_value: float = 0.0, out: Optional[torch.Tensor] = None,
                       meta_dev: Optional[torch.Tensor] = None, totals: Optional[BatchTotals] = None,
                       ) -> Tuple[torch.Tensor, np.ndarray]:
        """samples: 1-D CUDA tensor (float32 or int16) holding the cuts at `offsets` (element units;
        default: back to back with 4-element alignment — see `pack_device`).
        Returns (features, row_prefix): packed (sum T, F) or padded (B, Tmax, F)."""
        assert samples.is_cuda and samples.dim() == 1 and samples.is_contiguous()
        if samples.data_ptr() % 16:
            # a view with a storage offset (`wave[1:]` is contiguous, so .contiguous() is a no-op): the kernels pick their
            # 64/128-bit load path from the element offset relative to this pointer and need the pointer itself aligned
            samples = samples.clone()
        dt = {torch.float32: DT_F32, torch.int16: DT_I16}[samples.dtype]
        B = len(num_samples)
        if meta_dev is None or totals is None:
            meta, totals = self.plan_batch(num_samples, offsets, out_mode=out_mode)
            assert totals.span_samples <= samples.numel(), "sample buffer shorter than offsets + lengths"
            meta_dev = torch.from_numpy(meta).to(samples.device, non_blocking=False)
            row_prefix = meta[2 * B: 3 * B + 1]
        else:
            row_prefix = None
        shape = (B, totals.max_frames, self.feature_dim) if out_mode == OUT_PADDED else (totals.total_rows, self.feature_dim)
        if out is None:
            # one flat allocation of totals.out_floats: the feature rows, then (whisper-fbank) the library's scratch tail
            flat = torch.empty(int(totals.out_floats), dtype=torch.float32, device=samples.device)
        else:
            assert out.is_cuda and out.is_contiguous() and out.numel() >= totals.out_floats
            flat = out.view(-1)
        stream = torch.cuda.current_stream(samples.device).cuda_stream
        self._check(self.lib.b200feat_extract(self._h, samples.data_ptr(), dt, meta_dev.data_ptr(), B,
                                              C.byref(totals), flat.data_ptr(), out_mode, float(pad_value), stream))
        if out is None:
            out = flat[: shape[0] * shape[1] * (shape[2] if len(shape) == 3 else 1)].view(shape)
        return out, row_prefix

    # ------------------------------------------------------------------ host-to-host path
    def extract_host(self, samples: Union[np.ndarray, torch.Tensor], num_samples: Sequence[int],
                     out_mode: int = OUT_PACKED, pad_value: float = 0.0,
                     out: Optional[Union[np.ndarray, torch.Tensor]] = None,
                     offsets: Optional[Sequence[int]] = None):
        """samples: the cuts in ONE host buffer (numpy or CPU torch tensor, float32 or int16; pinned memory makes the
        H2D copies asynchronous), back to back or at the increasing element `offsets` (`stage_host` aligns them so
        that the kernels stay on their vector-load path).  Blocks until `out` is filled."""
        if isinstance(samples, torch.Tensor):
            assert not samples.is_cuda and samples.is_contiguous()
            dt = {torch.float32: DT_F32, torch.int16: DT_I16}[samples.dtype]
            sptr, numel = samples.data_ptr(), samples.numel()
        else:
            samples = np.ascontiguousarray(samples)
            dt = {np.dtype(np.float32): DT_F32, np.dtype(np.int16): DT_I16}[samples.dtype]
            sptr, numel = samples.ctypes.data, samples.size
        ns = np.ascontiguousarray(num_samples, dtype=np.int64)
        off = None if offsets is None else np.ascontiguousarray(offsets, dtype=np.int64)
        assert (int(ns.sum()) if off is None else int(off[-1] + ns[-1])) <= numel
        B = len(ns)
        p = self.plan
        if p.snip_edges and p.feature not in ("whisper-fbank", "librosa-fbank"):
            Ts = np.where(ns < p.L, 0, 1 + (ns - p.L) // p.S)
        else:
            Ts = (ns + p.S // 2) // p.S
        tmax = int(Ts.max())
        rows = B * tmax if out_mode == OUT_PADDED else int(Ts.sum())
        shape = (B, tmax, self.feature_dim) if out_mode == OUT_PADDED else (rows, self.feature_dim)
        if out is None:
            # pinned (page-locked) result: the D2H copies run asynchronously at full PCIe speed; torch's caching
            # host allocator makes repeated allocations of the same size cheap
            out = torch.empty(shape, dtype=torch.float32, pin_memory=True).numpy()
        optr = out.data_ptr() if isinstance(out, torch.Tensor) else out.ctypes.data
        rc = self.lib.b200feat_extract_host_at(self._h, sptr, dt, _ptr(ns), _ptr(off), B, optr, out_mode, float(pad_value))
        if rc == -5:
            raise ValueError(self.lib.b200feat_last_error(self._h).decode())
        self._check(rc)
        return out, np.concatenate(([0], np.cumsum(Ts))).astype(np.int64)

    def extract_host_list(self, arrays: Sequence[np.ndarray], dtype=np.float32, sub_bytes: int = 64 << 20):
        """A LIST of separately allocated host waveforms -> packed (sum T_i, F) features in pinned host memory + row prefix.
        One C call (`b200feat_extract_host_ptrs`): the library gathers the cuts into its pinned staging slots with its own
        thread pool (non-temporal stores) and overlaps that with the H2D / kernel / D2H pipeline; the GIL is released
        throughout.  `B200FEAT_PY_GATHER=1` selects the round-1 route (Python staging threads) for A/B measurements."""
        if os.environ.get("B200FEAT_PY_GATHER") != "1":
            want = np.dtype(dtype)
            arrs = [np.ascontiguousarray(a, dtype=want).reshape(-1) for a in arrays]
            B = len(arrs)
            ns = np.asarray([a.shape[0] for a in arrs], dtype=np.int64)
            p = self.plan
            if p.snip_edges and p.feature not in ("whisper-fbank", "librosa-fbank"):
                Ts = np.where(ns < p.L, 0, 1 + (ns - p.L) // p.S)
            else:
                Ts = (ns + p.S // 2) // p.S
            prefix = np.concatenate(([0], np.cumsum(Ts))).astype(np.int64)
            out = torch.empty((int(prefix[-1]), self.feature_dim), dtype=torch.float32, pin_memory=torch.cuda.is_available()).numpy()
            ptrs = (C.c_void_p * B)(*[a.ctypes.data for a in arrs])
            rc = self.lib.b200feat_extract_host_ptrs(self._h, ptrs, DT_I16 if want == np.int16 else DT_F32, _ptr(ns), B, out.ctypes.data,
                                                     OUT_PACKED, 0.0)
            if rc == -5:
                raise ValueError(self.lib.b200feat_last_error(self._h).decode())
            self._check(rc)
            return out, prefix
        lens = [int(a.shape[0]) for a in arrays]
        B = len(lens)
        p = self.plan
        ns = np.asarray(lens, dtype=np.int64)
        if p.snip_edges and p.feature not in ("whisper-fbank", "librosa-fbank"):
            Ts = np.where(ns < p.L, 0, 1 + (ns - p.L) // p.S)
        else:
            Ts = (ns + p.S // 2) // p.S
        prefix = np.concatenate(([0], np.cumsum(Ts))).astype(np.int64)
        pin = torch.cuda.is_available()
        out = torch.empty((int(prefix[-1]), self.feature_dim), dtype=torch.float32, pin_memory=pin).numpy()
        esz = 2 if np.dtype(dtype) == np.int16 else 4
        groups = _groups(lens, sub_bytes, esz, ramp=True)
        tdt = torch.int16 if esz == 2 else torch.float32
        cap = max(_aligned_offsets(lens[b0:b1], 4)[1] for b0, b1 in groups)
        bufs = [torch.empty(cap, dtype=tdt, pin_memory=pin) for _ in range(min(2, len(groups)))]
        stager = (lambda j: stage_host(arrays[groups[j][0]: groups[j][1]], dtype=dtype, out=bufs[j % 2]))
        cur, nxt = stager(0), None
        side = ThreadPoolExecutor(max_workers=1) if len(groups) > 1 else None  # drives the staging of j + 1 (fans out to the pool)
        try:
            for j, (b0, b1) in enumerate(groups):
                if side is not None and j + 1 < len(groups):
                    nxt = side.submit(stager, j + 1)
                buf, glens, goffs = cur
                self.extract_host(buf, glens, out=out[prefix[b0]: prefix[b1]], offsets=goffs)
                if nxt is not None:
                    cur, nxt = nxt.result(), None
        finally:
            if side is not None:
                side.shutdown(wait=True)
        return out, prefix

    def set_output_affine(self, scale: Optional[np.ndarray], shift: Optional[np.ndarray]) -> None:
        """Fuses `v * scale[c] + shift[c]` (per output column c; the padding value too) into the kernels' epilogue —
        e.g. GlobalMVN with scale = 1 / std, shift = -mean / std.  `None, None` switches it off."""
        if scale is None or shift is None:
            self._check(self.lib.b200feat_set_output_affine(self._h, None, None))
            return
        sc = np.ascontiguousarray(scale, dtype=np.float32).reshape(-1)
        sh = np.ascontiguousarray(shift, dtype=np.float32).reshape(-1)
        if sc.shape[0] != self.feature_dim or sh.shape[0] != self.feature_dim:
            raise ValueError(f"output affine needs {self.feature_dim} values per table, got {sc.shape[0]} / {sh.shape[0]}")
        self._check(self.lib.b200feat_set_output_affine(self._h, _ptr(sc), _ptr(sh)))

    # ------------------------------------------------------------------ introspection
    def get_table(self, which: int) -> np.ndarray:
        cap = max(self.plan.K * max(self.plan.num_filters, 1), self.plan.N * 2, 8192)
        buf = np.empty(cap, dtype=np.float32)
        n = int(self.lib.b200feat_get_table(self._h, which, _ptr(buf), cap))
        if n < 0:
            self._check(n)
        return buf[:n].copy()

    def stats(self) -> dict:
        s = Stats()
        self._check(self.lib.b200feat_get_stats(self._h, C.byref(s)))
        return {k: int(getattr(s, k)) for k, _ in Stats._fields_}


# ---- host staging --------------------------------------------------------------------------------------------------
# Gathering B separately allocated waveforms into one pinned buffer is a plain memcpy, and ONE host thread moves only a
# fraction of what PCIe takes, so the copies are spread over a small thread pool
# (numpy / torch copies release the GIL) and overlapped with the transfer of the previous group.
STAGING_THREADS = max(1, min(8, (os.cpu_count() or 2) // 2, int(os.environ.get("B200FEAT_STAGING_THREADS", "8"))))
_POOL = None
_POOL_PID = None


def _copy_pool() -> Optional[ThreadPoolExecutor]:
    """Per-process pool (threads do not survive fork(): DataLoader workers get their own on first use)."""
    global _POOL, _POOL_PID
    if STAGING_THREADS <= 1:
        return None
    if _POOL is None or _POOL_PID != os.getpid():
        _POOL, _POOL_PID = ThreadPoolExecutor(max_workers=STAGING_THREADS, thread_name_prefix="b200feat-stage"), os.getpid()
    return _POOL


def _groups(lens: Sequence[int], target_bytes: int, esz: int, ramp: bool = False) -> List[Tuple[int, int]]:
    """Consecutive index ranges [b0, b1) of roughly `target_bytes` each; with `ramp` the first two groups are 1/4 and 1/2
    of that (a software pipeline starts sooner on a small first stage)."""
    out, b0, acc = [], 0, 0
    for i, n in enumerate(lens):
        acc += n * esz
        if acc >= (target_bytes >> max(0, 2 - len(out)) if ramp else target_bytes):
            out.append((b0, i + 1))
            b0, acc = i + 1, 0
    if b0 < len(lens):
        out.append((b0, len(lens)))
    return out


def _aligned_offsets(lens: Sequence[int], align: int) -> Tuple[List[int], int]:
    offs, cur = [], 0
    for n in lens:
        cur = (cur + align - 1) // align * align
        offs.append(cur)
        cur += n
    return offs, cur


def pack_device(tensors: List[torch.Tensor], device: torch.device, align: int = 4,
                dtype: torch.dtype = torch.float32) -> Tuple[torch.Tensor, List[int], List[int]]:
    """Packs 1-D waveforms into one ragged device buffer (each start aligned to `align` elements).
    Host tensors are gathered into ONE pinned staging buffer by the staging threads, group by group, and every finished
    group is sent to the device at once (its H2D copy overlaps the gathering of the next group); device tensors are
    copied device-to-device."""
    lens = [int(t.numel()) for t in tensors]
    offs, total = _aligned_offsets(lens, align)
    if all(not t.is_cuda for t in tensors):
        cuda = torch.cuda.is_available()
        stage = torch.empty(total, dtype=dtype, pin_memory=cuda)
        pool = _copy_pool()
        esz = stage.element_size()

        view = stage.numpy()

        def gather(b0, b1):
            for i in range(b0, b1):
                if i > 0:
                    view[offs[i - 1] + lens[i - 1]: offs[i]] = 0  # alignment gap: defined bytes only
                t = tensors[i]
                if t.requires_grad or not t.is_contiguous():
                    stage[offs[i]: offs[i] + lens[i]].copy_(t.detach().reshape(-1))
                else:  # a numpy view of the tensor: plain memcpy (3x torch's CPU copy_ on this path), GIL released
                    view[offs[i]: offs[i] + lens[i]] = t.numpy().reshape(-1)

        if pool is None or total * esz < (8 << 20) or not cuda:
            gather(0, len(tensors))
            return stage.to(device, non_blocking=True), lens, offs
        dev = torch.empty(total, dtype=dtype, device=device)
        groups = _groups(lens, max(4 << 20, total * esz // (4 * STAGING_THREADS)), esz)
        futs = [pool.submit(gather, b0, b1) for b0, b1 in groups]
        for (b0, b1), f in zip(groups, futs):
            f.result()
            e0, e1 = offs[b0], offs[b1 - 1] + lens[b1 - 1]
            dev[e0:e1].copy_(stage[e0:e1], non_blocking=True)
        return dev, lens, offs
    buf = torch.empty(total, dtype=dtype, device=device)
    for t, o, n in zip(tensors, offs, lens):
        buf[o:o + n].copy_(t.reshape(-1), non_blocking=True)
    return buf, lens, offs


def stage_host(arrays: Sequence[np.ndarray], dtype=np.float32, align: int = 4,
               out: Optional[torch.Tensor] = None) -> Tuple[torch.Tensor, List[int], List[int]]:
    """Copies 1-D host waveforms into ONE pinned buffer (`out`, or a fresh one), each start aligned to `align` elements
    (gaps are zero-filled so that no uninitialised memory crosses PCIe), using the staging threads.
    Returns (buffer, lengths, offsets) for `Engine.extract_host(offsets=)`."""
    lens = [int(a.shape[0]) for a in arrays]
    offs, cur = _aligned_offsets(lens, align)
    tdt = torch.int16 if np.dtype(dtype) == np.int16 else torch.float32
    stage = out if out is not None else torch.empty(max(cur, 1), dtype=tdt, pin_memory=torch.cuda.is_available())
    assert stage.dtype == tdt and stage.numel() >= cur
    view = stage.numpy()

    def gather(b0, b1):
        for i in range(b0, b1):
            if i > 0:
                view[offs[i - 1] + lens[i - 1]: offs[i]] = 0
            view[offs[i]: offs[i] + lens[i]] = arrays[i]

    pool = _copy_pool()
    esz = 2 if tdt == torch.int16 else 4
    if pool is None or cur * esz < (8 << 20):
        gather(0, len(arrays))
    else:
        for f in [pool.submit(gather, b0, b1) for b0, b1 in _groups(lens, max(4 << 20, cur * esz // (2 * STAGING_THREADS)), esz)]:
            f.result()
    return stage[:max(cur, 1)], lens, offs
