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
from concurrent.futures import Future, ThreadPoolExecutor
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


class FlacStreamInfo(C.Structure):
    _fields_ = [("struct_size", C.c_int32), ("sample_rate", C.c_int32), ("channels", C.c_int32), ("bits_per_sample", C.c_int32),
                ("min_block_size", C.c_int32), ("max_block_size", C.c_int32), ("variable_blocking", C.c_int32),
                ("reserved", C.c_int32), ("total_samples", C.c_int64), ("audio_offset", C.c_int64), ("md5", C.c_uint8 * 16)]


# b200feat_flac_frame / b200feat_flac_job as numpy record layouts (the job table is built with vector operations)
FLAC_FRAME_DTYPE = np.dtype([("byte_offset", "<i8"), ("first_sample", "<i8"), ("block_size", "<i4"), ("byte_length", "<i4")])
FLAC_JOB_DTYPE = np.dtype([("src_byte", "<i8"), ("dst_elem", "<i8"), ("scratch_elem", "<i8"), ("coded_number", "<i8"),
                           ("byte_length", "<i4"), ("block_size", "<i4"), ("channels", "<i4"), ("want_channel", "<i4"),
                           ("skip", "<i4"), ("count", "<i4"), ("variable_blocking", "<i4"), ("reserved", "<i4")])
FLAC_STATUS = {1: "inconsistent job", 2: "bad frame header", 3: "CRC-16 mismatch", 4: "reserved code", 5: "invalid LPC precision",
               6: "negative LPC shift", 7: "partition order does not fit the block", 8: "sample out of range",
               9: "frame truncated", 10: "frame shorter than its byte range"}

# b200feat_mix_track / b200feat_mix_cut as numpy record layouts (the staged-mix tables are built with vector operations)
MIX_TRACK_DTYPE = np.dtype([("struct_size", "<i4"), ("source", "<i4"), ("src_elem", "<i8"), ("num_samples", "<i8"),
                            ("mix_offset", "<i8"), ("snr_factor", "<f8"), ("cut", "<i4"), ("role", "<i4")])
MIX_CUT_DTYPE = np.dtype([("struct_size", "<i4"), ("mode", "<i4"), ("out_elem", "<i8"), ("mix_len", "<i8"), ("target_len", "<i8"),
                          ("first_track", "<i4"), ("num_tracks", "<i4"), ("ref_track", "<i4"), ("reserved", "<i4")])
MIX_ROLE_MIXED, MIX_ROLE_ENERGY = 0, 1
MIX_F32, MIX_SCALED_FIRST = 0, 1
MIX_SRC_F32 = 2  # b200feat_mix_track.source of a track in the float32 track buffer (src2)

# b200feat_resample_stage as a numpy record layout (the transform route's stage table is built with vector operations)
RESAMPLE_STAGE_DTYPE = np.dtype([("struct_size", "<i4"), ("table", "<i4"), ("source", "<i4"), ("target", "<i4"), ("depth", "<i4"),
                                 ("scale_in", "<f4"), ("scale_out", "<f4"), ("reserved", "<i4"), ("in_elem", "<i8"),
                                 ("in_len", "<i8"), ("out_elem", "<i8"), ("out_len", "<i8"), ("target_len", "<i8")])
RESAMPLE_SRC0, RESAMPLE_SRC1, RESAMPLE_MID = 0, 1, 2
RESAMPLE_TO_MID, RESAMPLE_TO_OUT = 0, 1

# b200feat_reverb_rir / b200feat_reverb_cut as numpy record layouts
REVERB_RIR_DTYPE = np.dtype([("struct_size", "<i4"), ("source", "<i4"), ("src_elem", "<i8"), ("num_samples", "<i8")])
REVERB_CUT_DTYPE = np.dtype([("struct_size", "<i4"), ("rir", "<i4"), ("normalize", "<i4"), ("reserved", "<i4"), ("in_elem", "<i8"),
                             ("in_len", "<i8"), ("out_elem", "<i8"), ("target_len", "<i8")])
REVERB_MAX_RIR = 65536  # B200FEAT_REVERB_MAX_RIR
REVERB_RIR_F32 = 2      # B200FEAT_REVERB_RIR_F32: b200feat_reverb_ex's float32 RIR source

# b200feat_rir_gen as a numpy record layout
RIR_GEN_DTYPE = np.dtype([("struct_size", "<i4"), ("sampling_rate", "<i4"), ("t60", "<f8"), ("r", "<f8"), ("d0", "<f8"),
                          ("tau", "<f8"), ("b0", "<f4"), ("b1", "<f4"), ("b2", "<f4"), ("a1", "<f4"), ("a2", "<f4"),
                          ("reserved", "<i4"), ("cdf_elem", "<i8"), ("draw_elem", "<i8"), ("comb_len", "<i8"),
                          ("out_elem", "<i8"), ("out_len", "<i8")])
RIRGEN_TAPS = 106  # B200FEAT_RIRGEN_TAPS

# b200feat_specaug_warp / b200feat_specaug_mask as numpy record layouts
SPECAUG_WARP_DTYPE = np.dtype([("struct_size", "<i4"), ("seq", "<i4"), ("start", "<i4"), ("len", "<i4"), ("center", "<i4"),
                               ("warped", "<i4")])
SPECAUG_MASK_DTYPE = np.dtype([("struct_size", "<i4"), ("seq", "<i4"), ("axis", "<i4"), ("start", "<i4"), ("end", "<i4"),
                               ("reserved", "<i4")])
SPECAUG_TIME, SPECAUG_FEATURE = 0, 1

# b200feat_featmix_track / b200feat_featmix_cut as numpy record layouts
FEATMIX_TRACK_DTYPE = np.dtype([("struct_size", "<i4"), ("cut", "<i4"), ("flags", "<i4"), ("stored_rows", "<i4"), ("num_rows", "<i4"),
                                ("offset", "<i4"), ("value", "<f4"), ("reserved", "<i4"), ("src_elem", "<i8"), ("snr_factor", "<f8")])
FEATMIX_CUT_DTYPE = np.dtype([("struct_size", "<i4"), ("mode", "<i4"), ("law", "<i4"), ("num_rows", "<i4"), ("mix_rows", "<i4"),
                              ("first_track", "<i4"), ("num_tracks", "<i4"), ("ref_track", "<i4"), ("pad_value", "<f4"),
                              ("reserved", "<i4")])
FEATMIX_LOG, FEATMIX_LINEAR = 0, 1
FEATMIX_COPY, FEATMIX_MIX = 0, 1
FEATMIX_MIXED, FEATMIX_ENERGY = 1, 2


EXPORTS = [
    "b200feat_version", "b200feat_global_error", "b200feat_create", "b200feat_destroy",
    "b200feat_last_error", "b200feat_num_frames", "b200feat_feature_dim", "b200feat_kernel_kind",
    "b200feat_meta_words", "b200feat_plan_words", "b200feat_plan_batch", "b200feat_extract", "b200feat_extract_host",
    "b200feat_extract_host_at", "b200feat_desc_num_frames",
    "b200feat_get_table", "b200feat_get_stats", "b200feat_set_output_affine", "b200feat_extract_host_ptrs",
    "b200feat_flac_index", "b200feat_flac_decode", "b200feat_mix_work_bytes", "b200feat_mix",
    "b200feat_resample_table", "b200feat_resample_work_bytes", "b200feat_resample", "b200feat_mix_ex",
    "b200feat_reverb_work_bytes", "b200feat_reverb", "b200feat_specaug_work_bytes", "b200feat_specaug",
    "b200feat_reverb_ex", "b200feat_rir_generate_work_bytes", "b200feat_rir_generate",
    "b200feat_feature_mix_work_bytes", "b200feat_feature_mix", "b200feat_backward_work_bytes", "b200feat_backward",
    "b200feat_collate_audio_work_bytes", "b200feat_collate_audio", "b200feat_extract_keep_raw", "b200feat_whisper_backward",
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
        lib.b200feat_flac_index.restype = i64
        lib.b200feat_flac_index.argtypes = [vp, i64, C.POINTER(FlacStreamInfo), vp, i64]
        lib.b200feat_flac_decode.restype = C.c_int
        lib.b200feat_flac_decode.argtypes = [vp, vp, i32, vp, i64, vp, vp, i64, vp]
        lib.b200feat_mix_work_bytes.restype = i64
        lib.b200feat_mix_work_bytes.argtypes = [i32, i32]
        lib.b200feat_mix.restype = C.c_int
        lib.b200feat_mix.argtypes = [vp, vp, i64, vp, i64, vp, i32, vp, i32, vp, i64, vp, i64, vp]
        lib.b200feat_mix_ex.restype = C.c_int
        lib.b200feat_mix_ex.argtypes = [vp, vp, i64, vp, i64, vp, i64, vp, i32, vp, i32, vp, i64, vp, i64, vp]
        lib.b200feat_resample_table.restype = C.c_int
        lib.b200feat_resample_table.argtypes = [vp, i32, i32, vp, i32, i32, i32, C.POINTER(i32)]
        lib.b200feat_resample_work_bytes.restype = i64
        lib.b200feat_resample_work_bytes.argtypes = [i32]
        lib.b200feat_resample.restype = C.c_int
        lib.b200feat_resample.argtypes = [vp, vp, i64, vp, i64, vp, i64, vp, i32, vp, i64, vp, i64, vp]
        lib.b200feat_reverb_work_bytes.restype = i64
        lib.b200feat_reverb_work_bytes.argtypes = [vp, i32, vp, i32]
        lib.b200feat_reverb.restype = C.c_int
        lib.b200feat_reverb.argtypes = [vp, vp, i64, vp, i64, vp, i64, vp, i32, vp, i32, vp, i64, vp, i64, vp]
        lib.b200feat_reverb_ex.restype = C.c_int
        lib.b200feat_reverb_ex.argtypes = [vp, vp, i64, vp, i64, vp, i64, vp, i64, vp, i32, vp, i32, vp, i64, vp, i64, vp]
        lib.b200feat_rir_generate_work_bytes.restype = i64
        lib.b200feat_rir_generate_work_bytes.argtypes = [vp, i32]
        lib.b200feat_rir_generate.restype = C.c_int
        lib.b200feat_rir_generate.argtypes = [vp, vp, i64, vp, i64, vp, vp, i32, vp, i64, vp, i64, vp]
        lib.b200feat_specaug_work_bytes.restype = i64
        lib.b200feat_specaug_work_bytes.argtypes = [i32, i32, i32, i32, i32]
        lib.b200feat_specaug.restype = C.c_int
        lib.b200feat_specaug.argtypes = [vp, vp, vp, i32, i32, i32, vp, i32, vp, i32, vp, i64, vp]
        lib.b200feat_feature_mix_work_bytes.restype = i64
        lib.b200feat_feature_mix_work_bytes.argtypes = [i32, i32]
        lib.b200feat_feature_mix.restype = C.c_int
        lib.b200feat_feature_mix.argtypes = [vp, vp, i64, vp, i32, vp, i32, i32, vp, i32, C.c_float, vp, i64, vp]
        lib.b200feat_backward_work_bytes.restype = i64
        lib.b200feat_backward_work_bytes.argtypes = [vp, vp, i32]
        lib.b200feat_backward.restype = C.c_int
        lib.b200feat_backward.argtypes = [vp, vp, i32, vp, vp, i32, vp, vp, vp, vp, i64, vp]
        lib.b200feat_extract_keep_raw.restype = C.c_int
        lib.b200feat_extract_keep_raw.argtypes = [vp, vp, i32, vp, i32, C.POINTER(BatchTotals), vp, vp, vp]
        lib.b200feat_whisper_backward.restype = C.c_int
        lib.b200feat_whisper_backward.argtypes = [vp, vp, i32, vp, vp, i32, vp, vp, vp, vp, vp, vp, i64, vp]
        lib.b200feat_collate_audio_work_bytes.restype = i64
        lib.b200feat_collate_audio_work_bytes.argtypes = [i32]
        lib.b200feat_collate_audio.restype = C.c_int
        lib.b200feat_collate_audio.argtypes = [vp, vp, i32, i64, vp, vp, i32, i64, vp, vp, i64, vp]
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


def flac_index(data) -> Tuple[FlacStreamInfo, np.ndarray]:
    """`b200feat_flac_index` over a whole FLAC file in memory (bytes or a uint8 array): (STREAMINFO, frame table as a
    FLAC_FRAME_DTYPE array).  Pure host work (no device); ctypes releases the GIL for the scan.  Raises ValueError when the
    data is not a native FLAC stream."""
    lib = load_library()
    buf = np.frombuffer(data, dtype=np.uint8) if isinstance(data, (bytes, bytearray, memoryview)) else np.ascontiguousarray(data, np.uint8)
    info = FlacStreamInfo()
    info.struct_size = C.sizeof(FlacStreamInfo)
    cap = max(16, buf.size // 1024)
    while True:
        frames = np.empty(cap, dtype=FLAC_FRAME_DTYPE)
        n = int(lib.b200feat_flac_index(buf.ctypes.data, buf.size, C.byref(info), frames.ctypes.data, cap))
        if n < 0:
            raise ValueError(lib.b200feat_global_error().decode())
        if n <= cap:
            return info, frames[:n]
        cap = n


def flac_decode(bytes_dev: torch.Tensor, jobs_dev: torch.Tensor, njobs: int, out: torch.Tensor, status: torch.Tensor,
                scratch: Optional[torch.Tensor]) -> None:
    """Launches `b200feat_flac_decode` on the current stream of `out`'s device (asynchronous; `status` holds the per-job
    B200FEAT_FLAC_* codes once it has run)."""
    lib = load_library()
    stream = torch.cuda.current_stream(out.device).cuda_stream
    rc = lib.b200feat_flac_decode(bytes_dev.data_ptr(), jobs_dev.data_ptr(), int(njobs), out.data_ptr(), out.numel(),
                                  status.data_ptr(), None if scratch is None else scratch.data_ptr(),
                                  0 if scratch is None else scratch.numel() * 4, stream)
    if rc != 0:
        raise B200FeatError(rc, lib.b200feat_global_error().decode())


def mix(src0: Optional[torch.Tensor], src1: Optional[torch.Tensor], tracks: np.ndarray, cuts: np.ndarray, out: torch.Tensor,
        handle=None, src2: Optional[torch.Tensor] = None) -> None:
    """Launches `b200feat_mix_ex` on the current stream of `out`'s device (asynchronous): the int16 device sources and the
    float32 track buffer `src2` (None = empty), the host track / cut tables (MIX_TRACK_DTYPE / MIX_CUT_DTYPE arrays, pinned or
    not: they are read by a copy on the same stream, so a pinned table must not change until that copy has run) and the
    float32 output.  Raises B200FeatError when the library refuses the tables."""
    lib = load_library()
    stream = torch.cuda.current_stream(out.device).cuda_stream
    assert tracks.dtype == MIX_TRACK_DTYPE and cuts.dtype == MIX_CUT_DTYPE and out.dtype == torch.float32
    assert src2 is None or src2.dtype == torch.float32
    work = torch.empty(max(int(lib.b200feat_mix_work_bytes(len(tracks), len(cuts))), 1), dtype=torch.uint8, device=out.device)

    def src(t):
        return (None, 0) if t is None or t.numel() == 0 else (t.data_ptr(), t.numel())

    (p0, n0), (p1, n1), (p2, n2) = src(src0), src(src1), src(src2)
    rc = lib.b200feat_mix_ex(handle, p0, n0, p1, n1, p2, n2, tracks.ctypes.data, len(tracks), cuts.ctypes.data, len(cuts),
                             out.data_ptr(), out.numel(), work.data_ptr(), work.numel(), stream)
    if rc != 0:
        msg = (lib.b200feat_last_error(handle) if handle is not None else lib.b200feat_global_error()).decode()
        raise B200FeatError(rc, msg)


def _raise(lib, rc: int, handle) -> None:
    msg = (lib.b200feat_last_error(handle) if handle is not None else lib.b200feat_global_error()).decode()
    raise B200FeatError(rc, msg)


def resample_table(orig: int, new: int, kernel: np.ndarray, width: int, device, handle=None) -> int:
    """The id of the rate pair's table on `device` (`b200feat_resample_table`): `kernel` is the float32 [N][K] table, read
    only the first time the pair is seen on that device."""
    lib = load_library()
    kernel = np.ascontiguousarray(kernel, dtype=np.float32)
    tid = C.c_int32(-1)
    with torch.cuda.device(torch.device(device)):
        rc = lib.b200feat_resample_table(handle, int(orig), int(new), kernel.ctypes.data, kernel.shape[0], kernel.shape[1],
                                         int(width), C.byref(tid))
    if rc != 0:
        _raise(lib, rc, handle)
    return int(tid.value)


def resample(src0: Optional[torch.Tensor], src1: Optional[torch.Tensor], mid: Optional[torch.Tensor], stages: np.ndarray,
             out: torch.Tensor, handle=None) -> None:
    """Launches `b200feat_resample` on the current stream of `out`'s device (asynchronous): the int16 device sources and the
    float32 intermediate buffer (None = empty), the host stage table (RESAMPLE_STAGE_DTYPE, sorted by depth) and the float32
    output.  Raises B200FeatError when the library refuses the table."""
    lib = load_library()
    stream = torch.cuda.current_stream(out.device).cuda_stream
    assert stages.dtype == RESAMPLE_STAGE_DTYPE and out.dtype == torch.float32
    work = torch.empty(max(int(lib.b200feat_resample_work_bytes(len(stages))), 1), dtype=torch.uint8, device=out.device)

    def src(t):
        return (None, 0) if t is None or t.numel() == 0 else (t.data_ptr(), t.numel())

    (p0, n0), (p1, n1), (pm, nm) = src(src0), src(src1), src(mid)
    with torch.cuda.device(out.device):
        rc = lib.b200feat_resample(handle, p0, n0, p1, n1, pm, nm, stages.ctypes.data, len(stages), out.data_ptr(), out.numel(),
                                   work.data_ptr(), work.numel(), stream)
    if rc != 0:
        _raise(lib, rc, handle)


def reverb(src0: Optional[torch.Tensor], src1: Optional[torch.Tensor], x: torch.Tensor, rirs: np.ndarray, cuts: np.ndarray,
           out: torch.Tensor, handle=None, rir32: Optional[torch.Tensor] = None) -> None:
    """Launches `b200feat_reverb_ex` on the current stream of `out`'s device (asynchronous): the int16 device sources of the
    RIRs, the float32 input `x`, the host RIR / cut tables (REVERB_RIR_DTYPE / REVERB_CUT_DTYPE; copied before this returns)
    and the float32 output; `rir32`, the float32 RIRs of records whose source is REVERB_RIR_F32 (generated ones).  Raises
    B200FeatError when the library refuses the tables."""
    lib = load_library()
    stream = torch.cuda.current_stream(out.device).cuda_stream
    assert rirs.dtype == REVERB_RIR_DTYPE and cuts.dtype == REVERB_CUT_DTYPE
    assert x.dtype == torch.float32 and out.dtype == torch.float32
    rirs, cuts = np.ascontiguousarray(rirs), np.ascontiguousarray(cuts)
    nbytes = int(lib.b200feat_reverb_work_bytes(rirs.ctypes.data, len(rirs), cuts.ctypes.data, len(cuts)))
    work = torch.empty(max(nbytes, 1), dtype=torch.uint8, device=out.device)

    def src(t):
        return (None, 0) if t is None or t.numel() == 0 else (t.data_ptr(), t.numel())

    (p0, n0), (p1, n1), (p2, n2), (px, nx) = src(src0), src(src1), src(rir32), src(x)
    with torch.cuda.device(out.device):
        rc = lib.b200feat_reverb_ex(handle, p0, n0, p1, n1, p2, n2, px, nx, rirs.ctypes.data, len(rirs), cuts.ctypes.data,
                                    len(cuts), out.data_ptr(), out.numel(), work.data_ptr(), work.numel(), stream)
    if rc != 0:
        _raise(lib, rc, handle)


def rir_generate(draws: torch.Tensor, cdf: torch.Tensor, table: np.ndarray, rirs: np.ndarray, out: torch.Tensor,
                 handle=None) -> None:
    """Launches `b200feat_rir_generate` on the current stream of `out`'s device (asynchronous): the float64 device draws, the
    float32 device distributions, the host 8 -> 1 resampler table (RIRGEN_TAPS floats) and records (RIR_GEN_DTYPE; both
    copied before this returns) and the float32 output at 8 x sr.  Raises B200FeatError when the library refuses them."""
    lib = load_library()
    stream = torch.cuda.current_stream(out.device).cuda_stream
    assert rirs.dtype == RIR_GEN_DTYPE and draws.dtype == torch.float64 and cdf.dtype == torch.float32
    assert out.dtype == torch.float32
    rirs = np.ascontiguousarray(rirs)
    table = np.ascontiguousarray(table, dtype=np.float32)
    assert table.shape == (RIRGEN_TAPS,)
    with torch.cuda.device(out.device):  # the sort's scratch query depends on the device
        nbytes = int(lib.b200feat_rir_generate_work_bytes(rirs.ctypes.data, len(rirs)))
        work = torch.empty(max(nbytes, 1), dtype=torch.uint8, device=out.device)
        rc = lib.b200feat_rir_generate(handle, draws.data_ptr(), draws.numel(), cdf.data_ptr(), cdf.numel(),
                                       table.ctypes.data, rirs.ctypes.data, len(rirs), out.data_ptr(), out.numel(),
                                       work.data_ptr(), work.numel(), stream)
    if rc != 0:
        _raise(lib, rc, handle)


def specaug(x: torch.Tensor, out: torch.Tensor, warps: np.ndarray, masks: np.ndarray, handle=None) -> None:
    """Launches `b200feat_specaug` on the current stream of `out`'s device (asynchronous, no synchronisation): `x` and `out`
    are contiguous float32 (B, T, F) device tensors that share no memory, `warps` / `masks` the host tables
    (SPECAUG_WARP_DTYPE / SPECAUG_MASK_DTYPE; copied before this returns).  Raises B200FeatError when the library refuses
    the tables."""
    lib = load_library()
    stream = torch.cuda.current_stream(out.device).cuda_stream
    assert warps.dtype == SPECAUG_WARP_DTYPE and masks.dtype == SPECAUG_MASK_DTYPE
    assert x.dtype == torch.float32 and out.dtype == torch.float32 and x.dim() == 3 and x.shape == out.shape
    assert x.is_contiguous() and out.is_contiguous() and x.device == out.device
    warps, masks = np.ascontiguousarray(warps), np.ascontiguousarray(masks)
    B, T, F = x.shape
    nbytes = int(lib.b200feat_specaug_work_bytes(B, T, F, len(warps), len(masks)))
    work = torch.empty(max(nbytes, 1), dtype=torch.uint8, device=out.device)
    with torch.cuda.device(out.device):
        rc = lib.b200feat_specaug(handle, x.data_ptr(), out.data_ptr(), B, T, F, warps.ctypes.data, len(warps),
                                  masks.ctypes.data, len(masks), work.data_ptr(), work.numel(), stream)
    if rc != 0:
        _raise(lib, rc, handle)


def feature_mix(src: Optional[torch.Tensor], tracks: np.ndarray, cuts: np.ndarray, out: torch.Tensor, pad_value: float,
                handle=None) -> None:
    """Launches `b200feat_feature_mix` on the current stream of `out`'s device (asynchronous, no synchronisation): the float32
    device rows `src` (None = empty), the host track / cut tables (FEATMIX_TRACK_DTYPE / FEATMIX_CUT_DTYPE; copied before this
    returns) and the contiguous float32 (B, T_max, F) output, B = len(cuts).  Raises B200FeatError when the library refuses
    the tables."""
    lib = load_library()
    stream = torch.cuda.current_stream(out.device).cuda_stream
    assert tracks.dtype == FEATMIX_TRACK_DTYPE and cuts.dtype == FEATMIX_CUT_DTYPE
    assert out.dtype == torch.float32 and out.dim() == 3 and out.is_contiguous() and out.shape[0] == len(cuts)
    assert src is None or (src.dtype == torch.float32 and src.is_contiguous() and src.device == out.device)
    tracks, cuts = np.ascontiguousarray(tracks), np.ascontiguousarray(cuts)
    _, T, F = out.shape
    work = torch.empty(max(int(lib.b200feat_feature_mix_work_bytes(len(tracks), len(cuts))), 1), dtype=torch.uint8,
                       device=out.device)
    p, n = (None, 0) if src is None or src.numel() == 0 else (src.data_ptr(), src.numel())
    with torch.cuda.device(out.device):
        rc = lib.b200feat_feature_mix(handle, p, n, tracks.ctypes.data, len(tracks), cuts.ctypes.data, len(cuts), F,
                                      out.data_ptr(), T, float(pad_value), work.data_ptr(), work.numel(), stream)
    if rc != 0:
        _raise(lib, rc, handle)


def collate_audio(src: Optional[torch.Tensor], offsets: Sequence[int], lens: Sequence[int], out: torch.Tensor,
                  handle=None) -> None:
    """Launches `b200feat_collate_audio` on the current stream of `out`'s device (asynchronous, no synchronisation): row b of
    the contiguous float32 (B, T) output `out` is cut b's `lens[b]` samples from element `offsets[b]` of the 1-D int16 or
    float32 device buffer `src` (None = empty; int16 widened as q / 32768), then zeros.  Raises B200FeatError when the library
    refuses the tables."""
    lib = load_library()
    assert out.dtype == torch.float32 and out.dim() == 2 and out.is_contiguous() and out.shape[0] == len(lens) == len(offsets)
    assert src is None or (src.dim() == 1 and src.is_contiguous() and src.device == out.device)
    dt = DT_F32 if src is None else {torch.float32: DT_F32, torch.int16: DT_I16}[src.dtype]
    off = np.ascontiguousarray(offsets, dtype=np.int64)
    ln = np.ascontiguousarray(lens, dtype=np.int64)
    B, T = out.shape
    stream = torch.cuda.current_stream(out.device).cuda_stream
    work = torch.empty(max(int(lib.b200feat_collate_audio_work_bytes(B)), 1), dtype=torch.uint8, device=out.device)
    p, n = (None, 0) if src is None or src.numel() == 0 else (src.data_ptr(), src.numel())
    with torch.cuda.device(out.device):
        rc = lib.b200feat_collate_audio(handle, p, dt, n, off.ctypes.data, ln.ctypes.data, B, T, out.data_ptr(), work.data_ptr(),
                                        work.numel(), stream)
    if rc != 0:
        _raise(lib, rc, handle)


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

    def _check_cuts(self, rc: int):
        """`_check` for the calls that frame the caller's cuts: B200FEAT_ESHORT (-5, a cut too short to frame) is an input
        error and raises ValueError, as the reference does."""
        if rc == -5:
            raise ValueError(self.lib.b200feat_last_error(self._h).decode())
        self._check(rc)

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
        if words < 0:
            self._check_cuts(words)
        meta = np.empty(words, dtype=np.int64)
        tot = BatchTotals()
        self._check_cuts(self.lib.b200feat_plan_batch(self._h, _ptr(ns), _ptr(off), B, align, out_mode, _ptr(meta), words,
                                                      C.byref(tot)))
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

    def backward_device(self, samples: torch.Tensor, num_samples: Sequence[int], offsets: Sequence[int],
                        grad_out: torch.Tensor, row_prefix: Sequence[int]) -> torch.Tensor:
        """Gradient with respect to `samples` (1-D float32 CUDA tensor, cut i at offsets[i] with num_samples[i] samples) of a
        loss whose gradient with respect to the packed (sum T_i, F) features `extract_device` gave for them is `grad_out`
        (`row_prefix`: that call's row prefix).  Returns a float32 tensor shaped like `samples`: zero outside the cuts."""
        assert samples.is_cuda and samples.dim() == 1 and samples.is_contiguous() and samples.dtype == torch.float32
        B = len(num_samples)
        ns = np.ascontiguousarray(num_samples, dtype=np.int64)
        off = np.ascontiguousarray(offsets, dtype=np.int64)
        rows = np.ascontiguousarray(row_prefix, dtype=np.int64)
        g = grad_out.to(device=samples.device, dtype=torch.float32).contiguous()
        assert g.shape == (int(rows[-1]), self.feature_dim), (tuple(g.shape), int(rows[-1]), self.feature_dim)
        nbytes = int(self.lib.b200feat_backward_work_bytes(self._h, _ptr(ns), B))
        if nbytes < 0:
            self._check_cuts(nbytes)
        work = torch.empty(max(nbytes, 1), dtype=torch.uint8, device=samples.device)
        grad_in = torch.zeros_like(samples)
        stream = torch.cuda.current_stream(samples.device).cuda_stream
        self._check_cuts(self.lib.b200feat_backward(self._h, samples.data_ptr(), DT_F32, _ptr(ns), _ptr(off), B, g.data_ptr(),
                                                    _ptr(rows), grad_in.data_ptr(), work.data_ptr(), work.numel(), stream))
        return grad_in

    def extract_device_keep_raw(self, samples: torch.Tensor, num_samples: Sequence[int], offsets: Sequence[int]
                                ) -> Tuple[torch.Tensor, torch.Tensor, np.ndarray]:
        """`extract_device` (packed) for a whisper-fbank engine that also keeps what `whisper_backward_device` needs:
        (features (sum R_i, F), raw, row prefix), `raw` a flat float32 tensor holding the forward's (sum R_i, F) log-mel rows
        before the clamp and normalisation, then the B per-cut maxima.  The features are bitwise those of `extract_device`."""
        assert samples.is_cuda and samples.dim() == 1 and samples.is_contiguous()
        if samples.data_ptr() % 16:
            samples = samples.clone()
        dt = {torch.float32: DT_F32, torch.int16: DT_I16}[samples.dtype]
        B = len(num_samples)
        meta, totals = self.plan_batch(num_samples, offsets)
        assert totals.span_samples <= samples.numel(), "sample buffer shorter than offsets + lengths"
        meta_dev = torch.from_numpy(meta).to(samples.device, non_blocking=False)
        rows = int(totals.total_rows)
        out = torch.empty((rows, self.feature_dim), dtype=torch.float32, device=samples.device)
        raw = torch.empty(int(totals.out_floats), dtype=torch.float32, device=samples.device)
        stream = torch.cuda.current_stream(samples.device).cuda_stream
        self._check(self.lib.b200feat_extract_keep_raw(self._h, samples.data_ptr(), dt, meta_dev.data_ptr(), B, C.byref(totals),
                                                       out.data_ptr(), raw.data_ptr(), stream))
        return out, raw, meta[2 * B: 3 * B + 1]

    def whisper_backward_device(self, samples: torch.Tensor, num_samples: Sequence[int], offsets: Sequence[int],
                                grad_out: torch.Tensor, raw: torch.Tensor, row_prefix: Sequence[int]) -> torch.Tensor:
        """`backward_device` for a whisper-fbank engine: `raw` is the tensor `extract_device_keep_raw` returned for the same
        samples, whose features the loss's gradient `grad_out` ((sum R_i, F)) is taken with respect to."""
        assert samples.is_cuda and samples.dim() == 1 and samples.is_contiguous() and samples.dtype == torch.float32
        B = len(num_samples)
        ns = np.ascontiguousarray(num_samples, dtype=np.int64)
        off = np.ascontiguousarray(offsets, dtype=np.int64)
        rows = np.ascontiguousarray(row_prefix, dtype=np.int64)
        R = int(rows[-1])
        g = grad_out.to(device=samples.device, dtype=torch.float32).contiguous()
        assert g.shape == (R, self.feature_dim), (tuple(g.shape), R, self.feature_dim)
        assert raw.is_cuda and raw.dtype == torch.float32 and raw.numel() == R * self.feature_dim + B
        nbytes = int(self.lib.b200feat_backward_work_bytes(self._h, _ptr(ns), B))
        if nbytes < 0:
            self._check_cuts(nbytes)
        work = torch.empty(max(nbytes, 1), dtype=torch.uint8, device=samples.device)
        grad_in = torch.zeros_like(samples)
        stream = torch.cuda.current_stream(samples.device).cuda_stream
        self._check_cuts(self.lib.b200feat_whisper_backward(
            self._h, samples.data_ptr(), DT_F32, _ptr(ns), _ptr(off), B, g.data_ptr(), raw.data_ptr(),
            raw.data_ptr() + 4 * R * self.feature_dim, _ptr(rows), grad_in.data_ptr(), work.data_ptr(), work.numel(), stream))
        return grad_in

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
        Ts = self.plan.num_frames(ns)
        tmax = int(Ts.max())
        rows = B * tmax if out_mode == OUT_PADDED else int(Ts.sum())
        shape = (B, tmax, self.feature_dim) if out_mode == OUT_PADDED else (rows, self.feature_dim)
        if out is None:
            # pinned (page-locked) result: the D2H copies run asynchronously at full PCIe speed; torch's caching
            # host allocator makes repeated allocations of the same size cheap
            out = torch.empty(shape, dtype=torch.float32, pin_memory=True).numpy()
        optr = out.data_ptr() if isinstance(out, torch.Tensor) else out.ctypes.data
        self._check_cuts(self.lib.b200feat_extract_host_at(self._h, sptr, dt, _ptr(ns), _ptr(off), B, optr, out_mode,
                                                           float(pad_value)))
        return out, np.concatenate(([0], np.cumsum(Ts))).astype(np.int64)

    def extract_host_list(self, arrays: Sequence[np.ndarray], dtype=np.float32):
        """A LIST of separately allocated host waveforms -> packed (sum T_i, F) features in pinned host memory + row prefix.
        One C call (`b200feat_extract_host_ptrs`): the library gathers the cuts into its pinned staging slots with its own
        thread pool (non-temporal stores) and overlaps that with the H2D / kernel / D2H pipeline; the GIL is released
        throughout."""
        want = np.dtype(dtype)
        arrs = [np.ascontiguousarray(a, dtype=want).reshape(-1) for a in arrays]
        B = len(arrs)
        ns = np.asarray([a.shape[0] for a in arrs], dtype=np.int64)
        prefix = np.concatenate(([0], np.cumsum(self.plan.num_frames(ns)))).astype(np.int64)
        out = torch.empty((int(prefix[-1]), self.feature_dim), dtype=torch.float32, pin_memory=torch.cuda.is_available()).numpy()
        ptrs = (C.c_void_p * B)(*[a.ctypes.data for a in arrs])
        self._check_cuts(self.lib.b200feat_extract_host_ptrs(self._h, ptrs, DT_I16 if want == np.int16 else DT_F32, _ptr(ns), B,
                                                             out.ctypes.data, OUT_PACKED, 0.0))
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


def _groups(lens: Sequence[int], target_bytes: int, esz: int) -> List[Tuple[int, int]]:
    """Consecutive index ranges [b0, b1) of roughly `target_bytes` each."""
    out, b0, acc = [], 0, 0
    for i, n in enumerate(lens):
        acc += n * esz
        if acc >= target_bytes:
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


def _zero_gaps(view: np.ndarray, lens: Sequence[int], offs: Sequence[int], b0: int = 0, b1: Optional[int] = None) -> None:
    """Zero-fills the alignment gap in front of each cut b0 <= i < b1: defined bytes only cross PCIe."""
    for i in range(max(b0, 1), len(lens) if b1 is None else b1):
        view[offs[i - 1] + lens[i - 1]: offs[i]] = 0


def _gather(view: np.ndarray, arrays: Sequence[np.ndarray], lens: List[int], offs: List[int],
            split: int) -> List[Tuple[Tuple[int, int], Future]]:
    """Copies arrays[i] to view[offs[i]: offs[i] + lens[i]] and zero-fills the gaps.  Below 8 MB (or with one staging
    thread) the calling thread does it all and this returns [].  Above, the staging pool copies groups of consecutive cuts,
    each about 1 / (split * STAGING_THREADS) of the batch, and this returns [((b0, b1), future)] in batch order."""
    def copy(b0, b1):
        _zero_gaps(view, lens, offs, b0, b1)
        for i in range(b0, b1):
            view[offs[i]: offs[i] + lens[i]] = arrays[i]

    pool, esz = _copy_pool(), view.itemsize
    total = offs[-1] + lens[-1] if lens else 0
    if pool is None or total * esz < (8 << 20):
        copy(0, len(lens))
        return []
    return [(g, pool.submit(copy, *g)) for g in _groups(lens, max(4 << 20, total * esz // (split * STAGING_THREADS)), esz)]


def pack_device(tensors: List[torch.Tensor], device: torch.device, align: int = 4,
                dtype: torch.dtype = torch.float32) -> Tuple[torch.Tensor, List[int], List[int]]:
    """Packs 1-D waveforms into one ragged device buffer (each start aligned to `align` elements).
    Host tensors are gathered into ONE pinned staging buffer by the staging threads, group by group, and every finished
    group is sent to the device at once (its H2D copy overlaps the gathering of the next group); device tensors are
    copied device-to-device."""
    lens = [int(t.numel()) for t in tensors]
    offs, total = _aligned_offsets(lens, align)
    if any(t.is_cuda for t in tensors):
        buf = torch.empty(total, dtype=dtype, device=device)
        for t, o, n in zip(tensors, offs, lens):
            buf[o:o + n].copy_(t.reshape(-1), non_blocking=True)
        return buf, lens, offs
    stage = torch.empty(total, dtype=dtype, pin_memory=torch.cuda.is_available())
    # numpy views of the tensors: a plain memcpy (3x torch's CPU copy_ on this path) that releases the GIL
    groups = _gather(stage.numpy(), [t.detach().numpy().reshape(-1) for t in tensors], lens, offs, split=4)
    if not groups:
        return stage.to(device, non_blocking=True), lens, offs
    dev = torch.empty(total, dtype=dtype, device=device)
    for (b0, b1), f in groups:
        f.result()
        e0, e1 = offs[b0], offs[b1 - 1] + lens[b1 - 1]
        dev[e0:e1].copy_(stage[e0:e1], non_blocking=True)
    return dev, lens, offs


def stage_host(arrays: Sequence[np.ndarray], dtype=np.float32, align: int = 4) -> Tuple[torch.Tensor, List[int], List[int]]:
    """Copies 1-D host waveforms into ONE pinned buffer, each start aligned to `align` elements (gaps zero-filled), using
    the staging threads.  Returns (buffer, lengths, offsets) for `Engine.extract_host(offsets=)`."""
    lens = [int(a.shape[0]) for a in arrays]
    offs, total = _aligned_offsets(lens, align)
    stage = torch.empty(max(total, 1), dtype=torch.int16 if np.dtype(dtype) == np.int16 else torch.float32,
                        pin_memory=torch.cuda.is_available())
    for _, f in _gather(stage.numpy(), arrays, lens, offs, split=2):
        f.result()
    return stage, lens, offs
