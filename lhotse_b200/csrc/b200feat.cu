// b200feat — host side of the C ABI (include/b200feat.h) + kernel dispatch.  sm_90a only.
#include <cuda_runtime.h>
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <immintrin.h>

#include <algorithm>
#include <atomic>
#include <condition_variable>
#include <functional>
#include <map>
#include <mutex>
#include <string>
#include <thread>
#include <vector>

#include "common.cuh"
#include "generic.cuh"
#include "fast512.cuh"
#include "tc512.cuh"
#include "fast256.cuh"
#include "fast2048.cuh"
#include "fast1024.cuh"
#include "fast400.cuh"
#include "flac.cuh"
#include "mix.cuh"
#include "resample.cuh"
#include "reverb.cuh"
#include "specaug.cuh"
#include "rirgen.cuh"
#include "featmix.cuh"
#include "backward.cuh"
#include "collate.cuh"
#include "wpe.cuh"

#include <cub/device/device_segmented_radix_sort.cuh>

namespace {

thread_local std::string g_error;

struct HostRing {  // grow-only staging for b200feat_extract_host
  void *d_samples = nullptr; size_t d_samples_cap = 0;
  float *d_out = nullptr; size_t d_out_cap = 0;
  int64_t *d_meta = nullptr; size_t d_meta_cap = 0;  // bytes
  int64_t *h_meta = nullptr; size_t h_meta_cap = 0;  // pinned
  cudaStream_t streams[3] = {nullptr, nullptr, nullptr};
  cudaEvent_t meta_ready = nullptr;
  // b200feat_extract_host_ptrs: two pinned staging slots the gather threads fill while the previous slot is on its way over PCIe
  void *h_stage[2] = {nullptr, nullptr}; size_t h_stage_cap[2] = {0, 0};
  cudaEvent_t stage_free[2] = {nullptr, nullptr};
  std::mutex mu;
};

// A small persistent pool for the host-side gather (memcpy-class work: it only has to keep a few memory channels busy).
class GatherPool {
 public:
  explicit GatherPool(int n) : stop_(false), pending_(0) {
    for (int i = 0; i < n; ++i) workers_.emplace_back([this] { loop(); });
  }
  ~GatherPool() {
    { std::lock_guard<std::mutex> g(mu_); stop_ = true; }
    cv_.notify_all();
    for (auto &t : workers_) t.join();
  }
  int size() const { return (int)workers_.size(); }
  // runs fn(i) for i in [0, n) on the pool and the calling thread; returns when all are done
  void parallel_for(int n, const std::function<void(int)> &fn) {
    if (n <= 0) return;
    {
      std::lock_guard<std::mutex> g(mu_);
      fn_ = &fn; next_ = 0; total_ = n; pending_ = n;
    }
    cv_.notify_all();
    run_some();
    std::unique_lock<std::mutex> g(mu_);
    done_.wait(g, [this] { return pending_ == 0; });
    fn_ = nullptr;
  }

 private:
  void run_some() {
    for (;;) {
      int i;
      const std::function<void(int)> *fn;
      {
        std::lock_guard<std::mutex> g(mu_);
        if (!fn_ || next_ >= total_) return;
        i = next_++; fn = fn_;
      }
      (*fn)(i);
      std::lock_guard<std::mutex> g(mu_);
      if (--pending_ == 0) done_.notify_all();
    }
  }
  void loop() {
    for (;;) {
      {
        std::unique_lock<std::mutex> g(mu_);
        cv_.wait(g, [this] { return stop_ || (fn_ && next_ < total_); });
        if (stop_) return;
      }
      run_some();
    }
  }
  std::vector<std::thread> workers_;
  std::mutex mu_;
  std::condition_variable cv_, done_;
  const std::function<void(int)> *fn_ = nullptr;
  int next_ = 0, total_ = 0;
  bool stop_;
  int pending_;
};

// memcpy with non-temporal stores: the destination (pinned staging) is read next by the DMA engine, not by this core, so
// bypassing the cache saves the read-for-ownership of every destination line (a third of the gather's memory traffic)
static void stream_copy(void *dst, const void *src, size_t bytes) {
  unsigned char *d = static_cast<unsigned char *>(dst);
  const unsigned char *s = static_cast<const unsigned char *>(src);
  const size_t head = std::min(bytes, (size_t)((32 - ((uintptr_t)d & 31)) & 31));
  if (head) { memcpy(d, s, head); d += head; s += head; bytes -= head; }
  const size_t blocks = bytes / 128;
  for (size_t i = 0; i < blocks; ++i) {
    const __m256i a = _mm256_loadu_si256(reinterpret_cast<const __m256i *>(s)), b = _mm256_loadu_si256(reinterpret_cast<const __m256i *>(s + 32));
    const __m256i c = _mm256_loadu_si256(reinterpret_cast<const __m256i *>(s + 64)), e = _mm256_loadu_si256(reinterpret_cast<const __m256i *>(s + 96));
    _mm256_stream_si256(reinterpret_cast<__m256i *>(d), a); _mm256_stream_si256(reinterpret_cast<__m256i *>(d + 32), b);
    _mm256_stream_si256(reinterpret_cast<__m256i *>(d + 64), c); _mm256_stream_si256(reinterpret_cast<__m256i *>(d + 96), e);
    s += 128; d += 128;
  }
  bytes -= blocks * 128;
  if (bytes) memcpy(d, s, bytes);
  _mm_sfence();
}

// Makes `device` current for the guard's lifetime and then restores the caller's current device.
class DeviceGuard {
 public:
  explicit DeviceGuard(int device) : device_(device) {
    cudaGetDevice(&prev_);
    if (prev_ != device_) cudaSetDevice(device_);
  }
  ~DeviceGuard() {
    if (prev_ != device_) cudaSetDevice(prev_);
  }

 private:
  int device_, prev_ = 0;
};

// grow-only staging buffer (device or pinned host): reallocated with 25 % headroom when `need` bytes do not fit
cudaError_t grow(void **p, size_t *cap, size_t need, bool pinned) {
  if (*cap >= need) return cudaSuccess;
  if (*p) { if (pinned) cudaFreeHost(*p); else cudaFree(*p); }
  *p = nullptr; *cap = 0;
  const size_t want = need + need / 4;
  cudaError_t e = pinned ? cudaMallocHost(p, want) : cudaMalloc(p, want);
  if (e == cudaSuccess) *cap = want;
  return e;
}

}  // namespace

struct b200feat_handle {
  b200feat_plan_desc desc;
  DevPlan plan;
  int device = 0;
  int kernel = B200FEAT_KERNEL_GENERIC;
  int sm_count = 132;
  int frames_per_tile = 1;
  int generic_warps = 4;
  size_t generic_smem = 0;
  std::vector<void *> allocs;
  std::vector<float> h_window, h_bank, h_dct, h_lifter;
  std::vector<float2> h_tw;
  mutable std::string error;
  b200feat_stats stats{};
  std::mutex stats_mu;
  HostRing ring;
  Fast512Host fast;
  Tc512Host tc;
  float *d_affine = nullptr;  // [2][F] output affine (b200feat_set_output_affine)
  GatherPool *pool = nullptr;  // created on the first b200feat_extract_host_ptrs
  Fast256Host fast256;
  Fast1024Host fast1024;
  Fast2048Host fast2048;
  Fast400Host fast400;
};

namespace {

int fail(b200feat_handle *h, int code, const std::string &msg) {
  if (h) h->error = msg;
  g_error = msg;
  return code;
}

#define CU_TRY(h, expr)                                                                      \
  do {                                                                                       \
    cudaError_t _e = (expr);                                                                 \
    if (_e != cudaSuccess)                                                                   \
      return fail(h, B200FEAT_ECUDA, std::string(#expr) + ": " + cudaGetErrorString(_e));    \
  } while (0)

template <typename T>
int upload(b200feat_handle *h, const T *src, size_t count, const T **dst) {
  CU_TRY(h, upload_table(src, count, h->allocs, dst));
  return 0;
}

std::vector<int> factorize(int n) {
  std::vector<int> f;
  // radix 4 / 2 passes.  (A register radix-16 pass — a quarter of the shared-memory round trips — did not pay: at one warp
  // per frame and 8 warps per SM the generic kernel is bound by its instruction count and occupancy, not by the passes.)
  while (n % 4 == 0) { f.push_back(4); n /= 4; }
  while (n % 2 == 0) { f.push_back(2); n /= 2; }
  for (int p = 3; n > 1; p += 2)
    while (n % p == 0) { f.push_back(p); n /= p; }
  return f;
}

// Output rows of a cut.  For whisper-fbank this is compute_num_frames_from_samples (whisper_fbank.py:73-80, utils.py:424):
// the stft itself yields n / S frames (1 + n / S, last one dropped, :62-63); a missing last row is a zero row.
int64_t frames_for(const b200feat_plan_desc &d, int64_t n) {
  const int64_t L = d.frame_length, S = d.frame_shift;
  if (d.feature == B200FEAT_WHISPER_FBANK) return (n + S / 2) / S;
  if (d.feature == B200FEAT_LOG10_FBANK && d.pad_mode == B200FEAT_PAD_CENTER) return (n + S / 2) / S;  // librosa_fbank.py:128-134
  if (d.snip_edges) return n < L ? 0 : 1 + (n - L) / S;
  return (n + S / 2) / S;
}

// The reference can frame a cut only if one reflection per side suffices (layers.py:757-764).
bool framable(const b200feat_plan_desc &d, int64_t n, int64_t T) {
  if (T <= 0) return false;
  if (d.pad_mode == B200FEAT_PAD_CENTER) return n > d.fft_length / 2;  // torch's reflect padding needs pad < n
  if (d.snip_edges) return true;
  const int64_t L = d.frame_length, S = d.frame_shift;
  const int64_t left = (L - S) / 2;
  const int64_t right = (T - 1) * S + L - n - left;
  return left <= n && right <= n;
}

// Frames of cut i of n samples, or B200FEAT_ESHORT (naming the cut) if it is too short to be framed.
int64_t cut_frames(b200feat_handle *h, int i, int64_t n) {
  const int64_t T = frames_for(h->desc, n);
  if (!framable(h->desc, n, T))
    return fail(h, B200FEAT_ESHORT, "cut " + std::to_string(i) + " with " + std::to_string(n) + " samples is too short to be framed");
  return T;
}

// Everything of b200feat_create after its argument and device checks: derived plan, device tables, kernel choice.  On
// failure the caller destroys the half-built handle.
int setup_handle(b200feat_handle *h, const float *window, const float *mel_bank, const float *dct, const float *lifter) {
  const b200feat_plan_desc *desc = &h->desc;
  const int L = desc->frame_length, S = desc->frame_shift, N = desc->fft_length;
  const bool whisper = desc->feature == B200FEAT_WHISPER_FBANK;
  const bool log10fb = desc->feature == B200FEAT_LOG10_FBANK;
  const bool mel = desc->feature == B200FEAT_FBANK || desc->feature == B200FEAT_MFCC || whisper || log10fb;
  DevPlan &p = h->plan;
  memset(&p, 0, sizeof(p));
  p.feature = desc->feature; p.L = L; p.S = S; p.N = N; p.K = N / 2 + 1;
  p.M = mel ? desc->num_filters : 0;
  p.C = desc->feature == B200FEAT_MFCC ? desc->num_ceps : 0;
  p.packed = (N % 2 == 0);
  p.Nc = p.packed ? N / 2 : N;
  p.pad_mode = desc->pad_mode;
  p.whisper = whisper ? 1 : 0;
  p.log10_mel = (whisper || log10fb) ? 1 : 0;
  p.pad_left = desc->pad_mode == B200FEAT_PAD_CENTER ? N / 2 : (L - S) / 2;
  p.snip_edges = desc->snip_edges; p.remove_dc = desc->remove_dc_offset;
  p.use_energy = desc->use_energy != 0; p.raw_energy = desc->raw_energy; p.use_mag = desc->use_fft_mag;
  p.energy_last = desc->use_energy == 2 && (desc->feature == B200FEAT_FBANK || desc->feature == B200FEAT_MFCC);
  p.energy_style = desc->energy_style; p.use_lifter = desc->use_lifter;
  p.preemph = desc->preemph_coeff;
  const bool has_floor = desc->energy_style == B200FEAT_ENERGY_KALDI ? desc->energy_floor != 0.f
                                                                      : desc->energy_floor > 0.f;
  p.has_energy_floor = has_floor ? 1.f : 0.f;
  p.energy_floor_log = has_floor ? (float)log((double)desc->energy_floor) : 0.f;
  p.mel_floor = desc->mel_floor;
  p.log_spec_eps = desc->log_spec_eps < 0.f ? 0.f : desc->log_spec_eps;
  p.log_spec_floor = desc->log_spec_eps < 0.f ? -desc->log_spec_eps : 0.f;
  switch (desc->feature) {
    case B200FEAT_FBANK: p.F = p.M + (desc->use_energy ? 1 : 0); break;
    case B200FEAT_WHISPER_FBANK: p.F = p.M; break;
    case B200FEAT_LOG10_FBANK: p.F = p.M; break;
    case B200FEAT_MFCC: p.F = p.C; break;
    default: p.F = p.K;
  }
  std::vector<int> fac = factorize(p.Nc);
  if ((int)fac.size() > B200_MAX_STAGES) return fail(nullptr, B200FEAT_EUNSUPPORTED, "too many FFT stages");
  p.nstages = (int)fac.size();
  for (int i = 0; i < p.nstages; ++i) p.radix[i] = fac[i];

  // host copies kept for get_table and for the fast kernel's derived tables
  h->h_window.assign(window, window + L);
  if (mel) h->h_bank.assign(mel_bank, mel_bank + (size_t)p.K * p.M);
  if (p.C) h->h_dct.assign(dct, dct + (size_t)p.M * p.C);
  if (desc->use_lifter) h->h_lifter.assign(lifter, lifter + p.C);

  int rc = 0;
#define UP(expr) do { if ((rc = (expr))) return rc; } while (0)
  UP(upload(h, h->h_window.data(), (size_t)L, &p.window));
  // twiddles in double, rounded once
  h->h_tw.resize(p.Nc);
  for (int k = 0; k < p.Nc; ++k) {
    const double a = -2.0 * M_PI * (double)k / (double)p.Nc;
    h->h_tw[k] = make_float2((float)cos(a), (float)sin(a));
  }
  UP(upload(h, h->h_tw.data(), (size_t)p.Nc, &p.tw));
  if (p.packed) {
    std::vector<float2> tws(p.K);
    for (int k = 0; k < p.K; ++k) {
      const double a = -2.0 * M_PI * (double)k / (double)N;
      tws[k] = make_float2((float)cos(a), (float)sin(a));
    }
    UP(upload(h, tws.data(), tws.size(), &p.tws));
  }
  std::vector<int> mstart, mlen, mwoff;
  std::vector<float> mw;
  if (mel) {  // sparse form: contiguous support [first, last] of each filter column
    mstart.resize(p.M); mlen.resize(p.M); mwoff.resize(p.M);
    for (int m = 0; m < p.M; ++m) {
      int first, last;
      const bool any = filter_support(mel_bank, p.K, p.M, m, &first, &last);
      mstart[m] = any ? first : 0;
      mlen[m] = any ? last - first + 1 : 0;
      mwoff[m] = (int)mw.size();
      for (int k = 0; k < mlen[m]; ++k) mw.push_back(mel_bank[(size_t)(mstart[m] + k) * p.M + m]);
    }
    if (mw.empty()) mw.push_back(0.f);
    UP(upload(h, mstart.data(), mstart.size(), &p.mel_start));
    UP(upload(h, mlen.data(), mlen.size(), &p.mel_len));
    UP(upload(h, mwoff.data(), mwoff.size(), &p.mel_woff));
    UP(upload(h, mw.data(), mw.size(), &p.mel_w));
  }
  if (p.C) UP(upload(h, h->h_dct.data(), h->h_dct.size(), &p.dct));
  if (desc->use_lifter) UP(upload(h, h->h_lifter.data(), h->h_lifter.size(), &p.lifter));

  // ---- kernel selection
  // the whisper-fbank epilogue / centre padding exist in the generic and the fast400 kernels only; the tensor-core kernel
  // (tc512.cuh) serves the N = 512 fbank / mfcc plans without an energy column
  const bool tc_ok = !whisper && tc512_supported(p);
  if (desc->kernel == B200FEAT_KERNEL_TC && !tc_ok)
    return fail(nullptr, B200FEAT_EUNSUPPORTED, "the tensor-core kernel needs fft_length 512, fbank / mfcc without use_energy, Kaldi framing");
  const bool fast512_ok = !whisper && fast512_supported(p);
  const bool fast256_ok = !whisper && fast256_supported(p);
  const bool fast1024_ok = !whisper && fast1024_supported(p);
  const bool fast400_ok = fast400_supported(p);
  const bool fast2048_ok = !whisper && fast2048_supported(p);
  const bool fast_ok = fast512_ok || fast256_ok || fast1024_ok || fast2048_ok || fast400_ok;
  if (desc->kernel == B200FEAT_KERNEL_FAST && !fast_ok)
    return fail(nullptr, B200FEAT_EUNSUPPORTED, "fast kernels require fft_length 256, 512, 1024, 2048 or frame_length = fft_length = 400");
  bool auto_tc = false;  // AUTO prefers the tensor-core kernel where it is the faster one (B200FEAT_AUTO_TC=0/1 overrides)
  if (const char *e = getenv("B200FEAT_AUTO_TC")) auto_tc = atoi(e) != 0;
  if (desc->kernel == B200FEAT_KERNEL_TC || (desc->kernel == B200FEAT_KERNEL_AUTO && tc_ok && auto_tc)) h->kernel = B200FEAT_KERNEL_TC;
  else if (desc->kernel == B200FEAT_KERNEL_GENERIC || !fast_ok) h->kernel = B200FEAT_KERNEL_GENERIC;
  else h->kernel = B200FEAT_KERNEL_FAST;

  {  // generic launch shape (generic.cuh)
    if (!generic_launch_shape(p, &h->generic_warps, &h->generic_smem))
      return fail(nullptr, B200FEAT_EUNSUPPORTED, "fft_length too large for shared memory");
    if (h->generic_smem > 48 * 1024) {
      cudaError_t e1 = cudaFuncSetAttribute(b200feat_generic_kernel<B200FEAT_F32>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)h->generic_smem);
      cudaError_t e2 = cudaFuncSetAttribute(b200feat_generic_kernel<B200FEAT_I16>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)h->generic_smem);
      if (e1 != cudaSuccess || e2 != cudaSuccess)
        return fail(nullptr, B200FEAT_ECUDA, "cudaFuncSetAttribute(generic smem) failed");
    }
  }
  h->frames_per_tile = 1;
  if (h->kernel == B200FEAT_KERNEL_TC) {
    rc = tc512_prepare(h->plan, h->h_bank, h->allocs, &h->frames_per_tile, h->h_window, &h->tc);
    if (rc == B200FEAT_EUNSUPPORTED && desc->kernel == B200FEAT_KERNEL_AUTO) {
      h->kernel = fast_ok ? B200FEAT_KERNEL_FAST : B200FEAT_KERNEL_GENERIC;
      h->frames_per_tile = 1;
      rc = 0;
    } else if (rc)
      return fail(nullptr, rc, "tensor-core kernel cannot be prepared for this plan");
  }
  if (h->kernel == B200FEAT_KERNEL_FAST) {
    if (h->plan.N == 256) rc = fast256_prepare(h->plan, h->h_bank, h->allocs, &h->frames_per_tile, h->h_window, &h->fast256);
    else if (h->plan.N == 400) rc = fast400_prepare(h->plan, h->h_bank, h->allocs, &h->frames_per_tile, h->h_window, &h->fast400);
    else if (h->plan.N == 1024) rc = fast1024_prepare(h->plan, h->h_bank, h->allocs, &h->frames_per_tile, h->h_window, &h->fast1024);
    else if (h->plan.N == 2048) rc = fast2048_prepare(h->plan, h->h_bank, h->allocs, &h->frames_per_tile, h->h_window, &h->fast2048);
    else rc = fast512_prepare(h->plan, h->h_bank, h->allocs, &h->frames_per_tile, h->h_window, &h->fast);
    if (rc == B200FEAT_EUNSUPPORTED && desc->kernel == B200FEAT_KERNEL_AUTO) {
      h->kernel = B200FEAT_KERNEL_GENERIC;  // e.g. the plan's tables do not fit the fast kernel's shared memory
      h->frames_per_tile = 1;
    } else if (rc)
      return fail(nullptr, rc, "fast kernel cannot be prepared for this plan (shared-memory footprint?)");
  }
#undef UP
  return 0;
}

// launches the selected kernel over cuts [b0, b1) of a planned batch
int launch_range(b200feat_handle *h, const void *samples_dev, int32_t dt, const int64_t *meta_dev,
                        int32_t B, int32_t b0, int32_t b1, int64_t tile0, int64_t tile1,
                        int64_t max_frames, float *out_dev, int32_t out_mode, float pad_value,
                        cudaStream_t stream, float *cut_max_dev = nullptr, int64_t norm_rows = 0,
                        float *norm_out = nullptr) {
  DevBatch db;
  db.samples = samples_dev;
  db.samp_off = meta_dev + b0;
  db.nsamp = meta_dev + B + b0;
  db.row_off = meta_dev + 2 * (int64_t)B + b0;
  db.tile_off = meta_dev + 3 * (int64_t)B + 1 + b0;
  db.tile_cut = h->frames_per_tile > 1 ? reinterpret_cast<const int32_t *>(meta_dev + 4 * (int64_t)B + 2) : nullptr;
  db.out = out_dev;
  db.cut_max = cut_max_dev ? cut_max_dev + b0 : nullptr;
  db.tile_base = tile0;
  db.num_tiles = tile1 - tile0;
  db.max_frames = max_frames;
  db.batch_first = b0;
  db.B = b1 - b0;
  db.out_mode = out_mode;
  db.pad_value = pad_value;
  if (db.num_tiles <= 0) return 0;
  if (h->plan.whisper) {
    if (!cut_max_dev) return fail(h, B200FEAT_EINVAL, "whisper-fbank: scratch missing");
    cudaError_t e = cudaMemsetAsync(db.cut_max, 0xff, (size_t)db.B * sizeof(float), stream);  // "empty" (common.cuh)
    if (e != cudaSuccess) return fail(h, B200FEAT_ECUDA, std::string("memset(cut_max): ") + cudaGetErrorString(e));
  }
  if (h->kernel == B200FEAT_KERNEL_TC || h->kernel == B200FEAT_KERNEL_FAST) {
    const char *name;
    int rc;
    if (h->kernel == B200FEAT_KERNEL_TC) { name = "tc512"; rc = tc512_launch(h->plan, h->tc, db, dt, h->sm_count, stream); }
    else if (h->plan.N == 256) { name = "fast256"; rc = fast256_launch(h->plan, h->fast256, db, dt, h->sm_count, stream); }
    else if (h->plan.N == 400) { name = "fast400"; rc = fast400_launch(h->plan, h->fast400, db, dt, h->sm_count, stream); }
    else if (h->plan.N == 1024) { name = "fast1024"; rc = fast1024_launch(h->plan, h->fast1024, db, dt, h->sm_count, stream); }
    else if (h->plan.N == 2048) { name = "fast2048"; rc = fast2048_launch(h->plan, h->fast2048, db, dt, h->sm_count, stream); }
    else { name = "fast512"; rc = fast512_launch(h->plan, h->fast, db, dt, h->sm_count, stream); }
    if (rc) return fail(h, B200FEAT_ECUDA, std::string(name) + " launch: " + cudaGetErrorString((cudaError_t)rc));
  } else {
    const int w = h->generic_warps;
    const unsigned blocks = persistent_grid((db.num_tiles + w - 1) / w, h->sm_count, 8);
    if (dt == B200FEAT_I16)
      b200feat_generic_kernel<B200FEAT_I16><<<blocks, w * 32, h->generic_smem, stream>>>(h->plan, db);
    else
      b200feat_generic_kernel<B200FEAT_F32><<<blocks, w * 32, h->generic_smem, stream>>>(h->plan, db);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return fail(h, B200FEAT_ECUDA, std::string("generic launch: ") + cudaGetErrorString(e));
  }
  if (h->plan.whisper && norm_rows > 0) {  // second launch: clamp to the cut's maximum - 8, (x + 4) / 4, zero rows
    // norm_out: the fused kernel's log-mel rows stay where it wrote them, the normalised rows go to norm_out
    const float *src = out_dev;
    if (norm_out) db.out = norm_out;
    if (h->frames_per_tile > 1) {
      const unsigned blocks = persistent_grid(db.num_tiles, h->sm_count, 8);
      b200feat_whisper_normalize_tiled_kernel<<<blocks, 256, 0, stream>>>(h->plan, db, src, h->frames_per_tile);
    } else {
      const unsigned blocks = persistent_grid((norm_rows + 7) / 8, h->sm_count, 16);
      b200feat_whisper_normalize_kernel<<<blocks, 256, 0, stream>>>(h->plan, db, src, norm_rows);
    }
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return fail(h, B200FEAT_ECUDA, std::string("whisper normalise launch: ") + cudaGetErrorString(e));
  }
  return 0;
}

// Copies cuts [b0, b1) into the pinned slot `stage` at their planned offsets relative to the chunk's first sample, with
// the alignment gaps zeroed: one task per ~1 MB piece so that long and short cuts balance over the pool's threads.
void gather_chunk(GatherPool *pool, unsigned char *stage, const void *const *cuts, const int64_t *soff, const int64_t *num_samples,
                  int b0, int b1, size_t esz) {
  struct Piece { const unsigned char *src; unsigned char *dst; size_t bytes; };
  std::vector<Piece> pieces;
  const int64_t e0 = soff[b0];
  for (int i = b0; i < b1; ++i) {
    const unsigned char *src = static_cast<const unsigned char *>(cuts[i]);
    unsigned char *dst = stage + (size_t)(soff[i] - e0) * esz;
    size_t left = (size_t)num_samples[i] * esz;
    while (left) {
      const size_t take = std::min(left, (size_t)1 << 20);
      pieces.push_back({src, dst, take});
      src += take; dst += take; left -= take;
    }
    if (i + 1 < b1) {  // alignment gap before the next cut: defined bytes only
      const size_t gap = (size_t)(soff[i + 1] - soff[i] - num_samples[i]) * esz;
      if (gap) memset(stage + (size_t)(soff[i] + num_samples[i] - e0) * esz, 0, gap);
    }
  }
  const std::function<void(int)> job = [&](int k) { stream_copy(pieces[k].dst, pieces[k].src, pieces[k].bytes); };
  pool->parallel_for((int)pieces.size(), job);
}

// b200feat_extract_host_at / _ptrs after their argument checks.  The samples come either from one host buffer `src` laid
// out as the batch's offsets say (copied a chunk at a time, verbatim), or from one pointer per cut `cuts` (gathered a chunk
// at a time into one of two pinned slots while the other slot's copy is in flight).
int extract_staged(b200feat_handle *h, const void *src, const void *const *cuts, int32_t dt, const int64_t *num_samples,
                   const int64_t *sample_offsets, int32_t B, float *out_host, int32_t out_mode, float pad_value) {
  HostRing &r = h->ring;
  std::lock_guard<std::mutex> guard(r.mu);
  DeviceGuard on(h->device);

  const size_t esz = dt == B200FEAT_I16 ? 2 : 4;
  // gathered cuts start on a 16-byte boundary of the device buffer; a caller's buffer keeps its own layout on the device
  const int32_t align = cuts ? (dt == B200FEAT_I16 ? 8 : 4) : 1;
  const int64_t words = b200feat_plan_words(h, num_samples, B, out_mode);
  if (words < 0) return (int)words;
  if (r.h_meta_cap < (size_t)words) {
    if (r.h_meta) cudaFreeHost(r.h_meta);
    r.h_meta = nullptr; r.h_meta_cap = 0;
    CU_TRY(h, cudaMallocHost((void **)&r.h_meta, (size_t)words * 8));
    r.h_meta_cap = (size_t)words;
  }
  b200feat_batch_totals tot;
  int rc = b200feat_plan_batch(h, num_samples, sample_offsets, B, align, out_mode, r.h_meta, words, &tot);
  if (rc) return rc;
  for (auto &s : r.streams) if (!s) CU_TRY(h, cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking));
  if (!r.meta_ready) CU_TRY(h, cudaEventCreateWithFlags(&r.meta_ready, cudaEventDisableTiming));
  if (cuts) {
    for (int k = 0; k < 2; ++k)
      if (!r.stage_free[k]) CU_TRY(h, cudaEventCreateWithFlags(&r.stage_free[k], cudaEventDisableTiming));
    if (!h->pool) {
      int nthreads = 8;
      if (const char *e = getenv("B200FEAT_STAGING_THREADS")) nthreads = std::max(1, atoi(e));
      h->pool = new GatherPool(nthreads - 1);  // the calling thread works too
    }
  }
  CU_TRY(h, grow(&r.d_samples, &r.d_samples_cap, (size_t)tot.span_samples * esz + 16, false));
  CU_TRY(h, grow((void **)&r.d_out, &r.d_out_cap, (size_t)tot.out_floats * 4 + 16, false));
  CU_TRY(h, grow((void **)&r.d_meta, &r.d_meta_cap, (size_t)words * 8, false));
  CU_TRY(h, cudaMemcpyAsync(r.d_meta, r.h_meta, (size_t)words * 8, cudaMemcpyHostToDevice, r.streams[0]));
  CU_TRY(h, cudaEventRecord(r.meta_ready, r.streams[0]));

  // chunks of cuts with ~32 MB of samples each, round-robin over 3 streams so that H2D(i+1), kernel(i) and D2H(i-1)
  // overlap (PCIe is the end-to-end bound, SURVEY.md §7)
  const int64_t *soff = r.h_meta, *roff = r.h_meta + 2 * (int64_t)B, *toff = r.h_meta + 3 * (int64_t)B + 1;
  const int64_t chunk_elems = (32ll << 20) / (int64_t)esz;
  std::vector<int> cb{0};  // chunk boundaries
  for (int b0 = 0; b0 < B;) {
    int b1 = b0 + 1;
    while (b1 < B && (soff[b1] + num_samples[b1]) - soff[b0] <= chunk_elems) ++b1;
    cb.push_back(b1);
    b0 = b1;
  }
  const size_t nchunks = cb.size() - 1;
  if (cuts) {  // the staging slots must hold the largest chunk
    size_t max_bytes = 0;
    for (size_t c = 0; c < nchunks; ++c)
      max_bytes = std::max(max_bytes, (size_t)((soff[cb[c + 1] - 1] + num_samples[cb[c + 1] - 1]) - soff[cb[c]]) * esz);
    for (int k = 0; k < 2; ++k) CU_TRY(h, grow(&r.h_stage[k], &r.h_stage_cap[k], max_bytes + 64, true));
  }

  float *scratch = h->plan.whisper ? r.d_out + (tot.out_floats - B) : nullptr;
  int launches = 0;
  for (size_t c = 0; c < nchunks; ++c) {
    const int b0 = cb[c], b1 = cb[c + 1], slot = (int)(c & 1);
    cudaStream_t st = r.streams[c % 3];
    if (c < 3) CU_TRY(h, cudaStreamWaitEvent(st, r.meta_ready, 0));
    const int64_t e0 = soff[b0], e1 = soff[b1 - 1] + num_samples[b1 - 1];
    const void *chunk = static_cast<const char *>(src) + e0 * esz;
    if (cuts) {
      if (c >= 2) CU_TRY(h, cudaEventSynchronize(r.stage_free[slot]));  // the H2D copy out of this slot (chunk c - 2) is done
      gather_chunk(h->pool, static_cast<unsigned char *>(r.h_stage[slot]), cuts, soff, num_samples, b0, b1, esz);
      chunk = r.h_stage[slot];
    }
    CU_TRY(h, cudaMemcpyAsync((char *)r.d_samples + e0 * esz, chunk, (size_t)(e1 - e0) * esz, cudaMemcpyHostToDevice, st));
    if (cuts) CU_TRY(h, cudaEventRecord(r.stage_free[slot], st));
    int64_t f0, f1;
    if (out_mode == B200FEAT_OUT_PADDED) { f0 = (int64_t)b0 * tot.max_frames; f1 = (int64_t)b1 * tot.max_frames; }
    else { f0 = roff[b0]; f1 = roff[b1]; }
    rc = launch_range(h, r.d_samples, dt, r.d_meta, B, b0, b1, toff[b0], toff[b1], tot.max_frames, r.d_out, out_mode, pad_value, st,
                      scratch, f1 - f0);
    if (rc) return rc;
    launches += h->plan.whisper ? 2 : 1;
    CU_TRY(h, cudaMemcpyAsync(out_host + f0 * h->plan.F, r.d_out + f0 * h->plan.F, (size_t)(f1 - f0) * h->plan.F * 4,
                              cudaMemcpyDeviceToHost, st));
  }
  for (auto &s : r.streams) CU_TRY(h, cudaStreamSynchronize(s));
  {
    std::lock_guard<std::mutex> g(h->stats_mu);
    h->stats.calls++; h->stats.cuts += B; h->stats.frames += tot.total_rows;
    h->stats.samples += tot.span_samples; h->stats.kernel_launches += launches;
  }
  return B200FEAT_OK;
}


}  // namespace

extern "C" {

int b200feat_version(void) { return B200FEAT_ABI_VERSION; }
const char *b200feat_global_error(void) { return g_error.c_str(); }
const char *b200feat_last_error(const b200feat_handle *h) { return h ? h->error.c_str() : g_error.c_str(); }

int b200feat_create(const b200feat_plan_desc *desc, const float *window, const float *mel_bank,
                    const float *dct, const float *lifter, int device, b200feat_handle **out) {
  if (!desc || !out) return fail(nullptr, B200FEAT_EINVAL, "null desc/out");
  if (desc->struct_size != (int32_t)sizeof(b200feat_plan_desc))
    return fail(nullptr, B200FEAT_EINVAL, "b200feat_plan_desc size mismatch (ABI)");
  const int L = desc->frame_length, S = desc->frame_shift, N = desc->fft_length;
  if (L <= 0 || S <= 0 || N < L || N < 2) return fail(nullptr, B200FEAT_EINVAL, "bad L/S/N");
  if (!window) return fail(nullptr, B200FEAT_EINVAL, "window table is required");
  const bool whisper = desc->feature == B200FEAT_WHISPER_FBANK;
  const bool log10fb = desc->feature == B200FEAT_LOG10_FBANK;
  const bool mel = desc->feature == B200FEAT_FBANK || desc->feature == B200FEAT_MFCC || whisper || log10fb;
  if (desc->feature < 0 || desc->feature > 5) return fail(nullptr, B200FEAT_EINVAL, "bad feature kind");
  if (desc->pad_mode != B200FEAT_PAD_KALDI && desc->pad_mode != B200FEAT_PAD_CENTER)
    return fail(nullptr, B200FEAT_EINVAL, "bad pad_mode");
  if (whisper && desc->pad_mode != B200FEAT_PAD_CENTER)
    return fail(nullptr, B200FEAT_EINVAL, "whisper-fbank needs pad_mode CENTER");
  if (desc->pad_mode == B200FEAT_PAD_CENTER && !(whisper || log10fb))
    return fail(nullptr, B200FEAT_EINVAL, "pad_mode CENTER goes with the whisper-fbank and log10-fbank kinds only");
  if (log10fb && (desc->use_energy || desc->mel_floor <= 0.f || (desc->pad_mode == B200FEAT_PAD_CENTER && desc->snip_edges)))
    return fail(nullptr, B200FEAT_EINVAL, "log10-fbank: use_energy must be off, mel_floor > 0, no snip_edges with CENTER");
  if (whisper && (desc->snip_edges || desc->use_energy || desc->use_fft_mag || desc->mel_floor <= 0.f))
    return fail(nullptr, B200FEAT_EINVAL, "whisper-fbank: snip_edges / use_energy / use_fft_mag must be off, mel_floor > 0");
  if (mel && (desc->num_filters <= 0 || !mel_bank)) return fail(nullptr, B200FEAT_EINVAL, "mel bank required");
  if (desc->feature == B200FEAT_MFCC && (desc->num_ceps <= 0 || !dct))
    return fail(nullptr, B200FEAT_EINVAL, "dct required for mfcc");
  if (desc->use_lifter && !lifter) return fail(nullptr, B200FEAT_EINVAL, "lifter table missing");

  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0)
    return fail(nullptr, B200FEAT_ENODEVICE, "no CUDA device visible: b200feat has no CPU fallback");
  if (device < 0 || device >= ndev) return fail(nullptr, B200FEAT_EINVAL, "bad device index");
  cudaDeviceProp prop;
  if (cudaGetDeviceProperties(&prop, device) != cudaSuccess)
    return fail(nullptr, B200FEAT_ECUDA, "cudaGetDeviceProperties failed");
  if (prop.major != 9 || prop.minor != 0)
    return fail(nullptr, B200FEAT_ENODEVICE,
                std::string("device is sm_") + std::to_string(prop.major * 10 + prop.minor) +
                    "; this library carries sm_90a code only");

  b200feat_handle *h = new b200feat_handle();
  h->desc = *desc;
  h->device = device;
  h->sm_count = prop.multiProcessorCount;
  DeviceGuard on(device);
  const int rc = setup_handle(h, window, mel_bank, dct, lifter);
  if (rc) {
    b200feat_destroy(h);
    return rc;
  }
  *out = h;
  return B200FEAT_OK;
}

void b200feat_destroy(b200feat_handle *h) {
  if (!h) return;
  {
    DeviceGuard on(h->device);
    for (void *p : h->allocs) cudaFree(p);
    HostRing &r = h->ring;
    if (r.d_samples) cudaFree(r.d_samples);
    if (r.d_out) cudaFree(r.d_out);
    if (r.d_meta) cudaFree(r.d_meta);
    if (r.h_meta) cudaFreeHost(r.h_meta);
    for (auto &s : r.streams) if (s) cudaStreamDestroy(s);
    if (r.meta_ready) cudaEventDestroy(r.meta_ready);
    for (int k = 0; k < 2; ++k) {
      if (r.h_stage[k]) cudaFreeHost(r.h_stage[k]);
      if (r.stage_free[k]) cudaEventDestroy(r.stage_free[k]);
    }
    delete h->pool;
  }
  delete h;
}

int64_t b200feat_num_frames(const b200feat_handle *h, int64_t n) {
  if (!h) return B200FEAT_EINVAL;
  const int64_t T = frames_for(h->desc, n);
  if (!framable(h->desc, n, T)) return B200FEAT_ESHORT;
  return T;
}

int64_t b200feat_desc_num_frames(const b200feat_plan_desc *desc, int64_t n) {
  if (!desc || desc->struct_size != (int32_t)sizeof(b200feat_plan_desc) || desc->frame_length <= 0 || desc->frame_shift <= 0 ||
      desc->fft_length < desc->frame_length || n < 0)
    return B200FEAT_EINVAL;
  const int64_t T = frames_for(*desc, n);
  return framable(*desc, n, T) ? T : (int64_t)B200FEAT_ESHORT;
}

int32_t b200feat_feature_dim(const b200feat_handle *h) { return h ? h->plan.F : B200FEAT_EINVAL; }
int32_t b200feat_kernel_kind(const b200feat_handle *h) { return h ? h->kernel : B200FEAT_EINVAL; }
int64_t b200feat_meta_words(int32_t batch) { return 4 * (int64_t)batch + 2; }

int64_t b200feat_plan_words(const b200feat_handle *hc, const int64_t *num_samples, int32_t B, int32_t out_mode) {
  b200feat_handle *h = const_cast<b200feat_handle *>(hc);
  if (!h || !num_samples || B <= 0) return fail(h, B200FEAT_EINVAL, "plan_words: bad arguments");
  int64_t words = b200feat_meta_words(B);
  const int64_t ft = h->frames_per_tile;
  if (ft <= 1) return words;
  int64_t tmax = 0, tiles = 0;
  for (int i = 0; i < B; ++i) {
    const int64_t T = cut_frames(h, i, num_samples[i]);
    if (T < 0) return T;
    if (T > tmax) tmax = T;
    tiles += (T + ft - 1) / ft;
  }
  if (out_mode == B200FEAT_OUT_PADDED) tiles = (int64_t)B * ((tmax + ft - 1) / ft);
  return words + (tiles + 1) / 2;
}

int b200feat_plan_batch(const b200feat_handle *hc, const int64_t *num_samples,
                        const int64_t *sample_offsets, int32_t B, int32_t align, int32_t out_mode,
                        int64_t *meta, int64_t meta_capacity, b200feat_batch_totals *tot) {
  b200feat_handle *h = const_cast<b200feat_handle *>(hc);
  if (!h || !num_samples || !meta || !tot || B <= 0) return fail(h, B200FEAT_EINVAL, "plan_batch: bad arguments");
  if (out_mode != B200FEAT_OUT_PACKED && out_mode != B200FEAT_OUT_PADDED) return fail(h, B200FEAT_EINVAL, "bad out_mode");
  if (align < 1) align = 1;
  if (meta_capacity < b200feat_meta_words(B)) return fail(h, B200FEAT_EINVAL, "plan_batch: meta buffer too small");
  int64_t *soff = meta, *ns = meta + B, *roff = meta + 2 * (int64_t)B, *toff = meta + 3 * (int64_t)B + 1;
  int64_t cur = 0, rows = 0, tmax = 0, span = 0;
  for (int i = 0; i < B; ++i) {
    const int64_t n = num_samples[i];
    const int64_t T = cut_frames(h, i, n);
    if (T < 0) return (int)T;
    if (sample_offsets) soff[i] = sample_offsets[i];
    else { cur = (cur + align - 1) / align * align; soff[i] = cur; cur += n; }
    ns[i] = n;
    roff[i] = rows;
    rows += T;
    if (T > tmax) tmax = T;
    if (soff[i] + n > span) span = soff[i] + n;
  }
  roff[B] = rows;
  const int64_t ft = h->frames_per_tile;
  int64_t tiles = 0;
  for (int i = 0; i < B; ++i) {
    toff[i] = tiles;
    const int64_t r = out_mode == B200FEAT_OUT_PADDED ? tmax : roff[i + 1] - roff[i];
    tiles += (r + ft - 1) / ft;
  }
  toff[B] = tiles;
  int64_t words = b200feat_meta_words(B);
  if (ft > 1) {  // tile -> cut table for the tiled kernel
    if (meta_capacity < words + (tiles + 1) / 2) return fail(h, B200FEAT_EINVAL, "plan_batch: meta buffer too small for the tile table");
    int32_t *tc = reinterpret_cast<int32_t *>(meta + words);
    for (int i = 0; i < B; ++i)
      for (int64_t t = toff[i]; t < toff[i + 1]; ++t) tc[t] = i;
    if (tiles & 1) tc[tiles] = 0;
    words += (tiles + 1) / 2;
  }
  tot->meta_words = words;
  tot->total_rows = rows; tot->max_frames = tmax; tot->total_tiles = tiles; tot->span_samples = span;
  tot->out_floats = (out_mode == B200FEAT_OUT_PADDED ? (int64_t)B * tmax : rows) * h->plan.F;
  if (h->plan.whisper) tot->out_floats += B;  // scratch tail: per-cut maxima
  return B200FEAT_OK;
}


int b200feat_extract(b200feat_handle *h, const void *samples_dev, int32_t dt, const int64_t *meta_dev,
                     int32_t B, const b200feat_batch_totals *tot, float *out_dev, int32_t out_mode,
                     float pad_value, void *stream) {
  if (!h || !samples_dev || !meta_dev || !tot || !out_dev || B <= 0) return fail(h, B200FEAT_EINVAL, "extract: bad arguments");
  if (dt != B200FEAT_F32 && dt != B200FEAT_I16) return fail(h, B200FEAT_EINVAL, "bad sample dtype");
  DeviceGuard on(h->device);
  const int64_t all_rows = out_mode == B200FEAT_OUT_PADDED ? (int64_t)B * tot->max_frames : tot->total_rows;
  float *scratch = h->plan.whisper ? out_dev + all_rows * h->plan.F : nullptr;
  int rc = launch_range(h, samples_dev, dt, meta_dev, B, 0, B, 0, tot->total_tiles, tot->max_frames, out_dev,
                        out_mode, pad_value, (cudaStream_t)stream, scratch, all_rows);
  if (rc) return rc;
  {
    std::lock_guard<std::mutex> g(h->stats_mu);
    h->stats.calls++; h->stats.cuts += B; h->stats.frames += tot->total_rows;
    h->stats.kernel_launches += h->plan.whisper ? 2 : 1;
  }
  return B200FEAT_OK;
}


int b200feat_extract_keep_raw(b200feat_handle *h, const void *samples_dev, int32_t dt, const int64_t *meta_dev, int32_t B,
                              const b200feat_batch_totals *tot, float *out_dev, float *raw_dev, void *stream) {
  if (!h || !samples_dev || !meta_dev || !tot || !out_dev || !raw_dev || B <= 0)
    return fail(h, B200FEAT_EINVAL, "extract_keep_raw: bad arguments");
  if (!h->plan.whisper) return fail(h, B200FEAT_EINVAL, "extract_keep_raw: whisper-fbank handles only");
  if (dt != B200FEAT_F32 && dt != B200FEAT_I16) return fail(h, B200FEAT_EINVAL, "bad sample dtype");
  if (((uintptr_t)out_dev | (uintptr_t)raw_dev) & 15) return fail(h, B200FEAT_EINVAL, "extract_keep_raw: out and raw must be 16-byte aligned");
  DeviceGuard on(h->device);
  float *scratch = raw_dev + tot->total_rows * h->plan.F;
  int rc = launch_range(h, samples_dev, dt, meta_dev, B, 0, B, 0, tot->total_tiles, tot->max_frames, raw_dev,
                        B200FEAT_OUT_PACKED, 0.f, (cudaStream_t)stream, scratch, tot->total_rows, out_dev);
  if (rc) return rc;
  {
    std::lock_guard<std::mutex> g(h->stats_mu);
    h->stats.calls++; h->stats.cuts += B; h->stats.frames += tot->total_rows;
    h->stats.kernel_launches += 2;
  }
  return B200FEAT_OK;
}


int b200feat_extract_host(b200feat_handle *h, const void *samples_host, int32_t dt,
                          const int64_t *num_samples, int32_t B, float *out_host, int32_t out_mode,
                          float pad_value) {
  return b200feat_extract_host_at(h, samples_host, dt, num_samples, nullptr, B, out_host, out_mode, pad_value);
}

int b200feat_extract_host_at(b200feat_handle *h, const void *samples_host, int32_t dt,
                             const int64_t *num_samples, const int64_t *sample_offsets, int32_t B,
                             float *out_host, int32_t out_mode, float pad_value) {
  if (!h || !samples_host || !num_samples || !out_host || B <= 0) return fail(h, B200FEAT_EINVAL, "extract_host: bad arguments");
  if (sample_offsets) {
    int64_t end = 0;
    for (int i = 0; i < B; ++i) {
      if (sample_offsets[i] < end) return fail(h, B200FEAT_EINVAL, "extract_host_at: offsets must be increasing and non-overlapping");
      end = sample_offsets[i] + num_samples[i];
    }
  }
  if (dt != B200FEAT_F32 && dt != B200FEAT_I16) return fail(h, B200FEAT_EINVAL, "bad sample dtype");
  return extract_staged(h, samples_host, nullptr, dt, num_samples, sample_offsets, B, out_host, out_mode, pad_value);
}

int b200feat_extract_host_ptrs(b200feat_handle *h, const void *const *cuts, int32_t dt, const int64_t *num_samples, int32_t B,
                               float *out_host, int32_t out_mode, float pad_value) {
  if (!h || !cuts || !num_samples || !out_host || B <= 0) return fail(h, B200FEAT_EINVAL, "extract_host_ptrs: bad arguments");
  if (dt != B200FEAT_F32 && dt != B200FEAT_I16) return fail(h, B200FEAT_EINVAL, "bad sample dtype");
  for (int i = 0; i < B; ++i)
    if (!cuts[i] && num_samples[i] > 0) return fail(h, B200FEAT_EINVAL, "extract_host_ptrs: null cut pointer");
  return extract_staged(h, nullptr, cuts, dt, num_samples, nullptr, B, out_host, out_mode, pad_value);
}

int64_t b200feat_get_table(b200feat_handle *h, int32_t which, float *out, int64_t cap) {
  if (!h || !out) return B200FEAT_EINVAL;
  const DevPlan &p = h->plan;
  DeviceGuard on(h->device);
  auto pull = [&](const void *src, int64_t count) -> int64_t {
    if (count > cap) return fail(h, B200FEAT_EINVAL, "get_table: capacity too small");
    if (cudaMemcpy(out, src, (size_t)count * 4, cudaMemcpyDeviceToHost) != cudaSuccess)
      return fail(h, B200FEAT_ECUDA, "get_table: memcpy failed");
    return count;
  };
  switch (which) {
    case 0: return pull(p.window, p.L);
    case 1: {
      if (!p.M) return 0;
      const int64_t count = (int64_t)p.K * p.M;
      if (count > cap) return fail(h, B200FEAT_EINVAL, "get_table: capacity too small");
      std::vector<int> st(p.M), len(p.M), off(p.M);
      cudaMemcpy(st.data(), p.mel_start, p.M * 4, cudaMemcpyDeviceToHost);
      cudaMemcpy(len.data(), p.mel_len, p.M * 4, cudaMemcpyDeviceToHost);
      cudaMemcpy(off.data(), p.mel_woff, p.M * 4, cudaMemcpyDeviceToHost);
      int nnz = 1;
      for (int m = 0; m < p.M; ++m) nnz = off[m] + len[m] > nnz ? off[m] + len[m] : nnz;
      std::vector<float> w(nnz);
      cudaMemcpy(w.data(), p.mel_w, (size_t)nnz * 4, cudaMemcpyDeviceToHost);
      memset(out, 0, (size_t)count * 4);
      for (int m = 0; m < p.M; ++m)
        for (int i = 0; i < len[m]; ++i) out[(size_t)(st[m] + i) * p.M + m] = w[off[m] + i];
      return count;
    }
    case 2: return p.C ? pull(p.dct, (int64_t)p.M * p.C) : 0;
    case 3: return p.use_lifter ? pull(p.lifter, p.C) : 0;
    case 4: return pull(p.tw, (int64_t)p.Nc * 2);
    default: return fail(h, B200FEAT_EINVAL, "get_table: unknown table");
  }
}

int b200feat_set_output_affine(b200feat_handle *h, const float *scale, const float *shift) {
  if (!h) return B200FEAT_EINVAL;
  if (h->plan.whisper) return fail(h, B200FEAT_EUNSUPPORTED, "output affine: not available for whisper-fbank (its normalise pass is per cut)");
  if (!scale || !shift) {
    h->plan.post_scale = h->plan.post_shift = nullptr;
    return B200FEAT_OK;
  }
  DeviceGuard on(h->device);
  const size_t bytes = (size_t)h->plan.F * sizeof(float);
  if (!h->d_affine) {
    CU_TRY(h, cudaMalloc((void **)&h->d_affine, 2 * bytes));
    h->allocs.push_back(h->d_affine);
  }
  CU_TRY(h, cudaMemcpy(h->d_affine, scale, bytes, cudaMemcpyHostToDevice));
  CU_TRY(h, cudaMemcpy(h->d_affine + h->plan.F, shift, bytes, cudaMemcpyHostToDevice));
  h->plan.post_scale = h->d_affine;
  h->plan.post_shift = h->d_affine + h->plan.F;
  return B200FEAT_OK;
}

int b200feat_get_stats(const b200feat_handle *h, b200feat_stats *out) {
  if (!h || !out) return B200FEAT_EINVAL;
  *out = h->stats;
  return B200FEAT_OK;
}

int64_t b200feat_flac_index(const uint8_t *file, int64_t nbytes, b200feat_flac_stream *info, b200feat_flac_frame *frames,
                            int64_t capacity) {
  const int64_t r = flac_index(file, nbytes, info, frames, capacity);
  if (r < 0) fail(nullptr, (int)r, "flac_index: not a FLAC stream with a valid STREAMINFO block (or bad arguments)");
  return r;
}

int b200feat_flac_decode(const uint8_t *bytes_dev, const b200feat_flac_job *jobs_dev, int32_t njobs, int16_t *out_dev,
                         int64_t out_elems, int32_t *status_dev, void *scratch_dev, int64_t scratch_bytes, void *stream) {
  if (njobs < 0 || (njobs > 0 && (!bytes_dev || !jobs_dev || !out_dev || !status_dev)) || out_elems < 0 || scratch_bytes < 0)
    return fail(nullptr, B200FEAT_EINVAL, "flac_decode: bad arguments");
  if (njobs == 0) return B200FEAT_OK;
  flac_decode_kernel<<<(njobs + FLAC_THREADS - 1) / FLAC_THREADS, FLAC_THREADS, 0, (cudaStream_t)stream>>>(
      bytes_dev, jobs_dev, njobs, out_dev, out_elems, status_dev, (int32_t *)scratch_dev, scratch_dev ? scratch_bytes / 4 : 0);
  CU_TRY(nullptr, cudaGetLastError());
  return B200FEAT_OK;
}

int64_t b200feat_mix_work_bytes(int32_t ntracks, int32_t ncuts) {
  if (ntracks < 0 || ncuts < 0) return 0;
  auto up = [](int64_t b) { return (b + 255) / 256 * 256; };
  return up((int64_t)ntracks * (int64_t)sizeof(b200feat_mix_track)) + up((int64_t)ncuts * (int64_t)sizeof(b200feat_mix_cut)) +
         up((int64_t)ntracks * 8) + up((int64_t)ntracks * 4) + up((int64_t)ncuts * 8);
}

int b200feat_mix(b200feat_handle *h, const int16_t *src0_dev, int64_t src0_elems, const int16_t *src1_dev, int64_t src1_elems,
                 const b200feat_mix_track *tracks, int32_t ntracks, const b200feat_mix_cut *cuts, int32_t ncuts,
                 float *out_dev, int64_t out_elems, void *work_dev, int64_t work_bytes, void *stream) {
  return b200feat_mix_ex(h, src0_dev, src0_elems, src1_dev, src1_elems, nullptr, 0, tracks, ntracks, cuts, ncuts, out_dev,
                         out_elems, work_dev, work_bytes, stream);
}

int b200feat_mix_ex(b200feat_handle *h, const int16_t *src0_dev, int64_t src0_elems, const int16_t *src1_dev, int64_t src1_elems,
                    const float *src2_dev, int64_t src2_elems, const b200feat_mix_track *tracks, int32_t ntracks,
                    const b200feat_mix_cut *cuts, int32_t ncuts, float *out_dev, int64_t out_elems, void *work_dev,
                    int64_t work_bytes, void *stream) {
  if (ntracks < 0 || ncuts < 0 || (ncuts > 0 && (!tracks || !cuts || !out_dev || !work_dev)) || out_elems < 0 || src0_elems < 0 ||
      src1_elems < 0 || src2_elems < 0)
    return fail(h, B200FEAT_EINVAL, "mix: bad arguments");
  if (ncuts == 0) return B200FEAT_OK;
  if (ncuts > 65535) return fail(h, B200FEAT_EINVAL, "mix: more than 65535 cuts in one call");
  if (work_bytes < b200feat_mix_work_bytes(ntracks, ncuts)) return fail(h, B200FEAT_EINVAL, "mix: work buffer too small");
  const void *src[3] = {src0_dev, src1_dev, src2_dev};
  const int64_t src_elems[3] = {src0_elems, src1_elems, src2_elems};
  auto where = [](const char *what, int64_t i) { return std::string("mix: ") + what + " " + std::to_string(i) + ": "; };
  for (int32_t t = 0; t < ntracks; ++t) {
    const b200feat_mix_track &tr = tracks[t];
    if (tr.struct_size != (int32_t)sizeof(b200feat_mix_track))
      return fail(h, B200FEAT_EINVAL, where("track", t) + "b200feat_mix_track size mismatch (ABI)");
    if (tr.source < -1 || tr.source > B200FEAT_MIX_SRC_F32)
      return fail(h, B200FEAT_EINVAL, where("track", t) + "source must be 0, 1, 2 (float32) or -1 (padding)");
    if (tr.source == B200FEAT_MIX_SRC_F32 && !src2_dev)
      return fail(h, B200FEAT_EINVAL, where("track", t) + "a float32 track without the float32 source (src2)");
    if (tr.num_samples < 0 || tr.num_samples > ((int64_t)1 << 40) || tr.mix_offset < 0 || tr.mix_offset > ((int64_t)1 << 40))
      return fail(h, B200FEAT_EINVAL, where("track", t) + "bad length or mix offset");
    if (tr.source >= 0 && (!src[tr.source] || tr.src_elem < 0 || tr.src_elem > src_elems[tr.source] - tr.num_samples))
      return fail(h, B200FEAT_EINVAL, where("track", t) + "samples outside its source buffer");
    if (tr.role != B200FEAT_MIX_ROLE_MIXED && tr.role != B200FEAT_MIX_ROLE_ENERGY)
      return fail(h, B200FEAT_EINVAL, where("track", t) + "bad role");
    if (tr.cut < 0 || tr.cut >= ncuts) return fail(h, B200FEAT_EINVAL, where("track", t) + "cut index out of range");
  }
  for (int32_t c = 0; c < ncuts; ++c) {
    const b200feat_mix_cut &cu = cuts[c];
    if (cu.struct_size != (int32_t)sizeof(b200feat_mix_cut))
      return fail(h, B200FEAT_EINVAL, where("cut", c) + "b200feat_mix_cut size mismatch (ABI)");
    if (cu.mode != B200FEAT_MIX_F32 && cu.mode != B200FEAT_MIX_SCALED_FIRST) return fail(h, B200FEAT_EINVAL, where("cut", c) + "bad mode");
    if (cu.num_tracks < 1 || cu.first_track < 0 || (int64_t)cu.first_track + cu.num_tracks > ntracks)
      return fail(h, B200FEAT_EINVAL, where("cut", c) + "tracks outside the track table");
    if (cu.ref_track < 0 || cu.ref_track >= cu.num_tracks) return fail(h, B200FEAT_EINVAL, where("cut", c) + "reference index outside the cut's tracks");
    if (cu.out_elem < 0 || cu.target_len < 0 || cu.out_elem + cu.target_len > out_elems)
      return fail(h, B200FEAT_EINVAL, where("cut", c) + "outside the output buffer");
    int64_t len = 0;
    for (int32_t k = 0; k < cu.num_tracks; ++k) {
      const b200feat_mix_track &tr = tracks[cu.first_track + k];
      if (tr.cut != c) return fail(h, B200FEAT_EINVAL, where("cut", c) + "a track of another cut inside its range");
      if (k == 0 && tr.role != B200FEAT_MIX_ROLE_MIXED) return fail(h, B200FEAT_EINVAL, where("cut", c) + "the first track must be mixed");
      if (tr.role == B200FEAT_MIX_ROLE_MIXED) len = std::max(len, tr.mix_offset + tr.num_samples);
    }
    if (len != cu.mix_len) return fail(h, B200FEAT_EINVAL, where("cut", c) + "mix_len is not the end of its last track");
    if (cu.target_len > cu.mix_len && cu.target_len - cu.mix_len > cu.mix_len - 1)
      return fail(h, B200FEAT_EINVAL, where("cut", c) + "reflect padding longer than the mix");
  }
  auto up = [](int64_t b) { return (b + 255) / 256 * 256; };
  char *w = (char *)work_dev;
  b200feat_mix_track *d_tracks = (b200feat_mix_track *)w;
  w += up((int64_t)ntracks * (int64_t)sizeof(b200feat_mix_track));
  b200feat_mix_cut *d_cuts = (b200feat_mix_cut *)w;
  w += up((int64_t)ncuts * (int64_t)sizeof(b200feat_mix_cut));
  double *energy = (double *)w;
  w += up((int64_t)ntracks * 8);
  float *gain32 = (float *)w;
  w += up((int64_t)ntracks * 4);
  double *scale64 = (double *)w;
  const cudaStream_t st = (cudaStream_t)stream;
  if (ntracks) CU_TRY(h, cudaMemcpyAsync(d_tracks, tracks, (size_t)ntracks * sizeof(b200feat_mix_track), cudaMemcpyHostToDevice, st));
  CU_TRY(h, cudaMemcpyAsync(d_cuts, cuts, (size_t)ncuts * sizeof(b200feat_mix_cut), cudaMemcpyHostToDevice, st));
  mix_energy_kernel<<<ncuts, MIX_THREADS, 0, st>>>(src0_dev, src1_dev, src2_dev, d_tracks, d_cuts, energy, gain32, scale64);
  CU_TRY(h, cudaGetLastError());
  int64_t longest = 1;
  for (int32_t c = 0; c < ncuts; ++c) longest = std::max(longest, cuts[c].target_len);
  const int64_t gx = std::min<int64_t>((longest + 4 * MIX_MIX_THREADS - 1) / (4 * MIX_MIX_THREADS), 1024);
  mix_kernel<<<dim3((unsigned)gx, (unsigned)ncuts), MIX_MIX_THREADS, 0, st>>>(src0_dev, src1_dev, src2_dev, d_tracks, d_cuts, gain32, scale64,
                                                                              out_dev);
  CU_TRY(h, cudaGetLastError());
  return B200FEAT_OK;
}

}  // extern "C"

namespace {

// Resampling tables, [K][N] on the device, kept per (device, orig, new) for the life of the process: a table is a pure
// function of its pair, and a handle-free caller (lhotse_b200.transform_cuts) shares them with every extractor.
struct RsTable {
  int device;
  int32_t orig, new_rate, N, O, K, width;
  const float *dev;
};
std::mutex g_rs_mu;
std::vector<RsTable> g_rs_tables;  // the id of a table is its index
std::vector<void *> g_rs_allocs;

}  // namespace

extern "C" {

int b200feat_resample_table(b200feat_handle *h, int32_t orig, int32_t new_rate, const float *kernel, int32_t rows, int32_t taps,
                            int32_t width, int32_t *table_id) {
  if (orig <= 0 || new_rate <= 0 || orig == new_rate || !table_id) return fail(h, B200FEAT_EINVAL, "resample_table: bad arguments");
  int device = 0;
  CU_TRY(h, cudaGetDevice(&device));
  std::lock_guard<std::mutex> g(g_rs_mu);
  for (size_t i = 0; i < g_rs_tables.size(); ++i) {
    const RsTable &t = g_rs_tables[i];
    if (t.device == device && t.orig == orig && t.new_rate == new_rate) {
      *table_id = (int32_t)i;
      return B200FEAT_OK;
    }
  }
  int32_t a = orig, b = new_rate;
  while (b) { const int32_t r = a % b; a = b; b = r; }
  const int32_t O = orig / a, N = new_rate / a;
  if (!kernel || rows != N || width <= 0 || taps != 2 * width + O)
    return fail(h, B200FEAT_EINVAL, "resample_table: the table is not N x (2 * width + O) for the pair");
  if ((int64_t)taps + O > RS_WIN_FLOATS || (int64_t)rows * taps > ((int64_t)1 << 22))
    return fail(h, B200FEAT_EINVAL, "resample_table: table too large for the resampling kernel");
  std::vector<float> tr((size_t)rows * taps);
  for (int32_t p = 0; p < rows; ++p)
    for (int32_t t = 0; t < taps; ++t) tr[(size_t)t * rows + p] = kernel[(size_t)p * taps + t];
  const float *dev = nullptr;
  CU_TRY(h, upload_table(tr, g_rs_allocs, &dev));
  g_rs_tables.push_back(RsTable{device, orig, new_rate, N, O, taps, width, dev});
  *table_id = (int32_t)(g_rs_tables.size() - 1);
  return B200FEAT_OK;
}

int64_t b200feat_resample_work_bytes(int32_t nstages) {
  if (nstages < 0) return 0;
  return ((int64_t)nstages * (int64_t)sizeof(RsStage) + 255) / 256 * 256;
}

int b200feat_resample(b200feat_handle *h, const int16_t *src0_dev, int64_t src0_elems, const int16_t *src1_dev,
                      int64_t src1_elems, float *mid_dev, int64_t mid_elems, const b200feat_resample_stage *stages,
                      int32_t nstages, float *out_dev, int64_t out_elems, void *work_dev, int64_t work_bytes, void *stream) {
  if (nstages < 0 || (nstages > 0 && (!stages || !work_dev)) || src0_elems < 0 || src1_elems < 0 || mid_elems < 0 || out_elems < 0)
    return fail(h, B200FEAT_EINVAL, "resample: bad arguments");
  if (nstages == 0) return B200FEAT_OK;
  if (work_bytes < b200feat_resample_work_bytes(nstages)) return fail(h, B200FEAT_EINVAL, "resample: work buffer too small");
  int device = 0;
  CU_TRY(h, cudaGetDevice(&device));
  const void *src[3] = {src0_dev, src1_dev, mid_dev};
  const int64_t src_elems[3] = {src0_elems, src1_elems, mid_elems};
  float *dst[2] = {mid_dev, out_dev};
  const int64_t dst_elems[2] = {mid_elems, out_elems};
  auto where = [](int32_t i) { return std::string("resample: stage ") + std::to_string(i) + ": "; };
  std::vector<RsStage> rs((size_t)nstages);
  std::vector<int32_t> group_start;  // first record of every depth
  std::vector<size_t> group_smem;
  int64_t ctas = 0;
  {
    std::lock_guard<std::mutex> g(g_rs_mu);
    for (int32_t i = 0; i < nstages; ++i) {
      const b200feat_resample_stage &s = stages[i];
      if (s.struct_size != (int32_t)sizeof(b200feat_resample_stage))
        return fail(h, B200FEAT_EINVAL, where(i) + "b200feat_resample_stage size mismatch (ABI)");
      if (s.source < 0 || s.source > 2 || s.target < 0 || s.target > 1) return fail(h, B200FEAT_EINVAL, where(i) + "bad source or target");
      if (s.depth < 0 || (i > 0 && s.depth < stages[i - 1].depth)) return fail(h, B200FEAT_EINVAL, where(i) + "records not in depth order");
      const RsTable *t = nullptr;
      if (s.table != -1) {
        if (s.table < 0 || s.table >= (int32_t)g_rs_tables.size() || g_rs_tables[s.table].device != device)
          return fail(h, B200FEAT_EINVAL, where(i) + "unknown table id on this device");
        t = &g_rs_tables[s.table];
      }
      if (s.in_len < 1 || s.in_len > ((int64_t)1 << 40) || s.in_elem < 0 || !src[s.source] || s.in_elem > src_elems[s.source] - s.in_len)
        return fail(h, B200FEAT_EINVAL, where(i) + "input outside its source buffer");
      // lhotse keeps torch.ceil(torch.as_tensor(N * L / O)) outputs: the double quotient as a float32 tensor, then its ceil,
      // at most the N * (L / O + 1) the conv produces
      const int64_t want = t ? std::min((int64_t)ceilf((float)((double)((int64_t)t->N * s.in_len) / (double)t->O)),
                                        (int64_t)t->N * (s.in_len / t->O + 1))
                             : s.in_len;
      if (s.out_len != want) return fail(h, B200FEAT_EINVAL, where(i) + "out_len is not lhotse's ceil(f32(N * L / O))");
      if (s.target_len < 0 || (s.target == B200FEAT_RESAMPLE_TO_MID && s.target_len != s.out_len) ||
          (s.target_len > s.out_len && s.target_len - s.out_len > s.out_len - 1))
        return fail(h, B200FEAT_EINVAL, where(i) + "bad target_len (reflect padding longer than the stage output?)");
      if (s.out_elem < 0 || !dst[s.target] || s.out_elem > dst_elems[s.target] - s.target_len)
        return fail(h, B200FEAT_EINVAL, where(i) + "output outside its target buffer");
      if (i == 0 || s.depth != stages[i - 1].depth) {
        group_start.push_back(i);
        group_smem.push_back(0);
        ctas = 0;
      }
      RsStage &r = rs[i];
      r.tab = t ? t->dev : nullptr;
      r.src16 = s.source == B200FEAT_RESAMPLE_MID ? nullptr : (const int16_t *)src[s.source] + s.in_elem;
      r.src32 = s.source == B200FEAT_RESAMPLE_MID ? mid_dev + s.in_elem : nullptr;
      r.dst = dst[s.target] + s.out_elem;
      r.in_len = s.in_len;
      r.out_len = s.out_len;
      r.target_len = s.target_len;
      r.N = t ? t->N : 1;
      r.O = t ? t->O : 1;
      r.K = t ? t->K : 1;
      r.width = t ? t->width : 0;
      r.chunk = rs_chunk_outputs(r.N, r.O, r.K);
      r.tab_smem = t && (int64_t)r.N * r.K <= RS_SMEM_TAB_FLOATS;
      r.scale_in = s.scale_in;
      r.scale_out = s.scale_out;
      r.cta_begin = ctas;
      ctas += rs_stage_ctas(r);
      if (ctas > 0x7fffffff) return fail(h, B200FEAT_EINVAL, where(i) + "too many CTAs in one depth");
      if (t) group_smem.back() = std::max(group_smem.back(), sizeof(float) * (size_t)rs_smem_floats(r));
    }
  }
  const cudaStream_t st = (cudaStream_t)stream;
  RsStage *d_rs = (RsStage *)work_dev;
  // a pageable copy: the call returns once `rs` has been staged, so the vector may go when this function returns
  CU_TRY(h, cudaMemcpyAsync(d_rs, rs.data(), rs.size() * sizeof(RsStage), cudaMemcpyHostToDevice, st));
  group_start.push_back(nstages);
  for (size_t gi = 0; gi + 1 < group_start.size(); ++gi) {
    const int32_t a = group_start[gi], b = group_start[gi + 1];
    const RsStage &last = rs[b - 1];
    const int64_t n = last.cta_begin + rs_stage_ctas(last);
    if (n == 0) continue;
    resample_stage_kernel<<<(unsigned)n, RS_THREADS, group_smem[gi], st>>>(d_rs + a, b - a);
    CU_TRY(h, cudaGetLastError());
  }
  return B200FEAT_OK;
}

}  // extern "C"

namespace {

// The reverb work buffer: the kernels' RIR and cut tables, the shifts, the RIR spectra, y, the per-CTA partials and the gains
struct RvLayout {
  int64_t rirs, cuts, shift, twiddles, spectra, y, partial, gain, total;
  int64_t parts, samples, ctas;
};

RvLayout rv_layout(const b200feat_reverb_rir *rirs, int32_t nrirs, const b200feat_reverb_cut *cuts, int32_t ncuts) {
  auto up = [](int64_t b) { return (b + 255) / 256 * 256; };
  RvLayout l{};
  for (int32_t i = 0; i < nrirs; ++i) l.parts += rv_parts(std::min<int64_t>(std::max<int64_t>(rirs[i].num_samples, 0), RV_MAX_RIR));
  for (int32_t i = 0; i < ncuts; ++i) {
    const int64_t n = std::min<int64_t>(std::max<int64_t>(cuts[i].in_len, 0), (int64_t)1 << 40);
    l.samples += n;
    l.ctas += rv_cut_ctas(n);
  }
  l.rirs = 0;
  l.cuts = l.rirs + up((int64_t)nrirs * (int64_t)sizeof(RvRir));
  l.shift = l.cuts + up((int64_t)ncuts * (int64_t)sizeof(RvCut));
  l.twiddles = l.shift + up((int64_t)nrirs * 4);
  l.spectra = l.twiddles + up(RV_B * (int64_t)sizeof(rv_c));
  l.y = l.spectra + up(l.parts * RV_F * (int64_t)sizeof(rv_c));
  l.partial = l.y + up(l.samples * 4);
  l.gain = l.partial + up(l.ctas * 4);
  l.total = l.gain + up((int64_t)ncuts * 4);
  return l;
}

}  // namespace

extern "C" {

int64_t b200feat_reverb_work_bytes(const b200feat_reverb_rir *rirs, int32_t nrirs, const b200feat_reverb_cut *cuts, int32_t ncuts) {
  if (nrirs < 0 || ncuts < 0 || (nrirs > 0 && !rirs) || (ncuts > 0 && !cuts)) return 0;
  return rv_layout(rirs, nrirs, cuts, ncuts).total;
}

int b200feat_reverb(b200feat_handle *h, const int16_t *src0_dev, int64_t src0_elems, const int16_t *src1_dev, int64_t src1_elems,
                    const float *in_dev, int64_t in_elems, const b200feat_reverb_rir *rirs, int32_t nrirs,
                    const b200feat_reverb_cut *cuts, int32_t ncuts, float *out_dev, int64_t out_elems, void *work_dev,
                    int64_t work_bytes, void *stream) {
  return b200feat_reverb_ex(h, src0_dev, src0_elems, src1_dev, src1_elems, nullptr, 0, in_dev, in_elems, rirs, nrirs, cuts,
                            ncuts, out_dev, out_elems, work_dev, work_bytes, stream);
}

int b200feat_reverb_ex(b200feat_handle *h, const int16_t *src0_dev, int64_t src0_elems, const int16_t *src1_dev,
                       int64_t src1_elems, const float *rir32_dev, int64_t rir32_elems, const float *in_dev, int64_t in_elems,
                       const b200feat_reverb_rir *rirs, int32_t nrirs, const b200feat_reverb_cut *cuts, int32_t ncuts,
                       float *out_dev, int64_t out_elems, void *work_dev, int64_t work_bytes, void *stream) {
  if (nrirs < 0 || ncuts < 0 || (ncuts > 0 && (!rirs || !cuts || !in_dev || !out_dev || !work_dev || nrirs < 1)) ||
      src0_elems < 0 || src1_elems < 0 || rir32_elems < 0 || in_elems < 0 || out_elems < 0)
    return fail(h, B200FEAT_EINVAL, "reverb: bad arguments");
  if (ncuts == 0) return B200FEAT_OK;
  if (ncuts > 65535) return fail(h, B200FEAT_EINVAL, "reverb: more than 65535 cuts in one call");
  const int16_t *src[2] = {src0_dev, src1_dev};
  const int64_t src_elems[2] = {src0_elems, src1_elems};
  auto where = [](const char *what, int64_t i) { return std::string("reverb: ") + what + " " + std::to_string(i) + ": "; };
  for (int32_t i = 0; i < nrirs; ++i) {
    const b200feat_reverb_rir &r = rirs[i];
    if (r.struct_size != (int32_t)sizeof(b200feat_reverb_rir))
      return fail(h, B200FEAT_EINVAL, where("rir", i) + "b200feat_reverb_rir size mismatch (ABI)");
    if (r.source < 0 || r.source > 2) return fail(h, B200FEAT_EINVAL, where("rir", i) + "source must be 0, 1 or 2");
    if (r.num_samples < 1 || r.num_samples > B200FEAT_REVERB_MAX_RIR)
      return fail(h, B200FEAT_EINVAL, where("rir", i) + "length outside 1 .. B200FEAT_REVERB_MAX_RIR");
    const bool f32 = r.source == B200FEAT_REVERB_RIR_F32;
    if ((f32 ? !rir32_dev : !src[r.source]) || r.src_elem < 0 ||
        r.src_elem > (f32 ? rir32_elems : src_elems[r.source]) - r.num_samples)
      return fail(h, B200FEAT_EINVAL, where("rir", i) + "samples outside its source buffer");
  }
  for (int32_t c = 0; c < ncuts; ++c) {
    const b200feat_reverb_cut &cu = cuts[c];
    if (cu.struct_size != (int32_t)sizeof(b200feat_reverb_cut))
      return fail(h, B200FEAT_EINVAL, where("cut", c) + "b200feat_reverb_cut size mismatch (ABI)");
    if (cu.rir < 0 || cu.rir >= nrirs) return fail(h, B200FEAT_EINVAL, where("cut", c) + "RIR index out of range");
    if (cu.normalize != 0 && cu.normalize != 1) return fail(h, B200FEAT_EINVAL, where("cut", c) + "normalize must be 0 or 1");
    if (cu.in_len < 1 || cu.in_len > ((int64_t)1 << 40) || cu.in_elem < 0 || cu.in_elem > in_elems - cu.in_len)
      return fail(h, B200FEAT_EINVAL, where("cut", c) + "input outside the input buffer");
    if (cu.target_len < 0 || (cu.target_len > cu.in_len && cu.target_len - cu.in_len > cu.in_len - 1))
      return fail(h, B200FEAT_EINVAL, where("cut", c) + "bad target_len (reflect padding longer than the signal?)");
    if (cu.out_elem < 0 || cu.out_elem > out_elems - cu.target_len)
      return fail(h, B200FEAT_EINVAL, where("cut", c) + "output outside the output buffer");
  }
  {  // no cut's output window may overlap any cut's input window: the output kernel writes while others read
    std::vector<std::pair<uintptr_t, uintptr_t>> in(ncuts);
    for (int32_t c = 0; c < ncuts; ++c) {
      const uintptr_t a = (uintptr_t)(in_dev + cuts[c].in_elem);
      in[c] = {a, a + (uintptr_t)cuts[c].in_len * sizeof(float)};
    }
    std::sort(in.begin(), in.end());
    std::vector<uintptr_t> reach(ncuts);  // the furthest end among the first i + 1 windows
    for (int32_t c = 0; c < ncuts; ++c) reach[c] = std::max(in[c].second, c ? reach[c - 1] : 0);
    for (int32_t c = 0; c < ncuts; ++c) {
      if (cuts[c].target_len == 0) continue;
      const uintptr_t a = (uintptr_t)(out_dev + cuts[c].out_elem), b = a + (uintptr_t)cuts[c].target_len * sizeof(float);
      // the input windows that start before b: one of them overlaps [a, b) iff the furthest of their ends lies past a
      const auto it = std::lower_bound(in.begin(), in.end(), std::make_pair(b, (uintptr_t)0));
      if (it != in.begin() && reach[(it - in.begin()) - 1] > a)
        return fail(h, B200FEAT_EINVAL, where("cut", c) + "output overlaps an input window");
    }
  }
  const RvLayout l = rv_layout(rirs, nrirs, cuts, ncuts);
  if (work_bytes < l.total) return fail(h, B200FEAT_EINVAL, "reverb: work buffer too small");
  if (l.parts > 0x7fffffff || l.ctas > 0x7fffffff) return fail(h, B200FEAT_EINVAL, "reverb: too many CTAs in one call");
  char *w = (char *)work_dev;
  rv_c *spectra = (rv_c *)(w + l.spectra);
  float *y = (float *)(w + l.y);
  std::vector<RvRir> rv((size_t)nrirs);
  int64_t parts = 0;
  for (int32_t i = 0; i < nrirs; ++i) {
    const bool f32 = rirs[i].source == B200FEAT_REVERB_RIR_F32;
    rv[i] = RvRir{f32 ? nullptr : src[rirs[i].source] + rirs[i].src_elem, rirs[i].num_samples, parts,
                  (int32_t)rv_parts(rirs[i].num_samples), 0, f32 ? rir32_dev + rirs[i].src_elem : nullptr};
    parts += rv[i].nparts;
  }
  std::vector<RvCut> cv((size_t)ncuts);
  int64_t ctas = 0, samples = 0;
  int64_t longest = 1;
  for (int32_t c = 0; c < ncuts; ++c) {
    const b200feat_reverb_cut &cu = cuts[c];
    cv[c] = RvCut{in_dev + cu.in_elem, y + samples, out_dev + cu.out_elem, cu.in_len, cu.target_len, ctas, cu.rir, cu.normalize};
    samples += cu.in_len;
    ctas += rv_cut_ctas(cu.in_len);
    longest = std::max(longest, cu.target_len);
  }
  // just over the 48 KB a launch gets without asking; set on every call (the attribute belongs to the current device)
  CU_TRY(h, cudaFuncSetAttribute(reverb_rir_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, RV_SMEM_BYTES));
  CU_TRY(h, cudaFuncSetAttribute(reverb_conv_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, RV_SMEM_BYTES));
  const cudaStream_t st = (cudaStream_t)stream;
  RvRir *d_rirs = (RvRir *)(w + l.rirs);
  RvCut *d_cuts = (RvCut *)(w + l.cuts);
  int32_t *d_shift = (int32_t *)(w + l.shift);
  rv_c *d_twiddles = (rv_c *)(w + l.twiddles);
  float *d_partial = (float *)(w + l.partial);
  float *d_gain = (float *)(w + l.gain);
  static const std::vector<rv_c> twiddles = [] {
    std::vector<rv_c> t(RV_B);
    for (int k = 0; k < RV_B; ++k) t[k] = rv_twiddle(k);
    return t;
  }();
  // pageable copies: the call returns once the tables have been staged, so the vectors may go when this function returns
  CU_TRY(h, cudaMemcpyAsync(d_twiddles, twiddles.data(), RV_B * sizeof(rv_c), cudaMemcpyHostToDevice, st));
  CU_TRY(h, cudaMemcpyAsync(d_rirs, rv.data(), rv.size() * sizeof(RvRir), cudaMemcpyHostToDevice, st));
  CU_TRY(h, cudaMemcpyAsync(d_cuts, cv.data(), cv.size() * sizeof(RvCut), cudaMemcpyHostToDevice, st));
  reverb_rir_kernel<<<(unsigned)parts, RV_THREADS, RV_SMEM_BYTES, st>>>(d_rirs, nrirs, spectra, d_shift, d_twiddles);
  CU_TRY(h, cudaGetLastError());
  reverb_conv_kernel<<<(unsigned)ctas, RV_THREADS, RV_SMEM_BYTES, st>>>(d_cuts, ncuts, d_rirs, spectra, d_shift, d_twiddles, d_partial);
  CU_TRY(h, cudaGetLastError());
  reverb_gain_kernel<<<(unsigned)ncuts, RV_GAIN_THREADS, 0, st>>>(d_cuts, d_partial, d_gain);
  CU_TRY(h, cudaGetLastError());
  const int64_t gx = std::min<int64_t>((longest + 4 * RV_OUT_THREADS - 1) / (4 * RV_OUT_THREADS), 1024);
  reverb_out_kernel<<<dim3((unsigned)gx, (unsigned)ncuts), RV_OUT_THREADS, 0, st>>>(d_cuts, d_gain);
  CU_TRY(h, cudaGetLastError());
  return B200FEAT_OK;
}

}  // extern "C"

namespace {

// The WPE work buffer: the kernels' cut table, the window, the twiddles, then every cut's [bin][frame] spectra
struct WpeLayout {
  int64_t cuts, window, twiddles, spectra, total;
  int64_t frames;
};

WpeLayout wpe_layout(const b200feat_wpe_cut *cuts, int32_t ncuts) {
  auto up = [](int64_t b) { return (b + 255) / 256 * 256; };
  WpeLayout l{};
  for (int32_t i = 0; i < ncuts; ++i)
    l.frames += wpe_frames(std::min<int64_t>(std::max<int64_t>(cuts[i].in_len, 0), (int64_t)1 << 40));
  l.cuts = 0;
  l.window = l.cuts + up((int64_t)ncuts * (int64_t)sizeof(WpeCut));
  l.twiddles = l.window + up(WPE_NFFT * (int64_t)sizeof(float));
  l.spectra = l.twiddles + up(WPE_NFFT / 2 * (int64_t)sizeof(wpe_c));
  l.total = l.spectra + up(l.frames * WPE_BINS * (int64_t)sizeof(wpe_c));
  return l;
}

}  // namespace

extern "C" {

int64_t b200feat_wpe_work_bytes(const b200feat_wpe_cut *cuts, int32_t ncuts) {
  if (ncuts < 0 || (ncuts > 0 && !cuts)) return 0;
  return wpe_layout(cuts, ncuts).total;
}

int b200feat_wpe(b200feat_handle *h, const float *in_dev, int64_t in_elems, const b200feat_wpe_cut *cuts, int32_t ncuts,
                 const b200feat_wpe_params *params, const float *window, float *out_dev, int64_t out_elems, void *work_dev,
                 int64_t work_bytes, void *stream) {
  if (ncuts < 0 || !params || in_elems < 0 || out_elems < 0 ||
      (ncuts > 0 && (!cuts || !window || !in_dev || !out_dev || !work_dev)))
    return fail(h, B200FEAT_EINVAL, "wpe: bad arguments");
  const b200feat_wpe_params &pm = *params;
  if (pm.struct_size != (int32_t)sizeof(b200feat_wpe_params))
    return fail(h, B200FEAT_EINVAL, "wpe: b200feat_wpe_params size mismatch (ABI)");
  if (pm.n_fft != WPE_NFFT || pm.hop != WPE_HOP)
    return fail(h, B200FEAT_EUNSUPPORTED, "wpe: only n_fft = 512 and hop = 128 are supported");
  if (pm.taps < 1 || pm.taps > B200FEAT_WPE_MAX_TAPS) return fail(h, B200FEAT_EINVAL, "wpe: taps outside 1 .. B200FEAT_WPE_MAX_TAPS");
  if (pm.delay < 0 || pm.delay > B200FEAT_WPE_MAX_FRAMES) return fail(h, B200FEAT_EINVAL, "wpe: delay outside 0 .. B200FEAT_WPE_MAX_FRAMES");
  if (pm.iterations < 0 || pm.iterations > 64) return fail(h, B200FEAT_EINVAL, "wpe: iterations outside 0 .. 64");
  if (pm.statistics_mode != B200FEAT_WPE_FULL && pm.statistics_mode != B200FEAT_WPE_VALID)
    return fail(h, B200FEAT_EINVAL, "wpe: statistics_mode must be B200FEAT_WPE_FULL or B200FEAT_WPE_VALID");
  if (ncuts == 0) return B200FEAT_OK;
  if ((int64_t)ncuts * WPE_BINS > 0x7fffffff) return fail(h, B200FEAT_EINVAL, "wpe: too many cuts in one call");
  auto where = [](int64_t i) { return std::string("wpe: cut ") + std::to_string(i) + ": "; };
  for (int32_t c = 0; c < ncuts; ++c) {
    const b200feat_wpe_cut &cu = cuts[c];
    if (cu.struct_size != (int32_t)sizeof(b200feat_wpe_cut))
      return fail(h, B200FEAT_EINVAL, where(c) + "b200feat_wpe_cut size mismatch (ABI)");
    if (cu.in_len < 0 || cu.in_elem < 0 || cu.in_elem > in_elems - cu.in_len)
      return fail(h, B200FEAT_EINVAL, where(c) + "input outside the input buffer");
    if (cu.in_len <= WPE_NFFT / 2 || wpe_frames(cu.in_len) < (int64_t)pm.taps + pm.delay)
      return fail(h, B200FEAT_ESHORT, where(c) + "too short: L > 256 and 1 + L / 128 >= taps + delay are needed");
    if (wpe_frames(cu.in_len) > B200FEAT_WPE_MAX_FRAMES)
      return fail(h, B200FEAT_EINVAL, where(c) + "longer than B200FEAT_WPE_MAX_FRAMES frames");
    const int64_t lz = wpe_istft_len(cu.in_len);
    if (cu.target_len < 0 || (cu.target_len > lz && cu.target_len - lz > lz - 1))
      return fail(h, B200FEAT_EINVAL, where(c) + "bad target_len (reflect padding longer than the signal?)");
    if (cu.out_elem < 0 || cu.out_elem > out_elems - cu.target_len)
      return fail(h, B200FEAT_EINVAL, where(c) + "output outside the output buffer");
  }
  {  // no cut's output window may overlap any cut's input window (the header's contract: the input is left as it was)
    std::vector<std::pair<uintptr_t, uintptr_t>> in(ncuts);
    for (int32_t c = 0; c < ncuts; ++c) {
      const uintptr_t a = (uintptr_t)(in_dev + cuts[c].in_elem);
      in[c] = {a, a + (uintptr_t)cuts[c].in_len * sizeof(float)};
    }
    std::sort(in.begin(), in.end());
    std::vector<uintptr_t> reach(ncuts);  // the furthest end among the first i + 1 windows
    for (int32_t c = 0; c < ncuts; ++c) reach[c] = std::max(in[c].second, c ? reach[c - 1] : 0);
    for (int32_t c = 0; c < ncuts; ++c) {
      if (cuts[c].target_len == 0) continue;
      const uintptr_t a = (uintptr_t)(out_dev + cuts[c].out_elem), b = a + (uintptr_t)cuts[c].target_len * sizeof(float);
      const auto it = std::lower_bound(in.begin(), in.end(), std::make_pair(b, (uintptr_t)0));
      if (it != in.begin() && reach[(it - in.begin()) - 1] > a)
        return fail(h, B200FEAT_EINVAL, where(c) + "output overlaps an input window");
    }
  }
  const WpeLayout l = wpe_layout(cuts, ncuts);
  if (work_bytes < l.total) return fail(h, B200FEAT_EINVAL, "wpe: work buffer too small");
  char *w = (char *)work_dev;
  wpe_c *spectra = (wpe_c *)(w + l.spectra);
  std::vector<WpeCut> cv((size_t)ncuts);
  int64_t tiles = 0, outs = 0, frames = 0, longest = 1;
  for (int32_t c = 0; c < ncuts; ++c) {
    const b200feat_wpe_cut &cu = cuts[c];
    const int64_t T = wpe_frames(cu.in_len);
    cv[c] = WpeCut{in_dev + cu.in_elem, out_dev + cu.out_elem, spectra + frames * WPE_BINS, cu.in_len, cu.target_len, tiles,
                   outs, (int32_t)T, 0};
    tiles += wpe_stft_ctas(T);
    outs += wpe_istft_ctas(T);
    frames += T;
    longest = std::max(longest, T);
  }
  if (tiles > 0x7fffffff || outs > 0x7fffffff) return fail(h, B200FEAT_EINVAL, "wpe: too many CTAs in one call");
  // over the 48 KB a launch gets without asking; set on every call (the attribute belongs to the current device)
  CU_TRY(h, cudaFuncSetAttribute(wpe_stft_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, WPE_STFT_SMEM));
  CU_TRY(h, cudaFuncSetAttribute(wpe_istft_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, WPE_ISTFT_SMEM));
  CU_TRY(h, cudaFuncSetAttribute(wpe_bin_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                 WPE_BIN_SMEM(B200FEAT_WPE_MAX_FRAMES)));
  const cudaStream_t st = (cudaStream_t)stream;
  WpeCut *d_cuts = (WpeCut *)(w + l.cuts);
  float *d_window = (float *)(w + l.window);
  wpe_c *d_twiddles = (wpe_c *)(w + l.twiddles);
  static const std::vector<wpe_c> twiddles = [] {
    std::vector<wpe_c> t(WPE_NFFT / 2);
    for (int k = 0; k < WPE_NFFT / 2; ++k) t[k] = wpe_twiddle(k);
    return t;
  }();
  // pageable copies: the call returns once the tables have been staged, so the caller's arrays may go when it returns
  CU_TRY(h, cudaMemcpyAsync(d_twiddles, twiddles.data(), WPE_NFFT / 2 * sizeof(wpe_c), cudaMemcpyHostToDevice, st));
  CU_TRY(h, cudaMemcpyAsync(d_window, window, WPE_NFFT * sizeof(float), cudaMemcpyHostToDevice, st));
  CU_TRY(h, cudaMemcpyAsync(d_cuts, cv.data(), cv.size() * sizeof(WpeCut), cudaMemcpyHostToDevice, st));
  wpe_stft_kernel<<<(unsigned)tiles, WPE_THREADS, WPE_STFT_SMEM, st>>>(d_cuts, ncuts, d_window, d_twiddles);
  CU_TRY(h, cudaGetLastError());
  const WpeParams prm{pm.taps, pm.delay, pm.iterations, pm.statistics_mode == B200FEAT_WPE_VALID};
  wpe_bin_kernel<<<(unsigned)(ncuts * WPE_BINS), WPE_THREADS, WPE_BIN_SMEM(longest), st>>>(d_cuts, prm);
  CU_TRY(h, cudaGetLastError());
  wpe_istft_kernel<<<(unsigned)outs, WPE_THREADS, WPE_ISTFT_SMEM, st>>>(d_cuts, ncuts, d_window, d_twiddles);
  CU_TRY(h, cudaGetLastError());
  return B200FEAT_OK;
}

}  // extern "C"

namespace {

// The SpecAugment work buffer: the tables the kernels read (one copy), then the per-CTA partial sums and the means
struct SaLayout {
  int64_t warp_begin, warps, masks, tables_end, partial, mean, total;
  int64_t tiles;
};

SaLayout sa_layout(int32_t B, int32_t T, int32_t F, int32_t nwarps, int32_t nmasks) {
  auto up = [](int64_t b) { return (b + 255) / 256 * 256; };
  SaLayout l{};
  l.tiles = sa_tiles(T, F);
  l.warp_begin = 0;
  l.warps = l.warp_begin + up(((int64_t)B + 1) * 4);
  l.masks = l.warps + up((int64_t)nwarps * (int64_t)sizeof(SaWarp));
  l.tables_end = l.masks + up((int64_t)nmasks * (int64_t)sizeof(SaMask));
  l.partial = l.tables_end;
  l.mean = l.partial + up((int64_t)B * l.tiles * 8);
  l.total = l.mean + up((int64_t)B * 4);
  return l;
}

bool sa_shape_ok(int32_t B, int32_t T, int32_t F) {
  return B >= 1 && T >= 1 && F >= 1 && (int64_t)T * F <= 0x7fffffff && (int64_t)B * sa_tiles(T, F) <= 0x7fffffff;
}

}  // namespace

extern "C" {

int64_t b200feat_specaug_work_bytes(int32_t B, int32_t T, int32_t F, int32_t nwarps, int32_t nmasks) {
  if (!sa_shape_ok(B, T, F) || nwarps < 0 || nmasks < 0) return 0;
  return sa_layout(B, T, F, nwarps, nmasks).total;
}

int b200feat_specaug(b200feat_handle *h, const float *in_dev, float *out_dev, int32_t B, int32_t T, int32_t F,
                     const b200feat_specaug_warp *warps, int32_t nwarps, const b200feat_specaug_mask *masks, int32_t nmasks,
                     void *work_dev, int64_t work_bytes, void *stream) {
  if (!in_dev || !out_dev || !work_dev || nwarps < 0 || nmasks < 0 || (nwarps > 0 && !warps) || (nmasks > 0 && !masks))
    return fail(h, B200FEAT_EINVAL, "specaug: bad arguments");
  if (!sa_shape_ok(B, T, F)) return fail(h, B200FEAT_EINVAL, "specaug: B, T, F must be positive, T * F and the CTA count below 2^31");
  if (nmasks > 0x7fffffff / 2) return fail(h, B200FEAT_EINVAL, "specaug: too many masks in one call");
  {  // the warp reads rows of `in` that other CTAs have already overwritten in `out` if the two share memory
    const uintptr_t a = (uintptr_t)in_dev, b = (uintptr_t)out_dev, bytes = (uintptr_t)B * T * F * sizeof(float);
    if (a < b + bytes && b < a + bytes) return fail(h, B200FEAT_EINVAL, "specaug: the output overlaps the input");
  }
  const SaLayout l = sa_layout(B, T, F, nwarps, nmasks);
  if (work_bytes < l.total) return fail(h, B200FEAT_EINVAL, "specaug: work buffer too small");
  auto where = [](const char *what, int64_t i) { return std::string("specaug: ") + what + " " + std::to_string(i) + ": "; };
  std::vector<int32_t> order((size_t)nwarps);
  for (int32_t i = 0; i < nwarps; ++i) {
    const b200feat_specaug_warp &w = warps[i];
    if (w.struct_size != (int32_t)sizeof(b200feat_specaug_warp))
      return fail(h, B200FEAT_EINVAL, where("warp", i) + "b200feat_specaug_warp size mismatch (ABI)");
    if (w.seq < 0 || w.seq >= B) return fail(h, B200FEAT_EINVAL, where("warp", i) + "sequence index out of range");
    if (w.start < 0 || w.len < 1 || w.start > T - w.len) return fail(h, B200FEAT_EINVAL, where("warp", i) + "segment outside [0, T)");
    if (w.center < 1 || w.center >= w.len || w.warped < 1 || w.warped >= w.len)
      return fail(h, B200FEAT_EINVAL, where("warp", i) + "center and warped must lie in (0, len)");
    order[i] = i;
  }
  std::sort(order.begin(), order.end(), [&](int32_t a, int32_t b) {
    return warps[a].seq != warps[b].seq ? warps[a].seq < warps[b].seq : warps[a].start != warps[b].start ? warps[a].start < warps[b].start : a < b;
  });
  for (int32_t k = 1; k < nwarps; ++k) {
    const b200feat_specaug_warp &p = warps[order[k - 1]], &w = warps[order[k]];
    if (p.seq == w.seq && w.start < p.start + p.len)
      return fail(h, B200FEAT_EINVAL, where("warp", order[k]) + "overlaps another segment of its sequence");
  }
  for (int32_t i = 0; i < nmasks; ++i) {
    const b200feat_specaug_mask &m = masks[i];
    if (m.struct_size != (int32_t)sizeof(b200feat_specaug_mask))
      return fail(h, B200FEAT_EINVAL, where("mask", i) + "b200feat_specaug_mask size mismatch (ABI)");
    if (m.seq < 0 || m.seq >= B) return fail(h, B200FEAT_EINVAL, where("mask", i) + "sequence index out of range");
    if (m.axis != B200FEAT_SPECAUG_TIME && m.axis != B200FEAT_SPECAUG_FEATURE) return fail(h, B200FEAT_EINVAL, where("mask", i) + "bad axis");
    if (m.start < 0 || m.start > m.end || m.end > (m.axis == B200FEAT_SPECAUG_TIME ? T : F))
      return fail(h, B200FEAT_EINVAL, where("mask", i) + "rectangle outside its axis");
  }
  // the kernels' tables in one host block: segments per sequence sorted by start, rectangles as they came
  std::vector<char> tables((size_t)l.tables_end, 0);
  int32_t *warp_begin = (int32_t *)(tables.data() + l.warp_begin);
  SaWarp *sw = (SaWarp *)(tables.data() + l.warps);
  SaMask *sm = (SaMask *)(tables.data() + l.masks);
  for (int32_t k = 0; k < nwarps; ++k) {
    const b200feat_specaug_warp &w = warps[order[k]];
    sw[k] = SaWarp{w.start, w.len, w.center, w.warped};
    ++warp_begin[w.seq + 1];
  }
  for (int32_t b = 0; b < B; ++b) warp_begin[b + 1] += warp_begin[b];
  int64_t largest = 0;
  for (int32_t i = 0; i < nmasks; ++i) {
    sm[i] = SaMask{masks[i].seq, masks[i].axis, masks[i].start, masks[i].end};
    largest = std::max<int64_t>(largest, sa_mask_elems(sm[i], T, F));
  }
  char *w = (char *)work_dev;
  const cudaStream_t st = (cudaStream_t)stream;
  double *d_partial = (double *)(w + l.partial);
  float *d_mean = (float *)(w + l.mean);
  // a pageable copy: the call returns once the block has been staged, so it may go when this function returns
  CU_TRY(h, cudaMemcpyAsync(w, tables.data(), tables.size(), cudaMemcpyHostToDevice, st));
  const unsigned ctas = (unsigned)((int64_t)B * l.tiles);
  // 128-bit accesses need whole rows of float4 at 16-byte addresses
  if (F % 4 == 0 && (uintptr_t)in_dev % 16 == 0 && (uintptr_t)out_dev % 16 == 0)
    specaug_warp_kernel<4><<<ctas, SA_THREADS, 0, st>>>(in_dev, out_dev, T, F, (int)l.tiles, (const SaWarp *)(w + l.warps),
                                                        (const int32_t *)(w + l.warp_begin), d_partial);
  else
    specaug_warp_kernel<1><<<ctas, SA_THREADS, 0, st>>>(in_dev, out_dev, T, F, (int)l.tiles, (const SaWarp *)(w + l.warps),
                                                        (const int32_t *)(w + l.warp_begin), d_partial);
  CU_TRY(h, cudaGetLastError());
  if (nmasks == 0) return B200FEAT_OK;
  specaug_mean_kernel<<<(unsigned)((B + 127) / 128), 128, 0, st>>>(d_partial, B, (int)l.tiles, (int64_t)T * F, d_mean);
  CU_TRY(h, cudaGetLastError());
  const int64_t gy = std::min<int64_t>(std::max<int64_t>((largest + 8 * SA_FILL_THREADS - 1) / (8 * SA_FILL_THREADS), 1), 64);
  specaug_fill_kernel<<<dim3((unsigned)nmasks, (unsigned)gy), SA_FILL_THREADS, 0, st>>>(out_dev, T, F, (const SaMask *)(w + l.masks), d_mean);
  CU_TRY(h, cudaGetLastError());
  return B200FEAT_OK;
}

int64_t b200feat_feature_mix_work_bytes(int32_t ntracks, int32_t ncuts) {
  if (ntracks < 0 || ncuts < 0) return 0;
  auto up = [](int64_t b) { return (b + 255) / 256 * 256; };
  return up((int64_t)ntracks * (int64_t)sizeof(b200feat_featmix_track)) + up((int64_t)ncuts * (int64_t)sizeof(b200feat_featmix_cut)) +
         up((int64_t)ntracks * FM_PARTS * 8) + up((int64_t)ntracks * 8);
}

int b200feat_feature_mix(b200feat_handle *h, const float *src_dev, int64_t src_elems, const b200feat_featmix_track *tracks,
                         int32_t ntracks, const b200feat_featmix_cut *cuts, int32_t ncuts, int32_t F, float *out_dev,
                         int32_t T_max, float pad_value, void *work_dev, int64_t work_bytes, void *stream) {
  if (ntracks < 0 || ncuts < 0 || F < 1 || T_max < 0 || src_elems < 0 || (ncuts > 0 && (!cuts || !out_dev || !work_dev)) ||
      (ntracks > 0 && !tracks))
    return fail(h, B200FEAT_EINVAL, "feature_mix: bad arguments");
  if (ncuts == 0 || T_max == 0) return B200FEAT_OK;
  if ((int64_t)ntracks * FM_PARTS > 0x7fffffff) return fail(h, B200FEAT_EINVAL, "feature_mix: too many tracks in one call");
  const int64_t tiles = ((int64_t)T_max * F + FM_TILE - 1) / FM_TILE;
  if (tiles > 0x7fffffff) return fail(h, B200FEAT_EINVAL, "feature_mix: T_max * F too large");
  if (work_bytes < b200feat_feature_mix_work_bytes(ntracks, ncuts)) return fail(h, B200FEAT_EINVAL, "feature_mix: work buffer too small");
  auto where = [](const char *what, int64_t i) { return std::string("feature_mix: ") + what + " " + std::to_string(i) + ": "; };
  for (int32_t t = 0; t < ntracks; ++t) {
    const b200feat_featmix_track &tr = tracks[t];
    if (tr.struct_size != (int32_t)sizeof(b200feat_featmix_track))
      return fail(h, B200FEAT_EINVAL, where("track", t) + "b200feat_featmix_track size mismatch (ABI)");
    if (tr.cut < 0 || tr.cut >= ncuts) return fail(h, B200FEAT_EINVAL, where("track", t) + "cut index out of range");
    if (tr.flags & ~(B200FEAT_FEATMIX_MIXED | B200FEAT_FEATMIX_ENERGY)) return fail(h, B200FEAT_EINVAL, where("track", t) + "bad flags");
    if (tr.num_rows < 0 || tr.offset < 0 || tr.stored_rows < 0 ||
        (tr.stored_rows > 0 && tr.stored_rows != tr.num_rows && tr.stored_rows != tr.num_rows - 1))
      return fail(h, B200FEAT_EINVAL, where("track", t) + "bad row counts or offset (stored_rows is num_rows or num_rows - 1)");
    if (tr.stored_rows > 0 && (!src_dev || tr.src_elem < 0 || tr.src_elem > src_elems - (int64_t)tr.stored_rows * F))
      return fail(h, B200FEAT_EINVAL, where("track", t) + "rows outside the source buffer");
  }
  for (int32_t c = 0; c < ncuts; ++c) {
    const b200feat_featmix_cut &cu = cuts[c];
    if (cu.struct_size != (int32_t)sizeof(b200feat_featmix_cut))
      return fail(h, B200FEAT_EINVAL, where("cut", c) + "b200feat_featmix_cut size mismatch (ABI)");
    if (cu.mode != B200FEAT_FEATMIX_COPY && cu.mode != B200FEAT_FEATMIX_MIX) return fail(h, B200FEAT_EINVAL, where("cut", c) + "bad mode");
    if (cu.num_tracks < 1 || cu.first_track < 0 || (int64_t)cu.first_track + cu.num_tracks > ntracks)
      return fail(h, B200FEAT_EINVAL, where("cut", c) + "tracks outside the track table");
    if (cu.num_rows < 0 || cu.num_rows > T_max) return fail(h, B200FEAT_EINVAL, where("cut", c) + "num_rows outside [0, T_max]");
    for (int32_t k = 0; k < cu.num_tracks; ++k)
      if (tracks[cu.first_track + k].cut != c) return fail(h, B200FEAT_EINVAL, where("cut", c) + "a track of another cut inside its range");
    const b200feat_featmix_track &b = tracks[cu.first_track];
    if (!(b.flags & B200FEAT_FEATMIX_MIXED) || b.offset != 0)
      return fail(h, B200FEAT_EINVAL, where("cut", c) + "the first track must be mixed, at offset 0");
    if (cu.mode == B200FEAT_FEATMIX_COPY) {
      if (cu.num_tracks != 1 || b.num_rows > cu.num_rows) return fail(h, B200FEAT_EINVAL, where("cut", c) + "a copy is one track of at most num_rows rows");
      continue;
    }
    if (cu.law != B200FEAT_FEATMIX_LOG && cu.law != B200FEAT_FEATMIX_LINEAR) return fail(h, B200FEAT_EINVAL, where("cut", c) + "bad law");
    if (cu.ref_track < 0 || cu.ref_track >= cu.num_tracks) return fail(h, B200FEAT_EINVAL, where("cut", c) + "reference index outside the cut's tracks");
    if (!(tracks[cu.first_track + cu.ref_track].flags & B200FEAT_FEATMIX_ENERGY))
      return fail(h, B200FEAT_EINVAL, where("cut", c) + "the reference track needs the energy flag");
    int64_t rows = b.num_rows;
    for (int32_t k = 0; k < cu.num_tracks; ++k) {
      const b200feat_featmix_track &tr = tracks[cu.first_track + k];
      if (!(tr.flags & B200FEAT_FEATMIX_MIXED)) continue;
      if (tr.snr_factor == tr.snr_factor && (k > 0 || cu.ref_track != 0) && !(tr.flags & B200FEAT_FEATMIX_ENERGY))
        return fail(h, B200FEAT_EINVAL, where("cut", c) + "a mixed track with an SNR needs the energy flag");
      if (k == 0) continue;
      if (tr.num_rows < 1) return fail(h, B200FEAT_EINVAL, where("cut", c) + "a further mixed track without rows (the mixer skips those)");
      rows = std::max(rows, (int64_t)tr.offset + tr.num_rows);
    }
    if (rows != cu.mix_rows) return fail(h, B200FEAT_EINVAL, where("cut", c) + "mix_rows is not the end of its mixed tracks");
    if (cu.num_rows > 0 && (cu.mix_rows < 1 || cu.mix_rows < (int64_t)cu.num_rows - 1 || cu.mix_rows > (int64_t)cu.num_rows + 1))
      return fail(h, B200FEAT_EINVAL, where("cut", c) + "mix_rows more than one row away from num_rows");
  }
  auto up = [](int64_t b) { return (b + 255) / 256 * 256; };
  char *w = (char *)work_dev;
  b200feat_featmix_track *d_tracks = (b200feat_featmix_track *)w;
  w += up((int64_t)ntracks * (int64_t)sizeof(b200feat_featmix_track));
  b200feat_featmix_cut *d_cuts = (b200feat_featmix_cut *)w;
  w += up((int64_t)ncuts * (int64_t)sizeof(b200feat_featmix_cut));
  double *partial = (double *)w;
  w += up((int64_t)ntracks * FM_PARTS * 8);
  double *gain = (double *)w;
  const cudaStream_t st = (cudaStream_t)stream;
  // pageable copies: each returns once its table has been staged, so the tables may go when this function returns
  CU_TRY(h, cudaMemcpyAsync(d_tracks, tracks, (size_t)ntracks * sizeof(b200feat_featmix_track), cudaMemcpyHostToDevice, st));
  CU_TRY(h, cudaMemcpyAsync(d_cuts, cuts, (size_t)ncuts * sizeof(b200feat_featmix_cut), cudaMemcpyHostToDevice, st));
  if (ntracks) {
    featmix_energy_kernel<<<(unsigned)(ntracks * FM_PARTS), FM_THREADS, 0, st>>>(src_dev, d_tracks, d_cuts, F, partial);
    CU_TRY(h, cudaGetLastError());
  }
  featmix_gain_kernel<<<(unsigned)((ncuts + FM_GAIN_THREADS - 1) / FM_GAIN_THREADS), FM_GAIN_THREADS, 0, st>>>(d_tracks, d_cuts, ncuts,
                                                                                                               partial, gain);
  CU_TRY(h, cudaGetLastError());
  featmix_out_kernel<<<dim3((unsigned)tiles, (unsigned)std::min(ncuts, 65535)), FM_THREADS, 0, st>>>(src_dev, d_tracks, d_cuts, ncuts, gain,
                                                                                                     F, T_max, pad_value, out_dev);
  CU_TRY(h, cudaGetLastError());
  return B200FEAT_OK;
}

int64_t b200feat_collate_audio_work_bytes(int32_t B) { return B < 0 ? 0 : (int64_t)B * 2 * (int64_t)sizeof(int64_t); }

int b200feat_collate_audio(b200feat_handle *h, const void *src_dev, int32_t dt, int64_t src_elems, const int64_t *offsets,
                           const int64_t *lens, int32_t B, int64_t T, float *out_dev, void *work_dev, int64_t work_bytes,
                           void *stream) {
  if (dt != B200FEAT_F32 && dt != B200FEAT_I16) return fail(h, B200FEAT_EINVAL, "collate_audio: unknown dtype " + std::to_string(dt));
  if (B < 0 || T < 0 || src_elems < 0) return fail(h, B200FEAT_EINVAL, "collate_audio: negative B, T or source size");
  if (B > 0 && (!offsets || !lens)) return fail(h, B200FEAT_EINVAL, "collate_audio: missing offset or length table");
  auto where = [](int64_t b) { return std::string("collate_audio: cut ") + std::to_string(b) + ": "; };
  for (int32_t b = 0; b < B; ++b) {
    if (offsets[b] < 0) return fail(h, B200FEAT_EINVAL, where(b) + "negative offset " + std::to_string(offsets[b]));
    if (lens[b] < 0) return fail(h, B200FEAT_EINVAL, where(b) + "negative length " + std::to_string(lens[b]));
    if (lens[b] > T)
      return fail(h, B200FEAT_EINVAL, where(b) + "length " + std::to_string(lens[b]) + " above T = " + std::to_string(T));
    if (offsets[b] > src_elems - lens[b])
      return fail(h, B200FEAT_EINVAL, where(b) + "samples [" + std::to_string(offsets[b]) + ", " + std::to_string(offsets[b] + lens[b]) +
                                           ") outside the source buffer of " + std::to_string(src_elems) + " elements");
  }
  if (B == 0 || T == 0) return B200FEAT_OK;
  if (!out_dev || !work_dev) return fail(h, B200FEAT_EINVAL, "collate_audio: missing output or work buffer");
  if (src_elems > 0 && !src_dev) return fail(h, B200FEAT_EINVAL, "collate_audio: missing source buffer");
  if ((uintptr_t)src_dev % (dt == B200FEAT_F32 ? 16 : 8))
    return fail(h, B200FEAT_EINVAL, "collate_audio: source buffer not 16-byte (float32) / 8-byte (int16) aligned");
  if ((uintptr_t)out_dev % 4) return fail(h, B200FEAT_EINVAL, "collate_audio: output not 4-byte aligned");
  if (work_bytes < b200feat_collate_audio_work_bytes(B)) return fail(h, B200FEAT_EINVAL, "collate_audio: work buffer too small");
  // the units of the longest row (the head and tail units of every row included) over CTAs of CO_THREADS * CO_UNITS_PER_THREAD
  const int64_t tiles = (co_units(T / 4) + CO_THREADS * CO_UNITS_PER_THREAD - 1) / (CO_THREADS * CO_UNITS_PER_THREAD);
  if (tiles > 0x7fffffff) return fail(h, B200FEAT_EINVAL, "collate_audio: T too large");
  std::vector<int64_t> tab((size_t)B * 2);
  std::copy(offsets, offsets + B, tab.begin());
  std::copy(lens, lens + B, tab.begin() + B);
  const cudaStream_t st = (cudaStream_t)stream;
  // a pageable copy: it returns once the table has been staged, so the table may go when this function returns
  CU_TRY(h, cudaMemcpyAsync(work_dev, tab.data(), tab.size() * sizeof(int64_t), cudaMemcpyHostToDevice, st));
  const dim3 grid((unsigned)tiles, (unsigned)std::min(B, 65535));
  const int base_mod4 = (int)(((uintptr_t)out_dev / 4) % 4);
  if (dt == B200FEAT_F32)
    collate_audio_kernel<float><<<grid, CO_THREADS, 0, st>>>((const float *)src_dev, (const int64_t *)work_dev, B, T, base_mod4, out_dev);
  else
    collate_audio_kernel<int16_t><<<grid, CO_THREADS, 0, st>>>((const int16_t *)src_dev, (const int64_t *)work_dev, B, T, base_mod4, out_dev);
  CU_TRY(h, cudaGetLastError());
  return B200FEAT_OK;
}

}  // extern "C"

namespace {

// The generator's work buffer: the kernels' RIR table, the resampler table, the segment offsets, the entries before and after
// the sort, the sort's own scratch
struct RgLayout {
  int64_t rirs, table, offsets, pos_in, val_in, pos_out, val_out, temp, temp_bytes, total;
  int64_t entries;
  int end_bit;
};

// Whether every image ratio of the record is positive: rg_room's lin_end, the last one, computed by the same code.  With
// lin_end <= 0 (d0 >= 340 T60) some distances would be <= 0 and their comb positions negative, which the sort (keys of end_bit
// bits) and the window's table lookup do not take.
bool rg_ratios_ok(const b200feat_rir_gen &g) {
  RgRir r{};
  r.t60 = g.t60;
  r.d0 = g.d0;
  return rg_room(r).lin_end > 0.0f;
}

// Whether the record is one b200feat_rir_generate takes (the buffer bounds are checked by the call)
bool rg_record_ok(const b200feat_rir_gen &g) {
  return g.struct_size == (int32_t)sizeof(b200feat_rir_gen) && g.sampling_rate >= 1 && g.sampling_rate <= 192000 &&
         g.t60 > 0.0 && g.d0 > 0.0 && isfinite(g.t60) && isfinite(g.r) && isfinite(g.d0) && isfinite(g.tau) &&
         g.comb_len >= 1 && g.comb_len <= 0x7fffffff && g.out_len >= 1 && g.out_len <= g.comb_len / RG_O + 1 &&
         rg_ratios_ok(g);
}

// false when a record is malformed or the entries do not fit the sort's int offsets
bool rg_layout(const b200feat_rir_gen *rirs, int32_t n, RgLayout *l) {
  auto up = [](int64_t b) { return (b + 255) / 256 * 256; };
  *l = RgLayout{};
  int64_t longest = 1;
  for (int32_t i = 0; i < n; ++i) {
    if (!rg_record_ok(rirs[i])) return false;
    l->entries += 2 * (int64_t)rirs[i].sampling_rate + 1;
    longest = std::max(longest, rirs[i].comb_len);
  }
  if (l->entries > 0x7fffffff) return false;
  l->end_bit = 1;
  while (l->end_bit < 31 && ((int64_t)1 << l->end_bit) < longest) ++l->end_bit;
  size_t temp = 0;
  if (n > 0 && cub::DeviceSegmentedRadixSort::SortPairs(nullptr, temp, (const int32_t *)nullptr, (int32_t *)nullptr,
                                                        (const float *)nullptr, (float *)nullptr, (int)l->entries, n,
                                                        (const int *)nullptr, (const int *)nullptr + 1, 0, l->end_bit) != cudaSuccess)
    return false;
  l->temp_bytes = (int64_t)temp;
  l->rirs = 0;
  l->table = l->rirs + up((int64_t)n * (int64_t)sizeof(RgRir));
  l->offsets = l->table + up(RG_TAPS * 4);
  l->pos_in = l->offsets + up(((int64_t)n + 1) * 4);
  l->val_in = l->pos_in + up(l->entries * 4);
  l->pos_out = l->val_in + up(l->entries * 4);
  l->val_out = l->pos_out + up(l->entries * 4);
  l->temp = l->val_out + up(l->entries * 4);
  l->total = l->temp + up(std::max<int64_t>(l->temp_bytes, 1));
  return true;
}

}  // namespace

extern "C" {

int64_t b200feat_rir_generate_work_bytes(const b200feat_rir_gen *rirs, int32_t nrirs) {
  RgLayout l;
  if (nrirs < 0 || (nrirs > 0 && !rirs) || !rg_layout(rirs, nrirs, &l)) return 0;
  return l.total;
}

int b200feat_rir_generate(b200feat_handle *h, const double *draws_dev, int64_t draws_elems, const float *cdf_dev,
                          int64_t cdf_elems, const float *table, const b200feat_rir_gen *rirs, int32_t nrirs, float *out_dev,
                          int64_t out_elems, void *work_dev, int64_t work_bytes, void *stream) {
  if (nrirs < 0 || (nrirs > 0 && (!rirs || !draws_dev || !cdf_dev || !table || !out_dev || !work_dev)) || draws_elems < 0 ||
      cdf_elems < 0 || out_elems < 0)
    return fail(h, B200FEAT_EINVAL, "rir_generate: bad arguments");
  if (nrirs == 0) return B200FEAT_OK;
  auto where = [](int64_t i) { return std::string("rir_generate: rir ") + std::to_string(i) + ": "; };
  std::vector<std::pair<int64_t, int64_t>> outs((size_t)nrirs);
  for (int32_t i = 0; i < nrirs; ++i) {
    const b200feat_rir_gen &g = rirs[i];
    if (g.struct_size != (int32_t)sizeof(b200feat_rir_gen))
      return fail(h, B200FEAT_EINVAL, where(i) + "b200feat_rir_gen size mismatch (ABI)");
    if (g.t60 > 0.0 && g.d0 > 0.0 && isfinite(g.t60) && isfinite(g.d0) && !rg_ratios_ok(g))
      return fail(h, B200FEAT_EINVAL, where(i) + "d0 must be below 340 T60 (its last image ratio 340 T60 / d0 - 1 is not "
                                                 "positive)");
    if (!rg_record_ok(g))
      return fail(h, B200FEAT_EINVAL, where(i) + "bad sampling rate, draws or lengths (T60 and d0 must be positive, "
                                                 "out_len at most comb_len / 8 + 1)");
    const int64_t images = 2 * (int64_t)g.sampling_rate;
    if (g.cdf_elem < 0 || g.cdf_elem > cdf_elems - images)
      return fail(h, B200FEAT_EINVAL, where(i) + "distribution outside the cdf buffer");
    if (g.draw_elem < 0 || g.draw_elem > draws_elems - 2 * images)
      return fail(h, B200FEAT_EINVAL, where(i) + "draws outside the draws buffer");
    if (g.out_elem < 0 || g.out_elem > out_elems - g.out_len)
      return fail(h, B200FEAT_EINVAL, where(i) + "output outside the output buffer");
    outs[i] = {g.out_elem, g.out_elem + g.out_len};
  }
  std::sort(outs.begin(), outs.end());
  for (int32_t i = 1; i < nrirs; ++i)
    if (outs[i].first < outs[i - 1].second) return fail(h, B200FEAT_EINVAL, "rir_generate: two outputs overlap");
  RgLayout l;
  if (!rg_layout(rirs, nrirs, &l)) return fail(h, B200FEAT_EINVAL, "rir_generate: more than 2^31 - 1 entries in one call");
  if (work_bytes < l.total) return fail(h, B200FEAT_EINVAL, "rir_generate: work buffer too small");
  char *w = (char *)work_dev;
  std::vector<RgRir> rg((size_t)nrirs);
  std::vector<int32_t> offsets((size_t)nrirs + 1);
  int64_t entries = 0, ctas = 0;
  for (int32_t i = 0; i < nrirs; ++i) {
    const b200feat_rir_gen &g = rirs[i];
    const int32_t images = 2 * g.sampling_rate;
    rg[i] = RgRir{draws_dev + g.draw_elem, draws_dev + g.draw_elem + images, cdf_dev + g.cdf_elem, out_dev + g.out_elem,
                  g.t60, g.r, g.d0, g.tau, g.comb_len, g.out_len, entries, ctas, g.sampling_rate, images,
                  g.b0, g.b1, g.b2, g.a1, g.a2};
    offsets[i] = (int32_t)entries;
    entries += images + 1;
    ctas += (g.out_len + RG_THREADS - 1) / RG_THREADS;
  }
  offsets[nrirs] = (int32_t)entries;
  if (ctas > 0x7fffffff) return fail(h, B200FEAT_EINVAL, "rir_generate: too many CTAs in one call");
  const cudaStream_t st = (cudaStream_t)stream;
  RgRir *d_rirs = (RgRir *)(w + l.rirs);
  float *d_table = (float *)(w + l.table);
  int32_t *d_offsets = (int32_t *)(w + l.offsets);
  int32_t *pos_in = (int32_t *)(w + l.pos_in), *pos_out = (int32_t *)(w + l.pos_out);
  float *val_in = (float *)(w + l.val_in), *val_out = (float *)(w + l.val_out);
  // pageable copies: the call returns once the tables have been staged, so the vectors may go when this function returns
  CU_TRY(h, cudaMemcpyAsync(d_rirs, rg.data(), rg.size() * sizeof(RgRir), cudaMemcpyHostToDevice, st));
  CU_TRY(h, cudaMemcpyAsync(d_table, table, RG_TAPS * sizeof(float), cudaMemcpyHostToDevice, st));
  CU_TRY(h, cudaMemcpyAsync(d_offsets, offsets.data(), offsets.size() * sizeof(int32_t), cudaMemcpyHostToDevice, st));
  rirgen_entry_kernel<<<(unsigned)((entries + RG_THREADS - 1) / RG_THREADS), RG_THREADS, 0, st>>>(d_rirs, nrirs, entries,
                                                                                                 pos_in, val_in);
  CU_TRY(h, cudaGetLastError());
  size_t temp = (size_t)l.temp_bytes;
  // a stable sort: entries that share a position keep their entry order, so the window kernel can keep the last one
  CU_TRY(h, cub::DeviceSegmentedRadixSort::SortPairs(w + l.temp, temp, pos_in, pos_out, val_in, val_out, (int)entries, nrirs,
                                                     d_offsets, d_offsets + 1, 0, l.end_bit, st));
  if (ctas > 0) {
    rirgen_window_kernel<<<(unsigned)ctas, RG_THREADS, 0, st>>>(d_rirs, nrirs, pos_out, val_out, d_table);
    CU_TRY(h, cudaGetLastError());
  }
  rirgen_biquad_kernel<<<(unsigned)((nrirs + 31) / 32), 32, 0, st>>>(d_rirs, nrirs);
  CU_TRY(h, cudaGetLastError());
  return B200FEAT_OK;
}

}  // extern "C"

namespace {

// The backward's view of the handle's plan; false for a plan without a backward (log10-fbank).  whisper-fbank has one
// through b200feat_whisper_backward only, which asks for it with `whisper`.
bool bwd_plan(const b200feat_handle *h, BwdPlan *out, bool whisper = false) {
  const DevPlan &p = h->plan;
  const int f = p.feature;
  if (whisper != (p.whisper != 0)) return false;
  if (!whisper && ((f != B200FEAT_FBANK && f != B200FEAT_MFCC && f != B200FEAT_SPECTROGRAM && f != B200FEAT_LOG_SPECTROGRAM) ||
                   p.log10_mel || p.pad_mode != B200FEAT_PAD_KALDI))
    return false;
  BwdPlan b;
  memset(&b, 0, sizeof(b));
  b.feature = f; b.L = p.L; b.S = p.S; b.N = p.N; b.K = p.K; b.M = p.M; b.C = p.C; b.F = p.F; b.Nc = p.Nc; b.packed = p.packed;
  b.pad = p.pad_left; b.snip_edges = p.snip_edges; b.remove_dc = p.remove_dc; b.use_energy = p.use_energy;
  b.raw_energy = p.raw_energy; b.use_mag = p.use_mag; b.energy_style = p.energy_style; b.use_lifter = p.use_lifter;
  b.ecol = p.energy_last ? p.F - 1 : 0;
  b.shift = (f == B200FEAT_FBANK && p.use_energy && !p.energy_last) ? 1 : 0;
  b.preemph = p.preemph; b.energy_floor_log = p.energy_floor_log; b.has_energy_floor = p.has_energy_floor;
  b.mel_floor = p.mel_floor; b.log_spec_eps = p.log_spec_eps; b.log_spec_floor = p.log_spec_floor;
  b.window = p.window; b.tws = reinterpret_cast<const BwdC *>(p.tws);
  b.mel_start = p.mel_start; b.mel_len = p.mel_len; b.mel_woff = p.mel_woff; b.mel_w = p.mel_w;
  b.dct = p.dct; b.lifter = p.lifter; b.post_scale = p.post_scale;
  b.whisper = p.whisper; b.reflect = p.pad_mode == B200FEAT_PAD_CENTER ? 1 : 0;
  *out = b;
  return true;
}

// Tiles of every cut (tile_off, B + 1 entries) and the work buffer size; a negative code for a cut too short to be framed
int64_t bwd_layout(b200feat_handle *h, const BwdPlan &p, int ft, const int64_t *num_samples, int32_t B,
                   std::vector<int64_t> *tile_off) {
  int64_t tiles = 0;
  if (tile_off) tile_off->assign((size_t)B + 1, 0);
  for (int i = 0; i < B; ++i) {
    const int64_t T = cut_frames(h, i, num_samples[i]);
    if (T < 0) return T;
    const int64_t frames = bwd_frames(p, num_samples[i], T);
    tiles += (frames + ft - 1) / ft;
    if (tile_off) (*tile_off)[i + 1] = tiles;
  }
  return bwd_meta_bytes(B) + bwd_reduce_bytes(p, B) + tiles * bwd_span(p, ft) * (int64_t)sizeof(float);
}

// The refusal of a frame whose backward does not fit shared memory, with the numbers that decide it
std::string bwd_too_long(const BwdPlan &p) {
  return "backward: frame too long for shared memory: L = " + std::to_string(p.L) + ", N = " + std::to_string(p.N) + " needs " +
         std::to_string(bwd_smem(p, 1, 1)) + " bytes for one warp and one frame, over the backward's limit of " +
         std::to_string(BWD_SMEM_LIMIT) + " bytes (at 16 kHz, N = 8192 with frames up to about 0.4 s is the largest supported)";
}

// b200feat_backward / b200feat_whisper_backward after their kind checks: the argument and per-cut checks, the tables, and
// the launches (whisper-fbank: the per-cut reduction, then the frames and combine kernels of every kind)
int run_backward(b200feat_handle *h, const float *samples_dev, int32_t dt, const int64_t *num_samples, const int64_t *offsets,
                 int32_t B, const float *grad_out_dev, const float *raw_dev, const float *cut_max_dev, const int64_t *row_off,
                 float *grad_in_dev, void *work_dev, int64_t work_bytes, void *stream) {
  if (!samples_dev || !num_samples || !offsets || B <= 0 || !grad_out_dev || !row_off || !grad_in_dev || !work_dev)
    return fail(h, B200FEAT_EINVAL, "backward: bad arguments");
  if (dt != B200FEAT_F32) return fail(h, B200FEAT_EINVAL, "backward: float32 samples only");
  BwdPlan p;
  if (!bwd_plan(h, &p, raw_dev != nullptr))
    return fail(h, B200FEAT_EINVAL, "backward: only the fbank, mfcc, spectrogram, log-spectrogram and whisper-fbank kinds have one");
  int warps, ft;
  if (!bwd_launch_shape(p, &warps, &ft)) return fail(h, B200FEAT_EUNSUPPORTED, bwd_too_long(p));
  std::vector<int64_t> tile_off;
  const int64_t need = bwd_layout(h, p, ft, num_samples, B, &tile_off);
  if (need < 0) return (int)need;
  if (work_bytes < need) return fail(h, B200FEAT_EINVAL, "backward: work buffer too small");
  if (row_off[0] != 0) return fail(h, B200FEAT_EINVAL, "backward: row_off[0] must be 0");
  for (int i = 0; i < B; ++i) {
    if (offsets[i] < 0 || num_samples[i] < 0) return fail(h, B200FEAT_EINVAL, "backward: negative offset or length");
    if (row_off[i + 1] - row_off[i] != frames_for(h->desc, num_samples[i]))
      return fail(h, B200FEAT_EINVAL, "backward: row_off does not match cut " + std::to_string(i) + "'s frame count");
  }
  // the int64 tables in one host block: samp_off, nsamp, row_off, tile_off
  std::vector<int64_t> meta(4 * (size_t)B + 2);
  std::copy(offsets, offsets + B, meta.begin());
  std::copy(num_samples, num_samples + B, meta.begin() + B);
  std::copy(row_off, row_off + B + 1, meta.begin() + 2 * (size_t)B);
  std::copy(tile_off.begin(), tile_off.end(), meta.begin() + 3 * (size_t)B + 1);
  DeviceGuard on(h->device);
  const cudaStream_t st = (cudaStream_t)stream;
  unsigned char *w = (unsigned char *)work_dev;
  // a pageable copy: the call returns once the block has been staged, so the vector may go when this function returns
  CU_TRY(h, cudaMemcpyAsync(w, meta.data(), meta.size() * sizeof(int64_t), cudaMemcpyHostToDevice, st));
  const int64_t *dm = (const int64_t *)w;
  BwdBatch bb;
  memset(&bb, 0, sizeof(bb));
  bb.samples = samples_dev; bb.grad_out = grad_out_dev; bb.grad_in = grad_in_dev;
  bb.samp_off = dm; bb.nsamp = dm + B; bb.row_off = dm + 2 * (int64_t)B; bb.tile_off = dm + 3 * (int64_t)B + 1;
  bb.spans = (float *)(w + bwd_meta_bytes(B) + bwd_reduce_bytes(p, B));
  bb.B = B; bb.ft = ft;
  if (p.whisper) {
    bb.xrows = raw_dev; bb.cut_max = cut_max_dev;
    bb.routed = (float *)(w + bwd_meta_bytes(B));
    bb.ties = (int *)(bb.routed + B);
    const unsigned grid = (unsigned)std::min<int64_t>(B, (int64_t)h->sm_count * 8);
    b200feat_whisper_backward_reduce_kernel<<<grid, BWD_REDUCE_THREADS, 0, st>>>(p, bb);
    CU_TRY(h, cudaGetLastError());
  }
  const int64_t ntiles = tile_off[B];
  if (ntiles > 0) {
    const size_t smem = bwd_smem(p, warps, ft);
    CU_TRY(h, cudaFuncSetAttribute(b200feat_backward_frames_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    const unsigned grid = (unsigned)std::min<int64_t>(ntiles, (int64_t)h->sm_count * 64);
    b200feat_backward_frames_kernel<<<grid, warps * 32, smem, st>>>(p, h->plan, bb, ntiles);
    CU_TRY(h, cudaGetLastError());
  }
  int64_t nmax = 0;
  for (int i = 0; i < B; ++i) nmax = std::max(nmax, num_samples[i]);
  if (nmax > 0) {
    const int64_t gx = std::min<int64_t>((nmax + BWD_COMBINE_THREADS - 1) / BWD_COMBINE_THREADS, 4096);
    const dim3 grid((unsigned)gx, (unsigned)std::min<int32_t>(B, 65535));
    b200feat_backward_combine_kernel<<<grid, BWD_COMBINE_THREADS, 0, st>>>(p, bb);
    CU_TRY(h, cudaGetLastError());
  }
  return B200FEAT_OK;
}

}  // namespace

extern "C" {

int64_t b200feat_backward_work_bytes(b200feat_handle *h, const int64_t *num_samples, int32_t B) {
  if (!h || !num_samples || B <= 0) return fail(h, B200FEAT_EINVAL, "backward_work_bytes: bad arguments");
  BwdPlan p;
  if (!bwd_plan(h, &p, h->plan.whisper != 0))
    return fail(h, B200FEAT_EINVAL, "backward: only the fbank, mfcc, spectrogram, log-spectrogram and whisper-fbank kinds have one");
  int warps, ft;
  if (!bwd_launch_shape(p, &warps, &ft)) return fail(h, B200FEAT_EUNSUPPORTED, bwd_too_long(p));
  return bwd_layout(h, p, ft, num_samples, B, nullptr);
}

int b200feat_backward(b200feat_handle *h, const float *samples_dev, int32_t dt, const int64_t *num_samples, const int64_t *offsets,
                      int32_t B, const float *grad_out_dev, const int64_t *row_off, float *grad_in_dev, void *work_dev,
                      int64_t work_bytes, void *stream) {
  if (!h) return fail(nullptr, B200FEAT_EINVAL, "backward: null handle");
  if (h->plan.whisper)
    return fail(h, B200FEAT_EINVAL, "backward: whisper-fbank's backward needs the forward's log-mel rows: use b200feat_whisper_backward");
  return run_backward(h, samples_dev, dt, num_samples, offsets, B, grad_out_dev, nullptr, nullptr, row_off, grad_in_dev, work_dev,
                      work_bytes, stream);
}

int b200feat_whisper_backward(b200feat_handle *h, const float *samples_dev, int32_t dt, const int64_t *num_samples,
                              const int64_t *offsets, int32_t B, const float *grad_out_dev, const float *raw_dev,
                              const float *cut_max_dev, const int64_t *row_off, float *grad_in_dev, void *work_dev,
                              int64_t work_bytes, void *stream) {
  if (!h) return fail(nullptr, B200FEAT_EINVAL, "whisper_backward: null handle");
  if (!h->plan.whisper) return fail(h, B200FEAT_EINVAL, "whisper_backward: whisper-fbank handles only (b200feat_backward serves the others)");
  if (!raw_dev || !cut_max_dev) return fail(h, B200FEAT_EINVAL, "whisper_backward: bad arguments");
  return run_backward(h, samples_dev, dt, num_samples, offsets, B, grad_out_dev, raw_dev, cut_max_dev, row_off, grad_in_dev,
                      work_dev, work_bytes, stream);
}

}  // extern "C"
