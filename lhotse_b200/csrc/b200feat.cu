// b200feat — host side of the C ABI (include/b200feat.h) + kernel dispatch.  sm_90a only.
#include <cuda_runtime.h>
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <immintrin.h>

#include <atomic>
#include <condition_variable>
#include <functional>
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

namespace {

thread_local std::string g_error;

struct HostRing {  // grow-only staging for b200feat_extract_host
  void *d_samples = nullptr; size_t d_samples_cap = 0;
  float *d_out = nullptr; size_t d_out_cap = 0;
  int64_t *d_meta = nullptr; size_t d_meta_cap = 0;
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
  void *d = nullptr;
  if (count == 0) { *dst = nullptr; return 0; }
  CU_TRY(h, cudaMalloc(&d, count * sizeof(T)));
  h->allocs.push_back(d);
  CU_TRY(h, cudaMemcpy(d, src, count * sizeof(T), cudaMemcpyHostToDevice));
  *dst = reinterpret_cast<const T *>(d);
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
  int prev = 0;
  cudaGetDevice(&prev);
  cudaSetDevice(device);

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
  if ((int)fac.size() > B200_MAX_STAGES) { delete h; return fail(nullptr, B200FEAT_EUNSUPPORTED, "too many FFT stages"); }
  p.nstages = (int)fac.size();
  for (int i = 0; i < p.nstages; ++i) p.radix[i] = fac[i];

  // host copies kept for get_table and for the fast kernel's derived tables
  h->h_window.assign(window, window + L);
  if (mel) h->h_bank.assign(mel_bank, mel_bank + (size_t)p.K * p.M);
  if (p.C) h->h_dct.assign(dct, dct + (size_t)p.M * p.C);
  if (desc->use_lifter) h->h_lifter.assign(lifter, lifter + p.C);

  int rc = 0;
#define UP(expr) do { rc = (expr); if (rc) { cudaSetDevice(prev); b200feat_destroy(h); return rc; } } while (0)
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
      int first = -1, last = -1;
      for (int k = 0; k < p.K; ++k)
        if (mel_bank[(size_t)k * p.M + m] != 0.f) { if (first < 0) first = k; last = k; }
      mstart[m] = first < 0 ? 0 : first;
      mlen[m] = first < 0 ? 0 : last - first + 1;
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
  if (desc->kernel == B200FEAT_KERNEL_TC && !tc_ok) {
    cudaSetDevice(prev); b200feat_destroy(h);
    return fail(nullptr, B200FEAT_EUNSUPPORTED, "the tensor-core kernel needs fft_length 512, fbank / mfcc without use_energy, Kaldi framing");
  }
  const bool fast512_ok = !whisper && fast512_supported(p);
  const bool fast256_ok = !whisper && fast256_supported(p);
  const bool fast1024_ok = !whisper && fast1024_supported(p);
  const bool fast400_ok = fast400_supported(p);
  const bool fast2048_ok = !whisper && fast2048_supported(p);
  const bool fast_ok = fast512_ok || fast256_ok || fast1024_ok || fast2048_ok || fast400_ok;
  if (desc->kernel == B200FEAT_KERNEL_FAST && !fast_ok) {
    cudaSetDevice(prev); b200feat_destroy(h);
    return fail(nullptr, B200FEAT_EUNSUPPORTED, "fast kernels require fft_length 256, 512, 1024, 2048 or frame_length = fft_length = 400");
  }
  bool auto_tc = false;  // AUTO prefers the tensor-core kernel where it is the faster one (B200FEAT_AUTO_TC=0/1 overrides)
  if (const char *e = getenv("B200FEAT_AUTO_TC")) auto_tc = atoi(e) != 0;
  if (desc->kernel == B200FEAT_KERNEL_TC || (desc->kernel == B200FEAT_KERNEL_AUTO && tc_ok && auto_tc)) h->kernel = B200FEAT_KERNEL_TC;
  else if (desc->kernel == B200FEAT_KERNEL_GENERIC || !fast_ok) h->kernel = B200FEAT_KERNEL_GENERIC;
  else h->kernel = B200FEAT_KERNEL_FAST;

  {  // generic launch shape: as many warps per CTA as fit ~100 KB, CTA <= 8 warps
    const size_t per_warp = generic_smem_per_warp(p.N, p.Nc);
    int w = (int)((100 * 1024) / per_warp);
    if (w > 8) w = 8;
    if (w < 1) w = 1;
    h->generic_warps = w;
    h->generic_smem = per_warp * w;
    if (h->generic_smem > 227 * 1024) {
      cudaSetDevice(prev); b200feat_destroy(h);
      return fail(nullptr, B200FEAT_EUNSUPPORTED, "fft_length too large for shared memory");
    }
    if (h->generic_smem > 48 * 1024) {
      cudaError_t e1 = cudaFuncSetAttribute(b200feat_generic_kernel<B200FEAT_F32>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)h->generic_smem);
      cudaError_t e2 = cudaFuncSetAttribute(b200feat_generic_kernel<B200FEAT_I16>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)h->generic_smem);
      if (e1 != cudaSuccess || e2 != cudaSuccess) {
        cudaSetDevice(prev); b200feat_destroy(h);
        return fail(nullptr, B200FEAT_ECUDA, "cudaFuncSetAttribute(generic smem) failed");
      }
    }
  }
  h->frames_per_tile = 1;
  if (h->kernel == B200FEAT_KERNEL_TC) {
    rc = tc512_prepare(h->plan, h->h_bank, h->allocs, &h->frames_per_tile, h->h_window, &h->tc);
    if (rc == B200FEAT_EUNSUPPORTED && desc->kernel == B200FEAT_KERNEL_AUTO) {
      h->kernel = fast_ok ? B200FEAT_KERNEL_FAST : B200FEAT_KERNEL_GENERIC;
      h->frames_per_tile = 1;
      rc = 0;
    } else if (rc) {
      cudaSetDevice(prev); b200feat_destroy(h);
      return fail(nullptr, rc, "tensor-core kernel cannot be prepared for this plan");
    }
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
    } else if (rc) {
      cudaSetDevice(prev); b200feat_destroy(h);
      return fail(nullptr, rc, "fast kernel cannot be prepared for this plan (shared-memory footprint?)");
    }
  }
#undef UP
  cudaSetDevice(prev);
  *out = h;
  return B200FEAT_OK;
}

void b200feat_destroy(b200feat_handle *h) {
  if (!h) return;
  int prev = 0;
  cudaGetDevice(&prev);
  cudaSetDevice(h->device);
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
  cudaSetDevice(prev);
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
    const int64_t T = frames_for(h->desc, num_samples[i]);
    if (!framable(h->desc, num_samples[i], T))
      return fail(h, B200FEAT_ESHORT, "cut " + std::to_string(i) + " with " + std::to_string(num_samples[i]) +
                                          " samples is too short to be framed");
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
    const int64_t T = frames_for(h->desc, n);
    if (!framable(h->desc, n, T))
      return fail(h, B200FEAT_ESHORT, "cut " + std::to_string(i) + " with " + std::to_string(n) +
                                          " samples is too short to be framed");
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

// launches the selected kernel over cuts [b0, b1) of a planned batch
static int launch_range(b200feat_handle *h, const void *samples_dev, int32_t dt, const int64_t *meta_dev,
                        int32_t B, int32_t b0, int32_t b1, int64_t tile0, int64_t tile1,
                        int64_t max_frames, float *out_dev, int32_t out_mode, float pad_value,
                        cudaStream_t stream, float *cut_max_dev = nullptr, int64_t norm_rows = 0) {
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
  if (h->kernel == B200FEAT_KERNEL_TC) {
    int rc = tc512_launch(h->plan, h->tc, db, dt, h->sm_count, stream);
    if (rc) return fail(h, B200FEAT_ECUDA, std::string("tc512 launch: ") + cudaGetErrorString((cudaError_t)rc));
  } else if (h->kernel == B200FEAT_KERNEL_FAST && h->plan.N == 256) {
    int rc = fast256_launch(h->plan, h->fast256, db, dt, h->sm_count, stream);
    if (rc) return fail(h, B200FEAT_ECUDA, std::string("fast256 launch: ") + cudaGetErrorString((cudaError_t)rc));
  } else if (h->kernel == B200FEAT_KERNEL_FAST && h->plan.N == 400) {
    int rc = fast400_launch(h->plan, h->fast400, db, dt, h->sm_count, stream);
    if (rc) return fail(h, B200FEAT_ECUDA, std::string("fast400 launch: ") + cudaGetErrorString((cudaError_t)rc));
  } else if (h->kernel == B200FEAT_KERNEL_FAST && h->plan.N == 1024) {
    int rc = fast1024_launch(h->plan, h->fast1024, db, dt, h->sm_count, stream);
    if (rc) return fail(h, B200FEAT_ECUDA, std::string("fast1024 launch: ") + cudaGetErrorString((cudaError_t)rc));
  } else if (h->kernel == B200FEAT_KERNEL_FAST && h->plan.N == 2048) {
    int rc = fast2048_launch(h->plan, h->fast2048, db, dt, h->sm_count, stream);
    if (rc) return fail(h, B200FEAT_ECUDA, std::string("fast2048 launch: ") + cudaGetErrorString((cudaError_t)rc));
  } else if (h->kernel == B200FEAT_KERNEL_FAST) {
    int rc = fast512_launch(h->plan, h->fast, db, dt, h->sm_count, stream);
    if (rc) return fail(h, B200FEAT_ECUDA, std::string("fast512 launch: ") + cudaGetErrorString((cudaError_t)rc));
  } else {
    const int w = h->generic_warps;
    int64_t blocks = (db.num_tiles + w - 1) / w;
    const int64_t cap = (int64_t)h->sm_count * 8;
    if (blocks > cap) blocks = cap;
    if (dt == B200FEAT_I16)
      b200feat_generic_kernel<B200FEAT_I16><<<(unsigned)blocks, w * 32, h->generic_smem, stream>>>(h->plan, db);
    else
      b200feat_generic_kernel<B200FEAT_F32><<<(unsigned)blocks, w * 32, h->generic_smem, stream>>>(h->plan, db);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return fail(h, B200FEAT_ECUDA, std::string("generic launch: ") + cudaGetErrorString(e));
  }
  if (h->plan.whisper && norm_rows > 0) {  // second launch: clamp to the cut's maximum - 8, (x + 4) / 4, zero rows
    if (h->frames_per_tile > 1) {
      int64_t blocks = db.num_tiles;
      const int64_t cap = (int64_t)h->sm_count * 8;
      if (blocks > cap) blocks = cap;
      b200feat_whisper_normalize_tiled_kernel<<<(unsigned)blocks, 256, 0, stream>>>(h->plan, db, h->frames_per_tile);
    } else {
      int64_t blocks = (norm_rows + 7) / 8;
      const int64_t cap = (int64_t)h->sm_count * 16;
      if (blocks > cap) blocks = cap;
      b200feat_whisper_normalize_kernel<<<(unsigned)blocks, 256, 0, stream>>>(h->plan, db, norm_rows);
    }
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return fail(h, B200FEAT_ECUDA, std::string("whisper normalise launch: ") + cudaGetErrorString(e));
  }
  return 0;
}

int b200feat_extract(b200feat_handle *h, const void *samples_dev, int32_t dt, const int64_t *meta_dev,
                     int32_t B, const b200feat_batch_totals *tot, float *out_dev, int32_t out_mode,
                     float pad_value, void *stream) {
  if (!h || !samples_dev || !meta_dev || !tot || !out_dev || B <= 0) return fail(h, B200FEAT_EINVAL, "extract: bad arguments");
  if (dt != B200FEAT_F32 && dt != B200FEAT_I16) return fail(h, B200FEAT_EINVAL, "bad sample dtype");
  int prev = 0;
  cudaGetDevice(&prev);
  if (prev != h->device) cudaSetDevice(h->device);
  const int64_t all_rows = out_mode == B200FEAT_OUT_PADDED ? (int64_t)B * tot->max_frames : tot->total_rows;
  float *scratch = h->plan.whisper ? out_dev + all_rows * h->plan.F : nullptr;
  int rc = launch_range(h, samples_dev, dt, meta_dev, B, 0, B, 0, tot->total_tiles, tot->max_frames, out_dev,
                        out_mode, pad_value, (cudaStream_t)stream, scratch, all_rows);
  if (prev != h->device) cudaSetDevice(prev);
  if (rc) return rc;
  {
    std::lock_guard<std::mutex> g(h->stats_mu);
    h->stats.calls++; h->stats.cuts += B; h->stats.frames += tot->total_rows;
    h->stats.kernel_launches += h->plan.whisper ? 2 : 1;
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
  HostRing &r = h->ring;
  std::lock_guard<std::mutex> guard(r.mu);
  int prev = 0;
  cudaGetDevice(&prev);
  cudaSetDevice(h->device);
  struct Restore { int d; ~Restore() { cudaSetDevice(d); } } restore{prev};

  const size_t esz = dt == B200FEAT_I16 ? 2 : 4;
  const int64_t words = b200feat_plan_words(h, num_samples, B, out_mode);
  if (words < 0) return (int)words;
  if (r.h_meta_cap < (size_t)words) {
    if (r.h_meta) cudaFreeHost(r.h_meta);
    r.h_meta = nullptr; r.h_meta_cap = 0;
    CU_TRY(h, cudaMallocHost((void **)&r.h_meta, (size_t)words * 8));
    r.h_meta_cap = (size_t)words;
  }
  b200feat_batch_totals tot;
  // the host layout (back to back unless the caller supplied offsets) is kept on the device: chunks are copied verbatim
  int rc = b200feat_plan_batch(h, num_samples, sample_offsets, B, 1, out_mode, r.h_meta, words, &tot);
  if (rc) return rc;
  for (auto &s : r.streams) if (!s) CU_TRY(h, cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking));
  if (!r.meta_ready) CU_TRY(h, cudaEventCreateWithFlags(&r.meta_ready, cudaEventDisableTiming));
  auto grow = [&](void **p, size_t *cap, size_t need) -> cudaError_t {
    if (*cap >= need) return cudaSuccess;
    if (*p) cudaFree(*p);
    *p = nullptr; *cap = 0;
    size_t want = need + need / 4;
    cudaError_t e = cudaMalloc(p, want);
    if (e == cudaSuccess) *cap = want;
    return e;
  };
  CU_TRY(h, grow(&r.d_samples, &r.d_samples_cap, (size_t)tot.span_samples * esz + 16));
  CU_TRY(h, grow((void **)&r.d_out, &r.d_out_cap, (size_t)tot.out_floats * 4 + 16));
  {
    size_t capb = r.d_meta_cap * 8;
    CU_TRY(h, grow((void **)&r.d_meta, &capb, (size_t)words * 8));
    r.d_meta_cap = capb / 8;
  }
  CU_TRY(h, cudaMemcpyAsync(r.d_meta, r.h_meta, (size_t)words * 8, cudaMemcpyHostToDevice, r.streams[0]));
  CU_TRY(h, cudaEventRecord(r.meta_ready, r.streams[0]));

  // chunk over cuts: ~32 MB of samples per chunk, round-robin over 3 streams so that
  // H2D(i+1), kernel(i) and D2H(i-1) overlap (PCIe is the end-to-end bound, SURVEY.md §7)
  const int64_t *soff = r.h_meta, *roff = r.h_meta + 2 * (int64_t)B, *toff = r.h_meta + 3 * (int64_t)B + 1;
  const int64_t chunk_elems = (32ll << 20) / (int64_t)esz;
  float *scratch = h->plan.whisper ? r.d_out + (tot.out_floats - B) : nullptr;
  int b0 = 0, ci = 0, launches = 0;
  while (b0 < B) {
    int b1 = b0 + 1;
    while (b1 < B && (soff[b1] + num_samples[b1]) - soff[b0] <= chunk_elems) ++b1;
    cudaStream_t st = r.streams[ci % 3];
    if (ci < 3) CU_TRY(h, cudaStreamWaitEvent(st, r.meta_ready, 0));
    const int64_t e0 = soff[b0], e1 = soff[b1 - 1] + num_samples[b1 - 1];
    CU_TRY(h, cudaMemcpyAsync((char *)r.d_samples + e0 * esz, (const char *)samples_host + e0 * esz,
                              (size_t)(e1 - e0) * esz, cudaMemcpyHostToDevice, st));
    int64_t f0, f1;
    if (out_mode == B200FEAT_OUT_PADDED) { f0 = (int64_t)b0 * tot.max_frames; f1 = (int64_t)b1 * tot.max_frames; }
    else { f0 = roff[b0]; f1 = roff[b1]; }
    rc = launch_range(h, r.d_samples, dt, r.d_meta, B, b0, b1, toff[b0], toff[b1], tot.max_frames, r.d_out,
                      out_mode, pad_value, st, scratch, f1 - f0);
    if (rc) return rc;
    launches += h->plan.whisper ? 2 : 1;
    CU_TRY(h, cudaMemcpyAsync(out_host + f0 * h->plan.F, r.d_out + f0 * h->plan.F,
                              (size_t)(f1 - f0) * h->plan.F * 4, cudaMemcpyDeviceToHost, st));
    b0 = b1; ++ci;
  }
  for (auto &s : r.streams) CU_TRY(h, cudaStreamSynchronize(s));
  {
    std::lock_guard<std::mutex> g(h->stats_mu);
    h->stats.calls++; h->stats.cuts += B; h->stats.frames += tot.total_rows;
    h->stats.samples += tot.span_samples; h->stats.kernel_launches += launches;
  }
  return B200FEAT_OK;
}

int b200feat_extract_host_ptrs(b200feat_handle *h, const void *const *cuts, int32_t dt, const int64_t *num_samples, int32_t B,
                               float *out_host, int32_t out_mode, float pad_value) {
  if (!h || !cuts || !num_samples || !out_host || B <= 0) return fail(h, B200FEAT_EINVAL, "extract_host_ptrs: bad arguments");
  if (dt != B200FEAT_F32 && dt != B200FEAT_I16) return fail(h, B200FEAT_EINVAL, "bad sample dtype");
  for (int i = 0; i < B; ++i)
    if (!cuts[i] && num_samples[i] > 0) return fail(h, B200FEAT_EINVAL, "extract_host_ptrs: null cut pointer");
  HostRing &r = h->ring;
  std::lock_guard<std::mutex> guard(r.mu);
  int prev = 0;
  cudaGetDevice(&prev);
  cudaSetDevice(h->device);
  struct Restore { int d; ~Restore() { cudaSetDevice(d); } } restore{prev};

  const size_t esz = dt == B200FEAT_I16 ? 2 : 4;
  const int32_t align = dt == B200FEAT_I16 ? 8 : 4;  // every cut starts on a 16-byte boundary of the device buffer
  const int64_t words = b200feat_plan_words(h, num_samples, B, out_mode);
  if (words < 0) return (int)words;
  if (r.h_meta_cap < (size_t)words) {
    if (r.h_meta) cudaFreeHost(r.h_meta);
    r.h_meta = nullptr; r.h_meta_cap = 0;
    CU_TRY(h, cudaMallocHost((void **)&r.h_meta, (size_t)words * 8));
    r.h_meta_cap = (size_t)words;
  }
  b200feat_batch_totals tot;
  int rc = b200feat_plan_batch(h, num_samples, nullptr, B, align, out_mode, r.h_meta, words, &tot);
  if (rc) return rc;
  for (auto &s : r.streams) if (!s) CU_TRY(h, cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking));
  if (!r.meta_ready) CU_TRY(h, cudaEventCreateWithFlags(&r.meta_ready, cudaEventDisableTiming));
  for (int k = 0; k < 2; ++k)
    if (!r.stage_free[k]) CU_TRY(h, cudaEventCreateWithFlags(&r.stage_free[k], cudaEventDisableTiming));
  if (!h->pool) {
    int nthreads = 8;
    if (const char *e = getenv("B200FEAT_STAGING_THREADS")) nthreads = std::max(1, atoi(e));
    h->pool = new GatherPool(nthreads - 1);  // the calling thread works too
  }
  auto grow = [&](void **p, size_t *cap, size_t need, bool host) -> cudaError_t {
    if (*cap >= need) return cudaSuccess;
    if (*p) { if (host) cudaFreeHost(*p); else cudaFree(*p); }
    *p = nullptr; *cap = 0;
    const size_t want = need + need / 4;
    cudaError_t e = host ? cudaMallocHost(p, want) : cudaMalloc(p, want);
    if (e == cudaSuccess) *cap = want;
    return e;
  };
  CU_TRY(h, grow(&r.d_samples, &r.d_samples_cap, (size_t)tot.span_samples * esz + 16, false));
  CU_TRY(h, grow((void **)&r.d_out, &r.d_out_cap, (size_t)tot.out_floats * 4 + 16, false));
  {
    size_t capb = r.d_meta_cap * 8;
    CU_TRY(h, grow((void **)&r.d_meta, &capb, (size_t)words * 8, false));
    r.d_meta_cap = capb / 8;
  }
  CU_TRY(h, cudaMemcpyAsync(r.d_meta, r.h_meta, (size_t)words * 8, cudaMemcpyHostToDevice, r.streams[0]));
  CU_TRY(h, cudaEventRecord(r.meta_ready, r.streams[0]));

  const int64_t *soff = r.h_meta, *roff = r.h_meta + 2 * (int64_t)B, *toff = r.h_meta + 3 * (int64_t)B + 1;
  const int64_t chunk_elems = (32ll << 20) / (int64_t)esz;
  // chunk boundaries first: the staging slots must hold the largest chunk
  std::vector<int> cb{0};
  for (int b0 = 0; b0 < B;) {
    int b1 = b0 + 1;
    while (b1 < B && (soff[b1] + num_samples[b1]) - soff[b0] <= chunk_elems) ++b1;
    cb.push_back(b1);
    b0 = b1;
  }
  size_t max_bytes = 0;
  for (size_t c = 0; c + 1 < cb.size(); ++c)
    max_bytes = std::max(max_bytes, (size_t)((soff[cb[c + 1] - 1] + num_samples[cb[c + 1] - 1]) - soff[cb[c]]) * esz);
  for (int k = 0; k < 2; ++k) CU_TRY(h, grow(&r.h_stage[k], &r.h_stage_cap[k], max_bytes + 64, true));

  float *scratch = h->plan.whisper ? r.d_out + (tot.out_floats - B) : nullptr;
  int launches = 0;
  for (size_t c = 0; c + 1 < cb.size(); ++c) {
    const int b0 = cb[c], b1 = cb[c + 1], slot = (int)(c & 1);
    cudaStream_t st = r.streams[c % 3];
    if (c < 3) CU_TRY(h, cudaStreamWaitEvent(st, r.meta_ready, 0));
    if (c >= 2) CU_TRY(h, cudaEventSynchronize(r.stage_free[slot]));  // the H2D copy out of this slot (chunk c - 2) is done
    unsigned char *stage = static_cast<unsigned char *>(r.h_stage[slot]);
    const int64_t e0 = soff[b0], e1 = soff[b1 - 1] + num_samples[b1 - 1];
    // gather: one task per ~1 MB piece so that long and short cuts balance over the threads
    struct Piece { const unsigned char *src; unsigned char *dst; size_t bytes; };
    std::vector<Piece> pieces;
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
    h->pool->parallel_for((int)pieces.size(), job);
    CU_TRY(h, cudaMemcpyAsync((char *)r.d_samples + e0 * esz, stage, (size_t)(e1 - e0) * esz, cudaMemcpyHostToDevice, st));
    CU_TRY(h, cudaEventRecord(r.stage_free[slot], st));
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

int64_t b200feat_get_table(b200feat_handle *h, int32_t which, float *out, int64_t cap) {
  if (!h || !out) return B200FEAT_EINVAL;
  const DevPlan &p = h->plan;
  int prev = 0;
  cudaGetDevice(&prev);
  cudaSetDevice(h->device);
  struct Restore { int d; ~Restore() { cudaSetDevice(d); } } restore{prev};
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
  int prev = 0;
  cudaGetDevice(&prev);
  cudaSetDevice(h->device);
  struct Restore { int d; ~Restore() { cudaSetDevice(d); } } restore{prev};
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

}  // extern "C"
