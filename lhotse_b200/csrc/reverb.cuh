// Reverberation of mono audio with a room impulse response (lhotse's ReverbWithImpulseResponse with a recorded RIR) on the
// GPU, within a float32 tolerance of a float64 convolution (the float route's own FFT convolution is not bit-reproducible, so
// there is no bit pattern to match; DESIGN.md §3.1j).
//
// Per cut, with x[0, N) the signal and h[0, R) = f32(q / 32768) * 2^-15 the RIR (both exact):
//   shift    s = argmax(h), the first index of the maximum (found on the int16 samples: the widening is monotonic)
//   conv     y[j] = sum_k x[j + s - k] * h[k], j in [0, N), x = 0 outside [0, N)
//   gain     pb = f32(pairwise_sum(x^2)) / N (NumPy's float32 sum, as mix.cuh computes it), pa the same for y (a fixed-order
//            sum of per-CTA partials); with normalize_output and pa > 0, g = f32(sqrt(f32(pb / pa))), else g = 1
//   output   out[p] = f32(y[src(p)] * g), src the trim / reflect-pad of the cut's length fix (mix_source_pos)
//
// The convolution is uniformly partitioned overlap-save with blocks of RV_B samples and complex FFTs of RV_F = 2 * RV_B
// points.  The RIR is cut into P = ceil(R / RV_B) partitions whose spectra H_p (scaled by 1 / RV_F, exact) are computed once
// per RIR and call.  Output block c of y is the second half of IFFT(sum_p X_{c,p} H_p), X_{c,p} the FFT of the RV_F input
// samples that end where block c - p does (shifted by s), with the p sum in increasing order.  Two real blocks ride in one
// complex FFT: block 2q in the real part and block 2q + 1 in the imaginary part (H_p is the spectrum of a real signal, so the
// product keeps the two apart).  One CTA computes one such pair; it recomputes each X instead of keeping a delay line, so its
// shared memory is one transform and the twiddles whatever R is.
//
// The per-butterfly, per-bin and per-sample arithmetic is __host__ __device__ so that scripts/micro/reverb_host_check.cu runs
// exactly this code on the CPU, CTA by CTA.  Kernels at the end.
#pragma once
#include <math.h>
#include <stdint.h>

#include "mix.cuh"

#define RV_LOG_F 12
#define RV_F (1 << RV_LOG_F)       // transform size
#define RV_B (RV_F / 2)            // block and partition length
#define RV_THREADS 512
#define RV_BINS (RV_F / RV_THREADS)  // spectrum bins a thread accumulates
#define RV_MAX_RIR 65536           // the longest RIR taken (b200feat_reverb checks): 32 partitions

#if defined(__CUDA_ARCH__)
#define RV_FMA(a, b, c) __fmaf_rn(a, b, c)
#else
#define RV_FMA(a, b, c) fmaf(a, b, c)
#endif

struct rv_c { float x, y; };

// One RIR as the kernels read it (b200feat_reverb builds these from the b200feat_reverb_rir records)
struct RvRir {
  const int16_t *src;   // its R int16 samples
  int64_t len;          // R
  int64_t part_begin;   // its first partition in the spectra table (and in the RIR kernel's grid)
  int32_t nparts;       // ceil(R / RV_B)
  int32_t reserved;
  const float *src32;   // or, when set (b200feat_reverb_ex), its R float32 samples h / 2^-15 (a generated RIR)
};

// One cut as the kernels read it
struct RvCut {
  const float *x;       // the input, N samples
  float *y;             // the unscaled convolution, N samples (work buffer)
  float *out;           // the cut's first output sample
  int64_t n;            // N
  int64_t target_len;   // samples written: N, fewer (trim) or at most N - 1 more (reflect-pad)
  int64_t cta_begin;    // its first CTA in the convolution kernel's grid
  int32_t rir;          // index into the RIR table
  int32_t normalize;    // 1: lhotse's normalize_output
};

MIX_HD int64_t rv_parts(int64_t R) { return (R + RV_B - 1) / RV_B; }
MIX_HD int64_t rv_cut_ctas(int64_t n) { return (n + 2 * RV_B - 1) / (2 * RV_B); }

MIX_HD int rv_bitrev(int i) {
#if defined(__CUDA_ARCH__)
  return (int)(__brev((unsigned)i) >> (32 - RV_LOG_F));
#else
  int r = 0;
  for (int b = 0; b < RV_LOG_F; ++b) r |= ((i >> b) & 1) << (RV_LOG_F - 1 - b);
  return r;
#endif
}

// exp(-2 pi i k / RV_F), k < RV_F / 2, evaluated in double on the host and rounded once: b200feat_reverb uploads this table
// and the host harness uses the same function, so both sides run the same twiddle bits
inline rv_c rv_twiddle(int k) {
  return rv_c{(float)cos(-2.0 * M_PI * k / RV_F), (float)sin(-2.0 * M_PI * k / RV_F)};
}

// Butterfly j (< RV_F / 2) of the radix-2 decimation-in-time stage whose sub-transforms have `half` points, in place on a
// bit-reversed array; the inverse transform uses the conjugate twiddles (its 1 / RV_F sits in the RIR spectra)
MIX_HD void rv_butterfly(rv_c *a, const rv_c *tw, int half, int j, bool inverse) {
  const int pos = j & (half - 1);
  const int i0 = ((j - pos) << 1) + pos, i1 = i0 + half;
  const rv_c w = tw[pos * (RV_B / half)];
  const float wy = inverse ? -w.y : w.y;
  const rv_c b = a[i1];
  const rv_c t{RV_FMA(w.x, b.x, -(wy * b.y)), RV_FMA(w.x, b.y, wy * b.x)};
  const rv_c u = a[i0];
  a[i0] = rv_c{u.x + t.x, u.y + t.y};
  a[i1] = rv_c{u.x - t.x, u.y - t.y};
}

// acc + a * b, complex, two FMAs per component
MIX_HD rv_c rv_cmac(rv_c acc, rv_c a, rv_c b) {
  return rv_c{RV_FMA(a.x, b.x, RV_FMA(-a.y, b.y, acc.x)), RV_FMA(a.x, b.y, RV_FMA(a.y, b.x, acc.y))};
}

// RIR sample i before lhotse's 2^-15 scaling: f32(q / 32768) for an int16 RIR, the float32 sample itself otherwise
MIX_HD float rv_rir_value(const RvRir &r, int64_t i) { return r.src32 ? r.src32[i] : mix_widen(r.src[i]); }

// RIR sample k of partition p as its spectrum takes it: h * 2^-15 * (1 / RV_F), 0 past the RIR.  Exact for every int16 RIR
// and for float32 samples with |h| >= 2^-99; below that the product is subnormal and rounded once (no flush to zero: the
// library is built without -ftz or fast math, so the device rounds as the host does)
MIX_HD float rv_rir_sample(const RvRir &r, int p, int k) {
  const int64_t i = (int64_t)p * RV_B + k;
  if (k >= RV_B || i >= r.len) return 0.0f;
  return MIX_FMUL(rv_rir_value(r, i), 1.0f / (32768.0f * RV_F));
}

// The first input sample of the transform of CTA q's block pair for partition p (its real part; the imaginary part starts
// RV_B later): x[g + m] lands at transform position m, and positions [RV_B, RV_F) of the circular convolution with H_p are
// then the partition's contribution to y[2q * RV_B + i]
MIX_HD int64_t rv_seg_start(int64_t q, int p, int64_t shift) { return shift + 2 * q * RV_B - (int64_t)(p + 1) * RV_B; }

// whether partition p touches the cut's samples at all (otherwise its product is zero and is skipped)
MIX_HD bool rv_seg_live(int64_t g, int64_t n) { return g + RV_F + RV_B > 0 && g < n; }

MIX_HD rv_c rv_seg_load(const RvCut &c, int64_t g, int m) {
  const int64_t a = g + m, b = a + RV_B;
  return rv_c{a >= 0 && a < c.n ? c.x[a] : 0.0f, b >= 0 && b < c.n ? c.x[b] : 0.0f};
}

// The gain of a cut from pb = f32(S_x) / N and the float64 sum of y^2: lhotse's sqrt(pb / pa) in float32, 1 without it
MIX_HD float rv_gain(float pb, double sum_y2, int64_t n, int normalize) {
  const float pa = MIX_FDIV((float)sum_y2, (float)n);
  if (!normalize || !(pa > 0.0f)) return 1.0f;
#if defined(__CUDA_ARCH__)
  return __fsqrt_rn(MIX_FDIV(pb, pa));
#else
  return sqrtf(MIX_FDIV(pb, pa));
#endif
}

MIX_HD float rv_out(const RvCut &c, float g, int64_t p) { return MIX_FMUL(c.y[mix_source_pos(p, c.n)], g); }

#ifdef __CUDACC__
#define RV_SMEM_BYTES ((RV_F + RV_B) * (int)sizeof(rv_c) + 32 * (int)sizeof(float))
#define RV_GAIN_THREADS 128
#define RV_OUT_THREADS 256

__device__ __forceinline__ void rv_fft(rv_c *a, const rv_c *tw, bool inverse) {
  for (int half = 1; half < RV_F; half <<= 1) {
    __syncthreads();
    for (int j = threadIdx.x; j < RV_F / 2; j += RV_THREADS) rv_butterfly(a, tw, half, j, inverse);
  }
  __syncthreads();
}

// One CTA per RIR partition: the partition's spectrum; partition 0 also finds the RIR's shift.
__global__ void __launch_bounds__(RV_THREADS) reverb_rir_kernel(const RvRir *__restrict__ rirs, int nrirs, rv_c *__restrict__ spectra,
                                                                 int32_t *__restrict__ shift, const rv_c *__restrict__ twiddles) {
  extern __shared__ __align__(16) unsigned char rv_smem[];
  rv_c *a = (rv_c *)rv_smem, *tw = a + RV_F;
  int lo = 0, hi = nrirs - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (rirs[mid].part_begin <= (int64_t)blockIdx.x) lo = mid; else hi = mid - 1;
  }
  const RvRir r = rirs[lo];
  const int p = (int)((int64_t)blockIdx.x - r.part_begin);
  for (int k = threadIdx.x; k < RV_B; k += RV_THREADS) tw[k] = twiddles[k];
  for (int m = threadIdx.x; m < RV_F; m += RV_THREADS) a[rv_bitrev(m)] = rv_c{rv_rir_sample(r, p, m), 0.0f};
  rv_fft(a, tw, false);
  rv_c *dst = spectra + (r.part_begin + p) * RV_F;
  for (int k = threadIdx.x; k < RV_F; k += RV_THREADS) dst[k] = a[k];
  if (p != 0) return;
  // first index of the maximum: per thread, then a tree over (value, index) with ties to the lower index
  // (on the widened samples: the widening of an int16 RIR is monotonic, so its first maximum is the same)
  float best = -INFINITY;
  int at = 0x7fffffff;
  for (int64_t i = threadIdx.x; i < r.len; i += RV_THREADS) {
    const float v = rv_rir_value(r, i);
    if (v > best || at == 0x7fffffff) { best = v; at = (int)i; }
  }
  float *red = (float *)(tw + RV_B);
  int *red_at = (int *)(red + 16);
  for (int off = 16; off > 0; off >>= 1) {
    const float ob = __shfl_down_sync(0xffffffffu, best, off);
    const int oa = __shfl_down_sync(0xffffffffu, at, off);
    if (oa != 0x7fffffff && (ob > best || (ob == best && oa < at) || at == 0x7fffffff)) { best = ob; at = oa; }
  }
  __syncthreads();
  if ((threadIdx.x & 31) == 0) { red[threadIdx.x >> 5] = best; red_at[threadIdx.x >> 5] = at; }
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int w = 1; w < RV_THREADS / 32; ++w)
      if (red_at[w] != 0x7fffffff && (red[w] > best || (red[w] == best && red_at[w] < at) || at == 0x7fffffff)) {
        best = red[w];
        at = red_at[w];
      }
    shift[lo] = at;
  }
}

// One CTA per block pair of a cut: y over [2q * RV_B, 2q * RV_B + 2 * RV_B) and the CTA's sum of y^2 (fixed order).
__global__ void __launch_bounds__(RV_THREADS, 1) reverb_conv_kernel(const RvCut *__restrict__ cuts, int ncuts, const RvRir *__restrict__ rirs,
                                                                  const rv_c *__restrict__ spectra, const int32_t *__restrict__ shift,
                                                                  const rv_c *__restrict__ twiddles, float *__restrict__ partial) {
  extern __shared__ __align__(16) unsigned char rv_smem[];
  rv_c *a = (rv_c *)rv_smem, *tw = a + RV_F;
  float *red = (float *)(tw + RV_B);
  int lo = 0, hi = ncuts - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (cuts[mid].cta_begin <= (int64_t)blockIdx.x) lo = mid; else hi = mid - 1;
  }
  const RvCut c = cuts[lo];
  const RvRir r = rirs[c.rir];
  const int64_t q = (int64_t)blockIdx.x - c.cta_begin, s = shift[c.rir];
  for (int k = threadIdx.x; k < RV_B; k += RV_THREADS) tw[k] = twiddles[k];
  rv_c acc[RV_BINS];
#pragma unroll
  for (int i = 0; i < RV_BINS; ++i) acc[i] = rv_c{0.0f, 0.0f};
  for (int p = 0; p < r.nparts; ++p) {
    const int64_t g = rv_seg_start(q, p, s);
    if (!rv_seg_live(g, c.n)) continue;  // CTA-uniform
    __syncthreads();
    for (int m = threadIdx.x; m < RV_F; m += RV_THREADS) a[rv_bitrev(m)] = rv_seg_load(c, g, m);
    rv_fft(a, tw, false);
    const rv_c *H = spectra + (r.part_begin + p) * RV_F;
#pragma unroll
    for (int i = 0; i < RV_BINS; ++i) {
      const int k = threadIdx.x + i * RV_THREADS;
      acc[i] = rv_cmac(acc[i], a[k], H[k]);
    }
  }
  __syncthreads();
#pragma unroll
  for (int i = 0; i < RV_BINS; ++i) {
    const int k = threadIdx.x + i * RV_THREADS;
    a[rv_bitrev(k)] = acc[i];
  }
  rv_fft(a, tw, true);
  float e = 0.0f;
  const int64_t base = 2 * q * RV_B;
  for (int i = threadIdx.x; i < RV_B; i += RV_THREADS) {
    const rv_c v = a[RV_B + i];
    if (base + i < c.n) { c.y[base + i] = v.x; e = RV_FMA(v.x, v.x, e); }
    if (base + RV_B + i < c.n) { c.y[base + RV_B + i] = v.y; e = RV_FMA(v.y, v.y, e); }
  }
  for (int off = 16; off > 0; off >>= 1) e += __shfl_down_sync(0xffffffffu, e, off);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = e;
  __syncthreads();
  if (threadIdx.x == 0) {
    float t = 0.0f;
    for (int w = 0; w < RV_THREADS / 32; ++w) t += red[w];
    partial[blockIdx.x] = t;
  }
}

// One block per cut: pb (warp 0, NumPy's pairwise sum of x^2), the float64 sum of the cut's partials in CTA order (the other
// warps, then a fixed tree), the gain.
__global__ void __launch_bounds__(RV_GAIN_THREADS) reverb_gain_kernel(const RvCut *__restrict__ cuts, const float *__restrict__ partial,
                                                                      float *__restrict__ gain) {
  __shared__ double part[RV_GAIN_THREADS];
  __shared__ float pb;
  const RvCut c = cuts[blockIdx.x];
  const int64_t nctas = rv_cut_ctas(c.n);
  if (threadIdx.x < 32) {
    const float v = mix_warp_sum(c.x, c.n, threadIdx.x);
    if (threadIdx.x == 0) pb = MIX_FDIV(v, (float)c.n);
  }
  double t = 0.0;
  for (int64_t i = threadIdx.x; i < nctas; i += RV_GAIN_THREADS) t += (double)partial[c.cta_begin + i];
  part[threadIdx.x] = t;
  __syncthreads();
  for (int w = RV_GAIN_THREADS / 2; w > 0; w >>= 1) {
    if (threadIdx.x < w) part[threadIdx.x] += part[threadIdx.x + w];
    __syncthreads();
  }
  if (threadIdx.x == 0) gain[blockIdx.x] = rv_gain(pb, part[0], c.n, c.normalize);
}

// grid (x, cuts): out[p] = f32(y[src(p)] * g) over the cut's target length
__global__ void __launch_bounds__(RV_OUT_THREADS) reverb_out_kernel(const RvCut *__restrict__ cuts, const float *__restrict__ gain) {
  const RvCut c = cuts[blockIdx.y];
  const float g = gain[blockIdx.y];
  for (int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; p < c.target_len; p += (int64_t)gridDim.x * blockDim.x)
    c.out[p] = rv_out(c, g, p);
}
#endif
