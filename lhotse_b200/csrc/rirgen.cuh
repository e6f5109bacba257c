// lhotse's FastRandomRIRGenerator (nsource = 1) on the GPU, from draws made on the host (lhotse_b200/rir_draws.py), up to
// its output at 8 x the sampling rate; b200feat_resample then takes that to the sampling rate (DESIGN.md §3.1l).
//
// Per RIR, with T60, R, d0 the room and source draws, sr its rate, S = 64 sr, I = 2 sr image sources and L = ceil(S T60):
//   entries  entry 0 is the direct path (distance d0, reflections 0); entry i >= 1 is image k = i - 1:
//              idx    torch.multinomial's binary search of the uniform u[k] over the float32 normalised cumulative
//                     distribution of linspace(alpha, 1, I)^2 (built on the host)
//              ratio  torch.linspace(1, 340 T60 / d0 - 1, I)[idx] in float32 (rg_linspace, pinned against torch's CPU kernel)
//              dist   d0 * ratio, reflections max(rr + pert[k] * f32(ratio^tau), 1) with lhotse's float64 chain
//            position min(ceil(dist * S / 340), L - 1) (pure float64 multiplies and divides: exact), value f32(coef^refl / dist)
//   comb     rir[position] = value; where entries share a position the last one in entry order is kept (what lhotse's
//            `rir[idx] += decay` leaves with one torch thread).  The entries of an RIR are sorted by position with a stable
//            segmented radix sort and only the last of each run is used.
//   S -> 8 sr  output j is the FMA chain of resample_stage_kernel (csrc/resample.cuh, the O = 8 -> N = 1 table, K = 106 taps)
//            over the comb entries inside its window, in tap order: the zero taps it skips would leave the chain unchanged
//            (but for the sign of a zero), so this is the dense resampler without its L-sample input.
//   biquad   torchaudio's highpass_biquad(., 8 sr, 80): the 3-tap FIR, the IIR recurrence in lfilter's order with no FMA
//            contraction, then clamp(-1, 1); one sequential thread per RIR.
//
// The index arithmetic, the linspace, the entry chain, the window walk and the biquad step are __host__ __device__ and
// compile as plain C++ too, so that a host harness can run exactly this code on the CPU.  Kernels at the end.
#pragma once
#include <math.h>
#include <stdint.h>

#include "mix.cuh"

#define RG_THREADS 256
#define RG_O 8        // both resampling stages are 8 -> 1
#define RG_WIDTH 49   // ceil(6 * 8 / 0.99)
#define RG_TAPS 106   // 2 * RG_WIDTH + RG_O
#define RG_VELOCITY 340.0

#if defined(__CUDA_ARCH__)
#define RG_FMA(a, b, c) __fmaf_rn(a, b, c)
#define RG_FSUB(a, b) __fsub_rn(a, b)
#define RG_DSUB(a, b) __dsub_rn(a, b)
#else
#define RG_FMA(a, b, c) fmaf(a, b, c)
MIX_HD float rg_fsub_h(float a, float b) { volatile float r = a - b; return r; }
MIX_HD double rg_dsub_h(double a, double b) { volatile double r = a - b; return r; }
#define RG_FSUB(a, b) rg_fsub_h(a, b)
#define RG_DSUB(a, b) rg_dsub_h(a, b)
#endif

// One RIR as the kernels read it (b200feat_rir_generate builds these from the b200feat_rir_gen records)
struct RgRir {
  const double *u;       // I uniforms of the multinomial
  const double *pert;    // I perturbations, source_rng.uniform(a, b)
  const float *cdf;      // I entries of the normalised cumulative distribution, the last one 1
  float *out;            // out_len samples at 8 sr
  double t60, r, d0, tau;
  int64_t comb_len;      // L
  int64_t out_len;       // resampled_len(1, L, 8)
  int64_t entry_begin;   // its first entry in the entry arrays (I + 1 entries)
  int64_t cta_begin;     // its first CTA in the window kernel's grid
  int32_t sr, images;
  float b0, b1, b2, a1, a2;  // the biquad, normalised by a0
};

// The scalars every entry of an RIR shares, in lhotse's float64 order
struct RgRoom {
  double coef;         // (1 - (1 - exp(-0.16 R / T60))^2)^0.5
  double vt;           // 340 T60
  double reflect_max;  // (log10(340 T60) - log10(d0) - 3) / log10(coef + 2^-10), less 1
  double sample_sr;    // 64 sr
  float lin_end;       // f32(340 T60 / d0 - 1)
};

MIX_HD RgRoom rg_room(const RgRir &g) {
  RgRoom m;
  const double e = exp(MIX_DDIV(MIX_DMUL(-0.16, g.r), g.t60));
  const double q = RG_DSUB(1.0, e);
  m.coef = MIX_DSQRT(RG_DSUB(1.0, MIX_DMUL(q, q)));
  m.vt = MIX_DMUL(RG_VELOCITY, g.t60);
  const double num = RG_DSUB(RG_DSUB(log10(m.vt), log10(g.d0)), 3.0);
  m.reflect_max = RG_DSUB(MIX_DDIV(num, log10(MIX_DADD(m.coef, 0.0009765625))), 1.0);
  m.sample_sr = (double)g.sr * 64.0;
  m.lin_end = MIX_D2F(RG_DSUB(MIX_DDIV(m.vt, g.d0), 1.0));
  return m;
}

// torch.multinomial's slot for uniform u over cdf[0, n) (ATen's multinomial_with_replacement, with cdf[n - 1] = 1)
MIX_HD int rg_search(const float *cdf, int n, double u) {
  int lo = 0, hi = n;
  while (hi - lo > 0) {
    const int mid = lo + (hi - lo) / 2;
    if ((double)cdf[mid] < u) lo = mid + 1; else hi = mid;
  }
  return lo;
}

// torch.linspace(start, end, steps)[i] in float32 as ATen's CPU kernel computes it: step = f32(end - start) / (steps - 1),
// then one FMA from the nearer end
MIX_HD float rg_linspace(float start, float end, int steps, int i) {
  const float step = MIX_FDIV(RG_FSUB(end, start), (float)(steps - 1));
  return i < steps / 2 ? RG_FMA(step, (float)i, start) : RG_FMA(-step, (float)(steps - i - 1), end);
}

// Entry i (0: the direct path) of the RIR: its comb position and value
MIX_HD void rg_entry(const RgRir &g, const RgRoom &m, int i, int32_t *pos, float *val) {
  double dist, refl;
  if (i == 0) {
    dist = g.d0;
    refl = 0.0;
  } else {
    const int idx = rg_search(g.cdf, g.images, g.u[i - 1]);
    const float ratio = rg_linspace(1.0f, m.lin_end, g.images, idx);
    dist = MIX_DMUL(g.d0, (double)ratio);
    const double a = MIX_DDIV(dist, m.vt);
    const double rr = MIX_DADD(MIX_DMUL(MIX_DMUL(a, a), m.reflect_max), 1.0);
    const double pert = MIX_DMUL(g.pert[i - 1], (double)MIX_D2F(pow((double)ratio, g.tau)));  // float32 pow in torch
    refl = MIX_DADD(rr, pert);
    refl = refl > 1.0 ? refl : 1.0;
  }
  const double p = ceil(MIX_DDIV(MIX_DMUL(dist, m.sample_sr), RG_VELOCITY));
  const double last = (double)(g.comb_len - 1);
  *pos = (int32_t)(p < last ? p : last);
  *val = MIX_D2F(MIX_DDIV(pow(m.coef, refl), dist));
}

// Output j at 8 sr from the sorted entries [e0, e1) of an RIR (positions pos, values val, ties in entry order): the first
// entry inside the window by binary search, then the chain over the last entry of every position in the window
MIX_HD float rg_window(const int32_t *pos, const float *val, int64_t e0, int64_t e1, const float *tab, int64_t j) {
  const int64_t lo = j * RG_O - RG_WIDTH, hi = lo + RG_TAPS - 1;
  int64_t a = e0, b = e1;
  while (a < b) {
    const int64_t mid = a + (b - a) / 2;
    if (pos[mid] < lo) a = mid + 1; else b = mid;
  }
  float acc = 0.0f;
  for (int64_t e = a; e < e1 && pos[e] <= hi; ++e) {
    if (e + 1 < e1 && pos[e + 1] == pos[e]) continue;  // a later entry at this position wins
    acc = RG_FMA(val[e], tab[pos[e] - lo], acc);
  }
  return acc;
}

// One step of the biquad: x0 the input sample, x1 / x2 the previous two, y1 / y2 the previous two unclamped outputs
MIX_HD float rg_biquad_step(const RgRir &g, float x0, float x1, float x2, float y1, float y2) {
  float fir = RG_FMA(x2, g.b2, 0.0f);
  fir = RG_FMA(x1, g.b1, fir);
  fir = RG_FMA(x0, g.b0, fir);
  return RG_FSUB(RG_FSUB(fir, MIX_FMUL(y2, g.a2)), MIX_FMUL(y1, g.a1));
}

MIX_HD float rg_clamp(float y) { return y < -1.0f ? -1.0f : (y > 1.0f ? 1.0f : y); }

// The biquad over an RIR's out_len samples, in place
MIX_HD void rg_biquad(const RgRir &g) {
  float x1 = 0.0f, x2 = 0.0f, y1 = 0.0f, y2 = 0.0f;
  for (int64_t n = 0; n < g.out_len; ++n) {
    const float x0 = g.out[n];
    const float y0 = rg_biquad_step(g, x0, x1, x2, y1, y2);
    g.out[n] = rg_clamp(y0);
    x2 = x1; x1 = x0; y2 = y1; y1 = y0;
  }
}

#ifdef __CUDACC__
MIX_HD int rg_find(const RgRir *g, int n, int64_t x, bool by_cta) {
  int lo = 0, hi = n - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if ((by_cta ? g[mid].cta_begin : g[mid].entry_begin) <= x) lo = mid; else hi = mid - 1;
  }
  return lo;
}

// one thread per entry of every RIR
__global__ void __launch_bounds__(RG_THREADS) rirgen_entry_kernel(const RgRir *__restrict__ rirs, int n, int64_t entries,
                                                                  int32_t *__restrict__ pos, float *__restrict__ val) {
  const int64_t e = (int64_t)blockIdx.x * RG_THREADS + threadIdx.x;
  if (e >= entries) return;
  const RgRir g = rirs[rg_find(rirs, n, e, false)];
  const RgRoom m = rg_room(g);
  rg_entry(g, m, (int)(e - g.entry_begin), pos + e, val + e);
}

// one thread per output sample at 8 sr over the sorted entries
__global__ void __launch_bounds__(RG_THREADS) rirgen_window_kernel(const RgRir *__restrict__ rirs, int n,
                                                                   const int32_t *__restrict__ pos, const float *__restrict__ val,
                                                                   const float *__restrict__ table) {
  __shared__ float tab[RG_TAPS];
  if (threadIdx.x < RG_TAPS) tab[threadIdx.x] = table[threadIdx.x];
  __syncthreads();
  const RgRir g = rirs[rg_find(rirs, n, blockIdx.x, true)];
  const int64_t j = ((int64_t)blockIdx.x - g.cta_begin) * RG_THREADS + threadIdx.x;
  if (j >= g.out_len) return;
  g.out[j] = rg_window(pos, val, g.entry_begin, g.entry_begin + g.images + 1, tab, j);
}

// one thread per RIR, sequential over its samples
__global__ void __launch_bounds__(32) rirgen_biquad_kernel(const RgRir *__restrict__ rirs, int n) {
  const int i = blockIdx.x * 32 + threadIdx.x;
  if (i < n) rg_biquad(rirs[i]);
}
#endif
