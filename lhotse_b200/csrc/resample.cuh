// Resampling and volume scaling of mono audio (lhotse's Speed, Resample and Volume transforms) on the GPU, bit-identical to
// lhotse's CPU route wherever torch runs the resampler's conv1d through oneDNN.
//
// The arithmetic contract is DESIGN.md §3.1i.  In short, per resampling stage of a rate pair reduced to O -> N:
//   table    kernel[N][K], K = 2 * width + O, float32 (built on the host in float64 and rounded once, as lhotse builds it);
//            the device keeps it transposed, [K][N], so that the N phases of one tap are adjacent
//   input    the stage's segment x[0, L), zero-padded by `width` samples on the left and width + O on the right
//   output   j = b * N + p is ONE float32 FMA chain over all K taps in tap order, starting from +0:
//              acc = fma(xpad[b * O + t], kernel[p][t], acc),  t = 0 .. K - 1
//            (pad taps are real FMAs with +0, so signed zeros come out as on the CPU); lhotse's count of outputs
//            is kept: ceil of the float32-rounded N * L / O (b200feat.h, b200feat_resample_stage.out_len)
//   volume   f32(x * f32(factor)) at its place in the chain: a load scale before the resampler, a store scale after it
//   last     the cut's final stage is trimmed or reflect-padded to the cut's length (mix_source_pos, as the mix kernel does)
//
// The per-sample arithmetic is __host__ __device__ so that scripts/micro/resample_host_check.cu runs exactly this code on
// the CPU.  The kernel is at the end.
#pragma once
#include <math.h>
#include <stdint.h>

#include "mix.cuh"

#define RS_THREADS 256
#define RS_CHUNK 1024          // target outputs per CTA
#define RS_WIN_FLOATS 8192     // the input window a CTA stages in shared memory, at most (K + O <= this, checked per table)
#define RS_SMEM_TAB_FLOATS 2048  // a table of at most this many floats is staged in shared memory too

#if defined(__CUDA_ARCH__)
#define RS_FMA(a, b, c) __fmaf_rn(a, b, c)
#else
#define RS_FMA(a, b, c) fmaf(a, b, c)
#endif

// One stage of one cut as the kernel reads it (b200feat_resample builds these from the b200feat_resample_stage records)
struct RsStage {
  const float *tab;      // [K][N] table, nullptr: no resampling (the scales only)
  const int16_t *src16;  // the stage's input: int16 samples (widened as B200FEAT_I16 does) ...
  const float *src32;    // ... or float32 samples (exactly one of the two is set)
  float *dst;            // the stage's first output sample
  int64_t in_len;        // L
  int64_t out_len;       // the outputs lhotse keeps (b200feat_resample_stage.out_len), L without a table
  int64_t target_len;    // samples written: out_len, fewer (trim) or at most out_len - 1 more (reflect-pad)
  int64_t cta_begin;     // first CTA of the stage in its launch
  int32_t N, O, K, width;
  int32_t chunk;         // outputs per CTA: a multiple of N, so that the CTAs of the unpadded part start on a block
  int32_t tab_smem;      // 1: the CTA copies the table to shared memory
  float scale_in, scale_out;
};

// Outputs per CTA of a stage: about RS_CHUNK, a whole number nb of blocks, and an input window (nb * O + K floats, the extra
// block of a reflect chunk that does not start on a block included) of at most RS_WIN_FLOATS
MIX_HD int32_t rs_chunk_outputs(int32_t N, int32_t O, int32_t K) {
  int64_t nb = RS_CHUNK / N > 1 ? RS_CHUNK / N : 1;
  if (nb > (RS_WIN_FLOATS - K) / O) nb = (RS_WIN_FLOATS - K) / O;
  return (int32_t)((nb > 1 ? nb : 1) * N);
}

// shared memory of a CTA of a resampling stage: the table when it is small, then the input window
MIX_HD int64_t rs_smem_floats(const RsStage &s) {
  return (s.tab_smem ? (int64_t)s.N * s.K : 0) + (int64_t)s.chunk / s.N * s.O + s.K;
}

MIX_HD int64_t rs_natural_ctas(const RsStage &s) {
  const int64_t n = s.target_len < s.out_len ? s.target_len : s.out_len;
  return (n + s.chunk - 1) / s.chunk;
}

// CTAs of a stage: its outputs [0, min(target, out_len)) in chunks, then the reflect-padded tail [out_len, target) in chunks
MIX_HD int64_t rs_stage_ctas(const RsStage &s) {
  const int64_t pad = s.target_len > s.out_len ? s.target_len - s.out_len : 0;
  return rs_natural_ctas(s) + (pad + s.chunk - 1) / s.chunk;
}

// the written positions [*p0, *p1) of CTA c of the stage
MIX_HD void rs_chunk(const RsStage &s, int64_t c, int64_t *p0, int64_t *p1) {
  const int64_t nat = rs_natural_ctas(s);
  const int64_t end_nat = s.target_len < s.out_len ? s.target_len : s.out_len;
  if (c < nat) {
    *p0 = c * s.chunk;
    *p1 = *p0 + s.chunk < end_nat ? *p0 + s.chunk : end_nat;
  } else {
    *p0 = s.out_len + (c - nat) * s.chunk;
    *p1 = *p0 + s.chunk < s.target_len ? *p0 + s.chunk : s.target_len;
  }
}

// Input sample i of the stage after its load scale; +0 outside [0, L) (the zero padding, which Volume never sees)
MIX_HD float rs_load(const RsStage &s, int64_t i) {
  if (i < 0 || i >= s.in_len) return 0.0f;
  const float x = s.src16 ? mix_widen(s.src16[i]) : s.src32[i];
  return MIX_FMUL(x, s.scale_in);
}

// Output phase p of the block whose padded input starts at `win` (win[t] = xpad[b * O + t]); tab is [K][N]
MIX_HD float rs_output(const float *win, const float *tab, int N, int K, int p) {
  float acc = 0.0f;
  for (int t = 0; t < K; ++t) acc = RS_FMA(win[t], tab[(int64_t)t * N + p], acc);
  return acc;
}

// The padded-input window CTA positions [p0, p1) need: blocks [*b_lo, *b_hi] (its size is (b_hi - b_lo) * O + K)
MIX_HD void rs_window(const RsStage &s, int64_t p0, int64_t p1, int64_t *b_lo, int64_t *b_hi) {
  const int64_t a = mix_source_pos(p0, s.out_len), b = mix_source_pos(p1 - 1, s.out_len);
  *b_lo = (a < b ? a : b) / s.N;
  *b_hi = (a < b ? b : a) / s.N;
}

#ifdef __CUDACC__
// One launch per stage depth over every cut that has a stage at that depth; the CTA finds its stage by binary search over
// cta_begin.  A CTA stages its input window (load scale applied) in shared memory, so every input sample is read from
// HBM once; the N phases of a block sit on adjacent threads and share that window.
__global__ void __launch_bounds__(RS_THREADS) resample_stage_kernel(const RsStage *__restrict__ stages, int nstages) {
  extern __shared__ float rs_smem[];
  int lo = 0, hi = nstages - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (stages[mid].cta_begin <= (int64_t)blockIdx.x) lo = mid; else hi = mid - 1;
  }
  const RsStage s = stages[lo];
  int64_t p0, p1;
  rs_chunk(s, (int64_t)blockIdx.x - s.cta_begin, &p0, &p1);
  if (!s.tab) {  // scales only: out = f32(f32(x * scale_in) * scale_out)
    for (int64_t p = p0 + threadIdx.x; p < p1; p += RS_THREADS)
      s.dst[p] = MIX_FMUL(rs_load(s, mix_source_pos(p, s.out_len)), s.scale_out);
    return;
  }
  int64_t b_lo, b_hi;
  rs_window(s, p0, p1, &b_lo, &b_hi);
  const int W = (int)((b_hi - b_lo) * s.O + s.K);
  const int tab_floats = s.tab_smem ? s.N * s.K : 0;
  float *win = rs_smem + tab_floats;
  const int64_t first = b_lo * s.O - s.width;  // input index of win[0]
  for (int i = threadIdx.x; i < W; i += RS_THREADS) win[i] = rs_load(s, first + i);
  for (int i = threadIdx.x; i < tab_floats; i += RS_THREADS) rs_smem[i] = s.tab[i];
  __syncthreads();
  const float *tab = s.tab_smem ? rs_smem : s.tab;
  for (int64_t p = p0 + threadIdx.x; p < p1; p += RS_THREADS) {
    const int64_t j = mix_source_pos(p, s.out_len);
    const int64_t b = j / s.N;
    s.dst[p] = MIX_FMUL(rs_output(win + (b - b_lo) * s.O, tab, s.N, s.K, (int)(j - b * s.N)), s.scale_out);
  }
}
#endif
