// SpecAugment (lhotse.dataset.signal_transforms.SpecAugment) on a padded (B, T, F) float32 feature batch on the GPU, from a
// table of warps and mask rectangles the host planned with lhotse's own random draws (lhotse_b200/spec_augment.py).
//
// The arithmetic contract is DESIGN.md §3.1k.  In short, per sequence b:
//   warp     a segment [start, start + len) with 0 < center, warped < len: output rows [0, warped) are the bicubic resampling
//            of input rows [0, center), rows [warped, len) that of input rows [center, len) (F.interpolate(mode="bicubic",
//            align_corners=False) along time; the feature axis keeps its size, so its interpolation is the identity).  For
//            output row j of a part that maps len_in rows onto len_out rows: scale = f32(len_in) / f32(len_out),
//            src = fma(scale, j + 0.5, -0.5), i0 = floor(src), u = src - i0, taps i0 - 1 .. i0 + 2 clamped to the part, Keys
//            coefficients with A = -0.75, out = fma(w0, x0, fma(w1, x1, fma(w2, x2, w3 * x3))).  Rows outside every segment
//            are copied.  The warp reads `in` and writes `out`, so the disjoint segments of a sequence need no order.
//   mean     the float64 sum of the T * F output values (per thread in unit order, then a fixed tree per CTA, then the CTAs
//            of the sequence in order), divided by T * F, rounded to float32 once
//   masks    rows [start, end) (axis 0) or columns [start, end) of every row (axis 1) are set to the mean
//
// The per-unit, per-tap and per-rectangle arithmetic is __host__ __device__ with explicitly rounded operations, so that
// scripts/micro/specaug_host_check.cu runs exactly this code on the CPU, CTA by CTA, and the device result is bit-identical
// to it.  Kernels at the end.
#pragma once
#include <math.h>
#include <stdint.h>

#include "mix.cuh"

#define SA_THREADS 256
#define SA_TILE_ELEMS 8192  // elements of one sequence a CTA of the warp kernel copies (whole rows: at least one)
#define SA_FILL_THREADS 256

#if defined(__CUDA_ARCH__)
#define SA_FMA(a, b, c) __fmaf_rn(a, b, c)
#else
#define SA_FMA(a, b, c) fmaf(a, b, c)
#endif

// One warped segment as the kernels read it (b200feat_specaug sorts them by sequence and start)
struct SaWarp {
  int32_t start;   // first row of the segment in its sequence
  int32_t len;     // t
  int32_t center;  // input rows [0, center) make output rows [0, warped)
  int32_t warped;
};

// One mask rectangle
struct SaMask {
  int32_t seq;
  int32_t axis;    // 0: rows [start, end) of every column, 1: columns [start, end) of every row
  int32_t start;
  int32_t end;
};

// the four input rows (relative to the segment) and weights of output row j of a warped segment
struct SaTaps {
  int32_t row[4];
  float w[4];
};

MIX_HD int sa_tile_rows(int F) { return F >= SA_TILE_ELEMS ? 1 : SA_TILE_ELEMS / F; }
MIX_HD int sa_tiles(int T, int F) { return (T + sa_tile_rows(F) - 1) / sa_tile_rows(F); }

// Keys' cubic convolution, A = -0.75: |x| <= 1 and 1 < |x| < 2
MIX_HD float sa_cc1(float x) { return SA_FMA(MIX_FMUL(SA_FMA(1.25f, x, -2.25f), x), x, 1.0f); }
MIX_HD float sa_cc2(float x) { return SA_FMA(SA_FMA(SA_FMA(-0.75f, x, 3.75f), x, -6.0f), x, 3.0f); }

MIX_HD SaTaps sa_taps(const SaWarp &w, int j) {
  const bool left = j < w.warped;
  const int len_in = left ? w.center : w.len - w.center, len_out = left ? w.warped : w.len - w.warped;
  const int base = left ? 0 : w.center, jj = left ? j : j - w.warped;
  const float scale = MIX_FDIV((float)len_in, (float)len_out);
  const float src = SA_FMA(scale, (float)jj + 0.5f, -0.5f);
  const float fl = floorf(src);
  const float u = MIX_FADD(src, -fl);  // exact, in [0, 1]
  const int i0 = (int)fl;
  SaTaps t;
  for (int k = 0; k < 4; ++k) {
    int i = i0 - 1 + k;
    i = i < 0 ? 0 : i > len_in - 1 ? len_in - 1 : i;
    t.row[k] = base + i;
  }
  const float v = MIX_FADD(1.0f, -u);
  t.w[0] = sa_cc2(MIX_FADD(u, 1.0f));
  t.w[1] = sa_cc1(u);
  t.w[2] = sa_cc1(v);
  t.w[3] = sa_cc2(MIX_FADD(v, 1.0f));
  return t;
}

MIX_HD float sa_cubic(const SaTaps &t, float x0, float x1, float x2, float x3) {
  return SA_FMA(t.w[0], x0, SA_FMA(t.w[1], x1, SA_FMA(t.w[2], x2, MIX_FMUL(t.w[3], x3))));
}

template <int V>
MIX_HD void sa_load(const float *p, float *v) {
#if defined(__CUDA_ARCH__)
  if constexpr (V == 4) {
    const float4 q = __ldg((const float4 *)p);
    v[0] = q.x; v[1] = q.y; v[2] = q.z; v[3] = q.w;
  } else
#endif
  {
    for (int i = 0; i < V; ++i) v[i] = p[i];
  }
}

template <int V>
MIX_HD void sa_store(float *p, const float *v) {
#if defined(__CUDA_ARCH__)
  if constexpr (V == 4) {
    *(float4 *)p = make_float4(v[0], v[1], v[2], v[3]);
  } else
#endif
  {
    for (int i = 0; i < V; ++i) p[i] = v[i];
  }
}

// Unit `unit` (V consecutive elements of one row; V divides F) of a sequence's tile that starts at row `row0`: writes the
// V output values and returns `acc` plus them, added in element order.  `in` and `out` point at the sequence, warps
// [wb, we) are the sequence's segments.
template <int V>
MIX_HD double sa_unit(const float *in, float *out, int F, const SaWarp *warps, int wb, int we, int row0, int unit, double acc) {
  const int per_row = F / V;
  const int r = row0 + unit / per_row, c = (unit % per_row) * V;
  float v[V];
  int k = wb;
  while (k < we && !(r >= warps[k].start && r < warps[k].start + warps[k].len)) ++k;
  if (k == we) {
    sa_load<V>(in + (int64_t)r * F + c, v);
  } else {
    const SaWarp w = warps[k];
    const SaTaps t = sa_taps(w, r - w.start);
    float x[4][V];
    for (int i = 0; i < 4; ++i) sa_load<V>(in + (int64_t)(w.start + t.row[i]) * F + c, x[i]);
    for (int i = 0; i < V; ++i) v[i] = sa_cubic(t, x[0][i], x[1][i], x[2][i], x[3][i]);
  }
  sa_store<V>(out + (int64_t)r * F + c, v);
  for (int i = 0; i < V; ++i) acc = MIX_DADD(acc, (double)v[i]);
  return acc;
}

// units of tile `tile` of a sequence
MIX_HD int sa_tile_units(int T, int F, int V, int tile) {
  const int R = sa_tile_rows(F), row0 = tile * R;
  return (T - row0 < R ? T - row0 : R) * (F / V);
}

// the mean of a sequence from its CTAs' partial sums, in CTA order
MIX_HD float sa_mean(const double *partial, int tiles, int64_t count) {
  double s = 0.0;
  for (int i = 0; i < tiles; ++i) s = MIX_DADD(s, partial[i]);
  return MIX_D2F(MIX_DDIV(s, (double)count));
}

// T * F < 2^31 (b200feat_specaug checks), so a rectangle's element count and offsets fit an int
MIX_HD int sa_mask_elems(const SaMask &m, int T, int F) { return (m.end - m.start) * (m.axis == 0 ? F : T); }

// element i of a rectangle, as an offset into its sequence
MIX_HD int sa_mask_offset(const SaMask &m, int F, int i) {
  if (m.axis == 0) return m.start * F + i;
  const int w = m.end - m.start;
  return (i / w) * F + m.start + i % w;
}

#ifdef __CUDACC__
// grid (B * tiles): CTA x copies or warps tile x % tiles of sequence x / tiles and leaves the float64 sum of what it wrote.
template <int V>
__global__ void __launch_bounds__(SA_THREADS) specaug_warp_kernel(const float *__restrict__ in, float *__restrict__ out, int T, int F, int tiles,
                                                                  const SaWarp *__restrict__ warps, const int32_t *__restrict__ warp_begin,
                                                                  double *__restrict__ partial) {
  __shared__ double red[SA_THREADS];
  const int b = blockIdx.x / tiles, tile = blockIdx.x - b * tiles;
  const int R = sa_tile_rows(F), row0 = tile * R, row1 = min(row0 + R, T);
  // the sequence's segments that reach into this tile (sorted by start, disjoint)
  int wb = warp_begin[b], we = warp_begin[b + 1];
  while (wb < we && warps[wb].start + warps[wb].len <= row0) ++wb;
  while (we > wb && warps[we - 1].start >= row1) --we;
  const float *src = in + (int64_t)b * T * F;
  float *dst = out + (int64_t)b * T * F;
  const int units = sa_tile_units(T, F, V, tile);
  double acc = 0.0;
  for (int u = threadIdx.x; u < units; u += SA_THREADS) acc = sa_unit<V>(src, dst, F, warps, wb, we, row0, u, acc);
  red[threadIdx.x] = acc;
  __syncthreads();
  for (int w = SA_THREADS / 2; w > 0; w >>= 1) {
    if (threadIdx.x < w) red[threadIdx.x] = __dadd_rn(red[threadIdx.x], red[threadIdx.x + w]);
    __syncthreads();
  }
  if (threadIdx.x == 0) partial[blockIdx.x] = red[0];
}

// one thread per sequence
__global__ void __launch_bounds__(128) specaug_mean_kernel(const double *__restrict__ partial, int B, int tiles, int64_t count,
                                                           float *__restrict__ mean) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b < B) mean[b] = sa_mean(partial + (int64_t)b * tiles, tiles, count);
}

// grid (masks, y): the rectangle's elements, strided over y
__global__ void __launch_bounds__(SA_FILL_THREADS) specaug_fill_kernel(float *__restrict__ out, int T, int F, const SaMask *__restrict__ masks,
                                                                       const float *__restrict__ mean) {
  const SaMask m = masks[blockIdx.x];
  const float v = mean[m.seq];
  float *dst = out + (int64_t)m.seq * T * F;
  const int n = sa_mask_elems(m, T, F);
  for (int i = blockIdx.y * SA_FILL_THREADS + threadIdx.x; i < n; i += gridDim.y * SA_FILL_THREADS)
    dst[sa_mask_offset(m, F, i)] = v;
}
#endif
