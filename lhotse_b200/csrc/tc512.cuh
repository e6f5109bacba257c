// Tensor-core kernel for fft_length N = 512 (kernel = "tc"): the 512-point real DFT of every frame is a two-stage
// Cooley-Tukey factorisation 512 = 32 x 16 whose two stages are GEMMs on the Hopper tensor cores
// (wgmma.mma_async .tf32, fp32 accumulators in registers), made fp32-accurate by the 3xTF32 split
//     A*B ~= A_hi*B_hi + (A_hi*B_lo + A_lo*B_hi),   x_hi = rna_tf32(x),  x_lo = rna_tf32(x - x_hi).
//
//   sample n = 16*n1 + n2 of the pre-processed frame v (n1 = 0..31, zero for n >= L; n2 = 0..15), bin k = k1 + 32*k2:
//     stage 1   Y[n2][k1]  = sum_n1 v[16 n1 + n2] * W32^(n1 k1)          k1 = 0..16 (real input: the rest is the conjugate)
//     twiddle   Y'[n2][k1] = Y[n2][k1] * W512^(n2 k1)                     (CUDA cores, between the two GEMMs)
//     stage 2   X[k1 + 32 k2] = sum_n2 Y'[n2][k1] * W16^(n2 k2)           k2 = 0..15; k2 >= 8 is conj X[512 - k]
//
//   GEMM 1:  D1[(frame, n2)][.] = A1[(frame, n2)][n1 = 0..31] * B1[n1][.]
//            B1 columns: {Re Y0, Y16, Re Y1, Im Y1, ..., Re Y15, Im Y15} (Im Y0 = Im Y16 = 0).
//   GEMM 2:  D2[(frame, k1)][.] = A2[(frame, k1 = 0..15)][(n2, re/im)] * B2[(n2, re/im)][(k2, re/im)]
//            the k1 = 16 column (bins 16 + 32 k2, 8 of the 257) is a 16-tap real-input DFT done on CUDA cores.
//   Per K-step two instructions: A_hi x [B_hi | B_lo] (N = 64: columns 0..31 hi*hi, 32..63 hi*lo) and A_lo x B_hi (N = 32,
//   its own accumulator); the epilogue adds hi*hi + (hi*lo + lo*hi).
//
// wgmma takes tf32 operands from shared memory only in K-major order, and the frame is MN-major for GEMM 1 (consecutive
// samples are consecutive rows), so both A operands come from registers: every warp stages its frame (GEMM 1) or its
// twiddled stage-1 output (GEMM 2) in shared memory and loads the m64k8 fragments from there, splitting hi / lo on the
// way.  B1 and B2 (hi and lo) are K-major 128-byte-swizzled images in shared memory, fetched once per CTA by one bulk
// asynchronous copy (TMA) completing on an mbarrier.
//
// A tile is 8 consecutive frames of one cut.  A CTA is two warpgroups; warpgroup w computes frames 4 w .. 4 w + 3 of every
// tile of the CTA's contiguous tile range, one frame per warp: rows 16 q .. 16 q + 15 of an m64 operand belong to warp q,
// so between the warpgroup-wide MMAs a warp only ever exchanges data with itself.  A warp's tile step:
//   PRE    global (next tile's frame prefetched into registers) -> DC removal, pre-emphasis, window (layers.py:151-186) -> V
//   GEMM 1 V -> A1 fragments -> D1 (registers) -> twiddle -> Y' (shared), Y16
//   GEMM 2 Y' -> A2 fragments -> D2 -> |X|^2 -> P[bin] (layers.py:38-42) + the k1 = 16 bins from Y16
//   MEL    lane = filter: P x mel weights (layers.py:565-578) -> log -> the output row (or DCT + lifter for MFCC, :708-724)
// Several CTAs share an SM, so one warpgroup's global loads and MMAs overlap another's CUDA-core work.
// HBM traffic: 4*S bytes in (the frame overlap is served by L1/L2), 4*F bytes out per frame; no intermediate leaves the SM.
#pragma once
#include <string.h>

#include <algorithm>
#include <vector>

#include "common.cuh"

#define TC_NF 8                      // frames per tile
#define TC_THREADS 256               // two warpgroups, one frame per warp
#define TC_PP 260                    // floats per P row (257 bins + zeroed pad a 128-bit mel load may touch)
#define TC_VS 24                     // floats per 16-sample row of a staged frame (16 + 8 pad: the A1 fragment loads of a
                                     // warp hit 32 distinct banks)
#define TC_YS 36                     // floats per k1 row of Y' (32 + 4 pad: the A2 fragment loads hit 32 distinct banks)

struct Tc512Tables {
  const void *cblob;      // [B1hi 4K][B1lo 4K][B2hi 4K][B2lo 4K][tw 2K][mel descriptors][mel weights]
  int cblob_bytes;
  int off_tw, off_md, off_mw;  // byte offsets inside the blob
  int fpu;                // filters per unit = ceil(M / 16)
  int Mpad;               // M rounded up to 4
  int warp_bytes;         // shared memory of one warp: V, Y', P, Y16, log-mel row
  const float *win4;      // [512] window, zero beyond L
  const float *c16;       // [16][16]: cos / -sin of 2 pi n2 (1 + 2 k2) / 32 at [2 k2 + part][n2] (the k1 = 16 column)
};

// tf32 (10 explicit mantissa bits) nearest to x, in an fp32 container.  hi = rna(x) and lo = rna(x - hi) leave a
// representation error of 2^-24 |x| (masking the low bits instead would leave 2^-22: the tensor core truncates whatever it is
// given), which keeps bins 70 dB under a frame's peak within the fp32 reference's tolerance.
__device__ __forceinline__ float tc_hi(float x) {
  uint32_t u;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(u) : "f"(x));
  return __uint_as_float(u);
}
// hi / lo tf32 parts of four fragment elements
__device__ __forceinline__ void tc_split4(const float (&x)[4], uint32_t (&hi)[4], uint32_t (&lo)[4]) {
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float h = tc_hi(x[i]);
    hi[i] = __float_as_uint(h);
    lo[i] = __float_as_uint(tc_hi(x[i] - h));
  }
}

// wgmma shared-memory matrix descriptor of a K-major operand in the 128-byte swizzle: start >> 4 | LBO (unused: 1) << 16 |
// SBO (1024 B between 8-row groups) >> 4 << 32 | layout 1 (SWIZZLE_128B) << 62.  A K-step of 8 tf32 advances the start by 32 B.
__device__ __forceinline__ uint64_t tc_desc_k128(uint32_t saddr) {
  return (uint64_t)((saddr >> 4) & 0x3FFF) | (1ull << 16) | ((uint64_t)(1024 >> 4) << 32) | (1ull << 62);
}
// m64nNk8 tf32 MMAs, A from registers (fragment of lane l in warp q: rows 16 q + l / 4 (+ 8), columns l % 4 (+ 4)),
// fp32 accumulator d (lane l of warp q holds rows 16 q + l / 4 (+ 8) and columns 8 j + 2 (l % 4) (+ 1))
__device__ __forceinline__ void tc_wgmma_n64(float (&d)[32], const uint32_t (&a)[4], uint64_t bdesc, uint32_t accumulate) {
  asm volatile("{ .reg .pred p; setp.ne.b32 p, %37, 0;\n"
               "  wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}, {%32,%33,%34,%35}, %36, p, 1, 1; }\n"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bdesc), "r"(accumulate));
}
__device__ __forceinline__ void tc_wgmma_n32(float (&d)[16], const uint32_t (&a)[4], uint64_t bdesc, uint32_t accumulate) {
  asm volatile("{ .reg .pred p; setp.ne.b32 p, %21, 0;\n"
               "  wgmma.mma_async.sync.aligned.m64n32k8.f32.tf32.tf32 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15}, {%16,%17,%18,%19}, %20, p, 1, 1; }\n"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bdesc), "r"(accumulate));
}
__device__ __forceinline__ void tc_wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void tc_wgmma_commit_wait() {
  asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory");
  asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory");
}
// keeps the compiler from moving accesses of accumulator registers across the wgmma fence / wait above
template <int N>
__device__ __forceinline__ void tc_pin(float (&d)[N]) {
#pragma unroll
  for (int i = 0; i < N; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

template <int DT>
__device__ __forceinline__ float4 tc_ld_chunk(const void *base, int64_t i) {  // 4 consecutive samples, i % 4 == 0, aligned
  if (DT == B200FEAT_I16) {
    const short4 q = __ldg(reinterpret_cast<const short4 *>(reinterpret_cast<const int16_t *>(base) + i));
    const float k = 1.0f / 32768.0f;
    return make_float4((float)q.x * k, (float)q.y * k, (float)q.z * k, (float)q.w * k);
  } else {
    return __ldg(reinterpret_cast<const float4 *>(reinterpret_cast<const float *>(base) + i));
  }
}

struct TcTile {
  int64_t t0, T, n, xoff, row0;
  int nv, nrows;
};
// A CTA walks a CONTIGUOUS range of tiles (consecutive tiles of a cut share 240 of their samples: the re-reads hit this
// SM's L1), so the per-cut metadata is reloaded only when the walk crosses into the next cut.
struct TcCut {
  int cut;
  int64_t tile_lo, tile_hi, T, n, xoff, row_base;
};
__device__ __forceinline__ void tc_load_cut(const DevBatch &b, int cut, TcCut &m) {
  m.cut = cut;
  m.tile_lo = __ldg(b.tile_off + cut);
  m.tile_hi = __ldg(b.tile_off + cut + 1);
  const int64_t r0 = __ldg(b.row_off + cut);
  m.T = __ldg(b.row_off + cut + 1) - r0;
  m.n = __ldg(b.nsamp + cut);
  m.xoff = __ldg(b.samp_off + cut);
  m.row_base = b.out_mode == B200FEAT_OUT_PADDED ? (int64_t)(b.batch_first + cut) * b.max_frames : r0;
}
__device__ __forceinline__ void tc_first_cut(const DevBatch &b, int64_t tile, TcCut &m) {
  tc_load_cut(b, __ldg(b.tile_cut + tile) - b.batch_first, m);
}
__device__ __forceinline__ TcTile tc_tile(const DevBatch &b, TcCut &m, int64_t tile) {  // tiles are visited in increasing order
  while (tile >= m.tile_hi) tc_load_cut(b, m.cut + 1, m);
  TcTile t;
  t.t0 = (tile - m.tile_lo) * TC_NF;
  t.T = m.T; t.n = m.n; t.xoff = m.xoff;
  const int64_t rows_here = b.out_mode == B200FEAT_OUT_PADDED ? b.max_frames : m.T;
  t.nv = (int)max((int64_t)0, min((int64_t)TC_NF, m.T - t.t0));
  t.nrows = (int)max((int64_t)0, min((int64_t)TC_NF, rows_here - t.t0));
  t.row0 = m.row_base + t.t0;
  return t;
}

template <int DT>
__global__ void __launch_bounds__(TC_THREADS, 2)
b200feat_tc512_kernel(const DevPlan p, const Tc512Tables tt, const DevBatch b) {
  extern __shared__ unsigned char tc_smem_raw[];
  // the swizzled B images need a 1024-byte-aligned base (the launch reserves the slack)
  unsigned char *sC = tc_smem_raw + ((1024u - (smem_u32(tc_smem_raw) & 1023u)) & 1023u);
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int f = warp;                            // this warp's frame in every tile (warpgroup warp / 4 owns frames 4 (warp / 4) ..)
  const int g = lane >> 2, tq = lane & 3;        // fragment row (and row + 8) / fragment column (and column + 4)
  const uint32_t bar0 = smem_u32(sC + tt.cblob_bytes);
  float *V = reinterpret_cast<float *>(sC + tt.cblob_bytes + 16 + (size_t)warp * tt.warp_bytes);  // [32 n1][TC_VS]
  float *Yp = V + 32 * TC_VS;                    // [16 k1][TC_YS]: (Re, Im) Y'[n2][k1] at 2 n2
  float *Pf = Yp + 16 * TC_YS;                   // [TC_PP]
  float *Y16 = Pf + TC_PP;                       // [16]
  float *E = Y16 + 16;                           // [Mpad]

  blob_copy_start(bar0, sC, tt.cblob, tt.cblob_bytes);  // constant tables: one TMA bulk copy
  mbar_wait(bar0, 0);
  const int64_t tile_begin = b.tile_base + b.num_tiles * (int64_t)blockIdx.x / gridDim.x;
  const int64_t my_tiles = b.tile_base + b.num_tiles * (int64_t)(blockIdx.x + 1) / gridDim.x - tile_begin;

  const uint32_t cb = smem_u32(sC);
  const float2 *s_tw = reinterpret_cast<const float2 *>(sC + tt.off_tw);  // [k1 - 1][n2]: W512^(n2 k1), k1 = 1..16
  const int4 *s_md = reinterpret_cast<const int4 *>(sC + tt.off_md);      // [unit][slot] {first bin, float4 groups, weight index, filter}
  const float4 *s_mw4 = reinterpret_cast<const float4 *>(sC + tt.off_mw);
  const float lgk = p.log10_mel ? 0.30102999566398119521f : 0.69314718055994530942f;
  const int L = p.L, NCH = (L + 3) >> 2;
  const float inv_L = 1.0f / (float)L, pre = p.preemph;
  const int pad = p.snip_edges ? 0 : p.pad_left;
  float4 wreg[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) wreg[j] = __ldg(reinterpret_cast<const float4 *>(tt.win4) + lane + 32 * j);
  const float4 *c16 = reinterpret_cast<const float4 *>(tt.c16) + (lane & 15) * 4;  // row o = lane % 16: 2 k2 + part, part 0 = Re (cos), 1 = Im (-sin)

  float4 xn[4];
  bool inn = false;
  auto fetch = [&](const TcTile &t) {  // interior frames: 4 vector loads per lane, issued early; edge frames are gathered later
    const int64_t sb = (t.t0 + f) * p.S - pad;
    inn = f < t.nv && sb >= 0 && sb + 4 * NCH <= t.n && (((t.xoff + sb) & 3) == 0);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int c = lane + 32 * j;
      xn[j] = (inn && c < NCH) ? tc_ld_chunk<DT>(b.samples, t.xoff + sb + 4 * c) : make_float4(0.f, 0.f, 0.f, 0.f);
    }
  };
  TcTile cur{};
  TcCut cm{};
  if (my_tiles > 0) { tc_first_cut(b, tile_begin, cm); cur = tc_tile(b, cm, tile_begin); fetch(cur); }
  for (int64_t it = 0; it < my_tiles; ++it) {
    float4 x[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) x[j] = xn[j];
    const bool in = inn;
    const TcTile t = cur;
    if (it + 1 < my_tiles) { cur = tc_tile(b, cm, tile_begin + it + 1); fetch(cur); }  // next tile's samples fly while this one is processed

    // ---------------------------------------------------------------- PRE: frame f -> V (missing frames: zeros)
    if (f < t.nv && !in) {  // cut edge (or an unaligned cut): per-sample reflection (layers.py:753-772)
      const int64_t sb = (t.t0 + f) * p.S - pad;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int c = lane + 32 * j;
        float e[4];
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const int i = 4 * c + q;
          e[q] = 0.f;
          if (i < L) {
            int64_t s = sb + i;
            if (!p.snip_edges) s = reflect_index(s, t.n, p.pad_mode);
            e[q] = ld_sample<DT>(b.samples, t.xoff + s);
          }
        }
        x[j] = make_float4(e[0], e[1], e[2], e[3]);
      }
    }
    if (L & 3) {  // taps >= L inside the last chunk are not part of the frame
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int i0 = 4 * (lane + 32 * j);
        if (i0 + 1 >= L) x[j].y = 0.f;
        if (i0 + 2 >= L) x[j].z = 0.f;
        if (i0 + 3 >= L) x[j].w = 0.f;
      }
    }
    {
      // the tap before chunk c is the last tap of chunk c - 1: the neighbour lane's .w (lane 0: lane 31 of the round before)
      float pv[4];
      float last = x[0].x;  // lane 0, chunk 0: replicate-left (layers.py:166)
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float up = __shfl_up_sync(0xffffffffu, x[j].w, 1);
        pv[j] = lane == 0 ? last : up;
        last = __shfl_sync(0xffffffffu, x[j].w, 31);
      }
      float s = 0.f;
#pragma unroll
      for (int j = 0; j < 4; ++j) s += (x[j].x + x[j].y) + (x[j].z + x[j].w);
      const float mu = p.remove_dc ? warp_sum(s) * inv_L : 0.f;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float d0 = x[j].x - mu, d1 = x[j].y - mu, d2 = x[j].z - mu, d3 = x[j].w - mu, dp = pv[j] - mu;
        float4 v;
        v.x = fmaf(-pre, dp, d0) * wreg[j].x;
        v.y = fmaf(-pre, d0, d1) * wreg[j].y;
        v.z = fmaf(-pre, d1, d2) * wreg[j].z;
        v.w = fmaf(-pre, d2, d3) * wreg[j].w;
        const int c = lane + 32 * j;
        if (c >= NCH || f >= t.nv) v = make_float4(0.f, 0.f, 0.f, 0.f);  // K-rows beyond the frame are exact zeros
        *reinterpret_cast<float4 *>(V + (c >> 2) * TC_VS + 4 * (c & 3)) = v;
      }
    }
    __syncwarp();

    // ---------------------------------------------------------------- GEMM 1: rows (frame f, n2 = g / g + 8), K = n1
    float d1[32], e1[16];
    {
      uint32_t ah[4][4], al[4][4];
#pragma unroll
      for (int ks = 0; ks < 4; ++ks) {
        const float *v0 = V + (8 * ks + tq) * TC_VS + g, *v4 = v0 + 4 * TC_VS;
        const float a[4] = {v0[0], v0[8], v4[0], v4[8]};
        tc_split4(a, ah[ks], al[ks]);
      }
      tc_wgmma_fence();
#pragma unroll
      for (int ks = 0; ks < 4; ++ks) {
        const uint64_t db = tc_desc_k128(cb + ks * 32);  // rows 0..31 B1_hi, 32..63 B1_lo
        tc_wgmma_n64(d1, ah[ks], db, ks ? 1u : 0u);     // [hi*hi | hi*lo]
        tc_wgmma_n32(e1, al[ks], db, ks ? 1u : 0u);     // lo*hi
      }
      tc_wgmma_commit_wait();
      tc_pin(d1);
      tc_pin(e1);
    }
    // twiddle: lane holds Y[n2][k1] for n2 = g + 8 r, k1 = 4 j + tq (columns 2 k1, 2 k1 + 1)
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      const int n2 = g + 8 * r;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int k1 = 4 * j + tq, i = 4 * j + 2 * r;
        const float a = d1[i] + (d1[16 + i] + e1[i]), bq = d1[i + 1] + (d1[17 + i] + e1[i + 1]);
        float yr, yi;
        if (k1 == 0) { yr = a; yi = 0.f; Y16[n2] = bq; }  // the k1 = 16 column (real): finished on CUDA cores below
        else {
          const float2 w = s_tw[(k1 - 1) * 16 + n2];
          yr = fmaf(a, w.x, -bq * w.y);
          yi = fmaf(a, w.y, bq * w.x);
        }
        *reinterpret_cast<float2 *>(Yp + k1 * TC_YS + 2 * n2) = make_float2(yr, yi);
      }
    }
    __syncwarp();

    // ---------------------------------------------------------------- GEMM 2: rows (frame f, k1 = g / g + 8), K = (n2, re/im)
    float d2[32], e2[16];
    {
      uint32_t ah[4][4], al[4][4];
#pragma unroll
      for (int ks = 0; ks < 4; ++ks) {
        const float *y0 = Yp + g * TC_YS + 8 * ks + tq, *y8 = y0 + 8 * TC_YS;
        const float a[4] = {y0[0], y8[0], y0[4], y8[4]};
        tc_split4(a, ah[ks], al[ks]);
      }
      tc_wgmma_fence();
#pragma unroll
      for (int ks = 0; ks < 4; ++ks) {
        const uint64_t db = tc_desc_k128(cb + 8192 + ks * 32);  // rows 0..31 B2_hi, 32..63 B2_lo
        tc_wgmma_n64(d2, ah[ks], db, ks ? 1u : 0u);
        tc_wgmma_n32(e2, al[ks], db, ks ? 1u : 0u);
      }
      tc_wgmma_commit_wait();
      tc_pin(d2);
      tc_pin(e2);
    }
    // power: lane holds X[k1 + 32 k2] for k1 = g + 8 r, k2 = 4 j + tq
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      const int k1 = g + 8 * r;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int k2 = 4 * j + tq, i = 4 * j + 2 * r;
        const float re = d2[i] + (d2[16 + i] + e2[i]), im = d2[i + 1] + (d2[17 + i] + e2[i + 1]);
        float pw = fmaf(re, re, im * im);
        if (p.use_mag) pw = sqrtf(pw);
        const int bin = k2 < 8 ? k1 + 32 * k2 : 512 - k1 - 32 * k2;
        if (k1 != 0 || k2 <= 8) Pf[k1 == 0 ? 32 * k2 : bin] = pw;
      }
    }
    {  // bins 16 + 32 k2: lane o = lane % 16 computes part o % 2 of k2 = o / 2
      float v16 = 0.f;
      const float4 *y = reinterpret_cast<const float4 *>(Y16);
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const float4 a = y[q], c = __ldg(c16 + q);
        v16 = fmaf(a.x, c.x, fmaf(a.y, c.y, fmaf(a.z, c.z, fmaf(a.w, c.w, v16))));
      }
      const float o = __shfl_xor_sync(0xffffffffu, v16, 1);
      float pw = fmaf(v16, v16, o * o);
      if (p.use_mag) pw = sqrtf(pw);
      if (lane < 16 && (lane & 1) == 0) Pf[16 + 32 * (lane >> 1)] = pw;
      if (lane == 0) Pf[257] = Pf[258] = Pf[259] = 0.f;  // row padding a 128-bit mel load may touch (weight 0): never stale NaNs
    }
    __syncwarp();

    // ---------------------------------------------------------------- MEL: lane = filter (unit-major descriptor order)
    for (int idx = lane; idx < 16 * tt.fpu; idx += 32) {
      const int4 md = s_md[idx];
      if (md.w < 0) continue;
      const float4 *pp = reinterpret_cast<const float4 *>(Pf + md.x);
      const float4 *wp = s_mw4 + md.z;
      float a0 = 0.f, a1 = 0.f;
      int i = 0;
      for (; i + 1 < md.y; i += 2) {  // two independent chains
        const float4 w0 = wp[i], q0 = pp[i], w1 = wp[i + 1], q1 = pp[i + 1];
        a0 = fmaf(q0.w, w0.w, fmaf(q0.z, w0.z, fmaf(q0.y, w0.y, fmaf(q0.x, w0.x, a0))));
        a1 = fmaf(q1.w, w1.w, fmaf(q1.z, w1.z, fmaf(q1.y, w1.y, fmaf(q1.x, w1.x, a1))));
      }
      if (i < md.y) {
        const float4 w0 = wp[i], q0 = pp[i];
        a0 = fmaf(q0.w, w0.w, fmaf(q0.z, w0.z, fmaf(q0.y, w0.y, fmaf(q0.x, w0.x, a0))));
      }
      E[md.w] = fast_lg2_normal(nanmax(a0 + a1, p.mel_floor)) * lgk;
    }
    __syncwarp();
    float *out = b.out + (t.row0 + f) * p.F;
    if (f < t.nv) {
      if (p.feature == B200FEAT_MFCC) {
        for (int c = lane; c < p.C; c += 32) {
          float acc = 0.f;
          for (int m = 0; m < p.M; ++m) acc = fmaf(E[m], __ldg(p.dct + m * p.C + c), acc);
          if (p.use_lifter) acc *= __ldg(p.lifter + c);
          out[c] = post_affine(p, c, acc);
        }
      } else {
        for (int m = lane; m < p.M; m += 32) out[m] = post_affine(p, m, E[m]);
      }
    } else if (f < t.nrows) {
      for (int i = lane; i < p.F; i += 32) out[i] = post_affine(p, i, b.pad_value);
    }
  }
}

// ---------------------------------------------------------------------------------------------- host
struct Tc512Host {
  Tc512Tables t;
  size_t smem;
  int ctas_per_sm;  // resident CTAs per SM (the persistent grid is this many per SM)
};

static inline bool tc512_supported(const DevPlan &p) {
  return p.N == 512 && p.L >= 16 && p.L <= 512 && (p.feature == B200FEAT_FBANK || p.feature == B200FEAT_MFCC) && !p.use_energy &&
         p.pad_mode == B200FEAT_PAD_KALDI && p.M >= 1 && p.M <= 128 && p.C <= 128;
}

// element (row, k) of a K-major 128-byte-swizzle operand with 32 fp32 per row (one 128-byte row per matrix row), in floats
static inline int tc_k128_index(int row, int k) { return (row >> 3) * 256 + (row & 7) * 32 + ((((k >> 2) ^ (row & 7)) & 7) << 2) + (k & 3); }

static inline float tc_hi_host(float x) {  // cvt.rna.tf32.f32: round to nearest, ties away from zero, on the magnitude bits
  uint32_t u;
  memcpy(&u, &x, 4);
  u = (u + 0x1000u) & 0xFFFFE000u;
  float r;
  memcpy(&r, &u, 4);
  return r;
}

// host images of the constant tables
struct Tc512Image {
  ConstBlob blob;
  std::vector<float> win4, c16;
  int off_tw = 0, off_md = 0, off_mw = 0, fpu = 0, Mpad = 0;
};

static inline int tc512_build_image(const DevPlan &p, const std::vector<float> &bank, const std::vector<float> &window, Tc512Image *img) {
  std::vector<float> b1(32 * 32), b2(32 * 32);  // logical [col][k]
  for (int n1 = 0; n1 < 32; ++n1) {
    b1[0 * 32 + n1] = 1.f;
    b1[1 * 32 + n1] = (n1 & 1) ? -1.f : 1.f;
    for (int k1 = 1; k1 < 16; ++k1) {
      const double a = 2.0 * M_PI * (double)((n1 * k1) % 32) / 32.0;
      b1[(2 * k1) * 32 + n1] = (float)cos(a);
      b1[(2 * k1 + 1) * 32 + n1] = (float)(-sin(a));
    }
  }
  for (int n2 = 0; n2 < 16; ++n2)
    for (int k2 = 0; k2 < 16; ++k2) {
      const double a = 2.0 * M_PI * (double)((n2 * k2) % 16) / 16.0;
      const float c = (float)cos(a), s = (float)sin(a);
      b2[(2 * k2) * 32 + 2 * n2] = c;       // Re X += Re Y' * cos
      b2[(2 * k2) * 32 + 2 * n2 + 1] = s;   //        + Im Y' * sin
      b2[(2 * k2 + 1) * 32 + 2 * n2] = -s;  // Im X += -Re Y' * sin
      b2[(2 * k2 + 1) * 32 + 2 * n2 + 1] = c;
    }
  std::vector<float> img4(4 * 1024, 0.f);  // B1hi | B1lo | B2hi | B2lo, each 32 rows x 128 B swizzled
  for (int c = 0; c < 32; ++c)
    for (int k = 0; k < 32; ++k) {
      const int idx = tc_k128_index(c, k);
      const float v1 = b1[c * 32 + k], h1 = tc_hi_host(v1);
      img4[idx] = h1; img4[1024 + idx] = tc_hi_host(v1 - h1);
      const float v2 = b2[c * 32 + k], h2 = tc_hi_host(v2);
      img4[2048 + idx] = h2; img4[3072 + idx] = tc_hi_host(v2 - h2);
    }
  std::vector<float2> tw(256);  // [k1 - 1][n2]
  for (int k1 = 1; k1 <= 16; ++k1)
    for (int n2 = 0; n2 < 16; ++n2) {
      const double a = -2.0 * M_PI * (double)((n2 * k1) % 512) / 512.0;
      tw[(k1 - 1) * 16 + n2] = make_float2((float)cos(a), (float)sin(a));
    }
  // mel: unit u (16 of them) owns filters u, u + 16, ...; per filter a 4-aligned window of float4 weight groups inside [0, 260)
  const int fpu = std::max(1, (p.M + 15) / 16);
  std::vector<int> md((size_t)16 * fpu * 4, 0);
  std::vector<float> mw;
  for (int u = 0; u < 16; ++u)
    for (int j = 0; j < fpu; ++j) {
      int *d = &md[((size_t)u * fpu + j) * 4];
      const int m = u + 16 * j;
      d[3] = -1;
      if (m >= p.M) continue;
      int f0, f1;
      d[3] = m;
      d[2] = (int)(mw.size() / 4);
      if (!filter_support(bank.data(), p.K, p.M, m, &f0, &f1)) { d[0] = 0; d[1] = 0; continue; }
      const int s0 = f0 & ~3;
      const int g = (f1 - s0) / 4 + 1;
      d[0] = s0; d[1] = g;
      for (int i = 0; i < 4 * g; ++i) {
        const int k = s0 + i;
        mw.push_back(k < p.K ? bank[(size_t)k * p.M + m] : 0.f);  // bins 257..259 of a P row are written as zeros
      }
    }
  if (mw.empty()) mw.assign(4, 0.f);
  img->blob = ConstBlob();
  img->blob.append(img4);
  img->off_tw = img->blob.append(tw);
  img->off_md = img->blob.append(md);
  img->off_mw = img->blob.append(mw);
  img->fpu = fpu;
  img->Mpad = (p.M + 3) & ~3;
  img->win4.assign(512, 0.f);
  for (int i = 0; i < p.L; ++i) img->win4[i] = window[i];
  img->c16.assign(256, 0.f);  // [2 k2 + part][n2]: X[16 + 32 k2] = sum_n2 Y16[n2] exp(-2 pi i n2 (1 + 2 k2) / 32)
  for (int k2 = 0; k2 < 8; ++k2)
    for (int n2 = 0; n2 < 16; ++n2) {
      const double a = 2.0 * M_PI * (double)((n2 * (1 + 2 * k2)) % 32) / 32.0;
      img->c16[(2 * k2) * 16 + n2] = (float)cos(a);
      img->c16[(2 * k2 + 1) * 16 + n2] = (float)(-sin(a));
    }
  return 0;
}

static inline int tc512_warp_bytes(int Mpad) { return 4 * (32 * TC_VS + 16 * TC_YS + TC_PP + 16 + Mpad); }
static inline size_t tc512_smem_bytes(const Tc512Tables &t) {  // 1024 B of alignment slack + tables + mbarrier + per-warp buffers
  return 1024 + (size_t)t.cblob_bytes + 16 + (size_t)(TC_THREADS / 32) * (size_t)t.warp_bytes;
}

template <int DT>
static int tc512_go(bool launch, size_t smem, const DevPlan &p, const Tc512Tables &t, const DevBatch &b, dim3 grid, cudaStream_t stream,
                    int *ctas_per_sm) {
  auto kern = b200feat_tc512_kernel<DT>;
  if (configure_or_launch(kern, TC_THREADS, launch, smem, p, t, b, grid, stream)) return B200FEAT_ECUDA;
  if (!launch && (cudaOccupancyMaxActiveBlocksPerMultiprocessor(ctas_per_sm, kern, TC_THREADS, smem) != cudaSuccess || *ctas_per_sm < 1))
    return B200FEAT_ECUDA;
  return 0;
}

static inline int tc512_prepare(DevPlan &p, const std::vector<float> &bank, std::vector<void *> &allocs, int *frames_per_tile,
                                const std::vector<float> &window, Tc512Host *out) {
  Tc512Image img;
  tc512_build_image(p, bank, window, &img);
  Tc512Host hst;
  if (img.blob.upload(allocs, &hst.t.cblob, &hst.t.cblob_bytes)) return B200FEAT_ECUDA;
  hst.t.off_tw = img.off_tw; hst.t.off_md = img.off_md; hst.t.off_mw = img.off_mw; hst.t.fpu = img.fpu; hst.t.Mpad = img.Mpad;
  hst.t.warp_bytes = tc512_warp_bytes(img.Mpad);
  if (upload_table(img.win4, allocs, &hst.t.win4) || upload_table(img.c16, allocs, &hst.t.c16)) return B200FEAT_ECUDA;
  hst.smem = tc512_smem_bytes(hst.t);
  if (hst.smem > (size_t)227 * 1024) return B200FEAT_EUNSUPPORTED;
  DevBatch none{};
  int occ_f32 = 0, occ_i16 = 0;
  if (tc512_go<B200FEAT_F32>(false, hst.smem, p, hst.t, none, dim3(1), nullptr, &occ_f32)) return B200FEAT_ECUDA;
  if (tc512_go<B200FEAT_I16>(false, hst.smem, p, hst.t, none, dim3(1), nullptr, &occ_i16)) return B200FEAT_ECUDA;
  hst.ctas_per_sm = std::min(occ_f32, occ_i16);
  *out = hst;
  *frames_per_tile = TC_NF;
  return 0;
}

static inline int tc512_launch(const DevPlan &p, const Tc512Host &hst, const DevBatch &b, int dt, int sm_count, cudaStream_t stream) {
  // persistent: every resident CTA walks a contiguous tile range
  const dim3 grid(persistent_grid(b.num_tiles, sm_count, hst.ctas_per_sm));
  if (dt == B200FEAT_I16) tc512_go<B200FEAT_I16>(true, hst.smem, p, hst.t, b, grid, stream, nullptr);
  else tc512_go<B200FEAT_F32>(true, hst.smem, p, hst.t, b, grid, stream, nullptr);
  return (int)cudaGetLastError();
}
