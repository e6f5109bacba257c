// Fast fused kernel for fft_length N = 256 (8 kHz telephone audio: L = 200, S = 80, and any plan with
// 128 < L <= 256): the N = 512 design (fast512.cuh) one size down.
//
//   A QUARTER-WARP (8 lanes) owns one frame; the 256-point real FFT is a packed 128-point complex FFT, 16 x 8:
//   lane l holds z[8*n1 + l], n1 = 0..15      (z[n] = y[2n] + i*y[2n+1], y = windowed frame)
//   radix-16 DFT over n1 in registers -> Y[k1][l], times W128^(l*k1)
//   16x8 transpose through a padded shared-memory tile
//   lane l holds rows k1 = l and l + 8 (8 values each): two radix-8 DFTs -> Z[l + 16*k2], Z[l + 8 + 16*k2]
//   paired real-FFT split against the mirror lane 8 - l (its OTHER row: row r pairs with row 16 - r), lane 0
//   mirrors itself; |2X|^2 of 4 consecutive frames staged as P[frame][bin]; mel rounds of 8 filters; log.
//
// Replaces the same reference code as fast512.cuh (lhotse/features/kaldi/layers.py:151-186, :32-42, :565-578,
// :708-724, framing :727-772).  Helpers (packed complex arithmetic, dft4/dft16, W32 constants) come from fast512.cuh.
#pragma once
#include "fast512.cuh"

#define F256_WARPS 8
#define F256_QW (4 * F256_WARPS)            // quarter-warps per CTA
#define F256_SLOTS 4                        // frames per quarter-warp per tile
#define F256_TILE (F256_QW * F256_SLOTS)    // frames per tile (128)
#define F256_XROW 10                        // float2 per transpose row (8 + 2 pad: 80 B keeps the 8-lane LDS.128 conflict-free)
#define F256_XBUF (16 * F256_XROW)          // float2 per quarter-warp transpose tile
#define F256_PBINS 130                      // floats per P row (129 bins; 4*130 = 8 mod 32: the four quarter-warps of a
                                            // warp land on disjoint banks when they store the same bin)
#define F256_PBUF (F256_PBINS * F256_SLOTS)
#define F256_PTAIL 64

// forward 8-point DFT in registers, natural order in and out
__device__ __forceinline__ void dft8(float2 &x0, float2 &x1, float2 &x2, float2 &x3, float2 &x4, float2 &x5, float2 &x6, float2 &x7) {
  float2 e0 = x0, e1 = x2, e2 = x4, e3 = x6, o0 = x1, o1 = x3, o2 = x5, o3 = x7;
  dft4(e0, e1, e2, e3);
  dft4(o0, o1, o2, o3);
  o1 = f2mul_w8_1(o1);                              // W8^1
  o2 = f2mi(o2);                                    // W8^2 = -i
  o3 = f2mul_w8_3(o3);                              // W8^3
  x0 = f2add(e0, o0); x4 = f2sub(e0, o0);
  x1 = f2add(e1, o1); x5 = f2sub(e1, o1);
  x2 = f2add(e2, o2); x6 = f2sub(e2, o2);
  x3 = f2add(e3, o3); x7 = f2sub(e3, o3);
}

__device__ __forceinline__ float qw_sum(float v) {  // sum over the 8 lanes of each quarter-warp
#pragma unroll
  for (int o = 4; o > 0; o >>= 1) v += __shfl_xor_sync(F512_FULL, v, o, 8);
  return v;
}

struct Fast256Tables {
  // one 16-byte-aligned blob (TMA bulk copy): [win2: 16*8 float2 | rstart: rounds*8 int | rlen | rrow | wdense: rows*8 float]
  const void *cblob;
  int cblob_bytes;
  int off_rstart, off_rlen, off_rrow, off_mw;
  const float2 *tw1;    // [16][8] W128^(l*k1)
  const float2 *w256;   // [8]     W256^l
  int mel_rounds, mel_wrows;
};

static inline size_t fast256_smem_bytes(const Fast256Tables &t) {
  size_t b = (size_t)F256_QW * (F256_XBUF * 8 + F256_PBUF * 4) + F256_PTAIL * 4;
  b += (size_t)t.cblob_bytes + 16;
  return (b + 15) & ~(size_t)15;
}

template <int DT, int LCT>
__global__ void __launch_bounds__(F256_WARPS * 32, 2)
b200feat_fast256_kernel(const DevPlan p, const Fast256Tables ft, const DevBatch b) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int tid = threadIdx.x;
  const int l = tid & 7;            // lane within the quarter-warp
  const int qw = tid >> 3;          // quarter-warp within the CTA
  const int L = LCT ? LCT : p.L;
  constexpr int NP = LCT ? (LCT + 15) / 16 : 16;  // sample-pair rows that carry data

  float2 *xall = reinterpret_cast<float2 *>(smem_raw);
  float *pall = reinterpret_cast<float *>(xall + (size_t)F256_QW * F256_XBUF);
  unsigned char *s_const = reinterpret_cast<unsigned char *>(pall + (size_t)F256_QW * F256_PBUF + F256_PTAIL);
  const float2 *s_win = reinterpret_cast<const float2 *>(s_const);               // [n1][lane] window pairs
  const int *s_rstart = reinterpret_cast<const int *>(s_const + ft.off_rstart);   // [round][lane]
  const int *s_rlen = reinterpret_cast<const int *>(s_const + ft.off_rlen);
  const int *s_rrow = reinterpret_cast<const int *>(s_const + ft.off_rrow);
  const float *s_mw = reinterpret_cast<const float *>(s_const + ft.off_mw);       // [row][lane]
  unsigned long long *s_bar = reinterpret_cast<unsigned long long *>(s_const + ft.cblob_bytes);
  float2 *X = xall + (size_t)qw * F256_XBUF;
  float *P = pall + (size_t)qw * F256_PBUF;  // [slot][F256_PBINS]

  const unsigned bar = f512_smem_u32(s_bar);
  if (tid == 0) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(bar));
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  if (tid == 0) {  // constant tables: one TMA bulk copy
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(ft.cblob_bytes) : "memory");
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(f512_smem_u32(s_const)), "l"(ft.cblob), "r"(ft.cblob_bytes), "r"(bar) : "memory");
  }
  for (int i = tid; i < F256_QW * F256_PBUF + F256_PTAIL; i += blockDim.x) pall[i] = 0.f;  // never NaN under zero weights

  float2 tw1[16];
#pragma unroll
  for (int k1 = 1; k1 < 16; ++k1) tw1[k1] = __ldg(ft.tw1 + k1 * 8 + l);
  const float2 w256l = __ldg(ft.w256 + l);
  const int partner = (8 - l) & 7;
  const float inv_L = 1.0f / (float)L;
  {
    unsigned done = 0;
    while (!done)
      asm volatile("{ .reg .pred p; mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2; selp.u32 %0, 1, 0, p; }"
                   : "=r"(done) : "r"(bar), "r"(0u) : "memory");
  }
  __syncthreads();

  for (int64_t tg = blockIdx.x; tg < b.num_tiles; tg += gridDim.x) {
    const int64_t tile = b.tile_base + tg;
    const int cut = __ldg(b.tile_cut + tile) - b.batch_first;
    const int64_t t0 = (tile - __ldg(b.tile_off + cut)) * F256_TILE + (int64_t)qw * F256_SLOTS;
    const int64_t T = __ldg(b.row_off + cut + 1) - __ldg(b.row_off + cut);
    const int64_t rows_here = b.out_mode == B200FEAT_OUT_PADDED ? b.max_frames : T;
    if (!__any_sync(F512_FULL, t0 < rows_here)) continue;  // all four quarters idle for this tile
    const int64_t n = __ldg(b.nsamp + cut);
    const int64_t xoff = __ldg(b.samp_off + cut);
    const int64_t row0 = b.out_mode == B200FEAT_OUT_PADDED ? (int64_t)(b.batch_first + cut) * b.max_frames + t0
                                                           : __ldg(b.row_off + cut) + t0;
    float le[F256_SLOTS];
#pragma unroll
    for (int k = 0; k < F256_SLOTS; ++k) le[k] = 0.f;

#pragma unroll 1
    for (int f = 0; f < F256_SLOTS; ++f) {
      if (!__any_sync(F512_FULL, t0 + f < T)) continue;
      const int64_t t = min(max(t0 + f, (int64_t)0), T - 1);  // out-of-range quarters redo the last frame (not stored)
      const int64_t base = t * p.S - (p.snip_edges ? 0 : p.pad_left);
      float2 v[16];
      float prev[NP];
      const bool interior = base >= 0 && base + L <= n && (((xoff + base) & 1) == 0);
      if (__all_sync(F512_FULL, interior)) {
        if (DT == B200FEAT_I16) {
          const int16_t *xp = reinterpret_cast<const int16_t *>(b.samples) + (xoff + base + 2 * l);
#pragma unroll
          for (int n1 = 0; n1 < NP; ++n1) {
            const int j0 = 16 * n1 + 2 * l;
            v[n1] = make_float2(0.f, 0.f);
            prev[n1] = 0.f;
            if (j0 + 1 < L) {
              const short2 q = __ldg(reinterpret_cast<const short2 *>(xp + 16 * n1));
              v[n1] = make_float2((float)q.x * (1.0f / 32768.0f), (float)q.y * (1.0f / 32768.0f));
            } else if (j0 < L) {
              v[n1].x = (float)__ldg(xp + 16 * n1) * (1.0f / 32768.0f);
            }
          }
        } else {
          const float *xp = reinterpret_cast<const float *>(b.samples) + (xoff + base + 2 * l);
#pragma unroll
          for (int n1 = 0; n1 < NP; ++n1) {
            const int j0 = 16 * n1 + 2 * l;
            v[n1] = make_float2(0.f, 0.f);
            prev[n1] = 0.f;
            if (j0 + 1 < L) v[n1] = __ldg(reinterpret_cast<const float2 *>(xp + 16 * n1));
            else if (j0 < L) v[n1].x = __ldg(xp + 16 * n1);
          }
        }
      } else {  // a cut edge in this warp: per-tap reflection (layers.py:753-772)
#pragma unroll
        for (int n1 = 0; n1 < NP; ++n1) {
          const int j0 = 16 * n1 + 2 * l;
          float a = 0.f, c = 0.f, pr = 0.f;
          if (j0 < L) {
            int64_t i = base + j0;
            if (!p.snip_edges) i = reflect_index(i, n, p.pad_mode);
            a = ld_sample<DT>(b.samples, xoff + i);
          }
          if (j0 + 1 < L) {
            int64_t i = base + j0 + 1;
            if (!p.snip_edges) i = reflect_index(i, n, p.pad_mode);
            c = ld_sample<DT>(b.samples, xoff + i);
          }
          v[n1] = make_float2(a, c);
          prev[n1] = pr;
        }
      }
      {  // the tap before (16 n1 + 2l) is the neighbour lane's odd tap: one shuffle instead of a second load
        float carry = v[0].x;  // lane 0, row 0: replicate-left (layers.py:166)
#pragma unroll
        for (int n1 = 0; n1 < NP; ++n1) {
          const float up = __shfl_sync(F512_FULL, v[n1].y, (l + 7) & 7, 8);  // lane 0 receives lane 7's
          prev[n1] = l == 0 ? carry : up;
          carry = up;  // lane 7's odd tap of this row precedes lane 0's first tap of the next row
        }
      }
      // ---- DC removal, energy, pre-emphasis, window (layers.py:155-170)
      float s = 0.f;
#pragma unroll
      for (int n1 = 0; n1 < NP; ++n1) s += v[n1].x + v[n1].y;
      const float mu = p.remove_dc ? qw_sum(s) * inv_L : 0.f;
      float e = 0.f;
#pragma unroll
      for (int n1 = 0; n1 < 16; ++n1) {
        if (n1 < NP) {
          const int j0 = 16 * n1 + 2 * l;
          const float2 w = s_win[n1 * 8 + l];  // zero beyond L
          float2 d = f2add(v[n1], make_float2(-mu, -mu));
          const float dp = prev[n1] - mu;
          if (j0 >= L) d.x = 0.f;
          if (j0 + 1 >= L) d.y = 0.f;
          if (p.raw_energy) e = fmaf(d.x, d.x, fmaf(d.y, d.y, e));
          const float2 y = preemph_window2(d, dp, p.preemph, w);
          if (!p.raw_energy) e = fmaf(y.x, y.x, fmaf(y.y, y.y, e));
          v[n1] = y;
        } else {
          v[n1] = make_float2(0.f, 0.f);
        }
      }
      if (p.use_energy) {  // le[] stays in registers: no dynamic indexing
        const float lev = log_energy_value(p, qw_sum(e));
#pragma unroll
        for (int k = 0; k < F256_SLOTS; ++k) le[k] = (f == k) ? lev : le[k];
      }

      // ---- stage 1: radix-16 over n1, twiddle W128^(l*k1), 16x8 transpose
      dft16(v);
#pragma unroll
      for (int k1 = 0; k1 < 16; ++k1) {
        float2 y = v[F512_OUT(k1)];
        if (k1 > 0) y = f2mul(y, tw1[k1]);
        X[k1 * F256_XROW + l] = y;
      }
      __syncwarp();
      {
        const float4 *ra = reinterpret_cast<const float4 *>(X + l * F256_XROW);
        const float4 *rb = reinterpret_cast<const float4 *>(X + (l + 8) * F256_XROW);
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const float4 a4 = ra[q], b4 = rb[q];
          v[2 * q] = make_float2(a4.x, a4.y); v[2 * q + 1] = make_float2(a4.z, a4.w);
          v[8 + 2 * q] = make_float2(b4.x, b4.y); v[8 + 2 * q + 1] = make_float2(b4.z, b4.w);
        }
      }
      __syncwarp();
      // ---- stage 2: radix-8 over n2 for rows l (slots 0..7: Z[l + 16*k2]) and l + 8 (slots 8..15: Z[l + 8 + 16*k2])
      dft8(v[0], v[1], v[2], v[3], v[4], v[5], v[6], v[7]);
      dft8(v[8], v[9], v[10], v[11], v[12], v[13], v[14], v[15]);
      // ---- paired real-FFT split: row r pairs with row 16 - r, i.e. my row l with the mirror lane's row (8-l)+8 and my
      // row l + 8 with its row 8 - l; each lane does its even k2 and receives the mirror's odd slots (7 - k2).
      // Lane 0 pairs within itself: row 0 as (0,0) (1,7) (2,6) (3,5) (4,4), row 8 as (0,7) (1,6) (2,5) and (3,4) below.
      float *Pf = P + f * F256_PBINS;
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        constexpr int kOwnU[8] = {0, 2, 4, 6, 8, 10, 12, 14};        // a[0,2,4,6], b[0,2,4,6]
        constexpr int kSendU[8] = {15, 13, 11, 9, 7, 5, 3, 1};        // b[7,5,3,1], a[7,5,3,1]
        constexpr int kTwU[8] = {0, 4, 8, 12, 1, 5, 9, 13};           // W32 exponent of W256^(k - l)
        constexpr int kOwn0[8] = {0, 1, 2, 3, 4, 8, 9, 10};
        constexpr int kSend0[8] = {0, 7, 6, 5, 4, 15, 14, 13};
        constexpr int kTw0[8] = {0, 2, 4, 6, 8, 1, 3, 5};
        constexpr int kBin0[8] = {0, 16, 32, 48, 64, 8, 24, 40};
        const float2 zk = l == 0 ? v[kOwn0[i]] : v[kOwnU[i]];
        const float2 zs = l == 0 ? v[kSend0[i]] : v[kSendU[i]];
        const float2 cc = f2conj(make_float2(__shfl_sync(F512_FULL, zs.x, partner, 8), __shfl_sync(F512_FULL, zs.y, partner, 8)));
        const float2 E = f2add(zk, cc), O = f2sub(zk, cc);
        const float2 wu = w32_const(kTwU[i]), w0 = w32_const(kTw0[i]);
        const float2 wc = l == 0 ? w0 : wu;
        const float2 mit = f2mi(f2mul(f2mul(O, wc), w256l));  // -i*T
        const float2 a = f2add(E, mit), bq = f2sub(E, mit);   // 2*X[k], 2*conj(X[128-k])
        float pa = fmaf(a.x, a.x, a.y * a.y), pb = fmaf(bq.x, bq.x, bq.y * bq.y);
        if (p.use_mag) { pa = sqrtf(pa); pb = sqrtf(pb); }
        const int k = l == 0 ? kBin0[i] : (i < 4 ? l + 32 * i : l + 8 + 32 * (i - 4));
        Pf[k] = pa;
        Pf[128 - k] = pb;
      }
      if (l == 0) {  // lane 0's ninth pair: row 8 slots (3, 4) -> bins 56 and 72
        const float2 zk = v[11], cc = f2conj(v[12]);
        const float2 E = f2add(zk, cc), O = f2sub(zk, cc);
        const float2 mit = f2mi(f2mul(O, w32_const(7)));
        const float2 a = f2add(E, mit), bq = f2sub(E, mit);
        float pa = fmaf(a.x, a.x, a.y * a.y), pb = fmaf(bq.x, bq.x, bq.y * bq.y);
        if (p.use_mag) { pa = sqrtf(pa); pb = sqrtf(pb); }
        Pf[56] = pa;
        Pf[72] = pb;
      }
    }
    __syncwarp();

    // ---- epilogue over the (up to) 4 frames of this quarter-warp
    const int nvalid = (int)max((int64_t)0, min((int64_t)F256_SLOTS, T - t0));
    const int nrows = (int)max((int64_t)0, min((int64_t)F256_SLOTS, rows_here - t0));
    float *out = b.out + row0 * p.F;
    if (p.feature == B200FEAT_SPECTROGRAM || p.feature == B200FEAT_LOG_SPECTROGRAM) {
      for (int f = 0; f < nrows; ++f) {
        float *o = out + (int64_t)f * p.F;
        if (f >= nvalid) { for (int k = l; k < p.F; k += 8) o[k] = post_affine(p, k, b.pad_value); continue; }
        for (int k = l; k < p.K; k += 8) {
          float x = P[f * F256_PBINS + k] * (p.use_mag ? 0.5f : 0.25f);
          if (p.feature == B200FEAT_LOG_SPECTROGRAM) x = log_spec_value(p, x);
          if (k == 0 && p.use_energy) {
#pragma unroll
            for (int q = 0; q < F256_SLOTS; ++q) x = (f == q) ? le[q] : x;
          }
          o[k] = post_affine(p, k, x);
        }
      }
    } else {
      const int shift = mel_shift(p), ecol = energy_col(p);
      const float lgk = p.log10_mel ? 0.30102999566398119521f : 0.69314718055994530942f;  // log10 (librosa_fbank.py:126) or ln
      const int Mpad = (p.M + 3) & ~3;
      float *mlog = reinterpret_cast<float *>(X);  // the transpose tile is idle during the epilogue
      for (int j = 0; j < ft.mel_rounds; ++j) {
        const int m = l + 8 * j;
        const float *Pj = P + s_rstart[j * 8 + l];
        const float *wj = s_mw + s_rrow[j] * 8 + l;
        const int len = s_rlen[j];
        float acc[F256_SLOTS];
#pragma unroll
        for (int f = 0; f < F256_SLOTS; ++f) acc[f] = 0.f;
        const float2 *w2 = reinterpret_cast<const float2 *>(wj - l) + l;  // [row / 2][lane][2]
#pragma unroll 2
        for (int i = 0; i < len; i += 2) {
          const float2 wi = w2[i * 4];
#pragma unroll
          for (int f = 0; f < F256_SLOTS; ++f) {
            const float2 pv = *reinterpret_cast<const float2 *>(Pj + f * F256_PBINS + i);
            acc[f] = fmaf(pv.y, wi.y, fmaf(pv.x, wi.x, acc[f]));
          }
        }
        if (m < p.M) {
          float r[F256_SLOTS];
#pragma unroll
          for (int f = 0; f < F256_SLOTS; ++f) r[f] = fast_lg2_normal(nanmax(acc[f], p.mel_floor)) * lgk;
          if (p.feature != B200FEAT_MFCC) {
            float *orow = out + m + shift;
#pragma unroll
            for (int f = 0; f < F256_SLOTS; ++f)
              if (f < nvalid) orow[(int64_t)f * p.F] = post_affine(p, m + shift, r[f]);
          } else {
#pragma unroll
            for (int f = 0; f < F256_SLOTS; ++f) mlog[f * Mpad + m] = r[f];
          }
        }
      }
      if (p.feature == B200FEAT_FBANK) {
        if (p.use_energy && l < nvalid) {
          float v0 = 0.f;
#pragma unroll
          for (int f = 0; f < F256_SLOTS; ++f) v0 = (l == f) ? le[f] : v0;
          out[(int64_t)l * p.F + ecol] = post_affine(p, ecol, v0);
        }
      } else if (p.feature == B200FEAT_MFCC) {
        __syncwarp();
        for (int idx = l; idx < nvalid * p.C; idx += 8) {
          const int f = idx / p.C, c = idx - f * p.C;
          float acc = 0.f;
          for (int m = 0; m < p.M; ++m) acc = fmaf(mlog[f * Mpad + m], __ldg(p.dct + m * p.C + c), acc);
          if (p.use_lifter) acc *= __ldg(p.lifter + c);
          if (p.use_energy && c == ecol) {
#pragma unroll
            for (int g = 0; g < F256_SLOTS; ++g) acc = (f == g) ? le[g] : acc;
          }
          out[(int64_t)f * p.F + c] = post_affine(p, c, acc);
        }
      }
      for (int f = nvalid; f < nrows; ++f)
        for (int k = l; k < p.F; k += 8) out[(int64_t)f * p.F + k] = post_affine(p, k, b.pad_value);
    }
    __syncwarp();
  }
}

// ---------------------------------------------------------------------------------------------- host
struct Fast256Host {
  Fast256Tables t;
  size_t smem;
};

static inline bool fast256_supported(const DevPlan &p) {
  return p.N == 256 && p.packed && p.L >= 2 && p.L <= 256 && p.C <= 128 && F256_SLOTS * ((p.M + 3) & ~3) <= 2 * F256_XBUF;
}

template <int DT, int LCT>
static int f256_go(bool launch, size_t smem, const DevPlan &p, const Fast256Tables &t, const DevBatch &b, dim3 grid, cudaStream_t stream) {
  auto kern = b200feat_fast256_kernel<DT, LCT>;
  if (!launch)
    return cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) == cudaSuccess ? 0 : B200FEAT_ECUDA;
  kern<<<grid, dim3(F256_WARPS * 32), smem, stream>>>(p, t, b);
  return 0;
}

static int f256_dispatch(int dt, int L, bool launch, size_t smem, const DevPlan &p, const Fast256Tables &t, const DevBatch &b,
                         dim3 grid, cudaStream_t stream) {
  if (L == 200) return dt == B200FEAT_I16 ? f256_go<B200FEAT_I16, 200>(launch, smem, p, t, b, grid, stream)
                                          : f256_go<B200FEAT_F32, 200>(launch, smem, p, t, b, grid, stream);
  return dt == B200FEAT_I16 ? f256_go<B200FEAT_I16, 0>(launch, smem, p, t, b, grid, stream)
                            : f256_go<B200FEAT_F32, 0>(launch, smem, p, t, b, grid, stream);
}

static inline int fast256_prepare(DevPlan &p, const std::vector<float> &bank, std::vector<void *> &allocs,
                                  int *frames_per_tile, const std::vector<float> &window, Fast256Host *out) {
  Fast256Host hst;
  std::vector<float2> win2(16 * 8), tw1(16 * 8), w256(8);
  for (int n1 = 0; n1 < 16; ++n1)
    for (int l = 0; l < 8; ++l) {
      const int j0 = 16 * n1 + 2 * l;
      win2[n1 * 8 + l] = make_float2(j0 < p.L ? window[j0] : 0.f, j0 + 1 < p.L ? window[j0 + 1] : 0.f);
    }
  for (int k1 = 0; k1 < 16; ++k1)
    for (int l = 0; l < 8; ++l) {
      const double a = -2.0 * M_PI * (double)((l * k1) % 128) / 128.0;
      tw1[k1 * 8 + l] = make_float2((float)cos(a), (float)sin(a));
    }
  for (int l = 0; l < 8; ++l) {
    const double a = -2.0 * M_PI * (double)l / 256.0;
    w256[l] = make_float2((float)cos(a), (float)sin(a));
  }
  int rc;
  if ((rc = f512_upload(tw1, allocs, &hst.t.tw1))) return rc;
  if ((rc = f512_upload(w256, allocs, &hst.t.w256))) return rc;
  const MelRounds mr = pack_mel_rounds(bank, p.K, p.M, p.use_mag ? 0.5f : 0.25f, 8, 2, F256_PBINS);  // 64-bit mel loads
  if (mr.max_reach > F256_PBINS) return B200FEAT_EUNSUPPORTED;
  hst.t.mel_rounds = mr.rounds;
  hst.t.mel_wrows = mr.rows;
  {
    std::vector<unsigned char> blob;
    auto append = [&](const void *src, size_t bytes) -> int {
      const size_t off = blob.size();
      blob.resize(off + ((bytes + 15) & ~(size_t)15), 0);
      memcpy(blob.data() + off, src, bytes);
      return (int)off;
    };
    append(win2.data(), win2.size() * sizeof(float2));
    hst.t.off_rstart = append(mr.rstart.data(), mr.rstart.size() * sizeof(int));
    hst.t.off_rlen = append(mr.rlen.data(), mr.rlen.size() * sizeof(int));
    hst.t.off_rrow = append(mr.rrow.data(), mr.rrow.size() * sizeof(int));
    hst.t.off_mw = append(mr.wdense.data(), mr.wdense.size() * sizeof(float));
    const unsigned char *d = nullptr;
    if ((rc = f512_upload(blob, allocs, &d))) return rc;
    hst.t.cblob = d;
    hst.t.cblob_bytes = (int)blob.size();
  }
  hst.smem = fast256_smem_bytes(hst.t);
  if (hst.smem > 113 * 1024) return B200FEAT_EUNSUPPORTED;  // keep 2 CTAs per SM
  DevBatch none{};
  for (int dt = 0; dt < 2; ++dt)
    for (int L : {200, 0})
      if (f256_dispatch(dt, L, false, hst.smem, p, hst.t, none, dim3(1), nullptr)) return B200FEAT_ECUDA;
  *out = hst;
  *frames_per_tile = F256_TILE;
  return 0;
}

static inline int fast256_launch(const DevPlan &p, const Fast256Host &hst, const DevBatch &b, int dt, int sm_count, cudaStream_t stream) {
  int64_t blocks = b.num_tiles;
  const int64_t cap = (int64_t)sm_count * 2;
  if (blocks > cap) blocks = cap;
  f256_dispatch(dt, p.L == 200 ? 200 : 0, true, hst.smem, p, hst.t, b, dim3((unsigned)blocks), stream);
  return (int)cudaGetLastError();
}
