// Fast fused kernel for fft_length N = 1024 (22.05 / 24 kHz with 25 ms frames: L = 551 / 600, and any plan with
// 512 < L <= 1024), second generation, in the style of fast2048.cuh: one WARP per frame, the 1024-point real FFT as a packed
// 512-point complex FFT factored 16 x 8 x 4 with 16 complex points per lane in registers:
//
//   z[n] = y[2n] + i*y[2n+1], n = 32*n1 + 4*n2 + n3            k = k1 + 16*k2 + 128*k3
//   stage 1  lane owns column c = lane = 4*n2 + n3: radix-16 DFT over n1, times W128^(n2*k1) -> tile A[k1][c]   (STS.64)
//   stage 2  lane (k1 = lane & 15, h = lane >> 4) reads A[k1][n2][n3 = 2h, 2h+1] (LDS.128), two radix-8 DFTs over n2, times
//            W512^(n3*(k1 + 16*k2)) (per-lane register constants) -> tile B[h][k = k1 + 16*k2]                  (STS.128)
//   stage 3  fast2048.cuh's in-lane split with Q = 128: lane owns k in {lane + 32j, 128 - (lane + 32j)}, j = 0, 1
//   power spectra of SLOTS consecutive frames as P[slot][bin] (513 bins), mel bank as balanced 12-tap work items.
//
// It replaced a kernel that ran one half-warp per 512-point sub-FFT plus a radix-2 combination across the halves (spilling in
// its run-time-length variant).  The stage functions are __host__ __device__
// (scripts/micro/f2k_host_check.cu).  Replaces the same reference code as fast512.cuh (lhotse/features/kaldi/layers.py:151-186,
// :32-42, :565-578, :708-724, framing :727-772).
#pragma once
#include "fast2048.cuh"

#define F1W_PBINS 528                      // floats per P row: 513 bins + zero pad (a 12-tap mel piece may start at bin 512)
#define F1W_PTAIL 64
#define F1W_XROW 34                        // float2 per k1-row of tile A (32 + 2 pad = 17 float4: the LDS.128 of stage 2 is conflict-free)
#define F1W_XBUF (16 * F1W_XROW)           // float2 per warp (4352 B); tile B aliases it
#define F1W_PLANE 132                      // float4 per n3-pair plane of tile B (128 + 4 pad)
#define F1W_PIECE F2K_PIECE

// forward 8-point DFT, natural order in and out (host + device)
F512_HD void f1w_dft8(float2 (&x)[8]) {
  float2 e0 = x[0], e1 = x[2], e2 = x[4], e3 = x[6], o0 = x[1], o1 = x[3], o2 = x[5], o3 = x[7];
  dft4(e0, e1, e2, e3);
  dft4(o0, o1, o2, o3);
  o1 = f2mul_w8_1(o1);
  o2 = f2mi(o2);
  o3 = f2mul_w8_3(o3);
  x[0] = f2add(e0, o0); x[4] = f2sub(e0, o0);
  x[1] = f2add(e1, o1); x[5] = f2sub(e1, o1);
  x[2] = f2add(e2, o2); x[6] = f2sub(e2, o2);
  x[3] = f2add(e3, o3); x[7] = f2sub(e3, o3);
}

// ---- stage 1: v[n1] = z[32*n1 + lane]; tw1[k1*8 + n2] = W128^(n2*k1)
F512_HD void f1w_stage1(int lane, float2 (&v)[16], const float2 *tw1, float2 *xa) {
  dft16(v);
  const int n2 = lane >> 2;
#pragma unroll
  for (int k1 = 0; k1 < 16; ++k1) {
    float2 a = v[F512_OUT(k1)];
    if (k1 > 0) a = f2mul(a, tw1[k1 * 8 + n2]);
    xa[k1 * F1W_XROW + lane] = a;
  }
}

// ---- stage 2, first half: lane (k1 = lane & 15, h = lane >> 4) pulls A[k1][n2][n3 = 2h, 2h+1] into v[0..7] and u[0..7]
F512_HD void f1w_stage2_load(int lane, const float2 *xa, float2 (&v)[16], float2 (&u)[8]) {
  const float4 *row = reinterpret_cast<const float4 *>(xa + (lane & 15) * F1W_XROW) + (lane >> 4);  // float4 index 2*n2 + h
#pragma unroll
  for (int n2 = 0; n2 < 8; ++n2) {
    const float4 r = row[2 * n2];
    v[n2] = make_float2(r.x, r.y);
    u[n2] = make_float2(r.z, r.w);
  }
}

// ---- stage 2, second half: tw[k2] / tw[8 + k2] = W512^(n3*(k1 + 16*k2)) for n3 = 2h / 2h + 1 (register constants)
F512_HD void f1w_stage2_store(int lane, float2 (&v)[16], float2 (&u)[8], const float2 (&tw)[16], float4 *xb) {
  float2 a[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) a[i] = v[i];
  f1w_dft8(a);
  f1w_dft8(u);
  float4 *dst = xb + (lane >> 4) * F1W_PLANE + (lane & 15);
#pragma unroll
  for (int k2 = 0; k2 < 8; ++k2) {
    const float2 c0 = f2mul(a[k2], tw[k2]), c1 = f2mul(u[k2], tw[8 + k2]);
    dst[16 * k2] = make_float4(c0.x, c0.y, c1.x, c1.y);
  }
}

struct Fast1024Tables {
  // one 16-byte-aligned blob (TMA bulk copy):
  //   [win2: 16*32 float2 (w[64 n1 + 2 lane], w[.. + 1]), zero beyond L] [tw1: 16*8 float2 W128^(n2*k1) at [k1][n2]]
  //   [w1k: 64 float2 W1024^k] [rstart: rounds*32 int | fdesc: M int2 + ceil(M/32) int2 | wdense: rounds*3*32 float4]
  const void *cblob;
  int cblob_bytes;
  int off_tw1, off_w1k, off_rstart, off_fdesc, off_mw;
  const float2 *tw2;   // [32 lanes][16]  W512^(n3*(k1 + 16*k2)): [k2] for n3 = 2h, [8 + k2] for n3 = 2h + 1 (global: loaded into registers once)
  int mel_rounds;
  int xfloats;         // floats of per-warp scratch: the exchange tile, reused by the epilogue for SLOTS x (work-item sums + log-mel row)
};

static inline size_t fast1024_smem_bytes(const Fast1024Tables &t, int warps, int slots) {
  size_t b = (size_t)warps * t.xfloats * 4 + (size_t)warps * F1W_PBINS * slots * 4 + F1W_PTAIL * 4;
  b += (size_t)t.cblob_bytes + 16;
  return (b + 15) & ~(size_t)15;
}

template <int DT, int LCT, int WARPS, int SLOTS, int MINB>
__global__ void __launch_bounds__(WARPS * 32, MINB)
b200feat_fast1024_kernel(const DevPlan p, const Fast1024Tables ft, const DevBatch b) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int tid = threadIdx.x;
  const int lane = tid & 31;
  const int w = tid >> 5;            // warp = frame owner
  const int L = LCT ? LCT : p.L;
  constexpr int NP = LCT ? (LCT + 63) / 64 : 16;  // rows of 64 samples that carry data

  float *xall = reinterpret_cast<float *>(smem_raw);
  float *pall = xall + (size_t)WARPS * ft.xfloats;
  unsigned char *s_const = reinterpret_cast<unsigned char *>(pall + (size_t)WARPS * (F1W_PBINS * SLOTS) + F1W_PTAIL);
  const float2 *s_win = reinterpret_cast<const float2 *>(s_const);
  const float2 *s_tw1 = reinterpret_cast<const float2 *>(s_const + ft.off_tw1);
  const float2 *s_w1k = reinterpret_cast<const float2 *>(s_const + ft.off_w1k);
  const int *s_rstart = reinterpret_cast<const int *>(s_const + ft.off_rstart);
  const int2 *s_fdesc = reinterpret_cast<const int2 *>(s_const + ft.off_fdesc);
  const float4 *s_mw4 = reinterpret_cast<const float4 *>(s_const + ft.off_mw);
  unsigned long long *s_bar = reinterpret_cast<unsigned long long *>(s_const + ft.cblob_bytes);
  float2 *X = reinterpret_cast<float2 *>(xall + (size_t)w * ft.xfloats);  // per warp exchange tile (xfloats is a multiple of 4)
  float *P = pall + (size_t)w * (F1W_PBINS * SLOTS);             // per warp: [slot][F1W_PBINS]

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
  for (int i = tid; i < WARPS * (F1W_PBINS * SLOTS) + F1W_PTAIL; i += blockDim.x) pall[i] = 0.f;
  // per-lane twiddles kept in registers for the whole kernel
  float2 tw2[16];  // W512^(n3*(k1 + 16*k2)): [0..7] for n3 = 2h, [8..15] for n3 = 2h + 1
#pragma unroll
  for (int i = 0; i < 16; ++i) tw2[i] = __ldg(ft.tw2 + lane * 16 + i);
  const float inv_L = 1.0f / (float)L;
  const int up_lane = (lane + 31) & 31;
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
    const int64_t t0 = (tile - __ldg(b.tile_off + cut)) * (WARPS * SLOTS) + (int64_t)w * SLOTS;
    const int64_t T = __ldg(b.row_off + cut + 1) - __ldg(b.row_off + cut);
    const int64_t rows_here = b.out_mode == B200FEAT_OUT_PADDED ? b.max_frames : T;
    if (t0 >= rows_here) continue;  // warp-uniform: the whole warp owns these frames
    const int64_t n = __ldg(b.nsamp + cut);
    const int64_t xoff = __ldg(b.samp_off + cut);
    const int64_t row0 = b.out_mode == B200FEAT_OUT_PADDED ? (int64_t)(b.batch_first + cut) * b.max_frames + t0
                                                           : __ldg(b.row_off + cut) + t0;
    float le[SLOTS];
#pragma unroll
    for (int k = 0; k < SLOTS; ++k) le[k] = 0.f;

#pragma unroll 1
    for (int f = 0; f < SLOTS; ++f) {
      const int64_t t = t0 + f;
      if (t >= T) break;  // warp-uniform; the frames of a warp are consecutive
      const int64_t base = t * p.S - (p.snip_edges ? 0 : p.pad_left);
      float2 v[16], u[8];
      const bool interior = base >= 0 && base + L <= n;
      if (F512_PREFETCH && f + 1 < SLOTS && t + 1 < T) {  // one L1 prefetch per 32-byte sector of the next frame's new samples
        constexpr int PER = DT == B200FEAT_I16 ? 16 : 8;
        const int64_t q = base + L + PER * lane;
        if (PER * lane < p.S + PER && q >= 0 && q < n)
          asm volatile("prefetch.global.L1 [%0];" ::"l"(reinterpret_cast<const char *>(b.samples) + (xoff + q) * (DT == B200FEAT_I16 ? 2 : 4)));
      }
      if (interior && (((xoff + base) & 1) == 0)) {  // aligned 8-byte (4-byte for PCM16) pairs, coalesced
        if (DT == B200FEAT_I16) {
          const int16_t *xp = reinterpret_cast<const int16_t *>(b.samples) + (xoff + base + 2 * lane);
#pragma unroll
          for (int n1 = 0; n1 < NP; ++n1) {
            const int j = 64 * n1 + 2 * lane;
            float2 r = make_float2(0.f, 0.f);
            if (j + 1 < L) {
              const short2 q = __ldg(reinterpret_cast<const short2 *>(xp + 64 * n1));
              r = make_float2((float)q.x * (1.0f / 32768.0f), (float)q.y * (1.0f / 32768.0f));
            } else if (j < L) {
              r.x = (float)__ldg(xp + 64 * n1) * (1.0f / 32768.0f);
            }
            v[n1] = r;
          }
        } else {
          const float *xp = reinterpret_cast<const float *>(b.samples) + (xoff + base + 2 * lane);
#pragma unroll
          for (int n1 = 0; n1 < NP; ++n1) {
            const int j = 64 * n1 + 2 * lane;
            float2 r = make_float2(0.f, 0.f);
            if (j + 1 < L) r = __ldg(reinterpret_cast<const float2 *>(xp + 64 * n1));
            else if (j < L) r.x = __ldg(xp + 64 * n1);  // odd L: last tap alone
            v[n1] = r;
          }
        }
      } else if (interior) {  // odd element offset: two 4-byte loads per pair
        const int64_t x0 = xoff + base + 2 * lane;
#pragma unroll
        for (int n1 = 0; n1 < NP; ++n1) {
          const int j = 64 * n1 + 2 * lane;
          float2 r = make_float2(0.f, 0.f);
          if (j < L) r.x = ld_sample<DT>(b.samples, x0 + 64 * n1);
          if (j + 1 < L) r.y = ld_sample<DT>(b.samples, x0 + 64 * n1 + 1);
          v[n1] = r;
        }
      } else {  // a cut edge: per-tap reflection (layers.py:753-772)
#pragma unroll
        for (int n1 = 0; n1 < NP; ++n1) {
          const int j = 64 * n1 + 2 * lane;
          float2 r = make_float2(0.f, 0.f);
          if (j < L) {
            int64_t i = base + j;
            if (!p.snip_edges) i = reflect_index(i, n, p.pad_mode);
            r.x = ld_sample<DT>(b.samples, xoff + i);
          }
          if (j + 1 < L) {
            int64_t i = base + j + 1;
            if (!p.snip_edges) i = reflect_index(i, n, p.pad_mode);
            r.y = ld_sample<DT>(b.samples, xoff + i);
          }
          v[n1] = r;
        }
      }
      // ---- DC removal (layers.py:155-157)
      float s = 0.f, s2 = 0.f;
#pragma unroll
      for (int n1 = 0; n1 < NP; ++n1) {  // taps beyond L are exact zeros
        if (n1 & 1) s2 += v[n1].x + v[n1].y; else s += v[n1].x + v[n1].y;
      }
      const float mu = p.remove_dc ? warp_sum(s + s2) * inv_L : 0.f;
      // ---- energy, pre-emphasis, window (layers.py:159-170).  The tap before y[64 n1 + 2 lane] is the neighbour lane's odd tap;
      // lane 0 takes lane 31's of the previous row
      float e = 0.f;
      float carry = v[0].x;  // lane 0, row 0: replicate-left (layers.py:166)
#pragma unroll
      for (int n1 = 0; n1 < 16; ++n1) {
        if (n1 < NP) {
          const float up = __shfl_sync(F512_FULL, v[n1].y, up_lane);
          const float pr = lane == 0 ? carry : up;
          carry = up;
          const int j = 64 * n1 + 2 * lane;
          const float2 wv = s_win[n1 * 32 + lane];  // zero beyond L
          float2 d = f2add(v[n1], make_float2(-mu, -mu));
          const float dp = pr - mu;
          if (j >= L) d.x = 0.f;
          if (j + 1 >= L) d.y = 0.f;
          if (p.raw_energy) e = fmaf(d.x, d.x, fmaf(d.y, d.y, e));
          const float2 y = preemph_window2(d, dp, p.preemph, wv);
          if (!p.raw_energy) e = fmaf(y.x, y.x, fmaf(y.y, y.y, e));
          v[n1] = y;
        } else {
          v[n1] = make_float2(0.f, 0.f);
        }
      }
      if (p.use_energy) {  // le[] stays in registers: no dynamic indexing
        const float lev = log_energy_value(p, warp_sum(e));
#pragma unroll
        for (int k = 0; k < SLOTS; ++k) le[k] = (f == k) ? lev : le[k];
      }
      // ---- the 512-point complex FFT, 16 x 8 x 4, and the split
      f1w_stage1(lane, v, s_tw1, X);
      __syncwarp();
      f1w_stage2_load(lane, X, v, u);  // v[0..7] <- column n3 = 2h, u <- column n3 = 2h + 1
      __syncwarp();
      f1w_stage2_store(lane, v, u, tw2, reinterpret_cast<float4 *>(X));
      __syncwarp();
      f2k_stage3_t<128, F1W_PLANE>(lane, reinterpret_cast<const float4 *>(X), s_w1k, P + f * F1W_PBINS, p.use_mag != 0);
      __syncwarp();
    }

    // ---- epilogue: the warp's (up to) SLOTS frames
    const int nvalid = (int)max((int64_t)0, min((int64_t)SLOTS, T - t0));
    const int nrows = (int)max((int64_t)0, min((int64_t)SLOTS, rows_here - t0));
    float *out = b.out + row0 * p.F;
    if (p.feature == B200FEAT_SPECTROGRAM || p.feature == B200FEAT_LOG_SPECTROGRAM) {
      for (int f = 0; f < nrows; ++f) {
        float *o = out + (int64_t)f * p.F;
        if (f >= nvalid) { for (int k = lane; k < p.F; k += 32) o[k] = post_affine(p, k, b.pad_value); continue; }
        for (int k = lane; k < p.K; k += 32) {
          float x = P[f * F1W_PBINS + k] * (p.use_mag ? 0.5f : 0.25f);
          if (p.feature == B200FEAT_LOG_SPECTROGRAM) x = log_spec_value(p, x);
          if (k == 0 && p.use_energy) {
#pragma unroll
            for (int g = 0; g < SLOTS; ++g) x = (f == g) ? le[g] : x;
          }
          o[k] = post_affine(p, k, x);
        }
      }
    } else {
      const int shift = mel_shift(p), ecol = energy_col(p);
      const float lgk = p.log10_mel ? 0.30102999566398119521f : 0.69314718055994530942f;  // log10 (librosa_fbank.py:126) or ln
      const int Mpad = (p.M + 3) & ~3;
      // the exchange tile is idle during the epilogue: [SLOTS][NQ] partial sums of the mel work items, then the log-mel rows (MFCC)
      const int NQ = ft.mel_rounds * 32;
      float *part = reinterpret_cast<float *>(X);
      float *mlog = part + SLOTS * NQ;
      for (int j = 0; j < ft.mel_rounds; ++j) {  // pass 1: one work item (filter, piece of 12 taps) per lane
        const float4 *pa = reinterpret_cast<const float4 *>(P + s_rstart[j * 32 + lane]);
        const float4 *wa = s_mw4 + (j * (F1W_PIECE / 4)) * 32 + lane;  // [round][trip][lane][4]
        float acc[SLOTS];
#pragma unroll
        for (int f = 0; f < SLOTS; ++f) acc[f] = 0.f;
#pragma unroll
        for (int t = 0; t < F1W_PIECE / 4; ++t) {
          const float4 w4 = wa[t * 32];
#pragma unroll
          for (int f = 0; f < SLOTS; ++f) {
            const float4 p4 = pa[f * (F1W_PBINS / 4) + t];
            acc[f] = fmaf(p4.w, w4.w, fmaf(p4.z, w4.z, fmaf(p4.y, w4.y, fmaf(p4.x, w4.x, acc[f]))));
          }
        }
#pragma unroll
        for (int f = 0; f < SLOTS; ++f) part[f * NQ + j * 32 + lane] = acc[f];
      }
      __syncwarp();
      for (int m = lane; m < p.M; m += 32) {  // pass 2: one filter per lane adds its pieces in item order
        const int2 fd = s_fdesc[m];             // {first item, items}
        const int qn = s_fdesc[p.M + (m >> 5)].x;  // uniform bound: the item count of the widest filter among these 32
        float r[SLOTS];
#pragma unroll
        for (int f = 0; f < SLOTS; ++f) r[f] = 0.f;
        for (int q = 0; q < qn; ++q) {
#pragma unroll
          for (int f = 0; f < SLOTS; ++f) r[f] += q < fd.y ? part[f * NQ + fd.x + q] : 0.f;
        }
#pragma unroll
        for (int f = 0; f < SLOTS; ++f) r[f] = fast_lg2_normal(nanmax(r[f], p.mel_floor)) * lgk;
        if (p.feature != B200FEAT_MFCC) {
          float *orow = out + m + shift;
#pragma unroll
          for (int f = 0; f < SLOTS; ++f)
            if (f < nvalid) orow[(int64_t)f * p.F] = post_affine(p, m + shift, r[f]);
        } else {
#pragma unroll
          for (int f = 0; f < SLOTS; ++f) mlog[f * Mpad + m] = r[f];
        }
      }
      if (p.feature == B200FEAT_FBANK) {
        if (p.use_energy && lane < nvalid) {
          float v0 = 0.f;
#pragma unroll
          for (int f = 0; f < SLOTS; ++f) v0 = (lane == f) ? le[f] : v0;
          out[(int64_t)lane * p.F + ecol] = post_affine(p, ecol, v0);
        }
      } else if (p.feature == B200FEAT_MFCC) {
        __syncwarp();
        for (int idx = lane; idx < nvalid * p.C; idx += 32) {
          const int f = idx / p.C, c = idx - f * p.C;
          float acc = 0.f;
          for (int m = 0; m < p.M; ++m) acc = fmaf(mlog[f * Mpad + m], __ldg(p.dct + m * p.C + c), acc);
          if (p.use_lifter) acc *= __ldg(p.lifter + c);
          if (p.use_energy && c == ecol) {
#pragma unroll
            for (int g = 0; g < SLOTS; ++g) acc = (f == g) ? le[g] : acc;
          }
          out[(int64_t)f * p.F + c] = post_affine(p, c, acc);
        }
      }
      for (int f = nvalid; f < nrows; ++f)
        for (int k = lane; k < p.F; k += 32) out[(int64_t)f * p.F + k] = post_affine(p, k, b.pad_value);
    }
    __syncwarp();
  }
}

// ---------------------------------------------------------------------------------------------- host
struct Fast1024Host {
  Fast1024Tables t;
  size_t smem;
  int shape;
};

// launch shapes {warps per CTA, frames per warp, CTAs per SM}: B200FEAT_FAST1024W_SHAPE selects (A/B runs)
struct F1wShape { int warps, slots, minb; };
#define F1W_NUM_SHAPES 4
static const F1wShape kF1wShapes[F1W_NUM_SHAPES] = {{8, 3, 2}, {6, 4, 2}, {10, 2, 2}, {12, 3, 1}};

// the constant tables of the FFT stages (also used by scripts/micro/f2k_host_check.cu)
static inline void f1w_fft_tables(std::vector<float2> &tw1, std::vector<float2> &tw2, std::vector<float2> &w1k) {
  tw1.resize(16 * 8); tw2.resize(32 * 16); w1k.resize(64);
  for (int k1 = 0; k1 < 16; ++k1)
    for (int n2 = 0; n2 < 8; ++n2) {
      const double a = -2.0 * M_PI * (double)((n2 * k1) % 128) / 128.0;
      tw1[k1 * 8 + n2] = make_float2((float)cos(a), (float)sin(a));
    }
  for (int lane = 0; lane < 32; ++lane) {
    const int k1 = lane & 15, h = lane >> 4;
    for (int c = 0; c < 2; ++c)
      for (int k2 = 0; k2 < 8; ++k2) {
        const double a = -2.0 * M_PI * (double)(((2 * h + c) * (k1 + 16 * k2)) % 512) / 512.0;
        tw2[lane * 16 + 8 * c + k2] = make_float2((float)cos(a), (float)sin(a));
      }
  }
  for (int k = 0; k < 64; ++k) {
    const double a = -2.0 * M_PI * (double)k / 1024.0;
    w1k[k] = make_float2((float)cos(a), (float)sin(a));
  }
}

static inline bool fast1024_supported(const DevPlan &p) {
  return p.N == 1024 && p.packed && p.L > 2 && p.L <= 1024 && p.C <= 128 && p.M <= 128;
}

template <int DT, int LCT, int WARPS, int SLOTS, int MINB>
static int f1w_go(bool launch, size_t smem, const DevPlan &p, const Fast1024Tables &t, const DevBatch &b, dim3 grid, cudaStream_t stream) {
  auto kern = b200feat_fast1024_kernel<DT, LCT, WARPS, SLOTS, MINB>;
  if (!launch)
    return cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) == cudaSuccess ? 0 : B200FEAT_ECUDA;
  kern<<<grid, dim3(WARPS * 32), smem, stream>>>(p, t, b);
  return 0;
}

template <int DT, int LCT>
static int f1w_shape(int shape, bool launch, size_t smem, const DevPlan &p, const Fast1024Tables &t, const DevBatch &b, dim3 grid,
                     cudaStream_t stream) {
  if (shape == 1) return f1w_go<DT, LCT, 6, 4, 2>(launch, smem, p, t, b, grid, stream);
  if (shape == 2) return f1w_go<DT, LCT, 10, 2, 2>(launch, smem, p, t, b, grid, stream);
  if (shape == 3) return f1w_go<DT, LCT, 12, 3, 1>(launch, smem, p, t, b, grid, stream);
  return f1w_go<DT, LCT, 8, 3, 2>(launch, smem, p, t, b, grid, stream);
}

static inline int f1w_ct_length(int L) { return (L == 600 || L == 551) ? L : 0; }

static int f1w_dispatch(int dt, int L, int shape, bool launch, size_t smem, const DevPlan &p, const Fast1024Tables &t,
                        const DevBatch &b, dim3 grid, cudaStream_t stream) {
  if (L == 600) return dt == B200FEAT_I16 ? f1w_shape<B200FEAT_I16, 600>(shape, launch, smem, p, t, b, grid, stream)
                                          : f1w_shape<B200FEAT_F32, 600>(shape, launch, smem, p, t, b, grid, stream);
  if (L == 551) return dt == B200FEAT_I16 ? f1w_shape<B200FEAT_I16, 551>(shape, launch, smem, p, t, b, grid, stream)
                                          : f1w_shape<B200FEAT_F32, 551>(shape, launch, smem, p, t, b, grid, stream);
  return dt == B200FEAT_I16 ? f1w_shape<B200FEAT_I16, 0>(shape, launch, smem, p, t, b, grid, stream)
                            : f1w_shape<B200FEAT_F32, 0>(shape, launch, smem, p, t, b, grid, stream);
}

static inline int fast1024_prepare(DevPlan &p, const std::vector<float> &bank, std::vector<void *> &allocs,
                                    int *frames_per_tile, const std::vector<float> &window, Fast1024Host *out) {
  Fast1024Host hst;
  std::vector<float2> win2(16 * 32), tw1, tw2, w1k;
  for (int n1 = 0; n1 < 16; ++n1)
    for (int l = 0; l < 32; ++l) {
      const int j = 64 * n1 + 2 * l;
      win2[n1 * 32 + l] = make_float2(j < p.L ? window[j] : 0.f, j + 1 < p.L ? window[j + 1] : 0.f);
    }
  f1w_fft_tables(tw1, tw2, w1k);
  int rc;
  if ((rc = f512_upload(tw2, allocs, &hst.t.tw2))) return rc;
  MelItems mr = pack_mel_items_T(bank, p.K, p.M, p.use_mag ? 0.5f : 0.25f, 32, 4, F1W_PIECE, /*uniform=*/true);
  if (mr.max_reach > F1W_PBINS) return B200FEAT_EUNSUPPORTED;
  hst.t.mel_rounds = mr.rounds;
  {
    std::vector<unsigned char> blob;
    auto append = [&](const void *src, size_t bytes) -> int {
      const size_t off = blob.size();
      blob.resize(off + ((bytes + 15) & ~(size_t)15), 0);
      if (bytes) memcpy(blob.data() + off, src, bytes);
      return (int)off;
    };
    append(win2.data(), win2.size() * sizeof(float2));
    hst.t.off_tw1 = append(tw1.data(), tw1.size() * sizeof(float2));
    hst.t.off_w1k = append(w1k.data(), w1k.size() * sizeof(float2));
    hst.t.off_rstart = append(mr.rstart.data(), mr.rstart.size() * sizeof(int));
    std::vector<int> fdesc((size_t)(std::max(p.M, 1) + (p.M + 31) / 32 + 1) * 2, 0);  // M x {first item, items}, then per 32 filters {max items, 0}
    for (int m = 0; m < p.M; ++m) {
      fdesc[2 * m] = mr.qfirst[m]; fdesc[2 * m + 1] = mr.qcount[m];
      int &mx = fdesc[2 * (p.M + m / 32)];
      mx = std::max(mx, mr.qcount[m]);
    }
    hst.t.off_fdesc = append(fdesc.data(), fdesc.size() * sizeof(int));
    hst.t.off_mw = append(mr.wdense.data(), mr.wdense.size() * sizeof(float));
    const unsigned char *d = nullptr;
    if ((rc = f512_upload(blob, allocs, &d))) return rc;
    hst.t.cblob = d;
    hst.t.cblob_bytes = (int)blob.size();
  }
  int forced = -1;
  if (const char *e = getenv("B200FEAT_FAST1024_VARIANT")) forced = atoi(e);
  hst.shape = -1;
  for (int v = 0; v < F1W_NUM_SHAPES; ++v) {
    if (forced >= 0 && forced < F1W_NUM_SHAPES && v != forced) continue;
    const F1wShape sh = kF1wShapes[v];
    hst.t.xfloats = std::max(F1W_XBUF * 2, sh.slots * (mr.rounds * 32 + ((p.M + 3) & ~3)));
    if (fast1024_smem_bytes(hst.t, sh.warps, sh.slots) <= (size_t)(227 * 1024 / sh.minb) - 1024) { hst.shape = v; break; }
  }
  if (hst.shape < 0) return B200FEAT_EUNSUPPORTED;
  const F1wShape shape = kF1wShapes[hst.shape];
  hst.smem = fast1024_smem_bytes(hst.t, shape.warps, shape.slots);
  DevBatch none{};
  for (int dt = 0; dt < 2; ++dt)
    if (f1w_dispatch(dt, f1w_ct_length(p.L), hst.shape, false, hst.smem, p, hst.t, none, dim3(1), nullptr)) return B200FEAT_ECUDA;
  *out = hst;
  *frames_per_tile = shape.warps * shape.slots;
  return 0;
}

static inline int fast1024_launch(const DevPlan &p, const Fast1024Host &hst, const DevBatch &b, int dt, int sm_count, cudaStream_t stream) {
  const F1wShape shape = kF1wShapes[hst.shape];
  int64_t blocks = b.num_tiles;
  const int64_t cap = (int64_t)sm_count * shape.minb;
  if (blocks > cap) blocks = cap;
  f1w_dispatch(dt, f1w_ct_length(p.L), hst.shape, true, hst.smem, p, hst.t, b, dim3((unsigned)blocks), stream);
  return (int)cudaGetLastError();
}
