// Fast fused kernel for fft_length N = 2048 (24 kHz with 50 ms frames: L = 1200; 44.1 / 48 kHz with 25 ms frames: L = 1102 /
// 1200; librosa-style fft_size = 2048; any plan with 1024 < L <= 2048): one WARP per frame, the 2048-point real FFT as a packed
// 1024-point complex FFT factored 16 x 16 x 4 with the data in registers (32 complex points per lane) between two passes through
// a per-warp shared-memory exchange tile:
//
//   z[n] = y[2n] + i*y[2n+1], n = 64*n1 + 4*n2 + n3          k = k1 + 16*k2 + 256*k3
//   stage 1  lane owns columns c = lane, lane + 32 (c = 4*n2 + n3): radix-16 DFT over n1 in registers, times W256^(n2*k1)
//            -> exchange tile A[k1][c]                                              (STS.64, conflict-free)
//   stage 2  lane (k1 = lane & 15, h = lane >> 4) reads A[k1][n2][n3 = 2h, 2h+1] (LDS.128), radix-16 DFT over n2,
//            times W1024^(n3*(k1 + 16*k2)) -> exchange tile B[h][k = k1 + 16*k2] (two n3 per 128-bit slot)
//   stage 3  lane owns k in {lane + 32*j, 256 - (lane + 32*j)}, j = 0..3: radix-4 DFT over n3 gives Z[k + 256*k3]; the mirror
//            Z[1024 - kappa] of every kappa = k + 256*k3 is ALREADY IN THE SAME LANE ((256 - k) + 256*(3 - k3)), so the
//            real-FFT split needs no shuffle and no further exchange:  E = Z[kappa] + conj Z[1024-kappa], O = Z[kappa] - conj(..),
//            T = W2048^kappa * O, 2 X[kappa] = E - iT, 2 conj X[1024-kappa] = E + iT; W2048^kappa = W2048^k * W8^k3 (table x
//            immediates).  Lane 0 also owns the two self-mirrored residues k = 0 and k = 128.
//   power spectra of SLOTS consecutive frames staged as P[slot][bin] (1025 bins), mel bank as balanced 12-tap work items (below).
//
// Loads are coalesced 8-byte pairs (y[128*n1 + 2*lane], y[.. + 64]); the pre-emphasis neighbour comes from the adjacent lane
// by shuffle.  The stage functions are __host__ __device__: scripts/micro/f2k_host_check.cu runs them lane by lane on the CPU
// against a float64 DFT (tests/test_build_and_entry.py compiles and runs it).
//
// Replaces the same reference code as fast512.cuh (lhotse/features/kaldi/layers.py:151-186, :32-42, :565-578, :708-724,
// framing :727-772).
#pragma once
#include "fast512.cuh"

#define F2K_PBINS 1040                     // floats per P row: 1025 bins + zero pad (a mel piece starting at bin 1024 reads 12 taps)
#define F2K_PTAIL 64
#define F2K_XROW 66                        // float2 per k1-row of exchange tile A (64 + 2 pad = 33 float4: LDS.128 conflict-free)
#define F2K_XBUF (16 * F2K_XROW)           // float2 per warp (8448 B); tile B aliases it: 2 planes of F2K_PLANE float4
#define F2K_PLANE 264                      // float4 per n3-pair plane of exchange tile B (256 + 8 pad)
#define F2K_PIECE 12                       // taps per mel work item: 3 x 128-bit, an odd count spreads the pieces of a wide filter
                                           // over the 16-byte bank groups (simulated wavefronts per 2 frames: 318 vs 716 whole-filter)

// complex product with a table twiddle
F512_HD float2 f2k_mul(float2 a, float2 b) { return f2mul(a, b); }

// ---- stage 1: v0 = column `lane`, v1 = column `lane + 32` of z[64*n1 + c]; tw1[k1*16 + n2] = W256^(n2*k1)
F512_HD void f2k_stage1(int lane, float2 (&v0)[16], float2 (&v1)[16], const float2 *tw1, float2 *xa) {
  dft16(v0);
  dft16(v1);
  const int n2a = lane >> 2, n2b = 8 + (lane >> 2);
#pragma unroll
  for (int k1 = 0; k1 < 16; ++k1) {
    float2 a = v0[F512_OUT(k1)], c = v1[F512_OUT(k1)];
    if (k1 > 0) {
      a = f2k_mul(a, tw1[k1 * 16 + n2a]);
      c = f2k_mul(c, tw1[k1 * 16 + n2b]);
    }
    xa[k1 * F2K_XROW + lane] = a;
    xa[k1 * F2K_XROW + 32 + lane] = c;
  }
}

// ---- stage 2, first half: every lane pulls its 2 x 16 inputs out of tile A (the tile is overwritten by the second half)
F512_HD void f2k_stage2_load(int lane, const float2 *xa, float2 (&u0)[16], float2 (&u1)[16]) {
  const int k1 = lane & 15, h = lane >> 4;
  const float4 *row = reinterpret_cast<const float4 *>(xa + k1 * F2K_XROW) + h;  // float4 index 2*n2 + h <-> n3 = 2h, 2h+1
#pragma unroll
  for (int n2 = 0; n2 < 16; ++n2) {
    const float4 r = row[2 * n2];
    u0[n2] = make_float2(r.x, r.y);
    u1[n2] = make_float2(r.z, r.w);
  }
}

// ---- stage 2, second half: tw2[n3*256 + k] = W1024^(n3*k), k = k1 + 16*k2 < 256
F512_HD void f2k_stage2_store(int lane, float2 (&u0)[16], float2 (&u1)[16], const float2 *tw2, float4 *xb) {
  dft16(u0);
  dft16(u1);
  const int k1 = lane & 15, h = lane >> 4;
  const float2 *ta = tw2 + (2 * h) * 256 + k1, *tb = tw2 + (2 * h + 1) * 256 + k1;
#pragma unroll
  for (int k2 = 0; k2 < 16; ++k2) {
    const float2 a = f2k_mul(u0[F512_OUT(k2)], ta[16 * k2]);  // row n3 = 0 of the table is all ones (uniform code for both halves)
    const float2 c = f2k_mul(u1[F512_OUT(k2)], tb[16 * k2]);
    xb[h * F2K_PLANE + k1 + 16 * k2] = make_float4(a.x, a.y, c.x, c.y);
  }
}

// one (Z[kappa], Z[4Q - kappa]) pair -> |2 X[kappa]|^2 and |2 X[4Q - kappa]|^2 (or the moduli); wk = exp(-2 pi i (kappa - Q*k3) / (8Q))
F512_HD void f2k_pair(float2 zk, float2 zm, float2 wk, int k3, bool use_mag, float &pa, float &pb) {
  const float2 cc = f2conj(zm);
  const float2 E = f2add(zk, cc), O = f2sub(zk, cc);
  float2 T = f2k_mul(O, wk);
  if (k3 == 1) T = f2mul_w8_1(T);       // exp(-2 pi i Q*k3 / (8Q)) = W8^k3
  else if (k3 == 2) T = f2mi(T);
  else if (k3 == 3) T = f2mul_w8_3(T);
  const float2 mit = f2mi(T);           // -i*T
  const float2 a = f2add(E, mit), q = f2sub(E, mit);
  pa = fmaf(a.x, a.x, a.y * a.y);
  pb = fmaf(q.x, q.x, q.y * q.y);
  if (use_mag) { pa = sqrtf(pa); pb = sqrtf(pb); }
}

// ---- stage 3 + real-FFT split + power for a packed complex FFT of 4*Q points (Q = 256: N = 2048; Q = 128: N = 1024, fast1024.cuh):
// tile B holds Z'[k][n3] as two planes of float4 (n3 = 0,1 | 2,3), k < Q; wk[k] = exp(-2 pi i k / (8 Q)), k < Q / 2; Pf[0 .. 4Q]
template <int Q, int PLANE>
F512_HD void f2k_stage3_t(int lane, const float4 *xb, const float2 *wk_table, float *Pf, bool use_mag) {
#pragma unroll
  for (int j = 0; j < Q / 64; ++j) {
    const int ka = lane + 32 * j;
    const int kb = (j == 0 && lane == 0) ? Q / 2 : Q - ka;
    float2 a[4], q[4];
    {
      const float4 r0 = xb[ka], r1 = xb[PLANE + ka];
      a[0] = make_float2(r0.x, r0.y); a[1] = make_float2(r0.z, r0.w);
      a[2] = make_float2(r1.x, r1.y); a[3] = make_float2(r1.z, r1.w);
      dft4(a[0], a[1], a[2], a[3]);  // a[k3] = Z[ka + Q*k3]
      const float4 s0 = xb[kb], s1 = xb[PLANE + kb];
      q[0] = make_float2(s0.x, s0.y); q[1] = make_float2(s0.z, s0.w);
      q[2] = make_float2(s1.x, s1.y); q[3] = make_float2(s1.z, s1.w);
      dft4(q[0], q[1], q[2], q[3]);  // q[k3] = Z[kb + Q*k3]
    }
    // mirror of kappa = ka + Q*k3 is kb + Q*(3 - k3); lane 0, j = 0 (ka = 0): 4Q - Q*k3 = Q*(4 - k3), with Z[4Q] = Z[0]
    float2 m[4] = {q[3], q[2], q[1], q[0]};
    if (j == 0) {
      const bool z = lane == 0;
      m[0] = z ? a[0] : m[0];
      m[1] = z ? a[3] : m[1];
      m[2] = z ? a[2] : m[2];
      m[3] = z ? a[1] : m[3];
    }
    const float2 wk = wk_table[ka];
#pragma unroll
    for (int k3 = 0; k3 < 4; ++k3) {
      float pa, pb;
      f2k_pair(a[k3], m[k3], wk, k3, use_mag, pa, pb);
      const int kappa = ka + Q * k3;
      Pf[kappa] = pa;
      Pf[4 * Q - kappa] = pb;
    }
    if (j == 0 && lane == 0) {  // the other self-mirrored residue: kappa = Q/2 + Q*k3 <-> Q/2 + Q*(3 - k3)
#pragma unroll
      for (int k3 = 0; k3 < 2; ++k3) {
        float pa, pb;
        f2k_pair(q[k3], q[3 - k3], make_float2(F512_C1, -F512_S1), k3, use_mag, pa, pb);  // exp(-2 pi i (Q/2) / (8Q)) = W16^1
        const int kappa = Q / 2 + Q * k3;
        Pf[kappa] = pa;
        Pf[4 * Q - kappa] = pb;
      }
    }
  }
}

// w2k[k] = W2048^k, k < 128; Pf[0..1024]
F512_HD void f2k_stage3(int lane, const float4 *xb, const float2 *w2k, float *Pf, bool use_mag) {
  f2k_stage3_t<256, F2K_PLANE>(lane, xb, w2k, Pf, use_mag);
}

struct Fast2048Tables {
  // one 16-byte-aligned blob (TMA bulk copy):
  //   [win2: 16*2*32 float2 (w[128 n1 + 64 c + 2 lane], w[.. + 1]) indexed [n1][c][lane], zero beyond L]
  //   [tw1: 16*16 float2 W256^(n2*k1) at [k1][n2]] [tw2: 4*256 float2 W1024^(n3*k) at [n3][k]] [w2k: 128 float2 W2048^k]
  //   [rstart: rounds*32 int | fdesc: M int2 {first item, items} + ceil(M/32) int2 {max items of the 32 filters, 0} | wdense: rounds*3*32 float4, [round][trip][lane][4]]
  const void *cblob;
  int cblob_bytes;
  int off_tw1, off_tw2, off_w2k, off_rstart, off_fdesc, off_mw;
  int mel_rounds, mel_qmax;  // rounds (even) of 32 work items; the widest filter's item count (informational)
};

static inline size_t fast2048_smem_bytes(const Fast2048Tables &t, int warps, int slots) {
  size_t b = (size_t)warps * F2K_XBUF * 8 + (size_t)warps * F2K_PBINS * slots * 4 + F2K_PTAIL * 4;
  b += (size_t)t.cblob_bytes + 16;
  return (b + 15) & ~(size_t)15;
}

template <int DT, int LCT, int WARPS, int SLOTS>
__global__ void __launch_bounds__(WARPS * 32, 1)
b200feat_fast2048_kernel(const DevPlan p, const Fast2048Tables ft, const DevBatch b) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int tid = threadIdx.x;
  const int lane = tid & 31;
  const int w = tid >> 5;            // warp = frame owner
  const int L = LCT ? LCT : p.L;
  constexpr int NP = LCT ? (LCT + 127) / 128 : 16;  // rows of 128 samples that carry data

  float2 *xall = reinterpret_cast<float2 *>(smem_raw);
  float *pall = reinterpret_cast<float *>(xall + (size_t)WARPS * F2K_XBUF);
  unsigned char *s_const = reinterpret_cast<unsigned char *>(pall + (size_t)WARPS * (F2K_PBINS * SLOTS) + F2K_PTAIL);
  const float2 *s_win = reinterpret_cast<const float2 *>(s_const);
  const float2 *s_tw1 = reinterpret_cast<const float2 *>(s_const + ft.off_tw1);
  const float2 *s_tw2 = reinterpret_cast<const float2 *>(s_const + ft.off_tw2);
  const float2 *s_w2k = reinterpret_cast<const float2 *>(s_const + ft.off_w2k);
  const int *s_rstart = reinterpret_cast<const int *>(s_const + ft.off_rstart);
  const int2 *s_fdesc = reinterpret_cast<const int2 *>(s_const + ft.off_fdesc);
  const float *s_mw = reinterpret_cast<const float *>(s_const + ft.off_mw);
  unsigned long long *s_bar = reinterpret_cast<unsigned long long *>(s_const + ft.cblob_bytes);
  float2 *X = xall + (size_t)w * F2K_XBUF;                       // per warp exchange tile
  float *P = pall + (size_t)w * (F2K_PBINS * SLOTS);             // per warp: [slot][F2K_PBINS]

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
  for (int i = tid; i < WARPS * (F2K_PBINS * SLOTS) + F2K_PTAIL; i += blockDim.x) pall[i] = 0.f;
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

    // the raw samples of frame t as (y[128 n1 + 2 lane], +1) / (y[128 n1 + 64 + 2 lane], +1); zero beyond L
    auto load_frame = [&](int64_t t, float2 (&v0)[16], float2 (&v1)[16]) {
      const int64_t base = t * p.S - (p.snip_edges ? 0 : p.pad_left);
      const bool interior = base >= 0 && base + L <= n;
      if (interior && (((xoff + base) & 1) == 0)) {  // aligned 8-byte (4-byte for PCM16) pairs, coalesced
        if (DT == B200FEAT_I16) {
          const int16_t *xp = reinterpret_cast<const int16_t *>(b.samples) + (xoff + base + 2 * lane);
#pragma unroll
          for (int n1 = 0; n1 < NP; ++n1) {
#pragma unroll
            for (int c = 0; c < 2; ++c) {
              const int j = 128 * n1 + 64 * c + 2 * lane;
              float2 r = make_float2(0.f, 0.f);
              if (j + 1 < L) {
                const short2 q = __ldg(reinterpret_cast<const short2 *>(xp + 128 * n1 + 64 * c));
                r = make_float2((float)q.x * (1.0f / 32768.0f), (float)q.y * (1.0f / 32768.0f));
              } else if (j < L) {
                r.x = (float)__ldg(xp + 128 * n1 + 64 * c) * (1.0f / 32768.0f);
              }
              if (c == 0) v0[n1] = r; else v1[n1] = r;
            }
          }
        } else {
          const float *xp = reinterpret_cast<const float *>(b.samples) + (xoff + base + 2 * lane);
#pragma unroll
          for (int n1 = 0; n1 < NP; ++n1) {
#pragma unroll
            for (int c = 0; c < 2; ++c) {
              const int j = 128 * n1 + 64 * c + 2 * lane;
              float2 r = make_float2(0.f, 0.f);
              if (j + 1 < L) r = __ldg(reinterpret_cast<const float2 *>(xp + 128 * n1 + 64 * c));
              else if (j < L) r.x = __ldg(xp + 128 * n1 + 64 * c);  // odd L: last tap alone
              if (c == 0) v0[n1] = r; else v1[n1] = r;
            }
          }
        }
      } else if (interior) {  // odd element offset (every other frame when the shift is odd, e.g. 441 samples): two 4-byte loads
        const int64_t x0 = xoff + base + 2 * lane;
#pragma unroll
        for (int n1 = 0; n1 < NP; ++n1) {
#pragma unroll
          for (int c = 0; c < 2; ++c) {
            const int j = 128 * n1 + 64 * c + 2 * lane;
            float2 r = make_float2(0.f, 0.f);
            if (j < L) r.x = ld_sample<DT>(b.samples, x0 + 128 * n1 + 64 * c);
            if (j + 1 < L) r.y = ld_sample<DT>(b.samples, x0 + 128 * n1 + 64 * c + 1);
            if (c == 0) v0[n1] = r; else v1[n1] = r;
          }
        }
      } else {  // a cut edge: per-tap reflection (layers.py:753-772)
#pragma unroll
        for (int n1 = 0; n1 < NP; ++n1) {
#pragma unroll
          for (int c = 0; c < 2; ++c) {
            const int j = 128 * n1 + 64 * c + 2 * lane;
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
            if (c == 0) v0[n1] = r; else v1[n1] = r;
          }
        }
      }
    };
    float2 v0[16], v1[16];
#pragma unroll 1
    for (int f = 0; f < SLOTS; ++f) {
      const int64_t t = t0 + f;
      if (t >= T) break;  // warp-uniform; the frames of a warp are consecutive
      load_frame(t, v0, v1);
      // ---- DC removal (layers.py:155-157)
      float s = 0.f, s2 = 0.f;
#pragma unroll
      for (int n1 = 0; n1 < NP; ++n1) {  // taps beyond L are exact zeros
        s += v0[n1].x + v0[n1].y;
        s2 += v1[n1].x + v1[n1].y;
      }
      const float mu = p.remove_dc ? warp_sum(s + s2) * inv_L : 0.f;
      // ---- energy, pre-emphasis, window (layers.py:159-170).  The tap before y[128 n1 + 64 c + 2 lane] is the neighbour
      // lane's odd tap of the same (n1, c); lane 0 takes lane 31's of the previous half-row
      float e = 0.f;
      float carry = v0[0].x;  // lane 0, row 0: replicate-left (layers.py:166)
#pragma unroll
      for (int n1 = 0; n1 < 16; ++n1) {
        if (n1 < NP) {
          const float up0 = __shfl_sync(F512_FULL, v0[n1].y, up_lane);
          const float up1 = __shfl_sync(F512_FULL, v1[n1].y, up_lane);
          const float pr0 = lane == 0 ? carry : up0;
          const float pr1 = lane == 0 ? up0 : up1;
          carry = up1;
#pragma unroll
          for (int c = 0; c < 2; ++c) {
            const int j = 128 * n1 + 64 * c + 2 * lane;
            const float2 wv = s_win[(n1 * 2 + c) * 32 + lane];  // zero beyond L
            float2 d = f2add(c ? v1[n1] : v0[n1], make_float2(-mu, -mu));
            const float dp = (c ? pr1 : pr0) - mu;
            if (j >= L) d.x = 0.f;
            if (j + 1 >= L) d.y = 0.f;
            if (p.raw_energy) e = fmaf(d.x, d.x, fmaf(d.y, d.y, e));
            const float2 y = preemph_window2(d, dp, p.preemph, wv);
            if (!p.raw_energy) e = fmaf(y.x, y.x, fmaf(y.y, y.y, e));
            if (c) v1[n1] = y; else v0[n1] = y;
          }
        } else {
          v0[n1] = make_float2(0.f, 0.f);
          v1[n1] = make_float2(0.f, 0.f);
        }
      }
      if (p.use_energy) {  // le[] stays in registers: no dynamic indexing
        const float lev = log_energy_value(p, warp_sum(e));
#pragma unroll
        for (int k = 0; k < SLOTS; ++k) le[k] = (f == k) ? lev : le[k];
      }
      // ---- the 1024-point complex FFT, 16 x 16 x 4, and the split
      f2k_stage1(lane, v0, v1, s_tw1, X);
      __syncwarp();
      f2k_stage2_load(lane, X, v0, v1);
      __syncwarp();
      f2k_stage2_store(lane, v0, v1, s_tw2, reinterpret_cast<float4 *>(X));
      __syncwarp();
      f2k_stage3(lane, reinterpret_cast<const float4 *>(X), s_w2k, P + f * F2K_PBINS, p.use_mag != 0);
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
          float x = P[f * F2K_PBINS + k] * (p.use_mag ? 0.5f : 0.25f);
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
      // pass 1: one work item (filter, piece of F2K_PIECE taps) per lane (common.cuh, MelItems), two rounds in flight: all
      // 3 + 3 weight and 2 * 3 * SLOTS power loads of the pair are issued before the first FFMA
      const float4 *mw4 = reinterpret_cast<const float4 *>(s_mw);
      for (int j = 0; j < ft.mel_rounds; j += 2) {  // mel_rounds is even (the tables are padded with an all-zero round)
        const float4 *pa = reinterpret_cast<const float4 *>(P + s_rstart[j * 32 + lane]);
        const float4 *pb = reinterpret_cast<const float4 *>(P + s_rstart[j * 32 + 32 + lane]);
        const float4 *wa = mw4 + (j * (F2K_PIECE / 4)) * 32 + lane;  // [round][trip][lane][4]
        float4 wv[2][F2K_PIECE / 4], pv[2][SLOTS][F2K_PIECE / 4];
#pragma unroll
        for (int t = 0; t < F2K_PIECE / 4; ++t) {
          wv[0][t] = wa[t * 32];
          wv[1][t] = wa[(F2K_PIECE / 4 + t) * 32];
#pragma unroll
          for (int f = 0; f < SLOTS; ++f) {
            pv[0][f][t] = pa[f * (F2K_PBINS / 4) + t];
            pv[1][f][t] = pb[f * (F2K_PBINS / 4) + t];
          }
        }
#pragma unroll
        for (int r2 = 0; r2 < 2; ++r2)
#pragma unroll
          for (int f = 0; f < SLOTS; ++f) {
            float acc = 0.f;
#pragma unroll
            for (int t = 0; t < F2K_PIECE / 4; ++t) {
              const float4 w4 = wv[r2][t], p4 = pv[r2][f][t];
              acc = fmaf(p4.w, w4.w, fmaf(p4.z, w4.z, fmaf(p4.y, w4.y, fmaf(p4.x, w4.x, acc))));
            }
            part[f * NQ + (j + r2) * 32 + lane] = acc;
          }
      }
      __syncwarp();
      for (int m = lane; m < p.M; m += 32) {  // pass 2: one filter per lane adds its pieces in item order
        const int2 fd = s_fdesc[m];             // {first item, items}
        float r[SLOTS];
#pragma unroll
        for (int f = 0; f < SLOTS; ++f) r[f] = 0.f;
        const int qn = s_fdesc[p.M + (m >> 5)].x;  // uniform bound: the item count of the widest filter among these 32; + 0.f leaves a sum as it is
#pragma unroll 2
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
struct Fast2048Host {
  Fast2048Tables t;
  size_t smem;
  int variant;
};

// launch shapes {warps per CTA, frames per warp}, one CTA per SM (the data alone is 64 registers per lane); prepare() takes
// the first shape whose shared memory fits next to the plan's mel tables.  B200FEAT_FAST2048_VARIANT forces one.
// Measured on an H100 SXM with a 400 W power limit (h audio/s, 24 kHz / 50 ms and 44.1 kHz / 25 ms, scripts/bench_fast2048.py;
// profiles/h100_launch_shapes.jsonl):
//   {11, 2} 595 / 587    {10, 2} 562 / 556    {8, 2} 499 / 490    {14, 1} 581 / 588
// Tried and dropped: loading the next frame into the dead data registers during stage 3, an L1 prefetch of the warp's next tile
// before the mel stage.
struct F2kVariant { int warps, slots; };
#define F2K_NUM_VARIANTS 4
static const F2kVariant kF2kVariants[F2K_NUM_VARIANTS] = {{11, 2}, {10, 2}, {8, 2}, {14, 1}};

static inline bool fast2048_supported(const DevPlan &p) {
  return p.N == 2048 && p.packed && p.L > 2 && p.L <= 2048 && p.C <= 128 && p.M <= 256;
}

template <int DT, int LCT, int WARPS, int SLOTS>
static int f2k_go(bool launch, size_t smem, const DevPlan &p, const Fast2048Tables &t, const DevBatch &b, dim3 grid, cudaStream_t stream) {
  auto kern = b200feat_fast2048_kernel<DT, LCT, WARPS, SLOTS>;
  if (!launch)
    return cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) == cudaSuccess ? 0 : B200FEAT_ECUDA;
  kern<<<grid, dim3(WARPS * 32), smem, stream>>>(p, t, b);
  return 0;
}

template <int DT, int LCT>
static int f2k_shape(int variant, bool launch, size_t smem, const DevPlan &p, const Fast2048Tables &t, const DevBatch &b, dim3 grid,
                     cudaStream_t stream) {
  if (variant == 1) return f2k_go<DT, LCT, 10, 2>(launch, smem, p, t, b, grid, stream);
  if (variant == 2) return f2k_go<DT, LCT, 8, 2>(launch, smem, p, t, b, grid, stream);
  if (variant == 3) return f2k_go<DT, LCT, 14, 1>(launch, smem, p, t, b, grid, stream);
  return f2k_go<DT, LCT, 11, 2>(launch, smem, p, t, b, grid, stream);
}

static inline int f2k_ct_length(int L) { return (L == 1200 || L == 1102) ? L : 0; }

static int f2k_dispatch(int dt, int L, int variant, bool launch, size_t smem, const DevPlan &p, const Fast2048Tables &t,
                        const DevBatch &b, dim3 grid, cudaStream_t stream) {
  if (L == 1200) return dt == B200FEAT_I16 ? f2k_shape<B200FEAT_I16, 1200>(variant, launch, smem, p, t, b, grid, stream)
                                           : f2k_shape<B200FEAT_F32, 1200>(variant, launch, smem, p, t, b, grid, stream);
  if (L == 1102) return dt == B200FEAT_I16 ? f2k_shape<B200FEAT_I16, 1102>(variant, launch, smem, p, t, b, grid, stream)
                                           : f2k_shape<B200FEAT_F32, 1102>(variant, launch, smem, p, t, b, grid, stream);
  return dt == B200FEAT_I16 ? f2k_shape<B200FEAT_I16, 0>(variant, launch, smem, p, t, b, grid, stream)
                            : f2k_shape<B200FEAT_F32, 0>(variant, launch, smem, p, t, b, grid, stream);
}

// the constant tables of the FFT stages (also used by scripts/micro/f2k_host_check.cu)
static inline void f2k_fft_tables(std::vector<float2> &tw1, std::vector<float2> &tw2, std::vector<float2> &w2k) {
  tw1.resize(256); tw2.resize(4 * 256); w2k.resize(128);
  for (int k1 = 0; k1 < 16; ++k1)
    for (int n2 = 0; n2 < 16; ++n2) {
      const double a = -2.0 * M_PI * (double)((n2 * k1) % 256) / 256.0;
      tw1[k1 * 16 + n2] = make_float2((float)cos(a), (float)sin(a));
    }
  for (int n3 = 0; n3 < 4; ++n3)
    for (int k = 0; k < 256; ++k) {
      const double a = -2.0 * M_PI * (double)((n3 * k) % 1024) / 1024.0;
      tw2[n3 * 256 + k] = make_float2((float)cos(a), (float)sin(a));
    }
  for (int k = 0; k < 128; ++k) {
    const double a = -2.0 * M_PI * (double)k / 2048.0;
    w2k[k] = make_float2((float)cos(a), (float)sin(a));
  }
}

static inline int fast2048_prepare(DevPlan &p, const std::vector<float> &bank, std::vector<void *> &allocs,
                                   int *frames_per_tile, const std::vector<float> &window, Fast2048Host *out) {
  Fast2048Host hst;
  std::vector<float2> win2(16 * 2 * 32), tw1, tw2, w2k;
  for (int n1 = 0; n1 < 16; ++n1)
    for (int c = 0; c < 2; ++c)
      for (int l = 0; l < 32; ++l) {
        const int j = 128 * n1 + 64 * c + 2 * l;
        win2[(n1 * 2 + c) * 32 + l] = make_float2(j < p.L ? window[j] : 0.f, j + 1 < p.L ? window[j + 1] : 0.f);
      }
  f2k_fft_tables(tw1, tw2, w2k);
  // balanced work items of F2K_PIECE taps, every round padded to the full piece, an even number of rounds
  MelItems mr = pack_mel_items_T(bank, p.K, p.M, p.use_mag ? 0.5f : 0.25f, 32, 4, F2K_PIECE, /*uniform=*/true);
  if (mr.rounds & 1) {
    mr.rounds += 1;
    mr.rstart.resize((size_t)mr.rounds * 32, 0);
    mr.wdense.resize((size_t)mr.rounds * F2K_PIECE * 32, 0.f);
  }
  int qmax = 0;
  for (int m = 0; m < p.M; ++m) qmax = std::max(qmax, mr.qcount[m]);
  if (mr.max_reach > F2K_PBINS || 3 * (mr.rounds * 32 + ((p.M + 3) & ~3)) > F2K_XBUF * 2) return B200FEAT_EUNSUPPORTED;
  hst.t.mel_rounds = mr.rounds;
  hst.t.mel_qmax = qmax;
  int rc;
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
    hst.t.off_tw2 = append(tw2.data(), tw2.size() * sizeof(float2));
    hst.t.off_w2k = append(w2k.data(), w2k.size() * sizeof(float2));
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
  if (const char *e = getenv("B200FEAT_FAST2048_VARIANT")) forced = atoi(e);
  hst.variant = -1;
  for (int v = 0; v < F2K_NUM_VARIANTS; ++v) {
    if (forced >= 0 && forced < F2K_NUM_VARIANTS && v != forced) continue;
    if (fast2048_smem_bytes(hst.t, kF2kVariants[v].warps, kF2kVariants[v].slots) <= (size_t)226 * 1024) { hst.variant = v; break; }
  }
  if (hst.variant < 0) return B200FEAT_EUNSUPPORTED;
  const F2kVariant shape = kF2kVariants[hst.variant];
  hst.smem = fast2048_smem_bytes(hst.t, shape.warps, shape.slots);
  DevBatch none{};
  for (int dt = 0; dt < 2; ++dt)
    if (f2k_dispatch(dt, f2k_ct_length(p.L), hst.variant, false, hst.smem, p, hst.t, none, dim3(1), nullptr)) return B200FEAT_ECUDA;
  *out = hst;
  *frames_per_tile = shape.warps * shape.slots;
  return 0;
}

static inline int fast2048_launch(const DevPlan &p, const Fast2048Host &hst, const DevBatch &b, int dt, int sm_count, cudaStream_t stream) {
  int64_t blocks = b.num_tiles;
  if (blocks > sm_count) blocks = sm_count;
  f2k_dispatch(dt, f2k_ct_length(p.L), hst.variant, true, hst.smem, p, hst.t, b, dim3((unsigned)blocks), stream);
  return (int)cudaGetLastError();
}
