// Fast fused kernel for fft_length N = L = 400 (16 kHz, 25 ms frames with round_to_power_of_two=False — the
// "n_fft = 400" geometry): the 400-point real FFT is a packed 200-point complex FFT computed with the prime-factor
// (Good-Thomas) algorithm 200 = 8 x 25, which needs NO twiddles between its two stages.
//
//   A QUARTER-WARP (8 lanes) owns one frame.
//   1. the 8 lanes copy the frame's 400 raw samples global -> shared (coalesced 64 B per row), summing them for the DC mean;
//   2. lane a gathers z[m], m = (25a + 8b) mod 200, b = 0..24, from shared memory (bank-conflict-free: 50a + 16b words),
//      applies DC removal / pre-emphasis / window (window pairs stored in the same permuted order);
//   3. 25-point DFT over b in registers (5 x 5 Cooley-Tukey: ten 5-point Winograd-style butterflies, 16 constant twiddles);
//   4. 25 x 8 exchange through the same shared tile (rows of 80 B keep the 128-bit row reads conflict-free);
//      lane l runs the 8-point DFTs of rows l, l+8, l+16 (lane 0 also row 24) and writes them back in place:
//      Z[(25 k1 + 176 r) mod 200] = row r, element k1                                   (CRT output map)
//   5. real-FFT split: lane l takes element k1 = l of rows r = 0..12 and pairs it with element (8 - l) of row 25 - r
//      (bins k and 200 - k), twiddle W400^k from a [row][lane] table;  |2X|^2 -> P[frame][bin] (201 bins);
//   6. mel rounds of 16 filters (two per lane) on 128-bit loads, log, store.
//
// Replaces the same reference code as fast512.cuh (lhotse/features/kaldi/layers.py:151-186, :32-42, :565-578, :708-724,
// framing :727-772) for Wav2LogFilterBank(round_to_power_of_two=False) & co (layers.py:264-265).
#pragma once
#include "fast256.cuh"

#define F400_N 400
#ifndef F400_SLOTS
#define F400_SLOTS 2                        // frames per quarter-warp per tile
#endif
#define F400_XROW 10                        // float2 per exchange row (8 + 2 pad: 80 B)
#define F400_XBUF 264                        // float2 per quarter-warp tile: 25 rows (2000 B; also holds the 400 raw samples),
                                            // padded to 16 (mod 32) words so that neighbouring quarter-warps sit on disjoint banks
#define F400_PBINS 204                      // floats per P row (201 bins + pad, multiple of 4)
#define F400_PBUF (F400_PBINS * F400_SLOTS)
#define F400_PTAIL 64

// W25^e = exp(-2 pi i e / 25) for the exponents b2*c1 (b2, c1 = 1..4) of the 5 x 5 factorisation
__device__ __forceinline__ float2 w25_const(int e) {
  switch (e) {
    case 1: return make_float2(0.96858316112863107605f, -0.24868988716485479484f);
    case 2: return make_float2(0.87630668004386358394f, -0.48175367410171532345f);
    case 3: return make_float2(0.72896862742141155245f, -0.68454710592868861507f);
    case 4: return make_float2(0.53582679497899654564f, -0.84432792550201507531f);
    case 6: return make_float2(0.06279051952931352654f, -0.99802672842827155897f);
    case 8: return make_float2(-0.42577929156507271502f, -0.90482705246601946580f);
    case 9: return make_float2(-0.63742398974868974548f, -0.77051324277578925326f);
    case 12: return make_float2(-0.99211470131447776488f, -0.12533323356430453588f);
    default: return make_float2(-0.63742398974868952344f, 0.77051324277578936428f);  // 16
  }
}

// forward 5-point DFT in registers, natural order in and out
__device__ __forceinline__ void dft5(float2 &x0, float2 &x1, float2 &x2, float2 &x3, float2 &x4) {
  constexpr float C1 = 0.30901699437494742410f, C2 = -0.80901699437494742410f;   // cos(2pi/5), cos(4pi/5)
  constexpr float S1 = 0.95105651629515357212f, S2 = 0.58778525229247312917f;    // sin(2pi/5), sin(4pi/5)
  const float2 s1 = f2add(x1, x4), d1 = f2sub(x1, x4), s2 = f2add(x2, x3), d2 = f2sub(x2, x3);
  const float2 a1 = make_float2(__fmaf_rn(s2.x, C2, __fmaf_rn(s1.x, C1, x0.x)), __fmaf_rn(s2.y, C2, __fmaf_rn(s1.y, C1, x0.y)));
  const float2 a2 = make_float2(__fmaf_rn(s2.x, C1, __fmaf_rn(s1.x, C2, x0.x)), __fmaf_rn(s2.y, C1, __fmaf_rn(s1.y, C2, x0.y)));
  const float2 b1 = make_float2(__fmaf_rn(d2.x, S2, __fmul_rn(d1.x, S1)), __fmaf_rn(d2.y, S2, __fmul_rn(d1.y, S1)));
  const float2 b2 = make_float2(__fmaf_rn(d2.x, -S1, __fmul_rn(d1.x, S2)), __fmaf_rn(d2.y, -S1, __fmul_rn(d1.y, S2)));
  x0 = f2add(x0, f2add(s1, s2));
  x1 = f2add(a1, f2mi(b1));  // a1 - i*b1
  x4 = f2add(a1, f2pi(b1));  // a1 + i*b1
  x2 = f2add(a2, f2mi(b2));
  x3 = f2add(a2, f2pi(b2));
}

// forward 25-point DFT in registers: input v[b], output A[k] in v[k] (natural order)
__device__ __forceinline__ void dft25(float2 (&v)[25]) {
  // b = 5*b1 + b2, k = c1 + 5*c2:  A[c1 + 5 c2] = sum_b2 W25^(b2 c1) W5^(b2 c2) [ sum_b1 W5^(b1 c1) v[5 b1 + b2] ]
#pragma unroll
  for (int b2 = 0; b2 < 5; ++b2) dft5(v[b2], v[5 + b2], v[10 + b2], v[15 + b2], v[20 + b2]);  // -> v[5 c1 + b2]
#pragma unroll
  for (int c1 = 1; c1 < 5; ++c1)
#pragma unroll
    for (int b2 = 1; b2 < 5; ++b2) v[5 * c1 + b2] = f2mul(v[5 * c1 + b2], w25_const(b2 * c1));
#pragma unroll
  for (int c1 = 0; c1 < 5; ++c1) dft5(v[5 * c1], v[5 * c1 + 1], v[5 * c1 + 2], v[5 * c1 + 3], v[5 * c1 + 4]);  // -> v[5 c1 + c2]
  // v[5 c1 + c2] holds A[c1 + 5 c2]: transpose the 5 x 5 register block to natural order (register renaming only)
#pragma unroll
  for (int c1 = 0; c1 < 5; ++c1)
#pragma unroll
    for (int c2 = c1 + 1; c2 < 5; ++c2) {
      const float2 t = v[5 * c1 + c2];
      v[5 * c1 + c2] = v[5 * c2 + c1];
      v[5 * c2 + c1] = t;
    }
}

struct Fast400Tables {
  // one 16-byte-aligned blob (TMA bulk copy):
  //   [win2: 25*8 float2 (w[2m], w[2m+1]), m = (25 lane + 8 b) mod 200, indexed [b][lane]]
  //   [tws : 13*8 float2 W400^k, k = (25 lane + 176 r) mod 200, indexed [r][lane]]
  //   [rdesc: rounds*16 int4 {first bin, trips, weight index, 0} | wdense: [row/4][16][4] float]
  const void *cblob;
  int cblob_bytes;
  int off_tws, off_rdesc, off_mw;
  int mel_rounds;
};

static inline size_t fast400_smem_bytes(const Fast400Tables &t, int warps) {
  size_t b = (size_t)(4 * warps) * (F400_XBUF * 8 + F400_PBUF * 4) + F400_PTAIL * 4;
  b += (size_t)t.cblob_bytes + 16;
  return (b + 15) & ~(size_t)15;
}

template <int DT, int WARPS>
__global__ void __launch_bounds__(WARPS * 32, 2)
b200feat_fast400_kernel(const DevPlan p, const Fast400Tables ft, const DevBatch b) {
  constexpr int QW = 4 * WARPS, TILE = QW * F400_SLOTS, L = F400_N;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int tid = threadIdx.x;
  const int l = tid & 7;            // lane within the quarter-warp
  const int qw = tid >> 3;          // quarter-warp within the CTA

  float2 *xall = reinterpret_cast<float2 *>(smem_raw);
  float *pall = reinterpret_cast<float *>(xall + (size_t)QW * F400_XBUF);
  unsigned char *s_const = reinterpret_cast<unsigned char *>(pall + (size_t)QW * F400_PBUF + F400_PTAIL);
  const float2 *s_win = reinterpret_cast<const float2 *>(s_const);                 // [b][lane] window pairs (permuted)
  const float2 *s_tws = reinterpret_cast<const float2 *>(s_const + ft.off_tws);    // [r][lane] split twiddles
  const int4 *s_rdesc = reinterpret_cast<const int4 *>(s_const + ft.off_rdesc);    // [round][16 filters]
  const float4 *s_mw4 = reinterpret_cast<const float4 *>(s_const + ft.off_mw);     // [row / 4][16][4]
  unsigned long long *s_bar = reinterpret_cast<unsigned long long *>(s_const + ft.cblob_bytes);
  float2 *X = xall + (size_t)qw * F400_XBUF;
  float *S = reinterpret_cast<float *>(X);   // the same tile first holds the frame's raw samples
  float *P = pall + (size_t)qw * F400_PBUF;  // [slot][F400_PBINS]

  const unsigned bar = smem_u32(s_bar);
  blob_copy_start(bar, s_const, ft.cblob, ft.cblob_bytes);  // constant tables: one TMA bulk copy
  for (int i = tid; i < QW * F400_PBUF + F400_PTAIL; i += blockDim.x) pall[i] = 0.f;  // never NaN under zero weights
  const float inv_L = 1.0f / (float)L;
  mbar_wait(bar, 0);
  __syncthreads();

  for (int64_t tg = blockIdx.x; tg < b.num_tiles; tg += gridDim.x) {
    const int64_t tile = b.tile_base + tg;
    const int cut = __ldg(b.tile_cut + tile) - b.batch_first;
    const int64_t t0 = (tile - __ldg(b.tile_off + cut)) * TILE + (int64_t)qw * F400_SLOTS;
    const int64_t T = __ldg(b.row_off + cut + 1) - __ldg(b.row_off + cut);
    const int64_t rows_here = b.out_mode == B200FEAT_OUT_PADDED ? b.max_frames : T;
    if (!__any_sync(F512_FULL, t0 < rows_here)) continue;  // all four quarters idle for this tile
    const int64_t n = __ldg(b.nsamp + cut);
    const int64_t xoff = __ldg(b.samp_off + cut);
    const int64_t row0 = b.out_mode == B200FEAT_OUT_PADDED ? (int64_t)(b.batch_first + cut) * b.max_frames + t0
                                                           : __ldg(b.row_off + cut) + t0;
    const int nvalid = (int)max((int64_t)0, min((int64_t)F400_SLOTS, T - t0));
    // whisper-fbank: only the stft's n / S frames feed the cut-wide maximum (whisper_fbank.py:63-68)
    const int nmaxed = p.whisper ? (int)max((int64_t)0, min((int64_t)F400_SLOTS, n / p.S - t0)) : 0;
    float le[F400_SLOTS];
#pragma unroll
    for (int k = 0; k < F400_SLOTS; ++k) le[k] = 0.f;

#pragma unroll 1
    for (int f = 0; f < F400_SLOTS; ++f) {
      if (!__any_sync(F512_FULL, f < nvalid)) continue;
      const int64_t t = min(max(t0 + f, (int64_t)0), T - 1);  // out-of-range quarters redo the last frame (not stored)
      const int64_t base = t * p.S - (p.snip_edges ? 0 : p.pad_left);
      // ---- 1. raw samples -> shared, lane l copies the pairs (16 i + 2 l, +1), i = 0..24
      float s = 0.f;
      const bool interior = base >= 0 && base + L <= n && (((xoff + base) & 1) == 0);
      if (__all_sync(F512_FULL, interior)) {
        if (DT == B200FEAT_I16) {
          const int16_t *xp = reinterpret_cast<const int16_t *>(b.samples) + (xoff + base + 2 * l);
#pragma unroll
          for (int i = 0; i < 25; ++i) {
            const short2 q = __ldg(reinterpret_cast<const short2 *>(xp + 16 * i));
            const float2 x = make_float2((float)q.x * (1.0f / 32768.0f), (float)q.y * (1.0f / 32768.0f));
            *reinterpret_cast<float2 *>(S + 16 * i + 2 * l) = x;
            s += x.x + x.y;
          }
        } else {
          const float *xp = reinterpret_cast<const float *>(b.samples) + (xoff + base + 2 * l);
#pragma unroll
          for (int i = 0; i < 25; ++i) {
            const float2 x = __ldg(reinterpret_cast<const float2 *>(xp + 16 * i));
            *reinterpret_cast<float2 *>(S + 16 * i + 2 * l) = x;
            s += x.x + x.y;
          }
        }
      } else {  // a cut edge in this warp: per-tap reflection (layers.py:753-772)
#pragma unroll 5
        for (int i = 0; i < 25; ++i) {
          int64_t ia = base + 16 * i + 2 * l, ib = ia + 1;
          if (!p.snip_edges) { ia = reflect_index(ia, n, p.pad_mode); ib = reflect_index(ib, n, p.pad_mode); }
          const float2 x = make_float2(ld_sample<DT>(b.samples, xoff + ia), ld_sample<DT>(b.samples, xoff + ib));
          *reinterpret_cast<float2 *>(S + 16 * i + 2 * l) = x;
          s += x.x + x.y;
        }
      }
      const float mu = p.remove_dc ? qw_sum(s) * inv_L : 0.f;
      __syncwarp();
      // ---- 2. gather in prime-factor order, DC removal, energy, pre-emphasis, window (layers.py:155-170)
      float2 v[25];
      float e = 0.f;
      if (p.preemph != 0.f) {
        int m = 25 * l;  // (25 l + 8 b) mod 200
#pragma unroll
        for (int bb = 0; bb < 25; ++bb) {
          const float2 x = *reinterpret_cast<const float2 *>(S + 2 * m);
          const float xp = S[max(2 * m - 1, 0)];          // replicate-left for the frame's first tap (layers.py:166)
          const float2 w = s_win[bb * 8 + l];
          const float2 d = f2add(x, make_float2(-mu, -mu));
          const float dp = xp - mu;
          if (p.raw_energy) e = fmaf(d.x, d.x, fmaf(d.y, d.y, e));
          const float2 y = preemph_window2(d, dp, p.preemph, w);
          if (!p.raw_energy) e = fmaf(y.x, y.x, fmaf(y.y, y.y, e));
          v[bb] = y;
          m += 8;
          m = m >= 200 ? m - 200 : m;
        }
      } else {  // no pre-emphasis (whisper-fbank, librosa-fbank, preemph_coeff = 0): no neighbour tap to fetch
        int m = 25 * l;
#pragma unroll
        for (int bb = 0; bb < 25; ++bb) {
          const float2 x = *reinterpret_cast<const float2 *>(S + 2 * m);
          const float2 w = s_win[bb * 8 + l];
          const float2 d = f2add(x, make_float2(-mu, -mu));
          if (p.raw_energy) e = fmaf(d.x, d.x, fmaf(d.y, d.y, e));
          const float2 y = make_float2(__fmul_rn(d.x, w.x), __fmul_rn(d.y, w.y));
          if (!p.raw_energy) e = fmaf(y.x, y.x, fmaf(y.y, y.y, e));
          v[bb] = y;
          m += 8;
          m = m >= 200 ? m - 200 : m;
        }
      }
      if (p.use_energy) {
        const float lev = log_energy_value(p, qw_sum(e));
#pragma unroll
        for (int k = 0; k < F400_SLOTS; ++k) le[k] = (f == k) ? lev : le[k];
      }
      // ---- 3. 25-point DFT over b in registers
      dft25(v);
      __syncwarp();  // every lane has read its samples: the tile can be overwritten
      // ---- 4. exchange: T[k2][a], then the 8-point DFTs over a of rows l, l+8, l+16 (and 24), written back in place
#pragma unroll
      for (int k2 = 0; k2 < 25; ++k2) X[k2 * F400_XROW + l] = v[k2];
      __syncwarp();
#pragma unroll
      for (int rr = 0; rr < 4; ++rr) {
        const int r = rr < 3 ? l + 8 * rr : 24;  // the fourth pass is row 24: every lane reads it, lane 0 owns it
        float4 *row = reinterpret_cast<float4 *>(X + r * F400_XROW);
        float2 z[8];
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const float4 r4 = row[q];
          z[2 * q] = make_float2(r4.x, r4.y);
          z[2 * q + 1] = make_float2(r4.z, r4.w);
        }
        dft8(z[0], z[1], z[2], z[3], z[4], z[5], z[6], z[7]);
        if (rr == 3) __syncwarp();  // all lanes have read row 24 before lane 0 rewrites it
        if (rr < 3 || l == 0) {
#pragma unroll
          for (int q = 0; q < 4; ++q) row[q] = make_float4(z[2 * q].x, z[2 * q].y, z[2 * q + 1].x, z[2 * q + 1].y);
        }
      }
      __syncwarp();
      // ---- 5. real-FFT split + power (layers.py:38-42): element l of row r against element (8-l) of row 25-r
      float *Pf = P + f * F400_PBINS;
      {
        const int lm = (8 - l) & 7;
        int k = 25 * l;  // (25 l + 176 r) mod 200
#pragma unroll
        for (int r = 0; r < 13; ++r) {
          const float2 zk = X[r * F400_XROW + l];
          const float2 cc = f2conj(X[((25 - r) % 25) * F400_XROW + lm]);
          const float2 E = f2add(zk, cc), O = f2sub(zk, cc);
          const float2 mit = f2mi(f2mul(O, s_tws[r * 8 + l]));  // -i * W400^k * O
          const float2 a = f2add(E, mit), bq = f2sub(E, mit);   // 2*X[k], 2*conj(X[200-k])
          float pa = fmaf(a.x, a.x, a.y * a.y), pb = fmaf(bq.x, bq.x, bq.y * bq.y);
          if (p.use_mag) { pa = sqrtf(pa); pb = sqrtf(pb); }
          if (r > 0 || l <= 4) {  // row 0 pairs with itself: lanes 5..7 would repeat lanes 3..1
            Pf[k] = pa;
            Pf[200 - k] = pb;
          }
          k -= 24;
          k = k < 0 ? k + 200 : k;
        }
      }
      __syncwarp();  // the tile is free for the next frame's samples
    }

    // ---- 6. epilogue over the (up to) F400_SLOTS frames of this quarter-warp
    const int nrows = (int)max((int64_t)0, min((int64_t)F400_SLOTS, rows_here - t0));
    float *out = b.out + row0 * p.F;
    if (p.feature == B200FEAT_SPECTROGRAM || p.feature == B200FEAT_LOG_SPECTROGRAM) {
      for (int f = 0; f < nrows; ++f) {
        float *o = out + (int64_t)f * p.F;
        if (f >= nvalid) { for (int k = l; k < p.F; k += 8) o[k] = post_affine(p, k, b.pad_value); continue; }
        for (int k = l; k < p.K; k += 8) {
          float x = P[f * F400_PBINS + k] * (p.use_mag ? 0.5f : 0.25f);
          if (p.feature == B200FEAT_LOG_SPECTROGRAM) x = log_spec_value(p, x);
          if (k == 0 && p.use_energy) {
#pragma unroll
            for (int g = 0; g < F400_SLOTS; ++g) x = (f == g) ? le[g] : x;
          }
          o[k] = post_affine(p, k, x);
        }
      }
    } else {
      const int shift = mel_shift(p), ecol = energy_col(p);
      const int Mpad = (p.M + 3) & ~3;
      float *mlog = reinterpret_cast<float *>(X);  // the exchange tile is idle during the epilogue
      const float lgk = p.log10_mel ? 0.30102999566398119521f : 0.69314718055994530942f;  // log10 (whisper_fbank.py:67) or ln
      float vmax = __int_as_float(0xff800000);
      // rounds of 16 filters, two per lane (l and l + 8): the per-round overhead is shared by 2 filters x 2 frames
      for (int j = 0; j < ft.mel_rounds; ++j) {
        const int4 ra = s_rdesc[j * 16 + l], rb = s_rdesc[j * 16 + l + 8];
        const float4 *pa = reinterpret_cast<const float4 *>(P + ra.x), *pb = reinterpret_cast<const float4 *>(P + rb.x);
        const float4 *wa = s_mw4 + ra.z, *wb = s_mw4 + rb.z;
        float acc[2][F400_SLOTS];
#pragma unroll
        for (int f = 0; f < F400_SLOTS; ++f) acc[0][f] = acc[1][f] = 0.f;
#pragma unroll 1
        for (int i = ra.y; i > 0; i -= 4, ++pa, ++pb, wa += 16, wb += 16) {
          const float4 ua = *wa, ub = *wb;
#pragma unroll
          for (int f = 0; f < F400_SLOTS; ++f) {
            const float4 qa = pa[f * (F400_PBINS / 4)], qb = pb[f * (F400_PBINS / 4)];
            acc[0][f] = fmaf(qa.w, ua.w, fmaf(qa.z, ua.z, fmaf(qa.y, ua.y, fmaf(qa.x, ua.x, acc[0][f]))));
            acc[1][f] = fmaf(qb.w, ub.w, fmaf(qb.z, ub.z, fmaf(qb.y, ub.y, fmaf(qb.x, ub.x, acc[1][f]))));
          }
        }
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int m = l + 8 * h + 16 * j;
          if (m < p.M) {
            float r[F400_SLOTS];
#pragma unroll
            for (int f = 0; f < F400_SLOTS; ++f) {
              r[f] = fast_lg2_normal(nanmax(acc[h][f], p.mel_floor)) * lgk;
              if (f < nmaxed) vmax = nanmax(vmax, r[f]);
            }
            if (p.feature != B200FEAT_MFCC) {
              float *orow = out + m + shift;
#pragma unroll
              for (int f = 0; f < F400_SLOTS; ++f)
                if (f < nvalid) orow[(int64_t)f * p.F] = post_affine(p, m + shift, r[f]);
            } else {
#pragma unroll
              for (int f = 0; f < F400_SLOTS; ++f) mlog[f * Mpad + m] = r[f];
            }
          }
        }
      }
      if (p.whisper) {  // one atomic per warp: its four quarter-warps work on the same cut
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) vmax = nanmax(vmax, __shfl_xor_sync(F512_FULL, vmax, o));
        if ((tid & 31) == 0 && vmax != __int_as_float(0xff800000)) atomic_max_float(b.cut_max + cut, vmax);
      } else if (p.feature == B200FEAT_FBANK) {
        if (p.use_energy && l < nvalid) {
          float v0 = 0.f;
#pragma unroll
          for (int f = 0; f < F400_SLOTS; ++f) v0 = (l == f) ? le[f] : v0;
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
            for (int g = 0; g < F400_SLOTS; ++g) acc = (f == g) ? le[g] : acc;
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
#ifndef F400_WARPS
#define F400_WARPS 7
#endif
struct Fast400Host {
  Fast400Tables t;
  size_t smem;
};

static inline bool fast400_supported(const DevPlan &p) {
  return p.N == F400_N && p.L == F400_N && p.packed && p.C <= 128 && F400_SLOTS * ((p.M + 3) & ~3) <= 2 * F400_XBUF;
}

template <int DT>
static int f400_go(bool launch, size_t smem, const DevPlan &p, const Fast400Tables &t, const DevBatch &b, dim3 grid, cudaStream_t stream) {
  return configure_or_launch(b200feat_fast400_kernel<DT, F400_WARPS>, F400_WARPS * 32, launch, smem, p, t, b, grid, stream);
}

static inline int fast400_prepare(DevPlan &p, const std::vector<float> &bank, std::vector<void *> &allocs,
                                  int *frames_per_tile, const std::vector<float> &window, Fast400Host *out) {
  Fast400Host hst;
  std::vector<float2> win2(25 * 8), tws(13 * 8);
  for (int bb = 0; bb < 25; ++bb)
    for (int l = 0; l < 8; ++l) {
      const int m = (25 * l + 8 * bb) % 200;
      win2[bb * 8 + l] = make_float2(window[2 * m], window[2 * m + 1]);
    }
  for (int r = 0; r < 13; ++r)
    for (int l = 0; l < 8; ++l) {
      const int k = (25 * l + 176 * r) % 200;
      const double a = -2.0 * M_PI * (double)k / 400.0;
      tws[r * 8 + l] = make_float2((float)cos(a), (float)sin(a));
    }
  const MelRounds mr = pack_mel_rounds(bank, p.K, p.M, p.use_mag ? 0.5f : 0.25f, 16, 4, F400_PBINS / 4 * 4);  // 16 filters per round, two per lane
  if (mr.max_reach > F400_PBINS) return B200FEAT_EUNSUPPORTED;
  hst.t.mel_rounds = mr.rounds;
  ConstBlob blob;
  blob.append(win2);
  hst.t.off_tws = blob.append(tws);
  hst.t.off_rdesc = blob.append(mel_round_descs(mr));
  hst.t.off_mw = blob.append(mr.wdense);
  if (blob.upload(allocs, &hst.t.cblob, &hst.t.cblob_bytes)) return B200FEAT_ECUDA;
  hst.smem = fast400_smem_bytes(hst.t, F400_WARPS);
  if (hst.smem > 113 * 1024) return B200FEAT_EUNSUPPORTED;  // keep 2 CTAs per SM
  DevBatch none{};
  if (f400_go<B200FEAT_F32>(false, hst.smem, p, hst.t, none, dim3(1), nullptr)) return B200FEAT_ECUDA;
  if (f400_go<B200FEAT_I16>(false, hst.smem, p, hst.t, none, dim3(1), nullptr)) return B200FEAT_ECUDA;
  *out = hst;
  *frames_per_tile = 4 * F400_WARPS * F400_SLOTS;
  return 0;
}

static inline int fast400_launch(const DevPlan &p, const Fast400Host &hst, const DevBatch &b, int dt, int sm_count, cudaStream_t stream) {
  const dim3 grid(persistent_grid(b.num_tiles, sm_count, 2));
  if (dt == B200FEAT_I16) f400_go<B200FEAT_I16>(true, hst.smem, p, hst.t, b, grid, stream);
  else f400_go<B200FEAT_F32>(true, hst.smem, p, hst.t, b, grid, stream);
  return (int)cudaGetLastError();
}
