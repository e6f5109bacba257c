// Fast fused kernel for fft_length N = 512 (the 16 kHz / 25 ms headline geometry and every other
// plan with 256 < L <= 512): one HALF-WARP owns one frame; the 512-point real FFT is a packed
// 256-point complex FFT factored 16 x 16 and kept in registers:
//
//   lane l holds z[16*n1 + l], n1 = 0..15         (z[n] = y[2n] + i*y[2n+1], y = windowed frame)
//   radix-16 DFT over n1 in registers  -> Y[k1][l], times W256^(l*k1)
//   16x16 transpose through a padded shared-memory tile (the only FFT traffic that leaves registers)
//   lane k1 holds Y'[k1][0..15], radix-16 DFT over n2 -> Z[k1 + 16*k2]
//   real-FFT split against the mirrored lane (16 - k1), whose slots come through the idle transpose tile -> |X[k]|^2
//   power spectrum of 4 consecutive frames staged as P[k][4] -> sparse mel bank with the weights
//   shared by the 4 frames (LDS.128) -> log -> coalesced 64-byte row segments.
//
// Replaces, for one frame, lhotse/features/kaldi/layers.py:151-186 (Wav2Win._forward_strided),
// :32-42 (_rfft/_pow_spectrogram), :565-578 (mel+log), :708-724 (DCT/lifter), with the framing of
// :727-772 folded into the load addresses.  HBM traffic: 4*S bytes in, 4*F bytes out per frame.
#pragma once
#include <string.h>

#include <algorithm>
#include <vector>

#include "common.cuh"

// Launch shape is a template parameter set (see Fast512Variant below): WARPS per CTA, SLOTS = frames per half-warp
// per tile (the mel loop shares each weight across SLOTS frames), TWS = stage-1 twiddles in shared memory instead of
// 30 registers, MINB = CTAs per SM the register allocator must leave room for.
#define F512_XROW 18                        // float2 per transpose row (16 + 2 pad: 144 B, LDS.128 conflict-free)
#define F512_XBUF (16 * F512_XROW)          // float2 per half-warp transpose tile
// floats per P row: 257 bins + pad chosen so that SLOTS * PBINS = 16 (mod 32): the two half-warps of a warp then sit on
// disjoint banks when they store the same bin of their frames
#define F512_PBINS(SLOTS) ((SLOTS) == 4 ? 260 : 264)
// F512_PREV_SHFL 1: the pre-emphasis neighbour x[j-1] comes from the adjacent lane by shuffle instead of a second load
#ifndef F512_PREV_SHFL
#define F512_PREV_SHFL 1
#endif
#ifndef F512_PREFETCH
#define F512_PREFETCH 2
#endif
#define F512_PTAIL 64                       // zeroed slack after the last tile (mel reads run past short filters)

struct Fast512Tables {  // derived once per handle
  // All per-plan constants the kernel keeps in shared memory live in ONE 16-byte-aligned device blob so that a CTA
  // fetches them with a single bulk asynchronous copy (TMA unit, cp.async.bulk + mbarrier) at start-up:
  //   [win2: 256 float2 window pairs (w[32*n1+2l], w[32*n1+2l+1]), zero beyond L]
  //   [tw1 : 256 float2 W256^(l*k1) indexed [k1][l]        (only when the variant keeps them in shared memory)]
  //   [rstart: rounds*16 int | rlen: rounds int | rrow: rounds int (each padded to 16 B)]
  //   [wdense: rows*16 float zero-padded mel weights]
  const void *cblob;
  int cblob_bytes;
  int off_tw1, off_rdesc, off_mw;  // byte offsets inside the blob
  const float2 *tw1;    // [16][16] W256^(l*k1) (global copy: loaded into registers by the default variant)
  const float2 *w512;   // [8][16]  W512^(l + 16 i): the real-FFT split twiddle of lane l's pair i
  int mel_rounds;       // ceil(M / 16)
  int mel_wrows;        // sum of the rounds' trip counts
};

// (F512_HD: the pure arithmetic helpers also compile for the host, where scripts/micro/f2k_host_check.cu runs the FFT
// stages of fast2048.cuh lane by lane against a float64 DFT)
#define F512_HD __host__ __device__ __forceinline__
// Complex arithmetic on the (re, im) register pair.  On the device the complex adds are explicitly rounded
// (__fadd_rn): the compiler never fuses a preceding product into them, so every stage rounds where the code says.
F512_HD float2 f2add(float2 a, float2 b) {
#if defined(__CUDA_ARCH__)
  return make_float2(__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y));
#else
  return make_float2(a.x + b.x, a.y + b.y);
#endif
}
F512_HD float2 f2sub(float2 a, float2 b) {
#if defined(__CUDA_ARCH__)
  return make_float2(__fadd_rn(a.x, -b.x), __fadd_rn(a.y, -b.y));
#else
  return make_float2(a.x - b.x, a.y - b.y);
#endif
}
F512_HD float2 f2mi(float2 a) { return make_float2(a.y, -a.x); }   // a * (-i)
F512_HD float2 f2pi(float2 a) { return make_float2(-a.y, a.x); }   // a * (+i)
F512_HD float2 f2conj(float2 a) { return make_float2(a.x, -a.y); }
F512_HD float2 f2mul(float2 a, float2 b) {  // complex product a * b
  return make_float2(fmaf(a.x, b.x, -a.y * b.y), fmaf(a.x, b.y, a.y * b.x));
}

// forward 4-point DFT, in place, natural order: 8 complex adds (the two rotations by -/+ i are swaps and sign flips folded into them)
F512_HD void dft4(float2 &a0, float2 &a1, float2 &a2, float2 &a3) {
  const float2 s02 = f2add(a0, a2), d02 = f2sub(a0, a2);
  const float2 s13 = f2add(a1, a3), d13 = f2sub(a1, a3);
  a0 = f2add(s02, s13);
  a2 = f2sub(s02, s13);
  a1 = f2add(d02, f2mi(d13));  // d02 - i*d13
  a3 = f2add(d02, f2pi(d13));  // d02 + i*d13
}

#define F512_C1 0.92387953251128674f  // cos(pi/8)
#define F512_S1 0.38268343236508977f  // sin(pi/8)
#define F512_R2 0.70710678118654752f  // sqrt(1/2)

// Multiplications by the eighth roots of unity W8^1 = (1 - i)/sqrt2 and W8^3 = -(1 + i)/sqrt2: a*(1 -+ i) is one complex
// add with a rotated operand (a + (-i)a resp. a + (+i)a) followed by one real scale.
F512_HD float2 f2mul_w8_1(float2 a) {
  const float2 s = f2add(a, f2mi(a));
#if defined(__CUDA_ARCH__)
  return make_float2(__fmul_rn(s.x, F512_R2), __fmul_rn(s.y, F512_R2));
#else
  return make_float2(s.x * F512_R2, s.y * F512_R2);
#endif
}
F512_HD float2 f2mul_w8_3(float2 a) {
  const float2 s = f2add(a, f2pi(a));
#if defined(__CUDA_ARCH__)
  return make_float2(__fmul_rn(s.x, -F512_R2), __fmul_rn(s.y, -F512_R2));
#else
  return make_float2(s.x * -F512_R2, s.y * -F512_R2);
#endif
}

// dft4 whose inputs a2 (Z2) and / or a3 (Z3) are known to be +0: the adds with them are left out (x + 0 = x except
// for the sign of a zero, which no power spectrum keeps)
template <bool Z2, bool Z3>
F512_HD void dft4z(float2 &a0, float2 &a1, float2 &a2, float2 &a3) {
  const float2 s02 = Z2 ? a0 : f2add(a0, a2), d02 = Z2 ? a0 : f2sub(a0, a2);
  const float2 s13 = Z3 ? a1 : f2add(a1, a3), d13 = Z3 ? a1 : f2sub(a1, a3);
  a0 = f2add(s02, s13);
  a2 = f2sub(s02, s13);
  a1 = f2add(d02, f2mi(d13));
  a3 = f2add(d02, f2pi(d13));
}

// forward 16-point DFT in registers (radix 4x4).  Input v[n]; output X[k] lands in v[4*(k&3) + (k>>2)].
// Inputs v[NZ..15] are +0 (a frame shorter than 32 * 16 taps): the first radix-4 pass skips them.
template <int NZ = 16>
F512_HD void dft16(float2 (&v)[16]) {
#pragma unroll
  for (int b = 0; b < 4; ++b) {
    if (8 + b >= NZ) dft4z<true, true>(v[b], v[4 + b], v[8 + b], v[12 + b]);
    else if (12 + b >= NZ) dft4z<false, true>(v[b], v[4 + b], v[8 + b], v[12 + b]);
    else dft4(v[b], v[4 + b], v[8 + b], v[12 + b]);
  }
  // v[4c + b] = y[b][c]; twiddle by W16^(b*c), W16^m = (cos(pi m/8), -sin(pi m/8))
  v[5] = f2mul(v[5], make_float2(F512_C1, -F512_S1));    // W^1
  v[6] = f2mul_w8_1(v[6]);                               // W^2
  v[7] = f2mul(v[7], make_float2(F512_S1, -F512_C1));    // W^3
  v[9] = f2mul_w8_1(v[9]);                               // W^2
  v[10] = f2mi(v[10]);                                   // W^4 = -i
  v[11] = f2mul_w8_3(v[11]);                             // W^6
  v[13] = f2mul(v[13], make_float2(F512_S1, -F512_C1));  // W^3
  v[14] = f2mul_w8_3(v[14]);                             // W^6
  v[15] = f2mul(v[15], make_float2(-F512_C1, F512_S1));  // W^9
#pragma unroll
  for (int c = 0; c < 4; ++c) dft4(v[4 * c], v[4 * c + 1], v[4 * c + 2], v[4 * c + 3]);
}

// Pre-emphasis and window of the DC-free taps (x - mu), two adjacent taps per lane.  Pre-emphasis is linear, so
// pre(x - mu)[j] = x[j] - preemph * x[j-1] - cmu with cmu = mu * (1 - preemph), the replicate-left first tap included:
// three operations per tap, each rounded on its own.
F512_HD float2 preemph_window_dc(float2 x, float xp, float preemph, float cmu, float2 w) {
#if defined(__CUDA_ARCH__)
  return make_float2(__fmul_rn(__fadd_rn(__fmaf_rn(xp, -preemph, x.x), -cmu), w.x),
                     __fmul_rn(__fadd_rn(__fmaf_rn(x.x, -preemph, x.y), -cmu), w.y));
#else
  return make_float2((fmaf(xp, -preemph, x.x) - cmu) * w.x, (fmaf(x.x, -preemph, x.y) - cmu) * w.y);
#endif
}
// register holding output bin k of dft16
#define F512_OUT(k) (4 * ((k) & 3) + ((k) >> 2))

// W32^k2 = exp(-2*pi*i*k2/32), k2 = 0..15 (compile-time immediates after unrolling)
__device__ __forceinline__ float2 w32_const(int k2) {
  const float c[16] = {1.0f, 0.98078528040323043f, 0.92387953251128674f, 0.83146961230254524f,
                       0.70710678118654752f, 0.55557023301960218f, 0.38268343236508977f, 0.19509032201612825f,
                       0.0f, -0.19509032201612825f, -0.38268343236508977f, -0.55557023301960218f,
                       -0.70710678118654752f, -0.83146961230254524f, -0.92387953251128674f, -0.98078528040323043f};
  const float s[16] = {0.0f, 0.19509032201612825f, 0.38268343236508977f, 0.55557023301960218f,
                       0.70710678118654752f, 0.83146961230254524f, 0.92387953251128674f, 0.98078528040323043f,
                       1.0f, 0.98078528040323043f, 0.92387953251128674f, 0.83146961230254524f,
                       0.70710678118654752f, 0.55557023301960218f, 0.38268343236508977f, 0.19509032201612825f};
  return make_float2(c[k2], -s[k2]);
}

template <int DT>
__device__ __forceinline__ float2 ld_pair(const void *base, int64_t i) {  // i even, element index
  if (DT == B200FEAT_I16) {
    const short2 v = __ldg(reinterpret_cast<const short2 *>(reinterpret_cast<const int16_t *>(base) + i));
    return make_float2((float)v.x * (1.0f / 32768.0f), (float)v.y * (1.0f / 32768.0f));
  } else {
    return __ldg(reinterpret_cast<const float2 *>(reinterpret_cast<const float *>(base) + i));
  }
}

// The two half-warps of a warp process different frames but execute in LOCKSTEP: every branch below
// is warp-uniform (decided with __any_sync/__all_sync), so the full-mask shuffles (width 16) and
// __syncwarp() compile to single instructions (a runtime half-mask costs a MATCH/REDUX/VOTE
// sequence per shuffle).  A half whose frame lies beyond its cut recomputes the cut's last frame
// and simply does not store it.
#define F512_FULL 0xffffffffu
__device__ __forceinline__ float hw_sum(float v) {  // sum over the 16 lanes of each half-warp
#pragma unroll
  for (int o = 8; o > 0; o >>= 1) v += __shfl_xor_sync(F512_FULL, v, o, 16);
  return v;
}

static inline size_t fast512_smem_bytes(const DevPlan &p, const Fast512Tables &t, int warps, int slots, int tws) {
  size_t b = (size_t)(2 * warps) * (F512_XBUF * 8 + (size_t)F512_PBINS(slots) * slots * 4) + F512_PTAIL * 4;
  b += (size_t)t.cblob_bytes;  // constant blob (multiple of 16 B)
  b += 16;                     // mbarrier
  (void)p; (void)tws;
  return (b + 15) & ~(size_t)15;
}

// PLAIN: the host has established that the plan is a log-mel fbank without energy column or magnitude spectrum, that
// no output affine is set and that the output is packed; those options then cost no instructions or registers.
template <int DT, int LCT, int WARPS, int SLOTS, int TWS, int MINB, bool PLAIN>
__global__ void __launch_bounds__(WARPS * 32, MINB)
b200feat_fast512_kernel(const DevPlan p, const Fast512Tables ft, const DevBatch b) {
  const bool use_energy = !PLAIN && p.use_energy;
  const bool use_mag = !PLAIN && p.use_mag;
  const bool padded = !PLAIN && b.out_mode == B200FEAT_OUT_PADDED;
  const int feature = PLAIN ? B200FEAT_FBANK : p.feature;
  constexpr int HW = 2 * WARPS;               // half-warps per CTA
  constexpr int TILE = HW * SLOTS;            // frames per tile
  constexpr int PBINS = F512_PBINS(SLOTS);
  constexpr int PBUF = PBINS * SLOTS;         // floats per half-warp P tile, laid out [slot][bin]
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int tid = threadIdx.x;
  const int l = tid & 15;           // lane within the half-warp
  const int hw = tid >> 4;          // half-warp within the CTA
  const int L = LCT ? LCT : p.L;
  constexpr int NP = LCT ? (LCT + 31) / 32 : 16;  // sample-pair registers actually needed

  // ---- shared memory carve-up
  float2 *xall = reinterpret_cast<float2 *>(smem_raw);
  float *pall = reinterpret_cast<float *>(xall + (size_t)HW * F512_XBUF);
  unsigned char *s_const = reinterpret_cast<unsigned char *>(pall + (size_t)HW * PBUF + F512_PTAIL);
  const float2 *s_win = reinterpret_cast<const float2 *>(s_const);
  const float2 *s_tw1 = reinterpret_cast<const float2 *>(s_const + ft.off_tw1);   // [k1][lane] (TWS only)
  const int4 *s_rdesc = reinterpret_cast<const int4 *>(s_const + ft.off_rdesc);   // [round][lane] mel round descriptors
  const float4 *s_mw4 = reinterpret_cast<const float4 *>(s_const + ft.off_mw);    // [row / 4][lane][4] zero-padded weights
  unsigned long long *s_bar = reinterpret_cast<unsigned long long *>(s_const + ft.cblob_bytes);
  float2 *X = xall + (size_t)hw * F512_XBUF;
  float *P = pall + (size_t)hw * PBUF;                        // [slot][PBINS]

  // ---- constant tables: one TMA bulk copy global -> shared, completion signalled on an mbarrier
  const unsigned bar = smem_u32(s_bar);
  blob_copy_start(bar, s_const, ft.cblob, ft.cblob_bytes);
  // P is read past a filter's support with zero weights: it must never hold NaN patterns
  for (int i = tid; i < HW * PBUF + F512_PTAIL; i += blockDim.x) pall[i] = 0.f;

  // per-lane constants kept in registers for the whole kernel
  float2 tw1[TWS ? 1 : 16];
  if (!TWS) {
#pragma unroll
    for (int k1 = 1; k1 < 16; ++k1) tw1[TWS ? 0 : k1] = __ldg(ft.tw1 + k1 * 16 + l);
  }
  float2 wsplit[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) wsplit[i] = __ldg(ft.w512 + i * 16 + l);
  const int partner = (16 - l) & 15;
  const float inv_L = 1.0f / (float)L;
  mbar_wait(bar, 0);  // every thread observes the completion of the bulk copy before touching the tables
  __syncthreads();

  for (int64_t tg = blockIdx.x; tg < b.num_tiles; tg += gridDim.x) {
    const int64_t tile = b.tile_base + tg;
    const int cut = __ldg(b.tile_cut + tile) - b.batch_first;  // host-built tile->cut table: one load, no search
    // (fetching the next tile's cut one tile ahead and prefetching its four table rows into L1 before the mel stage did not pay:
    // the two-load chain of this prologue is already hidden by the other warps)
    const int64_t t0 = (tile - __ldg(b.tile_off + cut)) * TILE + (int64_t)hw * SLOTS;
    const int64_t T = __ldg(b.row_off + cut + 1) - __ldg(b.row_off + cut);
    const int64_t rows_here = padded ? b.max_frames : T;
    if (!__any_sync(F512_FULL, t0 < rows_here)) continue;  // both halves idle for this tile
    const int64_t n = __ldg(b.nsamp + cut);
    const int64_t xoff = __ldg(b.samp_off + cut);
    const int64_t row0 = padded
                             ? (int64_t)(b.batch_first + cut) * b.max_frames + t0
                             : __ldg(b.row_off + cut) + t0;
    // Everything per frame below is 32-bit arithmetic relative to the half-warp's first frame `tb`:
    //   frame t = tb + fl, fl = min(f, tmax)  (an out-of-range half redoes the cut's last frame and does not store it)
    //   first sample of the frame = base0 + rel, rel = fl * S
    const int64_t tb = min(t0, T - 1);
    const int tmax = (int)min(T - 1 - tb, (int64_t)(SLOTS - 1));
    const int nv = (int)max((int64_t)0, min((int64_t)SLOTS, T - t0));  // frames of this half that exist
    const int64_t base0 = tb * p.S - (p.snip_edges ? 0 : p.pad_left);
    constexpr int64_t kClamp = 1 << 30;
    const int rel_lo = (int)max(-kClamp, min(kClamp, -base0));           // frame starts inside the cut:  rel >= rel_lo
    const int rel_hi = (int)max(-kClamp, min(kClamp, n - L - base0));    // frame ends inside the cut:    rel <= rel_hi
    const int rel_end = (int)max(-kClamp, min(kClamp, n - 1 - base0));   // last sample of the cut, relative
    const int par0 = (int)((xoff + base0) & 1);                          // 8-byte alignment of the 64-bit loads
    const char *cut0 = reinterpret_cast<const char *>(b.samples) + (xoff + base0) * (DT == B200FEAT_I16 ? 2 : 4);
    float le[SLOTS];
#pragma unroll
    for (int k = 0; k < SLOTS; ++k) le[k] = 0.f;

#pragma unroll 1
    for (int f = 0; f < SLOTS; ++f) {
      if (!__any_sync(F512_FULL, f < nv)) continue;        // neither half has a frame in this slot
      const int rel = min(f, tmax) * p.S;
      const int64_t base = base0 + rel;                    // only the (rare) edge path uses the 64-bit form
      float2 v[16];
      float prev[NP];
      const bool interior = rel >= rel_lo && rel <= rel_hi && (((par0 + rel) & 1) == 0);
      if (F512_PREFETCH == 2) {  // one L1 prefetch per 32-byte sector of the next frame's new samples
        constexpr int PER = DT == B200FEAT_I16 ? 16 : 8;  // samples per sector
#pragma unroll
        for (int r = 0; r < (DT == B200FEAT_I16 ? 1 : 2); ++r) {
          const int q = rel + L + PER * (l + 16 * r);
          if (q >= rel_lo && q <= rel_end && PER * (l + 16 * r) < p.S + PER)
            asm volatile("prefetch.global.L1 [%0];" ::"l"(cut0 + (int64_t)q * (DT == B200FEAT_I16 ? 2 : 4)));
        }
      }
      if (__all_sync(F512_FULL, interior)) {
        if (DT == B200FEAT_I16) {
          const int16_t *xp = reinterpret_cast<const int16_t *>(cut0) + (rel + 2 * l);
#pragma unroll
          for (int n1 = 0; n1 < NP; ++n1) {
            const int j0 = 32 * n1 + 2 * l;
            v[n1] = make_float2(0.f, 0.f);
            prev[n1] = 0.f;
            if (j0 + 1 < L) {
              const short2 q = __ldg(reinterpret_cast<const short2 *>(xp + 32 * n1));
              v[n1] = make_float2((float)q.x * (1.0f / 32768.0f), (float)q.y * (1.0f / 32768.0f));
            } else if (j0 < L) {
              v[n1].x = (float)__ldg(xp + 32 * n1) * (1.0f / 32768.0f);
            }
            if (!F512_PREV_SHFL && j0 < L) prev[n1] = (float)__ldg(xp + 32 * n1 - (j0 > 0 ? 1 : 0)) * (1.0f / 32768.0f);
          }
        } else {
          const float *xp = reinterpret_cast<const float *>(cut0) + (rel + 2 * l);
#pragma unroll
          for (int n1 = 0; n1 < NP; ++n1) {
            const int j0 = 32 * n1 + 2 * l;
            v[n1] = make_float2(0.f, 0.f);
            prev[n1] = 0.f;
            if (j0 + 1 < L) v[n1] = __ldg(reinterpret_cast<const float2 *>(xp + 32 * n1));
            else if (j0 < L) v[n1].x = __ldg(xp + 32 * n1);  // odd L: last tap alone
            if (!F512_PREV_SHFL && j0 < L) prev[n1] = __ldg(xp + 32 * n1 - (j0 > 0 ? 1 : 0));
          }
        }
      } else {  // a cut edge in this warp: per-tap reflection (layers.py:753-772); ~3 frames per cut
#pragma unroll
        for (int n1 = 0; n1 < NP; ++n1) {
          const int j0 = 32 * n1 + 2 * l;
          float a = 0.f, c = 0.f, pr = 0.f;
          if (j0 < L) {
            int64_t i = base + j0;
            if (!p.snip_edges) i = reflect_index(i, n, p.pad_mode);
            a = ld_sample<DT>(b.samples, xoff + i);
            if (!F512_PREV_SHFL) {
              int64_t ip = base + (j0 > 0 ? j0 - 1 : 0);
              if (!p.snip_edges) ip = reflect_index(ip, n, p.pad_mode);
              pr = ld_sample<DT>(b.samples, xoff + ip);
            }
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
      if (F512_PREV_SHFL) {  // the tap before (32 n1 + 2l) is the neighbour lane's odd tap: one shuffle instead of a load
        float carry = v[0].x;  // lane 0, row 0: replicate-left (layers.py:166)
#pragma unroll
        for (int n1 = 0; n1 < NP; ++n1) {
          const float up = __shfl_sync(F512_FULL, v[n1].y, (l + 15) & 15, 16);  // lane 0 receives lane 15's
          prev[n1] = l == 0 ? carry : up;
          carry = up;  // lane 15's odd tap of this row precedes lane 0's first tap of the next row
        }
      }
      // ---- DC removal (layers.py:155-157)
      float s = 0.f;
#pragma unroll
      for (int n1 = 0; n1 < NP; ++n1) s += v[n1].x + v[n1].y;  // taps beyond L are exact zeros
      const float mu = p.remove_dc ? hw_sum(s) * inv_L : 0.f;
      const float cmu = __fmul_rn(mu, 1.0f - p.preemph);  // the DC offset after pre-emphasis
      // ---- energy, pre-emphasis, window (layers.py:159-170); zero padding is implicit
      float e = 0.f;
#pragma unroll
      for (int n1 = 0; n1 < 16; ++n1) {
        if (n1 < NP) {
          const int j0 = 32 * n1 + 2 * l;
          const float2 w = s_win[n1 * 16 + l];  // zero beyond L
          const float2 y = preemph_window_dc(v[n1], prev[n1], p.preemph, cmu, w);
          if (use_energy) {
            if (p.raw_energy) {
              float2 d = f2add(v[n1], make_float2(-mu, -mu));
              if (j0 >= L) d.x = 0.f;
              if (j0 + 1 >= L) d.y = 0.f;
              e = fmaf(d.x, d.x, fmaf(d.y, d.y, e));
            } else {
              e = fmaf(y.x, y.x, fmaf(y.y, y.y, e));
            }
          }
          v[n1] = y;
        } else {
          v[n1] = make_float2(0.f, 0.f);
        }
      }
      if (use_energy) {  // le[] stays in registers: no dynamic indexing
        const float lev = log_energy_value(p, hw_sum(e));
#pragma unroll
        for (int k = 0; k < SLOTS; ++k) le[k] = (f == k) ? lev : le[k];
      }

      // ---- stage 1: radix-16 over n1, twiddle, transpose
      dft16<NP>(v);
#pragma unroll
      for (int k1 = 0; k1 < 16; ++k1) {
        float2 y = v[F512_OUT(k1)];
        if (k1 > 0) y = f2mul(y, TWS ? s_tw1[k1 * 16 + l] : tw1[TWS ? 0 : k1]);
        X[k1 * F512_XROW + l] = y;
      }
      __syncwarp();
      {
        const float4 *row = reinterpret_cast<const float4 *>(X + l * F512_XROW);
#pragma unroll
        for (int q = 0; q < 8; ++q) {
          const float4 r = row[q];
          v[2 * q] = make_float2(r.x, r.y);
          v[2 * q + 1] = make_float2(r.z, r.w);
        }
      }
      __syncwarp();
      // ---- stage 2: radix-16 over n2 -> Z[l + 16*k2]
      dft16(v);
      // ---- real-FFT split + power (layers.py:38-42).  With E = Z[k] + conj(Z[256-k]), O = Z[k] - conj(Z[256-k]),
      // T = W512^k * O:   2*X[k] = E - i*T   and   2*conj(X[256-k]) = E + i*T, so one (E, O, T) serves two bins.
      // Lane l takes the pairs k = l + 16*i, i = 0..7: Z[k] is its own slot i, and Z[256-k] is slot 15-i of lane 16-l
      // (lanes 1..15) or lane 0's slot 16-i (mod 16).  The mirrored slots go through the transpose tile, which is idle
      // here: every lane stores slots 8..15 and then slot 0 at positions 8..16 of its row, lane 0 one position lower,
      // so that every lane finds its eight mirrors at positions 15..8 of its partner's row.  Bin 128 is left over.
      // The 1/4 of |X|^2 = |2X|^2/4 is folded into the mel weights / spectrogram epilogue.
      {
        float2 *xs = X + l * F512_XROW - (l == 0 ? 1 : 0);
#pragma unroll
        for (int s2 = 8; s2 < 16; ++s2) xs[s2] = v[F512_OUT(s2)];
        xs[16] = v[F512_OUT(0)];
      }
      __syncwarp();
      float *Pf = P + f * PBINS;
      const float4 *mirror = reinterpret_cast<const float4 *>(X + partner * F512_XROW);
#pragma unroll
      for (int i = 0; i < 8; i += 2) {
        const float4 m2 = mirror[7 - i / 2];  // positions 15 - i - 1 and 15 - i
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const float2 zk = v[F512_OUT(i + h)];
          const float2 cc = h == 0 ? make_float2(m2.z, -m2.w) : make_float2(m2.x, -m2.y);
          const float2 E = f2add(zk, cc), O = f2sub(zk, cc);
          const float2 mit = f2mi(f2mul(O, wsplit[i + h]));  // -i*T
          const float2 a = f2add(E, mit);                     // 2*X[k]
          const float2 bq = f2sub(E, mit);                    // 2*conj(X[256-k])
          float pa = fmaf(a.x, a.x, a.y * a.y), pb = fmaf(bq.x, bq.x, bq.y * bq.y);
          if (use_mag) { pa = sqrtf(pa); pb = sqrtf(pb); }
          Pf[l + 16 * (i + h)] = pa;
          Pf[256 - l - 16 * (i + h)] = pb;
        }
      }
      {  // bin 128 = lane 0's slot 8: X[128] = conj(Z[128]), so |2X[128]|^2 = |2 Z[128]|^2
        const float2 z = v[F512_OUT(8)];
        const float zx = 2.f * z.x, zy = 2.f * z.y;
        float pm = fmaf(zx, zx, zy * zy);
        if (use_mag) pm = sqrtf(pm);
        if (l == 0) Pf[128] = pm;
      }
      __syncwarp();  // the next frame's stage 1 overwrites the tile
    }
    __syncwarp();

    // ---- epilogue over the (up to) 4 frames of this half-warp
    const int nvalid = nv;
    const int nrows = (int)max((int64_t)0, min((int64_t)SLOTS, rows_here - t0));
    float *out = b.out + row0 * p.F;  // the rows below are 32-bit offsets from this per-tile base
    auto aff = [&](int col, float x) { return PLAIN ? x : post_affine(p, col, x); };
    if (feature == B200FEAT_SPECTROGRAM || feature == B200FEAT_LOG_SPECTROGRAM) {
      for (int f = 0; f < nrows; ++f) {
        float *o = out + f * p.F;
        if (f >= nvalid) { for (int k = l; k < p.F; k += 16) o[k] = aff(k, b.pad_value); continue; }
        for (int k = l; k < p.K; k += 16) {
          float x = P[f * PBINS + k] * (use_mag ? 0.5f : 0.25f);  // P holds |2X|^2 (or |2X|)
          if (feature == B200FEAT_LOG_SPECTROGRAM) x = log_spec_value(p, x);
          if (k == 0 && use_energy) {
#pragma unroll
            for (int g = 0; g < SLOTS; ++g) x = (f == g) ? le[g] : x;
          }
          o[k] = aff(k, x);
        }
      }
    } else {
      const int shift = PLAIN ? 0 : mel_shift(p), ecol = energy_col(p);
      const float lgk = p.log10_mel ? 0.30102999566398119521f : 0.69314718055994530942f;  // log10 (librosa_fbank.py:126) or ln
      const int Mpad = (p.M + 3) & ~3;
      float *mlog = reinterpret_cast<float *>(X);  // the transpose tile is idle during the epilogue
      for (int j = 0; j < ft.mel_rounds; ++j) {
        const int m = l + 16 * j;
        const int4 rd = s_rdesc[j * 16 + l];  // {first bin (multiple of 4), trip count (uniform), weight index, -}
        const float4 *pp = reinterpret_cast<const float4 *>(P + rd.x);
        const float4 *wp = s_mw4 + rd.z;      // weights [row / 4][lane][4]: one 128-bit load feeds 4 taps x SLOTS frames
        float acc[SLOTS];
#pragma unroll
        for (int f = 0; f < SLOTS; ++f) acc[f] = 0.f;
#pragma unroll 1
        for (int i = rd.y; i > 0; i -= 4, ++pp, wp += 16) {
          const float4 wi = *wp;
#pragma unroll
          for (int f = 0; f < SLOTS; ++f) {
            const float4 pv = pp[f * (PBINS / 4)];
            acc[f] = fmaf(pv.w, wi.w, fmaf(pv.z, wi.z, fmaf(pv.y, wi.y, fmaf(pv.x, wi.x, acc[f]))));
          }
        }
        if (m < p.M) {
          float r[SLOTS];
#pragma unroll
          for (int f = 0; f < SLOTS; ++f) r[f] = fast_lg2_normal(nanmax(acc[f], p.mel_floor)) * lgk;
          if (feature != B200FEAT_MFCC) {
            float *orow = out + m + shift;
            if (nvalid == SLOTS) {  // the common case: no per-row guards
#pragma unroll
              for (int f = 0; f < SLOTS; ++f) orow[f * p.F] = aff(m + shift, r[f]);
            } else {
#pragma unroll
              for (int f = 0; f < SLOTS; ++f)
                if (f < nvalid) orow[f * p.F] = aff(m + shift, r[f]);
            }
          } else {
#pragma unroll
            for (int f = 0; f < SLOTS; ++f) mlog[f * Mpad + m] = r[f];
          }
        }
      }
      if (feature == B200FEAT_FBANK) {
        if (use_energy && l < nvalid) { float v0 = 0.f;
#pragma unroll
          for (int f = 0; f < SLOTS; ++f) v0 = (l == f) ? le[f] : v0;
          out[l * p.F + ecol] = aff(ecol, v0); }
      } else if (feature == B200FEAT_MFCC) {
        __syncwarp();
        for (int idx = l; idx < nvalid * p.C; idx += 16) {
          const int f = idx / p.C, c = idx - f * p.C;
          float acc = 0.f;
          for (int m = 0; m < p.M; ++m) acc = fmaf(mlog[f * Mpad + m], __ldg(p.dct + m * p.C + c), acc);
          if (p.use_lifter) acc *= __ldg(p.lifter + c);
          if (use_energy && c == ecol) {
#pragma unroll
            for (int g = 0; g < SLOTS; ++g) acc = (f == g) ? le[g] : acc; }
          out[f * p.F + c] = aff(c, acc);
        }
      }
      // padded tail rows (packed output has none: nrows == nvalid)
      if (padded)
        for (int f = nvalid; f < nrows; ++f)
          for (int k = l; k < p.F; k += 16) out[f * p.F + k] = aff(k, b.pad_value);
    }
    __syncwarp();
  }
}

// ---------------------------------------------------------------------------------------------- host
// Launch shapes on the headline workload (kernel ms per launch of 2048 x 10 s cuts, scripts/variant_bench.py, H100 SXM with a
// 400 W power limit, profiles/h100_launch_shapes.jsonl):
//   {8 warps, 4 slots, twiddles in registers, 2 CTAs/SM}  1.796 / 1.767   <- shape 0, what ships
//   {10, 2, shared, 2}  (20 warps/SM, 96 registers)       1.859           <- shape 2
// B200FEAT_FAST_VARIANT=2 selects the high-occupancy shape for A/B runs; 0 and 1 select shape 0.
struct Fast512Variant { int warps, slots, tws, minb; };
static inline Fast512Variant f512_variant(int v) { return v == 2 ? Fast512Variant{10, 2, 1, 2} : Fast512Variant{8, 4, 0, 2}; }
#ifndef F512_DEFAULT_VARIANT
#define F512_DEFAULT_VARIANT 0
#endif

struct Fast512Host {
  Fast512Tables t;
  size_t smem;
  int variant;  // 0 or 2
};

static inline bool fast512_supported(const DevPlan &p) {
  return p.N == 512 && p.packed && p.L >= 2 && p.L <= 512 && p.C <= 128 &&
         4 * ((p.M + 3) & ~3) <= 2 * F512_XBUF;  // log-mel staging reuses the transpose tile
}

// one instantiation per (dtype, compile-time L, variant, plain log-mel or not); `launch` == false only raises the
// shared-memory limit
template <int DT, int LCT, int V, bool PLAIN>
static int f512_go(bool launch, size_t smem, const DevPlan &p, const Fast512Tables &t, const DevBatch &b, dim3 grid,
                   cudaStream_t stream) {
  constexpr int W = V == 2 ? 10 : 8;
  constexpr int S = V == 2 ? 2 : 4;
  constexpr int TW = V == 2 ? 1 : 0;
  constexpr int MB = 2;
  return configure_or_launch(b200feat_fast512_kernel<DT, LCT, W, S, TW, MB, PLAIN>, W * 32, launch, smem, p, t, b, grid, stream);
}

template <int DT, int LCT, bool PLAIN>
static int f512_dispatch_variant(int v, bool launch, size_t smem, const DevPlan &p, const Fast512Tables &t, const DevBatch &b,
                                 dim3 grid, cudaStream_t stream) {
  if (v == 2) return f512_go<DT, LCT, 2, PLAIN>(launch, smem, p, t, b, grid, stream);
  return f512_go<DT, LCT, 0, PLAIN>(launch, smem, p, t, b, grid, stream);
}

template <bool PLAIN>
static int f512_dispatch(int v, int dt, int L, bool launch, size_t smem, const DevPlan &p, const Fast512Tables &t,
                         const DevBatch &b, dim3 grid, cudaStream_t stream) {
  if (L == 400) {
    if (dt == B200FEAT_I16) return f512_dispatch_variant<B200FEAT_I16, 400, PLAIN>(v, launch, smem, p, t, b, grid, stream);
    return f512_dispatch_variant<B200FEAT_F32, 400, PLAIN>(v, launch, smem, p, t, b, grid, stream);
  }
  if (dt == B200FEAT_I16) return f512_dispatch_variant<B200FEAT_I16, 0, PLAIN>(v, launch, smem, p, t, b, grid, stream);
  return f512_dispatch_variant<B200FEAT_F32, 0, PLAIN>(v, launch, smem, p, t, b, grid, stream);
}

// The plain log-mel instantiation serves a launch when the plan has no energy column and no magnitude spectrum, no output
// affine is set (b200feat_set_output_affine) and the output is packed; everything else takes the general one.
static inline bool fast512_plain(const DevPlan &p, const DevBatch &b) {
  return p.feature == B200FEAT_FBANK && !p.use_energy && !p.use_mag && p.post_scale == nullptr &&
         b.out_mode == B200FEAT_OUT_PACKED;
}

static inline int fast512_prepare(DevPlan &p, const std::vector<float> &bank, std::vector<void *> &allocs,
                                  int *frames_per_tile, const std::vector<float> &window, Fast512Host *out) {
  Fast512Host hst;
  const int forced = launch_shape_override("B200FEAT_FAST_VARIANT", 3);
  hst.variant = (forced >= 0 ? forced : F512_DEFAULT_VARIANT) == 2 ? 2 : 0;
  const Fast512Variant var = f512_variant(hst.variant);
  std::vector<float2> win2(256), tw1(256), w512(128);
  for (int n1 = 0; n1 < 16; ++n1)
    for (int l = 0; l < 16; ++l) {
      const int j0 = 32 * n1 + 2 * l;
      win2[n1 * 16 + l] = make_float2(j0 < p.L ? window[j0] : 0.f, j0 + 1 < p.L ? window[j0 + 1] : 0.f);
    }
  for (int k1 = 0; k1 < 16; ++k1)
    for (int l = 0; l < 16; ++l) {
      const double a = -2.0 * M_PI * (double)((l * k1) % 256) / 256.0;
      tw1[k1 * 16 + l] = make_float2((float)cos(a), (float)sin(a));
    }
  for (int i = 0; i < 8; ++i)
    for (int l = 0; l < 16; ++l) {
      const double a = -2.0 * M_PI * (double)(l + 16 * i) / 512.0;
      w512[i * 16 + l] = make_float2((float)cos(a), (float)sin(a));
    }
  if (upload_table(tw1, allocs, &hst.t.tw1) || upload_table(w512, allocs, &hst.t.w512)) return B200FEAT_ECUDA;
  // mel bank re-packed for the epilogue (pack_mel_rounds, common.cuh); the kernel stores |2X|^2 (or |2X|), so the
  // exact power-of-two factor 1/4 (1/2) rides on the weights
  const MelRounds mr = pack_mel_rounds(bank, p.K, p.M, p.use_mag ? 0.5f : 0.25f, 16, 4, 260);  // 4-aligned filter starts: 128-bit mel loads
  if (mr.max_reach > 260) return B200FEAT_EUNSUPPORTED;  // zero-weight over-reads must stay inside the frame's own P row
  hst.t.mel_rounds = mr.rounds;
  hst.t.mel_wrows = mr.rounds ? (int)(mr.wdense.size() / 16) : 0;
  ConstBlob blob;
  blob.append(win2);
  hst.t.off_tw1 = var.tws ? blob.append(tw1) : 0;
  hst.t.off_rdesc = blob.append(mel_round_descs(mr));
  hst.t.off_mw = blob.append(mr.wdense);
  if (blob.upload(allocs, &hst.t.cblob, &hst.t.cblob_bytes)) return B200FEAT_ECUDA;
  hst.smem = fast512_smem_bytes(p, hst.t, var.warps, var.slots, var.tws);
  if (hst.smem > (size_t)(227 * 1024 / var.minb) - 1024) return B200FEAT_EUNSUPPORTED;  // keep MINB CTAs per SM
  DevBatch none{};
  for (int dt = 0; dt < 2; ++dt)
    for (int L : {400, 0})
      if (f512_dispatch<false>(hst.variant, dt, L, false, hst.smem, p, hst.t, none, dim3(1), nullptr) ||
          f512_dispatch<true>(hst.variant, dt, L, false, hst.smem, p, hst.t, none, dim3(1), nullptr))
        return B200FEAT_ECUDA;
  *out = hst;
  *frames_per_tile = 2 * var.warps * var.slots;
  return 0;
}

static inline int fast512_launch(const DevPlan &p, const Fast512Host &hst, const DevBatch &b, int dt, int sm_count,
                                 cudaStream_t stream) {
  const dim3 grid(persistent_grid(b.num_tiles, sm_count, f512_variant(hst.variant).minb));
  const int L = p.L == 400 ? 400 : 0;
  if (fast512_plain(p, b)) f512_dispatch<true>(hst.variant, dt, L, true, hst.smem, p, hst.t, b, grid, stream);
  else f512_dispatch<false>(hst.variant, dt, L, true, hst.smem, p, hst.t, b, grid, stream);
  return (int)cudaGetLastError();
}
