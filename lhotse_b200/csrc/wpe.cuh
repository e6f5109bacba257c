// Single-channel WPE dereverberation on the GPU: lhotse's DereverbWPE (torch.stft, nara_wpe's wpe_v8, torch.istft, then the
// cut's length fix), within a float32 tolerance of a float64 restatement (DESIGN.md §3.1q).  The float route runs wpe_v8 in
// complex64 through LAPACK, whose bits depend on the CPU's BLAS, so there is no bit pattern to match.
//
// Per cut, with x[0, L) the float32 signal (L > 256) and w the 512-point periodic Blackman window as torch computes it:
//   STFT    Y_t[k] = sum_m w[m] x~[128 t + m] e^{-2 pi i k m / 512}, k < 257, t < T = 1 + L / 128, x~ the signal reflect-padded
//           by 256 on each side (torch.stft's center=True)
//   WPE     per bin, on its own: X = Y; `iterations` times: power_t = |X_t|^2, eps = 1e-10 max_t power_t (over every frame of
//           the bin), inv_t = 1 when eps = 0 else 1 / max(power_t, eps); R = sum_{t in S} inv_t y~_t y~_t^H and
//           P = sum_{t in S} inv_t y~_t conj(Y_t), y~_t[k] = Y_{t - delay - k} (0 before the first frame), S every frame
//           ("full") or t >= delay + taps - 1 ("valid"); G = R^-1 P (0 when R is exactly singular, as lstsq gives for R = 0);
//           X_t = Y_t - G^H y~_t
//   iSTFT   z[j] = sum_t w[p - 128 t] x_t[p - 128 t] / sum_t w[p - 128 t]^2, p = j + 256, over the frames that cover p, x_t the
//           inverse real transform of X_t (imaginary parts of bins 0 and 256 ignored, as a C2R transform does); j < 128 (T - 1)
//   output  out[q] = z[mix_source_pos(q, 128 (T - 1))] over the cut's target length (trim or np.pad(mode="reflect"))
//
// Three kernels, no floating-point atomics, so results are identical from run to run and a cut's output does not depend on
// its batch:
//   wpe_stft_kernel   one CTA per tile of WPE_TILE frames: two real frames per 512-point complex radix-2 FFT (one warp per
//                     pair), the tile staged in shared memory and written bin-major ([bin][frame]) in rows of WPE_TILE frames
//   wpe_bin_kernel    one CTA per (cut, bin): the bin's row and inv_t in shared memory; R and P accumulated in float64 by
//                     fixed (entry, frame-slice) assignments and summed in slice order; G by one warp (LU with partial
//                     pivoting, one lane per column of [R | P]); X written over Y as float32
//   wpe_istft_kernel  one CTA per WPE_OUT_HOPS output hops: the WPE_OUT_HOPS + 3 frames that cover them (inverse FFTs, two
//                     frames per transform), the overlap-add per sample, the length fix
// A bin's row and inv_t take 16 bytes per frame of shared memory: WPE_MAX_FRAMES caps the frames at 128 KB.
//
// The per-bin and per-sample arithmetic is __host__ __device__ so that scripts/micro/wpe_host_check.cu runs exactly this code
// on the CPU (with a direct DFT in place of the FFTs).  Kernels at the end.
#pragma once
#include <math.h>
#include <stdint.h>

#include "mix.cuh"

#define WPE_NFFT 512
#define WPE_LOG_NFFT 9
#define WPE_HOP 128
#define WPE_BINS (WPE_NFFT / 2 + 1)
#define WPE_MAX_TAPS 16
#define WPE_MAX_FRAMES 8192  // T cap: 128 KB of shared memory per bin; 65.5 s at 16 kHz (L <= 1048575)
#define WPE_THREADS 256
#define WPE_WARPS (WPE_THREADS / 32)
#define WPE_TILE 32                         // STFT frames per CTA: a row of 256 bytes per bin
#define WPE_OUT_HOPS (WPE_TILE - 3)         // iSTFT output hops per CTA; they are covered by WPE_TILE frames
#define WPE_LD (WPE_MAX_TAPS + 1)           // row stride of the augmented matrix [R | P]

#if defined(__CUDA_ARCH__)
#define WPE_FMA(a, b, c) __fmaf_rn(a, b, c)
#else
#define WPE_FMA(a, b, c) fmaf(a, b, c)
#endif

struct wpe_c { float x, y; };
struct wpe_z { double x, y; };

// One cut as the kernels read it (b200feat_wpe builds these from the b200feat_wpe_cut records)
struct WpeCut {
  const float *x;       // the input, L samples
  float *out;           // the cut's first output sample
  wpe_c *Y;             // its spectra in the work buffer, [bin][frame], WPE_BINS * T
  int64_t n;            // L
  int64_t target_len;   // samples written: 128 (T - 1), fewer (trim) or at most 128 (T - 1) - 1 more (reflect-pad)
  int64_t tile_begin;   // its first CTA in the STFT kernel's grid
  int64_t out_begin;    // its first CTA in the iSTFT kernel's grid
  int32_t T;            // frames, 1 + L / 128
  int32_t reserved;
};

struct WpeParams {
  int32_t taps, delay, iterations, valid;  // valid: statistics_mode "valid"
};

MIX_HD int64_t wpe_frames(int64_t n) { return 1 + n / WPE_HOP; }
MIX_HD int64_t wpe_istft_len(int64_t n) { return WPE_HOP * (n / WPE_HOP); }  // 128 (T - 1)
MIX_HD int64_t wpe_stft_ctas(int64_t T) { return (T + WPE_TILE - 1) / WPE_TILE; }
MIX_HD int64_t wpe_istft_ctas(int64_t T) { return (T - 1 + WPE_OUT_HOPS - 1) / WPE_OUT_HOPS; }
MIX_HD int wpe_entries(int taps) { return taps * (taps + 1) / 2 + taps; }  // R's upper triangle, then P

MIX_HD int wpe_bitrev(int i) {
#if defined(__CUDA_ARCH__)
  return (int)(__brev((unsigned)i) >> (32 - WPE_LOG_NFFT));
#else
  int r = 0;
  for (int b = 0; b < WPE_LOG_NFFT; ++b) r |= ((i >> b) & 1) << (WPE_LOG_NFFT - 1 - b);
  return r;
#endif
}

// exp(-2 pi i k / 512), k < 256, evaluated in double on the host and rounded once (b200feat_wpe uploads this table)
inline wpe_c wpe_twiddle(int k) {
  return wpe_c{(float)cos(-2.0 * M_PI * k / WPE_NFFT), (float)sin(-2.0 * M_PI * k / WPE_NFFT)};
}

// Sample m of frame t of the centred, reflect-padded signal (torch.stft's center=True, pad_mode="reflect"; needs L > 256)
MIX_HD float wpe_frame_sample(const float *x, int64_t n, int64_t t, int m) {
  int64_t i = t * WPE_HOP + m - WPE_NFFT / 2;
  if (i < 0) i = -i;
  if (i >= n) i = 2 * (n - 1) - i;
  return x[i];
}

// Butterfly j (< 256) of the radix-2 decimation-in-time stage whose sub-transforms have `half` points, in place on a
// bit-reversed array; the inverse transform uses the conjugate twiddles (unscaled)
MIX_HD void wpe_butterfly(wpe_c *a, const wpe_c *tw, int half, int j, bool inverse) {
  const int pos = j & (half - 1);
  const int i0 = ((j - pos) << 1) + pos, i1 = i0 + half;
  const wpe_c w = tw[pos * (WPE_NFFT / 2 / half)];
  const float wy = inverse ? -w.y : w.y;
  const wpe_c b = a[i1];
  const wpe_c t{WPE_FMA(w.x, b.x, -(wy * b.y)), WPE_FMA(w.x, b.y, wy * b.x)};
  const wpe_c u = a[i0];
  a[i0] = wpe_c{u.x + t.x, u.y + t.y};
  a[i1] = wpe_c{u.x - t.x, u.y - t.y};
}

// Bin k (<= 256) of two real frames transformed together, frame a in the real part and frame b in the imaginary part:
// A = (Z[k] + conj(Z[-k])) / 2, B = (Z[k] - conj(Z[-k])) / 2i
MIX_HD void wpe_split(const wpe_c *Z, int k, wpe_c *A, wpe_c *B) {
  const wpe_c p = Z[k], q = Z[(WPE_NFFT - k) & (WPE_NFFT - 1)];
  *A = wpe_c{0.5f * (p.x + q.x), 0.5f * (p.y - q.y)};
  *B = wpe_c{0.5f * (p.y + q.y), 0.5f * (q.x - p.x)};
}

// Point m (< 512) of the spectrum whose inverse transform has frame a in its real part and frame b in its imaginary part,
// from their bins kk = min(m, 512 - m): the Hermitian extension, bins 0 and 256 real (a C2R transform ignores their
// imaginary parts)
MIX_HD wpe_c wpe_pack(wpe_c A, wpe_c B, int m) {
  const int kk = m <= WPE_NFFT / 2 ? m : WPE_NFFT - m;
  if (kk == 0 || kk == WPE_NFFT / 2) A.y = B.y = 0.0f;
  if (m > WPE_NFFT / 2) { A.y = -A.y; B.y = -B.y; }
  return wpe_c{A.x - B.y, A.y + B.x};
}

// Entry e (< wpe_entries(taps)) of the normal equations as the lags of its two factors, sum_t inv_t Y[t - la] conj(Y[t - lb]):
// R[i][j] (i <= j, row by row) has la = delay + i, lb = delay + j; P[i] (e past the triangle) has la = delay + i, lb = 0
MIX_HD void wpe_entry_lags(int e, int taps, int delay, int *la, int *lb) {
  const int nr = taps * (taps + 1) / 2;
  if (e >= nr) { *la = delay + (e - nr); *lb = 0; return; }
  int i = 0;
  while (e >= taps - i) { e -= taps - i; ++i; }
  *la = delay + i;
  *lb = delay + i + e;
}

// Slice s of S of an entry: the frames t = s (mod S) with t >= max(la, lb, t_min) (a factor before the first frame is 0), in
// increasing order, in float64
MIX_HD wpe_z wpe_entry_sum(const wpe_c *Y, const double *inv, int T, int la, int lb, int t_min, int s, int S) {
  int t0 = la > lb ? la : lb;
  if (t_min > t0) t0 = t_min;
  t0 += ((s - t0) % S + S) % S;
  double re = 0.0, im = 0.0;
  for (int t = t0; t < T; t += S) {
    const wpe_c a = Y[t - la], b = Y[t - lb];
    const double ar = inv[t] * (double)a.x, ai = inv[t] * (double)a.y;  // a conj(b) inv_t
    re = fma(ar, (double)b.x, fma(ai, (double)b.y, re));
    im = fma(ai, (double)b.x, fma(-ar, (double)b.y, im));
  }
  return wpe_z{re, im};
}

// X_t = Y_t - sum_k conj(G_k) Y_{t - delay - k}, in float64, k in increasing order
MIX_HD wpe_z wpe_filter(const wpe_c *Y, int t, const wpe_z *G, int taps, int delay) {
  double re = Y[t].x, im = Y[t].y;
  for (int k = 0; k < taps; ++k) {
    const int u = t - delay - k;
    if (u < 0) break;
    const double yx = Y[u].x, yy = Y[u].y;
    re -= fma(G[k].x, yx, G[k].y * yy);
    im -= fma(G[k].x, yy, -(G[k].y * yx));
  }
  return wpe_z{re, im};
}

MIX_HD double wpe_power(wpe_z x) { return fma(x.x, x.x, x.y * x.y); }

// nara_wpe's get_power_inverse for one frame, eps = 1e-10 times the bin's largest power
MIX_HD double wpe_inv(double power, double eps) { return eps == 0.0 ? 1.0 : 1.0 / (power > eps ? power : eps); }

MIX_HD double wpe_cabs1(wpe_z a) { return fabs(a.x) + fabs(a.y); }

MIX_HD wpe_z wpe_cdiv(wpe_z a, wpe_z b) {
  const double d = fma(b.x, b.x, b.y * b.y);
  return wpe_z{fma(a.x, b.x, a.y * b.y) / d, fma(a.y, b.x, -(a.x * b.y)) / d};
}

// The augmented n x (n + 1) matrix [R | P] of one bin, row stride WPE_LD: entry e's sum placed at R[i][j] and (conjugated)
// R[j][i], or at P[i]
MIX_HD void wpe_place(wpe_z *A, int taps, int delay, int e, wpe_z v) {
  int la, lb;
  wpe_entry_lags(e, taps, delay, &la, &lb);
  const int i = la - delay;
  if (e >= taps * (taps + 1) / 2) { A[i * WPE_LD + taps] = v; return; }
  const int j = lb - delay;
  A[i * WPE_LD + j] = v;
  if (j != i) A[j * WPE_LD + i] = wpe_z{v.x, -v.y};
}

// The pivot row of elimination step k: the first row i >= k with the largest |re| + |im| in column k (LAPACK's izamax); -1
// when they are all 0 (R is singular: the bin's G is 0)
MIX_HD int wpe_pivot(const wpe_z *A, int n, int k) {
  int p = -1;
  double best = 0.0;
  for (int i = k; i < n; ++i) {
    const double v = wpe_cabs1(A[i * WPE_LD + k]);
    if (v > best) { best = v; p = i; }
  }
  return p;
}

// Column c (k < c <= n) of elimination step k, the pivot row already swapped into row k: A[i][c] -= A[i][k] / A[k][k] * A[k][c]
// for i > k.  Column k is only read, so the columns of one step are independent (one lane each on the device).
MIX_HD void wpe_eliminate(wpe_z *A, int n, int k, int c) {
  const wpe_z d = A[k * WPE_LD + k], u = A[k * WPE_LD + c];
  for (int i = k + 1; i < n; ++i) {
    const wpe_z l = wpe_cdiv(A[i * WPE_LD + k], d);
    wpe_z &a = A[i * WPE_LD + c];
    a = wpe_z{a.x - fma(l.x, u.x, -(l.y * u.y)), a.y - fma(l.x, u.y, l.y * u.x)};
  }
}

// G from the triangular system left by the elimination (0 when it stopped at a zero pivot)
MIX_HD void wpe_back_substitute(const wpe_z *A, int n, bool regular, wpe_z *G) {
  for (int i = n - 1; i >= 0; --i) {
    if (!regular) { G[i] = wpe_z{0.0, 0.0}; continue; }
    wpe_z s = A[i * WPE_LD + n];
    for (int j = i + 1; j < n; ++j) {
      const wpe_z a = A[i * WPE_LD + j];
      s = wpe_z{s.x - fma(a.x, G[j].x, -(a.y * G[j].y)), s.y - fma(a.x, G[j].y, a.y * G[j].x)};
    }
    G[i] = wpe_cdiv(s, A[i * WPE_LD + i]);
  }
}

// Output sample j (< 128 (T - 1), after the n_fft / 2 trim) of the overlap-add: the windowed inverse transforms of the frames
// that cover it, in frame order, over the window-square envelope of the same frames.  frames[(f - f0) * 512 + m] holds
// sample m of frame f times the window.
MIX_HD float wpe_ola(const float *frames, int64_t f0, int64_t T, const float *win, int64_t j) {
  const int64_t p = j + WPE_NFFT / 2;
  const int64_t lo = p < WPE_NFFT ? 0 : (p - WPE_NFFT) / WPE_HOP + 1;
  const int64_t hi = p / WPE_HOP < T - 1 ? p / WPE_HOP : T - 1;
  float num = 0.0f, den = 0.0f;
  for (int64_t f = lo; f <= hi; ++f) {
    const int m = (int)(p - f * WPE_HOP);
    num = MIX_FADD(num, frames[(f - f0) * WPE_NFFT + m]);
    den = MIX_FADD(den, MIX_FMUL(win[m], win[m]));
  }
  return MIX_FDIV(num, den);
}

// The length fix: out[q] = z[mix_source_pos(q, Lz)] for q < target.  Sample j of z is the source of q = j and, when the cut
// is reflect-padded, of q = 2 (Lz - 1) - j >= Lz: whoever computes z[j] writes both.
MIX_HD void wpe_store(float *out, int64_t target, int64_t Lz, int64_t j, float v) {
  if (j < target) out[j] = v;
  const int64_t q = 2 * (Lz - 1) - j;
  if (q >= Lz && q < target) out[q] = v;
}

#ifdef __CUDACC__
#define WPE_FFT_SMEM (WPE_WARPS * WPE_NFFT * (int)sizeof(wpe_c))                       // one transform per warp
#define WPE_STFT_SMEM (WPE_BINS * (WPE_TILE + 1) * (int)sizeof(wpe_c) + WPE_FFT_SMEM)  // the tile's spectra, then the transforms
#define WPE_ISTFT_SMEM (WPE_TILE * WPE_NFFT * (int)sizeof(float) + WPE_FFT_SMEM)       // the windowed frames, then the transforms
#define WPE_BIN_SMEM(T) ((int)(T) * (int)(sizeof(double) + sizeof(wpe_c)))             // inv_t, then the bin's row

__device__ __forceinline__ int64_t wpe_find_cut(const WpeCut *__restrict__ cuts, int ncuts, bool out_grid) {
  int lo = 0, hi = ncuts - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if ((out_grid ? cuts[mid].out_begin : cuts[mid].tile_begin) <= (int64_t)blockIdx.x) lo = mid; else hi = mid - 1;
  }
  return lo;
}

// the warp's transform of its bit-reversed array, stage by stage
__device__ __forceinline__ void wpe_warp_fft(wpe_c *a, const wpe_c *tw, bool inverse, int lane) {
  for (int half = 1; half < WPE_NFFT; half <<= 1) {
    __syncwarp();
    for (int j = lane; j < WPE_NFFT / 2; j += 32) wpe_butterfly(a, tw, half, j, inverse);
  }
  __syncwarp();
}

// One CTA per tile of WPE_TILE frames of a cut: their spectra, written to the cut's [bin][frame] rows.
__global__ void __launch_bounds__(WPE_THREADS) wpe_stft_kernel(const WpeCut *__restrict__ cuts, int ncuts,
                                                               const float *__restrict__ window, const wpe_c *__restrict__ twiddles) {
  extern __shared__ __align__(16) unsigned char wpe_smem[];
  __shared__ wpe_c tw[WPE_NFFT / 2];
  __shared__ float win[WPE_NFFT];
  wpe_c *stage = (wpe_c *)wpe_smem;                       // [WPE_BINS][WPE_TILE + 1]
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  wpe_c *a = stage + WPE_BINS * (WPE_TILE + 1) + warp * WPE_NFFT;
  const WpeCut c = cuts[wpe_find_cut(cuts, ncuts, false)];
  const int64_t t0 = ((int64_t)blockIdx.x - c.tile_begin) * WPE_TILE;
  const int nf = (int)(c.T - t0 < WPE_TILE ? c.T - t0 : WPE_TILE);
  for (int k = threadIdx.x; k < WPE_NFFT / 2; k += WPE_THREADS) tw[k] = twiddles[k];
  for (int m = threadIdx.x; m < WPE_NFFT; m += WPE_THREADS) win[m] = window[m];
  __syncthreads();
  for (int pr = warp; 2 * pr < nf; pr += WPE_WARPS) {  // frames 2 pr and 2 pr + 1 of the tile
    const int64_t ta = t0 + 2 * pr;
    const bool has_b = 2 * pr + 1 < nf;
    for (int m = lane; m < WPE_NFFT; m += 32)
      a[wpe_bitrev(m)] = wpe_c{MIX_FMUL(wpe_frame_sample(c.x, c.n, ta, m), win[m]),
                               has_b ? MIX_FMUL(wpe_frame_sample(c.x, c.n, ta + 1, m), win[m]) : 0.0f};
    wpe_warp_fft(a, tw, false, lane);
    for (int k = lane; k < WPE_BINS; k += 32) {
      wpe_c A, B;
      wpe_split(a, k, &A, &B);
      stage[k * (WPE_TILE + 1) + 2 * pr] = A;
      stage[k * (WPE_TILE + 1) + 2 * pr + 1] = B;
    }
    __syncwarp();
  }
  __syncthreads();
  for (int i = threadIdx.x; i < WPE_BINS * WPE_TILE; i += WPE_THREADS) {
    const int k = i / WPE_TILE, f = i % WPE_TILE;
    if (f < nf) c.Y[(int64_t)k * c.T + t0 + f] = stage[k * (WPE_TILE + 1) + f];
  }
}

__device__ __forceinline__ double wpe_block_max(double v, double *red) {
  for (int off = 16; off > 0; off >>= 1) v = fmax(v, __shfl_down_sync(0xffffffffu, v, off));
  __syncthreads();  // `red` may still be read from the previous call
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  double m = red[0];
  for (int w = 1; w < WPE_WARPS; ++w) m = fmax(m, red[w]);
  return m;
}

// One CTA per (cut, bin): the bin's `iterations` weighted least-squares filters, then X over Y.
__global__ void __launch_bounds__(WPE_THREADS) wpe_bin_kernel(const WpeCut *__restrict__ cuts, WpeParams prm) {
  extern __shared__ __align__(16) unsigned char wpe_smem[];
  __shared__ wpe_z part[WPE_THREADS];
  __shared__ wpe_z A[WPE_MAX_TAPS * WPE_LD];
  __shared__ wpe_z G[WPE_MAX_TAPS];
  __shared__ double red[WPE_WARPS];
  const WpeCut c = cuts[blockIdx.x / WPE_BINS];
  const int bin = (int)(blockIdx.x % WPE_BINS), T = c.T;
  double *inv = (double *)wpe_smem;
  wpe_c *Y = (wpe_c *)(inv + T);
  wpe_c *row = c.Y + (int64_t)bin * T;
  for (int t = threadIdx.x; t < T; t += WPE_THREADS) Y[t] = row[t];
  const int n = prm.taps, E = wpe_entries(n), S = WPE_THREADS / E;
  const int e = threadIdx.x % E, s = threadIdx.x / E;  // this thread's entry and frame slice (none when s >= S)
  int la = 0, lb = 0;
  wpe_entry_lags(e, n, prm.delay, &la, &lb);
  const int t_min = prm.valid ? prm.delay + n - 1 : 0;
  for (int it = 0; it < prm.iterations; ++it) {
    __syncthreads();  // the row, or the previous iteration's G
    double mx = 0.0;
    for (int t = threadIdx.x; t < T; t += WPE_THREADS) {
      const double p = wpe_power(it == 0 ? wpe_z{Y[t].x, Y[t].y} : wpe_filter(Y, t, G, n, prm.delay));
      inv[t] = p;
      mx = fmax(mx, p);
    }
    const double eps = 1e-10 * wpe_block_max(mx, red);
    for (int t = threadIdx.x; t < T; t += WPE_THREADS) inv[t] = wpe_inv(inv[t], eps);
    __syncthreads();
    if (s < S) part[threadIdx.x] = wpe_entry_sum(Y, inv, T, la, lb, t_min, s, S);
    __syncthreads();
    if (threadIdx.x < E) {
      wpe_z v = part[threadIdx.x];
      for (int k = 1; k < S; ++k) v = wpe_z{v.x + part[threadIdx.x + k * E].x, v.y + part[threadIdx.x + k * E].y};
      wpe_place(A, n, prm.delay, threadIdx.x, v);
    }
    __syncthreads();
    if (threadIdx.x < 32) {  // [R | P] -> G by one warp: lane c owns column c
      const int lane = threadIdx.x;
      bool regular = true;
      for (int k = 0; k < n; ++k) {
        __syncwarp();
        const int p = wpe_pivot(A, n, k);
        if (p < 0) { regular = false; break; }  // warp-uniform
        if (p != k && lane >= k && lane <= n) {
          const wpe_z v = A[k * WPE_LD + lane];
          A[k * WPE_LD + lane] = A[p * WPE_LD + lane];
          A[p * WPE_LD + lane] = v;
        }
        __syncwarp();
        if (lane > k && lane <= n) wpe_eliminate(A, n, k, lane);
      }
      __syncwarp();
      if (lane == 0) wpe_back_substitute(A, n, regular, G);
    }
  }
  if (prm.iterations == 0) return;  // X = Y
  __syncthreads();
  for (int t = threadIdx.x; t < T; t += WPE_THREADS) {
    const wpe_z x = wpe_filter(Y, t, G, n, prm.delay);
    row[t] = wpe_c{(float)x.x, (float)x.y};
  }
}

// One CTA per WPE_OUT_HOPS output hops of a cut: the frames that cover them, then the overlap-add and the length fix.
__global__ void __launch_bounds__(WPE_THREADS) wpe_istft_kernel(const WpeCut *__restrict__ cuts, int ncuts,
                                                                const float *__restrict__ window, const wpe_c *__restrict__ twiddles) {
  extern __shared__ __align__(16) unsigned char wpe_smem[];
  __shared__ wpe_c tw[WPE_NFFT / 2];
  __shared__ float win[WPE_NFFT];
  float *frames = (float *)wpe_smem;                      // [WPE_TILE][512]
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  wpe_c *a = (wpe_c *)(frames + WPE_TILE * WPE_NFFT) + warp * WPE_NFFT;
  const WpeCut c = cuts[wpe_find_cut(cuts, ncuts, true)];
  const int64_t u0 = ((int64_t)blockIdx.x - c.out_begin) * WPE_OUT_HOPS;  // first output hop
  const int64_t f0 = u0 - 1;  // output hop u (samples 128 u .. 128 u + 127) is covered by frames u - 1 .. u + 2
  for (int k = threadIdx.x; k < WPE_NFFT / 2; k += WPE_THREADS) tw[k] = twiddles[k];
  for (int m = threadIdx.x; m < WPE_NFFT; m += WPE_THREADS) win[m] = window[m];
  __syncthreads();
  for (int pr = warp; pr < WPE_TILE / 2; pr += WPE_WARPS) {
    const int64_t fa = f0 + 2 * pr, fb = fa + 1;
    const bool ha = fa >= 0 && fa < c.T, hb = fb >= 0 && fb < c.T;
    if (!ha && !hb) continue;  // warp-uniform
    for (int m = lane; m < WPE_NFFT; m += 32) {
      const int kk = m <= WPE_NFFT / 2 ? m : WPE_NFFT - m;
      const wpe_c A = ha ? c.Y[(int64_t)kk * c.T + fa] : wpe_c{0.0f, 0.0f};
      const wpe_c B = hb ? c.Y[(int64_t)kk * c.T + fb] : wpe_c{0.0f, 0.0f};
      a[wpe_bitrev(m)] = wpe_pack(A, B, m);
    }
    wpe_warp_fft(a, tw, true, lane);
    for (int m = lane; m < WPE_NFFT; m += 32) {
      frames[(2 * pr) * WPE_NFFT + m] = MIX_FMUL(MIX_FMUL(a[m].x, 1.0f / WPE_NFFT), win[m]);
      frames[(2 * pr + 1) * WPE_NFFT + m] = MIX_FMUL(MIX_FMUL(a[m].y, 1.0f / WPE_NFFT), win[m]);
    }
    __syncwarp();
  }
  __syncthreads();
  const int64_t Lz = (int64_t)WPE_HOP * (c.T - 1);
  for (int i = threadIdx.x; i < WPE_OUT_HOPS * WPE_HOP; i += WPE_THREADS) {
    const int64_t j = u0 * WPE_HOP + i;
    if (j >= Lz) break;
    wpe_store(c.out, c.target_len, Lz, j, wpe_ola(frames, f0, c.T, win, j));
  }
}
#endif
