// Backward of the Kaldi-family features (fbank, mfcc, spectrogram, log-spectrogram): the gradient of a scalar loss with
// respect to the float32 waveform, given the gradient with respect to the packed (sum T_i, F) feature rows.
//
// The arithmetic contract is DESIGN.md §3.1n.  Per frame, in reverse order of the forward (generic.cuh):
//   log        log(max(v, floor)) passes g / v where v > floor, g / (2 v) on an exact tie (torch.max's rule), 0 below;
//              log(v + eps) passes g / (v + eps).  The same rules hold for the log-energy and its floor.
//   mel, mfcc  gM = fb^T gML (over the plan's filter ranges); for mfcc gML = dct (g * lifter); a column replaced by the
//              log-energy passes nothing into the spectrum
//   spectrum   Z_k = gP_k X_k (power) or gA_k X_k / (2 |X_k|) (magnitude, 0 where |X_k| = 0); the frame gradient is
//              2 Re sum_{k=0}^{N/2} Z_k e^{+2 pi i k n / N}: a real inverse FFT of Z with Z_0 and Z_{N/2} doubled, of which
//              the first L outputs are kept
//   frame      window, the adjoint of pre-emphasis with the replicated left sample, the energy term (raw or windowed),
//              then g - mean(g) for the DC removal
//   samples    the frames are summed back into the samples; a mirrored edge sample adds onto its source
// The frame kernel recomputes the windowed samples, the spectrum and the mel energies of each frame from the saved input
// (nothing of the forward is stored), runs both FFTs with generic.cuh's stockham_pass, and overlap-adds a tile of
// consecutive frames of one cut in shared memory into a per-tile span of the work buffer.  The combine kernel then sums,
// for every sample, the spans of the tiles that cover it in tile order.  No atomics: the result is bitwise reproducible
// and a cut's gradient does not depend on the other cuts of its batch.
//
// whisper-fbank (DESIGN.md §3.1p) runs the same chain with three differences.  The row gradient comes from the saved
// un-normalised log-mel rows x and the cut's maximum m: y = (maximum(x, m - 8) + 4) / 4 passes g / 4 to x above the
// threshold, half of it on a tie, and the rest to m, which max() spreads evenly over the elements equal to m; a reduction
// kernel sums that routed mass and counts the ties per cut before the frames kernel runs.  log10(clamp(v, 1e-10)) passes
// g / (v ln 10) where v >= 1e-10 and nothing below.  The frames are torch.stft's centred frames over the stft's n / S rows
// (the zero row gets no gradient), mirrored without repeating the edge sample.
//
// The per-frame and per-sample arithmetic is __host__ __device__, so that scripts/micro/backward_host_check.cu and
// scripts/micro/whisper_backward_host_check.cu run this code on the CPU.  Kernels at the end.
#pragma once
#include <math.h>
#include <stddef.h>
#include <stdint.h>

#include "../../include/b200feat.h"

#ifdef __CUDACC__
#define BWD_HD __host__ __device__ __forceinline__
#else
#define BWD_HD inline
#endif

#define BWD_MAX_WARPS 4   // warps of a frame-kernel CTA (fewer when a long frame does not fit shared memory)
#define BWD_MAX_TILE 16   // consecutive frames of one cut per CTA (fewer when a long frame does not fit)
#define BWD_SMEM_LIMIT (200 * 1024)
#define BWD_COMBINE_THREADS 256
#define BWD_REDUCE_THREADS 256  // per-cut reduction of whisper-fbank: fixed, so that its summation order is fixed

struct BwdC {  // same layout as float2
  float x, y;
};

// What the backward reads of the plan (built from the forward's DevPlan and device tables)
struct BwdPlan {
  int feature, L, S, N, K, M, C, F, Nc, packed;
  int pad, snip_edges, remove_dc, use_energy, raw_energy, use_mag, energy_style, use_lifter;
  int ecol;   // column of the log-energy (fbank / mfcc) when use_energy
  int shift;  // first mel column of an fbank row
  int whisper;  // whisper-fbank: row gradient from the saved log-mel rows, log10 with its clamp, n / S frames
  int reflect;  // mirror of the padded edges: 0 repeats the edge sample (Kaldi), 1 does not (torch's "reflect")
  float preemph, energy_floor_log, has_energy_floor, mel_floor, log_spec_eps, log_spec_floor;
  const float *window;     // [L]
  const BwdC *tws;         // [N/2 + 1] exp(-2 pi i k / N), even N
  const int *mel_start, *mel_len, *mel_woff;
  const float *mel_w, *dct, *lifter;
  const float *post_scale;  // [F] or null
};

// ---- launch shape --------------------------------------------------------------------------------------------------
BWD_HD int bwd_round4(int n) { return (n + 3) & ~3; }

// floats of one warp's frame buffers: X / Z [2K], two FFT buffers [2 Nc each], raw samples [L], spectrum values [K],
// mel gradient [M]
BWD_HD int bwd_warp_floats(const BwdPlan &p) {
  return bwd_round4(2 * p.K) + 4 * p.Nc + bwd_round4(p.L) + bwd_round4(p.K) + bwd_round4(p.M > 0 ? p.M : 1);
}
// floats of the span one tile of `ft` frames covers
BWD_HD int64_t bwd_span(const BwdPlan &p, int ft) { return (int64_t)(ft - 1) * p.S + p.L; }
// dynamic shared memory of a CTA: per-bin filter ranges [2 K ints], frame gradients [ft][L], the warps' buffers
BWD_HD size_t bwd_smem(const BwdPlan &p, int warps, int ft) {
  return (size_t)bwd_round4(2 * p.K) * 4 + (size_t)ft * bwd_round4(p.L) * 4 + (size_t)warps * bwd_warp_floats(p) * 4;
}
// largest shape within BWD_SMEM_LIMIT: tile first, then warps; false if even one warp and one frame do not fit
inline bool bwd_launch_shape(const BwdPlan &p, int *warps, int *ft) {
  int w = BWD_MAX_WARPS, f = BWD_MAX_TILE;
  while (bwd_smem(p, w, f) > BWD_SMEM_LIMIT && f > w) f /= 2;
  while (bwd_smem(p, w, f) > BWD_SMEM_LIMIT && w > 1) { w /= 2; if (f > w) f = w; }
  *warps = w; *ft = f;
  return bwd_smem(p, w, f) <= BWD_SMEM_LIMIT;
}

// ---- per-frame arithmetic ------------------------------------------------------------------------------------------
// d log(max(v, floor)) / dv, torch.max's rule at an exact tie
BWD_HD float bwd_dlog_max(float v, float floor_) { return v > floor_ ? 1.f / v : (v == floor_ ? 0.5f / v : 0.f); }

// d(log-energy) / d(sum of squares) at sum e (common.cuh log_energy_value)
BWD_HD float bwd_energy_scale(const BwdPlan &p, float e) {
  float lv, d;
  if (p.energy_style == B200FEAT_ENERGY_KALDI) {
    const float eps = 1.1920929e-07f;
    lv = logf(e > eps ? e : eps);
    d = bwd_dlog_max(e, eps);
  } else {
    lv = logf(e + 1e-15f);
    d = 1.f / (e + 1e-15f);
  }
  if (p.has_energy_floor != 0.f) d *= lv > p.energy_floor_log ? 1.f : (lv == p.energy_floor_log ? 0.5f : 0.f);
  return d;
}

BWD_HD float bwd_col_scale(const BwdPlan &p, int c) { return p.post_scale ? p.post_scale[c] : 1.f; }

// gradient of the row's log-energy column (0 without use_energy)
BWD_HD float bwd_energy_grad(const BwdPlan &p, const float *g) {
  if (!p.use_energy) return 0.f;
  return g[p.ecol] * bwd_col_scale(p, p.ecol);
}

// windowed, pre-emphasised sample j < L of a frame whose raw samples are raw[0, L) and mean mu (generic.cuh)
BWD_HD float bwd_y(const BwdPlan &p, const float *raw, float mu, int j) {
  const float d = raw[j] - mu;
  float g0 = d;
  if (p.preemph != 0.f) {
    const float dp = raw[j > 0 ? j - 1 : 0] - mu;
    g0 = d - p.preemph * dp;
  }
  return g0 * p.window[j];
}

// the energy term of sample j < L: d^2 (raw energy) or y^2
BWD_HD float bwd_energy_term(const BwdPlan &p, const float *raw, float mu, int j) {
  if (p.raw_energy) { const float d = raw[j] - mu; return d * d; }
  const float y = bwd_y(p, raw, mu, j);
  return y * y;
}

// bin k of the real spectrum from the FFT output (packed split for even N, generic.cuh)
BWD_HD BwdC bwd_bin(const BwdPlan &p, const BwdC *src, int k) {
  if (!p.packed) return src[k];
  const BwdC zk = src[k == p.Nc ? 0 : k];
  const BwdC zc = src[k == 0 ? 0 : p.Nc - k];
  const float er = zk.x + zc.x, ei = zk.y - zc.y;
  const float orr = zk.x - zc.x, oi = zk.y + zc.y;
  const BwdC w = p.tws[k];
  const float tr = w.x * orr - w.y * oi, ti = w.x * oi + w.y * orr;
  return BwdC{0.5f * (er + ti), 0.5f * (ei - tr)};
}

// the spectrum value the epilogue reads: |X|^2 or |X|
BWD_HD float bwd_value(const BwdPlan &p, BwdC X) {
  const float pw = X.x * X.x + X.y * X.y;
  return p.use_mag ? sqrtf(pw) : pw;
}

// mel energy of filter m from the spectrum values (generic.cuh's order)
BWD_HD float bwd_mel(const BwdPlan &p, const float *v, int m) {
  const int st = p.mel_start[m], len = p.mel_len[m];
  const float *w = p.mel_w + p.mel_woff[m];
  float acc = 0.f;
  for (int i = 0; i < len; ++i) acc += v[st + i] * w[i];
  return acc;
}

// gradient reaching mel energy m (fbank / mfcc) of a row with gradient g, mel energy mel
BWD_HD float bwd_gmel(const BwdPlan &p, const float *g, int m, float mel) {
  float gl;
  if (p.feature == B200FEAT_FBANK) {
    gl = g[m + p.shift] * bwd_col_scale(p, m + p.shift);
  } else {
    gl = 0.f;
    for (int c = 0; c < p.C; ++c) {
      if (p.use_energy && c == p.ecol) continue;
      float gc = g[c] * bwd_col_scale(p, c);
      if (p.use_lifter) gc *= p.lifter[c];
      gl += gc * p.dct[m * p.C + c];
    }
  }
  return gl * bwd_dlog_max(mel, p.mel_floor);
}

// first and one-past-last filter whose range holds bin k (lo >= hi: none)
BWD_HD void bwd_bin_filters(const BwdPlan &p, int k, int *lo, int *hi) {
  int a = p.M, b = 0;
  for (int m = 0; m < p.M; ++m)
    if (k >= p.mel_start[m] && k < p.mel_start[m] + p.mel_len[m]) { if (m < a) a = m; b = m + 1; }
  *lo = a; *hi = b;
}

// gradient reaching spectrum value k: the mel transpose over the filters [lo, hi), or the row's own column
BWD_HD float bwd_gvalue(const BwdPlan &p, const float *g, const float *v, const float *gm, int lo, int hi, int k) {
  if (p.feature == B200FEAT_FBANK || p.feature == B200FEAT_MFCC || p.whisper) {
    float acc = 0.f;
    for (int m = lo; m < hi; ++m) {
      const int i = k - p.mel_start[m];
      if (i >= 0 && i < p.mel_len[m]) acc += p.mel_w[p.mel_woff[m] + i] * gm[m];
    }
    return acc;
  }
  if (k == 0 && p.use_energy) return 0.f;
  const float gk = g[k] * bwd_col_scale(p, k);
  if (p.feature == B200FEAT_SPECTROGRAM) return gk;
  return gk * (p.log_spec_floor > 0.f ? bwd_dlog_max(v[k], p.log_spec_floor) : 1.f / (v[k] + p.log_spec_eps));
}

// Z_k from X_k, its spectrum value v (|X|^2 or |X|) and the gradient gv reaching v
BWD_HD BwdC bwd_z(const BwdPlan &p, BwdC X, float v, float gv) {
  if (p.use_mag) {
    if (!(v > 0.f)) return BwdC{0.f, 0.f};
    const float s = 0.5f * gv / v;
    return BwdC{s * X.x, s * X.y};
  }
  return BwdC{gv * X.x, gv * X.y};
}

// the Hermitian spectrum H of the inverse transform: H_0 = 2 Re Z_0, H_{N/2} = 2 Re Z_{N/2} (even N), H_k = Z_k else
BWD_HD BwdC bwd_h(const BwdPlan &p, const BwdC *Z, int k) {
  if (k == 0 || (p.packed && k == p.Nc)) return BwdC{2.f * Z[k].x, 0.f};
  return Z[k];
}

// entry k of the inverse FFT's input, taken through the forward (e^{-i}) transform: even N, conj(C_k), k < N/2, with
// C_k = (H_k + conj H_{N/2-k}) + i e^{+2 pi i k / N} (H_k - conj H_{N/2-k}); odd N, conj(H_k) for k < K, H_{N-k} above
BWD_HD BwdC bwd_inv_in(const BwdPlan &p, const BwdC *Z, int k) {
  if (!p.packed) {
    if (k < p.K) { const BwdC h = bwd_h(p, Z, k); return BwdC{h.x, -h.y}; }
    return bwd_h(p, Z, p.N - k);
  }
  const BwdC hk = bwd_h(p, Z, k), hm = bwd_h(p, Z, p.Nc - k);
  const float ex = hk.x + hm.x, ey = hk.y - hm.y;  // H_k + conj(H_{N/2-k})
  const float dx = hk.x - hm.x, dy = hk.y + hm.y;  // H_k - conj(H_{N/2-k})
  const BwdC w = p.tws[k];                         // conj(e^{+2 pi i k / N})
  const float ox = w.x * dx + w.y * dy, oy = w.x * dy - w.y * dx;
  return BwdC{ex - oy, -(ey + ox)};
}

// gradient of windowed sample j < L from the inverse FFT's output
BWD_HD float bwd_gy(const BwdPlan &p, const BwdC *out, int j) {
  if (!p.packed) return out[j].x;
  return (j & 1) ? -out[j >> 1].y : out[j >> 1].x;
}

// gradient of the pre-emphasised sample j: through the window, plus the windowed energy term
BWD_HD float bwd_gpre(const BwdPlan &p, const BwdC *out, const float *raw, float mu, float ge, int j) {
  float gy = bwd_gy(p, out, j);
  if (p.use_energy && !p.raw_energy) gy += 2.f * ge * bwd_y(p, raw, mu, j);
  return gy * p.window[j];
}

// gradient of the DC-removed sample j: the pre-emphasis adjoint (tap j feeds j and j + 1; tap 0 is also its own left
// neighbour) plus the raw energy term
BWD_HD float bwd_gd(const BwdPlan &p, const BwdC *out, const float *raw, float mu, float ge, int j) {
  float gd = bwd_gpre(p, out, raw, mu, ge, j);
  if (p.preemph != 0.f) {
    if (j + 1 < p.L) gd -= p.preemph * bwd_gpre(p, out, raw, mu, ge, j + 1);
    if (j == 0) gd -= p.preemph * bwd_gpre(p, out, raw, mu, ge, 0);
  }
  if (p.use_energy && p.raw_energy) gd += 2.f * ge * (raw[j] - mu);
  return gd;
}

// ---- whisper-fbank -------------------------------------------------------------------------------------------------
// frames of a cut of n samples the backward runs: the stft's n / S rows for whisper-fbank, else every row
BWD_HD int64_t bwd_frames(const BwdPlan &p, int64_t n, int64_t rows) { return p.whisper ? n / p.S : rows; }

// share of g / 4 that maximum(x, thr) passes to x: all above the threshold, half on a tie, none below (torch.maximum)
BWD_HD float bwd_whisper_weight(float x, float thr) { return x > thr ? 1.f : (x == thr ? 0.5f : 0.f); }

// what log-mel value x with row gradient g routes to the threshold m - 8, i.e. to the cut's maximum
BWD_HD float bwd_whisper_routed(float g, float x, float m) { return 0.25f * g * (1.f - bwd_whisper_weight(x, m - 8.f)); }

// gradient reaching log-mel value x: its own share of g / 4, plus the cut's routed mass over its `ties` maxima if x is one
BWD_HD float bwd_whisper_glog(float g, float x, float m, float routed, int ties) {
  float gx = 0.25f * g * bwd_whisper_weight(x, m - 8.f);
  if (x == m) gx += routed / (float)ties;
  return gx;
}

// d log10(clamp(v, min = floor)) / dv: torch.clamp passes the gradient where v >= floor, the tie included
BWD_HD float bwd_dlog10_clamp(float v, float floor_) { return v >= floor_ ? 1.f / (v * 2.30258509299404568402f) : 0.f; }

// gradient reaching mel energy m of a whisper-fbank row with gradient g and saved log-mel row x
BWD_HD float bwd_whisper_gmel(const BwdPlan &p, const float *g, const float *x, int m, float mel, float cmax, float routed,
                              int ties) {
  return bwd_whisper_glog(g[m], x[m], cmax, routed, ties) * bwd_dlog10_clamp(mel, p.mel_floor);
}

// ---- overlap-add ---------------------------------------------------------------------------------------------------
// position r of a tile's span: the sum, in frame order, of the gradients G[f][r - f S] of the tile's nf frames
BWD_HD float bwd_span_value(const float *G, int ldg, int nf, int S, int L, int r) {
  int f = r < L ? 0 : (r - L) / S + 1;
  const int f1 = r / S < nf - 1 ? r / S : nf - 1;
  float acc = 0.f;
  for (; f <= f1; ++f) acc += G[(size_t)f * ldg + (r - f * S)];
  return acc;
}

// the sum over the tiles of one cut (spans back to back in `ws`) at padded position q
BWD_HD float bwd_position(const float *ws, int64_t ntiles, int64_t span, int64_t stride, int64_t q) {
  int64_t t = q < span ? 0 : (q - span) / stride + 1;
  const int64_t t1 = q / stride < ntiles - 1 ? q / stride : ntiles - 1;
  float acc = 0.f;
  for (; t <= t1; ++t) acc += ws[t * span + (q - t * stride)];
  return acc;
}

// gradient of sample i of a cut of n samples and T frames: its own padded position, then its left and right mirror
// images.  layers.py:753-772 reflects once about either end, the edge sample repeated (reflect 0); torch.stft's "reflect"
// padding does not repeat it (reflect 1), so the edge samples have no image there.
BWD_HD float bwd_sample(const BwdPlan &p, const float *ws, int64_t ntiles, int ft, int64_t n, int64_t T, int64_t i) {
  const int64_t span = bwd_span(p, ft), stride = (int64_t)ft * p.S;
  const int64_t ext = (T - 1) * p.S + p.L, pad = p.snip_edges ? 0 : p.pad;
  float acc = 0.f;
  if (i + pad < ext) acc += bwd_position(ws, ntiles, span, stride, i + pad);
  if (!p.snip_edges) {
    const int64_t r = p.reflect;
    if (i >= r && i < pad + r) acc += bwd_position(ws, ntiles, span, stride, pad - 1 - i + r);
    const int64_t qr = 2 * n - 1 - r - i + pad;
    if (i < n - r && qr < ext) acc += bwd_position(ws, ntiles, span, stride, qr);
  }
  return acc;
}

// the work buffer: int64 tables [samp_off B][nsamp B][row_off B + 1][tile_off B + 1], then (whisper-fbank) the per-cut
// routed mass [B] and tie count [B], then the tiles' spans
BWD_HD int64_t bwd_meta_bytes(int32_t B) { return ((4 * (int64_t)B + 2) * 8 + 255) / 256 * 256; }
BWD_HD int64_t bwd_reduce_bytes(const BwdPlan &p, int32_t B) { return p.whisper ? (8 * (int64_t)B + 255) / 256 * 256 : 0; }

#if defined(__CUDACC__)
#include "generic.cuh"

struct BwdBatch {
  const float *samples;
  const float *grad_out;
  float *grad_in;
  const int64_t *samp_off, *nsamp, *row_off, *tile_off;
  float *spans;
  int B, ft;
  // whisper-fbank: the forward's un-normalised log-mel rows (laid out as grad_out) and per-cut maxima, and the reduction's
  // per-cut routed mass and tie count
  const float *xrows, *cut_max;
  float *routed;
  int *ties;
};

__device__ __forceinline__ int bwd_find(const int64_t *prefix, int B, int64_t g) {
  int lo = 0, hi = B;
  while (hi - lo > 1) {
    const int mid = (lo + hi) >> 1;
    if (prefix[mid] <= g) lo = mid; else hi = mid;
  }
  return lo;
}

// One CTA per tile of <= ft consecutive frames of one cut, one warp per frame at a time.
// `fp` is the forward's plan: its FFT twiddles and radix passes.
__global__ void __launch_bounds__(BWD_MAX_WARPS * 32, 1) b200feat_backward_frames_kernel(const BwdPlan p, const DevPlan fp,
                                                                                      const BwdBatch b, int64_t ntiles) {
  extern __shared__ __align__(16) float bsm[];
  __shared__ int radix[B200_MAX_STAGES];  // the passes' radices: a dynamically indexed parameter array would live in local memory
  if (threadIdx.x < B200_MAX_STAGES) radix[threadIdx.x] = fp.radix[threadIdx.x];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
  int *flo = reinterpret_cast<int *>(bsm), *fhi = flo + p.K;
  float *G = bsm + bwd_round4(2 * p.K);
  const int ldg = bwd_round4(p.L);
  float *mine = G + (size_t)b.ft * ldg + (size_t)warp * bwd_warp_floats(p);
  BwdC *xs = reinterpret_cast<BwdC *>(mine);
  float2 *bufA = reinterpret_cast<float2 *>(mine + bwd_round4(2 * p.K));
  float2 *bufB = bufA + p.Nc;
  float *raw = reinterpret_cast<float *>(bufB + p.Nc);
  float *v = raw + bwd_round4(p.L);
  float *gm = v + bwd_round4(p.K);
  const bool mel = p.feature == B200FEAT_FBANK || p.feature == B200FEAT_MFCC || p.whisper;
  if (mel)
    for (int k = threadIdx.x; k < p.K; k += blockDim.x) bwd_bin_filters(p, k, flo + k, fhi + k);
  const int64_t span = bwd_span(p, b.ft);

  for (int64_t tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    __syncthreads();  // the filter ranges are written; the previous tile's G has been read
    const int cut = bwd_find(b.tile_off, b.B, tile);
    const int64_t t0 = (tile - b.tile_off[cut]) * b.ft;
    const int64_t n = b.nsamp[cut];
    const int64_t T = bwd_frames(p, n, b.row_off[cut + 1] - b.row_off[cut]);
    const int nf = (int)min((int64_t)b.ft, T - t0);
    const float *x = b.samples + b.samp_off[cut];
    for (int f = warp; f < nf; f += nwarps) {
      const int64_t t = t0 + f;
      const float *g = b.grad_out + (b.row_off[cut] + t) * p.F;
      const int64_t base = t * p.S - (p.snip_edges ? 0 : p.pad);
      float s = 0.f;
      for (int j = lane; j < p.L; j += 32) {
        int64_t i = base + j;
        if (!p.snip_edges) i = reflect_index(i, n, p.reflect);
        const float r = __ldg(x + i);
        raw[j] = r;
        s += r;
      }
      s = warp_sum(s);
      const float mu = p.remove_dc ? s / (float)p.L : 0.f;
      __syncwarp();
      float e = 0.f;
      float *ybuf = reinterpret_cast<float *>(bufA);
      for (int j = lane; j < p.N; j += 32) {
        float y = 0.f;
        if (j < p.L) {
          y = bwd_y(p, raw, mu, j);
          if (p.use_energy) e += bwd_energy_term(p, raw, mu, j);
        }
        if (p.packed) ybuf[j] = y; else bufA[j] = make_float2(y, 0.f);
      }
      const float ge = p.use_energy ? bwd_energy_grad(p, g) * bwd_energy_scale(p, warp_sum(e)) : 0.f;
      __syncwarp();
      float2 *src = bufA, *dst = bufB;
      int Ns = 1;
      for (int st = 0; st < fp.nstages; ++st) {
        stockham_pass(src, dst, fp.tw, p.Nc, radix[st], Ns, lane);
        __syncwarp();
        float2 *tmp = src; src = dst; dst = tmp;
        Ns *= radix[st];
      }
      for (int k = lane; k < p.K; k += 32) {
        const BwdC X = bwd_bin(p, reinterpret_cast<const BwdC *>(src), k);
        xs[k] = X;
        v[k] = bwd_value(p, X);
      }
      __syncwarp();
      if (mel) {
        if (p.whisper) {
          const float *xr = b.xrows + (b.row_off[cut] + t) * p.F;
          const float cm = b.cut_max[cut], routed = b.routed[cut];
          const int ties = b.ties[cut];
          for (int m = lane; m < p.M; m += 32) gm[m] = bwd_whisper_gmel(p, g, xr, m, bwd_mel(p, v, m), cm, routed, ties);
        } else {
          for (int m = lane; m < p.M; m += 32) gm[m] = bwd_gmel(p, g, m, bwd_mel(p, v, m));
        }
        __syncwarp();
      }
      for (int k = lane; k < p.K; k += 32) {
        const float gv = bwd_gvalue(p, g, v, gm, mel ? flo[k] : 0, mel ? fhi[k] : 0, k);
        xs[k] = bwd_z(p, xs[k], v[k], gv);
      }
      __syncwarp();
      const int nin = p.packed ? p.Nc : p.N;
      for (int k = lane; k < nin; k += 32) {
        const BwdC c = bwd_inv_in(p, xs, k);
        bufA[k] = make_float2(c.x, c.y);
      }
      __syncwarp();
      src = bufA; dst = bufB; Ns = 1;
      for (int st = 0; st < fp.nstages; ++st) {
        stockham_pass(src, dst, fp.tw, p.Nc, radix[st], Ns, lane);
        __syncwarp();
        float2 *tmp = src; src = dst; dst = tmp;
        Ns *= radix[st];
      }
      float *Gf = G + (size_t)f * ldg;
      const BwdC *out = reinterpret_cast<const BwdC *>(src);
      float sum = 0.f;
      for (int j = lane; j < p.L; j += 32) {
        const float gd = bwd_gd(p, out, raw, mu, ge, j);
        Gf[j] = gd;
        sum += gd;
      }
      if (p.remove_dc) {
        const float mean = warp_sum(sum) / (float)p.L;
        for (int j = lane; j < p.L; j += 32) Gf[j] -= mean;
      }
      __syncwarp();
    }
    __syncthreads();
    float *ws = b.spans + tile * span;
    const int cover = (nf - 1) * p.S + p.L;
    for (int r = threadIdx.x; r < span; r += blockDim.x) ws[r] = r < cover ? bwd_span_value(G, ldg, nf, p.S, p.L, r) : 0.f;
  }
}

// whisper-fbank, before the frames kernel: one CTA per cut sums what its stft rows route to the cut's maximum and counts
// the elements equal to it.  Thread j takes elements j, j + 256, ... in order, then a fixed tree: the result depends on the
// cut alone.
__global__ void __launch_bounds__(BWD_REDUCE_THREADS) b200feat_whisper_backward_reduce_kernel(const BwdPlan p, const BwdBatch b) {
  __shared__ float s_mass[BWD_REDUCE_THREADS];
  __shared__ int s_ties[BWD_REDUCE_THREADS];
  for (int cut = blockIdx.x; cut < b.B; cut += gridDim.x) {
    const int64_t count = bwd_frames(p, b.nsamp[cut], 0) * p.F;
    const float *g = b.grad_out + b.row_off[cut] * p.F, *x = b.xrows + b.row_off[cut] * p.F;
    const float m = b.cut_max[cut];
    float mass = 0.f;
    int ties = 0;
    for (int64_t e = threadIdx.x; e < count; e += BWD_REDUCE_THREADS) {
      const float xv = x[e];
      mass += bwd_whisper_routed(g[e], xv, m);
      ties += xv == m;
    }
    s_mass[threadIdx.x] = mass;
    s_ties[threadIdx.x] = ties;
    __syncthreads();
    for (int h = BWD_REDUCE_THREADS / 2; h > 0; h >>= 1) {
      if (threadIdx.x < h) {
        s_mass[threadIdx.x] += s_mass[threadIdx.x + h];
        s_ties[threadIdx.x] += s_ties[threadIdx.x + h];
      }
      __syncthreads();
    }
    if (threadIdx.x == 0) {
      b.routed[cut] = s_mass[0];
      b.ties[cut] = s_ties[0];
    }
    __syncthreads();  // the next cut reuses the shared arrays
  }
}

// One thread per sample: the tiles' spans summed back into the cut's samples.
__global__ void __launch_bounds__(BWD_COMBINE_THREADS) b200feat_backward_combine_kernel(const BwdPlan p, const BwdBatch b) {
  for (int cut = blockIdx.y; cut < b.B; cut += gridDim.y) {
    const int64_t n = b.nsamp[cut], T = bwd_frames(p, n, b.row_off[cut + 1] - b.row_off[cut]);
    const int64_t t0 = b.tile_off[cut], ntiles = b.tile_off[cut + 1] - t0;
    const float *ws = b.spans + t0 * bwd_span(p, b.ft);
    float *gx = b.grad_in + b.samp_off[cut];
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
      gx[i] = bwd_sample(p, ws, ntiles, b.ft, n, T, i);
  }
}
#endif
