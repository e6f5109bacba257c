// Shared device/host definitions for the b200feat kernels (sm_90a).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <algorithm>
#include <vector>

#include "../../include/b200feat.h"

#define B200_MAX_STAGES 24

// Constant tables + plan, passed to kernels by value (lives in constant bank / param space).
struct DevPlan {
  int feature, L, S, N, K, M, C, F;  // F = output row width
  int Nc;                            // complex FFT length: N/2 (even N, packed real) or N (odd N)
  int packed;                        // 1 if even N
  int pad_left;                      // (L - S) / 2 when !snip_edges (B200FEAT_PAD_KALDI); N / 2 with B200FEAT_PAD_CENTER
  int pad_mode;                      // B200FEAT_PAD_*: 0 mirrors with the edge sample, 1 without (torch "reflect")
  int whisper;                       // feature == B200FEAT_WHISPER_FBANK: per-cut max + normalise pass, n / S valid frames
  int log10_mel;                     // mel epilogue in log10 (whisper-fbank, librosa-fbank) instead of ln
  int snip_edges, remove_dc, use_energy, raw_energy, use_mag, energy_style, use_lifter;
  int energy_last;                   // use_energy == 2 (htk_compat): the energy column is the LAST one (fbank: after the mel bins; mfcc: C0's place moved last)
  int nstages;
  int radix[B200_MAX_STAGES];
  float preemph, energy_floor_log, has_energy_floor, mel_floor, log_spec_eps;
  float log_spec_floor;             // > 0: log-spectrogram as log(max(P, floor)) (torchaudio kaldi.py spectrogram) instead of log(P + eps)
  const float *window;   // [L]
  const float2 *tw;      // [Nc]   exp(-2 pi i k / Nc)
  const float2 *tws;     // [N/2+1] exp(-2 pi i k / N) (packed split), even N only
  const int *mel_start;  // [M] first FFT bin of filter m
  const int *mel_len;    // [M] number of bins
  const int *mel_woff;   // [M] offset into mel_w
  const float *mel_w;    // [sum len]
  const float *dct;      // [M*C]
  const float *lifter;   // [C]
  const float *post_scale;  // [F] or nullptr: every stored value v of column c becomes v * post_scale[c] + post_shift[c]
  const float *post_shift;  //   (b200feat_set_output_affine: a fused GlobalMVN, lhotse/dataset/signal_transforms.py:16-58)
};

// One launch's view of the ragged batch (all device pointers).
struct DevBatch {
  const void *samples;
  const int64_t *samp_off;  // [B] element offsets
  const int64_t *nsamp;     // [B]
  const int64_t *row_off;   // [B+1] packed-row prefix (absolute rows)
  const int64_t *tile_off;  // [B+1] tile prefix (absolute)
  const int32_t *tile_cut;  // [total tiles] absolute tile -> absolute cut (tiled kernels), or nullptr
  float *out;
  float *cut_max;       // [B] per-cut running maximum (whisper-fbank only; bit pattern 0xffffffff = empty)
  int64_t tile_base;    // first tile of this launch (absolute)
  int64_t num_tiles;    // tiles in this launch
  int64_t max_frames;   // T_max (padded mode)
  int batch_first;      // absolute index of the first cut of this launch (padded mode row base)
  int B;                // cuts in this launch
  int out_mode;
  float pad_value;
};

template <int DT>
__device__ __forceinline__ float ld_sample(const void *base, int64_t i) {
  if (DT == B200FEAT_I16) {
    return (float)__ldg(reinterpret_cast<const int16_t *>(base) + i) * (1.0f / 32768.0f);
  } else {
    return __ldg(reinterpret_cast<const float *>(base) + i);
  }
}

// Optional per-column affine of the kernels' epilogues.  The padding value goes through it too: the reference transform
// sees the collated (B, T_max, F) batch, padding included (signal_transforms.py:52-57 after collation.py:506-533).
__device__ __forceinline__ float post_affine(const DevPlan &p, int col, float v) {
  return p.post_scale ? fmaf(v, __ldg(p.post_scale + col), __ldg(p.post_shift + col)) : v;
}

// column of the log-energy in an fbank / mfcc row: first (Kaldi default) or last (htk_compat)
__device__ __forceinline__ int energy_col(const DevPlan &p) { return p.energy_last ? p.F - 1 : 0; }
// first column of the mel bins in an fbank row
__device__ __forceinline__ int mel_shift(const DevPlan &p) { return (p.feature == B200FEAT_FBANK && p.use_energy && !p.energy_last) ? 1 : 0; }

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// index of the sample feeding (frame t, tap j): layers.py:753-772 in closed form (mode 0: the mirror repeats the edge
// sample); mode 1 is torch's "reflect" padding of torch.stft(center=True) (whisper_fbank.py:62): the edge is not repeated
__device__ __forceinline__ int64_t reflect_index(int64_t i, int64_t n, int mode = 0) {
  if (i < 0) i = -i - 1 + mode;
  if (i >= n) i = 2 * n - 1 - mode - i;
  return i;
}

// running float maximum in global memory with torch.max semantics (NaN wins): non-negative floats order like signed
// ints, negative floats like reversed unsigned ints; the slot starts as 0xffffffff (cudaMemset 0xff), which loses to
// every real value on both branches; the canonical NaN 0x7fffffff wins both
__device__ __forceinline__ void atomic_max_float(float *addr, float v) {
  if (v != v) v = __int_as_float(0x7fffffff);
  if (__float_as_int(v) >= 0) atomicMax(reinterpret_cast<int *>(addr), __float_as_int(v));
  else atomicMin(reinterpret_cast<unsigned int *>(addr), __float_as_uint(v));
}

// largest b in [0, B) with prefix[b] <= g   (prefix has B+1 entries, prefix[0] <= g < prefix[B])
__device__ __forceinline__ int find_segment(const int64_t *prefix, int B, int64_t g) {
  int lo = 0, hi = B;
  while (hi - lo > 1) {
    int mid = (lo + hi) >> 1;
    if (__ldg(prefix + mid) <= g) lo = mid; else hi = mid;
  }
  return lo;
}

// torch.max propagates NaN (fmaxf would drop it): max(x, floor) as the reference computes it
__device__ __forceinline__ float nanmax(float x, float floor_) {
  float r;
  asm("max.NaN.f32 %0, %1, %2;" : "=f"(r) : "f"(x), "f"(floor_));
  return r;
}

// log(x) for x known to be a normal float (the mel floor keeps it >= 1.19e-7): MUFU.LG2 * ln 2, i.e. __logf without its
// denormal-input fix-up (8 extra instructions per value); NaN and +inf pass through
__device__ __forceinline__ float fast_lg2_normal(float x) {
  float r;
  asm("lg2.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
  return r;
}
__device__ __forceinline__ float fast_log_normal(float x) { return fast_lg2_normal(x) * 0.69314718055994530942f; }

// Pre-emphasis and window of two adjacent taps: ((d.x - preemph * dp) * w.x, (d.y - preemph * d.x) * w.y), every
// operation rounded on its own (no contraction of the product into a neighbouring add)
__device__ __forceinline__ float2 preemph_window2(float2 d, float dp, float preemph, float2 w) {
  return make_float2(__fmul_rn(__fmaf_rn(dp, -preemph, d.x), w.x), __fmul_rn(__fmaf_rn(d.x, -preemph, d.y), w.y));
}

// one bin of the log-spectrogram: lhotse log(P + 1e-15) (layers.py:467) or Kaldi/torchaudio log(max(P, eps32))
__device__ __forceinline__ float log_spec_value(const DevPlan &p, float x) {
  return p.log_spec_floor > 0.f ? logf(nanmax(x, p.log_spec_floor)) : logf(x + p.log_spec_eps);
}

__device__ __forceinline__ float log_energy_value(const DevPlan &p, float e) {
  float le;
  if (p.energy_style == B200FEAT_ENERGY_KALDI) le = logf(nanmax(e, 1.1920929e-07f));
  else le = logf(e + 1e-15f);
  if (p.has_energy_floor != 0.0f) le = nanmax(le, p.energy_floor_log);
  return le;
}

// ---- host-side helper shared by the N = 512 kernels --------------------------------------------------------------
// The (K x M) mel bank re-packed for a `lanes`-wide epilogue (16 or 8): round j serves `lanes` consecutive filters, one per lane, with a common
// trip count (the round's longest filter); weights beyond a filter's own support are zero, so a shorter filter simply
// keeps accumulating zeros.  `scale` (an exact power of two) is folded into the weights.
struct MelRounds {
  std::vector<int> rstart;    // [rounds][lanes] first FFT bin of filter m = lane + lanes*round (0 if m >= M)
  std::vector<int> rlen;      // [rounds]     trip count
  std::vector<int> rrow;      // [rounds]     first row of the round in wdense
  std::vector<float> wdense;  // [rows][lanes]
  int rounds = 0, rows = 0;
  int max_reach = 0;          // max over lanes of (first bin + trip count): how far zero-weight over-reads go
};

static inline MelRounds pack_mel_rounds(const std::vector<float> &bank, int K, int M, float scale, int lanes = 16, int align = 1,
                                        int limit = 0) {
  // limit > 0: no lane may read past bin `limit` (the P row's padded length): a short filter at the top of the band that shares
  // its round with a wide one starts earlier instead, with zero weights in front (e.g. a 40-filter bank warped by VTLN 0.9)
  // align > 1: every filter starts on a multiple of `align` bins and trip counts are multiples of `align` (zero weights
  // fill the gaps), and the weights of `align` consecutive taps of one lane are adjacent: [row / align][lane][align],
  // so the epilogue can use 64/128-bit shared-memory loads for both operands.
  MelRounds r;
  r.rounds = (M + lanes - 1) / lanes;
  const int alloc = std::max(r.rounds, 1);
  r.rstart.assign(alloc * lanes, 0); r.rlen.assign(alloc, 0); r.rrow.assign(alloc, 0);
  for (int j = 0; j < r.rounds; ++j) {
    int first[32], len[32], mx = 0;  // lanes <= 32
    for (int l = 0; l < lanes; ++l) {
      const int m = l + lanes * j;
      first[l] = 0; len[l] = 0;
      if (m < M) {
        int f0 = -1, f1 = -1;
        for (int k = 0; k < K; ++k)
          if (bank[(size_t)k * M + m] != 0.f) { if (f0 < 0) f0 = k; f1 = k; }
        if (f0 >= 0) { first[l] = f0 / align * align; len[l] = f1 - first[l] + 1; }
      }
      mx = std::max(mx, len[l]);
      r.rstart[j * lanes + l] = first[l];
    }
    mx = (mx + align - 1) / align * align;
    if (limit > 0 && mx <= limit)
      for (int l = 0; l < lanes; ++l)
        if (len[l] > 0 && first[l] + mx > limit) {
          const int nf = (limit - mx) / align * align;
          len[l] += first[l] - nf;
          first[l] = nf;
          r.rstart[j * lanes + l] = nf;
        }
    for (int l = 0; l < lanes; ++l) r.max_reach = std::max(r.max_reach, first[l] + mx);
    r.rlen[j] = mx;
    r.rrow[j] = (int)(r.wdense.size() / lanes);
    for (int g = 0; g < mx; g += align)
      for (int l = 0; l < lanes; ++l)
        for (int e = 0; e < align; ++e) {
          const int m = l + lanes * j, i = g + e;
          r.wdense.push_back((m < M && i < len[l]) ? scale * bank[(size_t)(first[l] + i) * M + m] : 0.f);
        }
  }
  if (r.wdense.empty()) r.wdense.assign(lanes, 0.f);
  r.rows = r.rounds ? (int)(r.wdense.size() / lanes) : 0;
  return r;
}

// ---- the same bank cut into balanced work items (fast2048.cuh) -----------------------------------------------------
// pack_mel_rounds gives every lane one whole filter, so a round costs its WIDEST filter and the last round of a bank runs with
// idle lanes.  Here a filter wider than `T` taps is cut into pieces of at most T taps; items (filter, piece) are dealt to the
// lanes in filter order, a round costs its longest piece, and a second pass adds the (<= a few) pieces of each filter in a fixed
// order.  T is chosen on the host by simulating the shared-memory wavefronts of the epilogue's 128-bit loads (weights: one
// conflict-free wavefront per quarter-warp; P: per quarter-warp the largest number of distinct addresses in one 16-byte bank
// group), so piece offsets that spread over the bank groups win.
struct MelItems {
  std::vector<int> rstart;    // [rounds][lanes] first FFT bin of item q = lane + lanes*round (0 for idle lanes)
  std::vector<int> rlen;      // [rounds]        trip count in taps (multiple of align)
  std::vector<int> rrow;      // [rounds]        first row of the round in wdense
  std::vector<float> wdense;  // [row / align][lane][align]
  std::vector<int> qfirst;    // [M] first item of filter m
  std::vector<int> qcount;    // [M] number of items (0: the filter has no taps)
  int rounds = 0, rows = 0, items = 0, piece = 0;
  int max_reach = 0;
  long cost = 0;              // simulated wavefronts per frame group (slots = 2)
};

static inline MelItems pack_mel_items_T(const std::vector<float> &bank, int K, int M, float scale, int lanes, int align, int T,
                                        bool uniform = false) {  // uniform: every round runs the full T taps
  MelItems r;
  r.piece = T;
  struct Item { int m, first, len; };
  std::vector<Item> items;
  r.qfirst.assign(M, 0); r.qcount.assign(M, 0);
  for (int m = 0; m < M; ++m) {
    int f0 = -1, f1 = -1;
    for (int k = 0; k < K; ++k)
      if (bank[(size_t)k * M + m] != 0.f) { if (f0 < 0) f0 = k; f1 = k; }
    r.qfirst[m] = (int)items.size();
    if (f0 < 0) continue;
    const int s0 = f0 / align * align, end = f1 + 1;
    for (int a = s0; a < end; a += T) items.push_back({m, a, std::min(T, end - a)});
    r.qcount[m] = (int)items.size() - r.qfirst[m];
  }
  r.items = (int)items.size();
  r.rounds = (r.items + lanes - 1) / lanes;
  const int alloc = std::max(r.rounds, 1);
  r.rstart.assign(alloc * lanes, 0); r.rlen.assign(alloc, 0); r.rrow.assign(alloc, 0);
  for (int j = 0; j < r.rounds; ++j) {
    int mx = 0;
    for (int l = 0; l < lanes; ++l) {
      const int q = l + lanes * j;
      if (q < r.items) { r.rstart[q] = items[q].first; mx = std::max(mx, items[q].len); }
    }
    mx = uniform ? T : (mx + align - 1) / align * align;
    for (int l = 0; l < lanes; ++l) r.max_reach = std::max(r.max_reach, r.rstart[j * lanes + l] + mx);
    r.rlen[j] = mx;
    r.rrow[j] = (int)(r.wdense.size() / lanes);
    for (int g = 0; g < mx; g += align) {
      for (int l = 0; l < lanes; ++l)
        for (int e = 0; e < align; ++e) {
          const int q = l + lanes * j, i = g + e;
          r.wdense.push_back((q < r.items && i < items[q].len) ? scale * bank[(size_t)(items[q].first + i) * M + items[q].m] : 0.f);
        }
      // simulated cost of this trip: weights 4 wavefronts per 32 lanes, P loads per quarter-warp
      long wf = 0;
      for (int q0 = 0; q0 < lanes; q0 += 8) {
        int distinct[8][8], cnt[8] = {0, 0, 0, 0, 0, 0, 0, 0};
        for (int l = q0; l < q0 + 8 && l < lanes; ++l) {
          const int a = (r.rstart[j * lanes + l] + g) / 4, bg = a & 7;
          bool seen = false;
          for (int c = 0; c < cnt[bg]; ++c) seen |= distinct[bg][c] == a;
          if (!seen) distinct[bg][cnt[bg]++] = a;
        }
        int worst = 1;
        for (int bg = 0; bg < 8; ++bg) worst = std::max(worst, cnt[bg]);
        wf += worst;
      }
      r.cost += lanes / 8 + 2 * wf;
    }
  }
  if (r.wdense.empty()) r.wdense.assign(lanes * align, 0.f);
  r.rows = r.rounds ? (int)(r.wdense.size() / lanes) : 0;
  return r;
}

static inline MelItems pack_mel_items(const std::vector<float> &bank, int K, int M, float scale, int lanes = 32, int align = 4) {
  MelItems best;
  bool have = false;
  for (int T = 2 * align; T <= 1024; T += align) {
    MelItems c = pack_mel_items_T(bank, K, M, scale, lanes, align, T);
    if (c.rounds > 12) continue;  // the second pass keeps rounds * lanes partial sums per frame in shared memory
    if (!have || c.cost < best.cost) { best = c; have = true; }
    if (c.items == 0 || c.piece >= K) break;
  }
  if (!have) best = pack_mel_items_T(bank, K, M, scale, lanes, align, (K + align - 1) / align * align);
  return best;
}
