// Feature-domain mixing and right-padding collation of precomputed feature rows (lhotse's collate_features over cuts with
// stored features: MixedCut.load_features and its FeatureMixer, PaddingCut constants, the padding-only copy) on the GPU, from
// the tables lhotse_b200/precomputed.py plans.
//
// The arithmetic contract is DESIGN.md §3.1m.  In short, per cut:
//   energy   E_t = the float64 sum of e^x (log law) or x (linear law) over track t's rows: FM_PARTS CTAs per track, CTA p
//            summing chunks p, p + FM_PARTS, ... of FM_CHUNK elements, each thread in element order, then a fixed tree per
//            CTA; the gains fold the parts in order
//   gains    a later mixed track with an SNR: g = E_ref * factor / E_t when E_ref > 0 and E_t > 0, else 1 (FeatureMixer);
//            the first track with an SNR, only when the reference is another track: the same g unless E_ref <= 0 or E_t <= 0
//            (_scale_features_for_snr's rejections, so a NaN energy gives a NaN gain), stored as log g for the log law
//            (x + log g) and g for the linear law (g x)
//   output   per element in float64, rounded once: the base (the scaled first track, -1000 past its rows), then every further
//            mixed track folded in track order with -1000 outside its rows: s = max(EPSILON, s + g e^b) over s = e^base and a
//            final log (log law), or s + g b (linear law); a cut with no further track is its base.  Mix row m = min(r,
//            mix_rows - 1) (trimmed, or the last row repeated).  COPY cuts are their track's rows and then pad_value; rows
//            past a cut's num_rows are the call's pad value.
//   non-finite values  NaN and +-inf follow lhotse's float64 code element by element: the clamp keeps a NaN (np.maximum),
//            inf * 0 is NaN, and a COPY cut is its rows bit for bit.
//   cuts     any number: the output kernel's grid y is min(cuts, 65535) and strides over the rest.
//
// The per-element, per-thread and per-cut arithmetic is __host__ __device__, so that scripts/micro/featmix_host_check.cu runs
// exactly this code on the CPU.  Kernels at the end.
#pragma once
#include <math.h>
#include <stdint.h>

#include "mix.cuh"

#define FM_PARTS 8                  // energy CTAs per track
#define FM_THREADS 256              // energy and output CTAs
#define FM_CHUNK (FM_THREADS * 8)   // elements of one energy round of a CTA
#define FM_TILE 2048                // output elements of a cut one CTA writes
#define FM_GAIN_THREADS 128
#define FM_DUMMY (-1000.0)          // FeatureMixer's padding_value
#define FM_EPSILON 1e-10            // lhotse.utils.EPSILON

// CUDA's and the C library's float64 exp / log may differ in the last bit: the host check is held to a tolerance, not bits
#define FM_DEXP(a) exp(a)
#define FM_DLOG(a) log(a)

// element (r, c) of track t's rows (r < num_rows): a constant, or the stored row (the last one for a repeated last row)
MIX_HD float fm_track_x(const float *src, const b200feat_featmix_track &t, int F, int64_t r, int c) {
  if (t.stored_rows == 0) return t.value;
  const int64_t rr = r < t.stored_rows ? r : (int64_t)t.stored_rows - 1;
  return src[t.src_elem + rr * F + c];
}

MIX_HD double fm_energy_term(int law, float x) { return law == B200FEAT_FEATMIX_LOG ? FM_DEXP((double)x) : (double)x; }

// the float64 sum one thread of energy CTA `part` of track t makes, in element order
MIX_HD double fm_energy_thread(const float *src, const b200feat_featmix_track &t, int law, int F, int part, int tid) {
  const int64_t n = (int64_t)t.num_rows * F;
  double acc = 0.0;
  for (int64_t k = (int64_t)part * FM_CHUNK; k < n; k += (int64_t)FM_PARTS * FM_CHUNK)
    for (int j = 0; j < FM_CHUNK / FM_THREADS; ++j) {
      const int64_t e = k + (int64_t)j * FM_THREADS + tid;
      if (e < n) acc = MIX_DADD(acc, fm_energy_term(law, fm_track_x(src, t, F, e / F, (int)(e % F))));
    }
  return acc;
}

MIX_HD double fm_energy(const double *partial, int64_t t) {
  double s = 0.0;
  for (int p = 0; p < FM_PARTS; ++p) s = MIX_DADD(s, partial[t * FM_PARTS + p]);
  return s;
}

MIX_HD bool fm_has_snr(const b200feat_featmix_track &t) { return t.snr_factor == t.snr_factor; }

// gain[t] of every track of a MIX cut (the first track's as log g under the log law); COPY cuts leave 1.  The first track
// takes _scale_features_for_snr's rejections (E <= 0 keeps 1, so a NaN energy scales by NaN), later tracks FeatureMixer's
// acceptance (E > 0 scales, so a NaN energy keeps 1)
MIX_HD void fm_gains(const b200feat_featmix_cut &cu, const b200feat_featmix_track *tracks, const double *partial, double *gain) {
  const int64_t t0 = cu.first_track;
  const double e_ref = cu.mode == B200FEAT_FEATMIX_MIX ? fm_energy(partial, t0 + cu.ref_track) : 0.0;
  for (int k = 0; k < cu.num_tracks; ++k) {
    const b200feat_featmix_track &t = tracks[t0 + k];
    double g = 1.0;
    if (cu.mode == B200FEAT_FEATMIX_MIX && (t.flags & B200FEAT_FEATMIX_MIXED) && fm_has_snr(t) && (k > 0 || cu.ref_track != 0)) {
      const double e = fm_energy(partial, t0 + k);
      const bool scale = k == 0 ? !(e_ref <= 0.0) && !(e <= 0.0) : e_ref > 0.0 && e > 0.0;
      if (scale) g = MIX_DDIV(MIX_DMUL(e_ref, t.snr_factor), e);
    }
    gain[t0 + k] = (k == 0 && cu.law == B200FEAT_FEATMIX_LOG) ? FM_DLOG(g) : g;
  }
}

// output element (r, c) of a cut
MIX_HD float fm_output(const float *src, const b200feat_featmix_track *tracks, const b200feat_featmix_cut &cu, const double *gain,
                       int F, int64_t r, int c, float pad_value) {
  if (r >= cu.num_rows) return pad_value;
  const int64_t t0 = cu.first_track;
  const b200feat_featmix_track &b = tracks[t0];
  if (cu.mode == B200FEAT_FEATMIX_COPY) return r < b.num_rows ? fm_track_x(src, b, F, r, c) : cu.pad_value;
  const bool log_law = cu.law == B200FEAT_FEATMIX_LOG;
  const int64_t m = r < cu.mix_rows ? r : (int64_t)cu.mix_rows - 1;
  double base = FM_DUMMY;
  if (m < b.num_rows) {
    const double x = (double)fm_track_x(src, b, F, m, c);
    base = log_law ? MIX_DADD(x, gain[t0]) : MIX_DMUL(gain[t0], x);
  }
  double s = log_law ? FM_DEXP(base) : base;
  bool added = false;
  for (int k = 1; k < cu.num_tracks; ++k) {
    const b200feat_featmix_track &t = tracks[t0 + k];
    if (!(t.flags & B200FEAT_FEATMIX_MIXED)) continue;
    added = true;
    const bool inside = m >= t.offset && m < (int64_t)t.offset + t.num_rows;
    const double v = inside ? (double)fm_track_x(src, t, F, m - t.offset, c) : FM_DUMMY;
    if (log_law) {
      const double y = MIX_DADD(s, MIX_DMUL(gain[t0 + k], FM_DEXP(v)));
      s = y < FM_EPSILON ? FM_EPSILON : y;  // np.maximum: a NaN stays NaN
    } else {
      s = MIX_DADD(s, MIX_DMUL(gain[t0 + k], v));
    }
  }
  if (!added) return MIX_D2F(base);
  return MIX_D2F(log_law ? FM_DLOG(s) : s);
}

#ifdef __CUDACC__
// grid (ntracks * FM_PARTS): CTA x sums part x % FM_PARTS of track x / FM_PARTS (0 for a track whose energy no cut needs)
__global__ void __launch_bounds__(FM_THREADS) featmix_energy_kernel(const float *__restrict__ src,
                                                                    const b200feat_featmix_track *__restrict__ tracks,
                                                                    const b200feat_featmix_cut *__restrict__ cuts, int F,
                                                                    double *__restrict__ partial) {
  __shared__ double red[FM_THREADS];
  const int64_t t = blockIdx.x / FM_PARTS;
  const int part = blockIdx.x % FM_PARTS;
  const b200feat_featmix_track tr = tracks[t];
  double acc = 0.0;
  if (tr.flags & B200FEAT_FEATMIX_ENERGY) acc = fm_energy_thread(src, tr, cuts[tr.cut].law, F, part, threadIdx.x);
  red[threadIdx.x] = acc;
  __syncthreads();
  for (int w = FM_THREADS / 2; w > 0; w >>= 1) {
    if (threadIdx.x < w) red[threadIdx.x] = __dadd_rn(red[threadIdx.x], red[threadIdx.x + w]);
    __syncthreads();
  }
  if (threadIdx.x == 0) partial[blockIdx.x] = red[0];
}

// one thread per cut
__global__ void __launch_bounds__(FM_GAIN_THREADS) featmix_gain_kernel(const b200feat_featmix_track *__restrict__ tracks,
                                                                       const b200feat_featmix_cut *__restrict__ cuts, int ncuts,
                                                                       const double *__restrict__ partial, double *__restrict__ gain) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c < ncuts) fm_gains(cuts[c], tracks, partial, gain);
}

// grid (tiles, min(cuts, 65535)): CTA (x, y) writes elements [x * FM_TILE, (x + 1) * FM_TILE) of cuts y, y + gridDim.y, ...
// of the (T_max, F) outputs
__global__ void __launch_bounds__(FM_THREADS) featmix_out_kernel(const float *__restrict__ src,
                                                                 const b200feat_featmix_track *__restrict__ tracks,
                                                                 const b200feat_featmix_cut *__restrict__ cuts, int ncuts,
                                                                 const double *__restrict__ gain, int F, int T_max, float pad_value,
                                                                 float *__restrict__ out) {
  const int64_t n = (int64_t)T_max * F;
  const int64_t e1 = min(n, ((int64_t)blockIdx.x + 1) * FM_TILE);
  for (int c = blockIdx.y; c < ncuts; c += gridDim.y) {
    const b200feat_featmix_cut cu = cuts[c];
    float *dst = out + (int64_t)c * n;
    for (int64_t e = (int64_t)blockIdx.x * FM_TILE + threadIdx.x; e < e1; e += FM_THREADS)
      dst[e] = fm_output(src, tracks, cu, gain, F, e / F, (int)(e % F), pad_value);
  }
}
#endif
