// Audio-domain mixing of mono tracks (lhotse MixedCut.load_audio) on the GPU, bit-identical to lhotse under NumPy >= 2.  A
// track is int16 (x = q / 32768, sources 0 and 1) or float32 (x as it is, source 2: a perturbed track the resample kernel
// wrote into a track buffer).
//
// The arithmetic contract is DESIGN.md §3.1h.  In short, per cut:
//   energy   E = f32(S / n), S the float32 pairwise sum of f32(x)^2 in NumPy's order: n < 8 a sequential sum,
//            n <= 128 eight strided accumulators combined ((r0+r1)+(r2+r3))+((r4+r5)+(r6+r7)) then the tail, otherwise a split
//            at n2 = n/2 - (n/2 mod 8) and the two halves recursively.  The tree depends on n only.
//   gains    g = sqrt(E_ref * factor / E_track) in double (factor = 10 ** (-snr / 10), evaluated by the host); a further
//            track is added as f32(f32(g) * x), an SNR-scaled first track as f64(x) * g and then the whole mix is float64.
//   mix      a zero buffer of the mix's dtype, the tracks added in track order, then trimmed or reflect-padded to the cut.
//
// The per-element and per-leaf arithmetic is __host__ __device__ with explicitly rounded operations (no contraction into an
// FMA on either side), so that scripts/micro/mix_host_check.cu runs exactly this code on the CPU.  Kernels at the end.
#pragma once
#include <math.h>
#include <stdint.h>

#include "../../include/b200feat.h"

#ifdef __CUDACC__
#define MIX_HD __host__ __device__ __forceinline__
#else
#define MIX_HD inline
#endif

#if defined(__CUDA_ARCH__)
#define MIX_FMUL(a, b) __fmul_rn(a, b)
#define MIX_FADD(a, b) __fadd_rn(a, b)
#define MIX_FDIV(a, b) __fdiv_rn(a, b)
#define MIX_DMUL(a, b) __dmul_rn(a, b)
#define MIX_DADD(a, b) __dadd_rn(a, b)
#define MIX_DDIV(a, b) __ddiv_rn(a, b)
#define MIX_DSQRT(a) __dsqrt_rn(a)
#define MIX_D2F(a) __double2float_rn(a)
#else
// the host harness: volatile stores keep every operation a separately rounded IEEE one whatever -ffp-contract says
MIX_HD float mix_fmul_h(float a, float b) { volatile float r = a * b; return r; }
MIX_HD float mix_fadd_h(float a, float b) { volatile float r = a + b; return r; }
MIX_HD float mix_fdiv_h(float a, float b) { volatile float r = a / b; return r; }
MIX_HD double mix_dmul_h(double a, double b) { volatile double r = a * b; return r; }
MIX_HD double mix_dadd_h(double a, double b) { volatile double r = a + b; return r; }
MIX_HD double mix_ddiv_h(double a, double b) { volatile double r = a / b; return r; }
#define MIX_FMUL(a, b) mix_fmul_h(a, b)
#define MIX_FADD(a, b) mix_fadd_h(a, b)
#define MIX_FDIV(a, b) mix_fdiv_h(a, b)
#define MIX_DMUL(a, b) mix_dmul_h(a, b)
#define MIX_DADD(a, b) mix_dadd_h(a, b)
#define MIX_DDIV(a, b) mix_ddiv_h(a, b)
#define MIX_DSQRT(a) sqrt(a)
#define MIX_D2F(a) ((float)(a))
#endif

#define MIX_LEAF 128       // NumPy's PW_BLOCKSIZE
#define MIX_TOP_DEPTH 5    // one warp: lane l evaluates the subtree at depth 5 whose index is l
#define MIX_STACK 40       // the pairwise tree of n <= 2^40 samples (b200feat_mix checks) is at most 35 deep

// x = q / 32768 exactly as B200FEAT_I16 widens a sample; a float32 track sample (B200FEAT_MIX_SRC_F32) is x itself
MIX_HD float mix_widen(int16_t q) { return (float)q * (1.0f / 32768.0f); }
MIX_HD float mix_widen(float x) { return x; }

template <typename T>
MIX_HD float mix_sq(T q) {
  const float x = mix_widen(q);
  return MIX_FMUL(x, x);
}

// where NumPy splits a block of n > MIX_LEAF elements
MIX_HD int64_t mix_split(int64_t n) {
  int64_t n2 = n / 2;
  return n2 - n2 % 8;
}

// NumPy's pairwise_sum leaf (n <= 128) over the squares of q[0, n)
template <typename T>
MIX_HD float mix_leaf(const T *q, int64_t n) {
  if (n < 8) {
    float r = 0.0f;
    for (int64_t i = 0; i < n; ++i) r = MIX_FADD(r, mix_sq(q[i]));
    return r;
  }
  float r[8];
  for (int j = 0; j < 8; ++j) r[j] = mix_sq(q[j]);
  int64_t i = 8;
  for (; i < n - (n % 8); i += 8)
    for (int j = 0; j < 8; ++j) r[j] = MIX_FADD(r[j], mix_sq(q[i + j]));
  float res = MIX_FADD(MIX_FADD(MIX_FADD(r[0], r[1]), MIX_FADD(r[2], r[3])), MIX_FADD(MIX_FADD(r[4], r[5]), MIX_FADD(r[6], r[7])));
  for (; i < n; ++i) res = MIX_FADD(res, mix_sq(q[i]));
  return res;
}

// the pairwise sum of the squares of q[0, n), in NumPy's order, without recursion: a post-order walk with an explicit stack
// of the open nodes' lengths and left-half sums; bit k of `right` says the walk is in the right half of open node k
template <typename T>
MIX_HD float mix_pairwise(const T *q, int64_t n) {
  int64_t len[MIX_STACK];
  float left[MIX_STACK];
  uint64_t right = 0;
  int64_t s = 0;  // start of the current node
  int sp = 0;
  len[0] = n;
  for (;;) {
    if (len[sp] > MIX_LEAF) {  // descend into the left half
      len[sp + 1] = mix_split(len[sp]);
      right &= ~(1ull << sp);
      ++sp;
      continue;
    }
    float v = mix_leaf(q + s, len[sp]);
    for (;;) {  // hand v to the parent
      if (sp == 0) return v;
      --sp;
      const int64_t n2 = mix_split(len[sp]);
      if (!((right >> sp) & 1)) {  // the left half is done: the right half next
        left[sp] = v;
        right |= 1ull << sp;
        s += n2;
        len[sp + 1] = len[sp] - n2;
        ++sp;
        break;
      }
      v = MIX_FADD(left[sp], v);
      s -= n2;  // back to the parent's start
    }
  }
}

// The subtree at depth MIX_TOP_DEPTH with index `lane` (bits read MSB first: 0 = left half): its [start, start + len), or
// false when a leaf above that depth covers it and `lane` is not that leaf's leftmost descendant (the leftmost one
// evaluates the leaf, the others hold nothing).
MIX_HD bool mix_top_node(int64_t n, int lane, int64_t *start, int64_t *len) {
  int64_t s = 0, m = n;
  for (int k = 0; k < MIX_TOP_DEPTH; ++k) {
    if (m <= MIX_LEAF) {
      const int rest = lane & ((1 << (MIX_TOP_DEPTH - k)) - 1);
      if (rest) return false;
      break;
    }
    const int64_t n2 = mix_split(m);
    if ((lane >> (MIX_TOP_DEPTH - 1 - k)) & 1) { s += n2; m -= n2; } else { m = n2; }
  }
  *start = s; *len = m;
  return true;
}

// Combines the value of subtree `lane` (at depth MIX_TOP_DEPTH - k) with its sibling's into their parent's: both present =
// the sum (a single addition, so the order of its operands does not matter), one present = its value.
MIX_HD void mix_combine(float *v, bool *present, float other, bool other_present) {
  if (*present && other_present) *v = MIX_FADD(*v, other);
  else if (other_present) { *v = other; *present = true; }
}

// audio_energy = float(np.average(x ** 2)): the float32 mean, rounded once, widened to double
MIX_HD double mix_energy_of_sum(float s, int64_t n) { return n > 0 ? (double)MIX_FDIV(s, (float)n) : 0.0; }

// The whole energy on one thread in the same tree as the warp (the host harness; the kernel splits it over 32 lanes)
template <typename T>
MIX_HD double mix_energy(const T *q, int64_t n) {
  float v[1 << MIX_TOP_DEPTH];
  bool p[1 << MIX_TOP_DEPTH];
  for (int l = 0; l < (1 << MIX_TOP_DEPTH); ++l) {
    int64_t s, m;
    p[l] = mix_top_node(n, l, &s, &m);
    v[l] = p[l] ? mix_pairwise(q + s, m) : 0.0f;
  }
  for (int k = 0; k < MIX_TOP_DEPTH; ++k) {
    const int bit = 1 << k;
    for (int l = 0; l < (1 << MIX_TOP_DEPTH); ++l) {
      if (l & bit) continue;
      float a = v[l];
      bool pa = p[l];
      mix_combine(&a, &pa, v[l | bit], p[l | bit]);
      v[l] = v[l | bit] = a;
      p[l] = p[l | bit] = pa;
    }
  }
  return mix_energy_of_sum(v[0], n);
}

// The gain of a track whose SNR factor is `factor` (NaN: no SNR) against the reference energy, as add_to_mix /
// _scale_audio_for_snr decide it: 0 = no scaling (the track is added as it is), else sqrt(E_ref * factor / E_track).
MIX_HD double mix_gain(double e_ref, double factor, double e_track) {
  if (factor != factor || !(e_ref > 0.0) || !(e_track > 0.0)) return 0.0;
  return MIX_DSQRT(MIX_DDIV(MIX_DMUL(e_ref, factor), e_track));
}

// A further track's sample in a float32 mix: f32(f32(g) * x); gain32 = 1 for an unscaled track (1 * x = x exactly)
template <typename T>
MIX_HD float mix_added_sample(float gain32, T q) { return MIX_FMUL(gain32, mix_widen(q)); }

// The mix position read for output sample p of a mix of `mix_len` samples: p itself, or np.pad(mode="reflect") past the end
MIX_HD int64_t mix_source_pos(int64_t p, int64_t mix_len) { return p < mix_len ? p : 2 * (mix_len - 1) - p; }

// The gain state of a cut's track t (k = its place in the cut) once the energies are known: f32(g) of a further track (1 when
// it is not scaled), and for the first track the float64 factor of _scale_audio_for_snr in *scale64 (0: the mix is float32).
MIX_HD float mix_track_gain(const b200feat_mix_cut &cut, const b200feat_mix_track &tr, int k, double e_ref, double e_track,
                            double *scale64) {
  const double g = mix_gain(e_ref, tr.snr_factor, e_track);
  if (k == 0) {
    *scale64 = cut.mode == B200FEAT_MIX_SCALED_FIRST ? g : 0.0;
    return 1.0f;
  }
  return g > 0.0 ? MIX_D2F(g) : 1.0f;
}

// Sample x of track `tr` at mix position pos (inside the track): +0 for padding, q / 32768 of an int16 source, the float32
// sample of the track buffer as it is
MIX_HD float mix_track_x(const int16_t *src0, const int16_t *src1, const float *src2, const b200feat_mix_track &tr, int64_t pos) {
  const int64_t i = tr.src_elem + pos - tr.mix_offset;
  if (tr.source == B200FEAT_MIX_SRC_F32) return mix_widen(src2[i]);
  return mix_widen(tr.source < 0 ? (int16_t)0 : (tr.source == 0 ? src0 : src1)[i]);
}

// Output sample p of a cut: the tracks that cover its mix position added in track order to a zero of the mix's dtype,
// returned as float32 (a float64 mix is rounded once here).
MIX_HD float mix_sample(const int16_t *src0, const int16_t *src1, const float *src2, const b200feat_mix_track *tracks,
                        const b200feat_mix_cut &cut, const float *gain32, double scale, int64_t p) {
  const int64_t pos = mix_source_pos(p, cut.mix_len);
  const int64_t t0 = cut.first_track, t1 = cut.first_track + cut.num_tracks;
  if (scale > 0.0) {  // the first track went through _scale_audio_for_snr: a float64 mix
    double m = 0.0;
    for (int64_t t = t0; t < t1; ++t) {
      const b200feat_mix_track &tr = tracks[t];
      if (tr.role != B200FEAT_MIX_ROLE_MIXED || pos < tr.mix_offset || pos >= tr.mix_offset + tr.num_samples) continue;
      const float x = mix_track_x(src0, src1, src2, tr, pos);
      m = MIX_DADD(m, t == t0 ? MIX_DMUL((double)x, scale) : (double)mix_added_sample(gain32[t], x));
    }
    return MIX_D2F(m);
  }
  float m = 0.0f;
  for (int64_t t = t0; t < t1; ++t) {
    const b200feat_mix_track &tr = tracks[t];
    if (tr.role != B200FEAT_MIX_ROLE_MIXED || pos < tr.mix_offset || pos >= tr.mix_offset + tr.num_samples) continue;
    m = MIX_FADD(m, mix_added_sample(gain32[t], mix_track_x(src0, src1, src2, tr, pos)));
  }
  return m;
}

// whether the cut needs track t's energy: its SNR reference, or a track with an SNR
MIX_HD bool mix_needs_energy(const b200feat_mix_cut &cut, const b200feat_mix_track &tr, int64_t t) {
  return t == (int64_t)cut.first_track + cut.ref_track || tr.snr_factor == tr.snr_factor;
}

#ifdef __CUDACC__
#define MIX_THREADS 128
#define MIX_MIX_THREADS 256

// The warp's energy sum of one track: lane `lane` walks its subtree at depth MIX_TOP_DEPTH, the shuffles combine the subtrees
// in NumPy's order; every lane returns the whole sum.
template <typename T>
__device__ __forceinline__ float mix_warp_sum(const T *__restrict__ q, int64_t n, int lane) {
  int64_t s = 0, m = 0;
  bool present = mix_top_node(n, lane, &s, &m);
  float v = present ? mix_pairwise(q + s, m) : 0.0f;
  for (int b = 0; b < MIX_TOP_DEPTH; ++b) {  // siblings differ in bit b of the lane: the tree above depth 5, bottom up
    const float other = __shfl_xor_sync(0xffffffffu, v, 1 << b);
    const bool other_present = __shfl_xor_sync(0xffffffffu, (int)present, 1 << b) != 0;
    mix_combine(&v, &present, other, other_present);
  }
  return v;
}

// One block per cut, one warp per track: the energies the cut needs (its reference, every track with an SNR), then the gains.
__global__ void __launch_bounds__(MIX_THREADS) mix_energy_kernel(const int16_t *__restrict__ src0, const int16_t *__restrict__ src1,
                                                                  const float *__restrict__ src2,
                                                                  const b200feat_mix_track *__restrict__ tracks,
                                                                  const b200feat_mix_cut *__restrict__ cuts, double *__restrict__ energy,
                                                                  float *__restrict__ gain32, double *__restrict__ scale64) {
  const b200feat_mix_cut cut = cuts[blockIdx.x];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int k = warp; k < cut.num_tracks; k += MIX_THREADS / 32) {  // warp-uniform: the shuffles below see all 32 lanes
    const int64_t t = cut.first_track + k;
    const b200feat_mix_track tr = tracks[t];
    if (!mix_needs_energy(cut, tr, t) || tr.source < 0 || tr.num_samples <= 0) {  // padding is zeros: energy 0
      if (lane == 0) energy[t] = 0.0;
      continue;
    }
    const float v = tr.source == B200FEAT_MIX_SRC_F32  // warp-uniform: the source is chosen once per track
                        ? mix_warp_sum(src2 + tr.src_elem, tr.num_samples, lane)
                        : mix_warp_sum((tr.source == 0 ? src0 : src1) + tr.src_elem, tr.num_samples, lane);
    if (lane == 0) energy[t] = mix_energy_of_sum(v, tr.num_samples);
  }
  __syncthreads();
  const double e_ref = energy[cut.first_track + cut.ref_track];
  for (int k = threadIdx.x; k < cut.num_tracks; k += MIX_THREADS) {
    const int64_t t = cut.first_track + k;
    double sc = 0.0;
    gain32[t] = mix_track_gain(cut, tracks[t], k, e_ref, energy[t], &sc);
    if (k == 0) scale64[blockIdx.x] = sc;
  }
}

// grid (x, cuts), a grid-stride loop over each cut's output samples
__global__ void __launch_bounds__(MIX_MIX_THREADS) mix_kernel(const int16_t *__restrict__ src0, const int16_t *__restrict__ src1,
                                                              const float *__restrict__ src2,
                                                              const b200feat_mix_track *__restrict__ tracks,
                                                              const b200feat_mix_cut *__restrict__ cuts,
                                                              const float *__restrict__ gain32, const double *__restrict__ scale64,
                                                              float *__restrict__ out) {
  const b200feat_mix_cut cut = cuts[blockIdx.y];
  const double scale = scale64[blockIdx.y];
  for (int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; p < cut.target_len; p += (int64_t)gridDim.x * blockDim.x)
    out[cut.out_elem + p] = mix_sample(src0, src1, src2, tracks, cut, gain32, scale, p);
}
#endif
