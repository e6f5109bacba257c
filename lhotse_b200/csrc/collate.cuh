// Right-padding collation of a ragged audio buffer into lhotse's (B, T) waveform batch (collate_audio / AudioSamples) on the
// GPU: row b of the float32 output is cut b's samples, widened from int16 exactly as the feature kernels widen them (q / 32768,
// bit-identical to the float route), and then zeros up to T.  The contract is DESIGN.md §3.1o.
//
// Plan of a row.  The output is written once, zeros included (the caller allocates it with torch.empty, no memset pass), with
// 16-byte stores where the row allows them.  Row b starts at element b * T of the output, which is in general not on a 16-byte
// boundary, so each row is split into units:
//   unit 0              the head: the h = (4 - (base + b * T) % 4) % 4 elements (at most T) before the row's first 16-byte
//                       boundary, base the output pointer's 4-byte word index; scalar stores
//   units 1 .. nv       the body: nv = (T - h) / 4 aligned float4 stores
//   unit nv + 1         the tail: the (T - h) % 4 elements left; scalar stores
// The source is read with one vector load where the unit's first source element is on a 4-sample boundary (the row's source
// offset and h are both multiples of 4) and the unit is inside the cut, else with scalar loads.  Every index is 64-bit: B * T
// and the source offsets may pass 2^31.
//
// The per-unit and per-element index math is __host__ __device__ with no intrinsics, so that scripts/micro/collate_host_check.cu
// runs exactly this code on the CPU.  Kernel at the end.
#pragma once
#include <stdint.h>

#ifdef __CUDACC__
#define CO_HD __host__ __device__ __forceinline__
#else
#define CO_HD inline
#endif

#define CO_THREADS 256
#define CO_UNITS_PER_THREAD 4  // units of a row one thread writes per CTA (grid x covers a row in CTAs of this many units each)

// one unit of a row: `n` elements from row element `j`; `vec`: one aligned float4 store
struct CoUnit {
  int64_t j;
  int n;
  bool vec;
};

// elements before row b's first 16-byte boundary (at most T); `base_mod4` is the output pointer's 4-byte word index mod 4
CO_HD int co_head(int base_mod4, int64_t b, int64_t T) {
  const int64_t h = (4 - (int64_t)((base_mod4 + (b % 4) * (T % 4)) % 4)) % 4;
  return (int)(h < T ? h : T);
}

// aligned float4 stores of a row with head h
CO_HD int64_t co_vectors(int h, int64_t T) { return (T - h) / 4; }

// units of a row: head, body, tail (the head and tail units may hold no element)
CO_HD int64_t co_units(int64_t nv) { return nv + 2; }

CO_HD CoUnit co_unit(int64_t k, int h, int64_t nv, int64_t T) {
  CoUnit u;
  if (k == 0) {
    u.j = 0, u.n = h, u.vec = false;
  } else if (k <= nv) {
    u.j = h + 4 * (k - 1), u.n = 4, u.vec = true;
  } else {
    u.j = h + 4 * nv, u.n = (int)(T - h - 4 * nv), u.vec = false;
  }
  return u;
}

// row element j of a cut of `len` samples at source element `off`: the widened sample, or 0 past the cut
CO_HD float co_sample_f32(const float *src, int64_t off, int64_t len, int64_t j) { return j < len ? src[off + j] : 0.0f; }
CO_HD float co_sample_i16(const int16_t *src, int64_t off, int64_t len, int64_t j) {
  return j < len ? (float)src[off + j] * (1.0f / 32768.0f) : 0.0f;
}

// whether a unit reads its four samples with one vector load: a body unit wholly inside the cut, starting on a 4-sample boundary
CO_HD bool co_vector_load(const CoUnit &u, int64_t off, int64_t len) { return u.vec && u.j + 4 <= len && ((off + u.j) & 3) == 0; }

#ifdef __CUDACC__
template <typename S>
__device__ __forceinline__ float co_sample(const S *src, int64_t off, int64_t len, int64_t j);
template <>
__device__ __forceinline__ float co_sample<float>(const float *src, int64_t off, int64_t len, int64_t j) {
  return co_sample_f32(src, off, len, j);
}
template <>
__device__ __forceinline__ float co_sample<int16_t>(const int16_t *src, int64_t off, int64_t len, int64_t j) {
  return co_sample_i16(src, off, len, j);
}

__device__ __forceinline__ float4 co_load4(const float *p) { return __ldg(reinterpret_cast<const float4 *>(p)); }
__device__ __forceinline__ float4 co_load4(const int16_t *p) {
  const short4 q = __ldg(reinterpret_cast<const short4 *>(p));
  const float k = 1.0f / 32768.0f;
  return make_float4((float)q.x * k, (float)q.y * k, (float)q.z * k, (float)q.w * k);
}

// grid (ceil(max units / (CO_THREADS * CO_UNITS_PER_THREAD)), min(B, 65535)): CTA (x, y) writes units
// [x * CO_THREADS * CO_UNITS_PER_THREAD, (x + 1) * ...) of rows y, y + gridDim.y, ...  `cut_tab` holds the B source offsets,
// then the B lengths.  The source must be 16-byte aligned for float32 and 8-byte aligned for int16 (the host checks).
template <typename S>
__global__ void __launch_bounds__(CO_THREADS) collate_audio_kernel(const S *__restrict__ src, const int64_t *__restrict__ cut_tab,
                                                                   int32_t B, int64_t T, int base_mod4, float *__restrict__ out) {
  const int64_t k0 = (int64_t)blockIdx.x * (CO_THREADS * CO_UNITS_PER_THREAD) + threadIdx.x;
  for (int64_t b = blockIdx.y; b < B; b += gridDim.y) {
    const int64_t off = cut_tab[b], len = cut_tab[B + b];
    const int h = co_head(base_mod4, b, T);
    const int64_t nv = co_vectors(h, T), units = co_units(nv);
    float *row = out + b * T;
#pragma unroll
    for (int i = 0; i < CO_UNITS_PER_THREAD; ++i) {
      const int64_t k = k0 + (int64_t)i * CO_THREADS;
      if (k >= units) break;
      const CoUnit u = co_unit(k, h, nv, T);
      if (u.vec) {
        float4 v;
        if (co_vector_load(u, off, len)) {
          v = co_load4(src + off + u.j);
        } else {
          v = make_float4(co_sample<S>(src, off, len, u.j), co_sample<S>(src, off, len, u.j + 1),
                          co_sample<S>(src, off, len, u.j + 2), co_sample<S>(src, off, len, u.j + 3));
        }
        *reinterpret_cast<float4 *>(row + u.j) = v;
      } else {
        for (int e = 0; e < u.n; ++e) row[u.j + e] = co_sample<S>(src, off, len, u.j + e);
      }
    }
  }
}
#endif
