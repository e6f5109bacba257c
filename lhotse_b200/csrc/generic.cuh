// Generic fused kernel: any (L, S, N), any window, all four feature kinds.
// One warp owns one frame at a time: gather(reflect) -> DC -> pre-emphasis -> window ->
// mixed-radix Stockham FFT in shared memory (packed-real for even N) -> |X|^2 -> mel -> log
// (-> DCT/lifter).  Replaces the op chain of lhotse/features/kaldi/layers.py:151-186 (Wav2Win),
// :309-320 (rfft), :392-402 / :461-473 / :565-578 / :708-724 (spectrum epilogues) and the
// framing of :727-772, with no HBM intermediates: 4*S bytes read, 4*F bytes written per frame.
#pragma once
#include "common.cuh"

__device__ __forceinline__ float2 cmul(float2 a, float2 b) {
  return make_float2(a.x * b.x - a.y * b.y, a.x * b.y + a.y * b.x);
}

// One Stockham pass of radix R over a length-Nc complex sequence, executed by one warp.
// out[(j / Ns) * Ns * R + (j % Ns) + q * Ns] = sum_r in[j + r * Nc / R] * W^(r * (k*Nc/(Ns*R) + q*Nc/R))
__device__ __forceinline__ void stockham_pass(const float2 *__restrict__ src, float2 *__restrict__ dst,
                                              const float2 *__restrict__ tw, int Nc, int R, int Ns,
                                              int lane) {
  const int nb = Nc / R;
  const int tstep = Nc / (Ns * R);
  // Ns is a power of two for as long as only radix-4/2 passes have run (every pass of a power-of-two plan): j % Ns and
  // j / Ns are then a mask and a shift instead of two ~20-instruction integer divisions per butterfly
  const bool pow2 = (Ns & (Ns - 1)) == 0;
  const int sh = 31 - __clz(Ns), msk = Ns - 1;
  if (R == 4) {
    for (int j = lane; j < nb; j += 32) {
      const int k = pow2 ? (j & msk) : j % Ns;
      float2 v0 = src[j], v1 = src[j + nb], v2 = src[j + 2 * nb], v3 = src[j + 3 * nb];
      if (k != 0) {
        const int ti = k * tstep;
        v1 = cmul(v1, __ldg(tw + ti));
        v2 = cmul(v2, __ldg(tw + 2 * ti));
        v3 = cmul(v3, __ldg(tw + 3 * ti));
      }
      const float2 a = make_float2(v0.x + v2.x, v0.y + v2.y);
      const float2 b = make_float2(v0.x - v2.x, v0.y - v2.y);
      const float2 c = make_float2(v1.x + v3.x, v1.y + v3.y);
      const float2 d = make_float2(v1.y - v3.y, v3.x - v1.x);  // -i * (v1 - v3)
      const int o = (pow2 ? (j >> sh) : j / Ns) * Ns * 4 + k;
      dst[o] = make_float2(a.x + c.x, a.y + c.y);
      dst[o + Ns] = make_float2(b.x + d.x, b.y + d.y);
      dst[o + 2 * Ns] = make_float2(a.x - c.x, a.y - c.y);
      dst[o + 3 * Ns] = make_float2(b.x - d.x, b.y - d.y);
    }
  } else if (R == 2) {
    for (int j = lane; j < nb; j += 32) {
      const int k = pow2 ? (j & msk) : j % Ns;
      float2 v0 = src[j], v1 = src[j + nb];
      if (k != 0) v1 = cmul(v1, __ldg(tw + k * tstep));
      const int o = (pow2 ? (j >> sh) : j / Ns) * Ns * 2 + k;
      dst[o] = make_float2(v0.x + v1.x, v0.y + v1.y);
      dst[o + Ns] = make_float2(v0.x - v1.x, v0.y - v1.y);
    }
  } else {
    // arbitrary (prime) radix: O(R^2) direct DFT with exact table twiddles
    const int qstep = Nc / R;
    for (int j = lane; j < nb; j += 32) {
      const int k = j % Ns;
      const int o = (j / Ns) * Ns * R + k;
      for (int q = 0; q < R; ++q) {
        const int step = (k * tstep + q * qstep) % Nc;
        float2 acc = src[j];
        int ti = 0;
        for (int r = 1; r < R; ++r) {
          ti += step;
          if (ti >= Nc) ti -= Nc;
          const float2 w = __ldg(tw + ti);
          const float2 v = src[j + r * nb];
          acc.x += v.x * w.x - v.y * w.y;
          acc.y += v.x * w.y + v.y * w.x;
        }
        dst[o + q * Ns] = acc;
      }
    }
  }
}

// Per-warp region of the dynamic shared memory, in floats from the warp's base (the host sizes the launch from the same
// function, so the two cannot disagree):
//   raw   [0, bufA)              the frame's L samples, then its K <= N spectrum values
//   bufA  [bufA, bufA + 2 Nc)    the FFT's ping-pong buffers, Nc complex values each
//   bufB  [bufB, bufB + 2 Nc)
//   mlog  [bufA, bufA + M)       the MFCC epilogue's M log-mel values.  Both FFT buffers are dead once the spectrum is in
//                                raw, so mlog reuses them from bufA on, and the region grows past bufB only when M > 4 Nc
//                                (N = 16 with 40 filters, say).  Other features keep no scratch.
// Every region starts on 8 bytes and every warp's base on 16.
struct GenericLayout {
  int bufA, bufB, mlog, floats;
};
__host__ __device__ inline GenericLayout generic_layout(const DevPlan &p) {
  GenericLayout l;
  l.bufA = (p.N + 3) & ~3;
  l.bufB = l.bufA + 2 * p.Nc;
  l.mlog = l.bufA;
  const int scratch = p.feature == B200FEAT_MFCC ? (p.M + 3) & ~3 : 0;
  l.floats = l.bufA + (4 * p.Nc > scratch ? 4 * p.Nc : scratch);
  return l;
}

// The opt-in limit of dynamic shared memory per CTA on sm_90
#define GENERIC_SMEM_OPTIN_MAX (227 * 1024)

// Launch shape: as many warps per CTA as fit ~100 KB, at least 1 and at most 8.  False if one warp's region is over the
// opt-in limit: N > 16384 for even N, N > 11621 for odd N (20 N bytes per warp).
inline bool generic_launch_shape(const DevPlan &p, int *warps, size_t *smem) {
  const size_t per_warp = (size_t)generic_layout(p).floats * sizeof(float);
  int w = (int)((100 * 1024) / per_warp);
  if (w > 8) w = 8;
  if (w < 1) w = 1;
  *warps = w;
  *smem = per_warp * w;
  return *smem <= GENERIC_SMEM_OPTIN_MAX;
}

template <int DT>
__global__ void __launch_bounds__(256) b200feat_generic_kernel(const DevPlan p, const DevBatch b) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int lane = threadIdx.x & 31;
  const int warp = threadIdx.x >> 5;
  const int nwarps = blockDim.x >> 5;
  const GenericLayout lay = generic_layout(p);
  float *raw = reinterpret_cast<float *>(smem_raw) + (size_t)warp * lay.floats;
  float2 *bufA = reinterpret_cast<float2 *>(raw + lay.bufA);
  float2 *bufB = reinterpret_cast<float2 *>(raw + lay.bufB);
  float *mlog = raw + lay.mlog;

  // generic kernel: one tile == one output row
  for (int64_t g = (int64_t)blockIdx.x * nwarps + warp; g < b.num_tiles; g += (int64_t)gridDim.x * nwarps) {
    const int64_t tile = b.tile_base + g;
    int cut;
    int64_t t, out_row;
    if (b.out_mode == B200FEAT_OUT_PADDED) {
      cut = (int)(g / b.max_frames);
      t = g - (int64_t)cut * b.max_frames;
      out_row = (int64_t)(b.batch_first + cut) * b.max_frames + t;
    } else {
      cut = find_segment(b.row_off, b.B, tile);
      t = tile - __ldg(b.row_off + cut);
      out_row = tile;
    }
    float *out = b.out + out_row * p.F;
    const int64_t T = __ldg(b.row_off + cut + 1) - __ldg(b.row_off + cut);
    if (t >= T) {  // padded tail
      for (int c = lane; c < p.F; c += 32) out[c] = post_affine(p, c, b.pad_value);
      continue;
    }
    const int64_t n = __ldg(b.nsamp + cut);
    const int64_t xoff = __ldg(b.samp_off + cut);
    const int64_t base = t * p.S - (p.snip_edges ? 0 : p.pad_left);

    // ---- gather + mean (layers.py:753-772, :155-157)
    float s = 0.f;
    for (int j = lane; j < p.L; j += 32) {
      int64_t i = base + j;
      if (!p.snip_edges) i = reflect_index(i, n, p.pad_mode);
      const float v = ld_sample<DT>(b.samples, xoff + i);
      raw[j] = v;
      s += v;
    }
    s = warp_sum(s);
    const float mu = p.remove_dc ? s / (float)p.L : 0.f;
    __syncwarp();

    // ---- energy, pre-emphasis, window, zero-pad (layers.py:159-181)
    float e = 0.f;
    float *ybuf = reinterpret_cast<float *>(bufA);
    for (int j = lane; j < p.N; j += 32) {
      float y = 0.f;
      if (j < p.L) {
        const float d = raw[j] - mu;
        if (p.raw_energy) e += d * d;
        float g0 = d;
        if (p.preemph != 0.f) {
          const float dp = raw[j > 0 ? j - 1 : 0] - mu;
          g0 = __fsub_rn(d, __fmul_rn(p.preemph, dp));
        }
        y = g0 * __ldg(p.window + j);
        if (!p.raw_energy) e += y * y;
      }
      if (p.packed) ybuf[j] = y; else bufA[j] = make_float2(y, 0.f);
    }
    float le = 0.f;
    if (p.use_energy) le = log_energy_value(p, warp_sum(e));
    __syncwarp();

    // ---- FFT (layers.py:32-36)
    float2 *src = bufA, *dst = bufB;
    int Ns = 1;
    for (int st = 0; st < p.nstages; ++st) {
      const int R = p.radix[st];
      stockham_pass(src, dst, p.tw, p.Nc, R, Ns, lane);
      __syncwarp();
      float2 *tmp = src; src = dst; dst = tmp;
      Ns *= R;
    }

    // ---- spectrum (layers.py:38-42) into raw[0..K)
    for (int k = lane; k < p.K; k += 32) {
      float xr, xi;
      if (p.packed) {
        const float2 zk = src[k == p.Nc ? 0 : k];
        const float2 zc = src[k == 0 ? 0 : p.Nc - k];  // partner (to be conjugated)
        const float er = zk.x + zc.x, ei = zk.y - zc.y;
        const float orr = zk.x - zc.x, oi = zk.y + zc.y;
        const float2 w = __ldg(p.tws + k);
        const float tr = w.x * orr - w.y * oi, ti = w.x * oi + w.y * orr;
        xr = 0.5f * (er + ti);
        xi = 0.5f * (ei - tr);
      } else {
        const float2 z = src[k];
        xr = z.x; xi = z.y;
      }
      const float pw = xr * xr + xi * xi;
      raw[k] = p.use_mag ? sqrtf(pw) : pw;
    }
    __syncwarp();

    // ---- epilogue
    if (p.feature == B200FEAT_SPECTROGRAM) {
      for (int k = lane; k < p.K; k += 32) out[k] = post_affine(p, k, (k == 0 && p.use_energy) ? le : raw[k]);
    } else if (p.feature == B200FEAT_LOG_SPECTROGRAM) {
      for (int k = lane; k < p.K; k += 32)
        out[k] = post_affine(p, k, (k == 0 && p.use_energy) ? le : log_spec_value(p, raw[k]));
    } else {
      const int shift = mel_shift(p), ecol = energy_col(p);
      float vmax = __int_as_float(0xff800000);  // -inf
      for (int m = lane; m < p.M; m += 32) {
        const int st = __ldg(p.mel_start + m), len = __ldg(p.mel_len + m);
        const float *w = p.mel_w + __ldg(p.mel_woff + m);
        float acc = 0.f;
        for (int i = 0; i < len; ++i) acc += raw[st + i] * __ldg(w + i);
        const float fl = nanmax(acc, p.mel_floor);
        const float v = p.log10_mel ? log10f(fl) : logf(fl);  // whisper_fbank.py:67, librosa_fbank.py:126
        vmax = nanmax(vmax, v);
        if (p.feature == B200FEAT_MFCC) mlog[m] = v; else out[m + shift] = p.whisper ? v : post_affine(p, m + shift, v);
      }
      if (p.whisper) {
        // the cut-wide maximum the normalise pass clamps against (whisper_fbank.py:68); rows past the stft's n / S
        // frames exist only as zero rows (:73-80) and do not take part
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) vmax = nanmax(vmax, __shfl_xor_sync(0xffffffffu, vmax, o));
        if (lane == 0 && t < n / p.S) atomic_max_float(b.cut_max + cut, vmax);
      } else if (p.feature == B200FEAT_FBANK) {
        if (p.use_energy && lane == 0) out[ecol] = post_affine(p, ecol, le);
      } else if (p.feature == B200FEAT_MFCC) {
        __syncwarp();
        for (int c = lane; c < p.C; c += 32) {
          float acc = 0.f;
          for (int m = 0; m < p.M; ++m) acc += mlog[m] * __ldg(p.dct + m * p.C + c);
          if (p.use_lifter) acc *= __ldg(p.lifter + c);
          if (p.use_energy && c == ecol) acc = le;
          out[c] = post_affine(p, c, acc);
        }
      }
    }
    __syncwarp();
  }
}


// Second launch of the whisper-fbank path (whisper_fbank.py:68-80): x -> (max(x, cut_max - 8) + 4) / 4 for the rows the
// stft produced (t < n / S), 0 for the extra row `compute_num_frames_from_samples` asks for; padded rows keep pad_value.
// The log-mel rows x are read from `src` and the result written to b.out at the same offsets: src is b.out itself, or the
// rows the fused kernel wrote elsewhere when the caller keeps them (b200feat_extract_keep_raw, for the backward).
// One warp per output row; reads and writes 4*F bytes per row.
__global__ void __launch_bounds__(256) b200feat_whisper_normalize_kernel(const DevPlan p, const DevBatch b, const float *src,
                                                                         int64_t nrows) {
  const int lane = threadIdx.x & 31;
  const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  const int64_t first_row = __ldg(b.row_off);
  for (int64_t g = warp; g < nrows; g += nwarps) {
    int cut;
    int64_t t, out_row;
    if (b.out_mode == B200FEAT_OUT_PADDED) {
      cut = (int)(g / b.max_frames);
      t = g - (int64_t)cut * b.max_frames;
      out_row = (int64_t)(b.batch_first + cut) * b.max_frames + t;
      if (t >= __ldg(b.row_off + cut + 1) - __ldg(b.row_off + cut)) continue;  // pad row: already pad_value
    } else {
      out_row = first_row + g;
      cut = find_segment(b.row_off, b.B, out_row);
      t = out_row - __ldg(b.row_off + cut);
    }
    float *o = b.out + out_row * p.F;
    const float *x = src + out_row * p.F;
    if (t >= __ldg(b.nsamp + cut) / p.S) {
      for (int c = lane; c < p.F; c += 32) o[c] = 0.f;
    } else {
      const float thr = b.cut_max[cut] - 8.0f;
      for (int c = lane; c < p.F; c += 32) o[c] = (nanmax(x[c], thr) + 4.0f) * 0.25f;
    }
  }
}


// The same pass for the tiled kernels (fast400): one CTA per tile of `ft` consecutive rows of one cut, located through the
// host-built tile -> cut table exactly as the fused kernel does (no per-row search), rows processed as one contiguous run of
// 128-bit accesses.
__global__ void __launch_bounds__(256) b200feat_whisper_normalize_tiled_kernel(const DevPlan p, const DevBatch b, const float *src,
                                                                               int ft) {
  for (int64_t tg = blockIdx.x; tg < b.num_tiles; tg += gridDim.x) {
    const int64_t tile = b.tile_base + tg;
    const int cut = __ldg(b.tile_cut + tile) - b.batch_first;
    const int64_t t0 = (tile - __ldg(b.tile_off + cut)) * ft;
    const int64_t T = __ldg(b.row_off + cut + 1) - __ldg(b.row_off + cut);
    const int64_t rows = min((int64_t)ft, T - t0);  // rows past T (padded mode) keep pad_value
    if (rows <= 0) continue;
    const int64_t row0 = b.out_mode == B200FEAT_OUT_PADDED ? (int64_t)(b.batch_first + cut) * b.max_frames + t0
                                                           : __ldg(b.row_off + cut) + t0;
    const int total = (int)rows * p.F;
    const int live = (int)max((int64_t)0, min(rows, __ldg(b.nsamp + cut) / p.S - t0)) * p.F;  // floats of stft rows
    const float thr = b.cut_max[cut] - 8.0f;
    float *o = b.out + row0 * p.F;
    const float *x = src + row0 * p.F;
    if (((row0 * p.F) & 3) == 0 && (p.F & 3) == 0) {
      float4 *o4 = reinterpret_cast<float4 *>(o);
      const float4 *x4 = reinterpret_cast<const float4 *>(x);
      for (int i = threadIdx.x; 4 * i < total; i += blockDim.x) {
        float4 v = x4[i];
        const bool on = 4 * i < live;  // F is a multiple of 4: a float4 never straddles the live / zero boundary
        v.x = on ? (nanmax(v.x, thr) + 4.0f) * 0.25f : 0.f;
        v.y = on ? (nanmax(v.y, thr) + 4.0f) * 0.25f : 0.f;
        v.z = on ? (nanmax(v.z, thr) + 4.0f) * 0.25f : 0.f;
        v.w = on ? (nanmax(v.w, thr) + 4.0f) * 0.25f : 0.f;
        o4[i] = v;
      }
    } else {
      for (int i = threadIdx.x; i < total; i += blockDim.x) o[i] = i < live ? (nanmax(x[i], thr) + 4.0f) * 0.25f : 0.f;
    }
  }
}
