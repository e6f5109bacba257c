// FLAC (RFC 9639) decode of 16-bit streams: the host frame index and the per-frame decoder, one thread per frame.
//
// The per-frame decoder and the per-job checks are __host__ __device__ code with no CUDA intrinsics outside FLAC_CLZ64, so that
// scripts/micro/flac_host_check.cu runs exactly this code on the CPU (also under AddressSanitizer) against the oracle, on
// truncated / bit-flipped frames and on job tables.  The kernel at the end is the only device-only part.
//
//   bit reader   a 64-bit MSB-first window refilled byte by byte; bytes at or past the frame's byte_length read as zero, and
//                every loop that could spin on those zeros (unary codes) stops once the reader has passed the end.  The
//                CRC-16 is folded into the refill, so every byte of the frame is loaded once.
//   history      the last 32 samples of the current subframe in a ring indexed (i & 31), and the predictor coefficients,
//                both in caller memory with a stride: shared memory [32][blockDim] on the device (one bank per thread), a
//                plain array on the host — never a run-time-indexed local array.
//   channels     mono and independent channels decode straight into the output window; of a decorrelated pair the first
//                subframe goes to the job's int32 scratch (window samples only) and the second is combined with it there.
#pragma once
#include <stdint.h>
#include <string.h>

#include "../../include/b200feat.h"

#ifdef __CUDACC__
#define FLAC_HD __host__ __device__ __forceinline__
#else
#define FLAC_HD inline
#endif

#if defined(__CUDA_ARCH__)
#define FLAC_CLZ64(x) __clzll((long long)(x))
#else
#define FLAC_CLZ64(x) __builtin_clzll(x)
#endif

#define FLAC_MAX_ORDER 32

FLAC_HD uint32_t flac_crc16_byte(uint32_t crc, uint32_t b) {  // polynomial 0x8005, MSB first (table-free form)
  crc ^= b << 8;
  for (int k = 0; k < 8; ++k) crc = (crc & 0x8000u) ? ((crc << 1) ^ 0x8005u) : (crc << 1);
  return crc & 0xFFFFu;
}

FLAC_HD uint32_t flac_crc8(const uint8_t *p, int n) {  // polynomial 0x07
  uint32_t crc = 0;
  for (int i = 0; i < n; ++i) {
    crc ^= p[i];
    for (int k = 0; k < 8; ++k) crc = (crc & 0x80u) ? ((crc << 1) ^ 0x07u) & 0xFFu : (crc << 1) & 0xFFu;
  }
  return crc;
}

struct FlacHeader {
  int variable, block_size, ch_code, channels, ss_code, length;  // length: header bytes including the CRC-8
  int64_t number;
};

// Parses a frame header from at most `avail` bytes.  Returns 0 or B200FEAT_FLAC_EHEADER (sync, reserved codes, UTF-8 number,
// CRC-8; never reads past `avail`).
FLAC_HD int flac_parse_header(const uint8_t *p, int64_t avail, FlacHeader &h) {
  if (avail < 6 || p[0] != 0xFF || (p[1] & 0xFE) != 0xF8) return B200FEAT_FLAC_EHEADER;
  h.variable = p[1] & 1;
  const int bs = p[2] >> 4, sr = p[2] & 15, ch = p[3] >> 4, ss = (p[3] >> 1) & 7;
  if (bs == 0 || sr == 15 || ch > 10 || ss == 3 || (p[3] & 1)) return B200FEAT_FLAC_EHEADER;
  int pos = 4;
  const uint32_t b0 = p[pos++];
  int more;
  uint64_t v;
  if (b0 < 0x80) { more = 0; v = b0; }
  else if ((b0 & 0xE0) == 0xC0) { more = 1; v = b0 & 0x1F; }
  else if ((b0 & 0xF0) == 0xE0) { more = 2; v = b0 & 0x0F; }
  else if ((b0 & 0xF8) == 0xF0) { more = 3; v = b0 & 0x07; }
  else if ((b0 & 0xFC) == 0xF8) { more = 4; v = b0 & 0x03; }
  else if ((b0 & 0xFE) == 0xFC) { more = 5; v = b0 & 0x01; }
  else if (b0 == 0xFE) { more = 6; v = 0; }
  else return B200FEAT_FLAC_EHEADER;
  if (pos + more + 1 > avail) return B200FEAT_FLAC_EHEADER;
  for (int k = 0; k < more; ++k) {
    const uint32_t c = p[pos++];
    if ((c & 0xC0) != 0x80) return B200FEAT_FLAC_EHEADER;
    v = (v << 6) | (c & 0x3F);
  }
  int block = 0;
  if (bs == 1) block = 192;
  else if (bs <= 5) block = 576 << (bs - 2);
  else if (bs >= 8) block = 256 << (bs - 8);
  const int extra = (bs == 6 ? 1 : bs == 7 ? 2 : 0) + (sr == 12 ? 1 : (sr == 13 || sr == 14) ? 2 : 0);
  if (pos + extra + 1 > avail) return B200FEAT_FLAC_EHEADER;
  if (bs == 6) block = p[pos++] + 1;
  else if (bs == 7) { block = ((int)p[pos] << 8 | p[pos + 1]) + 1; pos += 2; }
  pos += (sr == 12 ? 1 : (sr == 13 || sr == 14) ? 2 : 0);
  if (flac_crc8(p, pos) != p[pos]) return B200FEAT_FLAC_EHEADER;
  h.block_size = block;
  h.ch_code = ch;
  h.channels = ch < 8 ? ch + 1 : 2;
  h.ss_code = ss;
  h.number = (int64_t)v;
  h.length = pos + 1;
  return 0;
}

struct FlacBits {
  const uint8_t *p;
  int32_t n, next, avail, crc_end;  // bytes [0, crc_end) feed the CRC-16
  uint32_t crc;
  uint64_t cache;                   // the next `avail` bits, MSB first; bits below them are zero
  const uint16_t *tab;              // CRC-16 byte table, or nullptr for the table-free form

  FLAC_HD void init(const uint8_t *p_, int32_t n_, int32_t start, const uint16_t *tab_) {
    p = p_; n = n_; next = start; avail = 0; cache = 0; tab = tab_; crc_end = n_ - 2; crc = 0;
    for (int32_t i = 0; i < start && i < crc_end; ++i) crc_byte(p[i]);
  }
  FLAC_HD void crc_byte(uint32_t b) {
    crc = tab ? ((crc << 8) ^ tab[((crc >> 8) ^ b) & 0xFF]) & 0xFFFFu : flac_crc16_byte(crc, b);
  }
  FLAC_HD void refill() {
    while (avail <= 56) {
      uint32_t b = 0;
      if (next < n) {
        b = p[next];
        if (next < crc_end) crc_byte(b);
      }
      cache |= (uint64_t)b << (56 - avail);
      avail += 8;
      ++next;
    }
  }
  FLAC_HD int64_t consumed() const { return (int64_t)next * 8 - avail; }
  FLAC_HD bool over() const { return consumed() > (int64_t)n * 8; }
  FLAC_HD uint32_t get(int k) {  // 0 <= k <= 32
    refill();
    if (k == 0) return 0;
    const uint32_t v = (uint32_t)(cache >> (64 - k));
    cache <<= k;
    avail -= k;
    return v;
  }
  FLAC_HD int32_t get_signed(int k) {  // 1 <= k <= 32, two's complement
    const uint32_t v = get(k);
    return k == 32 ? (int32_t)v : (int32_t)(v << (32 - k)) >> (32 - k);
  }
  // zeros before the next one bit (the one is consumed); false once past the end or above `limit`
  FLAC_HD bool unary(uint32_t &q, uint32_t limit) {
    q = 0;
    for (;;) {
      refill();
      if (cache) {
        const int z = FLAC_CLZ64(cache);
        q += z;
        cache <<= z;
        cache <<= 1;
        avail -= z + 1;
        return q <= limit;
      }
      q += avail;
      cache = 0;
      avail = 0;
      if (over() || q > limit) return false;
    }
  }
  FLAC_HD void align() {
    const int d = avail & 7;
    cache <<= d;
    avail -= d;
  }
  // CRC-16 over the rest of [0, crc_end) (bytes the reader has not loaded), then compared with the frame's last two bytes
  FLAC_HD bool crc_ok() {
    for (int32_t i = next; i < crc_end; ++i) crc_byte(p[i]);
    return n >= 2 && crc == ((uint32_t)p[n - 2] << 8 | p[n - 1]);
  }
};

// Where the samples of one subframe go.
enum { FLAC_SINK_NONE = 0, FLAC_SINK_OUT = 1, FLAC_SINK_SCRATCH = 2, FLAC_SINK_COMBINE = 3 };

struct FlacSink {
  int mode, shift, ch_code, want, skip, count;
  int16_t *out;
  int32_t *scratch;
  // returns 0 or B200FEAT_FLAC_ERANGE
  FLAC_HD int put(int i, int32_t s) const {
    const int w = i - skip;
    if ((unsigned)w >= (unsigned)count) return 0;
    const int32_t v = (int32_t)((uint32_t)s << shift);
    if (mode == FLAC_SINK_SCRATCH) {
      scratch[w] = v;
      return 0;
    }
    int32_t x = v;
    if (mode == FLAC_SINK_COMBINE) {
      const int32_t a = scratch[w], b = v;
      int32_t l, r;
      if (ch_code == 8) { l = a; r = a - b; }            // left / side
      else if (ch_code == 9) { l = a + b; r = b; }       // side / right
      else {                                             // mid / side
        const int32_t m = (int32_t)((uint32_t)a << 1) | (b & 1);
        l = (m + b) >> 1;
        r = (m - b) >> 1;
      }
      x = want == 0 ? l : r;
    }
    if (x < -32768 || x > 32767) return B200FEAT_FLAC_ERANGE;
    out[w] = (int16_t)x;
    return 0;
  }
};

// One subframe: header, warm-up, residual and prediction.  `hist` / `coef` are rings of FLAC_MAX_ORDER entries `stride` apart.
FLAC_HD int flac_subframe(FlacBits &br, int bs, int sbps, const FlacSink &sink_in, int32_t *hist, int32_t *coef, int stride) {
  if (br.get(1)) return B200FEAT_FLAC_ERESERVED;
  const int type = (int)br.get(6);
  FlacSink sink = sink_in;
  sink.shift = 0;
  if (br.get(1)) {  // wasted bits: k - 1 in unary
    uint32_t q;
    if (!br.unary(q, 32)) return br.over() ? B200FEAT_FLAC_ETRUNCATED : B200FEAT_FLAC_ERANGE;
    if ((int)q + 1 >= sbps) return B200FEAT_FLAC_ERANGE;
    sink.shift = (int)q + 1;
    sbps -= sink.shift;
  }
  const bool emit = sink.mode != FLAC_SINK_NONE;
  if (type == 0 || type == 1) {  // CONSTANT / VERBATIM
    int32_t v = br.get_signed(sbps);
    for (int i = 0; i < bs; ++i) {
      if (type == 1 && i) v = br.get_signed(sbps);
      if (emit) {
        const int e = sink.put(i, v);
        if (e) return e;
      }
      if ((i & 1023) == 1023 && br.over()) return B200FEAT_FLAC_ETRUNCATED;
    }
    return br.over() ? B200FEAT_FLAC_ETRUNCATED : 0;
  }
  int order, shift = 0, precision = 0;
  if (type >= 8 && type <= 12) order = type - 8;
  else if (type >= 32) order = type - 31;
  else return B200FEAT_FLAC_ERESERVED;
  if (order > bs) return B200FEAT_FLAC_EPARTITION;
  for (int i = 0; i < order; ++i) {
    const int32_t v = br.get_signed(sbps);
    hist[(i & (FLAC_MAX_ORDER - 1)) * stride] = v;
    if (emit) {
      const int e = sink.put(i, v);
      if (e) return e;
    }
  }
  if (type >= 32) {
    precision = (int)br.get(4) + 1;
    if (precision == 16) return B200FEAT_FLAC_EPRECISION;
    shift = br.get_signed(5);
    if (shift < 0) return B200FEAT_FLAC_ESHIFT;
    for (int j = 0; j < order; ++j) coef[j * stride] = br.get_signed(precision);
  } else {
    // the fixed predictors as coefficients (-1)^j C(order, j + 1): 1 | 2 -1 | 3 -3 1 | 4 -6 4 -1
    int32_t binom = 1;
    for (int j = 0; j < order; ++j) {
      binom = binom * (order - j) / (j + 1);
      coef[j * stride] = (j & 1) ? -binom : binom;
    }
    precision = 4;
  }
  // 32-bit accumulation is exact when |c| < 2^(precision-1), |s| <= 2^(sbps-1) and there are <= 2^ceil(log2 order) terms
  int lg = 0;
  while ((1 << lg) < order) ++lg;
  const bool wide = precision + sbps + lg > 32;
  // residual
  const uint32_t method = br.get(2);
  if (method > 1) return B200FEAT_FLAC_ERESERVED;
  const int pbits = method ? 5 : 4, esc = (1 << pbits) - 1;
  const int porder = (int)br.get(4);
  const int psize = bs >> porder;
  if ((porder && (bs & ((1 << porder) - 1))) || psize < order) return B200FEAT_FLAC_EPARTITION;
  const int64_t lo = -((int64_t)1 << (sbps - 1)), hi = ((int64_t)1 << (sbps - 1)) - 1;
  int i = order;
  for (int part = 0; part < (1 << porder); ++part) {
    const int end = (part + 1) * psize;
    const int param = (int)br.get(pbits);
    const int raw = param == esc ? (int)br.get(5) : -1;
    for (; i < end; ++i) {
      int32_t r;
      if (raw >= 0) {
        r = raw ? br.get_signed(raw) : 0;
      } else {
        uint32_t q;
        if (!br.unary(q, 0xFFFFFFFFu >> param)) return br.over() ? B200FEAT_FLAC_ETRUNCATED : B200FEAT_FLAC_ERANGE;
        const uint32_t u = (q << param) | br.get(param);
        r = (int32_t)(u >> 1) ^ -(int32_t)(u & 1);
      }
      if (!emit) continue;  // another channel's samples: only the bit stream has to be followed
      int64_t pred;
      if (wide) {
        int64_t acc = 0;
        for (int j = 0; j < order; ++j) acc += (int64_t)coef[j * stride] * hist[((i - 1 - j) & (FLAC_MAX_ORDER - 1)) * stride];
        pred = acc >> shift;
      } else {
        int32_t acc = 0;
        for (int j = 0; j < order; ++j) acc += coef[j * stride] * hist[((i - 1 - j) & (FLAC_MAX_ORDER - 1)) * stride];
        pred = (int64_t)(acc >> shift);
      }
      const int64_t s = (int64_t)r + pred;
      if (s < lo || s > hi) return B200FEAT_FLAC_ERANGE;
      hist[(i & (FLAC_MAX_ORDER - 1)) * stride] = (int32_t)s;
      const int e = sink.put(i, (int32_t)s);
      if (e) return e;
    }
    if (br.over()) return B200FEAT_FLAC_ETRUNCATED;
  }
  return 0;
}

// Decodes one job.  `p` points at the frame's first byte and holds job.byte_length bytes; `out` at the job's output window
// (job.count int16); `scratch` at job.count int32 or nullptr.  Returns a B200FEAT_FLAC_* status.  A frame whose CRC-16 does
// not hold reports B200FEAT_FLAC_ECRC whatever else went wrong in it (check_crc = false: the parser alone decides).
FLAC_HD int flac_decode_frame(const uint8_t *p, const b200feat_flac_job &job, int16_t *out, int32_t *scratch, int32_t *hist,
                              int32_t *coef, int stride, const uint16_t *crc_tab, bool check_crc) {
  const int bs = job.block_size, n = job.byte_length;
  if (bs < 1 || bs > 65536 || n < 8 || job.channels < 1 || job.channels > 8 || job.want_channel < 0 ||
      job.want_channel >= job.channels || job.skip < 0 || job.count < 0 || job.skip + job.count > bs)
    return B200FEAT_FLAC_EJOB;
  FlacHeader h;
  if (flac_parse_header(p, n - 2, h) || h.block_size != bs || h.channels != job.channels || h.variable != job.variable_blocking ||
      h.number != job.coded_number || (h.ss_code != 0 && h.ss_code != 4))
    return B200FEAT_FLAC_EHEADER;
  const bool pair = h.ch_code >= 8;
  if (pair && scratch == nullptr && job.count > 0) return B200FEAT_FLAC_EJOB;
  FlacBits br;
  br.init(p, n, h.length, crc_tab);
  int st = 0;
  for (int c = 0; c < h.channels && !st; ++c) {
    FlacSink sink;
    sink.ch_code = h.ch_code; sink.want = job.want_channel; sink.skip = job.skip; sink.count = job.count;
    sink.out = out; sink.scratch = scratch; sink.shift = 0;
    if (!pair) sink.mode = c == job.want_channel ? FLAC_SINK_OUT : FLAC_SINK_NONE;
    else sink.mode = c == 0 ? FLAC_SINK_SCRATCH : FLAC_SINK_COMBINE;
    const bool side = (h.ch_code == 8 && c == 1) || (h.ch_code == 9 && c == 0) || (h.ch_code == 10 && c == 1);
    st = flac_subframe(br, bs, 16 + (side ? 1 : 0), sink, hist, coef, stride);
  }
  if (!st) {
    br.align();
    const int64_t end = br.consumed();
    if (end > (int64_t)(n - 2) * 8) st = B200FEAT_FLAC_ETRUNCATED;
    else if (end < (int64_t)(n - 2) * 8) st = B200FEAT_FLAC_ELENGTH;
  }
  if (check_crc && !br.crc_ok()) return B200FEAT_FLAC_ECRC;
  return st;
}

// One job of a launch: the job's offsets checked against the launch's buffers (`out_elems` int16 of output, `scratch_elems`
// int32 of scratch; a job whose scratch range does not fit gets none), then the frame.  The kernel and the host check both
// run this, so they apply the same checks.
FLAC_HD int flac_decode_job(const uint8_t *bytes, const b200feat_flac_job &job, int16_t *out, int64_t out_elems, int32_t *scratch,
                            int64_t scratch_elems, int32_t *hist, int32_t *coef, int stride, const uint16_t *crc_tab) {
  if (job.src_byte < 0 || job.dst_elem < 0 || job.count < 0 || job.dst_elem + job.count > out_elems) return B200FEAT_FLAC_EJOB;
  int32_t *scr = nullptr;
  if (job.scratch_elem >= 0 && job.scratch_elem + job.count <= scratch_elems) scr = scratch + job.scratch_elem;
  return flac_decode_frame(bytes + job.src_byte, job, out + job.dst_elem, scr, hist, coef, stride, crc_tab, true);
}

// Host frame index (b200feat_flac_index).
inline int64_t flac_index(const uint8_t *f, int64_t nbytes, b200feat_flac_stream *info, b200feat_flac_frame *frames,
                          int64_t capacity) {
  if (!f || nbytes < 42 || !info || info->struct_size != (int32_t)sizeof(b200feat_flac_stream) || capacity < 0 ||
      (capacity > 0 && !frames) || memcmp(f, "fLaC", 4) != 0)
    return B200FEAT_EINVAL;
  int64_t pos = 4;
  bool have_info = false, last = false;
  while (!last) {
    if (pos + 4 > nbytes) return B200FEAT_EINVAL;
    last = f[pos] & 0x80;
    const int type = f[pos] & 0x7F;
    const int64_t len = (int64_t)f[pos + 1] << 16 | (int64_t)f[pos + 2] << 8 | f[pos + 3];
    pos += 4;
    if (pos + len > nbytes || type == 127) return B200FEAT_EINVAL;
    if (type == 0) {
      if (len < 34 || have_info) return B200FEAT_EINVAL;
      const uint8_t *s = f + pos;
      info->min_block_size = s[0] << 8 | s[1];
      info->max_block_size = s[2] << 8 | s[3];
      info->sample_rate = (int32_t)((uint32_t)s[10] << 12 | (uint32_t)s[11] << 4 | s[12] >> 4);
      info->channels = ((s[12] >> 1) & 7) + 1;
      info->bits_per_sample = ((s[12] & 1) << 4 | s[13] >> 4) + 1;
      info->total_samples = (int64_t)(s[13] & 15) << 32 | (int64_t)s[14] << 24 | (int64_t)s[15] << 16 | (int64_t)s[16] << 8 | s[17];
      memcpy(info->md5, s + 18, 16);
      have_info = true;
    } else if (!have_info) {
      return B200FEAT_EINVAL;  // STREAMINFO comes first
    }
    pos += len;
  }
  if (!have_info || info->max_block_size < 16 || info->min_block_size > info->max_block_size) return B200FEAT_EINVAL;
  info->audio_offset = pos;
  info->variable_blocking = 0;
  info->reserved = 0;
  static const int ss_bits[8] = {0, 8, 12, 0, 16, 20, 24, 32};
  int64_t count = 0, expect_number = 0, expect_sample = 0;
  while (pos + 1 < nbytes) {
    const uint8_t *hit = (const uint8_t *)memchr(f + pos, 0xFF, (size_t)(nbytes - pos - 1));
    if (!hit) break;
    const int64_t at = hit - f;
    FlacHeader h;
    if ((f[at + 1] & 0xFE) == 0xF8 && flac_parse_header(f + at, nbytes - at, h) == 0 &&
        (count > 0 ? h.variable == info->variable_blocking : true) &&
        h.number == (h.variable ? expect_sample : expect_number) && h.block_size <= info->max_block_size &&
        h.channels == info->channels && (h.ss_code == 0 || ss_bits[h.ss_code] == info->bits_per_sample)) {
      if (count == 0) info->variable_blocking = h.variable;
      if (count > 0 && count - 1 < capacity) frames[count - 1].byte_length = (int32_t)(at - frames[count - 1].byte_offset);
      if (count < capacity) {
        frames[count].byte_offset = at;
        frames[count].first_sample = expect_sample;
        frames[count].block_size = h.block_size;
        frames[count].byte_length = (int32_t)(nbytes - at);
      }
      ++count;
      ++expect_number;
      expect_sample += h.block_size;
      pos = at + h.length;
    } else {
      pos = at + 1;
    }
  }
  return count;
}

#ifdef __CUDACC__
#define FLAC_THREADS 128

// One thread per job.  Shared memory: the CRC-16 table, and per thread the 32-sample history ring and the coefficients
// ([32][FLAC_THREADS] each: thread t owns column t, so the run-time-indexed taps never leave shared memory).
__global__ void __launch_bounds__(FLAC_THREADS) flac_decode_kernel(const uint8_t *__restrict__ bytes,
                                                                  const b200feat_flac_job *__restrict__ jobs, int njobs,
                                                                  int16_t *__restrict__ out, int64_t out_elems,
                                                                  int32_t *__restrict__ status, int32_t *__restrict__ scratch,
                                                                  int64_t scratch_elems) {
  __shared__ uint16_t tab[256];
  __shared__ int32_t hist[FLAC_MAX_ORDER * FLAC_THREADS];
  __shared__ int32_t coef[FLAC_MAX_ORDER * FLAC_THREADS];
  for (int t = threadIdx.x; t < 256; t += blockDim.x) {
    uint32_t c = (uint32_t)t << 8;
    for (int k = 0; k < 8; ++k) c = (c & 0x8000u) ? ((c << 1) ^ 0x8005u) : (c << 1);
    tab[t] = (uint16_t)(c & 0xFFFFu);
  }
  __syncthreads();
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= njobs) return;
  const b200feat_flac_job job = jobs[j];
  status[j] = flac_decode_job(bytes, job, out, out_elems, scratch, scratch_elems, hist + threadIdx.x, coef + threadIdx.x,
                              FLAC_THREADS, tab);
}
#endif
