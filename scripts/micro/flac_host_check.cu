// CPU run of the FLAC decoder of lhotse_b200/csrc/flac.cuh: the same flac_index and __host__ __device__ flac_decode_frame the
// library and its kernel use, one frame at a time, every buffer allocated to its exact size so that AddressSanitizer sees any
// access outside a job's byte range or output window.  No GPU needed; the header also compiles as plain C++:
//   g++ -x c++ -std=c++17 -O1 -g -fsanitize=address -o flac_host_check scripts/micro/flac_host_check.cu
//   ./flac_host_check in.flac out.raw        whole-file decode -> interleaved int16 (out.raw); each frame and channel is also
//                                            decoded through a random window [skip, skip + count) and compared
//   ./flac_host_check in.flac - corrupt N    N rounds over every frame: truncated byte ranges and single bit flips must come
//                                            back as a status (with the CRC-16 check), and the parser alone (check off) must
//                                            stay inside the buffers whatever the bits say
//   ./flac_host_check jobs data.bin jobs.bin OUT_ELEMS SCRATCH_ELEMS OUT_FILL SCRATCH_FILL out.bin scratch.bin
//                                            one launch of a b200feat_flac_job table over the bytes of data.bin, as the kernel
//                                            runs it (flac_decode_job): an int16 output of OUT_ELEMS and an int32 scratch of
//                                            SCRATCH_ELEMS, filled with OUT_FILL / SCRATCH_FILL, each exactly sized; each job
//                                            reads an exactly sized copy of its byte range.  Prints one status per job and
//                                            writes both buffers.  A job whose byte range leaves data.bin refuses the table.
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <vector>

#include "../../lhotse_b200/csrc/flac.cuh"

static uint64_t rng = 88172645463325252ull;
static uint32_t rnd() {
  rng ^= rng << 13; rng ^= rng >> 7; rng ^= rng << 17;
  return (uint32_t)(rng >> 11);
}

// decodes `nbytes` of `src` as `job` with exactly sized copies of every buffer; returns the status, fills `got` (job.count)
static int run(const uint8_t *src, int nbytes, b200feat_flac_job job, std::vector<int16_t> &got, bool check_crc) {
  uint8_t *bytes = (uint8_t *)malloc(nbytes > 0 ? nbytes : 1);
  memcpy(bytes, src, nbytes);
  job.byte_length = nbytes;
  int16_t *out = (int16_t *)malloc(sizeof(int16_t) * (job.count > 0 ? job.count : 1));
  int32_t *scratch = job.channels > 1 ? (int32_t *)malloc(sizeof(int32_t) * (job.count > 0 ? job.count : 1)) : nullptr;
  int32_t *hist = (int32_t *)malloc(sizeof(int32_t) * FLAC_MAX_ORDER), *coef = (int32_t *)malloc(sizeof(int32_t) * FLAC_MAX_ORDER);
  const int st = flac_decode_frame(bytes, job, out, scratch, hist, coef, 1, nullptr, check_crc);
  got.assign(out, out + job.count);
  free(bytes); free(out); free(scratch); free(hist); free(coef);
  return st;
}

static bool read_file(const char *path, std::vector<uint8_t> &out) {
  FILE *f = fopen(path, "rb");
  if (!f) return false;
  uint8_t buf[65536];
  size_t k;
  while ((k = fread(buf, 1, sizeof buf, f)) > 0) out.insert(out.end(), buf, buf + k);
  fclose(f);
  return true;
}

static int jobs_main(int argc, char **argv) {
  if (argc != 10) {
    fprintf(stderr, "usage: %s jobs data.bin jobs.bin OUT_ELEMS SCRATCH_ELEMS OUT_FILL SCRATCH_FILL out.bin scratch.bin\n", argv[0]);
    return 2;
  }
  std::vector<uint8_t> data, table;
  if (!read_file(argv[2], data) || !read_file(argv[3], table) || table.size() % sizeof(b200feat_flac_job)) return 2;
  const int64_t out_elems = atoll(argv[4]), scratch_elems = atoll(argv[5]);
  const int16_t out_fill = (int16_t)atoi(argv[6]);
  const int32_t scratch_fill = (int32_t)strtol(argv[7], nullptr, 0);
  const size_t njobs = table.size() / sizeof(b200feat_flac_job);
  std::vector<b200feat_flac_job> jobs(njobs);
  memcpy(jobs.data(), table.data(), table.size());
  int16_t *out = (int16_t *)malloc(sizeof(int16_t) * (out_elems > 0 ? out_elems : 1));
  int32_t *scratch = scratch_elems > 0 ? (int32_t *)malloc(sizeof(int32_t) * scratch_elems) : nullptr;
  for (int64_t i = 0; i < out_elems; ++i) out[i] = out_fill;
  for (int64_t i = 0; i < scratch_elems; ++i) scratch[i] = scratch_fill;
  int32_t *hist = (int32_t *)malloc(sizeof(int32_t) * FLAC_MAX_ORDER), *coef = (int32_t *)malloc(sizeof(int32_t) * FLAC_MAX_ORDER);
  printf("statuses");
  for (size_t j = 0; j < njobs; ++j) {
    b200feat_flac_job job = jobs[j];
    const int64_t len = job.byte_length > 0 ? job.byte_length : 0;
    if (job.src_byte >= 0 && job.src_byte + len > (int64_t)data.size()) {
      fprintf(stderr, "job %zu: bytes [%lld, +%lld) outside the %zu bytes of data\n", j, (long long)job.src_byte,
              (long long)len, data.size());
      return 2;
    }
    uint8_t *bytes = (uint8_t *)malloc(len > 0 ? len : 1);
    if (job.src_byte >= 0) {
      memcpy(bytes, data.data() + job.src_byte, len);
      job.src_byte = 0;
    }
    printf(" %d", flac_decode_job(bytes, job, out, out_elems, scratch, scratch_elems, hist, coef, 1, nullptr));
    free(bytes);
  }
  printf("\n");
  FILE *o = fopen(argv[8], "wb"), *s = fopen(argv[9], "wb");
  if (!o || !s) return 2;
  fwrite(out, sizeof(int16_t), out_elems, o);
  if (scratch_elems > 0) fwrite(scratch, sizeof(int32_t), scratch_elems, s);
  fclose(o);
  fclose(s);
  free(out); free(scratch); free(hist); free(coef);
  return 0;
}

int main(int argc, char **argv) {
  if (argc >= 2 && !strcmp(argv[1], "jobs")) return jobs_main(argc, argv);
  if (argc < 3) {
    fprintf(stderr, "usage: %s in.flac out.raw|- [corrupt N]\n", argv[0]);
    return 2;
  }
  FILE *f = fopen(argv[1], "rb");
  if (!f) return 2;
  std::vector<uint8_t> file;
  uint8_t buf[65536];
  size_t k;
  while ((k = fread(buf, 1, sizeof buf, f)) > 0) file.insert(file.end(), buf, buf + k);
  fclose(f);
  b200feat_flac_stream info;
  info.struct_size = sizeof info;
  const int64_t nf = flac_index(file.data(), (int64_t)file.size(), &info, nullptr, 0);
  if (nf < 0) { printf("index failed %lld\n", (long long)nf); return 1; }
  std::vector<b200feat_flac_frame> frames(nf);
  flac_index(file.data(), (int64_t)file.size(), &info, frames.data(), nf);
  const int C = info.channels;
  auto job_of = [&](const b200feat_flac_frame &fr, int64_t index, int ch) {
    b200feat_flac_job j;
    memset(&j, 0, sizeof j);
    j.byte_length = fr.byte_length; j.block_size = fr.block_size; j.channels = C; j.want_channel = ch;
    j.skip = 0; j.count = fr.block_size; j.variable_blocking = info.variable_blocking;
    j.coded_number = info.variable_blocking ? fr.first_sample : index;
    j.scratch_elem = C > 1 ? 0 : -1;
    return j;
  };
  long bad = 0, checked = 0;
  if (argc >= 5 && !strcmp(argv[3], "corrupt")) {
    const int rounds = atoi(argv[4]);
    long flagged = 0, parser_only = 0;
    std::vector<int16_t> got;
    for (int r = 0; r < rounds; ++r)
      for (int64_t i = 0; i < nf; ++i) {
        const b200feat_flac_frame &fr = frames[i];
        const uint8_t *src = file.data() + fr.byte_offset;
        b200feat_flac_job j = job_of(fr, i, (int)(rnd() % C));
        j.skip = (int)(rnd() % fr.block_size);
        j.count = (int)(rnd() % (fr.block_size - j.skip + 1));
        // truncated: any shorter byte range is an error
        const int cut = (int)(rnd() % fr.byte_length);
        ++checked;
        if (run(src, cut, j, got, true) == 0) { ++bad; printf("truncated frame %lld to %d bytes decoded\n", (long long)i, cut); }
        // one flipped bit: the CRC-16 catches every single-bit error
        std::vector<uint8_t> flip(src, src + fr.byte_length);
        flip[rnd() % fr.byte_length] ^= (uint8_t)(1u << (rnd() % 8));
        ++checked;
        const int st = run(flip.data(), fr.byte_length, j, got, true);
        if (st == 0) { ++bad; printf("bit flip in frame %lld decoded\n", (long long)i); }
        flagged += st != 0;
        // the parser alone on flipped bits, and on a few flipped bytes: any status, no out-of-range access (ASan)
        run(flip.data(), fr.byte_length, j, got, false);
        for (int b = 0; b < 4; ++b) flip[rnd() % fr.byte_length] = (uint8_t)rnd();
        parser_only += run(flip.data(), fr.byte_length, j, got, false) != 0;
        run(flip.data(), (int)(rnd() % fr.byte_length), j, got, false);
      }
    printf("corrupt: %lld frames x %d rounds, %ld flagged flips, %ld parser-only errors, %ld checked, %ld bad\n", (long long)nf,
           rounds, flagged, parser_only, checked, bad);
    return bad ? 1 : 0;
  }
  std::vector<int16_t> pcm;
  int64_t total = 0;
  for (auto &fr : frames) total += fr.block_size;
  pcm.assign((size_t)total * C, 0);
  std::vector<int16_t> got, win;
  for (int64_t i = 0; i < nf; ++i) {
    const b200feat_flac_frame &fr = frames[i];
    for (int ch = 0; ch < C; ++ch) {
      b200feat_flac_job j = job_of(fr, i, ch);
      const int st = run(file.data() + fr.byte_offset, fr.byte_length, j, got, true);
      ++checked;
      if (st) { ++bad; printf("frame %lld channel %d: status %d\n", (long long)i, ch, st); continue; }
      for (int s = 0; s < fr.block_size; ++s) pcm[(size_t)(fr.first_sample + s) * C + ch] = got[s];
      j.skip = (int)(rnd() % fr.block_size);
      j.count = (int)(rnd() % (fr.block_size - j.skip + 1));
      const int st2 = run(file.data() + fr.byte_offset, fr.byte_length, j, win, true);
      ++checked;
      if (st2 || memcmp(win.data(), got.data() + j.skip, sizeof(int16_t) * j.count)) {
        ++bad; printf("frame %lld channel %d window [%d, +%d): status %d or samples differ\n", (long long)i, ch, j.skip, j.count, st2);
      }
    }
  }
  if (strcmp(argv[2], "-")) {
    FILE *o = fopen(argv[2], "wb");
    fwrite(pcm.data(), sizeof(int16_t), pcm.size(), o);
    fclose(o);
  }
  printf("frames %lld, samples %lld, channels %d, %ld checked, %ld bad\n", (long long)nf, (long long)total, C, checked, bad);
  return bad ? 1 : 0;
}
