/*
 * Plain-C client of include/b200feat.h — the drop-in boundary exercised without Python, torch or any C++ in the caller.
 *
 *   abi_smoke <dir>
 *
 * <dir> holds float32 little-endian files written by the test that drives this program (tests/test_c_abi.py):
 *   window.f32 (L), bank.f32 (K x M row-major), samples.f32 (the cuts back to back), lens.i64 (B cut lengths).
 * Writes <dir>/out.f32 (packed (sum T_i, F) features) and <dir>/rows.i64 (B frame counts).
 * Exit codes: 0 ok; 3 = b200feat_create said B200FEAT_ENODEVICE (no sm_90 GPU: the library has no CPU fallback);
 *             1 = anything else went wrong (message on stderr).
 */
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "b200feat.h"

static void *slurp(const char *dir, const char *name, size_t *bytes) {
  char path[4096];
  snprintf(path, sizeof path, "%s/%s", dir, name);
  FILE *f = fopen(path, "rb");
  if (!f) { fprintf(stderr, "cannot open %s\n", path); exit(1); }
  fseek(f, 0, SEEK_END);
  long n = ftell(f);
  fseek(f, 0, SEEK_SET);
  void *p = malloc(n > 0 ? (size_t)n : 1);
  if (fread(p, 1, (size_t)n, f) != (size_t)n) { fprintf(stderr, "short read on %s\n", path); exit(1); }
  fclose(f);
  *bytes = (size_t)n;
  return p;
}

static void dump(const char *dir, const char *name, const void *p, size_t bytes) {
  char path[4096];
  snprintf(path, sizeof path, "%s/%s", dir, name);
  FILE *f = fopen(path, "wb");
  if (!f || fwrite(p, 1, bytes, f) != bytes) { fprintf(stderr, "cannot write %s\n", path); exit(1); }
  fclose(f);
}

int main(int argc, char **argv) {
  if (argc < 2) { fprintf(stderr, "usage: abi_smoke <dir>\n"); return 1; }
  const char *dir = argv[1];
  if (b200feat_version() != B200FEAT_ABI_VERSION) { fprintf(stderr, "ABI version mismatch\n"); return 1; }

  size_t wb, bb, sb, lb;
  float *window = (float *)slurp(dir, "window.f32", &wb);
  float *bank = (float *)slurp(dir, "bank.f32", &bb);
  float *samples = (float *)slurp(dir, "samples.f32", &sb);
  int64_t *lens = (int64_t *)slurp(dir, "lens.i64", &lb);
  const int32_t B = (int32_t)(lb / sizeof(int64_t));

  /* the headline plan: Fbank-80, 16 kHz, 25 ms / 10 ms, N = 512 (lhotse FbankConfig defaults, extractors.py:24-44) */
  b200feat_plan_desc d;
  memset(&d, 0, sizeof d);
  d.struct_size = (int32_t)sizeof d;
  d.feature = B200FEAT_FBANK;
  d.frame_length = (int32_t)(wb / sizeof(float));
  d.frame_shift = 160;
  d.fft_length = 512;
  d.num_filters = (int32_t)(bb / sizeof(float) / (512 / 2 + 1));
  d.remove_dc_offset = 1;
  d.raw_energy = 1;
  d.energy_style = B200FEAT_ENERGY_LHOTSE;
  d.kernel = B200FEAT_KERNEL_AUTO;
  d.pad_mode = B200FEAT_PAD_KALDI;
  d.preemph_coeff = 0.97f;
  d.energy_floor = 1e-10f;
  d.mel_floor = 1.1920929e-07f;
  d.log_spec_eps = 1e-15f;

  b200feat_handle *h = NULL;
  int rc = b200feat_create(&d, window, bank, NULL, NULL, 0, &h);
  if (rc == B200FEAT_ENODEVICE) {
    fprintf(stderr, "no device: %s\n", b200feat_global_error());
    return 3;
  }
  if (rc != B200FEAT_OK) { fprintf(stderr, "create failed (%d): %s\n", rc, b200feat_global_error()); return 1; }

  const int32_t F = b200feat_feature_dim(h);
  int64_t *rows = (int64_t *)malloc(sizeof(int64_t) * (size_t)B);
  int64_t total = 0;
  for (int32_t i = 0; i < B; ++i) {
    rows[i] = b200feat_num_frames(h, lens[i]);
    if (rows[i] < 0) { fprintf(stderr, "cut %d cannot be framed\n", i); return 1; }
    total += rows[i];
  }
  float *out = (float *)malloc(sizeof(float) * (size_t)total * (size_t)F);
  rc = b200feat_extract_host(h, samples, B200FEAT_F32, lens, B, out, B200FEAT_OUT_PACKED, 0.0f);
  if (rc != B200FEAT_OK) { fprintf(stderr, "extract_host failed (%d): %s\n", rc, b200feat_last_error(h)); return 1; }

  /* error convention: a cut too short to be framed is refused with B200FEAT_ESHORT, nothing is launched */
  int64_t tiny = 10;
  float junk[80];
  if (b200feat_extract_host(h, samples, B200FEAT_F32, &tiny, 1, junk, B200FEAT_OUT_PACKED, 0.0f) != B200FEAT_ESHORT) {
    fprintf(stderr, "expected B200FEAT_ESHORT for a 10-sample cut\n");
    return 1;
  }
  b200feat_stats st;
  if (b200feat_get_stats(h, &st) != B200FEAT_OK || st.cuts != B || st.frames != total) {
    fprintf(stderr, "stats mismatch\n");
    return 1;
  }
  dump(dir, "out.f32", out, sizeof(float) * (size_t)total * (size_t)F);
  dump(dir, "rows.i64", rows, sizeof(int64_t) * (size_t)B);
  printf("abi_smoke: %d cuts, %lld rows x %d, kernel kind %d\n", B, (long long)total, F, b200feat_kernel_kind(h));
  b200feat_destroy(h);
  return 0;
}
