// CPU run of the SpecAugment arithmetic of lhotse_b200/csrc/specaug.cuh: the same per-unit warp-or-copy, partial sums, mean
// and rectangle fill the kernels use, CTA by CTA and thread by thread, with the input and the output allocated to their exact
// sizes so that AddressSanitizer sees any access outside them.  No GPU needed; the header also compiles as plain C++:
//   g++ -x c++ -std=c++17 -O1 -g -fsanitize=address -o specaug_host_check scripts/micro/specaug_host_check.cu
//   ./specaug_host_check in.f32 warps.bin masks.bin B T F out.f32 [means.f32]
//        b200feat_specaug over a (B, T, F) float32 batch and the b200feat_specaug_warp / b200feat_specaug_mask tables (no
//        argument checks: the tables are expected to be valid).  128-bit units when F % 4 == 0, as the library chooses for
//        16-byte aligned tensors.  means.f32 receives the B mask values.
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <vector>

#include "../../lhotse_b200/csrc/specaug.cuh"

template <typename T>
static std::vector<T> load(const char *path) {
  std::vector<T> v;
  FILE *f = fopen(path, "rb");
  if (!f) { fprintf(stderr, "cannot open %s\n", path); exit(2); }
  fseek(f, 0, SEEK_END);
  const long bytes = ftell(f);
  fseek(f, 0, SEEK_SET);
  v.resize((size_t)bytes / sizeof(T));
  if (!v.empty() && fread(v.data(), sizeof(T), v.size(), f) != v.size()) { fprintf(stderr, "short read %s\n", path); exit(2); }
  fclose(f);
  return v;
}

// one CTA of the warp kernel: the threads' units in thread order, then the kernel's reduction tree
template <int V>
static double warp_cta(const float *in, float *out, int T, int F, const SaWarp *warps, int wb, int we, int tile) {
  const int R = sa_tile_rows(F), row0 = tile * R, row1 = std::min(row0 + R, T);
  while (wb < we && warps[wb].start + warps[wb].len <= row0) ++wb;
  while (we > wb && warps[we - 1].start >= row1) --we;
  const int units = sa_tile_units(T, F, V, tile);
  double red[SA_THREADS];
  for (int t = 0; t < SA_THREADS; ++t) {
    double acc = 0.0;
    for (int u = t; u < units; u += SA_THREADS) acc = sa_unit<V>(in, out, F, warps, wb, we, row0, u, acc);
    red[t] = acc;
  }
  for (int w = SA_THREADS / 2; w > 0; w >>= 1)
    for (int t = 0; t < w; ++t) red[t] = MIX_DADD(red[t], red[t + w]);
  return red[0];
}

int main(int argc, char **argv) {
  if (argc != 8 && argc != 9) {
    fprintf(stderr, "usage: %s in.f32 warps.bin masks.bin B T F out.f32 [means.f32]\n", argv[0]);
    return 2;
  }
  const std::vector<float> in_v = load<float>(argv[1]);
  std::vector<b200feat_specaug_warp> warps = load<b200feat_specaug_warp>(argv[2]);
  const std::vector<b200feat_specaug_mask> masks = load<b200feat_specaug_mask>(argv[3]);
  const int B = atoi(argv[4]), T = atoi(argv[5]), F = atoi(argv[6]);
  const size_t n = (size_t)B * T * F;
  if (in_v.size() != n) { fprintf(stderr, "in.f32 is not B * T * F floats\n"); return 2; }
  float *in = (float *)malloc(sizeof(float) * n), *out = (float *)malloc(sizeof(float) * n);
  memcpy(in, in_v.data(), sizeof(float) * n);
  // the kernels' segment table: per sequence, sorted by start
  std::stable_sort(warps.begin(), warps.end(), [](const b200feat_specaug_warp &a, const b200feat_specaug_warp &b) {
    return a.seq != b.seq ? a.seq < b.seq : a.start < b.start;
  });
  std::vector<SaWarp> sw(warps.size());
  std::vector<int32_t> begin((size_t)B + 1, 0);
  for (size_t k = 0; k < warps.size(); ++k) {
    sw[k] = SaWarp{warps[k].start, warps[k].len, warps[k].center, warps[k].warped};
    ++begin[warps[k].seq + 1];
  }
  for (int b = 0; b < B; ++b) begin[b + 1] += begin[b];
  const int tiles = sa_tiles(T, F);
  double *partial = (double *)malloc(sizeof(double) * (size_t)B * tiles);
  float *mean = (float *)malloc(sizeof(float) * B);
  for (int b = 0; b < B; ++b)
    for (int tile = 0; tile < tiles; ++tile) {
      const float *src = in + (size_t)b * T * F;
      float *dst = out + (size_t)b * T * F;
      partial[(size_t)b * tiles + tile] = F % 4 == 0 ? warp_cta<4>(src, dst, T, F, sw.data(), begin[b], begin[b + 1], tile)
                                                     : warp_cta<1>(src, dst, T, F, sw.data(), begin[b], begin[b + 1], tile);
    }
  for (int b = 0; b < B; ++b) mean[b] = sa_mean(partial + (size_t)b * tiles, tiles, (int64_t)T * F);
  for (const b200feat_specaug_mask &pm : masks) {
    const SaMask m{pm.seq, pm.axis, pm.start, pm.end};
    float *dst = out + (size_t)m.seq * T * F;
    for (int i = 0; i < sa_mask_elems(m, T, F); ++i) dst[sa_mask_offset(m, F, i)] = mean[m.seq];
  }
  FILE *fo = fopen(argv[7], "wb");
  if (!fo || fwrite(out, sizeof(float), n, fo) != n) { fprintf(stderr, "cannot write %s\n", argv[7]); return 2; }
  fclose(fo);
  if (argc == 9) {
    FILE *fm = fopen(argv[8], "wb");
    if (!fm || fwrite(mean, sizeof(float), (size_t)B, fm) != (size_t)B) { fprintf(stderr, "cannot write %s\n", argv[8]); return 2; }
    fclose(fm);
  }
  free(in); free(out); free(partial); free(mean);
  printf("specaug: %d x %d x %d, %zu warps, %zu masks, %d ctas\n", B, T, F, warps.size(), masks.size(), B * tiles);
  return 0;
}
