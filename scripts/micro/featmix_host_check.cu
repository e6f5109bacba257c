// CPU run of the feature-mix arithmetic of lhotse_b200/csrc/featmix.cuh: the same per-thread energy sums and CTA reduction
// tree, per-cut gains and per-element output the kernels use, with the source and the output allocated to their exact sizes
// so that AddressSanitizer sees any access outside them.  No GPU needed; the header also compiles as plain C++:
//   g++ -x c++ -std=c++17 -O1 -g -fsanitize=address -o featmix_host_check scripts/micro/featmix_host_check.cu
//   ./featmix_host_check src.f32 tracks.bin cuts.bin F T_max pad_value out.f32
//        b200feat_feature_mix over the float32 rows in src.f32 and the b200feat_featmix_track / b200feat_featmix_cut tables
//        (no argument checks: the tables are expected to be valid); out.f32 receives the (B, T_max, F) batch.
#include <stdio.h>
#include <stdlib.h>

#include <algorithm>
#include <vector>

#include "../../lhotse_b200/csrc/featmix.cuh"

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

int main(int argc, char **argv) {
  if (argc != 8) {
    fprintf(stderr, "usage: %s src.f32 tracks.bin cuts.bin F T_max pad_value out.f32\n", argv[0]);
    return 2;
  }
  const std::vector<float> src_v = load<float>(argv[1]);
  const std::vector<b200feat_featmix_track> tracks = load<b200feat_featmix_track>(argv[2]);
  const std::vector<b200feat_featmix_cut> cuts = load<b200feat_featmix_cut>(argv[3]);
  const int F = atoi(argv[4]), T = atoi(argv[5]);
  const float pad_value = (float)atof(argv[6]);
  // exact-size copies: an access past the rows is a heap overflow under AddressSanitizer
  float *src = new float[src_v.size() > 0 ? src_v.size() : 1];
  std::copy(src_v.begin(), src_v.end(), src);
  const size_t n = cuts.size() * (size_t)T * F;
  float *out = new float[n > 0 ? n : 1];
  std::vector<double> partial(tracks.size() * FM_PARTS), gain(tracks.size());
  for (size_t t = 0; t < tracks.size(); ++t)
    for (int p = 0; p < FM_PARTS; ++p) {  // one energy CTA: the threads in order, then the kernel's tree
      double red[FM_THREADS];
      for (int i = 0; i < FM_THREADS; ++i)
        red[i] = (tracks[t].flags & B200FEAT_FEATMIX_ENERGY) ? fm_energy_thread(src, tracks[t], cuts[tracks[t].cut].law, F, p, i) : 0.0;
      for (int w = FM_THREADS / 2; w > 0; w >>= 1)
        for (int i = 0; i < w; ++i) red[i] = MIX_DADD(red[i], red[i + w]);
      partial[t * FM_PARTS + p] = red[0];
    }
  for (const b200feat_featmix_cut &cu : cuts) fm_gains(cu, tracks.data(), partial.data(), gain.data());
  for (size_t c = 0; c < cuts.size(); ++c)
    for (int64_t e = 0; e < (int64_t)T * F; ++e)
      out[c * (size_t)T * F + e] = fm_output(src, tracks.data(), cuts[c], gain.data(), F, e / F, (int)(e % F), pad_value);
  FILE *f = fopen(argv[7], "wb");
  if (!f || fwrite(out, sizeof(float), n, f) != n) { fprintf(stderr, "cannot write %s\n", argv[7]); return 2; }
  fclose(f);
  delete[] src;
  delete[] out;
  return 0;
}
