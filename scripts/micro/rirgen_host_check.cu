// CPU run of the RIR generator arithmetic of lhotse_b200/csrc/rirgen.cuh: the same entry chain (rg_room, rg_entry with its
// multinomial search and linspace), a stable sort by position, the window walk (rg_window) and the biquad (rg_biquad) the
// kernels use, with every buffer allocated to its exact size so that AddressSanitizer sees any access outside them.  No GPU
// needed; the header also compiles as plain C++:
//   g++ -x c++ -std=c++17 -O1 -g -fsanitize=address -o rirgen_host_check scripts/micro/rirgen_host_check.cu
//   ./rirgen_host_check recs.bin draws.f64 cdf.f32 table.f32 entries.bin out8.f32
//        recs.bin holds b200feat_rir_gen records (cdf_elem / draw_elem into the two buffers; out_elem is ignored), table.f32
//        the 106-tap 8 -> 1 resampler.  Per RIR, entries.bin gets: int64 kept, int32 direct-path position, int32 entries at
//        that position, float direct-path value, then the kept comb (the last entry of every position, in position order):
//        kept int32 positions and kept float values.  out8.f32 gets each RIR's out_len samples at 8 sr after the biquad.
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <numeric>
#include <vector>

#include "../../lhotse_b200/csrc/rirgen.cuh"

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

template <typename T>
static T *exact_copy(const std::vector<T> &v, int64_t a, int64_t n) {
  T *p = (T *)malloc(sizeof(T) * (n > 0 ? n : 1));
  if (n > 0) memcpy(p, v.data() + a, sizeof(T) * n);
  return p;
}

int main(int argc, char **argv) {
  if (argc != 7) {
    fprintf(stderr, "usage: %s recs.bin draws.f64 cdf.f32 table.f32 entries.bin out8.f32\n", argv[0]);
    return 2;
  }
  const std::vector<b200feat_rir_gen> recs = load<b200feat_rir_gen>(argv[1]);
  const std::vector<double> draws = load<double>(argv[2]);
  const std::vector<float> cdf = load<float>(argv[3]);
  const std::vector<float> table = load<float>(argv[4]);
  if (table.size() != RG_TAPS) { fprintf(stderr, "table must hold %d floats\n", RG_TAPS); return 2; }
  FILE *fe = fopen(argv[5], "wb"), *fo = fopen(argv[6], "wb");
  if (!fe || !fo) { fprintf(stderr, "cannot write the outputs\n"); return 2; }
  float *tab = exact_copy(table, 0, RG_TAPS);
  for (const b200feat_rir_gen &r : recs) {
    const int images = 2 * r.sampling_rate;
    double *u = exact_copy(draws, r.draw_elem, images), *pert = exact_copy(draws, r.draw_elem + images, images);
    float *dist = exact_copy(cdf, r.cdf_elem, images);
    float *out = (float *)malloc(sizeof(float) * (size_t)r.out_len);
    RgRir g{u, pert, dist, out, r.t60, r.r, r.d0, r.tau, r.comb_len, r.out_len, 0, 0, r.sampling_rate, images,
            r.b0, r.b1, r.b2, r.a1, r.a2};
    const RgRoom m = rg_room(g);
    const int n = images + 1;
    int32_t *pos = (int32_t *)malloc(sizeof(int32_t) * n);
    float *val = (float *)malloc(sizeof(float) * n);
    for (int i = 0; i < n; ++i) rg_entry(g, m, i, pos + i, val + i);
    // the kernels' stable segmented sort by position
    std::vector<int> order(n);
    std::iota(order.begin(), order.end(), 0);
    std::stable_sort(order.begin(), order.end(), [&](int a, int b) { return pos[a] < pos[b]; });
    int32_t *spos = (int32_t *)malloc(sizeof(int32_t) * n);
    float *sval = (float *)malloc(sizeof(float) * n);
    for (int i = 0; i < n; ++i) { spos[i] = pos[order[i]]; sval[i] = val[order[i]]; }
    std::vector<int32_t> kpos;
    std::vector<float> kval;
    for (int i = 0; i < n; ++i)
      if (i + 1 == n || spos[i + 1] != spos[i]) { kpos.push_back(spos[i]); kval.push_back(sval[i]); }
    const int32_t at_direct = (int32_t)std::count(pos, pos + n, pos[0]);
    const int64_t kept = (int64_t)kpos.size();
    fwrite(&kept, sizeof(kept), 1, fe);
    fwrite(&pos[0], sizeof(int32_t), 1, fe);
    fwrite(&at_direct, sizeof(int32_t), 1, fe);
    fwrite(&val[0], sizeof(float), 1, fe);
    fwrite(kpos.data(), sizeof(int32_t), kpos.size(), fe);
    fwrite(kval.data(), sizeof(float), kval.size(), fe);
    for (int64_t j = 0; j < r.out_len; ++j) out[j] = rg_window(spos, sval, 0, n, tab, j);
    rg_biquad(g);
    fwrite(out, sizeof(float), (size_t)r.out_len, fo);
    free(u); free(pert); free(dist); free(out); free(pos); free(val); free(spos); free(sval);
  }
  free(tab);
  fclose(fe);
  fclose(fo);
  return 0;
}
