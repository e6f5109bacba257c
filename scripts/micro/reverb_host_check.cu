// CPU run of the reverberation arithmetic of lhotse_b200/csrc/reverb.cuh: the same twiddle table (rv_twiddle), butterflies,
// partition multiply-accumulate, gain and output the kernels use, CTA by CTA, with every RIR, input and output window
// allocated to its exact size so that AddressSanitizer sees any access outside them.  No GPU needed; the header also
// compiles as plain C++:
//   g++ -x c++ -std=c++17 -O1 -g -fsanitize=address -o reverb_host_check scripts/micro/reverb_host_check.cu
//   ./reverb_host_check src0.i16 rirs.bin cuts.bin in.f32 out.f32
//        b200feat_reverb over the int16 RIR source (every RIR record's source 0), the b200feat_reverb_rir /
//        b200feat_reverb_cut tables and the float32 input buffer (no argument checks: the tables are expected to be valid);
//        each cut's target_len samples are written back to back to out.f32.  The per-CTA partial sums of y^2 are added in
//        thread order here (the kernel uses a shuffle tree), so pa may differ from the device in the last bits.
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <vector>

#include "../../lhotse_b200/csrc/reverb.cuh"

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

// the forward or inverse transform of the CTA's shared array, stage by stage, butterflies in thread order
static void fft(rv_c *a, const rv_c *tw, bool inverse) {
  for (int half = 1; half < RV_F; half <<= 1)
    for (int j = 0; j < RV_F / 2; ++j) rv_butterfly(a, tw, half, j, inverse);
}

int main(int argc, char **argv) {
  if (argc != 6) {
    fprintf(stderr, "usage: %s src0.i16 rirs.bin cuts.bin in.f32 out.f32\n", argv[0]);
    return 2;
  }
  const std::vector<int16_t> s0 = load<int16_t>(argv[1]);
  const std::vector<b200feat_reverb_rir> rirs = load<b200feat_reverb_rir>(argv[2]);
  const std::vector<b200feat_reverb_cut> cuts = load<b200feat_reverb_cut>(argv[3]);
  const std::vector<float> in = load<float>(argv[4]);
  std::vector<rv_c> tw(RV_B), a(RV_F);
  for (int k = 0; k < RV_B; ++k) tw[k] = rv_twiddle(k);
  // the RIR kernel: spectra and shifts
  std::vector<RvRir> rv(rirs.size());
  std::vector<int16_t *> rir_mem(rirs.size());
  std::vector<std::vector<rv_c>> spectra(rirs.size());
  std::vector<int64_t> shift(rirs.size());
  for (size_t i = 0; i < rirs.size(); ++i) {
    rir_mem[i] = exact_copy(s0, rirs[i].src_elem, rirs[i].num_samples);
    rv[i] = RvRir{rir_mem[i], rirs[i].num_samples, 0, (int32_t)rv_parts(rirs[i].num_samples), 0};
    spectra[i].resize((size_t)rv[i].nparts * RV_F);
    for (int p = 0; p < rv[i].nparts; ++p) {
      for (int m = 0; m < RV_F; ++m) a[rv_bitrev(m)] = rv_c{rv_rir_sample(rv[i], p, m), 0.0f};
      fft(a.data(), tw.data(), false);
      memcpy(&spectra[i][(size_t)p * RV_F], a.data(), sizeof(rv_c) * RV_F);
    }
    int best = -32769;
    for (int64_t k = 0; k < rv[i].len; ++k)
      if (rv[i].src[k] > best) { best = rv[i].src[k]; shift[i] = k; }
  }
  FILE *fo = fopen(argv[5], "wb");
  if (!fo) { fprintf(stderr, "cannot write %s\n", argv[5]); return 2; }
  int64_t ctas = 0;
  for (const b200feat_reverb_cut &cu : cuts) {
    const RvRir &r = rv[cu.rir];
    float *x = exact_copy(in, cu.in_elem, cu.in_len);
    float *y = (float *)malloc(sizeof(float) * cu.in_len);
    float *out = (float *)malloc(sizeof(float) * (cu.target_len > 0 ? cu.target_len : 1));
    RvCut c{x, y, out, cu.in_len, cu.target_len, 0, cu.rir, cu.normalize};
    double sum_y2 = 0.0;
    for (int64_t q = 0; q < rv_cut_ctas(c.n); ++q, ++ctas) {  // the convolution kernel's CTAs
      std::vector<rv_c> acc(RV_F, rv_c{0.0f, 0.0f});
      for (int p = 0; p < r.nparts; ++p) {
        const int64_t g = rv_seg_start(q, p, shift[cu.rir]);
        if (!rv_seg_live(g, c.n)) continue;
        for (int m = 0; m < RV_F; ++m) a[rv_bitrev(m)] = rv_seg_load(c, g, m);
        fft(a.data(), tw.data(), false);
        for (int k = 0; k < RV_F; ++k) acc[k] = rv_cmac(acc[k], a[k], spectra[cu.rir][(size_t)p * RV_F + k]);
      }
      for (int k = 0; k < RV_F; ++k) a[rv_bitrev(k)] = acc[k];
      fft(a.data(), tw.data(), true);
      float e = 0.0f;
      const int64_t base = 2 * q * RV_B;
      for (int i = 0; i < RV_B; ++i) {
        if (base + i < c.n) { y[base + i] = a[RV_B + i].x; e = RV_FMA(a[RV_B + i].x, a[RV_B + i].x, e); }
        if (base + RV_B + i < c.n) { y[base + RV_B + i] = a[RV_B + i].y; e = RV_FMA(a[RV_B + i].y, a[RV_B + i].y, e); }
      }
      sum_y2 += (double)e;
    }
    const float pb = (float)mix_energy(x, c.n);  // f32(S_x) / N, widened exactly by mix_energy_of_sum
    const float g = rv_gain(pb, sum_y2, c.n, c.normalize);
    for (int64_t p = 0; p < c.target_len; ++p) out[p] = rv_out(c, g, p);
    if (c.target_len > 0 && fwrite(out, sizeof(float), (size_t)c.target_len, fo) != (size_t)c.target_len) return 2;
    free(x); free(y); free(out);
  }
  fclose(fo);
  for (int16_t *p : rir_mem) free(p);
  printf("reverb: %zu cuts, %zu rirs, %lld ctas\n", cuts.size(), rirs.size(), (long long)ctas);
  return 0;
}
