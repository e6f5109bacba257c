// CPU run of the backward arithmetic of lhotse_b200/csrc/backward.cuh: the same per-frame adjoint chain, tile spans and
// per-sample combine the kernels use, frame by frame and sample by sample, with every buffer allocated to its exact size so
// that AddressSanitizer sees any access outside it.  The FFT passes of the kernel (generic.cuh's stockham_pass) are device
// code; here a direct DFT of the same length, input and sign (float64, rounded once) stands in for them.  No GPU needed:
//   g++ -x c++ -std=c++17 -O1 -g -fsanitize=address -o backward_host_check scripts/micro/backward_host_check.cu
//   ./backward_host_check in.bin out.f32
// in.bin: int32 header [feature L S N M C F snip_edges remove_dc use_energy raw_energy use_mag energy_style use_lifter
// ecol shift n T pad 0], float32 [preemph energy_floor_log has_energy_floor mel_floor log_spec_eps log_spec_floor], then
// float32 window [L], mel bank [K][M] (M > 0), dct [M][C] (C > 0), lifter [C] (use_lifter), samples [n], row gradient [T][F].
// out.f32: the gradient of the n samples.  Prints the launch shape (frames per tile, warps per CTA); exits with 3, writing
// nothing, for a frame the backward refuses.
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <vector>

#include "../../lhotse_b200/csrc/backward.cuh"

static std::vector<unsigned char> load(const char *path) {
  std::vector<unsigned char> v;
  FILE *f = fopen(path, "rb");
  if (!f) { fprintf(stderr, "cannot open %s\n", path); exit(2); }
  fseek(f, 0, SEEK_END);
  v.resize((size_t)ftell(f));
  fseek(f, 0, SEEK_SET);
  if (!v.empty() && fread(v.data(), 1, v.size(), f) != v.size()) { fprintf(stderr, "short read %s\n", path); exit(2); }
  fclose(f);
  return v;
}

template <typename T>
static T *take(const std::vector<unsigned char> &buf, size_t *pos, size_t count) {  // a copy at its exact size
  if (*pos + count * sizeof(T) > buf.size()) { fprintf(stderr, "input too short\n"); exit(2); }
  T *p = (T *)malloc(count * sizeof(T) + (count == 0));
  memcpy(p, buf.data() + *pos, count * sizeof(T));
  *pos += count * sizeof(T);
  return p;
}

// out[k] = sum_j in[j] exp(-2 pi i j k / Nc): the transform the kernel's Stockham passes compute
static void dft(const BwdC *in, BwdC *out, int Nc) {
  for (int k = 0; k < Nc; ++k) {
    double re = 0.0, im = 0.0;
    for (int j = 0; j < Nc; ++j) {
      const double a = -2.0 * M_PI * (double)(((int64_t)j * k) % Nc) / (double)Nc;
      re += in[j].x * cos(a) - in[j].y * sin(a);
      im += in[j].x * sin(a) + in[j].y * cos(a);
    }
    out[k] = BwdC{(float)re, (float)im};
  }
}

static int64_t reflect(int64_t i, int64_t n) {
  if (i < 0) i = -i - 1;
  if (i >= n) i = 2 * n - 1 - i;
  return i;
}

int main(int argc, char **argv) {
  if (argc != 3) { fprintf(stderr, "usage: %s in.bin out.f32\n", argv[0]); return 2; }
  const std::vector<unsigned char> buf = load(argv[1]);
  size_t pos = 0;
  int32_t *h = take<int32_t>(buf, &pos, 20);
  float *sc = take<float>(buf, &pos, 6);
  BwdPlan p;
  memset(&p, 0, sizeof(p));
  p.feature = h[0]; p.L = h[1]; p.S = h[2]; p.N = h[3]; p.M = h[4]; p.C = h[5]; p.F = h[6];
  p.snip_edges = h[7]; p.remove_dc = h[8]; p.use_energy = h[9]; p.raw_energy = h[10]; p.use_mag = h[11];
  p.energy_style = h[12]; p.use_lifter = h[13]; p.ecol = h[14]; p.shift = h[15];
  const int64_t n = h[16], T = h[17];
  p.pad = h[18];
  p.preemph = sc[0]; p.energy_floor_log = sc[1]; p.has_energy_floor = sc[2]; p.mel_floor = sc[3]; p.log_spec_eps = sc[4];
  p.log_spec_floor = sc[5];
  p.K = p.N / 2 + 1;
  p.packed = p.N % 2 == 0;
  p.Nc = p.packed ? p.N / 2 : p.N;
  float *window = take<float>(buf, &pos, p.L);
  p.window = window;
  float *bank = p.M ? take<float>(buf, &pos, (size_t)p.K * p.M) : nullptr;
  float *dct = p.C ? take<float>(buf, &pos, (size_t)p.M * p.C) : nullptr;
  float *lifter = p.use_lifter ? take<float>(buf, &pos, p.C) : nullptr;
  float *x = take<float>(buf, &pos, n);
  float *g = take<float>(buf, &pos, (size_t)T * p.F);
  p.dct = dct; p.lifter = lifter;
  // the library's tables: twiddles of the packed split, the filters' supports (b200feat.cu setup_handle)
  BwdC *tws = (BwdC *)malloc(sizeof(BwdC) * p.K);
  for (int k = 0; k < p.K; ++k) {
    const double a = -2.0 * M_PI * (double)k / (double)p.N;
    tws[k] = BwdC{(float)cos(a), (float)sin(a)};
  }
  p.tws = tws;
  std::vector<int> mstart(p.M > 0 ? p.M : 1), mlen(p.M > 0 ? p.M : 1), mwoff(p.M > 0 ? p.M : 1);
  std::vector<float> mw;
  for (int m = 0; m < p.M; ++m) {
    int first = -1, last = -1;
    for (int k = 0; k < p.K; ++k)
      if (bank[(size_t)k * p.M + m] != 0.f) { if (first < 0) first = k; last = k; }
    mstart[m] = first >= 0 ? first : 0;
    mlen[m] = first >= 0 ? last - first + 1 : 0;
    mwoff[m] = (int)mw.size();
    for (int k = 0; k < mlen[m]; ++k) mw.push_back(bank[(size_t)(mstart[m] + k) * p.M + m]);
  }
  if (mw.empty()) mw.push_back(0.f);
  p.mel_start = mstart.data(); p.mel_len = mlen.data(); p.mel_woff = mwoff.data(); p.mel_w = mw.data();

  int warps, ft;
  if (!bwd_launch_shape(p, &warps, &ft)) {
    printf("backward: frame too long, %zu bytes of shared memory for one warp and one frame, limit %d\n", bwd_smem(p, 1, 1),
           BWD_SMEM_LIMIT);
    free(h); free(sc); free(window); free(bank); free(dct); free(lifter); free(x); free(g); free(tws);
    return 3;
  }
  const bool mel = p.feature == B200FEAT_FBANK || p.feature == B200FEAT_MFCC;
  int *flo = (int *)malloc(sizeof(int) * p.K), *fhi = (int *)malloc(sizeof(int) * p.K);
  if (mel)
    for (int k = 0; k < p.K; ++k) bwd_bin_filters(p, k, flo + k, fhi + k);
  const int64_t ntiles = (T + ft - 1) / ft, span = bwd_span(p, ft);
  float *spans = (float *)malloc(sizeof(float) * (size_t)(ntiles * span));
  float *G = (float *)malloc(sizeof(float) * (size_t)ft * p.L);
  float *raw = (float *)malloc(sizeof(float) * p.L), *v = (float *)malloc(sizeof(float) * p.K);
  float *gm = (float *)malloc(sizeof(float) * (p.M > 0 ? p.M : 1));
  BwdC *xs = (BwdC *)malloc(sizeof(BwdC) * p.K);
  BwdC *fa = (BwdC *)malloc(sizeof(BwdC) * p.Nc), *fb = (BwdC *)malloc(sizeof(BwdC) * p.Nc);
  for (int64_t tile = 0; tile < ntiles; ++tile) {
    const int64_t t0 = tile * ft;
    const int nf = (int)(T - t0 < ft ? T - t0 : ft);
    for (int f = 0; f < nf; ++f) {
      const int64_t t = t0 + f;
      const float *gr = g + t * p.F;
      const int64_t base = t * p.S - (p.snip_edges ? 0 : p.pad);
      float s = 0.f;
      for (int j = 0; j < p.L; ++j) {
        const int64_t i = p.snip_edges ? base + j : reflect(base + j, n);
        raw[j] = x[i];
        s += raw[j];
      }
      const float mu = p.remove_dc ? s / (float)p.L : 0.f;
      float e = 0.f;
      float *ybuf = (float *)fa;
      for (int j = 0; j < p.N; ++j) {
        float y = 0.f;
        if (j < p.L) {
          y = bwd_y(p, raw, mu, j);
          if (p.use_energy) e += bwd_energy_term(p, raw, mu, j);
        }
        if (p.packed) ybuf[j] = y; else fa[j] = BwdC{y, 0.f};
      }
      const float ge = p.use_energy ? bwd_energy_grad(p, gr) * bwd_energy_scale(p, e) : 0.f;
      dft(fa, fb, p.Nc);
      for (int k = 0; k < p.K; ++k) {
        xs[k] = bwd_bin(p, fb, k);
        v[k] = bwd_value(p, xs[k]);
      }
      if (mel)
        for (int m = 0; m < p.M; ++m) gm[m] = bwd_gmel(p, gr, m, bwd_mel(p, v, m));
      for (int k = 0; k < p.K; ++k)
        xs[k] = bwd_z(p, xs[k], v[k], bwd_gvalue(p, gr, v, gm, mel ? flo[k] : 0, mel ? fhi[k] : 0, k));
      const int nin = p.packed ? p.Nc : p.N;
      for (int k = 0; k < nin; ++k) fa[k] = bwd_inv_in(p, xs, k);
      dft(fa, fb, p.Nc);
      float *Gf = G + (size_t)f * p.L;
      float sum = 0.f;
      for (int j = 0; j < p.L; ++j) { Gf[j] = bwd_gd(p, fb, raw, mu, ge, j); sum += Gf[j]; }
      if (p.remove_dc)
        for (int j = 0; j < p.L; ++j) Gf[j] -= sum / (float)p.L;
    }
    const int cover = (nf - 1) * p.S + p.L;
    for (int r = 0; r < span; ++r) spans[tile * span + r] = r < cover ? bwd_span_value(G, p.L, nf, p.S, p.L, r) : 0.f;
  }
  float *gx = (float *)malloc(sizeof(float) * (size_t)n);
  for (int64_t i = 0; i < n; ++i) gx[i] = bwd_sample(p, spans, ntiles, ft, n, T, i);
  FILE *fo = fopen(argv[2], "wb");
  if (!fo || fwrite(gx, sizeof(float), (size_t)n, fo) != (size_t)n) { fprintf(stderr, "cannot write %s\n", argv[2]); return 2; }
  fclose(fo);
  printf("backward: n %lld, T %lld, %lld tiles of %d frames, %d warps\n", (long long)n, (long long)T, (long long)ntiles, ft,
         warps);
  free(h); free(sc); free(window); free(bank); free(dct); free(lifter); free(x); free(g); free(tws); free(flo); free(fhi);
  free(spans); free(G); free(raw); free(v); free(gm); free(xs); free(fa); free(fb); free(gx);
  return 0;
}
