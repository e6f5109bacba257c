// CPU run of the whisper-fbank backward arithmetic of lhotse_b200/csrc/backward.cuh: the routed mass and tie count of the
// cut, the row-gradient rule, the log10 / clamp adjoint, the per-frame chain, the tile spans and the combine with torch's
// centre mirror, frame by frame and sample by sample, with every buffer allocated to its exact size so that
// AddressSanitizer sees any access outside it.  As in backward_host_check.cu, a direct DFT (float64, rounded once) stands in
// for the kernel's Stockham passes, and the reduction sums in element order.  No GPU needed:
//   g++ -x c++ -std=c++17 -O1 -g -fsanitize=address -o whisper_backward_host_check scripts/micro/whisper_backward_host_check.cu
//   ./whisper_backward_host_check in.bin out.f32
// in.bin: int32 [M n R], float32 [cut maximum m], then float32 window [400], mel bank [201][M], samples [n], log-mel rows
// [R][M] (the forward's, before the clamp), row gradient [R][M].  out.f32: the gradient of the n samples.
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

// common.cuh reflect_index, mode 1 (torch's "reflect")
static int64_t reflect1(int64_t i, int64_t n) {
  if (i < 0) i = -i;
  if (i >= n) i = 2 * n - 2 - i;
  return i;
}

int main(int argc, char **argv) {
  if (argc != 3) { fprintf(stderr, "usage: %s in.bin out.f32\n", argv[0]); return 2; }
  const std::vector<unsigned char> buf = load(argv[1]);
  size_t pos = 0;
  int32_t *h = take<int32_t>(buf, &pos, 3);
  float *mx = take<float>(buf, &pos, 1);
  BwdPlan p;
  memset(&p, 0, sizeof(p));
  // the whisper-fbank plan as b200feat.cu's bwd_plan builds it
  p.feature = B200FEAT_WHISPER_FBANK; p.whisper = 1; p.reflect = 1;
  p.L = 400; p.S = 160; p.N = 400; p.K = 201; p.Nc = 200; p.packed = 1; p.pad = 200;
  p.M = h[0]; p.F = h[0]; p.mel_floor = 1e-10f;
  const int64_t n = h[1], R = h[2], T = n / p.S;
  const float cmax = mx[0];
  float *window = take<float>(buf, &pos, p.L);
  p.window = window;
  float *bank = take<float>(buf, &pos, (size_t)p.K * p.M);
  float *x = take<float>(buf, &pos, n);
  float *xrows = take<float>(buf, &pos, (size_t)R * p.F);
  float *g = take<float>(buf, &pos, (size_t)R * p.F);
  BwdC *tws = (BwdC *)malloc(sizeof(BwdC) * p.K);
  for (int k = 0; k < p.K; ++k) {
    const double a = -2.0 * M_PI * (double)k / (double)p.N;
    tws[k] = BwdC{(float)cos(a), (float)sin(a)};
  }
  p.tws = tws;
  std::vector<int> mstart(p.M), mlen(p.M), mwoff(p.M);
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
  if (!bwd_launch_shape(p, &warps, &ft)) { fprintf(stderr, "launch shape refused\n"); return 2; }
  // the reduction kernel's per-cut sums, over the stft's T rows only
  float routed = 0.f;
  int ties = 0;
  for (int64_t e = 0; e < T * p.F; ++e) {
    routed += bwd_whisper_routed(g[e], xrows[e], cmax);
    ties += xrows[e] == cmax;
  }
  int *flo = (int *)malloc(sizeof(int) * p.K), *fhi = (int *)malloc(sizeof(int) * p.K);
  for (int k = 0; k < p.K; ++k) bwd_bin_filters(p, k, flo + k, fhi + k);
  const int64_t ntiles = (T + ft - 1) / ft, span = bwd_span(p, ft);
  float *spans = (float *)malloc(sizeof(float) * (size_t)(ntiles * span));
  float *G = (float *)malloc(sizeof(float) * (size_t)ft * p.L);
  float *raw = (float *)malloc(sizeof(float) * p.L), *v = (float *)malloc(sizeof(float) * p.K);
  float *gm = (float *)malloc(sizeof(float) * p.M);
  BwdC *xs = (BwdC *)malloc(sizeof(BwdC) * p.K);
  BwdC *fa = (BwdC *)malloc(sizeof(BwdC) * p.Nc), *fb = (BwdC *)malloc(sizeof(BwdC) * p.Nc);
  for (int64_t tile = 0; tile < ntiles; ++tile) {
    const int64_t t0 = tile * ft;
    const int nf = (int)(T - t0 < ft ? T - t0 : ft);
    for (int f = 0; f < nf; ++f) {
      const int64_t t = t0 + f;
      const float *gr = g + t * p.F, *xr = xrows + t * p.F;
      const int64_t base = t * p.S - p.pad;
      for (int j = 0; j < p.L; ++j) raw[j] = x[reflect1(base + j, n)];
      float *ybuf = (float *)fa;
      for (int j = 0; j < p.N; ++j) ybuf[j] = j < p.L ? bwd_y(p, raw, 0.f, j) : 0.f;
      dft(fa, fb, p.Nc);
      for (int k = 0; k < p.K; ++k) {
        xs[k] = bwd_bin(p, fb, k);
        v[k] = bwd_value(p, xs[k]);
      }
      for (int m = 0; m < p.M; ++m) gm[m] = bwd_whisper_gmel(p, gr, xr, m, bwd_mel(p, v, m), cmax, routed, ties);
      for (int k = 0; k < p.K; ++k) xs[k] = bwd_z(p, xs[k], v[k], bwd_gvalue(p, gr, v, gm, flo[k], fhi[k], k));
      for (int k = 0; k < p.Nc; ++k) fa[k] = bwd_inv_in(p, xs, k);
      dft(fa, fb, p.Nc);
      float *Gf = G + (size_t)f * p.L;
      for (int j = 0; j < p.L; ++j) Gf[j] = bwd_gd(p, fb, raw, 0.f, 0.f, j);
    }
    const int cover = (nf - 1) * p.S + p.L;
    for (int r = 0; r < span; ++r) spans[tile * span + r] = r < cover ? bwd_span_value(G, p.L, nf, p.S, p.L, r) : 0.f;
  }
  float *gx = (float *)malloc(sizeof(float) * (size_t)n);
  for (int64_t i = 0; i < n; ++i) gx[i] = bwd_sample(p, spans, ntiles, ft, n, T, i);
  FILE *fo = fopen(argv[2], "wb");
  if (!fo || fwrite(gx, sizeof(float), (size_t)n, fo) != (size_t)n) { fprintf(stderr, "cannot write %s\n", argv[2]); return 2; }
  fclose(fo);
  printf("whisper backward: n %lld, T %lld, R %lld, routed %g, ties %d, %lld tiles of %d frames, %d warps\n", (long long)n,
         (long long)T, (long long)R, routed, ties, (long long)ntiles, ft, warps);
  free(h); free(mx); free(window); free(bank); free(x); free(xrows); free(g); free(tws); free(flo); free(fhi); free(spans);
  free(G); free(raw); free(v); free(gm); free(xs); free(fa); free(fb); free(gx);
  return 0;
}
