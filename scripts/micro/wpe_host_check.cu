// CPU run of the WPE arithmetic of lhotse_b200/csrc/wpe.cuh: the per-bin statistics (the kernel's entry / frame-slice split
// and slice-order sums), the column-by-column LU solve, the filter, the overlap-add and the length fix, with a direct DFT
// (evaluated in double, rounded to float32) in place of the kernels' FFTs.  Every input, spectrum and output window is
// allocated to its exact size so that AddressSanitizer sees any access outside them.  No GPU needed; the header also compiles
// as plain C++:
//   g++ -x c++ -std=c++17 -O1 -g -fsanitize=address -o wpe_host_check scripts/micro/wpe_host_check.cu
//   ./wpe_host_check cuts.bin in.f32 window.f32 out.f32 taps delay iterations valid
//        b200feat_wpe over the b200feat_wpe_cut table and the float32 input buffer (no argument checks: the table is expected
//        to be valid); each cut's target_len samples are written back to back to out.f32.
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <vector>

#include "../../include/b200feat.h"
#include "../../lhotse_b200/csrc/wpe.cuh"

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
  if (argc != 9) {
    fprintf(stderr, "usage: %s cuts.bin in.f32 window.f32 out.f32 taps delay iterations valid\n", argv[0]);
    return 2;
  }
  const std::vector<b200feat_wpe_cut> cuts = load<b200feat_wpe_cut>(argv[1]);
  const std::vector<float> in = load<float>(argv[2]);
  const std::vector<float> win = load<float>(argv[3]);
  const WpeParams prm{atoi(argv[5]), atoi(argv[6]), atoi(argv[7]), atoi(argv[8])};
  if (win.size() != WPE_NFFT) { fprintf(stderr, "window must have 512 samples\n"); return 2; }
  FILE *fo = fopen(argv[4], "wb");
  if (!fo) { fprintf(stderr, "cannot write %s\n", argv[4]); return 2; }
  const int n = prm.taps, E = wpe_entries(n), S = WPE_THREADS / E;
  std::vector<double> cs(WPE_NFFT), sn(WPE_NFFT);
  for (int m = 0; m < WPE_NFFT; ++m) { cs[m] = cos(2.0 * M_PI * m / WPE_NFFT); sn[m] = sin(2.0 * M_PI * m / WPE_NFFT); }
  for (const b200feat_wpe_cut &cu : cuts) {
    float *x = (float *)malloc(sizeof(float) * cu.in_len);
    memcpy(x, in.data() + cu.in_elem, sizeof(float) * cu.in_len);
    const int T = (int)wpe_frames(cu.in_len);
    // STFT (direct DFT of the windowed frame)
    std::vector<std::vector<wpe_c>> Y(WPE_BINS, std::vector<wpe_c>(T));
    std::vector<float> fr(WPE_NFFT);
    for (int t = 0; t < T; ++t) {
      for (int m = 0; m < WPE_NFFT; ++m) fr[m] = MIX_FMUL(wpe_frame_sample(x, cu.in_len, t, m), win[m]);
      for (int k = 0; k < WPE_BINS; ++k) {
        double re = 0.0, im = 0.0;
        for (int m = 0; m < WPE_NFFT; ++m) {
          const int r = (int)(((int64_t)k * m) % WPE_NFFT);
          re += fr[m] * cs[r];
          im -= fr[m] * sn[r];
        }
        Y[k][t] = wpe_c{(float)re, (float)im};
      }
    }
    // per bin, as wpe_bin_kernel: the bin's row and inv_t in arrays of exactly T
    for (int k = 0; k < WPE_BINS && prm.iterations > 0; ++k) {
      wpe_c *row = (wpe_c *)malloc(sizeof(wpe_c) * T);
      double *inv = (double *)malloc(sizeof(double) * T);
      memcpy(row, Y[k].data(), sizeof(wpe_c) * T);
      wpe_z A[WPE_MAX_TAPS * WPE_LD], G[WPE_MAX_TAPS];
      std::vector<wpe_z> part((size_t)S * E);
      const int t_min = prm.valid ? prm.delay + n - 1 : 0;
      for (int it = 0; it < prm.iterations; ++it) {
        double mx = 0.0;
        for (int t = 0; t < T; ++t) {
          inv[t] = wpe_power(it == 0 ? wpe_z{row[t].x, row[t].y} : wpe_filter(row, t, G, n, prm.delay));
          mx = fmax(mx, inv[t]);
        }
        const double eps = 1e-10 * mx;
        for (int t = 0; t < T; ++t) inv[t] = wpe_inv(inv[t], eps);
        for (int th = 0; th < S * E; ++th) {
          int la, lb;
          wpe_entry_lags(th % E, n, prm.delay, &la, &lb);
          part[th] = wpe_entry_sum(row, inv, T, la, lb, t_min, th / E, S);
        }
        for (int e = 0; e < E; ++e) {
          wpe_z v = part[e];
          for (int s = 1; s < S; ++s) v = wpe_z{v.x + part[e + s * E].x, v.y + part[e + s * E].y};
          wpe_place(A, n, prm.delay, e, v);
        }
        bool regular = true;
        for (int kk = 0; kk < n; ++kk) {
          const int p = wpe_pivot(A, n, kk);
          if (p < 0) { regular = false; break; }
          if (p != kk)
            for (int c = kk; c <= n; ++c) { const wpe_z v = A[kk * WPE_LD + c]; A[kk * WPE_LD + c] = A[p * WPE_LD + c]; A[p * WPE_LD + c] = v; }
          for (int c = kk + 1; c <= n; ++c) wpe_eliminate(A, n, kk, c);
        }
        wpe_back_substitute(A, n, regular, G);
      }
      for (int t = 0; t < T; ++t) {
        const wpe_z v = wpe_filter(row, t, G, n, prm.delay);
        Y[k][t] = wpe_c{(float)v.x, (float)v.y};
      }
      free(row);
      free(inv);
    }
    // iSTFT: every frame's windowed C2R inverse (direct), then the kernel's overlap-add and length fix
    float *frames = (float *)malloc(sizeof(float) * (size_t)T * WPE_NFFT);
    for (int t = 0; t < T; ++t)
      for (int m = 0; m < WPE_NFFT; ++m) {
        double v = Y[0][t].x + ((m & 1) ? -1.0 : 1.0) * Y[WPE_NFFT / 2][t].x;
        for (int k = 1; k < WPE_NFFT / 2; ++k) {
          const int r = (int)(((int64_t)k * m) % WPE_NFFT);
          v += 2.0 * (Y[k][t].x * cs[r] - Y[k][t].y * sn[r]);
        }
        frames[(size_t)t * WPE_NFFT + m] = MIX_FMUL((float)(v / WPE_NFFT), win[m]);
      }
    float *out = (float *)malloc(sizeof(float) * (cu.target_len > 0 ? cu.target_len : 1));
    const int64_t Lz = wpe_istft_len(cu.in_len);
    for (int64_t j = 0; j < Lz; ++j) wpe_store(out, cu.target_len, Lz, j, wpe_ola(frames, 0, T, win.data(), j));
    if (cu.target_len > 0 && fwrite(out, sizeof(float), (size_t)cu.target_len, fo) != (size_t)cu.target_len) return 2;
    free(frames);
    free(out);
    free(x);
  }
  fclose(fo);
  printf("wpe: %zu cuts\n", cuts.size());
  return 0;
}
