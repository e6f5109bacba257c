// CPU check of the FFT stages of lhotse_b200/csrc/fast2048.cuh: the __host__ __device__ stage functions are run lane by lane
// (32 emulated lanes, the exchange tile a plain array) and the resulting |2 X[k]|^2, k = 0..1024, is compared with a float64
// DFT of the same 2048 real samples.  No GPU needed:
//   nvcc -gencode arch=compute_90a,code=sm_90a -o f2k_host_check scripts/micro/f2k_host_check.cu && ./f2k_host_check
#include <math.h>
#include <stdio.h>
#include <stdlib.h>

#include <vector>

#include "../../lhotse_b200/csrc/fast1024.cuh"

int main(int argc, char **argv) {
  const int L = argc > 1 ? atoi(argv[1]) : 2048;
  std::vector<float> y(2048, 0.f);
  srand(7);
  for (int i = 0; i < L; ++i) y[i] = (float)rand() / RAND_MAX - 0.5f + (i % 7 == 0 ? 0.3f : 0.f);
  std::vector<float2> tw1, tw2, w2k;
  f2k_fft_tables(tw1, tw2, w2k);
  std::vector<float2> X(F2K_XBUF, make_float2(NAN, NAN));
  std::vector<float> P(F2K_PBINS, NAN);
  static float2 v0[32][16], v1[32][16];
  for (int lane = 0; lane < 32; ++lane)
    for (int n1 = 0; n1 < 16; ++n1) {
      const int j = 128 * n1 + 2 * lane;
      v0[lane][n1] = make_float2(y[j], y[j + 1]);
      v1[lane][n1] = make_float2(y[j + 64], y[j + 65]);
    }
  for (int lane = 0; lane < 32; ++lane) f2k_stage1(lane, v0[lane], v1[lane], tw1.data(), X.data());
  for (int lane = 0; lane < 32; ++lane) f2k_stage2_load(lane, X.data(), v0[lane], v1[lane]);
  for (auto &x : X) x = make_float2(NAN, NAN);  // tile B overwrites tile A: nothing of A may be read afterwards
  for (int lane = 0; lane < 32; ++lane) f2k_stage2_store(lane, v0[lane], v1[lane], tw2.data(), reinterpret_cast<float4 *>(X.data()));
  for (int lane = 0; lane < 32; ++lane) f2k_stage3(lane, reinterpret_cast<const float4 *>(X.data()), w2k.data(), P.data(), false);
  double worst = 0.0, scale = 0.0;
  std::vector<double> ref(1025);
  for (int k = 0; k <= 1024; ++k) {
    double re = 0.0, im = 0.0;
    for (int n = 0; n < 2048; ++n) {
      const double a = -2.0 * M_PI * (double)((int64_t)n * k % 2048) / 2048.0;
      re += y[n] * cos(a); im += y[n] * sin(a);
    }
    ref[k] = 4.0 * (re * re + im * im);
    scale = fmax(scale, ref[k]);
  }
  int bad = 0;
  for (int k = 0; k <= 1024; ++k) {
    const double err = fabs((double)P[k] - ref[k]) / (ref[k] + 1e-3 * scale);
    if (!(err < 2e-5)) { if (bad < 10) printf("bin %d: got %.9g want %.9g\n", k, P[k], ref[k]); ++bad; }
    if (err > worst) worst = err;
  }
  printf("f2k_host_check L=%d: worst relative error %.3g over 1025 bins, %d bad\n", L, worst, bad);

  // ---- the balanced mel work items (common.cuh, MelItems) against the dense (K x M) product, on a warped triangular bank
  const int K = 1025, M = argc > 2 ? atoi(argv[2]) : 80;
  std::vector<float> bank((size_t)K * M, 0.f);
  std::vector<double> edge(M + 2);
  for (int m = 0; m < M + 2; ++m) edge[m] = 2.0 + 1020.0 * (exp(3.0 * m / (M + 1)) - 1.0) / (exp(3.0) - 1.0);
  for (int m = 0; m < M; ++m)
    for (int k = 0; k < K; ++k) {
      const double up = (k - edge[m]) / (edge[m + 1] - edge[m]), dn = (edge[m + 2] - k) / (edge[m + 2] - edge[m + 1]);
      const double w = fmin(up, dn);
      if (w > 0) bank[(size_t)k * M + m] = (float)w;
    }
  const MelItems mi = pack_mel_items_T(bank, K, M, 0.25f, 32, 4, F2K_PIECE, true);  // as fast2048_prepare
  const MelRounds mo = pack_mel_rounds(bank, K, M, 0.25f, 32, 4);
  std::vector<float> Pz(F2K_PBINS + 64, 0.f);
  for (int k = 0; k < K; ++k) Pz[k] = P[k];
  const int NQ = mi.rounds * 32;
  std::vector<float> part(NQ, 0.f);
  for (int j = 0; j < mi.rounds; ++j)
    for (int lane = 0; lane < 32; ++lane) {
      float acc = 0.f;
      const float *pp = Pz.data() + mi.rstart[j * 32 + lane];
      const float *wp = mi.wdense.data() + ((size_t)j * (F2K_PIECE / 4) * 32 + lane) * 4;  // [round][trip][lane][4]
      for (int t = 0; t < F2K_PIECE / 4; ++t, pp += 4, wp += 128)
        acc = fmaf(pp[3], wp[3], fmaf(pp[2], wp[2], fmaf(pp[1], wp[1], fmaf(pp[0], wp[0], acc))));
      part[j * 32 + lane] = acc;
    }
  int mbad = 0;
  double mworst = 0.0;
  for (int m = 0; m < M; ++m) {
    float a = 0.f;
    for (int q = 0; q < mi.qcount[m]; ++q) a += part[mi.qfirst[m] + q];
    double want = 0.0;
    for (int k = 0; k < K; ++k) want += 0.25 * (double)bank[(size_t)k * M + m] * (double)P[k];
    const double err = fabs(a - want) / (fabs(want) + 1e-30);
    mworst = fmax(mworst, err);
    if (!(err < 1e-5)) { if (mbad < 10) printf("filter %d: got %.9g want %.9g (items %d)\n", m, a, want, mi.qcount[m]); ++mbad; }
  }
  printf("mel items: piece %d taps, %d items in %d rounds, %d weight rows (whole-filter rounds: %d rows), simulated wavefronts %ld, "
         "reach %d; worst relative error %.3g, %d bad\n", mi.piece, mi.items, mi.rounds, mi.rows, mo.rows, mi.cost, mi.max_reach, mworst, mbad);

  // ---- whole-filter rounds (fast512 / fast256 / fast400 epilogues, pack_mel_rounds) with the over-read clamp: a short filter at the top
  // of the band that shares its round with a wide one must start earlier (zero weights in front) instead of reading past `limit`
  int rbad = 0;
  {
    const int K5 = 257, M5 = 40, limit = 260;
    std::vector<float> b5((size_t)K5 * M5, 0.f);
    std::vector<double> e5(M5 + 2);
    for (int m = 0; m < M5 + 2; ++m) e5[m] = 2.0 + 240.0 * (exp(2.2 * m / (M5 + 1)) - 1.0) / (exp(2.2) - 1.0);
    e5[M5] = 250.0; e5[M5 + 1] = 254.0;  // squeeze the last filter: ~8 taps next to ~30-tap neighbours (what VTLN 0.9 does to a 40-filter bank)
    for (int m = 0; m < M5; ++m)
      for (int k = 0; k < K5; ++k) {
        const double up = (k - e5[m]) / (e5[m + 1] - e5[m]), dn = (e5[m + 2] - k) / (e5[m + 2] - e5[m + 1]);
        const double w = fmin(up, dn);
        if (w > 0) b5[(size_t)k * M5 + m] = (float)w;
      }
    const MelRounds free_ = pack_mel_rounds(b5, K5, M5, 0.25f, 16, 4), clamped = pack_mel_rounds(b5, K5, M5, 0.25f, 16, 4, limit);
    std::vector<float> Pz(limit + 64, 0.f);
    for (int k = 0; k < K5; ++k) Pz[k] = 1.0f + 0.37f * (float)((k * 7919) % 101);
    for (int j = 0; j < clamped.rounds; ++j)
      for (int l = 0; l < 16; ++l) {
        const int m = l + 16 * j;
        if (m >= M5) continue;
        float acc = 0.f;
        const float *pp = Pz.data() + clamped.rstart[j * 16 + l];
        const float *wp = clamped.wdense.data() + (size_t)clamped.rrow[j] * 16 + l * 4;  // [row / 4][lane][4]
        for (int i = 0; i < clamped.rlen[j]; i += 4, pp += 4, wp += 64)
          acc = fmaf(pp[3], wp[3], fmaf(pp[2], wp[2], fmaf(pp[1], wp[1], fmaf(pp[0], wp[0], acc))));
        double want = 0.0;
        for (int k = 0; k < K5; ++k) want += 0.25 * (double)b5[(size_t)k * M5 + m] * (double)Pz[k];
        if (!(fabs(acc - want) <= 1e-5 * fabs(want) + 1e-6)) { if (rbad < 10) printf("clamped rounds, filter %d: got %.9g want %.9g\n", m, acc, want); ++rbad; }
      }
    if (!(free_.max_reach > limit) || clamped.max_reach > limit) { printf("clamp: reach %d -> %d (limit %d)\n", free_.max_reach, clamped.max_reach, limit); ++rbad; }
    printf("whole-filter rounds: reach %d without the clamp, %d with it (limit %d), %d bad\n", free_.max_reach, clamped.max_reach, limit, rbad);
  }

  // ---- the N = 1024 stages (fast1024.cuh): 512-point complex FFT as 16 x 8 x 4 + the same in-lane split with Q = 128
  int wbad = 0;
  {
    const int L1 = L > 1024 ? 600 : (L < 3 ? 3 : L);
    std::vector<float> y1(1024, 0.f);
    for (int i = 0; i < L1; ++i) y1[i] = (float)rand() / RAND_MAX - 0.5f + (i % 5 == 0 ? 0.25f : 0.f);
    std::vector<float2> t1, t2, wk;
    f1w_fft_tables(t1, t2, wk);
    std::vector<float2> X1(F1W_XBUF, make_float2(NAN, NAN));
    std::vector<float> P1(F1W_PBINS, NAN);
    static float2 v1w[32][16], u1w[32][8];
    for (int lane = 0; lane < 32; ++lane)
      for (int n1 = 0; n1 < 16; ++n1) v1w[lane][n1] = make_float2(y1[64 * n1 + 2 * lane], y1[64 * n1 + 2 * lane + 1]);
    for (int lane = 0; lane < 32; ++lane) f1w_stage1(lane, v1w[lane], t1.data(), X1.data());
    for (int lane = 0; lane < 32; ++lane) f1w_stage2_load(lane, X1.data(), v1w[lane], u1w[lane]);
    for (auto &x : X1) x = make_float2(NAN, NAN);
    for (int lane = 0; lane < 32; ++lane) {
      float2 tw[16];
      for (int i = 0; i < 16; ++i) tw[i] = t2[lane * 16 + i];
      f1w_stage2_store(lane, v1w[lane], u1w[lane], tw, reinterpret_cast<float4 *>(X1.data()));
    }
    for (int lane = 0; lane < 32; ++lane)
      f2k_stage3_t<128, F1W_PLANE>(lane, reinterpret_cast<const float4 *>(X1.data()), wk.data(), P1.data(), false);
    double w1 = 0.0, sc = 0.0;
    std::vector<double> r1(513);
    for (int k = 0; k <= 512; ++k) {
      double re = 0.0, im = 0.0;
      for (int n = 0; n < 1024; ++n) {
        const double a = -2.0 * M_PI * (double)((n * k) % 1024) / 1024.0;
        re += y1[n] * cos(a); im += y1[n] * sin(a);
      }
      r1[k] = 4.0 * (re * re + im * im);
      sc = fmax(sc, r1[k]);
    }
    for (int k = 0; k <= 512; ++k) {
      const double err = fabs((double)P1[k] - r1[k]) / (r1[k] + 1e-3 * sc);
      if (!(err < 2e-5)) { if (wbad < 10) printf("1024w bin %d: got %.9g want %.9g\n", k, P1[k], r1[k]); ++wbad; }
      w1 = fmax(w1, err);
    }
    printf("fast1024 stages L=%d: worst relative error %.3g over 513 bins, %d bad\n", L1, w1, wbad);
  }
  return (bad || mbad || wbad || rbad) ? 1 : 0;
}
