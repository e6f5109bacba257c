// CPU run of the mixing arithmetic of lhotse_b200/csrc/mix.cuh: the same __host__ __device__ energy tree, gains and per-sample
// mix the kernels use, every buffer allocated to its exact size so that AddressSanitizer sees any access outside a track's
// samples or a cut's output window.  No GPU needed; the header also compiles as plain C++:
//   g++ -x c++ -std=c++17 -O1 -g -fsanitize=address -o mix_host_check scripts/micro/mix_host_check.cu
//   ./mix_host_check energy in.i16 lens.i64 out.f64
//        audio_energy of consecutive segments of in.i16 (lengths in lens.i64), in the tree the energy kernel's warp uses
//   ./mix_host_check mix src0.i16 src1.i16 tracks.bin cuts.bin out_elems out.f32 [src2.f32]
//        b200feat_mix over the two sources and the b200feat_mix_track / b200feat_mix_cut tables (no argument checks: the
//        tables are expected to be valid), written as out_elems float32 (zeros between the cuts); with src2.f32, the
//        float32 track buffer of b200feat_mix_ex (source 2, perturbed tracks) as well
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <vector>

#include "../../lhotse_b200/csrc/mix.cuh"

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
static void save(const char *path, const T *p, size_t n) {
  FILE *f = fopen(path, "wb");
  if (!f || fwrite(p, sizeof(T), n, f) != n) { fprintf(stderr, "cannot write %s\n", path); exit(2); }
  fclose(f);
}

// an exactly sized heap copy of samples [a, a + n) (ASan catches a read past either end)
template <typename T>
static T *exact_copy(const std::vector<T> &v, int64_t a, int64_t n) {
  T *p = (T *)malloc(sizeof(T) * (n > 0 ? n : 1));
  if (n > 0) memcpy(p, v.data() + a, sizeof(T) * n);
  return p;
}

int main(int argc, char **argv) {
  if (argc >= 5 && !strcmp(argv[1], "energy")) {
    const std::vector<int16_t> pcm = load<int16_t>(argv[2]);
    const std::vector<int64_t> lens = load<int64_t>(argv[3]);
    std::vector<double> out(lens.size());
    int64_t a = 0;
    for (size_t i = 0; i < lens.size(); ++i) {
      if (a + lens[i] > (int64_t)pcm.size()) { fprintf(stderr, "segments past the samples\n"); return 2; }
      int16_t *q = exact_copy(pcm, a, lens[i]);
      out[i] = mix_energy(q, lens[i]);
      free(q);
      a += lens[i];
    }
    save(argv[4], out.data(), out.size());
    printf("energy: %zu segments\n", lens.size());
    return 0;
  }
  if (argc >= 8 && !strcmp(argv[1], "mix")) {
    const std::vector<int16_t> s0 = load<int16_t>(argv[2]), s1 = load<int16_t>(argv[3]);
    const std::vector<b200feat_mix_track> tracks = load<b200feat_mix_track>(argv[4]);
    const std::vector<b200feat_mix_cut> cuts = load<b200feat_mix_cut>(argv[5]);
    const int64_t out_elems = atoll(argv[6]);
    const std::vector<float> s2 = argc >= 9 ? load<float>(argv[8]) : std::vector<float>();
    int16_t *src0 = exact_copy(s0, 0, (int64_t)s0.size()), *src1 = exact_copy(s1, 0, (int64_t)s1.size());
    float *src2 = exact_copy(s2, 0, (int64_t)s2.size());
    float *out = (float *)calloc((size_t)(out_elems > 0 ? out_elems : 1), sizeof(float));
    std::vector<double> energy(tracks.size(), 0.0);
    std::vector<float> gain32(tracks.size(), 1.0f);
    for (const b200feat_mix_cut &cut : cuts) {  // the energy kernel's block
      for (int k = 0; k < cut.num_tracks; ++k) {
        const int64_t t = cut.first_track + k;
        const b200feat_mix_track &tr = tracks[t];
        if (!mix_needs_energy(cut, tr, t) || tr.source < 0 || tr.num_samples <= 0) continue;
        energy[t] = tr.source == B200FEAT_MIX_SRC_F32 ? mix_energy(src2 + tr.src_elem, tr.num_samples)
                                                      : mix_energy((tr.source == 0 ? src0 : src1) + tr.src_elem, tr.num_samples);
      }
      double scale = 0.0;
      const double e_ref = energy[cut.first_track + cut.ref_track];
      for (int k = 0; k < cut.num_tracks; ++k) {
        const int64_t t = cut.first_track + k;
        gain32[t] = mix_track_gain(cut, tracks[t], k, e_ref, energy[t], &scale);
      }
      for (int64_t p = 0; p < cut.target_len; ++p)  // the mix kernel's grid-stride loop
        out[cut.out_elem + p] = mix_sample(src0, src1, src2, tracks.data(), cut, gain32.data(), scale, p);
    }
    save(argv[7], out, (size_t)out_elems);
    free(src0); free(src1); free(src2); free(out);
    printf("mix: %zu cuts, %zu tracks\n", cuts.size(), tracks.size());
    return 0;
  }
  fprintf(stderr, "usage: %s energy in.i16 lens.i64 out.f64 | mix src0.i16 src1.i16 tracks.bin cuts.bin out_elems out.f32 [src2.f32]\n", argv[0]);
  return 2;
}
