// CPU run of the resampling arithmetic of lhotse_b200/csrc/resample.cuh: the same __host__ __device__ chunking, window and
// FMA chain the kernel uses, CTA by CTA, with every window, table and buffer allocated to its exact size so that
// AddressSanitizer sees any access outside them.  No GPU needed; the header also compiles as plain C++:
//   g++ -x c++ -std=c++17 -O1 -g -fsanitize=address -o resample_host_check scripts/micro/resample_host_check.cu
//   ./resample_host_check src0.i16 src1.i16 tables.bin stages.bin mid_elems out_elems out.f32
//        b200feat_resample over the two int16 sources and the b200feat_resample_stage records (no argument checks: the
//        records are expected to be valid; `table` indexes tables.bin, a sequence of int32 N, O, K, width followed by the
//        float32 table [N][K]), written as out_elems float32 (zeros between the cuts)
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <vector>

#include "../../lhotse_b200/csrc/resample.cuh"

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
static T *exact(size_t n) { return (T *)calloc(n > 0 ? n : 1, sizeof(T)); }

struct Table { int32_t N, O, K, width; float *tr; };  // tr: [K][N], exactly N * K floats

int main(int argc, char **argv) {
  if (argc != 8) {
    fprintf(stderr, "usage: %s src0.i16 src1.i16 tables.bin stages.bin mid_elems out_elems out.f32\n", argv[0]);
    return 2;
  }
  const std::vector<int16_t> s0 = load<int16_t>(argv[1]), s1 = load<int16_t>(argv[2]);
  const std::vector<unsigned char> tb = load<unsigned char>(argv[3]);
  const std::vector<b200feat_resample_stage> stages = load<b200feat_resample_stage>(argv[4]);
  const int64_t mid_elems = atoll(argv[5]), out_elems = atoll(argv[6]);
  int16_t *src[2] = {exact<int16_t>(s0.size()), exact<int16_t>(s1.size())};
  if (!s0.empty()) memcpy(src[0], s0.data(), s0.size() * 2);
  if (!s1.empty()) memcpy(src[1], s1.data(), s1.size() * 2);
  std::vector<Table> tables;
  for (size_t at = 0; at < tb.size();) {
    Table t;
    memcpy(&t, tb.data() + at, 16);
    at += 16;
    t.tr = exact<float>((size_t)t.N * t.K);
    for (int32_t p = 0; p < t.N; ++p)
      for (int32_t k = 0; k < t.K; ++k) memcpy(&t.tr[(size_t)k * t.N + p], tb.data() + at + 4 * ((size_t)p * t.K + k), 4);
    at += 4 * (size_t)t.N * t.K;
    tables.push_back(t);
  }
  float *mid = exact<float>((size_t)mid_elems), *out = exact<float>((size_t)out_elems);
  float *dst[2] = {mid, out};
  for (const b200feat_resample_stage &r : stages) {  // records in depth order, as the launches run them
    RsStage s{};
    const Table *t = r.table >= 0 ? &tables[r.table] : nullptr;
    s.tab = t ? t->tr : nullptr;
    s.src16 = r.source == B200FEAT_RESAMPLE_MID ? nullptr : src[r.source] + r.in_elem;
    s.src32 = r.source == B200FEAT_RESAMPLE_MID ? mid + r.in_elem : nullptr;
    s.dst = dst[r.target] + r.out_elem;
    s.in_len = r.in_len; s.out_len = r.out_len; s.target_len = r.target_len;
    s.N = t ? t->N : 1; s.O = t ? t->O : 1; s.K = t ? t->K : 1; s.width = t ? t->width : 0;
    s.chunk = rs_chunk_outputs(s.N, s.O, s.K);
    s.scale_in = r.scale_in; s.scale_out = r.scale_out;
    for (int64_t c = 0; c < rs_stage_ctas(s); ++c) {  // one CTA
      int64_t p0, p1;
      rs_chunk(s, c, &p0, &p1);
      if (!s.tab) {
        for (int64_t p = p0; p < p1; ++p) s.dst[p] = MIX_FMUL(rs_load(s, mix_source_pos(p, s.out_len)), s.scale_out);
        continue;
      }
      int64_t b_lo, b_hi;
      rs_window(s, p0, p1, &b_lo, &b_hi);
      const int64_t W = (b_hi - b_lo) * s.O + s.K;
      if (W > rs_smem_floats(s)) { fprintf(stderr, "window of %lld floats past the CTA's shared memory\n", (long long)W); return 3; }
      float *win = exact<float>((size_t)W);
      for (int64_t i = 0; i < W; ++i) win[i] = rs_load(s, b_lo * s.O - s.width + i);
      for (int64_t p = p0; p < p1; ++p) {
        const int64_t j = mix_source_pos(p, s.out_len), b = j / s.N;
        s.dst[p] = MIX_FMUL(rs_output(win + (b - b_lo) * s.O, s.tab, s.N, s.K, (int)(j - b * s.N)), s.scale_out);
      }
      free(win);
    }
  }
  FILE *f = fopen(argv[7], "wb");
  if (!f || fwrite(out, sizeof(float), (size_t)out_elems, f) != (size_t)out_elems) { fprintf(stderr, "cannot write\n"); return 2; }
  fclose(f);
  for (Table &t : tables) free(t.tr);
  free(src[0]); free(src[1]); free(mid); free(out);
  printf("resample: %zu stages, %zu tables\n", stages.size(), tables.size());
  return 0;
}
