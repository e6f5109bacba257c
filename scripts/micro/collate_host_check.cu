// CPU run of the audio collation index math of lhotse_b200/csrc/collate.cuh: the same row plan (head, float4 body, tail),
// unit order and per-element samples the kernel uses, with the source and every output row allocated to their exact sizes so
// that AddressSanitizer sees any access outside them.  No GPU needed; the header also compiles as plain C++:
//   g++ -x c++ -std=c++17 -O1 -g -fsanitize=address -o collate_host_check scripts/micro/collate_host_check.cu
//   ./collate_host_check src.bin dtype table.i64 T base_mod4 out.f32
//        src.bin holds the int16 (dtype 1) or float32 (dtype 0) source, table.i64 the B offsets and then the B lengths;
//        out.f32 receives the (B, T) batch.  Each element is written through a per-row write counter: an element written
//        twice or never is an error (exit 1).  Rows are kept apart (one allocation each), so a T past 2^31 / B is only
//        limited by memory per row.
//   ./collate_host_check --plan b T base_mod4
//        prints the row plan of row b (head, vectors, units and each unit's first element, count and kind) with 64-bit b
//        and T, so that rows past element 2^31 are checked without allocating them.
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <vector>

#include "../../lhotse_b200/csrc/collate.cuh"

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

// the units of one row as the kernel visits them (unit k of CTA k / (CO_THREADS * CO_UNITS_PER_THREAD)); checks that they tile
// [0, T) in order, that vector units start on a 16-byte boundary of the whole output, and returns false on any violation
static bool check_plan(int base_mod4, int64_t b, int64_t T, bool print) {
  const int h = co_head(base_mod4, b, T);
  const int64_t nv = co_vectors(h, T), units = co_units(nv);
  if (print) printf("head %d vectors %lld units %lld\n", h, (long long)nv, (long long)units);
  if (h < 0 || h > 3 || nv < 0 || (h < T &&(base_mod4 + (b % 4) * (T % 4) + h) % 4 != 0)) return false;
  int64_t next = 0;
  for (int64_t k = 0; k < units; ++k) {
    const CoUnit u = co_unit(k, h, nv, T);
    // print the head, the first and last two vectors and the tail (the rest follow the same rule)
    if (print && (k < 3 || k + 3 > units)) printf("unit %lld j %lld n %d vec %d\n", (long long)k, (long long)u.j, u.n, (int)u.vec);
    if (u.j != next || u.n < 0 || (u.vec && u.n != 4) || (!u.vec && u.n > 3)) return false;
    if (u.vec && (base_mod4 + (b % 4) * (T % 4) + (u.j % 4)) % 4 != 0) return false;
    next += u.n;
  }
  return next == T;
}

int main(int argc, char **argv) {
  if (argc == 5 && !strcmp(argv[1], "--plan")) {
    const int64_t b = atoll(argv[2]), T = atoll(argv[3]);
    return check_plan(atoi(argv[4]), b, T, true) ? 0 : 1;
  }
  if (argc != 7) {
    fprintf(stderr, "usage: %s src.bin dtype table.i64 T base_mod4 out.f32 | --plan b T base_mod4\n", argv[0]);
    return 2;
  }
  const int dt = atoi(argv[2]);
  const std::vector<int64_t> tab = load<int64_t>(argv[3]);
  const int64_t T = atoll(argv[4]);
  const int base_mod4 = atoi(argv[5]);
  const int64_t B = (int64_t)tab.size() / 2;
  // exact-size copies: an access past the source is a heap overflow under AddressSanitizer
  std::vector<char> raw = load<char>(argv[1]);
  const size_t esz = dt == 1 ? 2 : 4;
  char *src = (char *)malloc(raw.size() ? raw.size() : 1);
  memcpy(src, raw.data(), raw.size());
  FILE *fo = fopen(argv[6], "wb");
  if (!fo) { fprintf(stderr, "cannot open %s\n", argv[6]); return 2; }
  int bad = 0;
  for (int64_t b = 0; b < B; ++b) {
    const int64_t off = tab[b], len = tab[B + b];
    if (off < 0 || len < 0 || len > T || (uint64_t)(off + len) > raw.size() / esz) { fprintf(stderr, "bad table row %lld\n", (long long)b); return 2; }
    if (!check_plan(base_mod4, b, T, false)) { fprintf(stderr, "row %lld: plan does not tile [0, T)\n", (long long)b); bad = 1; }
    float *row = (float *)malloc((size_t)(T ? T : 1) * sizeof(float));
    std::vector<unsigned char> writes((size_t)T, 0);
    const int h = co_head(base_mod4, b, T);
    const int64_t nv = co_vectors(h, T), units = co_units(nv);
    for (int64_t k = 0; k < units; ++k) {
      const CoUnit u = co_unit(k, h, nv, T);
      for (int e = 0; e < u.n; ++e) {
        const int64_t j = u.j + e;
        row[j] = dt == 1 ? co_sample_i16((const int16_t *)src, off, len, j) : co_sample_f32((const float *)src, off, len, j);
        ++writes[(size_t)j];
      }
      // the vector-load test reads the same four samples the scalar path would
      if (co_vector_load(u, off, len) && (u.j + 4 > len || (off + u.j) % 4 != 0)) bad = 1;
    }
    for (int64_t j = 0; j < T; ++j)
      if (writes[(size_t)j] != 1) { fprintf(stderr, "row %lld element %lld written %d times\n", (long long)b, (long long)j, writes[(size_t)j]); bad = 1; break; }
    fwrite(row, sizeof(float), (size_t)T, fo);
    free(row);
  }
  fclose(fo);
  free(src);
  return bad;
}
