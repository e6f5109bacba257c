// The shared-memory layout and launch shape of the generic kernel (lhotse_b200/csrc/generic.cuh), as the host sizes the
// launch and the kernel addresses its warp's region: one line per plan on stdin, `feature N M` (feature: the
// B200FEAT_* kind, M: the number of mel filters, 0 for spectra), one line out per plan:
//   N Nc bufA bufB mlog floats warps smem fits
// (offsets and sizes of one warp's region in floats, warps per CTA, dynamic shared-memory bytes per CTA, and whether
// that is within the opt-in limit).  No GPU needed:
//   nvcc -std=c++17 -gencode arch=compute_90a,code=sm_90a -o generic_layout_check scripts/micro/generic_layout_check.cu
//   printf '1 32 40\n' | ./generic_layout_check
#include <stdio.h>
#include <string.h>

#include "../../lhotse_b200/csrc/generic.cuh"

int main() {
  int feature, N, M;
  while (scanf("%d %d %d", &feature, &N, &M) == 3) {
    DevPlan p;
    memset(&p, 0, sizeof(p));
    p.feature = feature;
    p.N = N;
    p.K = N / 2 + 1;
    p.M = M;
    p.packed = N % 2 == 0;
    p.Nc = p.packed ? N / 2 : N;
    const GenericLayout l = generic_layout(p);
    int warps = 0;
    size_t smem = 0;
    const bool fits = generic_launch_shape(p, &warps, &smem);
    printf("%d %d %d %d %d %d %d %zu %d\n", N, p.Nc, l.bufA, l.bufB, l.mlog, l.floats, warps, smem, fits ? 1 : 0);
  }
  return 0;
}
