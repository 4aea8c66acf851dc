// Triangle arithmetic shared by the surface sampling of recon_eval.cu and the mesh operations of mesh_ops.cu.  Every
// fp64 step uses an explicit-rounding intrinsic (nvcc would otherwise contract mul-adds into FMAs), so numpy, which
// rounds every elementwise operation, reproduces it.
#pragma once
#include <cuda_runtime.h>

namespace nslam {

// x = (b - a) × (c - a) of triangle (ia, ib, ic) of vertices [V,3] fp32, in fp64: e1 = b - a, e2 = c - a,
// x0 = e1y e2z - e1z e2y, x1 = e1z e2x - e1x e2z, x2 = e1x e2y - e1y e2x
__device__ __forceinline__ void tri_cross(const float* V, int ia, int ib, int ic, double x[3]) {
  double e1[3], e2[3];
#pragma unroll
  for (int c = 0; c < 3; c++) {
    const double a = V[3 * (size_t)ia + c];
    e1[c] = __dsub_rn((double)V[3 * (size_t)ib + c], a);
    e2[c] = __dsub_rn((double)V[3 * (size_t)ic + c], a);
  }
  x[0] = __dsub_rn(__dmul_rn(e1[1], e2[2]), __dmul_rn(e1[2], e2[1]));
  x[1] = __dsub_rn(__dmul_rn(e1[2], e2[0]), __dmul_rn(e1[0], e2[2]));
  x[2] = __dsub_rn(__dmul_rn(e1[0], e2[1]), __dmul_rn(e1[1], e2[0]));
}

// The integer area weight w = rint(area · 2^40) (round to nearest even) of a triangle whose indices are in range,
// area = 0.5 sqrt((x0² + x1²) + x2²).  Returns 0, or the flag that sets w = 0: 2 a non-finite area, 4 w > cap (the
// caller's bound, 2^62 / T, keeps every 64-bit sum of weights exact).
__device__ __forceinline__ unsigned tri_area_weight(const float* V, int ia, int ib, int ic, unsigned long long cap,
                                                    unsigned long long& w) {
  double x[3];
  tri_cross(V, ia, ib, ic, x);
  const double area =
      __dmul_rn(0.5, __dsqrt_rn(__dadd_rn(__dadd_rn(__dmul_rn(x[0], x[0]), __dmul_rn(x[1], x[1])), __dmul_rn(x[2], x[2]))));
  w = 0;
  if (!isfinite(area)) return 2u;
  const double s = __dmul_rn(area, 0x1p40);
  if (s > (double)cap) return 4u;
  w = __double2ull_rn(s);
  return 0u;
}

}  // namespace nslam
