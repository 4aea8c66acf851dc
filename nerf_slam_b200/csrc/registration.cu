// Rigid and similarity registration of a point set to a surface (ICP): the transform of points and normals, the unit
// face normals of surface samples, and the Gauss-Newton sums of the correspondences.  The rules below DEFINE the
// behaviour; tests/registration_oracle.py restates them (fp64 numpy).  Every fp64 step uses an explicit-rounding
// intrinsic (nvcc would otherwise contract mul-adds into FMAs), so numpy, which rounds every elementwise operation,
// reproduces it.  The correspondences themselves are nslam_eval_nearest's (recon_eval.cu), unchanged.
//
// Transform.  A similarity (s, R [3x3 row-major], t) in fp64 maps an fp32 point p to p' with q_r = ((R_r0 p0 + R_r1 p1) +
// R_r2 p2) and p'_r = s q_r + t_r per row, rounded to fp32 once.  The direction mode writes q_r (a rotated normal: no
// scale, no translation).
//
// Face normals.  Sample i on triangle k = tri[i] (a, b, c of vertices [V,3] fp32): x = (b - a) × (c - a) in fp64
// (mesh_rules.cuh's tri_cross), len = sqrt((x0² + x1²) + x2²), n_c = x_c / len rounded to fp32 once.  A triangle index
// outside [0, T) or a vertex index outside [0, V) gives 0 and flag 1; a zero or non-finite len gives 0 and flag 2
// (surface sampling never picks a zero-area triangle).
//
// Correspondence terms.  The frame (c, L) normalises coordinates: p~_r = (p_r - c_r) / L in fp64 for the transformed
// source point p and its nearest target point q (idx >= 0), d = p~ - q~.  The host sets c to the centre of the target's
// box and L to half its diagonal, so |q~| <= 1, and refuses a correspondence distance above L, so |d| <= 1 and
// |p~| <= 2.  Point-to-plane with the target normal n: one row, r = ((n0 d0 + n1 d1) + n2 d2) and
// J = [p~ × n, n | (p~0 n0 + p~1 n1) + p~2 n2], with (p~ × n)_0 = p~1 n2 - p~2 n1, _1 = p~2 n0 - p~0 n2,
// _2 = p~0 n1 - p~1 n0.  Point-to-point: three rows k, r_k = d_k and J_k = [(-[p~]×)_k, e_k | p~_k] with
// -[p~]× = [[0, p~2, -p~1], [-p~2, 0, p~0], [p~1, -p~0, 0]]; a sum over the rows is ((row 0 + row 1) + row 2).  The
// scale column after `|` exists only with `with_scale`.  Each correspondence contributes H_ab = J_a J_b (a <= b),
// g_a = J_a r, e = (d0² + d1²) + d2² and 1 to the count.  Every term is rounded to a 64-bit integer in units of 2^-27
// (rint(v · 2^27)) before it is summed; |J| <= 2 elementwise, so |term| < 16 < 2^4 and every term is below 2^31 units,
// and with fewer than 2^31 points every sum stays below 2^62: the sums are exact and no thread order can change them.
// A term that is not finite or not below 16 in magnitude (a bad normal, a broken frame) is left out and raises flag 2; a
// target index outside [0, n_target) raises flag 1.
//
// Output layout, int64 [38]: H's upper triangle over 7 unknowns (omega 0..2, tau 3..5, sigma 6) row by row (28;
// entries of column 6 stay 0 without scale), g [7], e, the count, the flags.
//
// Reduction: each thread sums its points (grid-stride), then integer warp shuffles, shared memory across the block's
// warps and one atomicAdd per block per sum.  No scratch: the kernels write only their outputs.
#include "nslam_eval.h"
#include "common.cuh"
#include "mesh_rules.cuh"

#include <algorithm>
#include <cmath>

namespace nslam {

constexpr int kRegSums = 38;
constexpr int kRegThreads = 256;

struct Sim3Arg {
  double s, R[9], t[3];
};

struct RegFrame {
  double c[3], L;
};

__global__ void __launch_bounds__(256) reg_transform_kernel(const float* in, int n, Sim3Arg T, int direction, float* out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const double p[3] = {(double)in[3 * (size_t)i], (double)in[3 * (size_t)i + 1], (double)in[3 * (size_t)i + 2]};
#pragma unroll
  for (int r = 0; r < 3; r++) {
    const double q = __dadd_rn(__dadd_rn(__dmul_rn(T.R[3 * r], p[0]), __dmul_rn(T.R[3 * r + 1], p[1])),
                               __dmul_rn(T.R[3 * r + 2], p[2]));
    out[3 * (size_t)i + r] = __double2float_rn(direction ? q : __dadd_rn(__dmul_rn(T.s, q), T.t[r]));
  }
}

__global__ void __launch_bounds__(256) reg_face_normals_kernel(const float* V, int nv, const int* T, int nt, const int* tri,
                                                               int n, float* normals, unsigned long long* flags) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int k = tri[i];
  double x[3] = {0.0, 0.0, 0.0}, len = 0.0;
  unsigned f = 0;
  if (k < 0 || k >= nt) {
    f = 1;
  } else {
    const int ia = T[3 * (size_t)k], ib = T[3 * (size_t)k + 1], ic = T[3 * (size_t)k + 2];
    if (ia < 0 || ia >= nv || ib < 0 || ib >= nv || ic < 0 || ic >= nv) {
      f = 1;
    } else {
      tri_cross(V, ia, ib, ic, x);
      len = __dsqrt_rn(__dadd_rn(__dadd_rn(__dmul_rn(x[0], x[0]), __dmul_rn(x[1], x[1])), __dmul_rn(x[2], x[2])));
      if (!(len > 0.0) || isinf(len)) f = 2;
    }
  }
#pragma unroll
  for (int c = 0; c < 3; c++) normals[3 * (size_t)i + c] = f ? 0.f : __double2float_rn(__ddiv_rn(x[c], len));
  if (f) atomicOr(flags, (unsigned long long)f);
}

// index of H_ab (a <= b) in the row-by-row upper triangle over 7 unknowns
__host__ __device__ constexpr int reg_h(int a, int b) { return a * 7 - a * (a - 1) / 2 + (b - a); }

__device__ __forceinline__ void reg_add(unsigned long long& acc, double v, unsigned& flag) {
  if (fabs(v) < 16.0)
    acc += (unsigned long long)__double2ll_rn(__dmul_rn(v, 0x1p27));
  else
    flag |= 2u;
}

template <bool P2P, bool SCALE>
__global__ void __launch_bounds__(kRegThreads) reg_accumulate_kernel(const float* src, int n, const long long* idx,
                                                                     const float* tgt, const float* nrm, int n_tgt,
                                                                     RegFrame fr, unsigned long long* out) {
  constexpr int D = SCALE ? 7 : 6;
  unsigned long long acc[kRegSums - 1];
#pragma unroll
  for (int k = 0; k < kRegSums - 1; k++) acc[k] = 0;
  unsigned flag = 0;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const long long j = idx[i];
    if (j < 0) continue;
    if (j >= n_tgt) {
      flag |= 1u;
      continue;
    }
    double p[3], d[3];
#pragma unroll
    for (int c = 0; c < 3; c++) {
      p[c] = __ddiv_rn(__dsub_rn((double)src[3 * (size_t)i + c], fr.c[c]), fr.L);
      const double q = __ddiv_rn(__dsub_rn((double)__ldg(tgt + 3 * (size_t)j + c), fr.c[c]), fr.L);
      d[c] = __dsub_rn(p[c], q);
    }
    if constexpr (!P2P) {
      const double nn[3] = {(double)__ldg(nrm + 3 * (size_t)j), (double)__ldg(nrm + 3 * (size_t)j + 1),
                            (double)__ldg(nrm + 3 * (size_t)j + 2)};
      double J[7];
      J[0] = __dsub_rn(__dmul_rn(p[1], nn[2]), __dmul_rn(p[2], nn[1]));
      J[1] = __dsub_rn(__dmul_rn(p[2], nn[0]), __dmul_rn(p[0], nn[2]));
      J[2] = __dsub_rn(__dmul_rn(p[0], nn[1]), __dmul_rn(p[1], nn[0]));
      J[3] = nn[0];
      J[4] = nn[1];
      J[5] = nn[2];
      J[6] = __dadd_rn(__dadd_rn(__dmul_rn(p[0], nn[0]), __dmul_rn(p[1], nn[1])), __dmul_rn(p[2], nn[2]));
      const double r = __dadd_rn(__dadd_rn(__dmul_rn(nn[0], d[0]), __dmul_rn(nn[1], d[1])), __dmul_rn(nn[2], d[2]));
#pragma unroll
      for (int a = 0; a < D; a++) {
#pragma unroll
        for (int b = a; b < D; b++) reg_add(acc[reg_h(a, b)], __dmul_rn(J[a], J[b]), flag);
        reg_add(acc[28 + a], __dmul_rn(J[a], r), flag);
      }
    } else {
      // rows k of [-[p~]x | I | p~]; column a of row k
      const double J[3][7] = {{0.0, p[2], -p[1], 1.0, 0.0, 0.0, p[0]},
                              {-p[2], 0.0, p[0], 0.0, 1.0, 0.0, p[1]},
                              {p[1], -p[0], 0.0, 0.0, 0.0, 1.0, p[2]}};
#pragma unroll
      for (int a = 0; a < D; a++) {
#pragma unroll
        for (int b = a; b < D; b++)
          reg_add(acc[reg_h(a, b)],
                  __dadd_rn(__dadd_rn(__dmul_rn(J[0][a], J[0][b]), __dmul_rn(J[1][a], J[1][b])), __dmul_rn(J[2][a], J[2][b])),
                  flag);
        reg_add(acc[28 + a], __dadd_rn(__dadd_rn(__dmul_rn(J[0][a], d[0]), __dmul_rn(J[1][a], d[1])), __dmul_rn(J[2][a], d[2])),
                flag);
      }
    }
    reg_add(acc[35], __dadd_rn(__dadd_rn(__dmul_rn(d[0], d[0]), __dmul_rn(d[1], d[1])), __dmul_rn(d[2], d[2])), flag);
    acc[36] += 1;
  }
  __shared__ unsigned long long red[kRegThreads / 32][kRegSums - 1];
  __shared__ unsigned sflag;
  if (threadIdx.x == 0) sflag = 0;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int k = 0; k < kRegSums - 1; k++) {
    unsigned long long v = acc[k];
#pragma unroll
    for (int m = 16; m; m >>= 1) v += __shfl_xor_sync(0xffffffffu, v, m);
    if (lane == 0) red[warp][k] = v;
  }
  __syncthreads();
  if (flag) atomicOr(&sflag, flag);
  if (threadIdx.x < kRegSums - 1) {
    unsigned long long s = 0;
#pragma unroll
    for (int w = 0; w < kRegThreads / 32; w++) s += red[w][threadIdx.x];
    if (s) atomicAdd(out + threadIdx.x, s);
  }
  __syncthreads();
  if (threadIdx.x == 0 && sflag) atomicOr(out + kRegSums - 1, (unsigned long long)sflag);
}

}  // namespace nslam

extern "C" {

int nslam_reg_transform(const float* points, int n, const double* sim3, int direction, float* out, void* stream) {
  using namespace nslam;
  if (n < 0 || !sim3) return (int)cudaErrorInvalidValue;
  if (n == 0) return 0;
  Sim3Arg T;
  T.s = sim3[0];
  for (int k = 0; k < 9; k++) T.R[k] = sim3[1 + k];
  for (int k = 0; k < 3; k++) T.t[k] = sim3[10 + k];
  reg_transform_kernel<<<(n + 255) / 256, 256, 0, (cudaStream_t)stream>>>(points, n, T, direction, out);
  NSLAM_CHECK_LAUNCH();
  return 0;
}

int nslam_reg_face_normals(const float* vertices, int n_vert, const int* triangles, int n_tri, const int* tri, int n,
                           float* normals, long long* flags, void* stream) {
  using namespace nslam;
  if (n < 0 || n_vert < 0 || n_tri < 0) return (int)cudaErrorInvalidValue;
  cudaStream_t st = (cudaStream_t)stream;
  cudaError_t e = cudaMemsetAsync(flags, 0, sizeof(long long), st);
  if (e != cudaSuccess) return (int)e;
  if (n == 0) return 0;
  reg_face_normals_kernel<<<(n + 255) / 256, 256, 0, st>>>(vertices, n_vert, triangles, n_tri, tri, n, normals,
                                                           (unsigned long long*)flags);
  NSLAM_CHECK_LAUNCH();
  return 0;
}

int nslam_reg_accumulate(const float* source, int n, const long long* idx, const float* target, const float* target_normals,
                         int n_target, const double* frame, int point_to_point, int with_scale, int num_sms, long long* sums,
                         void* stream) {
  using namespace nslam;
  if (n < 0 || n_target <= 0 || !frame || !(frame[3] > 0.0) || !std::isfinite(frame[3]) ||
      (!point_to_point && !target_normals))
    return (int)cudaErrorInvalidValue;
  cudaStream_t st = (cudaStream_t)stream;
  cudaError_t e = cudaMemsetAsync(sums, 0, kRegSums * sizeof(long long), st);
  if (e != cudaSuccess) return (int)e;
  if (n == 0) return 0;
  if (num_sms <= 0) {
    int dev = 0;
    if ((e = cudaGetDevice(&dev)) != cudaSuccess) return (int)e;
    if ((e = cudaDeviceGetAttribute(&num_sms, cudaDevAttrMultiProcessorCount, dev)) != cudaSuccess) return (int)e;
  }
  const RegFrame fr{{frame[0], frame[1], frame[2]}, frame[3]};
  const int grid = (int)std::min<long long>(((long long)n + kRegThreads - 1) / kRegThreads, 4ll * num_sms);
  unsigned long long* out = (unsigned long long*)sums;
  if (point_to_point) {
    if (with_scale)
      reg_accumulate_kernel<true, true><<<grid, kRegThreads, 0, st>>>(source, n, idx, target, nullptr, n_target, fr, out);
    else
      reg_accumulate_kernel<true, false><<<grid, kRegThreads, 0, st>>>(source, n, idx, target, nullptr, n_target, fr, out);
  } else {
    if (with_scale)
      reg_accumulate_kernel<false, true><<<grid, kRegThreads, 0, st>>>(source, n, idx, target, target_normals, n_target,
                                                                       fr, out);
    else
      reg_accumulate_kernel<false, false><<<grid, kRegThreads, 0, st>>>(source, n, idx, target, target_normals, n_target,
                                                                        fr, out);
  }
  NSLAM_CHECK_LAUNCH();
  return 0;
}

}  // extern "C"
