// Rules shared by the dense TSDF volume (tsdf.cu, tsdf_mesh.cu) and the sparse voxel-block volume (tsdf_blocks.cu):
// the per-voxel update of one keyframe and the ray march of the read-out.  Both volumes call these functions, so the
// arithmetic is written once; each volume only supplies how a voxel is addressed.  Every fp32 step uses an
// explicit-rounding intrinsic so that the numpy restatements (oracle/tsdf.py, tests/tsdf_readout_oracle.py) match bit
// for bit.
#pragma once
#include "common.cuh"

namespace nslam {

struct TsdfFrame {
  const float* idepth;      // [H,W] inverse depth (upsampled)
  const float* depth_cov;   // [H,W] depth variance, or NULL = uniform weight 1
  const unsigned char* rgb; // [3,H,W] u8
  int H, W;
  float fx, fy, cx, cy;
  const float* pose;        // cam_T_world [t, q_xyzw] on the DEVICE (x_cam = R(q) x_world + t): no host copy of the pose
  float max_depth, trunc, max_weight, max_sigma;
};

// SE3(poses).matrix() is a float32 matrix that build_volume promotes to float64 (reference :186, :209): the rotation is
// rounded to fp32, then promoted
__device__ __forceinline__ void tsdf_pose_rotation(const float* p, double R[9]) {
  const double qx = p[3], qy = p[4], qz = p[5], qw = p[6];
  const double r[9] = {1 - 2 * (qy * qy + qz * qz), 2 * (qx * qy - qz * qw), 2 * (qx * qz + qy * qw),
                       2 * (qx * qy + qz * qw), 1 - 2 * (qx * qx + qz * qz), 2 * (qy * qz - qx * qw),
                       2 * (qx * qz - qy * qw), 2 * (qy * qz + qx * qw), 1 - 2 * (qx * qx + qy * qy)};
  for (int i = 0; i < 9; i++) R[i] = (double)(float)r[i];
}

// depth of pixel `pix` as build_volume makes it: 1 / inverse depth, pushed beyond max_depth when the sigma test masks it
// (:192-203, :549); wr = its weight reading
__device__ __forceinline__ float tsdf_pixel_depth(const TsdfFrame& f, size_t pix, float& wr) {
  float depth = 1.0f / f.idepth[pix];
  wr = 1.0f;
  if (f.depth_cov) {
    const float cov = f.depth_cov[pix];
    wr = sqrtf(1.0f / cov);                                   // cov.pow(-1).sqrt()  (:196)
    if (!(sqrtf(cov) < f.max_sigma)) depth = f.max_depth + 1.0f;
  }
  return depth;
}

// One voxel, one keyframe (reference fusion/tsdf_fusion.py:231-296).  (wxf, wyf, wzf) = the voxel's fp32 world
// coordinate, promoted to fp64 with the pose and the intrinsics for the projection.  tsdf / weight point at the voxel,
// color at its 3 channels.
__device__ __forceinline__ void tsdf_update_voxel(const TsdfFrame& f, const double* sR, const double* st, float wxf,
                                                  float wyf, float wzf, float* tsdf, float* weight, float* color) {
  const double wx = wxf, wy = wyf, wz = wzf;
  const double x = sR[0] * wx + sR[1] * wy + sR[2] * wz + st[0];
  const double y = sR[3] * wx + sR[4] * wy + sR[5] * wz + st[1];
  const double d = sR[6] * wx + sR[7] * wy + sR[8] * wz + st[2];
  if (!(d > 0.0)) return;
  const long long u = llrint(((double)f.fx * x + (double)f.cx * d) / d);     // round-half-even, like Tensor.round()
  const long long v = llrint(((double)f.fy * y + (double)f.cy * d) / d);
  if (u < 0 || v < 0 || u >= f.W || v >= f.H) return;
  const size_t pix = (size_t)v * f.W + (size_t)u;
  float wr;
  const float depth = tsdf_pixel_depth(f, pix, wr);
  float sdf = depth - (float)d;
  if (!(depth > 0.f && depth < f.max_depth && sdf >= -f.trunc)) return;
  sdf = fminf(sdf, f.trunc) / f.trunc;
  const float w = *weight;
  const float wp = w + wr;
  // products and sum rounded separately, like the tensor expression (:280-281) — no FMA contraction
  *tsdf = __fdiv_rn(__fadd_rn(__fmul_rn(w, *tsdf), __fmul_rn(wr, sdf)), wp);
  const size_t hw = (size_t)f.H * f.W;
#pragma unroll
  for (int c = 0; c < 3; c++) {
    const float col = (float)f.rgb[(size_t)c * hw + pix];
    color[c] = __fdiv_rn(__fadd_rn(__fmul_rn(w, color[c]), __fmul_rn(wr, col)), wp);
  }
  *weight = fminf(wp, f.max_weight);
}

// ------------------------------------------------------------------------------------------------------------ ray march
__device__ __forceinline__ float lerp_rn(float a, float b, float t) { return __fadd_rn(a, __fmul_rn(t, __fsub_rn(b, a))); }

// trilinear interpolation of the 8 cell corners, corner n = dx + 2 dy + 4 dz
__device__ __forceinline__ float trilerp8(const float* c, float fx, float fy, float fz) {
  const float c0 = lerp_rn(lerp_rn(c[0], c[1], fx), lerp_rn(c[2], c[3], fx), fy);
  const float c1 = lerp_rn(lerp_rn(c[4], c[5], fx), lerp_rn(c[6], c[7], fx), fy);
  return lerp_rn(c0, c1, fz);
}

// the 8 corners of the cell that holds a hit: tsdf, weight, colour, and the fractions within the cell
struct RayCell {
  float fx, fy, fz;
  float t[8], w[8], c[3][8];
};

struct RayParams {
  float ox, oy, oz, voxel;  // world position of lattice index (0,0,0) and voxel size
  const float* pose;        // [n,7] cam_T_world (t, q_xyzw), DEVICE
  int H, W;
  float fx, fy, cx, cy, min_depth, max_depth, trunc;
  float* depth;             // [n,H,W]
  float* color;             // [n,H,W,3]
  float* weight;            // [n,H,W]
  float* normal;            // [n,H,W,3] or NULL
};

static inline RayParams ray_params(const float* origin3, float voxel, const float* pose, int H, int W, const float* intr4,
                                   float min_depth, float max_depth, float trunc, float* depth, float* color, float* weight,
                                   float* normal) {
  RayParams a{};
  a.ox = origin3[0]; a.oy = origin3[1]; a.oz = origin3[2]; a.voxel = voxel;
  a.pose = pose; a.H = H; a.W = W;
  a.fx = intr4[0]; a.fy = intr4[1]; a.cx = intr4[2]; a.cy = intr4[3];
  a.min_depth = min_depth; a.max_depth = max_depth; a.trunc = trunc;
  a.depth = depth; a.color = color; a.weight = weight; a.normal = normal;
  return a;
}

// One thread per pixel, views over blockIdx.y.  Pixel (u,v) casts z * ((u-cx)/fx, (v-cy)/fy, 1) (camera frame,
// z-depth) from min_depth to max_depth through the trilinear TSDF, in lattice coordinates (world - origin) / voxel.
// Steps: voxel while unobserved or not in front of the surface, max(f * sdf_trunc, voxel) in front of it; the hit is
// the first + -> (<= 0) transition between consecutive observed samples, linearly interpolated.  The volume is the
// accessor A:
//   bool A::sample(const float gq[3], float& f)  — false when the cell at gq is unobserved (a corner has weight
//                                                  <= min_weight); else f = trilinear tsdf
//   void A::hit(const float gq[3], RayCell& c)   — the corners of the hit's cell
template <class A>
__global__ void __launch_bounds__(128) tsdf_raycast_kernel(RayParams a, A vol) {
  __shared__ double sR[9];
  __shared__ float sgo[3];
  const int view = blockIdx.y;
  if (threadIdx.x == 0) {
    const float* p = a.pose + 7 * (size_t)view;
    tsdf_pose_rotation(p, sR);                                      // the fp32 rotation of the pose
    const double t0 = p[0], t1 = p[1], t2 = p[2];
    const float org[3] = {a.ox, a.oy, a.oz};
    for (int c = 0; c < 3; c++) {
      // camera centre -R^T t, then lattice coordinates (world - origin) / voxel
      const float cw = (float)-__dadd_rn(__dadd_rn(__dmul_rn(sR[c], t0), __dmul_rn(sR[3 + c], t1)), __dmul_rn(sR[6 + c], t2));
      sgo[c] = __fdiv_rn(__fsub_rn(cw, org[c]), a.voxel);
    }
  }
  __syncthreads();
  const int pix = blockIdx.x * blockDim.x + threadIdx.x;
  if (pix >= a.H * a.W) return;
  const int u = pix % a.W, v = pix / a.W;
  const float dxc = __fdiv_rn(__fsub_rn((float)u, a.cx), a.fx), dyc = __fdiv_rn(__fsub_rn((float)v, a.cy), a.fy);
  float gd[3];
#pragma unroll
  for (int c = 0; c < 3; c++)
    gd[c] = __fdiv_rn((float)__dadd_rn(__dadd_rn(__dmul_rn(sR[c], (double)dxc), __dmul_rn(sR[3 + c], (double)dyc)), sR[6 + c]),
                      a.voxel);
  const float len = __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(dxc, dxc), __fmul_rn(dyc, dyc)), 1.f));
  auto at = [&](float z, float* gq) {
#pragma unroll
    for (int q = 0; q < 3; q++) gq[q] = __fadd_rn(sgo[q], __fmul_rn(z, gd[q]));
  };

  const int max_steps = (int)ceilf(__fdiv_rn(__fmul_rn(__fsub_rn(a.max_depth, a.min_depth), len), a.voxel)) + 2;
  float z = a.min_depth, z_prev = 0.f, f_prev = 0.f, z_hit = 0.f;
  bool have_prev = false, hit = false;
  for (int s = 0; s < max_steps && z <= a.max_depth; s++) {
    float gq[3], f = 0.f;
    at(z, gq);
    const bool obs = vol.sample(gq, f);
    if (obs && have_prev && f_prev > 0.f && f <= 0.f) {
      z_hit = __fadd_rn(z_prev, __fdiv_rn(__fmul_rn(__fsub_rn(z, z_prev), f_prev), __fsub_rn(f_prev, f)));
      hit = true;
      break;
    }
    const float step = obs && f > 0.f ? fmaxf(__fmul_rn(f, a.trunc), a.voxel) : a.voxel;
    have_prev = obs; f_prev = f; z_prev = z;
    z = __fadd_rn(z, __fdiv_rn(step, len));
  }

  const size_t o = (size_t)view * a.H * a.W + pix;
  if (!hit) {
    a.depth[o] = 0.f; a.weight[o] = 0.f;
    for (int c = 0; c < 3; c++) a.color[3 * o + c] = 0.f;
    if (a.normal) for (int c = 0; c < 3; c++) a.normal[3 * o + c] = 0.f;
    return;
  }
  float gq[3];
  at(z_hit, gq);
  RayCell c;
  vol.hit(gq, c);
  a.depth[o] = z_hit;
  a.weight[o] = trilerp8(c.w, c.fx, c.fy, c.fz);
  for (int ch = 0; ch < 3; ch++) a.color[3 * o + ch] = __fdiv_rn(trilerp8(c.c[ch], c.fx, c.fy, c.fz), 255.f);
  if (a.normal) {
    auto T = [&](int dx, int dy, int dz) { return c.t[dx + 2 * dy + 4 * dz]; };
    auto d = [](float p, float q) { return __fsub_rn(p, q); };
    const float gx = lerp_rn(lerp_rn(d(T(1, 0, 0), T(0, 0, 0)), d(T(1, 1, 0), T(0, 1, 0)), c.fy),
                             lerp_rn(d(T(1, 0, 1), T(0, 0, 1)), d(T(1, 1, 1), T(0, 1, 1)), c.fy), c.fz);
    const float gy = lerp_rn(lerp_rn(d(T(0, 1, 0), T(0, 0, 0)), d(T(1, 1, 0), T(1, 0, 0)), c.fx),
                             lerp_rn(d(T(0, 1, 1), T(0, 0, 1)), d(T(1, 1, 1), T(1, 0, 1)), c.fx), c.fz);
    const float gz = lerp_rn(lerp_rn(d(T(0, 0, 1), T(0, 0, 0)), d(T(1, 0, 1), T(1, 0, 0)), c.fx),
                             lerp_rn(d(T(0, 1, 1), T(0, 1, 0)), d(T(1, 1, 1), T(1, 1, 0)), c.fx), c.fy);
    const float gl = __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(gx, gx), __fmul_rn(gy, gy)), __fmul_rn(gz, gz)));
    a.normal[3 * o + 0] = gl > 0.f ? __fdiv_rn(gx, gl) : 0.f;
    a.normal[3 * o + 1] = gl > 0.f ? __fdiv_rn(gy, gl) : 0.f;
    a.normal[3 * o + 2] = gl > 0.f ? __fdiv_rn(gz, gl) : 0.f;
  }
}

}  // namespace nslam
