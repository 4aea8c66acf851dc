// §8(f3) — Sigma- / TSDF-fusion consumer of the SLAM packet (upsampled depth + depth covariance per keyframe).
//
// Replaces TsdfFusion.custom_volume_integrate (reference fusion/tsdf_fusion.py:185-302), which drives Open3D's hashed
// VoxelBlockGrid from Python: per keyframe it activates the 16^3 blocks touched by the depth map, gathers their voxel
// coordinates, and runs ~40 Open3D tensor ops with four device synchronisations.  Open3D is absent from the reference
// tree and from this image (parity of its block activation is unpinned); the per-voxel update rule is in the reference's
// own Python and is followed statement by statement:
//     xyz = R v + t;  uvd = K xyz;  d = uvd.z;  u = round(uvd.x / d), v = round(uvd.y / d)            (:246-252)
//     keep  d > 0, 0 <= u < W, 0 <= v < H                                                               (:255)
//     sdf = depth[v,u] - d;  inlier = depth in (0, max_depth) and sdf >= -trunc                        (:259-262)
//     sdf = min(sdf, trunc) / trunc                                                                     (:264-265)
//     wr = weight_reading[v,u];  wp = w + wr                                                            (:274-277)
//     tsdf = (w tsdf + wr sdf) / wp;  color = (w color + wr rgb) / wp;  w = min(wp, max_weight)         (:280-294)
//
// Design: 80 GB of HBM make the hashing unnecessary for the reference's own extent ("a 6 m room with a dense
// 512^3 grid", :66) — the volume is a DENSE grid (tsdf, weight fp32 + colour 3 x fp32 = 20 B/voxel, 2.7 GB at 512^3),
// one thread per voxel, one launch per keyframe; depth = 1 / inverse depth, weight = 1 / sqrt(depth variance) and the
// depth mask are evaluated on the fly from the packet's tensors (the reference materialises three images per frame).
// The set of updated voxels is every grid voxel that passes the reference's own tests (a superset of its activated
// blocks: voxels far in front of the surface receive the saturated value +1 there only if their block was activated).
// HBM-bound: 20 B read + 20 B written per voxel inside the frustum, 4 B otherwise.
#include "common.cuh"

namespace nslam {

struct TsdfGrid {
  float* tsdf;      // [nz][ny][nx]
  float* weight;
  float* color;     // [nz][ny][nx][3]
  int nx, ny, nz;
  float ox, oy, oz; // world coordinates of voxel (0,0,0)
  float voxel;
};

struct TsdfFrame {
  const float* idepth;      // [H,W] inverse depth (upsampled)
  const float* depth_cov;   // [H,W] depth variance, or NULL = uniform weight 1
  const unsigned char* rgb; // [3,H,W] u8
  int H, W;
  float fx, fy, cx, cy;
  const float* pose;        // cam_T_world [t, q_xyzw] on the DEVICE (x_cam = R(q) x_world + t): no host copy of the pose
  float max_depth, trunc, max_weight, max_sigma;
};

__global__ void __launch_bounds__(256)
tsdf_integrate_kernel(TsdfGrid g, TsdfFrame f) {
  __shared__ double sR[9], st[3];
  if (threadIdx.x == 0) {
    // SE3(poses).matrix() is a float32 matrix that build_volume promotes to float64 (:186, :209): round the rotation to fp32
    const double qx = f.pose[3], qy = f.pose[4], qz = f.pose[5], qw = f.pose[6];
    const double R[9] = {1 - 2 * (qy * qy + qz * qz), 2 * (qx * qy - qz * qw), 2 * (qx * qz + qy * qw),
                         2 * (qx * qy + qz * qw), 1 - 2 * (qx * qx + qz * qz), 2 * (qy * qz - qx * qw),
                         2 * (qx * qz - qy * qw), 2 * (qy * qz + qx * qw), 1 - 2 * (qx * qx + qy * qy)};
    for (int i = 0; i < 9; i++) sR[i] = (double)(float)R[i];
    st[0] = f.pose[0]; st[1] = f.pose[1]; st[2] = f.pose[2];
  }
  __syncthreads();
  const int ix = blockIdx.x * blockDim.x + threadIdx.x;
  const int iy = blockIdx.y, iz = blockIdx.z;
  if (ix >= g.nx) return;
  // the reference's voxel coordinates are float32 tensors (metric: voxel_size * index, lattice through `origin`), promoted to
  // float64 together with extrinsic and intrinsic for the projection (:243-252): float32 product, float32 sum, no contraction
  const double wx = (double)__fadd_rn(__fmul_rn(g.voxel, (float)ix), g.ox), wy = (double)__fadd_rn(__fmul_rn(g.voxel, (float)iy), g.oy),
               wz = (double)__fadd_rn(__fmul_rn(g.voxel, (float)iz), g.oz);
  const double x = sR[0] * wx + sR[1] * wy + sR[2] * wz + st[0];
  const double y = sR[3] * wx + sR[4] * wy + sR[5] * wz + st[1];
  const double d = sR[6] * wx + sR[7] * wy + sR[8] * wz + st[2];
  if (!(d > 0.0)) return;
  const long long u = llrint(((double)f.fx * x + (double)f.cx * d) / d);     // round-half-even, like Tensor.round()
  const long long v = llrint(((double)f.fy * y + (double)f.cy * d) / d);
  if (u < 0 || v < 0 || u >= f.W || v >= f.H) return;
  const size_t pix = (size_t)v * f.W + (size_t)u;
  float depth = 1.0f / f.idepth[pix];
  float wr = 1.0f;
  if (f.depth_cov) {
    const float cov = f.depth_cov[pix];
    wr = sqrtf(1.0f / cov);                                   // cov.pow(-1).sqrt()  (:196)
    if (!(sqrtf(cov) < f.max_sigma)) depth = f.max_depth + 1.0f;   // masked pixels are pushed beyond max_depth (:201-203, :549)
  }
  float sdf = depth - (float)d;
  if (!(depth > 0.f && depth < f.max_depth && sdf >= -f.trunc)) return;
  sdf = fminf(sdf, f.trunc) / f.trunc;
  const size_t vi = ((size_t)iz * g.ny + iy) * g.nx + ix;
  const float w = g.weight[vi];
  const float wp = w + wr;
  // products and sum rounded separately, like the tensor expression (:280-281) — no FMA contraction
  g.tsdf[vi] = __fdiv_rn(__fadd_rn(__fmul_rn(w, g.tsdf[vi]), __fmul_rn(wr, sdf)), wp);
  const size_t hw = (size_t)f.H * f.W;
#pragma unroll
  for (int c = 0; c < 3; c++) {
    const float col = (float)f.rgb[(size_t)c * hw + pix];
    g.color[vi * 3 + c] = __fdiv_rn(__fadd_rn(__fmul_rn(w, g.color[vi * 3 + c]), __fmul_rn(wr, col)), wp);
  }
  g.weight[vi] = fminf(wp, f.max_weight);
}

}  // namespace nslam

extern "C" {

/* One keyframe into the dense volume (fusion/tsdf_fusion.py:185-302 per-voxel rule, see the head of this file).
 * tsdf / weight [nz,ny,nx] fp32, color [nz,ny,nx,3] fp32; origin = world position of voxel (0,0,0); cam_T_world: DEVICE
 * [7] = (t, q_xyzw) as the packet carries it; idepth_up [H,W], depth_cov_up [H,W] or NULL (uniform weights = "tsdf",
 * variance weights = "sigma"), rgb u8 [3,H,W]: DEVICE.  intr = fx, fy, cx, cy at full resolution (HOST). */
int nslam_tsdf_integrate(float* tsdf, float* weight, float* color, int nx, int ny, int nz, const float* origin3_host,
                         float voxel_size, const float* idepth_up, const float* depth_cov_up, const unsigned char* rgb_chw,
                         int H, int W, const float* intr4_host, const float* cam_T_world_tq, float max_depth,
                         float sdf_trunc, float max_weight, float max_depth_sigma, void* stream) {
  using namespace nslam;
  if (nx <= 0 || ny <= 0 || nz <= 0 || ny > 65535 || nz > 65535) return (int)cudaErrorInvalidValue;
  TsdfGrid g{tsdf, weight, color, nx, ny, nz, origin3_host[0], origin3_host[1], origin3_host[2], voxel_size};
  TsdfFrame f{};
  f.idepth = idepth_up; f.depth_cov = depth_cov_up; f.rgb = rgb_chw; f.H = H; f.W = W;
  f.fx = intr4_host[0]; f.fy = intr4_host[1]; f.cx = intr4_host[2]; f.cy = intr4_host[3];
  f.pose = cam_T_world_tq;
  f.max_depth = max_depth; f.trunc = sdf_trunc; f.max_weight = max_weight; f.max_sigma = max_depth_sigma;
  dim3 grid((nx + 255) / 256, ny, nz);
  tsdf_integrate_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(g, f);
  NSLAM_CHECK_LAUNCH();
  return 0;
}

}  // extern "C"
