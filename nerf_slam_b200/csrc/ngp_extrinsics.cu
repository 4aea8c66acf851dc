// B3 — camera-pose refinement of the NeRF trainer (`ngp.nerf.training.optimize_extrinsics = True`, reference
// fusion/nerf_fusion.py:99; the SLAM path trains with it ON, only process_data switches it off, :123).
//
// The fork's sources are absent (parity unpinned, see oracle/ngp.py); this follows the PUBLISHED instant-ngp scheme
// (testbed_nerf.cu: compute_cam_gradient_train_nerf + the per-camera Adam variables cam_pos_offset / cam_rot_offset):
//   * the photometric / depth loss reaches a camera only through the sample positions  p_k = o + t_k d
//     (the direction's own path through the spherical harmonics is ignored, as upstream does);
//   * dL/dp_k = (d enc / d p)^T dL/d enc : derivative of the trilinear hash-grid interpolation, 16 levels x 8 corners,
//     from the loss-scaled fp16 dL/d enc rows the tensor-core backward leaves in `denc` for the scatter kernel;
//   * per ray  g_o = sum_k dL/dp_k,  g_d = sum_k t_k dL/dp_k ;  per camera  dL/d(translation) += g_o,
//     dL/d(rotation vector) += d x g_d  (left perturbation of the camera orientation about its centre);
//   * Adam (beta 0.9 / 0.99, eps 1e-10, lr 1e-3, L2 1e-4 on the offsets — upstream defaults) on the 6 offsets per camera,
//     effective camera = [Exp(rot_offset) R_base | t_base + pos_offset];  a camera whose base pose is rewritten by the
//     SLAM hand-off starts again from zero offset / zero moments (ingest kernel).
// One WARP per ray (lanes = samples), table gathers from the L2-resident fp16 grid, one atomic per ray and component.
#include "ngp_common.cuh"

namespace ngp {

struct ExtrLevels {
  float scale[N_LEVELS];
  int res[N_LEVELS];
  uint32_t size[N_LEVELS];
  uint32_t offset[N_LEVELS];
  int dense[N_LEVELS];
};

// dL/dx (unit-cube coordinates) of one sample from its dL/d enc row
__device__ __forceinline__ void grid_input_grad(const float x[3], const __half2* __restrict__ grid, const ExtrLevels& lv,
                                                const __half* __restrict__ denc, float g[3]) {
  g[0] = g[1] = g[2] = 0.f;
#pragma unroll 2
  for (int l = 0; l < N_LEVELS; l++) {
    const float s = lv.scale[l];
    const float px = fmaf(x[0], s, 0.5f), py = fmaf(x[1], s, 0.5f), pz = fmaf(x[2], s, 0.5f);
    const float fx = floorf(px), fy = floorf(py), fz = floorf(pz);
    const float wx = px - fx, wy = py - fy, wz = pz - fz;
    const int ix = (int)fx, iy = (int)fy, iz = (int)fz;
    const float d0 = __half2float(denc[2 * l]), d1 = __half2float(denc[2 * l + 1]);
    if (d0 == 0.f && d1 == 0.f) continue;
    const __half2* gl = grid + lv.offset[l];
    float ax = 0.f, ay = 0.f, az = 0.f;
#pragma unroll
    for (int c = 0; c < 8; c++) {
      const int dx = c & 1, dy = (c >> 1) & 1, dz = c >> 2;
      const float2 v = __half22float2(__ldg(gl + grid_index(ix + dx, iy + dy, iz + dz, lv.res[l], lv.size[l], lv.dense[l])));
      const float f = d0 * v.x + d1 * v.y;
      const float ux = dx ? wx : 1.f - wx, uy = dy ? wy : 1.f - wy, uz = dz ? wz : 1.f - wz;
      ax += (dx ? f : -f) * uy * uz;
      ay += (dy ? f : -f) * ux * uz;
      az += (dz ? f : -f) * ux * uy;
    }
    g[0] = fmaf(s, ax, g[0]); g[1] = fmaf(s, ay, g[1]); g[2] = fmaf(s, az, g[2]);
  }
}

// rays [R,16] (see ngp_train.cu), coords [S,7] (unit-cube position, dt, direction), tdist [S], denc [S,32] fp16
// cam_acc [N,6]: += (dL/d translation, dL/d rotation vector) in fixed point (CAM_FX, order-independent sums).
// grid: one warp per ray.
constexpr float CAM_FX = 4294967296.f;            // 2^32: fixed-point scale of the camera-gradient accumulator

__global__ void __launch_bounds__(256)
cam_grad_kernel(const float* __restrict__ rays, int n_rays, const float* __restrict__ coords,
                const float* __restrict__ tdist, const __half* __restrict__ denc, const __half2* __restrict__ grid,
                ExtrLevels lv, float inv_extent, float inv_loss_scale, long long* __restrict__ cam_acc) {
  const int r = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (r >= n_rays) return;
  const float* R = rays + (size_t)r * 16;
  const int base = reinterpret_cast<const int*>(R)[12], n = reinterpret_cast<const int*>(R)[13];
  if (n <= 0) return;
  float go[3] = {0.f, 0.f, 0.f}, gd[3] = {0.f, 0.f, 0.f};
  for (int k = lane; k < n; k += 32) {
    const size_t s = (size_t)(base + k);
    const float x[3] = {coords[s * 7 + 0], coords[s * 7 + 1], coords[s * 7 + 2]};
    float g[3];
    grid_input_grad(x, grid, lv, denc + s * ENC_DIM, g);
    const float t = tdist[s];
#pragma unroll
    for (int a = 0; a < 3; a++) { go[a] += g[a]; gd[a] = fmaf(t, g[a], gd[a]); }
  }
#pragma unroll
  for (int off = 16; off >= 1; off >>= 1)
#pragma unroll
    for (int a = 0; a < 3; a++) {
      go[a] += __shfl_xor_sync(0xffffffffu, go[a], off);
      gd[a] += __shfl_xor_sync(0xffffffffu, gd[a], off);
    }
  if (lane != 0) return;
  // unit cube -> world: p_unit = (p_world - lo) * inv_extent
  const float sc = inv_extent * inv_loss_scale;
  const float d[3] = {R[3], R[4], R[5]};
  const int img = reinterpret_cast<const int*>(R)[14];
  long long* cg = cam_acc + (size_t)img * 6;
  fx_add(cg + 0, sc * go[0], CAM_FX); fx_add(cg + 1, sc * go[1], CAM_FX); fx_add(cg + 2, sc * go[2], CAM_FX);
  fx_add(cg + 3, sc * (d[1] * gd[2] - d[2] * gd[1]), CAM_FX);
  fx_add(cg + 4, sc * (d[2] * gd[0] - d[0] * gd[2]), CAM_FX);
  fx_add(cg + 5, sc * (d[0] * gd[1] - d[1] * gd[0]), CAM_FX);
}

// Adam on the [N,6] offsets + effective cameras.  One thread per camera.
__global__ void cam_adam_apply_kernel(const Camera* __restrict__ base, Camera* __restrict__ eff, float* __restrict__ off,
                                      float* __restrict__ grad, float* __restrict__ m, float* __restrict__ v,
                                      int* __restrict__ steps, int n, float lr, float b1, float b2, float eps, float l2) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  float* g = grad + (size_t)i * 6;
  bool any = false;
#pragma unroll
  for (int k = 0; k < 6; k++) any |= (g[k] != 0.f);
  if (any) {                                   // cameras no ray of this batch came from keep their state
    const int t = ++steps[i];
    const float c1 = 1.f - powf(b1, (float)t), c2 = 1.f - powf(b2, (float)t);
#pragma unroll
    for (int k = 0; k < 6; k++) {
      const size_t j = (size_t)i * 6 + k;
      const float gk = g[k] + l2 * off[j];
      m[j] = b1 * m[j] + (1.f - b1) * gk;
      v[j] = b2 * v[j] + (1.f - b2) * gk * gk;
      off[j] -= lr * (m[j] / c1) / (sqrtf(v[j] / c2) + eps);
      g[k] = 0.f;
    }
  }
  // effective camera: R = Exp(w) R_base, t = t_base + dt
  const float* o = off + (size_t)i * 6;
  const float wx = o[3], wy = o[4], wz = o[5];
  const float th2 = wx * wx + wy * wy + wz * wz, th = sqrtf(th2);
  const float A = th > 1e-6f ? sinf(th) / th : 1.f - th2 / 6.f;
  const float B = th > 1e-6f ? (1.f - cosf(th)) / th2 : 0.5f - th2 / 24.f;
  const float E[3][3] = {{1.f - B * (wy * wy + wz * wz), B * wx * wy - A * wz, B * wx * wz + A * wy},
                         {B * wx * wy + A * wz, 1.f - B * (wx * wx + wz * wz), B * wy * wz - A * wx},
                         {B * wx * wz - A * wy, B * wy * wz + A * wx, 1.f - B * (wx * wx + wy * wy)}};
  Camera c = base[i];
  Camera out = c;
#pragma unroll
  for (int r = 0; r < 3; r++) {
#pragma unroll
    for (int cc = 0; cc < 3; cc++)
      out.c2w[r * 4 + cc] = E[r][0] * c.c2w[0 * 4 + cc] + E[r][1] * c.c2w[1 * 4 + cc] + E[r][2] * c.c2w[2 * 4 + cc];
    out.c2w[r * 4 + 3] = c.c2w[r * 4 + 3] + o[r];
  }
  eff[i] = out;
}

}  // namespace ngp

extern "C" {

/* dL/d(camera) of the batch just back-propagated (rays / coords / tdist / denc of nslam_ngp_batch after
 * nslam_ngp_train_step_tc) accumulated into cam_grad [n_images,6] = (d translation, d rotation vector) through the
 * fixed-point accumulator cam_grad_fx [n_images,6] (zero on entry, zero on return).
 * grid_half / level tables as in nslam_ngp_model; loss_scale = the scale the backward applied to denc. */
int nslam_ngp_cam_grad(const void* grid_half, const float* scale16, const int* res16, const unsigned* size16,
                       const unsigned* offset16, const int* dense16, float aabb_scale, const float* rays, int max_rays,
                       const float* coords, const float* tdist, const void* denc, float loss_scale, float* cam_grad,
                       long long* cam_grad_fx, int n_images, void* stream) {
  using namespace ngp;
  ExtrLevels lv;
  for (int l = 0; l < N_LEVELS; l++) {
    lv.scale[l] = scale16[l]; lv.res[l] = res16[l]; lv.size[l] = size16[l]; lv.offset[l] = offset16[l]; lv.dense[l] = dense16[l];
  }
  if (max_rays <= 0 || n_images <= 0) return 0;
  const int threads = 256, warps_per_block = threads / 32;
  cam_grad_kernel<<<(max_rays + warps_per_block - 1) / warps_per_block, threads, 0, (cudaStream_t)stream>>>(
      rays, max_rays, coords, tdist, (const __half*)denc, (const __half2*)grid_half, lv, 1.f / aabb_scale, 1.f / loss_scale,
      cam_grad_fx);
  NSLAM_CHECK_LAUNCH();
  fx_flush_kernel<<<1, 256, 0, (cudaStream_t)stream>>>(cam_grad_fx, cam_grad, (size_t)n_images * 6, 1.f / CAM_FX);
  NSLAM_CHECK_LAUNCH();
  return 0;
}

/* Adam step on the per-camera offsets [n,6] (pos, rotation vector) from cam_grad (zeroed here), then the effective
 * cameras eff[i] = [Exp(rot_off) R_base | t_base + pos_off] that the ray sampler reads.  lr <= 0: only re-apply. */
int nslam_ngp_cam_adam_apply(const void* base_cams, void* eff_cams, float* offsets, float* cam_grad, float* m, float* v,
                             int* steps, int n, float lr, float beta1, float beta2, float eps, float l2, void* stream) {
  if (n <= 0) return 0;
  ngp::cam_adam_apply_kernel<<<(n + 63) / 64, 64, 0, (cudaStream_t)stream>>>(
      (const ngp::Camera*)base_cams, (ngp::Camera*)eff_cams, offsets, cam_grad, m, v, steps, n, lr, beta1, beta2, eps, l2);
  NSLAM_CHECK_LAUNCH();
  return 0;
}

}  // extern "C"
