// Shared device helpers for the nerf_slam_b200 kernels (sm_90a).
//
// Conventions (same as the reference's droid_backends, src/droid_kernels.cu):
//   pose      = [tx ty tz qx qy qz qw]  (camera-from-world, Hamilton quaternion, w last)
//   intrinsics= [fx fy cx cy] at 1/8 resolution
//   twist     = [tau(3) phi(3)] in "DROID order", [omega(3) t(3)] in "GTSAM order"
#pragma once
#include <cuda_runtime.h>
#include <cuda_fp16.h>
#include <stdint.h>
#include <atomic>

#define NSLAM_MIN_DEPTH 0.25f   // src/droid_kernels.cu:26
#define NSLAM_MAX_DEVICES 64    // per-device caches of kernel attributes (last slot = overflow: always re-set)

#define NSLAM_CHECK_LAUNCH()                         \
  do {                                               \
    cudaError_t e__ = cudaGetLastError();            \
    if (e__ != cudaSuccess) return (int)e__;         \
  } while (0)

namespace nslam {

// Lets `Kernel` launch with `smem` bytes of dynamic shared memory.  cudaFuncAttributeMaxDynamicSharedMemorySize is a
// PER-DEVICE attribute, so what was configured is remembered per device (a process may drive several GPUs, or reset
// one) instead of once per process; each instantiation owns its cache.
template <auto Kernel>
inline cudaError_t ensure_dyn_smem(size_t smem) {
  static std::atomic<size_t> cache[NSLAM_MAX_DEVICES];
  if (smem <= 48 * 1024) return cudaSuccess;
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) return e;
  if (dev < 0 || dev >= NSLAM_MAX_DEVICES) dev = NSLAM_MAX_DEVICES - 1, cache[dev] = 0;   // overflow slot: always set
  if (smem <= cache[dev].load(std::memory_order_acquire)) return cudaSuccess;
  e = cudaFuncSetAttribute(Kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e == cudaSuccess) cache[dev].store(smem, std::memory_order_release);
  return e;
}

// Lays out caller-owned scratch: take(bytes) hands out consecutive regions, each starting 256-byte aligned.  With a
// null base only the total `off` is computed (the size query) and every pointer is null.
struct ScratchCarver {
  char* base;
  size_t off = 0;
  explicit ScratchCarver(void* b) : base((char*)b) {}
  template <typename T = void>
  T* take(size_t bytes) {
    T* p = base ? (T*)(base + off) : nullptr;
    off += (bytes + 255) & ~(size_t)255;
    return p;
  }
};

struct Intr { float fx, fy, cx, cy; };

// ---------------------------------------------------------------- quaternion / SE3
// v' = R(q) v,  computed as v + w*uv + qv x uv with uv = 2 (qv x v)
// (operation order mirrors src/droid_kernels.cu:66-76 so that fp32 results agree)
__device__ __forceinline__ void rot_apply(const float* q, const float* v, float* out) {
  float ux = 2.0f * (q[1] * v[2] - q[2] * v[1]);
  float uy = 2.0f * (q[2] * v[0] - q[0] * v[2]);
  float uz = 2.0f * (q[0] * v[1] - q[1] * v[0]);
  float ox = v[0] + q[3] * ux + (q[1] * uz - q[2] * uy);
  float oy = v[1] + q[3] * uy + (q[2] * ux - q[0] * uz);
  float oz = v[2] + q[3] * uz + (q[0] * uy - q[1] * ux);
  out[0] = ox; out[1] = oy; out[2] = oz;
}

// homogeneous point action: X = [x y z d]  ->  [R xyz + d t, d]
__device__ __forceinline__ void se3_act4(const float* t, const float* q, const float* X, float* Y) {
  rot_apply(q, X, Y);
  Y[3] = X[3];
  Y[0] += X[3] * t[0];
  Y[1] += X[3] * t[1];
  Y[2] += X[3] * t[2];
}

// G_ij = G_j * G_i^{-1}   (src/droid_kernels.cu:107-120)
__device__ __forceinline__ void se3_rel(const float* ti, const float* qi, const float* tj,
                                        const float* qj, float* tij, float* qij) {
  qij[0] = -qj[3] * qi[0] + qj[0] * qi[3] - qj[1] * qi[2] + qj[2] * qi[1];
  qij[1] = -qj[3] * qi[1] + qj[1] * qi[3] - qj[2] * qi[0] + qj[0] * qi[2];
  qij[2] = -qj[3] * qi[2] + qj[2] * qi[3] - qj[0] * qi[1] + qj[1] * qi[0];
  qij[3] =  qj[3] * qi[3] + qj[0] * qi[0] + qj[1] * qi[1] + qj[2] * qi[2];
  float r[3];
  rot_apply(qij, ti, r);
  tij[0] = tj[0] - r[0];
  tij[1] = tj[1] - r[1];
  tij[2] = tj[2] - r[2];
}

// rotation matrix (row major) from quaternion
__device__ __forceinline__ void quat_to_R(const float* q, float* R) {
  const float x = q[0], y = q[1], z = q[2], w = q[3];
  R[0] = 1.f - 2.f * (y * y + z * z); R[1] = 2.f * (x * y - z * w);       R[2] = 2.f * (x * z + y * w);
  R[3] = 2.f * (x * y + z * w);       R[4] = 1.f - 2.f * (x * x + z * z); R[5] = 2.f * (y * z - x * w);
  R[6] = 2.f * (x * z - y * w);       R[7] = 2.f * (y * z + x * w);       R[8] = 1.f - 2.f * (x * x + y * y);
}

// A(6x6, row major) = Ad(G)^T for twist order (tau, phi):
//   Ad(G) = [[R, [t]x R], [0, R]]   =>   Ad^T = [[R^T, 0], [-R^T [t]x, R^T]]
// so that (Ad^T X)[0:3] = R^T Xa,  (Ad^T X)[3:6] = R^T Xb + R^T (Xa x t)
// (this is what adjSE3(t,q,X,Y) of src/droid_kernels.cu:87-104 evaluates per pixel).
__device__ __forceinline__ void se3_adjT_matrix(const float* t, const float* q, float* A) {
  float R[9];
  quat_to_R(q, R);
  // R^T
  float Rt[9] = {R[0], R[3], R[6], R[1], R[4], R[7], R[2], R[5], R[8]};
  // K = -[t]x  so that Xa x t = K Xa  (Xa x t = -(t x Xa))
  float K[9] = {0.f, t[2], -t[1], -t[2], 0.f, t[0], t[1], -t[0], 0.f};
  for (int r = 0; r < 3; r++)
    for (int c = 0; c < 3; c++) {
      A[r * 6 + c] = Rt[r * 3 + c];
      A[r * 6 + 3 + c] = 0.f;
      float s = 0.f;
      for (int k = 0; k < 3; k++) s += Rt[r * 3 + k] * K[k * 3 + c];
      A[(3 + r) * 6 + c] = s;
      A[(3 + r) * 6 + 3 + c] = Rt[r * 3 + c];
    }
}

// SO3 / SE3 exponential, twist = [tau, phi]   (src/droid_kernels.cu:123-188)
__device__ __forceinline__ void so3_exp(const float* phi, float* q) {
  float th2 = phi[0] * phi[0] + phi[1] * phi[1] + phi[2] * phi[2];
  float th4 = th2 * th2;
  float th = sqrtf(th2);
  float imag, real;
  if (th2 < 1e-8f) {
    imag = 0.5f - (1.0f / 48.0f) * th2 + (1.0f / 3840.0f) * th4;
    real = 1.0f - (1.0f / 8.0f) * th2 + (1.0f / 384.0f) * th4;
  } else {
    imag = sinf(0.5f * th) / th;
    real = cosf(0.5f * th);
  }
  q[0] = imag * phi[0]; q[1] = imag * phi[1]; q[2] = imag * phi[2]; q[3] = real;
}

__device__ __forceinline__ void cross3(const float* a, const float* b, float* c) {
  float x = a[1] * b[2] - a[2] * b[1];
  float y = a[2] * b[0] - a[0] * b[2];
  float z = a[0] * b[1] - a[1] * b[0];
  c[0] = x; c[1] = y; c[2] = z;
}

__device__ __forceinline__ void se3_exp(const float* xi, float* t, float* q) {
  so3_exp(xi + 3, q);
  float tau[3] = {xi[0], xi[1], xi[2]};
  const float* phi = xi + 3;
  float th2 = phi[0] * phi[0] + phi[1] * phi[1] + phi[2] * phi[2];
  float th = sqrtf(th2);
  t[0] = tau[0]; t[1] = tau[1]; t[2] = tau[2];
  if (th > 1e-4f) {
    float a = (1.f - cosf(th)) / th2;
    cross3(phi, tau, tau);
    t[0] += a * tau[0]; t[1] += a * tau[1]; t[2] += a * tau[2];
    float b = (th - sinf(th)) / (th * th2);
    cross3(phi, tau, tau);
    t[0] += b * tau[0]; t[1] += b * tau[1]; t[2] += b * tau[2];
  }
}

// quaternion product a*b (Hamilton, w last)
__device__ __forceinline__ void quat_mul(const float* a, const float* b, float* o) {
  float x = a[3] * b[0] + a[0] * b[3] + a[1] * b[2] - a[2] * b[1];
  float y = a[3] * b[1] + a[1] * b[3] + a[2] * b[0] - a[0] * b[2];
  float z = a[3] * b[2] + a[2] * b[3] + a[0] * b[1] - a[1] * b[0];
  float w = a[3] * b[3] - a[0] * b[0] - a[1] * b[1] - a[2] * b[2];
  o[0] = x; o[1] = y; o[2] = z; o[3] = w;
}

// ---------------------------------------------------------------- reductions
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// block-wide sum of NV values per thread; result valid in thread 0 (vals[] overwritten).
// smem must hold NV * (blockDim.x/32) floats.
template <int NV>
__device__ __forceinline__ void block_sum(float* vals, float* smem) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, nw = blockDim.x >> 5;
#pragma unroll
  for (int i = 0; i < NV; i++) {
    float v = warp_sum(vals[i]);
    if (lane == 0) smem[i * nw + wid] = v;
  }
  __syncthreads();
  if (threadIdx.x < 32) {
#pragma unroll 1
    for (int i = 0; i < NV; i++) {
      float v = (lane < nw) ? smem[i * nw + lane] : 0.f;
      v = warp_sum(v);
      if (lane == 0) smem[i * nw] = v;
    }
  }
  __syncthreads();
  if (threadIdx.x == 0) {
#pragma unroll
    for (int i = 0; i < NV; i++) vals[i] = smem[i * nw];
  }
  __syncthreads();
}

}  // namespace nslam
