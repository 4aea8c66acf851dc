// Path B (instant-NGP style hash-grid NeRF) — shared device code.
// Restates the published instant-ngp / tiny-cuda-nn algorithm (the fork's sources are absent from
// /root/reference, see oracle/ngp.py header: "parity unpinned"); call sites that fix the contract:
// fusion/nerf_fusion.py:57-101 (setup), :285-289 (update_training_images), :299 (frame), :411-424 (render).
#pragma once
#include <cuda_runtime.h>
#include <cuda_fp16.h>
#include <stdint.h>
#include "common.cuh"
#include "../../include/nslam_ngp.h"

namespace ngp {

constexpr int N_LEVELS = 16;
constexpr int N_FEAT = 2;
constexpr int ENC_DIM = N_LEVELS * N_FEAT;  // 32
constexpr int HID = 64;
constexpr int DOUT = 16;                    // density MLP output width (sigma = exp(out[0]))
constexpr int SH_DIM = 16;
constexpr int GRID = 128;                   // occupancy grid resolution per cascade
constexpr int MAX_STEPS = 1024;             // NERF_STEPS
constexpr float SQRT3 = 1.73205080757f;
constexpr float MIN_STEP = SQRT3 / MAX_STEPS;
constexpr float MAX_STEP = MIN_STEP * 128.f * 8.f;
constexpr float MIN_T = 1e-4f;              // transmittance cut-off

// MLP weight blob layout (row-major [in][out], fp32)
constexpr int W1_OFF = 0;                          // [32][64]
constexpr int W2_OFF = W1_OFF + ENC_DIM * HID;     // [64][16]
constexpr int W3_OFF = W2_OFF + HID * DOUT;        // [32][64]
constexpr int W4_OFF = W3_OFF + 32 * HID;          // [64][64]
constexpr int W5_OFF = W4_OFF + HID * HID;         // [64][16] (3 used)
constexpr int W_TOTAL = W5_OFF + HID * 16;         // 10240

struct LevelInfo {
  float scale[N_LEVELS];
  int res[N_LEVELS];
  uint32_t size[N_LEVELS];    // entries in level
  uint32_t offset[N_LEVELS];  // entry offset of level
  int dense[N_LEVELS];        // res^3 <= size
};

static inline LevelInfo level_info(const nslam_ngp_model* m) {
  LevelInfo lv;
  for (int l = 0; l < N_LEVELS; l++) {
    lv.scale[l] = m->scale[l]; lv.res[l] = m->res[l]; lv.size[l] = m->size[l];
    lv.offset[l] = m->offset[l]; lv.dense[l] = m->dense[l];
  }
  return lv;
}

struct Camera {      // per training image
  float c2w[12];     // 3x4 row-major
  float fx, fy, cx, cy;
  int w, h;
};

__device__ __forceinline__ uint32_t grid_index(int x, int y, int z, int res, uint32_t size, int dense) {
  if (dense) return ((uint32_t)x + (uint32_t)y * res + (uint32_t)z * res * res) % size;
  const uint32_t h = ((uint32_t)x * 1u) ^ ((uint32_t)y * 2654435761u) ^ ((uint32_t)z * 805459861u);
  return h % size;
}

// hash-grid encoding of one point (x in [0,1]^3) -> enc[32]
__device__ __forceinline__ void hash_encode(const float x[3], const __half2* __restrict__ grid,
                                            const LevelInfo& lv, float* enc) {
#pragma unroll 4
  for (int l = 0; l < N_LEVELS; l++) {
    const float s = lv.scale[l];
    const float px = fmaf(x[0], s, 0.5f), py = fmaf(x[1], s, 0.5f), pz = fmaf(x[2], s, 0.5f);
    const float fx = floorf(px), fy = floorf(py), fz = floorf(pz);
    const float wx = px - fx, wy = py - fy, wz = pz - fz;
    const int ix = (int)fx, iy = (int)fy, iz = (int)fz;
    const __half2* g = grid + lv.offset[l];
    float a0 = 0.f, a1 = 0.f;
#pragma unroll
    for (int c = 0; c < 8; c++) {
      const int dx = c & 1, dy = (c >> 1) & 1, dz = c >> 2;
      const float w = (dx ? wx : 1.f - wx) * (dy ? wy : 1.f - wy) * (dz ? wz : 1.f - wz);
      const float2 v = __half22float2(__ldg(g + grid_index(ix + dx, iy + dy, iz + dz, lv.res[l], lv.size[l], lv.dense[l])));
      a0 = fmaf(w, v.x, a0); a1 = fmaf(w, v.y, a1);
    }
    enc[2 * l] = a0; enc[2 * l + 1] = a1;
  }
}

// spherical harmonics, degree 4 (tiny-cuda-nn convention)
__device__ __forceinline__ void sh4(const float d[3], float* o) {
  const float x = d[0], y = d[1], z = d[2];
  const float xy = x * y, xz = x * z, yz = y * z, x2 = x * x, y2 = y * y, z2 = z * z;
  o[0] = 0.28209479177387814f;
  o[1] = -0.48860251190291987f * y; o[2] = 0.48860251190291987f * z; o[3] = -0.48860251190291987f * x;
  o[4] = 1.0925484305920792f * xy; o[5] = -1.0925484305920792f * yz;
  o[6] = 0.94617469575755997f * z2 - 0.31539156525251999f; o[7] = -1.0925484305920792f * xz;
  o[8] = 0.54627421529603959f * x2 - 0.54627421529603959f * y2;
  o[9] = 0.59004358992664352f * y * (-3.0f * x2 + y2); o[10] = 2.8906114426405538f * xy * z;
  o[11] = 0.45704579946446572f * y * (1.0f - 5.0f * z2); o[12] = 0.3731763325901154f * z * (5.0f * z2 - 3.0f);
  o[13] = 0.45704579946446572f * x * (1.0f - 5.0f * z2); o[14] = 1.4453057213202769f * z * (x2 - y2);
  o[15] = 0.59004358992664352f * x * (-x2 + 3.0f * y2);
}

// counter-based RNG (pcg hash), uniform in [0,1)
__device__ __forceinline__ uint32_t pcg(uint32_t v) {
  uint32_t s = v * 747796405u + 2891336453u;
  uint32_t w = ((s >> ((s >> 28u) + 4u)) ^ s) * 277803737u;
  return (w >> 22u) ^ w;
}
__device__ __forceinline__ float rnd01(uint32_t a, uint32_t b, uint32_t c) {
  return (float)(pcg(pcg(pcg(a) ^ b) ^ c) >> 8) * (1.0f / 16777216.0f);
}
// j-th cell (j < GRID^3) refreshed in cascade `mip` when only part of the occupancy grid is refreshed: an affine
// permutation of the GRID^3 cells (odd multiplier, power-of-two count) with seeded coefficients, so the cells of one
// refresh are distinct and no two threads update the same cell
static_assert((GRID & (GRID - 1)) == 0, "GRID^3 must be a power of two");
__device__ __forceinline__ uint32_t density_cell(uint32_t seed, int mip, int j) {
  const uint32_t a = pcg(pcg(seed) ^ (uint32_t)(2 * mip)) | 1u, b = pcg(pcg(seed) ^ (uint32_t)(2 * mip + 1));
  return (a * (uint32_t)j + b) & (uint32_t)(GRID * GRID * GRID - 1);
}

// ------------------------------------------------------------------ occupancy grid marching
__device__ __forceinline__ float calc_dt(float t, float cone) {
  return fminf(fmaxf(t * cone, MIN_STEP), MAX_STEP);
}
__device__ __forceinline__ int mip_from_pos(const float p[3], int cascades) {
  const float m = fmaxf(fabsf(p[0] - 0.5f), fmaxf(fabsf(p[1] - 0.5f), fabsf(p[2] - 0.5f)));
  int e;
  frexpf(m, &e);
  return min(max(e + 1, 0), cascades - 1);
}
__device__ __forceinline__ int mip_from_dt(float dt, const float p[3], int cascades) {
  const int mip = mip_from_pos(p, cascades);
  dt *= 2 * GRID;
  if (dt < 1.f) return mip;
  int e;
  frexpf(dt, &e);
  return min(max(max(e, mip), 0), cascades - 1);
}
// linear cell index inside cascade `mip`, or -1 when outside
__device__ __forceinline__ int cell_index(const float p[3], int mip) {
  const float s = scalbnf(1.0f, -mip);
  const int ix = (int)floorf(((p[0] - 0.5f) * s + 0.5f) * GRID);
  const int iy = (int)floorf(((p[1] - 0.5f) * s + 0.5f) * GRID);
  const int iz = (int)floorf(((p[2] - 0.5f) * s + 0.5f) * GRID);
  if (ix < 0 || iy < 0 || iz < 0 || ix >= GRID || iy >= GRID || iz >= GRID) return -1;
  return ix + GRID * (iy + GRID * iz);
}
__device__ __forceinline__ bool occupied(const float p[3], int mip, const uint8_t* __restrict__ bits) {
  const int c = cell_index(p, mip);
  if (c < 0) return false;
  const uint32_t i = (uint32_t)c + (uint32_t)mip * GRID * GRID * GRID;
  return (bits[i >> 3] >> (i & 7)) & 1;
}
// distance to the next voxel boundary of cascade `mip`, then snapped to the step lattice
__device__ __forceinline__ float advance_to_next_voxel(float t, float cone, const float p[3],
                                                       const float d[3], const float id[3], int mip) {
  const float res = scalbnf((float)GRID, -mip);
  float tt = 1e30f;
#pragma unroll
  for (int a = 0; a < 3; a++) {
    const float q = (p[a] - 0.5f) * res + 0.5f * GRID;          // position in cells of this cascade
    const float edge = floorf(q + 0.5f + 0.5f * copysignf(1.f, d[a]));
    tt = fminf(tt, (edge - q) * id[a] / res);
  }
  const float target = t + fmaxf(tt, 0.f);
  do { t += calc_dt(t, cone); } while (t < target);
  return t;
}
// slab intersection with [lo,hi]^3; returns (tmin,tmax), tmax < tmin when missed
__device__ __forceinline__ void ray_aabb(const float o[3], const float id[3], float lo, float hi,
                                         float& tmin, float& tmax) {
  tmin = -1e30f; tmax = 1e30f;
#pragma unroll
  for (int a = 0; a < 3; a++) {
    const float t0 = (lo - o[a]) * id[a], t1 = (hi - o[a]) * id[a];
    tmin = fmaxf(tmin, fminf(t0, t1));
    tmax = fminf(tmax, fmaxf(t0, t1));
  }
}

}  // namespace ngp

// ---- order-independent accumulation
// Float atomics add in whatever order the threads arrive, so their sums differ from run to run in the last bits, and
// training amplifies that.  Gradients that many threads scatter into the same entries are therefore accumulated as
// 64-bit fixed-point integers (integer addition is associative) and converted to fp32 once the scatter is done.
namespace ngp {
__device__ __forceinline__ void fx_add(long long* acc, float v, float scale) {
  const float x = fminf(fmaxf(v * scale, -9.2e18f), 9.2e18f);
  atomicAdd(reinterpret_cast<unsigned long long*>(acc), (unsigned long long)__float2ll_rn(x));
}
// out[i] += acc[i] / scale; acc[i] = 0
static __global__ void fx_flush_kernel(long long* __restrict__ acc, float* __restrict__ out, size_t n, float inv_scale) {
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    const long long v = acc[i];
    if (v != 0) { out[i] += (float)((double)v * (double)inv_scale); acc[i] = 0; }
  }
}
}  // namespace ngp
