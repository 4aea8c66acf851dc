// Path B — NeRF training step + rendering kernels (instant-NGP style), sm_90a.
//
//   B3  one training step (what pyngp's Testbed.frame() does per call, fusion/nerf_fusion.py:299):
//       sample rays over the training images -> occupancy-grid ray march -> hash-grid encode ->
//       density MLP -> SH -> rgb MLP -> volume rendering + Huber RGB loss + covariance-weighted
//       depth loss (fusion/nerf_fusion.py:99-101,285-289) -> backward -> Adam.
//   B4  rendering of a camera view (Testbed.render, fusion/nerf_fusion.py:411-424): same march,
//       forward and compositing without loss.
//
// Kernel structure (all launches are sized for the buffer capacity and read the live sample
// count from a device counter, so a step never synchronises the host):
//   ngp_sample_rays    warp per ray: 32 lattice points per iteration through the cascaded occupancy bitfield,
//                      contiguous sample ranges claimed with one atomic per ray
//   ngp_forward        thread per sample: 128 independent hash-table gathers (table is fp16 and
//                      L2-resident: 16 levels x 2^19 x 4 B = 33 MB << 126 MB), then the two tiny
//                      MLPs with weights broadcast from shared memory (float4 LDS, 64 register
//                      accumulators per thread), activations staged feature-major in smem
//   ngp_loss           thread per ray: compositing forward + closed-form backward (dL/d rgb,sigma)
//   ngp_backward       persistent CTAs over 128-sample tiles: recompute forward, back-propagate,
//                      weight gradients as 4x4 register-blocked outer products over the tile
//                      (kept in registers across tiles, one atomic flush per CTA), hash-grid
//                      gradients scattered with vector atomics (red.global.add.v2.f32)
//   ngp_adam           fused Adam (+L2 on the MLP, zero-gradient skip on hash entries) writing
//                      the fp32 master and the fp16 compute copy
#include "ngp_common.cuh"
#include "../../include/nslam_ngp.h"

#define NGP_CHECK_LAUNCH()                        \
  do {                                            \
    cudaError_t e__ = cudaGetLastError();         \
    if (e__ != cudaSuccess) return (int)e__;      \
  } while (0)

namespace ngp {

constexpr int TILE = 128;
constexpr int LD = TILE + 1;  // feature-major staging [feature][LD]

struct Scene {
  float aabb_lo, aabb_hi;   // render/training box in world units: 0.5 -/+ aabb_scale/2
  float inv_extent;         // 1/(hi-lo)
  int cascades;
  float cone;               // cone angle constant (1/256 when aabb_scale > 1)
  float near;               // near distance
};

// ------------------------------------------------------------------------------------------
// dense layer helpers (thread == sample, column `tid` of the feature-major staging buffer)
template <int K, int N, int WLD>
__device__ __forceinline__ void dense_fwd(const float* __restrict__ S, const float* __restrict__ W,
                                          float (&acc)[N], int tid) {
#pragma unroll
  for (int n = 0; n < N; n++) acc[n] = 0.f;
#pragma unroll 2
  for (int k = 0; k < K; k++) {
    const float a = S[k * LD + tid];
    const float4* w4 = reinterpret_cast<const float4*>(W + k * WLD);
#pragma unroll
    for (int n4 = 0; n4 < N / 4; n4++) {
      const float4 w = w4[n4];
      acc[4 * n4 + 0] = fmaf(a, w.x, acc[4 * n4 + 0]);
      acc[4 * n4 + 1] = fmaf(a, w.y, acc[4 * n4 + 1]);
      acc[4 * n4 + 2] = fmaf(a, w.z, acc[4 * n4 + 2]);
      acc[4 * n4 + 3] = fmaf(a, w.w, acc[4 * n4 + 3]);
    }
  }
}
// out[k] = sum_n W[k][n] d[n]  written to O[k][tid]  (d in registers)
template <int K, int N, int WLD>
__device__ __forceinline__ void dense_bwd_in(const float (&d)[N], const float* __restrict__ W,
                                             float* __restrict__ O, int tid) {
#pragma unroll 2
  for (int k = 0; k < K; k++) {
    const float4* w4 = reinterpret_cast<const float4*>(W + k * WLD);
    float s = 0.f;
#pragma unroll
    for (int n4 = 0; n4 < N / 4; n4++) {
      const float4 w = w4[n4];
      s = fmaf(w.x, d[4 * n4 + 0], s); s = fmaf(w.y, d[4 * n4 + 1], s);
      s = fmaf(w.z, d[4 * n4 + 2], s); s = fmaf(w.w, d[4 * n4 + 3], s);
    }
    O[k * LD + tid] = s;
  }
}
// dW[k][n] += sum_rows A[k][row] D[n][row], thread owns NB 4x4 blocks (block b = tid + j*TILE)
template <int K, int N, int NB>
__device__ __forceinline__ void outer_acc(const __half* __restrict__ A, const float* __restrict__ D,
                                          float (&acc)[NB][16], int tid, int rows) {
  constexpr int NBLK = (K / 4) * (N / 4);
#pragma unroll
  for (int j = 0; j < NB; j++) {
    const int b = tid + j * TILE;
    if (b < NBLK) {
      const int k0 = (b / (N / 4)) * 4, n0 = (b % (N / 4)) * 4;
      for (int r = 0; r < rows; r++) {
        float a[4], d[4];
#pragma unroll
        for (int i = 0; i < 4; i++) { a[i] = __half2float(A[(k0 + i) * LD + r]); d[i] = D[(n0 + i) * LD + r]; }
#pragma unroll
        for (int i = 0; i < 4; i++)
#pragma unroll
          for (int q = 0; q < 4; q++) acc[j][i * 4 + q] = fmaf(a[i], d[q], acc[j][i * 4 + q]);
      }
    }
  }
}
template <int K, int N, int NB, int WLD>
__device__ __forceinline__ void outer_flush(const float (&acc)[NB][16], float* __restrict__ G, int tid) {
  constexpr int NBLK = (K / 4) * (N / 4);
#pragma unroll
  for (int j = 0; j < NB; j++) {
    const int b = tid + j * TILE;
    if (b < NBLK) {
      const int k0 = (b / (N / 4)) * 4, n0 = (b % (N / 4)) * 4;
#pragma unroll
      for (int i = 0; i < 4; i++)
#pragma unroll
        for (int q = 0; q < 4; q++) atomicAdd(G + (k0 + i) * WLD + n0 + q, acc[j][i * 4 + q]);
    }
  }
}

// ------------------------------------------------------------------------------------------
// ray generation + marching.  rays: [R] records of 16 floats:
//   0-2 origin, 3-5 dir (unit), 6 inv_len (z-depth = t*inv_len), 7 target depth, 8 depth cov,
//   9-11 target rgb, 12 (int) sample base, 13 (int) n samples, 14 (int) image, 15 (int) pixel
struct ImageStore {
  const __half* rgba;     // [N,H,W,4] linear, premultiplied
  const float* depth;     // [N,H,W]  (<= 0: no depth)
  const float* depth_cov; // [N,H,W]
  const Camera* cams;     // [N]
  const int* active;      // [n_active] slot ids used for training
  int n_active, H, W;
};

__device__ __forceinline__ void make_ray(const Camera& c, float px, float py, float* o, float* d,
                                         float& inv_len) {
  const float dx = (px - c.cx) / c.fx, dy = (py - c.cy) / c.fy;
  const float len = sqrtf(dx * dx + dy * dy + 1.f);
  inv_len = 1.f / len;
  const float cx_ = dx * inv_len, cy_ = dy * inv_len, cz_ = inv_len;
  for (int r = 0; r < 3; r++) {
    d[r] = c.c2w[r * 4 + 0] * cx_ + c.c2w[r * 4 + 1] * cy_ + c.c2w[r * 4 + 2] * cz_;
    o[r] = c.c2w[r * 4 + 3];
  }
}

// Warp-cooperative march (one warp = one ray; all lanes hold identical o, d, jitter).
// The step lattice t_{k+1} = t_k + calc_dt(t_k) does not depend on occupancy, so the warp tests 32
// consecutive lattice points per iteration (one dependent bitfield load per 32 steps instead of one
// per step): lane l rebuilds t_{base+l} with the same serial recurrence a single thread would run
// (bit-identical t), the ballot of occupied points is kept in registers (lane c%32 holds chunk c),
// the ray's contiguous sample range is either reserved with ONE atomicAdd (render) or given by the caller
// (training: a count pass, an ordered scan, then this write pass, so that the sample layout is the same on every
// run), and the write pass replays the kept masks without touching the bitfield again.  A sample is emitted for every lattice point that
// lies in an occupied cell of its cascade, up to max_n samples / 4096 lattice points per ray.
constexpr int MW_SLOTS = 4;                 // 4 x 32 chunks x 32 points

__device__ __forceinline__ float lattice_t(float tbase, int lane, float cone) {
  float t = tbase;
  for (int i = 0; i < lane; i++) t += calc_dt(t, cone);
  return t;
}

// returns the number of samples (uniform over the warp); writes them at coords/tdist[base...].
// base_in: -1 = reserve the range with an atomic on counters[0]; -2 = count only (nothing is written);
// >= 0 = write at this offset
__device__ int march_warp(const float* o, const float* d, const Scene& sc, const uint8_t* __restrict__ bits,
                          float jitter, int max_n, int max_samples, int* __restrict__ counters,
                          float* __restrict__ coords, float* __restrict__ tdist, int& base_out, int base_in = -1) {
  const int lane = threadIdx.x & 31;
  const float id[3] = {1.f / d[0], 1.f / d[1], 1.f / d[2]};
  float tmin, tmax;
  ray_aabb(o, id, sc.aabb_lo, sc.aabb_hi, tmin, tmax);
  if (tmax <= fmaxf(tmin, 0.f)) return 0;
  float tbase = fmaxf(tmin, sc.near) + 1e-6f;
  tbase += calc_dt(tbase, sc.cone) * jitter;
  uint32_t mk[MW_SLOTS];
  float tb[MW_SLOTS];
  int n = 0, nchunks = 0;
  bool done = false;
#pragma unroll
  for (int slot = 0; slot < MW_SLOTS; slot++) {
    mk[slot] = 0u; tb[slot] = 0.f;
    for (int j = 0; j < 32 && !done; j++) {
      if (tbase >= tmax || n >= max_n) { done = true; break; }
      const float t = lattice_t(tbase, lane, sc.cone);
      const float dt = calc_dt(t, sc.cone);
      bool occ = false;
      if (t < tmax) {
        const float p[3] = {fmaf(d[0], t, o[0]), fmaf(d[1], t, o[1]), fmaf(d[2], t, o[2])};
        occ = occupied(p, mip_from_dt(dt, p, sc.cascades), bits);
      }
      uint32_t m = __ballot_sync(0xffffffffu, occ);
      const int c = __popc(m);
      if (n + c > max_n) m &= (1u << __fns(m, 0, max_n - n + 1)) - 1u;   // keep the first max_n - n points
      n += __popc(m);
      if (lane == j) { mk[slot] = m; tb[slot] = tbase; }
      nchunks++;
      tbase = __shfl_sync(0xffffffffu, t + dt, 31);
    }
  }
  if (n == 0 || base_in == -2) return n;
  int base = base_in;
  if (base_in == -1) {
    if (lane == 0) {
      base = atomicAdd(&counters[0], n);
      if (base + n > max_samples) { atomicSub(&counters[0], n); base = -1; }
    }
    base = __shfl_sync(0xffffffffu, base, 0);
  }
  if (base < 0) return 0;
  base_out = base;
  int off = 0, ci = 0;
#pragma unroll
  for (int slot = 0; slot < MW_SLOTS; slot++) {
    for (int j = 0; j < 32 && ci < nchunks; j++, ci++) {
      const uint32_t m = __shfl_sync(0xffffffffu, mk[slot], j);
      const float tbs = __shfl_sync(0xffffffffu, tb[slot], j);
      if (m == 0u) continue;
      if ((m >> lane) & 1u) {
        const float t = lattice_t(tbs, lane, sc.cone);
        const float dt = calc_dt(t, sc.cone);
        const int k = base + off + __popc(m & ((1u << lane) - 1u));
        float* s = coords + (size_t)k * 7;
        s[0] = (fmaf(d[0], t, o[0]) - sc.aabb_lo) * sc.inv_extent;
        s[1] = (fmaf(d[1], t, o[1]) - sc.aabb_lo) * sc.inv_extent;
        s[2] = (fmaf(d[2], t, o[2]) - sc.aabb_lo) * sc.inv_extent;
        s[3] = dt; s[4] = d[0]; s[5] = d[1]; s[6] = d[2];
        tdist[k] = t;
      }
      off += __popc(m);
    }
  }
  return n;
}

// counters: [0] samples used, [1] rays kept, [2] rays tried.  One WARP per ray.
// Two passes: count (R[13] = samples of ray i), then sample_scan_kernel, then write (at R[12], R[13] samples).
__global__ void sample_rays_kernel(ImageStore st, Scene sc, const uint8_t* __restrict__ bits,
                                   int n_rays, uint32_t seed, int max_samples,
                                   float* __restrict__ rays, float* __restrict__ coords,
                                   float* __restrict__ tdist, int* __restrict__ counters, int count_pass) {
  const int i = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (i >= n_rays) return;
  float* R = rays + (size_t)i * 16;
  const int planned = count_pass ? 0 : reinterpret_cast<const int*>(R)[13];
  __syncwarp();
  if (count_pass && lane == 0) reinterpret_cast<int*>(R)[13] = 0;
  if (st.n_active <= 0 || (!count_pass && planned == 0)) return;
  const int img = st.active[min((int)(rnd01(seed, i, 1) * st.n_active), st.n_active - 1)];
  const int px = min((int)(rnd01(seed, i, 2) * st.W), st.W - 1);
  const int py = min((int)(rnd01(seed, i, 3) * st.H), st.H - 1);
  float o[3], d[3], inv_len;
  make_ray(st.cams[img], px + 0.5f, py + 0.5f, o, d, inv_len);
  const float jit = rnd01(seed, i, 4);
  int base = 0;
  const int n = march_warp(o, d, sc, bits, jit, MAX_STEPS, max_samples, counters, coords, tdist, base,
                           count_pass ? -2 : reinterpret_cast<const int*>(R)[12]);
  if (count_pass) {
    if (lane == 0) reinterpret_cast<int*>(R)[13] = n;
    return;
  }
  if (n == 0 || lane != 0) return;
  const size_t pix = ((size_t)img * st.H + py) * st.W + px;
  R[0] = o[0]; R[1] = o[1]; R[2] = o[2]; R[3] = d[0]; R[4] = d[1]; R[5] = d[2]; R[6] = inv_len;
  R[7] = st.depth ? st.depth[pix] : -1.f;
  R[8] = st.depth_cov ? st.depth_cov[pix] : 1.f;
  const __half* c = st.rgba + pix * 4;
  R[9] = __half2float(c[0]); R[10] = __half2float(c[1]); R[11] = __half2float(c[2]);
  reinterpret_cast<int*>(R)[12] = base;
  reinterpret_cast<int*>(R)[13] = n;
  reinterpret_cast<int*>(R)[14] = img;
  reinterpret_cast<int*>(R)[15] = py * st.W + px;
}

// between the two passes of sample_rays_kernel: exclusive scan of the per-ray counts in ray order; rays are kept
// while the running total fits max_samples (R[12] = offset, R[13] = count, 0 = dropped); counters[0] / [1] =
// samples / rays kept.  One block.
__global__ void __launch_bounds__(1024)
sample_scan_kernel(float* __restrict__ rays, int n_rays, int max_samples, int* __restrict__ counters) {
  __shared__ int wsum[32];
  __shared__ int carry, kept, used;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  if (tid == 0) { carry = 0; kept = 0; used = 0; }
  __syncthreads();
  for (int c0 = 0; c0 < n_rays; c0 += 1024) {
    const int i = c0 + tid;
    int* R = reinterpret_cast<int*>(rays + (size_t)i * 16);
    const int n = i < n_rays ? R[13] : 0;
    int x = n;                                              // inclusive scan: warp, then across warps
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const int y = __shfl_up_sync(0xffffffffu, x, o); if (lane >= o) x += y; }
    if (lane == 31) wsum[warp] = x;
    __syncthreads();
    if (warp == 0) {
      int w = wsum[lane];
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) { const int y = __shfl_up_sync(0xffffffffu, w, o); if (lane >= o) w += y; }
      wsum[lane] = w;
    }
    __syncthreads();
    const int incl = carry + x + (warp ? wsum[warp - 1] : 0);
    const bool keep = n > 0 && incl <= max_samples;
    if (i < n_rays) { R[12] = incl - n; R[13] = keep ? n : 0; }
    if (keep) atomicMax(&used, incl);                       // kept rays form a prefix: the last one ends the range
    const int nk = __syncthreads_count(keep);
    if (tid == 1023) carry = incl;
    if (tid == 0) kept += nk;
    __syncthreads();
  }
  if (tid == 0) {
    counters[0] = used;
    counters[1] = kept;
  }
}

// rays of one image tile (render): ray r <-> pixel (x0 + r % tw, y0 + r / tw).  One WARP per ray.
__global__ void render_rays_kernel(Camera cam, Scene sc, const uint8_t* __restrict__ bits, int x0,
                                   int y0, int tw, int th, int max_samples, int max_per_ray,
                                   float* __restrict__ rays, float* __restrict__ coords,
                                   float* __restrict__ tdist, int* __restrict__ counters) {
  const int i = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (i >= tw * th) return;
  float* R = rays + (size_t)i * 16;
  if (lane == 0) reinterpret_cast<int*>(R)[13] = 0;
  const int px = x0 + i % tw, py = y0 + i / tw;
  if (px >= cam.w || py >= cam.h) return;
  float o[3], d[3], inv_len;
  make_ray(cam, px + 0.5f, py + 0.5f, o, d, inv_len);
  if (lane == 0) R[6] = inv_len;
  int base = 0;
  const int n = march_warp(o, d, sc, bits, 0.f, max_per_ray, max_samples, counters, coords, tdist, base);
  if (n == 0 || lane != 0) return;
  reinterpret_cast<int*>(R)[12] = base;
  reinterpret_cast<int*>(R)[13] = n;
}

// ------------------------------------------------------------------------------------------
// forward: one thread per sample. smem: weights (W_TOTAL floats) + staging S [64][LD]
struct NetState {
  float o[DOUT];    // density MLP output
  float rgbraw[4];  // rgb MLP output (pre-sigmoid), [3] unused
};

// runs the network for the calling thread's sample; leaves h3 (last hidden) in S.
// If KEEP != nullptr the layer inputs are additionally stored for the backward pass:
//   KEEP (fp16) rows: [0,32) enc, [32,96) h1, [96,128) in2, [128,192) h2, [192,256) h3  (feature-major, LD)
__device__ __forceinline__ void net_forward(const float* c7, const __half2* __restrict__ grid,
                                            const LevelInfo& lv, const float* __restrict__ sW,
                                            float* __restrict__ S, __half* __restrict__ KEEP, int tid,
                                            NetState& ns) {
  {
    float enc[ENC_DIM];
    hash_encode(c7, grid, lv, enc);
#pragma unroll
    for (int k = 0; k < ENC_DIM; k++) { S[k * LD + tid] = enc[k]; if (KEEP) KEEP[k * LD + tid] = __float2half_rn(enc[k]); }
  }
  {
    float h[HID];
    dense_fwd<ENC_DIM, HID, HID>(S, sW + W1_OFF, h, tid);
#pragma unroll
    for (int k = 0; k < HID; k++) { const float v = fmaxf(h[k], 0.f); S[k * LD + tid] = v; if (KEEP) KEEP[(32 + k) * LD + tid] = __float2half_rn(v); }
  }
  dense_fwd<HID, DOUT, DOUT>(S, sW + W2_OFF, ns.o, tid);
  {
    float sh[SH_DIM];
    sh4(c7 + 4, sh);
#pragma unroll
    for (int k = 0; k < DOUT; k++) { S[k * LD + tid] = ns.o[k]; if (KEEP) KEEP[(96 + k) * LD + tid] = __float2half_rn(ns.o[k]); }
#pragma unroll
    for (int k = 0; k < SH_DIM; k++) { S[(DOUT + k) * LD + tid] = sh[k]; if (KEEP) KEEP[(96 + DOUT + k) * LD + tid] = __float2half_rn(sh[k]); }
  }
  {
    float h[HID];
    dense_fwd<32, HID, HID>(S, sW + W3_OFF, h, tid);
#pragma unroll
    for (int k = 0; k < HID; k++) { const float v = fmaxf(h[k], 0.f); S[k * LD + tid] = v; if (KEEP) KEEP[(128 + k) * LD + tid] = __float2half_rn(v); }
  }
  {
    float h[HID];
    dense_fwd<HID, HID, HID>(S, sW + W4_OFF, h, tid);
#pragma unroll
    for (int k = 0; k < HID; k++) { const float v = fmaxf(h[k], 0.f); S[k * LD + tid] = v; if (KEEP) KEEP[(192 + k) * LD + tid] = __float2half_rn(v); }
  }
  dense_fwd<HID, 4, 16>(S, sW + W5_OFF, ns.rgbraw, tid);
}

__device__ __forceinline__ float sigmoidf(float x) { return 1.f / (1.f + __expf(-x)); }

__global__ void __launch_bounds__(TILE)
forward_kernel(const float* __restrict__ coords, const int* __restrict__ counters, int n_fixed,
               const __half2* __restrict__ grid, LevelInfo lv, const float* __restrict__ mlp,
               float* __restrict__ rgbsigma) {
  extern __shared__ float sm[];
  float* sW = sm;
  float* S = sm + W_TOTAL;
  const int n = n_fixed >= 0 ? n_fixed : counters[0];
  const int tid = threadIdx.x;
  if (blockIdx.x * TILE >= n) return;
  for (int i = tid; i < W_TOTAL; i += TILE) sW[i] = mlp[i];
  __syncthreads();
  const int s = blockIdx.x * TILE + tid;
  if (s >= n) return;
  float c7[7];
#pragma unroll
  for (int k = 0; k < 7; k++) c7[k] = coords[(size_t)s * 7 + k];
  NetState ns;
  net_forward(c7, grid, lv, sW, S, nullptr, tid, ns);
  float4 out;
  out.x = sigmoidf(ns.rgbraw[0]); out.y = sigmoidf(ns.rgbraw[1]); out.z = sigmoidf(ns.rgbraw[2]);
  out.w = __expf(ns.o[0]);
  reinterpret_cast<float4*>(rgbsigma)[s] = out;
}

// ------------------------------------------------------------------------------------------
// compositing + loss + closed-form backward of the volume rendering, one WARP per ray: the samples
// of a ray are processed 32 at a time, transmittance by a multiplicative warp scan, the suffix terms
// of d/d(sigma) as (ray total - inclusive prefix) from additive warp scans.  Loads and the dout
// stores are coalesced (consecutive lanes = consecutive samples).
//   mode 0: training (writes dL/d(rgb,sigma) per sample, accumulates loss)
//   mode 1: render   (writes out_rgbd[r] = (r,g,b,z-depth))
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_scan_mul(float v, int lane) {
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) { const float u = __shfl_up_sync(0xffffffffu, v, o); if (lane >= o) v *= u; }
  return v;
}
__device__ __forceinline__ float warp_scan_add(float v, int lane) {
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) { const float u = __shfl_up_sync(0xffffffffu, v, o); if (lane >= o) v += u; }
  return v;
}

constexpr float LOSS_FX = 4294967296.f;            // 2^32: fixed-point scale of the batch-loss accumulator

__global__ void loss_kernel(const float* __restrict__ rays, int n_rays, const float* __restrict__ coords,
                            const float* __restrict__ tdist, const float* __restrict__ rgbsigma,
                            const int* __restrict__ counters, float lambda_d, float3 bg, int mode,
                            float* __restrict__ dout, float* __restrict__ loss_acc,
                            float* __restrict__ out_rgbd, long long* __restrict__ loss_fx = nullptr) {
  const int r = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (r >= n_rays) return;
  const float* R = rays + (size_t)r * 16;
  const int base = reinterpret_cast<const int*>(R)[12], n = reinterpret_cast<const int*>(R)[13];
  const float inv_len = R[6];
  // ---- forward sweep: a sample is used while the transmittance in front of it is >= MIN_T
  float T = 1.f, cr = 0.f, cg = 0.f, cb = 0.f, dep = 0.f;
  int used = 0;
  for (int c0 = 0; c0 < n; c0 += 32) {
    const int k = c0 + lane;
    const bool valid = k < n;
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    float dt = 0.f, tz = 0.f;
    if (valid) {
      v = reinterpret_cast<const float4*>(rgbsigma)[base + k];
      dt = coords[(size_t)(base + k) * 7 + 3];
      tz = tdist[base + k] * inv_len;
    }
    const float e = valid ? __expf(-v.w * dt) : 1.f;
    const float pin = warp_scan_mul(e, lane);
    float pex = __shfl_up_sync(0xffffffffu, pin, 1);
    if (lane == 0) pex = 1.f;
    const float Tb = T * pex;                                    // transmittance in front of sample k
    const bool use = valid && Tb >= MIN_T;
    const float w = use ? (1.f - e) * Tb : 0.f;
    cr += w * v.x; cg += w * v.y; cb += w * v.z; dep += w * tz;
    const uint32_t um = __ballot_sync(0xffffffffu, use);
    const uint32_t vm = __ballot_sync(0xffffffffu, valid);
    used += __popc(um);
    if (um != vm) {                                               // cut inside this chunk
      T = __shfl_sync(0xffffffffu, Tb, __popc(um));               // T in front of the first unused sample
      break;
    }
    T *= __shfl_sync(0xffffffffu, pin, 31);
  }
  cr = warp_sum(cr); cg = warp_sum(cg); cb = warp_sum(cb); dep = warp_sum(dep);
  if (mode == 1) {
    if (lane == 0) reinterpret_cast<float4*>(out_rgbd)[r] = make_float4(cr + T * bg.x, cg + T * bg.y, cb + T * bg.z, dep);
    return;
  }
  if (n == 0) return;
  const int kept = max(counters[1], 1);
  const float invR = 1.f / (float)kept;
  cr += T * bg.x; cg += T * bg.y; cb += T * bg.z;
  const float tgt[3] = {R[9], R[10], R[11]};
  const float col[3] = {cr, cg, cb};
  float lg[3], loss = 0.f;
#pragma unroll
  for (int c = 0; c < 3; c++) {
    const float diff = col[c] - tgt[c], ad = fabsf(diff);
    // Huber(delta = 0.1) / 5, mean over the 3 channels
    loss += (ad < 0.1f ? 0.5f * diff * diff / 0.1f : ad - 0.05f) / 5.f / 3.f;
    lg[c] = (ad < 0.1f ? diff / 0.1f : copysignf(1.f, diff)) / 5.f / 3.f * invR;
  }
  const float td = R[7], cov = fmaxf(R[8], 1e-12f);
  float ld = 0.f;
  if (td > 0.f && lambda_d > 0.f) {
    const float e = dep - td;
    loss += lambda_d * e * e / cov;
    ld = 2.f * lambda_d * e / cov * invR;
  }
  if (lane == 0) {
    if (loss_fx) fx_add(loss_fx, loss * invR, LOSS_FX);      // order-independent; added to loss_acc by fx_flush_kernel
    else atomicAdd(loss_acc, loss * invR);
  }
  // ---- backward sweep
  float T2 = 1.f, r2 = 0.f, g2 = 0.f, b2 = 0.f, d2 = 0.f;       // carries: values after the previous chunk
  for (int c0 = 0; c0 < n; c0 += 32) {
    const int k = c0 + lane;
    float4 g = make_float4(0.f, 0.f, 0.f, 0.f);
    if (c0 < used) {                                              // warp-uniform
      const bool use = k < used;
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      float dt = 0.f, tz = 0.f;
      if (use) {
        v = reinterpret_cast<const float4*>(rgbsigma)[base + k];
        dt = coords[(size_t)(base + k) * 7 + 3];
        tz = tdist[base + k] * inv_len;
      }
      const float e = use ? __expf(-v.w * dt) : 1.f;
      const float pin = warp_scan_mul(e, lane);
      float pex = __shfl_up_sync(0xffffffffu, pin, 1);
      if (lane == 0) pex = 1.f;
      const float w = use ? (1.f - e) * (T2 * pex) : 0.f;
      const float Ta = T2 * pin;                                  // transmittance behind sample k
      const float sr = r2 + warp_scan_add(w * v.x, lane), sg = g2 + warp_scan_add(w * v.y, lane);
      const float sb = b2 + warp_scan_add(w * v.z, lane), sd = d2 + warp_scan_add(w * tz, lane);
      if (use) {
        // d(colour)/d(rgb_s) = w ;  d(C)/d(sigma_s) = dt (T_after c_s - suffix)
        g.x = lg[0] * w * v.x * (1.f - v.x);                      // through the sigmoid
        g.y = lg[1] * w * v.y * (1.f - v.y);
        g.z = lg[2] * w * v.z * (1.f - v.z);
        float ds = lg[0] * (Ta * v.x - (col[0] - sr)) + lg[1] * (Ta * v.y - (col[1] - sg)) + lg[2] * (Ta * v.z - (col[2] - sb));
        ds += ld * (Ta * tz - (dep - sd));
        g.w = ds * dt * v.w;                                      // through sigma = exp(o0)
      }
      T2 = __shfl_sync(0xffffffffu, Ta, 31);
      r2 = __shfl_sync(0xffffffffu, sr, 31); g2 = __shfl_sync(0xffffffffu, sg, 31);
      b2 = __shfl_sync(0xffffffffu, sb, 31); d2 = __shfl_sync(0xffffffffu, sd, 31);
    }
    if (k < n) reinterpret_cast<float4*>(dout)[base + k] = g;     // d/d(raw rgb outputs), d/d(o0)
  }
}

// ------------------------------------------------------------------------------------------
// backward: persistent CTAs, 128-sample tiles.  smem: weights | S | D | KEEP(256 rows)
__global__ void __launch_bounds__(TILE)
backward_kernel(const float* __restrict__ coords, const int* __restrict__ counters,
                const __half2* __restrict__ grid, LevelInfo lv, const float* __restrict__ mlp,
                const float* __restrict__ dout, float* __restrict__ mlp_grad,
                float* __restrict__ grid_grad) {
  extern __shared__ float sm[];
  float* sW = sm;
  float* S = sW + W_TOTAL;         // [64][LD]
  float* D = S + 64 * LD;          // [64][LD]
  __half* KEEP = reinterpret_cast<__half*>(D + 64 * LD);   // [256][LD] fp16
  const int tid = threadIdx.x;
  const int n = counters[0];
  for (int i = tid; i < W_TOTAL; i += TILE) sW[i] = mlp[i];
  float g5[1][16], g4[2][16], g3[1][16], g2[1][16], g1[1][16];
#pragma unroll
  for (int q = 0; q < 16; q++) { g5[0][q] = 0.f; g4[0][q] = 0.f; g4[1][q] = 0.f; g3[0][q] = 0.f; g2[0][q] = 0.f; g1[0][q] = 0.f; }
  __syncthreads();
  const int ntiles = (n + TILE - 1) / TILE;
  for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    const int s = tile * TILE + tid;
    const bool act = s < n;
    const int rows = min(TILE, n - tile * TILE);
    float c7[7] = {0.5f, 0.5f, 0.5f, 0.f, 0.f, 0.f, 1.f};
    float4 dg = make_float4(0.f, 0.f, 0.f, 0.f);
    if (act) {
#pragma unroll
      for (int k = 0; k < 7; k++) c7[k] = coords[(size_t)s * 7 + k];
      dg = reinterpret_cast<const float4*>(dout)[s];
    }
    NetState ns;
    net_forward(c7, grid, lv, sW, S, KEEP, tid, ns);       // S holds h3, KEEP all layer inputs
    // ---- layer 5 (64 -> 3): delta5 = dg.xyz
    D[0 * LD + tid] = dg.x; D[1 * LD + tid] = dg.y; D[2 * LD + tid] = dg.z; D[3 * LD + tid] = 0.f;
    __syncthreads();
    outer_acc<HID, 4, 1>(KEEP + 192 * LD, D, g5, tid, rows);
    float d64[HID];
    {
      float d4[4] = {dg.x, dg.y, dg.z, 0.f};
      __syncthreads();
      dense_bwd_in<HID, 4, 16>(d4, sW + W5_OFF, D, tid);    // D[k] = dL/dh3[k] (pre-mask)
#pragma unroll 4
      for (int k = 0; k < HID; k++) { const float v = (__half2float(KEEP[(192 + k) * LD + tid]) > 0.f) ? D[k * LD + tid] : 0.f; D[k * LD + tid] = v; }
    }
    __syncthreads();
    // ---- layer 4 (64 -> 64)
    outer_acc<HID, HID, 2>(KEEP + 128 * LD, D, g4, tid, rows);
#pragma unroll
    for (int k = 0; k < HID; k++) d64[k] = D[k * LD + tid];
    __syncthreads();
    dense_bwd_in<HID, HID, HID>(d64, sW + W4_OFF, D, tid);
#pragma unroll 4
    for (int k = 0; k < HID; k++) { const float v = (__half2float(KEEP[(128 + k) * LD + tid]) > 0.f) ? D[k * LD + tid] : 0.f; D[k * LD + tid] = v; }
    __syncthreads();
    // ---- layer 3 (32 -> 64)
    outer_acc<32, HID, 1>(KEEP + 96 * LD, D, g3, tid, rows);
#pragma unroll
    for (int k = 0; k < HID; k++) d64[k] = D[k * LD + tid];
    __syncthreads();
    dense_bwd_in<32, HID, HID>(d64, sW + W3_OFF, D, tid);    // D[0..31] = dL/d in2 ; first 16 -> density out
    float d16[DOUT];
#pragma unroll
    for (int k = 0; k < DOUT; k++) d16[k] = D[k * LD + tid];
    d16[0] += dg.w;                                           // sigma path
    __syncthreads();
#pragma unroll
    for (int k = 0; k < DOUT; k++) D[k * LD + tid] = d16[k];
    __syncthreads();
    // ---- layer 2 (64 -> 16)
    outer_acc<HID, DOUT, 1>(KEEP + 32 * LD, D, g2, tid, rows);
    __syncthreads();
    dense_bwd_in<HID, DOUT, DOUT>(d16, sW + W2_OFF, D, tid);
#pragma unroll 4
    for (int k = 0; k < HID; k++) { const float v = (__half2float(KEEP[(32 + k) * LD + tid]) > 0.f) ? D[k * LD + tid] : 0.f; D[k * LD + tid] = v; }
    __syncthreads();
    // ---- layer 1 (32 -> 64)
    outer_acc<ENC_DIM, HID, 1>(KEEP, D, g1, tid, rows);
#pragma unroll
    for (int k = 0; k < HID; k++) d64[k] = D[k * LD + tid];
    __syncthreads();
    dense_bwd_in<ENC_DIM, HID, HID>(d64, sW + W1_OFF, D, tid);  // D[0..31] = dL/d enc
    // ---- hash-grid gradient scatter
    if (act) {
#pragma unroll 2
      for (int l = 0; l < N_LEVELS; l++) {
        const float ga = D[(2 * l) * LD + tid], gb = D[(2 * l + 1) * LD + tid];
        if (ga == 0.f && gb == 0.f) continue;
        const float sc = lv.scale[l];
        const float px = fmaf(c7[0], sc, 0.5f), py = fmaf(c7[1], sc, 0.5f), pz = fmaf(c7[2], sc, 0.5f);
        const float fx = floorf(px), fy = floorf(py), fz = floorf(pz);
        const float wx = px - fx, wy = py - fy, wz = pz - fz;
        const int ix = (int)fx, iy = (int)fy, iz = (int)fz;
        float2* gg = reinterpret_cast<float2*>(grid_grad) + lv.offset[l];
#pragma unroll
        for (int c = 0; c < 8; c++) {
          const int dx = c & 1, dy = (c >> 1) & 1, dz = c >> 2;
          const float w = (dx ? wx : 1.f - wx) * (dy ? wy : 1.f - wy) * (dz ? wz : 1.f - wz);
          const uint32_t idx = grid_index(ix + dx, iy + dy, iz + dz, lv.res[l], lv.size[l], lv.dense[l]);
          atomicAdd(gg + idx, make_float2(w * ga, w * gb));
        }
      }
    }
    __syncthreads();
  }
  outer_flush<HID, 4, 1, 16>(g5, mlp_grad + W5_OFF, tid);
  outer_flush<HID, HID, 2, HID>(g4, mlp_grad + W4_OFF, tid);
  outer_flush<32, HID, 1, HID>(g3, mlp_grad + W3_OFF, tid);
  outer_flush<HID, DOUT, 1, DOUT>(g2, mlp_grad + W2_OFF, tid);
  outer_flush<ENC_DIM, HID, 1, HID>(g1, mlp_grad + W1_OFF, tid);
}

// ------------------------------------------------------------------------------------------
// Adam.  is_grid: skip entries with zero gradient (untouched hash slots), no L2.
// float4-vectorised; bias corrections (1/(1-b^t)) are computed once on the host.  Writes g = 0.
__global__ void adam_kernel(float4* __restrict__ p, float4* __restrict__ g, float4* __restrict__ m,
                            float4* __restrict__ v, __half2* __restrict__ p_half, size_t n4, float lr,
                            float b1, float b2, float eps, float l2, int is_grid, float bc1, float bc2) {
  const size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (i >= n4) return;
  const float4 g4 = g[i];
  if (g4.x == 0.f && g4.y == 0.f && g4.z == 0.f && g4.w == 0.f) {
    if (is_grid) return;           // untouched hash slots keep their moments (tiny-cuda-nn semantics)
  } else {
    g[i] = make_float4(0.f, 0.f, 0.f, 0.f);
  }
  float4 w4 = p[i], m4 = m[i], v4 = v[i];
  float* w = reinterpret_cast<float*>(&w4);
  float* mm = reinterpret_cast<float*>(&m4);
  float* vv = reinterpret_cast<float*>(&v4);
  const float* gg = reinterpret_cast<const float*>(&g4);
#pragma unroll
  for (int k = 0; k < 4; k++) {
    if (is_grid && gg[k] == 0.f) continue;
    const float grad = gg[k] + l2 * w[k];
    mm[k] = b1 * mm[k] + (1.f - b1) * grad;
    vv[k] = b2 * vv[k] + (1.f - b2) * grad * grad;
    w[k] -= lr * (mm[k] * bc1) / (sqrtf(vv[k] * bc2) + eps);
  }
  p[i] = w4; m[i] = m4; v[i] = v4;
  if (p_half) { p_half[2 * i] = __floats2half2_rn(w[0], w[1]); p_half[2 * i + 1] = __floats2half2_rn(w[2], w[3]); }
}

// ------------------------------------------------------------------------------------------
// occupancy grid maintenance
// sample `n` cells per cascade (all cells when n == GRID^3), evaluate the density MLP at a
// jittered point inside the cell, EMA-max into density[], cells that no camera sees stay at -1.
__global__ void __launch_bounds__(TILE)
density_sample_kernel(const __half2* __restrict__ grid, LevelInfo lv, const float* __restrict__ mlp,
                      Scene sc, int n_per_cascade, uint32_t seed, float decay,
                      float* __restrict__ density) {
  extern __shared__ float sm[];
  float* sW = sm;
  float* S = sm + W1_OFF + ENC_DIM * HID + HID * DOUT;  // only W1,W2 are needed
  const int tid = threadIdx.x;
  for (int i = tid; i < ENC_DIM * HID + HID * DOUT; i += TILE) sW[i] = mlp[i];
  __syncthreads();
  const int total = n_per_cascade * sc.cascades;
  const int i = blockIdx.x * TILE + tid;
  if (i >= total) return;
  const int mip = i / n_per_cascade, j = i % n_per_cascade;
  const int NC = GRID * GRID * GRID;
  const uint32_t cell = (n_per_cascade >= NC) ? (uint32_t)j : density_cell(seed, mip, j);
  const size_t gi = (size_t)mip * NC + cell;
  if (density[gi] < 0.f) return;   // never visible from a training camera
  const int ix = cell % GRID, iy = (cell / GRID) % GRID, iz = cell / (GRID * GRID);
  const float s = scalbnf(1.f, mip);
  float p[3] = {((ix + rnd01(seed, i, 11)) / GRID - 0.5f) * s + 0.5f,
                ((iy + rnd01(seed, i, 12)) / GRID - 0.5f) * s + 0.5f,
                ((iz + rnd01(seed, i, 13)) / GRID - 0.5f) * s + 0.5f};
  float x01[3] = {(p[0] - sc.aabb_lo) * sc.inv_extent, (p[1] - sc.aabb_lo) * sc.inv_extent,
                  (p[2] - sc.aabb_lo) * sc.inv_extent};
  float enc[ENC_DIM];
  hash_encode(x01, grid, lv, enc);
#pragma unroll
  for (int k = 0; k < ENC_DIM; k++) S[k * LD + tid] = enc[k];
  float h[HID];
  dense_fwd<ENC_DIM, HID, HID>(S, sW + W1_OFF, h, tid);
#pragma unroll
  for (int k = 0; k < HID; k++) S[k * LD + tid] = fmaxf(h[k], 0.f);
  float o[DOUT];
  dense_fwd<HID, DOUT, DOUT>(S, sW + W2_OFF, o, tid);
  const float thick = __expf(o[0]) * MIN_STEP * s;        // optical thickness of one minimal step
  density[gi] = fmaxf(density[gi] * decay, thick);
}

// visibility: mark cells that project inside at least one training image (in front of it)
__global__ void density_mark_kernel(const Camera* __restrict__ cams, const int* __restrict__ active,
                                    int n_active, int cascades, float* __restrict__ density) {
  const int NC = GRID * GRID * GRID;
  const size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (i >= (size_t)NC * cascades) return;
  if (density[i] >= 0.f) return;
  const int mip = (int)(i / NC);
  const int cell = (int)(i % NC);
  const int ix = cell % GRID, iy = (cell / GRID) % GRID, iz = cell / (GRID * GRID);
  const float s = scalbnf(1.f, mip);
  const float half = 0.5f * s / GRID * SQRT3;
  const float p[3] = {((ix + 0.5f) / GRID - 0.5f) * s + 0.5f, ((iy + 0.5f) / GRID - 0.5f) * s + 0.5f,
                      ((iz + 0.5f) / GRID - 0.5f) * s + 0.5f};
  for (int a = 0; a < n_active; a++) {
    const Camera& c = cams[active[a]];
    // world -> camera: R^T (p - t)
    const float q[3] = {p[0] - c.c2w[3], p[1] - c.c2w[7], p[2] - c.c2w[11]};
    const float xc = c.c2w[0] * q[0] + c.c2w[4] * q[1] + c.c2w[8] * q[2];
    const float yc = c.c2w[1] * q[0] + c.c2w[5] * q[1] + c.c2w[9] * q[2];
    const float zc = c.c2w[2] * q[0] + c.c2w[6] * q[1] + c.c2w[10] * q[2];
    if (zc + half <= 1e-3f) continue;
    const float z = fmaxf(zc, 1e-3f);
    const float u = c.fx * xc / z + c.cx, v = c.fy * yc / z + c.cy;
    const float mu = c.fx * half / z, mv = c.fy * half / z;
    if (u + mu >= 0.f && u - mu < c.w && v + mv >= 0.f && v - mv < c.h) { density[i] = 0.f; return; }
  }
}

// mean of the non-negative densities -> stats[0] = sum, stats[1] = count.  Fixed summation order (no atomics):
// each block writes its partial, density_mean_final_kernel adds the partials in block order.
constexpr int DM_BLOCKS = 592;
__device__ float g_density_partials[2 * DM_BLOCKS];
__global__ void __launch_bounds__(256) density_mean_kernel(const float* __restrict__ density, size_t n) {
  __shared__ float ws[2][8];
  float s = 0.f, c = 0.f;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    const float d = density[i];
    if (d >= 0.f) { s += d; c += 1.f; }
  }
  for (int o = 16; o > 0; o >>= 1) { s += __shfl_xor_sync(0xffffffffu, s, o); c += __shfl_xor_sync(0xffffffffu, c, o); }
  if ((threadIdx.x & 31) == 0) { ws[0][threadIdx.x >> 5] = s; ws[1][threadIdx.x >> 5] = c; }
  __syncthreads();
  if (threadIdx.x < 2) {
    float v = 0.f;
    for (int w = 0; w < 8; w++) v += ws[threadIdx.x][w];
    g_density_partials[2 * blockIdx.x + threadIdx.x] = v;
  }
}
__global__ void density_mean_final_kernel(float* __restrict__ stats) {
  if (threadIdx.x < 2) {
    float v = 0.f;
    for (int b = 0; b < DM_BLOCKS; b++) v += g_density_partials[2 * b + threadIdx.x];
    stats[threadIdx.x] = v;
  }
}
__global__ void density_bits_kernel(const float* __restrict__ density, size_t nbytes,
                                    const float* __restrict__ stats, float min_thick,
                                    uint8_t* __restrict__ bits) {
  const size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (i >= nbytes) return;
  const float thr = fminf(min_thick, stats[1] > 0.f ? stats[0] / stats[1] : 0.f);
  uint8_t b = 0;
#pragma unroll
  for (int k = 0; k < 8; k++) b |= (density[i * 8 + k] > thr) ? (1u << k) : 0u;
  bits[i] = b;
}

// training image upload helpers: sRGB u8 -> linear premultiplied half4 (process_slam,
// fusion/nerf_fusion.py:198-215, done on the GPU without the CPU round trip), depth = 1/idepth
__global__ void ingest_image_kernel(const uint8_t* __restrict__ rgb_chw, const float* __restrict__ idepth,
                                    const float* __restrict__ dcov, int H, int W, __half* __restrict__ rgba,
                                    float* __restrict__ depth, float* __restrict__ depth_cov) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= H * W) return;
  float c[3];
#pragma unroll
  for (int k = 0; k < 3; k++) {
    const float s = rgb_chw[(size_t)k * H * W + i] * (1.f / 255.f);
    c[k] = s > 0.04045f ? powf((s + 0.055f) / 1.055f, 2.4f) : s / 12.92f;
  }
  __half* o = rgba + (size_t)i * 4;
  o[0] = __float2half_rn(c[0]); o[1] = __float2half_rn(c[1]); o[2] = __float2half_rn(c[2]); o[3] = __float2half_rn(1.f);
  const float id = idepth[i];
  depth[i] = 1.0f / id;             // negative idepth sentinel -> negative depth = "no depth"
  depth_cov[i] = dcov[i];
}

// the whole SLAM packet in ONE launch (grid: pixel blocks x keyframes): images / depths / covariances into their
// slots `ids[k]`, and the camera record of each slot from the packet's cam_T_world pose [t, q_xyzw]:
// world_T_cam = inverse, 3x4 row-major (fusion/nerf_fusion.py:163-170: scale 1, offset 0), computed in fp64 like the
// host formulation it replaces.  No host copy of the poses is needed any more (that copy was a device sync per tick).
__global__ void ingest_batch_kernel(const uint8_t* __restrict__ rgb_chw, const float* __restrict__ idepth,
                                    const float* __restrict__ dcov, const long long* __restrict__ ids, int H, int W,
                                    __half* __restrict__ rgba, float* __restrict__ depth, float* __restrict__ depth_cov,
                                    const float* __restrict__ cam_T_world, float fx, float fy, float cx, float cy,
                                    Camera* __restrict__ cams, Camera* __restrict__ cams_base,
                                    float* __restrict__ cam_state /* [3][N][6] offsets | m | v */, int* __restrict__ cam_steps,
                                    int n_slots) {
  const int k = blockIdx.y;
  const size_t hw = (size_t)H * W;
  const size_t slot = (size_t)ids[k];
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (cams && blockIdx.x == 0 && threadIdx.x == 0) {
    const float* p = cam_T_world + (size_t)k * 7;
    const double t[3] = {p[0], p[1], p[2]};
    const double x = p[3], y = p[4], z = p[5], w = p[6];
    // R (cam <- world); world_T_cam = [R^T | -R^T t]
    const double R[3][3] = {{1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)},
                            {2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)},
                            {2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)}};
    Camera c;
    for (int r = 0; r < 3; r++) {
      for (int cc = 0; cc < 3; cc++) c.c2w[r * 4 + cc] = (float)R[cc][r];
      c.c2w[r * 4 + 3] = (float)(-(R[0][r] * t[0] + R[1][r] * t[1] + R[2][r] * t[2]));
    }
    c.fx = fx; c.fy = fy; c.cx = cx; c.cy = cy; c.w = W; c.h = H;
    cams[slot] = c;
    if (cams_base) {
      // a new base pose from SLAM: the pose refinement of this camera starts again from zero (offsets, Adam moments)
      cams_base[slot] = c;
      for (int part = 0; part < 3; part++)
        for (int q = 0; q < 6; q++) cam_state[((size_t)part * n_slots + slot) * 6 + q] = 0.f;
      cam_steps[slot] = 0;
    }
  }
  if (i >= H * W) return;
  const uint8_t* src = rgb_chw + (size_t)k * 3 * hw;
  float c[3];
#pragma unroll
  for (int ch = 0; ch < 3; ch++) {
    const float s = src[(size_t)ch * hw + i] * (1.f / 255.f);
    c[ch] = s > 0.04045f ? powf((s + 0.055f) / 1.055f, 2.4f) : s / 12.92f;
  }
  __half* o = rgba + (slot * hw + i) * 4;
  o[0] = __float2half_rn(c[0]); o[1] = __float2half_rn(c[1]); o[2] = __float2half_rn(c[2]); o[3] = __float2half_rn(1.f);
  depth[slot * hw + i] = 1.0f / idepth[(size_t)k * hw + i];
  depth_cov[slot * hw + i] = dcov[(size_t)k * hw + i];
}

}  // namespace ngp

// ============================================================================================
namespace ngp {
static LevelInfo make_lv(const nslam_ngp_model* m) {
  LevelInfo lv;
  for (int l = 0; l < N_LEVELS; l++) {
    lv.scale[l] = m->scale[l]; lv.res[l] = m->res[l]; lv.size[l] = m->size[l];
    lv.offset[l] = m->offset[l]; lv.dense[l] = m->dense[l];
  }
  return lv;
}
static Scene make_scene(const nslam_ngp_model* m) {
  Scene s;
  s.aabb_lo = 0.5f - 0.5f * m->aabb_scale; s.aabb_hi = 0.5f + 0.5f * m->aabb_scale;
  s.inv_extent = 1.f / m->aabb_scale; s.cascades = m->cascades; s.cone = m->cone; s.near = m->near_distance;
  return s;
}
static ImageStore make_store(const nslam_ngp_images* im) {
  ImageStore st;
  st.rgba = (const __half*)im->rgba; st.depth = im->depth; st.depth_cov = im->depth_cov;
  st.cams = (const Camera*)im->cams; st.active = im->active; st.n_active = im->n_active; st.H = im->H; st.W = im->W;
  return st;
}
constexpr size_t FWD_SMEM = (W_TOTAL + 64 * LD) * sizeof(float);
constexpr size_t BWD_SMEM = (W_TOTAL + (64 + 64) * LD) * sizeof(float) + 256 * LD * sizeof(__half);
static int ensure_attrs() {
  static bool done = false;
  if (done) return 0;
  cudaError_t e = cudaFuncSetAttribute(forward_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)FWD_SMEM);
  if (e != cudaSuccess) return (int)e;
  e = cudaFuncSetAttribute(backward_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)BWD_SMEM);
  if (e != cudaSuccess) return (int)e;
  e = cudaFuncSetAttribute(density_sample_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)FWD_SMEM);
  if (e != cudaSuccess) return (int)e;
  done = true;
  return 0;
}
}  // namespace ngp

extern "C" {

/* one training step WITHOUT the optimiser: sample rays, march, forward, loss, backward.
 * Gradients accumulate into model->*_grad (must be zero on entry; nslam_ngp_adam zeroes them). */
static void sample_rays(const nslam_ngp_model* m, const nslam_ngp_images* im, const nslam_ngp_batch* b, int n_rays,
                        unsigned seed, cudaStream_t st) {
  using namespace ngp;
  for (int pass = 1; pass >= 0; pass--) {
    sample_rays_kernel<<<(n_rays + 3) / 4, 128, 0, st>>>(make_store(im), make_scene(m), m->bits, n_rays, seed,
                                                           b->max_samples, b->rays, b->coords, b->tdist, b->counters, pass);
    if (pass) sample_scan_kernel<<<1, 1024, 0, st>>>(b->rays, n_rays, b->max_samples, b->counters);
  }
}

int nslam_ngp_train_step(const nslam_ngp_model* m, const nslam_ngp_images* im, const nslam_ngp_batch* b,
                         int n_rays, unsigned seed, float lambda_depth, float bg_r, float bg_g,
                         float bg_b, int num_sms, void* stream) {
  using namespace ngp;
  int r = ensure_attrs();
  if (r) return r;
  cudaStream_t st = (cudaStream_t)stream;
  if (n_rays > b->max_rays) return (int)cudaErrorInvalidValue;
  cudaMemsetAsync(b->counters, 0, 4 * sizeof(int), st);
  cudaMemsetAsync(b->loss, 0, sizeof(float), st);
  const LevelInfo lv = make_lv(m);
  const Scene sc = make_scene(m);
  sample_rays(m, im, b, n_rays, seed, st);
  NGP_CHECK_LAUNCH();
  forward_kernel<<<(b->max_samples + TILE - 1) / TILE, TILE, FWD_SMEM, st>>>(
      b->coords, b->counters, -1, (const __half2*)m->grid_half, lv, m->mlp, b->rgbsigma);
  NGP_CHECK_LAUNCH();
  long long* loss_fx = (long long*)ngp_scratch(NGP_SCRATCH_LOSS, sizeof(long long));
  if (!loss_fx) return (int)cudaErrorMemoryAllocation;
  loss_kernel<<<(n_rays + 3) / 4, 128, 0, st>>>(b->rays, n_rays, b->coords, b->tdist, b->rgbsigma,
                                                     b->counters, lambda_depth, make_float3(bg_r, bg_g, bg_b),
                                                     0, b->dout, b->loss, nullptr, loss_fx);
  fx_flush_kernel<<<1, 32, 0, (cudaStream_t)stream>>>(loss_fx, b->loss, 1, 1.f / LOSS_FX);
  NGP_CHECK_LAUNCH();
  backward_kernel<<<2 * num_sms, TILE, BWD_SMEM, st>>>(b->coords, b->counters, (const __half2*)m->grid_half,
                                                       lv, m->mlp, b->dout, m->mlp_grad, m->grid_grad);
  NGP_CHECK_LAUNCH();
  return 0;
}

/* the two non-network phases of a training step, exported so that the tensor-core step
 * (csrc/ngp_tc.cu: nslam_ngp_train_step_tc) can reuse them: ray/sample generation and the loss */
int nslam_ngp_sample_phase(const nslam_ngp_model* m, const nslam_ngp_images* im, const nslam_ngp_batch* b,
                           int n_rays, unsigned seed, void* stream) {
  using namespace ngp;
  cudaStream_t st = (cudaStream_t)stream;
  if (n_rays > b->max_rays) return (int)cudaErrorInvalidValue;
  cudaMemsetAsync(b->counters, 0, 4 * sizeof(int), st);
  cudaMemsetAsync(b->loss, 0, sizeof(float), st);
  sample_rays(m, im, b, n_rays, seed, st);
  NGP_CHECK_LAUNCH();
  return 0;
}

int nslam_ngp_loss_phase(const nslam_ngp_batch* b, int n_rays, float lambda_depth, float bg_r, float bg_g,
                         float bg_b, void* stream) {
  using namespace ngp;
  long long* loss_fx = (long long*)ngp_scratch(NGP_SCRATCH_LOSS, sizeof(long long));
  if (!loss_fx) return (int)cudaErrorMemoryAllocation;
  loss_kernel<<<(n_rays + 3) / 4, 128, 0, (cudaStream_t)stream>>>(b->rays, n_rays, b->coords, b->tdist, b->rgbsigma,
                                                                       b->counters, lambda_depth,
                                                                       make_float3(bg_r, bg_g, bg_b), 0, b->dout, b->loss, nullptr, loss_fx);
  fx_flush_kernel<<<1, 32, 0, (cudaStream_t)stream>>>(loss_fx, b->loss, 1, 1.f / LOSS_FX);
  NGP_CHECK_LAUNCH();
  return 0;
}

int nslam_ngp_adam(const nslam_ngp_model* m, int step, float lr, float beta1, float beta2, float eps,
                   float l2_mlp, void* stream) {
  using namespace ngp;
  cudaStream_t st = (cudaStream_t)stream;
  const size_t ng4 = (size_t)m->n_grid * 2 / 4;   // level sizes are multiples of 8 entries
  const float bc1 = 1.f / (1.f - powf(beta1, (float)step)), bc2 = 1.f / (1.f - powf(beta2, (float)step));
  adam_kernel<<<(unsigned)((ng4 + 255) / 256), 256, 0, st>>>((float4*)m->grid_master, (float4*)m->grid_grad, (float4*)m->grid_m,
                                                            (float4*)m->grid_v, (__half2*)m->grid_half, ng4, lr, beta1, beta2,
                                                            eps, 0.f, 1, bc1, bc2);
  NGP_CHECK_LAUNCH();
  adam_kernel<<<(W_TOTAL / 4 + 255) / 256, 256, 0, st>>>((float4*)m->mlp, (float4*)m->mlp_grad, (float4*)m->mlp_m,
                                                         (float4*)m->mlp_v, nullptr, W_TOTAL / 4, lr, beta1, beta2, eps,
                                                         l2_mlp, 0, bc1, bc2);
  NGP_CHECK_LAUNCH();
  return 0;
}

/* network forward on caller-provided samples (tests / density queries): coords [n,7] -> rgbsigma [n,4] */
int nslam_ngp_forward(const nslam_ngp_model* m, const float* coords, int n, float* rgbsigma, void* stream) {
  using namespace ngp;
  int r = ensure_attrs();
  if (r) return r;
  if (n == 0) return 0;
  forward_kernel<<<(n + TILE - 1) / TILE, TILE, FWD_SMEM, (cudaStream_t)stream>>>(
      coords, nullptr, n, (const __half2*)m->grid_half, make_lv(m), m->mlp, rgbsigma);
  NGP_CHECK_LAUNCH();
  return 0;
}

/* loss + gradients on caller-provided rays/samples (tests): rays [R,16] must carry base/n/targets */
int nslam_ngp_loss_backward(const nslam_ngp_model* m, const nslam_ngp_batch* b, int n_rays, int n_samples,
                            float lambda_depth, float bg_r, float bg_g, float bg_b, int num_sms, void* stream) {
  using namespace ngp;
  int r = ensure_attrs();
  if (r) return r;
  cudaStream_t st = (cudaStream_t)stream;
  int h[4] = {n_samples, n_rays, n_rays, 0};
  cudaMemcpyAsync(b->counters, h, sizeof(h), cudaMemcpyHostToDevice, st);
  cudaMemsetAsync(b->loss, 0, sizeof(float), st);
  const LevelInfo lv = make_lv(m);
  forward_kernel<<<(n_samples + TILE - 1) / TILE, TILE, FWD_SMEM, st>>>(b->coords, b->counters, -1,
                                                                       (const __half2*)m->grid_half, lv, m->mlp, b->rgbsigma);
  NGP_CHECK_LAUNCH();
  long long* loss_fx = (long long*)ngp_scratch(NGP_SCRATCH_LOSS, sizeof(long long));
  if (!loss_fx) return (int)cudaErrorMemoryAllocation;
  loss_kernel<<<(n_rays + 3) / 4, 128, 0, st>>>(b->rays, n_rays, b->coords, b->tdist, b->rgbsigma, b->counters,
                                                     lambda_depth, make_float3(bg_r, bg_g, bg_b), 0, b->dout, b->loss, nullptr, loss_fx);
  fx_flush_kernel<<<1, 32, 0, (cudaStream_t)stream>>>(loss_fx, b->loss, 1, 1.f / LOSS_FX);
  NGP_CHECK_LAUNCH();
  backward_kernel<<<2 * num_sms, TILE, BWD_SMEM, st>>>(b->coords, b->counters, (const __half2*)m->grid_half, lv,
                                                       m->mlp, b->dout, m->mlp_grad, m->grid_grad);
  NGP_CHECK_LAUNCH();
  return 0;
}

/* occupancy grid: mark visibility, sample densities (EMA-max), rebuild the bitfield */
int nslam_ngp_update_density_grid(const nslam_ngp_model* m, const nslam_ngp_images* im, int n_per_cascade,
                                  unsigned seed, float decay, float min_thickness, const void* packed, int num_sms,
                                  void* stream) {
  using namespace ngp;
  int r = ensure_attrs();
  if (r) return r;
  cudaStream_t st = (cudaStream_t)stream;
  const size_t NC = (size_t)GRID * GRID * GRID;
  const size_t total = NC * m->cascades;
  density_mark_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>((const Camera*)im->cams, im->active,
                                                                      im->n_active, m->cascades, m->density);
  NGP_CHECK_LAUNCH();
  const int n = n_per_cascade * m->cascades;
  if (packed) {
    r = nslam_ngp_density_sample_tc(m, packed, n_per_cascade, seed, decay, num_sms, stream);
    if (r) return r;
  } else {
    density_sample_kernel<<<(n + TILE - 1) / TILE, TILE, FWD_SMEM, st>>>((const __half2*)m->grid_half, make_lv(m), m->mlp,
                                                                       make_scene(m), n_per_cascade, seed, decay, m->density);
    NGP_CHECK_LAUNCH();
  }
  density_mean_kernel<<<DM_BLOCKS, 256, 0, st>>>(m->density, total);
  density_mean_final_kernel<<<1, 32, 0, st>>>(m->stats);
  NGP_CHECK_LAUNCH();
  density_bits_kernel<<<(unsigned)((total / 8 + 255) / 256), 256, 0, st>>>(m->density, total / 8, m->stats,
                                                                          min_thickness, m->bits);
  NGP_CHECK_LAUNCH();
  return 0;
}

/* render a tile of a camera view: out_rgbd [th*tw,4] = (r,g,b,z-depth).  packed != NULL: the network runs on tensor
 * cores (nslam_ngp_forward_tc, the kernel the trainer uses); NULL: the fp32 CUDA-core forward (the tests' cross-check). */
int nslam_ngp_render_tile(const nslam_ngp_model* m, const nslam_ngp_batch* b, const float* cam16,
                          int x0, int y0, int tw, int th, int max_per_ray, float bg_r, float bg_g,
                          float bg_b, float* out_rgbd, const void* packed, int num_sms, void* stream) {
  using namespace ngp;
  int r = ensure_attrs();
  if (r) return r;
  cudaStream_t st = (cudaStream_t)stream;
  if (tw * th > b->max_rays) return (int)cudaErrorInvalidValue;
  Camera cam;
  for (int i = 0; i < 12; i++) cam.c2w[i] = cam16[i];
  cam.fx = cam16[12]; cam.fy = cam16[13]; cam.cx = cam16[14]; cam.cy = cam16[15];
  cam.w = (int)cam16[16]; cam.h = (int)cam16[17];
  cudaMemsetAsync(b->counters, 0, 4 * sizeof(int), st);
  const LevelInfo lv = make_lv(m);
  render_rays_kernel<<<(tw * th + 3) / 4, 128, 0, st>>>(cam, make_scene(m), m->bits, x0, y0, tw, th,
                                                           b->max_samples, max_per_ray, b->rays, b->coords, b->tdist, b->counters);
  NGP_CHECK_LAUNCH();
  if (packed) {
    r = nslam_ngp_forward_tc(m, packed, b->coords, b->counters, -1, b->max_samples, b->rgbsigma, nullptr, num_sms, stream);
    if (r) return r;
  } else {
    forward_kernel<<<(b->max_samples + TILE - 1) / TILE, TILE, FWD_SMEM, st>>>(b->coords, b->counters, -1,
                                                                              (const __half2*)m->grid_half, lv, m->mlp, b->rgbsigma);
    NGP_CHECK_LAUNCH();
  }
  loss_kernel<<<(tw * th + 3) / 4, 128, 0, st>>>(b->rays, tw * th, b->coords, b->tdist, b->rgbsigma, b->counters,
                                                      0.f, make_float3(bg_r, bg_g, bg_b), 1, nullptr, nullptr, out_rgbd);
  NGP_CHECK_LAUNCH();
  return 0;
}

/* training-image slot upload from the SLAM packet, all on the device (B1/B2) */
int nslam_ngp_ingest_image(const unsigned char* rgb_chw, const float* idepth_up, const float* depth_cov_up,
                           int H, int W, void* rgba_slot, float* depth_slot, float* cov_slot, void* stream) {
  ngp::ingest_image_kernel<<<(H * W + 255) / 256, 256, 0, (cudaStream_t)stream>>>(
      rgb_chw, idepth_up, depth_cov_up, H, W, (__half*)rgba_slot, depth_slot, cov_slot);
  NGP_CHECK_LAUNCH();
  return 0;
}

/* B1/B2 in one launch: n keyframes of a SLAM packet (images u8 [n,3,H,W], idepth_up / depth_cov_up [n,H,W], slot ids
 * [n] int64, cam_T_world [n,7] or NULL) into the trainer's slot arrays (rgba [N,H,W,4] fp16, depth / depth_cov [N,H,W])
 * and camera records cams [N] (when cam_T_world is given).  cams_base / cam_state [3,N,6] / cam_steps [N] (or NULL): the
 * pose-refinement state of the trainer (csrc/ngp_extrinsics.cu) — base camera rewritten, offsets and moments reset.
 * All pointers DEVICE. */
int nslam_ngp_ingest_batch(const unsigned char* rgb_chw, const float* idepth_up, const float* depth_cov_up,
                           const long long* ids, int n, int H, int W, void* rgba, float* depth, float* depth_cov,
                           const float* cam_T_world, float fx, float fy, float cx, float cy, void* cams, void* cams_base,
                           float* cam_state, int* cam_steps, int n_slots, void* stream) {
  if (n <= 0) return 0;
  dim3 grid((H * W + 255) / 256, n);
  ngp::ingest_batch_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(
      rgb_chw, idepth_up, depth_cov_up, ids, H, W, (__half*)rgba, depth, depth_cov, cam_T_world, fx, fy, cx, cy,
      (ngp::Camera*)cams, (ngp::Camera*)cams_base, cam_state, cam_steps, n_slots);
  NGP_CHECK_LAUNCH();
  return 0;
}

}  // extern "C"
