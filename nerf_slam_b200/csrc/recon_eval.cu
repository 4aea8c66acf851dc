// Reconstruction evaluation against ground truth: area-uniform surface sampling, exact nearest neighbours through a
// linear BVH, the camera visibility mask of ground-truth points, and the metric sums.  The rules below DEFINE the
// behaviour; tests/recon_eval_oracle.py restates them (fp64 numpy, scipy's cKDTree for the neighbours).  Every fp64
// step uses an explicit-rounding intrinsic (nvcc would otherwise contract mul-adds into FMAs), so numpy, which rounds
// every elementwise operation, reproduces it.
//
// Surface sampling.  Triangle t = (a, b, c) of vertices [V,3] fp32: e1 = b - a, e2 = c - a (fp64), x = e1 × e2
// (x0 = e1y e2z - e1z e2y, x1 = e1z e2x - e1x e2z, x2 = e1x e2y - e1y e2x), area = 0.5 sqrt((x0² + x1²) + x2²), its
// weight w = rint(area · 2^40) as an unsigned 64-bit integer (round to nearest even).  A triangle with a vertex index
// outside [0, V), a non-finite area or w > 2^62 / T gets w = 0 and raises a flag.  cdf = inclusive scan of w (CUB,
// integers: exact), total = cdf[T-1] (must be > 0).  The hash of (seed, i, k) is splitmix64's finaliser of
// seed · 0x9E3779B97F4A7C15 + (3i + k + 1) · 0xD1B54A32D192ED03 (mod 2^64): x ^= x >> 30; x *= 0xBF58476D1CE4E5B9;
// x ^= x >> 27; x *= 0x94D049BB133111EB; x ^= x >> 31.  Sample i: target = floor(hash(seed, i, 0) · total / 2^64)
// (the high word of the 128-bit product); the triangle is the first j with cdf[j] > target (binary search), so a
// triangle is chosen with probability w / total and a zero-weight one never.  u = (hash(seed, i, 1) >> 11) · 2^-53,
// v = (hash(seed, i, 2) >> 11) · 2^-53, s = sqrt(u), p = ((1 - s) a + (s (1 - v)) b) + (s v) c per axis in fp64
// (each product and sum rounded), rounded to fp32 once.
//
// Nearest neighbour.  The distance of query q to reference r is sqrt(fp64 ((dx² + dy²) + dz²)) with d = q - r of the
// fp32 coordinates in fp64, rounded to fp32 once.  The nearest reference is the one with the smallest fp64 squared
// distance, ties to the smaller reference index; only references with squared distance < max_dist² (fp64) count
// (cKDTree's distance_upper_bound); none -> +inf and -1.  The BVH (Karras 2012; lbvh.cuh): 63-bit Morton keys of the points
// quantised to 2^21 cells per axis of their bounding box, CUB radix SortPairs of (key, index) (stable, so the index
// breaks ties), leaf buckets of `leaf_size` consecutive sorted points, L - 1 internal nodes from the buckets' first
// keys (equal keys split by bucket index), boxes bottom-up (min / max: exact, whatever order threads arrive in).
// The traversal keeps a stack, visits the nearer child first and skips a box whose fp64 squared distance, computed with
// the same rounded operations as the points' (so never larger than any point's inside it), exceeds the best so far.
// The search is exact, so neither the tree (leaf_size) nor the launch (num_sms) can change a result.  Queries are
// visited in Morton order of the same quantisation (a sort of their keys) so that a warp walks one part of the tree.
//
// Visibility.  Camera k: R = the rotation of q_xyzw rounded to fp32 (tsdf_pose_rotation, as the TSDF kernels take it),
// p_c = ((R0 x + R1 y) + R2 z) + t per row in fp64, u = fx (p_cx / p_cz) + cx, v = fy (p_cy / p_cz) + cy.  The point
// is seen when near < p_cz <= far, the nearest pixel (floor(u + 0.5), floor(v + 0.5)) lies in the W x H image and, with
// depth maps, d = depth[k, v, u] <= 0 (no measurement: not tested) or p_cz <= d + tol (fp64 sum).  Visible = seen by
// at least one camera.
//
// Metric sums.  For dist [n]: sum of rint(min(d, max_dist) · 2^32) as 64-bit integers (integer atomics: the same bits
// in every run), the count with d < threshold and the count with d = +inf.
//
// Scratch: sampling 16 B per triangle + CUB's scan storage; the BVH about 110 B per reference point (keys, indices, the
// sorted points, 2 L - 1 node boxes, links, CUB's sort storage); the queries 24 B per query + CUB's sort storage.
#include "nslam_eval.h"
#include "lbvh.cuh"
#include "mesh_rules.cuh"
#include "tsdf_rules.cuh"

#include <climits>
#include <cmath>
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>

namespace nslam {

// ------------------------------------------------------------------------------------------------------------ sampling
__device__ __forceinline__ unsigned long long ev_hash(unsigned long long seed, long long i, int k) {
  unsigned long long x = seed * 0x9E3779B97F4A7C15ull + ((unsigned long long)i * 3ull + (unsigned long long)k + 1ull) *
                                                            0xD1B54A32D192ED03ull;
  x ^= x >> 30;
  x *= 0xBF58476D1CE4E5B9ull;
  x ^= x >> 27;
  x *= 0x94D049BB133111EBull;
  x ^= x >> 31;
  return x;
}

__device__ __forceinline__ double ev_unit(unsigned long long h) { return (double)(h >> 11) * 0x1p-53; }

__global__ void __launch_bounds__(256) ev_area_kernel(const float* V, int nv, const int* T, int nt, unsigned long long cap,
                                                      unsigned long long* w, unsigned long long* flags) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= nt) return;
  const int ia = T[3 * (size_t)t], ib = T[3 * (size_t)t + 1], ic = T[3 * (size_t)t + 2];
  if (ia < 0 || ia >= nv || ib < 0 || ib >= nv || ic < 0 || ic >= nv) {
    w[t] = 0;
    atomicOr(flags, 1ull);
    return;
  }
  unsigned long long wt;
  const unsigned f = tri_area_weight(V, ia, ib, ic, cap, wt);
  w[t] = wt;
  if (f) atomicOr(flags, (unsigned long long)f);
}

__global__ void __launch_bounds__(256) ev_sample_kernel(const float* V, const int* T, const unsigned long long* cdf, int nt,
                                                        int n, unsigned long long seed, float* out, int* tri) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const unsigned long long total = cdf[nt - 1];
  const unsigned long long target = __umul64hi(ev_hash(seed, i, 0), total);
  int lo = 0, hi = nt - 1;                       // first j with cdf[j] > target (exists: cdf[nt-1] = total > target)
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (cdf[mid] > target) hi = mid; else lo = mid + 1;
  }
  const double u = ev_unit(ev_hash(seed, i, 1)), v = ev_unit(ev_hash(seed, i, 2));
  const double s = __dsqrt_rn(u);
  const double wa = __dsub_rn(1.0, s), wb = __dmul_rn(s, __dsub_rn(1.0, v)), wc = __dmul_rn(s, v);
  const size_t t3 = 3 * (size_t)lo;
  const int ia = T[t3], ib = T[t3 + 1], ic = T[t3 + 2];
#pragma unroll
  for (int c = 0; c < 3; c++) {
    const double p = __dadd_rn(__dadd_rn(__dmul_rn(wa, (double)V[3 * (size_t)ia + c]), __dmul_rn(wb, (double)V[3 * (size_t)ib + c])),
                               __dmul_rn(wc, (double)V[3 * (size_t)ic + c]));
    out[3 * (size_t)i + c] = __double2float_rn(p);
  }
  if (tri) tri[i] = lo;
}

struct SurfaceScratch {
  unsigned long long *w, *cdf;
  void* cub;
  size_t cub_bytes;
};

static size_t surface_scratch(int nt, void* base, SurfaceScratch* s) {
  size_t scan_bytes = 0;
  cub::DeviceScan::InclusiveSum((void*)nullptr, scan_bytes, (const unsigned long long*)nullptr, (unsigned long long*)nullptr, nt);
  ScratchCarver c(base);
  SurfaceScratch t;
  t.w = c.take<unsigned long long>(8 * (size_t)nt);
  t.cdf = c.take<unsigned long long>(8 * (size_t)nt);
  t.cub_bytes = scan_bytes;
  t.cub = c.take(scan_bytes);
  if (s) *s = t;
  return c.off;
}

// ----------------------------------------------------------------------------------------------------------------- BVH
constexpr int kStack = 96;      // > the deepest tree: 63 key bits + 31 bits of bucket index among equal keys

__global__ void __launch_bounds__(256) ev_gather_kernel(const float* P, const int* order, int n, float4* pts) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int j = order[i];
  pts[i] = make_float4(P[3 * (size_t)j], P[3 * (size_t)j + 1], P[3 * (size_t)j + 2], __int_as_float(j));
}

// the box of leaf bucket l: min / max of its sorted points
struct PointLeaf {
  const float4* pts;
  int n, B;
  __device__ void operator()(int l, float lo[3], float hi[3]) const {
    const int s = l * B, e = min(n, s + B);
    for (int j = s; j < e; j++) {
      const float4 p = pts[j];
      lo[0] = fminf(lo[0], p.x); lo[1] = fminf(lo[1], p.y); lo[2] = fminf(lo[2], p.z);
      hi[0] = fmaxf(hi[0], p.x); hi[1] = fmaxf(hi[1], p.y); hi[2] = fmaxf(hi[2], p.z);
    }
  }
};

struct BvhLayout {
  unsigned* bounds;              // [6] ordered fp32: lo xyz, hi xyz
  unsigned long long *keys, *sorted;
  int *index, *order;
  float4* pts;                   // sorted points, .w = the input index (int bits)
  float* box;                    // [2L-1][6]
  int2* child;                   // [L-1]
  int *parent, *flags;           // [2L-1], [L-1]
  void* cub;
  size_t cub_bytes;
  int L;
};

static size_t bvh_layout(int n, int B, void* base, BvhLayout* s) {
  BvhLayout t;
  t.L = (n + B - 1) / B;
  const size_t nodes = 2 * (size_t)t.L - 1;
  size_t sort_bytes = 0;
  cub::DeviceRadixSort::SortPairs((void*)nullptr, sort_bytes, (const unsigned long long*)nullptr, (unsigned long long*)nullptr,
                                  (const int*)nullptr, (int*)nullptr, n);
  ScratchCarver c(base);
  t.bounds = c.take<unsigned>(6 * 4);
  t.keys = c.take<unsigned long long>(8 * (size_t)n);
  t.sorted = c.take<unsigned long long>(8 * (size_t)n);
  t.index = c.take<int>(4 * (size_t)n);
  t.order = c.take<int>(4 * (size_t)n);
  t.pts = c.take<float4>(16 * (size_t)n);
  t.box = c.take<float>(24 * nodes);
  t.child = c.take<int2>(8 * (size_t)t.L);
  t.parent = c.take<int>(4 * nodes);
  t.flags = c.take<int>(4 * (size_t)t.L);
  t.cub_bytes = sort_bytes;
  t.cub = c.take(sort_bytes);
  if (s) *s = t;
  return c.off;
}

struct QueryScratch {
  unsigned long long *keys, *sorted;
  int *index, *order;
  void* cub;
  size_t cub_bytes;
};

static size_t query_scratch(int n, void* base, QueryScratch* s) {
  size_t sort_bytes = 0;
  cub::DeviceRadixSort::SortPairs((void*)nullptr, sort_bytes, (const unsigned long long*)nullptr, (unsigned long long*)nullptr,
                                  (const int*)nullptr, (int*)nullptr, n);
  ScratchCarver c(base);
  QueryScratch t;
  t.keys = c.take<unsigned long long>(8 * (size_t)n);
  t.sorted = c.take<unsigned long long>(8 * (size_t)n);
  t.index = c.take<int>(4 * (size_t)n);
  t.order = c.take<int>(4 * (size_t)n);
  t.cub_bytes = sort_bytes;
  t.cub = c.take(sort_bytes);
  if (s) *s = t;
  return c.off;
}

// fp64 squared distance of q to a box with the points' rounded operations: per axis the gap max(lo - q, q - hi, 0)
__device__ __forceinline__ double ev_box_d2(const float* b, const double q[3]) {
  double g[3];
#pragma unroll
  for (int c = 0; c < 3; c++) {
    const double lo = __dsub_rn((double)__ldg(b + c), q[c]), hi = __dsub_rn(q[c], (double)__ldg(b + 3 + c));
    g[c] = fmax(fmax(lo, hi), 0.0);
  }
  return __dadd_rn(__dadd_rn(__dmul_rn(g[0], g[0]), __dmul_rn(g[1], g[1])), __dmul_rn(g[2], g[2]));
}

__global__ void __launch_bounds__(128) ev_nearest_kernel(const float4* pts, const float* box, const int2* child, int n, int B,
                                                         int L, const float* Q, const int* order, int nq, double bound2,
                                                         float* dist, long long* idx) {
  int snode[kStack];
  float sd[kStack];
  for (int t = blockIdx.x * blockDim.x + threadIdx.x; t < nq; t += gridDim.x * blockDim.x) {
    const int qi = order[t];
    const double q[3] = {(double)Q[3 * (size_t)qi], (double)Q[3 * (size_t)qi + 1], (double)Q[3 * (size_t)qi + 2]};
    double best = bound2;
    int best_i = -1;
    int sp = 0;
    snode[sp] = 0;
    sd[sp++] = __double2float_rd(ev_box_d2(box, q));
    while (sp > 0) {
      --sp;
      int node = snode[sp];
      if ((double)sd[sp] > best) continue;            // rounded down: never skips a box that could hold the answer
      while (true) {
        if (node >= L - 1) {                          // leaf: its bucket of sorted points
          const int s = (node - (L - 1)) * B, e = min(n, s + B);
          for (int j = s; j < e; j++) {
            const float4 r = __ldg(pts + j);
            const double dx = __dsub_rn(q[0], (double)r.x), dy = __dsub_rn(q[1], (double)r.y), dz = __dsub_rn(q[2], (double)r.z);
            const double d2 = __dadd_rn(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)), __dmul_rn(dz, dz));
            const int ri = __float_as_int(r.w);
            if (d2 < best || (d2 == best && best_i >= 0 && ri < best_i)) {
              best = d2;
              best_i = ri;
            }
          }
          break;
        }
        const int2 ch = __ldg(child + node);
        const double d0 = ev_box_d2(box + 6 * (size_t)ch.x, q), d1 = ev_box_d2(box + 6 * (size_t)ch.y, q);
        const bool v0 = d0 <= best, v1 = d1 <= best;
        if (v0 && v1) {
          const bool first0 = d0 <= d1;
          snode[sp] = first0 ? ch.y : ch.x;
          sd[sp++] = __double2float_rd(first0 ? d1 : d0);
          node = first0 ? ch.x : ch.y;
        } else if (v0) {
          node = ch.x;
        } else if (v1) {
          node = ch.y;
        } else {
          break;
        }
      }
    }
    if (best_i >= 0) {
      dist[qi] = __double2float_rn(__dsqrt_rn(best));
      idx[qi] = best_i;
    } else {
      dist[qi] = INFINITY;
      idx[qi] = -1;
    }
  }
}

// ---------------------------------------------------------------------------------------------------------- visibility
constexpr int kVisThreads = 256;
constexpr int kVisCams = 64;    // cameras staged in shared memory per round

__global__ void __launch_bounds__(kVisThreads) ev_visible_kernel(const float* P, int n, const float* poses, int ncam,
                                                                 const float* intr, int W, int H, const float* depths,
                                                                 float tol, float near_z, float far_z, unsigned char* mask) {
  __shared__ double sR[kVisCams][12];           // rotation (fp32-rounded) and translation per camera
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  const bool active = i < n;
  double p[3] = {0.0, 0.0, 0.0};
  if (active)
    for (int c = 0; c < 3; c++) p[c] = (double)P[3 * (size_t)i + c];
  const double fx = intr[0], fy = intr[1], cx = intr[2], cy = intr[3];
  bool seen = false;
  for (int k0 = 0; k0 < ncam; k0 += kVisCams) {
    const int m = min(kVisCams, ncam - k0);
    __syncthreads();
    for (int k = threadIdx.x; k < m; k += blockDim.x) {
      const float* q = poses + 7 * (size_t)(k0 + k);
      tsdf_pose_rotation(q, sR[k]);
      for (int c = 0; c < 3; c++) sR[k][9 + c] = (double)q[c];
    }
    __syncthreads();
    if (!active || seen) continue;
    for (int k = 0; k < m && !seen; k++) {
      const double* R = sR[k];
      double pc[3];
#pragma unroll
      for (int r = 0; r < 3; r++)
        pc[r] = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(R[3 * r], p[0]), __dmul_rn(R[3 * r + 1], p[1])), __dmul_rn(R[3 * r + 2], p[2])),
                          R[9 + r]);
      if (!(pc[2] > (double)near_z && pc[2] <= (double)far_z)) continue;
      const double u = __dadd_rn(__dmul_rn(fx, __ddiv_rn(pc[0], pc[2])), cx);
      const double v = __dadd_rn(__dmul_rn(fy, __ddiv_rn(pc[1], pc[2])), cy);
      const double ui = floor(__dadd_rn(u, 0.5)), vi = floor(__dadd_rn(v, 0.5));
      if (!(ui >= 0.0 && ui < (double)W && vi >= 0.0 && vi < (double)H)) continue;
      if (depths) {
        const float d = depths[((size_t)(k0 + k) * H + (size_t)vi) * W + (size_t)ui];
        if (d > 0.f && !(pc[2] <= __dadd_rn((double)d, (double)tol))) continue;
      }
      seen = true;
    }
  }
  if (active) mask[i] = seen ? 1 : 0;
}

// ------------------------------------------------------------------------------------------------------------- metrics
__global__ void __launch_bounds__(256) ev_reduce_kernel(const float* dist, int n, float max_dist, float thr,
                                                        unsigned long long* out) {
  unsigned long long s = 0, below = 0, miss = 0;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const float d = dist[i];
    s += __double2ull_rn(__dmul_rn((double)fminf(d, max_dist), 0x1p32));
    below += d < thr;
    miss += isinf(d) && d > 0.f;
  }
  for (int m = 16; m; m >>= 1) {
    s += __shfl_xor_sync(0xffffffffu, s, m);
    below += __shfl_xor_sync(0xffffffffu, below, m);
    miss += __shfl_xor_sync(0xffffffffu, miss, m);
  }
  if ((threadIdx.x & 31) == 0) {
    atomicAdd(out, s);
    atomicAdd(out + 1, below);
    atomicAdd(out + 2, miss);
  }
}

}  // namespace nslam

extern "C" {

int nslam_eval_surface_scratch(int n_tri, long long* bytes) {
  using namespace nslam;
  if (n_tri <= 0) return (int)cudaErrorInvalidValue;
  *bytes = (long long)surface_scratch(n_tri, nullptr, nullptr);
  return 0;
}

int nslam_eval_surface_area(const float* vertices, int n_vert, const int* triangles, int n_tri, void* scratch,
                            long long scratch_bytes, long long* info, void* stream) {
  using namespace nslam;
  if (n_tri <= 0 || n_vert <= 0) return (int)cudaErrorInvalidValue;
  SurfaceScratch s;
  if ((long long)surface_scratch(n_tri, scratch, &s) > scratch_bytes) return (int)cudaErrorInvalidValue;
  cudaStream_t st = (cudaStream_t)stream;
  cudaError_t e = cudaMemsetAsync(info, 0, 2 * sizeof(long long), st);
  if (e != cudaSuccess) return (int)e;
  const unsigned long long cap = (1ull << 62) / (unsigned long long)n_tri;
  ev_area_kernel<<<(n_tri + 255) / 256, 256, 0, st>>>(vertices, n_vert, triangles, n_tri, cap, s.w,
                                                      (unsigned long long*)(info + 1));
  NSLAM_CHECK_LAUNCH();
  size_t tb = s.cub_bytes;
  if ((e = cub::DeviceScan::InclusiveSum(s.cub, tb, s.w, s.cdf, n_tri, st)) != cudaSuccess) return (int)e;
  return (int)cudaMemcpyAsync(info, s.cdf + n_tri - 1, sizeof(long long), cudaMemcpyDeviceToDevice, st);
}

int nslam_eval_sample_surface(const float* vertices, const int* triangles, int n_tri, int n, unsigned long long seed,
                              const void* scratch, long long scratch_bytes, float* points, int* tri, void* stream) {
  using namespace nslam;
  if (n_tri <= 0 || n < 0) return (int)cudaErrorInvalidValue;
  SurfaceScratch s;
  if ((long long)surface_scratch(n_tri, (void*)scratch, &s) > scratch_bytes) return (int)cudaErrorInvalidValue;
  if (n == 0) return 0;
  ev_sample_kernel<<<(n + 255) / 256, 256, 0, (cudaStream_t)stream>>>(vertices, triangles, s.cdf, n_tri, n, seed, points, tri);
  NSLAM_CHECK_LAUNCH();
  return 0;
}

int nslam_eval_bvh_scratch(int n_ref, int leaf_size, long long* bytes) {
  using namespace nslam;
  if (n_ref <= 0 || leaf_size < 1 || leaf_size > 32) return (int)cudaErrorInvalidValue;
  *bytes = (long long)bvh_layout(n_ref, leaf_size, nullptr, nullptr);
  return 0;
}

int nslam_eval_bvh_build(const float* ref, int n_ref, int leaf_size, void* bvh, long long bvh_bytes, void* stream) {
  using namespace nslam;
  if (n_ref <= 0 || leaf_size < 1 || leaf_size > 32) return (int)cudaErrorInvalidValue;
  BvhLayout s;
  if ((long long)bvh_layout(n_ref, leaf_size, bvh, &s) > bvh_bytes) return (int)cudaErrorInvalidValue;
  cudaStream_t st = (cudaStream_t)stream;
  cudaError_t e;
  if ((e = cudaMemsetAsync(s.bounds, 0xff, 3 * sizeof(unsigned), st)) != cudaSuccess) return (int)e;
  if ((e = cudaMemsetAsync(s.bounds + 3, 0, 3 * sizeof(unsigned), st)) != cudaSuccess) return (int)e;
  if ((e = cudaMemsetAsync(s.flags, 0, sizeof(int) * (size_t)s.L, st)) != cudaSuccess) return (int)e;
  const int nb = (n_ref + 255) / 256;
  ev_bounds_kernel<<<ev_grid(n_ref, 256, 1024), 256, 0, st>>>(ref, n_ref, s.bounds);
  NSLAM_CHECK_LAUNCH();
  ev_keys_kernel<<<nb, 256, 0, st>>>(ref, n_ref, s.bounds, s.keys, s.index);
  NSLAM_CHECK_LAUNCH();
  size_t tb = s.cub_bytes;
  if ((e = cub::DeviceRadixSort::SortPairs(s.cub, tb, s.keys, s.sorted, s.index, s.order, n_ref, 0, 3 * kMortonBits, st)) !=
      cudaSuccess)
    return (int)e;
  ev_gather_kernel<<<nb, 256, 0, st>>>(ref, s.order, n_ref, s.pts);
  NSLAM_CHECK_LAUNCH();
  if (s.L > 1) {
    ev_internal_kernel<<<(s.L - 1 + 255) / 256, 256, 0, st>>>(s.sorted, leaf_size, s.L, s.child, s.parent);
    NSLAM_CHECK_LAUNCH();
  } else if ((e = cudaMemsetAsync(s.parent, 0xff, sizeof(int), st)) != cudaSuccess) {
    return (int)e;
  }
  ev_boxes_kernel<<<(s.L + 255) / 256, 256, 0, st>>>(PointLeaf{s.pts, n_ref, leaf_size}, s.L, s.child, s.parent, s.flags,
                                                     s.box);
  NSLAM_CHECK_LAUNCH();
  return 0;
}

int nslam_eval_nearest_scratch(int n_query, long long* bytes) {
  using namespace nslam;
  if (n_query <= 0) return (int)cudaErrorInvalidValue;
  *bytes = (long long)query_scratch(n_query, nullptr, nullptr);
  return 0;
}

int nslam_eval_nearest(const void* bvh, long long bvh_bytes, int n_ref, int leaf_size, const float* query, int n_query,
                       float max_dist, int num_sms, void* scratch, long long scratch_bytes, float* dist, long long* idx,
                       void* stream) {
  using namespace nslam;
  if (n_ref <= 0 || leaf_size < 1 || leaf_size > 32 || n_query <= 0 || !(max_dist > 0.f)) return (int)cudaErrorInvalidValue;
  BvhLayout b;
  if ((long long)bvh_layout(n_ref, leaf_size, (void*)bvh, &b) > bvh_bytes) return (int)cudaErrorInvalidValue;
  QueryScratch s;
  if ((long long)query_scratch(n_query, scratch, &s) > scratch_bytes) return (int)cudaErrorInvalidValue;
  cudaStream_t st = (cudaStream_t)stream;
  cudaError_t e;
  if (num_sms <= 0) {
    int dev = 0;
    if ((e = cudaGetDevice(&dev)) != cudaSuccess) return (int)e;
    if ((e = cudaDeviceGetAttribute(&num_sms, cudaDevAttrMultiProcessorCount, dev)) != cudaSuccess) return (int)e;
  }
  const int nb = (n_query + 255) / 256;
  ev_keys_kernel<<<nb, 256, 0, st>>>(query, n_query, b.bounds, s.keys, s.index);
  NSLAM_CHECK_LAUNCH();
  size_t tb = s.cub_bytes;
  if ((e = cub::DeviceRadixSort::SortPairs(s.cub, tb, s.keys, s.sorted, s.index, s.order, n_query, 0, 3 * kMortonBits, st)) !=
      cudaSuccess)
    return (int)e;
  const double md = (double)max_dist;
  const double bound2 = std::isinf(md) ? (double)INFINITY : md * md;
  ev_nearest_kernel<<<ev_grid(n_query, 128, num_sms * 16), 128, 0, st>>>(b.pts, b.box, b.child, n_ref, leaf_size, b.L, query,
                                                                         s.order, n_query, bound2, dist, idx);
  NSLAM_CHECK_LAUNCH();
  return 0;
}

int nslam_eval_visible(const float* points, int n_points, const float* cam_T_world, int n_cams, const float* intr4, int W,
                       int H, const float* depths, float depth_tol, float near_z, float far_z, unsigned char* mask,
                       void* stream) {
  using namespace nslam;
  if (n_points < 0 || n_cams < 0 || W <= 0 || H <= 0) return (int)cudaErrorInvalidValue;
  if (n_points == 0) return 0;
  ev_visible_kernel<<<(n_points + kVisThreads - 1) / kVisThreads, kVisThreads, 0, (cudaStream_t)stream>>>(
      points, n_points, cam_T_world, n_cams, intr4, W, H, depths, depth_tol, near_z, far_z, mask);
  NSLAM_CHECK_LAUNCH();
  return 0;
}

int nslam_eval_reduce(const float* dist, int n, float max_dist, float threshold, long long* out, void* stream) {
  using namespace nslam;
  if (n < 0 || !(max_dist > 0.f) || !std::isfinite(max_dist) || (double)n * (double)max_dist >= 2147483648.0)
    return (int)cudaErrorInvalidValue;
  cudaStream_t st = (cudaStream_t)stream;
  cudaError_t e = cudaMemsetAsync(out, 0, 3 * sizeof(long long), st);
  if (e != cudaSuccess) return (int)e;
  if (n == 0) return 0;
  ev_reduce_kernel<<<ev_grid(n, 256, 1184), 256, 0, st>>>(dist, n, max_dist, threshold, (unsigned long long*)out);
  NSLAM_CHECK_LAUNCH();
  return 0;
}

}  // extern "C"
