// Building blocks of the linear BVH (Karras 2012) shared by the nearest-neighbour search (recon_eval.cu) and the mesh
// renderer (mesh_render.cu): ordered-float bounds, 63-bit Morton keys quantised to 2^21 cells per axis of the bounding
// box, the internal nodes from the sorted keys of the leaf buckets, and the bottom-up boxes.  Every box is a min / max of
// fp32 coordinates, so it is exact whatever order threads arrive in.
#pragma once
#include "common.cuh"

namespace nslam {

constexpr int kMortonBits = 21;

// order-preserving map of fp32 to u32, so that integer atomics give the exact min / max
__device__ __forceinline__ unsigned ev_ord(float f) {
  const unsigned b = __float_as_uint(f);
  return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}
__device__ __forceinline__ float ev_unord(unsigned o) {
  return __uint_as_float((o & 0x80000000u) ? (o & 0x7fffffffu) : ~o);
}

__device__ __forceinline__ unsigned long long ev_spread(unsigned v) {
  unsigned long long x = v & 0x1fffffu;
  x = (x | x << 32) & 0x1f00000000ffffull;
  x = (x | x << 16) & 0x1f0000ff0000ffull;
  x = (x | x << 8) & 0x100f00f00f00f00full;
  x = (x | x << 4) & 0x10c30c30c30c30c3ull;
  x = (x | x << 2) & 0x1249249249249249ull;
  return x;
}

// Morton key of p in the box bounds (ordered lo[3], hi[3]); outside points clamp to the nearest cell
__device__ __forceinline__ unsigned long long ev_morton(float x, float y, float z, const unsigned* bounds) {
  const float p[3] = {x, y, z};
  unsigned q[3];
#pragma unroll
  for (int c = 0; c < 3; c++) {
    const float lo = ev_unord(bounds[c]), hi = ev_unord(bounds[3 + c]);
    const float ext = hi - lo;
    float f = ext > 0.f ? (p[c] - lo) / ext * (float)(1 << kMortonBits) : 0.f;
    f = fminf(fmaxf(f, 0.f), (float)((1 << kMortonBits) - 1));   // NaN -> 0
    q[c] = (unsigned)f;
  }
  return ev_spread(q[0]) << 2 | ev_spread(q[1]) << 1 | ev_spread(q[2]);
}

// bounds [6] (ordered lo xyz, hi xyz; set to 0xff.. / 0 before) of the points P [n,3]
static __global__ void __launch_bounds__(256) ev_bounds_kernel(const float* P, int n, unsigned* bounds) {
  unsigned lo[3] = {0xffffffffu, 0xffffffffu, 0xffffffffu}, hi[3] = {0u, 0u, 0u};
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
#pragma unroll
    for (int c = 0; c < 3; c++) {
      const unsigned o = ev_ord(P[3 * (size_t)i + c]);
      lo[c] = min(lo[c], o);
      hi[c] = max(hi[c], o);
    }
  }
#pragma unroll
  for (int c = 0; c < 3; c++) {
    for (int m = 16; m; m >>= 1) {
      lo[c] = min(lo[c], __shfl_xor_sync(0xffffffffu, lo[c], m));
      hi[c] = max(hi[c], __shfl_xor_sync(0xffffffffu, hi[c], m));
    }
  }
  if ((threadIdx.x & 31) == 0) {
#pragma unroll
    for (int c = 0; c < 3; c++) {
      atomicMin(bounds + c, lo[c]);
      atomicMax(bounds + 3 + c, hi[c]);
    }
  }
}

static __global__ void __launch_bounds__(256) ev_keys_kernel(const float* P, int n, const unsigned* bounds, unsigned long long* keys,
                                                      int* index) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  keys[i] = ev_morton(P[3 * (size_t)i], P[3 * (size_t)i + 1], P[3 * (size_t)i + 2], bounds);
  index[i] = i;
}

// common-prefix length of buckets i and j (keys = the sorted keys, bucket b starts at sorted position b * B); -1 when
// j is outside [0, L)
__device__ __forceinline__ int ev_delta(const unsigned long long* keys, int B, long long L, long long i, long long j) {
  if (j < 0 || j >= L) return -1;
  const unsigned long long ki = keys[i * B], kj = keys[j * B];
  return ki == kj ? 64 + __clz((int)(i ^ j)) : __clzll((long long)(ki ^ kj));
}

// Karras 2012: node ids 0 .. L-2 internal, L-1 .. 2L-2 the leaves (leaf l = L-1+l); the root is node 0
static __global__ void __launch_bounds__(256) ev_internal_kernel(const unsigned long long* keys, int B, int L, int2* child,
                                                          int* parent) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= L - 1) return;
  const int d = ev_delta(keys, B, L, i, i + 1) - ev_delta(keys, B, L, i, i - 1) >= 0 ? 1 : -1;
  const int dmin = ev_delta(keys, B, L, i, i - d);
  long long lmax = 2;
  while (ev_delta(keys, B, L, i, i + lmax * d) > dmin) lmax *= 2;
  long long l = 0;
  for (long long t = lmax / 2; t >= 1; t /= 2)
    if (ev_delta(keys, B, L, i, i + (l + t) * d) > dmin) l += t;
  const long long j = i + l * d;
  const int dnode = ev_delta(keys, B, L, i, j);
  long long s = 0, t = l;
  do {
    t = (t + 1) >> 1;
    if (ev_delta(keys, B, L, i, i + (s + t) * d) > dnode) s += t;
  } while (t > 1);
  const int gamma = (int)(i + s * d + min(d, 0));
  const int lo = (int)min((long long)i, j), hi = (int)max((long long)i, j);
  const int left = lo == gamma ? L - 1 + gamma : gamma;
  const int right = hi == gamma + 1 ? L - 1 + gamma + 1 : gamma + 1;
  child[i] = make_int2(left, right);
  parent[left] = i;
  parent[right] = i;
  if (i == 0) parent[0] = -1;
}

// Leaf boxes, then up the tree: the second child to arrive at a node writes its box.  box [2L-1][6] (lo xyz, hi xyz);
// flags [L-1] zero before.  The leaf functor fills the box of leaf l:  void Leaf::operator()(int l, float lo[3],
// float hi[3]) const, with lo / hi set to +inf / -inf on entry.
template <class Leaf>
__global__ void __launch_bounds__(256) ev_boxes_kernel(Leaf leaf, int L, const int2* child, const int* parent, int* flags,
                                                       float* box) {
  const int l = blockIdx.x * blockDim.x + threadIdx.x;
  if (l >= L) return;
  float lo[3] = {INFINITY, INFINITY, INFINITY}, hi[3] = {-INFINITY, -INFINITY, -INFINITY};
  leaf(l, lo, hi);
  int node = L - 1 + l;
  float* b = box + 6 * (size_t)node;
  for (int c = 0; c < 3; c++) { b[c] = lo[c]; b[3 + c] = hi[c]; }
  __threadfence();
  node = parent[node];
  while (node >= 0) {
    if (atomicAdd(flags + node, 1) == 0) return;           // the sibling's box is not written yet: it goes on
    __threadfence();
    const int2 ch = child[node];
    const float* b0 = box + 6 * (size_t)ch.x;
    const float* b1 = box + 6 * (size_t)ch.y;
    float* bn = box + 6 * (size_t)node;
    for (int c = 0; c < 3; c++) {
      bn[c] = fminf(__ldcg(b0 + c), __ldcg(b1 + c));
      bn[3 + c] = fmaxf(__ldcg(b0 + 3 + c), __ldcg(b1 + 3 + c));
    }
    __threadfence();
    node = parent[node];
  }
}

static inline int ev_grid(long long n, int threads, int cap) {
  const long long b = (n + threads - 1) / threads;
  return (int)(b < cap ? (b > 0 ? b : 1) : cap);
}

}  // namespace nslam
