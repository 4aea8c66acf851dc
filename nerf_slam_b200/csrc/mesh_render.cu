// Depth, triangle-id, normal and colour views of a triangle mesh by exact ray casting through a linear BVH over the
// triangles.  The rules below DEFINE the behaviour; tests/mesh_render_oracle.py restates them in fp64 by brute force over
// all triangles.  Every fp64 step uses an explicit-rounding intrinsic (nvcc would otherwise contract mul-adds into
// FMAs), so numpy, which rounds every elementwise operation, reproduces it bit for bit.
//
// Rays.  View k: R = the rotation of cam_T_world[k] = (t, q_xyzw) rounded to fp32 (tsdf_pose_rotation, as the TSDF ray
// cast takes it), the origin o = -R^T t in fp64: o_c = -((R0c t0 + R1c t1) + R2c t2).  Pixel (u, v): dx = (u - cx) / fx,
// dy = (v - cy) / fy, each a fp32 subtraction and division (as tsdf_raycast_kernel), and the direction d_c =
// (R0c dx + R1c dy) + R2c in fp64.  The camera-frame direction is (dx, dy, 1), so the ray parameter t is the z-depth.
//
// Hit test (Woop, Benthin & Wald 2013, watertight), all in fp64 from the fp32 vertices: kz = the axis of the largest
// |d_c| (ties to the lower axis), kx = kz + 1, ky = kx + 1 (mod 3), kx and ky swapped when d_kz < 0; Sx = d_kx / d_kz,
// Sy = d_ky / d_kz, Sz = 1 / d_kz.  Per vertex p: P = p - o, X = P_kx - Sx P_kz, Y = P_ky - Sy P_kz, Z = Sz P_kz.  For
// the triangle (a, b, c) -> (A, B, C): U = Cx By - Cy Bx, V = Ax Cy - Ay Cx, W = Bx Ay - By Ax; a miss when U, V, W
// have mixed signs (some < 0 and some > 0) or det = (U + V) + W is 0; T = ((U Az + V Bz) + W Cz), t = T / det.  A
// shared edge gives both triangles the same products, so a ray through it hits one of them.  det > 0 exactly when the
// ray meets the side (b - a) x (c - a) points to (the front face); cull_backfaces keeps only those.
//
// Which hit wins.  Among triangles hit with near < t <= far: the smallest fp64 t, ties to the smaller input triangle
// index.  depth = t rounded to fp32 once, 0 on a miss; triangle = the input index, -1 on a miss.  normal = x / |x| with
// x = (b - a) x (c - a) (fp64: x0 = e1y e2z - e1z e2y, ..., |x| = sqrt((x0² + x1²) + x2²)), rounded to fp32, 0 on a
// miss.  colour = ((U ca + V cb) + W cc) / det per channel in fp64 from the fp32 vertex colours, rounded to fp32, 0 on
// a miss.
//
// Pruning.  The BVH (lbvh.cuh: Morton keys of the triangle centroids, CUB radix sort, leaf buckets of leaf_size
// triangles, Karras internal nodes, bottom-up min / max boxes of the buckets' vertices) is traversed with a stack, the
// nearer child first.  A child is skipped only when its slab interval [tn, tf], computed in fp32 with directed
// rounding (tn rounded down, tf rounded up, from bounds of o and of 1 / |d| that enclose the fp64 values), lies beyond
// the best hit (tn > best rounded up), before near (tf < near rounded down) or is empty (tn > tf).  The boxes are padded
// outward by 2^-20 of their largest coordinate (plus 2^-100 m), far more than the fp64 test's rounding, so a triangle
// the test hits is never in a skipped box; strict comparisons keep ties visited.  So the result does not depend on
// leaf_size, the tree or num_sms.  (The one case the pad does not cover is a sliver whose edges are shorter than about
// 2^-20 of its distance to the camera, where the fp64 edge functions themselves are rounding noise.)
//
// Layout.  A BVH2 whose internal node (64 B) holds both children's padded boxes as three float4 (x: lo0, hi0, lo1, hi1;
// y; z) and an int4 of the two child ids, read with __ldg: one node visit is four 16-byte loads and both children are
// tested from registers.  Leaf triangles are contiguous in leaf order, three float4 each (the vertices; a.w = the input
// index), 48 B per triangle; their vertex indices (int4: ia, ib, ic, input index) are read once per pixel for colours
// only.  One warp renders an 8 x 4 pixel tile, so its rays stay coherent; warps stride over the tiles of all views.
//
// Memory: the BVH buffer holds the sort keys and indices, the centroids, the leaf-ordered triangles and vertex indices,
// the node boxes and links and CUB's sort storage: about 112 B per triangle + 132 B per leaf + CUB's sort storage
// (nslam_render_bvh_scratch gives the exact size).
#include "nslam_render.h"
#include "lbvh.cuh"
#include "tsdf_rules.cuh"

#include <cmath>
#include <cub/device/device_radix_sort.cuh>

namespace nslam {

constexpr int kRenderStack = 96;   // > the deepest tree: 63 key bits + 31 bits of bucket index among equal keys
constexpr int kTileW = 8, kTileH = 4, kRenderThreads = 128;

// centroids of the triangles (for the Morton order only) and the validity flags: 1 a vertex index outside [0, nv),
// 2 a non-finite vertex coordinate
__global__ void __launch_bounds__(256) mr_centroid_kernel(const float* V, int nv, const int* T, int nt, float* cen,
                                                          unsigned long long* flags) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= nt) return;
  int id[3];
  bool bad = false;
  for (int k = 0; k < 3; k++) {
    id[k] = T[3 * (size_t)t + k];
    if (id[k] < 0 || id[k] >= nv) bad = true, id[k] = 0;
  }
  if (bad) atomicOr(flags, 1ull);
  bool finite = true;
  for (int c = 0; c < 3; c++) {
    float s = 0.f;
    for (int k = 0; k < 3; k++) {
      const float x = V[3 * (size_t)id[k] + c];
      finite = finite && isfinite(x);
      s += x;
    }
    cen[3 * (size_t)t + c] = s * (1.f / 3.f);
  }
  if (!finite) atomicOr(flags, 2ull);
}

// leaf-ordered copy: tri[3i + k] = vertex k of sorted triangle i (.w of k = 0: the input index), vid[i] = its vertex
// indices and input index
__global__ void __launch_bounds__(256) mr_gather_kernel(const float* V, int nv, const int* T, const int* order, int nt,
                                                        float4* tri, int4* vid) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= nt) return;
  const int j = order[i];
  int id[3];
  for (int k = 0; k < 3; k++) {
    id[k] = T[3 * (size_t)j + k];
    if (id[k] < 0 || id[k] >= nv) id[k] = 0;                 // flagged by the centroid pass: the host refuses the mesh
  }
  for (int k = 0; k < 3; k++) {
    const float* p = V + 3 * (size_t)id[k];
    tri[3 * (size_t)i + k] = make_float4(p[0], p[1], p[2], k == 0 ? __int_as_float(j) : 0.f);
  }
  vid[i] = make_int4(id[0], id[1], id[2], j);
}

// the box of leaf bucket l: min / max of its triangles' vertices
struct TriLeaf {
  const float4* tri;
  int n, B;
  __device__ void operator()(int l, float lo[3], float hi[3]) const {
    const int s = l * B, e = min(n, s + B);
    for (int j = 3 * s; j < 3 * e; j++) {
      const float4 p = tri[j];
      lo[0] = fminf(lo[0], p.x); lo[1] = fminf(lo[1], p.y); lo[2] = fminf(lo[2], p.z);
      hi[0] = fmaxf(hi[0], p.x); hi[1] = fmaxf(hi[1], p.y); hi[2] = fmaxf(hi[2], p.z);
    }
  }
};

__device__ __forceinline__ float mr_pad(float lo, float hi) {
  return __fadd_ru(__fmul_ru(fmaxf(fabsf(lo), fabsf(hi)), 0x1p-20f), 0x1p-100f);
}

// node i (internal): float4 x / y / z = (lo0, hi0, lo1, hi1) of its children's padded boxes, then int4 (child0, child1)
__global__ void __launch_bounds__(256) mr_pack_kernel(const float* box, const int2* child, int L, float4* nodes) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= L - 1) return;
  const int2 ch = child[i];
  const float* b0 = box + 6 * (size_t)ch.x;
  const float* b1 = box + 6 * (size_t)ch.y;
  for (int c = 0; c < 3; c++) {
    const float m0 = mr_pad(b0[c], b0[3 + c]), m1 = mr_pad(b1[c], b1[3 + c]);
    nodes[4 * (size_t)i + c] = make_float4(__fsub_rd(b0[c], m0), __fadd_ru(b0[3 + c], m0), __fsub_rd(b1[c], m1),
                                           __fadd_ru(b1[3 + c], m1));
  }
  nodes[4 * (size_t)i + 3] = make_float4(__int_as_float(ch.x), __int_as_float(ch.y), 0.f, 0.f);
}

struct MeshBvh {
  unsigned* bounds;              // [6] ordered fp32 of the centroids
  unsigned long long *keys, *sorted;
  int *index, *order;
  float* cen;                    // [n,3]
  float4* tri;                   // [3n] leaf-ordered vertices
  int4* vid;                     // [n] vertex indices + input index
  float* box;                    // [2L-1][6]
  int2* child;                   // [L-1]
  int *parent, *flags;           // [2L-1], [L]
  float4* nodes;                 // [L-1][4]
  void* cub;
  size_t cub_bytes;
  int L;
};

static size_t mesh_bvh_layout(int n, int B, void* base, MeshBvh* s) {
  MeshBvh t;
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
  t.cen = c.take<float>(12 * (size_t)n);
  t.tri = c.take<float4>(48 * (size_t)n);
  t.vid = c.take<int4>(16 * (size_t)n);
  t.box = c.take<float>(24 * nodes);
  t.child = c.take<int2>(8 * (size_t)t.L);
  t.parent = c.take<int>(4 * nodes);
  t.flags = c.take<int>(4 * (size_t)t.L);
  t.nodes = c.take<float4>(64 * (size_t)t.L);
  t.cub_bytes = sort_bytes;
  t.cub = c.take(sort_bytes);
  if (s) *s = t;
  return c.off;
}

// ------------------------------------------------------------------------------------------------------------ render
struct RenderArgs {
  const float4* nodes;
  const float4* tri;
  const int4* vid;
  int n, B, L;
  const float* colors;           // [V,3] or NULL
  const float* pose;             // [n_views,7]
  int H, W;
  float fx, fy, cx, cy;
  double near_z, far_z;
  int cull;
  long long tiles_x, tiles_per_view, n_tiles;
  float* depth;                  // [n,H,W]
  int* tri_out;                  // [n,H,W]
  float* normal;                 // [n,H,W,3] or NULL
  float* color;                  // [n,H,W,3] or NULL
};

__device__ __forceinline__ double sel3(const double* v, int k) { return k == 0 ? v[0] : (k == 1 ? v[1] : v[2]); }
__device__ __forceinline__ double sel3f(float4 p, int k) { return (double)(k == 0 ? p.x : (k == 1 ? p.y : p.z)); }

// the ray in Woop's sheared frame
struct ShearRay {
  int kx, ky, kz;
  double ox, oy, oz, Sx, Sy, Sz;
};

struct Sheared { double X, Y, Z; };

__device__ __forceinline__ Sheared shear(const ShearRay& r, float4 p) {
  const double px = __dsub_rn(sel3f(p, r.kx), r.ox), py = __dsub_rn(sel3f(p, r.ky), r.oy), pz = __dsub_rn(sel3f(p, r.kz), r.oz);
  return {__dsub_rn(px, __dmul_rn(r.Sx, pz)), __dsub_rn(py, __dmul_rn(r.Sy, pz)), __dmul_rn(r.Sz, pz)};
}

// the watertight test: false on a miss; else t and the edge functions
__device__ __forceinline__ bool hit_triangle(const ShearRay& r, float4 a, float4 b, float4 c, bool cull, double& t,
                                             double& U, double& V, double& W, double& det) {
  const Sheared A = shear(r, a), B = shear(r, b), C = shear(r, c);
  U = __dsub_rn(__dmul_rn(C.X, B.Y), __dmul_rn(C.Y, B.X));
  V = __dsub_rn(__dmul_rn(A.X, C.Y), __dmul_rn(A.Y, C.X));
  W = __dsub_rn(__dmul_rn(B.X, A.Y), __dmul_rn(B.Y, A.X));
  if ((U < 0.0 || V < 0.0 || W < 0.0) && (U > 0.0 || V > 0.0 || W > 0.0)) return false;
  det = __dadd_rn(__dadd_rn(U, V), W);
  if (det == 0.0 || (cull && !(det > 0.0))) return false;
  const double T = __dadd_rn(__dadd_rn(__dmul_rn(U, A.Z), __dmul_rn(V, B.Z)), __dmul_rn(W, C.Z));
  t = __ddiv_rn(T, det);
  return true;
}

// slab interval of one padded box along one axis: s = the sign of d (+-1), so_lo / so_hi enclose s o, a_lo / a_hi
// enclose 1 / |d|; tn rounded down, tf rounded up
__device__ __forceinline__ void slab(float lo, float hi, float s, float so_lo, float so_hi, float a_lo, float a_hi, float& tn,
                                     float& tf) {
  const float xn = s > 0.f ? lo : hi, xf = s > 0.f ? hi : lo;
  const float nn = __fsub_rd(s * xn, so_hi), nf = __fsub_ru(s * xf, so_lo);
  tn = __fmul_rd(nn, nn >= 0.f ? a_lo : a_hi);
  tf = __fmul_ru(nf, nf >= 0.f ? a_hi : a_lo);
}

__global__ void __launch_bounds__(kRenderThreads) mr_render_kernel(RenderArgs a) {
  const int lane = threadIdx.x & 31;
  const long long warps = (long long)gridDim.x * (kRenderThreads / 32);
  int stack[kRenderStack];
  float sdist[kRenderStack];
  for (long long tile = (long long)blockIdx.x * (kRenderThreads / 32) + (threadIdx.x >> 5); tile < a.n_tiles; tile += warps) {
    const long long view = tile / a.tiles_per_view, r = tile - view * a.tiles_per_view;
    const int u = (int)(r % a.tiles_x) * kTileW + (lane % kTileW), v = (int)(r / a.tiles_x) * kTileH + lane / kTileW;
    if (u >= a.W || v >= a.H) continue;
    double R[9];
    const float* p = a.pose + 7 * view;
    tsdf_pose_rotation(p, R);
    const double t0 = p[0], t1 = p[1], t2 = p[2];
    const float dxc = __fdiv_rn(__fsub_rn((float)u, a.cx), a.fx), dyc = __fdiv_rn(__fsub_rn((float)v, a.cy), a.fy);
    double o[3], d[3];
#pragma unroll
    for (int c = 0; c < 3; c++) {
      o[c] = -__dadd_rn(__dadd_rn(__dmul_rn(R[c], t0), __dmul_rn(R[3 + c], t1)), __dmul_rn(R[6 + c], t2));
      d[c] = __dadd_rn(__dadd_rn(__dmul_rn(R[c], (double)dxc), __dmul_rn(R[3 + c], (double)dyc)), R[6 + c]);
    }
    ShearRay ray;
    ray.kz = 0;
    if (fabs(d[1]) > fabs(d[0])) ray.kz = 1;
    if (fabs(d[2]) > fabs(sel3(d, ray.kz))) ray.kz = 2;
    ray.kx = ray.kz == 2 ? 0 : ray.kz + 1;
    ray.ky = ray.kx == 2 ? 0 : ray.kx + 1;
    const double dz = sel3(d, ray.kz);
    if (dz < 0.0) { const int k = ray.kx; ray.kx = ray.ky; ray.ky = k; }
    ray.Sx = __ddiv_rn(sel3(d, ray.kx), dz);
    ray.Sy = __ddiv_rn(sel3(d, ray.ky), dz);
    ray.Sz = __ddiv_rn(1.0, dz);
    ray.ox = sel3(o, ray.kx); ray.oy = sel3(o, ray.ky); ray.oz = sel3(o, ray.kz);
    // enclosing fp32 bounds for the slab test
    float sg[3], so_lo[3], so_hi[3], a_lo[3], a_hi[3];
#pragma unroll
    for (int c = 0; c < 3; c++) {
      sg[c] = d[c] >= 0.0 ? 1.f : -1.f;
      const double so = d[c] >= 0.0 ? o[c] : -o[c], ad = fabs(d[c]);
      so_lo[c] = __double2float_rd(so);
      so_hi[c] = __double2float_ru(so);
      a_lo[c] = __double2float_rd(__ddiv_rd(1.0, ad));
      a_hi[c] = __double2float_ru(__ddiv_ru(1.0, ad));
    }
    const float near_lo = __double2float_rd(a.near_z);
    const bool cull = a.cull != 0;

    double best = a.far_z;
    float best_hi = __double2float_ru(best);
    int best_i = -1, best_j = -1;
    int sp = 0, node = 0;
    while (true) {
      if (node >= a.L - 1) {                                   // leaf: its bucket of triangles
        const int s = (node - (a.L - 1)) * a.B, e = min(a.n, s + a.B);
        for (int j = s; j < e; j++) {
          const float4 va = __ldg(a.tri + 3 * (size_t)j), vb = __ldg(a.tri + 3 * (size_t)j + 1),
                       vc = __ldg(a.tri + 3 * (size_t)j + 2);
          double t, U, V, W, det;
          if (!hit_triangle(ray, va, vb, vc, cull, t, U, V, W, det)) continue;
          const int ti = __float_as_int(va.w);
          if (t > a.near_z && (t < best || (t == best && (best_i < 0 || ti < best_i)))) {
            best = t;
            best_i = ti;
            best_j = j;
            best_hi = __double2float_ru(best);
          }
        }
      } else {
        const float4 bx = __ldg(a.nodes + 4 * (size_t)node), by = __ldg(a.nodes + 4 * (size_t)node + 1),
                     bz = __ldg(a.nodes + 4 * (size_t)node + 2), lk = __ldg(a.nodes + 4 * (size_t)node + 3);
        float n0, f0, n1, f1, tn, tf;
        slab(bx.x, bx.y, sg[0], so_lo[0], so_hi[0], a_lo[0], a_hi[0], n0, f0);
        slab(bx.z, bx.w, sg[0], so_lo[0], so_hi[0], a_lo[0], a_hi[0], n1, f1);
        slab(by.x, by.y, sg[1], so_lo[1], so_hi[1], a_lo[1], a_hi[1], tn, tf);
        n0 = fmaxf(n0, tn); f0 = fminf(f0, tf);
        slab(by.z, by.w, sg[1], so_lo[1], so_hi[1], a_lo[1], a_hi[1], tn, tf);
        n1 = fmaxf(n1, tn); f1 = fminf(f1, tf);
        slab(bz.x, bz.y, sg[2], so_lo[2], so_hi[2], a_lo[2], a_hi[2], tn, tf);
        n0 = fmaxf(n0, tn); f0 = fminf(f0, tf);
        slab(bz.z, bz.w, sg[2], so_lo[2], so_hi[2], a_lo[2], a_hi[2], tn, tf);
        n1 = fmaxf(n1, tn); f1 = fminf(f1, tf);
        const bool v0 = !(n0 > f0 || n0 > best_hi || f0 < near_lo), v1 = !(n1 > f1 || n1 > best_hi || f1 < near_lo);
        const int c0 = __float_as_int(lk.x), c1 = __float_as_int(lk.y);
        if (v0 && v1) {
          const bool first0 = n0 <= n1;
          stack[sp] = first0 ? c1 : c0;
          sdist[sp++] = first0 ? n1 : n0;
          node = first0 ? c0 : c1;
          continue;
        }
        if (v0 || v1) {
          node = v0 ? c0 : c1;
          continue;
        }
      }
      bool found = false;                                      // pop the next box that may still hold a better hit
      while (sp > 0) {
        --sp;
        if (sdist[sp] > best_hi) continue;
        node = stack[sp];
        found = true;
        break;
      }
      if (!found) break;
    }

    const size_t o_px = ((size_t)view * a.H + v) * a.W + u;
    if (best_i < 0) {
      a.depth[o_px] = 0.f;
      a.tri_out[o_px] = -1;
      if (a.normal) for (int c = 0; c < 3; c++) a.normal[3 * o_px + c] = 0.f;
      if (a.color) for (int c = 0; c < 3; c++) a.color[3 * o_px + c] = 0.f;
      continue;
    }
    a.depth[o_px] = __double2float_rn(best);
    a.tri_out[o_px] = best_i;
    const float4 va = __ldg(a.tri + 3 * (size_t)best_j), vb = __ldg(a.tri + 3 * (size_t)best_j + 1),
                 vc = __ldg(a.tri + 3 * (size_t)best_j + 2);
    if (a.normal) {
      const double e1[3] = {__dsub_rn((double)vb.x, (double)va.x), __dsub_rn((double)vb.y, (double)va.y),
                            __dsub_rn((double)vb.z, (double)va.z)};
      const double e2[3] = {__dsub_rn((double)vc.x, (double)va.x), __dsub_rn((double)vc.y, (double)va.y),
                            __dsub_rn((double)vc.z, (double)va.z)};
      const double x[3] = {__dsub_rn(__dmul_rn(e1[1], e2[2]), __dmul_rn(e1[2], e2[1])),
                           __dsub_rn(__dmul_rn(e1[2], e2[0]), __dmul_rn(e1[0], e2[2])),
                           __dsub_rn(__dmul_rn(e1[0], e2[1]), __dmul_rn(e1[1], e2[0]))};
      const double len = __dsqrt_rn(__dadd_rn(__dadd_rn(__dmul_rn(x[0], x[0]), __dmul_rn(x[1], x[1])), __dmul_rn(x[2], x[2])));
      for (int c = 0; c < 3; c++) a.normal[3 * o_px + c] = len > 0.0 ? __double2float_rn(__ddiv_rn(x[c], len)) : 0.f;
    }
    if (a.color) {
      double t, U, V, W, det;
      hit_triangle(ray, va, vb, vc, cull, t, U, V, W, det);   // the winner again, for its edge functions
      const int4 id = __ldg(a.vid + best_j);
      for (int c = 0; c < 3; c++) {
        const double ca = a.colors[3 * (size_t)id.x + c], cb = a.colors[3 * (size_t)id.y + c], cc = a.colors[3 * (size_t)id.z + c];
        a.color[3 * o_px + c] =
            __double2float_rn(__ddiv_rn(__dadd_rn(__dadd_rn(__dmul_rn(U, ca), __dmul_rn(V, cb)), __dmul_rn(W, cc)), det));
      }
    }
  }
}

}  // namespace nslam

extern "C" {

int nslam_render_bvh_scratch(int n_tri, int leaf_size, long long* bytes) {
  using namespace nslam;
  if (n_tri <= 0 || leaf_size < 1 || leaf_size > 32) return (int)cudaErrorInvalidValue;
  *bytes = (long long)mesh_bvh_layout(n_tri, leaf_size, nullptr, nullptr);
  return 0;
}

int nslam_render_bvh_build(const float* vertices, int n_vert, const int* triangles, int n_tri, int leaf_size, void* bvh,
                           long long bvh_bytes, long long* info, void* stream) {
  using namespace nslam;
  if (n_tri <= 0 || n_vert <= 0 || leaf_size < 1 || leaf_size > 32) return (int)cudaErrorInvalidValue;
  MeshBvh s;
  if ((long long)mesh_bvh_layout(n_tri, leaf_size, bvh, &s) > bvh_bytes) return (int)cudaErrorInvalidValue;
  cudaStream_t st = (cudaStream_t)stream;
  cudaError_t e;
  if ((e = cudaMemsetAsync(info, 0, sizeof(long long), st)) != cudaSuccess) return (int)e;
  if ((e = cudaMemsetAsync(s.bounds, 0xff, 3 * sizeof(unsigned), st)) != cudaSuccess) return (int)e;
  if ((e = cudaMemsetAsync(s.bounds + 3, 0, 3 * sizeof(unsigned), st)) != cudaSuccess) return (int)e;
  if ((e = cudaMemsetAsync(s.flags, 0, sizeof(int) * (size_t)s.L, st)) != cudaSuccess) return (int)e;
  const int nb = (n_tri + 255) / 256;
  mr_centroid_kernel<<<nb, 256, 0, st>>>(vertices, n_vert, triangles, n_tri, s.cen, (unsigned long long*)info);
  NSLAM_CHECK_LAUNCH();
  ev_bounds_kernel<<<ev_grid(n_tri, 256, 1024), 256, 0, st>>>(s.cen, n_tri, s.bounds);
  NSLAM_CHECK_LAUNCH();
  ev_keys_kernel<<<nb, 256, 0, st>>>(s.cen, n_tri, s.bounds, s.keys, s.index);
  NSLAM_CHECK_LAUNCH();
  size_t tb = s.cub_bytes;
  if ((e = cub::DeviceRadixSort::SortPairs(s.cub, tb, s.keys, s.sorted, s.index, s.order, n_tri, 0, 3 * kMortonBits, st)) !=
      cudaSuccess)
    return (int)e;
  mr_gather_kernel<<<nb, 256, 0, st>>>(vertices, n_vert, triangles, s.order, n_tri, s.tri, s.vid);
  NSLAM_CHECK_LAUNCH();
  if (s.L > 1) {
    ev_internal_kernel<<<(s.L - 1 + 255) / 256, 256, 0, st>>>(s.sorted, leaf_size, s.L, s.child, s.parent);
    NSLAM_CHECK_LAUNCH();
  } else if ((e = cudaMemsetAsync(s.parent, 0xff, sizeof(int), st)) != cudaSuccess) {
    return (int)e;
  }
  ev_boxes_kernel<<<(s.L + 255) / 256, 256, 0, st>>>(TriLeaf{s.tri, n_tri, leaf_size}, s.L, s.child, s.parent, s.flags,
                                                     s.box);
  NSLAM_CHECK_LAUNCH();
  if (s.L > 1) {
    mr_pack_kernel<<<(s.L - 1 + 255) / 256, 256, 0, st>>>(s.box, s.child, s.L, s.nodes);
    NSLAM_CHECK_LAUNCH();
  }
  return 0;
}

int nslam_render_views(const void* bvh, long long bvh_bytes, int n_tri, int leaf_size, const float* vertex_colors,
                       const float* cam_T_world, int n_views, const float* intr4, int W, int H, float near_z, float far_z,
                       int cull_backfaces, int num_sms, float* depth, int* triangle, float* normal, float* color,
                       void* stream) {
  using namespace nslam;
  if (n_tri <= 0 || leaf_size < 1 || leaf_size > 32 || n_views < 0 || W <= 0 || H <= 0) return (int)cudaErrorInvalidValue;
  if (color && !vertex_colors) return (int)cudaErrorInvalidValue;
  if ((double)n_views * (double)H * (double)W * 3.0 >= 9.2e18) return (int)cudaErrorInvalidValue;   // int64 indices
  MeshBvh b;
  if ((long long)mesh_bvh_layout(n_tri, leaf_size, (void*)bvh, &b) > bvh_bytes) return (int)cudaErrorInvalidValue;
  if (n_views == 0) return 0;
  cudaError_t e;
  if (num_sms <= 0) {
    int dev = 0;
    if ((e = cudaGetDevice(&dev)) != cudaSuccess) return (int)e;
    if ((e = cudaDeviceGetAttribute(&num_sms, cudaDevAttrMultiProcessorCount, dev)) != cudaSuccess) return (int)e;
  }
  RenderArgs a{};
  a.nodes = b.nodes; a.tri = b.tri; a.vid = b.vid;
  a.n = n_tri; a.B = leaf_size; a.L = b.L;
  a.colors = vertex_colors; a.pose = cam_T_world; a.H = H; a.W = W;
  a.fx = intr4[0]; a.fy = intr4[1]; a.cx = intr4[2]; a.cy = intr4[3];
  a.near_z = (double)near_z; a.far_z = (double)far_z; a.cull = cull_backfaces;
  a.tiles_x = (W + kTileW - 1) / kTileW;
  a.tiles_per_view = a.tiles_x * ((H + kTileH - 1) / kTileH);
  a.n_tiles = a.tiles_per_view * n_views;
  a.depth = depth; a.tri_out = triangle; a.normal = normal; a.color = color;
  mr_render_kernel<<<ev_grid(a.n_tiles * 32, kRenderThreads, num_sms * 16), kRenderThreads, 0, (cudaStream_t)stream>>>(a);
  NSLAM_CHECK_LAUNCH();
  return 0;
}

}  // extern "C"
