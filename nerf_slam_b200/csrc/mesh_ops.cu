// Triangle-mesh operations: connected components, compaction to a triangle subset, the triangle mask of culling,
// area-weighted vertex normals and vertex clustering.  The rules below DEFINE the behaviour; tests/mesh_ops_oracle.py
// restates them in numpy fp64.  Every result is the same bits in every run, whatever order threads arrive in.
//
// Components.  Two triangles are connected when they share a vertex INDEX (positions are not compared).  Union-find over
// the vertices, lock-free: a union hooks the larger root under the smaller with atomicCAS, so every parent is smaller
// than its child and each tree's root is its minimum vertex index, whatever the arrival order; finds halve paths (a
// write of an ancestor, which only shortens a path).  Then one pass points every vertex at its root (a read-only walk:
// its only stores are roots, so no vertex can be left pointing at a non-root), an atomicMin per
// root keeps the lowest triangle index of its component, and an exclusive scan of the "lowest triangle of its
// component" marks numbers the components 0..C-1 in that order.  Area of a component: the sum of its triangles'
// weights rint(area 2^40) (mesh_rules.cuh, as surface sampling; each weight <= 2^62 / T so the 64-bit integer sums are
// exact), reported /2^40.
//
// Submesh.  Kept triangles stay in input order; the output vertices are the vertices kept triangles reference, in
// input order (two exclusive scans of 0/1 marks); indices are remapped, colours and normals copied.
//
// Cull mask.  keep[t] = seen[a] | seen[b] | seen[c] of the vertex mask of recon_eval.cu's visibility kernel; a
// triangle with a non-finite vertex raises a flag.
//
// Vertex normals (Open3D's compute_vertex_normals).  n_t = (b - a) × (c - a) in fp64 from the fp32 coordinates, not
// normalised.  The 3T corner keys (vertex, then triangle) go through a stable CUB radix sort, so each vertex's corners
// come in ascending triangle order; the vertex sums its corners' n_t in that order (a triangle that repeats an index
// adds n_t once per corner), l = sqrt((s_x² + s_y²) + s_z²) in fp64, and s / l is rounded to fp32 once; l = 0 gives 0.
//
// Vertex clustering.  Vertices that no triangle references are ignored.  The cell of a referenced vertex is
// floor(p / voxel) per axis in fp64, packed as the lattice keys of tsdf_rules.cuh (anchored at the world origin, as
// point-cloud downsampling); a vertex outside the key range has no cell.  A triangle is dropped when a corner has no cell
// or two corners share one.  Among triangles with the same unordered cell triple the lowest index is kept, with its
// winding (two stable radix sorts: by the largest cell, then by the two smaller ones, then a compare with the
// predecessor).  Kept triangles stay in input order.  One output vertex per cell that a kept triangle references, in
// ascending key order: position and colour are the means over all the referenced input vertices of that cell, fp64
// sums in vertex order divided by the count and rounded to fp32 once.
//
// Scratch: components 8 B per vertex + 16 B per triangle; submesh 8 B per vertex + 8 B per triangle; normals 8 B per
// vertex + 48 B per triangle (16 B per corner); clustering 52 B per vertex + 40 B per triangle; each plus CUB's
// temporary storage.
#include "nslam_mesh.h"
#include "common.cuh"
#include "mesh_rules.cuh"
#include "tsdf_rules.cuh"

#include <climits>
#include <cmath>
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>

namespace nslam {

constexpr int kMoThreads = 256;

static inline int mo_blocks(long long n) { return (int)((n + kMoThreads - 1) / kMoThreads); }

// the three indices of triangle t; false when one lies outside [0, nv)
__device__ __forceinline__ bool mo_tri(const int* T, int t, int nv, int& a, int& b, int& c) {
  a = T[3 * (size_t)t]; b = T[3 * (size_t)t + 1]; c = T[3 * (size_t)t + 2];
  return a >= 0 && a < nv && b >= 0 && b < nv && c >= 0 && c < nv;
}

__device__ __forceinline__ bool mo_finite(const float* V, int v) {
  return isfinite(V[3 * (size_t)v]) && isfinite(V[3 * (size_t)v + 1]) && isfinite(V[3 * (size_t)v + 2]);
}

static size_t scan_bytes(int n) {
  size_t b = 0;
  cub::DeviceScan::ExclusiveSum((void*)nullptr, b, (const int*)nullptr, (int*)nullptr, n);
  return b;
}

// ---------------------------------------------------------------------------------------------------------- components
__device__ __forceinline__ int uf_find(volatile int* p, int x) {
  while (true) {
    const int px = p[x];
    if (px == x) return x;
    const int gp = p[px];
    if (gp != px) p[x] = gp;         // path halving: gp is an ancestor of x (parents only ever move to ancestors)
    x = gp;
  }
}

__device__ __forceinline__ void uf_union(volatile int* p, int a, int b) {
  while (true) {
    a = uf_find(p, a);
    b = uf_find(p, b);
    if (a == b) return;
    if (a < b) { const int s = a; a = b; b = s; }
    if (atomicCAS((int*)&p[a], a, b) == a) return;   // hook the larger root under the smaller; retry if a moved
  }
}

__global__ void __launch_bounds__(kMoThreads) mo_cc_init_kernel(int nv, int* parent, int* first) {
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= nv) return;
  parent[v] = v;
  first[v] = INT_MAX;
}

__global__ void __launch_bounds__(kMoThreads) mo_cc_union_kernel(const float* V, int nv, const int* T, int nt,
                                                                 unsigned long long cap, int* parent,
                                                                 unsigned long long* w, unsigned long long* flags) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= nt) return;
  int a, b, c;
  if (!mo_tri(T, t, nv, a, b, c)) {
    w[t] = 0;
    atomicOr(flags, 1ull);
    return;
  }
  unsigned long long wt;
  const unsigned f = tri_area_weight(V, a, b, c, cap, wt);
  w[t] = wt;
  if (f) atomicOr(flags, (unsigned long long)f);
  uf_union(parent, a, b);
  uf_union(parent, a, c);
}

// Read-only walk to the root.  No halving here: a halving store could land after another thread's final store of its
// root and leave a non-root in that slot.  Every store of this pass is a root, so any value a walk reads is an ancestor.
__global__ void __launch_bounds__(kMoThreads) mo_cc_flatten_kernel(int nv, int* parent) {
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= nv) return;
  volatile const int* p = parent;
  int r = p[v], q;
  while ((q = p[r]) != r) r = q;
  parent[v] = r;
}

__global__ void __launch_bounds__(kMoThreads) mo_cc_first_kernel(const int* T, int nv, int nt, const int* parent,
                                                                 int* first) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= nt) return;
  int a, b, c;
  if (mo_tri(T, t, nv, a, b, c)) atomicMin(&first[parent[a]], t);
}

__global__ void __launch_bounds__(kMoThreads) mo_cc_head_kernel(const int* T, int nv, int nt, const int* parent,
                                                                const int* first, int* head) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t > nt) return;
  int a, b, c;
  head[t] = t < nt && mo_tri(T, t, nv, a, b, c) && first[parent[a]] == t;
}

__global__ void __launch_bounds__(kMoThreads) mo_cc_label_kernel(const int* T, int nv, int nt, const int* parent,
                                                                 const int* first, const int* cid,
                                                                 const unsigned long long* w, int* labels,
                                                                 unsigned long long* count, unsigned long long* area,
                                                                 long long* info) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= nt) return;
  if (t == 0) info[0] = cid[nt];
  int a, b, c;
  if (!mo_tri(T, t, nv, a, b, c)) {
    labels[t] = -1;
    return;
  }
  const int l = cid[first[parent[a]]];
  labels[t] = l;
  atomicAdd(&count[l], 1ull);
  atomicAdd(&area[l], w[t]);
}

struct CcScratch {
  int *parent, *first, *head, *cid;
  unsigned long long* w;
  void* cub;
  size_t cub_bytes;
};

static size_t cc_scratch(int nv, int nt, void* base, CcScratch* s) {
  ScratchCarver c(base);
  CcScratch t;
  t.parent = c.take<int>(4 * (size_t)nv);
  t.first = c.take<int>(4 * (size_t)nv);
  t.w = c.take<unsigned long long>(8 * (size_t)nt);
  t.head = c.take<int>(4 * ((size_t)nt + 1));
  t.cid = c.take<int>(4 * ((size_t)nt + 1));
  t.cub_bytes = scan_bytes(nt + 1);
  t.cub = c.take(t.cub_bytes);
  if (s) *s = t;
  return c.off;
}

// ------------------------------------------------------------------------------------------------------------- submesh
__global__ void __launch_bounds__(kMoThreads) mo_sub_mark_kernel(const int* T, int nv, int nt, const unsigned char* keep,
                                                                 int* tflag, int* vflag, int* bad) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t > nt) return;
  if (t == nt) {
    tflag[nt] = 0;
    return;
  }
  int a, b, c;
  const bool ok = mo_tri(T, t, nv, a, b, c);
  if (!ok) *bad = 1;
  const bool k = ok && keep[t];
  tflag[t] = k;
  if (k) vflag[a] = vflag[b] = vflag[c] = 1;
}

__global__ void mo_sub_counts_kernel(const int* vpos, int nv, const int* tpos, int nt, const int* bad, int* counts) {
  counts[0] = *bad ? -1 : vpos[nv];
  counts[1] = tpos[nt];
}

__global__ void __launch_bounds__(kMoThreads) mo_sub_tris_kernel(const int* T, int nt, const int* tflag, const int* tpos,
                                                                 const int* vpos, int* out) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= nt || !tflag[t]) return;
  const size_t o = 3 * (size_t)tpos[t];
#pragma unroll
  for (int k = 0; k < 3; k++) out[o + k] = vpos[T[3 * (size_t)t + k]];
}

__global__ void __launch_bounds__(kMoThreads) mo_sub_verts_kernel(const float* V, const float* C, const float* N, int nv,
                                                                  const int* vflag, const int* vpos, float* oV, float* oC,
                                                                  float* oN) {
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= nv || !vflag[v]) return;
  const size_t i = 3 * (size_t)v, o = 3 * (size_t)vpos[v];
#pragma unroll
  for (int k = 0; k < 3; k++) {
    oV[o + k] = V[i + k];
    if (C) oC[o + k] = C[i + k];
    if (N) oN[o + k] = N[i + k];
  }
}

__global__ void __launch_bounds__(kMoThreads) mo_any_vertex_kernel(const float* V, const int* T, int nv, int nt,
                                                                   const unsigned char* m, unsigned char* keep,
                                                                   int* flags) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= nt) return;
  int a, b, c;
  const bool ok = mo_tri(T, t, nv, a, b, c);
  if (!ok) atomicOr(flags, 1);
  else if (!(mo_finite(V, a) && mo_finite(V, b) && mo_finite(V, c))) atomicOr(flags, 2);
  keep[t] = ok && (m[a] || m[b] || m[c]);
}

struct SubScratch {
  int *vflag, *vpos, *tflag, *tpos, *bad;
  void* cub;
  size_t cub_bytes;
};

static size_t sub_scratch(int nv, int nt, void* base, SubScratch* s) {
  ScratchCarver c(base);
  SubScratch t;
  t.vflag = c.take<int>(4 * ((size_t)nv + 1));
  t.vpos = c.take<int>(4 * ((size_t)nv + 1));
  t.tflag = c.take<int>(4 * ((size_t)nt + 1));
  t.tpos = c.take<int>(4 * ((size_t)nt + 1));
  t.bad = c.take<int>(4);
  t.cub_bytes = scan_bytes((nv > nt ? nv : nt) + 1);
  t.cub = c.take(t.cub_bytes);
  if (s) *s = t;
  return c.off;
}

// ------------------------------------------------------------------------------------------------------ vertex normals
__global__ void __launch_bounds__(kMoThreads) mo_corner_kernel(const float* V, const int* T, int nv, int nt, int* key,
                                                               int* tri, int* count, unsigned long long* flags) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= nt) return;
  int a, b, c;
  const bool ok = mo_tri(T, t, nv, a, b, c);
  if (!ok) atomicOr(flags, 1ull);
  else if (!(mo_finite(V, a) && mo_finite(V, b) && mo_finite(V, c))) atomicOr(flags, 2ull);
  const int v[3] = {a, b, c};
#pragma unroll
  for (int k = 0; k < 3; k++) {
    key[3 * (size_t)t + k] = ok ? v[k] : nv;            // an invalid triangle's corners sort after every vertex
    tri[3 * (size_t)t + k] = t;
    if (ok) atomicAdd(&count[v[k]], 1);
  }
}

__global__ void __launch_bounds__(kMoThreads) mo_normals_kernel(const float* V, const int* T, int nv, const int* off,
                                                                const int* tri, float* N) {
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= nv) return;
  double s[3] = {0.0, 0.0, 0.0};
  for (int i = off[v], e = off[v + 1]; i < e; i++) {
    const int t = tri[i];
    double x[3];
    tri_cross(V, T[3 * (size_t)t], T[3 * (size_t)t + 1], T[3 * (size_t)t + 2], x);
#pragma unroll
    for (int k = 0; k < 3; k++) s[k] = __dadd_rn(s[k], x[k]);
  }
  const double l = __dsqrt_rn(__dadd_rn(__dadd_rn(__dmul_rn(s[0], s[0]), __dmul_rn(s[1], s[1])), __dmul_rn(s[2], s[2])));
#pragma unroll
  for (int k = 0; k < 3; k++) N[3 * (size_t)v + k] = l > 0.0 ? __double2float_rn(__ddiv_rn(s[k], l)) : 0.f;
}

static int bits_for(long long n) {       // the bits of every key in [0, n]
  int b = 1;
  while (b < 63 && (1ll << b) <= n) b++;
  return b;
}

struct NormalScratch {
  int *count, *off, *key[2], *tri[2];
  void* cub;
  size_t cub_bytes;
};

static size_t normal_scratch(int nv, int nt, void* base, NormalScratch* s) {
  const size_t nc = 3 * (size_t)nt;
  size_t sort_bytes = 0;
  cub::DoubleBuffer<int> k, v;
  cub::DeviceRadixSort::SortPairs((void*)nullptr, sort_bytes, k, v, (int)nc, 0, bits_for(nv));
  const size_t sb = scan_bytes(nv + 1);
  ScratchCarver c(base);
  NormalScratch t;
  t.count = c.take<int>(4 * ((size_t)nv + 1));
  t.off = c.take<int>(4 * ((size_t)nv + 1));
  for (int i = 0; i < 2; i++) {
    t.key[i] = c.take<int>(4 * nc);
    t.tri[i] = c.take<int>(4 * nc);
  }
  t.cub_bytes = sort_bytes > sb ? sort_bytes : sb;
  t.cub = c.take(t.cub_bytes);
  if (s) *s = t;
  return c.off;
}

// ---------------------------------------------------------------------------------------------------------- clustering
__global__ void __launch_bounds__(kMoThreads) mo_cl_used_kernel(const int* T, int nv, int nt, int* used,
                                                                int* flags) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= nt) return;
  int a, b, c;
  if (!mo_tri(T, t, nv, a, b, c)) {
    atomicOr(flags, 1);
    return;
  }
  used[a] = used[b] = used[c] = 1;
}

__global__ void __launch_bounds__(kMoThreads) mo_cl_keys_kernel(const float* V, int nv, float voxel, const int* used,
                                                                unsigned long long* key, int* idx, int* flags) {
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= nv) return;
  idx[v] = v;
  unsigned long long k = kEmpty;
  if (used[v]) {
    if (!mo_finite(V, v)) {
      atomicOr(flags, 2);
    } else {
      double q[3];
      bool ok = true;
#pragma unroll
      for (int c = 0; c < 3; c++) {
        q[c] = floor(__ddiv_rn((double)V[3 * (size_t)v + c], (double)voxel));
        ok = ok && block_in_range(q[c]);
      }
      if (ok) k = pack_block((long long)q[0], (long long)q[1], (long long)q[2]);
    }
  }
  key[v] = k;
}

__global__ void __launch_bounds__(kMoThreads) mo_cl_heads_kernel(const unsigned long long* sk, int nv, int* head) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i > nv) return;
  head[i] = i < nv && sk[i] != kEmpty && (i == 0 || sk[i - 1] != sk[i]);
}

// cell of every vertex (-1: none) and the sorted range [start[c], start[c+1]) of each cell's vertices
__global__ void __launch_bounds__(kMoThreads) mo_cl_cells_kernel(const unsigned long long* sk, const int* sv, int nv,
                                                                 const int* head, const int* hpos, int* cell_of,
                                                                 int* start) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= nv) return;
  const unsigned long long k = sk[i];
  if (k == kEmpty) {
    cell_of[sv[i]] = -1;
    return;
  }
  const int c = head[i] ? hpos[i] : hpos[i] - 1;
  cell_of[sv[i]] = c;
  if (head[i]) start[c] = i;
  if (i == nv - 1 || sk[i + 1] != k) start[c + 1] = i + 1;
}

// the cells of triangle t sorted ascending; false when a corner has no cell or two share one
__device__ __forceinline__ bool mo_cl_triple(const int* T, int t, const int* cell_of, int& c0, int& c1, int& c2) {
  int a = cell_of[T[3 * (size_t)t]], b = cell_of[T[3 * (size_t)t + 1]], c = cell_of[T[3 * (size_t)t + 2]];
  if (a < 0 || b < 0 || c < 0 || a == b || b == c || a == c) return false;
  if (a > b) { const int s = a; a = b; b = s; }
  if (b > c) { const int s = b; b = c; c = s; }
  if (a > b) { const int s = a; a = b; b = s; }
  c0 = a; c1 = b; c2 = c;
  return true;
}

__global__ void __launch_bounds__(kMoThreads) mo_cl_key32_kernel(const int* T, int nt, const int* cell_of,
                                                                 const int* bad, unsigned* key, int* tri) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= nt) return;
  int c0, c1, c2;
  key[t] = !(*bad & 1) && mo_cl_triple(T, t, cell_of, c0, c1, c2) ? (unsigned)c2 : UINT_MAX;
  tri[t] = t;
}

__global__ void __launch_bounds__(kMoThreads) mo_cl_key64_kernel(const int* T, int nt, const int* cell_of,
                                                                 const int* bad, const int* tri_in,
                                                                 unsigned long long* key, int* tri_out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= nt) return;
  const int t = tri_in[i];
  int c0, c1, c2;
  key[i] = !(*bad & 1) && mo_cl_triple(T, t, cell_of, c0, c1, c2)
               ? ((unsigned long long)c0 << 32) | (unsigned long long)c1 : ~0ull;
  tri_out[i] = t;
}

// keep the first (lowest-index) triangle of each run of equal cell triples; mark the cells it references
__global__ void __launch_bounds__(kMoThreads) mo_cl_dedup_kernel(const int* T, int nt, const int* cell_of,
                                                                 const int* bad, const int* tri, int* keep,
                                                                 int* cell_used) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i > nt) return;
  if (i == nt) {
    keep[nt] = 0;
    return;
  }
  const int t = tri[i];
  int c0, c1, c2, p0, p1, p2;
  bool k = !(*bad & 1) && mo_cl_triple(T, t, cell_of, c0, c1, c2);
  if (k && i > 0 && mo_cl_triple(T, tri[i - 1], cell_of, p0, p1, p2)) k = !(p0 == c0 && p1 == c1 && p2 == c2);
  keep[t] = k;
  if (k) cell_used[c0] = cell_used[c1] = cell_used[c2] = 1;
}

__global__ void mo_cl_info_kernel(const int* cell_out, int nv, const int* tpos, int nt, const int* flags, int* info) {
  info[0] = cell_out[nv];
  info[1] = tpos[nt];
  info[2] = *flags;
}

__global__ void __launch_bounds__(kMoThreads) mo_cl_tris_kernel(const int* T, int nt, const int* cell_of,
                                                                const int* cell_out, const int* keep, const int* tpos,
                                                                int* out) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= nt || !keep[t]) return;
  const size_t o = 3 * (size_t)tpos[t];
#pragma unroll
  for (int k = 0; k < 3; k++) out[o + k] = cell_out[cell_of[T[3 * (size_t)t + k]]];
}

__global__ void __launch_bounds__(kMoThreads) mo_cl_verts_kernel(const float* V, const float* C, int nv, const int* hpos,
                                                                 const int* start, const int* sv, const int* cell_used,
                                                                 const int* cell_out, float* oV, float* oC) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= hpos[nv] || !cell_used[c]) return;
  double p[3] = {0.0, 0.0, 0.0}, q[3] = {0.0, 0.0, 0.0};
  const int s = start[c], e = start[c + 1];
  for (int i = s; i < e; i++) {
    const size_t v = 3 * (size_t)sv[i];
#pragma unroll
    for (int k = 0; k < 3; k++) {
      p[k] = __dadd_rn(p[k], (double)V[v + k]);
      if (C) q[k] = __dadd_rn(q[k], (double)C[v + k]);
    }
  }
  const double n = (double)(e - s);
  const size_t o = 3 * (size_t)cell_out[c];
#pragma unroll
  for (int k = 0; k < 3; k++) {
    oV[o + k] = __double2float_rn(__ddiv_rn(p[k], n));
    oC[o + k] = __double2float_rn(__ddiv_rn(q[k], n));
  }
}

struct ClusterScratch {
  int *flags, *used, *idx[2], *head, *hpos, *cell_of, *start, *cell_used, *cell_out;
  unsigned long long* vkey[2];
  unsigned* k32[2];
  unsigned long long* k64[2];
  int *tri[2], *keep, *tpos;
  void* cub;
  size_t cub_bytes;
};

static size_t cluster_scratch(int nv, int nt, void* base, ClusterScratch* s) {
  size_t b1 = 0, b2 = 0, b3 = 0;
  {
    cub::DoubleBuffer<unsigned long long> k;
    cub::DoubleBuffer<int> v;
    cub::DeviceRadixSort::SortPairs((void*)nullptr, b1, k, v, nv);
    cub::DeviceRadixSort::SortPairs((void*)nullptr, b3, k, v, nt);
    cub::DoubleBuffer<unsigned> k32;
    cub::DeviceRadixSort::SortPairs((void*)nullptr, b2, k32, v, nt);
  }
  const size_t sb = scan_bytes((nv > nt ? nv : nt) + 1);
  ScratchCarver c(base);
  ClusterScratch t;
  const size_t v1 = (size_t)nv + 1, t1 = (size_t)nt + 1;
  t.flags = c.take<int>(4);
  t.used = c.take<int>(4 * (size_t)nv);
  for (int i = 0; i < 2; i++) {
    t.vkey[i] = c.take<unsigned long long>(8 * (size_t)nv);
    t.idx[i] = c.take<int>(4 * (size_t)nv);
  }
  t.head = c.take<int>(4 * v1);
  t.hpos = c.take<int>(4 * v1);
  t.cell_of = c.take<int>(4 * (size_t)nv);
  t.start = c.take<int>(4 * v1);
  t.cell_used = c.take<int>(4 * v1);
  t.cell_out = c.take<int>(4 * v1);
  for (int i = 0; i < 2; i++) {
    t.k32[i] = c.take<unsigned>(4 * (size_t)nt);
    t.k64[i] = c.take<unsigned long long>(8 * (size_t)nt);
    t.tri[i] = c.take<int>(4 * (size_t)nt);
  }
  t.keep = c.take<int>(4 * t1);
  t.tpos = c.take<int>(4 * t1);
  size_t m = sb;
  for (size_t x : {b1, b2, b3}) m = x > m ? x : m;
  t.cub_bytes = m;
  t.cub = c.take(m);
  if (s) *s = t;
  return c.off;
}

// n_vert < INT_MAX and 3 n_tri <= INT_MAX: every count + 1 and every corner index fits an int
static bool mesh_ok(int nv, int nt) { return nv > 0 && nv < INT_MAX && nt > 0 && 3ll * nt <= INT_MAX; }

}  // namespace nslam

#define MO_TRY(x)                                 \
  do {                                            \
    cudaError_t e__ = (x);                        \
    if (e__ != cudaSuccess) return (int)e__;      \
  } while (0)

extern "C" {

int nslam_mesh_components_scratch(int n_vert, int n_tri, long long* bytes) {
  using namespace nslam;
  if (!mesh_ok(n_vert, n_tri)) return (int)cudaErrorInvalidValue;
  *bytes = (long long)cc_scratch(n_vert, n_tri, nullptr, nullptr);
  return 0;
}

int nslam_mesh_components(const float* vertices, int n_vert, const int* triangles, int n_tri, void* scratch,
                          long long scratch_bytes, int* labels, long long* n_triangles, long long* area_fixed,
                          long long* info, void* stream) {
  using namespace nslam;
  if (!mesh_ok(n_vert, n_tri)) return (int)cudaErrorInvalidValue;
  CcScratch s;
  if ((long long)cc_scratch(n_vert, n_tri, scratch, &s) > scratch_bytes) return (int)cudaErrorInvalidValue;
  cudaStream_t st = (cudaStream_t)stream;
  MO_TRY(cudaMemsetAsync(info, 0, 2 * sizeof(long long), st));
  MO_TRY(cudaMemsetAsync(n_triangles, 0, sizeof(long long) * (size_t)n_tri, st));
  MO_TRY(cudaMemsetAsync(area_fixed, 0, sizeof(long long) * (size_t)n_tri, st));
  const unsigned long long cap = (1ull << 62) / (unsigned long long)n_tri;
  mo_cc_init_kernel<<<mo_blocks(n_vert), kMoThreads, 0, st>>>(n_vert, s.parent, s.first);
  NSLAM_CHECK_LAUNCH();
  mo_cc_union_kernel<<<mo_blocks(n_tri), kMoThreads, 0, st>>>(vertices, n_vert, triangles, n_tri, cap, s.parent, s.w,
                                                              (unsigned long long*)(info + 1));
  NSLAM_CHECK_LAUNCH();
  mo_cc_flatten_kernel<<<mo_blocks(n_vert), kMoThreads, 0, st>>>(n_vert, s.parent);
  NSLAM_CHECK_LAUNCH();
  mo_cc_first_kernel<<<mo_blocks(n_tri), kMoThreads, 0, st>>>(triangles, n_vert, n_tri, s.parent, s.first);
  NSLAM_CHECK_LAUNCH();
  mo_cc_head_kernel<<<mo_blocks(n_tri + 1ll), kMoThreads, 0, st>>>(triangles, n_vert, n_tri, s.parent, s.first, s.head);
  NSLAM_CHECK_LAUNCH();
  size_t tb = s.cub_bytes;
  MO_TRY(cub::DeviceScan::ExclusiveSum(s.cub, tb, s.head, s.cid, n_tri + 1, st));
  mo_cc_label_kernel<<<mo_blocks(n_tri), kMoThreads, 0, st>>>(triangles, n_vert, n_tri, s.parent, s.first, s.cid, s.w,
                                                              labels, (unsigned long long*)n_triangles,
                                                              (unsigned long long*)area_fixed, info);
  NSLAM_CHECK_LAUNCH();
  return 0;
}

int nslam_mesh_submesh_scratch(int n_vert, int n_tri, long long* bytes) {
  using namespace nslam;
  if (!mesh_ok(n_vert, n_tri)) return (int)cudaErrorInvalidValue;
  *bytes = (long long)sub_scratch(n_vert, n_tri, nullptr, nullptr);
  return 0;
}

int nslam_mesh_submesh_count(const int* triangles, int n_vert, int n_tri, const unsigned char* keep, void* scratch,
                             long long scratch_bytes, int* counts, void* stream) {
  using namespace nslam;
  if (!mesh_ok(n_vert, n_tri)) return (int)cudaErrorInvalidValue;
  SubScratch s;
  if ((long long)sub_scratch(n_vert, n_tri, scratch, &s) > scratch_bytes) return (int)cudaErrorInvalidValue;
  cudaStream_t st = (cudaStream_t)stream;
  MO_TRY(cudaMemsetAsync(s.vflag, 0, 4 * ((size_t)n_vert + 1), st));
  MO_TRY(cudaMemsetAsync(s.bad, 0, 4, st));
  mo_sub_mark_kernel<<<mo_blocks(n_tri + 1ll), kMoThreads, 0, st>>>(triangles, n_vert, n_tri, keep, s.tflag, s.vflag,
                                                                    s.bad);
  NSLAM_CHECK_LAUNCH();
  size_t tb = s.cub_bytes;
  MO_TRY(cub::DeviceScan::ExclusiveSum(s.cub, tb, s.vflag, s.vpos, n_vert + 1, st));
  tb = s.cub_bytes;
  MO_TRY(cub::DeviceScan::ExclusiveSum(s.cub, tb, s.tflag, s.tpos, n_tri + 1, st));
  mo_sub_counts_kernel<<<1, 1, 0, st>>>(s.vpos, n_vert, s.tpos, n_tri, s.bad, counts);
  NSLAM_CHECK_LAUNCH();
  return 0;
}

int nslam_mesh_submesh_emit(const float* vertices, const float* colors, const float* normals, int n_vert,
                            const int* triangles, int n_tri, const void* scratch, long long scratch_bytes,
                            float* out_vertices, float* out_colors, float* out_normals, int* out_triangles,
                            void* stream) {
  using namespace nslam;
  if (!mesh_ok(n_vert, n_tri)) return (int)cudaErrorInvalidValue;
  SubScratch s;
  if ((long long)sub_scratch(n_vert, n_tri, (void*)scratch, &s) > scratch_bytes) return (int)cudaErrorInvalidValue;
  cudaStream_t st = (cudaStream_t)stream;
  mo_sub_tris_kernel<<<mo_blocks(n_tri), kMoThreads, 0, st>>>(triangles, n_tri, s.tflag, s.tpos, s.vpos, out_triangles);
  NSLAM_CHECK_LAUNCH();
  mo_sub_verts_kernel<<<mo_blocks(n_vert), kMoThreads, 0, st>>>(vertices, colors, normals, n_vert, s.vflag, s.vpos,
                                                                out_vertices, out_colors, out_normals);
  NSLAM_CHECK_LAUNCH();
  return 0;
}

int nslam_mesh_any_vertex(const float* vertices, const int* triangles, int n_vert, int n_tri,
                          const unsigned char* vertex_mask, unsigned char* keep, int* flags, void* stream) {
  using namespace nslam;
  if (!mesh_ok(n_vert, n_tri)) return (int)cudaErrorInvalidValue;
  cudaStream_t st = (cudaStream_t)stream;
  MO_TRY(cudaMemsetAsync(flags, 0, sizeof(int), st));
  mo_any_vertex_kernel<<<mo_blocks(n_tri), kMoThreads, 0, st>>>(vertices, triangles, n_vert, n_tri, vertex_mask,
                                                                keep, flags);
  NSLAM_CHECK_LAUNCH();
  return 0;
}

int nslam_mesh_vertex_normals_scratch(int n_vert, int n_tri, long long* bytes) {
  using namespace nslam;
  if (!mesh_ok(n_vert, n_tri)) return (int)cudaErrorInvalidValue;
  *bytes = (long long)normal_scratch(n_vert, n_tri, nullptr, nullptr);
  return 0;
}

int nslam_mesh_vertex_normals(const float* vertices, int n_vert, const int* triangles, int n_tri, void* scratch,
                              long long scratch_bytes, float* normals, long long* info, void* stream) {
  using namespace nslam;
  if (!mesh_ok(n_vert, n_tri)) return (int)cudaErrorInvalidValue;
  NormalScratch s;
  if ((long long)normal_scratch(n_vert, n_tri, scratch, &s) > scratch_bytes) return (int)cudaErrorInvalidValue;
  cudaStream_t st = (cudaStream_t)stream;
  MO_TRY(cudaMemsetAsync(info, 0, sizeof(long long), st));
  MO_TRY(cudaMemsetAsync(s.count, 0, 4 * ((size_t)n_vert + 1), st));
  mo_corner_kernel<<<mo_blocks(n_tri), kMoThreads, 0, st>>>(vertices, triangles, n_vert, n_tri, s.key[0], s.tri[0],
                                                            s.count, (unsigned long long*)info);
  NSLAM_CHECK_LAUNCH();
  size_t tb = s.cub_bytes;
  MO_TRY(cub::DeviceScan::ExclusiveSum(s.cub, tb, s.count, s.off, n_vert + 1, st));
  cub::DoubleBuffer<int> k(s.key[0], s.key[1]), v(s.tri[0], s.tri[1]);
  tb = s.cub_bytes;
  MO_TRY(cub::DeviceRadixSort::SortPairs(s.cub, tb, k, v, 3 * n_tri, 0, bits_for(n_vert), st));
  mo_normals_kernel<<<mo_blocks(n_vert), kMoThreads, 0, st>>>(vertices, triangles, n_vert, s.off, v.Current(), normals);
  NSLAM_CHECK_LAUNCH();
  return 0;
}

int nslam_mesh_cluster_scratch(int n_vert, int n_tri, long long* bytes) {
  using namespace nslam;
  if (!mesh_ok(n_vert, n_tri)) return (int)cudaErrorInvalidValue;
  *bytes = (long long)cluster_scratch(n_vert, n_tri, nullptr, nullptr);
  return 0;
}

int nslam_mesh_cluster_count(const float* vertices, int n_vert, const int* triangles, int n_tri, float voxel_size,
                             void* scratch, long long scratch_bytes, int* info, void* stream) {
  using namespace nslam;
  if (!mesh_ok(n_vert, n_tri) || !(voxel_size > 0.f) || !std::isfinite(voxel_size)) return (int)cudaErrorInvalidValue;
  ClusterScratch s;
  if ((long long)cluster_scratch(n_vert, n_tri, scratch, &s) > scratch_bytes) return (int)cudaErrorInvalidValue;
  cudaStream_t st = (cudaStream_t)stream;
  MO_TRY(cudaMemsetAsync(s.flags, 0, 4, st));
  MO_TRY(cudaMemsetAsync(s.used, 0, 4 * (size_t)n_vert, st));
  MO_TRY(cudaMemsetAsync(s.cell_used, 0, 4 * ((size_t)n_vert + 1), st));
  mo_cl_used_kernel<<<mo_blocks(n_tri), kMoThreads, 0, st>>>(triangles, n_vert, n_tri, s.used, s.flags);
  NSLAM_CHECK_LAUNCH();
  mo_cl_keys_kernel<<<mo_blocks(n_vert), kMoThreads, 0, st>>>(vertices, n_vert, voxel_size, s.used, s.vkey[0], s.idx[0],
                                                              s.flags);
  NSLAM_CHECK_LAUNCH();
  cub::DoubleBuffer<unsigned long long> vk(s.vkey[0], s.vkey[1]);
  cub::DoubleBuffer<int> vi(s.idx[0], s.idx[1]);
  size_t tb = s.cub_bytes;
  MO_TRY(cub::DeviceRadixSort::SortPairs(s.cub, tb, vk, vi, n_vert, 0, 64, st));
  if (vi.selector)                       // the emit pass reads the sorted vertex order from idx[0]
    MO_TRY(cudaMemcpyAsync(s.idx[0], s.idx[1], 4 * (size_t)n_vert, cudaMemcpyDeviceToDevice, st));
  mo_cl_heads_kernel<<<mo_blocks(n_vert + 1ll), kMoThreads, 0, st>>>(vk.Current(), n_vert, s.head);
  NSLAM_CHECK_LAUNCH();
  tb = s.cub_bytes;
  MO_TRY(cub::DeviceScan::ExclusiveSum(s.cub, tb, s.head, s.hpos, n_vert + 1, st));
  mo_cl_cells_kernel<<<mo_blocks(n_vert), kMoThreads, 0, st>>>(vk.Current(), s.idx[0], n_vert, s.head, s.hpos, s.cell_of,
                                                               s.start);
  NSLAM_CHECK_LAUNCH();
  mo_cl_key32_kernel<<<mo_blocks(n_tri), kMoThreads, 0, st>>>(triangles, n_tri, s.cell_of, s.flags, s.k32[0], s.tri[0]);
  NSLAM_CHECK_LAUNCH();
  cub::DoubleBuffer<unsigned> k32(s.k32[0], s.k32[1]);
  cub::DoubleBuffer<int> t32(s.tri[0], s.tri[1]);
  tb = s.cub_bytes;
  MO_TRY(cub::DeviceRadixSort::SortPairs(s.cub, tb, k32, t32, n_tri, 0, 32, st));
  mo_cl_key64_kernel<<<mo_blocks(n_tri), kMoThreads, 0, st>>>(triangles, n_tri, s.cell_of, s.flags, t32.Current(),
                                                              s.k64[0], t32.Alternate());
  NSLAM_CHECK_LAUNCH();
  cub::DoubleBuffer<unsigned long long> k64(s.k64[0], s.k64[1]);
  cub::DoubleBuffer<int> t64(t32.Alternate(), t32.Current());
  tb = s.cub_bytes;
  MO_TRY(cub::DeviceRadixSort::SortPairs(s.cub, tb, k64, t64, n_tri, 0, 64, st));
  mo_cl_dedup_kernel<<<mo_blocks(n_tri + 1ll), kMoThreads, 0, st>>>(triangles, n_tri, s.cell_of, s.flags, t64.Current(),
                                                                    s.keep, s.cell_used);
  NSLAM_CHECK_LAUNCH();
  tb = s.cub_bytes;
  MO_TRY(cub::DeviceScan::ExclusiveSum(s.cub, tb, s.keep, s.tpos, n_tri + 1, st));
  tb = s.cub_bytes;
  MO_TRY(cub::DeviceScan::ExclusiveSum(s.cub, tb, s.cell_used, s.cell_out, n_vert + 1, st));
  mo_cl_info_kernel<<<1, 1, 0, st>>>(s.cell_out, n_vert, s.tpos, n_tri, s.flags, info);
  NSLAM_CHECK_LAUNCH();
  return 0;
}

int nslam_mesh_cluster_emit(const float* vertices, const float* colors, int n_vert, const int* triangles, int n_tri,
                            const void* scratch, long long scratch_bytes, float* out_vertices, float* out_colors,
                            int* out_triangles, void* stream) {
  using namespace nslam;
  if (!mesh_ok(n_vert, n_tri)) return (int)cudaErrorInvalidValue;
  ClusterScratch s;
  if ((long long)cluster_scratch(n_vert, n_tri, (void*)scratch, &s) > scratch_bytes) return (int)cudaErrorInvalidValue;
  cudaStream_t st = (cudaStream_t)stream;
  mo_cl_tris_kernel<<<mo_blocks(n_tri), kMoThreads, 0, st>>>(triangles, n_tri, s.cell_of, s.cell_out, s.keep, s.tpos,
                                                             out_triangles);
  NSLAM_CHECK_LAUNCH();
  mo_cl_verts_kernel<<<mo_blocks(n_vert), kMoThreads, 0, st>>>(vertices, colors, n_vert, s.hpos, s.start, s.idx[0],
                                                               s.cell_used, s.cell_out, out_vertices, out_colors);
  NSLAM_CHECK_LAUNCH();
  return 0;
}

}  // extern "C"
