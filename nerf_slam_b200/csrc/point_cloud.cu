// Coloured point clouds of the SLAM keyframe map: what the reference's GUI draws (gui/open3d_gui.py, build_pcls
// :646-678 and get_depth_masks :289-299, through Open3D's create_from_rgbd_image) plus Open3D's voxel_down_sample.
// Open3D's sources are not part of the reference, so the rules below DEFINE the behaviour; tests/point_cloud_oracle.py
// restates them operation for operation.
//
// Input: n keyframes of a SLAM packet, all DEVICE: cam_T_world [n,7] (t, q_xyzw), inverse depths [n,H,W] fp32, depth
// variances [n,H,W] fp32 or NULL (the "uniform" mask), images [n,3,H,W] u8, intrinsics fx, fy, cx, cy at full resolution.
//
// Pixel (u, v) of keyframe k (u the integer column, v the row):
//   d = 1 / idepth in fp32; with variances d := max_depth + 1 where !(sqrt(cov) < max_sigma) (tsdf_pixel_depth, the
//   integration's own mask).  Kept when 0 < d < max_depth, the integration's validity test (NaN, 0, negative and
//   infinite inverse depths drop out), and, with the multi-view filter, when views[k,v,u] >= min_views.
//   views = droid_backends.depth_filter (csrc/geom.cu, unchanged) on the packet's full-resolution inverse depths:
//   neighbours i-1, i-2, i-3, i+3, i+4, i+5 by packet position, one threshold for every frame, agreement in depth units.
//   It sees the raw maps, as DROID's filter does: the sigma mask is not applied to the neighbours.
//   p_c = ((u - cx) d / fx, (v - cy) d / fy, d) in fp64 from the fp32 inputs (Open3D's operation order);
//   p_w = R^T p_c + c_w with R the rotation of the pose rounded to fp32 and c_w = -R^T t rounded to fp32 (as the ray
//   cast takes them), sums left to right, rounded to fp32 once.  Colour = image[:, v, u] / 255 in fp32, channel order as
//   in the packet.  Order: keyframes in packet order, then pixels row-major.  Every step uses an explicit-rounding
//   intrinsic (nvcc would otherwise contract the fp64 mul-adds into FMAs).
//
// Voxel downsampling (voxel_size > 0, finite): the voxel of a point is floor(p / voxel) per axis in fp64, packed as the
// lattice keys of tsdf_rules.cuh (points whose voxel lies outside [-2^20, 2^20)^3 are dropped, never wrapped).  One
// point per occupied voxel in ascending key order: the mean position and mean colour (fp64 sums in the cloud's order,
// divided by the count, rounded to fp32) and the count.  This is Open3D's voxel_down_sample averaging, except that its
// lattice is anchored at the cloud's minimum bound; here it passes through the world origin, so repeated exports of a
// growing map put their points on the same lattice.
//
// Passes.  Cloud: classify (a thread per pixel, every keyframe in one launch, CTAs never straddle two keyframes,
// per-CTA counts) -> CUB exclusive scan of the counts, whose last entry is the total -> ONE host read of the total ->
// emit (the same predicate, an in-CTA ballot scan, each kept pixel writes its point and colour at its slot).  No
// atomics, so the output order is the defined one.  Downsampling: keys + indices -> CUB radix SortPairs (stable: input
// order kept inside a voxel) -> segment heads -> CUB exclusive scan -> segment starts and the voxel count -> ONE host
// read of the count -> a thread per voxel sums its segment in order.
//
// Scratch (bytes, nslam_point_cloud_scratch / _voxel_scratch): the cloud 8 per 256 candidate pixels + CUB's scan
// storage; the downsampling 36 per kept point + CUB's radix-sort storage (about 12 per point: <= 52 in all) on top of
// the full-resolution cloud (24 per kept point).  The depth_filter counter (4 per candidate pixel)
// and the outputs are the caller's.  Nothing is kept between calls.
#include "tsdf_rules.cuh"

#include <climits>
#include <cmath>
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>

namespace nslam {

constexpr int kPcThreads = 256;

struct CloudArgs {
  const float* pose;         // [n,7]
  const float* idepth;       // [n,H,W]
  const float* cov;          // [n,H,W] or NULL
  const float* views;        // [n,H,W] depth_filter counts or NULL
  const unsigned char* rgb;  // [n,3,H,W]
  const float* intr;         // [4]
  int H, W, bpf;             // bpf = CTAs per keyframe
  float max_depth, max_sigma, min_views;
};

// the keep rule of pixel g (index over [n,H,W]) and its depth
__device__ __forceinline__ bool pc_keep(const CloudArgs& a, size_t g, float& d) {
  TsdfFrame f{};
  f.idepth = a.idepth;                 // the whole packet: tsdf_pixel_depth only indexes idepth / depth_cov by g
  f.depth_cov = a.cov;
  f.max_depth = a.max_depth;
  f.max_sigma = a.max_sigma;
  float wr;
  d = tsdf_pixel_depth(f, g, wr);
  return d > 0.f && d < a.max_depth && (!a.views || a.views[g] >= a.min_views);
}

// counts[b] = kept pixels of CTA b; counts[gridDim.x] = 0 (the exclusive scan's last entry becomes the total)
__global__ void __launch_bounds__(kPcThreads) pc_classify_kernel(CloudArgs a, int* counts) {
  const int k = blockIdx.x / a.bpf;
  const int p = (blockIdx.x - k * a.bpf) * kPcThreads + threadIdx.x;
  const int hw = a.H * a.W;
  float d;
  const bool keep = p < hw && pc_keep(a, (size_t)k * hw + p, d);
  const int c = __syncthreads_count(keep);
  if (threadIdx.x == 0) {
    counts[blockIdx.x] = c;
    if (blockIdx.x == gridDim.x - 1) counts[gridDim.x] = 0;
  }
}

__global__ void __launch_bounds__(kPcThreads) pc_emit_kernel(CloudArgs a, const int* offsets, float* points, float* colors) {
  __shared__ double sR[9];
  __shared__ float sc[3], sk[4];
  __shared__ int warp_count[kPcThreads / 32];
  const int k = blockIdx.x / a.bpf;
  if (threadIdx.x == 0) {
    const float* q = a.pose + 7 * (size_t)k;
    tsdf_pose_rotation(q, sR);
    const double t0 = q[0], t1 = q[1], t2 = q[2];
    for (int c = 0; c < 3; c++)
      sc[c] = (float)-__dadd_rn(__dadd_rn(__dmul_rn(sR[c], t0), __dmul_rn(sR[3 + c], t1)), __dmul_rn(sR[6 + c], t2));
    for (int c = 0; c < 4; c++) sk[c] = a.intr[c];
  }
  const int p = (blockIdx.x - k * a.bpf) * kPcThreads + threadIdx.x;
  const int hw = a.H * a.W;
  const size_t g = (size_t)k * hw + p;
  float d = 0.f;
  const bool keep = p < hw && pc_keep(a, g, d);
  const unsigned lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const unsigned ballot = __ballot_sync(0xffffffffu, keep);
  if (lane == 0) warp_count[warp] = __popc(ballot);
  __syncthreads();
  if (!keep) return;
  int slot = offsets[blockIdx.x] + __popc(ballot & ((1u << lane) - 1u));
  for (unsigned w = 0; w < warp; w++) slot += warp_count[w];
  const int u = p % a.W, v = p / a.W;
  const double z = (double)d;
  const double pc[3] = {__ddiv_rn(__dmul_rn(__dsub_rn((double)u, (double)sk[2]), z), (double)sk[0]),
                        __ddiv_rn(__dmul_rn(__dsub_rn((double)v, (double)sk[3]), z), (double)sk[1]), z};
  float* po = points + 3 * (size_t)slot;
  float* co = colors + 3 * (size_t)slot;
  const unsigned char* rgb = a.rgb + (size_t)k * 3 * hw + p;
#pragma unroll
  for (int c = 0; c < 3; c++) {
    const double w = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(sR[c], pc[0]), __dmul_rn(sR[3 + c], pc[1])),
                                         __dmul_rn(sR[6 + c], pc[2])), (double)sc[c]);
    po[c] = __double2float_rn(w);
    co[c] = __fdiv_rn((float)rgb[(size_t)c * hw], 255.f);
  }
}

// ------------------------------------------------------------------------------------------------------ downsampling
__global__ void __launch_bounds__(256) pc_voxel_keys_kernel(const float* points, int n, float voxel, unsigned long long* keys,
                                                            int* index) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  double q[3];
  bool ok = true;
#pragma unroll
  for (int c = 0; c < 3; c++) {
    q[c] = floor(__ddiv_rn((double)points[3 * (size_t)i + c], (double)voxel));
    ok = ok && block_in_range(q[c]);
  }
  keys[i] = ok ? pack_block((long long)q[0], (long long)q[1], (long long)q[2]) : kEmpty;
  index[i] = i;
}

__global__ void __launch_bounds__(256) pc_voxel_heads_kernel(const unsigned long long* sorted, int n, int* head) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const unsigned long long k = sorted[i];
  head[i] = k != kEmpty && (i == 0 || sorted[i - 1] != k);
}

// starts[r] = first sorted position of voxel r; starts[V] = end of the last voxel; *n_voxels = V (0 when every key was
// dropped: the caller zeroes it first)
__global__ void __launch_bounds__(256) pc_voxel_starts_kernel(const unsigned long long* sorted, const int* head,
                                                              const int* rank, int n, int* starts, int* n_voxels) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  if (head[i]) starts[rank[i]] = i;
  if (sorted[i] != kEmpty && (i == n - 1 || sorted[i + 1] == kEmpty)) {
    const int V = rank[i] + head[i];
    starts[V] = i + 1;
    *n_voxels = V;
  }
}

// one thread per voxel: fp64 sums in the sorted (= cloud) order
__global__ void __launch_bounds__(256) pc_voxel_reduce_kernel(const float* points, const float* colors, const int* order,
                                                              const int* starts, int V, float* out_points,
                                                              float* out_colors, int* out_counts) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= V) return;
  const int s = starts[r], e = starts[r + 1];
  double sp[3] = {0.0, 0.0, 0.0}, sc[3] = {0.0, 0.0, 0.0};
  for (int j = s; j < e; j++) {
    const size_t i = 3 * (size_t)order[j];
#pragma unroll
    for (int c = 0; c < 3; c++) {
      sp[c] = __dadd_rn(sp[c], (double)points[i + c]);
      sc[c] = __dadd_rn(sc[c], (double)colors[i + c]);
    }
  }
  const double m = (double)(e - s);
#pragma unroll
  for (int c = 0; c < 3; c++) {
    out_points[3 * (size_t)r + c] = __double2float_rn(__ddiv_rn(sp[c], m));
    out_colors[3 * (size_t)r + c] = __double2float_rn(__ddiv_rn(sc[c], m));
  }
  out_counts[r] = e - s;
}

static size_t pc_align(size_t x) { return (x + 255) & ~(size_t)255; }

static bool pc_shape_ok(int n, int H, int W) { return n > 0 && H > 0 && W > 0 && (long long)n * H * W <= INT_MAX; }

// cloud scratch: counts, offsets [nblk + 1] int; CUB scan storage
struct CloudScratch {
  int *counts, *offsets;
  void* cub;
  size_t cub_bytes;
  int nblk, bpf;
};

static size_t cloud_scratch(int n, int H, int W, void* base, CloudScratch* s) {
  CloudScratch t;
  t.bpf = (H * W + kPcThreads - 1) / kPcThreads;
  t.nblk = n * t.bpf;
  size_t scan_bytes = 0;
  cub::DeviceScan::ExclusiveSum((void*)nullptr, scan_bytes, (const int*)nullptr, (int*)nullptr, t.nblk + 1);
  size_t off = 0;
  char* b = (char*)base;
  auto take = [&](size_t bytes) { void* p = b ? b + off : nullptr; off += pc_align(bytes); return p; };
  t.counts = (int*)take(4 * ((size_t)t.nblk + 1));
  t.offsets = (int*)take(4 * ((size_t)t.nblk + 1));
  t.cub_bytes = scan_bytes;
  t.cub = take(scan_bytes);
  if (s) *s = t;
  return off;
}

// downsampling scratch: keys, sorted keys [N] u64; index, order, head, rank [N] int; starts [N + 1] int; CUB storage
struct VoxelScratch {
  unsigned long long *keys, *sorted;
  int *index, *order, *head, *rank, *starts;
  void* cub;
  size_t cub_bytes;
};

static size_t voxel_scratch(int N, void* base, VoxelScratch* s) {
  size_t sort_bytes = 0, scan_bytes = 0;
  cub::DeviceRadixSort::SortPairs((void*)nullptr, sort_bytes, (const unsigned long long*)nullptr, (unsigned long long*)nullptr,
                                  (const int*)nullptr, (int*)nullptr, N);
  cub::DeviceScan::ExclusiveSum((void*)nullptr, scan_bytes, (const int*)nullptr, (int*)nullptr, N);
  size_t off = 0;
  char* b = (char*)base;
  auto take = [&](size_t bytes) { void* p = b ? b + off : nullptr; off += pc_align(bytes); return p; };
  VoxelScratch t;
  t.keys = (unsigned long long*)take(8 * (size_t)N);
  t.sorted = (unsigned long long*)take(8 * (size_t)N);
  t.index = (int*)take(4 * (size_t)N);
  t.order = (int*)take(4 * (size_t)N);
  t.head = (int*)take(4 * (size_t)N);
  t.rank = (int*)take(4 * (size_t)N);
  t.starts = (int*)take(4 * ((size_t)N + 1));
  t.cub_bytes = sort_bytes > scan_bytes ? sort_bytes : scan_bytes;
  t.cub = take(t.cub_bytes);
  if (s) *s = t;
  return off;
}

static CloudArgs cloud_args(const float* pose, const float* idepth, const float* cov, const float* views, int min_views,
                            const unsigned char* rgb, const float* intr4, int H, int W, int bpf, float max_depth,
                            float max_sigma) {
  CloudArgs a{};
  a.pose = pose; a.idepth = idepth; a.cov = cov; a.views = views; a.rgb = rgb; a.intr = intr4;
  a.H = H; a.W = W; a.bpf = bpf;
  a.max_depth = max_depth; a.max_sigma = max_sigma; a.min_views = (float)min_views;
  return a;
}

}  // namespace nslam

extern "C" {

/* Device scratch (bytes) of nslam_point_cloud_count / _emit for n keyframes of H x W. */
int nslam_point_cloud_scratch(int n, int H, int W, long long* bytes) {
  using namespace nslam;
  if (!pc_shape_ok(n, H, W)) return (int)cudaErrorInvalidValue;
  *bytes = (long long)cloud_scratch(n, H, W, nullptr, nullptr);
  return 0;
}

/* Classify + scan (rules at the head of csrc/point_cloud.cu): *total (DEVICE int) = the number of kept pixels.  views
 * (DEVICE [n,H,W], depth_filter's counter) or NULL = no multi-view filter; min_views in 1..6 when views is given.
 * n H W <= INT32_MAX.  The scratch keeps the per-CTA offsets for nslam_point_cloud_emit. */
int nslam_point_cloud_count(const float* idepth_up, const float* depth_cov_up, const float* views, int min_views, int n,
                            int H, int W, float max_depth, float max_depth_sigma, void* scratch, long long scratch_bytes,
                            int* total, void* stream) {
  using namespace nslam;
  if (!pc_shape_ok(n, H, W) || (views && (min_views < 1 || min_views > 6))) return (int)cudaErrorInvalidValue;
  CloudScratch s;
  if ((long long)cloud_scratch(n, H, W, scratch, &s) > scratch_bytes) return (int)cudaErrorInvalidValue;
  cudaStream_t st = (cudaStream_t)stream;
  const CloudArgs a = cloud_args(nullptr, idepth_up, depth_cov_up, views, min_views, nullptr, nullptr, H, W, s.bpf, max_depth,
                                 max_depth_sigma);
  pc_classify_kernel<<<s.nblk, kPcThreads, 0, st>>>(a, s.counts);
  NSLAM_CHECK_LAUNCH();
  size_t tb = s.cub_bytes;
  cudaError_t e = cub::DeviceScan::ExclusiveSum(s.cub, tb, s.counts, s.offsets, s.nblk + 1, st);
  if (e != cudaSuccess) return (int)e;
  return (int)cudaMemcpyAsync(total, s.offsets + s.nblk, sizeof(int), cudaMemcpyDeviceToDevice, st);
}

/* Emit after nslam_point_cloud_count with the same inputs and scratch: points [total,3] (world, fp32) and colors
 * [total,3] ([0,1]) in keyframe then row-major pixel order.  cam_T_world_tq [n,7], rgb_chw [n,3,H,W] u8 and intr4 =
 * fx, fy, cx, cy at full resolution, all DEVICE. */
int nslam_point_cloud_emit(const float* cam_T_world_tq, const float* idepth_up, const float* depth_cov_up, const float* views,
                           int min_views, const unsigned char* rgb_chw, const float* intr4, int n, int H, int W,
                           float max_depth, float max_depth_sigma, const void* scratch, long long scratch_bytes,
                           float* points, float* colors, void* stream) {
  using namespace nslam;
  if (!pc_shape_ok(n, H, W) || (views && (min_views < 1 || min_views > 6))) return (int)cudaErrorInvalidValue;
  CloudScratch s;
  if ((long long)cloud_scratch(n, H, W, (void*)scratch, &s) > scratch_bytes) return (int)cudaErrorInvalidValue;
  const CloudArgs a = cloud_args(cam_T_world_tq, idepth_up, depth_cov_up, views, min_views, rgb_chw, intr4, H, W, s.bpf,
                                 max_depth, max_depth_sigma);
  pc_emit_kernel<<<s.nblk, kPcThreads, 0, (cudaStream_t)stream>>>(a, s.offsets, points, colors);
  NSLAM_CHECK_LAUNCH();
  return 0;
}

/* Device scratch (bytes) of nslam_point_cloud_voxel_sort / _reduce for n_points points. */
int nslam_point_cloud_voxel_scratch(int n_points, long long* bytes) {
  using namespace nslam;
  if (n_points <= 0) return (int)cudaErrorInvalidValue;
  *bytes = (long long)voxel_scratch(n_points, nullptr, nullptr);
  return 0;
}

/* Voxel keys of points [n_points,3] (DEVICE) at voxel_size (> 0, finite), stable sort, segments: *n_voxels (DEVICE int)
 * = the number of occupied voxels.  The scratch keeps the order and the segments for nslam_point_cloud_voxel_reduce. */
int nslam_point_cloud_voxel_sort(const float* points, int n_points, float voxel_size, void* scratch, long long scratch_bytes,
                                 int* n_voxels, void* stream) {
  using namespace nslam;
  if (n_points <= 0 || !(voxel_size > 0.f) || !std::isfinite(voxel_size)) return (int)cudaErrorInvalidValue;
  VoxelScratch s;
  if ((long long)voxel_scratch(n_points, scratch, &s) > scratch_bytes) return (int)cudaErrorInvalidValue;
  cudaStream_t st = (cudaStream_t)stream;
  cudaError_t e = cudaMemsetAsync(n_voxels, 0, sizeof(int), st);
  if (e != cudaSuccess) return (int)e;
  const int nb = (n_points + 255) / 256;
  pc_voxel_keys_kernel<<<nb, 256, 0, st>>>(points, n_points, voxel_size, s.keys, s.index);
  NSLAM_CHECK_LAUNCH();
  size_t tb = s.cub_bytes;
  if ((e = cub::DeviceRadixSort::SortPairs(s.cub, tb, s.keys, s.sorted, s.index, s.order, n_points, 0, 64, st)) != cudaSuccess)
    return (int)e;
  pc_voxel_heads_kernel<<<nb, 256, 0, st>>>(s.sorted, n_points, s.head);
  NSLAM_CHECK_LAUNCH();
  tb = s.cub_bytes;
  if ((e = cub::DeviceScan::ExclusiveSum(s.cub, tb, s.head, s.rank, n_points, st)) != cudaSuccess) return (int)e;
  pc_voxel_starts_kernel<<<nb, 256, 0, st>>>(s.sorted, s.head, s.rank, n_points, s.starts, n_voxels);
  NSLAM_CHECK_LAUNCH();
  return 0;
}

/* Per-voxel means after nslam_point_cloud_voxel_sort with the same points and scratch: out_points, out_colors
 * [n_voxels,3] fp32 and out_counts [n_voxels] int32 (DEVICE), voxels in ascending key order. */
int nslam_point_cloud_voxel_reduce(const float* points, const float* colors, int n_points, const void* scratch,
                                   long long scratch_bytes, int n_voxels, float* out_points, float* out_colors,
                                   int* out_counts, void* stream) {
  using namespace nslam;
  if (n_points <= 0 || n_voxels < 0 || n_voxels > n_points) return (int)cudaErrorInvalidValue;
  VoxelScratch s;
  if ((long long)voxel_scratch(n_points, (void*)scratch, &s) > scratch_bytes) return (int)cudaErrorInvalidValue;
  if (n_voxels == 0) return 0;
  pc_voxel_reduce_kernel<<<(n_voxels + 255) / 256, 256, 0, (cudaStream_t)stream>>>(points, colors, s.order, s.starts, n_voxels,
                                                                                   out_points, out_colors, out_counts);
  NSLAM_CHECK_LAUNCH();
  return 0;
}

}  // extern "C"
