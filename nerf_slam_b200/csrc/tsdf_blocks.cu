// Sparse voxel-block TSDF volume: unbounded Sigma / TSDF fusion that allocates 16^3 blocks where the depth maps reach
// (the reference's Open3D VoxelBlockGrid, fusion/tsdf_fusion.py:64-86, 231-296, block_resolution 16, block_count 5000).
//
// Lattice.  Block b = (bx,by,bz) (int32) holds the voxels of global index g = 16 b + l, l in [0,16)^3.  A voxel's world
// coordinate is the fp32 product voxel_size * g, promoted to fp64 for the projection (Open3D's "integer index x voxel
// size"; the dense grid's origin + voxel * i gives the same bits when its origin is 0).  A block is a 63-bit key:
// (bx + 2^20) | (by + 2^20) << 21 | (bz + 2^20) << 42, so ascending keys run z-major; blocks outside [-2^20, 2^20)^3
// (for example from non-finite coordinates) are dropped, never wrapped.
//
// Activation, per keyframe (Open3D's compute_unique_block_coordinates(depth, K, T, depth_scale=1, depth_max=max_depth)
// with its default trunc_voxel_multiplier 8, restated; oracle/tsdf_blocks.py follows it operation for operation):
//   d = 1 / idepth (fp32); a pixel the sigma test masks gets max_depth + 1; the pixel is valid when 0 < d < max_depth.
//   trunc_a = 8 voxel_size (fp32).  In fp64, from the fp32-rounded rotation R and the translation t of cam_T_world:
//   o = -R^T t, p = ((u - cx) / fx, (v - cy) / fy, 1), x1 = R^T (p - t), dir = x1 - o (sums left to right, no FMA).
//   In fp32: t_min = max(d - trunc_a, 0), t_max = min(d + trunc_a, max_depth), t_k = t_min + (k (t_max - t_min)) / 3,
//   k = 0..3.  The block of sample k is floor((o + t_k dir) / (16 voxel_size)) in fp64.
//   The keyframe's touched set is the unique set of those blocks over all valid pixels.
// Integration applies the per-voxel rule (tsdf_rules.cuh) to every voxel of every touched block and to no other voxel,
// so voxels in free space outside the band get the saturated +1 only where their block was touched (the reference's
// activate -> find -> update).
//
// Pool.  Blocks that are new in a keyframe are appended in ascending key order, so pool order is the same on every run;
// the pool (tsdf, weight [cap,16,16,16] fp32, colour [cap,16,16,16,3] fp32, 80 KB per block) grows on the host and keeps
// every index.  The block -> pool index lookup is an open-addressing hash table (linear probing, load <= 1/2, rebuilt
// from the pool's key array when it would pass 1/2); slot placement may vary between runs, nothing observable does.
//
// Passes per keyframe: touch (one thread per pixel, <= 4 keys, consecutive equal keys dropped) -> radix sort (CUB) ->
// unique + hash lookup -> ordered exclusive scan of the missing keys -> scatter of the touched pool indices and the
// sorted new keys -> ONE pinned read of (touched, new) on the host, which grows the pool and sizes the launch -> insert
// (pool keys, zeroed blocks, hash) -> integrate (one CTA per touched block).
//
// Read-outs are DEFINED as the dense read-outs (tsdf_mesh.cu) of the volume's dense embedding, where every voxel outside
// an allocated block has tsdf 0, weight 0 and colour 0: the mesh kernels run over the pool in tsdf_mesh.cu (they share
// the triangle table there); the ray cast below visits the same samples as the dense march and only skips the memory
// reads of unallocated blocks.  Both read cross-block neighbours through a [B,27] neighbour table built per call.
#include "tsdf_rules.cuh"

#include <climits>
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>

namespace nslam {

// block keys: pack_block / block_in_range / kEmpty in tsdf_rules.cuh

__device__ __forceinline__ unsigned hash_slot(unsigned long long k, unsigned mask) {
  k ^= k >> 33; k *= 0xff51afd7ed558ccdull; k ^= k >> 33; k *= 0xc4ceb9fe1a85ec53ull; k ^= k >> 33;
  return (unsigned)k & mask;
}

struct BlockHash {
  const unsigned long long* keys;   // [cap], kEmpty = free
  const int* vals;                  // [cap] pool index
  unsigned mask;                    // cap - 1 (cap a power of two, load <= 1/2)
  __device__ __forceinline__ int find(unsigned long long key) const {
    for (unsigned s = hash_slot(key, mask);; s = (s + 1) & mask) {
      const unsigned long long k = keys[s];
      if (k == key) return vals[s];
      if (k == kEmpty) return -1;
    }
  }
};

__device__ __forceinline__ void hash_insert(unsigned long long* keys, int* vals, unsigned mask, unsigned long long key, int val) {
  for (unsigned s = hash_slot(key, mask);; s = (s + 1) & mask) {
    const unsigned long long old = atomicCAS(keys + s, kEmpty, key);
    if (old == kEmpty || old == key) { vals[s] = val; return; }
  }
}

// ---------------------------------------------------------------------------------------------------------- activation
__global__ void __launch_bounds__(256) blocks_touch_kernel(TsdfFrame f, float voxel, unsigned long long* keys) {
  __shared__ double sR[9], so[3];
  __shared__ float st32[3];
  if (threadIdx.x == 0) {
    tsdf_pose_rotation(f.pose, sR);
    for (int c = 0; c < 3; c++) st32[c] = f.pose[c];
    const double t0 = f.pose[0], t1 = f.pose[1], t2 = f.pose[2];
    for (int c = 0; c < 3; c++)
      so[c] = -__dadd_rn(__dadd_rn(__dmul_rn(sR[c], t0), __dmul_rn(sR[3 + c], t1)), __dmul_rn(sR[6 + c], t2));
  }
  __syncthreads();
  const int pix = blockIdx.x * blockDim.x + threadIdx.x;
  if (pix >= f.H * f.W) return;
  unsigned long long* out = keys + 4 * (size_t)pix;
  float wr;
  const float d = tsdf_pixel_depth(f, pix, wr);
  int n = 0;
  if (d > 0.f && d < f.max_depth) {
    const int u = pix % f.W, v = pix / f.W;
    const double p[3] = {__ddiv_rn(__dsub_rn((double)u, (double)f.cx), (double)f.fx),
                         __ddiv_rn(__dsub_rn((double)v, (double)f.cy), (double)f.fy), 1.0};
    const double q[3] = {__dsub_rn(p[0], (double)st32[0]), __dsub_rn(p[1], (double)st32[1]), __dsub_rn(p[2], (double)st32[2])};
    double dir[3];
    for (int c = 0; c < 3; c++) {
      const double x1 = __dadd_rn(__dadd_rn(__dmul_rn(sR[c], q[0]), __dmul_rn(sR[3 + c], q[1])), __dmul_rn(sR[6 + c], q[2]));
      dir[c] = __dsub_rn(x1, so[c]);
    }
    const float ta = __fmul_rn(8.f, voxel);
    const float t_min = fmaxf(__fsub_rn(d, ta), 0.f), t_max = fminf(__fadd_rn(d, ta), f.max_depth);
    const float dt = __fsub_rn(t_max, t_min);
    const double bl = (double)__fmul_rn(16.f, voxel);
    unsigned long long last = kEmpty;
    for (int k = 0; k < 4; k++) {
      const double tk = (double)__fadd_rn(t_min, __fdiv_rn(__fmul_rn((float)k, dt), 3.f));
      double b[3];
      bool ok = true;
      for (int c = 0; c < 3; c++) {
        b[c] = floor(__ddiv_rn(__dadd_rn(so[c], __dmul_rn(tk, dir[c])), bl));
        ok = ok && block_in_range(b[c]);
      }
      if (!ok) continue;
      const unsigned long long key = pack_block((long long)b[0], (long long)b[1], (long long)b[2]);
      if (key == last) continue;
      out[n++] = last = key;
    }
  }
  for (; n < 4; n++) out[n] = kEmpty;
}

// sorted keys -> per position: new-block flag (first of its run, valid, not in the table) and the run's pool index
__global__ void __launch_bounds__(256) blocks_lookup_kernel(const unsigned long long* sorted, int n, BlockHash h, int* is_new,
                                                            int* pool) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const unsigned long long k = sorted[i];
  const bool head = k != kEmpty && (i == 0 || sorted[i - 1] != k);
  const int p = head ? h.find(k) : -1;
  is_new[i] = head && p < 0;
  pool[i] = head ? p : -2;                     // -2: not the first of a run
}

// scatter: touched pool indices in ascending key order (new blocks -> n_blocks + rank), new keys in ascending order,
// counts[0..1] = touched, new.  `head_rank` = exclusive scan of the heads
__global__ void __launch_bounds__(256) blocks_scatter_kernel(const unsigned long long* sorted, int n, const int* is_new,
                                                             const int* new_rank, const int* pool, const int* head_rank,
                                                             int n_blocks, int* touched, unsigned long long* new_keys,
                                                             int* counts) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int p = pool[i];
  if (p != -2) {
    const int r = new_rank[i];
    touched[head_rank[i]] = p >= 0 ? p : n_blocks + r;
    if (p < 0) new_keys[r] = sorted[i];
  }
  if (i == n - 1) {
    counts[0] = head_rank[i] + (p != -2);
    counts[1] = new_rank[i] + is_new[i];
  }
}

__global__ void __launch_bounds__(256) blocks_head_kernel(const int* pool, int n, int* head) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) head[i] = pool[i] != -2;
}

// ---------------------------------------------------------------------------------------------------- insert / rehash
__global__ void __launch_bounds__(256) blocks_insert_kernel(const unsigned long long* new_keys, int n_new, int first,
                                                            unsigned long long* pool_keys, int* pool_coords, float* tsdf,
                                                            float* weight, float* color, unsigned long long* hkeys, int* hvals,
                                                            unsigned mask) {
  const int r = blockIdx.x;
  if (r >= n_new) return;
  const int p = first + r;
  const unsigned long long key = new_keys[r];
  float* t = tsdf + ((size_t)p << 12);
  float* w = weight + ((size_t)p << 12);
  float* c = color + 3 * ((size_t)p << 12);
  for (int l = threadIdx.x; l < 4096; l += blockDim.x) { t[l] = 0.f; w[l] = 0.f; }
  for (int l = threadIdx.x; l < 3 * 4096; l += blockDim.x) c[l] = 0.f;
  if (threadIdx.x == 0) {
    pool_keys[p] = key;
    pool_coords[3 * (size_t)p + 0] = (int)(key & 0x1FFFFF) - kBias;
    pool_coords[3 * (size_t)p + 1] = (int)((key >> 21) & 0x1FFFFF) - kBias;
    pool_coords[3 * (size_t)p + 2] = (int)((key >> 42) & 0x1FFFFF) - kBias;
    hash_insert(hkeys, hvals, mask, key, p);
  }
}

__global__ void __launch_bounds__(256) blocks_rehash_kernel(const unsigned long long* pool_keys, int n_blocks,
                                                            unsigned long long* hkeys, int* hvals, unsigned mask) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p < n_blocks) hash_insert(hkeys, hvals, mask, pool_keys[p], p);
}

// ---------------------------------------------------------------------------------------------------------- integrate
__global__ void __launch_bounds__(256) blocks_integrate_kernel(float* tsdf, float* weight, float* color, const int* pool_coords,
                                                               const int* touched, float voxel, TsdfFrame f) {
  __shared__ double sR[9], st[3];
  if (threadIdx.x == 0) {
    tsdf_pose_rotation(f.pose, sR);
    st[0] = f.pose[0]; st[1] = f.pose[1]; st[2] = f.pose[2];
  }
  __syncthreads();
  const int p = touched[blockIdx.x];
  const int bx = 16 * pool_coords[3 * (size_t)p], by = 16 * pool_coords[3 * (size_t)p + 1], bz = 16 * pool_coords[3 * (size_t)p + 2];
  for (int l = threadIdx.x; l < 4096; l += blockDim.x) {
    const size_t vi = ((size_t)p << 12) + l;
    tsdf_update_voxel(f, sR, st, __fmul_rn(voxel, (float)(bx + (l & 15))), __fmul_rn(voxel, (float)(by + ((l >> 4) & 15))),
                      __fmul_rn(voxel, (float)(bz + (l >> 8))), tsdf + vi, weight + vi, color + 3 * vi);
  }
}

// ------------------------------------------------------------------------------------------------------ neighbour table
__global__ void __launch_bounds__(256) blocks_neighbours_kernel(const int* pool_coords, int n_blocks, BlockHash h, int* nbr) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= 27LL * n_blocks) return;
  const int p = (int)(i / 27), o = (int)(i % 27);
  const long long x = pool_coords[3 * (size_t)p] + o % 3 - 1, y = pool_coords[3 * (size_t)p + 1] + (o / 3) % 3 - 1,
                  z = pool_coords[3 * (size_t)p + 2] + o / 9 - 1;
  const bool ok = x >= -kBias && x < kBias && y >= -kBias && y < kBias && z >= -kBias && z < kBias;
  nbr[i] = ok ? h.find(pack_block(x, y, z)) : -1;
}

// ------------------------------------------------------------------------------------------------------------ ray cast
// Samples and hits address the embedding through the hash (the current block is cached in registers) and the neighbour
// table; a cell with a corner in an unallocated block (weight 0 <= min_weight) is unobserved, and its reads are skipped.
struct BlockRay {
  const float* tsdf;
  const float* weight;
  const float* color;
  const int* nbr;
  BlockHash h;
  float min_weight;
  unsigned long long ck = kEmpty;  // cached block key and pool index
  int cp = -1;

  __device__ __forceinline__ static bool packable(int bx, int by, int bz) {
    return bx >= -kBias && bx < kBias && by >= -kBias && by < kBias && bz >= -kBias && bz < kBias;
  }
  __device__ __forceinline__ int find(int bx, int by, int bz) const {
    return packable(bx, by, bz) ? h.find(pack_block(bx, by, bz)) : -1;
  }
  __device__ __forceinline__ int block(int bx, int by, int bz) {
    if (!packable(bx, by, bz)) return -1;
    const unsigned long long key = pack_block(bx, by, bz);
    if (key != ck) { ck = key; cp = h.find(key); }
    return cp;
  }
  // cell at gq: pool voxel index of its 8 corners (-1 = unallocated) and the fractions; false when its corner (0,0,0)
  // lies outside the packable lattice
  __device__ __forceinline__ bool cell(const float* gq, long long* vox, float* fr, bool all_by_hash) {
    int g[3];
#pragma unroll
    for (int q = 0; q < 3; q++) {
      const float fl = floorf(gq[q]);
      if (!(fl >= -(float)(16 * kBias) && fl < (float)(16 * kBias - 1))) return false;
      g[q] = (int)fl;
      fr[q] = __fsub_rn(gq[q], fl);
    }
    const int b[3] = {g[0] >> 4, g[1] >> 4, g[2] >> 4};
    const int p0 = block(b[0], b[1], b[2]);
    if (p0 < 0 && !all_by_hash) return false;
    for (int n = 0; n < 8; n++) {
      const int x = g[0] + (n & 1), y = g[1] + ((n >> 1) & 1), z = g[2] + (n >> 2);
      const int ox = (x >> 4) - b[0], oy = (y >> 4) - b[1], oz = (z >> 4) - b[2];
      int p;
      if (p0 >= 0) p = nbr[27 * (size_t)p0 + (ox + 1) + 3 * (oy + 1) + 9 * (oz + 1)];
      else p = (ox | oy | oz) == 0 ? -1 : find(b[0] + ox, b[1] + oy, b[2] + oz);
      vox[n] = p < 0 ? -1 : ((long long)p << 12) + ((z & 15) << 8) + ((y & 15) << 4) + (x & 15);
    }
    return true;
  }
  __device__ __forceinline__ bool sample(const float* gq, float& f) {
    long long vox[8];
    float fr[3];
    if (!cell(gq, vox, fr, false)) return false;
    for (int n = 0; n < 8; n++)
      if (vox[n] < 0 || !(weight[vox[n]] > min_weight)) return false;
    float t[8];
#pragma unroll
    for (int n = 0; n < 8; n++) t[n] = tsdf[vox[n]];
    f = trilerp8(t, fr[0], fr[1], fr[2]);
    return true;
  }
  __device__ __forceinline__ void hit(const float* gq, RayCell& c) {
    long long vox[8];
    float fr[3] = {0.f, 0.f, 0.f};
    for (int n = 0; n < 8; n++) vox[n] = -1;
    cell(gq, vox, fr, true);
    c.fx = fr[0]; c.fy = fr[1]; c.fz = fr[2];
    for (int n = 0; n < 8; n++) {
      const long long v = vox[n];
      c.t[n] = v < 0 ? 0.f : tsdf[v];
      c.w[n] = v < 0 ? 0.f : weight[v];
      for (int ch = 0; ch < 3; ch++) c.c[ch][n] = v < 0 ? 0.f : color[3 * v + ch];
    }
  }
};

static bool hash_ok(int cap) { return cap >= 2 && (cap & (cap - 1)) == 0; }

static TsdfFrame make_frame(const float* idepth, const float* cov, const unsigned char* rgb, int H, int W, const float* intr4,
                            const float* pose, float max_depth, float trunc, float max_weight, float max_sigma) {
  TsdfFrame f{};
  f.idepth = idepth; f.depth_cov = cov; f.rgb = rgb; f.H = H; f.W = W;
  f.fx = intr4[0]; f.fy = intr4[1]; f.cx = intr4[2]; f.cy = intr4[3];
  f.pose = pose;
  f.max_depth = max_depth; f.trunc = trunc; f.max_weight = max_weight; f.max_sigma = max_sigma;
  return f;
}

// activation scratch layout for n = 4 H W keys: keys, sorted keys [n] u64; is_new, new_rank, pool, head, head_rank [n] int;
// CUB temporary storage
struct ActScratch {
  unsigned long long *keys, *sorted;
  int *is_new, *new_rank, *pool, *head, *head_rank;
  void* cub;
  size_t cub_bytes;
};

static size_t align256(size_t x) { return (x + 255) & ~(size_t)255; }

static size_t act_scratch(int n, void* base, ActScratch* s) {
  size_t sort_bytes = 0, scan_bytes = 0;
  cub::DeviceRadixSort::SortKeys((void*)nullptr, sort_bytes, (const unsigned long long*)nullptr, (unsigned long long*)nullptr, n);
  cub::DeviceScan::ExclusiveSum((void*)nullptr, scan_bytes, (const int*)nullptr, (int*)nullptr, n);
  const size_t cub_bytes = sort_bytes > scan_bytes ? sort_bytes : scan_bytes;
  size_t off = 0;
  char* b = (char*)base;
  auto take = [&](size_t bytes) { void* p = b ? b + off : nullptr; off += align256(bytes); return p; };
  ActScratch t;
  t.keys = (unsigned long long*)take(8 * (size_t)n);
  t.sorted = (unsigned long long*)take(8 * (size_t)n);
  t.is_new = (int*)take(4 * (size_t)n);
  t.new_rank = (int*)take(4 * (size_t)n);
  t.pool = (int*)take(4 * (size_t)n);
  t.head = (int*)take(4 * (size_t)n);
  t.head_rank = (int*)take(4 * (size_t)n);
  t.cub_bytes = cub_bytes;
  t.cub = take(cub_bytes);
  if (s) *s = t;
  return off;
}

}  // namespace nslam

extern "C" {

/* Device scratch (bytes) of nslam_tsdf_blocks_activate for an H x W frame. */
int nslam_tsdf_blocks_scratch(int H, int W, long long* bytes) {
  using namespace nslam;
  if (H <= 0 || W <= 0 || 4LL * H * W > INT_MAX) return (int)cudaErrorInvalidValue;
  *bytes = (long long)act_scratch(4 * H * W, nullptr, nullptr);
  return 0;
}

/* Activation of one keyframe (rule at the head of csrc/tsdf_blocks.cu).  Frame arguments as nslam_tsdf_integrate.
 * hash_keys / hash_vals [hash_cap] (DEVICE; hash_cap a power of two) map block keys to the n_blocks pool indices.
 * Outputs (DEVICE, 4 H W entries each): touched = pool indices of the touched blocks in ascending key order, blocks not
 * yet in the pool numbered n_blocks, n_blocks + 1, ... in that order; new_keys = their keys, ascending.  counts_host
 * (pinned HOST, 2 ints) = (touched, new): the stream is synchronised for it, the one host read of a keyframe. */
int nslam_tsdf_blocks_activate(const float* idepth_up, const float* depth_cov_up, int H, int W, const float* intr4_host,
                               const float* cam_T_world_tq, float voxel_size, float max_depth, float max_depth_sigma,
                               const long long* hash_keys, const int* hash_vals, int hash_cap, int n_blocks, void* scratch,
                               long long scratch_bytes, int* touched, long long* new_keys, int* counts_dev,
                               int* counts_host, void* stream) {
  using namespace nslam;
  if (H <= 0 || W <= 0 || 4LL * H * W > INT_MAX || !hash_ok(hash_cap) || n_blocks < 0) return (int)cudaErrorInvalidValue;
  const int n = 4 * H * W;
  ActScratch s;
  if ((long long)act_scratch(n, scratch, &s) > scratch_bytes) return (int)cudaErrorInvalidValue;
  cudaStream_t st = (cudaStream_t)stream;
  const TsdfFrame f = make_frame(idepth_up, depth_cov_up, nullptr, H, W, intr4_host, cam_T_world_tq, max_depth, 0.f, 0.f,
                                 max_depth_sigma);
  const BlockHash h{(const unsigned long long*)hash_keys, hash_vals, (unsigned)hash_cap - 1};
  blocks_touch_kernel<<<(H * W + 255) / 256, 256, 0, st>>>(f, voxel_size, s.keys);
  NSLAM_CHECK_LAUNCH();
  size_t tb = s.cub_bytes;
  cudaError_t e = cub::DeviceRadixSort::SortKeys(s.cub, tb, s.keys, s.sorted, n, 0, 64, st);
  if (e != cudaSuccess) return (int)e;
  const int nb = (n + 255) / 256;
  blocks_lookup_kernel<<<nb, 256, 0, st>>>(s.sorted, n, h, s.is_new, s.pool);
  NSLAM_CHECK_LAUNCH();
  blocks_head_kernel<<<nb, 256, 0, st>>>(s.pool, n, s.head);
  NSLAM_CHECK_LAUNCH();
  tb = s.cub_bytes;
  if ((e = cub::DeviceScan::ExclusiveSum(s.cub, tb, s.is_new, s.new_rank, n, st)) != cudaSuccess) return (int)e;
  tb = s.cub_bytes;
  if ((e = cub::DeviceScan::ExclusiveSum(s.cub, tb, s.head, s.head_rank, n, st)) != cudaSuccess) return (int)e;
  blocks_scatter_kernel<<<nb, 256, 0, st>>>(s.sorted, n, s.is_new, s.new_rank, s.pool, s.head_rank, n_blocks, touched,
                                             (unsigned long long*)new_keys, counts_dev);
  NSLAM_CHECK_LAUNCH();
  if ((e = cudaMemcpyAsync(counts_host, counts_dev, 2 * sizeof(int), cudaMemcpyDeviceToHost, st)) != cudaSuccess) return (int)e;
  return (int)cudaStreamSynchronize(st);
}

/* Append n_new blocks (keys ascending, from nslam_tsdf_blocks_activate) at pool index n_blocks: their keys, block
 * coordinates [B,3] int32 and zeroed voxels, and their hash entries.  The caller keeps the table's load <= 1/2. */
int nslam_tsdf_blocks_insert(const long long* new_keys, int n_new, int n_blocks, long long* pool_keys, int* pool_coords,
                             float* tsdf, float* weight, float* color, long long* hash_keys, int* hash_vals, int hash_cap,
                             void* stream) {
  using namespace nslam;
  if (n_new < 0 || n_blocks < 0 || !hash_ok(hash_cap) || 2LL * (n_blocks + n_new) > hash_cap) return (int)cudaErrorInvalidValue;
  if (n_new == 0) return 0;
  blocks_insert_kernel<<<n_new, 256, 0, (cudaStream_t)stream>>>((const unsigned long long*)new_keys, n_new, n_blocks,
                                                                (unsigned long long*)pool_keys, pool_coords, tsdf, weight, color,
                                                                (unsigned long long*)hash_keys, hash_vals, (unsigned)hash_cap - 1);
  NSLAM_CHECK_LAUNCH();
  return 0;
}

/* Rebuild the hash table from the pool's keys: hash_keys must be all -1 (empty) on entry; 2 n_blocks <= hash_cap. */
int nslam_tsdf_blocks_rehash(const long long* pool_keys, int n_blocks, long long* hash_keys, int* hash_vals, int hash_cap,
                             void* stream) {
  using namespace nslam;
  if (n_blocks < 0 || !hash_ok(hash_cap) || 2LL * n_blocks > hash_cap) return (int)cudaErrorInvalidValue;
  if (n_blocks == 0) return 0;
  blocks_rehash_kernel<<<(n_blocks + 255) / 256, 256, 0, (cudaStream_t)stream>>>(
      (const unsigned long long*)pool_keys, n_blocks, (unsigned long long*)hash_keys, hash_vals, (unsigned)hash_cap - 1);
  NSLAM_CHECK_LAUNCH();
  return 0;
}

/* Per-voxel update of one keyframe on every voxel of the n_touched blocks `touched` (DEVICE pool indices): one CTA per
 * block.  Pool tsdf / weight [B,16,16,16], color [B,16,16,16,3], block coordinates [B,3] int32 (DEVICE); frame
 * arguments as nslam_tsdf_integrate. */
int nslam_tsdf_blocks_integrate(float* tsdf, float* weight, float* color, const int* pool_coords, const int* touched,
                                int n_touched, float voxel_size, const float* idepth_up, const float* depth_cov_up,
                                const unsigned char* rgb_chw, int H, int W, const float* intr4_host,
                                const float* cam_T_world_tq, float max_depth, float sdf_trunc, float max_weight,
                                float max_depth_sigma, void* stream) {
  using namespace nslam;
  if (n_touched < 0 || H <= 0 || W <= 0) return (int)cudaErrorInvalidValue;
  if (n_touched == 0) return 0;
  const TsdfFrame f = make_frame(idepth_up, depth_cov_up, rgb_chw, H, W, intr4_host, cam_T_world_tq, max_depth, sdf_trunc,
                                 max_weight, max_depth_sigma);
  blocks_integrate_kernel<<<n_touched, 256, 0, (cudaStream_t)stream>>>(tsdf, weight, color, pool_coords, touched, voxel_size, f);
  NSLAM_CHECK_LAUNCH();
  return 0;
}

/* Neighbour table [B,27] int32 (DEVICE): entry (a+1) + 3(b+1) + 9(c+1) of block p = pool index of block p + (a,b,c),
 * or -1 when it is not allocated. */
int nslam_tsdf_blocks_neighbours(const int* pool_coords, int n_blocks, const long long* hash_keys, const int* hash_vals,
                                 int hash_cap, int* neighbours, void* stream) {
  using namespace nslam;
  if (n_blocks < 0 || !hash_ok(hash_cap) || 27LL * n_blocks > INT_MAX) return (int)cudaErrorInvalidValue;
  if (n_blocks == 0) return 0;
  const BlockHash h{(const unsigned long long*)hash_keys, hash_vals, (unsigned)hash_cap - 1};
  blocks_neighbours_kernel<<<(27 * n_blocks + 255) / 256, 256, 0, (cudaStream_t)stream>>>(pool_coords, n_blocks, h, neighbours);
  NSLAM_CHECK_LAUNCH();
  return 0;
}

/* Ray cast n views of the block volume in one launch, as nslam_tsdf_raycast on the volume's dense embedding at lattice
 * origin 0 (same samples, same bits).  min_weight >= 0. */
int nslam_tsdf_blocks_raycast(const float* tsdf, const float* weight, const float* color, const int* neighbours,
                              const long long* hash_keys, const int* hash_vals, int hash_cap, float voxel_size,
                              const float* cam_T_world_tq, int n, int H, int W, const float* intr4_host, float min_depth,
                              float max_depth, float sdf_trunc, float min_weight, float* depth, float* color_out,
                              float* weight_out, float* normal_out, void* stream) {
  using namespace nslam;
  if (n < 0 || H <= 0 || W <= 0 || n > 65535 || (long long)H * W > INT_MAX || !hash_ok(hash_cap) || !(min_weight >= 0.f))
    return (int)cudaErrorInvalidValue;
  if (n == 0) return 0;
  const float zero[3] = {0.f, 0.f, 0.f};
  const RayParams a = ray_params(zero, voxel_size, cam_T_world_tq, H, W, intr4_host, min_depth, max_depth, sdf_trunc, depth,
                                 color_out, weight_out, normal_out);
  BlockRay vol{tsdf, weight, color, neighbours, BlockHash{(const unsigned long long*)hash_keys, hash_vals, (unsigned)hash_cap - 1},
               min_weight};
  dim3 grid((unsigned)(((long long)H * W + 127) / 128), n);
  tsdf_raycast_kernel<<<grid, 128, 0, (cudaStream_t)stream>>>(a, vol);
  NSLAM_CHECK_LAUNCH();
  return 0;
}

}  // extern "C"
