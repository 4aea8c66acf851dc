/* C ABI of libnslam_sm90a.so — hand-written sm_90a kernels behind the reference's
 * `droid_backends` operator surface (reference src/droid.cpp:347-363) and the Python-side hot
 * loops around it.  Every entry point takes raw DEVICE pointers, sizes and a cudaStream_t
 * (as void*), launches on that stream, never synchronises the host and returns 0 or a
 * cudaError_t value.  dtype codes: 0 = fp16, 1 = fp32.
 *
 * Each function cites the reference interface it replaces (paths relative to /root/reference).
 * The BA entry points live in nslam_ba.h, the conv/update-operator ones in nslam_nn.h, the
 * NeRF ones in nslam_ngp.h.
 */
#ifndef NSLAM_H_
#define NSLAM_H_

#include "nslam_ba.h"

#ifdef __cplusplus
extern "C" {
#endif

/* droid_backends.corr_index_forward (src/droid.cpp:280-288; kernel src/correlation_kernels.cu:19-70)
 * volume [n,h1,w1,h2,w2], coords [n,2,h1,w1] fp32, out [n,2r+1,2r+1,h1,w1] (dtype of volume). */
int nslam_corr_index_forward(const void* volume, int dtype, const float* coords, void* out, int n,
                             int h1, int w1, int h2, int w2, int radius, void* stream);

/* droid_backends.corr_index_backward (src/droid.cpp:290-301; kernel src/correlation_kernels.cu:73-124, host :157-185)
 * coords [n,2,h1,w1] fp32, corr_grad [n,2r+1,2r+1,h1,w1] and volume_grad [n,h1,w1,h2,w2] in `dtype` (0 fp16, 1 fp32).
 * Every element of volume_grad is written (zeros outside the windows); volume_grad must be 16-byte aligned. */
int nslam_corr_index_backward(const float* coords, const void* corr_grad, int dtype, void* volume_grad, int n, int h1,
                              int w1, int h2, int w2, int radius, void* stream);

/* CorrBlock.__call__ (networks/modules/corr.py:40-50) fused over the pyramid:
 * volumes: HOST array of num_levels device pointers, h2s/w2s: HOST int arrays;
 * coords [n,2,h1,w1] in level-0 pixels (level l samples coords/2^l); out [n,L*(2r+1)^2,h1,w1].
 * slots: optional DEVICE int32 [n]: edge n reads volume slots[n] (correlation arena), NULL = n.
 * nhwc_stride > 0: out is channels-last [n,h1,w1,nhwc_stride] (tail channels zero-filled);
 * coords_nhwc != 0: coords are [n,h1,w1,2]. */
int nslam_corr_lookup_pyramid(const void* const* volumes, const int* h2s, const int* w2s,
                              int num_levels, int dtype, const float* coords, void* out, int n,
                              int h1, int w1, int radius, const int* slots, int nhwc_stride,
                              int coords_nhwc, void* stream);

/* CorrBlock.__init__ + CorrBlock.corr (networks/modules/corr.py:23-38,63-72): all-pairs
 * correlation (f1/4).(f2/4) and the 3 avg-pooled levels, fp16, in one tensor-core kernel.
 * fmaps [NF,H,W,C=128] fp16 channels-last; ii/jj [E] int32 DEVICE frame indices;
 * out_l [E,H,W,H>>l,W>>l] fp16. */
int nslam_corr_volume_build(const void* fmaps, int NF, int H, int W, int C, const int* ii,
                            const int* jj, int E, void* out0, void* out1, void* out2, void* out3,
                            void* stream);
/* same contract, plain SIMT kernels (test cross-check only) */
int nslam_corr_volume_build_simt(const void* fmaps, int NF, int H, int W, int C, const int* ii,
                                 const int* jj, int E, void* out0, void* out1, void* out2,
                                 void* out3, void* stream);

/* The same operation with row-pair tiles (the default for the shapes it covers; bit-identical output,
 * tests/test_gpu_parity.py) — level 0 leaves the SM as 320 contiguous bytes per source pixel instead of
 * 32-byte pieces (csrc/corr_volume_rows.cu).  C = 128, H even, W in {64, 80}; cudaErrorNotSupported otherwise. */
int nslam_corr_volume_build_rows(const void* fmaps, int NF, int H, int W, int C, const int* ii, const int* jj,
                                 int E, void* out0, void* out1, void* out2, void* out3, void* stream);
/* the same kernel writing edge e into slot slots[e] of pyramid ARENAS out0..3 = [n_slots,H,W,H>>l,W>>l]: all new edges of
 * a keyframe in one launch (CorrPool.build); cudaErrorNotSupported for shapes the row-pair kernel does not cover. */
int nslam_corr_volume_build_slots(const void* fmaps, int NF, int H, int W, int C, const int* ii, const int* jj,
                                  const int* slots, int E, int n_slots, void* out0, void* out1, void* out2, void* out3,
                                  void* stream);

/* droid_backends.altcorr_forward (src/droid.cpp:303-313; kernel src/altcorr_kernel.cu:27-149)
 * fmap1 [B,H1,W1,C], fmap2 [B,H2,W2,C], coords [B,N,H1,W1,2] fp32, corr [B,N,(2r+1)^2,H1,W1]. */
int nslam_altcorr_forward(const void* fmap1, const void* fmap2, int dtype, const float* coords,
                          void* corr, int B, int N, int H1, int W1, int H2, int W2, int C,
                          int radius, void* stream);

/* droid_backends.altcorr_backward (src/droid.cpp:315-327; kernel src/altcorr_kernel.cu:152-286, host :321-356), fp32:
 * fmap1 [B,H1,W1,C], fmap2 [B,H2,W2,C], coords [B,N,H1,W1,2], corr_grad [B,N,(2r+1)^2,H1,W1] ->
 * fmap1_grad [B,H1,W1,C], fmap2_grad [B,H2,W2,C], both fully written.  Deterministic: no float atomics, the scatter
 * into fmap2_grad goes through bucket lists in `scratch` (DEVICE, at least the bytes that
 * nslam_altcorr_backward_scratch returns for the same shapes).  C % 4 == 0, C <= 512, 1 <= r <= 4.
 * The coordinate gradient is not computed (the reference returns zeros). */
int nslam_altcorr_backward_scratch(int B, int N, int H1, int W1, int H2, int W2, int C, int radius,
                                   unsigned long long* bytes);
int nslam_altcorr_backward(const float* fmap1, const float* fmap2, const float* coords, const float* corr_grad,
                           float* fmap1_grad, float* fmap2_grad, void* scratch, unsigned long long scratch_bytes, int B,
                           int N, int H1, int W1, int H2, int W2, int C, int radius, void* stream);

/* pops.projective_transform, jacobian=False (networks/geom/projective_ops.py:98-145) as used by
 * RaftVisualFrontend.reproject (slam/visual_frontends/visual_frontend.py:909-918).
 * poses [N,7], disps [N,ht,wd], intrinsics [N,4] (intr_stride=4) or [4] (intr_stride=0),
 * ii/jj [E] int64; coords [E,ht,wd,2], valid [E,ht,wd,1] (may be NULL). */
int nslam_reproject(const float* poses, const float* disps, const float* intrinsics,
                    int intr_stride, const long long* ii, const long long* jj, int num_edges,
                    int ht, int wd, float* coords, float* valid, void* stream);

/* droid_backends.frame_distance (src/droid.cpp:230-246; kernel src/droid_kernels.cu:630-769) */
int nslam_frame_distance(const float* poses, const float* disps, const float* intrinsics,
                         const long long* ii, const long long* jj, int num, int ht, int wd,
                         float beta, float* dist, void* stream);

/* droid_backends.projmap (src/droid.cpp:249-264): coords [n,ht,wd,3], valid [n,ht,wd,1] */
int nslam_projmap(const float* poses, const float* disps, const float* intrinsics,
                  const long long* ii, const long long* jj, int num, int ht, int wd,
                  float* coords, float* valid, void* stream);

/* droid_backends.iproj (src/droid.cpp:267-276): points [N,ht,wd,3] */
int nslam_iproj(const float* poses, const float* disps, const float* intrinsics, int num, int ht,
                int wd, float* points, void* stream);

/* droid_backends.depth_filter (src/droid.cpp:330-344): counter [n,ht,wd] */
int nslam_depth_filter(const float* poses, const float* disps, const float* intrinsics,
                       const long long* inds, const float* thresh, int num_inds, int num_frames,
                       int ht, int wd, float* counter, void* stream);

/* cvx_upsample (utils/flow_viz.py:166-183): data [K,ht,wd] fp32, mask [K,576,ht,wd]
 * (or [K,ht,wd,576] when mask_nhwc != 0), out [K,8ht,8wd] */
int nslam_cvx_upsample(const float* data, const void* mask, int mask_dtype, float* out, int K,
                       int ht, int wd, float pw, int mask_nhwc, void* stream);
/* two planes through one softmax (inverse depths and their covariances share the mask,
 * visual_frontend.py:444-446); data2/out2 may be NULL.  index (int64 [K], or NULL = identity): mask plane
 * k is applied to row index[k] of the data and out planes (x[kx] = cvx_upsample(y[kx], mask) gather/scatter). */
int nslam_cvx_upsample2(const float* data, const float* data2, const void* mask, int mask_dtype,
                        float* out, float* out2, const long long* index, int K, int ht, int wd, float pw,
                        int mask_nhwc, void* stream);

/* §8(f3) Sigma / TSDF fusion of the SLAM packet into a DENSE voxel grid — the per-voxel update of
 * TsdfFusion.custom_volume_integrate (reference fusion/tsdf_fusion.py:185-302; Open3D VoxelBlockGrid there).
 * tsdf, weight [nz,ny,nx] fp32, color [nz,ny,nx,3] fp32 (DEVICE, updated in place); origin3 = world position of voxel
 * (0,0,0) (HOST); idepth_up / depth_cov_up [H,W] fp32, rgb u8 [3,H,W] (DEVICE; depth_cov_up NULL = uniform weights,
 * the "tsdf" mode; given = weights 1/sqrt(variance), the "sigma" mode); intr4 = fx, fy, cx, cy at full resolution (HOST);
 * cam_T_world_tq = the packet's pose [t, q_xyzw] (DEVICE, 7 floats: no host copy of the pose). */
int nslam_tsdf_integrate(float* tsdf, float* weight, float* color, int nx, int ny, int nz, const float* origin3_host,
                         float voxel_size, const float* idepth_up, const float* depth_cov_up, const unsigned char* rgb_chw,
                         int H, int W, const float* intr4_host, const float* cam_T_world_tq, float max_depth,
                         float sdf_trunc, float max_weight, float max_depth_sigma, void* stream);

/* Read-outs of that volume (csrc/tsdf_mesh.cu; TsdfFusion.build_mesh / render_volume, reference :556-573, :319-484).
 * Marching cubes in three calls: _plan -> int32 scratch size (cudaErrorInvalidValue when the grid's worst-case vertex or
 * triangle count overflows int32); _count -> scratch[0..2] = vertices, triangles, active voxels (DEVICE); _emit with the
 * same volume and min_weight -> active [A,4] int32 scratch, vertices / vertex_colors ([0,1]) / vertex_normals [V,3] fp32,
 * triangles [T,3] int32 in a fixed order (vertices by owning voxel then axis, triangles by cube then table order).
 * A cube is meshed when its 8 corners have weight > min_weight.  origin3 (HOST) as above.  color may be NULL (a volume
 * without colours, such as the NeRF mesh lattice): vertex colours are then 0. */
int nslam_tsdf_mesh_plan(int nx, int ny, int nz, long long* scratch_ints);
int nslam_tsdf_mesh_count(const float* tsdf, const float* weight, int nx, int ny, int nz, float min_weight, int* scratch,
                          void* stream);
int nslam_tsdf_mesh_emit(const float* tsdf, const float* weight, const float* color, int nx, int ny, int nz,
                         const float* origin3_host, float voxel_size, float min_weight, const int* scratch, int n_active,
                         int* active, float* vertices, float* vertex_colors, float* vertex_normals, int* triangles,
                         void* stream);
/* Ray cast n views in one launch: cam_T_world_tq [n,7] (DEVICE, the packet's poses), intr4 = fx, fy, cx, cy (HOST);
 * z-depth march from min_depth to max_depth, hit = first + -> - transition of the trilinear TSDF between samples whose
 * 8 corners have weight > min_weight.  depth [n,H,W] (0 = miss), color [n,H,W,3] in [0,1], weight [n,H,W], normal
 * [n,H,W,3] or NULL (DEVICE). */
int nslam_tsdf_raycast(const float* tsdf, const float* weight, const float* color, int nx, int ny, int nz,
                       const float* origin3_host, float voxel_size, const float* cam_T_world_tq, int n, int H, int W,
                       const float* intr4_host, float min_depth, float max_depth, float sdf_trunc, float min_weight,
                       float* depth, float* color_out, float* weight_out, float* normal_out, void* stream);

/* §8(f3) sparse voxel-block volume (csrc/tsdf_blocks.cu; semantics at its head): 16^3 blocks allocated where the depth
 * maps reach, a pool [B,16,16,16] (tsdf, weight fp32, colour x3 fp32) in a fixed order, an open-addressing hash table
 * of block keys (int64, -1 = empty; capacity a power of two, load <= 1/2).  Per keyframe: _activate (one pinned read of
 * the touched / new block counts) -> _insert (or _rehash into a larger table) -> _integrate.  Read-outs: _neighbours
 * [B,27] -> _mesh_plan / _mesh_count / _mesh_emit (csrc/tsdf_mesh.cu) and _raycast, equal to the dense read-outs of
 * the volume's dense embedding at lattice origin 0. */
int nslam_tsdf_blocks_scratch(int H, int W, long long* bytes);
int nslam_tsdf_blocks_activate(const float* idepth_up, const float* depth_cov_up, int H, int W, const float* intr4_host,
                               const float* cam_T_world_tq, float voxel_size, float max_depth, float max_depth_sigma,
                               const long long* hash_keys, const int* hash_vals, int hash_cap, int n_blocks, void* scratch,
                               long long scratch_bytes, int* touched, long long* new_keys, int* counts_dev,
                               int* counts_host, void* stream);
int nslam_tsdf_blocks_insert(const long long* new_keys, int n_new, int n_blocks, long long* pool_keys, int* pool_coords,
                             float* tsdf, float* weight, float* color, long long* hash_keys, int* hash_vals, int hash_cap,
                             void* stream);
int nslam_tsdf_blocks_rehash(const long long* pool_keys, int n_blocks, long long* hash_keys, int* hash_vals, int hash_cap,
                             void* stream);
int nslam_tsdf_blocks_integrate(float* tsdf, float* weight, float* color, const int* pool_coords, const int* touched,
                                int n_touched, float voxel_size, const float* idepth_up, const float* depth_cov_up,
                                const unsigned char* rgb_chw, int H, int W, const float* intr4_host,
                                const float* cam_T_world_tq, float max_depth, float sdf_trunc, float max_weight,
                                float max_depth_sigma, void* stream);
int nslam_tsdf_blocks_neighbours(const int* pool_coords, int n_blocks, const long long* hash_keys, const int* hash_vals,
                                 int hash_cap, int* neighbours, void* stream);
int nslam_tsdf_blocks_mesh_plan(int n_blocks, long long* scratch_ints);
int nslam_tsdf_blocks_mesh_count(const float* tsdf, const float* weight, const int* neighbours, const int* block_coords,
                                 int n_blocks, float min_weight, int* scratch, void* stream);
int nslam_tsdf_blocks_mesh_emit(const float* tsdf, const float* weight, const float* color, const int* neighbours,
                                const int* block_coords, int n_blocks, float voxel_size, float min_weight, const int* scratch,
                                int n_active, int* active, float* vertices, float* vertex_colors, float* vertex_normals,
                                int* triangles, void* stream);
int nslam_tsdf_blocks_raycast(const float* tsdf, const float* weight, const float* color, const int* neighbours,
                              const long long* hash_keys, const int* hash_vals, int hash_cap, float voxel_size,
                              const float* cam_T_world_tq, int n, int H, int W, const float* intr4_host, float min_depth,
                              float max_depth, float sdf_trunc, float min_weight, float* depth, float* color_out,
                              float* weight_out, float* normal_out, void* stream);

#ifdef __cplusplus
}
#endif
#endif
