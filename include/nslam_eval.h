/* C ABI of the reconstruction evaluation (nerf_slam_b200/csrc/recon_eval.cu, rules at its head): area-uniform surface
 * sampling of a triangle mesh, exact nearest neighbours through a linear BVH, the camera visibility mask of ground-truth
 * points and the metric sums.  The reference has no such code (it writes ground-truth paths but never scores against
 * them).  Every pointer is a DEVICE pointer unless said otherwise; every entry point launches on `stream`, never
 * synchronises the host and returns 0 or a cudaError_t value.  Scratch sizes come back through a HOST long long.
 */
#ifndef NSLAM_EVAL_H_
#define NSLAM_EVAL_H_

#ifdef __cplusplus
extern "C" {
#endif

/* Device scratch (bytes) of nslam_eval_surface_area / nslam_eval_sample_surface for n_tri triangles. */
int nslam_eval_surface_scratch(int n_tri, long long* bytes);

/* Triangle weights (fixed-point fp64 areas) and their inclusive scan into the scratch.  vertices [n_vert,3] fp32,
 * triangles [n_tri,3] int32.  info [2] (DEVICE int64): info[0] = the total weight (2^-40 m^2 units), info[1] = flags:
 * 1 a vertex index outside [0, n_vert), 2 a non-finite area, 4 a triangle too large for the 64-bit scan.  Triangles
 * that raise a flag get weight 0. */
int nslam_eval_surface_area(const float* vertices, int n_vert, const int* triangles, int n_tri, void* scratch,
                            long long scratch_bytes, long long* info, void* stream);

/* n points sampled uniformly by area after nslam_eval_surface_area with the same mesh and scratch (its total must be
 * > 0): points [n,3] fp32, tri [n] int32 (the chosen triangle) or NULL.  Sample i depends on (seed, i) only. */
int nslam_eval_sample_surface(const float* vertices, const int* triangles, int n_tri, int n, unsigned long long seed,
                              const void* scratch, long long scratch_bytes, float* points, int* tri, void* stream);

/* Bytes of the BVH over n_ref reference points with leaf buckets of leaf_size (1..32) points. */
int nslam_eval_bvh_scratch(int n_ref, int leaf_size, long long* bytes);

/* Build the BVH over ref [n_ref,3] fp32 (finite coordinates) into `bvh`; it holds a sorted copy of the points, so `ref`
 * may be freed afterwards. */
int nslam_eval_bvh_build(const float* ref, int n_ref, int leaf_size, void* bvh, long long bvh_bytes, void* stream);

/* Device scratch (bytes) of nslam_eval_nearest for n_query queries. */
int nslam_eval_nearest_scratch(int n_query, long long* bytes);

/* Exact nearest reference point of every query [n_query,3] fp32 within max_dist (> 0, +inf allowed): dist [n_query] fp32
 * and idx [n_query] int64 (the reference's input index); +inf and -1 when no reference lies strictly closer than
 * max_dist.  bvh from nslam_eval_bvh_build with the same n_ref and leaf_size.  num_sms bounds the grid (<= 0: every
 * SM); the results do not depend on it nor on leaf_size. */
int nslam_eval_nearest(const void* bvh, long long bvh_bytes, int n_ref, int leaf_size, const float* query, int n_query,
                       float max_dist, int num_sms, void* scratch, long long scratch_bytes, float* dist, long long* idx,
                       void* stream);

/* Visibility of points [n_points,3] fp32 from n_cams cameras cam_T_world [n_cams,7] (t, q_xyzw) with intr4 = fx, fy,
 * cx, cy, images W x H: mask [n_points] u8 = 1 where some camera sees the point.  depths [n_cams,H,W] fp32 or NULL
 * (no occlusion test); depth_tol, near, far in metres (far may be +inf). */
int nslam_eval_visible(const float* points, int n_points, const float* cam_T_world, int n_cams, const float* intr4, int W,
                       int H, const float* depths, float depth_tol, float near_z, float far_z, unsigned char* mask,
                       void* stream);

/* Metric sums over dist [n] fp32 (nearest's output): out [3] (DEVICE int64) = sum of min(d, max_dist) in 2^-32 m
 * fixed point, the count with d < threshold, the count with d = +inf (no neighbour).  max_dist finite and > 0 with
 * n * max_dist < 2^31 (the fixed-point sum then fits in 63 bits). */
int nslam_eval_reduce(const float* dist, int n, float max_dist, float threshold, long long* out, void* stream);

/* ---- registration (nerf_slam_b200/csrc/registration.cu, rules at its head): ICP against the BVH above. ---- */

/* points [n,3] fp32 -> out [n,3] fp32 under the similarity sim3 (a HOST array of 13 doubles: s, R [3x3 row-major], t):
 * s (R p) + t in fp64, rounded once; direction != 0 writes R p only (normals).  out may not alias points. */
int nslam_reg_transform(const float* points, int n, const double* sim3, int direction, float* out, void* stream);

/* normals [n,3] fp32: the unit (b - a) x (c - a) of triangle tri[i] of the mesh (vertices [n_vert,3] fp32, triangles
 * [n_tri,3] int32), e.g. the triangles nslam_eval_sample_surface returns.  flags [1] (DEVICE int64): 1 an index out of
 * range, 2 a zero or non-finite normal; such samples get 0. */
int nslam_reg_face_normals(const float* vertices, int n_vert, const int* triangles, int n_tri, const int* tri, int n,
                           float* normals, long long* flags, void* stream);

/* The Gauss-Newton sums of one ICP iteration -> sums [38] (DEVICE int64, integers of 2^-27): source [n,3] fp32 (the
 * transformed points), idx [n] int64 (nslam_eval_nearest's, -1: no correspondence) into target [n_target,3] fp32 and,
 * unless point_to_point, target_normals [n_target,3] fp32 (unit).  frame is a HOST array of 4 doubles, the centre c and
 * half-diagonal L of the target's box (L > 0, finite); correspondences must lie within L.  with_scale adds the scale
 * unknown.  Layout: H's upper triangle over (omega, tau, sigma) row by row [28], g [7], the squared-residual sum, the
 * count, flags (1 a target index out of range, 2 a term not below 16).  num_sms bounds the grid (<= 0: every SM); the
 * sums do not depend on it. */
int nslam_reg_accumulate(const float* source, int n, const long long* idx, const float* target, const float* target_normals,
                         int n_target, const double* frame, int point_to_point, int with_scale, int num_sms, long long* sums,
                         void* stream);

#ifdef __cplusplus
}
#endif

#endif  // NSLAM_EVAL_H_
