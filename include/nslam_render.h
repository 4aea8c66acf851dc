/* C ABI of the triangle-mesh renderer (nerf_slam_b200/csrc/mesh_render.cu, rules at its head): a linear BVH over the
 * triangles and exact, watertight ray casting of depth, triangle-id, normal and colour views.  It replaces the
 * reference's MeshRenderer (utils/evaluation.py, Open3D's OpenGL visualiser), which renders the ground-truth mesh at
 * the ground-truth poses.  Every pointer is a DEVICE pointer unless said otherwise; every entry point launches on
 * `stream`, never synchronises the host and returns 0 or a cudaError_t value.  Sizes come back through a HOST long long.
 */
#ifndef NSLAM_RENDER_H_
#define NSLAM_RENDER_H_

#ifdef __cplusplus
extern "C" {
#endif

/* Bytes of the BVH over n_tri triangles with leaf buckets of leaf_size (1..32) triangles. */
int nslam_render_bvh_scratch(int n_tri, int leaf_size, long long* bytes);

/* Build the BVH over vertices [n_vert,3] fp32 and triangles [n_tri,3] int32 into `bvh`.  It keeps a leaf-ordered copy
 * of the triangles' vertices and their vertex indices, so the mesh may be freed afterwards.  info [1] (DEVICE int64) =
 * flags: 1 a vertex index outside [0, n_vert), 2 a non-finite coordinate of a vertex some triangle uses.  A BVH built
 * with a flag set must not be rendered. */
int nslam_render_bvh_build(const float* vertices, int n_vert, const int* triangles, int n_tri, int leaf_size, void* bvh,
                           long long bvh_bytes, long long* info, void* stream);

/* Render n_views views cam_T_world [n_views,7] (t, q_xyzw) with intr4 = fx, fy, cx, cy (HOST fp32 [4]) at W x H:
 * depth [n,H,W] fp32 (0 on a miss) and triangle [n,H,W] int32 (the input index, -1 on a miss); normal [n,H,W,3] fp32
 * (unit geometric normal (b - a) x (c - a), world frame) or NULL; color [n,H,W,3] fp32 (barycentric blend of
 * vertex_colors [V,3] fp32, which must then be given; it is read here, not copied by the build) or NULL.  Only hits with
 * near_z < t <= far_z count (far_z may be +inf); cull_backfaces != 0 keeps only hits on the side the normal points to.
 * bvh from nslam_render_bvh_build with the same n_tri and leaf_size.  num_sms bounds the grid (<= 0: every SM); the
 * results do not depend on it nor on leaf_size. */
int nslam_render_views(const void* bvh, long long bvh_bytes, int n_tri, int leaf_size, const float* vertex_colors,
                       const float* cam_T_world, int n_views, const float* intr4, int W, int H, float near_z, float far_z,
                       int cull_backfaces, int num_sms, float* depth, int* triangle, float* normal, float* color,
                       void* stream);

#ifdef __cplusplus
}
#endif

#endif  // NSLAM_RENDER_H_
