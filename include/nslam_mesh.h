/* C ABI of the triangle-mesh operations (nerf_slam_b200/csrc/mesh_ops.cu, rules at its head): connected components,
 * compaction to a triangle subset, the any-vertex triangle mask of culling, area-weighted vertex normals and vertex
 * clustering.  Every pointer is a DEVICE pointer unless said otherwise; every entry point launches on `stream`, never
 * synchronises the host and returns 0 or a cudaError_t value.  Scratch sizes come back through a HOST long long.
 * Meshes are vertices [n_vert,3] fp32 and triangles [n_tri,3] int32 with 1 <= n_vert < INT32_MAX, n_tri >= 1 and
 * 3 n_tri <= INT32_MAX.
 * Flags: 1 a vertex index outside [0, n_vert), 2 a non-finite coordinate of a vertex some triangle uses, 4 a mesh too
 * large for the 64-bit area sums (2^22 m^2 in all).  A result computed with a flag set is meaningless.
 */
#ifndef NSLAM_MESH_H_
#define NSLAM_MESH_H_

#ifdef __cplusplus
extern "C" {
#endif

/* Device scratch (bytes) of nslam_mesh_components. */
int nslam_mesh_components_scratch(int n_vert, int n_tri, long long* bytes);

/* Connected components of the triangles (two triangles are connected when they share a vertex index): labels [n_tri]
 * int32 in 0..C-1, numbered in the order of each component's lowest triangle index; n_triangles [n_tri] int64 and
 * area_fixed [n_tri] int64 hold in their first C entries each component's triangle count and the sum of its
 * triangles' weights rint(area 2^40) (the rest is zero).  info [2] (DEVICE int64) = C, flags. */
int nslam_mesh_components(const float* vertices, int n_vert, const int* triangles, int n_tri, void* scratch,
                          long long scratch_bytes, int* labels, long long* n_triangles, long long* area_fixed,
                          long long* info, void* stream);

/* Device scratch (bytes) of nslam_mesh_submesh_count / _emit. */
int nslam_mesh_submesh_scratch(int n_vert, int n_tri, long long* bytes);

/* Sizes of the submesh of the triangles with keep[t] != 0 (u8 [n_tri]): counts [2] (DEVICE int32) = the vertices the
 * kept triangles reference (-1 when any triangle has a vertex index outside [0, n_vert)) and the kept triangles. */
int nslam_mesh_submesh_count(const int* triangles, int n_vert, int n_tri, const unsigned char* keep, void* scratch,
                             long long scratch_bytes, int* counts, void* stream);

/* After nslam_mesh_submesh_count with the same mesh, mask and scratch: the kept triangles in input order with their
 * indices remapped, out_triangles [counts[1],3], and their vertices in input order, out_vertices [counts[0],3]; the
 * vertex colours / normals [n_vert,3] fp32 of the kept vertices go to out_colors / out_normals (both may be NULL). */
int nslam_mesh_submesh_emit(const float* vertices, const float* colors, const float* normals, int n_vert,
                            const int* triangles, int n_tri, const void* scratch, long long scratch_bytes,
                            float* out_vertices, float* out_colors, float* out_normals, int* out_triangles,
                            void* stream);

/* keep[t] = 1 when a vertex of triangle t has vertex_mask[v] != 0 (u8 [n_vert]), else 0 (also for a triangle with an
 * index outside [0, n_vert)).  flags [1] (DEVICE int32) = flags 1 and 2 of the triangles (a vertex index outside the
 * mesh, a non-finite vertex of vertices [n_vert,3]). */
int nslam_mesh_any_vertex(const float* vertices, const int* triangles, int n_vert, int n_tri,
                          const unsigned char* vertex_mask, unsigned char* keep, int* flags, void* stream);

/* Device scratch (bytes) of nslam_mesh_vertex_normals. */
int nslam_mesh_vertex_normals_scratch(int n_vert, int n_tri, long long* bytes);

/* Area-weighted vertex normals [n_vert,3] fp32: the normalised sum, in ascending triangle order, of the unnormalised
 * (b - a) x (c - a) of the triangles that use the vertex ((0,0,0) for a zero sum).  info [1] (DEVICE int64) = flags. */
int nslam_mesh_vertex_normals(const float* vertices, int n_vert, const int* triangles, int n_tri, void* scratch,
                              long long scratch_bytes, float* normals, long long* info, void* stream);

/* Device scratch (bytes) of nslam_mesh_cluster_count / _emit. */
int nslam_mesh_cluster_scratch(int n_vert, int n_tri, long long* bytes);

/* Vertex clustering on the lattice of cells voxel_size (> 0, finite) anchored at the origin: info [3] (DEVICE int32) =
 * the output vertices (cells a kept triangle references), the kept triangles, flags. */
int nslam_mesh_cluster_count(const float* vertices, int n_vert, const int* triangles, int n_tri, float voxel_size,
                             void* scratch, long long scratch_bytes, int* info, void* stream);

/* After nslam_mesh_cluster_count with the same mesh and scratch: out_vertices / out_colors [info[0],3] fp32 (the means
 * of each cell's referenced vertices and of their colors [n_vert,3]; 0 when colors is NULL) in ascending cell key
 * order, out_triangles [info[1],3] in input order. */
int nslam_mesh_cluster_emit(const float* vertices, const float* colors, int n_vert, const int* triangles, int n_tri,
                            const void* scratch, long long scratch_bytes, float* out_vertices, float* out_colors,
                            int* out_triangles, void* stream);

#ifdef __cplusplus
}
#endif

#endif  // NSLAM_MESH_H_
