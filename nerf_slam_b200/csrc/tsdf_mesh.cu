// §8(f3) read-outs of the dense TSDF volume that nslam_tsdf_integrate writes (tsdf.cu): marching-cubes triangle mesh and
// ray-cast depth / colour / weight / normal views.  They stand in for Open3D's VoxelBlockGrid.extract_triangle_mesh and
// .ray_cast used by TsdfFusion.build_mesh / render_volume (reference fusion/tsdf_fusion.py:556-573, :319-484).  Open3D is
// absent from the reference tree, so parity with it is unpinned; the rules below define the behaviour and
// tests/tsdf_readout_oracle.py restates them in numpy.  Every fp32 step uses an explicit-rounding intrinsic (no FMA
// contraction, no approximate reciprocal / square root) so that the restatement matches the mesh bit for bit.
//
// Volume: tsdf, weight [nz,ny,nx] fp32, color [nz,ny,nx,3] fp32 on the u8 scale; voxel (i,j,k) at origin + voxel*(i,j,k);
// tsdf > 0 is free space in front of the surface; unobserved voxels have weight 0.
//
// Marching cubes.  Cube (i,j,k) spans voxels i..i+1, j..j+1, k..k+1 and is valid when its 8 corners have weight > min_weight.
// Corner bit n of the case is set when tsdf < 0 there (Lorensen / Bourke corner and edge numbering).  A vertex sits on every
// lattice edge whose endpoints differ in sign and that belongs to at least one valid cube (so none is unreferenced), at
// t = f0 / (f0 - f1); its normal is the lerp of the central-difference TSDF gradients at the endpoints, normalised (toward
// +tsdf); triangles are wound so that (b - a) x (c - a) points toward +tsdf.  Output order is fixed, with no atomics:
// vertices by the linear index of the voxel owning their edge (a voxel owns its +x, +y, +z edges), then axis; triangles by
// linear cube index, then table order.  Passes: classify (per-block counts) -> ordered scan in one CTA -> compaction (the
// sorted list of ACTIVE voxels, those owning a vertex or emitting a triangle, with their vertex / triangle bases; vertices
// written here) -> triangles (each edge resolved to its owner by binary search in the active list).  Scratch is
// 3 ints per 256 voxels plus 4 ints per active voxel: it grows with the surface, not with the grid.
//
// Ray cast.  One thread per pixel, views batched over blockIdx.y.  Pixel (u,v) casts z * ((u-cx)/fx, (v-cy)/fy, 1) (camera
// frame, z-depth) from min_depth to max_depth through the trilinear TSDF.  A sample is observed when its 8 cell corners have
// weight > min_weight.  Steps along the ray: voxel while unobserved or not in front of the surface, max(f * sdf_trunc, voxel)
// in front of it.  The hit is the first + -> (<= 0) transition between consecutive observed samples, linearly interpolated.
#include "tsdf_rules.cuh"

#include <climits>

namespace nslam {

// triangle table: case -> up to 5 triangles of cube edges, -1 terminated.  Face rule: on every cube face the iso-line cuts
// off each inside corner (on an ambiguous face, whose inside corners are diagonal, each gets its own segment), so the two
// cubes sharing a face agree and the surface is closed; loops are fanned from their lowest edge.
__constant__ signed char c_tri[256][16] = {
    {-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1}, {0,3,8,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1}, {0,9,1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1}, {1,3,8,1,8,9,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1},
    {1,10,2,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1}, {0,3,8,1,10,2,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1}, {0,9,10,0,10,2,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1}, {2,3,8,2,8,9,2,9,10,-1,-1,-1,-1,-1,-1,-1},
    {2,11,3,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1}, {0,2,11,0,11,8,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1}, {0,9,1,2,11,3,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1}, {1,2,11,1,11,8,1,8,9,-1,-1,-1,-1,-1,-1,-1},
    {1,10,11,1,11,3,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1}, {0,1,10,0,10,11,0,11,8,-1,-1,-1,-1,-1,-1,-1}, {0,9,10,0,10,11,0,11,3,-1,-1,-1,-1,-1,-1,-1}, {8,9,10,8,10,11,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1},
    {4,8,7,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1}, {0,3,7,0,7,4,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1}, {0,9,1,4,8,7,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1}, {1,3,7,1,7,4,1,4,9,-1,-1,-1,-1,-1,-1,-1},
    {1,10,2,4,8,7,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1}, {0,3,7,0,7,4,1,10,2,-1,-1,-1,-1,-1,-1,-1}, {0,9,10,0,10,2,4,8,7,-1,-1,-1,-1,-1,-1,-1}, {2,3,7,2,7,4,2,4,9,2,9,10,-1,-1,-1,-1},
    {2,11,3,4,8,7,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1}, {0,2,11,0,11,7,0,7,4,-1,-1,-1,-1,-1,-1,-1}, {0,9,1,2,11,3,4,8,7,-1,-1,-1,-1,-1,-1,-1}, {1,2,11,1,11,7,1,7,4,1,4,9,-1,-1,-1,-1},
    {1,10,11,1,11,3,4,8,7,-1,-1,-1,-1,-1,-1,-1}, {0,1,10,0,10,11,0,11,7,0,7,4,-1,-1,-1,-1}, {0,9,10,0,10,11,0,11,3,4,8,7,-1,-1,-1,-1}, {4,9,10,4,10,11,4,11,7,-1,-1,-1,-1,-1,-1,-1},
    {4,5,9,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1}, {0,3,8,4,5,9,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1}, {0,4,5,0,5,1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1}, {1,3,8,1,8,4,1,4,5,-1,-1,-1,-1,-1,-1,-1},
    {1,10,2,4,5,9,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1}, {0,3,8,1,10,2,4,5,9,-1,-1,-1,-1,-1,-1,-1}, {0,4,5,0,5,10,0,10,2,-1,-1,-1,-1,-1,-1,-1}, {2,3,8,2,8,4,2,4,5,2,5,10,-1,-1,-1,-1},
    {2,11,3,4,5,9,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1}, {0,2,11,0,11,8,4,5,9,-1,-1,-1,-1,-1,-1,-1}, {0,4,5,0,5,1,2,11,3,-1,-1,-1,-1,-1,-1,-1}, {1,2,11,1,11,8,1,8,4,1,4,5,-1,-1,-1,-1},
    {1,10,11,1,11,3,4,5,9,-1,-1,-1,-1,-1,-1,-1}, {0,1,10,0,10,11,0,11,8,4,5,9,-1,-1,-1,-1}, {0,4,5,0,5,10,0,10,11,0,11,3,-1,-1,-1,-1}, {4,5,10,4,10,11,4,11,8,-1,-1,-1,-1,-1,-1,-1},
    {5,9,8,5,8,7,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1}, {0,3,7,0,7,5,0,5,9,-1,-1,-1,-1,-1,-1,-1}, {0,8,7,0,7,5,0,5,1,-1,-1,-1,-1,-1,-1,-1}, {1,3,7,1,7,5,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1},
    {1,10,2,5,9,8,5,8,7,-1,-1,-1,-1,-1,-1,-1}, {0,3,7,0,7,5,0,5,9,1,10,2,-1,-1,-1,-1}, {0,8,7,0,7,5,0,5,10,0,10,2,-1,-1,-1,-1}, {2,3,7,2,7,5,2,5,10,-1,-1,-1,-1,-1,-1,-1},
    {2,11,3,5,9,8,5,8,7,-1,-1,-1,-1,-1,-1,-1}, {0,2,11,0,11,7,0,7,5,0,5,9,-1,-1,-1,-1}, {0,8,7,0,7,5,0,5,1,2,11,3,-1,-1,-1,-1}, {1,2,11,1,11,7,1,7,5,-1,-1,-1,-1,-1,-1,-1},
    {1,10,11,1,11,3,5,9,8,5,8,7,-1,-1,-1,-1}, {0,1,10,0,10,11,0,11,7,0,7,5,0,5,9,-1}, {0,8,7,0,7,5,0,5,10,0,10,11,0,11,3,-1}, {5,10,11,5,11,7,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1},
    {5,6,10,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1}, {0,3,8,5,6,10,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1}, {0,9,1,5,6,10,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1}, {1,3,8,1,8,9,5,6,10,-1,-1,-1,-1,-1,-1,-1},
    {1,5,6,1,6,2,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1}, {0,3,8,1,5,6,1,6,2,-1,-1,-1,-1,-1,-1,-1}, {0,9,5,0,5,6,0,6,2,-1,-1,-1,-1,-1,-1,-1}, {2,3,8,2,8,9,2,9,5,2,5,6,-1,-1,-1,-1},
    {2,11,3,5,6,10,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1}, {0,2,11,0,11,8,5,6,10,-1,-1,-1,-1,-1,-1,-1}, {0,9,1,2,11,3,5,6,10,-1,-1,-1,-1,-1,-1,-1}, {1,2,11,1,11,8,1,8,9,5,6,10,-1,-1,-1,-1},
    {1,5,6,1,6,11,1,11,3,-1,-1,-1,-1,-1,-1,-1}, {0,1,5,0,5,6,0,6,11,0,11,8,-1,-1,-1,-1}, {0,9,5,0,5,6,0,6,11,0,11,3,-1,-1,-1,-1}, {5,6,11,5,11,8,5,8,9,-1,-1,-1,-1,-1,-1,-1},
    {4,8,7,5,6,10,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1}, {0,3,7,0,7,4,5,6,10,-1,-1,-1,-1,-1,-1,-1}, {0,9,1,4,8,7,5,6,10,-1,-1,-1,-1,-1,-1,-1}, {1,3,7,1,7,4,1,4,9,5,6,10,-1,-1,-1,-1},
    {1,5,6,1,6,2,4,8,7,-1,-1,-1,-1,-1,-1,-1}, {0,3,7,0,7,4,1,5,6,1,6,2,-1,-1,-1,-1}, {0,9,5,0,5,6,0,6,2,4,8,7,-1,-1,-1,-1}, {2,3,7,2,7,4,2,4,9,2,9,5,2,5,6,-1},
    {2,11,3,4,8,7,5,6,10,-1,-1,-1,-1,-1,-1,-1}, {0,2,11,0,11,7,0,7,4,5,6,10,-1,-1,-1,-1}, {0,9,1,2,11,3,4,8,7,5,6,10,-1,-1,-1,-1}, {1,2,11,1,11,7,1,7,4,1,4,9,5,6,10,-1},
    {1,5,6,1,6,11,1,11,3,4,8,7,-1,-1,-1,-1}, {0,1,5,0,5,6,0,6,11,0,11,7,0,7,4,-1}, {0,9,5,0,5,6,0,6,11,0,11,3,4,8,7,-1}, {4,9,5,4,5,6,4,6,11,4,11,7,-1,-1,-1,-1},
    {4,6,10,4,10,9,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1}, {0,3,8,4,6,10,4,10,9,-1,-1,-1,-1,-1,-1,-1}, {0,4,6,0,6,10,0,10,1,-1,-1,-1,-1,-1,-1,-1}, {1,3,8,1,8,4,1,4,6,1,6,10,-1,-1,-1,-1},
    {1,9,4,1,4,6,1,6,2,-1,-1,-1,-1,-1,-1,-1}, {0,3,8,1,9,4,1,4,6,1,6,2,-1,-1,-1,-1}, {0,4,6,0,6,2,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1}, {2,3,8,2,8,4,2,4,6,-1,-1,-1,-1,-1,-1,-1},
    {2,11,3,4,6,10,4,10,9,-1,-1,-1,-1,-1,-1,-1}, {0,2,11,0,11,8,4,6,10,4,10,9,-1,-1,-1,-1}, {0,4,6,0,6,10,0,10,1,2,11,3,-1,-1,-1,-1}, {1,2,11,1,11,8,1,8,4,1,4,6,1,6,10,-1},
    {1,9,4,1,4,6,1,6,11,1,11,3,-1,-1,-1,-1}, {0,1,9,0,9,4,0,4,6,0,6,11,0,11,8,-1}, {0,4,6,0,6,11,0,11,3,-1,-1,-1,-1,-1,-1,-1}, {4,6,11,4,11,8,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1},
    {6,10,9,6,9,8,6,8,7,-1,-1,-1,-1,-1,-1,-1}, {0,3,7,0,7,6,0,6,10,0,10,9,-1,-1,-1,-1}, {0,8,7,0,7,6,0,6,10,0,10,1,-1,-1,-1,-1}, {1,3,7,1,7,6,1,6,10,-1,-1,-1,-1,-1,-1,-1},
    {1,9,8,1,8,7,1,7,6,1,6,2,-1,-1,-1,-1}, {0,3,7,0,7,6,0,6,2,0,2,1,0,1,9,-1}, {0,8,7,0,7,6,0,6,2,-1,-1,-1,-1,-1,-1,-1}, {2,3,7,2,7,6,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1},
    {2,11,3,6,10,9,6,9,8,6,8,7,-1,-1,-1,-1}, {0,2,11,0,11,7,0,7,6,0,6,10,0,10,9,-1}, {0,8,7,0,7,6,0,6,10,0,10,1,2,11,3,-1}, {1,2,11,1,11,7,1,7,6,1,6,10,-1,-1,-1,-1},
    {1,9,8,1,8,7,1,7,6,1,6,11,1,11,3,-1}, {0,1,9,6,11,7,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1}, {0,8,7,0,7,6,0,6,11,0,11,3,-1,-1,-1,-1}, {6,11,7,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1},
    {6,7,11,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1}, {0,3,8,6,7,11,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1}, {0,9,1,6,7,11,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1}, {1,3,8,1,8,9,6,7,11,-1,-1,-1,-1,-1,-1,-1},
    {1,10,2,6,7,11,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1}, {0,3,8,1,10,2,6,7,11,-1,-1,-1,-1,-1,-1,-1}, {0,9,10,0,10,2,6,7,11,-1,-1,-1,-1,-1,-1,-1}, {2,3,8,2,8,9,2,9,10,6,7,11,-1,-1,-1,-1},
    {2,6,7,2,7,3,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1}, {0,2,6,0,6,7,0,7,8,-1,-1,-1,-1,-1,-1,-1}, {0,9,1,2,6,7,2,7,3,-1,-1,-1,-1,-1,-1,-1}, {1,2,6,1,6,7,1,7,8,1,8,9,-1,-1,-1,-1},
    {1,10,6,1,6,7,1,7,3,-1,-1,-1,-1,-1,-1,-1}, {0,1,10,0,10,6,0,6,7,0,7,8,-1,-1,-1,-1}, {0,9,10,0,10,6,0,6,7,0,7,3,-1,-1,-1,-1}, {6,7,8,6,8,9,6,9,10,-1,-1,-1,-1,-1,-1,-1},
    {4,8,11,4,11,6,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1}, {0,3,11,0,11,6,0,6,4,-1,-1,-1,-1,-1,-1,-1}, {0,9,1,4,8,11,4,11,6,-1,-1,-1,-1,-1,-1,-1}, {1,3,11,1,11,6,1,6,4,1,4,9,-1,-1,-1,-1},
    {1,10,2,4,8,11,4,11,6,-1,-1,-1,-1,-1,-1,-1}, {0,3,11,0,11,6,0,6,4,1,10,2,-1,-1,-1,-1}, {0,9,10,0,10,2,4,8,11,4,11,6,-1,-1,-1,-1}, {2,3,11,2,11,6,2,6,4,2,4,9,2,9,10,-1},
    {2,6,4,2,4,8,2,8,3,-1,-1,-1,-1,-1,-1,-1}, {0,2,6,0,6,4,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1}, {0,9,1,2,6,4,2,4,8,2,8,3,-1,-1,-1,-1}, {1,2,6,1,6,4,1,4,9,-1,-1,-1,-1,-1,-1,-1},
    {1,10,6,1,6,4,1,4,8,1,8,3,-1,-1,-1,-1}, {0,1,10,0,10,6,0,6,4,-1,-1,-1,-1,-1,-1,-1}, {0,9,10,0,10,6,0,6,4,0,4,8,0,8,3,-1}, {4,9,10,4,10,6,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1},
    {4,5,9,6,7,11,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1}, {0,3,8,4,5,9,6,7,11,-1,-1,-1,-1,-1,-1,-1}, {0,4,5,0,5,1,6,7,11,-1,-1,-1,-1,-1,-1,-1}, {1,3,8,1,8,4,1,4,5,6,7,11,-1,-1,-1,-1},
    {1,10,2,4,5,9,6,7,11,-1,-1,-1,-1,-1,-1,-1}, {0,3,8,1,10,2,4,5,9,6,7,11,-1,-1,-1,-1}, {0,4,5,0,5,10,0,10,2,6,7,11,-1,-1,-1,-1}, {2,3,8,2,8,4,2,4,5,2,5,10,6,7,11,-1},
    {2,6,7,2,7,3,4,5,9,-1,-1,-1,-1,-1,-1,-1}, {0,2,6,0,6,7,0,7,8,4,5,9,-1,-1,-1,-1}, {0,4,5,0,5,1,2,6,7,2,7,3,-1,-1,-1,-1}, {1,2,6,1,6,7,1,7,8,1,8,4,1,4,5,-1},
    {1,10,6,1,6,7,1,7,3,4,5,9,-1,-1,-1,-1}, {0,1,10,0,10,6,0,6,7,0,7,8,4,5,9,-1}, {0,4,5,0,5,10,0,10,6,0,6,7,0,7,3,-1}, {4,5,10,4,10,6,4,6,7,4,7,8,-1,-1,-1,-1},
    {5,9,8,5,8,11,5,11,6,-1,-1,-1,-1,-1,-1,-1}, {0,3,11,0,11,6,0,6,5,0,5,9,-1,-1,-1,-1}, {0,8,11,0,11,6,0,6,5,0,5,1,-1,-1,-1,-1}, {1,3,11,1,11,6,1,6,5,-1,-1,-1,-1,-1,-1,-1},
    {1,10,2,5,9,8,5,8,11,5,11,6,-1,-1,-1,-1}, {0,3,11,0,11,6,0,6,5,0,5,9,1,10,2,-1}, {0,8,11,0,11,6,0,6,5,0,5,10,0,10,2,-1}, {2,3,11,2,11,6,2,6,5,2,5,10,-1,-1,-1,-1},
    {2,6,5,2,5,9,2,9,8,2,8,3,-1,-1,-1,-1}, {0,2,6,0,6,5,0,5,9,-1,-1,-1,-1,-1,-1,-1}, {0,8,3,0,3,2,0,2,6,0,6,5,0,5,1,-1}, {1,2,6,1,6,5,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1},
    {1,10,6,1,6,5,1,5,9,1,9,8,1,8,3,-1}, {0,1,10,0,10,6,0,6,5,0,5,9,-1,-1,-1,-1}, {0,8,3,5,10,6,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1}, {5,10,6,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1},
    {5,7,11,5,11,10,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1}, {0,3,8,5,7,11,5,11,10,-1,-1,-1,-1,-1,-1,-1}, {0,9,1,5,7,11,5,11,10,-1,-1,-1,-1,-1,-1,-1}, {1,3,8,1,8,9,5,7,11,5,11,10,-1,-1,-1,-1},
    {1,5,7,1,7,11,1,11,2,-1,-1,-1,-1,-1,-1,-1}, {0,3,8,1,5,7,1,7,11,1,11,2,-1,-1,-1,-1}, {0,9,5,0,5,7,0,7,11,0,11,2,-1,-1,-1,-1}, {2,3,8,2,8,9,2,9,5,2,5,7,2,7,11,-1},
    {2,10,5,2,5,7,2,7,3,-1,-1,-1,-1,-1,-1,-1}, {0,2,10,0,10,5,0,5,7,0,7,8,-1,-1,-1,-1}, {0,9,1,2,10,5,2,5,7,2,7,3,-1,-1,-1,-1}, {1,2,10,1,10,5,1,5,7,1,7,8,1,8,9,-1},
    {1,5,7,1,7,3,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1}, {0,1,5,0,5,7,0,7,8,-1,-1,-1,-1,-1,-1,-1}, {0,9,5,0,5,7,0,7,3,-1,-1,-1,-1,-1,-1,-1}, {5,7,8,5,8,9,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1},
    {4,8,11,4,11,10,4,10,5,-1,-1,-1,-1,-1,-1,-1}, {0,3,11,0,11,10,0,10,5,0,5,4,-1,-1,-1,-1}, {0,9,1,4,8,11,4,11,10,4,10,5,-1,-1,-1,-1}, {1,3,11,1,11,10,1,10,5,1,5,4,1,4,9,-1},
    {1,5,4,1,4,8,1,8,11,1,11,2,-1,-1,-1,-1}, {0,3,11,0,11,2,0,2,1,0,1,5,0,5,4,-1}, {0,9,5,0,5,4,0,4,8,0,8,11,0,11,2,-1}, {2,3,11,4,9,5,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1},
    {2,10,5,2,5,4,2,4,8,2,8,3,-1,-1,-1,-1}, {0,2,10,0,10,5,0,5,4,-1,-1,-1,-1,-1,-1,-1}, {0,9,1,2,10,5,2,5,4,2,4,8,2,8,3,-1}, {1,2,10,1,10,5,1,5,4,1,4,9,-1,-1,-1,-1},
    {1,5,4,1,4,8,1,8,3,-1,-1,-1,-1,-1,-1,-1}, {0,1,5,0,5,4,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1}, {0,9,5,0,5,4,0,4,8,0,8,3,-1,-1,-1,-1}, {4,9,5,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1},
    {4,7,11,4,11,10,4,10,9,-1,-1,-1,-1,-1,-1,-1}, {0,3,8,4,7,11,4,11,10,4,10,9,-1,-1,-1,-1}, {0,4,7,0,7,11,0,11,10,0,10,1,-1,-1,-1,-1}, {1,3,8,1,8,4,1,4,7,1,7,11,1,11,10,-1},
    {1,9,4,1,4,7,1,7,11,1,11,2,-1,-1,-1,-1}, {0,3,8,1,9,4,1,4,7,1,7,11,1,11,2,-1}, {0,4,7,0,7,11,0,11,2,-1,-1,-1,-1,-1,-1,-1}, {2,3,8,2,8,4,2,4,7,2,7,11,-1,-1,-1,-1},
    {2,10,9,2,9,4,2,4,7,2,7,3,-1,-1,-1,-1}, {0,2,10,0,10,9,0,9,4,0,4,7,0,7,8,-1}, {0,4,7,0,7,3,0,3,2,0,2,10,0,10,1,-1}, {1,2,10,4,7,8,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1},
    {1,9,4,1,4,7,1,7,3,-1,-1,-1,-1,-1,-1,-1}, {0,1,9,0,9,4,0,4,7,0,7,8,-1,-1,-1,-1}, {0,4,7,0,7,3,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1}, {4,7,8,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1},
    {8,11,10,8,10,9,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1}, {0,3,11,0,11,10,0,10,9,-1,-1,-1,-1,-1,-1,-1}, {0,8,11,0,11,10,0,10,1,-1,-1,-1,-1,-1,-1,-1}, {1,3,11,1,11,10,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1},
    {1,9,8,1,8,11,1,11,2,-1,-1,-1,-1,-1,-1,-1}, {0,3,11,0,11,2,0,2,1,0,1,9,-1,-1,-1,-1}, {0,8,11,0,11,2,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1}, {2,3,11,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1},
    {2,10,9,2,9,8,2,8,3,-1,-1,-1,-1,-1,-1,-1}, {0,2,10,0,10,9,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1}, {0,8,3,0,3,2,0,2,10,0,10,1,-1,-1,-1,-1}, {1,2,10,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1},
    {1,9,8,1,8,3,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1}, {0,1,9,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1}, {0,8,3,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1}, {-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1},
};

// cube edge -> owner corner offset (dx | dy << 1 | dz << 2) and axis (<< 3)
__constant__ unsigned char c_edge_owner[12] = {
    0 | (0 << 3), 1 | (1 << 3), 2 | (0 << 3), 0 | (1 << 3), 4 | (0 << 3), 5 | (1 << 3),
    6 | (0 << 3), 4 | (1 << 3), 0 | (2 << 3), 1 | (2 << 3), 3 | (2 << 3), 2 | (2 << 3)};

constexpr int kMeshBlock = 256;
constexpr int kScanThreads = 1024;
constexpr int kScanItems = 4;          // block counts per scan thread per chunk

// Voxel accessors of the two volumes.  The passes below address voxels by accessor coordinates (i,j,k) relative to a
// voxel bound with `bind`, read tsdf / weight / colour there, and ask whether a voxel exists (`inside`: the dense grid has
// borders, the block volume has none — its unallocated voxels read as tsdf 0, weight 0, colour 0).  `pos` gives the
// lattice index a vertex position is formed from.

// dense grid [nz,ny,nx]: accessor coordinates are grid indices, records keyed by the linear voxel index
struct DenseVox {
  const float* tsdf;
  const float* weight;
  const float* color;
  int nx, ny, nz;
  __device__ __forceinline__ size_t idx(int i, int j, int k) const { return ((size_t)k * ny + j) * nx + i; }
  __device__ __forceinline__ bool inside(int i, int j, int k) const {
    return i >= 0 && j >= 0 && k >= 0 && i < nx && j < ny && k < nz;
  }
  __device__ __forceinline__ float t(int i, int j, int k) const { return tsdf[idx(i, j, k)]; }
  __device__ __forceinline__ float w(int i, int j, int k) const { return weight[idx(i, j, k)]; }
  // color == nullptr: a volume without colours (the NeRF mesh lattice), colour 0
  __device__ __forceinline__ float c(int i, int j, int k, int ch) const { return color ? color[idx(i, j, k) * 3 + ch] : 0.f; }
  __device__ __forceinline__ DenseVox bind(size_t v, int& i, int& j, int& k) const {
    i = (int)(v % nx);
    j = (int)((v / nx) % ny);
    k = (int)(v / ((size_t)nx * ny));
    return *this;
  }
  __device__ __forceinline__ void pos(int i, int j, int k, int* p) const { p[0] = i; p[1] = j; p[2] = k; }
  // record key of the voxel at offset (dx,dy,dz) in {0,1}^3 from record key `key`, and the records to search for it:
  // keys are distinct and ascending, so it lies within (owner - key) places after r
  __device__ __forceinline__ int owner(int key, int dx, int dy, int dz, int r, int n, int& lo, int& hi) const {
    const int own = key + dx + dy * nx + dz * nx * ny;     // grids are limited to < 2^31 voxels
    lo = r; hi = min(n - 1, r + (own - key));
    return own;
  }
};

// block volume: pool [B,16,16,16] (x fastest); record key = pool index * 4096 + local voxel.  A bound accessor holds the
// pool block's row of the neighbour table [B,27] (-1 = unallocated; offset (a,b,c) in {-1,0,1}^3 at (a+1)+3(b+1)+9(c+1))
// and reads any voxel at accessor coordinates in [-16, 32) through it.
struct BlockVox {
  const float* tsdf;
  const float* weight;
  const float* color;
  const int* nbr;           // [B,27]
  const int* coords;        // [B,3] block coordinates
  const int* row;           // bound: nbr + 27 * pool index
  int bc[3];                // bound: block coordinate
  __device__ __forceinline__ long long idx(int i, int j, int k) const {
    const int q = row[((i >> 4) + 1) + 3 * ((j >> 4) + 1) + 9 * ((k >> 4) + 1)];
    return q < 0 ? -1 : ((long long)q << 12) + ((k & 15) << 8) + ((j & 15) << 4) + (i & 15);
  }
  __device__ __forceinline__ bool inside(int, int, int) const { return true; }
  __device__ __forceinline__ float t(int i, int j, int k) const { const long long v = idx(i, j, k); return v < 0 ? 0.f : tsdf[v]; }
  __device__ __forceinline__ float w(int i, int j, int k) const { const long long v = idx(i, j, k); return v < 0 ? 0.f : weight[v]; }
  __device__ __forceinline__ float c(int i, int j, int k, int ch) const {
    const long long v = idx(i, j, k);
    return v < 0 ? 0.f : color[v * 3 + ch];
  }
  __device__ __forceinline__ BlockVox bind(size_t v, int& i, int& j, int& k) const {
    const int p = (int)(v >> 12), l = (int)(v & 4095);
    i = l & 15; j = (l >> 4) & 15; k = l >> 8;
    BlockVox b = *this;
    b.row = nbr + 27 * (size_t)p;
    for (int q = 0; q < 3; q++) b.bc[q] = coords[3 * (size_t)p + q];
    return b;
  }
  __device__ __forceinline__ void pos(int i, int j, int k, int* p) const { p[0] = 16 * bc[0] + i; p[1] = 16 * bc[1] + j; p[2] = 16 * bc[2] + k; }
  // the owner may sit in a block of lower pool index: search below r or above it
  __device__ __forceinline__ int owner(int key, int dx, int dy, int dz, int r, int n, int& lo, int& hi) const {
    const int l = key & 4095, i = (l & 15) + dx, j = ((l >> 4) & 15) + dy, k = (l >> 8) + dz;
    const int q = nbr[27 * (size_t)(key >> 12) + ((i >> 4) + 1) + 3 * ((j >> 4) + 1) + 9 * ((k >> 4) + 1)];
    const int own = q < 0 ? -1 : (q << 12) + ((k & 15) << 8) + ((j & 15) << 4) + (i & 15);
    if (own >= key) { lo = r; hi = min(n - 1, r + (own - key)); } else { lo = 0; hi = r; }
    return own;
  }
};

__device__ __forceinline__ int tri_count(int cs) {
  int n = 0;
  while (n < 5 && c_tri[cs][3 * n] >= 0) n++;
  return n;
}

// voxel (i,j,k) -> vertex mask (bits 0-2: its +x, +y, +z edges carry a vertex) | case << 3 | cube valid << 11
template <class V>
__device__ int mesh_classify(const V& g, int i, int j, int k, float min_weight) {
  const bool hx = g.inside(i + 1, j, k), hy = g.inside(i, j + 1, k), hz = g.inside(i, j, k + 1);
  const bool n0 = g.t(i, j, k) < 0.f;
  const bool cx = hx && ((g.t(i + 1, j, k) < 0.f) != n0);
  const bool cy = hy && ((g.t(i, j + 1, k) < 0.f) != n0);
  const bool cz = hz && ((g.t(i, j, k + 1) < 0.f) != n0);
  int cs = 0;
  if (hx && hy && hz) {
#pragma unroll
    for (int n = 0; n < 8; n++) {
      const int dx = (n == 1 || n == 2 || n == 5 || n == 6), dy = (n == 2 || n == 3 || n == 6 || n == 7), dz = n >= 4;
      cs |= (g.t(i + dx, j + dy, k + dz) < 0.f) << n;
    }
  }
  if (!(cx || cy || cz) && (cs == 0 || cs == 255)) return 0;
  // weight test over the 3x3x3 neighbourhood: bit (a+1) + 3(b+1) + 9(c+1) for offset (a,b,c); a missing voxel fails
  unsigned ok = 0;
  for (int c = -1; c <= 1; c++)
    for (int b = -1; b <= 1; b++)
      for (int a = -1; a <= 1; a++) {
        const int ii = i + a, jj = j + b, kk = k + c;
        if (!g.inside(ii, jj, kk)) continue;
        if (g.w(ii, jj, kk) > min_weight) ok |= 1u << ((a + 1) + 3 * (b + 1) + 9 * (c + 1));
      }
  // cube at offset (a,b,c) in {-1,0}^3 is valid when its 8 corner bits are set: mask 0x361B shifted by (a+1)+3(b+1)+9(c+1)
  auto cube = [ok](int s) { return ((ok >> s) & 0x361Bu) == 0x361Bu; };
  const bool c000 = cube(13);
  int vm = 0;
  if (cx && (c000 || cube(10) || cube(4) || cube(1))) vm |= 1;
  if (cy && (c000 || cube(12) || cube(4) || cube(3))) vm |= 2;
  if (cz && (c000 || cube(12) || cube(10) || cube(9))) vm |= 4;
  return vm | (cs << 3) | ((c000 && hx && hy && hz) << 11);
}

__device__ __forceinline__ void mesh_counts(int bits, int& nv, int& nt, int& na) {
  nv = __popc(bits & 7);
  nt = (bits >> 11) & 1 ? tri_count((bits >> 3) & 255) : 0;
  na = (nv | nt) != 0;
}

// exclusive scan of (x, y, z) over the block; totals returned in tx, ty, tz.  blockDim.x = NT, a multiple of 32
template <int NT>
__device__ __forceinline__ void block_scan3(int& x, int& y, int& z, int& tx, int& ty, int& tz) {
  __shared__ int sw[3][NT / 32];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  int ix = x, iy = y, iz = z;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int ax = __shfl_up_sync(0xffffffffu, ix, o), ay = __shfl_up_sync(0xffffffffu, iy, o),
              az = __shfl_up_sync(0xffffffffu, iz, o);
    if (lane >= o) { ix += ax; iy += ay; iz += az; }
  }
  if (lane == 31) { sw[0][wid] = ix; sw[1][wid] = iy; sw[2][wid] = iz; }
  __syncthreads();
  if (wid == 0) {
    int wx = lane < NT / 32 ? sw[0][lane] : 0, wy = lane < NT / 32 ? sw[1][lane] : 0, wz = lane < NT / 32 ? sw[2][lane] : 0;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int ax = __shfl_up_sync(0xffffffffu, wx, o), ay = __shfl_up_sync(0xffffffffu, wy, o),
                az = __shfl_up_sync(0xffffffffu, wz, o);
      if (lane >= o) { wx += ax; wy += ay; wz += az; }
    }
    if (lane < NT / 32) { sw[0][lane] = wx; sw[1][lane] = wy; sw[2][lane] = wz; }   // inclusive over warps
  }
  __syncthreads();
  const int bx = wid ? sw[0][wid - 1] : 0, by = wid ? sw[1][wid - 1] : 0, bz = wid ? sw[2][wid - 1] : 0;
  x = bx + ix - x; y = by + iy - y; z = bz + iz - z;
  tx = sw[0][NT / 32 - 1]; ty = sw[1][NT / 32 - 1]; tz = sw[2][NT / 32 - 1];
  __syncthreads();                                        // sw is reused by the next call
}

// pass 1: per-block counts of vertices, triangles, active voxels -> scratch[4 + 3 * block + {0,1,2}]
template <class V>
__global__ void __launch_bounds__(kMeshBlock, 4) tsdf_mesh_classify_kernel(V g, size_t nvox, float min_weight, int* scratch) {
  const size_t v = (size_t)blockIdx.x * kMeshBlock + threadIdx.x;
  int nv = 0, nt = 0, na = 0;
  if (v < nvox) {
    int i, j, k;
    const V b = g.bind(v, i, j, k);
    mesh_counts(mesh_classify(b, i, j, k, min_weight), nv, nt, na);
  }
  int tv, tt, ta;
  block_scan3<kMeshBlock>(nv, nt, na, tv, tt, ta);
  if (threadIdx.x == 0) {
    int* c = scratch + 4 + 3 * (size_t)blockIdx.x;
    c[0] = tv; c[1] = tt; c[2] = ta;
  }
}

// pass 2: exclusive scan of the block counts in block order (one CTA), totals -> scratch[0..2]
__global__ void __launch_bounds__(kScanThreads) tsdf_mesh_scan_kernel(int* scratch, int nblocks) {
  int* c = scratch + 4;
  int carry[3] = {0, 0, 0};
  for (int base = 0; base < nblocks; base += kScanThreads * kScanItems) {
    const int first = base + threadIdx.x * kScanItems;
    int s[3] = {0, 0, 0};
    for (int q = 0; q < kScanItems; q++)
      if (first + q < nblocks)
        for (int ch = 0; ch < 3; ch++) s[ch] += c[3 * (size_t)(first + q) + ch];
    int t[3];
    block_scan3<kScanThreads>(s[0], s[1], s[2], t[0], t[1], t[2]);
    for (int ch = 0; ch < 3; ch++) s[ch] += carry[ch];
    for (int q = 0; q < kScanItems; q++)
      if (first + q < nblocks)
        for (int ch = 0; ch < 3; ch++) {
          const int x = c[3 * (size_t)(first + q) + ch];
          c[3 * (size_t)(first + q) + ch] = s[ch];
          s[ch] += x;
        }
    for (int ch = 0; ch < 3; ch++) carry[ch] += t[ch];
  }
  if (threadIdx.x == 0) { scratch[0] = carry[0]; scratch[1] = carry[1]; scratch[2] = carry[2]; scratch[3] = 0; }
}

struct MeshOut {
  float ox, oy, oz, voxel;
  float min_weight;
  int4* active;             // [A] (record key, vertex base, triangle base, classify bits)
  int n_active;
  float* vertices;          // [V,3]
  float* colors;            // [V,3] in [0,1]
  float* normals;           // [V,3]
  int* triangles;           // [T,3]
};

// TSDF gradient component along `axis` at voxel p: central difference, one-sided where a neighbour is missing
template <class V>
__device__ __forceinline__ float tsdf_grad(const V& g, const int* p, int axis) {
  int lo[3] = {p[0], p[1], p[2]}, hi[3] = {p[0], p[1], p[2]};
  lo[axis] -= 1; hi[axis] += 1;
  const bool has_lo = g.inside(lo[0], lo[1], lo[2]), has_hi = g.inside(hi[0], hi[1], hi[2]);
  if (!has_lo && !has_hi) return 0.f;
  if (!has_lo) return __fsub_rn(g.t(hi[0], hi[1], hi[2]), g.t(p[0], p[1], p[2]));
  if (!has_hi) return __fsub_rn(g.t(p[0], p[1], p[2]), g.t(lo[0], lo[1], lo[2]));
  return __fmul_rn(__fsub_rn(g.t(hi[0], hi[1], hi[2]), g.t(lo[0], lo[1], lo[2])), 0.5f);
}

template <class V>
__device__ void emit_vertex(const V& g, const MeshOut& o, int i, int j, int k, int axis, int id) {
  int p0[3] = {i, j, k}, p1[3] = {i, j, k};
  p1[axis] += 1;
  const float f0 = g.t(i, j, k), f1 = g.t(p1[0], p1[1], p1[2]);
  const float t = __fdiv_rn(f0, __fsub_rn(f0, f1));
  int li[3];
  g.pos(i, j, k, li);
  float idx[3] = {(float)li[0], (float)li[1], (float)li[2]};
  idx[axis] = __fadd_rn(idx[axis], t);
  const float org[3] = {o.ox, o.oy, o.oz};
  const size_t w = (size_t)id * 3;
#pragma unroll
  for (int a = 0; a < 3; a++) o.vertices[w + a] = __fadd_rn(org[a], __fmul_rn(o.voxel, idx[a]));
#pragma unroll
  for (int c = 0; c < 3; c++) o.colors[w + c] = __fdiv_rn(lerp_rn(g.c(i, j, k, c), g.c(p1[0], p1[1], p1[2], c), t), 255.f);
  float n[3];
#pragma unroll
  for (int a = 0; a < 3; a++) n[a] = lerp_rn(tsdf_grad(g, p0, a), tsdf_grad(g, p1, a), t);
  const float len = __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(n[0], n[0]), __fmul_rn(n[1], n[1])), __fmul_rn(n[2], n[2])));
#pragma unroll
  for (int a = 0; a < 3; a++) o.normals[w + a] = len > 0.f ? __fdiv_rn(n[a], len) : 0.f;
}

// pass 3: active-voxel records in ascending key order and the vertices
template <class V>
__global__ void __launch_bounds__(kMeshBlock) tsdf_mesh_compact_kernel(V g, size_t nvox, const int* scratch, MeshOut o) {
  const size_t v = (size_t)blockIdx.x * kMeshBlock + threadIdx.x;
  int bits = 0, i = 0, j = 0, k = 0;
  V b = g;
  if (v < nvox) {
    b = g.bind(v, i, j, k);
    bits = mesh_classify(b, i, j, k, o.min_weight);
  }
  int nv, nt, na;
  mesh_counts(bits, nv, nt, na);
  const bool is_active = na;
  int tv, tt, ta;
  block_scan3<kMeshBlock>(nv, nt, na, tv, tt, ta);
  if (!is_active) return;
  const int* c = scratch + 4 + 3 * (size_t)blockIdx.x;
  const int vbase = c[0] + nv, tbase = c[1] + nt, r = c[2] + na;
  o.active[r] = make_int4((int)v, vbase, tbase, bits);
  int id = vbase;
  for (int a = 0; a < 3; a++)
    if ((bits >> a) & 1) emit_vertex(b, o, i, j, k, a, id++);
}

// pass 4: triangles of every active voxel whose cube is valid; each edge resolved to its owner's record by binary search
template <class V>
__global__ void __launch_bounds__(kMeshBlock) tsdf_mesh_triangles_kernel(V g, MeshOut o) {
  const int r = blockIdx.x * kMeshBlock + threadIdx.x;
  if (r >= o.n_active) return;
  const int4 rec = o.active[r];
  if (!((rec.w >> 11) & 1)) return;
  const int cs = (rec.w >> 3) & 255;
  const int nt = tri_count(cs);
  for (int s = 0; s < nt; s++)
    for (int q = 0; q < 3; q++) {
      const int eo = c_edge_owner[c_tri[cs][3 * s + q]];
      const int axis = eo >> 3;
      int lo, hi;
      const int owner = g.owner(rec.x, eo & 1, (eo >> 1) & 1, (eo >> 2) & 1, r, o.n_active, lo, hi);
      while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (o.active[mid].x < owner) lo = mid + 1; else hi = mid;
      }
      const int4 own = o.active[lo];
      o.triangles[3 * ((size_t)rec.z + s) + q] = own.x == owner ? own.y + __popc(own.w & ((1 << axis) - 1)) : -1;
    }
}

// ---------------------------------------------------------------------------------------------------------------- ray cast
// dense grid: a sample outside the grid is unobserved; the hit's cell is clamped into the grid
struct DenseRay {
  DenseVox g;
  float min_weight;
  __device__ __forceinline__ bool locate(const float* gq, size_t& v, float* fr, bool clamp) const {
    const int dims[3] = {g.nx, g.ny, g.nz};
    int ix[3];
    bool inb = true;
#pragma unroll
    for (int q = 0; q < 3; q++) {
      float fl = floorf(gq[q]);
      if (clamp) fl = fminf(fmaxf(fl, 0.f), (float)(dims[q] - 2));
      inb = inb && fl >= 0.f && fl <= (float)(dims[q] - 2);
      ix[q] = inb ? (int)fl : 0;
      fr[q] = __fsub_rn(gq[q], fl);
    }
    v = g.idx(ix[0], ix[1], ix[2]);
    return inb;
  }
  __device__ __forceinline__ size_t corner(size_t v, int n) const {
    return v + (n & 1) + ((n >> 1) & 1) * (size_t)g.nx + (n >> 2) * (size_t)g.nx * g.ny;
  }
  __device__ __forceinline__ bool sample(const float* gq, float& f) const {
    size_t v;
    float fr[3];
    if (!locate(gq, v, fr, false)) return false;
    for (int n = 0; n < 8; n++)
      if (!(g.weight[corner(v, n)] > min_weight)) return false;
    float t[8];
#pragma unroll
    for (int n = 0; n < 8; n++) t[n] = g.tsdf[corner(v, n)];
    f = trilerp8(t, fr[0], fr[1], fr[2]);
    return true;
  }
  __device__ __forceinline__ void hit(const float* gq, RayCell& c) const {
    size_t v;
    float fr[3];
    locate(gq, v, fr, true);
    c.fx = fr[0]; c.fy = fr[1]; c.fz = fr[2];
#pragma unroll
    for (int n = 0; n < 8; n++) {
      const size_t q = corner(v, n);
      c.t[n] = g.tsdf[q]; c.w[n] = g.weight[q];
      for (int ch = 0; ch < 3; ch++) c.c[ch][n] = g.color[q * 3 + ch];
    }
  }
};

// grids whose worst-case vertex (3 per voxel) and triangle (5 per cube) counts fit int32
static bool mesh_grid_ok(int nx, int ny, int nz) {
  if (nx <= 0 || ny <= 0 || nz <= 0) return false;
  const long long n = (long long)nx * ny * nz;
  const long long cubes = (long long)(nx - 1) * (ny - 1) * (nz - 1);
  return 3 * n <= INT_MAX && 5 * cubes <= INT_MAX;
}

// block pools whose worst-case vertex and triangle counts (3 and 5 per voxel) fit int32
static bool mesh_blocks_ok(int n_blocks) { return n_blocks >= 0 && 5LL * 4096 * n_blocks <= INT_MAX; }

template <class V>
static int mesh_count(const V& g, size_t n, float min_weight, int* scratch, void* stream) {
  const int nblocks = (int)((n + kMeshBlock - 1) / kMeshBlock);
  tsdf_mesh_classify_kernel<<<nblocks, kMeshBlock, 0, (cudaStream_t)stream>>>(g, n, min_weight, scratch);
  NSLAM_CHECK_LAUNCH();
  tsdf_mesh_scan_kernel<<<1, kScanThreads, 0, (cudaStream_t)stream>>>(scratch, nblocks);
  NSLAM_CHECK_LAUNCH();
  return 0;
}

template <class V>
static int mesh_emit(const V& g, size_t n, const int* scratch, const MeshOut& o, void* stream) {
  if (o.n_active == 0) return 0;
  const int nblocks = (int)((n + kMeshBlock - 1) / kMeshBlock);
  tsdf_mesh_compact_kernel<<<nblocks, kMeshBlock, 0, (cudaStream_t)stream>>>(g, n, scratch, o);
  NSLAM_CHECK_LAUNCH();
  tsdf_mesh_triangles_kernel<<<(o.n_active + kMeshBlock - 1) / kMeshBlock, kMeshBlock, 0, (cudaStream_t)stream>>>(g, o);
  NSLAM_CHECK_LAUNCH();
  return 0;
}

}  // namespace nslam

extern "C" {

/* Scratch size (int32 elements) of nslam_tsdf_mesh_count for a [nz,ny,nx] grid: 4 + 3 per 256 voxels.
 * cudaErrorInvalidValue when the worst-case vertex or triangle count of the grid overflows int32. */
int nslam_tsdf_mesh_plan(int nx, int ny, int nz, long long* scratch_ints) {
  using namespace nslam;
  if (!mesh_grid_ok(nx, ny, nz)) return (int)cudaErrorInvalidValue;
  const long long n = (long long)nx * ny * nz;
  *scratch_ints = 4 + 3 * ((n + kMeshBlock - 1) / kMeshBlock);
  return 0;
}

/* Marching cubes, counting passes: scratch (DEVICE, nslam_tsdf_mesh_plan ints) receives the per-block offsets and, in
 * scratch[0..2], the numbers of vertices, triangles and active voxels. */
int nslam_tsdf_mesh_count(const float* tsdf, const float* weight, int nx, int ny, int nz, float min_weight, int* scratch,
                          void* stream) {
  using namespace nslam;
  if (!mesh_grid_ok(nx, ny, nz)) return (int)cudaErrorInvalidValue;
  return mesh_count(DenseVox{tsdf, weight, nullptr, nx, ny, nz}, (size_t)nx * ny * nz, min_weight, scratch, stream);
}

/* Marching cubes, emission passes after nslam_tsdf_mesh_count with the same volume and min_weight: active [n_active,4]
 * int32 scratch; vertices / vertex_colors ([0,1]) / vertex_normals [V,3] fp32, triangles [T,3] int32 (DEVICE, sized
 * from the counts).  origin3 = world position of voxel (0,0,0) (HOST).  Launches nothing when n_active is 0. */
int nslam_tsdf_mesh_emit(const float* tsdf, const float* weight, const float* color, int nx, int ny, int nz,
                         const float* origin3_host, float voxel_size, float min_weight, const int* scratch, int n_active,
                         int* active, float* vertices, float* vertex_colors, float* vertex_normals, int* triangles,
                         void* stream) {
  using namespace nslam;
  if (!mesh_grid_ok(nx, ny, nz) || n_active < 0) return (int)cudaErrorInvalidValue;
  MeshOut o{origin3_host[0], origin3_host[1], origin3_host[2], voxel_size, min_weight, (int4*)active, n_active,
            vertices, vertex_colors, vertex_normals, triangles};
  return mesh_emit(DenseVox{tsdf, weight, color, nx, ny, nz}, (size_t)nx * ny * nz, scratch, o, stream);
}

/* Ray cast n views of the volume in one launch: cam_T_world_tq [n,7] (t, q_xyzw) DEVICE; intr4 = fx, fy, cx, cy (HOST);
 * outputs [n,H,W] depth (z, 0 on a miss), [n,H,W,3] colour in [0,1], [n,H,W] weight, [n,H,W,3] unit normal toward
 * +tsdf or NULL (DEVICE). */
int nslam_tsdf_raycast(const float* tsdf, const float* weight, const float* color, int nx, int ny, int nz,
                       const float* origin3_host, float voxel_size, const float* cam_T_world_tq, int n, int H, int W,
                       const float* intr4_host, float min_depth, float max_depth, float sdf_trunc, float min_weight,
                       float* depth, float* color_out, float* weight_out, float* normal_out, void* stream) {
  using namespace nslam;
  if (nx < 2 || ny < 2 || nz < 2 || n < 0 || H <= 0 || W <= 0 || n > 65535 || (long long)H * W > INT_MAX)
    return (int)cudaErrorInvalidValue;
  if (n == 0) return 0;
  const RayParams a = ray_params(origin3_host, voxel_size, cam_T_world_tq, H, W, intr4_host, min_depth, max_depth,
                                 sdf_trunc, depth, color_out, weight_out, normal_out);
  dim3 grid((unsigned)(((long long)H * W + 127) / 128), n);
  tsdf_raycast_kernel<<<grid, 128, 0, (cudaStream_t)stream>>>(a, DenseRay{DenseVox{tsdf, weight, color, nx, ny, nz}, min_weight});
  NSLAM_CHECK_LAUNCH();
  return 0;
}

/* Marching cubes over a voxel-block volume (csrc/tsdf_blocks.cu): the dense read-out of the volume's dense embedding
 * (tsdf, weight, colour 0 outside its blocks) at lattice origin 0.  Scratch size (int32 elements): 4 + 48 per block;
 * cudaErrorInvalidValue when the worst-case vertex or triangle count of n_blocks blocks overflows int32. */
int nslam_tsdf_blocks_mesh_plan(int n_blocks, long long* scratch_ints) {
  using namespace nslam;
  if (!mesh_blocks_ok(n_blocks)) return (int)cudaErrorInvalidValue;
  *scratch_ints = 4 + 3 * ((4096LL * n_blocks + kMeshBlock - 1) / kMeshBlock);
  return 0;
}

/* Counting passes over the pool: tsdf / weight [B,16,16,16], neighbours [B,27] (nslam_tsdf_blocks_neighbours), block
 * coordinates [B,3] int32 (DEVICE).  min_weight >= 0, so that no voxel outside the blocks is observed. */
int nslam_tsdf_blocks_mesh_count(const float* tsdf, const float* weight, const int* neighbours, const int* block_coords,
                                 int n_blocks, float min_weight, int* scratch, void* stream) {
  using namespace nslam;
  if (!mesh_blocks_ok(n_blocks) || !(min_weight >= 0.f)) return (int)cudaErrorInvalidValue;
  if (n_blocks == 0) {
    cudaMemsetAsync(scratch, 0, 4 * sizeof(int), (cudaStream_t)stream);
    NSLAM_CHECK_LAUNCH();
    return 0;
  }
  return mesh_count(BlockVox{tsdf, weight, nullptr, neighbours, block_coords, nullptr, {0, 0, 0}}, 4096 * (size_t)n_blocks,
                    min_weight, scratch, stream);
}

/* Emission passes after nslam_tsdf_blocks_mesh_count, as nslam_tsdf_mesh_emit.  Vertices are ordered by (pool index,
 * local voxel, axis), triangles by (pool index, local cube, table order); positions are voxel_size * lattice index. */
int nslam_tsdf_blocks_mesh_emit(const float* tsdf, const float* weight, const float* color, const int* neighbours,
                                const int* block_coords, int n_blocks, float voxel_size, float min_weight, const int* scratch,
                                int n_active, int* active, float* vertices, float* vertex_colors, float* vertex_normals,
                                int* triangles, void* stream) {
  using namespace nslam;
  if (!mesh_blocks_ok(n_blocks) || n_active < 0 || !(min_weight >= 0.f)) return (int)cudaErrorInvalidValue;
  MeshOut o{0.f, 0.f, 0.f, voxel_size, min_weight, (int4*)active, n_active, vertices, vertex_colors, vertex_normals, triangles};
  return mesh_emit(BlockVox{tsdf, weight, color, neighbours, block_coords, nullptr, {0, 0, 0}}, 4096 * (size_t)n_blocks,
                   scratch, o, stream);
}

}  // extern "C"
