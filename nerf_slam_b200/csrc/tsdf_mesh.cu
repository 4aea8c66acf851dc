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
#include "common.cuh"

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

struct MeshVolume {
  const float* tsdf;
  const float* weight;
  const float* color;
  int nx, ny, nz;
  float min_weight;
};

__device__ __forceinline__ int tri_count(int cs) {
  int n = 0;
  while (n < 5 && c_tri[cs][3 * n] >= 0) n++;
  return n;
}

// voxel (i,j,k) -> vertex mask (bits 0-2: its +x, +y, +z edges carry a vertex) | case << 3 | cube valid << 11
__device__ int mesh_classify(const MeshVolume& g, int i, int j, int k) {
  const size_t sy = (size_t)g.nx, sz = (size_t)g.nx * g.ny;
  const size_t v = (size_t)k * sz + (size_t)j * sy + i;
  const bool hx = i + 1 < g.nx, hy = j + 1 < g.ny, hz = k + 1 < g.nz;
  const bool n0 = g.tsdf[v] < 0.f;
  const bool cx = hx && ((g.tsdf[v + 1] < 0.f) != n0);
  const bool cy = hy && ((g.tsdf[v + sy] < 0.f) != n0);
  const bool cz = hz && ((g.tsdf[v + sz] < 0.f) != n0);
  int cs = 0;
  if (hx && hy && hz) {
#pragma unroll
    for (int n = 0; n < 8; n++) {
      const int dx = (n == 1 || n == 2 || n == 5 || n == 6), dy = (n == 2 || n == 3 || n == 6 || n == 7), dz = n >= 4;
      cs |= (g.tsdf[v + dx + dy * sy + dz * sz] < 0.f) << n;
    }
  }
  if (!(cx || cy || cz) && (cs == 0 || cs == 255)) return 0;
  // weight test over the 3x3x3 neighbourhood: bit (a+1) + 3(b+1) + 9(c+1) for offset (a,b,c); outside the grid = fails
  unsigned ok = 0;
  for (int c = -1; c <= 1; c++)
    for (int b = -1; b <= 1; b++)
      for (int a = -1; a <= 1; a++) {
        const int ii = i + a, jj = j + b, kk = k + c;
        if (ii < 0 || jj < 0 || kk < 0 || ii >= g.nx || jj >= g.ny || kk >= g.nz) continue;
        if (g.weight[(size_t)kk * sz + (size_t)jj * sy + ii] > g.min_weight) ok |= 1u << ((a + 1) + 3 * (b + 1) + 9 * (c + 1));
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

__device__ __forceinline__ void voxel_ijk(const MeshVolume& g, size_t v, int& i, int& j, int& k) {
  i = (int)(v % g.nx);
  j = (int)((v / g.nx) % g.ny);
  k = (int)(v / ((size_t)g.nx * g.ny));
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
__global__ void __launch_bounds__(kMeshBlock, 4) tsdf_mesh_classify_kernel(MeshVolume g, size_t nvox, int* scratch) {
  const size_t v = (size_t)blockIdx.x * kMeshBlock + threadIdx.x;
  int nv = 0, nt = 0, na = 0;
  if (v < nvox) {
    int i, j, k;
    voxel_ijk(g, v, i, j, k);
    mesh_counts(mesh_classify(g, i, j, k), nv, nt, na);
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
  int4* active;             // [A] (voxel index, vertex base, triangle base, classify bits)
  int n_active;
  float* vertices;          // [V,3]
  float* colors;            // [V,3] in [0,1]
  float* normals;           // [V,3]
  int* triangles;           // [T,3]
};

// TSDF gradient component along one axis at voxel (i,j,k): central difference, one-sided at the border
__device__ __forceinline__ float tsdf_grad(const MeshVolume& g, size_t v, int idx, int n, size_t stride) {
  if (n < 2) return 0.f;
  if (idx == 0) return __fsub_rn(g.tsdf[v + stride], g.tsdf[v]);
  if (idx == n - 1) return __fsub_rn(g.tsdf[v], g.tsdf[v - stride]);
  return __fmul_rn(__fsub_rn(g.tsdf[v + stride], g.tsdf[v - stride]), 0.5f);
}

__device__ __forceinline__ float lerp_rn(float a, float b, float t) { return __fadd_rn(a, __fmul_rn(t, __fsub_rn(b, a))); }

__device__ void emit_vertex(const MeshVolume& g, const MeshOut& o, int i, int j, int k, size_t v, int axis, int id) {
  const size_t sy = (size_t)g.nx, sz = (size_t)g.nx * g.ny;
  const size_t s = axis == 0 ? 1 : axis == 1 ? sy : sz;
  const float f0 = g.tsdf[v], f1 = g.tsdf[v + s];
  const float t = __fdiv_rn(f0, __fsub_rn(f0, f1));
  float idx[3] = {(float)i, (float)j, (float)k};
  idx[axis] = __fadd_rn(idx[axis], t);
  const float org[3] = {o.ox, o.oy, o.oz};
  const size_t w = (size_t)id * 3;
#pragma unroll
  for (int a = 0; a < 3; a++) o.vertices[w + a] = __fadd_rn(org[a], __fmul_rn(o.voxel, idx[a]));
#pragma unroll
  for (int c = 0; c < 3; c++) o.colors[w + c] = __fdiv_rn(lerp_rn(g.color[v * 3 + c], g.color[(v + s) * 3 + c], t), 255.f);
  int p0[3] = {i, j, k}, p1[3] = {i, j, k};
  p1[axis] += 1;
  const int dims[3] = {g.nx, g.ny, g.nz};
  const size_t str[3] = {1, sy, sz};
  float n[3];
#pragma unroll
  for (int a = 0; a < 3; a++) {
    const float g0 = tsdf_grad(g, v, p0[a], dims[a], str[a]);
    const float g1 = tsdf_grad(g, v + s, p1[a], dims[a], str[a]);
    n[a] = lerp_rn(g0, g1, t);
  }
  const float len = __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(n[0], n[0]), __fmul_rn(n[1], n[1])), __fmul_rn(n[2], n[2])));
#pragma unroll
  for (int a = 0; a < 3; a++) o.normals[w + a] = len > 0.f ? __fdiv_rn(n[a], len) : 0.f;
}

// pass 3: active-voxel records in ascending voxel order and the vertices
__global__ void __launch_bounds__(kMeshBlock) tsdf_mesh_compact_kernel(MeshVolume g, size_t nvox, const int* scratch,
                                                                       MeshOut o) {
  const size_t v = (size_t)blockIdx.x * kMeshBlock + threadIdx.x;
  int bits = 0, i = 0, j = 0, k = 0;
  if (v < nvox) {
    voxel_ijk(g, v, i, j, k);
    bits = mesh_classify(g, i, j, k);
  }
  int nv, nt, na;
  mesh_counts(bits, nv, nt, na);
  const bool is_active = na;
  int tv, tt, ta;
  block_scan3<kMeshBlock>(nv, nt, na, tv, tt, ta);
  if (!is_active) return;
  const int* b = scratch + 4 + 3 * (size_t)blockIdx.x;
  const int vbase = b[0] + nv, tbase = b[1] + nt, r = b[2] + na;
  o.active[r] = make_int4((int)v, vbase, tbase, bits);
  int id = vbase;
  for (int a = 0; a < 3; a++)
    if ((bits >> a) & 1) emit_vertex(g, o, i, j, k, v, a, id++);
}

// pass 4: triangles of every active voxel whose cube is valid
__global__ void __launch_bounds__(kMeshBlock) tsdf_mesh_triangles_kernel(MeshVolume g, MeshOut o) {
  const int r = blockIdx.x * kMeshBlock + threadIdx.x;
  if (r >= o.n_active) return;
  const int4 rec = o.active[r];
  if (!((rec.w >> 11) & 1)) return;
  const int cs = (rec.w >> 3) & 255;
  const int nt = tri_count(cs);
  const int sy = g.nx, sz = g.nx * g.ny;                 // grids are limited to < 2^31 voxels
  for (int s = 0; s < nt; s++)
    for (int q = 0; q < 3; q++) {
      const int eo = c_edge_owner[c_tri[cs][3 * s + q]];
      const int owner = rec.x + (eo & 1) + ((eo >> 1) & 1) * sy + ((eo >> 2) & 1) * sz, axis = eo >> 3;
      // records are sorted by distinct voxel index, so the owner's record lies within owner - voxel places after r
      int lo = r, hi = min(o.n_active - 1, r + (owner - rec.x));
      while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (o.active[mid].x < owner) lo = mid + 1; else hi = mid;
      }
      const int4 own = o.active[lo];
      o.triangles[3 * ((size_t)rec.z + s) + q] = own.x == owner ? own.y + __popc(own.w & ((1 << axis) - 1)) : -1;
    }
}

// ---------------------------------------------------------------------------------------------------------------- ray cast
struct RayArgs {
  MeshVolume g;
  float ox, oy, oz, voxel;
  const float* pose;        // [n,7] cam_T_world (t, q_xyzw), DEVICE
  int H, W;
  float fx, fy, cx, cy, min_depth, max_depth, trunc;
  float* depth;             // [n,H,W]
  float* color;             // [n,H,W,3]
  float* weight;            // [n,H,W]
  float* normal;            // [n,H,W,3] or NULL
};

struct Cell {
  size_t v;                 // linear index of the cell's corner (0,0,0)
  float fx, fy, fz;         // fractions within the cell
};

__device__ __forceinline__ float tri_lerp(const float* a, size_t sy, size_t sz, size_t v, int ch, int nch, const Cell& c) {
  auto at = [&](int dx, int dy, int dz) { return a[(v + dx + dy * sy + dz * sz) * nch + ch]; };
  const float c0 = lerp_rn(lerp_rn(at(0, 0, 0), at(1, 0, 0), c.fx), lerp_rn(at(0, 1, 0), at(1, 1, 0), c.fx), c.fy);
  const float c1 = lerp_rn(lerp_rn(at(0, 0, 1), at(1, 0, 1), c.fx), lerp_rn(at(0, 1, 1), at(1, 1, 1), c.fx), c.fy);
  return lerp_rn(c0, c1, c.fz);
}

__global__ void __launch_bounds__(128) tsdf_raycast_kernel(RayArgs a) {
  __shared__ double sR[9];
  __shared__ float sgo[3];
  const int view = blockIdx.y;
  if (threadIdx.x == 0) {
    const float* p = a.pose + 7 * (size_t)view;
    const double qx = p[3], qy = p[4], qz = p[5], qw = p[6];
    const double R[9] = {1 - 2 * (qy * qy + qz * qz), 2 * (qx * qy - qz * qw), 2 * (qx * qz + qy * qw),
                         2 * (qx * qy + qz * qw), 1 - 2 * (qx * qx + qz * qz), 2 * (qy * qz - qx * qw),
                         2 * (qx * qz - qy * qw), 2 * (qy * qz + qx * qw), 1 - 2 * (qx * qx + qy * qy)};
    for (int i = 0; i < 9; i++) sR[i] = (double)(float)R[i];       // the fp32 rotation of the pose, as tsdf.cu
    const double t0 = p[0], t1 = p[1], t2 = p[2];
    const float org[3] = {a.ox, a.oy, a.oz};
    for (int c = 0; c < 3; c++) {
      // camera centre -R^T t, then grid coordinates (world - origin) / voxel
      const float cw = (float)-__dadd_rn(__dadd_rn(__dmul_rn((double)(float)R[c], t0), __dmul_rn((double)(float)R[3 + c], t1)),
                                         __dmul_rn((double)(float)R[6 + c], t2));
      sgo[c] = __fdiv_rn(__fsub_rn(cw, org[c]), a.voxel);
    }
  }
  __syncthreads();
  const int pix = blockIdx.x * blockDim.x + threadIdx.x;
  if (pix >= a.H * a.W) return;
  const int u = pix % a.W, v = pix / a.W;
  const float dxc = __fdiv_rn(__fsub_rn((float)u, a.cx), a.fx), dyc = __fdiv_rn(__fsub_rn((float)v, a.cy), a.fy);
  float gd[3];
#pragma unroll
  for (int c = 0; c < 3; c++)
    gd[c] = __fdiv_rn((float)__dadd_rn(__dadd_rn(__dmul_rn(sR[c], (double)dxc), __dmul_rn(sR[3 + c], (double)dyc)), sR[6 + c]),
                      a.voxel);
  const float len = __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(dxc, dxc), __fmul_rn(dyc, dyc)), 1.f));
  const MeshVolume& g = a.g;
  const int dims[3] = {g.nx, g.ny, g.nz};
  const size_t sy = (size_t)g.nx, sz = (size_t)g.nx * g.ny;

  // grid cell of depth z; false outside the grid
  auto locate = [&](float z, Cell& c, bool clamp) {
    float fr[3];
    int ix[3];
    bool inb = true;
#pragma unroll
    for (int q = 0; q < 3; q++) {
      const float gq = __fadd_rn(sgo[q], __fmul_rn(z, gd[q]));
      float fl = floorf(gq);
      if (clamp) fl = fminf(fmaxf(fl, 0.f), (float)(dims[q] - 2));
      inb = inb && fl >= 0.f && fl <= (float)(dims[q] - 2);
      ix[q] = inb ? (int)fl : 0;
      fr[q] = __fsub_rn(gq, fl);
    }
    c.v = (size_t)ix[2] * sz + (size_t)ix[1] * sy + ix[0];
    c.fx = fr[0]; c.fy = fr[1]; c.fz = fr[2];
    return inb;
  };
  auto observed = [&](size_t v0) {
    bool ok = true;
#pragma unroll
    for (int n = 0; n < 8; n++) ok = ok && g.weight[v0 + (n & 1) + ((n >> 1) & 1) * sy + (n >> 2) * sz] > g.min_weight;
    return ok;
  };

  const int max_steps = (int)ceilf(__fdiv_rn(__fmul_rn(__fsub_rn(a.max_depth, a.min_depth), len), a.voxel)) + 2;
  float z = a.min_depth, z_prev = 0.f, f_prev = 0.f, z_hit = 0.f;
  bool have_prev = false, hit = false;
  for (int s = 0; s < max_steps && z <= a.max_depth; s++) {
    Cell c;
    const bool obs = locate(z, c, false) && observed(c.v);
    const float f = tri_lerp(g.tsdf, sy, sz, c.v, 0, 1, c);
    if (obs && have_prev && f_prev > 0.f && f <= 0.f) {
      z_hit = __fadd_rn(z_prev, __fdiv_rn(__fmul_rn(__fsub_rn(z, z_prev), f_prev), __fsub_rn(f_prev, f)));
      hit = true;
      break;
    }
    const float step = obs && f > 0.f ? fmaxf(__fmul_rn(f, a.trunc), a.voxel) : a.voxel;
    have_prev = obs; f_prev = f; z_prev = z;
    z = __fadd_rn(z, __fdiv_rn(step, len));
  }

  const size_t o = (size_t)view * a.H * a.W + pix;
  if (!hit) {
    a.depth[o] = 0.f; a.weight[o] = 0.f;
    for (int c = 0; c < 3; c++) a.color[3 * o + c] = 0.f;
    if (a.normal) for (int c = 0; c < 3; c++) a.normal[3 * o + c] = 0.f;
    return;
  }
  Cell c;
  locate(z_hit, c, true);
  a.depth[o] = z_hit;
  a.weight[o] = tri_lerp(g.weight, sy, sz, c.v, 0, 1, c);
  for (int ch = 0; ch < 3; ch++) a.color[3 * o + ch] = __fdiv_rn(tri_lerp(g.color, sy, sz, c.v, ch, 3, c), 255.f);
  if (a.normal) {
    auto T = [&](int dx, int dy, int dz) { return g.tsdf[c.v + dx + dy * sy + dz * sz]; };
    auto d = [](float p, float q) { return __fsub_rn(p, q); };
    const float gx = lerp_rn(lerp_rn(d(T(1, 0, 0), T(0, 0, 0)), d(T(1, 1, 0), T(0, 1, 0)), c.fy),
                             lerp_rn(d(T(1, 0, 1), T(0, 0, 1)), d(T(1, 1, 1), T(0, 1, 1)), c.fy), c.fz);
    const float gy = lerp_rn(lerp_rn(d(T(0, 1, 0), T(0, 0, 0)), d(T(1, 1, 0), T(1, 0, 0)), c.fx),
                             lerp_rn(d(T(0, 1, 1), T(0, 0, 1)), d(T(1, 1, 1), T(1, 0, 1)), c.fx), c.fz);
    const float gz = lerp_rn(lerp_rn(d(T(0, 0, 1), T(0, 0, 0)), d(T(1, 0, 1), T(1, 0, 0)), c.fx),
                             lerp_rn(d(T(0, 1, 1), T(0, 1, 0)), d(T(1, 1, 1), T(1, 1, 0)), c.fx), c.fy);
    const float gl = __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(gx, gx), __fmul_rn(gy, gy)), __fmul_rn(gz, gz)));
    a.normal[3 * o + 0] = gl > 0.f ? __fdiv_rn(gx, gl) : 0.f;
    a.normal[3 * o + 1] = gl > 0.f ? __fdiv_rn(gy, gl) : 0.f;
    a.normal[3 * o + 2] = gl > 0.f ? __fdiv_rn(gz, gl) : 0.f;
  }
}

// grids whose worst-case vertex (3 per voxel) and triangle (5 per cube) counts fit int32
static bool mesh_grid_ok(int nx, int ny, int nz) {
  if (nx <= 0 || ny <= 0 || nz <= 0) return false;
  const long long n = (long long)nx * ny * nz;
  const long long cubes = (long long)(nx - 1) * (ny - 1) * (nz - 1);
  return 3 * n <= INT_MAX && 5 * cubes <= INT_MAX;
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
  const size_t n = (size_t)nx * ny * nz;
  const int nblocks = (int)((n + kMeshBlock - 1) / kMeshBlock);
  MeshVolume g{tsdf, weight, nullptr, nx, ny, nz, min_weight};
  tsdf_mesh_classify_kernel<<<nblocks, kMeshBlock, 0, (cudaStream_t)stream>>>(g, n, scratch);
  NSLAM_CHECK_LAUNCH();
  tsdf_mesh_scan_kernel<<<1, kScanThreads, 0, (cudaStream_t)stream>>>(scratch, nblocks);
  NSLAM_CHECK_LAUNCH();
  return 0;
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
  if (n_active == 0) return 0;
  const size_t n = (size_t)nx * ny * nz;
  const int nblocks = (int)((n + kMeshBlock - 1) / kMeshBlock);
  MeshVolume g{tsdf, weight, color, nx, ny, nz, min_weight};
  MeshOut o{origin3_host[0], origin3_host[1], origin3_host[2], voxel_size, (int4*)active, n_active,
            vertices, vertex_colors, vertex_normals, triangles};
  tsdf_mesh_compact_kernel<<<nblocks, kMeshBlock, 0, (cudaStream_t)stream>>>(g, n, scratch, o);
  NSLAM_CHECK_LAUNCH();
  tsdf_mesh_triangles_kernel<<<(n_active + kMeshBlock - 1) / kMeshBlock, kMeshBlock, 0, (cudaStream_t)stream>>>(g, o);
  NSLAM_CHECK_LAUNCH();
  return 0;
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
  RayArgs a{};
  a.g = MeshVolume{tsdf, weight, color, nx, ny, nz, min_weight};
  a.ox = origin3_host[0]; a.oy = origin3_host[1]; a.oz = origin3_host[2]; a.voxel = voxel_size;
  a.pose = cam_T_world_tq; a.H = H; a.W = W;
  a.fx = intr4_host[0]; a.fy = intr4_host[1]; a.cx = intr4_host[2]; a.cy = intr4_host[3];
  a.min_depth = min_depth; a.max_depth = max_depth; a.trunc = sdf_trunc;
  a.depth = depth; a.color = color_out; a.weight = weight_out; a.normal = normal_out;
  dim3 grid((unsigned)(((long long)H * W + 127) / 128), n);
  tsdf_raycast_kernel<<<grid, 128, 0, (cudaStream_t)stream>>>(a);
  NSLAM_CHECK_LAUNCH();
  return 0;
}

}  // extern "C"
