"""Cleaning and simplifying triangle meshes on the GPU (csrc/mesh_ops.cu, rules at its head; DESIGN §4h): connected
components, small-component removal, culling to what cameras saw, compaction to a triangle subset, Open3D-style
area-weighted vertex normals and vertex clustering.

    mesh = nerf.build_mesh(resolution=256, thresh=10.0)
    mesh = cull(mesh, cam_T_world, intrinsics, W, H, depths=MeshScene(mesh).render(cam_T_world, intrinsics, W, H).depth)
    mesh = remove_small_components(mesh, min_area=0.01)
    mesh = simplify_vertex_clustering(mesh, voxel_size=0.02)

Every operation takes a `TsdfMesh` (TsdfFusion / NerfFusion.build_mesh) or a (vertices [V,3], triangles [T,3]) pair;
numpy arrays are uploaded to the current device, CPU tensors are refused (there is no CPU path).  An operation that
returns a mesh returns a `TsdfMesh` of device tensors, or None when no triangle remains.  Kept vertices keep their
colours and normals; a pair has no colours, so its output gets colours 0 and `vertex_normals` of the output.  Every
result is the same bits in every run.  A vertex index outside [0, V) and, where positions are used (areas, culling,
normals, clustering), a non-finite vertex of a triangle are refused with a ValueError."""
import math

import numpy as np
import torch

from . import _lib
from .evaluation import INT32_MAX, _cuda_tensor, _mesh_arrays, visible
from .tsdf_fusion import TsdfMesh

FIXED_AREA = 2.0 ** 40          # component areas: integers of 2^-40 m^2 (the weights of evaluation.sample_surface)


def _arrays(mesh):
    """-> V [V,3] fp32, T [T,3] int32, colours and normals [V,3] fp32 (None for a pair)"""
    V, T = _mesh_arrays(mesh)
    if V.shape[0] >= INT32_MAX:
        raise ValueError(f"{V.shape[0]} vertices: the kernels' counts need fewer than 2^31 - 1")
    if 3 * T.shape[0] > INT32_MAX:
        raise ValueError(f"{T.shape[0]} triangles exceed the int32 corner count")
    C = N = None
    if hasattr(mesh, "vertices") and hasattr(mesh, "triangles"):
        C = _cuda_tensor(mesh.vertex_colors, torch.float32, "vertex colors")
        N = _cuda_tensor(mesh.vertex_normals, torch.float32, "vertex normals")
        for x, name in ((C, "vertex colors"), (N, "vertex normals")):
            if tuple(x.shape) != tuple(V.shape):
                raise ValueError(f"{name} must be [{V.shape[0]},3], got {tuple(x.shape)}")
            if x.device != V.device:
                raise ValueError(f"{name} and vertices must be on one device")
    return V, T, C, N


def _refuse(flags):
    if flags & 1:
        raise ValueError("a triangle indexes a vertex outside the mesh")
    if flags & 2:
        raise ValueError("the mesh has non-finite vertex coordinates")
    if flags & 4:
        raise ValueError("the mesh is too large for the 64-bit area sums (2^22 m^2 in all)")


def connected_components(mesh):
    """-> (labels [T] int32, n_triangles [C] int64, area [C] float64) device tensors: the component of every triangle,
    numbered 0..C-1 in the order of each component's lowest triangle index, and each component's triangle count and
    area (m^2, the sum of the fixed-point triangle weights rint(area 2^40) / 2^40; 2^22 m^2 in all at most).  Two
    triangles are connected when they share a vertex INDEX: positions are not compared, so unwelded duplicate vertices
    stay apart.  Every mesh this project emits shares its vertices between cubes and blocks, so for those the
    components are the geometric ones.  One host read (C and the validity flags)."""
    V, T, _, _ = _arrays(mesh)
    lib = _lib.load()
    nv, nt, dev = int(V.shape[0]), int(T.shape[0]), V.device
    if nt == 0:
        return (torch.empty(0, dtype=torch.int32, device=dev), torch.empty(0, dtype=torch.int64, device=dev),
                torch.empty(0, dtype=torch.float64, device=dev))
    if nv == 0:
        raise ValueError("a triangle indexes a vertex outside the mesh")
    scratch = torch.empty(_lib.query_size("nslam_mesh_components_scratch", nv, nt), dtype=torch.uint8, device=dev)
    labels = torch.empty(nt, dtype=torch.int32, device=dev)
    counts = torch.empty(nt, dtype=torch.int64, device=dev)
    area = torch.empty(nt, dtype=torch.int64, device=dev)
    info = torch.empty(2, dtype=torch.int64, device=dev)
    with _lib.fixed_stream():
        _lib.check(lib.nslam_mesh_components(_lib.ptr(V), nv, _lib.ptr(T), nt, _lib.ptr(scratch), scratch.numel(),
                                             _lib.ptr(labels), _lib.ptr(counts), _lib.ptr(area), _lib.ptr(info),
                                             _lib.stream_ptr()), "mesh_components")
        n_comp, flags = info.tolist()
    _refuse(flags)
    return labels, counts[:n_comp].clone(), area[:n_comp].to(torch.float64) / FIXED_AREA


def _normals(V, T):
    lib = _lib.load()
    nv, nt = int(V.shape[0]), int(T.shape[0])
    out = torch.zeros(nv, 3, dtype=torch.float32, device=V.device)
    if nt == 0:
        return out
    if nv == 0:
        raise ValueError("a triangle indexes a vertex outside the mesh")
    scratch = torch.empty(_lib.query_size("nslam_mesh_vertex_normals_scratch", nv, nt), dtype=torch.uint8,
                          device=V.device)
    info = torch.empty(1, dtype=torch.int64, device=V.device)
    _lib.check(lib.nslam_mesh_vertex_normals(_lib.ptr(V), nv, _lib.ptr(T), nt, _lib.ptr(scratch), scratch.numel(),
                                             _lib.ptr(out), _lib.ptr(info), _lib.stream_ptr()), "mesh_vertex_normals")
    _refuse(int(info.item()))
    return out


def vertex_normals(mesh):
    """-> [V,3] fp32 device tensor, the rule of Open3D's compute_vertex_normals (what the reference calls on its TSDF
    meshes): each vertex sums the unnormalised (b - a) x (c - a) of its triangles (fp64, ascending triangle order), and
    the sum is normalised in fp64 and rounded once; a zero sum (e.g. an unreferenced vertex) gives (0, 0, 0).  One host
    read (the validity flags)."""
    V, T, _, _ = _arrays(mesh)
    return _normals(V, T)


def submesh(mesh, keep):
    """-> TsdfMesh of the triangles with keep [T] bool set, or None when there is none.  Kept triangles stay in input
    order; the output vertices are the vertices they reference, in input order, with their colours and normals.  One
    8-byte host read (the output sizes)."""
    V, T, C, N = _arrays(mesh)
    if torch.is_tensor(keep):
        if not keep.is_cuda:
            raise RuntimeError("keep must be a CUDA tensor: mesh operations run on sm_90a kernels, there is no CPU path")
        keep = keep.contiguous()
    else:
        keep = _lib.h2d(np.asarray(keep, bool), V.device)
    if keep.dtype != torch.bool or tuple(keep.shape) != (T.shape[0],):
        raise ValueError(f"keep must be a bool mask of shape ({T.shape[0]},), got {keep.dtype} {tuple(keep.shape)}")
    if keep.device != V.device:
        raise ValueError("keep and the mesh must be on one device")
    return _compact(V, T, C, N, keep)


def _compact(V, T, C, N, keep):
    lib = _lib.load()
    nv, nt, dev = int(V.shape[0]), int(T.shape[0]), V.device
    if nt == 0:
        return None
    if nv == 0:
        raise ValueError("a triangle indexes a vertex outside the mesh")
    scratch = torch.empty(_lib.query_size("nslam_mesh_submesh_scratch", nv, nt), dtype=torch.uint8, device=dev)
    counts = torch.empty(2, dtype=torch.int32, device=dev)
    with _lib.fixed_stream():
        _lib.check(lib.nslam_mesh_submesh_count(_lib.ptr(T), nv, nt, _lib.ptr(keep), _lib.ptr(scratch), scratch.numel(),
                                                _lib.ptr(counts), _lib.stream_ptr()), "mesh_submesh_count")
        n_vert, n_tri = counts.tolist()
        if n_vert < 0:
            raise ValueError("a triangle indexes a vertex outside the mesh")
        if n_tri == 0:
            return None
        verts = torch.empty(n_vert, 3, dtype=torch.float32, device=dev)
        cols = torch.zeros(n_vert, 3, dtype=torch.float32, device=dev) if C is None else torch.empty_like(verts)
        nrms = torch.empty_like(verts) if N is not None else None
        tris = torch.empty(n_tri, 3, dtype=torch.int32, device=dev)
        _lib.check(lib.nslam_mesh_submesh_emit(_lib.ptr(V), _lib.ptr(C), _lib.ptr(N), nv, _lib.ptr(T), nt,
                                               _lib.ptr(scratch), scratch.numel(), _lib.ptr(verts),
                                               _lib.ptr(cols if C is not None else None), _lib.ptr(nrms), _lib.ptr(tris),
                                               _lib.stream_ptr()), "mesh_submesh_emit")
        del scratch
        if nrms is None:
            nrms = _normals(verts, tris)
    return TsdfMesh(verts, tris, cols, nrms)


def remove_small_components(mesh, min_area):
    """-> TsdfMesh of the triangles whose connected component (connected_components) has an area >= min_area (m^2),
    or None.  Two host reads (the component count and flags, the output sizes)."""
    min_area = float(min_area)
    if math.isnan(min_area):
        raise ValueError("min_area must be a number")
    V, T, C, N = _arrays(mesh)
    if T.shape[0] == 0:
        return None
    labels, _, area = connected_components((V, T))
    keep = torch.index_select(area >= min_area, 0, labels)
    del labels
    return _compact(V, T, C, N, keep)


def cull(mesh, cam_T_world, intrinsics, width, height, depths=None, depth_tol=0.05, near=0.0, far=math.inf):
    """-> TsdfMesh of the triangles with at least one vertex seen by a camera, or None: the culling step of
    NICE-SLAM-style evaluation (a face goes only when none of its vertices is seen).  Seen is evaluation.visible with
    the same arguments: cam_T_world [n,7] (t, q_xyzw), intrinsics fx, fy, cx, cy at width x height, near < z <= far
    and, with depth maps [n,H,W], z <= depth + depth_tol (e.g. depth rendered from the mesh itself, for occlusion).
    A triangle with a non-finite vertex is refused.  Two host reads (the validity flags, the output sizes)."""
    V, T, C, N = _arrays(mesh)
    lib = _lib.load()
    nv, nt = int(V.shape[0]), int(T.shape[0])
    if nt == 0:
        return None
    if nv == 0:
        raise ValueError("a triangle indexes a vertex outside the mesh")
    seen = visible(V, cam_T_world, intrinsics, width, height, depths, depth_tol, near, far)
    keep = torch.empty(nt, dtype=torch.bool, device=V.device)
    flags = torch.empty(1, dtype=torch.int32, device=V.device)
    _lib.check(lib.nslam_mesh_any_vertex(_lib.ptr(V), _lib.ptr(T), nv, nt, _lib.ptr(seen), _lib.ptr(keep),
                                         _lib.ptr(flags), _lib.stream_ptr()), "mesh_any_vertex")
    del seen
    _refuse(int(flags.item()))
    return _compact(V, T, C, N, keep)


def _voxel(voxel_size):
    with np.errstate(over="ignore"):
        v32 = float(np.float32(float(voxel_size)))
    if not (math.isfinite(v32) and v32 > 0):
        raise ValueError(f"voxel_size must be positive and finite in fp32, got {voxel_size}")
    return v32


def simplify_vertex_clustering(mesh, voxel_size):
    """-> TsdfMesh of the mesh clustered on cells of voxel_size (metres; the fp32 value is used) anchored at the world
    origin, or None.  The cell of a vertex is floor(p / voxel) per axis in fp64, keyed as point-cloud downsampling; a
    vertex outside the key range (2^20 cells from the origin per axis) is dropped with its triangles.  Vertices no
    triangle references are ignored.  A triangle with two corners in one cell is dropped; of triangles with the same
    unordered cell triple the lowest-index one is kept, with its winding; kept triangles stay in input order.  One
    output vertex per cell a kept triangle references, in ascending key order: the mean position and colour of the
    cell's referenced input vertices (fp64 sums in vertex order, rounded once); normals are vertex_normals of the
    output.  One host read (the output sizes and the validity flags)."""
    voxel = _voxel(voxel_size)
    V, T, C, _ = _arrays(mesh)
    lib = _lib.load()
    nv, nt, dev = int(V.shape[0]), int(T.shape[0]), V.device
    if nt == 0:
        return None
    if nv == 0:
        raise ValueError("a triangle indexes a vertex outside the mesh")
    scratch = torch.empty(_lib.query_size("nslam_mesh_cluster_scratch", nv, nt), dtype=torch.uint8, device=dev)
    info = torch.empty(3, dtype=torch.int32, device=dev)
    with _lib.fixed_stream():
        _lib.check(lib.nslam_mesh_cluster_count(_lib.ptr(V), nv, _lib.ptr(T), nt, voxel, _lib.ptr(scratch),
                                                scratch.numel(), _lib.ptr(info), _lib.stream_ptr()), "mesh_cluster_count")
        n_vert, n_tri, flags = info.tolist()
        _refuse(flags)
        if n_tri == 0:
            return None
        verts = torch.empty(n_vert, 3, dtype=torch.float32, device=dev)
        cols = torch.empty_like(verts)
        tris = torch.empty(n_tri, 3, dtype=torch.int32, device=dev)
        _lib.check(lib.nslam_mesh_cluster_emit(_lib.ptr(V), _lib.ptr(C), nv, _lib.ptr(T), nt, _lib.ptr(scratch),
                                               scratch.numel(), _lib.ptr(verts), _lib.ptr(cols), _lib.ptr(tris),
                                               _lib.stream_ptr()), "mesh_cluster_emit")
        del scratch
        nrms = _normals(verts, tris)
    return TsdfMesh(verts, tris, cols, nrms)
