"""Depth, triangle-id, normal and colour views of triangle meshes on the GPU (csrc/mesh_render.cu, rules at its head;
DESIGN §4g).  The reference renders its ground-truth mesh through Open3D's OpenGL visualiser (utils/evaluation.py,
MeshRenderer); here a linear BVH over the triangles is ray cast exactly, with the cameras of the TSDF ray cast:

    scene = MeshScene(mesh, leaf_size=4)          # TsdfMesh, NeRF mesh, or (vertices, triangles[, vertex_colors])
    out = scene.render(cam_T_world, intrinsics, width, height, normals=True, colors=True)
    out.depth, out.triangle, out.normal, out.color

Pixel (u, v) of view k casts the ray from the camera centre along R^T ((u - cx) / fx, (v - cy) / fy, 1), so depth is the
z-depth, as in `TsdfFusion.render_volume` and the synthetic room.  Every hit is exact (a watertight fp64 test, the
nearest hit, ties to the smaller triangle index), so the views do not depend on the tree or the launch.  Inputs are
CUDA tensors or numpy arrays (uploaded to the current device); there is no CPU path."""
import math
from dataclasses import dataclass
from typing import Optional

import numpy as np
import torch

from . import _lib
from .evaluation import INT32_MAX, _cuda_tensor, _mesh_arrays

LEAF_SIZE = 4                   # triangles per BVH leaf
INT64_MAX = 2 ** 63 - 1


@dataclass
class MeshViews:
    """device tensors: depth [n,H,W] fp32 (0 on a miss), triangle [n,H,W] int32 (-1 on a miss), normal / color
    [n,H,W,3] fp32 or None when not asked for"""
    depth: torch.Tensor
    triangle: torch.Tensor
    normal: Optional[torch.Tensor] = None
    color: Optional[torch.Tensor] = None


def _check_host_side(x, name, cols):
    """what can be refused before any device work: a CPU tensor, a shape other than [N, cols]"""
    if torch.is_tensor(x) and not x.is_cuda:
        raise RuntimeError(f"{name} must be a CUDA tensor: rendering runs on sm_90a kernels, there is no CPU path")
    shape = tuple(x.shape) if torch.is_tensor(x) else np.shape(x)
    if len(shape) != 2 or shape[1] != cols:
        raise ValueError(f"{name} must be [N,{cols}], got {shape}")


def _mesh_colors(mesh, n_vert, device):
    if hasattr(mesh, "vertices") and hasattr(mesh, "triangles"):
        c = getattr(mesh, "vertex_colors", None)
    else:
        c = mesh[2] if len(mesh) > 2 else None
    if c is None:
        return None
    c = _cuda_tensor(c, torch.float32, "vertex colors")
    if tuple(c.shape) != (n_vert, 3):
        raise ValueError(f"vertex colors must be [{n_vert},3], got {tuple(c.shape)}")
    if c.device != device:
        raise ValueError("vertex colors and vertices must be on one device")
    return c


class MeshScene:
    """a triangle mesh ready to render: a linear BVH over its triangles with leaf buckets of `leaf_size` (1..32)
    triangles, built once.  `mesh`: TsdfMesh / NeRF mesh (vertices, triangles, vertex_colors) or a (vertices [V,3],
    triangles [T,3][, vertex_colors [V,3]]) tuple.  The BVH keeps its own copy of the triangles' vertices; the vertex
    colours stay referenced and are read when a view asks for colours.  One host read, for the build's validity flags
    (a vertex index outside the mesh, a non-finite vertex): both are refused with a ValueError."""

    def __init__(self, mesh, leaf_size=LEAF_SIZE):
        V, T = (mesh.vertices, mesh.triangles) if hasattr(mesh, "vertices") else (mesh[0], mesh[1])
        _check_host_side(V, "mesh vertices", 3)
        _check_host_side(T, "mesh triangles", 3)
        lib = _lib.load()
        V, T = _mesh_arrays((V, T))
        self.n_vert, self.n_tri, self.leaf_size, self.device = int(V.shape[0]), int(T.shape[0]), int(leaf_size), V.device
        if self.n_tri == 0 or self.n_vert == 0:
            raise ValueError("the mesh has no triangle")
        if self.n_tri > INT32_MAX:
            raise ValueError(f"{self.n_tri} triangles exceed int32")
        if not 1 <= self.leaf_size <= 32:
            raise ValueError(f"leaf_size must be in 1..32, got {leaf_size}")
        self.vertex_colors = _mesh_colors(mesh, self.n_vert, self.device)
        self.bvh = torch.empty(_lib.query_size("nslam_render_bvh_scratch", self.n_tri, self.leaf_size), dtype=torch.uint8,
                               device=self.device)
        info = torch.empty(1, dtype=torch.int64, device=self.device)
        _lib.check(lib.nslam_render_bvh_build(_lib.ptr(V), self.n_vert, _lib.ptr(T), self.n_tri, self.leaf_size,
                                              _lib.ptr(self.bvh), self.bvh.numel(), _lib.ptr(info), _lib.stream_ptr()),
                   "render_bvh_build")
        flags = int(info.item())
        if flags & 1:
            raise ValueError("a triangle indexes a vertex outside the mesh")
        if flags & 2:
            raise ValueError("the mesh has non-finite vertex coordinates")

    def render(self, cam_T_world, intrinsics, width, height, near=0.0, far=math.inf, normals=False, colors=False,
               cull_backfaces=False, num_sms=0):
        """-> MeshViews of the views cam_T_world [n,7] (t, q_xyzw) with pinhole intrinsics fx, fy, cx, cy at width x
        height.  Only hits with near < depth <= far count.  Back faces count unless `cull_backfaces`, which keeps only
        hits on the side (b - a) x (c - a) points to (free space for a TsdfMesh).  `normals`: the unit geometric normal
        of the hit triangle, world frame, as wound; `colors`: the barycentric blend of the vertex colours (the mesh must
        have them).  num_sms bounds the grid (0: every SM); no result depends on it.  No host read."""
        _check_host_side(cam_T_world, "cam_T_world", 7)
        lib = _lib.load()
        poses = _cuda_tensor(cam_T_world, torch.float32, "cam_T_world")
        if poses.dim() != 2 or poses.shape[1] != 7:
            raise ValueError(f"cam_T_world must be [n,7] (t, q_xyzw), got {tuple(poses.shape)}")
        if poses.device != self.device:
            raise ValueError("cam_T_world and the mesh must be on one device")
        W, H, n = int(width), int(height), int(poses.shape[0])
        if not (0 < W <= INT32_MAX and 0 < H <= INT32_MAX):
            raise ValueError(f"image size must be positive, got {W} x {H}")
        if 3 * n * H * W > INT64_MAX:
            raise ValueError(f"{n} x {H} x {W} pixels exceed the kernels' int64 indexing")
        if colors and self.vertex_colors is None:
            raise ValueError("colors=True needs a mesh with vertex colours")
        if not float(far) > float(near):
            raise ValueError(f"far ({far}) must exceed near ({near})")
        intr = np.ascontiguousarray(np.asarray(intrinsics.detach().cpu() if torch.is_tensor(intrinsics) else intrinsics,
                                               np.float32).reshape(-1))
        if intr.size != 4:
            raise ValueError(f"intrinsics must be fx, fy, cx, cy, got {intr.size} values")
        dev = self.device
        out = MeshViews(torch.empty(n, H, W, dtype=torch.float32, device=dev),
                        torch.empty(n, H, W, dtype=torch.int32, device=dev),
                        torch.empty(n, H, W, 3, dtype=torch.float32, device=dev) if normals else None,
                        torch.empty(n, H, W, 3, dtype=torch.float32, device=dev) if colors else None)
        if n == 0:
            return out
        _lib.check(lib.nslam_render_views(_lib.ptr(self.bvh), self.bvh.numel(), self.n_tri, self.leaf_size,
                                          _lib.ptr(self.vertex_colors if colors else None), _lib.ptr(poses), n,
                                          intr.ctypes.data, W, H, float(near), float(far), int(bool(cull_backfaces)),
                                          int(num_sms), _lib.ptr(out.depth), _lib.ptr(out.triangle), _lib.ptr(out.normal),
                                          _lib.ptr(out.color), _lib.stream_ptr()), "render_views")
        return out


def render_mesh(mesh, cam_T_world, intrinsics, width, height, **kwargs):
    """MeshScene(mesh).render(...) for a one-off view set"""
    return MeshScene(mesh).render(cam_T_world, intrinsics, width, height, **kwargs)
