"""Coloured point clouds of the SLAM keyframe map on the GPU (csrc/point_cloud.cu, rules at its head).

The reference shows this map in its Open3D GUI (gui/open3d_gui.py: `get_depth_masks` :289-299, `build_pcls` :646-678):
every keyframe's upsampled inverse depth, masked by the depth sigma in the "uncertainty" mode, back-projected through its
BA pose and coloured by its image.  Here the whole packet goes through two kernel passes with one host read, optionally
through DROID's multi-view depth filter (`droid_backends.depth_filter`) first and Open3D-style voxel averaging after.

    cloud = build_point_cloud(packet, intrinsics, voxel_size=0.01)      # -> PointCloud or None
    cloud.write_ply("map.ply")

`TsdfFusion.build_point_cloud` (and its GUI packet key "build_pcl") and `RaftVisualFrontend.point_cloud` call it."""
import math

import numpy as np
import torch

from . import _lib

INT32_MAX = 2 ** 31 - 1
_PLY_TYPES = {"<f4": "float", "<i4": "int"}


def write_binary_ply(path, columns, triangles=None):
    """binary little-endian PLY: one vertex property per (name, 1-D array) of `columns` (float32 -> float, int32 -> int),
    and with `triangles` [T,3] a face element (uchar count, int vertex indices)"""
    cols = [(k, np.ascontiguousarray(a, np.dtype(a.dtype).newbyteorder("<"))) for k, a in columns]
    vt = np.empty(len(cols[0][1]), [(k, a.dtype.str) for k, a in cols])
    for k, a in cols:
        vt[k] = a
    head = ["ply", "format binary_little_endian 1.0", f"element vertex {len(vt)}"] + \
           [f"property {_PLY_TYPES[a.dtype.str]} {k}" for k, a in cols]
    ft = None
    if triangles is not None:
        t = np.asarray(triangles).astype("<i4")
        ft = np.empty(t.shape[0], [("n", "u1"), ("v", "<i4", (3,))])
        ft["n"], ft["v"] = 3, t
        head += [f"element face {t.shape[0]}", "property list uchar int vertex_indices"]
    head.append("end_header")
    with open(path, "wb") as f:
        f.write(("\n".join(head) + "\n").encode("ascii"))
        f.write(vt.tobytes())
        if ft is not None:
            f.write(ft.tobytes())


class PointCloud:
    """device tensors: points [N,3] fp32 (world, metres), colors [N,3] fp32 in [0,1]; after voxel downsampling also
    counts [N] int32, the number of points merged into each"""

    def __init__(self, points, colors, counts=None):
        self.points, self.colors, self.counts = points, colors, counts

    def __len__(self):
        return int(self.points.shape[0])

    def write_ply(self, path):
        """binary little-endian PLY: float x y z red green blue (colours in [0,1]), plus int count when downsampled"""
        p = self.points.detach().float().cpu().numpy()
        c = self.colors.detach().float().cpu().numpy()
        cols = [(k, p[:, i]) for i, k in enumerate("xyz")] + [(k, c[:, i]) for i, k in enumerate(("red", "green", "blue"))]
        if self.counts is not None:
            cols.append(("count", self.counts.detach().cpu().numpy().astype(np.int32)))
        write_binary_ply(path, cols)


class _CloudKernels:
    """the device passes of build_point_cloud (tests substitute the numpy restatement, tests/point_cloud_oracle.py)"""

    @staticmethod
    def _cuda(*ts):
        for t in ts:
            if t is not None and not t.is_cuda:
                raise RuntimeError("point clouds (sm_90a) need CUDA tensors; there is no CPU path")

    def filter_counts(self, poses, idepths, intr, thresh):
        """droid_backends.depth_filter of every keyframe against its packet neighbours (i-1, i-2, i-3, i+3, i+4, i+5),
        one threshold for all -> [n,H,W] fp32 counts"""
        from . import droid_backends as db
        n = poses.shape[0]
        ix = torch.arange(n, dtype=torch.int64, device=poses.device)
        th = torch.full((n,), float(thresh), dtype=torch.float32, device=poses.device)
        return db.depth_filter(poses, idepths, intr, ix, th)

    def cloud(self, poses, idepths, covs, images, intr, max_depth, max_sigma, views, min_views):
        """-> points, colors [N,3] fp32 (N may be 0).  One host read: the kept total."""
        self._cuda(poses, idepths, covs, images, intr, views)
        lib = _lib.load()
        n, H, W = idepths.shape
        dev = idepths.device
        nb = np.zeros(1, np.int64)
        _lib.check(lib.nslam_point_cloud_scratch(n, H, W, nb.ctypes.data), "point_cloud_scratch")
        scratch = torch.empty(int(nb[0]), dtype=torch.uint8, device=dev)
        total = torch.empty(1, dtype=torch.int32, device=dev)
        mv = int(min_views) if views is not None else 0
        with _lib.fixed_stream():
            _lib.check(lib.nslam_point_cloud_count(_lib.ptr(idepths), _lib.ptr(covs), _lib.ptr(views), mv, n, H, W,
                                                   float(max_depth), float(max_sigma), _lib.ptr(scratch), int(nb[0]),
                                                   _lib.ptr(total), _lib.stream_ptr()), "point_cloud_count")
            N = int(total.item())
            points = torch.empty(N, 3, dtype=torch.float32, device=dev)
            colors = torch.empty(N, 3, dtype=torch.float32, device=dev)
            if N:
                _lib.check(lib.nslam_point_cloud_emit(
                    _lib.ptr(poses), _lib.ptr(idepths), _lib.ptr(covs), _lib.ptr(views), mv, _lib.ptr(images), _lib.ptr(intr),
                    n, H, W, float(max_depth), float(max_sigma), _lib.ptr(scratch), int(nb[0]), _lib.ptr(points),
                    _lib.ptr(colors), _lib.stream_ptr()), "point_cloud_emit")
        return points, colors

    def downsample(self, points, colors, voxel_size):
        """-> per occupied voxel (ascending key order): mean points, mean colors [V,3] fp32, counts [V] int32.  One host
        read: the voxel count."""
        self._cuda(points, colors)
        lib = _lib.load()
        N = int(points.shape[0])
        dev = points.device
        nb = np.zeros(1, np.int64)
        _lib.check(lib.nslam_point_cloud_voxel_scratch(N, nb.ctypes.data), "point_cloud_voxel_scratch")
        scratch = torch.empty(int(nb[0]), dtype=torch.uint8, device=dev)
        nv = torch.empty(1, dtype=torch.int32, device=dev)
        with _lib.fixed_stream():
            _lib.check(lib.nslam_point_cloud_voxel_sort(_lib.ptr(points), N, float(voxel_size), _lib.ptr(scratch), int(nb[0]),
                                                        _lib.ptr(nv), _lib.stream_ptr()), "point_cloud_voxel_sort")
            V = int(nv.item())
            out_p = torch.empty(V, 3, dtype=torch.float32, device=dev)
            out_c = torch.empty(V, 3, dtype=torch.float32, device=dev)
            out_n = torch.empty(V, dtype=torch.int32, device=dev)
            _lib.check(lib.nslam_point_cloud_voxel_reduce(_lib.ptr(points), _lib.ptr(colors), N, _lib.ptr(scratch), int(nb[0]),
                                                          V, _lib.ptr(out_p), _lib.ptr(out_c), _lib.ptr(out_n),
                                                          _lib.stream_ptr()), "point_cloud_voxel_reduce")
        return out_p, out_c, out_n


kernels = _CloudKernels()


def _check(name, t, dtype, shape):
    if not torch.is_tensor(t) or t.dtype != dtype or tuple(t.shape) != tuple(shape):
        got = (t.dtype, tuple(t.shape)) if torch.is_tensor(t) else type(t).__name__
        raise ValueError(f"{name} must be a {dtype} tensor of shape {tuple(shape)}, got {got}")
    if not t.is_contiguous():
        raise RuntimeError(f"{name} must be contiguous")


def _intrinsics(intrinsics, device):
    """fx, fy, cx, cy at full resolution (tensor, array or sequence) -> fp32 [4] on `device`, without a host round trip
    for a device tensor"""
    if torch.is_tensor(intrinsics):
        t = intrinsics.detach().to(device=device, dtype=torch.float32).reshape(-1).contiguous()
    else:
        a = np.ascontiguousarray(np.asarray(intrinsics, np.float32).reshape(-1))
        t = _lib.h2d(a, device) if device.type == "cuda" else torch.from_numpy(a.copy())
    if t.numel() != 4:
        raise ValueError(f"intrinsics must be fx, fy, cx, cy, got {t.numel()} values")
    return t


def build_point_cloud(packet, intrinsics, *, max_depth=6.0, max_depth_sigma=10.0, filter_thresh=None, min_views=2,
                      voxel_size=None):
    """The keyframes of a SLAM packet as one coloured point cloud -> PointCloud, or None when no point survives.

    packet: "cam0_poses" [n,7] fp32 cam_T_world (t, q_xyzw), "cam0_idepths_up" [n,H,W] fp32, "cam0_depths_cov_up"
    [n,H,W] fp32 or None (None = the "uniform" mask: no sigma test), "cam0_images" [n,3,H,W] u8 — contiguous, one device.
    intrinsics: fx, fy, cx, cy at full resolution (the reference: dsf * cam0_intrinsics[0]).
    A pixel is kept when 0 < d < max_depth, d = 1/idepth pushed past max_depth where sqrt(cov) >= max_depth_sigma.
    filter_thresh: also keep only pixels on which at least `min_views` (1..6) packet neighbours agree within
    filter_thresh (depth units), by droid_backends.depth_filter on the raw maps.  voxel_size: average the points of each
    occupied voxel floor(p / voxel_size) of the world-origin lattice (PointCloud.counts = points merged)."""
    poses, idepths = packet["cam0_poses"], packet["cam0_idepths_up"]
    covs, images = packet.get("cam0_depths_cov_up"), packet["cam0_images"]
    if not torch.is_tensor(idepths) or idepths.dim() != 3:
        raise ValueError("cam0_idepths_up must be a [n,H,W] tensor")
    n, H, W = idepths.shape
    _check("cam0_idepths_up", idepths, torch.float32, (n, H, W))
    _check("cam0_poses", poses, torch.float32, (n, 7))
    _check("cam0_images", images, torch.uint8, (n, 3, H, W))
    if covs is not None:
        _check("cam0_depths_cov_up", covs, torch.float32, (n, H, W))
    dev = idepths.device
    if any(t is not None and t.device != dev for t in (poses, covs, images)):
        raise ValueError("the packet's tensors must be on one device")
    if n * H * W > INT32_MAX:
        raise ValueError(f"{n} x {H} x {W} candidate pixels exceed int32")
    if voxel_size is not None and not (math.isfinite(float(voxel_size)) and float(voxel_size) > 0):
        raise ValueError(f"voxel_size must be positive and finite, got {voxel_size}")
    if filter_thresh is not None and (int(min_views) != min_views or not 1 <= int(min_views) <= 6):
        raise ValueError(f"min_views must be an integer in 1..6 (six neighbours), got {min_views}")
    intr = _intrinsics(intrinsics, dev)
    if n == 0 or H == 0 or W == 0:
        return None
    views = kernels.filter_counts(poses, idepths, intr, filter_thresh) if filter_thresh is not None else None
    points, colors = kernels.cloud(poses, idepths, covs, images, intr, max_depth, max_depth_sigma, views, min_views)
    if points.shape[0] == 0:
        return None
    if voxel_size is None:
        return PointCloud(points, colors)
    points, colors, counts = kernels.downsample(points, colors, voxel_size)
    return PointCloud(points, colors, counts) if points.shape[0] else None
