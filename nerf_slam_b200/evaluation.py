"""Reconstruction quality against ground truth on the GPU (csrc/recon_eval.cu, rules at its head; DESIGN §4f).

Dense-SLAM reconstructions are judged by their distance to the true surface: accuracy (reconstruction -> ground truth),
completion (ground truth -> reconstruction), precision / recall (completion ratio) / F-score at a threshold, and the
trajectory error of the camera centres.  Meshes are compared through area-uniform samples of their surfaces, point
clouds as they are; every nearest-neighbour distance is exact (a linear BVH, not an approximate grid).

    gt_vertices, gt_triangles = read_ply("gt_mesh.ply")
    m = reconstruction_metrics(fusion.build_mesh(0.5), (gt_vertices, gt_triangles), threshold=0.05)
    m["accuracy"], m["completion"], m["f_score"]
    trajectory_error(estimated_cam_T_world, gt_cam_T_world, align="sim3")["rmse"]

Ground truth given only as a mesh is culled for occlusion with depth rendered from it (mesh_render.MeshScene):

    gt = MeshScene((gt_vertices, gt_triangles))
    m = reconstruction_metrics(rec, gt_mesh, gt_mask=lambda p: visible(p, poses, intr, W, H,
                                                                          depths=gt.render(poses, intr, W, H).depth))

and the depth metric of dense neural SLAM compares rendered views of two meshes:

    mesh_depth_l1(fusion.build_mesh(0.5), (gt_vertices, gt_triangles), poses, intr, W, H)["depth_l1"]

Inputs: `TsdfMesh` (TsdfFusion / NerfFusion.build_mesh), `point_cloud.PointCloud`, a (vertices, triangles) pair or a
[N,3] point tensor.  Tensors must be CUDA tensors (there is no CPU path); numpy arrays are uploaded to the current
device.  `read_ply` and `trajectory_error` are host code."""
import math

import numpy as np
import torch

from . import _lib
from .point_cloud import PointCloud, _intrinsics

INT32_MAX = 2 ** 31 - 1
FIXED_POINT = 2.0 ** 32          # metric sums: integers of 2^-32 m
LEAF_SIZE = 4                    # reference points per BVH leaf


def _cuda_tensor(x, dtype, name):
    """a CUDA tensor of `dtype`, contiguous; numpy arrays / sequences go to the current device"""
    if torch.is_tensor(x):
        if not x.is_cuda:
            raise RuntimeError(f"{name} must be a CUDA tensor: the evaluation runs on sm_90a kernels, there is no CPU path")
        return x.detach().to(dtype).contiguous()
    np_dtype = {torch.float32: np.float32, torch.int32: np.int32}[dtype]
    a = np.ascontiguousarray(np.asarray(x), np_dtype)
    return _lib.h2d(a, torch.device("cuda", torch.cuda.current_device()))


def _points3(x, name):
    t = _cuda_tensor(x, torch.float32, name)
    if t.dim() != 2 or t.shape[1] != 3:
        raise ValueError(f"{name} must be [N,3], got {tuple(t.shape)}")
    if t.shape[0] > INT32_MAX:
        raise ValueError(f"{name}: {t.shape[0]} points exceed int32")
    return t


def _mesh_arrays(mesh):
    if hasattr(mesh, "vertices") and hasattr(mesh, "triangles"):
        V, T = mesh.vertices, mesh.triangles
    else:
        V, T = mesh
    V = _points3(V, "mesh vertices")
    T = _cuda_tensor(T, torch.int32, "mesh triangles")
    if T.dim() != 2 or T.shape[1] != 3:
        raise ValueError(f"mesh triangles must be [T,3], got {tuple(T.shape)}")
    if T.device != V.device:
        raise ValueError("mesh vertices and triangles must be on one device")
    return V, T


def sample_surface(mesh, n, seed=0, return_triangles=False):
    """`n` points sampled uniformly by area from a triangle mesh -> [n,3] fp32 device tensor (and with
    `return_triangles` the [n] int32 index of each point's triangle).  `mesh`: TsdfMesh or (vertices [V,3],
    triangles [T,3]).  Sample i depends on (seed, i) only: the same call gives the same bits.  Zero-area triangles are
    never chosen.  One host read (the total area, and whether the mesh is valid)."""
    lib = _lib.load()
    V, T = _mesh_arrays(mesh)
    n = int(n)
    if not 0 <= n <= INT32_MAX:
        raise ValueError(f"n must be in [0, 2^31), got {n}")
    nv, nt = int(V.shape[0]), int(T.shape[0])
    if nt == 0 or nv == 0:
        raise ValueError("the mesh has no triangle")
    dev = V.device
    scratch = torch.empty(_lib.query_size("nslam_eval_surface_scratch", nt), dtype=torch.uint8, device=dev)
    info = torch.empty(2, dtype=torch.int64, device=dev)
    points = torch.empty(n, 3, dtype=torch.float32, device=dev)
    tri = torch.empty(n, dtype=torch.int32, device=dev) if return_triangles else None
    with _lib.fixed_stream():
        _lib.check(lib.nslam_eval_surface_area(_lib.ptr(V), nv, _lib.ptr(T), nt, _lib.ptr(scratch), scratch.numel(),
                                               _lib.ptr(info), _lib.stream_ptr()), "eval_surface_area")
        total, flags = info.tolist()
        if flags & 1:
            raise ValueError("a triangle indexes a vertex outside the mesh")
        if flags & 2:
            raise ValueError("the mesh has non-finite vertex coordinates")
        if flags & 4:
            raise ValueError("the mesh is too large for the 64-bit area weights (2^22 m^2 in all)")
        if total <= 0:
            raise ValueError("the mesh has no area to sample")
        if n:
            _lib.check(lib.nslam_eval_sample_surface(_lib.ptr(V), _lib.ptr(T), nt, n, int(seed) % (1 << 64),
                                                     _lib.ptr(scratch), scratch.numel(), _lib.ptr(points), _lib.ptr(tri),
                                                     _lib.stream_ptr()), "eval_sample_surface")
    return (points, tri) if return_triangles else points


class PointIndex:
    """exact nearest-neighbour index over reference points [N,3] fp32 on the GPU: a linear BVH with leaf buckets of
    `leaf_size` (1..32) points.  It keeps its own sorted copy of the points."""

    def __init__(self, reference, leaf_size=LEAF_SIZE):
        lib = _lib.load()
        ref = _points3(reference, "reference")
        self.n, self.leaf_size, self.device = int(ref.shape[0]), int(leaf_size), ref.device
        if self.n == 0:
            raise ValueError("the reference has no point")
        if not 1 <= self.leaf_size <= 32:
            raise ValueError(f"leaf_size must be in 1..32, got {leaf_size}")
        self.bvh = torch.empty(_lib.query_size("nslam_eval_bvh_scratch", self.n, self.leaf_size), dtype=torch.uint8,
                               device=self.device)
        _lib.check(lib.nslam_eval_bvh_build(_lib.ptr(ref), self.n, self.leaf_size, _lib.ptr(self.bvh), self.bvh.numel(),
                                            _lib.stream_ptr()), "eval_bvh_build")

    def query(self, query, max_dist=math.inf, num_sms=0):
        """-> dist [M] fp32, idx [M] int64 of the nearest reference point strictly closer than max_dist (+inf / -1 when
        there is none).  dist = sqrt of the fp64 squared distance of the fp32 coordinates, rounded to fp32 once; ties
        go to the smaller reference index.  num_sms bounds the grid (0: every SM); no result depends on it."""
        lib = _lib.load()
        q = _points3(query, "query")
        if q.device != self.device:
            raise ValueError("query and reference must be on one device")
        if not float(max_dist) > 0:
            raise ValueError(f"max_dist must be > 0, got {max_dist}")
        m = int(q.shape[0])
        dist = torch.empty(m, dtype=torch.float32, device=self.device)
        idx = torch.empty(m, dtype=torch.int64, device=self.device)
        if m == 0:
            return dist, idx
        scratch = torch.empty(_lib.query_size("nslam_eval_nearest_scratch", m), dtype=torch.uint8, device=self.device)
        _lib.check(lib.nslam_eval_nearest(_lib.ptr(self.bvh), self.bvh.numel(), self.n, self.leaf_size, _lib.ptr(q), m,
                                          float(max_dist), int(num_sms), _lib.ptr(scratch), scratch.numel(), _lib.ptr(dist),
                                          _lib.ptr(idx), _lib.stream_ptr()), "eval_nearest")
        return dist, idx


def nearest(query, reference, max_dist=math.inf, leaf_size=LEAF_SIZE, num_sms=0):
    """exact nearest neighbour in `reference` [N,3] of every `query` point [M,3] -> (dist [M] fp32, idx [M] int64), device
    tensors; +inf and -1 where no reference point is strictly closer than max_dist (PointIndex.query)"""
    return PointIndex(reference, leaf_size).query(query, max_dist, num_sms)


def visible(points, cam_T_world, intrinsics, width, height, depths=None, depth_tol=0.05, near=0.0, far=math.inf):
    """-> bool [N] device mask of the points [N,3] seen by at least one camera: cam_T_world [n,7] (t, q_xyzw), pinhole
    intrinsics fx, fy, cx, cy for width x height images.  Seen: near < z <= far, the nearest pixel lies in the image and,
    with depth maps [n,H,W] (metres), z <= depth + depth_tol there, a depth <= 0 meaning no measurement (not tested).
    The usual protocol to cull ground truth to what the cameras saw."""
    lib = _lib.load()
    P = _points3(points, "points")
    poses = _cuda_tensor(cam_T_world, torch.float32, "cam_T_world")
    if poses.dim() != 2 or poses.shape[1] != 7:
        raise ValueError(f"cam_T_world must be [n,7] (t, q_xyzw), got {tuple(poses.shape)}")
    W, H = int(width), int(height)
    if W <= 0 or H <= 0:
        raise ValueError(f"image size must be positive, got {W} x {H}")
    n = int(poses.shape[0])
    if depths is not None:
        depths = _cuda_tensor(depths, torch.float32, "depths")
        if tuple(depths.shape) != (n, H, W):
            raise ValueError(f"depths must be [{n},{H},{W}], got {tuple(depths.shape)}")
    if any(t is not None and t.device != P.device for t in (poses, depths)):
        raise ValueError("points, poses and depths must be on one device")
    intr = _intrinsics(intrinsics, P.device)
    mask = torch.empty(P.shape[0], dtype=torch.bool, device=P.device)
    _lib.check(lib.nslam_eval_visible(_lib.ptr(P), int(P.shape[0]), _lib.ptr(poses), n, _lib.ptr(intr), W, H,
                                      _lib.ptr(depths), float(depth_tol), float(near), float(far), _lib.ptr(mask),
                                      _lib.stream_ptr()), "eval_visible")
    return mask


def _as_points(x, n_samples, seed, name):
    if isinstance(x, PointCloud):
        return _points3(x.points, name)
    if hasattr(x, "vertices") and hasattr(x, "triangles") or isinstance(x, tuple) and len(x) == 2:
        return sample_surface(x, n_samples, seed)
    return _points3(x, name)


def _metric_sums(dist, max_dist, threshold, out):
    _lib.check(_lib.load().nslam_eval_reduce(_lib.ptr(dist), int(dist.shape[0]), float(max_dist), float(threshold),
                                             _lib.ptr(out), _lib.stream_ptr()), "eval_reduce")


def reconstruction_metrics(reconstruction, ground_truth, threshold=0.05, n_samples=200_000, max_dist=1.0, seed=0,
                           gt_mask=None, leaf_size=LEAF_SIZE):
    """Accuracy, completion and F-score of a reconstruction against ground truth -> dict.

    Each side is a TsdfMesh or (vertices, triangles) pair (sampled: `n_samples` points, the reconstruction with `seed`,
    the ground truth with seed + 1), a PointCloud or a [N,3] tensor (used as is).  gt_mask: a bool [M] mask of the
    ground-truth points (after sampling) or a function of them returning one, e.g. `lambda p: visible(p, ...)`.

      accuracy    mean over reconstruction points of min(d(p, GT), max_dist)
      completion  mean over ground-truth points of min(d(g, reconstruction), max_dist)
      chamfer_l1  (accuracy + completion) / 2
      precision   share of reconstruction points with d < threshold;  recall (completion ratio): same for GT points
      f_score     2 precision recall / (precision + recall), 0 when both are 0
    Distances are clamped at max_dist (metres, finite) in the means, so a far outlier counts max_dist; points with no
    neighbour within max_dist are counted as unmatched.  The sums are 64-bit fixed-point integers of 2^-32 m
    (`accuracy_fixed`, `completion_fixed`): the same bits in every run.  One host read for the ground-truth mask, one for
    the six sums (and one per sampled mesh)."""
    _lib.load()
    if not (math.isfinite(float(max_dist)) and float(max_dist) > 0):
        raise ValueError(f"max_dist must be positive and finite, got {max_dist}")
    rec = _as_points(reconstruction, n_samples, seed, "reconstruction")
    gt = _as_points(ground_truth, n_samples, seed + 1, "ground_truth")
    if gt_mask is not None:
        m = gt_mask(gt) if callable(gt_mask) else gt_mask
        if not torch.is_tensor(m) or m.dtype != torch.bool or tuple(m.shape) != (gt.shape[0],):
            raise ValueError(f"gt_mask must be a bool tensor of shape ({gt.shape[0]},)")
        gt = gt[m.to(gt.device)].contiguous()
    n_rec, n_gt = int(rec.shape[0]), int(gt.shape[0])
    if n_rec == 0 or n_gt == 0:
        raise ValueError(f"nothing to compare: {n_rec} reconstruction and {n_gt} ground-truth points")
    if max(n_rec, n_gt) * float(max_dist) >= 2.0 ** 31:
        raise ValueError("points x max_dist must stay below 2^31 for the 64-bit fixed-point sums")
    sums = torch.empty(2, 3, dtype=torch.int64, device=rec.device)
    with _lib.fixed_stream():
        d_acc, _ = nearest(rec, gt, max_dist, leaf_size)
        _metric_sums(d_acc, max_dist, threshold, sums[0])
        d_comp, _ = nearest(gt, rec, max_dist, leaf_size)
        _metric_sums(d_comp, max_dist, threshold, sums[1])
        (s_acc, in_acc, miss_acc), (s_comp, in_comp, miss_comp) = sums.tolist()
    accuracy = s_acc / FIXED_POINT / n_rec
    completion = s_comp / FIXED_POINT / n_gt
    precision, recall = in_acc / n_rec, in_comp / n_gt
    f_score = 2 * precision * recall / (precision + recall) if precision + recall > 0 else 0.0
    return {"accuracy": accuracy, "completion": completion, "chamfer_l1": 0.5 * (accuracy + completion),
            "precision": precision, "recall": recall, "f_score": f_score, "threshold": float(threshold),
            "max_dist": float(max_dist), "n_reconstruction": n_rec, "n_ground_truth": n_gt,
            "unmatched_reconstruction": miss_acc, "unmatched_ground_truth": miss_comp,
            "accuracy_fixed": s_acc, "completion_fixed": s_comp}


def mesh_depth_l1(reconstruction, ground_truth, cam_T_world, intrinsics, width, height, max_dist=1.0, near=0.0,
                  far=math.inf):
    """Depth L1 between rendered views of two meshes -> dict: both are rendered (mesh_render.MeshScene, back faces
    included) at the views cam_T_world [n,7] (t, q_xyzw) with intrinsics fx, fy, cx, cy at width x height, and

      depth_l1        mean over the pixels both meshes hit of min(|d_rec - d_gt|, max_dist), metres
      gt_hits         pixels the ground truth hits;  both_hits: pixels both hit
      missing         pixels only the ground truth hits;  extra: pixels only the reconstruction hits
      depth_l1_fixed  the sum of min(|d_rec - d_gt|, max_dist) as a 64-bit integer of 2^-32 m (nslam_eval_reduce):
                      the same bits in every run
    Each side is a TsdfMesh / NeRF mesh, a (vertices, triangles) pair or a MeshScene built before.  |d_rec - d_gt| is
    the fp32 difference of the fp32 depths.  Views go in chunks of at most 2^31 / max_dist pixels (the fixed-point
    sum's bound).  One host read (the sums), plus one per mesh given as a mesh (its build's validity flags)."""
    from .mesh_render import MeshScene
    md = float(max_dist)
    if not (math.isfinite(md) and md > 0):
        raise ValueError(f"max_dist must be positive and finite, got {max_dist}")
    rec = reconstruction if isinstance(reconstruction, MeshScene) else MeshScene(reconstruction)
    gt = ground_truth if isinstance(ground_truth, MeshScene) else MeshScene(ground_truth)
    if rec.device != gt.device:
        raise ValueError("reconstruction and ground truth must be on one device")
    poses = _cuda_tensor(cam_T_world, torch.float32, "cam_T_world")
    if poses.dim() != 2 or poses.shape[1] != 7:
        raise ValueError(f"cam_T_world must be [n,7] (t, q_xyzw), got {tuple(poses.shape)}")
    W, H, n = int(width), int(height), int(poses.shape[0])
    if W <= 0 or H <= 0 or n == 0:
        raise ValueError(f"need at least one view of positive size, got {n} views of {W} x {H}")
    per_chunk = min(INT32_MAX, int(math.ceil(2.0 ** 31 / md)) - 1) // (H * W)
    if per_chunk < 1:
        raise ValueError(f"one {W} x {H} view exceeds the fixed-point sum's 2^31 / max_dist pixels")
    chunks = range(0, n, per_chunk)
    sums = torch.empty(len(chunks), 3, dtype=torch.int64, device=rec.device)
    counts = torch.zeros(4, dtype=torch.int64, device=rec.device)
    with _lib.fixed_stream():
        for c, k0 in enumerate(chunks):
            p = poses[k0:k0 + per_chunk]
            a = rec.render(p, intrinsics, W, H, near, far)
            b = gt.render(p, intrinsics, W, H, near, far)
            hit_rec, hit_gt = a.triangle >= 0, b.triangle >= 0
            both = hit_rec & hit_gt
            diff = torch.where(both, (a.depth - b.depth).abs(), torch.zeros((), device=rec.device)).reshape(-1)
            _metric_sums(diff, md, md, sums[c])
            counts += torch.stack([hit_gt.sum(), both.sum(), (hit_gt & ~hit_rec).sum(), (hit_rec & ~hit_gt).sum()])
        total = torch.cat([sums[:, 0].sum().reshape(1), counts]).tolist()
    s, gt_hits, both_hits, missing, extra = total
    return {"depth_l1": s / FIXED_POINT / both_hits if both_hits else math.nan, "gt_hits": gt_hits,
            "both_hits": both_hits, "missing": missing, "extra": extra, "pixels": n * H * W, "max_dist": md,
            "depth_l1_fixed": s}


# ---------------------------------------------------------------------------------------------------------------- PLY
_PLY_DTYPES = {"char": "i1", "int8": "i1", "uchar": "u1", "uint8": "u1", "short": "i2", "int16": "i2", "ushort": "u2",
               "uint16": "u2", "int": "i4", "int32": "i4", "uint": "u4", "uint32": "u4", "float": "f4", "float32": "f4",
               "double": "f8", "float64": "f8"}


def _ply_header(data):
    end = data.find(b"end_header")
    if not data.startswith(b"ply") or end < 0:
        raise ValueError("not a PLY file")
    body = data.index(b"\n", end) + 1
    fmt, elements = None, []
    for line in data[:end].decode("ascii").splitlines()[1:]:
        w = line.split()
        if not w or w[0] in ("comment", "obj_info"):
            continue
        if w[0] == "format":
            fmt = w[1]
        elif w[0] == "element":
            elements.append((w[1], int(w[2]), []))
        elif w[0] == "property":
            if w[1] == "list":
                elements[-1][2].append((w[4], _PLY_DTYPES[w[2]], _PLY_DTYPES[w[3]]))
            else:
                elements[-1][2].append((w[2], _PLY_DTYPES[w[1]], None))
    if fmt not in ("ascii", "binary_little_endian", "binary_big_endian"):
        raise ValueError(f"unsupported PLY format {fmt!r}")
    return fmt, elements, body


def _ply_binary_element(buf, pos, count, props, endian):
    """-> ({name: array or list of arrays}, new position)"""
    if all(p[2] is None for p in props):
        dt = np.dtype([(n, endian + t) for n, t, _ in props])
        rec = np.frombuffer(buf, dt, count, pos)
        return {n: rec[n] for n, _, _ in props}, pos + count * dt.itemsize
    if len(props) == 1:                                    # one list, every row a triangle: one structured read
        name, ct, it = props[0]
        dt = np.dtype([("n", endian + ct), ("v", endian + it, (3,))])
        if pos + count * dt.itemsize <= len(buf):
            rec = np.frombuffer(buf, dt, count, pos)
            if np.all(rec["n"] == 3):
                return {name: rec["v"]}, pos + count * dt.itemsize
    out = {n: [] for n, _, _ in props}
    for _ in range(count):
        for n, t, it in props:
            if it is None:
                out[n].append(np.frombuffer(buf, endian + t, 1, pos)[0])
                pos += np.dtype(t).itemsize
            else:
                k = int(np.frombuffer(buf, endian + t, 1, pos)[0])
                pos += np.dtype(t).itemsize
                out[n].append(np.frombuffer(buf, endian + it, k, pos))
                pos += k * np.dtype(it).itemsize
    return out, pos


def _ply_ascii_element(tokens, pos, count, props):
    if all(p[2] is None for p in props):
        k = len(props)
        a = np.asarray(tokens[pos:pos + count * k], np.float64).reshape(count, k)
        return {n: a[:, i].astype(t) for i, (n, t, _) in enumerate(props)}, pos + count * k
    out = {n: [] for n, _, _ in props}
    for _ in range(count):
        for n, t, it in props:
            if it is None:
                out[n].append(float(tokens[pos]))
                pos += 1
            else:
                k = int(tokens[pos])
                out[n].append(np.asarray(tokens[pos + 1:pos + 1 + k], np.int64))
                pos += 1 + k
    return out, pos


def _triangles(faces):
    """face vertex lists (an [F,3] array, or a list of index arrays: polygons fan-triangulated) -> [T,3] int32"""
    if isinstance(faces, np.ndarray) and faces.ndim == 2:
        return np.ascontiguousarray(faces, np.int32)
    tris = [np.stack([np.full(len(f) - 2, f[0]), f[1:-1], f[2:]], 1) for f in faces if len(f) >= 3]
    return np.concatenate(tris).astype(np.int32) if tris else np.zeros((0, 3), np.int32)


def read_ply(path, return_colors=False):
    """vertices [V,3] float32 and triangles [T,3] int32 (None when the file has no face element) of a PLY file: binary
    little- or big-endian or ASCII, x / y / z vertex properties of any numeric type, faces as a `vertex_indices` (or
    `vertex_index`) list, polygons fan-triangulated.  What TsdfMesh.write_ply / PointCloud.write_ply write, and the usual
    ground-truth meshes and scans.  Other elements and properties are skipped.  With `return_colors`, also the vertex
    colours [V,3] float32 in [0,1] from red / green / blue (integer types divided by their maximum, 255 for uchar;
    floats as stored), None when the file has none."""
    with open(path, "rb") as f:
        data = f.read()
    fmt, elements, body = _ply_header(data)
    endian = {"binary_little_endian": "<", "binary_big_endian": ">"}.get(fmt)
    tokens = data[body:].split() if fmt == "ascii" else None
    pos = body if endian else 0
    vertices = triangles = colors = None
    for name, count, props in elements:
        if endian:
            vals, pos = _ply_binary_element(data, pos, count, props, endian)
        else:
            vals, pos = _ply_ascii_element(tokens, pos, count, props)
        if name == "vertex":
            if not all(k in vals for k in "xyz"):
                raise ValueError("the vertex element has no x, y, z")
            vertices = np.stack([np.asarray(vals[k], np.float32) for k in "xyz"], 1)
            if all(k in vals for k in ("red", "green", "blue")):
                types = {n: t for n, t, _ in props}
                colors = np.stack([_unit_color(vals[k], types[k]) for k in ("red", "green", "blue")], 1)
        elif name == "face":
            key = "vertex_indices" if "vertex_indices" in vals else "vertex_index"
            if key not in vals:
                raise ValueError("the face element has no vertex_indices list")
            triangles = _triangles(vals[key])
    if vertices is None:
        raise ValueError("the PLY file has no vertex element")
    return (vertices, triangles, colors) if return_colors else (vertices, triangles)


def _unit_color(values, ply_type):
    """a colour channel on [0,1]: integers over their type's maximum, floats as stored"""
    dt = np.dtype(ply_type)
    a = np.asarray(values, np.float64)
    if dt.kind in "iu":
        return (a / np.iinfo(dt).max).astype(np.float32)
    return a.astype(np.float32)


# ------------------------------------------------------------------------------------------------------ trajectory error
def _camera_centres(poses):
    """cam_T_world [N,7] (t, q_xyzw; q normalised here) or [N,4,4] -> camera centres -R^T t [N,3], fp64"""
    P = np.asarray(poses.detach().cpu().numpy() if torch.is_tensor(poses) else poses, np.float64)
    if P.ndim == 2 and P.shape[1] == 7:
        t = P[:, :3]
        q = P[:, 3:] / np.linalg.norm(P[:, 3:], axis=1, keepdims=True)
        x, y, z, w = q.T
        R = np.stack([1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w),
                      2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w),
                      2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)], 1).reshape(-1, 3, 3)
    elif P.ndim == 3 and P.shape[1:] == (4, 4):
        R, t = P[:, :3, :3], P[:, :3, 3]
    else:
        raise ValueError(f"poses must be [N,7] (t, q_xyzw) or [N,4,4] cam_T_world, got {P.shape}")
    return -np.einsum("nji,nj->ni", R, t)


def umeyama(src, dst, with_scale=True):
    """closed-form least-squares similarity (Umeyama 1991) with dst ~ s R src + t, fp64 -> (s, R [3,3], t [3])"""
    src, dst = np.asarray(src, np.float64), np.asarray(dst, np.float64)
    mu_s, mu_d = src.mean(0), dst.mean(0)
    X, Y = src - mu_s, dst - mu_d
    U, D, Vt = np.linalg.svd(Y.T @ X / len(src))
    S = np.eye(3)
    if np.linalg.det(U) * np.linalg.det(Vt) < 0:
        S[2, 2] = -1.0
    R = U @ S @ Vt
    var = (X ** 2).sum() / len(src)
    s = float(np.trace(np.diag(D) @ S) / var) if with_scale and var > 0 else 1.0
    return s, R, mu_d - s * R @ mu_s


def trajectory_error(est, gt, align="sim3"):
    """absolute trajectory error of the camera centres of `est` against `gt` (cam_T_world, [N,7] t q_xyzw or [N,4,4],
    frame i against frame i) after aligning est to gt: "sim3" (rotation, translation, scale), "se3" (no scale) or
    "none" -> {rmse, mean, median, max, scale, n} in gt's units.  Host code in fp64."""
    ce, cg = _camera_centres(est), _camera_centres(gt)
    if ce.shape != cg.shape or len(ce) == 0:
        raise ValueError(f"est and gt must hold the same number (> 0) of poses, got {len(ce)} and {len(cg)}")
    if align == "none":
        s, R, t = 1.0, np.eye(3), np.zeros(3)
    elif align in ("sim3", "se3"):
        s, R, t = umeyama(ce, cg, with_scale=align == "sim3")
    else:
        raise ValueError(f"align must be 'sim3', 'se3' or 'none', not {align!r}")
    e = np.linalg.norm(s * ce @ R.T + t - cg, axis=1)
    return {"rmse": float(np.sqrt(np.mean(e ** 2))), "mean": float(e.mean()), "median": float(np.median(e)),
            "max": float(e.max()), "scale": float(s), "n": int(len(e))}
