"""Aligning a reconstruction to ground truth on the GPU (csrc/registration.cu, rules at its head; DESIGN §4i).

A reconstruction built from SLAM poses lives in the SLAM frame: a monocular map has an arbitrary scale and its poses
drift.  The usual neural-SLAM protocol first fits a similarity between the estimated and true trajectories, then refines
it with ICP between the reconstruction and the true surface, and only then scores accuracy and completion:

    init = trajectory_alignment(est_cam_T_world, gt_cam_T_world, "sim3")
    r = icp(slam_cloud, gt_mesh, init=init, with_scale=True)
    m = evaluation.reconstruction_metrics(transform(slam_cloud, r.transform), gt_mesh)

The correspondences are exact nearest neighbours (evaluation.PointIndex, built once over the target samples); the
Gauss-Newton sums are 64-bit fixed-point integers, so every run gives the same bits, and the fp64 solve and update run on
the host, one 38-integer read per iteration.  Tensors must be CUDA tensors (there is no CPU path); numpy arrays are
uploaded to the current device."""
import ctypes
import math
from dataclasses import dataclass, field

import numpy as np
import torch

from . import _lib
from .evaluation import _as_points, _camera_centres, _mesh_arrays, _points3, PointIndex, sample_surface, umeyama
from .point_cloud import PointCloud
from .tsdf_fusion import TsdfMesh

FIXED = 2.0 ** 27                # Gauss-Newton sums: integers of 2^-27
N_SUMS = 38
METRICS = ("point_to_plane", "point_to_point")
PIVOT_RTOL = 1e-12               # a Cholesky pivot below this share of H's largest diagonal entry is degenerate


def _is_mesh(x):
    return hasattr(x, "vertices") and hasattr(x, "triangles") or isinstance(x, tuple) and len(x) == 2


# ------------------------------------------------------------------------------------------------------------ host maths
def rodrigues(w):
    """exp([w]x): the rotation by |w| radians about w / |w| (fp64 [3,3])"""
    w = np.asarray(w, np.float64)
    th = math.sqrt(float(w @ w))
    K = np.array([[0.0, -w[2], w[1]], [w[2], 0.0, -w[0]], [-w[1], w[0], 0.0]])
    if th < 1e-12:
        return np.eye(3) + K
    return np.eye(3) + (math.sin(th) / th) * K + ((1.0 - math.cos(th)) / (th * th)) * (K @ K)


def compose(s, R, t):
    """the 4x4 fp64 matrix of p -> s R p + t"""
    T = np.eye(4)
    T[:3, :3] = float(s) * np.asarray(R, np.float64)
    T[:3, 3] = np.asarray(t, np.float64)
    return T


def decompose(T, name="transform"):
    """a 4x4 similarity -> (s, R, t); refuses anything else (non-finite, a bottom row other than 0 0 0 1, a 3x3 block
    that is not s times a rotation with s > 0)"""
    M = np.asarray(T.detach().cpu().numpy() if torch.is_tensor(T) else T, np.float64)
    if M.shape != (4, 4) or not np.all(np.isfinite(M)):
        raise ValueError(f"{name} must be a finite 4x4 matrix")
    if not np.allclose(M[3], [0.0, 0.0, 0.0, 1.0], rtol=0.0, atol=1e-9):
        raise ValueError(f"{name} must have the bottom row 0 0 0 1")
    det = float(np.linalg.det(M[:3, :3]))
    if not det > 0:
        raise ValueError(f"{name} is not a similarity: det = {det}")
    s = det ** (1.0 / 3.0)
    R = M[:3, :3] / s
    if np.abs(R.T @ R - np.eye(3)).max() > 1e-6:
        raise ValueError(f"{name} is not a similarity: its 3x3 block is not a scaled rotation")
    return s, R, M[:3, 3].copy()


def target_frame(lo, hi):
    """the normalisation of the correspondence terms from the target's box (fp32 min / max): its centre c = (lo + hi) / 2
    and half its diagonal L = sqrt((dx^2 + dy^2) + dz^2) / 2, fp64"""
    lo, hi = [float(v) for v in lo], [float(v) for v in hi]
    c = [(a + b) * 0.5 for a, b in zip(lo, hi)]
    d = [b - a for a, b in zip(lo, hi)]
    return c, math.sqrt((d[0] * d[0] + d[1] * d[1]) + d[2] * d[2]) * 0.5


def unpack_sums(sums):
    """38 integers of nslam_reg_accumulate -> H [7,7] and g [7] (fp64, 2^-27 units removed), the squared-residual sum
    (normalised units), the count and the flags"""
    v = [int(x) for x in sums]
    H = np.zeros((7, 7))
    k = 0
    for a in range(7):
        for b in range(a, 7):
            H[a, b] = H[b, a] = v[k] / FIXED
            k += 1
    return H, np.array(v[28:35], np.float64) / FIXED, v[35] / FIXED, v[36], v[37]


def gauss_newton_step(sums, with_scale):
    """solve H x = -g in fp64 by Cholesky over (omega, tau[, sigma]) -> x [7] (sigma = 0 without scale), or None when the
    system is degenerate: fewer correspondences than unknowns, or a pivot that is not positive or below PIVOT_RTOL of
    H's largest diagonal entry"""
    H, g, _, count, _ = unpack_sums(sums)
    dof = 7 if with_scale else 6
    if count < dof:
        return None
    A = H[:dof, :dof]
    try:
        Lc = np.linalg.cholesky(A)
    except np.linalg.LinAlgError:
        return None
    if not np.all(np.diag(Lc) ** 2 > PIVOT_RTOL * np.max(np.diag(A))):
        return None
    x = np.zeros(7)
    x[:dof] = np.linalg.solve(Lc.T, np.linalg.solve(Lc, -g[:dof]))
    return x


def apply_step(s, R, t, x, c, L):
    """the update of the normalised step x = (omega, tau, sigma): s <- e^sigma s, R <- exp([omega]x) R,
    t <- e^sigma R_d (t - c) + c + L tau (the step acts on (p - c) / L)"""
    Rd = rodrigues(x[:3])
    e = math.exp(x[6])
    c = np.asarray(c, np.float64)
    return e * s, Rd @ R, e * (Rd @ (np.asarray(t, np.float64) - c)) + c + L * x[3:6]


# ----------------------------------------------------------------------------------------------------------------- kernels
def _sim3(s, R, t):
    return (ctypes.c_double * 13)(float(s), *[float(v) for v in np.asarray(R, np.float64).reshape(-1)],
                                  *[float(v) for v in np.asarray(t, np.float64)])


def _transform_points(P, s, R, t, direction=False):
    out = torch.empty_like(P)
    _lib.check(_lib.load().nslam_reg_transform(_lib.ptr(P), int(P.shape[0]), _sim3(s, R, t), int(direction),
                                               _lib.ptr(out), _lib.stream_ptr()), "reg_transform")
    return out


class _Correspondences:
    """the BVH over the target and the buffers of one ICP iteration (transform, nearest, sums), allocated once"""

    def __init__(self, source, target, normals, frame):
        self.src, self.tgt, self.nrm = source, target, normals
        self.index = PointIndex(target)
        n, dev = int(source.shape[0]), source.device
        self.moved = torch.empty_like(source)
        self.dist = torch.empty(n, dtype=torch.float32, device=dev)
        self.idx = torch.empty(n, dtype=torch.int64, device=dev)
        self.scratch = torch.empty(_lib.query_size("nslam_eval_nearest_scratch", n), dtype=torch.uint8, device=dev)
        self.sums = torch.empty(N_SUMS, dtype=torch.int64, device=dev)
        self.frame = (ctypes.c_double * 4)(*frame[0], frame[1])

    def sums_at(self, s, R, t, max_dist, point_to_point, with_scale):
        """-> the 38 integers at the transform (s, R, t), correspondences closer than max_dist (one host read)"""
        lib, ix, n = _lib.load(), self.index, int(self.src.shape[0])
        _lib.check(lib.nslam_reg_transform(_lib.ptr(self.src), n, _sim3(s, R, t), 0, _lib.ptr(self.moved),
                                           _lib.stream_ptr()), "reg_transform")
        _lib.check(lib.nslam_eval_nearest(_lib.ptr(ix.bvh), ix.bvh.numel(), ix.n, ix.leaf_size, _lib.ptr(self.moved), n,
                                          float(max_dist), 0, _lib.ptr(self.scratch), self.scratch.numel(),
                                          _lib.ptr(self.dist), _lib.ptr(self.idx), _lib.stream_ptr()), "eval_nearest")
        _lib.check(lib.nslam_reg_accumulate(_lib.ptr(self.moved), n, _lib.ptr(self.idx), _lib.ptr(self.tgt),
                                            _lib.ptr(None if point_to_point else self.nrm), int(self.tgt.shape[0]),
                                            self.frame, int(point_to_point), int(with_scale), 0, _lib.ptr(self.sums),
                                            _lib.stream_ptr()), "reg_accumulate")
        v = self.sums.tolist()
        if v[37] & 1:
            raise RuntimeError("registration: a correspondence index outside the target")
        if v[37] & 2:
            raise ValueError("registration: a correspondence term is out of bounds (non-unit target normals?)")
        return v


def _target(target, metric, n_samples, seed):
    """-> target points [M,3] and, for point-to-plane, their unit face normals [M,3] (a device flag word to check)"""
    if not _is_mesh(target) or isinstance(target, PointCloud):
        if metric == "point_to_plane":
            raise ValueError("point-to-plane ICP needs a mesh target (its face normals); give a mesh or use "
                             "metric='point_to_point'")
        return _as_points(target, n_samples, seed, "target"), None, None
    pts, tri = sample_surface(target, n_samples, seed, return_triangles=True)
    if metric == "point_to_point":
        return pts, None, None
    V, T = _mesh_arrays(target)
    nrm = torch.empty_like(pts)
    flags = torch.empty(1, dtype=torch.int64, device=pts.device)
    _lib.check(_lib.load().nslam_reg_face_normals(_lib.ptr(V), int(V.shape[0]), _lib.ptr(T), int(T.shape[0]),
                                                  _lib.ptr(tri), int(pts.shape[0]), _lib.ptr(nrm), _lib.ptr(flags),
                                                  _lib.stream_ptr()), "reg_face_normals")
    return pts, nrm, flags


def _prepare(source, target, metric, n_samples, seed, max_corr_dist):
    """-> source and target points, target normals, the frame (c, L) and the correspondence distances; validates"""
    if metric not in METRICS:
        raise ValueError(f"metric must be one of {METRICS}, not {metric!r}")
    dists = [float(d) for d in (max_corr_dist if np.ndim(max_corr_dist) else [max_corr_dist])]
    if not dists:
        raise ValueError("max_corr_dist needs at least one distance")
    src = _as_points(source, n_samples, seed, "source")
    tgt, nrm, nflags = _target(target, metric, n_samples, seed + 1)
    if src.device != tgt.device:
        raise ValueError("source and target must be on one device")
    if src.shape[0] == 0 or tgt.shape[0] == 0:
        raise ValueError(f"nothing to register: {src.shape[0]} source and {tgt.shape[0]} target points")
    lo, hi = torch.aminmax(tgt, dim=0)
    checks = torch.stack([torch.isfinite(src).all().to(torch.float64), torch.isfinite(tgt).all().to(torch.float64),
                          (nflags[0] if nflags is not None else torch.zeros((), dtype=torch.int64,
                                                                            device=src.device)).to(torch.float64)])
    info = torch.cat([checks, lo.to(torch.float64), hi.to(torch.float64)]).tolist()
    if not info[0]:
        raise ValueError("the source has non-finite points")
    if not info[1]:
        raise ValueError("the target has non-finite points")
    if int(info[2]):
        raise ValueError("the target mesh has a degenerate sampled triangle (no face normal)")
    frame = target_frame(info[3:6], info[6:9])
    if not frame[1] > 0:
        raise ValueError("the target has no extent (all points coincide)")
    for d in dists:
        if not 0 < d <= frame[1]:
            raise ValueError(f"max_corr_dist {d} must lie in (0, {frame[1]:.6g}], half the target's box diagonal")
    return src, tgt, nrm, frame, dists


@dataclass
class IcpResult:
    """the result of icp(): transform (4x4 fp64, source -> target) = [s R | t]; fitness (share of source points with a
    correspondence within the last max_corr_dist) and inlier_rmse (metres, over those) from one final pass, as Open3D's
    registration_icp reports them; iterations (Gauss-Newton steps taken), converged (the last stage's step fell below
    tol), degenerate (a system could not be solved: the transform is the one before it); history: one dict per
    iteration (stage, max_corr_dist, correspondences, rmse in metres at the iteration's transform, step = |x|inf or None,
    and the 38 integer sums)"""
    transform: np.ndarray
    scale: float
    rotation: np.ndarray
    translation: np.ndarray
    fitness: float
    inlier_rmse: float
    iterations: int
    converged: bool
    degenerate: bool
    history: list = field(default_factory=list)


def _fit(count, sse_fixed, n, L):
    return count / n, (L * math.sqrt(sse_fixed / FIXED / count) if count else 0.0)


def icp(source, target, init=None, metric="point_to_plane", with_scale=False, max_corr_dist=(0.2, 0.1, 0.05),
        max_iters=30, tol=1e-7, n_samples=200_000, seed=0):
    """Iterative closest point from `source` to `target` -> IcpResult.

    source: a mesh (TsdfMesh or (vertices, triangles): `n_samples` points sampled with `seed`), a PointCloud or [N,3]
    points (used as they are).  target: a mesh, sampled with seed + 1; point-to-point also takes a cloud or points.
    init: a 4x4 similarity (default identity).  metric: "point_to_plane" (the target's face normals at its samples) or
    "point_to_point".  with_scale adds the scale (Sim3).  Each entry of max_corr_dist (metres, in (0, L], L half the
    target's box diagonal) is one coarse-to-fine stage of at most max_iters Gauss-Newton steps; a stage ends when the
    normalised step's largest component is below tol.  The target's BVH is built once; each iteration is transform,
    nearest, accumulate and one host read of the 38 integer sums."""
    if metric not in METRICS:
        raise ValueError(f"metric must be one of {METRICS}, not {metric!r}")
    if int(max_iters) < 1:
        raise ValueError(f"max_iters must be >= 1, got {max_iters}")
    if not float(tol) >= 0:
        raise ValueError(f"tol must be >= 0, got {tol}")
    s, R, t = decompose(init, "init") if init is not None else (1.0, np.eye(3), np.zeros(3))
    _lib.load()
    p2p = metric == "point_to_point"
    with _lib.fixed_stream():
        src, tgt, nrm, frame, dists = _prepare(source, target, metric, n_samples, seed, max_corr_dist)
        c, L = frame
        corr = _Correspondences(src, tgt, nrm, frame)
        history, iterations, converged, degenerate = [], 0, False, False
        for stage, d in enumerate(dists):
            converged = False
            for _ in range(int(max_iters)):
                sums = corr.sums_at(s, R, t, d, p2p, with_scale)
                x = gauss_newton_step(sums, with_scale)
                count = sums[36]
                history.append({"stage": stage, "max_corr_dist": d, "correspondences": count,
                                "rmse": _fit(count, sums[35], 1, L)[1], "step": None if x is None else float(np.abs(x).max()),
                                "sums": sums})
                if x is None:
                    degenerate = True
                    break
                s, R, t = apply_step(s, R, t, x, c, L)
                iterations += 1
                if np.abs(x).max() < tol:
                    converged = True
                    break
            if degenerate:
                break
        final = corr.sums_at(s, R, t, dists[-1], True, False)
    fitness, rmse = _fit(final[36], final[35], int(src.shape[0]), L)
    return IcpResult(compose(s, R, t), float(s), R, np.asarray(t, np.float64), fitness, rmse, iterations, converged,
                     degenerate, history)


def evaluate_registration(source, target, transform, max_corr_dist, n_samples=200_000, seed=0):
    """the final pass of icp() alone -> {fitness, inlier_rmse, correspondences}: `source` (sampled with `seed` when a
    mesh) moved by the 4x4 similarity `transform`, matched to `target` (a mesh sampled with seed + 1, a cloud or points)
    within max_corr_dist (metres, in (0, L])"""
    _lib.load()
    s, R, t = decompose(transform)
    with _lib.fixed_stream():
        src, tgt, _, frame, dists = _prepare(source, target, "point_to_point", n_samples, seed, [max_corr_dist])
        v = _Correspondences(src, tgt, None, frame).sums_at(s, R, t, dists[0], True, False)
    fitness, rmse = _fit(v[36], v[35], int(src.shape[0]), frame[1])
    return {"fitness": fitness, "inlier_rmse": rmse, "correspondences": v[36]}


# ------------------------------------------------------------------------------------------------------------ transform
def transform(x, T):
    """x moved by the 4x4 similarity T, the same type back: a TsdfMesh (vertices moved, normals rotated, triangles and
    colours kept), a PointCloud (points moved, colours and counts kept), a (vertices, triangles) pair or [N,3] points.
    Each point is s (R p) + t in fp64, rounded to fp32 once (nslam_reg_transform)."""
    _lib.load()
    s, R, t = decompose(T)
    with _lib.fixed_stream():
        if isinstance(x, PointCloud):
            return PointCloud(_transform_points(_points3(x.points, "points"), s, R, t), x.colors, x.counts)
        if hasattr(x, "vertices") and hasattr(x, "triangles"):
            V = _transform_points(_points3(x.vertices, "vertices"), s, R, t)
            N = _transform_points(_points3(x.vertex_normals, "vertex normals"), s, R, t, direction=True)
            return TsdfMesh(V, x.triangles, x.vertex_colors, N)
        if isinstance(x, tuple) and len(x) == 2:
            return _transform_points(_points3(x[0], "vertices"), s, R, t), x[1]
        return _transform_points(_points3(x, "points"), s, R, t)


def trajectory_alignment(est, gt, align="sim3"):
    """the 4x4 fp64 similarity (align "sim3") or rigid transform ("se3") that evaluation.umeyama fits from the camera
    centres of `est` to those of `gt` (cam_T_world, [N,7] t q_xyzw or [N,4,4], frame i against frame i): an `init` for
    icp() of a reconstruction built from `est`"""
    if align not in ("sim3", "se3"):
        raise ValueError(f"align must be 'sim3' or 'se3', not {align!r}")
    ce, cg = _camera_centres(est), _camera_centres(gt)
    if ce.shape != cg.shape or len(ce) < 3:
        raise ValueError(f"est and gt must hold the same number (>= 3) of poses, got {len(ce)} and {len(cg)}")
    return compose(*umeyama(ce, cg, with_scale=align == "sim3"))
