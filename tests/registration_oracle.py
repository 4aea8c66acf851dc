"""ORACLE (test infrastructure only — never imported by the product path).

Restatement of nerf_slam_b200/csrc/registration.cu in fp64 numpy (numpy rounds every elementwise operation and never
fuses a multiply-add, the kernels use explicit-rounding intrinsics):

- `transform(...)`: s (R p) + t per row, rounded to fp32 once; the direction mode R p;
- `face_normals(...)`: the unit (b - a) x (c - a) of each sample's triangle;
- `accumulate(...)`: the correspondence terms in the target's normalised frame, each rounded to an integer of 2^-27;
- `icp(...)`: a whole ICP on the CPU: recon_eval_oracle.nearest for the correspondences (cKDTree, strictly closer than
  the fp32 max_corr_dist) and the product's host step (registration.gauss_newton_step / apply_step), which both sides
  share, so the integer sums and every transform must agree bit for bit."""
import math

import numpy as np

from nerf_slam_b200 import registration as reg
from tests import recon_eval_oracle as rorc

F32 = np.float32
FIXED = 2.0 ** 27


def transform(points, s, R, t, direction=False):
    P = np.asarray(points, F32).astype(np.float64)
    R = np.asarray(R, np.float64)
    q = [(R[r, 0] * P[:, 0] + R[r, 1] * P[:, 1]) + R[r, 2] * P[:, 2] for r in range(3)]
    if not direction:
        q = [float(s) * q[r] + float(t[r]) for r in range(3)]
    return np.stack(q, 1).astype(F32)


def face_normals(vertices, triangles, tri):
    """-> normals [n,3] fp32, flags (1 an index out of range, 2 a zero or non-finite normal; such samples get 0)"""
    V = np.asarray(vertices, F32).astype(np.float64)
    T = np.asarray(triangles, np.int64)
    tri = np.asarray(tri, np.int64)
    bad_t = (tri < 0) | (tri >= len(T))
    Ti = T[np.where(bad_t, 0, tri)]
    bad = bad_t | np.any((Ti < 0) | (Ti >= len(V)), axis=1)
    Ti = np.where(bad[:, None], 0, Ti)
    a, b, c = V[Ti[:, 0]], V[Ti[:, 1]], V[Ti[:, 2]]
    e1, e2 = b - a, c - a
    x = np.stack([e1[:, 1] * e2[:, 2] - e1[:, 2] * e2[:, 1], e1[:, 2] * e2[:, 0] - e1[:, 0] * e2[:, 2],
                  e1[:, 0] * e2[:, 1] - e1[:, 1] * e2[:, 0]], 1)
    with np.errstate(invalid="ignore", over="ignore", divide="ignore"):
        length = np.sqrt((x[:, 0] * x[:, 0] + x[:, 1] * x[:, 1]) + x[:, 2] * x[:, 2])
        zero = ~bad & ~((length > 0) & np.isfinite(length))
        n = x / length[:, None]
    n[bad | zero] = 0
    return n.astype(F32), (1 if bad.any() else 0) | (2 if zero.any() else 0)


def frame(target):
    """the product's frame (registration.target_frame) of the target's exact fp32 box"""
    P = np.asarray(target, F32)
    return reg.target_frame(P.min(0), P.max(0))


def accumulate(moved, idx, target, normals, frame_, point_to_point, with_scale):
    """-> the 38 integers of nslam_reg_accumulate (a list of Python ints)"""
    (c, L), D = frame_, 7 if with_scale else 6
    idx = np.asarray(idx, np.int64)
    out = [0] * 38
    bad_idx = idx >= len(target)
    ok = (idx >= 0) & ~bad_idx
    j = idx[ok]
    cc = np.asarray(c, np.float64)
    p = (np.asarray(moved, F32)[ok].astype(np.float64) - cc) / L
    q = (np.asarray(target, F32)[j].astype(np.float64) - cc) / L
    d = p - q
    zero = np.zeros(len(p))
    flag = 1 if bad_idx.any() else 0

    def add(k, v):
        nonlocal flag
        good = np.abs(v) < 16.0
        if not good.all():
            flag |= 2
        out[k] += int(np.rint(v[good] * FIXED).astype(np.int64).sum(dtype=np.int64))

    if not point_to_point:
        n = np.asarray(normals, F32)[j].astype(np.float64)
        J = [p[:, 1] * n[:, 2] - p[:, 2] * n[:, 1], p[:, 2] * n[:, 0] - p[:, 0] * n[:, 2],
             p[:, 0] * n[:, 1] - p[:, 1] * n[:, 0], n[:, 0], n[:, 1], n[:, 2],
             (p[:, 0] * n[:, 0] + p[:, 1] * n[:, 1]) + p[:, 2] * n[:, 2]]
        r = (n[:, 0] * d[:, 0] + n[:, 1] * d[:, 1]) + n[:, 2] * d[:, 2]
        k = 0
        for a in range(7):
            for b in range(a, 7):
                if b < D and a < D:
                    add(k, J[a] * J[b])
                k += 1
            if a < D:
                add(28 + a, J[a] * r)
    else:
        J = [[zero, p[:, 2], -p[:, 1], zero + 1, zero, zero, p[:, 0]],
             [-p[:, 2], zero, p[:, 0], zero, zero + 1, zero, p[:, 1]],
             [p[:, 1], -p[:, 0], zero, zero, zero, zero + 1, p[:, 2]]]
        k = 0
        for a in range(7):
            for b in range(a, 7):
                if b < D:
                    add(k, (J[0][a] * J[0][b] + J[1][a] * J[1][b]) + J[2][a] * J[2][b])
                k += 1
            if a < D:
                add(28 + a, (J[0][a] * d[:, 0] + J[1][a] * d[:, 1]) + J[2][a] * d[:, 2])
    add(35, (d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2])
    out[36] = int(len(p))
    out[37] = flag
    return out


def sums_at(source, target, normals, frame_, s, R, t, max_dist, point_to_point, with_scale):
    moved = transform(source, s, R, t)
    _, idx, _ = rorc.nearest(moved, target, max_dist)
    return accumulate(moved, idx, target, normals, frame_, point_to_point, with_scale)


def icp(source, target, normals, init=(1.0, np.eye(3), np.zeros(3)), metric="point_to_plane", with_scale=False,
        max_corr_dist=(0.2, 0.1, 0.05), max_iters=30, tol=1e-7):
    """registration.icp on given point sets (source [N,3], target [M,3] fp32 and its unit normals for point-to-plane)
    -> dict with the fields of IcpResult"""
    p2p = metric == "point_to_point"
    fr = frame(target)
    c, L = fr
    s, R, t = init
    history, iterations, converged, degenerate = [], 0, False, False
    for stage, d in enumerate(float(v) for v in max_corr_dist):
        converged = False
        for _ in range(max_iters):
            sums = sums_at(source, target, normals, fr, s, R, t, d, p2p, with_scale)
            assert sums[37] == 0
            x = reg.gauss_newton_step(sums, with_scale)
            count = sums[36]
            history.append({"stage": stage, "max_corr_dist": d, "correspondences": count,
                            "rmse": L * math.sqrt(sums[35] / FIXED / count) if count else 0.0,
                            "step": None if x is None else float(np.abs(x).max()), "sums": sums})
            if x is None:
                degenerate = True
                break
            s, R, t = reg.apply_step(s, R, t, x, c, L)
            iterations += 1
            if np.abs(x).max() < tol:
                converged = True
                break
        if degenerate:
            break
    final = sums_at(source, target, None, fr, s, R, t, float(max_corr_dist[-1]), True, False)
    count = final[36]
    return {"transform": reg.compose(s, R, t), "scale": s, "rotation": R, "translation": np.asarray(t, np.float64),
            "fitness": count / len(source), "inlier_rmse": L * math.sqrt(final[35] / FIXED / count) if count else 0.0,
            "iterations": iterations, "converged": converged, "degenerate": degenerate, "history": history}


def sample_with_normals(vertices, triangles, n, seed):
    """the target of icp(): `n` surface samples (seed) and their face normals"""
    pts, tri = rorc.surface_samples(vertices, triangles, n, seed)
    nrm, flags = face_normals(vertices, triangles, tri)
    assert flags == 0
    return pts, nrm
