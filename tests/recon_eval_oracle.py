"""ORACLE (test infrastructure only — never imported by the product path).

Restatement of nerf_slam_b200/csrc/recon_eval.cu in fp64 numpy (numpy rounds every elementwise operation and never fuses
a multiply-add, the kernel uses explicit-rounding intrinsics):

- `surface_samples(...)`: triangle weights, their exact integer scan, the counter-based hash, the triangle search and
  the barycentric point;
- `nearest(...)`: scipy's cKDTree with distance_upper_bound (strictly closer, as the kernel), the distance of the found
  index recomputed by the kernel's rule and rounded to fp32;
- `visible(...)`: the camera projection and depth test;
- `metric_sums(...)` / `metrics(...)`: the fixed-point sums and the counts, and the metric dict built from them;
- `umeyama(...)`: an independent closed-form similarity (Horn's quaternion method), so that the product's SVD form is
  checked against a different derivation."""
import numpy as np
from scipy.spatial import cKDTree

F32 = np.float32
M64 = (1 << 64) - 1
FIXED = 2.0 ** 32


def _rotation_f32(q):
    """tsdf_pose_rotation: the fp64 rotation of q_xyzw, each entry rounded to fp32 (no normalisation)"""
    x, y, z, w = (np.float64(v) for v in np.asarray(q, F32))
    r = np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                  [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                  [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])
    return r.astype(F32).astype(np.float64)


# ------------------------------------------------------------------------------------------------------------ sampling
def hash64(seed, i, k):
    """splitmix64's finaliser of seed * 0x9E3779B97F4A7C15 + (3 i + k + 1) * 0xD1B54A32D192ED03 (mod 2^64)"""
    i = np.asarray(i, np.uint64)
    with np.errstate(over="ignore"):
        x = np.uint64(seed % (1 << 64)) * np.uint64(0x9E3779B97F4A7C15) + \
            (i * np.uint64(3) + np.uint64(k + 1)) * np.uint64(0xD1B54A32D192ED03)
        x = np.asarray(x, np.uint64)
        x ^= x >> np.uint64(30)
        x *= np.uint64(0xBF58476D1CE4E5B9)
        x ^= x >> np.uint64(27)
        x *= np.uint64(0x94D049BB133111EB)
        x ^= x >> np.uint64(31)
    return x


def _mulhi64(a, b):
    """high 64 bits of the 128-bit products a * b (uint64 arrays / scalar)"""
    a = np.asarray(a, np.uint64)
    b = np.uint64(b)
    m32 = np.uint64(0xFFFFFFFF)
    s32 = np.uint64(32)
    a_lo, a_hi = a & m32, a >> s32
    b_lo, b_hi = b & m32, b >> s32
    with np.errstate(over="ignore"):
        ll, lh, hl, hh = a_lo * b_lo, a_lo * b_hi, a_hi * b_lo, a_hi * b_hi
        mid = (ll >> s32) + (lh & m32) + (hl & m32)
        return hh + (lh >> s32) + (hl >> s32) + (mid >> s32)


def triangle_weights(vertices, triangles):
    """-> uint64 weights rint(area * 2^40) (0 for an index out of range or a non-finite area), flags"""
    V = np.asarray(vertices, F32).astype(np.float64)
    T = np.asarray(triangles, np.int64)
    bad_idx = np.any((T < 0) | (T >= len(V)), axis=1)
    Ts = np.where(bad_idx[:, None], 0, T)
    a, b, c = V[Ts[:, 0]], V[Ts[:, 1]], V[Ts[:, 2]]
    e1, e2 = b - a, c - a
    x0 = e1[:, 1] * e2[:, 2] - e1[:, 2] * e2[:, 1]
    x1 = e1[:, 2] * e2[:, 0] - e1[:, 0] * e2[:, 2]
    x2 = e1[:, 0] * e2[:, 1] - e1[:, 1] * e2[:, 0]
    with np.errstate(invalid="ignore", over="ignore"):
        area = 0.5 * np.sqrt((x0 * x0 + x1 * x1) + x2 * x2)
        bad_area = ~np.isfinite(area) & ~bad_idx
        s = area * 2.0 ** 40
    cap = (1 << 62) // len(T)
    big = ~bad_idx & ~bad_area & (s > float(cap))
    ok = ~(bad_idx | bad_area | big)
    w = np.zeros(len(T), np.uint64)
    w[ok] = np.rint(s[ok]).astype(np.uint64)
    flags = (1 if bad_idx.any() else 0) | (2 if bad_area.any() else 0) | (4 if big.any() else 0)
    return w, flags


def surface_samples(vertices, triangles, n, seed=0):
    """-> points [n,3] fp32, triangle index [n]"""
    V = np.asarray(vertices, F32).astype(np.float64)
    T = np.asarray(triangles, np.int64)
    w, _ = triangle_weights(vertices, triangles)
    cdf = np.cumsum(w, dtype=np.uint64)
    total = int(cdf[-1])
    i = np.arange(n, dtype=np.uint64)
    target = _mulhi64(hash64(seed, i, 0), total)
    tri = np.searchsorted(cdf, target, side="right")          # first j with cdf[j] > target
    u = (hash64(seed, i, 1) >> np.uint64(11)).astype(np.float64) * 2.0 ** -53
    v = (hash64(seed, i, 2) >> np.uint64(11)).astype(np.float64) * 2.0 ** -53
    s = np.sqrt(u)
    wa, wb, wc = 1.0 - s, s * (1.0 - v), s * v
    a, b, c = V[T[tri, 0]], V[T[tri, 1]], V[T[tri, 2]]
    p = (wa[:, None] * a + wb[:, None] * b) + wc[:, None] * c
    return p.astype(F32), tri.astype(np.int64)


# ----------------------------------------------------------------------------------------------------------- neighbours
def distance(query, reference, idx):
    """the kernel's distance of query i to reference idx[i]: sqrt((dx^2 + dy^2) + dz^2) in fp64, rounded to fp32"""
    q = np.asarray(query, F32).astype(np.float64)
    r = np.asarray(reference, F32).astype(np.float64)[idx]
    d = q - r
    return np.sqrt((d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2]).astype(F32)


def nearest(query, reference, max_dist=np.inf):
    """-> dist [M] fp32 (+inf without a neighbour), idx [M] int64 (-1), second-neighbour fp64 distance [M] (to tell
    ties: the index is defined by the smaller index only where the two nearest are equally far)"""
    q = np.asarray(query, F32).astype(np.float64)
    tree = cKDTree(np.asarray(reference, F32).astype(np.float64))
    k = 2 if len(reference) > 1 else 1
    dd, ii = tree.query(q, k=k, distance_upper_bound=float(np.float64(F32(max_dist))))
    dd, ii = dd.reshape(len(q), k), ii.reshape(len(q), k)
    idx = np.where(np.isinf(dd[:, 0]), -1, ii[:, 0]).astype(np.int64)
    dist = np.full(len(q), np.inf, F32)
    hit = idx >= 0
    dist[hit] = distance(q[hit], reference, idx[hit])
    second = dd[:, 1] if k == 2 else np.full(len(q), np.inf)
    return dist, idx, second


# ----------------------------------------------------------------------------------------------------------- visibility
def visible(points, poses, intr, W, H, depths=None, tol=0.05, near=0.0, far=np.inf):
    P = np.asarray(points, F32).astype(np.float64)
    fx, fy, cx, cy = (np.float64(F32(v)) for v in intr)
    seen = np.zeros(len(P), bool)
    for k, pose in enumerate(np.asarray(poses, F32)):
        R = _rotation_f32(pose[3:])
        t = pose[:3].astype(np.float64)
        pc = [((R[r, 0] * P[:, 0] + R[r, 1] * P[:, 1]) + R[r, 2] * P[:, 2]) + t[r] for r in range(3)]
        with np.errstate(divide="ignore", invalid="ignore"):
            u = fx * (pc[0] / pc[2]) + cx
            v = fy * (pc[1] / pc[2]) + cy
            ui, vi = np.floor(u + 0.5), np.floor(v + 0.5)
            ok = (pc[2] > np.float64(F32(near))) & (pc[2] <= np.float64(F32(far)))
            ok &= (ui >= 0) & (ui < W) & (vi >= 0) & (vi < H)
        if depths is not None:
            d = np.zeros(len(P), F32)
            d[ok] = np.asarray(depths[k], F32)[vi[ok].astype(np.int64), ui[ok].astype(np.int64)]
            dd = d.astype(np.float64) + np.float64(F32(tol))
            ok &= ~(d > 0) | (pc[2] <= dd)
        seen |= ok
    return seen


# -------------------------------------------------------------------------------------------------------------- metrics
def metric_sums(dist, max_dist, threshold):
    """-> (sum of rint(min(d, max_dist) 2^32) as a Python int, count d < threshold, count d = +inf)"""
    d = np.asarray(dist, F32)
    m = np.minimum(d, F32(max_dist)).astype(np.float64)
    s = int(np.rint(m * FIXED).astype(np.uint64).sum(dtype=np.uint64))
    return s, int(np.sum(d < F32(threshold))), int(np.sum(np.isposinf(d)))


def metrics(rec_points, gt_points, threshold=0.05, max_dist=1.0):
    """reconstruction_metrics on given point sets (no sampling, no mask)"""
    d_acc, _, _ = nearest(rec_points, gt_points, max_dist)
    d_comp, _, _ = nearest(gt_points, rec_points, max_dist)
    sa, ia, ma = metric_sums(d_acc, max_dist, threshold)
    sc, ic, mc = metric_sums(d_comp, max_dist, threshold)
    n_rec, n_gt = len(d_acc), len(d_comp)
    acc, comp = sa / FIXED / n_rec, sc / FIXED / n_gt
    p, r = ia / n_rec, ic / n_gt
    return {"accuracy": acc, "completion": comp, "chamfer_l1": 0.5 * (acc + comp), "precision": p, "recall": r,
            "f_score": 2 * p * r / (p + r) if p + r > 0 else 0.0, "n_reconstruction": n_rec, "n_ground_truth": n_gt,
            "unmatched_reconstruction": ma, "unmatched_ground_truth": mc, "accuracy_fixed": sa, "completion_fixed": sc}


# ----------------------------------------------------------------------------------------------------------- trajectory
def umeyama(src, dst, with_scale=True):
    """dst ~ s R src + t by Horn's closed form: R from the top eigenvector of the 4x4 quaternion matrix of the
    cross-covariance, s = sum(y . R x) / sum(|x|^2) -> (s, R, t)"""
    src, dst = np.asarray(src, np.float64), np.asarray(dst, np.float64)
    ms, md = src.mean(0), dst.mean(0)
    X, Y = src - ms, dst - md
    S = X.T @ Y
    Sxx, Sxy, Sxz, Syx, Syy, Syz, Szx, Szy, Szz = S.reshape(-1)
    N = np.array([[Sxx + Syy + Szz, Syz - Szy, Szx - Sxz, Sxy - Syx],
                  [Syz - Szy, Sxx - Syy - Szz, Sxy + Syx, Szx + Sxz],
                  [Szx - Sxz, Sxy + Syx, -Sxx + Syy - Szz, Syz + Szy],
                  [Sxy - Syx, Szx + Sxz, Syz + Szy, -Sxx - Syy + Szz]])
    w, V = np.linalg.eigh(N)
    q0, qx, qy, qz = V[:, -1]
    R = np.array([[q0 * q0 + qx * qx - qy * qy - qz * qz, 2 * (qx * qy - q0 * qz), 2 * (qx * qz + q0 * qy)],
                  [2 * (qy * qx + q0 * qz), q0 * q0 - qx * qx + qy * qy - qz * qz, 2 * (qy * qz - q0 * qx)],
                  [2 * (qz * qx - q0 * qy), 2 * (qz * qy + q0 * qx), q0 * q0 - qx * qx - qy * qy + qz * qz]])
    s = float(np.sum(Y * (X @ R.T)) / np.sum(X * X)) if with_scale else 1.0
    return s, R, md - s * R @ ms
