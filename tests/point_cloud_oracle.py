"""ORACLE (test infrastructure only — never imported by the product path).

numpy restatement of nerf_slam_b200/csrc/point_cloud.cu, rule for rule and operation for operation (numpy rounds every
elementwise operation and never fuses a multiply-add, the kernel uses explicit-rounding intrinsics), so that the kernel's
points can be compared bit for bit:

- `point_cloud(...)`: pixel depth and sigma mask, the keep test, fp64 back-projection, fp32 colours, packet / row-major
  order;
- `filter_counts(...)`: the multi-view agreement count of every keyframe against its packet neighbours (the
  droid_backends.depth_filter rule, in fp64);
- `downsample(...)`: lattice keys, stable order, per-voxel fp64 sums in cloud order."""
import numpy as np

from oracle import se3
from tests.tsdf_readout_oracle import _pose_rotation_center

F32 = np.float32
KBIAS = 1 << 20
NEIGHBOURS = (-1, -2, -3, 3, 4, 5)


def pixel_depth(idepths, covs, max_depth, max_sigma):
    """d = 1/idepth (fp32); max_depth + 1 where !(sqrt(cov) < max_sigma)"""
    with np.errstate(divide="ignore", invalid="ignore"):
        d = (F32(1) / np.asarray(idepths, F32)).astype(F32)
        if covs is not None:
            masked = ~(np.sqrt(np.asarray(covs, F32)) < F32(max_sigma))
            d = np.where(masked, F32(max_depth) + F32(1), d).astype(F32)
    return d


def keep_mask(idepths, covs, max_depth, max_sigma, views=None, min_views=2):
    d = pixel_depth(idepths, covs, max_depth, max_sigma)
    keep = (d > 0) & (d < F32(max_depth))
    if views is not None:
        keep &= np.asarray(views, F32) >= F32(min_views)
    return keep, d


def point_cloud(poses, idepths, covs, images, intr, max_depth=6.0, max_sigma=10.0, views=None, min_views=2):
    """-> points, colors [N,3] fp32 (the kernel's rules; `views` = the filter counts or None)"""
    n, H, W = np.shape(idepths)
    keep, d = keep_mask(idepths, covs, max_depth, max_sigma, views, min_views)
    fx, fy, cx, cy = [np.float64(F32(x)) for x in np.asarray(intr).reshape(-1)]
    v, u = np.meshgrid(np.arange(H, dtype=np.float64), np.arange(W, dtype=np.float64), indexing="ij")
    pts, cols = [np.zeros((0, 3), F32)], [np.zeros((0, 3), F32)]
    for k in range(n):
        m = keep[k]
        z = d[k][m].astype(np.float64)
        x = (u[m] - cx) * z / fx
        y = (v[m] - cy) * z / fy
        R, cw = _pose_rotation_center(np.asarray(poses, F32)[k])
        pts.append(np.stack([((R[0, c] * x + R[1, c] * y) + R[2, c] * z) + np.float64(cw[c]) for c in range(3)], -1).astype(F32))
        cols.append((np.asarray(images)[k][:, m].T.astype(F32) / F32(255)).astype(F32))
    return np.concatenate(pts), np.concatenate(cols)


def filter_counts(poses, idepths, intr, thresh):
    """[n,H,W]: for every keyframe i of the packet, how many of its neighbours j = i-1, i-2, i-3, i+3, i+4, i+5 (by packet
    position, inside the packet) see the pixel's point at a depth that agrees within `thresh` with one of the four
    inverse depths around its projection (u0 in [0, W-2], v0 in [0, H-2]); in fp64 on the full-resolution maps"""
    poses = np.asarray(poses, np.float64)
    disps = np.asarray(idepths, np.float64)
    n, H, W = disps.shape
    fx, fy, cx, cy = [np.float64(F32(x)) for x in np.asarray(intr).reshape(-1)]
    v, u = np.meshgrid(np.arange(H, dtype=np.float64), np.arange(W, dtype=np.float64), indexing="ij")
    th = np.float64(F32(thresh))
    out = np.zeros((n, H, W))
    for i in range(n):
        Xi = np.stack([(u - cx) / fx, (v - cy) / fy, np.ones((H, W)), disps[i]], -1)
        for o in NEIGHBOURS:
            j = i + o
            if not 0 <= j < n:
                continue
            t, q = se3.rel_se3(poses[i, :3], poses[i, 3:], poses[j, :3], poses[j, 3:])
            Xj = se3.act_se3(t, q, Xi)
            with np.errstate(divide="ignore", invalid="ignore"):
                uj, vj = fx * (Xj[..., 0] / Xj[..., 2]) + cx, fy * (Xj[..., 1] / Xj[..., 2]) + cy
                depth_j = 1.0 / (Xj[..., 3] / Xj[..., 2])
                u0, v0 = np.floor(uj), np.floor(vj)
                inside = (u0 >= 0) & (v0 >= 0) & (u0 < W - 1) & (v0 < H - 1)
                a = np.where(inside, v0, 0).astype(int)
                b = np.where(inside, u0, 0).astype(int)
                agree = np.zeros((H, W), bool)
                for dv, du in ((0, 0), (0, 1), (1, 0), (1, 1)):
                    agree |= np.abs(depth_j - 1.0 / disps[j][a + dv, b + du]) < th
            out[i] += inside & agree
    return out


def voxel_keys(points, voxel):
    """-> packed keys (uint64; the block keys of tsdf_rules.cuh) and the in-range mask"""
    with np.errstate(invalid="ignore"):
        q = np.floor(np.asarray(points, F32).astype(np.float64) / np.float64(F32(voxel)))
        ok = np.all((q >= -KBIAS) & (q < KBIAS), axis=1)
    qi = np.where(ok[:, None], q, 0).astype(np.int64) + KBIAS
    keys = (qi[:, 0] | (qi[:, 1] << 21) | (qi[:, 2] << 42)).astype(np.uint64)
    return keys, ok


def downsample(points, colors, voxel):
    """-> mean points, mean colors [V,3] fp32, counts [V] int32, keys [V] (ascending); sums in fp64 in cloud order"""
    keys, ok = voxel_keys(points, voxel)
    idx = np.nonzero(ok)[0]
    order = idx[np.argsort(keys[idx], kind="stable")]
    ks = keys[order]
    heads = np.r_[True, ks[1:] != ks[:-1]] if len(ks) else np.zeros(0, bool)
    starts = np.r_[np.nonzero(heads)[0], len(ks)]
    counts = np.diff(starts)
    V = len(counts)
    P, C = np.asarray(points, F32).astype(np.float64), np.asarray(colors, F32).astype(np.float64)
    sp, sc = np.zeros((V, 3)), np.zeros((V, 3))
    for j in range(int(counts.max()) if V else 0):     # the j-th point of every voxel that has one: sequential sums
        live = counts > j
        src = order[starts[:-1][live] + j]
        sp[live] = sp[live] + P[src]
        sc[live] = sc[live] + C[src]
    m = counts[:, None].astype(np.float64)
    return (sp / m).astype(F32), (sc / m).astype(F32), counts.astype(np.int32), ks[heads]
