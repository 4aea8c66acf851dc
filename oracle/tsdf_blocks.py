"""ORACLE (test infrastructure only — never imported by the product path).

numpy restatement of the sparse voxel-block volume of nerf_slam_b200/csrc/tsdf_blocks.cu (rules at the head of that
file): block keys, the activation rule (Open3D's compute_unique_block_coordinates with trunc_voxel_multiplier 8, as the
kernel defines it — Open3D itself is unavailable, so this set is not pinned against it), the pool order, and the
integration of every voxel of the touched blocks.

The per-voxel update is oracle.tsdf's, restated on explicit voxel coordinates: oracle.tsdf.integrate forms a voxel's
coordinate as fp32(origin + fp32(voxel * i)), which equals the block lattice's fp32(voxel * g) only for origin 0, so it
cannot be run on a scratch grid around blocks at negative indices.  tests/test_cpu_tsdf_blocks.py checks the two
restatements against each other, bit for bit, on an origin-0 grid."""
import numpy as np

from oracle.tsdf import F32, pose_tq_to_matrix

BIAS = 1 << 20
BLOCK = 16


def pack(b):
    """int block coordinates [...,3] -> (int64 keys, in-range mask); keys outside [-2^20, 2^20)^3 are not packable"""
    b = np.asarray(b, np.int64)
    ok = np.all((b >= -BIAS) & (b < BIAS), -1)
    c = np.where(ok[..., None], b + BIAS, 0)
    return c[..., 0] | (c[..., 1] << 21) | (c[..., 2] << 42), ok


def unpack(keys):
    k = np.asarray(keys, np.int64)
    return np.stack([(k & 0x1FFFFF) - BIAS, ((k >> 21) & 0x1FFFFF) - BIAS, ((k >> 42) & 0x1FFFFF) - BIAS], -1).astype(np.int32)


def pixel_depth(idepth_up, depth_cov_up, max_depth=6.0, max_depth_sigma=10000.0):
    """build_volume's depth: 1 / inverse depth, pushed to max_depth + 1 where the sigma test masks the pixel"""
    depth = (F32(1.0) / idepth_up.astype(F32)).astype(F32)
    if depth_cov_up is not None:
        cov = depth_cov_up.astype(F32)
        depth = np.where(np.sqrt(cov) < F32(max_depth_sigma), depth, F32(max_depth) + F32(1.0)).astype(F32)
    return depth


def touched_keys_from_depth(depth, intr4, T, voxel_size, max_depth=6.0):
    """sorted unique int64 keys of the blocks a depth map touches.  T = the fp64 cam_T_world matrix with the fp32-rounded
    rotation (oracle.tsdf.pose_tq_to_matrix); intr4 = fx, fy, cx, cy (fp32)"""
    H, W = depth.shape
    fx, fy, cx, cy = [np.float64(F32(v)) for v in intr4]
    R, t = T[:3, :3], T[:3, 3]
    v, u = np.meshgrid(np.arange(H, dtype=np.float64), np.arange(W, dtype=np.float64), indexing="ij")
    valid = (depth > 0) & (depth < F32(max_depth))
    d = depth[valid]
    q = [(u[valid] - cx) / fx - t[0], (v[valid] - cy) / fy - t[1], np.float64(1.0) - t[2]]
    o = [-((R[0, c] * t[0] + R[1, c] * t[1]) + R[2, c] * t[2]) for c in range(3)]
    dirs = [((R[0, c] * q[0] + R[1, c] * q[1]) + R[2, c] * q[2]) - o[c] for c in range(3)]
    vs = F32(voxel_size)
    ta = F32(8) * vs
    t_min = np.maximum((d - ta).astype(F32), F32(0))
    t_max = np.minimum((d + ta).astype(F32), F32(max_depth))
    dt = (t_max - t_min).astype(F32)
    bl = np.float64(F32(16) * vs)
    keys = []
    for k in range(4):
        tk = (t_min + ((F32(k) * dt).astype(F32) / F32(3)).astype(F32)).astype(F32).astype(np.float64)
        with np.errstate(invalid="ignore", over="ignore"):
            b = np.stack([np.floor((o[c] + tk * dirs[c]) / bl) for c in range(3)], -1)
            ok = np.all((b >= -BIAS) & (b < BIAS), -1)
        key, _ = pack(np.where(ok[:, None], b, 0).astype(np.int64))
        keys.append(key[ok])
    return np.unique(np.concatenate(keys)) if keys else np.zeros(0, np.int64)


def touched_keys(idepth_up, depth_cov_up, intr4, cam_T_world_tq, voxel_size, max_depth=6.0, max_depth_sigma=10000.0):
    """the activation of one keyframe from the packet's tensors, as nslam_tsdf_blocks_activate computes it"""
    depth = pixel_depth(idepth_up, depth_cov_up, max_depth, max_depth_sigma)
    return touched_keys_from_depth(depth, intr4, pose_tq_to_matrix(np.asarray(cam_T_world_tq, np.float32)), voxel_size, max_depth)


def voxel_world(coords, voxel_size):
    """fp32 world coordinates voxel_size * (16 b + l) of every voxel of the blocks `coords` [n,3] -> [n,16,16,16,3]
    (local voxel l = lx + 16 ly + 256 lz, array order [lz][ly][lx])"""
    lz, ly, lx = np.meshgrid(np.arange(BLOCK), np.arange(BLOCK), np.arange(BLOCK), indexing="ij")
    loc = np.stack([lx, ly, lz], -1)
    g = BLOCK * np.asarray(coords, np.int64)[:, None, None, None, :] + loc[None]
    return (F32(voxel_size) * g.astype(F32)).astype(F32)


def update_voxels(tsdf, weight, color, world, idepth_up, depth_cov_up, rgb_chw, intr, cam_T_world_tq, max_depth=6.0,
                  sdf_trunc=0.10, max_weight=20.0, max_depth_sigma=10000.0):
    """oracle.tsdf.integrate's per-voxel rule on voxels at fp32 world coordinates `world` [...,3]; tsdf / weight [...]
    and color [...,3] fp32 are updated in place.  Returns the number of voxels updated."""
    H, W = idepth_up.shape
    depth = pixel_depth(idepth_up, depth_cov_up, max_depth, max_depth_sigma)
    wimg = np.ones((H, W), F32) if depth_cov_up is None else np.sqrt(F32(1.0) / depth_cov_up.astype(F32)).astype(F32)
    T = pose_tq_to_matrix(np.asarray(cam_T_world_tq, np.float32))
    fx, fy, cx, cy = [float(F32(v)) for v in intr]
    wx, wy, wz = [world[..., c].astype(np.float64) for c in range(3)]
    x = T[0, 0] * wx + T[0, 1] * wy + T[0, 2] * wz + T[0, 3]
    y = T[1, 0] * wx + T[1, 1] * wy + T[1, 2] * wz + T[1, 3]
    d = T[2, 0] * wx + T[2, 1] * wy + T[2, 2] * wz + T[2, 3]
    with np.errstate(divide="ignore", invalid="ignore"):
        u = np.rint((fx * x + cx * d) / d)
        v = np.rint((fy * y + cy * d) / d)
    proj = (d > 0) & (u >= 0) & (v >= 0) & (u < W) & (v < H)
    ui = np.where(proj, u, 0).astype(np.int64); vi = np.where(proj, v, 0).astype(np.int64)
    dr = depth[vi, ui]
    sdf = (dr - d.astype(F32)).astype(F32)
    inl = proj & (dr > 0) & (dr < F32(max_depth)) & (sdf >= -F32(sdf_trunc))
    sdf = (np.minimum(sdf, F32(sdf_trunc)) / F32(sdf_trunc)).astype(F32)
    wr = wimg[vi, ui]
    w = weight
    wp = (w + wr).astype(F32)
    with np.errstate(divide="ignore", invalid="ignore"):
        new_t = ((w * tsdf + wr * sdf) / wp).astype(F32)
        rgb = rgb_chw.astype(F32)
        new_c = ((w[..., None] * color + wr[..., None] * np.stack([rgb[c][vi, ui] for c in range(3)], -1)) / wp[..., None]).astype(F32)
    tsdf[inl] = new_t[inl]
    color[inl] = new_c[inl]
    weight[inl] = np.minimum(wp, F32(max_weight))[inl]
    return int(inl.sum())


class BlockVolume:
    """the block volume in numpy: pool arrays in pool order, new blocks appended in ascending key order"""

    def __init__(self, voxel_size):
        self.voxel_size = F32(voxel_size)
        self.keys = np.zeros(0, np.int64)
        self.tsdf = np.zeros((0, BLOCK, BLOCK, BLOCK), F32)
        self.weight = np.zeros((0, BLOCK, BLOCK, BLOCK), F32)
        self.color = np.zeros((0, BLOCK, BLOCK, BLOCK, 3), F32)

    @property
    def coords(self):
        return unpack(self.keys)

    def activate(self, keys):
        """append the blocks of `keys` (sorted, unique) that are new -> (pool indices of `keys`, new keys)"""
        new = np.setdiff1d(keys, self.keys)                      # sorted
        n0 = len(self.keys)
        self.keys = np.concatenate([self.keys, new])
        z = np.zeros((len(new), BLOCK, BLOCK, BLOCK), F32)
        self.tsdf = np.concatenate([self.tsdf, z]); self.weight = np.concatenate([self.weight, z])
        self.color = np.concatenate([self.color, np.zeros(z.shape + (3,), F32)])
        index = {int(k): i for i, k in enumerate(self.keys)}
        return np.array([index[int(k)] for k in keys], np.int64), new

    def integrate_blocks(self, pool, idepth_up, depth_cov_up, rgb_chw, intr, cam_T_world_tq, **kw):
        """the per-voxel rule on every voxel of the pool blocks `pool`, on scratch copies merged back"""
        t, w, c = self.tsdf[pool].copy(), self.weight[pool].copy(), self.color[pool].copy()
        n = update_voxels(t, w, c, voxel_world(self.coords[pool], self.voxel_size), idepth_up, depth_cov_up, rgb_chw,
                          intr, cam_T_world_tq, **kw)
        self.tsdf[pool], self.weight[pool], self.color[pool] = t, w, c
        return n

    def integrate(self, idepth_up, depth_cov_up, rgb_chw, intr, cam_T_world_tq, max_depth=6.0, sdf_trunc=0.10,
                  max_weight=20.0, max_depth_sigma=10000.0):
        """one keyframe -> its touched keys"""
        keys = touched_keys(idepth_up, depth_cov_up, intr, cam_T_world_tq, self.voxel_size, max_depth, max_depth_sigma)
        pool, _ = self.activate(keys)
        self.integrate_blocks(pool, idepth_up, depth_cov_up, rgb_chw, intr, cam_T_world_tq, max_depth=max_depth,
                              sdf_trunc=sdf_trunc, max_weight=max_weight, max_depth_sigma=max_depth_sigma)
        return keys


def to_dense(coords, tsdf, weight, color, voxel_size, margin_blocks=1, lo=None):
    """dense embedding [nz,ny,nx] of pool arrays (0 outside the blocks) from block `lo` (default: the smallest block
    coordinate minus the margin) -> tsdf, weight, color, fp32 origin voxel_size * 16 lo"""
    coords = np.asarray(coords, np.int64).reshape(-1, 3)
    lo = coords.min(0) - margin_blocks if lo is None else np.asarray(lo, np.int64)
    hi = coords.max(0) + margin_blocks + 1
    nb = hi - lo
    dims = (BLOCK * nb[2], BLOCK * nb[1], BLOCK * nb[0])
    t = np.zeros(dims, F32); w = np.zeros(dims, F32); c = np.zeros(dims + (3,), F32)
    for i, b in enumerate(coords - lo):
        s = np.s_[BLOCK * b[2]:BLOCK * b[2] + BLOCK, BLOCK * b[1]:BLOCK * b[1] + BLOCK, BLOCK * b[0]:BLOCK * b[0] + BLOCK]
        t[s], w[s], c[s] = tsdf[i], weight[i], color[i]
    return t, w, c, (F32(voxel_size) * (BLOCK * lo).astype(F32)).astype(F32)
