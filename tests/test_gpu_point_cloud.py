"""SLAM point clouds on the GPU (csrc/point_cloud.cu): the kernels against the numpy restatement
(tests/point_cloud_oracle.py) bit for bit on seeded packets, the filter counts against droid_backends.depth_filter,
determinism, the ground-truth synthetic room (walls, a corrupted patch, downsampling invariants), the live front end's
arenas, and the peak memory of a 100-keyframe 640x480 map against the documented scratch bound."""
import os
import types

import numpy as np
import pytest
import torch

from oracle import se3
from tests import point_cloud_oracle as opc

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
WEIGHTS = os.path.join(ROOT, "oracle", "_ref", "droid.pth")
DEV = "cuda:0"
F32 = np.float32


def _seeded_packet(seed, n, H, W):
    """a slowly moving camera over a wavy surface at 0.8-2.5 m, 2 % depth noise, special inverse depths (0, negative,
    NaN, inf, beyond max_depth) and sigma-masked pixels"""
    rng = np.random.default_rng(seed)
    poses = se3.random_poses(rng, n, trans=0.03, rot_deg=1.5).astype(F32)
    v, u = np.meshgrid(np.arange(H), np.arange(W), indexing="ij")
    depth = 1.6 + 0.5 * np.sin(u / 23.0 + 0.3 * seed) * np.cos(v / 31.0)
    idepth = (1.0 / (depth[None] * rng.uniform(0.99, 1.01, (n, H, W)))).astype(F32)
    flat = idepth.reshape(-1)
    m = flat.size
    for val in (0.0, -0.5, np.nan, np.inf, 1.0 / 7.0):
        flat[rng.integers(0, m, max(1, m // 200))] = val
    cov = rng.uniform(0.0, 120.0, (n, H, W)).astype(F32)             # sigma up to 11: about a sixth masked
    cov.reshape(-1)[rng.integers(0, m, max(1, m // 500))] = np.nan
    images = rng.integers(0, 256, (n, 3, H, W)).astype(np.uint8)
    f = 0.8 * W
    intr = np.array([f, f * 1.01, (W - 1) / 2 + 0.25, (H - 1) / 2 - 0.5], F32)
    return poses, idepth, cov, images, intr


def _t(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def _packet(poses, idepth, cov, images):
    return {"cam0_poses": _t(poses), "cam0_idepths_up": _t(idepth), "cam0_depths_cov_up": None if cov is None else _t(cov),
            "cam0_images": _t(images)}


SHAPES = [(3, 480, 640), (7, 37, 53), (2, 1, 301)]


@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: "x".join(map(str, s)))
@pytest.mark.parametrize("mask", ["uncertainty", "uniform"])
@pytest.mark.parametrize("filt", [None, 0.05], ids=["nofilter", "filter"])
@pytest.mark.parametrize("voxel", [None, 0.05], ids=["full", "voxel"])
def test_kernel_matches_oracle(shape, mask, filt, voxel):
    """points bit-exact, colours and counts exact; downsampled means bit-exact (the oracle restates the fp64 sums in
    cloud order).  With the filter, the oracle takes the kernel's counts: they are droid_backends.depth_filter's
    (compared with it below), whose fp32 arithmetic the fp64 oracle does not restate bit for bit."""
    from nerf_slam_b200.point_cloud import build_point_cloud, kernels
    poses, idepth, cov, images, intr = _seeded_packet(sum(shape), *shape)
    cov = cov if mask == "uncertainty" else None
    pk = _packet(poses, idepth, cov, images)
    pc = build_point_cloud(pk, intr, filter_thresh=filt, min_views=2, voxel_size=voxel)
    views = None
    if filt is not None:
        views = kernels.filter_counts(pk["cam0_poses"], pk["cam0_idepths_up"], _t(intr), filt).cpu().numpy()
    P, C = opc.point_cloud(poses, idepth, cov, images, intr, 6.0, 10.0, views, 2)
    if voxel is not None:
        P, C, N, _ = opc.downsample(P, C, voxel)
    if len(P) == 0:
        assert pc is None
        return
    assert np.array_equal(pc.points.cpu().numpy(), P)
    assert np.array_equal(pc.colors.cpu().numpy(), C)
    if voxel is not None:
        assert pc.counts.dtype == torch.int32 and np.array_equal(pc.counts.cpu().numpy(), N)
    else:
        assert pc.counts is None


def test_filter_counts_are_depth_filter():
    from nerf_slam_b200 import droid_backends as db
    from nerf_slam_b200.point_cloud import kernels
    poses, idepth, _, _, intr = _seeded_packet(5, 9, 120, 160)
    P, D, K = _t(poses), _t(idepth), _t(intr)
    got = kernels.filter_counts(P, D, K, 0.05)
    ref = db.depth_filter(P, D, K, torch.arange(9, device=DEV), torch.full((9,), 0.05, device=DEV))
    assert torch.equal(got, ref)
    orc = opc.filter_counts(poses, idepth, intr, 0.05)                  # fp64 restatement: agreement up to rounding
    assert (got.cpu().numpy() == orc).mean() > 0.999 and orc.max() >= 4


def test_two_fresh_calls_give_the_same_bytes():
    from nerf_slam_b200.point_cloud import build_point_cloud
    poses, idepth, cov, images, intr = _seeded_packet(11, 6, 240, 320)
    out = []
    for _ in range(2):
        pc = build_point_cloud(_packet(poses, idepth, cov, images), intr, filter_thresh=0.05, voxel_size=0.02)
        out.append([t.cpu().numpy().tobytes() for t in (pc.points, pc.colors, pc.counts)])
        pc2 = build_point_cloud(_packet(poses, idepth, cov, images), intr)
        out[-1] += [t.cpu().numpy().tobytes() for t in (pc2.points, pc2.colors)]
    assert out[0] == out[1]


# --------------------------------------------------------------------------------------------- synthetic room (GT)
def _room_packet(n, step=4, W=640, H=480):
    """ground-truth keyframes of the synthetic room: inverse depths from the u16 depth, a synthetic variance
    (0.1 d^2)^2, images, cam_T_world"""
    from nerf_slam_b200.frontend import matrix_to_tq
    from nerf_slam_b200.synthetic import SyntheticRoom
    room = SyntheticRoom(W, H, n * step, seed=0)
    poses, idepth, images = [], [], []
    for k in range(0, n * step, step):
        rgba, d16, w2c = room.render(k)
        depth = d16[..., 0].astype(np.float32) * np.float32(room.calib.depth_scale)
        poses.append(matrix_to_tq(np.asarray(w2c, np.float64)).astype(F32))
        idepth.append((1.0 / depth).astype(F32))
        images.append(np.ascontiguousarray(rgba[..., :3].transpose(2, 0, 1)))
    idepth = np.stack(idepth)
    cov = ((0.1 / idepth ** 2) ** 2).astype(F32)
    return room, np.stack(poses), idepth, cov, np.stack(images), room.calib.camera_model.numpy().astype(F32)


def _wall_distance(room, P):
    return np.min(np.abs(room.ext[None] - np.abs(P.astype(np.float64))), axis=1)


@pytest.fixture(scope="module")
def room10():
    return _room_packet(10)


def test_room_points_lie_on_the_walls(room10):
    from nerf_slam_b200.point_cloud import build_point_cloud
    room, poses, idepth, cov, images, intr = room10
    pc = build_point_cloud(_packet(poses, idepth, cov, images), intr)
    P = pc.points.cpu().numpy()
    keep, _ = opc.keep_mask(idepth, cov, 6.0, 10.0)
    assert len(P) == keep.sum() and len(P) > 0.9 * idepth.size
    # depth quantisation: the u16 depth truncates by < depth_scale along z, i.e. < depth_scale * |ray| in space
    ray = np.sqrt(1 + ((np.array([room.W, room.H]) / 2) / intr[:2]) ** 2 @ np.ones(2))
    assert _wall_distance(room, P).max() < room.calib.depth_scale * ray + 1e-4


def test_room_filter_removes_a_corrupted_patch(room10):
    from nerf_slam_b200.point_cloud import build_point_cloud, kernels
    room, poses, idepth, cov, images, intr = room10
    bad = idepth.copy()
    k, (v0, v1, u0, u1) = 5, (200, 260, 300, 380)
    bad[k, v0:v1, u0:u1] /= 0.6                                          # 40 % too close: off the walls
    thresh, min_views = 0.05, 2
    # thresholds from the oracle on the same data: the patch has fewer than min_views agreeing neighbours, the clean
    # part of the keyframe mostly more
    orc = opc.filter_counts(poses[k - 3:k + 6], bad[k - 3:k + 6], intr, thresh)[3]
    assert orc[v0:v1, u0:u1].max() < min_views
    clean = np.ones(orc.shape, bool)
    clean[v0:v1, u0:u1] = False
    assert (orc[clean] >= min_views).mean() > 0.9
    pk = _packet(poses, bad, cov, images)
    pc = build_point_cloud(pk, intr, filter_thresh=thresh, min_views=min_views)
    views = kernels.filter_counts(pk["cam0_poses"], pk["cam0_idepths_up"], _t(intr), thresh).cpu().numpy()
    keep, _ = opc.keep_mask(bad, cov, 6.0, 10.0, views, min_views)
    assert not keep[k, v0:v1, u0:u1].any() and keep[k][clean].mean() > 0.9
    assert len(pc.points) == keep.sum()
    ray = np.sqrt(1 + ((np.array([room.W, room.H]) / 2) / intr[:2]) ** 2 @ np.ones(2))
    assert _wall_distance(room, pc.points.cpu().numpy()).max() < room.calib.depth_scale * ray + 1e-4
    unfiltered = build_point_cloud(pk, intr)
    assert _wall_distance(room, unfiltered.points.cpu().numpy()).max() > 0.5            # the patch is there without it


def test_room_downsampling_invariants(room10):
    from nerf_slam_b200.point_cloud import build_point_cloud
    room, poses, idepth, cov, images, intr = room10
    pk = _packet(poses, idepth, cov, images)
    full = build_point_cloud(pk, intr)
    pc = build_point_cloud(pk, intr, voxel_size=0.01)
    cnt = pc.counts.cpu().numpy()
    assert cnt.sum() == len(full.points) and len(cnt) < len(full.points) / 4
    keys, ok = opc.voxel_keys(pc.points.cpu().numpy(), 0.01)
    assert ok.all() and np.all(keys[1:] > keys[:-1])                    # one output per voxel, ascending keys
    _, _, _, member_keys = opc.downsample(full.points.cpu().numpy(), full.colors.cpu().numpy(), 0.01)
    assert np.array_equal(keys, member_keys)                            # each mean inside the voxel of its points
    assert ((pc.colors >= 0) & (pc.colors <= 1)).all()


# --------------------------------------------------------------------------------------------------- live front end
def test_frontend_point_cloud_from_the_arenas():
    if not os.path.exists(WEIGHTS):
        pytest.skip("oracle/_ref/droid.pth not built")
    from nerf_slam_b200.frontend import RaftVisualFrontend
    from nerf_slam_b200.synthetic import SyntheticRoom
    args = types.SimpleNamespace(buffer=24, stereo=False, multi_gpu=False, weights=WEIGHTS)
    room = SyntheticRoom(320, 240, 40, seed=0, step=0.03)
    fe = RaftVisualFrontend(np.linalg.inv(room.packet(0)["poses"][0]), np.eye(4), args, DEV)
    for k in range(40):
        fe.forward(room.packet(k))
        if fe.stop_condition():
            break
    assert fe.is_initialized
    pc = fe.point_cloud()
    assert pc is not None and len(pc) > 1000
    n = fe.kf_idx + 1 if fe.stop else fe.kf_idx
    idepth = fe.cam0_idepths_up[:n].cpu().numpy()
    cov = fe.cam0_depths_cov_up[:n].cpu().numpy()
    keep, _ = opc.keep_mask(idepth, cov, 6.0, 10.0)
    assert keep.sum() == len(pc)
    P = pc.points.cpu().numpy().astype(np.float64)
    poses = fe.cam0_T_world[:n].cpu().numpy().astype(np.float64)
    s = 0
    for k in range(n):
        m = int(keep[k].sum())
        t, q = poses[k, :3], poses[k, 3:]
        z = (P[s:s + m] @ se3.to_matrix(t, q)[:3, :3].T + t)[:, 2]
        assert (z > 0).all() and (z < 6.0 * (1 + 1e-5)).all()
        s += m
    pc_u = fe.point_cloud(mask_type="uniform", voxel_size=0.05)
    assert pc_u is not None and int(pc_u.counts.sum()) >= len(pc)


# ----------------------------------------------------------------------------------------------------- memory bound
def test_peak_memory_of_a_100_keyframe_map_is_within_the_scratch_bound(room10):
    """100 x 640x480 keyframes (ten ground-truth views, each ten times), uncertainty mask, filter and 1 cm
    downsampling: the device memory added by the call stays within the bound csrc/point_cloud.cu documents — 4 B per
    candidate pixel for the filter counts, 1 B per 32 candidate pixels, 24 B per kept point (the cloud), 52 B per kept
    point (downsampling), 28 B per voxel (the result) and 4 MiB of fixed and rounding slack"""
    from nerf_slam_b200.point_cloud import build_point_cloud
    room, poses, idepth, cov, images, intr = room10
    rep = lambda a: np.ascontiguousarray(np.tile(a, (10,) + (1,) * (a.ndim - 1)))
    pk = _packet(rep(poses), rep(idepth), rep(cov), rep(images))
    K = _t(intr)
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    pc = build_point_cloud(pk, K, filter_thresh=0.05, min_views=2, voxel_size=0.01)
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    n_pix = idepth.size * 10
    keep, _ = opc.keep_mask(idepth, cov, 6.0, 10.0)
    n_max = int(keep.sum()) * 10                                        # the filter only removes points
    bound = 4 * n_pix + n_pix // 32 + (24 + 52) * n_max + 28 * len(pc) + (4 << 20)
    assert peak <= bound, (peak, bound)
    assert 1e7 < n_pix and int(pc.counts.sum()) <= n_max
