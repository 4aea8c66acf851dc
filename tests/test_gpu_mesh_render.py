"""The triangle-mesh renderer on the GPU (csrc/mesh_render.cu through nerf_slam_b200/mesh_render.py) against the
brute-force oracle (tests/mesh_render_oracle.py, run on torch fp64 for the large cases) bit for bit, its independence of
the tree and the grid, the synthetic room's closed form, watertightness, agreement with the TSDF ray cast, and the
depth metric built on it."""
import types

import numpy as np
import pytest
import torch

from tests import mesh_render_oracle as orc
from tests import recon_eval_oracle as eval_orc

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
F32 = np.float32


def _t(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def _look_at(eye, target):
    """cam_T_world [7] (t, q_xyzw) of a camera at eye looking at target, y down (the synthetic room's convention)"""
    from nerf_slam_b200.frontend import matrix_to_tq
    eye, target = np.asarray(eye, np.float64), np.asarray(target, np.float64)
    fwd = (target - eye) / np.linalg.norm(target - eye)
    right = np.cross(fwd, [0.0, -1.0, 0.0])
    right /= np.linalg.norm(right)
    down = np.cross(fwd, right)
    c2w = np.eye(4)
    c2w[:3, 0], c2w[:3, 1], c2w[:3, 2], c2w[:3, 3] = right, down, fwd, eye
    return matrix_to_tq(np.linalg.inv(c2w)).astype(F32)


def _check_exact(V, T, C, poses, intr, W, H, pixels=None, **kw):
    from nerf_slam_b200.mesh_render import MeshScene
    out = MeshScene((_t(V), _t(T), _t(C))).render(_t(poses), intr, W, H, normals=True, colors=True, **kw)
    d, t, n, c = orc.render(_t(V), T, poses, intr, W, H, colors=C, pixels=pixels, xp="torch",
                            near=kw.get("near", 0.0), far=kw.get("far", np.inf), cull=kw.get("cull_backfaces", False))
    sel = (slice(None),) if pixels is None else (slice(None), np.asarray(pixels))
    got = [x.reshape(len(poses), H * W, *x.shape[3:]).cpu().numpy()[sel] for x in (out.depth, out.triangle, out.normal,
                                                                                     out.color)]
    assert np.array_equal(got[1], t), np.argwhere(got[1] != t)[:10]
    for g, w in zip((got[0], got[2], got[3]), (d, n, c)):
        assert np.array_equal(g, w)
    return out, t


def _soup(rng, nt=3000):
    """triangles of very different sizes about (0, 0, 0), some of zero area (repeated or collinear vertices)"""
    V = rng.normal(0, 1, (2 * nt, 3)).astype(F32)
    T = rng.integers(0, len(V), (nt, 3)).astype(np.int32)
    scale = np.exp(rng.uniform(-4, 1, nt))
    V[T[:, 1]] = V[T[:, 0]] + (V[T[:, 1]] - V[T[:, 0]]) * scale[:, None].astype(F32)
    T[::97, 1] = T[::97, 0]                                 # zero area
    T[1::89, 2] = T[1::89, 1]
    C = rng.uniform(0, 1, (len(V), 3)).astype(F32)
    return V, T, C


SOUP_POSES = [((0, 0, -4), (0, 0, 0)), ((3, 1, 2), (0.2, 0, 0)), ((0.3, 0.2, 0.1), (1, 0.5, 2))]   # the last inside


def test_random_soup_matches_the_oracle_bit_for_bit():
    rng = np.random.default_rng(0)
    V, T, C = _soup(rng)
    poses = np.stack([_look_at(e, c) for e, c in SOUP_POSES])
    intr = [60.0, 60.0, 47.5, 35.5]
    _, tri = _check_exact(V, T, C, poses, intr, 96, 72)
    assert (tri >= 0).mean() > 0.3
    _, tri = _check_exact(V, T, C, poses, intr, 96, 72, cull_backfaces=True, near=0.5, far=4.0)
    assert (tri >= 0).any() and (tri < 0).any()


def test_nerf_mesh_matches_the_oracle_bit_for_bit():
    from nerf_slam_b200 import pyngp
    from nerf_slam_b200.pyngp import mesh_lattice
    tb = pyngp.Testbed(seed=4, max_samples=1 << 16, max_rays=1 << 13)
    tb.create_empty_nerf_dataset(8, 1.0, None, 4, None)
    g = torch.Generator().manual_seed(4)
    tb.grid_master.copy_(((torch.rand(tb.grid_master.shape, generator=g) * 2 - 1) * 0.5).to(DEV))
    tb.grid_half.copy_(tb.grid_master.half())
    tb.pack_weights()
    tb.density.copy_(torch.where(torch.rand(tb.density.shape, generator=g) < 0.7, 0.0, -1.0).to(DEV))
    lo, h, dims = mesh_lattice(48, None, tb.aabb_scale)
    field, weight = tb.mesh_kernels.lattice(tb, lo, h, dims, 0.0)
    mesh = tb.marching_cubes(48, None, float(torch.quantile(-field[weight > 0], 0.5)))
    assert mesh is not None
    V, T, C = (x.cpu().numpy() for x in (mesh.vertices, mesh.triangles, mesh.vertex_colors))
    centre, ext = (V.min(0) + V.max(0)) / 2, float((V.max(0) - V.min(0)).max())
    poses = np.stack([_look_at(centre + ext * np.array(e), centre) for e in ((0, 0.3, -1.5), (1.2, -0.4, 0.6))])
    _, tri = _check_exact(V, T, C, poses, [70.0, 70.0, 39.5, 29.5], 80, 60)
    assert (tri >= 0).mean() > 0.1


def test_large_mesh_matches_the_oracle_on_sampled_pixels():
    rng = np.random.default_rng(1)
    V, T, C = _soup(rng, 300_000)
    V *= F32(3)
    poses = np.stack([_look_at((0.5, 0.4, -9), (0, 0, 0)), _look_at((0.2, 0.1, 0.3), (4, 1, 1))])
    W, H = 320, 240
    pixels = rng.choice(W * H, 1500, replace=False)
    _, tri = _check_exact(V, T, C, poses, [200.0, 200.0, 159.5, 119.5], W, H, pixels=pixels)
    assert (tri >= 0).mean() > 0.5


def test_same_bits_for_every_leaf_size_and_grid():
    from nerf_slam_b200.mesh_render import MeshScene
    rng = np.random.default_rng(2)
    V, T, C = _soup(rng, 20_000)
    poses = _t(np.stack([_look_at(e, c) for e, c in SOUP_POSES]))
    mesh = (_t(V), _t(T), _t(C))
    ref = None
    for leaf in (1, 4, 16):
        scene = MeshScene(mesh, leaf)
        for sms in (0, 7, 0):
            out = scene.render(poses, [150.0, 150.0, 159.5, 119.5], 320, 240, normals=True, colors=True, num_sms=sms)
            got = (out.depth, out.triangle, out.normal, out.color)
            if ref is None:
                ref = got
                assert (out.triangle >= 0).any()
            assert all(torch.equal(a, b) for a, b in zip(got, ref)), (leaf, sms)


# ----------------------------------------------------------------------------------------------------- synthetic room
def _room(n_views=10, W=640, H=480, frames=40):
    from nerf_slam_b200.frontend import matrix_to_tq
    from nerf_slam_b200.synthetic import SyntheticRoom
    room = SyntheticRoom(W, H, frames, seed=0)
    ks = list(range(0, frames, frames // n_views))[:n_views]
    poses = np.asarray([matrix_to_tq(np.asarray(room.render(k)[2], np.float64)) for k in ks], F32)
    return room, ks, poses, room.calib.camera_model.numpy().astype(F32)


def _room_depth(room, k):
    """the room's closed-form ray cast of view k in fp64 (SyntheticRoom.render's t)"""
    T = room.c2w(k)
    d = room.dirs_cam @ T[:3, :3].T
    o = T[:3, 3]
    with np.errstate(divide="ignore"):
        tt = np.where(d > 0, (room.ext - o) / d, (-room.ext - o) / d)
    return tt.min(-1)


def test_room_mesh_against_the_closed_form():
    from nerf_slam_b200.mesh_render import MeshScene
    room, ks, poses, intr = _room()
    out = MeshScene(room.surface_mesh()).render(_t(poses), intr, room.W, room.H)
    depth = out.depth.cpu().numpy().astype(np.float64)
    assert (out.triangle >= 0).all()
    scale = room.calib.depth_scale
    for i, k in enumerate(ks):
        exact = _room_depth(room, k)
        assert np.abs(depth[i] - exact).max() <= 1e-5
        d16 = room.render(k)[1][..., 0].astype(np.float64)
        assert np.all(d16 * scale <= depth[i] + 1e-5) and np.all(depth[i] < (d16 + 1) * scale + 1e-5)


def test_watertight_grid_and_closed_icosphere():
    from nerf_slam_b200.mesh_render import MeshScene
    # a 32 x 32 grid of squares at z = 2 whose vertices and edges lie exactly on the pixel rays of a 33 x 33 view
    n = 32
    g = (np.arange(n + 1) - n // 2) / 8.0
    X, Y = np.meshgrid(g, g)
    V = np.stack([X, Y, np.full_like(X, 2.0)], -1).reshape(-1, 3).astype(F32)
    i = np.arange(n)[:, None] * (n + 1) + np.arange(n)[None, :]
    q = np.stack([i, i + 1, i + n + 2, i + n + 1], -1).reshape(-1, 4)
    T = np.concatenate([q[:, [0, 1, 2]], q[:, [0, 2, 3]]]).astype(np.int32)
    out = MeshScene((V, T)).render(_t(np.array([[0, 0, 0, 0, 0, 0, 1]], F32)), [16.0, 16.0, 16.0, 16.0], 33, 33)
    assert (out.triangle >= 0).all() and (out.depth == 2.0).all()

    # an icosphere (4 subdivisions) seen from inside: no ray escapes
    t = (1 + 5 ** 0.5) / 2
    Vs = [(-1, t, 0), (1, t, 0), (-1, -t, 0), (1, -t, 0), (0, -1, t), (0, 1, t), (0, -1, -t), (0, 1, -t), (t, 0, -1),
          (t, 0, 1), (-t, 0, -1), (-t, 0, 1)]
    Fs = [(0, 11, 5), (0, 5, 1), (0, 1, 7), (0, 7, 10), (0, 10, 11), (1, 5, 9), (5, 11, 4), (11, 10, 2), (10, 7, 6),
          (7, 1, 8), (3, 9, 4), (3, 4, 2), (3, 2, 6), (3, 6, 8), (3, 8, 9), (4, 9, 5), (2, 4, 11), (6, 2, 10), (8, 6, 7),
          (9, 8, 1)]
    Vs = [np.asarray(v, np.float64) / np.linalg.norm(v) for v in Vs]
    for _ in range(4):
        mid, F2 = {}, []

        def m(a, b):
            key = (min(a, b), max(a, b))
            if key not in mid:
                p = Vs[a] + Vs[b]
                Vs.append(p / np.linalg.norm(p))
                mid[key] = len(Vs) - 1
            return mid[key]
        for a, b, c in Fs:
            ab, bc, ca = m(a, b), m(b, c), m(c, a)
            F2 += [(a, ab, ca), (b, bc, ab), (c, ca, bc), (ab, bc, ca)]
        Fs = F2
    Vs, Fs = np.asarray(Vs, F32), np.asarray(Fs, np.int32)
    rng = np.random.default_rng(3)
    poses = np.concatenate([rng.uniform(-0.2, 0.2, (6, 3)), rng.normal(0, 1, (6, 4))], 1).astype(F32)
    poses[:, 3:] /= np.linalg.norm(poses[:, 3:], axis=1, keepdims=True)
    out = MeshScene((Vs, Fs)).render(_t(poses), [100.0, 100.0, 127.5, 95.5], 256, 192)
    assert (out.triangle >= 0).all()


# -------------------------------------------------------------------------------------------------- TSDF and metrics
def _fused_room_mesh(room, ks, poses, intr):
    from nerf_slam_b200.tsdf_fusion import TsdfFusion
    depths = np.stack([room.render(k)[1][..., 0].astype(F32) * F32(room.calib.depth_scale) for k in ks])
    images = np.stack([room.render(k)[0][..., :3].transpose(2, 0, 1) for k in ks])
    fus = TsdfFusion("tsdf", types.SimpleNamespace(eval=False, tsdf_volume="dense", tsdf_resolution=512), DEV)
    fus.voxel_size = 8.0 / 512
    fus.initialize()
    pk = {"cam0_poses": _t(poses), "cam0_idepths_up": _t(1.0 / depths), "cam0_depths_cov_up": None,
          "cam0_images": _t(images)}
    fus.build_volume(pk, intr, None)
    return fus, pk, depths


def test_tsdf_mesh_agrees_with_the_tsdf_ray_cast_and_the_depth_metric_with_the_oracle():
    from nerf_slam_b200.evaluation import mesh_depth_l1
    from nerf_slam_b200.mesh_render import MeshScene
    room, ks, poses, intr = _room()
    fus, pk, _ = _fused_room_mesh(room, ks, poses, intr)
    mesh = fus.build_mesh(0.5)
    ray_depth, _ = fus.render_volume(pk, intr, fus.min_weight_for_render, fus.max_depth_sigma_thresh)
    scene = MeshScene(mesh)
    out = scene.render(_t(poses), intr, room.W, room.H)
    both = (out.triangle >= 0) & (ray_depth > 0)
    assert float(both.float().mean()) > 0.5
    assert float((out.depth - ray_depth).abs()[both].median()) < fus.voxel_size / 2

    # the metric against the room's surface: its fixed-point sum equals the oracle's over the same depths
    gt = MeshScene(room.surface_mesh())
    m = mesh_depth_l1(scene, gt, _t(poses), intr, room.W, room.H, max_dist=1.0)
    g = gt.render(_t(poses), intr, room.W, room.H)
    dr, dg = out.depth.cpu().numpy(), g.depth.cpu().numpy()
    hr, hg = out.triangle.cpu().numpy() >= 0, g.triangle.cpu().numpy() >= 0
    diff = np.where(hr & hg, np.abs(dr - dg), F32(0)).astype(F32)
    s, _, _ = eval_orc.metric_sums(diff.reshape(-1), 1.0, 1.0)
    assert m["depth_l1_fixed"] == s and m["both_hits"] == int((hr & hg).sum()) and m["gt_hits"] == int(hg.sum())
    assert m["missing"] == int((hg & ~hr).sum()) and m["extra"] == int((hr & ~hg).sum())
    assert 0 < m["depth_l1"] < fus.voxel_size
    # the rendered TSDF mesh itself against the brute-force oracle on sampled pixels
    rng = np.random.default_rng(4)
    pixels = rng.choice(room.W * room.H, 800, replace=False)
    V, T = mesh.vertices, mesh.triangles
    od, ot, _, _ = orc.render(V, T.cpu().numpy(), poses[:2], intr, room.W, room.H, pixels=pixels, xp="torch")
    assert np.array_equal(dr[:2].reshape(2, -1)[:, pixels], od)
    assert np.array_equal(out.triangle.cpu().numpy()[:2].reshape(2, -1)[:, pixels], ot)


def test_room_metric_against_itself_and_culling_with_rendered_depth():
    from nerf_slam_b200.evaluation import mesh_depth_l1, sample_surface, visible
    from nerf_slam_b200.mesh_render import MeshScene
    room, ks, poses, intr = _room(6, 320, 240, 30)
    m = mesh_depth_l1(room.surface_mesh(), room.surface_mesh(), _t(poses), intr, room.W, room.H)
    assert m["depth_l1"] == 0 and m["depth_l1_fixed"] == 0 and m["missing"] == m["extra"] == 0
    assert m["gt_hits"] == m["both_hits"] == 6 * room.W * room.H

    rendered = MeshScene(room.surface_mesh()).render(_t(poses), intr, room.W, room.H).depth
    exact = np.stack([_room_depth(room, k) for k in ks]).astype(F32)
    P = sample_surface(room.surface_mesh(), 200_000, seed=5)
    tol = 0.05
    a = visible(P, _t(poses), intr, room.W, room.H, depths=rendered, depth_tol=tol).cpu().numpy()
    b = visible(P, _t(poses), intr, room.W, room.H, depths=_t(exact), depth_tol=tol).cpu().numpy()
    assert 0.1 < a.mean() < 0.95
    differ = np.flatnonzero(a != b)
    if len(differ):                                         # only points at the tolerance boundary, within one quantum
        Pn = P.cpu().numpy()[differ].astype(np.float64)
        quantum = room.calib.depth_scale
        near_boundary = np.zeros(len(differ), bool)
        for k, pose in enumerate(poses):
            R = eval_orc._rotation_f32(pose[3:])
            pc = Pn @ R.T + pose[:3].astype(np.float64)
            u = np.floor(intr[0] * pc[:, 0] / pc[:, 2] + intr[2] + 0.5)
            v = np.floor(intr[1] * pc[:, 1] / pc[:, 2] + intr[3] + 0.5)
            ok = (pc[:, 2] > 0) & (u >= 0) & (u < room.W) & (v >= 0) & (v < room.H)
            d = np.zeros(len(differ))
            d[ok] = exact[k][v[ok].astype(int), u[ok].astype(int)]
            near_boundary |= ok & (np.abs(pc[:, 2] - (d + tol)) <= quantum)
        assert near_boundary.all(), differ[~near_boundary][:10]
    assert len(differ) < 1e-3 * len(a)
