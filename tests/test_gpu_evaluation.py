"""Reconstruction evaluation on the GPU (csrc/recon_eval.cu through nerf_slam_b200/evaluation.py) against the oracle
(tests/recon_eval_oracle.py: cKDTree, fp64 numpy): exact nearest neighbours on uniform, clustered, coincident and
far-away points and at 1 M x 4 M, invariance to the leaf size and the grid, bit-exact surface samples with a chi^2 test
of the area weighting, visibility, the fixed-point metric sums, and end to end on the synthetic room."""
import types

import numpy as np
import pytest
import torch
from scipy import stats

from tests import recon_eval_oracle as orc

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
F32 = np.float32


def _t(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def _cloud(rng, kind, n):
    if kind == "uniform":
        return rng.uniform(-2, 2, (n, 3)).astype(F32)
    if kind == "clustered":                                 # tight blobs, a few far outliers
        c = rng.uniform(-5, 5, (12, 3))
        p = c[rng.integers(0, 12, n)] + rng.normal(0, 0.01, (n, 3))
        p[rng.integers(0, n, max(1, n // 100))] *= 30
        return p.astype(F32)
    if kind == "coincident":                                # every point repeated 1-4 times, shuffled; a coarse grid
        base = rng.integers(-20, 20, (n // 3, 3)).astype(F32) * F32(0.05)
        p = base[rng.integers(0, len(base), n)]
        return p
    raise ValueError(kind)


def _check_nearest(query, ref, max_dist, dist, idx):
    od, oi, second = orc.nearest(query, ref, max_dist)
    d, i = dist.cpu().numpy(), idx.cpu().numpy()
    assert d.dtype == np.float32 and i.dtype == np.int64
    assert np.array_equal(d, od), np.flatnonzero(d != od)[:10]
    assert np.array_equal(i < 0, oi < 0)
    first = np.where(oi >= 0, od.astype(np.float64), np.inf)
    clear = (oi >= 0) & (second > first * (1 + 1e-6))       # the second neighbour strictly farther: index defined
    assert np.array_equal(i[clear], oi[clear])
    # ties: the smallest index among the reference points at exactly the kernel's distance
    tied = np.flatnonzero((oi >= 0) & ~clear)[:2000]
    if len(tied):
        q = query[tied].astype(np.float64)
        r = ref.astype(np.float64)
        for k, qi in enumerate(tied):
            e = q[k] - r
            d2 = (e[:, 0] * e[:, 0] + e[:, 1] * e[:, 1]) + e[:, 2] * e[:, 2]
            assert i[qi] == int(np.flatnonzero(d2 == d2.min())[0])
    return d, i


@pytest.mark.parametrize("kind", ["uniform", "clustered", "coincident"])
@pytest.mark.parametrize("max_dist", [np.inf, 0.05])
def test_nearest_matches_ckdtree(kind, max_dist):
    from nerf_slam_b200.evaluation import nearest
    rng = np.random.default_rng(11)
    ref = _cloud(rng, kind, 30000)
    query = np.concatenate([_cloud(rng, kind, 20000), ref[:500]])      # exact hits too
    dist, idx = nearest(_t(query), _t(ref), max_dist)
    d, _ = _check_nearest(query, ref, max_dist, dist, idx)
    if np.isfinite(max_dist):
        assert np.isinf(d).any() and np.isfinite(d).any()


def test_nearest_queries_beyond_max_dist_and_one_reference():
    from nerf_slam_b200.evaluation import nearest
    rng = np.random.default_rng(5)
    ref = np.array([[0.25, -1.0, 2.0]], F32)
    query = rng.uniform(-3, 3, (5000, 3)).astype(F32)
    for md in (np.inf, 2.0, 1e-3):
        dist, idx = nearest(_t(query), _t(ref), md)
        _check_nearest(query, ref, md, dist, idx)
    far = ref + F32(10)
    dist, idx = nearest(_t(far), _t(ref), 1.0)
    assert np.isinf(dist.cpu().numpy()).all() and (idx.cpu().numpy() == -1).all()
    # exactly at max_dist: not counted (strictly closer only, as cKDTree)
    dist, idx = nearest(_t(np.array([[1.25, -1.0, 2.0]], F32)), _t(ref), 1.0)
    assert int(idx[0]) == -1


def test_nearest_one_million_by_four_million():
    from nerf_slam_b200.evaluation import nearest
    rng = np.random.default_rng(2)
    ref = np.concatenate([rng.uniform(-3, 3, (700_000, 3)), _cloud(rng, "clustered", 300_000)]).astype(F32)
    query = rng.uniform(-3.5, 3.5, (4_000_000, 3)).astype(F32)
    dist, idx = nearest(_t(query), _t(ref), 0.5)
    od, oi, second = orc.nearest(query, ref, 0.5)
    d, i = dist.cpu().numpy(), idx.cpu().numpy()
    assert np.array_equal(d, od)
    clear = (oi >= 0) & (second > od.astype(np.float64) * (1 + 1e-6))
    assert clear.sum() > 0.99 * (oi >= 0).sum() and (oi < 0).any()
    assert np.array_equal(i[clear], oi[clear]) and np.array_equal(i < 0, oi < 0)


def test_nearest_is_invariant_to_leaf_size_and_grid():
    from nerf_slam_b200.evaluation import PointIndex
    rng = np.random.default_rng(8)
    ref = _t(np.concatenate([_cloud(rng, "coincident", 200_000), _cloud(rng, "clustered", 100_000)]))
    query = _t(np.concatenate([_cloud(rng, "uniform", 300_000), _cloud(rng, "clustered", 100_000)]))
    results = []
    for leaf in (1, 8):
        index = PointIndex(ref, leaf)
        for sms in (0, 7):
            results.append(index.query(query, 0.2, num_sms=sms))
    for d, i in results[1:]:
        assert torch.equal(d, results[0][0]) and torch.equal(i, results[0][1])


# ------------------------------------------------------------------------------------------------------------ sampling
def _random_mesh(rng, nt=3000):
    """triangles of very different sizes, some of zero area (repeated or collinear vertices)"""
    V = rng.normal(0, 1, (2 * nt, 3)).astype(F32)
    T = rng.integers(0, len(V), (nt, 3)).astype(np.int32)
    scale = np.exp(rng.uniform(-4, 1, nt))
    V[T[:, 1]] = V[T[:, 0]] + (V[T[:, 1]] - V[T[:, 0]]) * scale[:, None].astype(F32)
    T[::97, 1] = T[::97, 0]                                 # zero area
    return V, T


def test_sampling_is_deterministic_and_matches_the_oracle():
    from nerf_slam_b200.evaluation import sample_surface
    rng = np.random.default_rng(4)
    V, T = _random_mesh(rng)
    n = 1_000_000
    p1, t1 = sample_surface((_t(V), _t(T)), n, seed=9, return_triangles=True)
    p2, t2 = sample_surface((V, T), n, seed=9, return_triangles=True)
    assert torch.equal(p1, p2) and torch.equal(t1, t2)
    P, tri = p1.cpu().numpy(), t1.cpu().numpy()
    OP, otri = orc.surface_samples(V, T, n, seed=9)
    assert np.array_equal(tri, otri)
    ulp = np.spacing(np.maximum(np.abs(OP), np.abs(P)))
    assert np.all(np.abs(P - OP) <= ulp)
    assert not torch.equal(sample_surface((V, T), 1000, seed=10), p1[:1000])

    # on its triangle: barycentric coordinates of the fp64 least-squares fit in [0, 1], residual at fp32 rounding
    a, b, c = (V[T[tri, k]].astype(np.float64) for k in range(3))
    A = np.stack([b - a, c - a], 2)
    sol = np.linalg.solve(np.einsum("nij,nik->njk", A, A), np.einsum("nij,ni->nj", A, P - a)[..., None])[..., 0]
    res = np.linalg.norm(np.einsum("nij,nj->ni", A, sol) + a - P, axis=1)
    scale = np.abs(np.stack([a, b, c])).max((0, 2))
    assert np.all(res <= 4 * np.spacing(F32(1)) * scale + 1e-30)
    cross = np.linalg.norm(np.cross(b - a, c - a), axis=1)
    sane = cross > 1e-3 * np.linalg.norm(b - a, axis=1) * np.linalg.norm(c - a, axis=1)   # not near-collinear
    assert sane.mean() > 0.9
    assert sol[sane].min() >= -1e-4 and sol[sane].sum(1).max() <= 1 + 1e-4

    # area weighting: per-triangle counts against area (chi^2), zero-area triangles never chosen
    w, _ = orc.triangle_weights(V, T)
    counts = np.bincount(tri, minlength=len(T))
    assert counts[w == 0].sum() == 0 and (w == 0).sum() >= len(T) // 97
    exp = n * w.astype(np.float64) / w.astype(np.float64).sum()
    keep = exp >= 5
    chi2 = np.sum((counts[keep] - exp[keep]) ** 2 / exp[keep])
    assert stats.chi2.sf(chi2, keep.sum() - 1) > 1e-4


def test_sampling_refuses_bad_meshes():
    from nerf_slam_b200.evaluation import sample_surface
    V = np.zeros((3, 3), F32)
    with pytest.raises(ValueError, match="no area"):
        sample_surface((V, np.array([[0, 1, 2]], np.int32)), 10)
    with pytest.raises(ValueError, match="outside"):
        sample_surface((np.eye(3, dtype=F32), np.array([[0, 1, 3]], np.int32)), 10)
    Vn = np.eye(3, dtype=F32)
    Vn[0, 0] = np.nan
    with pytest.raises(ValueError, match="non-finite"):
        sample_surface((Vn, np.array([[0, 1, 2]], np.int32)), 10)


# --------------------------------------------------------------------------------------------- visibility and metrics
def _room_views(n_views=10, W=320, H=240, frames=40):
    """ground-truth views of the synthetic room -> room, cam_T_world [n,7], depths [n,H,W] (metres), images, intrinsics"""
    from nerf_slam_b200.frontend import matrix_to_tq
    from nerf_slam_b200.synthetic import SyntheticRoom
    room = SyntheticRoom(W, H, frames, seed=0)
    ks = range(0, frames, frames // n_views)
    poses, depths, images = [], [], []
    for k in ks:
        rgba, d16, w2c = room.render(k)
        poses.append(matrix_to_tq(np.asarray(w2c, np.float64)))
        depths.append(d16[..., 0].astype(F32) * F32(room.calib.depth_scale))
        images.append(rgba[..., :3].transpose(2, 0, 1))
    return (room, np.asarray(poses, F32), np.asarray(depths, F32), np.asarray(images, np.uint8),
            room.calib.camera_model.numpy().astype(F32))


def test_visibility_matches_the_oracle():
    from nerf_slam_b200.evaluation import sample_surface, visible
    room, poses, depths, _, intr = _room_views(12)
    P = sample_surface(room.surface_mesh(), 300_000, seed=1)
    Pn = P.cpu().numpy()
    rng = np.random.default_rng(0)
    inner = rng.uniform(-2.5, 2.5, (50_000, 3)).astype(F32)            # free space: occluded by nothing, seen or not
    for depth, tol, far in ((None, 0.05, np.inf), (depths, 0.05, np.inf), (depths, 0.0, 3.0)):
        for pts, pn in ((P, Pn), (_t(inner), inner)):
            got = visible(pts, _t(poses), intr, room.W, room.H, None if depth is None else _t(depth), tol, 0.0, far)
            ref = orc.visible(pn, poses, intr, room.W, room.H, depth, tol, 0.0, far)
            assert got.dtype == torch.bool and np.array_equal(got.cpu().numpy(), ref)
    m = visible(P, _t(poses), intr, room.W, room.H, _t(depths))
    assert 0.2 < float(m.float().mean()) < 0.9


def test_metrics_match_the_oracle_and_repeat_bit_for_bit():
    from nerf_slam_b200.evaluation import reconstruction_metrics
    rng = np.random.default_rng(3)
    gt = rng.uniform(-1, 1, (150_000, 3)).astype(F32)
    rec = (gt[:120_000] + rng.normal(0, 0.03, (120_000, 3))).astype(F32)
    rec[:500] += F32(5)                                     # outliers: clamped at max_dist, unmatched
    for thr, md in ((0.05, 1.0), (0.02, 0.1)):
        a = reconstruction_metrics(_t(rec), _t(gt), thr, max_dist=md)
        b = reconstruction_metrics(_t(rec), _t(gt), thr, max_dist=md)
        o = orc.metrics(rec, gt, thr, md)
        assert a == b
        for k, v in o.items():
            assert a[k] == v, k
        assert a["unmatched_reconstruction"] >= 500


# ---------------------------------------------------------------------------------------------------------- end to end
def _fused_room_meshes():
    from nerf_slam_b200.tsdf_fusion import TsdfFusion
    room, poses, depths, images, intr = _room_views(10, 640, 480, 40)
    meshes = {}
    for kind in ("dense", "blocks"):
        fus = TsdfFusion("tsdf", types.SimpleNamespace(eval=False, tsdf_volume=kind, tsdf_resolution=512), DEV)
        fus.voxel_size = 8.0 / 512                          # the 6 x 4 x 6 m room inside the dense grid's 8 m
        fus.initialize()
        pk = {"cam0_poses": _t(poses), "cam0_idepths_up": _t(1.0 / depths), "cam0_depths_cov_up": None,
              "cam0_images": _t(images)}
        fus.build_volume(pk, intr, None)
        meshes[kind] = fus.build_mesh(0.5)
        del fus
        torch.cuda.empty_cache()
    return room, poses, depths, intr, meshes


def test_tsdf_meshes_of_the_room_against_its_true_surface():
    """Dense and block TSDF (1.5625 cm voxels) fused from the ground-truth depth of 10 views of the synthetic room at
    640x480; their meshes against `surface_mesh()` culled to what those views saw (visible with the depth maps), 2 M
    samples a side (the culled ground truth keeps about a fifth), threshold 5 cm.  First run on an H100: dense accuracy
    4.64 mm, completion 2.27 mm, blocks 4.63 / 2.26 mm, precision = recall = 1.0 for both (accuracy is mostly the
    spacing of the culled ground-truth samples).  Bounds with margin: half a voxel (7.8 mm) and 0.99."""
    from nerf_slam_b200.evaluation import reconstruction_metrics, visible
    room, poses, depths, intr, meshes = _fused_room_meshes()
    cull = lambda p: visible(p, _t(poses), intr, room.W, room.H, _t(depths), 0.05)    # noqa: E731
    voxel = 8.0 / 512
    for kind, mesh in meshes.items():
        assert mesh is not None
        m = reconstruction_metrics(mesh, room.surface_mesh(), 0.05, n_samples=2_000_000, gt_mask=cull)
        print(kind, {k: (round(v, 6) if isinstance(v, float) else v) for k, v in m.items()})
        assert m["accuracy"] < voxel / 2 and m["completion"] < voxel / 2, (kind, m)
        assert m["recall"] >= 0.99 and m["precision"] >= 0.99, (kind, m)
        assert m["unmatched_reconstruction"] == m["unmatched_ground_truth"] == 0


def test_nerf_mesh_and_slam_cloud_metrics_equal_the_oracle():
    """the NeRF mesh (a random network's level set) and the SLAM point cloud of ground-truth keyframes, scored against
    the room's surface: reconstruction_metrics equals the oracle on the same downloaded inputs (samples bit-exact, so
    the fixed-point sums and counts are equal)"""
    from nerf_slam_b200 import pyngp
    from nerf_slam_b200.evaluation import reconstruction_metrics
    from nerf_slam_b200.point_cloud import build_point_cloud
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

    room, poses, depths, images, intr = _room_views(6, 160, 120, 30)
    cloud = build_point_cloud({"cam0_poses": _t(poses), "cam0_idepths_up": _t(1.0 / depths), "cam0_depths_cov_up": None,
                               "cam0_images": _t(images)}, intr, voxel_size=0.02)
    V, T = room.surface_mesh()
    n = 100_000
    gt = orc.surface_samples(V, T, n, seed=1)[0]
    for rec, rec_np in ((mesh, orc.surface_samples(mesh.vertices.cpu().numpy(), mesh.triangles.cpu().numpy(), n, 0)[0]),
                        (cloud, cloud.points.cpu().numpy())):
        got = reconstruction_metrics(rec, (V, T), 0.05, n_samples=n, max_dist=2.0, seed=0)
        want = orc.metrics(rec_np, gt, 0.05, 2.0)
        for k, v in want.items():
            assert got[k] == v, (k, got[k], v)
