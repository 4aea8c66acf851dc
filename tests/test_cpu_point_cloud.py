"""SLAM point clouds without a GPU: the numpy restatement (tests/point_cloud_oracle.py) against the reference GUI's own
build_pcls (golden), against brute force and oracle/geom.py; the host paths of point_cloud.py, TsdfFusion and the GUI
packet with the oracle in place of the device passes; the PLY writer."""
import os
import types

import numpy as np
import pytest
import torch

from oracle import geom as ogeom
from tests import point_cloud_oracle as opc

HERE = os.path.dirname(os.path.abspath(__file__))
F32 = np.float32


def _golden():
    return dict(np.load(os.path.join(HERE, "golden", "ref_point_cloud.npz")))


@pytest.mark.parametrize("mode", ["uncertainty", "uniform"])
def test_oracle_reproduces_the_reference_build_pcls(mode):
    """selection and order exact, colours exact; positions to 1e-5 relative — the golden's pose comes from an fp32
    SE3 inverse (the lietorch stand-in), the oracle's from the fp32 rotation and fp32 centre -R^T t with fp64 products,
    so the last bits differ"""
    g = _golden()
    covs = g["covs"] if mode == "uncertainty" else None
    keep, _ = opc.keep_mask(g["idepths"], covs, g["max_depth"], g["max_depth_sigma"])
    kf, pix = np.nonzero(keep.reshape(len(keep), -1))
    assert np.array_equal(kf, g[f"{mode}_kf"]) and np.array_equal(pix, g[f"{mode}_pix"])
    P, C = opc.point_cloud(g["poses"], g["idepths"], covs, g["images"], g["intrinsics"], g["max_depth"], g["max_depth_sigma"])
    assert np.array_equal(C, g[f"{mode}_colors"])
    ref = g[f"{mode}_points"]
    assert np.abs(P - ref).max() <= 1e-5 * np.abs(ref).max()
    if mode == "uncertainty":
        assert (g["uncertainty_kf"] != 1).all()                    # the fully masked keyframe contributes nothing
    assert len(ref) < g["idepths"].size                             # zero / negative / NaN / beyond max_depth dropped


def test_oracle_downsampling_is_brute_force_grouping(rng):
    P = rng.normal(0, 0.4, (3000, 3)).astype(F32)
    P[:5] = np.nan                                                   # no voxel: dropped
    P[5] = [3.0e6, 0, 0]                                             # voxel beyond 2^20: dropped, not wrapped
    C = rng.uniform(0, 1, (3000, 3)).astype(F32)
    voxel = 0.1
    mp, mc, cnt, keys = opc.downsample(P, C, voxel)
    groups = {}
    for i, p in enumerate(P.astype(np.float64)):
        q = np.floor(p / np.float64(F32(voxel)))
        if not np.all(np.isfinite(q)) or np.any(np.abs(q) >= 2 ** 20):
            continue
        groups.setdefault((int(q[2]), int(q[1]), int(q[0])), []).append(i)     # z-major, as the packed key
    order = sorted(groups)
    assert len(order) == len(cnt) and cnt.sum() == 2994
    assert np.array_equal(cnt, [len(groups[k]) for k in order])
    assert np.all(keys[1:] > keys[:-1])
    for r, k in enumerate(order):
        assert ((int(keys[r]) >> 42) - 2 ** 20, ((int(keys[r]) >> 21) & 0x1FFFFF) - 2 ** 20, (int(keys[r]) & 0x1FFFFF) - 2 ** 20) == k
        idx = groups[k]
        assert np.allclose(mp[r], P[idx].astype(np.float64).mean(0), rtol=0, atol=1e-6)
        assert np.allclose(mc[r], C[idx].astype(np.float64).mean(0), rtol=0, atol=1e-6)
        assert np.all(np.floor(mp[r].astype(np.float64) / F32(voxel)) == [k[2], k[1], k[0]])


def _window(rng, n=8, H=20, W=24):
    from oracle import se3
    poses = se3.random_poses(rng, n, trans=0.05, rot_deg=2.0)
    idepth = rng.uniform(0.4, 0.6, (n, H, W)).astype(F32)
    return poses.astype(F32), idepth


def test_oracle_filter_counts_are_depth_filter_on_every_keyframe(rng):
    poses, idepth = _window(rng)
    intr = np.array([20.0, 20.0, 11.5, 9.5], F32)
    for thresh in (0.005, 0.05, 1.0):
        mine = opc.filter_counts(poses, idepth, intr, thresh)
        ref = ogeom.depth_filter(poses, idepth, intr, np.arange(len(poses)), np.full(len(poses), thresh, F32))
        assert np.array_equal(mine, ref)
        assert mine.max() <= 6
    assert opc.filter_counts(poses, idepth, intr, 1.0)[0].max() == 3     # frame 0 has the forward neighbours only


# ------------------------------------------------------------------------------------------------ host paths (oracle)
class OracleKernels:
    """point_cloud._CloudKernels restated on host tensors with the oracle; records its calls"""

    def __init__(self):
        self.calls = []

    def filter_counts(self, poses, idepths, intr, thresh):
        self.calls.append(("filter", float(thresh)))
        return torch.from_numpy(opc.filter_counts(poses.numpy(), idepths.numpy(), intr.numpy(), thresh).astype(F32))

    def cloud(self, poses, idepths, covs, images, intr, max_depth, max_sigma, views, min_views):
        self.calls.append(("cloud", covs is not None, intr.numpy().tolist(), float(max_depth), float(max_sigma),
                           views is not None, min_views))
        P, C = opc.point_cloud(poses.numpy(), idepths.numpy(), None if covs is None else covs.numpy(), images.numpy(),
                               intr.numpy(), max_depth, max_sigma, None if views is None else views.numpy(), min_views)
        return torch.from_numpy(P), torch.from_numpy(C)

    def downsample(self, points, colors, voxel_size):
        self.calls.append(("downsample", float(voxel_size)))
        p, c, n, _ = opc.downsample(points.numpy(), colors.numpy(), voxel_size)
        return torch.from_numpy(p), torch.from_numpy(c), torch.from_numpy(n)


@pytest.fixture
def kern(monkeypatch):
    from nerf_slam_b200 import point_cloud
    k = OracleKernels()
    monkeypatch.setattr(point_cloud, "kernels", k)
    return k


def _packet(rng, n=8, H=20, W=24, cov=True):
    poses, idepth = _window(rng, n, H, W)
    return {"cam0_poses": torch.from_numpy(poses), "cam0_idepths_up": torch.from_numpy(idepth),
            "cam0_depths_cov_up": torch.from_numpy(rng.uniform(0, 200, (n, H, W)).astype(F32)) if cov else None,
            "cam0_images": torch.from_numpy(rng.integers(0, 256, (n, 3, H, W)).astype(np.uint8))}


INTR = [20.0, 20.0, 11.5, 9.5]


def test_build_point_cloud_host_path_and_options(kern, rng):
    from nerf_slam_b200.point_cloud import build_point_cloud
    pk = _packet(rng)
    pc = build_point_cloud(pk, INTR)
    P, C = opc.point_cloud(pk["cam0_poses"].numpy(), pk["cam0_idepths_up"].numpy(), pk["cam0_depths_cov_up"].numpy(),
                           pk["cam0_images"].numpy(), INTR, 6.0, 10.0)
    assert pc.counts is None and np.array_equal(pc.points.numpy(), P) and np.array_equal(pc.colors.numpy(), C)
    assert 0 < len(pc) < pk["cam0_idepths_up"].numel()                              # the sigma mask dropped some
    assert kern.calls[-1] == ("cloud", True, INTR, 6.0, 10.0, False, 2)
    pc = build_point_cloud(pk, torch.tensor(INTR), filter_thresh=0.05, min_views=3, voxel_size=0.02, max_depth=2.2)
    assert [c[0] for c in kern.calls[-3:]] == ["filter", "cloud", "downsample"]
    assert kern.calls[-2][5:] == (True, 3) and abs(kern.calls[-3][1] - 0.05) < 1e-9
    assert pc.counts.dtype == torch.int32 and int(pc.counts.sum()) <= pk["cam0_idepths_up"].numel()


def test_build_point_cloud_refuses_bad_input(kern, rng):
    from nerf_slam_b200.point_cloud import build_point_cloud
    pk = _packet(rng)
    for v in (0.0, -0.01, float("nan"), float("inf")):
        with pytest.raises(ValueError, match="voxel_size"):
            build_point_cloud(pk, INTR, voxel_size=v)
    for m in (0, 7, 2.5):
        with pytest.raises(ValueError, match="min_views"):
            build_point_cloud(pk, INTR, filter_thresh=0.1, min_views=m)
    with pytest.raises(ValueError, match="cam0_poses"):
        build_point_cloud(dict(pk, cam0_poses=pk["cam0_poses"].double()), INTR)
    with pytest.raises(ValueError, match="cam0_images"):
        build_point_cloud(dict(pk, cam0_images=pk["cam0_images"][:, :, :-1]), INTR)
    with pytest.raises(ValueError, match="cam0_depths_cov_up"):
        build_point_cloud(dict(pk, cam0_depths_cov_up=pk["cam0_depths_cov_up"][:-1]), INTR)
    with pytest.raises(RuntimeError, match="contiguous"):
        build_point_cloud(dict(pk, cam0_idepths_up=pk["cam0_idepths_up"].transpose(1, 2).contiguous().transpose(1, 2)), INTR)
    with pytest.raises(ValueError, match="intrinsics"):
        build_point_cloud(pk, INTR[:3])
    big = {"cam0_poses": torch.empty(3, 7, device="meta"), "cam0_idepths_up": torch.empty(3, 30000, 30000, device="meta"),
           "cam0_depths_cov_up": None, "cam0_images": torch.empty(3, 3, 30000, 30000, dtype=torch.uint8, device="meta")}
    with pytest.raises(ValueError, match="int32"):
        build_point_cloud(big, INTR)
    assert kern.calls == []


def test_build_point_cloud_none_when_nothing_survives(kern, rng):
    from nerf_slam_b200.point_cloud import build_point_cloud
    pk = _packet(rng)
    assert build_point_cloud(dict(pk, cam0_idepths_up=torch.zeros_like(pk["cam0_idepths_up"])), INTR) is None
    assert build_point_cloud(dict(pk, cam0_depths_cov_up=torch.full_like(pk["cam0_depths_cov_up"], 1e4)), INTR) is None
    far = dict(pk, cam0_poses=torch.tensor([[0, 0, 0, 0, 0, 0, 1.0]]).repeat(8, 1).contiguous(),
               cam0_idepths_up=torch.full_like(pk["cam0_idepths_up"], 1e-7))
    assert build_point_cloud(far, INTR, max_depth=1e8, voxel_size=1.0) is None       # every voxel beyond 2^20: dropped
    assert build_point_cloud({k: v[:0] for k, v in pk.items()}, INTR) is None


def _fusion(rng, mode="sigma"):
    from nerf_slam_b200.tsdf_fusion import TsdfFusion
    fus = TsdfFusion(mode, types.SimpleNamespace(eval=False, tsdf_resolution=8), device="cpu")
    pk = _packet(rng, n=5)
    slam = dict(pk, is_last_frame=False, kf_idx=4, viz_idx=torch.arange(5), kf_idx_to_f_idx={i: 10 * i for i in range(5)},
                cam0_intrinsics=torch.tensor([INTR]).repeat(5, 1) / 8, gt_depths=torch.zeros(5, 1, 20, 24),
                calibs=[types.SimpleNamespace(depth_scale=1.0)])
    fus.fuse({"slam": [None, slam]})
    return fus, pk


@pytest.mark.parametrize("mode", ["sigma", "tsdf"])
def test_tsdf_fusion_point_cloud_from_history(kern, rng, monkeypatch, mode):
    from nerf_slam_b200.tsdf_fusion import TsdfFusion
    monkeypatch.setattr(TsdfFusion, "build_volume", lambda self, *a, **k: None)      # the volume is not read
    fus, pk = _fusion(rng, mode)
    pc = fus.build_point_cloud(voxel_size=0.05)
    covs = pk["cam0_depths_cov_up"].numpy() if mode == "sigma" else None
    P, C = opc.point_cloud(pk["cam0_poses"].numpy(), pk["cam0_idepths_up"].numpy(), covs, pk["cam0_images"].numpy(),
                           fus.intrinsics, fus.max_depth, fus.max_depth_sigma_thresh)
    p, c, n, _ = opc.downsample(P, C, 0.05)
    assert np.array_equal(pc.points.numpy(), p) and np.array_equal(pc.counts.numpy(), n)
    assert kern.calls[-2] == ("cloud", mode == "sigma", INTR, 6.0, 10000.0, False, 2)
    # the GUI packet: {"pcl": PointCloud} next to the mesh; without the key nothing changes
    out = fus.handle_gui_packet({"build_pcl": {"filter_thresh": 0.1, "min_views": 1}})
    assert list(out) == ["pcl"] and kern.calls[-1][0] == "cloud" and kern.calls[-1][5:] == (True, 1)
    n_calls = len(kern.calls)
    assert fus.handle_gui_packet({"depth_mask_type": "uniform"}) is None and len(kern.calls) == n_calls
    fus.handle_gui_packet({"build_pcl": True})
    assert kern.calls[-1][1] is False                                               # uniform: no sigma test
    fus.history.clear()
    assert fus.build_point_cloud() is None


def test_point_cloud_ply_round_trip(tmp_path, rng):
    from nerf_slam_b200.point_cloud import PointCloud
    P = rng.normal(size=(41, 3)).astype(F32)
    C = rng.uniform(size=(41, 3)).astype(F32)
    N = rng.integers(1, 100, 41).astype(np.int32)
    for counts in (None, N):
        path = str(tmp_path / "c.ply")
        PointCloud(torch.from_numpy(P), torch.from_numpy(C), None if counts is None else torch.from_numpy(counts)).write_ply(path)
        head, body = open(path, "rb").read().split(b"end_header\n", 1)
        lines = head.decode().splitlines()
        assert lines[:3] == ["ply", "format binary_little_endian 1.0", "element vertex 41"]
        props = [tuple(l.split()[1:]) for l in lines if l.startswith("property")]
        want = [("float", k) for k in ("x", "y", "z", "red", "green", "blue")] + ([("int", "count")] if counts is not None else [])
        assert props == want and not any(l.startswith("element face") for l in lines)
        vt = np.frombuffer(body, [(k, "<f4" if t == "float" else "<i4") for t, k in props])
        assert len(vt) == 41
        assert np.array_equal(np.stack([vt["x"], vt["y"], vt["z"]], 1), P)
        assert np.array_equal(np.stack([vt["red"], vt["green"], vt["blue"]], 1), C)
        if counts is not None:
            assert np.array_equal(vt["count"], N)
