"""NeRF mesh read-out without a GPU: the lattice rules of pyngp.mesh_lattice, the numpy restatement of lattice -> field
-> visibility -> mesh -> colour (tests/nerf_mesh_oracle.py) on analytic densities and the oracle network, and the host
paths of Testbed.marching_cubes / compute_*_marching_cubes_mesh / NerfFusion.build_mesh with that restatement standing in
for the kernels."""
import math
import types

import numpy as np
import pytest
import torch

from oracle import ngp as ongp
from tests import nerf_mesh_oracle as onm
from tests.test_cpu_tsdf_mesh import _edges

F32 = np.float32


# ---------------------------------------------------------------------------------------------------------- lattice rules
def test_lattice_spacing_and_dims():
    from nerf_slam_b200.pyngp import BoundingBox, mesh_lattice
    lo, h, dims = mesh_lattice(256, None, 4.0)                  # training box [-1.5, 2.5]^3
    assert lo.dtype == np.float32 and lo.tolist() == [-1.5] * 3
    assert h == np.float32(4.0 / 255) and dims == (256, 256, 256)
    lo, h, dims = mesh_lattice([33, 65, 17], BoundingBox([0.0, 0.1, 0.2], [1.0, 0.6, 0.45]), 4.0)
    assert h == np.float32(1.0 / 64)
    assert dims == (65, math.floor(0.5 * 64 + 1e-9) + 1, math.floor(0.25 * 64 + 1e-9) + 1) == (65, 33, 17)
    assert np.allclose(lo, [0.0, 0.1, 0.2])
    # extent not a multiple of h: floor
    _, h, dims = mesh_lattice(11, np.array([[0, 0, 0], [1.0, 0.35, 0.999]]), 1.0)
    assert h == np.float32(0.1) and dims == (11, 4, 10)


def test_lattice_clips_to_the_training_box():
    from nerf_slam_b200.pyngp import mesh_lattice
    lo, h, dims = mesh_lattice(101, [[-10, 0.0, -10], [10, 1.0, 0.5]], 2.0)     # box [-0.5, 1.5]^3
    assert lo.tolist() == [-0.5, 0.0, -0.5]
    assert h == np.float32(0.02) and dims == (101, 51, 51)


@pytest.mark.parametrize("resolution,aabb", [(1, None), (0, None), ([1, 1, 1], None), (64, [[3, 0, 0], [4, 1, 1]]),
                                             (64, [[0, 0, 0], [1, 0, 1]]), (64, [[0, 0.5, 0], [1, 0.2, 1]]),
                                             (64, [[np.nan, 0, 0], [1, 1, 1]])])
def test_lattice_rejects_empty_boxes_and_tiny_resolutions(resolution, aabb):
    from nerf_slam_b200.pyngp import mesh_lattice
    with pytest.raises(ValueError):
        mesh_lattice(resolution, aabb, 4.0)


def test_lattice_int32_guard():
    """worst case 3 vertices per point and 5 triangles per cube must fit int32: 750^3 passes, 760^3 and 800^3 fail"""
    from nerf_slam_b200.pyngp import mesh_lattice
    assert mesh_lattice(750, None, 4.0)[2] == (750, 750, 750)
    for r in (760, 800, 1024):
        with pytest.raises(ValueError, match="int32"):
            mesh_lattice(r, None, 4.0)
    assert mesh_lattice(1024, [[0, 0, 0], [1, 1, 0.1]], 4.0)[2] == (1024, 1024, 103)      # flat boxes may be finer


# ---------------------------------------------------------------------------------------------- restatement on analytic σ
def _ball_sigma(c, r0, k):
    return lambda p: np.exp(F32(k) * (F32(r0) - np.linalg.norm(np.asarray(p, np.float64) - c, axis=-1))).astype(F32)


def test_analytic_ball_mesh_is_closed_and_on_the_level_set():
    """sigma = exp(k (r0 - |p - c|)) with thresh 1: the level set is the sphere |p - c| = r0; every point observed ->
    a closed, consistently wound surface with Euler characteristic 2, vertices within h of r0, normals outward"""
    c, r0 = np.array([0.47, 0.52, 0.55]), 0.31
    lo, h, dims = np.array([0.1, 0.12, 0.15], F32), F32(0.02), (38, 39, 40)
    p = onm.lattice_points(lo, h, dims)
    fld = onm.field(_ball_sigma(c, r0, 6.0)(p), 1.0)
    V, F, C, N = onm.mesh(fld, np.ones_like(fld), lo, h)
    assert len(F) > 500 and np.all(C == 0)
    directed, undirected = _edges(F)
    assert all(m == 2 for m in undirected.values()) and all(m == 1 for m in directed.values())
    assert len(V) - len(undirected) + len(F) == 2
    rad = np.linalg.norm(V - c, axis=1)
    assert np.abs(rad - r0).max() < h
    assert np.all(np.sum(N * (V - c), 1) > 0)                                     # toward lower density
    a, b, cc = V[F[:, 0]], V[F[:, 1]], V[F[:, 2]]
    cr = np.cross(b - a, cc - a)
    area = np.linalg.norm(cr, axis=1)                       # 0 where a corner lies on the level set: coincident vertices
    assert (area > 0).mean() > 0.95
    assert np.all(np.sum(cr * ((a + b + cc) / 3 - c), 1)[area > 0] > 0)              # wound outward


def test_visibility_rule_on_a_hand_built_occupancy_array():
    """3 cascades (aabb_scale 4): a point reads the cell of cascade mip_from_pos(p); only that cell decides"""
    cascades, NC = 3, 128 ** 3
    dens = -np.ones(cascades * NC, F32)
    p = np.array([[0.25, 0.25, 0.25],          # cascade 0, cell (32,32,32)
                  [1.25, 0.5, 0.5],            # cascade 1: |p - 0.5| = 0.75 -> cell (((0.75 / 2) + 0.5) * 128 = 112, 64, 64)
                  [2.4, 0.5, 0.5],             # cascade 2, cell (((1.9 / 4) + 0.5) * 128 = 124.8 -> 124, 64, 64)
                  [2.6, 0.5, 0.5],             # outside every cascade
                  [0.25, 0.25, 0.75]], F32)    # cascade 0, cell (32,32,96): left unseen
    dens[32 + 128 * (32 + 128 * 32)] = 0.0
    dens[NC + 112 + 128 * (64 + 128 * 64)] = 3.0
    dens[2 * NC + 124 + 128 * (64 + 128 * 64)] = 0.0
    dens[32 + 128 * (32 + 128 * 96) + NC] = 0.0                                  # same cell, wrong cascade: no effect
    assert onm.visibility(p, dens, cascades).tolist() == [1, 1, 1, 0, 0]
    # the same rule as the ray marcher's cascade choice and cell lookup (oracle/ngp.py)
    rng = np.random.default_rng(0)
    q = rng.uniform(-1.7, 2.7, (400, 3)).astype(F32)
    dens2 = np.where(rng.uniform(size=dens.shape) < 0.5, 0.0, -1.0).astype(F32)
    bits = np.packbits(dens2 >= 0, bitorder="little")
    ref = [float(ongp.occupied(x, ongp._mip_from_pos(x, cascades), bits)) for x in q]
    assert onm.visibility(q, dens2, cascades).tolist() == ref


def test_unobserved_corners_are_not_meshed():
    c, r0 = np.array([0.5, 0.5, 0.5]), 0.3
    lo, h, dims = np.array([0.1, 0.1, 0.1], F32), F32(0.025), (33, 33, 33)
    p = onm.lattice_points(lo, h, dims)
    fld = onm.field(_ball_sigma(c, r0, 5.0)(p), 1.0)
    w = (p[..., 0] < 0.5).astype(F32)                                            # half the lattice observed
    V, F, _, _ = onm.mesh(fld, w, lo, h)
    assert len(F) > 100 and V[:, 0].max() < 0.5
    assert len(np.unique(F)) == len(V)                                           # no unreferenced vertex


def test_network_restatement_colours_and_srgb():
    P = ongp.init_params(4.0, seed=3)
    P["grid"] = P["grid"].half().float()
    V = np.array([[0.3, 0.4, 0.5], [0.6, 0.1, 0.2]], F32)
    N = np.array([[0, 0, 1], [0, 0, 0]], F32)
    rec = onm.color_records(V, N, 4.0)
    assert rec[:, 3].tolist() == [0, 0] and rec[0, 4:].tolist() == [0, 0, -1] and rec[1, 4:].tolist() == [0, 0, 1]
    assert np.array_equal(rec[:, :3], ((V - F32(-1.5)) * F32(0.25)).astype(F32))
    lin = onm.network_colors(P, 4.0, V, N)
    srgb = onm.network_colors(P, 4.0, V, N, srgb=True)
    back = ongp.srgb_to_linear(torch.from_numpy(srgb)).numpy()
    assert np.allclose(back, lin, rtol=1e-5, atol=1e-7)
    x = np.array([0.0, 0.002, 0.0031308, 0.01, 0.5, 1.0], F32)
    assert np.allclose(onm.linear_to_srgb(x), [0, 0.002 * 12.92, 0.0031308 * 12.92, 1.055 * 0.01 ** (1 / 2.4) - 0.055,
                                               1.055 * 0.5 ** (1 / 2.4) - 0.055, 1.0], atol=1e-6)


# ------------------------------------------------------------------------------------ host paths with the restatement
class OracleMeshKernels:
    """the three device passes of Testbed.marching_cubes on CPU tensors, computed by the restatement; `sigma` maps
    points [...,3] to densities (default: the oracle network of the testbed's weights)"""

    def __init__(self, sigma=None):
        self.sigma = sigma
        self.calls = []

    def lattice(self, tb, lo, h, dims, thresh):
        self.calls.append(("lattice", tuple(lo.tolist()), float(h), dims, thresh))
        p = onm.lattice_points(lo, h, dims)
        sig = self.sigma or onm.network_sigma(onm.network_params(tb.grid_half, tb.mlp), tb.aabb_scale)
        return (torch.from_numpy(onm.field(sig(p), thresh)),
                torch.from_numpy(onm.visibility(p, tb.density.numpy(), tb.cascades)))

    def mesh(self, field, weight, lo, h):
        from nerf_slam_b200.tsdf_fusion import TsdfMesh
        V, F, C, N = onm.mesh(field.numpy(), weight.numpy(), lo, h)
        self.calls.append(("mesh", len(F)))
        if len(F) == 0:
            return None
        return TsdfMesh(*(torch.from_numpy(a) for a in (V, F, C, N)))

    def colors(self, tb, mesh, srgb):
        self.calls.append(("colors", srgb))
        P = onm.network_params(tb.grid_half, tb.mlp)
        mesh.vertex_colors = torch.from_numpy(onm.network_colors(P, tb.aabb_scale, mesh.vertices.numpy(),
                                                                 mesh.vertex_normals.numpy(), srgb))


def _cpu_testbed(monkeypatch, sigma=None, seen=True):
    from nerf_slam_b200 import pyngp
    tb = object.__new__(pyngp.Testbed)
    tb.aabb_scale, tb.cascades = 4.0, 3
    P = ongp.init_params(4.0, seed=1)
    tb.grid_half = P["grid"].reshape(-1).half()
    tb.mlp = torch.cat([P[k].reshape(-1) for k in ("W1", "W2", "W3", "W4", "W5")])
    tb.density = torch.full((3 * 128 ** 3,), 0.0 if seen else -1.0)
    monkeypatch.setattr(pyngp.Testbed, "mesh_kernels", OracleMeshKernels(sigma))
    return tb


def _ball(c=(0.45, 0.55, 0.5), r0=0.3):
    return _ball_sigma(np.asarray(c), r0, 8.0)


def test_testbed_mesh_front_doors(monkeypatch, tmp_path):
    tb = _cpu_testbed(monkeypatch, sigma=_ball())
    out = tb.compute_marching_cubes_mesh(resolution=[20, 41, 3], aabb=[[0.05, 0.1, 0.1], [0.85, 0.95, 0.9]], thresh=1.0)
    assert sorted(out) == ["C", "F", "N", "V"]
    assert out["F"].dtype == np.int32 and out["V"].dtype == np.float32 and out["V"].shape == out["C"].shape == out["N"].shape
    assert len(out["F"]) > 100
    assert np.abs(np.linalg.norm(out["V"] - np.array([0.45, 0.55, 0.5]), axis=1) - 0.3).max() < 0.85 / 40
    calls = tb.mesh_kernels.calls
    assert calls[0][0] == "lattice" and calls[0][2] == np.float32(0.85 / 40) and calls[0][4] == 1.0
    assert calls[-1] == ("colors", False)                                         # linear: what the network outputs
    P = onm.network_params(tb.grid_half, tb.mlp)
    assert np.array_equal(out["C"], onm.network_colors(P, 4.0, out["V"], out["N"]))
    path = str(tmp_path / "m.ply")
    tb.compute_and_save_marching_cubes_mesh(path, resolution=[20, 41, 3], aabb=[[0.05, 0.1, 0.1], [0.85, 0.95, 0.9]],
                                            thresh=1.0)
    V, N, C, F = onm.read_ply(path)
    assert np.array_equal(V, out["V"]) and np.array_equal(N, out["N"]) and np.array_equal(C, out["C"])
    assert np.array_equal(F, out["F"])
    with pytest.raises(ValueError):
        tb.compute_marching_cubes_mesh(resolution=1)


def test_testbed_network_density_and_the_empty_mesh(monkeypatch, tmp_path):
    """the oracle network's own density: with nothing observed no cube is meshed -> empty arrays and an empty PLY"""
    tb = _cpu_testbed(monkeypatch, seen=False)
    out = tb.compute_marching_cubes_mesh(resolution=24, thresh=0.5)
    assert out["V"].shape == (0, 3) and out["F"].shape == (0, 3) and out["F"].dtype == np.int32
    assert tb.mesh_kernels.calls[-1] == ("mesh", 0)
    assert tb.marching_cubes(24, None, 0.5) is None
    path = str(tmp_path / "empty.ply")
    tb.compute_and_save_marching_cubes_mesh(path, resolution=24, thresh=0.5)
    V, N, C, F = onm.read_ply(path)
    assert V.shape == (0, 3) and F.shape == (0, 3)
    # observed everywhere: the random network's level set at its median density gives a mesh whose colours follow it
    tb = _cpu_testbed(monkeypatch)
    sig = onm.network_sigma(onm.network_params(tb.grid_half, tb.mlp), 4.0)(onm.lattice_points([-1.5] * 3, 4 / 23, (24,) * 3))
    out = tb.compute_marching_cubes_mesh(resolution=24, thresh=float(np.median(sig)))
    assert len(out["F"]) > 0 and np.all((out["C"] > 0) & (out["C"] < 1))


def _nerf_fusion(tb):
    from nerf_slam_b200.nerf_fusion import NerfFusion
    nf = object.__new__(NerfFusion)
    nf.ngp, nf.mask_type, nf.ref_frames, nf.evaluate = tb, "ours", {}, False
    nf.linear_training_colors = True
    return nf


def test_nerf_fusion_build_mesh_colour_convention_per_ingest_path(monkeypatch):
    from nerf_slam_b200 import pyngp
    tb = _cpu_testbed(monkeypatch, sigma=_ball())
    tb.device = "cpu"
    ingested = []
    tb.nerf = types.SimpleNamespace(training=types.SimpleNamespace(
        optimize_extrinsics=True,
        update_training_images=lambda *a: ingested.append("data"),
        update_training_images_device=lambda *a, **k: ingested.append("slam")))
    nf = _nerf_fusion(tb)
    H, W = 4, 5
    calib = types.SimpleNamespace(camera_model=torch.tensor([3.0, 3.0, 2.0, 1.5]), depth_scale=1.0,
                                  aabb=np.array([[-1.0, -1, -1], [1, 1, 1]]), resolution=torch.tensor([W, H]))
    data = {"calibs": [calib], "poses": np.eye(4)[None], "depths": np.ones((1, H, W), F32), "k": np.array([0]),
            "images": np.full((1, H, W, 4), 128, np.uint8)}
    slam = {"viz_idx": torch.tensor([0]), "cam0_images": torch.zeros(1, 3, H, W, dtype=torch.uint8),
            "cam0_idepths_up": torch.ones(1, H, W), "cam0_depths_cov_up": torch.ones(1, H, W), "calibs": [calib],
            "cam0_poses": torch.tensor([[0, 0, 0, 0, 0, 0, 1.0]])}
    args = dict(resolution=24, thresh=1.0, aabb=[[0.0, 0.1, 0.1], [0.9, 0.9, 0.95]])
    for ingest, convention, srgb in [(nf.process_data, "reference", False), (nf.process_slam, None, True),
                                     (nf.process_data, "metric", True), (nf.process_data, "reference", False)]:
        if convention:
            nf.gt_fit_convention = convention
        ingest(data if ingest == nf.process_data else [None, slam])
        mesh = nf.build_mesh(**args)
        assert tb.mesh_kernels.calls[-1] == ("colors", srgb)
        assert isinstance(mesh.vertices, torch.Tensor) and mesh.triangles.dtype == torch.int32
        P = onm.network_params(tb.grid_half, tb.mlp)
        ref = onm.network_colors(P, 4.0, mesh.vertices.numpy(), mesh.vertex_normals.numpy(), srgb)
        assert np.array_equal(mesh.vertex_colors.numpy(), ref)
    assert ingested == ["data", "slam", "data", "data"]
    # nothing observed: None, like TsdfFusion.build_mesh
    tb.density.fill_(-1.0)
    assert nf.build_mesh(**args) is None
    assert isinstance(tb, pyngp.Testbed)
