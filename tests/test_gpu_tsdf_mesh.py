"""TSDF read-outs on the GPU (csrc/tsdf_mesh.cu via TsdfFusion.build_mesh / render_volume) against the numpy restatements in
tests/tsdf_readout_oracle.py, and end to end on the synthetic room."""
import csv
import os
import types

import numpy as np
import pytest
import torch
from scipy.spatial.transform import Rotation

from tests import tsdf_readout_oracle as orc

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
F32 = np.float32
HERE = os.path.dirname(os.path.abspath(__file__))


def _fusion(t, w, c, origin, vs):
    from nerf_slam_b200.tsdf_fusion import DenseVolume, TsdfFusion
    fus = TsdfFusion("tsdf", types.SimpleNamespace(eval=False, tsdf_resolution=2), DEV)
    T = lambda a: torch.from_numpy(np.ascontiguousarray(a, F32)).to(DEV)
    fus.volume, fus.voxel_size = DenseVolume.from_tensors(T(t), T(w), T(c), origin, vs), float(vs)
    return fus


def _sphere_partial():
    nz, ny, nx, vs = 43, 41, 37, 0.05
    c, r = np.array([18.3, 20.6, 21.2]), 9.3
    k, j, i = np.meshgrid(np.arange(nz), np.arange(ny), np.arange(nx), indexing="ij")
    d = np.sqrt((i - c[0]) ** 2 + (j - c[1]) ** 2 + (k - c[2]) ** 2)
    rng = np.random.default_rng(11)
    w = rng.uniform(0, 2, d.shape).astype(F32)
    w[rng.uniform(size=d.shape) < 0.6] = 5.0
    col = rng.uniform(0, 255, d.shape + (3,)).astype(F32)
    t = np.clip((d - r) * vs / 0.10, -1, 1).astype(F32)
    return t, w, col, np.array([-0.9, -1.0, 0.3], F32), vs


def _golden(tag):
    g = np.load(os.path.join(HERE, "golden", "ref_tsdf_integrate.npz"))
    return (g[f"{tag}_w20.0_tsdf_2"], g[f"{tag}_w20.0_weight_2"], g[f"{tag}_w20.0_color_2"], g["origin"],
            float(g["voxel_size"]))


def _sin_dense():
    nz, ny, nx = 100, 96, 128                             # > 4096 blocks of 256 voxels: the scan runs over two chunks
    k, j, i = np.meshgrid(np.arange(nz), np.arange(ny), np.arange(nx), indexing="ij")
    t = (np.sin(0.9 * i + 0.3) * np.sin(0.7 * j + 0.1) * np.sin(1.1 * k + 0.2)).astype(F32)
    rng = np.random.default_rng(5)
    w = np.ones_like(t)
    col = rng.uniform(0, 255, t.shape + (3,)).astype(F32)
    return t, w, col, np.array([-3.0, -2.4, 0.5], F32), 0.05


VOLUMES = {"sphere_partial": _sphere_partial, "golden_sigma": lambda: _golden("sigma"),
           "golden_tsdf": lambda: _golden("tsdf"), "sin_dense": _sin_dense}
MIN_W = 0.5


@pytest.mark.parametrize("name", sorted(VOLUMES))
def test_dense_volume_mesh_matches_oracle(name):
    t, w, c, origin, vs = VOLUMES[name]()
    V, T, C, N = orc.marching_cubes(t, w, c, origin, vs, MIN_W)
    assert len(T) > 50
    mesh = _fusion(t, w, c, origin, vs).build_mesh(MIN_W)
    torch.cuda.synchronize()
    gv, gt = mesh.vertices.cpu().numpy(), mesh.triangles.cpu().numpy()
    gc, gn = mesh.vertex_colors.cpu().numpy(), mesh.vertex_normals.cpu().numpy()
    assert gv.shape == V.shape and gt.shape == T.shape
    assert np.array_equal(gt, T)
    assert np.array_equal(gv, V) and np.array_equal(gc, C)
    assert np.abs(gn - N).max() <= 1e-6


def test_empty_volume_gives_no_mesh():
    n = 20
    fus = _fusion(np.ones((n, n, n), F32), np.ones((n, n, n), F32), np.zeros((n, n, n, 3), F32), np.zeros(3, F32), 0.1)
    assert fus.build_mesh(0.5) is None
    assert fus.fuse({"gui": {"build_mesh": {"min_weight_for_mesh": 0.5}}}) is None


def _look_at_tq(cam, target, up=(0, -1.0, 0)):
    fwd = np.asarray(target, float) - cam
    fwd /= np.linalg.norm(fwd)
    right = np.cross(fwd, up); right /= np.linalg.norm(right)
    down = np.cross(fwd, right)
    R = np.stack([right, down, fwd])                      # world -> camera rows
    return np.concatenate([-R @ cam, Rotation.from_matrix(R).as_quat()]).astype(F32)


def _poses(origin, vs, shape, rng, n):
    nz, ny, nx = shape
    centre = np.asarray(origin, float) + vs * (np.array([nx, ny, nz]) - 1) / 2
    ext = vs * max(shape)
    out = []
    for _ in range(n):
        d = rng.normal(size=3); d /= np.linalg.norm(d)
        out.append(_look_at_tq(centre + d * ext * rng.uniform(0.9, 1.4), centre + rng.normal(size=3) * 0.1 * ext))
    return out


@pytest.mark.parametrize("name", sorted(VOLUMES))
def test_raycast_matches_oracle(name):
    from nerf_slam_b200 import _lib
    t, w, c, origin, vs = VOLUMES[name]()
    vol = _fusion(t, w, c, origin, vs).volume
    lib = _lib.load()
    if name.startswith("golden"):
        # the golden volume is observed only from its own three keyframes (30 x 40, fx = 22): view it from those
        g = np.load(os.path.join(HERE, "golden", "ref_tsdf_integrate.npz"))
        poses = [g["poses"][k] for k in (0, 1, 2, 1)]
        lens = lambda W: 22.0 / 40 * W
    else:
        poses = _poses(origin, vs, t.shape, np.random.default_rng(sorted(VOLUMES).index(name)), 4)
        lens = lambda W: 0.8 * W
    both, agree = 0, 0
    for H, W, tqs in ((48, 64, poses[:3]), (480, 640, poses[3:])):
        intr = np.array([lens(W), lens(W), W / 2 - 0.5, H / 2 - 0.5], F32)
        n = len(tqs)
        d_tq = torch.from_numpy(np.stack(tqs)).to(DEV)
        out = [torch.empty(n, H, W, device=DEV), torch.empty(n, H, W, 3, device=DEV), torch.empty(n, H, W, device=DEV),
               torch.empty(n, H, W, 3, device=DEV)]
        _lib.check(lib.nslam_tsdf_raycast(_lib.ptr(vol.tsdf), _lib.ptr(vol.weight), _lib.ptr(vol.color), t.shape[2], t.shape[1],
                                          t.shape[0], vol.origin.ctypes.data, vs, _lib.ptr(d_tq), n, H, W, intr.ctypes.data,
                                          0.01, 6.0, 0.10, 0.01, *[_lib.ptr(o) for o in out], _lib.stream_ptr()), "raycast")
        torch.cuda.synchronize()
        gd, gc, gw, gn = [o.cpu().numpy() for o in out]
        for q, tq in enumerate(tqs):
            D, C, Wt, N = orc.raycast(t, w, c, origin, vs, tq, H, W, intr, 0.01, 6.0, 0.10, 0.01)
            agree += int(((D > 0) == (gd[q] > 0)).sum())
            both += D.size
            m = (D > 0) & (gd[q] > 0)
            assert m.sum() > 0.02 * D.size, (name, q)
            assert np.allclose(gd[q][m], D[m], rtol=1e-5, atol=0)
            close = np.isclose(gd[q][m], D[m], rtol=1e-6, atol=0)
            assert np.allclose(gc[q][m][close], C[m][close], atol=1e-5)
            assert np.allclose(gw[q][m][close], Wt[m][close], rtol=1e-5, atol=1e-5)
            assert np.allclose(gn[q][m][close], N[m][close], atol=1e-4)
            assert (gd[q][~(gd[q] > 0)] == 0).all() and (gc[q][~(gd[q] > 0)] == 0).all()
    assert agree >= 0.999 * both, agree / both


# ------------------------------------------------------------------------------------------------------------ end to end
H, W = 240, 320


def _room_packets(room, frames):
    from nerf_slam_b200.frontend import matrix_to_tq
    for k in frames:
        p = room.packet(k)
        calib = p["calibs"][0]
        raw = torch.from_numpy(p["depths"][0, ..., 0].astype(np.float32)).to(DEV)     # u16 units, as datasets deliver
        depth = raw * calib.depth_scale
        yield k, {"is_last_frame": False, "kf_idx": k, "viz_idx": torch.tensor([k], device=DEV), "viz_idx_host": [k],
                  "kf_idx_to_f_idx": {k: k}, "calibs": p["calibs"],
                  "cam0_poses": torch.from_numpy(matrix_to_tq(np.asarray(p["poses"][0], np.float64))[None]).float().to(DEV),
                  "cam0_idepths_up": (1.0 / depth)[None], "cam0_depths_cov_up": torch.full((1, H, W), 0.04, device=DEV),
                  "cam0_images": torch.from_numpy(p["images"][..., :3]).permute(0, 3, 1, 2).contiguous().to(DEV),
                  "cam0_intrinsics": torch.from_numpy(calib.camera_model.numpy() / 8.0)[None].float().to(DEV),
                  "gt_depths": raw[None, None]}


@pytest.fixture(scope="module")
def room_fusion():
    from nerf_slam_b200.synthetic import SyntheticRoom
    from nerf_slam_b200.tsdf_fusion import TsdfFusion
    room = SyntheticRoom(W, H, 40, seed=0)
    fus = TsdfFusion("sigma", types.SimpleNamespace(eval=False, tsdf_resolution=256, tsdf_center=(0.0, 0.0, 0.0)), DEV)
    fus.voxel_size = 8.0 / 256; fus.initialize()                                  # the room is 6 x 4 x 6 m
    for _, pkt in _room_packets(room, range(0, 40, 4)):
        fus.fuse({"slam": [None, pkt]})
    torch.cuda.synchronize()
    return room, fus


def test_room_mesh_lies_on_the_walls_and_is_deterministic(room_fusion):
    room, fus = room_fusion
    mesh = fus.build_mesh(0.5)
    v = mesh.vertices
    assert v.shape[0] > 20000 and mesh.triangles.shape[0] > 20000
    he = torch.tensor(room.ext, device=DEV, dtype=torch.float32)
    dist_to_wall = (he - v.abs()).abs().min(dim=1).values
    assert float((dist_to_wall < 2.5 * fus.voxel_size).float().mean()) > 0.97
    assert int(mesh.triangles.min()) >= 0 and int(mesh.triangles.max()) < v.shape[0]
    again = fus.build_mesh(0.5)
    for a, b in ((mesh.vertices, again.vertices), (mesh.triangles, again.triangles),
                 (mesh.vertex_colors, again.vertex_colors), (mesh.vertex_normals, again.vertex_normals)):
        assert a.cpu().numpy().tobytes() == b.cpu().numpy().tobytes()


def test_room_renders_at_the_fused_views(room_fusion):
    """thresholds from a CPU rehearsal of this configuration with the numpy oracle (oracle.tsdf.integrate of the same ten
    packets into the same 256^3 grid, then tsdf_readout_oracle.raycast at each view): hit fraction 0.981 .. 0.997,
    median |depth - GT| 0.00014 .. 0.00027 m (voxel 0.031 m), PSNR 24.3 .. 30.8 dB; the limits leave margin"""
    from nerf_slam_b200.tsdf_fusion import color_psnr
    room, fus = room_fusion
    packet = fus.get_history_packet()
    depth, color = fus.render_volume(packet, fus.intrinsics, fus.min_weight_for_render, fus.max_depth_sigma_thresh)
    gt = packet["gt_depths"][:, 0]
    for i in range(depth.shape[0]):
        m = depth[i] > 0
        assert float(m.float().mean()) > HIT_MIN, i
        assert float((depth[i][m] - gt[i][m]).abs().median()) < MEDIAN_MAX, i
        assert color_psnr(color[i], packet["cam0_images"][i]) > PSNR_MIN, i
    d2, c2 = fus.render_volume(packet, fus.intrinsics, fus.min_weight_for_render, fus.max_depth_sigma_thresh)
    assert depth.cpu().numpy().tobytes() == d2.cpu().numpy().tobytes()
    assert color.cpu().numpy().tobytes() == c2.cpu().numpy().tobytes()


def test_gui_packet_builds_a_mesh_and_writes_results_csv(room_fusion, tmp_path, monkeypatch):
    from nerf_slam_b200.tsdf_fusion import TsdfMesh
    room, fus = room_fusion
    monkeypatch.chdir(tmp_path)
    out = fus.fuse({"gui": {"build_mesh": {"min_weight_for_mesh": 0.5}, "eval_metrics": True,
                            "depth_mask_type": "uncertainty", "rebuild_volume": False}})
    assert isinstance(out["mesh"], TsdfMesh) and out["mesh"].triangles.shape[0] > 0
    rows = list(csv.reader(open(tmp_path / "results.csv")))
    assert rows[0] == ["", "Dt", "PSNR", "L1"] and len(rows) == 2 and rows[1][:2] == ["0", "0.0"]
    psnr, l1 = float(rows[1][2]), float(rows[1][3])
    assert np.isfinite(psnr) and np.isfinite(l1) and psnr > PSNR_MIN and l1 < 10.0


def test_dense_volume_mesh_scratch_grows_with_the_surface_not_the_grid():
    from nerf_slam_b200.synthetic import SyntheticRoom
    from nerf_slam_b200.tsdf_fusion import TsdfFusion
    room = SyntheticRoom(W, H, 40, seed=0)
    fus = TsdfFusion("sigma", types.SimpleNamespace(eval=False, tsdf_resolution=512, tsdf_center=(0.0, 0.0, 0.0)), DEV)
    fus.voxel_size = 8.0 / 512; fus.initialize()
    for _, pkt in _room_packets(room, range(0, 40, 8)):
        fus.fuse({"slam": [None, pkt]})
    torch.cuda.synchronize()
    volume_bytes = fus.volume.memory_bytes()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    mesh = fus.build_mesh(0.5)
    torch.cuda.synchronize()
    rise = torch.cuda.max_memory_allocated() - base
    out_bytes = sum(x.numel() * x.element_size() for x in (mesh.vertices, mesh.triangles, mesh.vertex_colors,
                                                           mesh.vertex_normals))
    assert mesh.triangles.shape[0] > 50000
    assert rise < out_bytes + volume_bytes / 16, (rise, out_bytes, volume_bytes)


HIT_MIN, MEDIAN_MAX, PSNR_MIN = 0.95, 0.002, 22.0
