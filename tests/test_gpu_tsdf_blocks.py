"""The sparse voxel-block volume on the GPU (csrc/tsdf_blocks.cu, csrc/tsdf_mesh.cu via nerf_slam_b200/tsdf_blocks.py)
against the reference method executed on a block stand-in (tests/golden/ref_tsdf_blocks.npz), the numpy oracle
(oracle/tsdf_blocks.py), and the dense kernels applied to the volume's dense embedding."""
import csv
import os
import types

import numpy as np
import pytest
import torch

from oracle import tsdf as otsdf
from oracle import tsdf_blocks as otb

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
F32 = np.float32
T = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def _recording():
    from nerf_slam_b200.tsdf_blocks import _CudaKernels

    class Rec(_CudaKernels):
        def __init__(self):
            self.touched = []

        def activate(self, vol, f):
            touched, new = super().activate(vol, f)
            self.touched.append(touched.clone())
            return touched, new
    return Rec()


def _volume(vs, block_count=5000):
    from nerf_slam_b200.tsdf_blocks import VoxelBlockVolume
    vol = VoxelBlockVolume(vs, block_count, DEV)
    vol.kernels = _recording()
    return vol


def _integrate(vol, frame, **kw):
    idepth, cov, rgb, intr, tq = frame
    n = vol.integrate(T(idepth), T(cov) if cov is not None else None, T(rgb), intr, T(tq), **kw)
    keys = vol._keys[vol.kernels.touched[-1].long()].cpu().numpy()
    return n, keys


def _pool(vol):
    n = vol.n_blocks
    return (vol._keys[:n].cpu().numpy(), vol.tsdf[:n].cpu().numpy(), vol.weight[:n].cpu().numpy(), vol.color[:n].cpu().numpy())


@pytest.mark.parametrize("tag", ["tsdf", "sigma"])
def test_blocks_match_the_reference_method_executed_verbatim(tag):
    """touched keys and pool order exactly; voxels bit for bit against the oracle in both flavours and against the golden
    in "tsdf"; "sigma" holds the dense golden test's allowance for torch's CPU sqrt"""
    g = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_tsdf_blocks.npz"))
    K = g["intr"]
    intr4 = np.array([K[0, 0], K[1, 1], K[0, 2], K[1, 2]], F32)
    vol = _volume(float(g["voxel_size"]), block_count=4)
    ref = otb.BlockVolume(g["voxel_size"])
    for k in range(3):
        cov = g["covs"][k] if tag == "sigma" else None
        _, keys = _integrate(vol, (g["idepths"][k], cov, g["imgs"][k], intr4, g["poses"][k]))
        ref.integrate(g["idepths"][k], cov, g["imgs"][k], intr4, g["poses"][k])
        torch.cuda.synchronize()
        pk, pt, pw, pc = _pool(vol)
        assert np.array_equal(keys, g[f"{tag}_touched_{k}"]) and np.array_equal(pk, g[f"{tag}_keys_{k}"]), k
        assert np.array_equal(pt, ref.tsdf) and np.array_equal(pw, ref.weight) and np.array_equal(pc, ref.color), k
        t, w, c = g[f"{tag}_tsdf_{k}"], g[f"{tag}_weight_{k}"], g[f"{tag}_color_{k}"]
        assert np.array_equal(pw > 0, w > 0), k
        if tag == "tsdf":
            assert np.array_equal(pt, t) and np.array_equal(pw, w) and np.array_equal(pc, c), k
        else:
            assert np.allclose(pw, w, rtol=3e-7, atol=0) and np.allclose(pt, t, rtol=0, atol=3e-7) and np.allclose(pc, c, rtol=0, atol=1e-4), k
    assert vol.capacity > 4 and vol.capacity >= vol.n_blocks and vol.capacity % 4 == 0    # grown by doubling


def _frame(rng, H=48, W=64, with_cov=True, centre=(0.0, 0.0, 0.0), depth=(0.5, 2.5)):
    idepth = rng.uniform(1 / depth[1], 1 / depth[0], (H, W)).astype(F32)
    cov = rng.uniform(0.01, 0.5, (H, W)).astype(F32) if with_cov else None
    if with_cov:
        cov[:4] = 3e8
        idepth[4:6] = -1.0                                                       # invalid pixels
    rgb = rng.integers(0, 255, (3, H, W), dtype=np.uint8)
    q = rng.normal(size=4) * 0.1 + np.array([0, 0, 0, 1.0]); q /= np.linalg.norm(q)
    R = otsdf.pose_tq_to_matrix(np.concatenate([np.zeros(3), q]).astype(F32))[:3, :3]
    tq = np.concatenate([-R @ np.asarray(centre, np.float64), q]).astype(F32)
    intr = np.array([W * 0.6, W * 0.6, W / 2 - 0.5, H / 2 - 0.5], F32)
    return idepth, cov, rgb, intr, tq


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_activation_matches_the_oracle(seed):
    rng = np.random.default_rng(seed)
    for k in range(3):
        vs = float(rng.uniform(0.01, 0.08))
        fr = _frame(rng, with_cov=bool(k % 2), centre=rng.uniform(-3, 3, 3))
        vol = _volume(vs)
        _, keys = _integrate(vol, fr)
        ref = otb.touched_keys(fr[0], fr[1], fr[3], fr[4], F32(vs))
        assert len(ref) > 20 and np.array_equal(keys, ref), (seed, k)


def _dense_integrate(n, vs, frame):
    """nslam_tsdf_integrate on an origin-0 grid [n2,n1,n0]"""
    from nerf_slam_b200 import _lib
    lib = _lib.load()
    t = torch.zeros(n[2], n[1], n[0], device=DEV); w = torch.zeros_like(t); c = torch.zeros(n[2], n[1], n[0], 3, device=DEV)
    idepth, cov, rgb, intr, tq = frame
    d = [T(idepth), T(cov) if cov is not None else None, T(rgb), T(tq)]
    org = np.zeros(3, F32)
    _lib.check(lib.nslam_tsdf_integrate(_lib.ptr(t), _lib.ptr(w), _lib.ptr(c), n[0], n[1], n[2], org.ctypes.data, vs,
                                        _lib.ptr(d[0]), _lib.ptr(d[1]), _lib.ptr(d[2]), idepth.shape[0], idepth.shape[1],
                                        intr.ctypes.data, _lib.ptr(d[3]), 6.0, 0.10, 20.0, 10000.0, _lib.stream_ptr()), "tsdf")
    torch.cuda.synchronize()
    return t.cpu().numpy(), w.cpu().numpy(), c.cpu().numpy()


@pytest.mark.parametrize("mode", ["sigma", "tsdf"])
def test_integration_equals_the_dense_kernel_on_touched_blocks(mode):
    rng = np.random.default_rng(8)
    vs = 0.05
    fr = _frame(rng, with_cov=(mode == "sigma"), centre=(2.5, 2.5, 1.0), depth=(0.4, 1.5))
    vol = _volume(vs)
    _integrate(vol, fr)
    torch.cuda.synchronize()
    keys, pt, pw, pc = _pool(vol)
    coords = otb.unpack(keys)
    assert (coords >= 0).all() and len(coords) > 20
    dt, dw, dc = _dense_integrate(16 * (coords.max(0) + 2), vs, fr)
    for i, b in enumerate(coords):
        s = np.s_[16 * b[2]:16 * b[2] + 16, 16 * b[1]:16 * b[1] + 16, 16 * b[0]:16 * b[0] + 16]
        assert np.array_equal(pt[i], dt[s]) and np.array_equal(pw[i], dw[s]) and np.array_equal(pc[i], dc[s]), i
    # several keyframes against the block oracle, with test_tsdf_integrate_matches_oracle's allowance
    ref = otb.BlockVolume(vs)
    ref.integrate(*fr)
    for k in range(3):
        f = _frame(rng, with_cov=(mode == "sigma"), centre=(2.5 + 0.2 * k, 2.4, 1.1))
        _integrate(vol, f)
        ref.integrate(*f)
    torch.cuda.synchronize()
    keys, pt, pw, pc = _pool(vol)
    assert np.array_equal(keys, ref.keys)
    ok = ((pw > 0) == (ref.weight > 0)) & np.isclose(pw, ref.weight, rtol=1e-6, atol=0) \
        & np.isclose(pt, ref.tsdf, rtol=1e-5, atol=1e-5) & np.isclose(pc, ref.color, rtol=1e-5, atol=5e-3).all(-1)
    assert ok.mean() > 0.999, ok.mean()


def _fused(block_count=5000, frames=4, seed=12):
    rng = np.random.default_rng(seed)
    vol = _volume(0.04, block_count)
    for k in range(frames):
        _integrate(vol, _frame(rng, H=96, W=128, centre=(3.0 + 0.1 * k, 3.0, 1.0), depth=(0.8, 1.6)))
    torch.cuda.synchronize()
    return vol


def test_growth_gives_the_same_pool():
    a, b = _fused(8), _fused(5000)
    assert a.capacity >= a.n_blocks > 8 and b.capacity == 5000
    for x, y in zip(_pool(a), _pool(b)):
        assert x.tobytes() == y.tobytes()


def _embed0(vol):
    """the dense embedding from lattice index 0 (the volume must lie at non-negative block coordinates)"""
    t, w, c, org = vol.to_dense(margin_blocks=1)
    lo = np.rint(org / F32(vol.voxel_size)).astype(np.int64)
    assert (lo >= 0).all()
    pad = lambda a: torch.nn.functional.pad(a, (0, 0) * (a.dim() - 3) + (int(lo[0]), 0, int(lo[1]), 0, int(lo[2]), 0))
    return pad(t).contiguous(), pad(w).contiguous(), pad(c).contiguous()


def _canonical_triangles(v, tri):
    """triangles as sets of vertex positions, each rotated to start at its smallest vertex key"""
    key = [tuple(p) for p in v.view(np.int32).reshape(-1, 3)]
    out = set()
    for a, b, c in tri:
        t = [key[a], key[b], key[c]]
        r = t.index(min(t))
        out.add(tuple(t[r:] + t[:r]))
    return out


def test_block_mesh_equals_the_dense_volume_mesh_of_the_embedding():
    from nerf_slam_b200.tsdf_fusion import DenseVolume
    vol = _fused()
    mesh = vol.build_mesh(0.5)
    t, w, c = _embed0(vol)
    dense = DenseVolume.from_tensors(t, w, c, np.zeros(3, F32), vol.voxel_size).build_mesh(0.5)
    torch.cuda.synchronize()
    v, dv = mesh.vertices.cpu().numpy(), dense.vertices.cpu().numpy()
    assert v.shape == dv.shape and mesh.triangles.shape == dense.triangles.shape and len(v) > 1000
    order = np.lexsort(v.view(np.int32).T[::-1]); dorder = np.lexsort(dv.view(np.int32).T[::-1])
    assert np.array_equal(v[order], dv[dorder])
    assert np.array_equal(mesh.vertex_colors.cpu().numpy()[order], dense.vertex_colors.cpu().numpy()[dorder])
    assert np.abs(mesh.vertex_normals.cpu().numpy()[order] - dense.vertex_normals.cpu().numpy()[dorder]).max() <= 1e-6
    assert _canonical_triangles(v, mesh.triangles.cpu().numpy()) == _canonical_triangles(dv, dense.triangles.cpu().numpy())
    assert _volume(0.05).build_mesh(0.5) is None


def _views(n=3):
    from scipy.spatial.transform import Rotation
    out = []
    for k in range(n):
        cam = np.array([3.0 + 0.1 * k, 3.0 - 0.05 * k, 0.9])
        R = Rotation.from_euler("xyz", [0.05 * k, -0.04 * k, 0.02]).as_matrix()
        out.append(np.concatenate([-R @ cam, Rotation.from_matrix(R).as_quat()]).astype(F32))
    return np.stack(out)


def test_raycast_equals_the_dense_raycast_of_the_embedding():
    from nerf_slam_b200 import _lib
    vol = _fused()
    t, w, c = _embed0(vol)
    poses = T(_views())
    H, W = 96, 128
    intr = np.array([0.6 * W, 0.6 * W, W / 2 - 0.5, H / 2 - 0.5], F32)
    bd, bc, bw, bn = vol.raycast(poses, H, W, intr, 0.01, 6.0, 0.10, 0.01, normals=True)
    out = [torch.empty(3, H, W, device=DEV), torch.empty(3, H, W, 3, device=DEV), torch.empty(3, H, W, device=DEV),
           torch.empty(3, H, W, 3, device=DEV)]
    org = np.zeros(3, F32)
    _lib.check(_lib.load().nslam_tsdf_raycast(_lib.ptr(t), _lib.ptr(w), _lib.ptr(c), t.shape[2], t.shape[1], t.shape[0],
                                              org.ctypes.data, vol.voxel_size, _lib.ptr(poses), 3, H, W, intr.ctypes.data,
                                              0.01, 6.0, 0.10, 0.01, *[_lib.ptr(o) for o in out], _lib.stream_ptr()), "raycast")
    torch.cuda.synchronize()
    assert float((bd > 0).float().mean()) > 0.05
    for a, b in zip((bd, bc, bw, bn), out):
        assert a.cpu().numpy().tobytes() == b.cpu().numpy().tobytes()


def test_two_fresh_runs_give_the_same_bytes():
    runs = []
    for _ in range(2):
        vol = _fused()
        mesh = vol.build_mesh(0.5)
        d, c, _, _ = vol.raycast(T(_views()), 96, 128, np.array([77, 77, 63.5, 47.5], F32), 0.01, 6.0, 0.10, 0.01)
        torch.cuda.synchronize()
        runs.append([x.tobytes() for x in _pool(vol)] +
                    [x.cpu().numpy().tobytes() for x in (mesh.vertices, mesh.triangles, mesh.vertex_colors, mesh.vertex_normals, d, c)])
    assert runs[0] == runs[1]


# ------------------------------------------------------------------------------------------------------------ end to end
H, W = 240, 320
ROOM_FRAMES = range(0, 40, 4)
MEMORY_MAX = 1 << 30          # the dense grid for this room at 6/512 m would take ~12.5 GB
HIT_MIN, MEDIAN_MAX, PSNR_MIN = 0.95, 0.002, 24.0


def _room_packets(room, frames):
    from nerf_slam_b200.frontend import matrix_to_tq
    for k in frames:
        p = room.packet(k)
        calib = p["calibs"][0]
        raw = torch.from_numpy(p["depths"][0, ..., 0].astype(np.float32)).to(DEV)
        depth = raw * calib.depth_scale
        yield {"is_last_frame": False, "kf_idx": k, "viz_idx": torch.tensor([k], device=DEV), "viz_idx_host": [k],
               "kf_idx_to_f_idx": {k: k}, "calibs": p["calibs"],
               "cam0_poses": torch.from_numpy(matrix_to_tq(np.asarray(p["poses"][0], np.float64))[None]).float().to(DEV),
               "cam0_idepths_up": (1.0 / depth)[None], "cam0_depths_cov_up": torch.full((1, H, W), 0.04, device=DEV),
               "cam0_images": torch.from_numpy(p["images"][..., :3]).permute(0, 3, 1, 2).contiguous().to(DEV),
               "cam0_intrinsics": torch.from_numpy(calib.camera_model.numpy() / 8.0)[None].float().to(DEV),
               "gt_depths": raw[None, None]}


@pytest.fixture(scope="module")
def big_room():
    """a 10 x 4 x 10 m room at the reference's 6/512 m voxel, which the default dense grid (6 m cube) cannot hold"""
    from nerf_slam_b200.synthetic import SyntheticRoom
    from nerf_slam_b200.tsdf_fusion import TsdfFusion
    room = SyntheticRoom(W, H, 40, seed=0, half_extent=(5, 2, 5))
    fus = TsdfFusion("sigma", types.SimpleNamespace(eval=False, tsdf_volume="blocks", tsdf_block_count=5000), DEV)
    for pkt in _room_packets(room, ROOM_FRAMES):
        fus.fuse({"slam": [None, pkt]})
    torch.cuda.synchronize()
    return room, fus


def test_big_room_fuses_meshes_and_renders(big_room):
    """limits set with margin from a run on an H100: 4825 blocks in a 5000-block pool (0.38 GiB), every mesh vertex
    within 2.5 voxels of a wall, per view hit fraction 0.987 .. 0.999, median |depth - GT| 0.00044 .. 0.00051 m (voxel
    0.0117 m), PSNR 27.9 .. 36.8 dB.  A CPU rehearsal with the numpy oracle is not practical here: the read-out oracle
    needs the dense embedding, 853 x 341 x 853 voxels."""
    from nerf_slam_b200.tsdf_fusion import color_psnr
    room, fus = big_room
    vol = fus.volume
    print(f"blocks {vol.n_blocks} capacity {vol.capacity} memory {vol.memory_bytes() / 2**30:.2f} GiB")
    assert fus.integrated_frames == len(ROOM_FRAMES) and vol.memory_bytes() < MEMORY_MAX
    mesh = fus.build_mesh(0.5)
    v = mesh.vertices
    dist = (torch.tensor(room.ext, device=DEV, dtype=torch.float32) - v.abs()).abs().min(dim=1).values
    near = float((dist < 2.5 * fus.voxel_size).float().mean())
    print(f"vertices {v.shape[0]} near walls {near:.4f}")
    assert v.shape[0] > 20000 and near >= 0.97
    assert int(mesh.triangles.min()) >= 0 and int(mesh.triangles.max()) < v.shape[0]
    packet = fus.get_history_packet()
    depth, color = fus.render_volume(packet, fus.intrinsics, fus.min_weight_for_render, fus.max_depth_sigma_thresh)
    gt = packet["gt_depths"][:, 0]
    for i in range(depth.shape[0]):
        m = depth[i] > 0
        hit, med = float(m.float().mean()), float((depth[i][m] - gt[i][m]).abs().median())
        psnr = color_psnr(color[i], packet["cam0_images"][i])
        print(f"view {i}: hit {hit:.3f} median {med:.5f} psnr {psnr:.2f}")
        assert hit > HIT_MIN and med < MEDIAN_MAX and psnr > PSNR_MIN, i


def test_block_mode_gui_packets_results_csv_and_rebuild(big_room, tmp_path, monkeypatch):
    from nerf_slam_b200.tsdf_fusion import TsdfMesh
    room, fus = big_room
    monkeypatch.chdir(tmp_path)
    out = fus.fuse({"gui": {"build_mesh": {"min_weight_for_mesh": 0.5}, "eval_metrics": True}})
    assert isinstance(out["mesh"], TsdfMesh) and out["mesh"].triangles.shape[0] > 0
    rows = list(csv.reader(open(tmp_path / "results.csv")))
    assert rows[0] == ["", "Dt", "PSNR", "L1"] and len(rows) == 2
    assert np.isfinite(float(rows[1][2])) and np.isfinite(float(rows[1][3]))
    vs, cap = fus.voxel_size, fus.volume.capacity
    fus.fuse({"gui": {"rebuild_volume": True}})                                    # reset (half voxel) + history
    torch.cuda.synchronize()
    assert fus.voxel_size == vs / 2 and fus.volume.capacity >= cap
    mesh = fus.build_mesh(0.5)
    v = mesh.vertices
    dist = (torch.tensor(room.ext, device=DEV, dtype=torch.float32) - v.abs()).abs().min(dim=1).values
    assert float((dist < 2.5 * fus.voxel_size).float().mean()) >= 0.97
    # the whole room is still covered: vertices reach every wall the views saw, out to ~5 m
    assert float(v[:, 0].abs().max()) > 4.5 and float(v[:, 2].abs().max()) > 4.5
