"""§8(f3): Sigma / TSDF fusion consumer (nerf_slam_b200/tsdf_fusion.py, csrc/tsdf.cu) against the numpy restatement of the
reference's per-voxel update (oracle/tsdf.py <- fusion/tsdf_fusion.py:231-296), and end to end on ground-truth geometry."""
import types

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _frame(rng, H=48, W=64, with_cov=True):
    idepth = rng.uniform(0.4, 1.2, (H, W)).astype(np.float32)
    cov = rng.uniform(0.01, 0.5, (H, W)).astype(np.float32) if with_cov else None
    if with_cov:
        cov[:4] = 3e8                                   # sqrt > 10000: masked out by the sigma threshold
    rgb = rng.integers(0, 255, (3, H, W), dtype=np.uint8)
    q = rng.normal(size=4); q /= np.linalg.norm(q)
    q = 0.1 * q + np.array([0, 0, 0, 1.0]); q /= np.linalg.norm(q)
    tq = np.concatenate([rng.uniform(-0.1, 0.1, 3), q]).astype(np.float32)
    intr = np.array([W * 0.6, W * 0.6, W / 2 - 0.5, H / 2 - 0.5], np.float32)
    return idepth, cov, rgb, tq, intr


@pytest.mark.parametrize("mode", ["sigma", "tsdf"])
def test_tsdf_integrate_matches_oracle(mode):
    """three keyframes integrated one after the other into a 40^3 grid (running averages, weight saturation at 20)"""
    from nerf_slam_b200 import _lib
    from oracle import tsdf as otsdf
    lib = _lib.load()
    rng = np.random.default_rng(7)
    n, vs = 40, 0.06
    origin = np.array([-1.2, -1.2, 0.2], np.float32)
    T = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(DEV)
    tsdf = torch.zeros(n, n, n, device=DEV); weight = torch.zeros(n, n, n, device=DEV); color = torch.zeros(n, n, n, 3, device=DEV)
    rt, rw, rc = np.zeros((n, n, n), np.float32), np.zeros((n, n, n), np.float32), np.zeros((n, n, n, 3), np.float32)
    touched = 0
    for k in range(3):
        idepth, cov, rgb, tq, intr = _frame(rng, with_cov=(mode == "sigma"))
        if k == 2:
            rw[rw > 0] = 19.9; weight.copy_(T(rw))      # next reading saturates the weight
        d_tq = T(tq)
        d_idepth, d_cov, d_rgb = T(idepth), (T(cov) if cov is not None else None), T(rgb)   # named: they must outlive the launch
        _lib.check(lib.nslam_tsdf_integrate(_lib.ptr(tsdf), _lib.ptr(weight), _lib.ptr(color), n, n, n, origin.ctypes.data, vs,
                                            _lib.ptr(d_idepth), _lib.ptr(d_cov) if d_cov is not None else None, _lib.ptr(d_rgb),
                                            idepth.shape[0], idepth.shape[1], intr.ctypes.data, _lib.ptr(d_tq), 6.0, 0.10, 20.0,
                                            10000.0, _lib.stream_ptr()), "tsdf")
        touched += otsdf.integrate(rt, rw, rc, origin, vs, idepth, cov, rgb, intr, tq)
    torch.cuda.synchronize()
    assert touched > 5000
    gw, gt, gc = weight.cpu().numpy(), tsdf.cpu().numpy(), color.cpu().numpy()
    # random poses / depths at 40^3 (the golden scenario of the next test is checked bit for bit; this one keeps a small
    # allowance for voxels whose pixel coordinate sits within fp64 rounding of .5)
    ok = ((gw > 0) == (rw > 0)) & np.isclose(gw, rw, rtol=1e-6, atol=0) & np.isclose(gt, rt, rtol=1e-5, atol=1e-5) \
        & np.isclose(gc, rc, rtol=1e-5, atol=5e-3).all(-1)
    assert ok.mean() > 0.999, ok.mean()                                           # boundary voxels: < 0.1 %
    assert rw.max() == 20.0 and gw.max() == 20.0


@pytest.mark.parametrize("tag,mw", [("sigma", 20.0), ("sigma", 2.5), ("tsdf", 20.0), ("tsdf", 2.5)])
def test_tsdf_kernel_matches_the_reference_methods_executed_verbatim(tag, mw):
    """nslam_tsdf_integrate against tests/golden/ref_tsdf_integrate.npz = the reference's own build_volume +
    custom_volume_integrate executed verbatim on stand-ins for Open3D's tensors (tests/golden/make_golden_tsdf.py): three
    keyframes, checked after each.  The kernel performs the reference's operations in the reference's order (float32 voxel
    coordinates and pose matrix promoted to fp64, round-half-even, separately rounded products): bit-exact against the numpy
    oracle in both flavours and against the golden in "tsdf"; in "sigma" the golden's weights carry the last-bit error of
    torch's vectorised CPU sqrt (see tests/test_cpu_golden.py), hence 3e-7."""
    import os
    from nerf_slam_b200 import _lib
    from oracle import tsdf as otsdf
    lib = _lib.load()
    g = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_tsdf_integrate.npz"))
    n, vs, org, intr = int(g["n"]), float(g["voxel_size"]), g["origin"], g["intr"]
    intr4 = np.array([intr[0, 0], intr[1, 1], intr[0, 2], intr[1, 2]], np.float32)
    T = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(DEV)
    tsdf = torch.zeros(n, n, n, device=DEV); weight = torch.zeros(n, n, n, device=DEV); color = torch.zeros(n, n, n, 3, device=DEV)
    ot, ow, oc = np.zeros((n, n, n), np.float32), np.zeros((n, n, n), np.float32), np.zeros((n, n, n, 3), np.float32)
    for k in range(3):
        cov = g["covs"][k] if tag == "sigma" else None
        d_idepth, d_cov, d_rgb, d_tq = T(g["idepths"][k]), (T(cov) if cov is not None else None), T(g["imgs"][k]), T(g["poses"][k])
        H, W = g["idepths"][k].shape
        _lib.check(lib.nslam_tsdf_integrate(_lib.ptr(tsdf), _lib.ptr(weight), _lib.ptr(color), n, n, n, org.ctypes.data, vs,
                                            _lib.ptr(d_idepth), _lib.ptr(d_cov) if d_cov is not None else None, _lib.ptr(d_rgb),
                                            H, W, intr4.ctypes.data, _lib.ptr(d_tq), 6.0, 0.10, mw, 10000.0, _lib.stream_ptr()), "tsdf")
        torch.cuda.synchronize()
        otsdf.integrate(ot, ow, oc, org, vs, g["idepths"][k], cov, g["imgs"][k], intr4, g["poses"][k], max_weight=mw)
        gt, gw, gc = tsdf.cpu().numpy(), weight.cpu().numpy(), color.cpu().numpy()
        assert np.array_equal(gw, ow) and np.array_equal(gt, ot) and np.array_equal(gc, oc), (k, float(np.abs(gt - ot).max()))
        rt, rw, rc = g[f"{tag}_w{mw}_tsdf_{k}"], g[f"{tag}_w{mw}_weight_{k}"], g[f"{tag}_w{mw}_color_{k}"]
        assert np.array_equal(gw > 0, rw > 0), k
        if tag == "tsdf":
            assert np.array_equal(gt, rt) and np.array_equal(gw, rw) and np.array_equal(gc, rc), k
        else:
            assert np.allclose(gw, rw, rtol=3e-7, atol=0) and np.allclose(gt, rt, rtol=0, atol=3e-7) and np.allclose(gc, rc, rtol=0, atol=1e-4), k


def test_tsdf_fusion_volume_of_ground_truth_packets_recovers_the_room():
    """TsdfFusion('sigma') fed SLAM-shaped packets built from the synthetic room's ground-truth poses and depths: the
    zero crossings of the fused TSDF lie on the room's walls (within two voxels), history / rebuild work"""
    from nerf_slam_b200.synthetic import SyntheticRoom
    from nerf_slam_b200.frontend import matrix_to_tq
    from nerf_slam_b200.tsdf_fusion import TsdfFusion
    H, W = 240, 320
    room = SyntheticRoom(W, H, 40, seed=0)
    args = types.SimpleNamespace(eval=False, tsdf_resolution=256, tsdf_center=(0.0, 0.0, 0.0))
    fus = TsdfFusion("sigma", args, DEV)
    fus.voxel_size = 8.0 / 256; fus.initialize()                                  # the room is 6 x 4 x 6 m
    for k in range(0, 40, 4):
        p = room.packet(k)
        calib = p["calibs"][0]
        depth = torch.from_numpy(p["depths"][0, ..., 0].astype(np.float32) * calib.depth_scale).to(DEV)
        pkt = {"is_last_frame": False, "kf_idx": k, "viz_idx": torch.tensor([k], device=DEV), "viz_idx_host": [k],
               "kf_idx_to_f_idx": {k: k}, "calibs": p["calibs"],
               "cam0_poses": torch.from_numpy(matrix_to_tq(np.asarray(p["poses"][0], np.float64))[None]).float().to(DEV),
               "cam0_idepths_up": (1.0 / depth)[None], "cam0_depths_cov_up": torch.full((1, H, W), 0.04, device=DEV),
               "cam0_images": torch.from_numpy(p["images"][..., :3]).permute(0, 3, 1, 2).contiguous().to(DEV),
               "cam0_intrinsics": torch.from_numpy(calib.camera_model.numpy() / 8.0)[None].float().to(DEV),
               "gt_depths": depth[None, None]}
        assert fus.fuse({"slam": [None, pkt]}) is None
    torch.cuda.synchronize()
    assert fus.integrated_frames == 10 and len(fus.history) == 10
    pts, cols = fus.surface_points(min_weight=0.5)
    assert pts.shape[0] > 20000
    he = torch.tensor(room.ext, device=DEV, dtype=torch.float32)
    dist_to_wall = (he - pts.abs()).abs().min(dim=1).values
    assert float((dist_to_wall < 2.5 * fus.voxel_size).float().mean()) > 0.97
    assert float(cols.mean()) > 5.0                                                # colours were fused (u8 scale)
    w0 = float(fus.volume.weight.sum())
    fus.rebuild_volume()                                                           # history -> fresh volume at half the voxel size (:304-316)
    torch.cuda.synchronize()
    assert fus.voxel_size == pytest.approx(8.0 / 512) and float(fus.volume.weight.sum()) > 0 and w0 > 0
