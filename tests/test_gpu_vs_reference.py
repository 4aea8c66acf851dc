"""GPU parity against the REFERENCE'S OWN CUDA kernels, compiled for sm_90a from /root/reference
by oracle/build_ref.py into oracle/_ref/*.so (shipped to the GPU box; skipped if absent).
This is what pins the parity claim: same seeded inputs through both implementations."""
import numpy as np
import pytest
import torch

from oracle import build_ref
from tests.test_gpu_parity import T, _ba_problem, DEV
from tests.util import make_window

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def refcorr():
    m = build_ref.load("nslam_ref_corr")
    if m is None:
        pytest.skip("oracle/_ref/nslam_ref_corr.so not built")
    return m


@pytest.fixture(scope="module")
def refdroid():
    m = build_ref.load("nslam_ref_droid")
    if m is None:
        pytest.skip("oracle/_ref/nslam_ref_droid.so not built")
    return m


@pytest.fixture(scope="module")
def db():
    from nerf_slam_b200 import droid_backends
    return droid_backends


@pytest.mark.parametrize("dtype", [torch.float16, torch.float32])
def test_corr_index_forward_vs_reference(db, refcorr, dtype):
    g = torch.Generator(device="cpu").manual_seed(1235)
    n, h, w = 4, 30, 40
    vol = torch.randn(n, h, w, h, w, generator=g).to(DEV, dtype)
    yy, xx = torch.meshgrid(torch.arange(h), torch.arange(w), indexing="ij")
    coords = (torch.stack([xx, yy], 0)[None].float() + (torch.rand(n, 2, h, w, generator=g) * 16 - 8)).to(DEV).contiguous()
    ref, = refcorr.corr_index_forward(vol, coords, 3)
    got, = db.corr_index_forward(vol, coords, 3)
    if dtype == torch.float16:
        assert torch.equal(got.float(), ref.float()), (got.float() - ref.float()).abs().max()   # bit-exact
    else:
        assert torch.allclose(got, ref, atol=1e-6)


def test_altcorr_vs_reference(db, refcorr):
    g = torch.Generator(device="cpu").manual_seed(1236)
    B, H, W, C = 2, 24, 32, 128
    f1 = (torch.randn(B, H, W, C, generator=g) / 4).to(DEV)
    f2 = (torch.randn(B, H // 2, W // 2, C, generator=g) / 4).to(DEV)
    yy, xx = torch.meshgrid(torch.arange(H), torch.arange(W), indexing="ij")
    coords = (torch.stack([xx, yy], -1)[None, None].float() / 2 + torch.rand(B, 1, H, W, 2, generator=g) * 8 - 4).to(DEV).contiguous()
    ref, = refcorr.altcorr_forward(f1, f2, coords, 3)
    got, = db.altcorr_forward(f1, f2, coords, 3)
    assert torch.allclose(got, ref, atol=2e-4, rtol=1e-4), (got - ref).abs().max()


def test_frame_distance_bit_exact_vs_reference(db, refdroid):
    """same summation tree and expression order => identical fp32 distances => identical edge
    ordering under argsort (the 'bit-exact edge indices' contract)"""
    rng = np.random.default_rng(1237)
    poses, disps, intr, _, _ = make_window(rng, 12, 60, 80)
    ii, jj = np.meshgrid(np.arange(12), np.arange(12), indexing="ij")
    args = (T(poses), T(disps), T(intr), T(ii.reshape(-1)), T(jj.reshape(-1)), 0.3)
    ref = refdroid.frame_distance(*args)
    got = db.frame_distance(*args)
    assert torch.equal(got, ref), (got - ref).abs().max()
    assert torch.equal(torch.argsort(got, stable=True), torch.argsort(ref, stable=True))


@pytest.mark.parametrize("cfg", [dict(seed=71), dict(seed=72, kf0=2), dict(seed=73, with_sensor=True),
                                 dict(seed=74, nframes=10, ht=60, wd=80)])
def test_reduced_camera_matrix_vs_reference(db, refdroid, cfg):
    p = _ba_problem(**cfg)
    args = (T(p["poses"]), T(p["poses"]), T(p["disps"]), T(p["intr"]), T(p["ext"]), T(p["sens"]),
            T(p["target"]), T(p["weight"]), T(p["eta"]), T(p["ii"]), T(p["jj"]), p["kf0"], p["kf1"])
    rH, rv, rQ, rE, rw, rHs, rvs = refdroid.reduced_camera_matrix(*args)
    H, v, Q, E, w = db.reduced_camera_matrix(*args)
    prob = db.reduced_camera_matrix.last_problem

    def close(a, b, rel, name):
        scale = b.abs().max().item() + 1e-12
        err = (a.reshape(b.shape) - b).abs().max().item() / scale
        assert err < rel, f"{name}: rel err {err:.3e}"
    close(prob.Hs, rHs, 2e-4, "Hs"); close(prob.vs, rvs, 2e-4, "vs")
    close(Q, rQ, 1e-4, "Q"); close(w, rw, 2e-4, "w"); close(E, rE, 2e-4, "E")
    close(H, rH, 5e-4, "H"); close(v, rv, 5e-4, "v")
    # depth back-substitution with the reference kernel vs ours, same dx
    dx = T((np.random.default_rng(0).normal(0, 1e-2, (p["kf1"] - p["kf0"], 6))).astype(np.float32))
    d_ref = T(p["disps"].copy()); d_got = T(p["disps"].copy())
    refdroid.solve_depth(dx, d_ref, rQ, rE, rw, T(p["ii"]), T(p["jj"]), p["kf0"], p["kf1"])
    db.solve_depth(dx, d_got, Q, E, w, T(p["ii"]), T(p["jj"]), p["kf0"], p["kf1"])
    assert torch.allclose(d_got, d_ref, rtol=2e-4, atol=2e-5)


def test_ba_all_in_one_loop_vs_reference_kernels(db, refdroid):
    """A15: droid_backends.ba vs ba_cuda (src/droid_kernels.cu:1441-1568) rebuilt from the reference's OWN kernels in its
    own order — per iteration: reference linearisation + Schur (projective_transform / accum / EEt6x6 / Ev6x1 kernels),
    SparseBlock::solve's `diag += ep + lm*diag` Cholesky (:1320-1337, dense fp64 here), reference solve_depth
    (EvT6x1 + accum + disp_retr kernels), reference solve_poses (pose_retr_kernel).  In-place state after 2 iterations."""
    p = _ba_problem(75, nframes=7)
    lm, ep, iters = 1e-4, 0.1, 2
    ii, jj = T(p["ii"]), T(p["jj"])
    fixed = (T(p["intr"]), T(p["ext"]), T(p["sens"]), T(p["target"]), T(p["weight"]), T(p["eta"]))
    poses, disps = T(p["poses"].copy()), T(p["disps"].copy())
    dx, dz = db.ba(poses, T(p["poses"].copy()), disps, *fixed, ii, jj, p["kf0"], p["kf1"], iters, lm, ep, False)
    rposes, rdisps = T(p["poses"].copy()), T(p["disps"].copy())
    for _ in range(iters):
        rH, rv, rQ, rE, rw, _, _ = refdroid.reduced_camera_matrix(rposes, rposes, rdisps, *fixed, ii, jj, p["kf0"], p["kf1"])
        A = rH.double().cpu()
        A = A + torch.diag(ep + lm * torch.diagonal(A))
        rdx = torch.cholesky_solve(rv.double().cpu(), torch.linalg.cholesky(A)).float().view(-1, 6).to(DEV).contiguous()
        refdroid.solve_depth(rdx, rdisps, rQ, rE, rw, ii, jj, p["kf0"], p["kf1"])
        refdroid.solve_poses(rposes, rdx, p["kf0"], p["kf1"])
    assert torch.allclose(dx, rdx, rtol=2e-3, atol=2e-6)
    sgn = torch.sign((poses[:, 3:] * rposes[:, 3:]).sum(-1, keepdim=True))
    assert torch.allclose(poses[:, :3], rposes[:, :3], atol=2e-5) and torch.allclose(poses[:, 3:] * sgn, rposes[:, 3:], atol=2e-5)
    assert torch.allclose(disps, rdisps, rtol=5e-4, atol=5e-5)


def test_misc_geometry_vs_reference(db, refdroid):
    rng = np.random.default_rng(1238)
    poses, disps, intr, ii, jj = make_window(rng, 8, 30, 40)
    a = (T(poses), T(disps), T(intr), T(ii), T(jj))
    rc, rv = refdroid.projmap(*a)
    c, v = db.projmap(*a)
    assert torch.allclose(c[..., :2], rc[..., :2], atol=1e-3) and torch.equal(v, rv)
    assert torch.allclose(db.iproj(*a[:3]), refdroid.iproj(*a[:3]), rtol=1e-5, atol=1e-5)
    inds = T(np.array([1, 4])); th = T(np.array([0.05, 0.1], np.float32))
    assert torch.equal(db.depth_filter(a[0], a[1], a[2], inds, th), refdroid.depth_filter(a[0], a[1], a[2], inds, th))
    dxp = T(np.random.default_rng(1).normal(0, 1e-2, (8, 6)).astype(np.float32))
    p1 = T(poses.copy()); p2 = T(poses.copy())
    refdroid.solve_poses(p1, dxp, 0, 8); db.solve_poses(p2, dxp, 0, 8)
    assert torch.allclose(p1, p2, atol=1e-6)
