"""GPU parity tests: hand-written sm_90a kernels (through the C ABI) vs the CPU oracle on the same
seeded inputs.  Tolerances are stated per test (SURVEY.md §8c / north_star: bit-exact for the
fp16 lookup and integer work, fp32 tolerances elsewhere)."""
import os

import numpy as np
import pytest
import torch

from oracle import ba as oba
from oracle import corr as ocorr
from oracle import geom as ogeom
from oracle import se3
from tests.util import make_targets, make_window

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def T(x, dtype=None):
    t = torch.from_numpy(np.ascontiguousarray(x)).to(DEV)
    return t if dtype is None else t.to(dtype)


@pytest.fixture(scope="module")
def db():
    from nerf_slam_b200 import droid_backends
    return droid_backends


# ------------------------------------------------------------------------------------------ A3
@pytest.mark.parametrize("shape", [(2, 6, 8, 6, 8), (3, 30, 40, 30, 40), (1, 5, 7, 3, 2)])
def test_corr_lookup_fp16_bit_exact(db, shape):
    rng = np.random.default_rng(11)
    n, h1, w1, h2, w2 = shape
    vol = rng.normal(0, 1, shape).astype(np.float16)
    base = np.stack(np.meshgrid(np.arange(w1), np.arange(h1)), 0)[None].astype(np.float32) * (w2 / w1)
    coords = (base + rng.uniform(-8, 8, (n, 2, h1, w1))).astype(np.float32)
    ref = ocorr.corr_index_forward(vol, coords, 3)
    out, = db.corr_index_forward(T(vol), T(coords), 3)
    got = out.cpu().numpy()
    assert got.dtype == np.float16 and got.shape == ref.shape
    # bit-exact up to the sign of zero
    assert np.array_equal(got.astype(np.float32), ref.astype(np.float32))


def test_corr_lookup_fp32(db):
    rng = np.random.default_rng(12)
    vol = rng.normal(0, 1, (2, 6, 8, 6, 8)).astype(np.float32)
    coords = rng.uniform(-3, 10, (2, 2, 6, 8)).astype(np.float32)
    ref = ocorr.corr_index_forward(vol, coords, 3)
    out, = db.corr_index_forward(T(vol), T(coords), 3)
    assert np.allclose(out.cpu().numpy(), ref, atol=1e-6)


def test_corr_lookup_pyramid_fused_equals_per_level(db):
    rng = np.random.default_rng(13)
    E, C, H, W = 2, 16, 16, 24
    f = rng.normal(0, 1, (2 * E, C, H, W)).astype(np.float16)
    pyr = ocorr.corr_volume_pyramid(f[:E], f[E:])
    coords = (np.stack(np.meshgrid(np.arange(W), np.arange(H)), 0)[None] + rng.uniform(-6, 6, (E, 2, H, W))).astype(np.float32)
    ref = ocorr.corr_lookup_pyramid(pyr, coords, 3)
    got = db.corr_lookup_pyramid([T(p) for p in pyr], T(coords), 3).cpu().numpy()
    assert np.array_equal(got.astype(np.float32), ref.astype(np.float32))


def test_corr_lookup_empty(db):
    out, = db.corr_index_forward(torch.zeros(0, 4, 4, 4, 4, dtype=torch.float16, device=DEV),
                                 torch.zeros(0, 2, 4, 4, device=DEV), 3)
    assert out.shape == (0, 7, 7, 4, 4)


# ------------------------------------------------------------------------------------------ A2
@pytest.mark.parametrize("hw", [(16, 32), (30, 40), (60, 80), (43, 77)])
@pytest.mark.parametrize("simt", [True, False])
def test_corr_volume_pyramid(db, hw, simt):
    """fp16 volume: tensor-core accumulation order differs from the oracle's -> allow 1 fp16 ulp
    on level 0 (|x| <~ 8 => 2^-8 abs... use 2e-2 abs) and on the pooled levels."""
    rng = np.random.default_rng(21)
    H, W = hw
    C, NF = 128, 3
    fm = rng.normal(0, 1, (NF, C, H, W)).astype(np.float16)
    ii = np.array([0, 1, 2, 0], np.int32); jj = np.array([1, 0, 2, 2], np.int32)
    ref = ocorr.corr_volume_pyramid(fm[ii], fm[jj])
    nhwc = T(np.ascontiguousarray(fm.transpose(0, 2, 3, 1)))
    outs = db.corr_volume_build(nhwc, T(ii), T(jj), simt=simt)
    torch.cuda.synchronize()
    for l in range(4):
        got = outs[l].cpu().numpy().astype(np.float32)
        r = ref[l].astype(np.float32)
        assert got.shape == r.shape
        if r.size:
            err = np.abs(got - r).max()
            assert err <= 2e-2, f"level {l}: max err {err}"
            assert (got == r).mean() > 0.98, f"level {l}: only {(got == r).mean():.4f} bit-equal"


# ------------------------------------------------------------------------------------------ A4
@pytest.mark.parametrize("dtype", [np.float32, np.float16])
def test_altcorr(db, dtype):
    rng = np.random.default_rng(31)
    B, H, W, C = 2, 12, 16, 128
    f1 = (rng.normal(0, 1, (B, H, W, C)) / 4).astype(dtype)
    f2 = (rng.normal(0, 1, (B, H // 2, W // 2, C)) / 4).astype(dtype)
    coords = (np.stack(np.meshgrid(np.arange(W), np.arange(H)), -1)[None, None] / 2 + rng.uniform(-4, 4, (B, 1, H, W, 2))).astype(np.float32)
    ref = ocorr.altcorr_forward(f1, f2, coords, 3).astype(np.float32)
    out, = db.altcorr_forward(T(f1), T(f2), T(coords), 3)
    got = out.float().cpu().numpy()
    tol = 1e-4 if dtype == np.float32 else 2e-2
    assert np.allclose(got, ref, atol=tol), np.abs(got - ref).max()


# ------------------------------------------------------------------------------------------ A6 / A16 / misc geometry
def test_reproject(db):
    rng = np.random.default_rng(41)
    poses, disps, intr, ii, jj = make_window(rng, 6, 30, 40)
    ii = np.concatenate([ii, [2]]); jj = np.concatenate([jj, [2]])   # a stereo edge
    K = np.tile(intr, (6, 1)) * rng.uniform(0.95, 1.05, (6, 1)).astype(np.float32)
    ref_c, ref_v = ogeom.reproject(poses, disps, K, ii, jj)
    c, v = db.reproject(T(poses), T(disps), T(K.astype(np.float32)), T(ii), T(jj))
    assert np.allclose(c.cpu().numpy(), ref_c, atol=2e-3)
    assert (v.cpu().numpy() == ref_v).mean() > 0.999


def test_frame_distance(db):
    rng = np.random.default_rng(42)
    poses, disps, intr, _, _ = make_window(rng, 8, 60, 80)
    ii, jj = np.meshgrid(np.arange(8), np.arange(8), indexing="ij")
    ii, jj = ii.reshape(-1), jj.reshape(-1)
    ref = ogeom.frame_distance(poses, disps, intr, ii, jj, 0.3, np.float32)
    got = db.frame_distance(T(poses), T(disps), T(intr), T(ii), T(jj), 0.3).cpu().numpy()
    assert np.allclose(got, ref, rtol=2e-5, atol=1e-6)
    # ordering contract (SURVEY.md §9.20): argsort agrees wherever the oracle gap exceeds fp32 noise
    o = np.argsort(ref, kind="stable")
    gaps = np.diff(ref[o])
    safe = gaps > 1e-4 * np.maximum(1, ref[o][1:])
    assert np.all(np.diff(got[o])[safe] > 0)


def test_frame_distance_invalid_returns_1000(db):
    poses = np.array([[0, 0, 0, 0, 0, 0, 1], [0, 0, -10, 0, 0, 0, 1]], np.float32)  # target far behind
    disps = np.ones((2, 8, 8), np.float32)
    intr = np.array([8, 8, 3.5, 3.5], np.float32)
    got = db.frame_distance(T(poses), T(disps), T(intr), T(np.array([0])), T(np.array([1])), 0.3).cpu().numpy()
    assert got[0] == 1000.0


def test_projmap_iproj_depth_filter(db):
    rng = np.random.default_rng(43)
    poses, disps, intr, ii, jj = make_window(rng, 7, 20, 24)
    c, v = db.projmap(T(poses), T(disps), T(intr), T(ii), T(jj))
    rc, rv = ogeom.projmap(poses, disps, intr, ii, jj)
    assert np.allclose(c.cpu().numpy(), rc, atol=2e-3) and (v.cpu().numpy() == rv).mean() > 0.999
    p = db.iproj(T(poses), T(disps), T(intr)).cpu().numpy()
    assert np.allclose(p, ogeom.iproj(poses, disps, intr), rtol=1e-4, atol=1e-4)
    inds = np.array([0, 3, 6]); th = np.array([0.05, 0.1, 0.2], np.float32)
    cnt = db.depth_filter(T(poses), T(disps), T(intr), T(inds), T(th)).cpu().numpy()
    rc = ogeom.depth_filter(poses, disps, intr, inds, th)
    assert (cnt == rc).mean() > 0.995


# ------------------------------------------------------------------------------------------ A17
@pytest.mark.parametrize("mdt", [np.float32, np.float16])
def test_cvx_upsample(db, mdt):
    rng = np.random.default_rng(51)
    K, ht, wd = 3, 30, 40
    data = rng.uniform(0.1, 2, (K, ht, wd)).astype(np.float32)
    mask = rng.normal(0, 2, (K, 576, ht, wd)).astype(mdt)
    ref = ogeom.cvx_upsample(data, mask, 1.0, half_weights=(mdt == np.float16))
    m = T(mask)
    got = db.cvx_upsample(T(data).unsqueeze(-1), m, 1.0).squeeze(-1).cpu().numpy()
    assert np.allclose(got, ref, atol=2e-3 if mdt == np.float16 else 1e-5)
    assert torch.isfinite(m.float()).all()   # caller's mask is not mutated (the reference writes -inf)
    got2 = db.cvx_upsample(T(data).unsqueeze(-1), m, 0.5).squeeze(-1).cpu().numpy()
    ref2 = ogeom.cvx_upsample(data, mask, 0.5, half_weights=(mdt == np.float16))
    assert np.allclose(got2, ref2, atol=5e-3 if mdt == np.float16 else 1e-4)


# ------------------------------------------------------------------------------------------ A7-A14
def _ba_problem(seed, nframes=6, ht=30, wd=40, kf0=0, with_sensor=False, ext=None):
    rng = np.random.default_rng(seed)
    poses, disps, intr, ii, jj = make_window(rng, nframes, ht, wd)
    target, weight = make_targets(rng, poses, disps, intr, ii, jj)
    if ext is None:
        ext = np.array([0, 0, 0, 0, 0, 0, 1], np.float32)
    kf1 = int(max(ii.max(), jj.max())) + 1
    kx = np.unique(np.concatenate([np.arange(kf0, kf1), ii]))
    eta = rng.uniform(1e-3, 1e-1, (len(kx), ht, wd)).astype(np.float32)
    sens = np.zeros_like(disps)
    if with_sensor:
        sens[::2] = disps[::2] * rng.uniform(0.9, 1.1, disps[::2].shape).astype(np.float32)
        sens[:, :3] = 0
    return dict(poses=poses, disps=disps, intr=intr, ii=ii, jj=jj, target=target, weight=weight,
                ext=ext, kf0=kf0, kf1=kf1, eta=eta, sens=sens)


@pytest.mark.parametrize("cfg", [dict(seed=61), dict(seed=62, kf0=2), dict(seed=63, with_sensor=True),
                                 dict(seed=64, ext=np.array([0.06, -0.02, -0.01, 0.0077, -0.0105, -0.7018, 0.7123], np.float32)),
                                 dict(seed=65, nframes=10, ht=60, wd=80)])
def test_reduced_camera_matrix(db, cfg):
    """H, v, Q, E, w against the fp64 oracle. fp32 kernels: rel 2e-4 of the block scale."""
    p = _ba_problem(**cfg)
    ref = oba.reduced_camera_matrix(p["poses"], p["disps"], p["intr"], p["ext"], p["sens"], p["target"],
                                    p["weight"], p["eta"], p["ii"], p["jj"], p["kf0"], p["kf1"])
    H, v, Q, E, w = db.reduced_camera_matrix(
        T(p["poses"]), T(p["poses"]), T(p["disps"]), T(p["intr"]), T(p["ext"]), T(p["sens"]),
        T(p["target"]), T(p["weight"]), T(p["eta"]), T(p["ii"]), T(p["jj"]), p["kf0"], p["kf1"])
    prob = db.reduced_camera_matrix.last_problem

    def close(a, b, rel, name):
        a = a.cpu().numpy().reshape(b.shape)
        scale = np.abs(b).max() + 1e-12
        err = np.abs(a - b).max() / scale
        assert err < rel, f"{name}: rel err {err:.3e}"
    close(prob.Hs, ref["Hs"], 2e-4, "Hs")
    close(prob.vs, ref["vs"], 2e-4, "vs")
    close(Q, ref["Q"], 1e-4, "Q")
    close(w, ref["w"], 2e-4, "w")
    close(E, ref["E"], 2e-4, "E")
    close(H, ref["H"], 5e-4, "H")
    close(v, ref["v"].reshape(-1, 1), 5e-4, "v")


def test_ba_full_iteration(db):
    """linearise -> solve (+prior) -> retract -> depth update, vs oracle; then covariances."""
    p = _ba_problem(66, nframes=7)
    dev_poses = T(p["poses"])
    wTb0 = np.stack([np.concatenate(se3.inv_se3(q[:3].astype(np.float64), q[3:].astype(np.float64))) for q in p["poses"]]).astype(np.float32)
    disps = T(p["disps"])
    prob = db.BAProblem(dev_poses, disps, T(p["intr"]), T(p["ext"]), T(p["sens"]), T(p["target"]),
                        T(p["weight"]), T(p["eta"]), p["ii"], p["jj"], p["kf0"], p["kf1"])
    prob.linearize()
    ref = oba.reduced_camera_matrix(p["poses"], p["disps"], p["intr"], p["ext"], p["sens"], p["target"],
                                    p["weight"], p["eta"], p["ii"], p["jj"], p["kf0"], p["kf1"])
    err6 = torch.zeros(6, device=DEV)
    dx, linv, status = prob.solve(prior_idx=0, prior_err=err6, prior_info=1e8, want_linv=True)
    assert int(status.item()) == 0
    # the solve is checked against the system the GPU itself assembled (fp32 H -> fp64 Cholesky)
    Hg = prob.H.double().cpu().numpy(); vg = prob.v.double().cpu().numpy().reshape(-1)
    rdx, L = oba.dense_solve(Hg, vg, 0, np.zeros(6), 1e8)
    assert np.allclose(dx.cpu().numpy(), rdx, rtol=1e-4, atol=1e-7)
    Hp = Hg.copy(); Hp[:6, :6] += 1e8 * np.eye(6)
    res = Hp @ dx.double().cpu().numpy().reshape(-1) - vg
    assert np.abs(res).max() <= 1e-5 * max(1.0, np.abs(vg).max())
    # and against the oracle's own linearisation (looser: fp32 assembly)
    odx, _ = oba.dense_solve(ref["H"], ref["v"], 0, np.zeros(6), 1e8)
    assert np.allclose(dx.cpu().numpy(), odx, rtol=5e-2, atol=5e-5)
    # L^-1
    Li = np.linalg.inv(L)
    assert np.allclose(linv.cpu().numpy(), Li, rtol=1e-3, atol=1e-6 * np.abs(Li).max())
    # retract
    from nerf_slam_b200 import _lib
    lib = _lib.load()
    wTb = T(wTb0.copy()); cTw = T(p["poses"].copy()); ext = T(p["ext"])
    _lib.check(lib.nslam_ba_retract(_lib.ptr(wTb), _lib.ptr(cTw), _lib.ptr(ext), _lib.ptr(dx),
                                    p["kf0"], prob.gh.P, _lib.stream_ptr()), "retract")
    rw, rc = oba.gtsam_retract(wTb0, p["ext"], dx.cpu().numpy(), p["kf0"])

    def pose_close(a, b, tol):
        a = a.astype(np.float64); sgn = np.sign((a[:, 3:] * b[:, 3:]).sum(-1, keepdims=True))
        return np.allclose(a[:, :3], b[:, :3], atol=tol) and np.allclose(a[:, 3:] * sgn, b[:, 3:], atol=tol)
    assert pose_close(wTb.cpu().numpy(), rw, 1e-6) and pose_close(cTw.cpu().numpy(), rc, 1e-5)
    # depth update (uses the GPU's own Q,E,w; oracle formula)
    rd, _ = oba.solve_depth(dx.cpu().numpy(), p["disps"], prob.Q.cpu().numpy(), prob.E.cpu().numpy(),
                            prob.w.cpu().numpy(), p["ii"], p["jj"], p["kf0"], p["kf1"])
    prob.depth_update(dx, clamp_min=1e-3)
    assert np.allclose(disps.cpu().numpy(), np.maximum(rd, 1e-3), rtol=1e-4, atol=1e-5)
    # covariances
    sg, zc, dc = prob.covariances(linv, reference=False)             # the kernel alone = the intended formula
    rsg, rzc, rdc = oba.covariances(L, prob.E.double().cpu().numpy(), prob.Q.double().cpu().numpy(),
                                    p["ii"], p["jj"], p["kf0"], p["kf1"], disps.cpu().numpy())
    assert np.allclose(sg.cpu().numpy(), rsg, rtol=2e-3, atol=1e-9)
    assert np.allclose(zc.cpu().numpy().reshape(rzc.shape), rzc, rtol=2e-3, atol=1e-9)
    assert np.allclose(dc.cpu().numpy().reshape(rdc.shape), rdc, rtol=2e-3, atol=1e-9)


def test_ba_covariances_reference_exact(db):
    """A14, csrc/ba_cov_ref.cu: the reference's covariance block as it really behaves (Ei broadcast over the pose rows of
    optimised frames, visual_frontend.py:1214) vs oracle.covariances_reference, which is pinned on the CPU against the
    reference's own code (tests/golden/ref_covariances.npz); and on the golden's own inputs."""
    p = _ba_problem(66, nframes=7)
    disps = T(p["disps"])
    prob = db.BAProblem(T(p["poses"]), disps, T(p["intr"]), T(p["ext"]), T(p["sens"]), T(p["target"]),
                        T(p["weight"]), T(p["eta"]), p["ii"], p["jj"], p["kf0"], p["kf1"])
    prob.linearize()
    dx, linv, status = prob.solve(prior_idx=0, prior_err=torch.zeros(6, device=DEV), prior_info=1e8, want_linv=True)
    assert int(status.item()) == 0
    Hg = prob.H.double().cpu().numpy(); vg = prob.v.double().cpu().numpy().reshape(-1)
    _, L = oba.dense_solve(Hg, vg, 0, np.zeros(6), 1e8)
    rsg, rzc, rdc = oba.covariances_reference(L, prob.E.double().cpu().numpy(), prob.Q.double().cpu().numpy(),
                                              p["ii"], p["jj"], p["kf0"], p["kf1"], disps.cpu().numpy())
    assert prob.gh.K == rzc.shape[0]                      # every frame of the window has outgoing edges in this problem
    for mode in ("1", "kernel"):                          # kernel + torch fix-up (the default) / one CUDA kernel
        sg, zc, dc = prob.covariances(linv, reference=mode)
        assert np.allclose(sg.cpu().numpy(), rsg, rtol=2e-3, atol=1e-9), mode
        assert np.allclose(zc.cpu().numpy().reshape(rzc.shape), rzc, rtol=2e-3, atol=1e-9), mode
        assert np.allclose(dc.cpu().numpy().reshape(rdc.shape), rdc, rtol=2e-3, atol=1e-9), mode
    _, zi, _ = prob.covariances(linv, reference=False)
    assert not np.allclose(zi.cpu().numpy().reshape(rzc.shape), rzc, rtol=1e-2)          # the two formulas do differ


@pytest.mark.parametrize("cov_mode", [1, 0])
def test_ba_frontend_update_matches_piecewise_path(db, cov_mode):
    """nslam_ba_frontend_update (the live path's one-call BA step: 2 Gauss-Newton iterations + covariances written into
    the keyframe arenas) vs the piecewise entry points each validated above (gauss_newton, covariances)."""
    p = _ba_problem(68, nframes=7)
    wTb0 = np.stack([np.concatenate(se3.inv_se3(q[:3].astype(np.float64), q[3:].astype(np.float64))) for q in p["poses"]]).astype(np.float32)
    N, (ht, wd) = p["disps"].shape[0], p["disps"].shape[1:]
    prior = T(wTb0[p["kf0"]].copy())

    def fresh():
        cTw, wTb, disps = T(p["poses"].copy()), T(wTb0.copy()), T(p["disps"].copy())
        prob = db.BAProblem(cTw, disps, T(p["intr"]), T(p["ext"]), T(p["sens"]), T(p["target"]), T(p["weight"]), T(p["eta"]),
                            p["ii"], p["jj"], p["kf0"], p["kf1"])
        return prob, cTw, wTb, disps
    # piecewise
    prob, cTw, wTb, disps = fresh()
    dx, linv, status = prob.gauss_newton(2, wTb, cTw, T(p["ext"]), prior_idx=0, prior_pose=prior, prior_info=1e8, want_linv=True)
    assert int(status.item()) == 0
    sg, zc, dc = prob.covariances(linv, reference="1" if cov_mode else "0")
    kx = prob.gh.tables["kx"].astype(np.int64)
    # one call, arenas
    prob2, cTw2, wTb2, disps2 = fresh()
    st = torch.zeros(2, dtype=torch.int32, device=DEV)
    zarena = torch.full((N, ht, wd), -7.0, device=DEV); darena = torch.full((N, ht, wd), -7.0, device=DEV)
    parena = torch.full((N, 6, 6), -7.0, device=DEV)
    dx2, _ = prob2.frontend_update(2, wTb2, cTw2, T(p["ext"]), st, prior_idx=0, prior_pose=prior, prior_info=1e8,
                                   cov_mode=cov_mode, idepths_cov=zarena, depths_cov=darena, pose_cov=parena)
    assert st.tolist() == [0, 0]
    assert torch.equal(dx, dx2) and torch.equal(cTw, cTw2) and torch.equal(wTb, wTb2) and torch.equal(disps, disps2)
    assert np.allclose(zarena[kx].cpu().numpy(), zc.cpu().numpy(), rtol=2e-5, atol=1e-12)
    assert np.allclose(darena[kx].cpu().numpy(), dc.cpu().numpy(), rtol=2e-5, atol=1e-12)
    assert np.allclose(parena[p["kf0"]:p["kf1"]].cpu().numpy(), sg.cpu().numpy(), rtol=1e-6, atol=0)
    rest = np.setdiff1d(np.arange(N), kx)
    assert (zarena[rest] == -7.0).all() and (darena[rest] == -7.0).all()          # rows of untouched frames stay
    outside = np.setdiff1d(np.arange(N), np.arange(p["kf0"], p["kf1"]))
    assert (parena[outside] == -7.0).all()


def test_ba_frontend_update_failed_factorisation_changes_nothing(db):
    """ADVICE r1: a singular window (zero confidence weights, no prior, no damping of the poses) must not corrupt the
    state: poses, depths and covariance arenas stay as they were, status = [1, #failures]."""
    p = _ba_problem(69, nframes=6)
    wTb0 = np.stack([np.concatenate(se3.inv_se3(q[:3].astype(np.float64), q[3:].astype(np.float64))) for q in p["poses"]]).astype(np.float32)
    N, (ht, wd) = p["disps"].shape[0], p["disps"].shape[1:]
    cTw, wTb, disps = T(p["poses"].copy()), T(wTb0.copy()), T(p["disps"].copy())
    prob = db.BAProblem(cTw, disps, T(p["intr"]), T(p["ext"]), T(p["sens"]), T(p["target"]), T(np.zeros_like(p["weight"])),
                        T(p["eta"]), p["ii"], p["jj"], p["kf0"], p["kf1"])
    st = torch.zeros(2, dtype=torch.int32, device=DEV)
    zarena = torch.full((N, ht, wd), -7.0, device=DEV); darena = zarena.clone(); parena = torch.full((N, 6, 6), -7.0, device=DEV)
    prob.frontend_update(2, wTb, cTw, T(p["ext"]), st, prior_idx=-1, cov_mode=1, idepths_cov=zarena, depths_cov=darena, pose_cov=parena)
    assert st.tolist() == [1, 2]
    assert np.array_equal(cTw.cpu().numpy(), p["poses"]) and np.array_equal(wTb.cpu().numpy(), wTb0)
    assert np.array_equal(disps.cpu().numpy(), p["disps"])
    assert (zarena == -7.0).all() and (darena == -7.0).all() and (parena == -7.0).all()


def test_solve_depth_and_poses_api(db):
    p = _ba_problem(67)
    H, v, Q, E, w = db.reduced_camera_matrix(
        T(p["poses"]), T(p["poses"]), T(p["disps"]), T(p["intr"]), T(p["ext"]), T(p["sens"]),
        T(p["target"]), T(p["weight"]), T(p["eta"]), T(p["ii"]), T(p["jj"]), p["kf0"], p["kf1"])
    rng = np.random.default_rng(0)
    dx = (rng.normal(0, 1e-2, (p["kf1"] - p["kf0"], 6))).astype(np.float32)
    disps = T(p["disps"].copy())
    db.solve_depth(T(dx), disps, Q, E, w, T(p["ii"]), T(p["jj"]), p["kf0"], p["kf1"])
    rd, _ = oba.solve_depth(dx, p["disps"], Q.cpu().numpy(), E.cpu().numpy(), w.cpu().numpy(),
                            p["ii"], p["jj"], p["kf0"], p["kf1"])
    assert np.allclose(disps.cpu().numpy(), rd, rtol=1e-4, atol=1e-5)
    poses = T(p["poses"].copy())
    db.solve_poses(poses, T(dx), p["kf0"], p["kf1"])
    t, q = se3.retr_se3(dx.astype(np.float64), p["poses"][:, :3].astype(np.float64), p["poses"][:, 3:].astype(np.float64))
    assert np.allclose(poses.cpu().numpy(), np.concatenate([t, q], -1), atol=1e-5)


def test_solver_failure_zeroes_update(db):
    """Cholesky failure => zero step, never crash (SURVEY.md §5; src/droid_kernels.cu:1333-1337)"""
    from nerf_slam_b200 import _lib
    lib = _lib.load()
    H = -torch.eye(12, device=DEV); v = torch.ones(12, 1, device=DEV)
    work = torch.empty(2 * 144 + 24, dtype=torch.float64, device=DEV)
    dx = torch.ones(2, 6, device=DEV); st = torch.zeros(1, dtype=torch.int32, device=DEV)
    _lib.check(lib.nslam_ba_solve(_lib.ptr(H), _lib.ptr(v), 2, -1, None, 0.0, 0.0, 0.0, _lib.ptr(work),
                                  _lib.ptr(dx), None, _lib.ptr(st), _lib.stream_ptr()), "solve")
    assert int(st.item()) == 1 and float(dx.abs().max()) == 0.0


def test_pose_prior_error(db):
    from nerf_slam_b200 import _lib
    lib = _lib.load()
    rng = np.random.default_rng(5)
    p = se3.random_poses(rng, 2, 0.3, 20, np.float32)
    err = torch.zeros(6, device=DEV)
    x_d, pr_d = T(p[0]), T(p[1])      # keep both alive: temporaries would alias after being freed
    _lib.check(lib.nslam_pose_prior_error(_lib.ptr(x_d), _lib.ptr(pr_d), _lib.ptr(err), _lib.stream_ptr()), "prior")
    assert np.allclose(err.cpu().numpy(), oba.pose_prior_error(p[0], p[1]), atol=1e-5)
    # retract(prior, err) == x
    t, q = se3.pose3_retract(p[1, :3].astype(np.float64), p[1, 3:].astype(np.float64), err.double().cpu().numpy())
    assert np.allclose(t, p[0, :3], atol=1e-5)


@pytest.mark.parametrize("H,W,spread", [(30, 41, 6), (60, 80, 12), (16, 64, 40), (21, 48, 9)])
def test_corr_lookup_nhwc_equals_reference_layout(db, H, W, spread):
    """channels-last / slot-indirected variant == reference-layout kernel (bit for bit).  (30,41): odd width, partial
    32-pixel groups, scalar gathers; (60,80), (16,64), (22,48): level widths multiples of 8 -> the 128-bit kernel
    (aligned chunk pairs + select network on levels 0/1, staged slices on levels 2/3; (21,48) has a partial last CTA
    and odd pooled sizes); spread 40 px sends many windows partly or wholly out of the volume."""
    rng = np.random.default_rng(14)
    E, C = 3, 16
    f = rng.normal(0, 1, (2 * E, C, H, W)).astype(np.float16)
    pyr = [T(p) for p in ocorr.corr_volume_pyramid(f[:E], f[E:])]
    coords = (np.stack(np.meshgrid(np.arange(W), np.arange(H)), 0)[None] + rng.uniform(-spread, spread, (E, 2, H, W))).astype(np.float32)
    ref = db.corr_lookup_pyramid(pyr, T(coords), 3)                                     # [E,196,H,W]
    slots = T(np.array([2, 0, 1], np.int32))
    perm = [pyr_l[[1, 2, 0]] for pyr_l in pyr]                                         # slot s holds edge perm^-1
    got = db.corr_lookup_pyramid([p.contiguous() for p in perm], T(np.ascontiguousarray(coords.transpose(0, 2, 3, 1))), 3,
                                 slots=slots, nhwc_stride=200, coords_nhwc=True)        # [E,H,W,200]
    assert torch.equal(got[..., :196].permute(0, 3, 1, 2).float(), ref.float())
    assert float(got[..., 196:].abs().max()) == 0.0


def test_corr_pool_builds_scattered_slots_in_one_launch():
    """CorrPool.build: all new edges of a keyframe in ONE launch, each volume into the arena slot it was given
    (nslam_corr_volume_build_slots) == one build per edge; other slots untouched"""
    from nerf_slam_b200 import droid_backends as db
    from nerf_slam_b200.corr import CorrPool
    g = torch.Generator().manual_seed(78)
    H, W, NF = 16, 64, 5
    fm = torch.randn(NF, H, W, 128, generator=g).half().to("cuda:0")
    pool = CorrPool(9, H, W, "cuda:0")
    for lv in pool.levels:
        lv.fill_(-3.0)
    fi, fj, slots = [0, 3, 1, 4], [1, 3, 2, 0], [7, 2, 5, 0]
    pool.build(fm, fi, fj, slots)
    torch.cuda.synchronize()
    ref = db.corr_volume_build(fm, torch.tensor(fi, dtype=torch.int32, device="cuda:0"), torch.tensor(fj, dtype=torch.int32, device="cuda:0"))
    for l in range(4):
        assert torch.equal(pool.levels[l][slots], ref[l])
        rest = [s for s in range(9) if s not in slots]
        assert bool((pool.levels[l][rest] == -3.0).all())


@pytest.mark.parametrize("H,W,E", [(60, 80, 3), (16, 64, 2), (30, 80, 1)])
def test_corr_volume_rows_matches_tiled_kernel(H, W, E):
    """csrc/corr_volume_rows.cu (two full target rows per MMA tile) must reproduce csrc/corr_volume.cu bit for
    bit: same K order in the fp32 accumulation, same fp16 rounding chain of the pyramid"""
    import ctypes
    from nerf_slam_b200 import _lib
    lib = _lib.load()
    g = torch.Generator().manual_seed(77)
    NF = 4
    fm = torch.randn(NF, H, W, 128, generator=g).half().to("cuda:0")
    ii = torch.randint(0, NF, (E,), generator=g).int().to("cuda:0"); jj = torch.randint(0, NF, (E,), generator=g).int().to("cuda:0")
    mk = lambda: [torch.zeros(E, H, W, H >> l, W >> l, dtype=torch.float16, device="cuda:0") for l in range(4)]
    a, b = mk(), mk()
    _lib.check(lib.nslam_corr_volume_build(_lib.ptr(fm), NF, H, W, 128, _lib.ptr(ii), _lib.ptr(jj), E,
                                           *[_lib.ptr(o) for o in a], _lib.stream_ptr()), "tiled")
    _lib.check(lib.nslam_corr_volume_build_rows(_lib.ptr(fm), NF, H, W, 128, _lib.ptr(ii), _lib.ptr(jj), E,
                                                *[_lib.ptr(o) for o in b], _lib.stream_ptr()), "rows")
    torch.cuda.synchronize()
    for l in range(4):
        assert torch.equal(a[l], b[l]), (l, float((a[l].float() - b[l].float()).abs().max()))


def test_droid_backends_ba_all_in_one_loop(db):
    """A15: droid_backends.ba (ba_cuda, src/droid_kernels.cu:1441-1568, motion_only=False) = per iteration
    linearise -> (A - S) solve with `ep + lm*diag` damping -> depth back-substitution -> left pose retraction, all
    in place.  Oracle: the same composition of oracle/ba.py + oracle/se3.py pieces, 2 iterations."""
    p = _ba_problem(71, nframes=6)
    lm, ep, iters = 1e-4, 0.1, 2
    poses = T(p["poses"].copy()); disps = T(p["disps"].copy())
    dx, dz = db.ba(poses, T(p["poses"].copy()), disps, T(p["intr"]), T(p["ext"]), T(p["sens"]), T(p["target"]),
                   T(p["weight"]), T(p["eta"]), T(p["ii"]), T(p["jj"]), p["kf0"], p["kf1"], iters, lm, ep, False)
    rp = p["poses"].astype(np.float64).copy(); rd = p["disps"].astype(np.float64).copy()
    for _ in range(iters):
        r = oba.reduced_camera_matrix(rp.astype(np.float32), rd.astype(np.float32), p["intr"], p["ext"], p["sens"], p["target"],
                                      p["weight"], p["eta"], p["ii"], p["jj"], p["kf0"], p["kf1"])
        rdx, _ = oba.dense_solve(r["H"], r["v"], lm=lm, ep=ep)
        rd, _ = oba.solve_depth(rdx, rd, r["Q"], r["E"], r["w"], p["ii"], p["jj"], p["kf0"], p["kf1"])
        t, q = se3.retr_se3(rdx.astype(np.float64), rp[p["kf0"]:p["kf1"], :3], rp[p["kf0"]:p["kf1"], 3:])
        rp[p["kf0"]:p["kf1"]] = np.concatenate([t, q], -1)
    got_p = poses.cpu().numpy().astype(np.float64)
    sgn = np.sign((got_p[:, 3:] * rp[:, 3:]).sum(-1, keepdims=True))
    assert np.allclose(got_p[:, :3], rp[:, :3], atol=2e-4) and np.allclose(got_p[:, 3:] * sgn, rp[:, 3:], atol=2e-4)
    assert np.allclose(disps.cpu().numpy(), rd, rtol=2e-3, atol=2e-4)
    assert dx.shape == (p["kf1"] - p["kf0"], 6) and torch.isfinite(dx).all() and torch.isfinite(dz).all()
