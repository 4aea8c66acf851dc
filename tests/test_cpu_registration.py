"""ICP without a GPU: the oracle (tests/registration_oracle.py) recovers known transforms of the synthetic room's surface
and of a sphere-plus-torus mesh with the product's host step; the host maths; a degenerate plane; the refusals; the
argument checks of tools/eval_reconstruction.py's alignment flags."""
import json
import math
import os
import sys

import numpy as np
import pytest

from nerf_slam_b200 import registration as reg
from tests import recon_eval_oracle as rorc
from tests import registration_oracle as ro

F32 = np.float32
TOOLS = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools")
ROOM_DISTS = {False: (0.2, 0.1, 0.05), True: (0.5, 0.2, 0.1, 0.05)}    # a 0.9 scale moves the room's walls by 0.3 m


# ------------------------------------------------------------------------------------------------------------- inputs
def room_mesh():
    from nerf_slam_b200.synthetic import SyntheticRoom
    return SyntheticRoom(64, 48, 2).surface_mesh()


def sphere_torus():
    """a UV sphere of radius 0.8 at (2.2, 0, 0) and a torus (R 1, r 0.3) about z at the origin: (vertices, triangles)"""
    def grid(f, nu, nv, wrap_v):
        u, v = np.meshgrid(np.arange(nu) * 2 * np.pi / nu, np.arange(nv + (0 if wrap_v else 1)) * (2 * np.pi / nv if wrap_v
                                                                                               else np.pi / nv), indexing="ij")
        V = f(u, v).reshape(-1, 3)
        m = v.shape[1]
        i, j = np.meshgrid(np.arange(nu), np.arange(nv), indexing="ij")
        a, b = i * m + j, ((i + 1) % nu) * m + j
        c, d = ((i + 1) % nu) * m + (j + 1) % m, i * m + (j + 1) % m
        return V, np.concatenate([np.stack([a, b, c], -1).reshape(-1, 3), np.stack([a, c, d], -1).reshape(-1, 3)])
    sV, sF = grid(lambda u, v: np.stack([2.2 + 0.8 * np.sin(v) * np.cos(u), 0.8 * np.sin(v) * np.sin(u), 0.8 * np.cos(v)], -1),
                  48, 24, False)
    tV, tF = grid(lambda u, v: np.stack([(1 + 0.3 * np.cos(v)) * np.cos(u), (1 + 0.3 * np.cos(v)) * np.sin(u), 0.3 * np.sin(v)],
                                        -1), 64, 24, True)
    return np.concatenate([sV, tV]).astype(F32), np.concatenate([sF, tF + len(sV)]).astype(np.int32)


def perturbation(scale=1.0, degrees=7.0):
    """a known similarity of about `degrees` about a tilted axis and 0.1 m: (s, R, t)"""
    axis = np.array([0.3, 1.0, 0.2])
    return scale, reg.rodrigues(np.deg2rad(degrees) * axis / np.linalg.norm(axis)), np.array([0.1, -0.05, 0.08])


def transform_error(T, s, R, t):
    """-> (largest translation error (m), rotation error (degrees), relative scale error) of T against the inverse of
    p -> s R p + t"""
    E = T @ reg.compose(s, R, t)
    se = np.cbrt(np.linalg.det(E[:3, :3]))
    ang = math.degrees(math.acos(min(1.0, max(-1.0, (np.trace(E[:3, :3] / se) - 1) / 2))))
    return float(np.abs(E[:3, 3]).max()), ang, abs(se - 1.0)


# ---------------------------------------------------------------------------------------------------- oracle recovery
# tolerances from the oracle runs (20 k samples each side) with a margin of about 5x: point-to-plane ends within
# 6e-5 m / 0.004 deg / 1e-4 of scale on the room, point-to-point within 1.3e-3 m / 0.024 deg / 5e-5
TOL = {"point_to_plane": (5e-4, 0.02, 5e-4), "point_to_point": (5e-3, 0.1, 5e-4)}


@pytest.mark.parametrize("metric", ["point_to_plane", "point_to_point"])
@pytest.mark.parametrize("with_scale", [False, True])
@pytest.mark.parametrize("shape", ["room", "sphere_torus"])
def test_oracle_icp_recovers_a_known_transform(metric, with_scale, shape):
    V, T = room_mesh() if shape == "room" else sphere_torus()
    src, _ = rorc.surface_samples(V, T, 20_000, 0)
    tgt, nrm = ro.sample_with_normals(V, T, 20_000, 1)
    s, R, t = perturbation(0.9 if with_scale else 1.0)
    dists = ROOM_DISTS[with_scale] if shape == "room" else (0.3, 0.1, 0.05)
    r = ro.icp(ro.transform(src, s, R, t), tgt, nrm if metric == "point_to_plane" else None, metric=metric,
               with_scale=with_scale, max_corr_dist=dists, max_iters=40)
    assert r["converged"] and not r["degenerate"]
    te, re, se = transform_error(r["transform"], s, R, t)
    tol = TOL[metric]
    assert te < tol[0] and re < tol[1] and se < tol[2], (te, re, se)
    if not with_scale:
        assert r["scale"] == 1.0
    assert r["fitness"] > 0.5 and r["inlier_rmse"] < 0.05


def test_a_single_plane_is_degenerate_under_point_to_plane():
    V = np.array([[-1, -1, 0], [1, -1, 0], [1, 1, 0], [-1, 1, 0]], F32)
    T = np.array([[0, 1, 2], [0, 2, 3]], np.int32)
    src, _ = rorc.surface_samples(V, T, 2000, 0)
    tgt, nrm = ro.sample_with_normals(V, T, 2000, 1)
    r = ro.icp(ro.transform(src, 1.0, np.eye(3), [0.0, 0.0, 0.05]), tgt, nrm, max_corr_dist=(0.2,))
    assert r["degenerate"] and r["iterations"] == 0 and not r["converged"]
    assert np.array_equal(r["transform"], np.eye(4))


# ---------------------------------------------------------------------------------------------------------- host maths
def test_rodrigues_is_a_rotation_about_its_axis():
    w = np.array([0.2, -0.4, 0.9])
    R = reg.rodrigues(w)
    assert np.allclose(R.T @ R, np.eye(3), atol=1e-15) and np.isclose(np.linalg.det(R), 1.0)
    assert np.allclose(R @ w, w, atol=1e-15)
    th = np.linalg.norm(w)
    assert np.isclose(np.trace(R), 1 + 2 * np.cos(th))
    Rz = reg.rodrigues([0, 0, np.pi / 2])
    assert np.allclose(Rz @ [1, 0, 0], [0, 1, 0], atol=1e-15)
    assert np.array_equal(reg.rodrigues([0, 0, 0]), np.eye(3))
    small = np.array([1e-13, 0, 0])
    assert np.allclose(reg.rodrigues(small), np.eye(3) + np.array([[0, 0, 0], [0, 0, -1e-13], [0, 1e-13, 0]]))


def test_compose_and_decompose_are_inverse_and_compose_like_maps():
    s, R, t = perturbation(0.9)
    T = reg.compose(s, R, t)
    s2, R2, t2 = reg.decompose(T)
    assert np.isclose(s2, s) and np.allclose(R2, R, atol=1e-15) and np.array_equal(t2, t)
    p = np.array([0.3, -1.2, 2.0])
    assert np.allclose(T[:3, :3] @ p + T[:3, 3], s * R @ p + t)
    U = reg.compose(1.3, reg.rodrigues([0.1, 0.2, -0.3]), [1.0, 2.0, 3.0])
    a, b, c = reg.decompose(U @ T)
    assert np.allclose(a * b @ p + c, U[:3, :3] @ (s * R @ p + t) + U[:3, 3])


def test_the_step_acts_on_normalised_coordinates():
    """apply_step moves world points as the normalised step moves (p - c) / L: p'' = L (e^sigma R_d p~ + tau) + c"""
    s, R, t = perturbation(0.9)
    c, L = [0.5, -0.2, 1.0], 3.7
    x = np.array([0.01, -0.02, 0.03, 0.004, -0.005, 0.006, 0.05])
    s2, R2, t2 = reg.apply_step(s, R, t, x, c, L)
    p = np.array([1.0, 2.0, -0.5])
    moved = s * R @ p + t
    pt = (moved - c) / L
    want = L * (math.exp(x[6]) * reg.rodrigues(x[:3]) @ pt + x[3:6]) + np.asarray(c)
    assert np.allclose(s2 * R2 @ p + t2, want, atol=1e-14)


def test_target_frame_and_sums_unpack():
    c, L = reg.target_frame([-3, -2, -3], [3, 2, 3])
    assert c == [0.0, 0.0, 0.0] and L == math.sqrt(22.0)
    sums = list(range(38))
    H, g, e, count, flags = reg.unpack_sums(sums)
    assert H[0, 0] == 0 and H[0, 6] == 6 / 2 ** 27 and H[6, 0] == H[0, 6] and H[1, 1] == 7 / 2 ** 27
    assert H[6, 6] == 27 / 2 ** 27 and g[0] == 28 / 2 ** 27 and e == 35 / 2 ** 27 and (count, flags) == (36, 37)


def test_fewer_correspondences_than_unknowns_is_degenerate():
    sums = [0] * 38
    k = 0
    for a in range(7):
        for b in range(a, 7):
            sums[k] = 2 ** 27 if a == b else 0
            k += 1
    sums[36] = 6
    assert reg.gauss_newton_step(sums, False) is not None and reg.gauss_newton_step(sums, True) is None


def test_terms_outside_their_bound_raise_the_flag():
    tgt = np.array([[0, 0, 0], [1, 0, 0]], F32)
    moved = np.array([[0.1, 0, 0]], F32)
    assert ro.accumulate(moved, [1], tgt, None, ((0.5, 0.0, 0.0), 0.5), True, True)[37] == 0
    assert ro.accumulate(moved, [1], tgt, np.full((2, 3), 30.0, F32), ((0.5, 0.0, 0.0), 0.5), False, False)[37] == 2
    assert ro.accumulate(moved, [5], tgt, None, ((0.5, 0.0, 0.0), 0.5), True, False)[37] == 1


# ------------------------------------------------------------------------------------------------------------ refusals
def test_invalid_similarities_are_refused():
    for T, match in ((np.eye(3), "4x4"), (np.full((4, 4), np.nan), "finite"), (np.diag([1.0, 1.0, 1.0, 2.0]), "bottom"),
                     (np.diag([1.0, 1.0, -1.0, 1.0]), "similarity"), (np.diag([1.0, 2.0, 1.0, 1.0]), "scaled rotation"),
                     (np.diag([0.0, 0.0, 0.0, 1.0]), "similarity")):
        with pytest.raises(ValueError, match=match):
            reg.decompose(T)


def test_host_refusals_before_any_kernel():
    import torch
    V, T = room_mesh()
    mesh = (torch.from_numpy(V), torch.from_numpy(T))
    with pytest.raises(RuntimeError, match="CUDA"):
        reg.icp(torch.zeros(10, 3), mesh)
    with pytest.raises(ValueError, match="metric"):
        reg.icp(torch.zeros(10, 3), mesh, metric="plane")
    with pytest.raises(ValueError, match="max_iters"):
        reg.icp(torch.zeros(10, 3), mesh, max_iters=0)
    with pytest.raises(ValueError, match="tol"):
        reg.icp(torch.zeros(10, 3), mesh, tol=float("nan"))
    with pytest.raises(ValueError, match="similarity"):
        reg.icp(torch.zeros(10, 3), mesh, init=np.diag([1.0, 1.0, -1.0, 1.0]))
    with pytest.raises(ValueError, match="align"):
        reg.trajectory_alignment(np.zeros((4, 7)), np.zeros((4, 7)), "none")
    with pytest.raises(RuntimeError, match="CUDA"):
        reg.transform(torch.zeros(4, 3), np.eye(4))


def test_trajectory_alignment_maps_the_estimated_centres_onto_the_true_ones():
    rng = np.random.default_rng(0)
    c_gt = rng.normal(0, 1, (20, 3))
    s, R, t = perturbation(0.5, 20.0)
    c_est = (c_gt - t) @ R / s                               # c_gt = s R c_est + t
    gt, est = np.tile(np.eye(4), (20, 1, 1)), np.tile(np.eye(4), (20, 1, 1))
    gt[:, :3, 3], est[:, :3, 3] = -c_gt, -c_est              # cam_T_world with identity rotations: centre = -t
    assert np.allclose(reg.trajectory_alignment(est, gt, "sim3"), reg.compose(s, R, t), atol=1e-9)
    B = reg.trajectory_alignment(est, gt, "se3")
    assert np.isclose(np.linalg.det(B[:3, :3]), 1.0) and np.allclose(B[:3, :3], R, atol=1e-9)


# ----------------------------------------------------------------------------------------------------------- the tool
def _tool(name):
    sys.path.insert(0, TOOLS)
    try:
        return __import__(name)
    finally:
        sys.path.remove(TOOLS)


@pytest.mark.parametrize("argv", [["r.ply", "g.ply", "--align", "sim3"],
                                  ["r.ply", "g.ply", "--align_metric", "point_to_point"],
                                  ["r.ply", "g.ply", "--align", "icp", "--align_metric", "plane"],
                                  ["r.ply", "g.ply", "--align", "icp", "--align_max_dist", "0.1,-0.05"],
                                  ["r.ply", "g.ply", "--align", "icp", "--align_max_dist", "0.1,nan"],
                                  ["r.ply", "g.ply", "--align", "icp", "--align_max_dist", ""],
                                  ["r.ply", "g.ply", "--align_max_dist", "0.1"],
                                  ["r.ply", "g.ply", "--init", "t.json"],
                                  ["r.ply", "g.ply", "--align", "icp", "--init", "/nonexistent/t.json"]])
def test_eval_reconstruction_alignment_argument_checks(argv):
    with pytest.raises(SystemExit):
        _tool("eval_reconstruction").main(argv)


def test_eval_reconstruction_init_file_checks(tmp_path):
    tool = _tool("eval_reconstruction")
    good = tmp_path / "good.json"
    good.write_text(json.dumps(reg.compose(*perturbation(0.9)).tolist()))
    assert np.allclose(tool.read_init(str(good)), reg.compose(*perturbation(0.9)))
    for bad in ([[1, 0, 0], [0, 1, 0], [0, 0, 1]], [[1, 0, 0, 0], [0, 1, 0, 0], [0, 0, -1, 0], [0, 0, 0, 1]], "x"):
        p = tmp_path / "bad.json"
        p.write_text(json.dumps(bad))
        with pytest.raises(SystemExit):
            tool.main(["r.ply", "g.ply", "--align", "icp", "--init", str(p)])
