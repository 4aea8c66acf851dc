"""Reconstruction evaluation, host side (nerf_slam_b200/evaluation.py) and the oracle it is tested against
(tests/recon_eval_oracle.py): PLY reading through both writers, trajectory alignment and error, the synthetic room's
ground-truth surface, the oracle's metrics on a known offset, and the GPU entry points refusing to run without CUDA."""
import os

import numpy as np
import pytest
import torch

from tests import recon_eval_oracle as orc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F32 = np.float32


# ------------------------------------------------------------------------------------------------------------------ PLY
def test_ply_round_trip_through_the_mesh_writer(tmp_path, rng):
    from nerf_slam_b200.evaluation import read_ply
    from nerf_slam_b200.tsdf_fusion import TsdfMesh
    V = rng.normal(0, 2, (57, 3)).astype(F32)
    T = rng.integers(0, 57, (91, 3)).astype(np.int32)
    C = rng.uniform(0, 1, (57, 3)).astype(F32)
    N = rng.normal(0, 1, (57, 3)).astype(F32)
    TsdfMesh(*(torch.from_numpy(a) for a in (V, T, C, N))).write_ply(str(tmp_path / "m.ply"))
    v, t = read_ply(str(tmp_path / "m.ply"))
    assert v.dtype == np.float32 and np.array_equal(v, V)
    assert t.dtype == np.int32 and np.array_equal(t, T)


def test_ply_round_trip_through_the_point_cloud_writer(tmp_path, rng):
    from nerf_slam_b200.evaluation import read_ply
    from nerf_slam_b200.point_cloud import PointCloud
    P = rng.normal(0, 3, (1000, 3)).astype(F32)
    C = rng.uniform(0, 1, (1000, 3)).astype(F32)
    for counts in (None, torch.from_numpy(rng.integers(1, 9, 1000).astype(np.int32))):
        PointCloud(torch.from_numpy(P), torch.from_numpy(C), counts).write_ply(str(tmp_path / "c.ply"))
        v, t = read_ply(str(tmp_path / "c.ply"))
        assert np.array_equal(v, P) and t is None


def test_ply_ascii_polygons_and_other_elements(tmp_path):
    """ASCII, double coordinates, an extra element before the faces, a quad (fan-triangulated), `vertex_index`"""
    from nerf_slam_b200.evaluation import read_ply
    txt = """ply
format ascii 1.0
comment hand written
element vertex 5
property double x
property double y
property double z
property uchar red
element camera 1
property float k
element face 2
property list uchar uint vertex_index
end_header
0 0 0 1
1 0 0 2
1 1 0 3
0 1 0 4
0.5 0.5 1.25 5
7.5
4 0 1 2 3
3 0 1 4
"""
    (tmp_path / "a.ply").write_text(txt)
    v, t = read_ply(str(tmp_path / "a.ply"))
    assert np.array_equal(v, np.array([[0, 0, 0], [1, 0, 0], [1, 1, 0], [0, 1, 0], [0.5, 0.5, 1.25]], F32))
    assert np.array_equal(t, np.array([[0, 1, 2], [0, 2, 3], [0, 1, 4]], np.int32))


def test_ply_binary_big_endian_and_mixed_face_sizes(tmp_path):
    from nerf_slam_b200.evaluation import read_ply
    V = np.array([[0, 0, 0], [1, 0, 0], [1, 1, 0], [0, 1, 0]], ">f4")
    head = b"ply\nformat binary_big_endian 1.0\nelement vertex 4\nproperty float x\nproperty float y\nproperty float z\n" \
           b"element face 2\nproperty list uchar int vertex_indices\nend_header\n"
    faces = np.array([3], "u1").tobytes() + np.array([0, 1, 2], ">i4").tobytes() + \
        np.array([4], "u1").tobytes() + np.array([0, 1, 2, 3], ">i4").tobytes()
    (tmp_path / "b.ply").write_bytes(head + V.tobytes() + faces)
    v, t = read_ply(str(tmp_path / "b.ply"))
    assert np.array_equal(v, V.astype(F32))
    assert np.array_equal(t, np.array([[0, 1, 2], [0, 1, 2], [0, 2, 3]], np.int32))


def test_ply_refuses_what_it_cannot_read(tmp_path):
    from nerf_slam_b200.evaluation import read_ply
    (tmp_path / "x.ply").write_bytes(b"not a ply")
    with pytest.raises(ValueError):
        read_ply(str(tmp_path / "x.ply"))
    (tmp_path / "y.ply").write_bytes(b"ply\nformat ascii 1.0\nelement face 0\nproperty list uchar int vertex_indices\n"
                                     b"end_header\n")
    with pytest.raises(ValueError):
        read_ply(str(tmp_path / "y.ply"))


# ----------------------------------------------------------------------------------------------------------- trajectory
def _random_rotation(rng):
    q = rng.normal(size=4)
    q /= np.linalg.norm(q)
    x, y, z, w = q
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                     [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                     [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])


def _poses_with_centres(rng, centres):
    """cam_T_world [N,4,4] with random rotations and the given camera centres"""
    P = np.tile(np.eye(4), (len(centres), 1, 1))
    for i, c in enumerate(centres):
        R = _random_rotation(rng)
        P[i, :3, :3], P[i, :3, 3] = R, -R @ c
    return P


def test_umeyama_recovers_a_known_similarity(rng):
    from nerf_slam_b200.evaluation import umeyama
    src = rng.normal(0, 1, (40, 3))
    R = _random_rotation(rng)
    t = np.array([0.3, -1.2, 2.0])
    for s, with_scale in ((2.7, True), (1.0, False)):
        dst = s * src @ R.T + t
        for fit in (umeyama, orc.umeyama):
            s_, R_, t_ = fit(src, dst, with_scale)
            assert abs(s_ - s) < 1e-10 and np.abs(R_ - R).max() < 1e-10 and np.abs(t_ - t).max() < 1e-9


def test_product_umeyama_agrees_with_the_oracle_on_noisy_data(rng):
    from nerf_slam_b200.evaluation import umeyama
    src = rng.normal(0, 1, (50, 3))
    dst = 0.8 * src @ _random_rotation(rng).T + 0.5 + rng.normal(0, 0.05, (50, 3))
    for with_scale in (True, False):
        a, b = umeyama(src, dst, with_scale), orc.umeyama(src, dst, with_scale)
        assert abs(a[0] - b[0]) < 1e-10 and np.abs(a[1] - b[1]).max() < 1e-10 and np.abs(a[2] - b[2]).max() < 1e-10


@pytest.mark.parametrize("layout", ["tq", "matrix"])
def test_ate_is_zero_on_transformed_copies(rng, layout):
    from nerf_slam_b200.evaluation import trajectory_error
    from nerf_slam_b200.frontend import matrix_to_tq
    c = np.cumsum(rng.normal(0, 0.1, (30, 3)), 0)
    R, t = _random_rotation(rng), np.array([1.0, 2.0, -0.5])
    gt = _poses_with_centres(rng, c)
    sim = _poses_with_centres(rng, 0.4 * c @ R.T + t)
    rigid = _poses_with_centres(rng, c @ R.T + t)
    if layout == "tq":
        gt, sim, rigid = (np.stack([matrix_to_tq(p) for p in P]) for P in (gt, sim, rigid))
    e = trajectory_error(sim, gt, "sim3")
    assert e["rmse"] < 1e-9 and abs(e["scale"] - 2.5) < 1e-9 and e["n"] == 30
    e = trajectory_error(rigid, gt, "se3")
    assert e["rmse"] < 1e-9 and e["scale"] == 1.0
    assert trajectory_error(sim, gt, "se3")["rmse"] > 1e-3        # a scaled copy does not align without scale
    assert trajectory_error(torch.from_numpy(gt), torch.from_numpy(gt), "none")["max"] < 1e-12


def test_ate_by_hand():
    """identity rotations, centres on the x axis, estimates off by 0, 0.3 and 0.4 m in z, no alignment"""
    from nerf_slam_b200.evaluation import trajectory_error
    c = np.array([[0.0, 0, 0], [1, 0, 0], [2, 0, 0]])
    off = np.array([[0.0, 0, 0], [0, 0, 0.3], [0, 0, 0.4]])
    q = np.array([0, 0, 0, 1.0])
    gt = np.concatenate([-c, np.tile(q, (3, 1))], 1)
    est = np.concatenate([-(c + off), np.tile(q, (3, 1))], 1)
    e = trajectory_error(est, gt, "none")
    assert e["rmse"] == pytest.approx(np.sqrt(0.25 / 3), abs=1e-12)
    assert e["mean"] == pytest.approx(0.7 / 3, abs=1e-12)
    assert e["median"] == pytest.approx(0.3, abs=1e-12) and e["max"] == pytest.approx(0.4, abs=1e-12)
    with pytest.raises(ValueError):
        trajectory_error(est, gt, "affine")
    with pytest.raises(ValueError):
        trajectory_error(est[:2], gt, "none")


# ------------------------------------------------------------------------------------------------- ground-truth surface
@pytest.mark.parametrize("ext", [(3.0, 2.0, 3.0), (1.4, 1.0, 1.4), (0.5, 2.25, 1.0)])
def test_surface_mesh_area_and_winding(ext):
    from nerf_slam_b200.synthetic import SyntheticRoom
    V, T = SyntheticRoom(8, 6, 1, half_extent=ext).surface_mesh()
    assert V.dtype == np.float32 and V.shape == (8, 3) and T.dtype == np.int32 and T.shape == (12, 3)
    a, b, c = 2 * np.asarray(ext, F32).astype(np.float64)            # the fp32 corners' box
    x = np.cross(V[T[:, 1]].astype(np.float64) - V[T[:, 0]], V[T[:, 2]].astype(np.float64) - V[T[:, 0]])
    assert np.linalg.norm(x, axis=1).sum() / 2 == pytest.approx(2 * (a * b + b * c + c * a), rel=1e-12)
    centroid = V[T].astype(np.float64).mean(1)
    assert np.all(np.einsum("ij,ij->i", x, -centroid) > 0)            # normals point into the room (free space)
    edges = {}
    for tri in T:
        for i in range(3):
            e = (int(tri[i]), int(tri[(i + 1) % 3]))
            edges[e] = edges.get(e, 0) + 1
    assert all(n == 1 for n in edges.values()) and all((b_, a_) in edges for a_, b_ in edges)   # closed, consistent
    assert np.all(np.abs(np.abs(V) - np.asarray(ext, F32)) == 0)


# --------------------------------------------------------------------------------------------------------------- oracle
def test_oracle_mulhi_and_hash():
    a = np.array([0, 1, 2 ** 63, 2 ** 64 - 1, 0x123456789ABCDEF0], np.uint64)
    for b in (0, 1, 2 ** 40 + 7, 2 ** 64 - 1):
        assert [int(x) for x in orc._mulhi64(a, b)] == [(int(x) * b) >> 64 for x in a]
    h = orc.hash64(5, np.arange(1000), 1)
    assert len(np.unique(h)) == 1000 and np.array_equal(h, orc.hash64(5, np.arange(1000), 1))


def test_oracle_samples_lie_on_their_triangles():
    from nerf_slam_b200.synthetic import SyntheticRoom
    V, T = SyntheticRoom(8, 6, 1).surface_mesh()
    P, tri = orc.surface_samples(V, T, 20000, seed=3)
    ext = np.array([3.0, 2.0, 3.0])
    assert np.all(np.min(np.abs(np.abs(P) - ext), 1) == 0) and np.all(np.abs(P) <= ext)
    counts = np.bincount(tri, minlength=12)
    w, _ = orc.triangle_weights(V, T)
    expected = 20000 * w.astype(np.float64) / w.astype(np.float64).sum()
    assert np.sum((counts - expected) ** 2 / expected) < 40              # chi^2, 11 dof: p < 1e-4 above 35


def test_oracle_zero_area_triangles_are_never_chosen():
    V = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0], [2, 2, 2]], F32)
    T = np.array([[0, 0, 1], [0, 1, 2], [3, 3, 3], [1, 1, 1], [0, 1, 2]], np.int32)
    _, tri = orc.surface_samples(V, T, 5000, seed=1)
    assert set(np.unique(tri)) == {1, 4}


@pytest.mark.parametrize("delta", [0.004, 0.01, 0.03])
def test_oracle_metrics_of_a_face_shifted_along_its_normal(delta):
    """GT: samples of the room's +x wall; reconstruction: the same points moved delta into the room.  Each point's
    nearest neighbour is its partner, so accuracy = completion = delta, and the threshold splits precision / recall"""
    from nerf_slam_b200.synthetic import SyntheticRoom
    V, T = SyntheticRoom(8, 6, 1).surface_mesh()
    wall = T[np.all(V[T][:, :, 0] == 3.0, axis=1)]
    assert len(wall) == 2
    gt, _ = orc.surface_samples(V, wall, 5000, seed=0)
    rec = gt.copy()
    rec[:, 0] = gt[:, 0] - F32(delta)
    d = np.float64(F32(3.0) - F32(F32(3.0) - F32(delta)))              # the shift after fp32 rounding
    m = orc.metrics(rec, gt, threshold=0.02, max_dist=1.0)
    assert m["accuracy"] == pytest.approx(d, abs=1e-9) and m["completion"] == pytest.approx(d, abs=1e-9)
    inside = 1.0 if delta < 0.02 else 0.0
    assert m["precision"] == m["recall"] == m["f_score"] == inside
    assert m["unmatched_reconstruction"] == m["unmatched_ground_truth"] == 0
    far = orc.metrics(rec, gt, threshold=0.02, max_dist=delta / 2)     # every distance clamped: all unmatched
    assert far["accuracy"] == pytest.approx(np.float64(F32(delta / 2)), abs=1e-9)
    assert far["unmatched_reconstruction"] == 5000


def test_oracle_visibility_by_hand():
    """a camera at the origin looking down +z (identity pose), 4 x 3 image, f = 2, c = (1.5, 1)"""
    P = np.array([[0, 0, 1.0], [0, 0, -1.0], [10, 0, 1.0], [0, 0, 5.0], [0.99, 0, 1.0], [1.01, 0, 1.0]], F32)
    pose = np.array([[0, 0, 0, 0, 0, 0, 1]], F32)
    intr = (2.0, 2.0, 1.5, 1.0)
    assert orc.visible(P, pose, intr, 4, 3).tolist() == [True, False, False, True, True, False]
    depth = np.full((1, 3, 4), 2.0, F32)
    depth[0, 1, 1] = 0.0                                               # no measurement at (1, 1): not tested
    got = orc.visible(P, pose, intr, 4, 3, depth, tol=0.05)
    assert got.tolist() == [True, False, False, False, True, False]
    P2 = np.array([[-0.5, 0, 1.0], [0, 0, 5.0]], F32)                    # u = 0.5 -> pixel 1, no depth there: not tested
    assert orc.visible(P2, pose, intr, 4, 3, depth, tol=0.05).tolist() == [True, False]
    assert orc.visible(P, pose, intr, 4, 3, far=2.0).tolist() == [True, False, False, False, True, False]


# -------------------------------------------------------------------------------------------------------- no CUDA, no run
def test_entry_points_fail_loudly_without_cuda():
    if torch.cuda.is_available():
        pytest.skip("CUDA present")
    from nerf_slam_b200 import evaluation as ev
    from nerf_slam_b200.synthetic import SyntheticRoom
    V, T = SyntheticRoom(8, 6, 1).surface_mesh()
    pts = torch.zeros(4, 3)
    calls = [lambda: ev.sample_surface((torch.from_numpy(V), torch.from_numpy(T)), 10),
             lambda: ev.sample_surface((V, T), 10),
             lambda: ev.nearest(pts, pts, 1.0),
             lambda: ev.PointIndex(pts),
             lambda: ev.visible(pts, torch.zeros(1, 7), (1.0, 1.0, 0.0, 0.0), 4, 4),
             lambda: ev.reconstruction_metrics(pts, pts),
             lambda: ev.reconstruction_metrics((V, T), (V, T))]
    for call in calls:
        with pytest.raises(RuntimeError):
            call()


def test_cpu_tensors_are_refused_even_where_cuda_exists(monkeypatch):
    """the CUDA check of every tensor input, independent of whether this machine has a device"""
    from nerf_slam_b200 import _lib
    from nerf_slam_b200 import evaluation as ev
    monkeypatch.setattr(_lib, "load", lambda require_cuda=True: None)
    pts = torch.zeros(4, 3)
    for call in (lambda: ev.nearest(pts, pts), lambda: ev.sample_surface((pts, torch.zeros(1, 3, dtype=torch.int32)), 3),
                 lambda: ev.visible(pts, torch.zeros(1, 7), (1.0, 1.0, 0.0, 0.0), 4, 4)):
        with pytest.raises(RuntimeError, match="CUDA tensor"):
            call()


def test_product_code_never_imports_the_evaluation_oracle():
    pkg = os.path.join(ROOT, "nerf_slam_b200")
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith(".py"):
                assert "recon_eval_oracle" not in open(os.path.join(dirpath, f)).read(), f
