"""The mesh renderer's oracle (tests/mesh_render_oracle.py) on hand-made cases, the PLY colour reader, and MeshScene's
argument checks, without a GPU."""
import numpy as np
import pytest
import torch

from tests import mesh_render_oracle as orc

F32 = np.float32
IDENTITY = np.array([0, 0, 0, 0, 0, 0, 1], F32)
INTR = [4.0, 4.0, 2.0, 2.0]                       # 5 x 5 pixels, pixel (2, 2) on the optical axis


def _one(V, T, u, v, **kw):
    o, d = orc.rays(IDENTITY, INTR, 5, 5, [v * 5 + u])
    depth, tri, normal, color = orc.cast(V, T, o, d, **kw)
    return depth[0], tri[0], normal[0], (None if color is None else color[0])


# a triangle at z = 2 whose edge a-b runs along the row v = 0 and whose vertex a is pixel (0, 0)
TRI_V = np.array([[-1, -1, 2], [1, -1, 2], [0, 1, 2]], F32)
TRI_T = np.array([[0, 1, 2]], np.int32)


@pytest.mark.parametrize("u,v,hit", [(2, 2, True),       # interior
                                     (2, 0, True),       # on the edge a-b
                                     (0, 0, True),       # on the vertex a
                                     (2, 4, True),       # on the vertex c
                                     (1, 4, False),      # beside the vertex c
                                     (0, 2, False)])     # just outside the edge c-a
def test_single_triangle_interior_edge_vertex_and_outside(u, v, hit):
    depth, tri, normal, color = _one(TRI_V, TRI_T, u, v, colors=np.eye(3, dtype=F32))
    if hit:
        assert depth == F32(2) and tri == 0
        assert np.array_equal(normal, np.array([0, 0, 1], F32))
        assert abs(float(color.sum()) - 1) < 1e-6 and color.min() >= 0
    else:
        assert depth == 0 and tri == -1 and not normal.any() and not color.any()


def test_barycentric_colour_at_the_centre():
    _, _, _, color = _one(TRI_V, TRI_T, 2, 2, colors=np.eye(3, dtype=F32))
    assert np.array_equal(color, np.array([0.25, 0.25, 0.5], F32))


def test_backface_culling_keeps_the_side_the_normal_points_to():
    # (b - a) x (c - a) = +z points away from the camera: a back face
    assert _one(TRI_V, TRI_T, 2, 2, cull=True)[1] == -1
    assert _one(TRI_V, TRI_T, 2, 2, cull=False)[1] == 0
    flipped = TRI_T[:, ::-1].copy()
    assert _one(TRI_V, flipped, 2, 2, cull=True)[1] == 0


def test_near_and_far_bound_the_hit():
    assert _one(TRI_V, TRI_T, 2, 2, near=1.9)[1] == 0
    assert _one(TRI_V, TRI_T, 2, 2, near=2.0)[1] == -1            # near < t
    assert _one(TRI_V, TRI_T, 2, 2, far=2.0)[1] == 0              # t <= far
    assert _one(TRI_V, TRI_T, 2, 2, far=1.99)[1] == -1


def test_coincident_triangles_tie_to_the_smaller_index_and_the_nearer_wins():
    V = np.concatenate([TRI_V, TRI_V, TRI_V + np.array([0, 0, -0.5], F32)])
    T = np.array([[3, 4, 5], [0, 1, 2], [6, 7, 8]], np.int32)     # 0 and 1 coincide at z = 2; 2 is nearer
    assert _one(V, T[:2], 2, 2)[1] == 0
    assert _one(V, T[[1, 0]], 2, 2)[1] == 0
    d, t, _, _ = _one(V, T, 2, 2)
    assert t == 2 and d == F32(1.5)


def test_shared_edge_is_watertight():
    # a square of two triangles split along its diagonal; rays through the diagonal hit exactly one depth
    V = np.array([[-1, -1, 2], [1, -1, 2], [1, 1, 2], [-1, 1, 2]], F32)
    T = np.array([[0, 1, 2], [0, 2, 3]], np.int32)
    o, d = orc.rays(IDENTITY, INTR, 5, 5)                              # pixels at x, y = -1, -0.5, 0, 0.5, 1 on the square
    depth, tri, _, _ = orc.cast(V, T, o, d)
    assert np.all(tri >= 0) and np.all(depth == F32(2))
    diagonal = np.arange(5) * 6                                        # u = v: on the shared edge
    assert np.all(tri[diagonal] == 0)                                  # both hit at the same t: the smaller index


def test_degenerate_triangles_never_hit():
    V = np.array([[-1, -1, 2], [1, 1, 2], [0, 0, 2], [0, 0, 2]], F32)
    T = np.array([[0, 1, 2], [2, 3, 3]], np.int32)                   # collinear, and a point
    o, d = orc.rays(IDENTITY, INTR, 5, 5)
    assert np.all(orc.cast(V, T, o, d)[1] == -1)


def test_oracle_agrees_with_itself_in_chunks_and_on_torch():
    rng = np.random.default_rng(0)
    V = rng.normal(0, 1, (300, 3)).astype(F32) + np.array([0, 0, 4], F32)
    T = rng.integers(0, 300, (100, 3)).astype(np.int32)
    C = rng.uniform(0, 1, (300, 3)).astype(F32)
    o, d = orc.rays(IDENTITY, [8.0, 8.0, 8.0, 6.0], 16, 12)
    a = orc.cast(V, T, o, d, colors=C)
    b = orc.cast(V, T, o, d, colors=C, chunk=1000)
    c = orc.cast(V, T, o, d, colors=C, xp="torch")
    assert (a[1] >= 0).sum() > 20
    for x, y, z in zip(a, b, c):
        assert np.array_equal(x, y) and np.array_equal(x, z)


# ----------------------------------------------------------------------------------------------------------------- PLY
def test_read_ply_colours_round_trip_tsdf_mesh_write_ply(tmp_path):
    from nerf_slam_b200.evaluation import read_ply
    from nerf_slam_b200.tsdf_fusion import TsdfMesh
    rng = np.random.default_rng(1)
    V, C, N = (torch.from_numpy(rng.uniform(0, 1, (7, 3)).astype(F32)) for _ in range(3))
    T = torch.from_numpy(rng.integers(0, 7, (5, 3)).astype(np.int32))
    TsdfMesh(V, T, C, N).write_ply(str(tmp_path / "m.ply"))
    v, t, c = read_ply(str(tmp_path / "m.ply"), return_colors=True)
    assert np.array_equal(v, V.numpy()) and np.array_equal(t, T.numpy()) and np.array_equal(c, C.numpy())
    v2, t2 = read_ply(str(tmp_path / "m.ply"))                         # the default return is unchanged
    assert np.array_equal(v2, v) and np.array_equal(t2, t)


def test_read_ply_ascii_uchar_colours(tmp_path):
    from nerf_slam_b200.evaluation import read_ply
    p = tmp_path / "c.ply"
    p.write_text("ply\nformat ascii 1.0\nelement vertex 3\nproperty float x\nproperty float y\nproperty float z\n"
                 "property uchar red\nproperty uchar green\nproperty uchar blue\nelement face 1\n"
                 "property list uchar int vertex_indices\nend_header\n"
                 "0 0 0 255 0 0\n1 0 0 0 128 0\n0 1 0 0 0 51\n3 0 1 2\n")
    v, t, c = read_ply(str(p), return_colors=True)
    assert np.array_equal(t, [[0, 1, 2]])
    assert np.array_equal(c, np.array([[1, 0, 0], [0, 128 / 255, 0], [0, 0, 0.2]], F32))
    q = tmp_path / "n.ply"
    q.write_text("ply\nformat ascii 1.0\nelement vertex 1\nproperty float x\nproperty float y\nproperty float z\n"
                 "end_header\n0 0 0\n")
    assert read_ply(str(q), return_colors=True)[2] is None


# --------------------------------------------------------------------------------------------------------- MeshScene
def test_mesh_scene_refuses_cpu_tensors_and_bad_shapes():
    from nerf_slam_b200.mesh_render import MeshScene
    with pytest.raises(RuntimeError, match="CUDA tensor"):
        MeshScene((torch.zeros(3, 3), torch.zeros(1, 3, dtype=torch.int32)))
    with pytest.raises(ValueError, match=r"vertices must be \[N,3\]"):
        MeshScene((np.zeros((3, 2), F32), np.zeros((1, 3), np.int32)))
    with pytest.raises(ValueError, match=r"triangles must be \[N,3\]"):
        MeshScene((np.zeros((3, 3), F32), np.zeros(3, np.int32)))
    scene = MeshScene.__new__(MeshScene)                  # render's checks come before any device work too
    with pytest.raises(ValueError, match=r"cam_T_world must be \[N,7\]"):
        scene.render(np.zeros((2, 4, 4), F32), INTR, 5, 5)
    with pytest.raises(RuntimeError, match="CUDA tensor"):
        scene.render(torch.zeros(2, 7), INTR, 5, 5)
