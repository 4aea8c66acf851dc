"""The mesh operations' oracle (tests/mesh_ops_oracle.py) on hand-made meshes, the refusals, and the argument checks of
tools/clean_mesh.py and tools/eval_reconstruction.py, without a GPU."""
import os
import sys

import numpy as np
import pytest

from tests import mesh_ops_oracle as orc

F32 = np.float32
TOOLS = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools")


def test_two_triangles_sharing_one_vertex_form_one_component():
    V = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0], [-1, 0, 0], [0, -1, 0]], F32)
    T = np.array([[0, 1, 2], [0, 3, 4]], np.int32)
    labels, counts, area = orc.connected_components(V, T)
    assert labels.tolist() == [0, 0] and counts.tolist() == [2] and area.tolist() == [1.0]


def test_coincident_but_distinct_vertices_form_two_components():
    V = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0], [0, 0, 0], [-1, 0, 0], [0, -1, 0]], F32)
    T = np.array([[0, 1, 2], [3, 4, 5]], np.int32)
    labels, counts, area = orc.connected_components(V, T)
    assert labels.tolist() == [0, 1] and counts.tolist() == [1, 1] and area.tolist() == [0.5, 0.5]


def test_components_are_numbered_by_their_lowest_triangle():
    V = np.zeros((9, 3), F32)
    V[:, 0] = np.arange(9)
    V[:, 1] = np.arange(9) % 2
    T = np.array([[6, 7, 8], [0, 1, 2], [8, 7, 6], [2, 1, 0], [3, 4, 5]], np.int32)
    labels, counts, _ = orc.connected_components(V, T)
    assert labels.tolist() == [0, 1, 0, 1, 2] and counts.tolist() == [2, 2, 1]


def test_degenerate_triangle_with_a_repeated_index():
    V = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0], [5, 5, 5], [6, 5, 5]], F32)
    T = np.array([[0, 1, 2], [3, 3, 4], [4, 3, 3]], np.int32)
    labels, counts, area = orc.connected_components(V, T)
    assert labels.tolist() == [0, 1, 1] and counts.tolist() == [1, 2] and area.tolist() == [0.5, 0.0]
    N = orc.vertex_normals(V, T)
    assert np.array_equal(N[:3], np.tile(np.array([0, 0, 1], F32), (3, 1))) and not N[3:].any()
    assert orc.remove_small_components(V, T, 1e-3)[1].tolist() == [[0, 1, 2]]


def test_submesh_drops_isolated_vertices_and_keeps_order():
    V = np.arange(24, dtype=F32).reshape(8, 3)
    T = np.array([[1, 3, 5], [2, 6, 7], [7, 5, 1]], np.int32)
    C = V / 100
    Nn = -V
    Vo, To, Co, No = orc.submesh(V, T, [True, False, True], C, Nn)
    assert np.array_equal(Vo, V[[1, 3, 5, 7]]) and To.tolist() == [[0, 1, 2], [3, 2, 0]]
    assert np.array_equal(Co, C[[1, 3, 5, 7]]) and np.array_equal(No, Nn[[1, 3, 5, 7]])
    assert orc.submesh(V, T, [False] * 3) is None
    Vo, To, Co, No = orc.submesh(V, T, [True, True, True])          # a pair: colours 0, normals of the output
    assert len(Vo) == 6 and not Co.any() and np.array_equal(No, orc.vertex_normals(Vo, To))


def test_a_triangle_with_one_seen_vertex_survives_cull():
    pose = np.array([[0, 0, 0, 0, 0, 0, 1]], F32)                   # identity: looking along +z
    V = np.array([[0, 0, 2], [100, 0, 2], [0, 100, 2], [100, 100, 2], [-100, 0, 2], [0, 0, -2]], F32)
    T = np.array([[0, 1, 2], [1, 3, 2], [4, 5, 1]], np.int32)
    out = orc.cull(V, T, pose, [4.0, 4.0, 2.0, 2.0], 5, 5)
    assert out[1].tolist() == [[0, 1, 2]]
    depth = np.full((1, 5, 5), 1.0, F32)                            # a wall in front of vertex 0: occluded
    assert orc.cull(V, T, pose, [4.0, 4.0, 2.0, 2.0], 5, 5, depths=depth) is None


def test_vertex_normals_sum_area_weighted_face_normals():
    V = np.array([[0, 0, 0], [2, 0, 0], [0, 2, 0], [0, 0, 1]], F32)
    T = np.array([[0, 1, 2], [0, 3, 1]], np.int32)                  # (b - a) x (c - a) = (0, 0, 4) and (0, 2, 0)
    N = orc.vertex_normals(V, T)
    s = np.array([0.0, 2.0, 4.0])
    assert np.array_equal(N[0], (s / np.sqrt(20.0)).astype(F32)) and np.array_equal(N[1], N[0])
    assert np.array_equal(N[2], np.array([0, 0, 1], F32)) and np.array_equal(N[3], np.array([0, 1, 0], F32))


def _grid(n, s):
    i, j = np.meshgrid(np.arange(n + 1), np.arange(n + 1), indexing="xy")
    V = np.stack([(i + 0.5) * s, (j + 0.5) * s, np.full(i.shape, 0.5 * s)], -1).reshape(-1, 3).astype(F32)
    q = (np.arange(n)[:, None] * (n + 1) + np.arange(n)[None, :]).reshape(-1)
    T = np.concatenate([np.stack([q, q + 1, q + n + 2], 1), np.stack([q, q + n + 2, q + n + 1], 1)]).astype(np.int32)
    return V, T


def test_clustering_a_regular_grid_at_twice_its_spacing():
    """9 x 9 vertices at (i + 0.5) s: cells floor((i + 0.5) / 2) = 0 0 1 1 2 2 3 3 4, so 5 x 5 cells; only the quads
    that straddle a cell boundary in x and in y keep both triangles: 4 x 4 coarse quads, 32 triangles"""
    V, T = _grid(8, 0.25)
    Vo, To, Co, No = orc.simplify_vertex_clustering(V, T, 0.5)
    assert len(Vo) == 25 and len(To) == 32 and not Co.any()
    assert np.array_equal(Vo[0], np.array([0.25, 0.25, 0.125], F32))          # mean of (0.125, 0.375)^2
    assert np.array_equal(Vo[-1], np.array([2.125, 2.125, 0.125], F32))       # the last row / column alone
    assert np.all(No[:, 2] == 1) and np.all(No[:, :2] == 0)


def test_duplicate_cell_triples_are_removed_and_the_winding_kept():
    V = np.array([[0.1, 0.1, 0], [1.1, 0.1, 0], [0.1, 1.1, 0], [0.2, 0.2, 0], [0.3, 1.3, 0], [5, 5, 5]], F32)
    T = np.array([[3, 2, 1],      # cells (0, 2, 1): the lowest index of the triple, wound clockwise
                  [0, 1, 2],      # the same cells
                  [1, 4, 3],      # the same cells again
                  [0, 3, 1]],     # two corners in cell 0: dropped
                 np.int32)
    Vo, To, Co, No = orc.simplify_vertex_clustering(V, T, 1.0, colors=np.arange(18, dtype=F32).reshape(6, 3))
    assert To.tolist() == [[0, 2, 1]]
    mean = ((np.float64(F32(0.1)) + np.float64(F32(0.2))) / 2).astype(F32)  # vertices 0 and 3 share cell 0
    assert np.array_equal(Vo[0], np.array([mean, mean, 0], F32))
    assert np.array_equal(Co[0], np.array([4.5, 5.5, 6.5], F32))
    assert np.array_equal(No, np.tile(np.array([0, 0, -1], F32), (3, 1)))


def test_refusals():
    V = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0]], F32)
    for T in ([[0, 1, 3]], [[0, -1, 2]]):
        for fn in (orc.connected_components, orc.vertex_normals):
            with pytest.raises(ValueError, match="outside"):
                fn(V, T)
        with pytest.raises(ValueError, match="outside"):
            orc.simplify_vertex_clustering(V, T, 0.1)
    bad = V.copy()
    bad[2, 1] = np.nan
    for fn in (orc.connected_components, orc.vertex_normals, lambda v, t: orc.simplify_vertex_clustering(v, t, 0.1)):
        with pytest.raises(ValueError, match="non-finite"):
            fn(bad, [[0, 1, 2]])
    pose = np.array([[0, 0, 0, 0, 0, 0, 1]], F32)
    with pytest.raises(ValueError, match="non-finite"):
        orc.cull(bad, [[0, 1, 2]], pose, [4.0, 4.0, 2.0, 2.0], 5, 5)
    with pytest.raises(ValueError, match="outside"):
        orc.cull(V, [[0, 1, 3]], pose, [4.0, 4.0, 2.0, 2.0], 5, 5)
    Vu = np.concatenate([V, [[np.inf, 0, 0]]]).astype(F32)                     # unreferenced: ignored
    assert orc.simplify_vertex_clustering(Vu, [[0, 1, 2]], 0.5) is not None
    from nerf_slam_b200 import mesh_ops
    for voxel in (0.0, -1.0, np.nan, np.inf, 1e-50, 1e39):
        with pytest.raises(ValueError, match="voxel_size"):
            orc.simplify_vertex_clustering(V, [[0, 1, 2]], voxel)
        with pytest.raises(ValueError, match="voxel_size"):
            mesh_ops.simplify_vertex_clustering((V, np.array([[0, 1, 2]], np.int32)), voxel)


def test_cpu_tensors_are_refused():
    import torch
    from nerf_slam_b200 import mesh_ops
    V, T = torch.zeros(3, 3), torch.tensor([[0, 1, 2]], dtype=torch.int32)
    for fn in (mesh_ops.connected_components, mesh_ops.vertex_normals, lambda m: mesh_ops.submesh(m, [True]),
               lambda m: mesh_ops.simplify_vertex_clustering(m, 0.1)):
        with pytest.raises(RuntimeError, match="CUDA"):
            fn((V, T))


def _tool(name):
    sys.path.insert(0, TOOLS)
    try:
        return __import__(name)
    finally:
        sys.path.remove(TOOLS)


@pytest.mark.parametrize("argv", [["a.ply", "b.ply", "--voxel", "0"], ["a.ply", "b.ply", "--voxel", "-0.1"],
                                  ["a.ply", "b.ply", "--voxel", "nan"], ["a.ply", "b.ply", "--min_component_area", "-1"],
                                  ["a.ply", "b.ply", "--min_component_area", "inf"], ["a.ply"]])
def test_clean_mesh_argument_checks(argv):
    with pytest.raises(SystemExit):
        _tool("clean_mesh").parse_args(argv)


def test_clean_mesh_accepts_its_flags():
    a = _tool("clean_mesh").parse_args(["a.ply", "b.ply", "--views", "t.json", "--min_component_area", "0.01",
                                        "--voxel", "0.02"])
    assert (a.views, a.min_component_area, a.voxel) == ("t.json", 0.01, 0.02)


@pytest.mark.parametrize("argv", [["r.ply", "g.ply", "--cull"], ["r.ply", "g.ply", "--min_component_area", "-1"],
                                  ["r.ply", "g.ply", "--views", "t.json", "--cull", "--min_component_area", "nan"]])
def test_eval_reconstruction_argument_checks(argv):
    with pytest.raises(SystemExit):
        _tool("eval_reconstruction").main(argv)
