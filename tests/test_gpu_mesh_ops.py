"""The mesh operations on the GPU (csrc/mesh_ops.cu through nerf_slam_b200/mesh_ops.py) against the numpy restatement
(tests/mesh_ops_oracle.py) bit for bit, their determinism, cleaning that gives back the original mesh, cleaning the
trained NeRF room, and their peak memory at 512^3."""
import types

import numpy as np
import pytest
import torch

from tests import mesh_ops_oracle as orc

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
F32 = np.float32


def _t(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def _np(x):
    return x.cpu().numpy()


def _look_at(eye, target):
    """cam_T_world [7] (t, q_xyzw) of a camera at eye looking at target, y down"""
    from nerf_slam_b200.frontend import matrix_to_tq
    eye, target = np.asarray(eye, np.float64), np.asarray(target, np.float64)
    fwd = (target - eye) / np.linalg.norm(target - eye)
    right = np.cross(fwd, [0.0, -1.0, 0.0])
    right /= np.linalg.norm(right)
    down = np.cross(fwd, right)
    c2w = np.eye(4)
    c2w[:3, 0], c2w[:3, 1], c2w[:3, 2], c2w[:3, 3] = right, down, fwd, eye
    return matrix_to_tq(np.linalg.inv(c2w)).astype(F32)


# ------------------------------------------------------------------------------------------------------------- inputs
def _soup():
    """triangles inside 300 groups of 8 vertices, 400 triangles across the first 150 groups, degenerate triangles
    (repeated and collinear vertices) and 500 vertices no triangle references; a (vertices, triangles) pair"""
    rng = np.random.default_rng(0)
    V = rng.normal(0, 1, (2900, 3)).astype(F32)
    g = rng.integers(0, 300, 3000)
    T = (8 * g[:, None] + rng.integers(0, 8, (3000, 3))).astype(np.int32)
    cross = rng.integers(0, 1200, (400, 3)).astype(np.int32)
    T = np.concatenate([T, cross])
    T[::53, 2] = T[::53, 0]
    V[2401:2410] = V[2400] + np.arange(1, 10, dtype=F32)[:, None] * F32(0.5)   # collinear
    T = np.concatenate([T, [[2400, 2401, 2402], [2403, 2400, 2409]]]).astype(np.int32)
    return V, T


def _icosphere(n_sub):
    t = (1 + 5 ** 0.5) / 2
    Vs = [(-1, t, 0), (1, t, 0), (-1, -t, 0), (1, -t, 0), (0, -1, t), (0, 1, t), (0, -1, -t), (0, 1, -t), (t, 0, -1),
          (t, 0, 1), (-t, 0, -1), (-t, 0, 1)]
    Fs = [(0, 11, 5), (0, 5, 1), (0, 1, 7), (0, 7, 10), (0, 10, 11), (1, 5, 9), (5, 11, 4), (11, 10, 2), (10, 7, 6),
          (7, 1, 8), (3, 9, 4), (3, 4, 2), (3, 2, 6), (3, 6, 8), (3, 8, 9), (4, 9, 5), (2, 4, 11), (6, 2, 10), (8, 6, 7),
          (9, 8, 1)]
    Vs = [np.asarray(v, np.float64) / np.linalg.norm(v) for v in Vs]
    for _ in range(n_sub):
        mid, F2 = {}, []

        def m(a, b):
            key = (min(a, b), max(a, b))
            if key not in mid:
                p = Vs[a] + Vs[b]
                Vs.append(p / np.linalg.norm(p))
                mid[key] = len(Vs) - 1
            return mid[key]
        for a, b, c in Fs:
            ab, bc, ca = m(a, b), m(b, c), m(c, a)
            F2 += [(a, ab, ca), (b, bc, ab), (c, ca, bc), (ab, bc, ca)]
        Fs = F2
    return np.asarray(Vs), np.asarray(Fs, np.int64)


def _torus(R, r, nu, nv):
    u, v = np.meshgrid(np.arange(nu) * 2 * np.pi / nu, np.arange(nv) * 2 * np.pi / nv, indexing="ij")
    V = np.stack([(R + r * np.cos(v)) * np.cos(u), (R + r * np.cos(v)) * np.sin(u), r * np.sin(v)], -1).reshape(-1, 3)
    i, j = np.meshgrid(np.arange(nu), np.arange(nv), indexing="ij")
    a, b = i * nv + j, ((i + 1) % nu) * nv + j
    c, d = ((i + 1) % nu) * nv + (j + 1) % nv, i * nv + (j + 1) % nv
    F = np.concatenate([np.stack([a, b, c], -1).reshape(-1, 3), np.stack([a, c, d], -1).reshape(-1, 3)])
    return V, F


def _octahedron(centre, r):
    V = np.asarray(centre, np.float64) + r * np.array([[1, 0, 0], [-1, 0, 0], [0, 1, 0], [0, -1, 0], [0, 0, 1], [0, 0, -1]])
    F = np.array([[0, 2, 4], [2, 1, 4], [1, 3, 4], [3, 0, 4], [2, 0, 5], [1, 2, 5], [3, 1, 5], [0, 3, 5]])
    return V, F


def _join(parts):
    Vs, Fs, off = [], [], 0
    for V, F in parts:
        Vs.append(V)
        Fs.append(F + off)
        off += len(V)
    return np.concatenate(Vs).astype(F32), np.concatenate(Fs).astype(np.int32)


def _shapes():
    """a sphere, a torus and 40 scattered octahedra of random size in one mesh, with colours (a TsdfMesh)"""
    from nerf_slam_b200.tsdf_fusion import TsdfMesh
    rng = np.random.default_rng(1)
    sV, sF = _icosphere(4)
    tV, tF = _torus(1.0, 0.3, 48, 24)
    blobs = [_octahedron(rng.uniform(-3, 3, 3), rng.uniform(0.005, 0.2)) for _ in range(40)]
    V, T = _join([(sV * 0.8 + [2.5, 0, 0], sF), (tV, tF)] + blobs)
    C = rng.uniform(0, 1, V.shape).astype(F32)
    N = rng.normal(0, 1, V.shape).astype(F32)
    return TsdfMesh(_t(V), _t(T), _t(C), _t(N))


def _nerf_mesh48():
    from nerf_slam_b200 import pyngp
    from nerf_slam_b200.pyngp import mesh_lattice
    tb = pyngp.Testbed(seed=4, max_samples=1 << 16, max_rays=1 << 13)
    tb.create_empty_nerf_dataset(8, 1.0, None, 4, None)
    g = torch.Generator().manual_seed(4)
    tb.grid_master.copy_(((torch.rand(tb.grid_master.shape, generator=g) * 2 - 1) * 0.5).to(DEV))
    tb.grid_half.copy_(tb.grid_master.half())
    tb.pack_weights()
    tb.density.copy_(torch.where(torch.rand(tb.density.shape, generator=g) < 0.7, 0.0, -1.0).to(DEV))
    lo, h, dims = mesh_lattice(48, None, tb.aabb_scale)
    field, weight = tb.mesh_kernels.lattice(tb, lo, h, dims, 0.0)
    mesh = tb.marching_cubes(48, None, float(torch.quantile(-field[weight > 0], 0.5)))
    assert mesh is not None
    return mesh


def _room(n_views=10, frames=40):
    from nerf_slam_b200.frontend import matrix_to_tq
    from nerf_slam_b200.synthetic import SyntheticRoom
    room = SyntheticRoom(640, 480, frames, seed=0)
    ks = list(range(0, frames, frames // n_views))[:n_views]
    poses = np.asarray([matrix_to_tq(np.asarray(room.render(k)[2], np.float64)) for k in ks], F32)
    return room, ks, poses, room.calib.camera_model.numpy().astype(F32)


@pytest.fixture(scope="module")
def tsdf_room():
    """the dense 512^3 TSDF mesh of the synthetic room fused from 10 of its views, with the views"""
    from nerf_slam_b200.tsdf_fusion import TsdfFusion
    room, ks, poses, intr = _room()
    depths = np.stack([room.render(k)[1][..., 0].astype(F32) * F32(room.calib.depth_scale) for k in ks])
    images = np.stack([room.render(k)[0][..., :3].transpose(2, 0, 1) for k in ks])
    fus = TsdfFusion("tsdf", types.SimpleNamespace(eval=False, tsdf_volume="dense", tsdf_resolution=512), DEV)
    fus.voxel_size = 8.0 / 512
    fus.initialize()
    fus.build_volume({"cam0_poses": _t(poses), "cam0_idepths_up": _t(1.0 / depths), "cam0_depths_cov_up": None,
                      "cam0_images": _t(images)}, intr, None)
    mesh = fus.build_mesh(0.5)
    del fus
    torch.cuda.empty_cache()
    return room, poses, intr, mesh


def _arrays(mesh):
    if hasattr(mesh, "vertices"):
        return tuple(_np(x) for x in (mesh.vertices, mesh.triangles, mesh.vertex_colors, mesh.vertex_normals))
    return mesh[0], mesh[1], None, None


def _same(got, want):
    if want is None:
        assert got is None
        return
    assert got is not None
    for g, w, name in zip((got.vertices, got.triangles, got.vertex_colors, got.vertex_normals), want,
                          ("vertices", "triangles", "colors", "normals")):
        g = _np(g)
        assert g.shape == w.shape and g.dtype == w.dtype, name
        assert np.array_equal(g, w), (name, np.argwhere(g != w)[:5])


def _views(V):
    """three cameras around the mesh's box, 160 x 120"""
    lo, hi = V.min(0), V.max(0)
    c, e = (lo + hi) / 2, float((hi - lo).max())
    poses = np.stack([_look_at(c + e * np.asarray(d), c) for d in ((0, 0.3, -1.2), (1.1, -0.4, 0.5), (-0.7, 0.2, 0.9))])
    return poses, [100.0, 100.0, 79.5, 59.5], 160, 120


def _check_all(mesh):
    """every operation bit for bit against the oracle"""
    from nerf_slam_b200 import mesh_ops
    from nerf_slam_b200.mesh_render import MeshScene
    V, T, C, N = _arrays(mesh)
    labels, counts, area = mesh_ops.connected_components(mesh)
    ol, oc, oa = orc.connected_components(V, T)
    assert np.array_equal(_np(labels), ol) and np.array_equal(_np(counts), oc) and np.array_equal(_np(area), oa)
    assert area.dtype == torch.float64 and counts.dtype == torch.int64 and labels.dtype == torch.int32
    assert np.array_equal(_np(mesh_ops.vertex_normals(mesh)), orc.vertex_normals(V, T))

    keep = np.random.default_rng(5).random(len(T)) < 0.6
    _same(mesh_ops.submesh(mesh, _t(keep)), orc.submesh(V, T, keep, C, N))
    min_area = float(np.median(oa))
    _same(mesh_ops.remove_small_components(mesh, min_area), orc.remove_small_components(V, T, min_area, C, N))

    poses, intr, W, H = _views(V)
    depth = MeshScene(mesh).render(_t(poses), intr, W, H).depth
    got = mesh_ops.cull(mesh, _t(poses), intr, W, H, depths=depth, depth_tol=0.02)
    want = orc.cull(V, T, poses, intr, W, H, depths=_np(depth), tol=0.02, colors=C, normals=N)
    _same(got, want)
    assert want is not None and 0 < len(want[1]) < len(T)

    ext = float((V.max(0) - V.min(0)).max())
    for voxel in (ext / 40, ext / 7):
        got = mesh_ops.simplify_vertex_clustering(mesh, voxel)
        want = orc.simplify_vertex_clustering(V, T, voxel, C)
        _same(got, want)
        assert len(want[1]) < len(T)
    return len(oc)


def test_random_soup_matches_the_oracle_bit_for_bit():
    V, T = _soup()
    n_comp = _check_all((V, T))
    assert n_comp > 50


def test_sphere_torus_and_blobs_match_the_oracle_bit_for_bit():
    assert _check_all(_shapes()) == 42


def test_nerf_mesh_matches_the_oracle_bit_for_bit():
    _check_all(_nerf_mesh48())


def test_tsdf_room_mesh_matches_the_oracle_bit_for_bit(tsdf_room):
    _check_all(tsdf_room[3])


def test_refusals_on_the_device():
    from nerf_slam_b200 import mesh_ops
    V, T = _soup()
    bad = T.copy()
    bad[17, 1] = len(V)
    poses, intr, W, H = _views(V)
    cull = lambda m: mesh_ops.cull(m, _t(poses), intr, W, H)  # noqa: E731
    for fn in (mesh_ops.connected_components, mesh_ops.vertex_normals, lambda m: mesh_ops.submesh(m, [True] * len(T)),
               lambda m: mesh_ops.simplify_vertex_clustering(m, 0.1), lambda m: mesh_ops.remove_small_components(m, 0),
               cull):
        with pytest.raises(ValueError, match="outside"):
            fn((V, bad))
    Vn = V.copy()
    Vn[T[5, 0], 2] = np.nan
    for fn in (mesh_ops.connected_components, mesh_ops.vertex_normals,
               lambda m: mesh_ops.simplify_vertex_clustering(m, 0.1), cull):
        with pytest.raises(ValueError, match="non-finite"):
            fn((Vn, T))
    Vu = np.concatenate([V, [[np.nan, 0, 0]]]).astype(F32)               # a vertex no triangle uses: not refused
    assert cull((Vu, T)) is not None


def test_repeated_calls_give_identical_bytes(tsdf_room):
    """union-find arrival order, atomics and sorts must not leak into any result"""
    from nerf_slam_b200 import mesh_ops
    mesh = tsdf_room[3]
    runs = []
    for _ in range(3):
        labels, counts, area = mesh_ops.connected_components(mesh)
        s = mesh_ops.simplify_vertex_clustering(mesh, 0.05)
        runs.append([_np(x).tobytes() for x in (labels, counts, area, mesh_ops.vertex_normals(mesh), s.vertices,
                                                 s.triangles, s.vertex_colors, s.vertex_normals)])
    assert runs[0] == runs[1] == runs[2]


def _strips(n_strips=64, length=30_000, seed=3):
    """long triangle strips whose vertex indices are a random permutation: the union phase builds long parent chains"""
    rng = np.random.default_rng(seed)
    n = n_strips * (length + 2)
    perm = rng.permutation(n).astype(np.int32)
    k = np.arange(length)
    base = (np.arange(n_strips) * (length + 2))[:, None]
    T = perm[np.stack([base + k, base + k + 1, base + k + 2], -1).reshape(-1, 3)]
    i = np.arange(n)
    V = np.empty((n, 3), F32)                                           # strip vertex i of strip j at its place
    V[perm] = np.stack([(i % (length + 2)) * 0.01, (i % 2) * 0.01, (i // (length + 2)) * 0.1], 1)
    return V, np.ascontiguousarray(T[rng.permutation(len(T))])


def test_components_of_long_shuffled_strips_match_the_oracle_on_every_call():
    """64 strips of 30 000 triangles over permuted vertex indices, in shuffled triangle order: every find walks long
    parent chains while other threads hook and halve them.  Every vertex must end at its root, so three calls all give
    the oracle's labels, counts and areas"""
    from nerf_slam_b200 import mesh_ops
    V, T = _strips()
    ol, oc, oa = orc.connected_components(V, T)
    assert len(oc) == 64
    mesh = (_t(V), _t(T))
    for _ in range(3):
        labels, counts, area = mesh_ops.connected_components(mesh)
        assert np.array_equal(_np(labels), ol) and np.array_equal(_np(counts), oc) and np.array_equal(_np(area), oa)


def test_centimetre_floaters_are_removed_and_the_room_survives(tsdf_room):
    """floaters of a NeRF-like size (octahedra of radius 2 to 5 cm, 2.8e-3 to 1.7e-2 m^2) in the room's TSDF mesh:
    removing components under 0.05 m^2 drops every floater triangle and gives exactly what it gives on the mesh
    without them; the room's own slivers under that size go too, but they hold under 0.1 % of its triangles"""
    from nerf_slam_b200 import mesh_ops
    from nerf_slam_b200.tsdf_fusion import TsdfMesh
    room, poses, intr, mesh = tsdf_room
    V, T, C, N = _arrays(mesh)
    ext = np.asarray(room.ext, np.float64)
    rng = np.random.default_rng(8)
    xV, xF = _join([_octahedron(rng.uniform(-0.6, 0.6, 3) * ext, rng.uniform(0.02, 0.05)) for _ in range(30)])
    dirty = TsdfMesh(_t(np.concatenate([V, xV])), _t(np.concatenate([T, xF + len(V)]).astype(np.int32)),
                     _t(np.concatenate([C, np.full((len(xV), 3), 0.5, F32)])),
                     _t(np.concatenate([N, np.zeros((len(xV), 3), F32)])))
    _, _, area = mesh_ops.connected_components(dirty)
    assert int((area < 0.05).sum()) >= 30 and float(area.max()) > 30.0       # the floaters, and the room in one piece
    clean = mesh_ops.remove_small_components(dirty, 0.05)
    want = mesh_ops.remove_small_components(mesh, 0.05)
    _same(clean, _arrays(want))
    assert want.triangles.shape[0] > 0.999 * len(T)


def test_cleaning_floaters_and_a_hidden_box_gives_back_the_original_mesh(tsdf_room):
    """the room's TSDF mesh with small closed floaters in the room and a closed shape hidden 0.2 m and more behind the +x
    wall appended: culling with the room's depth and removing small components returns the original mesh bit for bit,
    and the metrics against the room's surface are the original's.  The TSDF mesh has slivers of its own (first H100
    run: 50 components, the smallest 3.0e-9 m^2), so to give back every original triangle the floaters here are
    octahedra of radius 10 um (6.9e-10 m^2); test_centimetre_floaters_are_removed_and_the_room_survives covers floaters
    of a realistic size."""
    from nerf_slam_b200 import mesh_ops
    from nerf_slam_b200.evaluation import reconstruction_metrics
    from nerf_slam_b200.mesh_render import MeshScene
    from nerf_slam_b200.tsdf_fusion import TsdfMesh
    room, poses, intr, mesh = tsdf_room
    V, T, C, N = _arrays(mesh)
    ext = np.asarray(room.ext, np.float64)
    rng = np.random.default_rng(7)
    r = 1e-5
    floaters = [_octahedron(rng.uniform(-0.6, 0.6, 3) * ext, r) for _ in range(20)]
    bV, bF = _torus(0.2, 0.1, 16, 8)                                    # a closed "box" far behind the wall
    box = (bV + [ext[0] + 0.5, 0.0, 0.0], bF)
    xV, xF = _join(floaters + [box])
    V2 = np.concatenate([V, xV]).astype(F32)
    T2 = np.concatenate([T, xF + len(V)]).astype(np.int32)
    extra = len(xV)
    C2 = np.concatenate([C, np.full((extra, 3), 0.5, F32)])
    N2 = np.concatenate([N, np.zeros((extra, 3), F32)])
    dirty = TsdfMesh(_t(V2), _t(T2), _t(C2), _t(N2))

    _, _, area = mesh_ops.connected_components(mesh)
    floater_area = float(mesh_ops.connected_components(_octahedron((0, 0, 0), r))[2][0])
    min_area = 2 * floater_area
    print(f"room mesh: {len(V)} vertices, {len(T)} triangles, {area.shape[0]} components, smallest "
          f"{float(area.min()):.3e} m^2; floater {floater_area:.3e} m^2")
    assert float(area.min()) >= min_area
    depth = MeshScene(room.surface_mesh()).render(_t(poses), intr, room.W, room.H).depth
    culled = mesh_ops.cull(dirty, _t(poses), intr, room.W, room.H, depths=depth, depth_tol=0.1)
    print(f"culled: {culled.triangles.shape[0]} of {len(T2)} triangles kept ({len(T)} original)")
    clean = mesh_ops.remove_small_components(culled, min_area)
    _same(clean, (V, T, C, N))
    gt = room.surface_mesh()
    assert reconstruction_metrics(clean, gt) == reconstruction_metrics(mesh, gt)


# ------------------------------------------------------------------------------------------------------- trained room
ROOM_RES, ROOM_THRESH, ROOM_EXT = 256, 10.0, (1.4, 1.0, 1.4)


@pytest.fixture(scope="module")
def nerf_room():
    """the room of test_gpu_nerf_mesh.py's trained-room fixture: 12 views, 300 tensor-core steps, metric poses"""
    from nerf_slam_b200.nerf_fusion import NerfFusion
    from nerf_slam_b200.synthetic import SyntheticRoom
    room = SyntheticRoom(160, 120, 12, seed=0, half_extent=ROOM_EXT, orbit_radius=0.3, step=0.25)
    nf = NerfFusion("nerf", types.SimpleNamespace(buffer=12, eval=False, mask_type="ours"), DEV)
    nf.ngp.nerf.training.depth_supervision_lambda = 1.0
    nf.gt_fit_convention = "metric"
    pk = [room.packet(k) for k in range(12)]
    nf.fuse({"data": {"k": np.arange(12), "poses": np.stack([p["poses"][0] for p in pk]),
                      "images": np.stack([p["images"][0] for p in pk]), "depths": np.stack([p["depths"][0] for p in pk]),
                      "calibs": pk[0]["calibs"]}})
    for _ in range(300):
        nf.fit_volume_once()
    torch.cuda.synchronize()
    return room, nf


def _near_walls(V):
    return float((np.min(np.abs(np.abs(V) - np.asarray(ROOM_EXT)), axis=1) < 0.10).mean())


def test_cleaning_the_trained_room_removes_floaters(nerf_room):
    """culling the 256^3 mesh to the 12 training views (occlusion from its own rendered depth) and removing components
    under 0.05 m^2 raises the share of vertices within 10 cm of a wall and lowers the accuracy against the room's
    surface.  First H100 run: 424 502 -> 166 213 vertices, within 10 cm of a wall 62.2 % -> 97.7 %, accuracy 17.7 ->
    2.5 cm, completion 35.6 -> 35.7 cm.  Asserted: strictly better share and accuracy (no absolute threshold yet)."""
    from nerf_slam_b200 import mesh_ops
    from nerf_slam_b200.evaluation import reconstruction_metrics
    from nerf_slam_b200.frontend import matrix_to_tq
    from nerf_slam_b200.mesh_render import MeshScene
    room, nf = nerf_room
    mesh = nf.build_mesh(resolution=ROOM_RES, thresh=ROOM_THRESH)
    poses = _t(np.asarray([matrix_to_tq(np.asarray(room.render(k)[2], np.float64)) for k in range(12)], F32))
    intr = room.calib.camera_model.numpy().astype(F32)
    depth = MeshScene(mesh).render(poses, intr, room.W, room.H).depth
    clean = mesh_ops.remove_small_components(mesh_ops.cull(mesh, poses, intr, room.W, room.H, depths=depth), 0.05)
    gt = room.surface_mesh()
    before, after = reconstruction_metrics(mesh, gt), reconstruction_metrics(clean, gt)
    near0, near1 = _near_walls(_np(mesh.vertices)), _near_walls(_np(clean.vertices))
    print(f"trained room: {mesh.vertices.shape[0]} -> {clean.vertices.shape[0]} vertices, within 10 cm of a wall "
          f"{near0:.4f} -> {near1:.4f}, accuracy {before['accuracy']:.4f} -> {after['accuracy']:.4f} m, completion "
          f"{before['completion']:.4f} -> {after['completion']:.4f} m")
    assert near1 > near0 and after["accuracy"] < before["accuracy"]


def test_memory_at_512(nerf_room):
    """peak device memory of each operation on the 512^3 room NeRF mesh is at most its allocations: the scratch its size
    query reports, its outputs and its temporaries (listed per operation below), plus a 1 MiB margin for allocator
    rounding and the host reads"""
    from nerf_slam_b200 import _lib, mesh_ops
    from nerf_slam_b200.frontend import matrix_to_tq
    room, nf = nerf_room
    mesh = nf.ngp.marching_cubes(512, None, ROOM_THRESH)
    nv, nt = int(mesh.vertices.shape[0]), int(mesh.triangles.shape[0])
    q = lambda name: _lib.query_size(name, nv, nt)  # noqa: E731
    keep = torch.ones(nt, dtype=torch.bool, device=DEV)
    poses = _t(np.asarray([matrix_to_tq(np.asarray(room.render(k)[2], np.float64)) for k in range(12)], F32))
    intr = room.calib.camera_model.numpy().astype(F32)
    out_mesh = 36 * nv + 12 * nt                                     # an output no larger than the input
    cc = q("nslam_mesh_components_scratch") + 20 * nt + 24 * nt      # labels, counts, fixed areas; their [C] copies
    sub = q("nslam_mesh_submesh_scratch") + out_mesh
    bounds = {"connected_components": (lambda: mesh_ops.connected_components(mesh), cc),
              "vertex_normals": (lambda: mesh_ops.vertex_normals(mesh), q("nslam_mesh_vertex_normals_scratch") + 12 * nv),
              "submesh": (lambda: mesh_ops.submesh(mesh, keep), sub),
              "cull": (lambda: mesh_ops.cull(mesh, poses, intr, room.W, room.H), nv + nt + sub),
              "remove_small_components": (lambda: mesh_ops.remove_small_components(mesh, 0.05), cc + nt + sub),
              "simplify_vertex_clustering": (lambda: mesh_ops.simplify_vertex_clustering(mesh, 0.01),
                                             q("nslam_mesh_cluster_scratch") + out_mesh +
                                             q("nslam_mesh_vertex_normals_scratch"))}
    for name, (fn, bound) in bounds.items():
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        out = fn()
        torch.cuda.synchronize()
        peak = torch.cuda.max_memory_allocated() - base
        bound += 1 << 20
        print(f"512^3 {name}: peak {peak / 2**20:.1f} MiB, bound {bound / 2**20:.1f} MiB ({nv} vertices, {nt} triangles)")
        assert peak <= bound, (name, peak, bound)
        del out
