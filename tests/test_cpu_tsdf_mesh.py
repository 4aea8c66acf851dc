"""TSDF read-outs without a GPU: the numpy restatements of marching cubes and ray casting (tests/tsdf_readout_oracle.py)
on analytic fields, the case table compiled into csrc/tsdf_mesh.cu, the PLY writer and the evaluation metrics."""
import os
import re
from collections import Counter

import numpy as np
import torch

from tests import tsdf_readout_oracle as orc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F32 = np.float32


def _sphere(n=32, c=(15.3, 16.1, 15.7), r=9.3, trunc=4.0):
    k, j, i = np.meshgrid(np.arange(n), np.arange(n), np.arange(n), indexing="ij")
    d = np.sqrt((i - c[0]) ** 2 + (j - c[1]) ** 2 + (k - c[2]) ** 2)
    return np.clip((d - r) / trunc, -1, 1).astype(F32), np.asarray(c), r


def _mesh(t, w=None, min_weight=0.5):
    w = np.ones_like(t) if w is None else w
    return orc.marching_cubes(t, w, np.zeros(t.shape + (3,), F32), np.zeros(3, F32), 1.0, min_weight)


def _edges(F):
    directed = Counter()
    for a, b, c in F.tolist():
        directed.update([(a, b), (b, c), (c, a)])
    undirected = Counter()
    for (a, b), m in directed.items():
        undirected[(min(a, b), max(a, b))] += m
    return directed, undirected


def test_kernel_table_is_the_oracle_table():
    src = open(os.path.join(ROOT, "nerf_slam_b200", "csrc", "tsdf_mesh.cu")).read()
    body = src[src.index("c_tri[256][16] = {"):]
    body = body[:body.index("};")]
    rows = re.findall(r"\{([-0-9,\s]+)\}", body)
    assert len(rows) == 256
    for case, row in enumerate(rows):
        vals = [int(x) for x in row.split(",")]
        tris = [tuple(vals[3 * s:3 * s + 3]) for s in range(5) if vals[3 * s] >= 0]
        assert tris == orc.TRI_TABLE[case], case
        assert all(v == -1 for v in vals[3 * len(tris):])


def test_table_cases_cover_exactly_the_crossed_edges():
    for case, tris in enumerate(orc.TRI_TABLE):
        crossed = {e for e, (a, b) in enumerate(orc.EDGES) if ((case >> a) & 1) != ((case >> b) & 1)}
        assert {e for t in tris for e in t} == crossed, case
        assert len(tris) <= 5


def test_sphere_mesh_is_closed_oriented_and_on_the_surface():
    t, c, r = _sphere()
    V, F, _, N = _mesh(t)
    directed, undirected = _edges(F)
    assert set(directed.values()) == {1} and set(undirected.values()) == {2}
    assert len(V) - len(undirected) + len(F) == 2
    assert np.abs(np.linalg.norm(V - c, axis=1) - r).max() < 0.1
    cr = np.cross(V[F[:, 1]] - V[F[:, 0]], V[F[:, 2]] - V[F[:, 0]])
    area = 0.5 * np.linalg.norm(cr, axis=1).sum()
    assert abs(area / (4 * np.pi * r * r) - 1) < 0.02
    assert ((cr * (V[F].mean(1) - c)).sum(1) > 0).all()
    assert ((N * (V - c)).sum(1) > 0).all() and np.allclose(np.linalg.norm(N, axis=1), 1, atol=1e-6)


def test_torus_mesh_has_euler_characteristic_zero():
    n, R, rr = 40, 11.0, 4.3
    c = np.array([19.6, 20.2, 19.4])
    k, j, i = np.meshgrid(np.arange(n), np.arange(n), np.arange(n), indexing="ij")
    x, y, z = i - c[0], j - c[1], k - c[2]
    d = np.sqrt((np.sqrt(x * x + y * y) - R) ** 2 + z * z) - rr
    V, F, _, _ = _mesh(np.clip(d / 4, -1, 1).astype(F32))
    directed, undirected = _edges(F)
    assert set(directed.values()) == {1}
    assert len(V) - len(undirected) + len(F) == 0


def test_partial_weights_mesh_only_valid_cubes_and_reference_every_vertex():
    t, _, _ = _sphere()
    rng = np.random.default_rng(3)
    w = rng.uniform(0, 1, t.shape).astype(F32)
    w[rng.uniform(size=t.shape) < 0.5] = 1.0
    mw = 0.3
    V, F, _, _ = _mesh(t, w, mw)
    assert len(F) > 100
    assert np.array_equal(np.unique(F), np.arange(len(V)))
    # every triangle lies inside a cube whose 8 corners pass the weight test
    lo = np.floor(V[F].min(1) + 1e-4).astype(int)
    hi = np.ceil(V[F].max(1) - 1e-4).astype(int)
    assert (hi - lo <= 1).all()
    for (i, j, k) in lo:
        assert (w[k:k + 2, j:j + 2, i:i + 2] > mw).all()


def _plane_volume(n=24, vs=0.05, z0=0.7):
    zw = (np.arange(n) * vs)[:, None, None] * np.ones((1, n, n))
    t = np.clip((z0 - zw) / 0.5, -1, 1).astype(F32)
    return t, np.ones_like(t), np.full(t.shape + (3,), 100, F32)


def test_raycast_plane_hits_at_the_analytic_depth():
    vs = 0.05
    t, w, col = _plane_volume(vs=vs)
    tq = np.array([-0.6, -0.6, 0.1, 0, 0, 0, 1], np.float32)          # camera at (0.6, 0.6, -0.1), looking along +z
    D, C, Wt, N = orc.raycast(t, w, col, np.zeros(3, F32), vs, tq, 16, 20, [20, 20, 9.5, 7.5], 0.01, 3.0, 0.1, 0.5)
    assert (D > 0).all()
    assert np.abs(D - 0.8).max() < 1e-3 * vs
    assert np.allclose(C, 100 / 255.0) and np.allclose(Wt, 1.0)
    assert np.allclose(N, [0, 0, -1], atol=1e-6)


def test_raycast_sphere_hits_within_a_tenth_of_a_voxel_and_misses_give_zeros():
    t, c, r = _sphere(trunc=3.0)
    w = np.ones_like(t)
    col = np.full(t.shape + (3,), 50, F32)
    # grid coordinates = world coordinates (voxel 1, origin 0); camera on the -z side of the sphere looking along +z
    cam = np.array([c[0], c[1], c[2] - 14.0])
    tq = np.concatenate([-cam, [0, 0, 0, 1]]).astype(F32)
    H, W, f = 40, 40, 12.0
    intr = [f, f, 19.5, 19.5]
    D, C, Wt, N = orc.raycast(t, w, col, np.zeros(3, F32), 1.0, tq, H, W, intr, 0.5, 40.0, 3.0, 0.5)
    v, u = np.meshgrid(np.arange(H), np.arange(W), indexing="ij")
    d = np.stack([(u - 19.5) / f, (v - 19.5) / f, np.ones_like(u, float)], -1)
    oc = cam - c
    b = (d @ oc)
    a = (d * d).sum(-1)
    disc = b * b - a * ((oc * oc).sum() - r * r)
    hit = disc > 0
    z = (-b - np.sqrt(np.where(hit, disc, 0))) / a
    inner = disc > 0.2 * a * r * r                                       # away from the silhouette
    assert (D[inner] > 0).all()
    assert np.abs(D[inner] - z[inner]).max() * np.sqrt(a[inner]).max() < 0.1
    far = ~hit
    assert far.sum() > 100
    assert (D[far] == 0).all() and (C[far] == 0).all() and (Wt[far] == 0).all() and (N[far] == 0).all()


def test_ply_round_trip():
    from nerf_slam_b200.tsdf_fusion import TsdfMesh
    rng = np.random.default_rng(0)
    V, T = 37, 50
    m = TsdfMesh(torch.from_numpy(rng.normal(size=(V, 3)).astype(F32)),
                 torch.from_numpy(rng.integers(0, V, (T, 3)).astype(np.int32)),
                 torch.from_numpy(rng.uniform(size=(V, 3)).astype(F32)),
                 torch.from_numpy(rng.normal(size=(V, 3)).astype(F32)))
    import tempfile
    with tempfile.TemporaryDirectory() as d:
        p = os.path.join(d, "m.ply")
        m.write_ply(p)
        raw = open(p, "rb").read()
    head, body = raw.split(b"end_header\n", 1)
    lines = head.decode().splitlines()
    assert lines[:2] == ["ply", "format binary_little_endian 1.0"]
    props = [l.split()[-1] for l in lines if l.startswith("property float")]
    nv = int(next(l for l in lines if l.startswith("element vertex")).split()[-1])
    nf = int(next(l for l in lines if l.startswith("element face")).split()[-1])
    vt = np.frombuffer(body[:nv * 4 * len(props)], [(p, "<f4") for p in props])
    ft = np.frombuffer(body[nv * 4 * len(props):], [("n", "u1"), ("v", "<i4", (3,))])
    assert len(ft) == nf == T and (ft["n"] == 3).all()
    assert np.array_equal(np.stack([vt["x"], vt["y"], vt["z"]], 1), m.vertices.numpy())
    assert np.array_equal(np.stack([vt["nx"], vt["ny"], vt["nz"]], 1), m.vertex_normals.numpy())
    assert np.array_equal(np.stack([vt["red"], vt["green"], vt["blue"]], 1), m.vertex_colors.numpy())
    assert np.array_equal(ft["v"], m.triangles.numpy())


def test_depth_l1_and_psnr_by_hand():
    from nerf_slam_b200.tsdf_fusion import color_psnr, depth_l1_cm
    gt = torch.full((10, 10), 2.0)
    r = torch.full((10, 10), 1.0)
    r[0, 0] = 3.0                                                         # scale = 2 / mean(r) over the 2x2 crop
    r[9, 9] = 100.0                                                       # cropped away
    crop = r[:2, :2]
    s = 2.0 / float(crop.mean())
    err = np.abs(s * crop.numpy() - 2.0)
    err[err > 2.0] = 2.0
    assert abs(float(depth_l1_cm(r, gt)) - err.mean() * 100) < 1e-4
    img = torch.zeros(3, 4, 4, dtype=torch.uint8)
    img[0] = 255
    rc = torch.zeros(4, 4, 3)
    rc[..., 0] = 0.5
    # mse = mean over pixels of the channel mean: (0.25 + 0 + 0) / 3
    assert abs(color_psnr(rc, img) - (-10 * np.log10(0.25 / 3))) < 1e-5                 # fp32 error map
