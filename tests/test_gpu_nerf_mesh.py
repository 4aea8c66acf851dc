"""NeRF mesh read-out on the GPU (pyngp.Testbed.marching_cubes; csrc/ngp_tc.cu + csrc/tsdf_mesh.cu) against the
tensor-core forward, the fp32 oracle network and the numpy restatement of tests/nerf_mesh_oracle.py, and end to end on
the synthetic room."""
import ctypes
import types

import numpy as np
import pytest
import torch

from tests import nerf_mesh_oracle as onm

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
F32 = np.float32


def _testbed(seed=3, seen=0.7):
    """random network (table values +-0.5 so that the encoding matters), occupancy cells seen with probability `seen`"""
    from nerf_slam_b200 import pyngp
    tb = pyngp.Testbed(seed=seed, max_samples=1 << 16, max_rays=1 << 13)
    tb.create_empty_nerf_dataset(8, 1.0, None, 4, None)
    g = torch.Generator().manual_seed(seed)
    tb.grid_master.copy_(((torch.rand(tb.grid_master.shape, generator=g) * 2 - 1) * 0.5).to(DEV))
    tb.grid_half.copy_(tb.grid_master.half())
    tb.pack_weights()
    dens = torch.where(torch.rand(tb.density.shape, generator=g) < seen, 0.0, -1.0)
    tb.density.copy_(dens.to(DEV))
    return tb


def _forward_tc(tb, coords):
    from nerf_slam_b200 import _lib
    n = coords.shape[0]
    out = torch.zeros(n, 4, device=DEV)
    _lib.check(_lib.load().nslam_ngp_forward_tc(ctypes.byref(tb.model), _lib.ptr(tb.packed), _lib.ptr(coords.contiguous()),
                                                None, n, n, _lib.ptr(out), None, tb.num_sms, _lib.stream_ptr()), "fwd_tc")
    return out


def _lattice(tb, resolution=48, aabb=None, thresh=0.0):
    from nerf_slam_b200.pyngp import mesh_lattice
    lo, h, dims = mesh_lattice(resolution, aabb, tb.aabb_scale)
    field, weight = tb.mesh_kernels.lattice(tb, lo, h, dims, thresh)
    torch.cuda.synchronize()
    return lo, h, dims, field, weight


def test_lattice_sigma_and_visibility():
    """sigma (field at thresh 0 = -sigma exactly) bit-identical to the tensor-core forward at the same x01 built in torch
    with the same roundings, within 3e-2 relative of the fp32 oracle network; weights equal the numpy visibility rule
    on the device's occupancy array"""
    tb = _testbed()
    lo, h, dims, field, weight = _lattice(tb)
    nx, ny, nz = dims
    k, j, i = torch.meshgrid(*(torch.arange(n, dtype=torch.float32, device=DEV) for n in (nz, ny, nx)), indexing="ij")
    hh = torch.tensor(float(h), device=DEV)
    p = torch.stack([torch.add(torch.mul(hh, a), float(lo[q])) for q, a in enumerate((i, j, k))], -1)
    pn = onm.lattice_points(lo, h, dims)
    assert np.array_equal(p.cpu().numpy(), pn)
    x01 = torch.mul(torch.sub(p, F32(0.5 - 0.5 * tb.aabb_scale).item()), F32(1.0 / tb.aabb_scale).item()).reshape(-1, 3)
    assert np.array_equal(x01.cpu().numpy(), onm.hash_input(pn, tb.aabb_scale).reshape(-1, 3))
    d = torch.nn.functional.normalize(torch.randn(x01.shape[0], 3, generator=torch.Generator().manual_seed(1)), dim=-1)
    coords = torch.cat([x01, torch.zeros_like(x01[:, :1]), d.to(DEV)], -1)
    sigma_tc = _forward_tc(tb, coords)[:, 3]
    sigma = -field.reshape(-1)
    assert torch.equal(sigma, sigma_tc)
    P = onm.network_params(tb.grid_half, tb.mlp)
    ref = onm.network_sigma(P, tb.aabb_scale)(pn).reshape(-1)
    rel = np.abs(sigma.cpu().numpy() - ref) / ref
    assert rel.max() < 3e-2, rel.max()
    assert np.ptp(np.log(ref)) > 0.1                                    # the field is not constant
    w = weight.cpu().numpy()
    assert np.array_equal(w, onm.visibility(pn, tb.density.cpu().numpy(), tb.cascades))
    assert 0.3 < w.mean() < 0.9


def _median_thresh(tb, resolution=48):
    _, _, _, field, weight = _lattice(tb, resolution)
    return float(torch.quantile(-field[weight > 0], 0.5))


def test_mesh_matches_the_readout_oracle():
    """marching cubes on the field / weights the GPU produced: positions and triangles bit-exact to
    tests/tsdf_readout_oracle.py (min_weight 0, no colour volume), normals within 1e-6"""
    tb = _testbed(seed=4)
    thresh = _median_thresh(tb)
    lo, h, dims, field, weight = _lattice(tb, 48, None, thresh)
    mesh = tb.mesh_kernels.mesh(field, weight, lo, h)
    V, F, C, N = onm.mesh(field.cpu().numpy(), weight.cpu().numpy(), lo, h)
    assert len(F) > 1000
    assert np.array_equal(mesh.vertices.cpu().numpy(), V) and np.array_equal(mesh.triangles.cpu().numpy(), F)
    assert np.abs(mesh.vertex_normals.cpu().numpy() - N).max() <= 1e-6
    assert float(mesh.vertex_colors.abs().max()) == 0.0                 # no colour volume: colour 0 until the colour pass


def test_colors_match_the_forward_and_srgb():
    """colours bit-identical to the tensor-core forward at [x01, 0, -n] (+z where n = 0); the sRGB variant within 2e-6
    of numpy's encoding of the linear colours"""
    tb = _testbed(seed=5)
    thresh = _median_thresh(tb)
    mesh = tb.marching_cubes(48, None, thresh, srgb=False)
    V, N = mesh.vertices, mesh.vertex_normals.clone()
    N[:7] = 0                                                            # exercise the n = 0 rule
    mesh.vertex_normals = N
    tb.mesh_kernels.colors(tb, mesh, False)
    lin = mesh.vertex_colors.clone()
    x01 = torch.mul(torch.sub(V, F32(0.5 - 0.5 * tb.aabb_scale).item()), F32(1.0 / tb.aabb_scale).item())
    dirs = -N
    dirs[(N == 0).all(1)] = torch.tensor([0.0, 0.0, 1.0], device=DEV)
    ref = _forward_tc(tb, torch.cat([x01, torch.zeros_like(x01[:, :1]), dirs], -1))[:, :3]
    assert len(V) > 1000 and torch.equal(lin, ref)
    assert np.array_equal(torch.cat([x01, torch.zeros_like(x01[:, :1]), dirs], -1).cpu().numpy(),
                          onm.color_records(V.cpu().numpy(), N.cpu().numpy(), tb.aabb_scale))
    tb.mesh_kernels.colors(tb, mesh, True)
    srgb = mesh.vertex_colors.cpu().numpy()
    assert np.abs(srgb - onm.linear_to_srgb(lin.cpu().numpy())).max() <= 2e-6
    # against the fp32 oracle network, within the tensor-core tolerance on colours
    P = onm.network_params(tb.grid_half, tb.mlp)
    assert np.abs(lin.cpu().numpy() - onm.network_colors(P, tb.aabb_scale, V.cpu().numpy(), N.cpu().numpy())).max() < 1e-2


def test_chunked_colours_over_many_vertices():
    """more vertices than one chunk of the colour pass (2^18): every chunk lands at its own rows"""
    tb = _testbed(seed=6)
    from nerf_slam_b200.tsdf_fusion import TsdfMesh
    n = (1 << 18) + 12345
    g = torch.Generator().manual_seed(2)
    V = (torch.rand(n, 3, generator=g) * 2 - 0.5).to(DEV)
    N = torch.nn.functional.normalize(torch.randn(n, 3, generator=g), dim=-1).to(DEV)
    mesh = TsdfMesh(V, torch.zeros(0, 3, dtype=torch.int32, device=DEV), torch.empty(n, 3, device=DEV), N)
    tb.mesh_kernels.colors(tb, mesh, False)
    x01 = torch.mul(torch.sub(V, F32(-1.5).item()), F32(0.25).item())
    ref = _forward_tc(tb, torch.cat([x01, torch.zeros_like(x01[:, :1]), -N], -1))[:, :3]
    assert torch.equal(mesh.vertex_colors, ref)


def test_edge_cases_untrained_and_ply_round_trip(tmp_path):
    """an untrained testbed has nothing observed: None / empty arrays / an empty PLY; a mesh written by
    compute_and_save_marching_cubes_mesh reads back equal to compute_marching_cubes_mesh"""
    from nerf_slam_b200 import pyngp
    tb = pyngp.Testbed(seed=1)
    tb.create_empty_nerf_dataset(4, 1.0, None, 4, None)
    assert tb.marching_cubes(32) is None
    out = tb.compute_marching_cubes_mesh(resolution=32)
    assert all(out[k].shape == (0, 3) for k in "VNCF") and out["F"].dtype == np.int32
    path = str(tmp_path / "empty.ply")
    tb.compute_and_save_marching_cubes_mesh(path, resolution=32)
    assert all(a.shape == (0, 3) for a in onm.read_ply(path))
    tb = _testbed(seed=7)
    thresh = _median_thresh(tb, 40)
    box = [[-0.5, -0.2, 0.0], [1.5, 1.2, 1.1]]
    out = tb.compute_marching_cubes_mesh(resolution=40, aabb=box, thresh=thresh)
    path = str(tmp_path / "mesh.ply")
    tb.compute_and_save_marching_cubes_mesh(path, resolution=40, aabb=pyngp.BoundingBox(*box), thresh=thresh)
    V, N, C, F = onm.read_ply(path)
    assert len(F) > 100 and out["F"].dtype == np.int32 and out["V"].dtype == np.float32
    for a, b in ((V, out["V"]), (N, out["N"]), (C, out["C"]), (F, out["F"])):
        assert np.array_equal(a, b)
    lo, hi = np.array(box[0], F32), np.array(box[1], F32)
    assert np.all(out["V"].min(0) >= lo) and np.all(out["V"].max(0) <= hi + 1e-6)


# ------------------------------------------------------------------------------------------------------- trained room
ROOM_RES, ROOM_THRESH = 256, 10.0           # see test_room_mesh_lies_on_the_walls


@pytest.fixture(scope="module")
def room():
    """the room of test_gpu_ngp.py::test_nerf_fits_synthetic_room: half extent (1.4, 1.0, 1.4) m, 12 views, 300
    tensor-core steps, metric poses and linear colours"""
    from nerf_slam_b200.nerf_fusion import NerfFusion
    from nerf_slam_b200.synthetic import SyntheticRoom
    room = SyntheticRoom(160, 120, 12, seed=0, half_extent=(1.4, 1.0, 1.4), orbit_radius=0.3, step=0.25)
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
    return nf


def _wall_distance(V, ext=(1.4, 1.0, 1.4)):
    """distance of each vertex to the nearest of the six wall planes x, y, z = +-ext"""
    return np.min(np.abs(np.abs(V) - np.asarray(ext)), axis=1)


def test_room_mesh_lies_on_the_walls(room):
    """NerfFusion.build_mesh of the trained room (sRGB colours: the metric ingest is linear) is not empty and lies on
    the walls.  First H100 run: the observed lattice points of this room have sigma 0.03 / 1.2 / 14 / 64 at the 10 / 50
    / 90 / 99th percentile, so the default thresh 2.5 cuts through the soft density in front of the walls (17 % of the
    vertices within 4 lattice steps of a wall at 256^3); thresh 10 is the best of 0.5 ... 100 there.  At resolution 256
    and thresh 10 (h = 15.7 mm) that run gave 424 502 vertices, 825 494 triangles, 62.2 % of the vertices within 10 cm of
    one of the six wall planes, 52.5 % within 4 h, median distance 5.3 cm.  Asserted: > 100 000 vertices, > 55 % within
    10 cm, > 45 % within 4 h, median < 8 cm.  The rest are floaters of a 300-step fit behind the walls and in the room."""
    mesh = room.build_mesh(resolution=ROOM_RES, thresh=ROOM_THRESH)
    assert mesh is not None
    V = mesh.vertices.cpu().numpy()
    dist = _wall_distance(V)
    h = 4.0 / (ROOM_RES - 1)
    near, near_h, med = float((dist < 0.10).mean()), float((dist < 4 * h).mean()), float(np.median(dist))
    print(f"room mesh: {len(V)} vertices, {mesh.triangles.shape[0]} triangles, within 10 cm {near:.4f}, within 4h "
          f"{near_h:.4f}, median distance {med:.4f} m")
    assert len(V) > 100_000 and near > 0.55 and near_h > 0.45 and med < 0.08
    C = mesh.vertex_colors.cpu().numpy()
    assert np.all((C >= 0) & (C <= 1))


def test_room_mesh_is_deterministic(room):
    a = room.ngp.compute_marching_cubes_mesh(resolution=ROOM_RES, thresh=ROOM_THRESH)
    b = room.ngp.compute_marching_cubes_mesh(resolution=ROOM_RES, thresh=ROOM_THRESH)
    assert len(a["F"]) > 0
    for k in "VFNC":
        assert a[k].tobytes() == b[k].tobytes(), k


def test_memory_at_512(room):
    """peak device memory added by a 512^3 read-out: 8 B per lattice point (field + weight), the marching cubes'
    scratch (4 + 3 ints per 256 points, 16 B per active voxel <= vertices + triangles) and outputs (36 B per vertex,
    12 B per triangle), plus a 1 MiB margin (allocator rounding, count read-back).  The colour pass's chunk scratch (44 B
    per vertex of a chunk of at most 2^18, 11.5 MB) is allocated after the field and weight are freed, so the peak
    does not include it."""
    tb = room.ngp
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    mesh = tb.marching_cubes(512, None, ROOM_THRESH)
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    n = 512 ** 3
    nv, nt = mesh.vertices.shape[0], mesh.triangles.shape[0]
    bound = 8 * n + 4 * (4 + 3 * ((n + 255) // 256)) + 16 * (nv + nt) + 36 * nv + 12 * nt + (1 << 20)
    print(f"512^3: peak {peak / 2**20:.1f} MiB, bound {bound / 2**20:.1f} MiB, {nv} vertices, {nt} triangles")
    assert peak <= bound, (peak, bound)
