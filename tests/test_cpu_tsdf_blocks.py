"""CPU checks of the sparse voxel-block volume: the numpy oracle (oracle/tsdf_blocks.py) against the reference's own
integration method run on a block stand-in (tests/golden/ref_tsdf_blocks.npz) and against the dense oracle, the
activation rule's edge cases, key packing, and the host logic of VoxelBlockVolume / TsdfFusion with the oracle standing
in for the kernels."""
import os
import types

import numpy as np
import pytest
import torch

from oracle import tsdf as otsdf
from oracle import tsdf_blocks as otb

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_tsdf_blocks.npz")


def _golden():
    g = np.load(GOLDEN)
    K = g["intr"]
    return g, np.array([K[0, 0], K[1, 1], K[0, 2], K[1, 2]], np.float32)


@pytest.mark.parametrize("tag", ["tsdf", "sigma"])
def test_oracle_reproduces_the_reference_method_on_blocks(tag):
    """touched keys and pool order exactly; voxels bit for bit in "tsdf"; in "sigma" the golden's weights carry the
    last-bit error of torch's CPU sqrt, held to the dense golden's allowance (tests/test_cpu_golden.py)"""
    g, intr4 = _golden()
    vol = otb.BlockVolume(g["voxel_size"])
    for k in range(3):
        cov = g["covs"][k] if tag == "sigma" else None
        keys = vol.integrate(g["idepths"][k], cov, g["imgs"][k], intr4, g["poses"][k])
        assert np.array_equal(keys, g[f"{tag}_touched_{k}"]), k
        assert np.array_equal(vol.keys, g[f"{tag}_keys_{k}"]), k
        t, w, c = g[f"{tag}_tsdf_{k}"], g[f"{tag}_weight_{k}"], g[f"{tag}_color_{k}"]
        assert np.array_equal(vol.weight > 0, w > 0), k
        if tag == "tsdf":
            assert np.array_equal(vol.tsdf, t) and np.array_equal(vol.weight, w) and np.array_equal(vol.color, c), k
        else:
            assert np.allclose(vol.weight, w, rtol=3e-7, atol=0) and np.allclose(vol.tsdf, t, rtol=0, atol=3e-7) \
                and np.allclose(vol.color, c, rtol=0, atol=1e-4), k
    coords = vol.coords
    assert len(coords) >= 8 and (coords < 0).any() and (coords >= 0).any()
    assert (vol.weight > 0).sum() > 2000


def _frame(rng, H=30, W=40, with_cov=True, depth=(0.5, 2.5)):
    idepth = rng.uniform(1 / depth[1], 1 / depth[0], (H, W)).astype(np.float32)
    cov = rng.uniform(0.01, 0.5, (H, W)).astype(np.float32) if with_cov else None
    if with_cov:
        cov[:3] = 3e8
    rgb = rng.integers(0, 255, (3, H, W), dtype=np.uint8)
    q = rng.normal(size=4) * 0.05 + np.array([0, 0, 0, 1.0]); q /= np.linalg.norm(q)
    intr = np.array([W * 0.6, W * 0.6, W / 2 - 0.5, H / 2 - 0.5], np.float32)
    return idepth, cov, rgb, intr, q


def _pose_at(centre, q):
    """cam_T_world (t, q) of a camera at world position `centre` with rotation q"""
    R = otsdf.pose_tq_to_matrix(np.concatenate([np.zeros(3), q]).astype(np.float32))[:3, :3]
    return np.concatenate([-R @ np.asarray(centre, np.float64), q]).astype(np.float32)


@pytest.mark.parametrize("mode", ["sigma", "tsdf"])
def test_block_update_equals_the_dense_oracle_on_the_touched_blocks(mode):
    """one keyframe at non-negative voxel indices: the block update equals oracle.tsdf.integrate on an origin-0 dense grid
    on every voxel of the touched blocks, and the two per-voxel restatements agree on the whole grid"""
    rng = np.random.default_rng(3)
    vs = np.float32(0.06)
    idepth, cov, rgb, intr, q = _frame(rng, with_cov=(mode == "sigma"), depth=(0.4, 1.2))
    tq = _pose_at((2.0, 2.0, 0.5), q)
    vol = otb.BlockVolume(vs)
    keys = vol.integrate(idepth, cov, rgb, intr, tq)
    coords = vol.coords
    assert len(keys) > 10 and (coords >= 0).all()
    n = 16 * (coords.max(0) + 2)
    dt, dw, dc = np.zeros(n[::-1], np.float32), np.zeros(n[::-1], np.float32), np.zeros(tuple(n[::-1]) + (3,), np.float32)
    otsdf.integrate(dt, dw, dc, np.zeros(3, np.float32), vs, idepth, cov, rgb, intr, tq)
    for i, b in enumerate(coords):
        s = np.s_[16 * b[2]:16 * b[2] + 16, 16 * b[1]:16 * b[1] + 16, 16 * b[0]:16 * b[0] + 16]
        assert np.array_equal(vol.tsdf[i], dt[s]) and np.array_equal(vol.weight[i], dw[s]) and np.array_equal(vol.color[i], dc[s])
    # the explicit-coordinate restatement on the whole origin-0 grid
    t, w, c = np.zeros_like(dt), np.zeros_like(dw), np.zeros_like(dc)
    iz, iy, ix = np.meshgrid(*(np.arange(m) for m in n[::-1]), indexing="ij")
    world = (vs * np.stack([ix, iy, iz], -1).astype(np.float32)).astype(np.float32)
    otb.update_voxels(t, w, c, world, idepth, cov, rgb, intr, tq)
    assert np.array_equal(t, dt) and np.array_equal(w, dw) and np.array_equal(c, dc)


def test_touched_set_skips_invalid_and_masked_pixels():
    rng = np.random.default_rng(4)
    vs = np.float32(0.05)
    idepth, cov, rgb, intr, q = _frame(rng)
    tq = _pose_at((0.3, -0.2, 0.1), q)
    bad = idepth.copy()
    bad[5:10] = 0.0                                      # depth inf
    bad[10:12] = -1.0                                    # negative depth
    bad[12:14] = 1 / 7.0                                 # beyond max_depth
    bad[14:16] = np.nan
    masked = cov.copy()
    masked[16:20] = 1e9                                  # sigma test masks them
    keys = otb.touched_keys(bad, masked, intr, tq, vs)
    ok = np.ones(idepth.shape, bool)
    ok[5:16] = False; ok[16:20] = False; ok[:3] = False
    only = np.where(ok, idepth, np.float32(-1.0))
    assert np.array_equal(keys, otb.touched_keys(only, None, intr, tq, vs))
    assert len(keys) > 0
    assert len(otb.touched_keys(np.full_like(idepth, -1.0), None, intr, tq, vs)) == 0
    assert len(otb.touched_keys(idepth, np.full_like(cov, 1e9), intr, tq, vs)) == 0


def test_key_packing_round_trips_and_rejects_out_of_range():
    b = np.array([[0, 0, 0], [-1, 2, -3], [2 ** 20 - 1, -2 ** 20, 5], [2 ** 20, 0, 0], [0, -2 ** 20 - 1, 0]])
    keys, ok = otb.pack(b)
    assert ok.tolist() == [True, True, True, False, False]
    assert np.array_equal(otb.unpack(keys[ok]), b[ok])
    assert (keys[ok] >= 0).all()
    # ascending keys run z-major, then y, then x
    s = np.array([[1, 0, 0], [0, 1, 0], [0, 0, 1], [-1, -1, 1]])
    assert np.argsort(otb.pack(s)[0]).tolist() == [0, 1, 3, 2]
    # a pose far away puts every sample outside the packable range: nothing is touched
    rng = np.random.default_rng(5)
    idepth, _, _, intr, q = _frame(rng, with_cov=False)
    far = np.concatenate([[0, 0, -1e9], [0, 0, 0, 1]]).astype(np.float32)
    assert len(otb.touched_keys(idepth, None, intr, far, np.float32(0.01))) == 0


class OracleKernels:
    """the four passes of VoxelBlockVolume on CPU tensors, computed by the numpy oracle"""

    def __init__(self):
        self.rehashes = 0

    def activate(self, vol, f):
        keys = otb.touched_keys(f["idepth"].numpy(), None if f["cov"] is None else f["cov"].numpy(), f["intr"],
                                f["pose"].numpy(), vol.voxel_size, f["max_depth"], f["max_depth_sigma"])
        pool = vol._keys[:vol.n_blocks].numpy()
        index = {int(k): i for i, k in enumerate(pool)}
        new = np.setdiff1d(keys, pool)
        rank = {int(k): vol.n_blocks + i for i, k in enumerate(new)}
        touched = [index.get(int(k), rank.get(int(k))) for k in keys]
        return torch.tensor(touched, dtype=torch.int32), torch.from_numpy(new)

    def insert(self, vol, new_keys):
        n0, m = vol.n_blocks, new_keys.shape[0]
        vol._keys[n0:n0 + m] = new_keys
        vol._coords[n0:n0 + m] = torch.from_numpy(otb.unpack(new_keys.numpy()))
        for t in (vol.tsdf, vol.weight, vol.color):
            t[n0:n0 + m] = 0

    def rehash(self, vol):
        self.rehashes += 1

    def integrate(self, vol, touched, f):
        p = touched.long().numpy()
        t, w, c = vol.tsdf.numpy()[p], vol.weight.numpy()[p], vol.color.numpy()[p]
        otb.update_voxels(t, w, c, otb.voxel_world(vol._coords[p].numpy(), vol.voxel_size), f["idepth"].numpy(),
                          None if f["cov"] is None else f["cov"].numpy(), f["rgb"].numpy(), f["intr"], f["pose"].numpy(),
                          f["max_depth"], f["sdf_trunc"], f["max_weight"], f["max_depth_sigma"])
        vol.tsdf[touched.long()], vol.weight[touched.long()], vol.color[touched.long()] = \
            torch.from_numpy(t), torch.from_numpy(w), torch.from_numpy(c)


def _frames(n=3):
    rng = np.random.default_rng(9)
    out = []
    for k in range(n):
        idepth, cov, rgb, intr, q = _frame(rng)
        out.append((torch.from_numpy(idepth), torch.from_numpy(cov), torch.from_numpy(rgb), intr,
                    torch.from_numpy(_pose_at((0.4 * k - 0.3, 0.1, -0.2), q))))
    return out


def test_growth_keeps_indices_and_order(monkeypatch):
    from nerf_slam_b200 import tsdf_blocks as tb
    monkeypatch.setattr(tb.VoxelBlockVolume, "kernels", OracleKernels())
    small, big = tb.VoxelBlockVolume(0.05, 2, "cpu"), tb.VoxelBlockVolume(0.05, 5000, "cpu")
    ref = otb.BlockVolume(0.05)
    for idepth, cov, rgb, intr, tq in _frames():
        before = small._keys[:small.n_blocks].clone(), small.tsdf[:small.n_blocks].clone()
        small.integrate(idepth, cov, rgb, intr, tq)
        big.integrate(idepth, cov, rgb, intr, tq)
        ref.integrate(idepth.numpy(), cov.numpy(), rgb.numpy(), intr, tq.numpy())
        assert torch.equal(small._keys[:before[0].shape[0]], before[0])          # earlier blocks keep their index
    assert small.kernels.rehashes >= 1 and small.capacity >= small.n_blocks and small.capacity & (small.capacity - 1) == 0
    assert big.capacity == 5000 and small.n_blocks == big.n_blocks == len(ref.keys)
    n = small.n_blocks
    assert np.array_equal(small._keys[:n].numpy(), ref.keys) and torch.equal(small.block_coords, big.block_coords)
    for a in ("tsdf", "weight", "color"):
        assert torch.equal(getattr(small, a)[:n], getattr(big, a)[:n])
        assert np.array_equal(getattr(small, a)[:n].numpy(), getattr(ref, a))
    t, w, c, org = small.to_dense(margin_blocks=1)
    rt, rw, rc, rorg = otb.to_dense(ref.coords, ref.tsdf, ref.weight, ref.color, 0.05)
    assert np.array_equal(t.numpy(), rt) and np.array_equal(w.numpy(), rw) and np.array_equal(c.numpy(), rc)
    assert np.array_equal(org, rorg)
    assert small.memory_bytes() > small.capacity * 80 * 1024


def test_tsdf_fusion_holds_one_volume_of_either_kind(monkeypatch):
    from nerf_slam_b200 import tsdf_blocks as tb
    from nerf_slam_b200.tsdf_fusion import DenseVolume, TsdfFusion
    monkeypatch.setattr(tb.VoxelBlockVolume, "kernels", OracleKernels())
    with pytest.raises(ValueError):
        TsdfFusion("sigma", types.SimpleNamespace(tsdf_volume="hashed"), "cpu")
    args = types.SimpleNamespace(eval=False, tsdf_volume="blocks", tsdf_block_count=3)
    fus = TsdfFusion("sigma", args, "cpu")
    assert isinstance(fus.volume, tb.VoxelBlockVolume) and fus.volume.capacity == 3
    assert not any(hasattr(fus, a) for a in ("tsdf", "weight", "color", "origin"))
    fr = _frames(2)
    packet = {"cam0_poses": torch.stack([f[4] for f in fr]), "cam0_idepths_up": torch.stack([f[0] for f in fr]),
              "cam0_depths_cov_up": torch.stack([f[1] for f in fr]), "cam0_images": torch.stack([f[2] for f in fr])}
    fus.build_volume(packet, fr[0][3])
    ref = otb.BlockVolume(fus.voxel_size)
    for idepth, cov, rgb, intr, tq in fr:
        ref.integrate(idepth.numpy(), cov.numpy(), rgb.numpy(), intr, tq.numpy())
    n = fus.volume.n_blocks
    assert fus.integrated_frames == 2 and n == len(ref.keys) and np.array_equal(fus.volume.tsdf[:n].numpy(), ref.tsdf)
    with pytest.raises(NotImplementedError, match="build_mesh"):
        fus.surface_points()
    cap, vs = fus.volume.capacity, fus.voxel_size
    fus.reset_volume()
    assert fus.voxel_size == vs / 2 and fus.volume.voxel_size == float(np.float32(vs / 2))
    assert fus.volume.n_blocks == 0 and fus.volume.capacity == cap
    dense = TsdfFusion("sigma", types.SimpleNamespace(eval=False, tsdf_resolution=8), "cpu")
    assert isinstance(dense.volume, DenseVolume) and dense.volume.tsdf.shape == (8, 8, 8)
    assert not any(hasattr(dense, a) for a in ("tsdf", "weight", "color", "origin"))


def test_dense_volume_resets_in_place():
    """reset_volume zeroes the dense grid's own tensors (no second grid) and moves the origin to the halved voxel"""
    from nerf_slam_b200.tsdf_fusion import DenseVolume, TsdfFusion
    centre = np.array([0.31, -0.52, 1.07], np.float32)
    fus = TsdfFusion("sigma", types.SimpleNamespace(eval=False, tsdf_resolution=8, tsdf_center=tuple(centre)), "cpu")
    vol = fus.volume
    assert isinstance(vol, DenseVolume) and vol.device == "cpu" and vol.voxel_size == float(np.float32(6.0 / 512))
    lattice = lambda vs: ((np.round(centre / np.float32(vs)) - 4) * np.float32(vs)).astype(np.float32)
    assert vol.origin.dtype == np.float32 and np.array_equal(vol.origin, lattice(6.0 / 512))
    assert vol.color.shape == (8, 8, 8, 3) and all(not t.any() for t in (vol.tsdf, vol.weight, vol.color))
    assert vol.memory_bytes() == 8 ** 3 * 5 * 4
    tensors = (vol.tsdf, vol.weight, vol.color)
    ptrs = [t.data_ptr() for t in tensors]
    for t in tensors:
        t.fill_(1.5)
    fus.reset_volume()
    assert fus.volume is vol and fus.voxel_size == 3.0 / 512 and vol.voxel_size == float(np.float32(3.0 / 512))
    assert all(a is b for a, b in zip((vol.tsdf, vol.weight, vol.color), tensors))
    assert [t.data_ptr() for t in tensors] == ptrs and all(not t.any() for t in tensors)
    assert np.array_equal(vol.origin, lattice(3.0 / 512)) and not np.array_equal(lattice(3.0 / 512), lattice(6.0 / 512))
    t, w, c, org = vol.to_dense()
    assert t is vol.tsdf and w is vol.weight and c is vol.color and org is vol.origin
