"""Golden vectors for the sparse voxel-block volume, produced by EXECUTING the reference's own integration method.

    python tests/golden/make_golden_tsdf_blocks.py   (needs /root/reference; writes tests/golden/ref_tsdf_blocks.npz)

As make_golden_tsdf.py (whose stand-ins and `reference_class()` are imported unchanged), the source text of the
reference's `TsdfFusion.build_volume`, `custom_volume_integrate` and `get_depth_masks` is compiled unchanged and run on
stand-ins for Open3D.  Here `self.volume` is a BLOCK volume, standing in for Open3D's VoxelBlockGrid:
  * `compute_unique_block_coordinates` is the activation rule of oracle/tsdf_blocks.py (Open3D's own is unavailable, so
    the touched set is defined by that rule, not pinned against Open3D);
  * `hashmap().activate` appends the blocks that are new in ascending key order, `find` returns their pool indices;
  * `voxel_coordinates_and_flattened_indices` returns the float32 coordinates voxel_size * (16 b + l) and the flat
    indices pool * 4096 + l (l = lx + 16 ly + 256 lz) into attributes of shape [pool * 4096, channels].
The scenario's depth maps span several 16^3 blocks at negative and non-negative block coordinates.  Stored: the inputs,
per flavour ("sigma": variance weights and the sigma mask; "tsdf": uniform weights) and keyframe k the touched keys
(`{tag}_touched_{k}`), and after each keyframe the pool keys in pool order (`{tag}_keys_{k}`) and the pool's tsdf /
weight [B,16,16,16] and color [B,16,16,16,3] (`{tag}_tsdf_{k}`, ...)."""
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

import make_golden_tsdf as mgt                       # noqa: E402
from oracle import tsdf_blocks as otb                # noqa: E402

VOX = otb.BLOCK ** 3


class BlockVolume:
    """the VoxelBlockGrid stand-in: pool attributes [B * 4096, channels], blocks appended in ascending key order"""

    def __init__(self, voxel_size):
        self.vs = np.float32(voxel_size)
        self.keys = np.zeros(0, np.int64)
        self.attr = {"tsdf": torch.zeros(0, 1), "weight": torch.zeros(0, 1), "color": torch.zeros(0, 3)}
        self.touched = []

    def compute_unique_block_coordinates(self, depth, intrinsic, extrinsic, depth_scale, max_depth):
        assert depth_scale == 1.0
        K = np.asarray(intrinsic)
        intr4 = np.array([K[0, 0], K[1, 1], K[0, 2], K[1, 2]], np.float32)
        keys = otb.touched_keys_from_depth(depth.as_tensor().t[..., 0].numpy(), intr4, extrinsic.t.numpy(), self.vs, max_depth)
        self.touched.append(keys)
        return keys

    def hashmap(self):
        vol = self

        class H:
            def activate(self, keys):
                new = np.setdiff1d(keys, vol.keys)
                vol.keys = np.concatenate([vol.keys, new])
                for k, t in vol.attr.items():
                    vol.attr[k] = torch.cat([t, torch.zeros(len(new) * VOX, t.shape[1])])

            def find(self, keys):
                index = {int(k): i for i, k in enumerate(vol.keys)}
                return np.array([index[int(k)] for k in keys], np.int64), None
        return H()

    def voxel_coordinates_and_flattened_indices(self, buf_indices):
        coords = otb.voxel_world(otb.unpack(self.keys[buf_indices]), self.vs).reshape(-1, 3)
        flat = (buf_indices[:, None] * VOX + np.arange(VOX)[None]).reshape(-1)
        return mgt.T(torch.from_numpy(coords)), mgt.T(torch.from_numpy(flat))

    def attribute(self, name):
        return mgt.T(self.attr[name])


def scenario(seed=5, H=24, W=32, frames=3):
    """camera near the world origin looking down +z: with 0.12 m voxels (1.92 m blocks) and depths of 0.6-2.2 m the touched
    blocks straddle 0 on every axis"""
    rng = np.random.default_rng(seed)
    vs = np.float32(0.12)
    idepths = rng.uniform(1 / 2.2, 1 / 0.6, (frames, H, W)).astype(np.float32)
    covs = rng.uniform(0.004, 0.6, (frames, H, W)).astype(np.float32)
    covs[:, :3] = 4e8                                    # masked in "sigma"
    imgs = rng.integers(0, 255, (frames, 3, H, W), dtype=np.uint8)
    q = rng.normal(size=(frames, 4)) * 0.08 + np.array([0, 0, 0, 1.0]); q /= np.linalg.norm(q, axis=1, keepdims=True)
    poses = np.concatenate([rng.uniform(-0.3, 0.3, (frames, 3)), q], 1).astype(np.float32)
    intr = np.array([[W * 0.55, 0, W / 2 - 0.5], [0, W * 0.55, H / 2 - 0.5], [0, 0, 1]], np.float64)
    return dict(voxel_size=vs, idepths=idepths, covs=covs, imgs=imgs, poses=poses, intr=intr)


def run_reference(sc, mask_type):
    Ref = mgt.reference_class()
    self = Ref.__new__(Ref)
    self.device, self.o3d_device = "cpu", "cpu"
    self.depth_scale, self.max_depth, self.sdf_trunc, self.max_weight = 1.0, 6.0, 0.10, 20.0
    self.max_depth_sigma_thresh, self.use_old_volume, self.depth_mask_type = 10000, False, mask_type
    self.volume = BlockVolume(sc["voxel_size"])
    out = []
    for k in range(len(sc["poses"])):
        packet = {"cam0_poses": torch.from_numpy(sc["poses"][k:k + 1]), "cam0_idepths_up": torch.from_numpy(sc["idepths"][k:k + 1]),
                  "cam0_depths_cov_up": torch.from_numpy(sc["covs"][k:k + 1].copy()), "cam0_images": torch.from_numpy(sc["imgs"][k:k + 1])}
        if mask_type == "uniform":
            packet["cam0_depths_cov_up"] = torch.ones_like(packet["cam0_depths_cov_up"])
        self.build_volume(packet, types.SimpleNamespace(intrinsic_matrix=sc["intr"]), self.get_depth_masks(packet))
        B = len(self.volume.keys)
        out.append({"touched": self.volume.touched[-1], "keys": self.volume.keys.copy(),
                    "tsdf": self.volume.attr["tsdf"].numpy().reshape(B, 16, 16, 16).copy(),
                    "weight": self.volume.attr["weight"].numpy().reshape(B, 16, 16, 16).copy(),
                    "color": self.volume.attr["color"].numpy().reshape(B, 16, 16, 16, 3).copy()})
    return out


def main():
    sc = scenario()
    out = dict(sc)
    for mask_type, tag in (("uncertainty", "sigma"), ("uniform", "tsdf")):
        for k, s in enumerate(run_reference(sc, mask_type)):
            for name, v in s.items():
                out[f"{tag}_{name}_{k}"] = v
        print(tag, "blocks", otb.unpack(out[f"{tag}_keys_2"]).tolist())
    path = os.path.join(HERE, "ref_tsdf_blocks.npz")
    np.savez_compressed(path, **out)
    print("wrote ref_tsdf_blocks.npz", os.path.getsize(path) // 1024, "KB")


if __name__ == "__main__":
    main()
