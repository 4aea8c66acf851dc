"""VoxelBlockVolume — the sparse voxel-block TSDF volume (csrc/tsdf_blocks.cu; rules at the head of that file).

Unbounded Sigma / TSDF fusion in 16^3 blocks allocated where the depth maps reach, as the reference's Open3D
VoxelBlockGrid (fusion/tsdf_fusion.py:64-86, block_resolution 16, block_count 5000).  Per keyframe only the voxels of
the blocks that the keyframe touches are updated (the reference's activate -> find -> update, :231-296), so this volume
and the dense grid of tsdf_fusion.py update different voxel sets; TsdfFusion selects one with `tsdf_volume`.

The pool (tsdf, weight, colour: 80 KB per block) starts at `block_count` blocks and doubles when a keyframe's new
blocks do not fit; every block keeps its pool index, and new blocks are appended in ascending key order, so the pool is
the same on every run.  Each keyframe costs one small host read (the numbers of touched and new blocks), which sizes
the growth and the launch.  Read-outs equal the dense read-outs of the volume's dense embedding (`to_dense`).
tsdf_fusion.DenseVolume, the dense grid, has the same surface."""
from functools import partial

import numpy as np
import torch

from . import _lib

BLOCK = 16


def _pow2_at_least(n):
    return 1 << max(1, int(n - 1).bit_length())


def raycast_outputs(n, H, W, device, normals, depth=None, color=None, weight=None):
    """depth [n,H,W], colour [n,H,W,3], weight [n,H,W] and normal [n,H,W,3] (None without `normals`): the caller's
    tensors where given (the kernels write them through raw pointers, hence the check), else new ones"""
    def out(t, *ch):
        if t is not None and (t.shape != (n, H, W, *ch) or t.dtype != torch.float32 or not t.is_contiguous()):
            raise ValueError(f"ray-cast output {tuple(t.shape)} {t.dtype}: wants a contiguous fp32 {(n, H, W, *ch)}")
        return torch.empty(n, H, W, *ch, dtype=torch.float32, device=device) if t is None else t
    return out(depth), out(color, 3), out(weight), out(None, 3) if normals else None


class _CudaKernels:
    """the sm_90a entry points the volume drives, one method per pass"""

    def activate(self, vol, f):
        """-> (pool indices of the touched blocks in ascending key order, new block keys ascending), device tensors"""
        lib = _lib.load()
        H, W = f["idepth"].shape
        n = 4 * H * W
        if vol._act is None or vol._act[0] != (H, W):
            dev = vol.device
            vol._act = ((H, W), torch.empty(_lib.query_size("nslam_tsdf_blocks_scratch", H, W), dtype=torch.uint8, device=dev),
                        torch.empty(n, dtype=torch.int32, device=dev), torch.empty(n, dtype=torch.int64, device=dev),
                        torch.empty(2, dtype=torch.int32, device=dev), torch.empty(2, dtype=torch.int32).pin_memory())
        _, scratch, touched, new_keys, counts_dev, counts_host = vol._act
        _lib.check(lib.nslam_tsdf_blocks_activate(
            _lib.ptr(f["idepth"]), _lib.ptr(f["cov"]), H, W, f["intr"].ctypes.data, _lib.ptr(f["pose"]), float(vol.voxel_size),
            float(f["max_depth"]), float(f["max_depth_sigma"]), _lib.ptr(vol._hkeys), _lib.ptr(vol._hvals), vol._hkeys.numel(),
            vol.n_blocks, _lib.ptr(scratch), scratch.numel(), _lib.ptr(touched), _lib.ptr(new_keys), _lib.ptr(counts_dev),
            _lib.ptr(counts_host), _lib.stream_ptr()), "tsdf_blocks_activate")
        n_touched, n_new = (int(v) for v in counts_host)
        return touched[:n_touched], new_keys[:n_new]

    def insert(self, vol, new_keys):
        _lib.check(_lib.load().nslam_tsdf_blocks_insert(
            _lib.ptr(new_keys), new_keys.numel(), vol.n_blocks, _lib.ptr(vol._keys), _lib.ptr(vol._coords), _lib.ptr(vol.tsdf),
            _lib.ptr(vol.weight), _lib.ptr(vol.color), _lib.ptr(vol._hkeys), _lib.ptr(vol._hvals), vol._hkeys.numel(),
            _lib.stream_ptr()), "tsdf_blocks_insert")

    def rehash(self, vol):
        vol._hkeys.fill_(-1)
        _lib.check(_lib.load().nslam_tsdf_blocks_rehash(_lib.ptr(vol._keys), vol.n_blocks, _lib.ptr(vol._hkeys),
                                                        _lib.ptr(vol._hvals), vol._hkeys.numel(), _lib.stream_ptr()),
                   "tsdf_blocks_rehash")

    def integrate(self, vol, touched, f):
        _lib.check(_lib.load().nslam_tsdf_blocks_integrate(
            _lib.ptr(vol.tsdf), _lib.ptr(vol.weight), _lib.ptr(vol.color), _lib.ptr(vol._coords), _lib.ptr(touched),
            touched.numel(), float(vol.voxel_size), _lib.ptr(f["idepth"]), _lib.ptr(f["cov"]), _lib.ptr(f["rgb"]),
            f["idepth"].shape[0], f["idepth"].shape[1], f["intr"].ctypes.data, _lib.ptr(f["pose"]), float(f["max_depth"]),
            float(f["sdf_trunc"]), float(f["max_weight"]), float(f["max_depth_sigma"]), _lib.stream_ptr()), "tsdf_blocks_integrate")


class VoxelBlockVolume:
    """tsdf / weight [capacity,16,16,16] fp32 and color [capacity,16,16,16,3] fp32 (u8 scale) on `device`; the first
    `n_blocks` blocks are allocated, block p holds the voxels 16 * block_coords[p] + (x, y, z) at world position
    voxel_size * index, stored [z][y][x]"""

    kernels = _CudaKernels()

    def __init__(self, voxel_size, block_count=5000, device="cuda:0"):
        self.device = device
        self._act = None                                 # activation buffers of the last frame size
        self._alloc(max(1, int(block_count)))
        self.reset(voxel_size)

    def _alloc(self, cap, keep=0):
        dev = self.device
        old = getattr(self, "tsdf", None)
        tsdf = torch.empty(cap, BLOCK, BLOCK, BLOCK, dtype=torch.float32, device=dev)
        weight = torch.empty_like(tsdf)
        color = torch.empty(cap, BLOCK, BLOCK, BLOCK, 3, dtype=torch.float32, device=dev)
        keys = torch.empty(cap, dtype=torch.int64, device=dev)
        coords = torch.empty(cap, 3, dtype=torch.int32, device=dev)
        if old is not None and keep:
            for new, cur in ((tsdf, self.tsdf), (weight, self.weight), (color, self.color), (keys, self._keys),
                             (coords, self._coords)):
                new[:keep].copy_(cur[:keep])
        self.tsdf, self.weight, self.color, self._keys, self._coords = tsdf, weight, color, keys, coords
        # hash table at load <= 1/2 for a full pool
        self._hkeys = torch.full((_pow2_at_least(2 * cap),), -1, dtype=torch.int64, device=dev)
        self._hvals = torch.empty(self._hkeys.numel(), dtype=torch.int32, device=dev)

    def reset(self, voxel_size):
        """empty the volume at a new voxel size; the capacity stays"""
        self.voxel_size = float(np.float32(voxel_size))
        self.n_blocks = 0
        self._hkeys.fill_(-1)

    @property
    def capacity(self):
        return self.tsdf.shape[0]

    @property
    def block_coords(self):
        """[n_blocks,3] int32 block coordinates in pool order"""
        return self._coords[:self.n_blocks]

    def memory_bytes(self):
        """device bytes held by the pool, its keys and the hash table (the activation scratch excluded)"""
        held = [self.tsdf, self.weight, self.color, self._keys, self._coords, self._hkeys, self._hvals]
        return sum(t.numel() * t.element_size() for t in held)

    # ------------------------------------------------------------------ integration
    def integrate(self, idepth_up, depth_cov_up, rgb_chw, intrinsics, cam_T_world_tq, max_depth=6.0, sdf_trunc=0.10,
                  max_weight=20.0, max_depth_sigma=10000.0):
        """one keyframe, arguments as nslam_tsdf_integrate: idepth_up / depth_cov_up (None = uniform weights) [H,W] fp32,
        rgb_chw u8 [3,H,W], cam_T_world_tq [7] device tensors; intrinsics fx, fy, cx, cy.  -> number of touched blocks"""
        f = {"idepth": idepth_up, "cov": depth_cov_up, "rgb": rgb_chw, "pose": cam_T_world_tq,
             "intr": np.ascontiguousarray(np.asarray(intrinsics, np.float32)), "max_depth": max_depth, "sdf_trunc": sdf_trunc,
             "max_weight": max_weight, "max_depth_sigma": max_depth_sigma}
        touched, new_keys = self.kernels.activate(self, f)
        n_new = int(new_keys.shape[0])
        if self.n_blocks + n_new > self.capacity:
            cap = self.capacity
            while self.n_blocks + n_new > cap:
                cap *= 2
            self._alloc(cap, keep=self.n_blocks)
            self.kernels.rehash(self)
        self.kernels.insert(self, new_keys)
        self.n_blocks += n_new
        self.kernels.integrate(self, touched, f)
        return int(touched.shape[0])

    # ------------------------------------------------------------------ read-outs
    def _neighbours(self):
        nbr = torch.empty(max(1, self.n_blocks), 27, dtype=torch.int32, device=self.device)
        _lib.check(_lib.load().nslam_tsdf_blocks_neighbours(_lib.ptr(self._coords), self.n_blocks, _lib.ptr(self._hkeys),
                                                            _lib.ptr(self._hvals), self._hkeys.numel(), _lib.ptr(nbr),
                                                            _lib.stream_ptr()), "tsdf_blocks_neighbours")
        return nbr

    def build_mesh(self, min_weight):
        """marching cubes over the cubes whose 8 corners have weight > min_weight (>= 0) -> TsdfMesh or None.  Vertices by
        (pool index, local voxel, axis)."""
        from .tsdf_fusion import marching_cubes
        lib = _lib.load()
        if not min_weight >= 0:
            raise ValueError("min_weight must be >= 0: voxels outside the blocks have weight 0")
        if self.n_blocks == 0:
            return None
        nbr = self._neighbours()
        head = (_lib.ptr(self.tsdf), _lib.ptr(self.weight))
        blocks = (_lib.ptr(nbr), _lib.ptr(self._coords), self.n_blocks)
        mw = float(min_weight)
        return marching_cubes("tsdf_blocks_mesh", (self.n_blocks,),
                              partial(lib.nslam_tsdf_blocks_mesh_count, *head, *blocks, mw),
                              partial(lib.nslam_tsdf_blocks_mesh_emit, *head, _lib.ptr(self.color), *blocks,
                                      float(self.voxel_size), mw), self.device)

    def raycast(self, cam_T_world_tq, H, W, intrinsics, min_depth, max_depth, sdf_trunc, min_weight, normals=False,
                depth=None, color=None, weight=None):
        """ray-cast the views cam_T_world_tq [n,7] in one launch -> depth [n,H,W] (0 = miss), colour [n,H,W,3] in [0,1],
        weight [n,H,W] and, with `normals`, unit normals [n,H,W,3] (else None).  `depth`, `color` and `weight` may be given
        as outputs."""
        if not min_weight >= 0:
            raise ValueError("min_weight must be >= 0: voxels outside the blocks have weight 0")
        poses = cam_T_world_tq.to(self.device, torch.float32).contiguous()
        n = poses.shape[0]
        out = raycast_outputs(n, H, W, self.device, normals, depth, color, weight)
        intr = np.ascontiguousarray(np.asarray(intrinsics, np.float32))
        with _lib.fixed_stream():
            nbr = self._neighbours()
            _lib.check(_lib.load().nslam_tsdf_blocks_raycast(
                _lib.ptr(self.tsdf), _lib.ptr(self.weight), _lib.ptr(self.color), _lib.ptr(nbr), _lib.ptr(self._hkeys),
                _lib.ptr(self._hvals), self._hkeys.numel(), float(self.voxel_size), _lib.ptr(poses), n, H, W, intr.ctypes.data,
                float(min_depth), float(max_depth), float(sdf_trunc), float(min_weight), *[_lib.ptr(t) for t in out],
                _lib.stream_ptr()), "tsdf_blocks_raycast")
        return out

    def to_dense(self, margin_blocks=1):
        """dense embedding of the volume (0 outside its blocks), for small volumes and export: tsdf, weight [nz,ny,nx],
        color [nz,ny,nx,3] device tensors over the blocks' bounding box grown by `margin_blocks`, and the fp32 world
        position of its voxel (0,0,0), voxel_size * 16 * (smallest block - margin)"""
        dev = self.device
        if self.n_blocks == 0:
            z = torch.zeros(0, 0, 0, dtype=torch.float32, device=dev)
            return z, z.clone(), torch.zeros(0, 0, 0, 3, dtype=torch.float32, device=dev), np.zeros(3, np.float32)
        c = self.block_coords.long()
        lo = c.min(0).values - margin_blocks
        nb = (c.max(0).values + margin_blocks + 1 - lo).tolist()
        b = (c - lo).T                                                       # x, y, z
        out = []
        for src, ch in ((self.tsdf, ()), (self.weight, ()), (self.color, (3,))):
            d = torch.zeros(nb[2], nb[1], nb[0], BLOCK, BLOCK, BLOCK, *ch, dtype=torch.float32, device=dev)
            d[b[2], b[1], b[0]] = src[:self.n_blocks]
            perm = (0, 3, 1, 4, 2, 5) + ((6,) if ch else ())
            out.append(d.permute(*perm).reshape(BLOCK * nb[2], BLOCK * nb[1], BLOCK * nb[0], *ch).contiguous())
        origin = (np.float32(self.voxel_size) * (BLOCK * lo.cpu().numpy()).astype(np.float32)).astype(np.float32)
        return out[0], out[1], out[2], origin
