"""TsdfFusion — the reference's fusion/tsdf_fusion.py (`--fusion=tsdf` / `--fusion=sigma`, SURVEY.md §8 f3) on a dense
sm_90a voxel grid.

Same surface: TsdfFusion(name, args, device)  .fuse(data_packets)  .stop_condition()
              .handle_slam_packet / .update_history / .get_history_packet / .get_depth_masks / .build_volume /
              .rebuild_volume / .reset_volume        (the Open3D GUI / mesh / ray-cast rendering paths are out of scope)
name "tsdf": uniform weights; "sigma": weights 1 / sqrt(depth variance) from the SLAM packet's covariances
(Rosinol22wacv; tsdf_fusion.py:46-49,196).

Differences by design: Open3D's hashed VoxelBlockGrid driven from Python (~40 tensor ops and four device
synchronisations per keyframe, :185-302) becomes one kernel launch per keyframe on a DENSE grid (csrc/tsdf.cu) —
the reference's own extent "6 m / 512 voxels" is 2.7 GB at 20 B per voxel on an 80 GB part; poses, depths, weights and
masks are consumed where the SLAM packet holds them (device tensors; the reference converts each frame to three Open3D
images and copies the poses to the host)."""
import numpy as np
import torch

from . import _lib


class TsdfFusion:
    def __init__(self, name, args, device="cuda:0"):
        self.name, self.args, self.device = name, args, device
        self.dsf = 8.0                                   # :32
        self.depth_scale = 1.0
        self.min_depth, self.max_depth = 0.01, 6.0       # :35-36
        self.evaluate = bool(getattr(args, "eval", False))
        self.history = {}
        self.intrinsics = None                           # fx, fy, cx, cy at full resolution (o3d_intrinsics, :133-137)
        self.max_depth_sigma_thresh = 10000.0            # :44
        self.min_weight_for_render = 0.01
        self.depth_mask_type = "uncertainty" if name == "sigma" else "uniform"     # :46-49
        self.max_weight = 20.0                           # :62
        self.voxel_size = 6.0 / 512                      # :64
        self.sdf_trunc = 0.10                            # :68
        # dense grid: `grid_resolution` voxels of `voxel_size` centred on `grid_center` (reference: unbounded hashed blocks,
        # 5000 x 16^3 voxels of capacity; the default here covers its "6 m room")
        self.grid_resolution = int(getattr(args, "tsdf_resolution", 512))
        self.grid_center = np.asarray(getattr(args, "tsdf_center", (0.0, 0.0, 0.0)), np.float32)
        self.integrated_frames = 0
        self.initialize()

    def initialize(self):
        n = self.grid_resolution
        dev = self.device
        self.tsdf = torch.zeros(n, n, n, dtype=torch.float32, device=dev)
        self.weight = torch.zeros(n, n, n, dtype=torch.float32, device=dev)
        self.color = torch.zeros(n, n, n, 3, dtype=torch.float32, device=dev)
        # voxel (i, j, k) sits at origin + voxel_size * (i, j, k) with the lattice passing through the world origin, like the
        # metric voxel coordinates Open3D's VoxelBlockGrid hands out (integer index x voxel_size): same sample points as the
        # reference wherever both volumes have a voxel
        vs = np.float32(self.voxel_size)
        self.origin = ((np.round(self.grid_center / vs) - n // 2) * vs).astype(np.float32)

    def reset_volume(self):
        """:304-316 — NB the reference re-creates its volume with HALF the voxel size here; kept"""
        self.voxel_size = self.voxel_size / 2
        self.initialize()

    # ------------------------------------------------------------------ main loop (:84-98)
    def fuse(self, data_packets):
        gui_output = None
        if data_packets:
            for name, packet in data_packets.items():
                if name == "slam":
                    self.handle_slam_packet(packet)
                elif name == "gui":
                    gui_output = self.handle_gui_packet(packet)
                else:
                    raise NotImplementedError("Unrecognized input packet for TsdfFusion Module")
        return gui_output if gui_output else None

    def stop_condition(self):
        return False                                     # :575-576

    def handle_gui_packet(self, packet):
        """:151-170 without the mesh branch (Open3D): mask type switch, volume rebuild"""
        if not packet:
            return None
        self.depth_mask_type = packet.get("depth_mask_type", self.depth_mask_type)
        if packet.get("build_mesh"):
            raise NotImplementedError("mesh extraction is an Open3D GUI feature (out of the hot-path scope)")
        if packet.get("rebuild_volume"):
            self.rebuild_volume()
        return None

    def handle_slam_packet(self, packet):
        """:100-149"""
        if not packet:
            return True
        packet = packet[1]
        if packet is None:
            return True
        if self.evaluate and packet["is_last_frame"] and "cam0_images" not in packet:
            return True
        if not self.update_history(packet):
            return True
        if self.intrinsics is None:
            self.intrinsics = (self.dsf * packet["cam0_intrinsics"][0].float().cpu().numpy()).astype(np.float32)   # once
        if self.depth_mask_type == "uniform":
            packet = dict(packet)
            packet["cam0_depths_cov_up"] = None          # = torch.ones_like(...) in the reference (:141): weight 1, mask all
        self.build_volume(packet, self.intrinsics, None)
        return False

    # ------------------------------------------------------------------ history (:486-543)
    def update_history(self, packet):
        if packet["is_last_frame"]:
            return False
        ids = packet["viz_idx_host"] if "viz_idx_host" in packet else packet["viz_idx"].tolist()
        k2f = packet["kf_idx_to_f_idx"]
        for i, ix in enumerate(ids):
            h = self.history.setdefault(k2f[int(ix)], {})
            h["kf_idx"] = packet["kf_idx"]
            h["viz_idx"] = packet["viz_idx"][i]
            for key in ("cam0_poses", "cam0_depths_cov_up", "cam0_idepths_up", "cam0_images", "cam0_intrinsics", "gt_depths"):
                h[key] = packet[key][i]
            h["calibs"] = packet["calibs"][0]
        return True

    def get_history_packet(self):
        keys = ("viz_idx", "cam0_poses", "cam0_depths_cov_up", "cam0_idepths_up", "cam0_images", "cam0_intrinsics")
        packet = {k: torch.stack([h[k] for h in self.history.values()]) for k in keys}
        packet["calibs"] = [h["calibs"] for h in self.history.values()]
        packet["gt_depths"] = torch.stack([h["gt_depths"].float() * h["calibs"].depth_scale for h in self.history.values()])
        return packet

    def get_depth_masks(self, packet):
        """:545-554 (evaluated inside the kernel during integration; this is the tensor form for callers)"""
        cov = packet["cam0_depths_cov_up"]
        if self.depth_mask_type == "uncertainty":
            return cov.sqrt() < self.max_depth_sigma_thresh
        if self.depth_mask_type == "uniform":
            return torch.ones_like(cov).to(torch.bool)
        raise NotImplementedError(f"Unknown depth mask type: {self.depth_mask_type}")

    # ------------------------------------------------------------------ integration (:185-302)
    def build_volume(self, packet, intrinsics, masks=None):
        """every keyframe of the packet into the volume: one kernel launch each, no host synchronisation"""
        lib = _lib.load()
        poses = packet["cam0_poses"].to(self.device, torch.float32).contiguous()
        idepths = packet["cam0_idepths_up"].to(self.device, torch.float32).contiguous()
        covs = packet["cam0_depths_cov_up"]
        covs = None if covs is None else covs.to(self.device, torch.float32).contiguous()
        images = packet["cam0_images"].to(self.device).contiguous()
        assert images.dtype == torch.uint8 and images.shape[1] == 3
        n, _, H, W = images.shape
        intr = np.ascontiguousarray(np.asarray(intrinsics, np.float32))
        n3 = self.grid_resolution
        with _lib.fixed_stream():
            for k in range(n):
                _lib.check(lib.nslam_tsdf_integrate(
                    _lib.ptr(self.tsdf), _lib.ptr(self.weight), _lib.ptr(self.color), n3, n3, n3, self.origin.ctypes.data,
                    float(self.voxel_size), _lib.ptr(idepths[k]), _lib.ptr(covs[k]) if covs is not None else None,
                    _lib.ptr(images[k]), H, W, intr.ctypes.data, _lib.ptr(poses[k]), float(self.max_depth), float(self.sdf_trunc),
                    float(self.max_weight), float(self.max_depth_sigma_thresh), _lib.stream_ptr()), "tsdf_integrate")
        self.integrated_frames += n

    def rebuild_volume(self):
        """:172-183"""
        packet = self.get_history_packet()
        self.reset_volume()
        if self.depth_mask_type == "uniform":
            packet["cam0_depths_cov_up"] = None
        self.build_volume(packet, self.intrinsics, None)

    # ------------------------------------------------------------------ read-out
    def surface_points(self, min_weight=0.01, max_points=2_000_000):
        """voxel centres next to a zero crossing of the TSDF along x / y / z with enough weight (a light-weight stand-in
        for the reference's mesh / ray-cast read-outs, which need Open3D) -> [m,3] world points, [m,3] colours"""
        t, w = self.tsdf, self.weight
        ok = w > min_weight
        m = torch.zeros_like(ok)
        for d in range(3):
            a = t.narrow(d, 0, t.shape[d] - 1); b = t.narrow(d, 1, t.shape[d] - 1)
            cross = ((a * b) < 0) & ok.narrow(d, 0, t.shape[d] - 1) & ok.narrow(d, 1, t.shape[d] - 1)
            m.narrow(d, 0, t.shape[d] - 1).logical_or_(cross)
        idx = m.nonzero()[:max_points]
        pts = torch.as_tensor(self.origin, device=t.device) + self.voxel_size * idx[:, [2, 1, 0]].float()
        return pts, self.color[idx[:, 0], idx[:, 1], idx[:, 2]]
