"""TsdfFusion — the reference's fusion/tsdf_fusion.py (`--fusion=tsdf` / `--fusion=sigma`, SURVEY.md §8 f3) on a dense
sm_90a voxel grid.

Same surface: TsdfFusion(name, args, device)  .fuse(data_packets)  .stop_condition()
              .handle_slam_packet / .handle_gui_packet / .update_history / .get_history_packet / .get_depth_masks /
              .build_volume / .rebuild_volume / .reset_volume / .build_mesh / .render_volume / .evaluate_metrics
              .build_point_cloud (the GUI's point clouds; the Open3D GUI itself is out of scope)
name "tsdf": uniform weights; "sigma": weights 1 / sqrt(depth variance) from the SLAM packet's covariances
(Rosinol22wacv; tsdf_fusion.py:46-49,196).

Read-outs (csrc/tsdf_mesh.cu): `build_mesh` is marching cubes over the cubes whose 8 corners are observed, with vertex
colours and TSDF-gradient normals (not the area-weighted face normals of Open3D's compute_vertex_normals, :561,565);
`render_volume` ray-casts depth and colour at every keyframe of a packet and, with `evaluate`, writes the PSNR / depth-L1
row of `results.csv` (:319-484).  One deliberate deviation there: the reference compares its 0-255 colour attribute with
image / 255 (:406, :459-461); here both sides are on [0, 1], as in its own `sum_colors` path (:413-415).

Differences by design: Open3D's hashed VoxelBlockGrid driven from Python (~40 tensor ops and four device
synchronisations per keyframe, :185-302) becomes one kernel launch per keyframe on a DENSE grid (DenseVolume,
csrc/tsdf.cu) — the reference's own extent "6 m / 512 voxels" is 2.7 GB at 20 B per voxel on an 80 GB part; poses,
depths, weights and masks are consumed where the SLAM packet holds them (device tensors; the reference converts each
frame to three Open3D images and copies the poses to the host).

TsdfFusion holds one `volume`: a DenseVolume, or with `args.tsdf_volume = "blocks"` (default "dense") the sparse
voxel-block volume of tsdf_blocks.py: unbounded, 16^3 blocks allocated where the depth maps reach (`args.tsdf_block_count`
to start with, default 5000, the reference's block_count), only the voxels of the blocks a keyframe touches updated, as in
the reference — so the two volumes update different voxel sets, and the choice is the user's.  Both have the same surface
(reset, integrate, build_mesh, raycast, memory_bytes, to_dense), so integration, the history rebuild, the reset, both
read-outs, the GUI packets and `--eval` work on either; `surface_points` is dense-only."""
import csv
from functools import partial

import numpy as np
import torch

from . import _lib
from .point_cloud import build_point_cloud as _build_point_cloud, write_binary_ply
from .tsdf_blocks import VoxelBlockVolume, raycast_outputs


class TsdfMesh:
    """triangle mesh read out of the volume, device tensors: vertices [V,3] (world, metres), triangles [T,3] int32 wound so
    that (b - a) x (c - a) points into free space, vertex_colors [V,3] in [0,1], vertex_normals [V,3] (unit, toward free
    space)"""

    def __init__(self, vertices, triangles, vertex_colors, vertex_normals):
        self.vertices, self.triangles = vertices, triangles
        self.vertex_colors, self.vertex_normals = vertex_colors, vertex_normals

    def write_ply(self, path):
        """binary little-endian PLY: float x y z nx ny nz red green blue (colours in [0,1]), int32 vertex indices"""
        arrays = [(("x", "y", "z"), self.vertices), (("nx", "ny", "nz"), self.vertex_normals),
                  (("red", "green", "blue"), self.vertex_colors)]
        cols = []
        for names, t in arrays:
            a = t.detach().float().cpu().numpy()
            cols += [(k, a[:, i]) for i, k in enumerate(names)]
        write_binary_ply(path, cols, self.triangles.detach().cpu().numpy())


def marching_cubes(name, plan_args, count, emit, device):
    """the host side of both marching-cubes read-outs: `plan_args` are the arguments of nslam_<name>_plan, `count` and
    `emit` are nslam_<name>_count / _emit with the volume's leading arguments bound.  The count passes leave the vertex, triangle and active-voxel totals at the
    head of the scratch; their one host read sizes the outputs of the emit passes -> TsdfMesh of device tensors, or None
    when there is no triangle."""
    scratch = torch.empty(_lib.query_size(f"nslam_{name}_plan", *plan_args), dtype=torch.int32, device=device)
    with _lib.fixed_stream():
        _lib.check(count(_lib.ptr(scratch), _lib.stream_ptr()), name + "_count")
        n_vert, n_tri, n_active = scratch[:3].tolist()
        if n_tri == 0:
            return None
        active = torch.empty(n_active, 4, dtype=torch.int32, device=device)
        verts, cols, nrms = (torch.empty(n_vert, 3, dtype=torch.float32, device=device) for _ in range(3))
        tris = torch.empty(n_tri, 3, dtype=torch.int32, device=device)
        _lib.check(emit(_lib.ptr(scratch), n_active, _lib.ptr(active), _lib.ptr(verts), _lib.ptr(cols), _lib.ptr(nrms),
                        _lib.ptr(tris), _lib.stream_ptr()), name + "_emit")
    return TsdfMesh(verts, tris, cols, nrms)


def mesh_dense(tsdf, weight, color, origin, voxel_size, min_weight):
    """marching cubes (csrc/tsdf_mesh.cu) over a dense [nz,ny,nx] volume whose voxel (i,j,k) sits at origin + voxel_size *
    (i,j,k), over the cubes whose 8 corners have weight > min_weight -> TsdfMesh of device tensors, or None when there is
    no triangle.  `color` [nz,ny,nx,3] on the u8 scale, or None for a volume without colours (vertex colours 0).  One host
    read of the three counts sizes the outputs."""
    lib = _lib.load()
    nz, ny, nx = tsdf.shape
    org = np.ascontiguousarray(np.asarray(origin, np.float32))
    mw = float(min_weight)
    return marching_cubes(
        "tsdf_mesh", (nx, ny, nz),
        partial(lib.nslam_tsdf_mesh_count, _lib.ptr(tsdf), _lib.ptr(weight), nx, ny, nz, mw),
        partial(lib.nslam_tsdf_mesh_emit, _lib.ptr(tsdf), _lib.ptr(weight), _lib.ptr(color), nx, ny, nz, org.ctypes.data,
                float(voxel_size), mw), tsdf.device)


class DenseVolume:
    """the dense grid, tsdf / weight [nz,ny,nx] fp32 and color [nz,ny,nx,3] fp32 (u8 scale) on `device` with voxel (i,j,k)
    at origin + voxel_size * (i,j,k); the surface of tsdf_blocks.VoxelBlockVolume.  Built as resolution^3 about `center`."""

    def __init__(self, resolution, center, voxel_size, device="cuda:0"):
        n = int(resolution)
        self.device, self.center = device, np.asarray(center, np.float32)
        self.tsdf = torch.empty(n, n, n, dtype=torch.float32, device=device)
        self.weight = torch.empty_like(self.tsdf)
        self.color = torch.empty(n, n, n, 3, dtype=torch.float32, device=device)
        self.reset(voxel_size)

    @classmethod
    def from_tensors(cls, tsdf, weight, color, origin, voxel_size):
        """a volume over existing tensors of any [nz,ny,nx]; without a centre it has no `reset`"""
        vol = cls.__new__(cls)
        vol.device, vol.tsdf, vol.weight, vol.color = tsdf.device, tsdf, weight, color
        vol.origin, vol.voxel_size = np.asarray(origin, np.float32), float(np.float32(voxel_size))
        return vol

    def reset(self, voxel_size):
        """empty the grid in place at a new voxel size.  Voxel (i,j,k) sits at origin + voxel_size * (i,j,k) with the lattice
        passing through the world origin, like the metric voxel coordinates Open3D's VoxelBlockGrid hands out (integer index
        x voxel_size): same sample points as the reference wherever both volumes have a voxel"""
        for t in (self.tsdf, self.weight, self.color):
            t.zero_()
        vs = np.float32(voxel_size)
        self.voxel_size = float(vs)
        self.origin = ((np.round(self.center / vs) - self.tsdf.shape[0] // 2) * vs).astype(np.float32)

    def memory_bytes(self):
        return sum(t.numel() * t.element_size() for t in (self.tsdf, self.weight, self.color))

    def integrate(self, idepth_up, depth_cov_up, rgb_chw, intrinsics, cam_T_world_tq, max_depth=6.0, sdf_trunc=0.10,
                  max_weight=20.0, max_depth_sigma=10000.0):
        """one keyframe, arguments as VoxelBlockVolume.integrate: one nslam_tsdf_integrate launch over the grid"""
        nz, ny, nx = self.tsdf.shape
        H, W = rgb_chw.shape[-2:]
        intr = np.ascontiguousarray(np.asarray(intrinsics, np.float32))
        _lib.check(_lib.load().nslam_tsdf_integrate(
            _lib.ptr(self.tsdf), _lib.ptr(self.weight), _lib.ptr(self.color), nx, ny, nz, self.origin.ctypes.data,
            self.voxel_size, _lib.ptr(idepth_up), _lib.ptr(depth_cov_up), _lib.ptr(rgb_chw), H, W, intr.ctypes.data,
            _lib.ptr(cam_T_world_tq), float(max_depth), float(sdf_trunc), float(max_weight), float(max_depth_sigma),
            _lib.stream_ptr()), "tsdf_integrate")

    def build_mesh(self, min_weight):
        """marching cubes over the cubes whose 8 corners have weight > min_weight -> TsdfMesh or None (mesh_dense)"""
        return mesh_dense(self.tsdf, self.weight, self.color, self.origin, self.voxel_size, min_weight)

    def raycast(self, cam_T_world_tq, H, W, intrinsics, min_depth, max_depth, sdf_trunc, min_weight, normals=False,
                depth=None, color=None, weight=None):
        """as VoxelBlockVolume.raycast: the views cam_T_world_tq [n,7] in one launch -> depth, colour, weight, normal"""
        poses = cam_T_world_tq.to(self.device, torch.float32).contiguous()
        n = poses.shape[0]
        out = raycast_outputs(n, H, W, self.device, normals, depth, color, weight)
        intr = np.ascontiguousarray(np.asarray(intrinsics, np.float32))
        nz, ny, nx = self.tsdf.shape
        _lib.check(_lib.load().nslam_tsdf_raycast(
            _lib.ptr(self.tsdf), _lib.ptr(self.weight), _lib.ptr(self.color), nx, ny, nz, self.origin.ctypes.data,
            self.voxel_size, _lib.ptr(poses), n, H, W, intr.ctypes.data, float(min_depth), float(max_depth),
            float(sdf_trunc), float(min_weight), *[_lib.ptr(t) for t in out], _lib.stream_ptr()), "tsdf_raycast")
        return out

    def to_dense(self):
        """tsdf, weight, color and origin: the grid itself"""
        return self.tsdf, self.weight, self.color, self.origin


def depth_l1_cm(rendered_depth, gt_depth):
    """depth error of one view (:466-474): the last 8 rows and columns dropped, the rendering scaled by the ratio of the
    means, |error| clamped at 2.0, mean x 100 (cm)"""
    r = rendered_depth[:-8, :-8]
    g = gt_depth[:-8, :-8].to(r)
    diff = torch.abs(g.mean() / r.mean() * r - g)
    diff[diff > 2.0] = 2.0
    return diff.mean().cpu().numpy() * 100


def color_psnr(rendered_color, image_chw_u8):
    """PSNR of one view (:458-462) with both sides on [0, 1]: rendered [H,W,3] against the u8 image [3,H,W] / 255"""
    from .nerf_fusion import compute_error, mse2psnr
    ref = image_chw_u8.permute(1, 2, 0).float() / 255.0
    return mse2psnr(compute_error(rendered_color.cpu().numpy(), ref.cpu().numpy()))


class TsdfFusion:
    def __init__(self, name, args, device="cuda:0"):
        self.name, self.args, self.device = name, args, device
        self.dsf = 8.0                                   # :32
        self.depth_scale = 1.0
        self.min_depth, self.max_depth = 0.01, 6.0       # :35-36
        self.evaluate = bool(getattr(args, "eval", False))
        self.do_render_volume = False                    # :47
        self.render_views_per_launch = 8                 # render_volume's chunk of views (bounds its scratch)
        self.history = {}
        self.intrinsics = None                           # fx, fy, cx, cy at full resolution (o3d_intrinsics, :133-137)
        self.max_depth_sigma_thresh = 10000.0            # :44
        self.min_weight_for_render = 0.01
        self.depth_mask_type = "uncertainty" if name == "sigma" else "uniform"     # :46-49
        self.max_weight = 20.0                           # :62
        self.voxel_size = 6.0 / 512                      # :64
        self.sdf_trunc = 0.10                            # :68
        kind = getattr(args, "tsdf_volume", "dense")
        if kind == "dense":
            # `tsdf_resolution`^3 voxels centred on `tsdf_center` (reference: unbounded hashed blocks, 5000 x 16^3 voxels of
            # capacity; the default here covers its "6 m room")
            self.volume = DenseVolume(int(getattr(args, "tsdf_resolution", 512)), getattr(args, "tsdf_center", (0.0, 0.0, 0.0)),
                                      self.voxel_size, device)
        elif kind == "blocks":
            self.volume = VoxelBlockVolume(self.voxel_size, int(getattr(args, "tsdf_block_count", 5000)), device)
        else:
            raise ValueError(f"tsdf_volume must be 'dense' or 'blocks', not {kind!r}")
        self.integrated_frames = 0

    def initialize(self):
        """empty the volume at the current voxel size, in place (the block volume keeps its capacity)"""
        self.volume.reset(self.voxel_size)

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
        """:149-169: mask type switch, mesh (-> {"mesh": TsdfMesh}), volume rebuild, evaluation"""
        if not packet:
            return None
        output = None
        self.depth_mask_type = packet.get("depth_mask_type", self.depth_mask_type)
        if packet.get("build_mesh"):
            mesh = self.build_mesh(packet["build_mesh"]["min_weight_for_mesh"])
            if mesh is not None:
                output = {"mesh": mesh}
            else:
                print("Could not build a mesh...")
        pcl_opts = packet.get("build_pcl")
        if pcl_opts is not None and pcl_opts is not False:
            # {"build_pcl": {}} or True; options: voxel_size, filter_thresh, min_views
            pcl = self.build_point_cloud(**(pcl_opts if isinstance(pcl_opts, dict) else {}))
            if pcl is not None:
                output = dict(output or {}, pcl=pcl)
            else:
                print("Could not build a point cloud...")
        if packet.get("rebuild_volume"):
            self.rebuild_volume()
        if packet.get("eval_metrics"):
            self.evaluate_metrics()
        return output

    def handle_slam_packet(self, packet):
        """:100-149"""
        if not packet:
            return True
        packet = packet[1]
        if packet is None:
            return True
        if self.evaluate and packet["is_last_frame"] and "cam0_images" not in packet:
            if self.history:
                self.evaluate_metrics()
            else:
                print("Can't evaluate volume since there is no history!")
            return True
        if not self.update_history(packet):
            return True
        if self.intrinsics is None:
            self.intrinsics = (self.dsf * packet["cam0_intrinsics"][0].float().cpu().numpy()).astype(np.float32)   # once
        if self.depth_mask_type == "uniform":
            packet = dict(packet)
            packet["cam0_depths_cov_up"] = None          # = torch.ones_like(...) in the reference (:141): weight 1, mask all
        self.build_volume(packet, self.intrinsics, None)
        if self.do_render_volume:
            self.render_volume(packet, self.intrinsics, self.min_weight_for_render, self.max_depth_sigma_thresh)
        if self.evaluate and packet["is_last_frame"]:
            self.evaluate_metrics()
        return False

    def evaluate_metrics(self):
        """:171-182: render every keyframe of the history and write results.csv"""
        self.render_volume(self.get_history_packet(), self.intrinsics, self.min_weight_for_render,
                           self.max_depth_sigma_thresh, evaluate=True)

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
        """every keyframe of the packet into the volume: one kernel launch each and no host synchronisation on the dense
        grid; activation, insertion and integration with one host read each on the block volume"""
        poses = packet["cam0_poses"].to(self.device, torch.float32).contiguous()
        idepths = packet["cam0_idepths_up"].to(self.device, torch.float32).contiguous()
        covs = packet["cam0_depths_cov_up"]
        covs = None if covs is None else covs.to(self.device, torch.float32).contiguous()
        images = packet["cam0_images"].to(self.device).contiguous()
        assert images.dtype == torch.uint8 and images.shape[1] == 3
        intr = np.ascontiguousarray(np.asarray(intrinsics, np.float32))
        for k in range(images.shape[0]):
            self.volume.integrate(idepths[k], covs[k] if covs is not None else None, images[k], intr, poses[k],
                                  self.max_depth, self.sdf_trunc, self.max_weight, self.max_depth_sigma_thresh)
        self.integrated_frames += images.shape[0]

    def rebuild_volume(self):
        """:172-183"""
        packet = self.get_history_packet()
        self.reset_volume()
        if self.depth_mask_type == "uniform":
            packet["cam0_depths_cov_up"] = None
        self.build_volume(packet, self.intrinsics, None)

    # ------------------------------------------------------------------ read-out
    def surface_points(self, min_weight=0.01, max_points=2_000_000):
        """voxel centres next to a zero crossing of the TSDF along x / y / z with enough weight (a quick look at the
        surface in plain torch; build_mesh is the full read-out) -> [m,3] world points, [m,3] colours.  Dense grid only."""
        vol = self.volume
        if not isinstance(vol, DenseVolume):
            raise NotImplementedError("surface_points reads the dense grid; use build_mesh with tsdf_volume='blocks'")
        t, w = vol.tsdf, vol.weight
        ok = w > min_weight
        m = torch.zeros_like(ok)
        for d in range(3):
            a = t.narrow(d, 0, t.shape[d] - 1); b = t.narrow(d, 1, t.shape[d] - 1)
            cross = ((a * b) < 0) & ok.narrow(d, 0, t.shape[d] - 1) & ok.narrow(d, 1, t.shape[d] - 1)
            m.narrow(d, 0, t.shape[d] - 1).logical_or_(cross)
        idx = m.nonzero()[:max_points]
        pts = torch.as_tensor(vol.origin, device=t.device) + vol.voxel_size * idx[:, [2, 1, 0]].float()
        return pts, vol.color[idx[:, 0], idx[:, 1], idx[:, 2]]

    def build_mesh(self, min_weight_for_mesh):
        """:556-573: marching cubes over the cubes whose 8 corners have weight > min_weight_for_mesh -> TsdfMesh, or None
        when there is no triangle.  One host read of the three counts sizes the outputs."""
        return self.volume.build_mesh(min_weight_for_mesh)

    def build_point_cloud(self, voxel_size=None, filter_thresh=None, min_views=2):
        """the GUI's build_pcls(None), "rebuild from history" (gui/open3d_gui.py:646-678): every keyframe of the history
        as one coloured point cloud (point_cloud.build_point_cloud) with this fusion's depth_mask_type,
        max_depth_sigma_thresh, max_depth and intrinsics -> PointCloud, or None when there is no history or no point.
        Reads the history, not the volume, so it works for both tsdf_volume modes."""
        if not self.history:
            return None
        packet = self.get_history_packet()
        if self.depth_mask_type == "uniform":
            packet["cam0_depths_cov_up"] = None
        elif self.depth_mask_type != "uncertainty":
            raise NotImplementedError(f"Unknown depth mask type: {self.depth_mask_type}")
        dev = packet["cam0_idepths_up"].device
        for k in ("cam0_poses", "cam0_idepths_up", "cam0_depths_cov_up"):
            if packet[k] is not None:
                packet[k] = packet[k].to(dev, torch.float32).contiguous()
        return _build_point_cloud(packet, self.intrinsics, max_depth=self.max_depth,
                                  max_depth_sigma=self.max_depth_sigma_thresh, filter_thresh=filter_thresh,
                                  min_views=min_views, voxel_size=voxel_size)

    def render_volume(self, packet, intrinsics, min_weight_for_render, max_depth_sigma_thresh, evaluate=False):
        """:319-484: ray-cast depth and colour at every keyframe of the packet -> (depth [n,H,W], colour [n,H,W,3] in [0,1]);
        0 where a ray misses.  Views go `render_views_per_launch` per launch.  With `evaluate`, the mean PSNR and depth L1
        over the views go to results.csv in the working directory as pandas' DataFrame.to_csv writes the reference's row.
        `max_depth_sigma_thresh` only feeds the reference's debug views; it is accepted for the same call."""
        if not packet:
            print("Error: asked to render volume, but packet is None.")
            return None
        dev = self.volume.device
        poses = packet["cam0_poses"].to(dev, torch.float32).contiguous()
        images = packet["cam0_images"]
        n, (H, W) = poses.shape[0], images.shape[-2:]
        intr = np.ascontiguousarray(np.asarray(intrinsics, np.float32))
        depth = torch.empty(n, H, W, dtype=torch.float32, device=dev)
        color = torch.empty(n, H, W, 3, dtype=torch.float32, device=dev)
        chunk = max(1, int(self.render_views_per_launch))
        weight = torch.empty(min(n, chunk), H, W, dtype=torch.float32, device=dev)
        total_psnr, total_l1 = 0.0, np.float32(0)
        with _lib.fixed_stream():
            for s in range(0, n, chunk):
                m = min(chunk, n - s)
                self.volume.raycast(poses[s:s + m], H, W, intr, self.min_depth, self.max_depth, self.sdf_trunc,
                                    min_weight_for_render, depth=depth[s:s + m], color=color[s:s + m], weight=weight[:m])
                if evaluate:
                    for i in range(s, s + m):
                        total_psnr += color_psnr(color[i], images[i])
                        total_l1 += depth_l1_cm(depth[i], packet["gt_depths"][i].squeeze())
        if evaluate:
            dt = 0
            psnr, l1 = total_psnr / (n or 1), total_l1 / (n or 1)
            print(f"Dt={dt}; PSNR={psnr}; L1={l1}")
            with open("results.csv", "w", newline="") as f:
                w = csv.writer(f, lineterminator="\n")
                w.writerow(["", "Dt", "PSNR", "L1"])
                w.writerow([0, repr(float(dt)), repr(float(psnr)), repr(float(l1))])
        return depth, color
