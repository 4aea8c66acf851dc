"""TsdfFusion — the reference's fusion/tsdf_fusion.py (`--fusion=tsdf` / `--fusion=sigma`, SURVEY.md §8 f3) on a dense
sm_90a voxel grid.

Same surface: TsdfFusion(name, args, device)  .fuse(data_packets)  .stop_condition()
              .handle_slam_packet / .handle_gui_packet / .update_history / .get_history_packet / .get_depth_masks /
              .build_volume / .rebuild_volume / .reset_volume / .build_mesh / .render_volume / .evaluate_metrics
              (the Open3D GUI itself is out of scope)
name "tsdf": uniform weights; "sigma": weights 1 / sqrt(depth variance) from the SLAM packet's covariances
(Rosinol22wacv; tsdf_fusion.py:46-49,196).

Read-outs (csrc/tsdf_mesh.cu): `build_mesh` is marching cubes over the cubes whose 8 corners are observed, with vertex
colours and TSDF-gradient normals (not the area-weighted face normals of Open3D's compute_vertex_normals, :561,565);
`render_volume` ray-casts depth and colour at every keyframe of a packet and, with `evaluate`, writes the PSNR / depth-L1
row of `results.csv` (:319-484).  One deliberate deviation there: the reference compares its 0-255 colour attribute with
image / 255 (:406, :459-461); here both sides are on [0, 1], as in its own `sum_colors` path (:413-415).

Differences by design: Open3D's hashed VoxelBlockGrid driven from Python (~40 tensor ops and four device
synchronisations per keyframe, :185-302) becomes one kernel launch per keyframe on a DENSE grid (csrc/tsdf.cu) —
the reference's own extent "6 m / 512 voxels" is 2.7 GB at 20 B per voxel on an 80 GB part; poses, depths, weights and
masks are consumed where the SLAM packet holds them (device tensors; the reference converts each frame to three Open3D
images and copies the poses to the host).

`args.tsdf_volume = "blocks"` (default "dense") selects the sparse voxel-block volume of tsdf_blocks.py instead: unbounded,
16^3 blocks allocated where the depth maps reach (`args.tsdf_block_count` to start with, default 5000, the reference's
block_count), only the voxels of the blocks a keyframe touches updated, as in the reference — so the two volumes update
different voxel sets, and the choice is the user's.  Integration, the history rebuild, the reset, both read-outs, the
GUI packets and `--eval` work on either; `surface_points` is dense-only."""
import csv

import numpy as np
import torch

from . import _lib
from .tsdf_blocks import VoxelBlockVolume


class TsdfMesh:
    """triangle mesh read out of the volume, device tensors: vertices [V,3] (world, metres), triangles [T,3] int32 wound so
    that (b - a) x (c - a) points into free space, vertex_colors [V,3] in [0,1], vertex_normals [V,3] (unit, toward free
    space)"""

    def __init__(self, vertices, triangles, vertex_colors, vertex_normals):
        self.vertices, self.triangles = vertices, triangles
        self.vertex_colors, self.vertex_normals = vertex_colors, vertex_normals

    def write_ply(self, path):
        """binary little-endian PLY: float x y z nx ny nz red green blue (colours in [0,1]), int32 vertex indices"""
        v = self.vertices.detach().float().cpu().numpy()
        vt = np.empty(v.shape[0], [(k, "<f4") for k in ("x", "y", "z", "nx", "ny", "nz", "red", "green", "blue")])
        for k, (src, c) in zip(vt.dtype.names, [(v, 0), (v, 1), (v, 2)] +
                               [(self.vertex_normals.detach().float().cpu().numpy(), c) for c in range(3)] +
                               [(self.vertex_colors.detach().float().cpu().numpy(), c) for c in range(3)]):
            vt[k] = src[:, c]
        t = self.triangles.detach().cpu().numpy().astype("<i4")
        ft = np.empty(t.shape[0], [("n", "u1"), ("v", "<i4", (3,))])
        ft["n"], ft["v"] = 3, t
        head = ["ply", "format binary_little_endian 1.0", f"element vertex {v.shape[0]}"] + \
               [f"property float {k}" for k in vt.dtype.names] + \
               [f"element face {t.shape[0]}", "property list uchar int vertex_indices", "end_header"]
        with open(path, "wb") as f:
            f.write(("\n".join(head) + "\n").encode("ascii"))
            f.write(vt.tobytes())
            f.write(ft.tobytes())


def mesh_dense(tsdf, weight, color, origin, voxel_size, min_weight):
    """marching cubes (csrc/tsdf_mesh.cu) over a dense [nz,ny,nx] volume whose voxel (i,j,k) sits at origin + voxel_size *
    (i,j,k), over the cubes whose 8 corners have weight > min_weight -> TsdfMesh of device tensors, or None when there is
    no triangle.  `color` [nz,ny,nx,3] on the u8 scale, or None for a volume without colours (vertex colours 0).  One host
    read of the three counts sizes the outputs."""
    lib = _lib.load()
    nz, ny, nx = tsdf.shape
    dev = tsdf.device
    org = np.ascontiguousarray(np.asarray(origin, np.float32))
    n_scratch = np.zeros(1, np.int64)
    _lib.check(lib.nslam_tsdf_mesh_plan(nx, ny, nz, n_scratch.ctypes.data), "tsdf_mesh_plan")
    scratch = torch.empty(int(n_scratch[0]), dtype=torch.int32, device=dev)
    mw = float(min_weight)
    with _lib.fixed_stream():
        _lib.check(lib.nslam_tsdf_mesh_count(_lib.ptr(tsdf), _lib.ptr(weight), nx, ny, nz, mw, _lib.ptr(scratch),
                                             _lib.stream_ptr()), "tsdf_mesh_count")
        n_vert, n_tri, n_active = scratch[:3].tolist()
        if n_tri == 0:
            return None
        active = torch.empty(n_active, 4, dtype=torch.int32, device=dev)
        verts = torch.empty(n_vert, 3, dtype=torch.float32, device=dev)
        cols = torch.empty(n_vert, 3, dtype=torch.float32, device=dev)
        nrms = torch.empty(n_vert, 3, dtype=torch.float32, device=dev)
        tris = torch.empty(n_tri, 3, dtype=torch.int32, device=dev)
        _lib.check(lib.nslam_tsdf_mesh_emit(
            _lib.ptr(tsdf), _lib.ptr(weight), _lib.ptr(color), nx, ny, nz, org.ctypes.data, float(voxel_size), mw,
            _lib.ptr(scratch), n_active, _lib.ptr(active), _lib.ptr(verts), _lib.ptr(cols), _lib.ptr(nrms), _lib.ptr(tris),
            _lib.stream_ptr()), "tsdf_mesh_emit")
    return TsdfMesh(verts, tris, cols, nrms)


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
        # dense grid: `grid_resolution` voxels of `voxel_size` centred on `grid_center` (reference: unbounded hashed blocks,
        # 5000 x 16^3 voxels of capacity; the default here covers its "6 m room")
        self.grid_resolution = int(getattr(args, "tsdf_resolution", 512))
        self.grid_center = np.asarray(getattr(args, "tsdf_center", (0.0, 0.0, 0.0)), np.float32)
        self.volume_type = getattr(args, "tsdf_volume", "dense")
        if self.volume_type not in ("dense", "blocks"):
            raise ValueError(f"tsdf_volume must be 'dense' or 'blocks', not {self.volume_type!r}")
        self.block_count = int(getattr(args, "tsdf_block_count", 5000))
        self.volume = None                               # the VoxelBlockVolume in "blocks" mode
        self.integrated_frames = 0
        self.initialize()

    def initialize(self):
        if self.volume_type == "blocks":
            if self.volume is None:
                self.volume = VoxelBlockVolume(self.voxel_size, self.block_count, self.device)
            else:
                self.volume.reset(self.voxel_size)       # capacity kept
            return
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
        n, _, H, W = images.shape
        intr = np.ascontiguousarray(np.asarray(intrinsics, np.float32))
        if self.volume is not None:
            for k in range(n):                           # one host read of the block counts per keyframe
                self.volume.integrate(idepths[k], covs[k] if covs is not None else None, images[k], intr, poses[k],
                                      self.max_depth, self.sdf_trunc, self.max_weight, self.max_depth_sigma_thresh)
            self.integrated_frames += n
            return
        lib = _lib.load()
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
        """voxel centres next to a zero crossing of the TSDF along x / y / z with enough weight (a quick look at the
        surface in plain torch; build_mesh is the full read-out) -> [m,3] world points, [m,3] colours.  Dense grid only."""
        if self.volume is not None:
            raise NotImplementedError("surface_points reads the dense grid; use build_mesh with tsdf_volume='blocks'")
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

    def build_mesh(self, min_weight_for_mesh):
        """:556-573: marching cubes over the cubes whose 8 corners have weight > min_weight_for_mesh -> TsdfMesh, or None
        when there is no triangle.  One host read of the three counts sizes the outputs."""
        if self.volume is not None:
            return self.volume.build_mesh(min_weight_for_mesh)
        return mesh_dense(self.tsdf, self.weight, self.color, self.origin, self.voxel_size, min_weight_for_mesh)

    def render_volume(self, packet, intrinsics, min_weight_for_render, max_depth_sigma_thresh, evaluate=False):
        """:319-484: ray-cast depth and colour at every keyframe of the packet -> (depth [n,H,W], colour [n,H,W,3] in [0,1]);
        0 where a ray misses.  Views go `render_views_per_launch` per launch.  With `evaluate`, the mean PSNR and depth L1
        over the views go to results.csv in the working directory as pandas' DataFrame.to_csv writes the reference's row.
        `max_depth_sigma_thresh` only feeds the reference's debug views; it is accepted for the same call."""
        if not packet:
            print("Error: asked to render volume, but packet is None.")
            return None
        dev = torch.device(self.device) if self.volume is not None else self.tsdf.device
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
                if self.volume is not None:
                    depth[s:s + m], color[s:s + m] = self.volume.raycast(
                        poses[s:s + m], H, W, intr, self.min_depth, self.max_depth, self.sdf_trunc, min_weight_for_render)[:2]
                else:
                    nz, ny, nx = self.tsdf.shape
                    _lib.check(_lib.load().nslam_tsdf_raycast(
                        _lib.ptr(self.tsdf), _lib.ptr(self.weight), _lib.ptr(self.color), nx, ny, nz, self.origin.ctypes.data,
                        float(self.voxel_size), _lib.ptr(poses[s:s + m]), m, H, W, intr.ctypes.data, float(self.min_depth),
                        float(self.max_depth), float(self.sdf_trunc), float(min_weight_for_render), _lib.ptr(depth[s:s + m]),
                        _lib.ptr(color[s:s + m]), _lib.ptr(weight), None, _lib.stream_ptr()), "tsdf_raycast")
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
