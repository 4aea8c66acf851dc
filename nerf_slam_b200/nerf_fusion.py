"""NerfFusion — the reference's fusion/nerf_fusion.py:29-485 on the sm_90a NeRF kernels.

Same surface: NerfFusion(name, args, device) .fuse(data_packets) .stop_condition()
              .process_slam / .process_data / .send_data / .fit_volume / .fit_volume_once / .eval_gt_traj
Beyond the reference: `build_mesh` reads the trained NeRF out as a coloured marching-cubes mesh (pyngp.Testbed.marching_cubes).
Differences by design: the SLAM packet's CUDA tensors go straight into the trainer's device slots
(sRGB->linear, premultiply, 1/idepth fused in one kernel) — the reference converts on the GPU,
copies to the CPU, to numpy, into pyngp and back to the GPU ("extremely slow", :209).
"""
import numpy as np
import torch

from . import pyngp as ngp


def _pose_tq_to_c2w(tq):
    """cam_T_world [n,7] (t, q_xyzw) -> world_T_cam 4x4 (fp64 on the host; n is small)"""
    tq = tq.detach().double().cpu().numpy() if torch.is_tensor(tq) else np.asarray(tq, np.float64)
    out = np.zeros((tq.shape[0], 4, 4))
    for k, v in enumerate(tq):
        x, y, z, w = v[3:]
        R = np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                      [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                      [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])
        T = np.eye(4); T[:3, :3] = R; T[:3, 3] = v[:3]
        out[k] = np.linalg.inv(T)
    return out


def get_scale_and_offset(aabb):
    """utils/utils.py:147-160: isotropic scale + offset that map the aabb [[min],[max]] into the unit cube around 0.5"""
    aabb = np.array(aabb, dtype=np.float64)
    ext = aabb[1] - aabb[0]
    scale = 1.0 / max(0.000001, float(np.abs(ext).max()))
    return scale, (aabb[1] + aabb[0]) * 0.5 * -scale + 0.5


def mse2psnr(x):
    return -10. * np.log(x) / np.log(10.)


def compute_error(img, ref):
    """utils/utils.py:176-188: mean squared error over ALL channels of the image (RGBA: the alpha channel counts),
    estimate clamped at 0, non-finite values of the estimate and of the error map count as 0"""
    img = np.array(img, dtype=np.float32, copy=True)
    img[~np.isfinite(img)] = 0
    err = (np.maximum(img, 0.) - ref) ** 2
    err[~np.isfinite(err)] = 0
    if err.ndim == 3:
        err = err.mean(axis=2)
    return float(err.mean())


class NerfFusion:
    def __init__(self, name, args, device):
        self.name, self.args, self.device = name, args, device
        self.iters = 1
        self.total_iters = 0
        self.stop_iters = 25000
        self.ngp = ngp.Testbed(ngp.TestbedMode.Nerf, 0)
        aabb_scale = 4
        self.ngp.create_empty_nerf_dataset(args.buffer, 1.0, np.array([np.inf] * 3), aabb_scale,
                                           ngp.BoundingBox(-np.inf * np.ones(3), np.inf * np.ones(3)))
        self.ngp.nerf.training.n_images_for_training = 0
        self.ngp.reload_network_from_file(getattr(args, "network", None))
        self.ngp.shall_train = True
        self.ngp.nerf.training.optimize_extrinsics = True      # :99 — per-camera pose refinement (csrc/ngp_extrinsics.cu)
        self.ngp.nerf.training.depth_supervision_lambda = 1.0
        self.ngp.nerf.training.depth_loss_type = ngp.LossType.L2
        self.mask_type = getattr(args, "mask_type", "ours")
        # ground-truth depth of the ingested keyframes, for eval_gt_traj only: ONE preallocated [buffer,H,W] device
        # tensor filled per frame id (allocated on first use when args.eval is set) + the depth scale; the SLAM packets
        # themselves are not retained (they hold full-resolution images / depths of the whole BA window)
        self.ref_frames = {}            # fid -> depth_scale (membership = "a GT depth is stored for this frame id")
        self._gt_depths = None
        self.anneal, self.anneal_every_iters, self.annealing_rate = False, 200, 0.95      # :108-110
        self.evaluate = bool(getattr(args, "eval", False))
        self.eval_every_iters = 200
        self.results = []
        # the training colours are linear (process_slam, process_data "metric") or sRGB values / 255 (process_data
        # "reference"); build_mesh hands its vertex colours back in the images' own encoding
        self.linear_training_colors = True
        self.fit_volume_once()

    # ------------------------------------------------------------------ B1
    def process_slam(self, packet):
        """fusion/nerf_fusion.py:140-235"""
        if not packet:
            return True
        slam = packet[1] if isinstance(packet, (list, tuple)) else packet
        if slam is None or slam.get("is_last_frame", False):      # the last packet is not ingested (:154-155): just fit
            return True
        viz_idx = slam["viz_idx"]
        images = slam["cam0_images"]
        idepths_up = slam["cam0_idepths_up"]
        depths_cov_up = slam["cam0_depths_cov_up"]
        calib = slam["calibs"][0]
        assert images.dtype == torch.uint8 and idepths_up.dtype == torch.float32
        self.linear_training_colors = True                          # sRGB -> linear in the ingest kernel
        if self.mask_type == "raw":
            depths_cov_up = torch.ones_like(depths_cov_up)
        elif self.mask_type == "ours_w_thresh":
            idepths_up = torch.where(depths_cov_up.sqrt() > depths_cov_up.quantile(0.50), -torch.ones_like(idepths_up), idepths_up)
        elif self.mask_type == "no_depth":
            idepths_up = -torch.ones_like(idepths_up)
        elif self.mask_type != "ours":
            raise NotImplementedError(f"Unknown mask type: {self.mask_type}")
        ids = slam["viz_idx_host"] if "viz_idx_host" in slam else viz_idx.tolist()
        poses = slam["cam0_poses"]                                  # cam_T_world [n,7]; scale 1.0, offset 0 (:167-170)
        on_device = torch.is_tensor(poses) and poses.is_cuda
        c2w = None if on_device else _pose_tq_to_c2w(poses)[:, :3, :4]
        intr = calib.camera_model.numpy()
        dev = self.ngp.device
        images, idepths_up, depths_cov_up = images.to(dev), idepths_up.to(dev), depths_cov_up.to(dev)
        # the packet was allocated on the SLAM stream and is read here by kernels of the (possibly different) current
        # stream: tell the caching allocator, so that the blocks are not handed back to the producer stream while the
        # ingest kernels are still pending
        cur = torch.cuda.current_stream(dev) if images.is_cuda else None
        if cur is not None:
            for t in (images, idepths_up, depths_cov_up):
                t.record_stream(cur)
        # world_T_cam records are computed on the device from the packet's poses (no host copy, no sync)
        self.ngp.nerf.training.update_training_images_device(
            ids, c2w, images, idepths_up, depths_cov_up, intr[:2], intr[2:],
            cam_T_world=poses.to(dev) if on_device else None,
            ids_device=viz_idx.to(dev) if torch.is_tensor(viz_idx) and viz_idx.is_cuda and viz_idx.dtype == torch.int64 else None)
        if getattr(self, "evaluate", False) and "gt_depths" in slam:
            gt = slam["gt_depths"].to(dev)
            if cur is not None:
                gt.record_stream(cur)
            if self._gt_depths is None:
                self._gt_depths = torch.zeros(self.args.buffer, gt.shape[-2], gt.shape[-1], device=dev)
            self._gt_depths[torch.as_tensor(ids, device=dev, dtype=torch.long)] = gt[:, 0].float()
            for fid in ids:
                self.ref_frames[fid] = float(calib.depth_scale)
        return False

    def process_data(self, packet):
        """ground-truth fitting (fusion/nerf_fusion.py:121-138).  `gt_fit_convention`:
        "reference" (default) = exactly the tuples the reference hands to the trainer — world_T_cam scaled and offset into
        the unit cube by the calibration's aabb (get_scale_and_offset), colours = u8 / 255 (NOT linearised, NOT
        premultiplied, unlike process_slam), depth scale = calib.depth_scale * scale;
        "metric" = poses as they are, linear premultiplied colours (consistent with process_slam's convention)."""
        calib = packet["calibs"][0]
        c2w = np.linalg.inv(np.asarray(packet["poses"], np.float64))
        dep = np.asarray(packet["depths"]).astype(np.float32)
        intr = calib.camera_model.numpy()
        reference = getattr(self, "gt_fit_convention", "reference") == "reference"
        self.linear_training_colors = not reference
        if reference:
            scale, offset = get_scale_and_offset(calib.aabb)
            c2w[:, :3, 3] = c2w[:, :3, 3] * scale + offset
            rgba = np.asarray(packet["images"]).astype(np.float32) / 255.0
            depth_scale = calib.depth_scale * scale
        else:
            imgs = torch.as_tensor(np.asarray(packet["images"])).float() / 255.0
            rgb = torch.where(imgs[..., :3] > 0.04045, ((imgs[..., :3] + 0.055) / 1.055) ** 2.4, imgs[..., :3] / 12.92)
            rgba = torch.cat([rgb * imgs[..., 3:4], imgs[..., 3:4]], -1).numpy()
            depth_scale = calib.depth_scale
        self.ngp.nerf.training.optimize_extrinsics = False
        k = packet["k"]
        ids = k.tolist() if hasattr(k, "tolist") else list(k)
        self.ngp.nerf.training.update_training_images(
            [int(i) for i in ids], list(c2w[:, :3, :4]), list(rgba), list(dep),
            list(np.ones_like(dep)), calib.resolution.numpy(), intr[2:], intr[:2], depth_scale, 1.0)
        return False

    def send_data(self, batch):
        raise NotImplementedError("use process_slam/process_data; kept for surface compatibility")

    # ------------------------------------------------------------------ main loop
    def fuse(self, data_packets):
        fit = False
        if data_packets:
            for name, packet in data_packets.items():
                if name == "data":
                    fit = self.process_data(packet)
                elif name == "slam":
                    fit = self.process_slam(packet)
                else:
                    raise NotImplementedError(f"process_{name} not implemented...")
            if fit:
                self.fit_volume()
        else:
            self.fit_volume()
        return True

    def stop_condition(self):
        return self.total_iters > self.stop_iters if self.evaluate else False

    def fit_volume(self):
        for _ in range(self.iters):
            self.fit_volume_once()

    def fit_volume_once(self):
        """:298-307"""
        self.ngp.frame()
        if self.anneal and self.total_iters % self.anneal_every_iters == 0:
            self.ngp.nerf.training.depth_supervision_lambda *= self.annealing_rate
        if self.evaluate and self.total_iters % self.eval_every_iters == 0 and self.ngp.rgba is not None:
            self.eval_gt_traj()
        self.total_iters += 1

    # ------------------------------------------------------------------ mesh read-out
    def build_mesh(self, resolution=256, thresh=2.5, aabb=None):
        """marching-cubes mesh of the NeRF's density level set sigma = thresh (pyngp.Testbed.marching_cubes) -> TsdfMesh of
        device tensors in the training cameras' world frame, or None when no triangle results (as TsdfFusion.build_mesh).
        Vertex colours come back in the encoding of the training images: sRGB when the ingest linearised them
        (process_slam, process_data with gt_fit_convention "metric"), the network's values for the reference convention."""
        return self.ngp.marching_cubes(resolution, aabb, thresh, srgb=self.linear_training_colors)

    # ------------------------------------------------------------------ B4
    def eval_gt_traj(self, stride=2):
        """PSNR / depth-L1 over the training views (fusion/nerf_fusion.py:379-485)"""
        tb = self.ngp
        saved = (tb.shall_train, list(tb.background_color), tb.render_mode, tb.camera_matrix.copy())
        tb.background_color = [0.0, 0.0, 0.0, 1.0]
        tb.shall_train = False
        tot_psnr = tot_l1 = 0.0
        count = 0
        n = tb.nerf.training.n_images_for_training
        for i in range(0, n, stride):
            tb.set_camera_to_training_view(i)
            fid = tb.active_set[i]
            ref = tb.rgba[fid].float().cpu().numpy()
            tb.render_mode = ngp.Shade
            est = tb.render(ref.shape[1], ref.shape[0], 1, True)
            mse = compute_error(est, ref)                       # over RGBA, like the reference (:424)
            tot_psnr += mse2psnr(max(mse, 1e-12))
            if fid in self.ref_frames:
                gt = self._gt_depths[fid].cpu().numpy() * self.ref_frames[fid]
                tb.render_mode = ngp.Depth
                d = tb.render(ref.shape[1], ref.shape[0], 1, True)[..., 0]
                s = gt.mean() / max(d.mean(), 1e-9)
                tot_l1 += float(np.minimum(np.abs(s * d - gt), 2.0).mean() * 100)
            count += 1
        tb.shall_train, tb.background_color, tb.render_mode, tb.camera_matrix = saved
        res = dict(iter=self.total_iters, dt=tb.elapsed_training_time, psnr=tot_psnr / max(count, 1),
                   l1=tot_l1 / max(count, 1), count=count)
        self.results.append(res)
        return res
