"""`pyngp`-shaped façade over the sm_90a NeRF kernels (Path B).

Exposes exactly the surface that the reference's fusion/nerf_fusion.py uses of the instant-ngp
fork's python module (SURVEY.md §8b "pyngp surface used"):

  TestbedMode.Nerf, Testbed(mode, 0), BoundingBox(min, max), LossType.L2, Shade / Depth,
  .create_empty_nerf_dataset(n_images, nerf_scale, offset, aabb_scale, render_aabb)
  .reload_network_from_file(path)      (no-op: the base.json architecture is built in)
  .shall_train .dynamic_res .dynamic_res_target_fps .camera_smoothing .display_gui ...
  .nerf.training.{n_images_for_training, optimize_extrinsics, depth_supervision_lambda,
                  depth_loss_type, update_training_images(...)}
  .frame()  .loss  .elapsed_training_time  .apply_camera_smoothing(ms)
  .background_color .snap_to_pixel_centers .nerf.rendering_min_transmittance .camera_matrix
  .render_mode .set_camera_to_training_view(i) .render(w, h, spp, linear, fps=)

plus a device-side fast path (`update_training_images_device`) that takes the SLAM packet's CUDA
tensors directly (no CPU round trip, cf. fusion/nerf_fusion.py:198-223).
"""
import ctypes
import math
import time

import numpy as np
import torch

from . import _lib

N_LEVELS, LOG2_T, BASE_RES = 16, 19, 16
W_TOTAL = 10240
GRID = 128


class TestbedMode:
    Nerf = 0


class LossType:
    L2 = 0
    L1 = 1
    Huber = 2


Shade, Depth = 0, 1


class BoundingBox:
    def __init__(self, mn, mx):
        self.min, self.max = np.asarray(mn, dtype=np.float64), np.asarray(mx, dtype=np.float64)


class NgpModel(ctypes.Structure):
    _fields_ = [(n, ctypes.c_void_p) for n in ("grid_half", "grid_master", "grid_grad", "grid_m", "grid_v",
                                               "mlp", "mlp_grad", "mlp_m", "mlp_v", "density", "bits", "stats")] + \
               [("aabb_scale", ctypes.c_float), ("cascades", ctypes.c_int), ("cone", ctypes.c_float),
                ("near_distance", ctypes.c_float),
                ("scale", ctypes.c_float * 16), ("res", ctypes.c_int * 16), ("size", ctypes.c_uint * 16),
                ("offset", ctypes.c_uint * 16), ("dense", ctypes.c_int * 16), ("n_grid", ctypes.c_uint)]


class NgpImages(ctypes.Structure):
    _fields_ = [(n, ctypes.c_void_p) for n in ("rgba", "depth", "depth_cov", "cams", "active")] + \
               [(n, ctypes.c_int) for n in ("n_active", "H", "W")]


class NgpBatch(ctypes.Structure):
    _fields_ = [(n, ctypes.c_void_p) for n in ("rays", "coords", "tdist", "rgbsigma", "dout", "counters", "loss")] + \
               [(n, ctypes.c_int) for n in ("max_rays", "max_samples")] + \
               [(n, ctypes.c_void_p) for n in ("enc", "denc")]


def level_table(aabb_scale):
    b = math.exp(math.log(2048.0 * aabb_scale / BASE_RES) / (N_LEVELS - 1))
    T = 1 << LOG2_T
    rows, off = [], 0
    for l in range(N_LEVELS):
        scale = BASE_RES * (b ** l) - 1.0
        res = int(math.ceil(scale)) + 1
        n = min(((res ** 3 + 7) // 8) * 8, T)
        rows.append((float(np.float32(scale)), res, n, off, int(res ** 3 <= n)))
        off += n
    return rows, off


class _Training:
    def __init__(self, tb):
        self._tb = tb
        self.n_images_for_training = 0
        self.optimize_extrinsics = False
        self.depth_supervision_lambda = 0.0
        self.depth_loss_type = LossType.L2
        self.near_distance = 0.05
        self.density_grid_decay = 0.95
        # camera-pose refinement (instant-ngp's published defaults; active when optimize_extrinsics is set)
        self.extrinsic_learning_rate = 1e-3
        self.extrinsic_l2_reg = 1e-4

    def update_training_images(self, frame_ids, poses, images, depths, depths_cov, resolution,
                               principal_point, focal_length, depth_scale, depth_cov_scale):
        """reference signature (fusion/nerf_fusion.py:285-289): lists of numpy arrays from the host."""
        tb = self._tb
        dev = tb.device
        for k, fid in enumerate(frame_ids):
            img = torch.as_tensor(np.asarray(images[k]), device=dev).float()      # [H,W,4] linear premult
            dep = torch.as_tensor(np.asarray(depths[k]), device=dev).float().reshape(img.shape[0], img.shape[1]) * depth_scale
            cov = torch.as_tensor(np.asarray(depths_cov[k]), device=dev).float().reshape(img.shape[0], img.shape[1]) * depth_cov_scale
            tb._ensure_store(img.shape[0], img.shape[1])
            tb.rgba[fid] = img.half()
            tb.depth[fid] = dep
            tb.depth_cov[fid] = cov
            tb._set_camera(fid, np.asarray(poses[k], np.float64), focal_length, principal_point, resolution)
        tb._activate(frame_ids)

    def update_training_images_device(self, frame_ids, c2w, images_u8_chw, idepths_up, depths_cov_up,
                                      focal_length, principal_point, cam_T_world=None, ids_device=None):
        """device fast path: images uint8 [n,3,H,W] (sRGB), idepths_up / depths_cov_up [n,H,W] CUDA tensors; ONE kernel
        launch for the whole packet (sRGB->linear, premultiply, 1/idepth, slot scatter).
        Cameras: `cam_T_world` [n,7] (t, q_xyzw) CUDA tensor -> world_T_cam records computed by the same kernel (no host
        copy of the poses: that copy was a device synchronisation per SLAM tick); else `c2w` [n,3,4] host matrices.
        frame_ids: host list (the slot ids are known on the host: dirty flags live there); ids_device: the same ids as
        an int64 CUDA tensor when the caller already has it."""
        tb = self._tb
        lib = _lib.load()
        n, _, H, W = images_u8_chw.shape
        tb._ensure_store(H, W)
        ids = [int(f) for f in frame_ids]
        if n:
            ids_d = ids_device if ids_device is not None else _lib.h2d(np.asarray(ids, np.int64), tb.device)
            fl = np.asarray(focal_length, np.float32).reshape(-1); pp = np.asarray(principal_point, np.float32).reshape(-1)
            pose = None
            if cam_T_world is not None:
                pose = cam_T_world.to(torch.float32).contiguous()
                assert pose.shape == (n, 7) and pose.is_cuda
            _lib.check(lib.nslam_ngp_ingest_batch(
                _lib.ptr(images_u8_chw.contiguous()), _lib.ptr(idepths_up.contiguous()), _lib.ptr(depths_cov_up.contiguous()),
                _lib.ptr(ids_d), n, H, W, _lib.ptr(tb.rgba), _lib.ptr(tb.depth), _lib.ptr(tb.depth_cov), _lib.ptr(pose),
                float(fl[0]), float(fl[1]), float(pp[0]), float(pp[1]), _lib.ptr(tb.cams) if pose is not None else None,
                _lib.ptr(tb.cams_base) if pose is not None else None, _lib.ptr(tb.cam_state), _lib.ptr(tb.cam_steps),
                tb.n_images, _lib.stream_ptr()), "ngp_ingest_batch")
            if pose is not None:
                tb._cams_host_stale = True
            else:
                for k, fid in enumerate(ids):
                    tb._set_camera(fid, np.asarray(c2w[k], np.float64), focal_length, principal_point, (W, H))
        tb._activate(ids)


class _Nerf:
    def __init__(self, tb):
        self.training = _Training(tb)
        self.visualize_cameras = False
        self.rendering_min_transmittance = 1e-4


class Testbed:
    def __init__(self, mode=TestbedMode.Nerf, device_index=0, seed=1337, max_samples=1 << 18, max_rays=1 << 16):
        self.device = torch.device("cuda", torch.cuda.current_device())
        self.nerf = _Nerf(self)
        self.shall_train = True
        self.dynamic_res = False
        self.dynamic_res_target_fps = 15
        self.camera_smoothing = False
        self.display_gui = False
        self.visualize_unit_cube = False
        self.background_color = [0.0, 0.0, 0.0, 1.0]
        self.snap_to_pixel_centers = True
        self.render_mode = Shade
        self.camera_matrix = np.eye(4)[:3]
        self.loss = float("nan")
        self.elapsed_training_time = 0.0
        self.training_step = 0
        self.seed = seed
        self.max_samples, self.max_rays = max_samples, max_rays
        self.rays_per_batch = 1 << 12
        self.n_images = 0
        self.rgba = None
        self.lr, self.beta1, self.beta2, self.eps, self.l2 = 1e-2, 0.9, 0.99, 1e-15, 1e-6
        self._t0 = None
        from .conv import _sm_budget
        self.num_sms = _sm_budget(self.device, "NSLAM_NERF_SMS")
        self._measured = None
        self.grad_hook = None        # e.g. dist.allreduce_grads for data-parallel training
        self._ctr_event = None; self._ctr_host = None; self._loss_host = None; self._ctr_rays = 0
        # "tcgen05" (the historical name of the tensor-core path): MLP forward/backward on tensor cores (wgmma,
        # csrc/ngp_tc.cu); "simt": fp32 CUDA-core kernels
        self.mlp_backend = "tcgen05"
        self.loss_scale = 1024.0

    # ---------------------------------------------------------------- setup
    def init_window(self, *a, **k):
        pass

    def reload_network_from_file(self, path=None):
        """configs/nerf/base.json of the fork is absent; its (published) architecture is built in:
        HashGrid 16x2, T=2^19, base 16; density 1x64 -> 16; SH4; rgb 2x64 -> 3; Adam 1e-2."""
        return None

    def create_empty_nerf_dataset(self, n_images, nerf_scale=1.0, offset=None, aabb_scale=4, render_aabb=None):
        dev = self.device
        self.n_images = int(n_images)
        self.aabb_scale = float(aabb_scale)
        self.cascades = 1 + int(math.ceil(math.log2(aabb_scale))) if aabb_scale > 1 else 1
        rows, total = level_table(self.aabb_scale)
        g = torch.Generator(device="cpu").manual_seed(self.seed)
        f = dict(dtype=torch.float32, device=dev)
        self.grid_master = ((torch.rand(total * 2, generator=g) * 2 - 1) * 1e-4).to(dev)
        self.grid_half = self.grid_master.half()
        self.grid_grad = torch.zeros(total * 2, **f); self.grid_m = torch.zeros(total * 2, **f); self.grid_v = torch.zeros(total * 2, **f)
        ws = []
        for (i, o) in ((32, 64), (64, 16), (32, 64), (64, 64), (64, 16)):
            s = math.sqrt(6.0 / (i + o))
            ws.append(((torch.rand(i, o, generator=g) * 2 - 1) * s).reshape(-1))
        self.mlp = torch.cat(ws).to(dev)
        self.mlp_grad = torch.zeros(W_TOTAL, **f); self.mlp_m = torch.zeros(W_TOTAL, **f); self.mlp_v = torch.zeros(W_TOTAL, **f)
        ncell = GRID ** 3 * self.cascades
        self.density = -torch.ones(ncell, **f)
        self.bits = torch.zeros(ncell // 8, dtype=torch.uint8, device=dev)
        self.stats = torch.zeros(2, **f)
        m = NgpModel()
        for name in ("grid_half", "grid_master", "grid_grad", "grid_m", "grid_v", "mlp", "mlp_grad", "mlp_m",
                     "mlp_v", "density", "bits", "stats"):
            setattr(m, name, getattr(self, name).data_ptr())
        m.aabb_scale = self.aabb_scale; m.cascades = self.cascades
        m.cone = 1.0 / 256.0 if aabb_scale > 1 else 0.0
        m.near_distance = self.nerf.training.near_distance
        for l, (sc, res, n, off, dense) in enumerate(rows):
            m.scale[l], m.res[l], m.size[l], m.offset[l], m.dense[l] = sc, res, n, off, dense
        m.n_grid = total
        self.model = m
        self._cams_h = np.zeros((self.n_images, 18), np.float32)
        self._cams_host_stale, self._cams_upload = False, []
        self.cams = torch.zeros(self.n_images, 18, **f)          # effective cameras (base pose (+) refinement offsets)
        # pose refinement (nerf.training.optimize_extrinsics, csrc/ngp_extrinsics.cu): base cameras as SLAM sent them,
        # per-camera offsets / Adam moments [3,N,6] = (translation, rotation vector), gradient accumulator, step counts
        self.cams_base = torch.zeros(self.n_images, 18, **f)
        self.cam_state = torch.zeros(3, self.n_images, 6, **f)
        self.cam_grad = torch.zeros(self.n_images, 6, **f)
        self.cam_steps = torch.zeros(self.n_images, dtype=torch.int32, device=dev)
        self._lv = {k: np.ascontiguousarray(np.asarray([r[i] for r in rows], dt)) for i, (k, dt) in
                    enumerate((("scale", np.float32), ("res", np.int32), ("size", np.uint32), ("offset", np.uint32), ("dense", np.int32)))}
        self.active = torch.zeros(self.n_images, dtype=torch.int32, device=dev)
        self.active_set = []
        b = NgpBatch()
        self._bufs = dict(rays=torch.zeros(self.max_rays, 16, **f), coords=torch.zeros(self.max_samples, 7, **f),
                          tdist=torch.zeros(self.max_samples, **f), rgbsigma=torch.zeros(self.max_samples, 4, **f),
                          dout=torch.zeros(self.max_samples, 4, **f),
                          counters=torch.zeros(4, dtype=torch.int32, device=dev), loss=torch.zeros(1, **f),
                          enc=torch.zeros(self.max_samples, 32, dtype=torch.float16, device=dev),
                          denc=torch.zeros(self.max_samples, 32, dtype=torch.float16, device=dev))
        for k, v in self._bufs.items():
            setattr(b, k, v.data_ptr())
        b.max_rays, b.max_samples = self.max_rays, self.max_samples
        self.batch = b
        self.packed = torch.zeros(61440, dtype=torch.uint8, device=dev)
        self.pack_weights()

    def pack_weights(self):
        """fp16 wgmma-ready images of the current fp32 MLP weights (after init / every optimiser step)"""
        _lib.check(_lib.load().nslam_ngp_pack_mlp(_lib.ptr(self.mlp), _lib.ptr(self.packed), _lib.stream_ptr()), "ngp_pack_mlp")

    def _ensure_store(self, H, W):
        if self.rgba is None:
            dev = self.device
            self.H, self.W = H, W
            self.rgba = torch.zeros(self.n_images, H, W, 4, dtype=torch.float16, device=dev)
            self.depth = -torch.ones(self.n_images, H, W, dtype=torch.float32, device=dev)
            self.depth_cov = torch.ones(self.n_images, H, W, dtype=torch.float32, device=dev)
        assert (H, W) == (self.H, self.W), "all training images share one resolution"

    @property
    def cams_h(self):
        """host mirror of the camera records [n_images,18]; refreshed from the device (one synchronising copy) when the
        device-side ingest wrote cameras since the last read — evaluation / tests only, never in the training loop"""
        if self._cams_host_stale:
            self._cams_h[:] = self.cams.cpu().numpy()
            self._cams_host_stale = False
        return self._cams_h

    def _set_camera(self, fid, c2w34, focal, pp, resolution):
        row = np.zeros(18, np.float32)
        row[:12] = np.asarray(c2w34, np.float32)[:3, :4].reshape(-1)
        row[12:14] = np.asarray(focal, np.float32).reshape(-1)[:2]
        row[14:16] = np.asarray(pp, np.float32).reshape(-1)[:2]
        # the camera record holds w,h as int32 in the last two slots
        row[16:18] = np.array([int(resolution[0]), int(resolution[1])], np.int32).view(np.float32)
        self.cams_h[fid] = row
        self._cams_upload.append(int(fid))

    def _activate(self, ids):
        for i in ids:
            if int(i) not in self.active_set:
                self.active_set.append(int(i))
        if self._cams_upload:                       # host-set camera rows only (device-written rows are not touched)
            rows = sorted(set(self._cams_upload))
            rd, vals = _lib.h2d(np.asarray(rows, np.int64), self.device), _lib.h2d(self._cams_h[rows], self.device)
            self.cams.index_copy_(0, rd, vals)
            self.cams_base.index_copy_(0, rd, vals)          # new base pose: the refinement of these cameras restarts
            self.cam_state[:, rd] = 0
            self.cam_steps[rd] = 0
            self._cams_upload = []
        n = len(self.active_set)
        self.active[:n].copy_(torch.as_tensor(self.active_set, dtype=torch.int32).pin_memory(), non_blocking=True)
        self.nerf.training.n_images_for_training = n

    def _images(self):
        im = NgpImages()
        im.rgba, im.depth, im.depth_cov = self.rgba.data_ptr(), self.depth.data_ptr(), self.depth_cov.data_ptr()
        im.cams, im.active = self.cams.data_ptr(), self.active.data_ptr()
        im.n_active, im.H, im.W = len(self.active_set), self.H, self.W
        return im

    # ---------------------------------------------------------------- training
    def update_density_grid(self, full=False):
        lib = _lib.load()
        n = GRID ** 3 if full else GRID ** 3 // 4
        im = self._images()
        _lib.check(lib.nslam_ngp_update_density_grid(ctypes.byref(self.model), ctypes.byref(im), n,
                                                     (self.seed * 7919 + self.training_step) & 0xFFFFFFFF,
                                                     self.nerf.training.density_grid_decay, 0.01,
                                                     _lib.ptr(self.packed) if self.mlp_backend == "tcgen05" else None,
                                                     self.num_sms, _lib.stream_ptr()), "ngp_update_density_grid")

    def train_step(self):
        """one optimisation step; no host synchronisation"""
        with _lib.fixed_stream():
            self._train_step_impl()

    def _train_step_impl(self):
        lib = _lib.load()
        if self._t0 is None:
            self._t0 = time.perf_counter()
        if self.training_step % 16 == 0:
            self.update_density_grid(full=self.training_step < 256)
        im = self._images()
        bg = self.background_color
        seed = (self.seed + 0x9E3779B1 * (self.training_step + 1)) & 0xFFFFFFFF
        lam = float(self.nerf.training.depth_supervision_lambda)
        if self.mlp_backend == "tcgen05":
            _lib.check(lib.nslam_ngp_train_step_tc(ctypes.byref(self.model), ctypes.byref(im), ctypes.byref(self.batch),
                                                   _lib.ptr(self.packed), self.rays_per_batch, seed, lam, bg[0], bg[1], bg[2],
                                                   float(self.loss_scale), self.num_sms, _lib.stream_ptr()), "ngp_train_step_tc")
        else:
            _lib.check(lib.nslam_ngp_train_step(ctypes.byref(self.model), ctypes.byref(im), ctypes.byref(self.batch),
                                                self.rays_per_batch, seed, lam, bg[0], bg[1], bg[2], self.num_sms,
                                                _lib.stream_ptr()), "ngp_train_step")
        tr = self.nerf.training
        refine = tr.optimize_extrinsics and self.mlp_backend == "tcgen05" and tr.extrinsic_learning_rate > 0
        if refine:
            lv = self._lv
            _lib.check(lib.nslam_ngp_cam_grad(_lib.ptr(self.grid_half), lv["scale"].ctypes.data, lv["res"].ctypes.data,
                                              lv["size"].ctypes.data, lv["offset"].ctypes.data, lv["dense"].ctypes.data,
                                              float(self.aabb_scale), _lib.ptr(self._bufs["rays"]), int(self.rays_per_batch),
                                              _lib.ptr(self._bufs["coords"]), _lib.ptr(self._bufs["tdist"]), _lib.ptr(self._bufs["denc"]),
                                              float(self.loss_scale), _lib.ptr(self.cam_grad), int(self.cam_grad.shape[0]),
                                              _lib.stream_ptr()), "ngp_cam_grad")
        if self.grad_hook is not None:
            self.grad_hook(self)
        if refine:
            _lib.check(lib.nslam_ngp_cam_adam_apply(_lib.ptr(self.cams_base), _lib.ptr(self.cams), _lib.ptr(self.cam_state[0]),
                                                    _lib.ptr(self.cam_grad), _lib.ptr(self.cam_state[1]), _lib.ptr(self.cam_state[2]),
                                                    _lib.ptr(self.cam_steps), self.n_images, float(tr.extrinsic_learning_rate),
                                                    0.9, 0.99, 1e-10, float(tr.extrinsic_l2_reg), _lib.stream_ptr()), "ngp_cam_adam")
            self._cams_host_stale = True
        self.training_step += 1
        decay = 0.33 ** max(0, (self.training_step - 20000) // 10000 + (1 if self.training_step >= 20000 else 0))
        _lib.check(lib.nslam_ngp_adam(ctypes.byref(self.model), self.training_step, self.lr * decay, self.beta1,
                                      self.beta2, self.eps, self.l2, _lib.stream_ptr()), "ngp_adam")
        self.pack_weights()
        # adapt the ray count so that a batch holds ~max_samples samples.  The device counters are copied to
        # pinned memory every 16 steps and consumed whenever that copy has completed: the host never waits.
        if self._ctr_event is not None and self._ctr_event.query():
            used, kept = int(self._ctr_host[0]), max(int(self._ctr_host[1]), 1)
            self.loss = float(self._loss_host[0])
            self._ctr_event = None
            self._measured = (used, kept)
            target = int(0.9 * self.max_samples)
            new = int(self._ctr_rays * target / max(used, 1))
            self.rays_per_batch = int(min(self.max_rays, max(256, (new // 128) * 128)))
        if self.training_step % 16 == 0 and self._ctr_event is None:
            if self._ctr_host is None:
                self._ctr_host = torch.zeros(4, dtype=torch.int32).pin_memory()
                self._loss_host = torch.zeros(1, dtype=torch.float32).pin_memory()
            self._ctr_host.copy_(self._bufs["counters"], non_blocking=True)
            self._loss_host.copy_(self._bufs["loss"], non_blocking=True)
            self._ctr_rays = self.rays_per_batch
            self._ctr_event = torch.cuda.Event()
            self._ctr_event.record()

    def sync_stats(self):
        """block until the last asynchronous counter/loss readback has landed (tests, reporting)"""
        torch.cuda.current_stream().synchronize()
        if self._ctr_event is not None:
            self._ctr_event.synchronize()
            self.loss = float(self._loss_host[0])
            self._measured = (int(self._ctr_host[0]), max(int(self._ctr_host[1]), 1))
        else:
            self.loss = float(self._bufs["loss"].item())
        return self.loss

    def frame(self):
        """Testbed.frame(): one training step when shall_train and data is present (fusion/nerf_fusion.py:299)"""
        if self.shall_train and self.rgba is not None and len(self.active_set) > 0:
            self.train_step()
            self.elapsed_training_time = time.perf_counter() - self._t0
        return True

    def apply_camera_smoothing(self, ms):
        pass

    # ---------------------------------------------------------------- rendering
    def set_camera_to_training_view(self, i):
        self.camera_matrix = self.cams_h[self.active_set[i] if i < len(self.active_set) else i, :12].reshape(3, 4).astype(np.float64).copy()
        self._view_intr = self.cams_h[self.active_set[i] if i < len(self.active_set) else i, 12:16].copy()

    def render(self, width, height, spp=1, linear=True, fps=None, tile_rows=32):
        """-> numpy [H,W,4] float32: Shade = (r,g,b,1) linear; Depth = (d,d,d,1) z-depth"""
        lib = _lib.load()
        dev = self.device
        intr = getattr(self, "_view_intr", None)
        if intr is None:
            intr = np.array([width / 2, width / 2, width / 2 - 0.5, height / 2 - 0.5], np.float32)
        sx, sy = width / float(self.W if self.rgba is not None else width), height / float(self.H if self.rgba is not None else height)
        cam = (ctypes.c_float * 18)()
        c2w = np.asarray(self.camera_matrix, np.float32)[:3, :4].reshape(-1)
        for k in range(12):
            cam[k] = float(c2w[k])
        cam[12], cam[13], cam[14], cam[15] = float(intr[0] * sx), float(intr[1] * sy), float((intr[2] + 0.5) * sx - 0.5), float((intr[3] + 0.5) * sy - 0.5)
        cam[16], cam[17] = float(width), float(height)
        out = torch.zeros(height, width, 4, dtype=torch.float32, device=dev)
        rows = max(1, min(tile_rows, self.max_rays // width))
        per_ray = max(8, min(1024, self.max_samples // (rows * width)))
        bg = self.background_color
        for y0 in range(0, height, rows):
            th = min(rows, height - y0)
            _lib.check(lib.nslam_ngp_render_tile(ctypes.byref(self.model), ctypes.byref(self.batch), cam, 0, y0, width, th,
                                                 per_ray, bg[0], bg[1], bg[2], _lib.ptr(out[y0]),
                                                 _lib.ptr(self.packed) if self.mlp_backend == "tcgen05" else None, self.num_sms,
                                                 _lib.stream_ptr()),
                       "ngp_render_tile")
        o = out.cpu().numpy()
        if self.render_mode == Depth:
            d = o[..., 3:4]
            return np.concatenate([d, d, d, np.ones_like(d)], -1)
        o[..., 3] = 1.0
        return o
