"""RaftVisualFrontend — the live SLAM front-end of the reference
(slam/visual_frontends/visual_frontend.py:62-1391) re-hosted on the sm_90a kernels.

Same public surface: RaftVisualFrontend(world_T_body_t0, body_T_cam0, args, device)
  .forward(batch) -> (x0, factors, viz_out)      .update(...)      .ba(...)      .stop_condition()
Same algorithm and constants (SURVEY.md §5 "Config", §9): warm-up 8 keyframes, motion filter
2.4 px, neighbourhood radius 3 at init, proximity edges (thresh 16, radius 2, nms 1, beta 0.3),
max 48 factors, max age 25, 4+2 update iterations, keyframe threshold 4.0, BA window
kf0 = max(0, min(ii)), 1e-4-sigma prior on frame 0, inactive edges >= kf0-3 prepended.

What is different (GPU-first design, not a translation):
  * state lives in pre-allocated device arenas; correlation pyramids in a slot pool (CorrPool)
    so edges are added/removed without re-copying volumes (reference: torch.cat per add);
  * features are stored channels-last fp16 — the layout the tensor-core kernels consume;
  * the whole BA iteration (linearise -> Schur -> dense fp64 Cholesky -> SE3 retract -> depth
    update -> covariances) runs on the GPU stream: no Eigen, no gtsam, no per-block
    .cpu().numpy() HessianFactor loop, no host synchronisation inside update();
  * the edge list is mirrored on the host, so graph bookkeeping (the bit-exact contract of
    add_proximity_factors) costs no device round-trips except the distance read-back that the
    reference also does.
gtsam is not required: poses may be given as gtsam.Pose3, 4x4 matrices or [t, q_xyzw] vectors.
"""
import numpy as np
import torch

from . import droid_backends as db
from . import _lib
from .corr import CorrPool, AltCorrBlock, coords_grid
from .graph import EdgeList, agg_tables, neighborhood_edges, proximity_edges
from .conv import CORR_PAD as CORR_PAD_
from .networks import BasicEncoder, UpdateModule, load_droid_weights


# ------------------------------------------------------------------------------------------ pose utils
def _as_matrix(p):
    if p is None:
        return np.eye(4)
    if hasattr(p, "matrix"):
        return np.asarray(p.matrix(), dtype=np.float64)
    p = np.asarray(p, dtype=np.float64)
    if p.shape == (4, 4):
        return p
    if p.shape == (7,):
        return tq_to_matrix(p)
    raise ValueError("pose must be gtsam.Pose3, 4x4 or [t,q]")


def tq_to_matrix(v):
    x, y, z, w = v[3:]
    R = np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                  [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                  [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])
    T = np.eye(4)
    T[:3, :3] = R
    T[:3, 3] = v[:3]
    return T


def matrix_to_tq(T):
    R = T[:3, :3]
    tr = np.trace(R)
    if tr > 0:
        s = np.sqrt(tr + 1.0) * 2
        w = 0.25 * s; x = (R[2, 1] - R[1, 2]) / s; y = (R[0, 2] - R[2, 0]) / s; z = (R[1, 0] - R[0, 1]) / s
    elif R[0, 0] > R[1, 1] and R[0, 0] > R[2, 2]:
        s = np.sqrt(1.0 + R[0, 0] - R[1, 1] - R[2, 2]) * 2
        w = (R[2, 1] - R[1, 2]) / s; x = 0.25 * s; y = (R[0, 1] + R[1, 0]) / s; z = (R[0, 2] + R[2, 0]) / s
    elif R[1, 1] > R[2, 2]:
        s = np.sqrt(1.0 + R[1, 1] - R[0, 0] - R[2, 2]) * 2
        w = (R[0, 2] - R[2, 0]) / s; x = (R[0, 1] + R[1, 0]) / s; y = 0.25 * s; z = (R[1, 2] + R[2, 1]) / s
    else:
        s = np.sqrt(1.0 + R[2, 2] - R[0, 0] - R[1, 1]) * 2
        w = (R[1, 0] - R[0, 1]) / s; x = (R[0, 2] + R[2, 0]) / s; y = (R[1, 2] + R[2, 1]) / s; z = 0.25 * s
    return np.array([T[0, 3], T[1, 3], T[2, 3], x, y, z, w])


def types_ns(**kw):
    import types
    return types.SimpleNamespace(**kw)


class _Timers:
    """optional wall-clock section timers of the HOST thread (NSLAM_TIMERS=1); no device syncs are added"""

    def __init__(self):
        import os
        self.on = os.environ.get("NSLAM_TIMERS", "0") == "1"
        self.t = {}

    def section(self, name):
        return _Section(self, name)

    def report(self):
        return {k: (round(v[0] * 1e3, 2), v[1]) for k, v in sorted(self.t.items(), key=lambda kv: -kv[1][0])}


class _Section:
    def __init__(self, timers, name):
        self.tm, self.name = timers, name

    def __enter__(self):
        if self.tm.on:
            import time
            self.t0 = time.perf_counter()

    def __exit__(self, *a):
        if self.tm.on:
            import time
            e = self.tm.t.setdefault(self.name, [0.0, 0])
            e[0] += time.perf_counter() - self.t0; e[1] += 1
        return False


def _edge_attr(name):
    """attribute `name` of the edge list (`self.edges`), readable and assignable on the front end"""
    return property(lambda self: getattr(self.edges, name), lambda self, v: setattr(self.edges, name, v))


class EmptyValues:
    """what the reference's forward() hands to its (no-op) back-end: an EMPTY gtsam.Values / NonlinearFactorGraph
    (visual_frontend.py:248-249).  They must not be None — VioSLAM._frontend stops the pipeline on `x0 is None`
    (slam/vio_slam.py:112-113) — but nothing is ever read from them; gtsam is not a dependency here."""

    def size(self):
        return 0

    def __len__(self):
        return 0

    def __bool__(self):
        return True


class EmptyFactorGraph(EmptyValues):
    pass


class RaftVisualFrontend:
    # the edge list (graph.EdgeList) under this class' names: host index lists *_h, per-edge state gru_* (the reference's
    # names; gru_hidden_states is [E,ht,wd,128] fp16 channels-last).  ii / jj / slots_d are their device copies.
    ii_h, jj_h, age_h, slots_h = _edge_attr("ii"), _edge_attr("jj"), _edge_attr("age"), _edge_attr("slots")
    ii_inactive_h, jj_inactive_h = _edge_attr("ii_inac"), _edge_attr("jj_inac")
    ii_bad_h, jj_bad_h = _edge_attr("ii_bad"), _edge_attr("jj_bad")
    gru_hidden_states, gru_estimated_flow, gru_estimated_flow_weight = _edge_attr("net"), _edge_attr("flow"), _edge_attr("weight")
    gru_estimated_flow_inactive, gru_estimated_flow_weight_inactive = _edge_attr("flow_inac"), _edge_attr("weight_inac")

    def __init__(self, world_T_body_t0, body_T_cam0, args, device="cuda:0"):
        self.args = args
        self.device = device
        self.kf_idx = 0
        self.kf_idx_to_f_idx = {}
        self.f_idx_to_kf_idx = {}
        self.last_kf_idx = 0
        self.last_k = None
        self.global_ba = bool(getattr(args, "global_ba", False))
        self.stop = False
        self.compute_covariances = True
        self.buffer = args.buffer
        self.stereo = bool(getattr(args, "stereo", False))
        self.is_initialized = False

        # constants: visual_frontend.py:92-131
        self.keyframe_warmup = 8
        self.max_age = 25
        self.max_factors = 48
        self.kf_init_count = 8
        self.motion_filter_thresh = 2.4
        self.keyframe_thresh = 4.0
        self.frontend_thresh = 16.0
        self.frontend_window = 25
        self.frontend_radius = 2
        self.frontend_nms = 1
        self.beta = 0.3
        self.backend_thresh = 22.0
        self.backend_radius = 2
        self.backend_nms = 3
        self.iters1 = 4
        self.iters2 = 2
        self.dsf = 8
        self.corr_impl = "volume"

        Twb = _as_matrix(world_T_body_t0)
        Tbc = _as_matrix(body_T_cam0)
        self.world_T_body_t0 = matrix_to_tq(Twb)
        self.world_T_cam0_t0 = matrix_to_tq(Twb @ Tbc)
        self.cam0_t0_T_world = matrix_to_tq(np.linalg.inv(Twb @ Tbc))
        self.cam0_T_body = torch.tensor(matrix_to_tq(np.linalg.inv(Tbc)), device=device, dtype=torch.float32)

        # networks (A1, A5); weights: args.weights (droid.pth) or seeded random init
        self.feature_net = BasicEncoder(128, "instance", torch.Generator().manual_seed(10))
        self.context_net = BasicEncoder(256, "none", torch.Generator().manual_seed(11))
        self.update_net = UpdateModule(torch.Generator().manual_seed(12))
        wpath = getattr(args, "weights", None)
        self.weights_source = "random-init(seeded)"
        if wpath:
            sd = load_droid_weights(wpath)
            self.feature_net.load_state_dict(sd, "feature_net.")
            self.context_net.load_state_dict(sd, "context_net.")
            self.update_net.load_state_dict(sd, "update_net.")
            self.weights_source = wpath
        for m in (self.feature_net, self.context_net, self.update_net):
            m.to(device=device, dtype=torch.float16)
        # encoders and update operator: hand-written wgmma implicit-GEMM convolutions.  There is no library / CPU
        # alternative in the product (the cuDNN formulation of the same networks lives with the reference arm,
        # oracle/ref_cuda_frontend.py, and in the parity tests).
        from .conv import EncoderTC, UpdateOperatorTC
        self.timers = _Timers()
        self.update_tc = UpdateOperatorTC(self.update_net, device)
        self.feature_tc = EncoderTC(self.feature_net, device)
        self.context_tc = EncoderTC(self.context_net, device)

        # prior sigmas (visual_frontend.py:142-153)
        self.g_prior_cov = torch.block_diag(0.01 ** 2 * torch.eye(3), 0.01 ** 2 * torch.eye(3)).to(device)
        self.idepth_prior_cov = 0.1 ** 2
        self.prior_info = 1.0 / (1e-4 ** 2)   # PriorFactorPose3 sigma 1e-4 (:1240-1241)
        self._mean = torch.tensor([0.485, 0.456, 0.406], device=device)[:, None, None]
        self._std = torch.tensor([0.229, 0.224, 0.225], device=device)[:, None, None]
        self.stats = {"updates": 0, "ba_fail": 0}
        # A14 semantics (DESIGN.md §2): 1 = what the reference's covariance block really computes (default), 0 = the
        # formula its comments describe
        self.cov_mode = int(getattr(args, "cov_reference", 1))
        self.use_cuda_graphs = bool(getattr(args, "cuda_graphs", True))
        self._static = None
        self._img_static = None
        # the update operator as one C call per update() (csrc/update_step.cu) instead of ~45 ctypes/torch calls
        self.use_op_step = bool(getattr(args, "op_step", True))
        self._graph_pool = torch.cuda.graph_pool_handle() if self.use_cuda_graphs else None
        # kernel nodes inherit the priority of the stream they were captured on: keep the SLAM chain high
        self._capture_stream = torch.cuda.Stream(priority=-1) if self.use_cuda_graphs else None

    def stop_condition(self):
        return self.stop

    def ba_failures(self, wait=False):
        """number of failed BA factorisations so far (stats['ba_fail']).  The counter lives on the device; each call
        consumes the previous asynchronous read-back (if it has landed, or `wait`) and starts the next one, so the hot
        loop never synchronises on it."""
        if not self._ba_status.is_cuda:          # CPU harness of the reference-trace tests
            self.stats["ba_fail"] = int(self._ba_status[1])
            return self.stats["ba_fail"]
        ev = self._ba_status_event
        if ev is not None and (wait or ev.query()):
            ev.synchronize()
            self.stats["ba_fail"] = int(self._ba_status_host[1])
            ev = None
        if ev is None:
            self._ba_status_host.copy_(self._ba_status, non_blocking=True)
            ev = torch.cuda.Event(); ev.record()
            if wait:
                ev.synchronize()
                self.stats["ba_fail"] = int(self._ba_status_host[1])
                ev = None
        self._ba_status_event = ev
        return self.stats["ba_fail"]

    # ------------------------------------------------------------------ buffers
    def initialize_buffers(self, image_size):
        dev, B = self.device, self.buffer
        self.img_height = h = int(image_size[0])
        self.img_width = w = int(image_size[1])
        self.ht, self.wd = h // self.dsf, w // self.dsf
        ht, wd = self.ht, self.wd
        self.coords0 = coords_grid(ht, wd, dev)
        f = dict(dtype=torch.float32, device=dev)
        self.cam0_timestamps = torch.zeros(B, **f)
        self.cam0_images = torch.zeros(B, 3, h, w, dtype=torch.uint8, device=dev)
        self.cam0_intrinsics = torch.zeros(B, 4, **f)
        self.gt_poses = torch.zeros(B, 4, 4, **f)
        self.gt_depths = torch.zeros(B, 1, h, w, **f)
        self.cam0_T_world = torch.zeros(B, 7, **f)
        self.world_T_body = torch.zeros(B, 7, **f)
        self.world_T_body_cov = torch.zeros(B, 6, 6, **f)
        self.cam0_idepths = torch.ones(B, ht, wd, **f)
        self.cam0_idepths_cov = torch.ones(B, ht, wd, **f) * self.idepth_prior_cov
        self.cam0_depths_cov = torch.ones(B, ht, wd, **f)
        self.cam0_idepths_sensed = torch.zeros(B, ht, wd, **f)
        self.cam0_idepths_up = torch.zeros(B, h, w, **f)
        self.cam0_depths_cov_up = torch.ones(B, h, w, **f)
        self.cam0_T_world[:] = torch.tensor(self.cam0_t0_T_world, **f)
        self.world_T_body[:] = torch.tensor(self.world_T_body_t0, **f)
        self.world_T_body_cov[:] = self.g_prior_cov * torch.eye(6, device=dev)
        self.prior_pose = torch.tensor(self.world_T_cam0_t0, **f)   # prior mean (visual_frontend.py:1235)
        cams = 2 if self.stereo else 1
        self.cameras = cams
        # features channels-last fp16 (wgmma operand layout); contexts channels-first views of NHWC storage
        self.features_imgs = torch.zeros(B, cams, ht, wd, 128, dtype=torch.float16, device=dev)
        self.contexts_imgs = torch.zeros(B, cams, ht, wd, 128, dtype=torch.float16, device=dev)       # NHWC
        self.cst_contexts_imgs = torch.zeros(B, cams, ht, wd, 128, dtype=torch.float16, device=dev)   # NHWC
        self.intr0 = self.cam0_intrinsics[0]      # the kernels only ever see the first keyframe's intrinsics (SURVEY.md §9.22)
        self.corr_pool = CorrPool(int(getattr(self.args, "corr_slots", 2 * self.max_factors)), ht, wd, dev)
        self._reset_graph()
        # BA status: [0] = last factorisation failed, [1] = cumulative failures (read back asynchronously: ba_failures())
        self._ba_status = torch.zeros(2, dtype=torch.int32, device=dev)
        self._ba_status_host = torch.zeros(2, dtype=torch.int32).pin_memory() if torch.cuda.is_available() else torch.zeros(2, dtype=torch.int32)
        self._ba_status_event = None
        self.viz_idx = np.zeros(B, dtype=bool)          # host-side dirty flags (a device mask would need a sync to read)

    def _reset_graph(self):
        self.edges = EdgeList(self.device, self.ht, self.wd)
        self._sync_edges()
        self.damping = 1e-6 * torch.ones_like(self.cam0_idepths)
        if hasattr(self, "corr_pool"):
            self.corr_pool.free = list(range(self.corr_pool.capacity - 1, -1, -1))

    def _sync_edges(self):
        self._static = None            # edge set changed: static part / CUDA graph of update() is stale
        self.ii = _lib.h2d(self.ii_h, self.device)
        self.jj = _lib.h2d(self.jj_h, self.device)
        self.slots_d = _lib.h2d(self.slots_h.astype(np.int32), self.device)

    # ------------------------------------------------------------------ per-frame entry
    def _normalize_imgs(self, images):
        x = images[:, :, :3].float() / 255.0
        return (x - self._mean) / self._std

    def _store_frame(self, idx, batch, imgs_k):
        dev = self.device
        self.gt_poses[idx] = _lib.h2d(np.asarray(batch["poses"][0]), dev, torch.float32)
        if batch["depths"][0] is not None:
            d = torch.as_tensor(np.asarray(batch["depths"][0]), device=dev).float()
            self.gt_depths[idx] = d.permute(2, 0, 1)
        self.cam0_timestamps[idx] = float(batch["t_cams"][0])
        self.cam0_images[idx] = imgs_k[0, 0, :3]
        cm = batch["calibs"][0].camera_model.numpy()
        self.cam0_intrinsics[idx] = (1.0 / self.dsf) * _lib.h2d(np.asarray(cm), dev, torch.float32)

    def _feature_encoder(self, imgs_norm):
        return self.feature_tc(imgs_norm[0])           # [cams,128,ht,wd] fp16 (NHWC storage)

    def _context_encoder(self, imgs_norm):
        """-> (tanh(context), relu(gru input)), both channels-last [cams,ht,wd,128]"""
        c = self.context_tc(imgs_norm[0]).permute(0, 2, 3, 1)
        return torch.tanh(c[..., :128]), torch.relu(c[..., 128:])

    def _run_update_net(self, net, inp, corr_nhwc, coords1, target, ii_host=None):
        """update operator on NHWC tensors: net/inp [E,ht,wd,128], corr [E,ht,wd,CORR_PAD], coords1/target
        [E,ht,wd,2] (target None -> zero residual) -> net' [E,ht,wd,128], delta/weight [E,ht,wd,2] fp32
        (, eta [K,ht,wd], upmask NHWC [K,ht,wd,576]) — the reference's UpdateModule return convention
        (droid_net.py:118-150).  ii_host: numpy source indices of the edges (enables GraphAgg)."""
        agg = None if ii_host is None else agg_tables(ii_host, self.device)
        out = self.update_tc(net, inp, corr_nhwc, coords1.contiguous(), self.coords0, target=target, agg=agg)
        delta = out[1] - coords1
        if ii_host is None:
            return out[0], delta, out[2]
        eta = 0.01 * torch.nn.functional.softplus(out[3][..., 0].float())
        return out[0], delta, out[2], eta, out[4]

    def _put_features(self, idx, feats):
        self.features_imgs[idx] = feats.permute(0, 2, 3, 1)

    @torch.no_grad()
    def forward(self, batch):
        """visual_frontend.py:240-365"""
        k = int(batch["k"][0])
        x0, factors, viz_out = EmptyValues(), EmptyFactorGraph(), None
        img = batch["images"]
        if not torch.is_tensor(img):
            img = torch.as_tensor(np.asarray(img))
        imgs_k = img.to(self.device, non_blocking=True)[None].permute(0, 1, 4, 2, 3)   # H2D when host-resident

        if self.last_k is None:
            assert k == 0 and self.kf_idx == 0
            imgs_norm = self._normalize_imgs(imgs_k)
            self.initialize_buffers(imgs_k.shape[-2:])
            self._store_frame(0, batch, imgs_k)
            self._put_features(0, self._feature_encoder(imgs_norm))
            self.contexts_imgs[0], self.cst_contexts_imgs[0] = self._context_encoder(imgs_norm)
            self.last_k, self.last_kf_idx = k, 0
            self.kf_idx_to_f_idx[0] = k; self.f_idx_to_kf_idx[k] = 0
            viz_out = self.get_viz_out(batch)
            self.kf_idx += 1
            return x0, factors, viz_out

        assert k > 0 and self.kf_idx < self.buffer
        with _lib.fixed_stream():              # one stream lookup per frame instead of one per operator call (~14 us each)
            return self._forward_steady(batch, k, imgs_k, x0, factors, viz_out)

    def _forward_steady(self, batch, k, imgs_k, x0, factors, viz_out):
        with self.timers.section("frame.front issue"):
            feats = self._frame_front(imgs_k)          # feature encoder + motion filter (CUDA graph)
        with self.timers.section("frame.motion item (device wait)"):
            enough = self.last_motion.item() > self.motion_filter_thresh
        if not enough:
            if batch["is_last_frame"]:
                self.kf_idx -= 1
                self.terminate()
                viz_out = self.get_viz_out(batch)
            return x0, factors, viz_out

        self._store_frame(self.kf_idx, batch, imgs_k)
        self._put_features(self.kf_idx, feats)
        self._context_front(self.kf_idx)           # context encoder of the frame already in the static image buffer
        self.kf_idx_to_f_idx[self.kf_idx] = k; self.f_idx_to_kf_idx[k] = self.kf_idx

        if not self.is_initialized:
            if self.kf_idx >= self.keyframe_warmup:
                self._initialize()
        else:
            if not self._update():
                self.rm_keyframe(self.kf_idx - 1)
                self._prefetch_proximity()
                return x0, factors, viz_out

        self.last_k, self.last_kf_idx = k, self.kf_idx
        viz_out = self.get_viz_out(batch)
        if self.kf_idx + 1 >= self.buffer or batch["is_last_frame"]:
            self.terminate()
            viz_out = self.get_viz_out(batch)
            return x0, factors, viz_out
        self.kf_idx += 1
        self._prefetch_proximity()
        return x0, factors, viz_out

    __call__ = forward

    # ------------------------------------------------------------------ per-frame front (A1 + motion filter)
    def _frame_front_body(self):
        """device-only: static image buffer -> fnet -> motion filter (1 update iteration on
        (last keyframe -> current frame), visual_frontend.py:976-1007) -> self.last_motion"""
        from .conv import CORR_PAD
        with _lib.fixed_stream():
            self._frame_front_impl(CORR_PAD)

    def _frame_front_impl(self, CORR_PAD):
        imgs_norm = self._normalize_imgs(self._img_static)
        feats = self._feature_encoder(imgs_norm)                       # [cams,128,ht,wd]
        self._feats_cur.copy_(feats)
        idx = self._last_kf_d
        self._pair[0].copy_(self.features_imgs[:, 0].index_select(0, idx)[0])
        self._pair[1].copy_(feats[0].permute(1, 2, 0))
        pyr = db.corr_volume_build(self._pair, self._i32_0, self._i32_1)
        corr = db.corr_lookup_pyramid(pyr, self._coords0_b, 3, nhwc_stride=CORR_PAD, coords_nhwc=True)
        net = self.contexts_imgs[:, 0].index_select(0, idx)
        inp = self.cst_contexts_imgs[:, 0].index_select(0, idx)
        _, delta, _ = self._run_update_net(net, inp, corr, self._coords0_b, None)
        self.last_motion.copy_(delta.float().norm(dim=-1).mean())

    def _frame_front(self, imgs_k):
        """imgs_k [1,cams,C,H,W] uint8 on the device -> features [cams,128,ht,wd]; sets self.last_motion"""
        if self._img_static is None:
            dev = self.device
            self._img_static = torch.zeros_like(imgs_k)
            self._feats_cur = torch.zeros(self.cameras, 128, self.ht, self.wd, dtype=torch.float16, device=dev)
            self._pair = torch.zeros(2, self.ht, self.wd, 128, dtype=torch.float16, device=dev)
            self._last_kf_d = torch.zeros(1, dtype=torch.long, device=dev)
            self._i32_0 = torch.zeros(1, dtype=torch.int32, device=dev); self._i32_1 = torch.ones(1, dtype=torch.int32, device=dev)
            self._coords0_b = self.coords0[None].contiguous()
            self.last_motion = torch.zeros((), device=dev)
            self._front_graph, self._front_calls = None, 0
        self._img_static.copy_(imgs_k)
        self._last_kf_d.fill_(self.last_kf_idx)
        if self.use_cuda_graphs and self._front_calls >= 2:
            if self._front_graph is None:
                g = torch.cuda.CUDAGraph()
                cs = self._capture_stream
                cs.wait_stream(torch.cuda.current_stream())
                with torch.cuda.stream(cs):
                    g.capture_begin(pool=self._graph_pool)
                    self._frame_front_body()
                    g.capture_end()
                torch.cuda.current_stream().wait_stream(cs)
                self._front_graph = g
            self._front_graph.replay()
        else:
            self._frame_front_body()
        self._front_calls += 1
        return self._feats_cur

    def _context_front(self, slot):
        """context encoder (cnet) of the current frame — the image `_frame_front` left in the static buffer — into the
        keyframe arenas at `slot`.  Like the per-frame front it is a replayed CUDA graph (26 launches, one host call)."""
        if not hasattr(self, "_ctx_cur"):
            self._ctx_cur = torch.zeros(self.cameras, self.ht, self.wd, 128, dtype=torch.float16, device=self.device)
            self._inp_cur = torch.zeros_like(self._ctx_cur)
            self._ctx_graph, self._ctx_calls = None, 0

        def body():
            with _lib.fixed_stream():
                c, g = self._context_encoder(self._normalize_imgs(self._img_static))
                self._ctx_cur.copy_(c); self._inp_cur.copy_(g)
        if self.use_cuda_graphs and self._ctx_calls >= 2:
            if self._ctx_graph is None:
                gr = torch.cuda.CUDAGraph()
                cs = self._capture_stream
                cs.wait_stream(torch.cuda.current_stream())
                with torch.cuda.stream(cs):
                    gr.capture_begin(pool=self._graph_pool)
                    body()
                    gr.capture_end()
                torch.cuda.current_stream().wait_stream(cs)
                self._ctx_graph = gr
            self._ctx_graph.replay()
        else:
            body()
        self._ctx_calls += 1
        self.contexts_imgs[slot] = self._ctx_cur
        self.cst_contexts_imgs[slot] = self._inp_cur

    def has_enough_motion(self, feats=None):
        return self.last_motion.item() > self.motion_filter_thresh

    # ------------------------------------------------------------------ graph management (A18)
    def add_neighborhood_factors(self, kf0, kf1, radius=3):
        """visual_frontend.py:690-708 (keyframes kf0..kf1 inclusive)"""
        self.add_factors(*neighborhood_edges(kf0, kf1 + 1, radius, self.stereo))

    def distance(self, ii, jj, beta=0.3, bidirectional=True):
        """visual_frontend.py:778-799"""
        ii = _lib.h2d(np.asarray(ii).reshape(-1), self.device, torch.long)
        jj = _lib.h2d(np.asarray(jj).reshape(-1), self.device, torch.long)
        if bidirectional:
            poses = self.cam0_T_world[:self.kf_idx + 1].clone()
            d1 = db.frame_distance(poses, self.cam0_idepths, self.cam0_intrinsics[0], ii, jj, beta)
            d2 = db.frame_distance(poses, self.cam0_idepths, self.cam0_intrinsics[0], jj, ii, beta)
            return .5 * (d1 + d2)
        return db.frame_distance(self.cam0_T_world, self.cam0_idepths, self.cam0_intrinsics[0], ii, jj, beta)

    def add_proximity_factors(self, kf0=0, kf1=0, rad=2, nms=2, beta=0.25, thresh=16.0, remove=False):
        """visual_frontend.py:712-775 — the order-sensitive edge selection (SURVEY.md §9.20);
        the selection logic is kept loop for loop, on the host copy of the distances."""
        t = self.kf_idx + 1
        ix = np.arange(kf0, t); jx = np.arange(kf1, t)
        ii, jj = np.meshgrid(ix, jx, indexing="ij")
        ii, jj = ii.reshape(-1), jj.reshape(-1)
        with self.timers.section("prox.distance + cpu (device wait)"):
            d = self._take_prefetched_distances(kf0, kf1, t, beta)
            if d is None:
                d = self.distance(ii, jj, beta=beta).cpu().numpy().copy()
        with self.timers.section("prox.selection (host)"):
            es = proximity_edges(d, ii, jj, *self.edges.known(), kf0, kf1, t, rad, nms, thresh, self.max_factors, self.stereo)
        if es.shape[0] == 0:
            return
        with self.timers.section("prox.add_factors"):
            self.add_factors(es[:, 0], es[:, 1], remove)

    # The pairwise distances of the NEXT keyframe candidate's proximity search depend only on poses / inverse depths
    # that are final once the current candidate has been processed (the new slot's initial guess is written at the end
    # of __update / __initialize; a rejected candidate ends with rm_keyframe).  They are therefore computed and copied
    # to pinned host memory asynchronously at the end of forward(), behind the updates still queued on the stream,
    # and are simply there when the next candidate arrives: no device round trip in front of the edge selection.
    # `_state_version` guards the cache: anything that changes poses or depths after the prefetch invalidates it.
    def _touch_state(self):
        self._state_version = getattr(self, "_state_version", 0) + 1

    def _prefetch_proximity(self):
        if not self.is_initialized or self.kf_idx >= self.buffer or not self.cam0_T_world.is_cuda:
            self._prox_prefetch = None
            return
        k = self.kf_idx
        kf0, kf1, t = k - 4, max(k + 1 - self.frontend_window, 0), k + 1
        ii, jj = np.meshgrid(np.arange(kf0, t), np.arange(kf1, t), indexing="ij")
        d = self.distance(ii.reshape(-1), jj.reshape(-1), beta=self.beta)
        n = d.numel()
        if getattr(self, "_prox_host", None) is None or self._prox_host.numel() < n:
            self._prox_host = torch.empty(max(n, 1024), dtype=torch.float32).pin_memory()
        self._prox_host[:n].copy_(d, non_blocking=True)
        ev = torch.cuda.Event()
        ev.record()
        self._prox_prefetch = (getattr(self, "_state_version", 0), (kf0, kf1, t, float(self.beta)), n, ev)

    def _take_prefetched_distances(self, kf0, kf1, t, beta):
        pf, self._prox_prefetch = getattr(self, "_prox_prefetch", None), None
        if pf is None or pf[0] != getattr(self, "_state_version", 0) or pf[1] != (kf0, kf1, t, float(beta)):
            return None
        pf[3].synchronize()
        return self._prox_host[:pf[2]].numpy().copy()

    def add_factors(self, ii, jj, remove=False):
        """visual_frontend.py:807-862"""
        ii = np.asarray(ii, np.int64).reshape(-1); jj = np.asarray(jj, np.int64).reshape(-1)
        ii, jj = self.edges.filter_repeated(ii, jj)
        new = ii.shape[0]
        if new == 0:
            return
        if remove and self.gru_hidden_states is not None:
            self.rm_factors(self.edges.retire_mask(new, self.max_factors), store=True)
        slots = np.zeros(new, np.int64)
        if self.corr_impl == "volume":
            slots = np.asarray(self.corr_pool.alloc(new), np.int64)
            cams = self.cameras
            fi = (ii * cams).tolist()
            fj = (jj * cams + (ii == jj)).tolist()
            fm = self.features_imgs.view(self.buffer * cams, self.ht, self.wd, 128)
            self.corr_pool.build(fm, fi, fj, slots.tolist())
        hid = self.contexts_imgs[_lib.h2d(ii, self.device), 0]
        target, _ = self.reproject(ii, jj)
        self.edges.append(ii, jj, slots, hid, target, torch.zeros_like(target))
        self._sync_edges()

    def rm_factors(self, mask, store=False):
        """visual_frontend.py:868-892; mask: host bool array over the active edges"""
        mask = np.asarray(mask, dtype=bool)
        if not mask.any():
            return
        slots = self.edges.remove(mask, store)
        if self.corr_impl == "volume":
            self.corr_pool.release(slots.tolist())
        self._sync_edges()

    def rm_keyframe(self, kf):
        """visual_frontend.py:530-574"""
        self._touch_state()
        for buf in (self.gt_poses, self.gt_depths, self.cam0_images, self.cam0_timestamps, self.cam0_T_world,
                    self.world_T_body, self.world_T_body_cov, self.cam0_idepths, self.cam0_idepths_cov,
                    self.cam0_depths_cov, self.cam0_idepths_sensed, self.cam0_intrinsics, self.features_imgs,
                    self.contexts_imgs, self.cst_contexts_imgs):
            buf[kf] = buf[kf + 1]
        m = self.edges.remove_keyframe(kf)
        if m.any():
            self.rm_factors(m, store=False)
        else:
            self._sync_edges()          # indices above kf moved down: the device copies must follow even if no edge leaves

    def reproject(self, ii, jj):
        """visual_frontend.py:909-918 -> coords [E,ht,wd,2], valid"""
        ii = ii.to(self.device, torch.long).reshape(-1) if torch.is_tensor(ii) else _lib.h2d(np.asarray(ii).reshape(-1), self.device, torch.long)
        jj = jj.to(self.device, torch.long).reshape(-1) if torch.is_tensor(jj) else _lib.h2d(np.asarray(jj).reshape(-1), self.device, torch.long)
        return db.reproject(self.cam0_T_world, self.cam0_idepths, self.cam0_intrinsics, ii, jj)

    # ------------------------------------------------------------------ init / steady state
    def _initialize(self):
        """visual_frontend.py:641-688"""
        assert self.kf_idx > 4 and self.kf_idx >= self.keyframe_warmup
        self.add_neighborhood_factors(0, self.kf_idx, radius=3)
        for _ in range(8):
            self.update(use_inactive=True)
        self.add_proximity_factors(kf0=0, kf1=0, rad=2, nms=2, thresh=self.frontend_thresh, remove=False)
        for _ in range(8):
            self.update(use_inactive=True)
        k = self.kf_idx
        self._touch_state()
        self.cam0_T_world[k + 1] = self.cam0_T_world[k].clone()
        self.world_T_body[k + 1] = self.world_T_body[k].clone()
        self.world_T_body_cov[k + 1] = self.world_T_body_cov[k].clone()
        self.cam0_idepths[k + 1] = self.cam0_idepths[k - 3:k + 1].mean()
        self.cam0_idepths_cov[k + 1] = self.cam0_idepths_cov[k - 3:k + 1].mean()
        self.cam0_depths_cov[k + 1] = self.cam0_depths_cov[k - 3:k + 1].mean()
        self.is_initialized = True
        self.viz_idx[:k + 1] = True
        self.rm_factors(self.ii_h < (self.keyframe_warmup - 4), store=True)

    def _update(self):
        """visual_frontend.py:577-638"""
        T = self.timers.section
        with T("kf.rm_factors(age)"):
            if self.gru_hidden_states is not None:
                self.rm_factors(self.age_h > self.max_age, store=True)
        with T("kf.add_proximity_factors"):
            self.add_proximity_factors(kf0=self.kf_idx - 4, kf1=max(self.kf_idx + 1 - self.frontend_window, 0),
                                       rad=self.frontend_radius, nms=self.frontend_nms,
                                       thresh=self.frontend_thresh, beta=self.beta, remove=True)
        k = self.kf_idx
        self._touch_state()
        self.cam0_idepths[k] = torch.where(self.cam0_idepths_sensed[k] > 0, self.cam0_idepths_sensed[k], self.cam0_idepths[k])
        with T("kf.updates iters1 (host issue)"):
            for _ in range(self.iters1):
                self.update(use_inactive=True)
        with T("kf.distance + item (device wait)"):
            d = self.distance([k - 2], [k - 1], beta=self.beta, bidirectional=True)
            dv = d.item()
        if dv < self.keyframe_thresh:
            return False
        with T("kf.updates iters2 (host issue)"):
            for _ in range(self.iters2):
                self.update(use_inactive=True)
        nk = k + 1
        self._touch_state()
        if nk < self.buffer:
            self.cam0_T_world[nk] = self.cam0_T_world[k]
            self.world_T_body[nk] = self.world_T_body[k]
            self.world_T_body_cov[nk] = self.world_T_body_cov[k]
            self.cam0_idepths[nk] = self.cam0_idepths[k].mean()
            self.cam0_idepths_cov[nk] = self.cam0_idepths_cov[k]
            self.cam0_depths_cov[nk] = self.cam0_depths_cov[k]
        return True

    # ------------------------------------------------------------------ the hot loop (A19)
    def _prepare_static(self, use_inactive, EP):
        """Everything of update() that depends only on the EDGE SET (not on the evolving state) is
        computed once here: device index tensors, gathered GRU inputs, the BA window (graph tables,
        buffers) with the stored flows of the inactive edges already in place.  The per-call body
        (_update_body) then issues only device work on these fixed buffers, for each of the 4+2 (or 8+8)
        updates that share the edge set."""
        import types
        dev, ht, wd = self.device, self.ht, self.wd
        st = types.SimpleNamespace()
        ii_h, jj_h = self.ii_h, self.jj_h
        kf0 = max(0, int(ii_h.min()))
        st.kf0, st.EP = kf0, EP
        ux, inv = np.unique(ii_h, return_inverse=True)
        st.ux = _lib.h2d(ux, dev); st.ix = _lib.h2d(inv, dev); st.K = len(ux)
        st.agg = agg_tables(ii_h, dev)
        st.op_ctx = None
        st.inp = self.cst_contexts_imgs[self.ii, 0].contiguous()
        if use_inactive:
            m = (self.ii_inactive_h >= kf0 - 3) & (self.jj_inactive_h >= kf0 - 3)
            md = _lib.h2d(np.nonzero(m)[0], dev)                   # integer indices: no device->host sync
            ii = np.concatenate([self.ii_inactive_h[m], ii_h]); jj = np.concatenate([self.jj_inactive_h[m], jj_h])
            tin = self.gru_estimated_flow_inactive.index_select(0, md); win = self.gru_estimated_flow_weight_inactive.index_select(0, md)
        else:
            ii, jj = ii_h, jj_h
            tin = win = torch.zeros(0, ht, wd, 2, device=dev)
        st.n_in = int(tin.shape[0])
        Eba = len(ii)
        st.target = torch.empty(Eba, 2, ht, wd, device=dev); st.weight = torch.empty(Eba, 2, ht, wd, device=dev)
        st.target[:st.n_in] = tin.permute(0, 3, 1, 2); st.weight[:st.n_in] = win.permute(0, 3, 1, 2)
        kxb = np.unique(ii)
        st.kx_ba = _lib.h2d(kxb, dev)
        st.damp = torch.empty(len(kxb), ht, wd, device=dev)
        kf1 = int(max(ii.max(), jj.max())) + 1
        st.kf1 = kf1
        st.prob = db.BAProblem(self.cam0_T_world, self.cam0_idepths, self.intr0, self.cam0_T_body,
                               self.cam0_idepths_sensed, st.target, st.weight, st.damp, ii, jj, kf0, kf1)
        st.has_prior = self.kf_idx_to_f_idx.get(kf0, -1) == 0
        if self.use_op_step:
            # the whole update operator as one host call on fixed buffers (csrc/update_step.cu)
            E = int(self.ii.shape[0])
            c, st.op_ws = self.update_tc.make_step(E, st.K, ht, wd, dev)
            st.coords1 = torch.empty(E, ht, wd, 2, device=dev)
            st.corr = torch.zeros(E, ht, wd, CORR_PAD_, dtype=torch.float16, device=dev)
            st.upmask = torch.empty(st.K, ht, wd, 576, dtype=torch.float16, device=dev)
            c.net = c.net_out = self.gru_hidden_states.data_ptr()
            c.inp, c.corr, c.coords1, c.coords0 = st.inp.data_ptr(), st.corr.data_ptr(), st.coords1.data_ptr(), self.coords0.data_ptr()
            c.target = c.flow = self.gru_estimated_flow.data_ptr()
            c.conf = self.gru_estimated_flow_weight.data_ptr()
            c.ba_target, c.ba_weight = st.target[st.n_in:].data_ptr(), st.weight[st.n_in:].data_ptr()
            c.seg_ptr, c.seg_edges = st.agg[0].data_ptr(), st.agg[1].data_ptr()
            c.upmask = st.upmask.data_ptr()
            c.ux, c.damping, c.kx_ba, c.ba_damp = st.ux.data_ptr(), self.damping.data_ptr(), st.kx_ba.data_ptr(), st.damp.data_ptr()
            c.Kba, c.ep = int(st.kx_ba.numel()), float(EP)
            st.op_ctx = c
        return st

    def _update_body(self, st, itrs, compute_covariances):
        """device-only part of update() (visual_frontend.py:371-470); no host<->device traffic, no syncs"""
        with _lib.fixed_stream():
            self._update_body_impl(st, itrs, compute_covariances)

    def _update_body_impl(self, st, itrs, compute_covariances):
        if st.op_ctx is not None:
            db.reproject(self.cam0_T_world, self.cam0_idepths, self.cam0_intrinsics, self.ii, self.jj, want_valid=False,
                         out=st.coords1)
            self.corr_pool.lookup(self.slots_d, st.coords1, nhwc=True, out=st.corr)
            self.update_tc.step(st.op_ctx)          # hidden state, flow, confidence, BA inputs, damping: all in place
            upmask = st.upmask
            coords1 = None
        else:
            coords1, _ = db.reproject(self.cam0_T_world, self.cam0_idepths, self.cam0_intrinsics, self.ii, self.jj, want_valid=False)
            corr = self.corr_pool.lookup(self.slots_d, coords1, nhwc=True)          # [E,ht,wd,CORR_PAD] fp16
        if st.op_ctx is None and self.update_tc is None:
            # test harness only (tests/test_cpu_droid.py replays the reference's update() traces on the CPU with a stand-in
            # operator in `_run_update_net`; the constructor never selects this): the bookkeeping of
            # visual_frontend.py:390-452 spelled out in tensor ops — what the fused kernels below do in place
            net, delta, weight, damping, upmask = self._run_update_net(self.gru_hidden_states, st.inp, corr, coords1,
                                                                       self.gru_estimated_flow, self.ii_h)
            self.gru_hidden_states.copy_(net)
            torch.add(coords1, delta, out=self.gru_estimated_flow)
            self.gru_estimated_flow_weight.copy_(weight)
            self.damping[st.ux] = damping
            st.target[st.n_in:].copy_(self.gru_estimated_flow.permute(0, 3, 1, 2))
            st.weight[st.n_in:].copy_(self.gru_estimated_flow_weight.permute(0, 3, 1, 2))
            torch.mul(self.damping[st.kx_ba], 0.2, out=st.damp)
            st.damp.add_(st.EP)
        elif st.op_ctx is None:
            # the same operator sequenced from Python (kept for the test that ties the fused C call to this sequencing):
            # flow/confidence land directly in the frontend state AND in the BA's planar input buffers
            net, _, _, e16, upmask = self.update_tc(
                self.gru_hidden_states, st.inp, corr, coords1, self.coords0, target=self.gru_estimated_flow, agg=st.agg,
                post=(self.gru_estimated_flow, self.gru_estimated_flow_weight, st.target[st.n_in:], st.weight[st.n_in:]))
            self.gru_hidden_states.copy_(net)
            _lib.check(_lib.load().nslam_eta_damping(_lib.ptr(e16), _lib.ptr(st.ux), _lib.ptr(self.damping), st.K,
                                                     _lib.ptr(st.kx_ba), _lib.ptr(st.damp), int(st.kx_ba.numel()),
                                                     self.ht * self.wd, float(st.EP), _lib.stream_ptr()), "eta_damping")
        # the whole BA step (2 Gauss-Newton iterations + covariance block) is one host call; results land in place
        # in the pose / depth / covariance arenas; a failed factorisation changes nothing and bumps _ba_status[1]
        st.prob.frontend_update(itrs, self.world_T_body, self.cam0_T_world, self.cam0_T_body, self._ba_status,
                                prior_idx=0 if st.has_prior else -1,
                                prior_pose=self.prior_pose if st.has_prior else None,
                                prior_info=self.prior_info if st.has_prior else 0.0, clamp_min=1e-3,
                                cov_mode=self.cov_mode if compute_covariances else None,
                                idepths_cov=self.cam0_idepths_cov, depths_cov=self.cam0_depths_cov,
                                pose_cov=self.world_T_body_cov)
        # inverse depths and depth covariances of the K source keyframes through one softmax, gathered /
        # scattered by keyframe index inside the kernel
        db.cvx_upsample2(self.cam0_idepths, self.cam0_depths_cov, upmask, self.cam0_idepths_up, self.cam0_depths_cov_up,
                         index=st.ux)

    @torch.no_grad()
    def update(self, kf0=None, kf1=None, itrs=2, use_inactive=False, EP=1e-7, motion_only=False):
        """visual_frontend.py:371-470.  The first call after an edge-set change prepares the static part
        (index tables, BA window, operator workspace); every call then issues ~10 host calls (reproject,
        lookup, nslam_update_op_step, BA Gauss-Newton, covariances, upsample)."""
        st = self._static
        if st is None or st.use_inactive != use_inactive:
            with self.timers.section("update.prepare_static"):
                st = self._prepare_static(use_inactive, EP)
            st.use_inactive = use_inactive
            self._static = st
        self._update_body(st, itrs, self.compute_covariances)
        self._touch_state()
        self.viz_idx[st.kf0:self.kf_idx + 1] = True
        self.age_h += 1
        self.stats["updates"] += 1
        self.last_ba = st.prob

    def ba(self, target, weight, damping, ii, jj, kf0=0, kf1=None, itrs=2, lm=1e-4, ep=0.1,
           motion_only=False, compute_covariances=True):
        """dense bundle adjustment (visual_frontend.py:1071-1232) — all on the device stream.
        `lm`, `ep` are accepted and unused, exactly like the reference's live path."""
        ii = np.asarray(ii, np.int64); jj = np.asarray(jj, np.int64)
        if kf1 is None:
            kf1 = int(max(ii.max(), jj.max())) + 1
        prob = db.BAProblem(self.cam0_T_world, self.cam0_idepths, self.intr0, self.cam0_T_body,
                            self.cam0_idepths_sensed, target, weight, damping, ii, jj, kf0, kf1)
        has_prior = self.kf_idx_to_f_idx.get(kf0, -1) == 0
        self._touch_state()
        prob.frontend_update(itrs, self.world_T_body, self.cam0_T_world, self.cam0_T_body, self._ba_status,
                             prior_idx=0 if has_prior else -1, prior_pose=self.prior_pose if has_prior else None,
                             prior_info=self.prior_info if has_prior else 0.0, clamp_min=1e-3,
                             cov_mode=self.cov_mode if compute_covariances else None,
                             idepths_cov=self.cam0_idepths_cov, depths_cov=self.cam0_depths_cov,
                             pose_cov=self.world_T_body_cov)
        self.last_ba = prob
        return None, None

    # ------------------------------------------------------------------ global BA (backend)
    def normalize(self, last_kf=-1):
        self._touch_state()
        s = self.cam0_idepths[:last_kf].mean()
        self.cam0_idepths[:last_kf] /= s
        self.cam0_T_world[:last_kf, :3] *= s
        self.viz_idx[:last_kf] = True

    def clear_edges(self):
        self.rm_factors(self.ii_h >= 0)
        self.gru_hidden_states = None

    @torch.no_grad()
    def update_lowmem(self, itrs=2, EP=1e-7, steps=8):
        """visual_frontend.py:474-526: global-BA path — correlation features computed on the fly (alt-corr, no stored
        volumes), edges processed in chunks of 8 source frames, then one BA over the whole window per step.
        Chunk membership and all gather / scatter indices are built on the host (the edge list lives there): no boolean
        device masks, no device synchronisation inside the loop.  Rows of the damping / upsampling maps of a chunk are
        its unique SOURCE frames (DROID's semantics, networks/factor_graph.py:259-303; see DESIGN.md on the reference's
        own variant, which raises)."""
        from .conv import CORR_PAD
        dev, cams = self.device, self.cameras
        fm = self.features_imgs.permute(0, 1, 4, 2, 3).reshape(1, self.buffer * cams, 128, self.ht, self.wd)
        corr_op = AltCorrBlock(fm)
        ii_h, jj_h = self.ii_h, self.jj_h
        s = 8
        chunks = []
        for i in range(0, int(jj_h.max()) + 1, s):
            sel = np.nonzero((ii_h >= i) & (ii_h < i + s))[0]
            if sel.size:
                iis, jjs = ii_h[sel], jj_h[sel]
                chunks.append(types_ns(sel=_lib.h2d(sel, dev), iis_h=iis, iis=_lib.h2d(iis, dev),
                                       fi=_lib.h2d(cams * iis, dev), fj=_lib.h2d(cams * jjs + (iis == jjs), dev),
                                       kx=_lib.h2d(np.unique(iis), dev)))
        ux_all = _lib.h2d(np.unique(ii_h), dev)
        for _ in range(steps):
            coords1, _ = self.reproject(self.ii, self.jj)
            for c in chunks:
                c1 = coords1.index_select(0, c.sel)
                corr = corr_op(c1[None], c.fi, c.fj)[0]                                  # [e,196,ht,wd] fp32
                corr = torch.nn.functional.pad(corr.permute(0, 2, 3, 1), (0, CORR_PAD - 196)).half().contiguous()
                net, delta, weight, damping, upmask = self._run_update_net(
                    self.gru_hidden_states.index_select(0, c.sel), self.cst_contexts_imgs[:, 0].index_select(0, c.iis),
                    corr, c1.contiguous(), self.gru_estimated_flow.index_select(0, c.sel), c.iis_h)
                self.gru_hidden_states.index_copy_(0, c.sel, net)
                self.gru_estimated_flow.index_copy_(0, c.sel, c1 + delta)
                self.gru_estimated_flow_weight.index_copy_(0, c.sel, weight)
                self.damping.index_copy_(0, c.kx, damping)
                up = db.cvx_upsample(self.cam0_idepths.index_select(0, c.kx).unsqueeze(-1), upmask, mask_nhwc=True).squeeze(-1)
                self.cam0_idepths_up.index_copy_(0, c.kx, up)
                upc = db.cvx_upsample(self.cam0_depths_cov.index_select(0, c.kx).unsqueeze(-1), upmask, mask_nhwc=True).squeeze(-1)
                self.cam0_depths_cov_up.index_copy_(0, c.kx, upc)
            dmp = (.2 * self.damping.index_select(0, ux_all) + EP).contiguous()
            target = self.gru_estimated_flow.permute(0, 3, 1, 2).contiguous()
            wgt = self.gru_estimated_flow_weight.permute(0, 3, 1, 2).contiguous()
            self.ba(target, wgt, dmp, ii_h, jj_h, kf0=0, kf1=None, itrs=itrs, compute_covariances=False)

    def backend(self, steps=12):
        """visual_frontend.py:1255-1306"""
        if not self.stereo and not torch.any(self.cam0_idepths_sensed):
            self.normalize(self.kf_idx)
        self.max_factors = 16 * self.kf_idx
        self.corr_impl = "alt"
        self._reset_graph()
        self.add_proximity_factors(rad=self.backend_radius, nms=self.backend_nms, thresh=self.backend_thresh, beta=self.beta)
        self.update_lowmem(steps=steps)
        self.clear_edges()
        self.viz_idx[:self.kf_idx] = True

    def terminate(self):
        """visual_frontend.py:1308-1335"""
        if self.global_ba:
            self.backend(7)
            self.backend(12)
            self.backend(0)
        self.stop = True

    # ------------------------------------------------------------------ output packet (B1 contract)
    def get_viz_out(self, batch):
        """visual_frontend.py:1337-1391.  Tensors stay on the device: the NeRF side receives them
        through NCCL / peer copies (nerf_slam_b200.dist), never through the CPU."""
        self.ba_failures()                      # asynchronous read-back of the BA failure counter (no sync)
        idx_h = np.nonzero(self.viz_idx)[0]
        if len(idx_h) == 0:
            return {"is_last_frame": True} if batch["is_last_frame"] else None
        idx = _lib.h2d(idx_h, self.device)
        sel = lambda t: torch.index_select(t, 0, idx)
        out = {"cam0_poses": sel(self.cam0_T_world), "gt_poses": sel(self.gt_poses), "gt_depths": sel(self.gt_depths),
               "world_T_body": sel(self.world_T_body), "world_T_body_cov": sel(self.world_T_body_cov),
               "cam0_idepths": sel(self.cam0_idepths), "cam0_idepths_up": sel(self.cam0_idepths_up),
               "cam0_idepths_sensed": sel(self.cam0_idepths_sensed), "cam0_idepths_cov": sel(self.cam0_idepths_cov),
               "cam0_depths_cov": sel(self.cam0_depths_cov), "cam0_depths_cov_up": sel(self.cam0_depths_cov_up),
               "cam0_images": sel(self.cam0_images), "cam0_intrinsics": sel(self.cam0_intrinsics),
               "calibs": batch["calibs"], "viz_idx": idx, "viz_idx_host": idx_h.tolist(), "kf_idx": self.kf_idx,
               "kf_idx_to_f_idx": dict(self.kf_idx_to_f_idx), "is_last_frame": batch["is_last_frame"]}
        self.viz_idx[:] = False
        return out

    def point_cloud(self, mask_type="uncertainty", voxel_size=None, filter_thresh=None, min_views=2, max_depth=6.0,
                    max_depth_sigma=10.0):
        """every keyframe the buffer holds as one coloured point cloud (point_cloud.build_point_cloud; the reference
        GUI's build_pcls, gui/open3d_gui.py:646-678, whose defaults max_depth 6 and max_depth_sigma_thresh 10 are kept)
        -> PointCloud, or None.  Reads the arenas in place (cam0_T_world, cam0_idepths_up, cam0_depths_cov_up,
        cam0_images, dsf * cam0_intrinsics[0]) on the current stream; the only host reads are the point and voxel
        counts.  mask_type "uncertainty" (the demo's --mask_type ours) or "uniform"."""
        from .point_cloud import build_point_cloud
        if mask_type not in ("uncertainty", "uniform"):
            raise ValueError(f"Unknown depth mask type: {mask_type}")
        if not hasattr(self, "cam0_T_world"):
            return None
        n = min(self.kf_idx + 1 if self.stop else self.kf_idx, self.buffer)    # slot kf_idx is the next keyframe's until stop
        packet = {"cam0_poses": self.cam0_T_world[:n], "cam0_idepths_up": self.cam0_idepths_up[:n],
                  "cam0_depths_cov_up": self.cam0_depths_cov_up[:n] if mask_type == "uncertainty" else None,
                  "cam0_images": self.cam0_images[:n]}
        return build_point_cloud(packet, self.dsf * self.cam0_intrinsics[0], max_depth=max_depth,
                                 max_depth_sigma=max_depth_sigma, filter_thresh=filter_thresh, min_views=min_views,
                                 voxel_size=voxel_size)
