"""ORACLE / reference arm (test + measurement infrastructure only — never imported by the product path).

`RefCudaFrontend`: the reference's OWN CUDA build of Path A, re-assembled so that it runs in this image, for
`bench.py --impl reference-cuda` (frames/s of the same synthetic stream, next to the product's) and for A/B tests.

What executes:
  * the reference's own CUDA kernels, compiled unmodified from /root/reference/src by oracle/build_ref.py into
    oracle/_ref/*.so: corr_index_forward_kernel (A3), projective_transform / accum / EEt6x6 / Ev6x1 / EvT6x1 /
    disp_retr kernels (A7-A11, A13), frame_distance_kernel (A16);
  * library PyTorch for everything the reference itself runs through PyTorch: BasicEncoder / UpdateModule / ConvGRU /
    GraphAgg as cuDNN fp16 convolutions (its autocast path, visual_frontend.py:370,950-959), CorrBlock's
    `torch.matmul` + 3x `avg_pool2d` and its `torch.cat` pool (networks/modules/corr.py:23-72), the covariance block as
    dense torch ops (visual_frontend.py:1164-1230), cvx_upsample with `F.unfold` (utils/flow_viz.py:166-183);
  * the reference's sequencing of update() / ba() (visual_frontend.py:371-470, 1071-1232) and its graph management
    (inherited host logic, pinned bit for bit against the reference's traces).
What is FAVOURABLE to the reference (absent third-party code replaced by something at least as fast):
  * gtsam: the Python loop that builds one HessianFactor per 6x6 block with a `.cpu().numpy()` each (:1127-1133,
    "this is quite slow") + optimizeDensely + retract becomes ONE device->host copy of H, v, a dense fp64 Cholesky on the
    host and a vectorised numpy retraction;
  * lietorch: `pops.projective_transform` with Jacobians (~30 small kernels, :377-380) becomes this repo's single
    reprojection kernel;
  * torch_scatter -> index_add_.
No CUDA graphs, no fused operator, no arenas: what is measured is the reference's launch / synchronisation structure
with its own kernels, on the same GPU.
"""
import numpy as np
import torch
import torch.nn.functional as F

from nerf_slam_b200 import _lib
from nerf_slam_b200 import droid_backends as db
from nerf_slam_b200.frontend import RaftVisualFrontend
from oracle import build_ref, se3


def cvx_upsample_torch(data, mask, pow=1.0):
    """utils/flow_viz.py:166-183 restated: data [K,ht,wd,1], mask [K,576,ht,wd] -> [K,8ht,8wd,1]"""
    batch, ht, wd, dim = data.shape
    data = data.permute(0, 3, 1, 2)
    mask = mask.view(batch, 1, 9, 8, 8, ht, wd).clone()
    mask[:, :, [0, 1, 2], :, :, 0, :] = -float("inf")       # border handling (:172-177)
    mask[:, :, [6, 7, 8], :, :, -1, :] = -float("inf")
    mask[:, :, [0, 3, 6], :, :, :, 0] = -float("inf")
    mask[:, :, [2, 5, 8], :, :, :, -1] = -float("inf")
    mask = torch.softmax(mask, dim=2)
    mask = torch.pow(mask, pow)
    up = F.unfold(data, [3, 3], padding=1).view(batch, dim, 9, 1, 1, ht, wd)
    up = torch.sum(mask * up, dim=2).permute(0, 4, 2, 5, 3, 1)
    return up.reshape(batch, 8 * ht, 8 * wd, dim)


class RefCorrPool:
    """CorrBlock + `.cat` + `__getitem__` (networks/modules/corr.py:23-60): four tensors [n,h,w,h>>l,w>>l] that are
    re-concatenated on every add and mask-indexed on every removal; lookup = the reference kernel per level"""

    def __init__(self, ht, wd, device, refcorr):
        self.ht, self.wd, self.device, self.ref = ht, wd, device, refcorr
        self.pyr, self.ids, self._next = None, [], 0
        self.free, self.capacity = [], 0

    def alloc(self, n):
        ids = list(range(self._next, self._next + n))
        self._next += n
        return ids

    def build(self, fm, fi, fj, slots):
        dev = self.device
        f1 = fm[torch.as_tensor(fi, device=dev)].permute(0, 3, 1, 2)           # [n,128,h,w] fp16
        f2 = fm[torch.as_tensor(fj, device=dev)].permute(0, 3, 1, 2)
        n, c, h, w = f1.shape
        corr = torch.matmul((f1 / 4.0).reshape(n, c, h * w).transpose(1, 2), (f2 / 4.0).reshape(n, c, h * w))
        corr = corr.view(n * h * w, 1, h, w)
        new = []
        for i in range(4):
            new.append(corr.view(n, h, w, h // 2 ** i, w // 2 ** i))
            corr = F.avg_pool2d(corr, 2, stride=2)
        self.pyr = new if self.pyr is None else [torch.cat([a, b], 0) for a, b in zip(self.pyr, new)]
        self.ids += list(slots)

    def release(self, slots):
        drop = set(int(s) for s in slots)
        keep = torch.as_tensor([i not in drop for i in self.ids], device=self.device)
        self.pyr = [p[keep] for p in self.pyr]
        self.ids = [i for i in self.ids if i not in drop]

    def lookup(self, slots_d, coords1, nhwc=True, out=None):
        """coords1 [n,h,w,2] -> [n,196,h,w] (CorrBlock.__call__, corr.py:40-50)"""
        c = coords1.permute(0, 3, 1, 2).contiguous()
        outs = []
        for i in range(4):
            o, = self.ref.corr_index_forward(self.pyr[i], (c / 2 ** i).contiguous(), 3)
            outs.append(o.view(o.shape[0], -1, self.ht, self.wd))
        return torch.cat(outs, 1)


class RefCudaFrontend(RaftVisualFrontend):
    def __init__(self, world_T_body_t0, body_T_cam0, args, device="cuda:0"):
        super().__init__(world_T_body_t0, body_T_cam0, args, device)
        self.refcorr = build_ref.load("nslam_ref_corr")
        self.refdroid = build_ref.load("nslam_ref_droid")
        if self.refcorr is None or self.refdroid is None:
            raise RuntimeError("oracle/_ref/*.so not built (python -m oracle.build_ref in the build container)")
        self.update_tc = self.feature_tc = self.context_tc = None      # library convolutions (cuDNN, fp16)
        self.use_cuda_graphs = self.use_op_step = False
        torch.backends.cudnn.benchmark = True

    # ---- buffers: the reference's growing correlation pool instead of the slot arena
    def initialize_buffers(self, image_size):
        super().initialize_buffers(image_size)
        self.corr_pool = RefCorrPool(self.ht, self.wd, self.device, self.refcorr)

    def _reset_graph(self):
        super()._reset_graph()
        if isinstance(getattr(self, "corr_pool", None), RefCorrPool):
            self.corr_pool = RefCorrPool(self.ht, self.wd, self.device, self.refcorr)

    def _prefetch_proximity(self):
        self._prox_prefetch = None           # the reference computes the distances when it needs them (:745)

    # ---- networks through the library
    def _feature_encoder(self, imgs_norm):
        return self.feature_net(imgs_norm)[0]

    def _context_encoder(self, imgs_norm):
        c = self.context_net(imgs_norm)[0].permute(0, 2, 3, 1)
        return torch.tanh(c[..., :128]), torch.relu(c[..., 128:])

    def _net(self, net, inp, corr196, coords1, target, ii_host=None):
        """UpdateModule.forward on the reference's layouts; state stays channels-last in the base class"""
        tgt = coords1 if target is None else target
        motion = torch.cat([coords1 - self.coords0, tgt - coords1], dim=-1).permute(0, 3, 1, 2).clamp(-64.0, 64.0)
        nchw = lambda t: t.permute(0, 3, 1, 2)
        ii = None if ii_host is None else torch.as_tensor(np.asarray(ii_host), device=self.device)
        out = self.update_net(nchw(net)[None], nchw(inp)[None], corr196[None], motion[None], ii, ii)
        net2 = out[0][0].permute(0, 2, 3, 1).contiguous()
        if ii is None:
            return net2, out[1][0].float(), out[2][0].float()
        return net2, out[1][0].float(), out[2][0].float(), out[3][0].float(), out[4][0]

    # ---- per-frame front (motion filter, visual_frontend.py:976-1007), eager
    def _frame_front(self, imgs_k):
        self._img_static = imgs_k                                               # the base class' context encoder reads it
        feats = self._feature_encoder(self._normalize_imgs(imgs_k))             # [cams,128,ht,wd]
        k = self.last_kf_idx
        pool = RefCorrPool(self.ht, self.wd, self.device, self.refcorr)
        fm = torch.stack([self.features_imgs[k, 0], feats[0].permute(1, 2, 0)])
        pool.build(fm, [0], [1], [0])
        c0 = self.coords0[None].contiguous()
        corr = pool.lookup(None, c0)
        _, delta, _ = self._net(self.contexts_imgs[k:k + 1, 0], self.cst_contexts_imgs[k:k + 1, 0], corr, c0, None)
        self.last_motion = delta.float().norm(dim=-1).mean()
        return feats

    def distance(self, ii, jj, beta=0.3, bidirectional=True):
        ii = torch.as_tensor(np.asarray(ii).reshape(-1), device=self.device)
        jj = torch.as_tensor(np.asarray(jj).reshape(-1), device=self.device)
        fd = self.refdroid.frame_distance
        if bidirectional:
            poses = self.cam0_T_world[:self.kf_idx + 1].clone()
            return .5 * (fd(poses, self.cam0_idepths, self.cam0_intrinsics[0], ii, jj, beta) +
                         fd(poses, self.cam0_idepths, self.cam0_intrinsics[0], jj, ii, beta))
        return fd(self.cam0_T_world, self.cam0_idepths, self.cam0_intrinsics[0], ii, jj, beta)

    # ---- update() / ba() with the reference's sequencing
    @torch.no_grad()
    def update(self, kf0=None, kf1=None, itrs=2, use_inactive=False, EP=1e-7, motion_only=False):
        dev = self.device
        coords1, _ = db.reproject(self.cam0_T_world, self.cam0_idepths, self.cam0_intrinsics, self.ii, self.jj)
        corr = self.corr_pool.lookup(None, coords1)
        net, delta, weight, damping, upmask = self._net(self.gru_hidden_states, self.cst_contexts_imgs[self.ii, 0], corr, coords1,
                                                        self.gru_estimated_flow, self.ii_h)
        self.gru_hidden_states = net
        kf0 = max(0, int(self.ii.min().item()))                               # `.item()`: a sync, as in the reference (:402)
        self.gru_estimated_flow = coords1 + delta
        self.gru_estimated_flow_weight = weight
        self.damping[torch.unique(self.ii)] = damping
        if use_inactive:
            ii_in = torch.as_tensor(self.ii_inactive_h, device=dev); jj_in = torch.as_tensor(self.jj_inactive_h, device=dev)
            mask = (ii_in >= kf0 - 3) & (jj_in >= kf0 - 3)
            ii = torch.cat([ii_in[mask], self.ii], 0); jj = torch.cat([jj_in[mask], self.jj], 0)
            flow = torch.cat([self.gru_estimated_flow_inactive[mask], self.gru_estimated_flow], 0)
            wgt = torch.cat([self.gru_estimated_flow_weight_inactive[mask], self.gru_estimated_flow_weight], 0)
        else:
            ii, jj, flow, wgt = self.ii, self.jj, self.gru_estimated_flow, self.gru_estimated_flow_weight
        damp = .2 * self.damping[torch.unique(ii)].contiguous() + EP
        flow = flow.permute(0, 3, 1, 2).contiguous(); wgt = wgt.permute(0, 3, 1, 2).contiguous()
        self.ba(flow, wgt, damp, ii, jj, kf0, None, itrs=itrs, compute_covariances=self.compute_covariances)
        kx = torch.unique(self.ii)
        self.cam0_idepths_up[kx] = cvx_upsample_torch(self.cam0_idepths[kx].unsqueeze(-1), upmask.float()).squeeze(-1)
        self.cam0_depths_cov_up[kx] = cvx_upsample_torch(self.cam0_depths_cov[kx].unsqueeze(-1), upmask.float(), pow=1.0).squeeze(-1)
        self._touch_state()
        self.viz_idx[kf0:self.kf_idx + 1] = True
        self.age_h += 1
        self.stats["updates"] += 1

    def ba(self, target, weight, damping, ii, jj, kf0=0, kf1=None, itrs=2, lm=1e-4, ep=0.1, motion_only=False,
           compute_covariances=True):
        dev = self.device
        if not torch.is_tensor(ii):
            ii = torch.as_tensor(np.asarray(ii), device=dev); jj = torch.as_tensor(np.asarray(jj), device=dev)
        if kf1 is None:
            kf1 = max(ii.max().item(), jj.max().item()) + 1
        N, HW = kf1 - kf0, self.ht * self.wd
        from oracle import ba as oba
        has_prior = self.kf_idx_to_f_idx.get(kf0, -1) == 0
        cTb = self.cam0_T_body.double().cpu().numpy()
        prior = self.prior_pose.double().cpu().numpy()
        Hn = L = None
        for _ in range(itrs):
            H, v, Q, E, w, _, _ = self.refdroid.reduced_camera_matrix(
                self.cam0_T_world, self.world_T_body, self.cam0_idepths, self.cam0_intrinsics[0].contiguous(), self.cam0_T_body,
                self.cam0_idepths_sensed, target, weight, damping, ii, jj, kf0, kf1)
            Hn = H.double().cpu().numpy(); vn = v.double().cpu().numpy().reshape(-1)          # ONE copy (reference: one per block)
            wTb = self.world_T_body.double().cpu().numpy()
            err = oba.pose_prior_error(wTb[kf0], prior) if has_prior else None                 # PriorFactorPose3, sigma 1e-4
            dx, L = oba.dense_solve(Hn, vn, 0 if has_prior else -1, err, self.prior_info if has_prior else 0.0)
            if has_prior:
                Hn[:6, :6] += self.prior_info * np.eye(6)                                       # the graph's hessian() includes the prior
            wTb_new, cTw_new = oba.gtsam_retract(wTb, cTb, dx, kf0)                             # right retraction, [omega, t]
            self.world_T_body[kf0:kf1] = torch.as_tensor(wTb_new[kf0:kf1], device=dev, dtype=torch.float32)
            self.cam0_T_world[kf0:kf1] = torch.as_tensor(cTw_new[kf0:kf1], device=dev, dtype=torch.float32)
            xi = torch.as_tensor(dx, device=dev, dtype=torch.float32).contiguous()
            self.refdroid.solve_depth(xi, self.cam0_idepths, Q, E, w, ii, jj, kf0, kf1)
            self.cam0_idepths.clamp_(min=0.001)
        if compute_covariances and L is not None:
            self._covariances(torch.as_tensor(Hn, device=dev, dtype=torch.float32), Q, E, ii, jj, kf0, kf1, N, HW)
        return None, None

    def _covariances(self, H, Q, E, ii, jj, kf0, kf1, P, HW):
        """visual_frontend.py:1164-1230 with dense torch ops, statement for statement (incl. the K x K x 6 x HW scratch)"""
        L = torch.linalg.cholesky(H)
        L_inv = torch.linalg.solve_triangular(L, torch.eye(L.shape[0], device=L.device), upper=False)
        sigma_gg = (L_inv.transpose(-2, -1) @ L_inv).view(P, 6, P, 6).permute(0, 2, 1, 3)
        sigma_g = torch.diagonal(sigma_gg, dim1=0, dim2=1).permute(2, 0, 1).view(P, 6, 6)
        Ei, Ejz = E[:P], E[P:P + ii.shape[0]]
        kx, _ = torch.unique(ii, return_inverse=True)
        K = kx.shape[0]
        m = int(min(ii.min(), jj.min()))
        Ej = torch.zeros(K, K, 6, HW, device=self.device)
        Ej[jj - m, ii - m] = Ejz
        Ej = Ej[kf0 - m:kf1 - m].view(P, K, 6, HW)
        Ej[range(P), kf0 - m:kf1 - m, :, :] = Ei[range(P), :, :]
        E_sum = Ej.permute(0, 2, 1, 3).reshape(P * 6, K * HW)
        Q_ = Q.view(K * HW, 1)
        Fm = torch.matmul(Q_ * E_sum.t(), L_inv)
        z_cov = (Q_.squeeze() + torch.pow(Fm, 2).sum(dim=-1)).view(K, self.ht, self.wd)
        self.world_T_body_cov[kf0:kf1] = sigma_g
        self.cam0_idepths_cov[kx] = z_cov
        self.cam0_depths_cov[kx] = z_cov / self.cam0_idepths[kx] ** 4
