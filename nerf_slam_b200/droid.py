"""DROID-style plugin surface of the reference on top of the sm_90a kernels (SURVEY.md §8 row A19 "API twins",
§8b "Python class surface to keep"):

  DroidNet                      .feature_net/.fnet  .context_net/.cnet  .update_net/.update   (networks/droid_net.py:153-158)
  DepthVideo                    the `video` object the classes below talk to (attribute list: SURVEY.md §8b)
  FactorGraph(video, update_net, device, corr_impl, max_factors)                     (networks/factor_graph.py:11-387)
      .update .update_lowmem .add_factors .rm_factors .rm_keyframe .add_neighborhood_factors
      .add_proximity_factors .filter_edges .clear_edges .print_edges
  MotionFilter(net, video, min_flow_thresh, device)   .track(k, tstamp, image, depth, intrinsics)   (networks/motion_filter.py)
  DroidFrontend(droid_net, video, args)               .__call__()                                   (networks/droid_frontend.py)

The reference ships these classes without the `video` they need and with one hole (`gru_contexts_input` is
never filled, networks/factor_graph.py:128-131 vs :219-220); both are closed here.

Layout decisions (GPU-first, not the reference's):
  * edge lists are CONTROL data and live on the host (`ii`, `jj`, `age`, ... are CPU int64 tensors sharing
    memory with numpy arrays); device copies are made once per edge-set change.  The reference keeps them
    on the GPU and pays a device->host sync for every `.item()` in its Python loops.
  * per-edge state is channels-last fp16 (`[E,ht,wd,128]`, the wgmma operand layout); the reference-shaped
    `[1,E,128,ht,wd]` tensors are exposed as views.
  * correlation volumes sit in a slot arena (`CorrPool`): adding/removing edges never copies volumes.
Every kernel call goes through `droid_backends` / `conv` (the C-ABI library); nothing here computes on the CPU.
"""
import threading
import types

import numpy as np
import torch
import torch.nn.functional as F

from . import _lib
from . import droid_backends as db
from .corr import AltCorrBlock, CorrPool
from .graph import proximity_edges


# ----------------------------------------------------------------------------------------------- helpers
def _se3_inverse(tq):
    """[N,7] (t, q xyzw) -> inverse transforms, same layout"""
    t, q = tq[:, :3], tq[:, 3:]
    qi = torch.cat([-q[:, :3], q[:, 3:]], dim=1)
    u = qi[:, :3]
    c = torch.cross(u, t, dim=1)
    rt = t + 2.0 * (qi[:, 3:] * c + torch.cross(u, c, dim=1))          # R(qi) t
    return torch.cat([-rt, qi], dim=1).contiguous()


def coords_grid(ht, wd, device):
    """networks/geom/projective_ops.py:14-19 -> [ht,wd,2] (x,y)"""
    y, x = torch.meshgrid(torch.arange(ht, device=device).float(), torch.arange(wd, device=device).float(), indexing="ij")
    return torch.stack([x, y], dim=-1)


def _host_index(v):
    """edge index argument (list / numpy / tensor on any device, ints or 0-dim tensors) -> int64 numpy [n]"""
    if torch.is_tensor(v):
        return v.detach().to("cpu", torch.long).reshape(-1).numpy().copy()
    return np.asarray([int(x) for x in v], dtype=np.int64).reshape(-1) if not isinstance(v, np.ndarray) \
        else v.astype(np.int64).reshape(-1)


def _host_mask(m):
    if torch.is_tensor(m):
        return m.detach().to("cpu").reshape(-1).numpy().astype(bool)
    return np.asarray(m, dtype=bool).reshape(-1)


def _to_dev(a, device, dtype=torch.long):
    """host index array -> tensor on `device` (pinned, non-blocking upload on CUDA)"""
    if torch.device(device).type == "cuda":
        return _lib.h2d(np.ascontiguousarray(a), device, dtype)
    return torch.from_numpy(np.ascontiguousarray(a)).to(dtype)


def _dev_index(v, device):
    if torch.is_tensor(v) and v.device.type == torch.device(device).type:
        return v.reshape(-1).long()
    return _to_dev(_host_index(v), device)


def _nhwc(t):
    """[n,C,h,w] (any strides) -> contiguous [n,h,w,C]"""
    return t.permute(0, 2, 3, 1).contiguous()


class _Value:
    """`multiprocessing.Value` stand-in (`video.counter.value`, `video.ready.value`): one process per GPU here"""

    def __init__(self, v=0):
        self.value = v


# ----------------------------------------------------------------------------------------------- networks
class EncoderNetTC:
    """BasicEncoder's call convention ([b,n,3,H,W] normalised image -> [b,n,C,H/8,W/8] fp16,
    networks/modules/extractor.py:183-198) on the tensor-core encoder (conv.EncoderTC)."""

    def __init__(self, params, device):
        from .conv import EncoderTC
        self.params = params
        self.tc = EncoderTC(params, device)

    def __call__(self, x):
        b, n = x.shape[:2]
        y = self.tc(x.reshape(b * n, *x.shape[2:]).float())
        return y.unflatten(0, (b, n))


class UpdateNetTC:
    """UpdateModule.forward's convention (networks/droid_net.py:118-150) on the fused tensor-core update operator:
    net, inp [1,E,128,ht,wd]; corr [1,E,196,ht,wd]; flow [1,E,4,ht,wd] | None; ii (GraphAgg) | None
      -> net [1,E,128,ht,wd], delta [1,E,ht,wd,2], weight [1,E,ht,wd,2] (, eta [1,K,ht,wd], upmask [1,K,576,ht,wd]).
    `fused` is the channels-last operator itself; `FactorGraph` calls it directly (no layout round trip)."""

    def __init__(self, params, device):
        from .conv import UpdateOperatorTC
        self.params = params
        self.fused = UpdateOperatorTC(params, device)

    def __call__(self, net, inp, corr, flow=None, ii=None, jj=None):
        from .conv import CORR_PAD
        b, n, _, h, w = net.shape
        assert b == 1, "batch of graphs: one graph per call"
        net_ = _nhwc(net.reshape(n, -1, h, w).half())
        inp_ = _nhwc(inp.reshape(n, -1, h, w).half())
        corr_ = F.pad(corr.reshape(n, -1, h, w).permute(0, 2, 3, 1), (0, CORR_PAD - corr.shape[2])).half().contiguous()
        motion = torch.zeros(n, 4, h, w, device=net.device) if flow is None else flow.reshape(n, 4, h, w)
        out = self.fused.call_reference_convention(net_, inp_, corr_, motion, ii)
        net2 = out[0].permute(0, 3, 1, 2)[None]
        if ii is None:
            return net2, out[1][None], out[2][None]
        return net2, out[1][None], out[2][None], out[3][None], out[4].permute(0, 3, 1, 2)[None]


class DroidNet:
    """networks/droid_net.py:153-158 (inference part): the three networks, weights from `droid.pth`
    (key remap of visual_frontend.py:1051-1068) or seeded random init."""

    def __init__(self, weights=None, device="cuda:0"):
        from .networks import BasicEncoder, UpdateModule, load_droid_weights
        fnet = BasicEncoder(128, "instance", torch.Generator().manual_seed(10))
        cnet = BasicEncoder(256, "none", torch.Generator().manual_seed(11))
        upd = UpdateModule(torch.Generator().manual_seed(12))
        self.weights_source = "random-init(seeded)"
        if weights:
            sd = load_droid_weights(weights)
            fnet.load_state_dict(sd, "feature_net.")
            cnet.load_state_dict(sd, "context_net.")
            upd.load_state_dict(sd, "update_net.")
            self.weights_source = weights
        for m in (fnet, cnet, upd):
            m.to(device=device, dtype=torch.float16)
        self.device = device
        self.feature_net = self.fnet = EncoderNetTC(fnet, device)
        self.context_net = self.cnet = EncoderNetTC(cnet, device)
        self.update_net = self.update = UpdateNetTC(upd, device)


# ----------------------------------------------------------------------------------------------- video
class DepthVideo:
    """The keyframe store the DROID-style classes operate on.  Attribute contract: SURVEY.md §8b
    (usage at networks/factor_graph.py:20-29,122-135,173-182,207,251-253,263-266,300-303,313,326,334;
    networks/droid_frontend.py:47-109; networks/motion_filter.py:81-85).

    poses [N,7] (t, q xyzw) camera-from-world; disps [N,h/8,w/8] inverse depth; intrinsics [N,4] at 1/8 resolution.
    fmaps/nets/inps are channels-first VIEWS of channels-last fp16 storage."""

    def __init__(self, image_size=(480, 640), buffer=512, stereo=False, device="cuda:0"):
        self.counter, self.ready = _Value(0), _Value(0)
        self._lock = threading.RLock()
        self.ht, self.wd = ht, wd = int(image_size[0]), int(image_size[1])
        self.stereo, self.device = bool(stereo), device
        h8, w8 = ht // 8, wd // 8
        f32 = dict(dtype=torch.float32, device=device)
        self.tstamp = torch.zeros(buffer, dtype=torch.float64, device=device)
        self.images = torch.zeros(buffer, 3, ht, wd, dtype=torch.uint8, device=device)
        self.dirty = torch.zeros(buffer, dtype=torch.bool, device=device)
        self.poses = torch.zeros(buffer, 7, **f32)
        self.poses[:, 6] = 1.0                                   # identity (t = 0, q = (0,0,0,1))
        self.extrinsics = torch.tensor([0, 0, 0, 0, 0, 0, 1.0], **f32)
        self.disps = torch.ones(buffer, h8, w8, **f32)
        self.disps_sens = torch.zeros(buffer, h8, w8, **f32)
        self.disps_up = torch.zeros(buffer, ht, wd, **f32)
        self.intrinsics = torch.zeros(buffer, 4, **f32)
        c = 2 if stereo else 1
        h16 = dict(dtype=torch.float16, device=device)
        self._fmaps = torch.zeros(buffer, c, h8, w8, 128, **h16)
        self._nets = torch.zeros(buffer, h8, w8, 128, **h16)
        self._inps = torch.zeros(buffer, h8, w8, 128, **h16)
        self.fmaps = self._fmaps.permute(0, 1, 4, 2, 3)          # [N,c,128,h8,w8]
        self.nets = self._nets.permute(0, 3, 1, 2)               # [N,128,h8,w8]
        self.inps = self._inps.permute(0, 3, 1, 2)

    def get_lock(self):
        return self._lock

    # ---- item access (networks/motion_filter.py:81-85 appends
    #      (tstamp, image, pose, disp, depth, intrinsics/8, fmap, net, inp))
    def _set_item(self, index, item):
        if isinstance(index, int) and index >= self.counter.value:
            self.counter.value = index + 1
        elif torch.is_tensor(index) and int(index.max()) >= self.counter.value:
            self.counter.value = int(index.max()) + 1
        dev = self.device
        self.tstamp[index] = float(item[0]) if not torch.is_tensor(item[0]) else item[0].to(dev)
        self.images[index] = torch.as_tensor(item[1]).to(dev)
        if item[2] is not None:
            self.poses[index] = torch.as_tensor(item[2], dtype=torch.float32).to(dev)
        if item[3] is not None:
            self.disps[index] = item[3] if not torch.is_tensor(item[3]) else item[3].to(dev)
        if item[4] is not None:
            depth = torch.as_tensor(item[4]).to(dev).float()[..., 3::8, 3::8]
            self.disps_sens[index] = torch.where(depth > 0, 1.0 / depth, depth)
        if item[5] is not None:
            self.intrinsics[index] = torch.as_tensor(item[5], dtype=torch.float32).to(dev)
        if len(item) > 6:
            self.fmaps[index] = item[6].to(dev)
        if len(item) > 7:
            self.nets[index] = item[7].to(dev)
        if len(item) > 8:
            self.inps[index] = item[8].to(dev)

    def __setitem__(self, index, item):
        with self.get_lock():
            self._set_item(index, item)

    def __getitem__(self, index):
        with self.get_lock():
            if isinstance(index, int) and index < 0:
                index = self.counter.value + index
            return (self.poses[index], self.disps[index], self.intrinsics[index], self.fmaps[index],
                    self.nets[index], self.inps[index])

    def append(self, *item):
        with self.get_lock():
            self._set_item(self.counter.value, item)

    # ---- geometry
    @staticmethod
    def format_indicies(ii, jj, device):
        """-> flat int64 tensors on `device` (tensors already there are used as they are: no host round trip)"""
        return _dev_index(ii, device), _dev_index(jj, device)

    def normalize(self):
        """scale the map to unit mean inverse depth (mono gauge)"""
        with self.get_lock():
            n = self.counter.value
            s = self.disps[:n].mean()
            self.disps[:n] /= s
            self.poses[:n, :3] *= s
            self.dirty[:n] = True

    def reproject(self, ii, jj):
        """A6: -> coords [1,E,h8,w8,2], valid [1,E,h8,w8,1]"""
        ii, jj = self.format_indicies(ii, jj, self.device)
        coords, valid = db.reproject(self.poses, self.disps, self.intrinsics, ii, jj)
        return coords[None], valid[None]

    def distance(self, ii=None, jj=None, beta=0.3, bidirectional=True):
        """A16: mean flow magnitude between frame pairs; all pairs of the first `counter` frames when ii is None"""
        return_matrix = ii is None
        if return_matrix:
            n = self.counter.value
            a, b = np.meshgrid(np.arange(n), np.arange(n), indexing="ij")
            ii, jj = a.reshape(-1), b.reshape(-1)
        ii, jj = self.format_indicies(ii, jj, self.device)
        if bidirectional:
            poses = self.poses[:self.counter.value + 1].clone()
            d1 = db.frame_distance(poses, self.disps, self.intrinsics[0], ii, jj, beta)
            d2 = db.frame_distance(poses, self.disps, self.intrinsics[0], jj, ii, beta)
            d = .5 * (d1 + d2)
        else:
            d = db.frame_distance(self.poses, self.disps, self.intrinsics[0], ii, jj, beta)
        return d.reshape(n, n) if return_matrix else d

    def ba(self, target, weight, eta, ii, jj, t0=1, t1=None, itrs=2, lm=1e-4, ep=0.1, motion_only=False):
        """dense bundle adjustment of poses [t0,t1) and the depths of the edges' source frames, in place — what
        networks/factor_graph.py:251-253,300-301 call on the `video` object (which the reference does not ship).

        Default (`ba_mode = "consistent"`): the linearisation of this code base (body-frame Jacobians in [omega, t]
        order, src/droid_kernels.cu:376-403) with the matching retraction (right perturbation of world_T_cam, the one
        the live path's gtsam step applies) and DROID's Levenberg damping `ep + lm*diag` — one host call, edge list
        stays on the host.  `ba_mode = "reference"` runs droid_backends.ba (A15: ba_cuda, src/droid_kernels.cu:1441-1568)
        as it is in the reference: the SAME body-frame Jacobians followed by the ORIGINAL DROID left retraction
        `exp([tau,phi]) * T` (`pose_retr_kernel`) — the two do not belong together (the reference's own comment on
        `body_poses`: "SEND IDENTITY, this is not supposed to work otw"), the pose step has the wrong parametrisation and
        the iteration diverges on real data; ba_cuda has no live caller in the reference.  Parity of that loop is kept
        at the operator level (tests/test_gpu_parity.py::test_droid_backends_ba_all_in_one_loop)."""
        with self.get_lock():
            ih, jh = _host_index(ii), _host_index(jj)
            if t1 is None:
                t1 = int(max(ih.max(), jh.max())) + 1
            if getattr(self, "ba_mode", "consistent") == "reference" or motion_only:
                db.ba_host_edges(self.poses, self.disps, self.intrinsics[0], self.extrinsics, self.disps_sens,
                                 target.contiguous(), weight.contiguous(), eta, ih, jh, t0, t1, itrs, lm, ep, motion_only)
            else:
                prob = db.BAProblem(self.poses, self.disps, self.intrinsics[0], self.extrinsics, self.disps_sens,
                                    target.contiguous(), weight.contiguous(), eta.contiguous(), ih, jh, t0, t1)
                if getattr(self, "_ba_status", None) is None:
                    self._ba_status = torch.zeros(2, dtype=torch.int32, device=self.device)
                wTc = _se3_inverse(self.poses)                     # body == camera (extrinsics = identity)
                prob.frontend_update(itrs, wTc, self.poses, self.extrinsics, self._ba_status, clamp_min=0.0, lm=lm, ep=ep)
            self.disps.clamp_(min=0.001)

    def upsample(self, ix, mask):
        """A17: full-resolution inverse depth of keyframes `ix` from the convex-combination mask [K,576,h8,w8]"""
        ix = _dev_index(ix, self.device)
        up = db.cvx_upsample(self.disps[ix].unsqueeze(-1), mask.reshape(ix.shape[0], 576, *mask.shape[-2:]))
        self.disps_up[ix] = up.squeeze(-1)


# ----------------------------------------------------------------------------------------------- correlation store
def _make_pool(capacity, ht, wd, device):
    return CorrPool(capacity, ht, wd, device)


class _VolumeStore:
    """`FactorGraph.correlation_volumes` for corr_impl == "volume": a growable slot arena of 4-level pyramids.
    Callable like the reference's CorrBlock: store(coords [1,E,ht,wd,2]) -> [1,E,196,ht,wd]."""

    def __init__(self, ht, wd, device, capacity):
        self.ht, self.wd, self.device = ht, wd, device
        self.pool = _make_pool(capacity, ht, wd, device)
        self.slots = np.zeros(0, np.int64)       # slot of every active edge, in edge order
        self._slots_d = None

    def __len__(self):
        return int(self.slots.shape[0])

    def _grow(self, need):
        old = self.pool
        cap = max(2 * old.capacity, old.capacity + need)
        new = _make_pool(cap, self.ht, self.wd, self.device)
        used = sorted(set(range(old.capacity)) - set(old.free))
        if used and hasattr(old, "levels"):
            idx = _to_dev(np.asarray(used, np.int64), self.device)
            for a, b in zip(new.levels, old.levels):
                a.index_copy_(0, idx, b.index_select(0, idx))
        new.free = [s for s in range(cap - 1, -1, -1) if s not in set(used)]
        self.pool = new

    def add(self, fmaps, fi, fj):
        """fmaps [N,rig,128,h,w] (any strides); fi/fj flat frame indices (host) of the new edges"""
        n = len(fi)
        if n > len(self.pool.free):
            self._grow(n)
        slots = np.asarray(self.pool.alloc(n), np.int64)
        # only the frames these edges touch are brought into the operand layout (channels-last fp16)
        frames, inv = np.unique(np.concatenate([fi, fj]), return_inverse=True)
        N, rig = fmaps.shape[:2]
        sel = fmaps.reshape(N * rig, *fmaps.shape[2:]) if fmaps.is_contiguous() else fmaps.flatten(0, 1)
        f = _nhwc(sel[_to_dev(frames, fmaps.device)].to(self.device)).half()
        self.pool.build(f, inv[:n].tolist(), inv[n:].tolist(), slots.tolist())
        self.slots = np.concatenate([self.slots, slots])
        self._slots_d = None

    def keep(self, keep_mask):
        self.pool.release(self.slots[~keep_mask].tolist())
        self.slots = self.slots[keep_mask]
        self._slots_d = None

    def slots_dev(self):
        if self._slots_d is None:
            self._slots_d = _to_dev(self.slots.astype(np.int32), self.device, torch.int32)
        return self._slots_d

    def lookup_nhwc(self, coords, out=None):
        """coords [E,ht,wd,2] -> [E,ht,wd,CORR_PAD] fp16 (operand of the fused update operator)"""
        return self.pool.lookup(self.slots_dev(), coords, nhwc=True, out=out)

    def __call__(self, coords):
        b, n, ht, wd, _ = coords.shape
        c = coords.reshape(n, ht, wd, 2).permute(0, 3, 1, 2).contiguous().float()
        return self.pool.lookup(self.slots_dev(), c)[None]


# ----------------------------------------------------------------------------------------------- factor graph
class FactorGraph:
    """networks/factor_graph.py:11-387.  Same constructor, methods, attribute names and edge semantics
    (bit-exact edge sets: tests/test_cpu_droid.py replays traces recorded from the reference's own class)."""

    def __init__(self, video, update_net, device="cuda:0", corr_impl="volume", max_factors=-1, upsample=False):
        self.video, self.update_net, self.device = video, update_net, device
        self.max_factors, self.corr_impl, self.upsample = max_factors, corr_impl, upsample
        self.ht = ht = video.ht // 8
        self.wd = wd = video.wd // 8
        self.coords0 = coords_grid(ht, wd, device)
        z = lambda: np.zeros(0, np.int64)
        self._ii, self._jj, self._age = z(), z(), z()
        self._ii_inac, self._jj_inac, self._ii_bad, self._jj_bad = z(), z(), z(), z()
        self.correlation_volumes = None            # _VolumeStore, created by the first add_factors ("volume")
        self._net = self._inp = None               # [E,ht,wd,C] channels-last
        e = lambda: torch.zeros(0, ht, wd, 2, device=device, dtype=torch.float32)
        self._flow, self._conf, self._target_inac, self._weight_inac = e(), e(), e(), e()
        self.damping = 1e-6 * torch.ones_like(video.disps)
        self._dev = None                           # device copies of the edge lists (per edge set)

    # ---- reference-shaped views of the state
    def _idx_prop(name):
        def get(self):
            return torch.from_numpy(getattr(self, name))            # shares memory: `graph.age += 1` works in place

        def set_(self, v):
            setattr(self, name, np.ascontiguousarray(_host_index(v)))
            self._dev = None
        return property(get, set_)

    ii, jj, age = _idx_prop("_ii"), _idx_prop("_jj"), _idx_prop("_age")
    ii_inac, jj_inac = _idx_prop("_ii_inac"), _idx_prop("_jj_inac")
    ii_bad, jj_bad = _idx_prop("_ii_bad"), _idx_prop("_jj_bad")

    def _edge_prop(name):
        def get(self):
            return getattr(self, name)[None]                        # [1,E,ht,wd,2]

        def set_(self, v):
            setattr(self, name, v.reshape(-1, self.ht, self.wd, 2).to(self.device, torch.float32))
        return property(get, set_)

    gru_estimated_flow, gru_estimated_flow_weight = _edge_prop("_flow"), _edge_prop("_conf")
    target_inac, weight_inac = _edge_prop("_target_inac"), _edge_prop("_weight_inac")

    def _state_prop(name):
        def get(self):
            t = getattr(self, name)
            return None if t is None else t.permute(0, 3, 1, 2)[None]     # [1,E,C,ht,wd] view

        def set_(self, v):
            setattr(self, name, None if v is None else _nhwc(v.reshape(-1, *v.shape[-3:])))
        return property(get, set_)

    gru_hidden_states, gru_contexts_input = _state_prop("_net"), _state_prop("_inp")
    del _idx_prop, _edge_prop, _state_prop

    def _edges_dev(self):
        """(ii, jj) on the device + GraphAgg tables, built once per edge set"""
        if self._dev is None:
            d = types.SimpleNamespace()
            d.ii, d.jj = _to_dev(self._ii, self.device), _to_dev(self._jj, self.device)
            d.ux, inv = np.unique(self._ii, return_inverse=True)
            order = np.argsort(inv, kind="stable").astype(np.int32)
            ptr = np.zeros(len(d.ux) + 1, np.int32)
            np.cumsum(np.bincount(inv, minlength=len(d.ux)), out=ptr[1:])
            d.agg = (_to_dev(ptr, self.device, torch.int32), _to_dev(order, self.device, torch.int32), len(d.ux))
            d.ux_d = _to_dev(d.ux, self.device)
            self._dev = d
        return self._dev

    # ---- edge bookkeeping
    def _filter_repeated_edges(self, ii, jj):
        """:43-54 — drop edges that are already active or inactive"""
        have = np.concatenate([self._ii * 65536 + self._jj, self._ii_inac * 65536 + self._jj_inac])
        keep = ~np.isin(ii * 65536 + jj, have)
        return ii[keep], jj[keep]

    def print_edges(self):
        """:56-68"""
        ix = np.argsort(self._ii, kind="stable")
        w = self._conf.mean(dim=[1, 2, 3]).cpu().numpy()
        for e in zip(self._ii[ix], self._jj[ix], w[ix]):
            print(e)
        print()

    def filter_edges(self):
        """:70-77 — retire long-range edges the network has no confidence in"""
        conf = self._conf.mean(dim=[1, 2, 3]).cpu().numpy()
        mask = (np.abs(self._ii - self._jj) > 2) & (conf < 0.001)
        self._ii_bad = np.concatenate([self._ii_bad, self._ii[mask]])
        self._jj_bad = np.concatenate([self._jj_bad, self._jj[mask]])
        self.rm_factors(mask, store=False)

    def clear_edges(self):
        """:79-82"""
        self.rm_factors(self._ii >= 0)
        self._net = self._inp = None

    @torch.no_grad()
    def add_factors(self, ii, jj, remove=False):
        """:85-139"""
        ii, jj = _host_index(ii), _host_index(jj)
        ii, jj = self._filter_repeated_edges(ii, jj)
        if ii.shape[0] == 0:
            return
        old, new = self._ii.shape[0], ii.shape[0]
        if self.max_factors > 0 and old + new > self.max_factors and self.correlation_volumes is not None and remove:
            # `ix` is argsort(age) (ties in index order, as torch's CPU sort yields); the mask is then applied
            # POSITIONALLY to the edges — the reference's own quirk (:107-108), kept
            ix = np.argsort(self._age, kind="stable")
            self.rm_factors(ix >= self.max_factors - new, store=True)
        self._ii = np.concatenate([self._ii, ii]); self._jj = np.concatenate([self._jj, jj])
        self._age = np.concatenate([self._age, np.zeros(new, np.int64)])
        self._dev = None
        video = self.video
        if self.corr_impl == "volume":
            rig = video.fmaps.shape[1]
            if self.correlation_volumes is None:
                cap = 2 * self.max_factors if self.max_factors > 0 else max(64, 2 * new)
                self.correlation_volumes = _VolumeStore(self.ht, self.wd, self.device, max(cap, new))
            self.correlation_volumes.add(video.fmaps, ii * rig, jj * rig + (ii == jj))
        vi = _to_dev(ii, video.nets.device)
        net = _nhwc(video.nets[vi]).to(self.device)
        inp = _nhwc(video.inps[vi]).to(self.device)
        self._net = net if self._net is None else torch.cat([self._net, net], 0)
        self._inp = inp if self._inp is None else torch.cat([self._inp, inp], 0)
        target, _ = video.reproject(ii, jj)                              # flow initialised with the reprojection
        target = target.reshape(new, self.ht, self.wd, 2).to(self.device, torch.float32)
        self._flow = torch.cat([self._flow, target], 0)
        self._conf = torch.cat([self._conf, torch.zeros_like(target)], 0)

    @torch.no_grad()
    def rm_factors(self, mask, store=False):
        """:144-167"""
        mask = _host_mask(mask)
        if mask.shape[0] == 0 or not mask.any():
            return
        keep = ~mask
        kd = _to_dev(np.nonzero(keep)[0], self.device)
        if store:
            rd = _to_dev(np.nonzero(mask)[0], self.device)
            self._ii_inac = np.concatenate([self._ii_inac, self._ii[mask]])
            self._jj_inac = np.concatenate([self._jj_inac, self._jj[mask]])
            self._target_inac = torch.cat([self._target_inac, self._flow.index_select(0, rd)], 0)
            self._weight_inac = torch.cat([self._weight_inac, self._conf.index_select(0, rd)], 0)
        self._ii, self._jj, self._age = self._ii[keep], self._jj[keep], self._age[keep]
        self._dev = None
        if self.corr_impl == "volume" and self.correlation_volumes is not None:
            self.correlation_volumes.keep(keep)
        if self._net is not None:
            self._net = self._net.index_select(0, kd)
        if self._inp is not None:
            self._inp = self._inp.index_select(0, kd)
        self._flow = self._flow.index_select(0, kd)
        self._conf = self._conf.index_select(0, kd)

    @torch.no_grad()
    def rm_keyframe(self, ix):
        """:171-198 — slot ix takes the content of slot ix+1; edges touching ix are dropped, later indices shift"""
        video = self.video
        with video.get_lock():
            for name in ("images", "poses", "disps", "disps_sens", "intrinsics", "nets", "inps", "fmaps"):
                buf = getattr(video, name)
                buf[ix] = buf[ix + 1]
        m = (self._ii_inac == ix) | (self._jj_inac == ix)
        self._ii_inac[self._ii_inac >= ix] -= 1
        self._jj_inac[self._jj_inac >= ix] -= 1
        if m.any():
            kd = _to_dev(np.nonzero(~m)[0], self.device)
            self._ii_inac, self._jj_inac = self._ii_inac[~m], self._jj_inac[~m]
            self._target_inac = self._target_inac.index_select(0, kd)
            self._weight_inac = self._weight_inac.index_select(0, kd)
        m = (self._ii == ix) | (self._jj == ix)
        self._ii[self._ii >= ix] -= 1
        self._jj[self._jj >= ix] -= 1
        self._dev = None
        self.rm_factors(m, store=False)

    # ---- the update operator + BA
    def _ba_inputs(self, t0, use_inactive, EP):
        """:229-244 -> (ii, jj, target [E,2,ht,wd], weight [E,2,ht,wd], damping [K,ht,wd])"""
        if use_inactive:
            m = (self._ii_inac >= t0 - 3) & (self._jj_inac >= t0 - 3)
            md = _to_dev(np.nonzero(m)[0], self.device)
            ii = np.concatenate([self._ii_inac[m], self._ii]); jj = np.concatenate([self._jj_inac[m], self._jj])
            flow = torch.cat([self._target_inac.index_select(0, md), self._flow], 0)
            conf = torch.cat([self._weight_inac.index_select(0, md), self._conf], 0)
        else:
            ii, jj, flow, conf = self._ii, self._jj, self._flow, self._conf
        damping = .2 * self.damping[_to_dev(np.unique(ii), self.device)].contiguous() + EP
        return ii, jj, flow.permute(0, 3, 1, 2).contiguous(), conf.permute(0, 3, 1, 2).contiguous(), damping

    def _operator(self, net, inp, corr_fn, coords1, flow, ii_host, agg=None):
        """one application of the update operator on channels-last state.
        coords1/flow [e,ht,wd,2]; corr_fn(coords1, nhwc) -> correlation features
          -> net' [e,ht,wd,128], flow' [e,ht,wd,2], conf [e,ht,wd,2], eta [K,ht,wd], upmask [K,576,ht,wd]"""
        fused = getattr(self.update_net, "fused", None)
        if fused is not None:
            if agg is None:
                ux, inv = np.unique(ii_host, return_inverse=True)
                order = np.argsort(inv, kind="stable").astype(np.int32)
                ptr = np.zeros(len(ux) + 1, np.int32)
                np.cumsum(np.bincount(inv, minlength=len(ux)), out=ptr[1:])
                agg = (_to_dev(ptr, self.device, torch.int32), _to_dev(order, self.device, torch.int32), len(ux))
            out = fused(net, inp, corr_fn(coords1, True), coords1.contiguous(), self.coords0, target=flow.contiguous(), agg=agg)
            eta = 0.01 * F.softplus(out[3][..., 0].float())
            return out[0], out[1], out[2], eta, out[4].permute(0, 3, 1, 2)
        # any callable with UpdateModule.forward's convention (networks/droid_net.py:118-150)
        motion = torch.cat([coords1 - self.coords0, flow - coords1], dim=-1).permute(0, 3, 1, 2).clamp(-64.0, 64.0)
        ii_t = _to_dev(ii_host, self.device)
        net2, delta, weight, eta, upmask = self.update_net(net.permute(0, 3, 1, 2)[None], inp.permute(0, 3, 1, 2)[None],
                                                           corr_fn(coords1, False), motion[None], ii_t, ii_t)
        return _nhwc(net2[0]), coords1 + delta[0].float(), weight[0].float(), eta[0].float(), upmask[0]

    @torch.no_grad()
    def update(self, t0=None, t1=None, itrs=2, use_inactive=False, EP=1e-7, motion_only=False):
        """:202-255 — reproject, correlation lookup, update operator, dense BA"""
        video, d = self.video, self._edges_dev()
        coords1, _ = video.reproject(d.ii, d.jj)
        coords1 = coords1.reshape(-1, self.ht, self.wd, 2)
        store = self.correlation_volumes
        corr_fn = lambda c, nhwc: store.lookup_nhwc(c) if nhwc else store(c[None])
        net, flow, conf, eta, upmask = self._operator(self._net, self._inp, corr_fn, coords1, self._flow, self._ii, d.agg)
        self._net, self._flow, self._conf = net, flow, conf
        if t0 is None:
            t0 = max(1, int(self._ii.min()) + 1)
        self.damping[d.ux_d] = eta
        ii, jj, target, weight, damping = self._ba_inputs(t0, use_inactive, EP)
        video.ba(target, weight, damping, ii, jj, t0, t1, itrs=itrs, lm=1e-4, ep=0.1, motion_only=motion_only)
        if self.upsample:
            video.upsample(d.ux_d, upmask)
        self._age += 1

    @torch.no_grad()
    def update_lowmem(self, t0=None, t1=None, itrs=2, use_inactive=False, EP=1e-7, steps=8):
        """:259-303 — global BA: on-the-fly correlation (alt-corr), edges in chunks of 8 source frames"""
        video = self.video
        t = video.counter.value
        num, rig, ch, ht, wd = video.fmaps.shape
        corr_op = AltCorrBlock(video.fmaps.reshape(1, num * rig, ch, ht, wd))
        from .conv import CORR_PAD
        for step in range(steps):
            coords1, _ = video.reproject(self._ii, self._jj)
            coords1 = coords1.reshape(-1, self.ht, self.wd, 2)
            s = 8
            for i in range(0, int(self._jj.max()) + 1, s):
                v = (self._ii >= i) & (self._ii < i + s)
                if not v.any():
                    continue
                vd = _to_dev(np.nonzero(v)[0], self.device)
                iis, jjs = self._ii[v], self._jj[v]
                fi = _to_dev(rig * iis, self.device); fj = _to_dev(rig * jjs + (iis == jjs), self.device)
                c1 = coords1.index_select(0, vd)

                def corr_fn(c, nhwc, fi=fi, fj=fj):
                    corr = corr_op(c[None], fi, fj)                            # [1,e,196,ht,wd] fp32
                    if not nhwc:
                        return corr
                    return F.pad(corr[0].permute(0, 2, 3, 1), (0, CORR_PAD - corr.shape[2])).half().contiguous()
                inp = _nhwc(video.inps[_to_dev(iis, video.inps.device)]).to(self.device)
                net, flow, conf, eta, upmask = self._operator(self._net.index_select(0, vd), inp, corr_fn, c1,
                                                              self._flow.index_select(0, vd), iis)
                self._net.index_copy_(0, vd, net)
                self._flow.index_copy_(0, vd, flow)
                self._conf.index_copy_(0, vd, conf)
                self.damping[_to_dev(np.unique(iis), self.device)] = eta
            damping = .2 * self.damping[_to_dev(np.unique(self._ii), self.device)].contiguous() + EP
            target = self._flow.permute(0, 3, 1, 2).contiguous()
            weight = self._conf.permute(0, 3, 1, 2).contiguous()
            video.ba(target, weight, damping, self._ii, self._jj, 1, t, itrs=itrs, lm=1e-5, ep=1e-2, motion_only=False)
            video.dirty[:t] = True

    # ---- edge creation
    def add_neighborhood_factors(self, t0, t1, r=3):
        """:305-320 — edges between frames of [t0,t1) whose index distance is in (c, r]"""
        ii, jj = np.meshgrid(np.arange(t0, t1), np.arange(t0, t1), indexing="ij")
        ii, jj = ii.reshape(-1), jj.reshape(-1)
        c = 1 if self.video.stereo else 0
        d = np.abs(ii - jj)
        keep = (d > c) & (d <= r)
        self.add_factors(ii[keep], jj[keep])

    def add_proximity_factors(self, t0=0, t1=0, rad=2, nms=2, beta=0.25, thresh=16.0, remove=False):
        """:323-387 — edges to frames that are close in mean-flow distance, with non-maximum suppression around
        existing and newly chosen edges.  Order-sensitive; the selection runs on the host copy of the distances
        (graph.proximity_edges, bit-exact against the reference's loops)."""
        t = self.video.counter.value
        ii, jj = np.meshgrid(np.arange(t0, t), np.arange(t1, t), indexing="ij")
        ii, jj = ii.reshape(-1), jj.reshape(-1)
        d = self.video.distance(ii, jj, beta=beta)
        d = d.detach().float().cpu().numpy().copy()
        ii1 = np.concatenate([self._ii, self._ii_bad, self._ii_inac])
        jj1 = np.concatenate([self._jj, self._jj_bad, self._jj_inac])
        es = proximity_edges(d, ii, jj, ii1, jj1, t0, t1, t, rad, nms, thresh, self.max_factors, self.video.stereo)
        if es.shape[0] == 0:
            return
        self.add_factors(es[:, 0], es[:, 1], remove)


# ----------------------------------------------------------------------------------------------- motion filter
class MotionFilter:
    """networks/motion_filter.py:11-85 — feature extraction for every frame; a frame enters the video when one
    application of the update operator on (last kept frame -> this frame) predicts enough flow."""

    def __init__(self, net, video, min_flow_thresh=2.5, device="cuda:0"):
        self.context_net, self.feature_net, self.update_net = net.cnet, net.fnet, net.update
        self.video, self.min_flow_thresh, self.device = video, min_flow_thresh, device
        self.skipped_frames = 0
        self.MEAN = torch.as_tensor([0.485, 0.456, 0.406], device=device)[:, None, None]
        self.STDV = torch.as_tensor([0.229, 0.224, 0.225], device=device)[:, None, None]

    def _context_encoder(self, image):
        c = self.context_net(image)
        context_maps, gru_input_maps = c.split([128, 128], dim=2)
        return context_maps.tanh().squeeze(0), gru_input_maps.relu().squeeze(0)

    def _feature_encoder(self, image):
        return self.feature_net(image).squeeze(0)

    @torch.no_grad()
    def track(self, k, timestamp, image, depth=None, intrinsics=None):
        """image [cams,3,H,W] u8 (BGR, as the reference's loaders deliver it); -> True when the frame was kept"""
        from .corr import CorrBlock
        img_normalized = image[None, :, [2, 1, 0]].to(self.device) / 255.0
        img_normalized = img_normalized.sub_(self.MEAN).div_(self.STDV)
        feature_map = self._feature_encoder(img_normalized)
        if k == 0:
            self.add_frame_to_video(timestamp, image, img_normalized, feature_map, depth, intrinsics, first=True)
            return True
        ht, wd = image.shape[-2] // 8, image.shape[-1] // 8
        coords0 = coords_grid(ht, wd, self.device)[None, None]
        corr = CorrBlock(self.feature_maps[None, [0]], feature_map[None, [0]])(coords0)
        _, delta, weight = self.update_net(self.context_maps[None], self.gru_input_maps[None], corr)
        if delta.norm(dim=-1).mean().item() > self.min_flow_thresh:
            self.add_frame_to_video(timestamp, image, img_normalized, feature_map, depth, intrinsics)      # pose/disp: keep
            self.skipped_frames = 0
            return True
        self.skipped_frames += 1
        return False

    def add_frame_to_video(self, timestamp, image, img_normalized, feature_map, depth_img=None, intrinsics=None, first=False):
        """:76-85, with two defects of the (never executed) reference method not reproduced:
        * it appends `context_maps[0,0]` / `gru_input_maps[0,0]` — after its own `.squeeze(0)` that is ONE channel
          plane [h,w], which `video.nets[k] = ...` would broadcast over all 128 channels; the full [128,h,w] maps of
          camera 0 are stored here (what the live path does, visual_frontend.py:300-330);
        * it appends the identity pose and disparity 1.0 for EVERY kept frame, which would overwrite the initial guess
          DroidFrontend writes into the next slot (`video.poses[t1] = video.poses[t1-1]`, droid_frontend.py:72-73); here
          only the first frame sets them, later frames pass None (keep what the front end prepared)."""
        context_maps, gru_input_maps = self._context_encoder(img_normalized[:, [0]])
        self.context_maps, self.gru_input_maps, self.feature_maps = context_maps, gru_input_maps, feature_map
        identity_pose = torch.tensor([0, 0, 0, 0, 0, 0, 1.0]) if first else None
        intr = None if intrinsics is None else torch.as_tensor(intrinsics, dtype=torch.float32) / 8.0
        self.video.append(timestamp, image[0], identity_pose, 1.0 if first else None, depth_img, intr,
                          feature_map, context_maps[0], gru_input_maps[0])


# ----------------------------------------------------------------------------------------------- front end
class DroidFrontend:
    """networks/droid_frontend.py:9-121 — keyframe loop over a `video` that a MotionFilter fills"""

    def __init__(self, droid_net, video, args):
        self.video = video
        self.update_net = droid_net.update_net
        self.graph = FactorGraph(video, droid_net.update_net, device=getattr(video, "device", "cuda:0"), max_factors=48,
                                 upsample=bool(getattr(args, "upsample", False)))
        self.t0 = self.t1 = 0
        self.is_initialized = False
        self.count = 0
        self.max_age, self.iters1, self.iters2 = 25, 4, 2
        self.warmup = args.warmup
        self.beta = args.beta
        self.frontend_nms = args.frontend_nms
        self.keyframe_thresh = args.keyframe_thresh
        self.frontend_window = args.frontend_window
        self.frontend_thresh = args.frontend_thresh
        self.frontend_radius = args.frontend_radius

    def _update(self):
        """:35-78 — add edges, run the operator, decide whether the previous frame stays a keyframe"""
        video, graph = self.video, self.graph
        self.count += 1
        self.t1 += 1
        if graph.correlation_volumes is not None:
            graph.rm_factors(graph.age > self.max_age, store=True)
        graph.add_proximity_factors(self.t1 - 5, max(self.t1 - self.frontend_window, 0), rad=self.frontend_radius,
                                    nms=self.frontend_nms, thresh=self.frontend_thresh, beta=self.beta, remove=True)
        k = self.t1 - 1
        video.disps[k] = torch.where(video.disps_sens[k] > 0, video.disps_sens[k], video.disps[k])
        for _ in range(self.iters1):
            graph.update(None, None, use_inactive=True)
        d = video.distance([self.t1 - 3], [self.t1 - 2], beta=self.beta, bidirectional=True)
        if d.item() < self.keyframe_thresh:
            graph.rm_keyframe(self.t1 - 2)
            with video.get_lock():
                video.counter.value -= 1
                self.t1 -= 1
        else:
            for _ in range(self.iters2):
                graph.update(None, None, use_inactive=True)
        video.poses[self.t1] = video.poses[self.t1 - 1]
        video.disps[self.t1] = video.disps[self.t1 - 1].mean()
        video.dirty[int(graph.ii.min()):self.t1] = True

    def _initialize(self):
        """:81-110"""
        video, graph = self.video, self.graph
        self.t0, self.t1 = 0, video.counter.value
        graph.add_neighborhood_factors(self.t0, self.t1, r=3)
        for _ in range(8):
            graph.update(1, use_inactive=True)
        graph.add_proximity_factors(0, 0, rad=2, nms=2, thresh=self.frontend_thresh, remove=False)
        for _ in range(8):
            graph.update(1, use_inactive=True)
        video.poses[self.t1] = video.poses[self.t1 - 1].clone()
        video.disps[self.t1] = video.disps[self.t1 - 4:self.t1].mean()
        self.is_initialized = True
        self.last_pose = video.poses[self.t1 - 1].clone()
        self.last_disp = video.disps[self.t1 - 1].clone()
        self.last_time = video.tstamp[self.t1 - 1].clone()
        with video.get_lock():
            video.ready.value = 1
            video.dirty[:self.t1] = True
        graph.rm_factors(graph.ii < self.warmup - 4, store=True)

    def __call__(self):
        """:112-121"""
        if not self.is_initialized and self.video.counter.value == self.warmup:
            self._initialize()
        elif self.is_initialized and self.t1 < self.video.counter.value:
            self._update()
