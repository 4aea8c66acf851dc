"""Tensor-core (wgmma) execution of the update operator — host side.

`UpdateOperatorTC` evaluates the reference's UpdateModule.forward (networks/droid_net.py:118-150;
ConvGRU networks/modules/gru.py:19-32; GraphAgg networks/droid_net.py:59-75) with every 3x3 / 1x1
convolution on the hand-written implicit-GEMM kernel (csrc/conv_igemm.cu, C ABI
include/nslam_nn.h).  Activations are NHWC fp16 end to end; `torch.cat` inputs are never
materialised (multi-source K loop); sigmoid/tanh/GRU gating/global-context reduction are epilogues.

Fusions (what replaces what):
  z, r gates      : ONE conv with N=256 over [net|inp|corr|flow] -> z and r*net    (2 convs + cat + 3 elementwise)
  q + state update: ONE conv, epilogue (1-z)*net + z*tanh(.)                      (conv + cat + 3 elementwise)
  glo             : 1x1 conv with epilogue sigmoid(.)*net and per-image column sums (conv + mul + mean)
  delta.0|weight.0: ONE conv with N=256 from the shared input
  delta.2|weight.2: ONE block-diagonal conv with N=16
The 7x7 conv on the 4-channel motion input runs as a 1x1 GEMM on an im2col tile written by
nslam_motion_im2col together with the motion features themselves; the head outputs, GraphAgg's
scatter-mean and the damping update are small fused kernels (csrc/update_glue.cu).
"""
import ctypes

import torch

from . import _lib


def pack_weights(w, src_channels, n_pad=None):
    """w [N, sum(src_channels), KH, KW] (torch conv layout) -> packed fp16 image for conv_igemm:
    [KH*KW * sum(ceil(C_s/64))] blocks of [N_pad][64], each row 128-B swizzled (16-B chunk j of row n
    stored at chunk j ^ (n & 7)).  Channels beyond a source's real count are zero."""
    N, Cin, KH, KW = w.shape
    assert Cin == sum(src_channels)
    Np = n_pad or N
    dev = w.device
    blocks = []
    wf = w.float()
    rows = torch.arange(Np, device=dev)
    perm = (torch.arange(8, device=dev)[None, :] ^ (rows % 8)[:, None])        # [Np,8]: dest chunk of src chunk j
    for ky in range(KH):
        for kx in range(KW):
            off = 0
            for C in src_channels:
                for cb in range((C + 63) // 64):
                    blk = torch.zeros(Np, 64, device=dev)
                    cs, ce = cb * 64, min(C, cb * 64 + 64)
                    blk[:N, :ce - cs] = wf[:, off + cs:off + ce, ky, kx]
                    src = blk.view(Np, 8, 8)
                    dst = torch.empty_like(src)
                    dst.scatter_(1, perm[:, :, None].expand(Np, 8, 8), src)
                    blocks.append(dst.reshape(-1))
                off += C
    return torch.cat(blocks).half().contiguous()


def conv_partials(B, H, W, N, k, device):
    """scratch of the per-tile column sums (mode 3: k = 1; mode 4 statistics: k = 2) that the kernel reduces in a
    fixed order, 4 row quarters per 8x16-pixel tile (include/nslam_nn.h)"""
    T = ((H + 7) // 8) * ((W + 15) // 16)
    return torch.empty(B * T * 4 * N * k, dtype=torch.float32, device=device)


def conv_tc(srcs, wpacked, bias, B, H, W, KH, pad, N, mode=0, act=0, gctx=None, net=None, zbuf=None,
            gsum=None, out0=None, out0_channels=None, out1=None, num_sms=132):
    lib = _lib.load()
    part = conv_partials(B, H, W, N, 1, srcs[0].device) if mode == 3 else None
    n = len(srcs)
    ptrs = (ctypes.c_void_p * n)(*[s.data_ptr() for s in srcs])
    chans = (ctypes.c_int * n)(*[s.shape[-1] for s in srcs])
    _lib.check(lib.nslam_conv_igemm(ctypes.cast(ptrs, ctypes.c_void_p), ctypes.cast(chans, ctypes.c_void_p), n,
                                    B, H, W, KH, KH, pad, N, _lib.ptr(wpacked), _lib.ptr(bias), mode, act,
                                    _lib.ptr(gctx), _lib.ptr(net), _lib.ptr(zbuf), _lib.ptr(gsum), _lib.ptr(out0),
                                    int(out0_channels or 0), _lib.ptr(out1), _lib.ptr(part), num_sms, _lib.stream_ptr()),
               "conv_igemm")


def _sm_budget(device, env):
    """number of SMs a family of PERSISTENT kernels may occupy (grid size).  SLAM and NeRF run on two streams
    of one GPU; their persistent CTAs do not pre-empt each other, so a static split (e.g. NSLAM_SLAM_SMS=108,
    NSLAM_NERF_SMS=40) keeps the latency-critical SLAM kernels from waiting for a NeRF CTA to retire."""
    import os
    n = torch.cuda.get_device_properties(device).multi_processor_count
    v = int(os.environ.get(env, "0"))
    return max(1, min(n, v)) if v > 0 else n


CORR_PAD = 200      # 196 correlation channels padded to a multiple of 8 (TMA stride rule), zero tail
MOTION_COLS = 200   # 7x7x4 im2col of the motion input (196) padded the same way


class UpdateOperatorTC:
    """drop-in for networks.UpdateModule.__call__ with NHWC tensors.

    see __call__.
    """

    def __init__(self, params, device):
        """params: networks.UpdateModule (its state_dict tensors)"""
        sd = {k: v.to(device).float() for k, v in params.state_dict().items()}
        self.dev = device
        self.num_sms = _sm_budget(device, "NSLAM_SLAM_SMS")
        f32 = lambda t: t.float().contiguous()
        P = {}
        P["ce0"] = (pack_weights(sd["corr_encoder.0.weight"], [196]), f32(sd["corr_encoder.0.bias"]))
        # the packed block layout depends on the channel count of the SOURCE TENSOR (CORR_PAD), whose
        # 64-blocks coincide with those of 196 real channels (4 blocks either way)
        P["ce2"] = (pack_weights(sd["corr_encoder.2.weight"], [128]), f32(sd["corr_encoder.2.bias"]))
        P["fe2"] = (pack_weights(sd["flow_encoder.2.weight"], [128]), f32(sd["flow_encoder.2.bias"]))
        # 7x7 conv on the 4-channel motion input = 1x1 GEMM on its im2col (csrc/update_glue.cu): K index = tap*4 + c
        w0 = torch.zeros(128, MOTION_COLS, 1, 1, device=device)
        w0[:, :196, 0, 0] = sd["flow_encoder.0.weight"].permute(0, 2, 3, 1).reshape(128, 196)
        P["fe0"] = (pack_weights(w0, [MOTION_COLS]), f32(sd["flow_encoder.0.bias"]))
        P["glo"] = (pack_weights(sd["gru.w.weight"], [128]), f32(sd["gru.w.bias"]))
        src4 = [128, 128, 128, 64]
        P["zr"] = (pack_weights(torch.cat([sd["gru.convz.weight"], sd["gru.convr.weight"]], 0), src4),
                   f32(torch.cat([sd["gru.convz.bias"], sd["gru.convr.bias"]])))
        P["q"] = (pack_weights(sd["gru.convq.weight"], src4), f32(sd["gru.convq.bias"]))
        self.glo_w = torch.cat([sd["gru.convz_glo.weight"], sd["gru.convr_glo.weight"], sd["gru.convq_glo.weight"]], 0)[:, :, 0, 0].contiguous()
        self.glo_b = torch.cat([sd["gru.convz_glo.bias"], sd["gru.convr_glo.bias"], sd["gru.convq_glo.bias"]]).contiguous()
        P["h0"] = (pack_weights(torch.cat([sd["delta.0.weight"], sd["weight.0.weight"]], 0), [128]),
                   f32(torch.cat([sd["delta.0.bias"], sd["weight.0.bias"]])))
        w2 = torch.zeros(16, 256, 3, 3, device=device)
        w2[0:2, 0:128] = sd["delta.2.weight"]; w2[2:4, 128:256] = sd["weight.2.weight"]
        b2 = torch.zeros(16, device=device); b2[0:2] = sd["delta.2.bias"]; b2[2:4] = sd["weight.2.bias"]
        P["h2"] = (pack_weights(w2, [256]), b2)
        P["a1"] = (pack_weights(sd["agg.conv1.weight"], [128]), f32(sd["agg.conv1.bias"]))
        P["a2"] = (pack_weights(sd["agg.conv2.weight"], [128]), f32(sd["agg.conv2.bias"]))
        we = torch.zeros(16, 128, 3, 3, device=device); we[0:1] = sd["agg.eta.0.weight"]
        be = torch.zeros(16, device=device); be[0:1] = sd["agg.eta.0.bias"]
        P["eta"] = (pack_weights(we, [128]), be)
        um_w, um_b = sd["agg.upmask.0.weight"], sd["agg.upmask.0.bias"]
        P["um"] = [(pack_weights(um_w[c0:c0 + n], [128]), f32(um_b[c0:c0 + n]), c0, n) for c0, n in ((0, 256), (256, 256), (512, 64))]
        self.P = P

    def _conv(self, key, srcs, B, H, W, k, N, out, **kw):
        wp, b = self.P[key][:2]
        conv_tc(srcs, wp, b, B, H, W, k, k // 2, N, out0=out, out0_channels=out.shape[-1] if out is not None else 0,
                num_sms=self.num_sms, **kw)

    def __call__(self, net, inp, corr, coords1, coords0, target=None, agg=None, post=None):
        """net, inp [E,ht,wd,128] f16; corr [E,ht,wd,CORR_PAD] f16; coords1 [E,ht,wd,2] f32 (reprojected
        grid), coords0 [ht,wd,2] f32, target [E,ht,wd,2] f32 or None (-> zero flow residual).
        agg = (seg_ptr int32 [K+1], seg_edges int32 [E], K): CSR of the edges per source keyframe, or None.
        post = (flow, conf, ba_target, ba_weight) output tensors ([E,ht,wd,2] x2, planar [E,2,ht,wd] x2
        or None x2), or None to allocate flow/conf.
        -> net' [E,ht,wd,128] f16, flow = coords1 + delta, conf = sigmoid(weight logits)
           (, e16 [K,ht,wd,16] f16 with the eta logit in column 0, upmask [K,ht,wd,576] f16)"""
        lib = _lib.load()
        E, H, W, _ = net.shape
        dev = net.device
        h16 = dict(dtype=torch.float16, device=dev)
        new = lambda c: torch.empty(E, H, W, c, **h16)
        sp = _lib.stream_ptr()
        # correlation / motion encoders
        c1 = new(128); self._conv("ce0", [corr], E, H, W, 1, 128, c1, act=1)
        c2 = new(128); self._conv("ce2", [c1], E, H, W, 3, 128, c2, act=1)
        mcol = new(MOTION_COLS)
        _lib.check(lib.nslam_motion_im2col(_lib.ptr(coords1), _lib.ptr(coords0), _lib.ptr(target), _lib.ptr(mcol),
                                           E, H, W, sp), "motion_im2col")
        f1 = new(128); self._conv("fe0", [mcol], E, H, W, 1, 128, f1, act=1)
        f2 = new(64); self._conv("fe2", [f1], E, H, W, 3, 64, f2, act=1)
        # global context: glo = mean_hw(sigmoid(w(net)) * net) ; then the three 1x1 "glo" convs as one GEMV batch
        gsum = torch.zeros(E, 128, dtype=torch.float32, device=dev)
        self._conv("glo", [net], E, H, W, 1, 128, None, mode=3, net=net, gsum=gsum)
        glo = (gsum * (1.0 / (H * W))).half().float()               # the reference's glo is an fp16 tensor
        g3 = torch.addmm(self.glo_b, glo, self.glo_w.t())           # [E,384] = z|r|q context terms
        gzr = g3[:, :256].contiguous(); gq = g3[:, 256:].contiguous()
        # GRU
        z = new(128); rnet = new(128)
        srcs = [net, inp, c2, f2]
        wp, b = self.P["zr"]
        conv_tc(srcs, wp, b, E, H, W, 3, 1, 256, mode=1, gctx=gzr, net=net, out0=z, out0_channels=128, out1=rnet, num_sms=self.num_sms)
        net2 = new(128)
        wp, b = self.P["q"]
        conv_tc([rnet, inp, c2, f2], wp, b, E, H, W, 3, 1, 128, mode=2, gctx=gq, net=net, zbuf=z, out0=net2, out0_channels=128,
                num_sms=self.num_sms)
        # heads
        h0 = new(256); self._conv("h0", [net2], E, H, W, 3, 256, h0, act=1)
        h2 = new(16); self._conv("h2", [h0], E, H, W, 3, 16, h2, act=0)
        if post is None:
            post = (torch.empty(E, H, W, 2, device=dev), torch.empty(E, H, W, 2, device=dev), None, None)
        flow, conf, ba_t, ba_w = post
        _lib.check(lib.nslam_flow_heads_post(_lib.ptr(h2), _lib.ptr(coords1), _lib.ptr(flow), _lib.ptr(conf),
                                             _lib.ptr(ba_t), _lib.ptr(ba_w), E, H * W, sp), "flow_heads_post")
        if agg is None:
            return net2, flow, conf
        # GraphAgg
        seg_ptr, seg_edges, K = agg
        a1 = new(128); self._conv("a1", [net2], E, H, W, 3, 128, a1, act=1)
        am = torch.empty(K, H, W, 128, **h16)
        _lib.check(lib.nslam_segment_mean(_lib.ptr(a1), _lib.ptr(seg_ptr), _lib.ptr(seg_edges), _lib.ptr(am), K, H * W, sp),
                   "segment_mean")
        a2 = torch.empty(K, H, W, 128, **h16); self._conv("a2", [am], K, H, W, 3, 128, a2, act=1)
        e16 = torch.empty(K, H, W, 16, **h16); self._conv("eta", [a2], K, H, W, 3, 16, e16, act=0)
        upmask = torch.empty(K, H, W, 576, **h16)
        for wp, b, c0, n in self.P["um"]:
            conv_tc([a2], wp, b, K, H, W, 1, 0, n, out0=upmask[..., c0:], out0_channels=576, num_sms=self.num_sms)
        return net2, flow, conf, e16, upmask

    W_ORDER = ("ce0", "ce2", "fe0", "fe2", "glo", "zr", "q", "h0", "h2", "a1", "a2", "eta", "um0", "um1", "um2")

    def make_step(self, E, K, H, W, device):
        """-> (ctx, keep): a `nslam_update_ctx` for a fixed (E, K) with all intermediates in ONE workspace
        tensor; the caller fills the input/output pointers and calls `step(ctx)`.  `keep` holds the tensors the
        ctx points into."""
        ctx = _lib.UpdateCtx()
        ctx.E, ctx.K, ctx.H, ctx.W, ctx.num_sms, ctx.corr_channels = E, K, H, W, self.num_sms, CORR_PAD
        um = {f"um{i}": (wp, b) for i, (wp, b, c0, n) in enumerate(self.P["um"])}
        for i, name in enumerate(self.W_ORDER):
            wp, b = (um[name] if name in um else self.P[name][:2])
            ctx.wp[i] = wp.data_ptr(); ctx.bias[i] = b.data_ptr() if b is not None else None
        ctx.glo_w, ctx.glo_b = self.glo_w.data_ptr(), self.glo_b.data_ptr()
        hw = H * W
        tiles = ((H + 7) // 8) * ((W + 15) // 16)               # gsum is followed by the glo convolution's partials
        sizes = dict(c1=E * hw * 128 * 2, c2=E * hw * 128 * 2, mcol=E * hw * MOTION_COLS * 2, f1=E * hw * 128 * 2,
                     f2=E * hw * 64 * 2, gsum=E * 128 * 4 * (1 + 4 * tiles), gzr=E * 256 * 4, gq=E * 128 * 4, z=E * hw * 128 * 2,
                     rnet=E * hw * 128 * 2, h0=E * hw * 256 * 2, h2=E * hw * 16 * 2, a1=E * hw * 128 * 2,
                     am=max(K, 1) * hw * 128 * 2, a2=max(K, 1) * hw * 128 * 2, e16=max(K, 1) * hw * 16 * 2)
        total = sum((v + 255) // 256 * 256 for v in sizes.values())
        ws = torch.empty(total, dtype=torch.uint8, device=device)
        off = 0
        for name, v in sizes.items():
            setattr(ctx, name, ws.data_ptr() + off)
            off += (v + 255) // 256 * 256
        return ctx, ws

    @staticmethod
    def step(ctx):
        _lib.check(_lib.load().nslam_update_op_step(ctypes.byref(ctx), _lib.stream_ptr()), "update_op_step")

    def call_reference_convention(self, net, inp, corr, motion, ii=None):
        """UpdateModule.forward's own argument/return convention (droid_net.py:118-150) on top of the fused
        operator — used by the parity tests: motion [E,4,ht,wd] (|.| < 64) is turned into the coordinate
        tensors it is derived from in the frontend; returns net, delta, weight (, eta, upmask NHWC)."""
        import numpy as np
        E, H, W, _ = net.shape
        dev = net.device
        yy, xx = torch.meshgrid(torch.arange(H, device=dev).float(), torch.arange(W, device=dev).float(), indexing="ij")
        coords0 = torch.stack([xx, yy], -1).contiguous()
        m = motion.float().permute(0, 2, 3, 1)
        coords1 = (coords0[None] + m[..., 0:2]).contiguous()
        target = (coords1 + m[..., 2:4]).contiguous()
        agg = None
        if ii is not None:
            ux, inv = np.unique(ii.cpu().numpy(), return_inverse=True)
            order = np.argsort(inv, kind="stable").astype(np.int32)
            ptr = np.zeros(len(ux) + 1, np.int32); np.cumsum(np.bincount(inv, minlength=len(ux)), out=ptr[1:])
            agg = (torch.as_tensor(ptr, device=dev), torch.as_tensor(order, device=dev), len(ux))
        out = self(net, inp, corr, coords1, coords0, target=target, agg=agg)
        delta = out[1] - coords1
        if ii is None:
            return out[0], delta, out[2]
        eta = 0.01 * torch.nn.functional.softplus(out[3][..., 0].float())
        return out[0], delta, out[2], eta, out[4]


def conv_enc(srcs, wpacked, bias, B, H, W, k, N, out, act=0, stats=None, sub=1, num_sms=132):
    """encoder layer on the tensor-core kernel (mode 4): NHWC fp16 in/out, optional channel statistics for the
    instance norm that follows, optional stride 2 (out is then [B,ceil(H/2),ceil(W/2),N])"""
    lib = _lib.load()
    n = len(srcs)
    ptrs = (ctypes.c_void_p * n)(*[s.data_ptr() for s in srcs])
    chans = (ctypes.c_int * n)(*[s.shape[-1] for s in srcs])
    part = conv_partials(B, H, W, N, 2, out.device) if stats is not None else None
    _lib.check(lib.nslam_conv_igemm_ex(ctypes.cast(ptrs, ctypes.c_void_p), ctypes.cast(chans, ctypes.c_void_p), n,
                                       B, H, W, k, k, k // 2, N, _lib.ptr(wpacked), _lib.ptr(bias), 4, act,
                                       None, None, None, None, _lib.ptr(out), out.shape[-1], None, _lib.ptr(stats), sub,
                                       _lib.ptr(part), num_sms, _lib.stream_ptr()), "conv_igemm_ex")


class EncoderTC:
    """BasicEncoder.forward (networks/modules/extractor.py:183-198, ResidualBlock :6-55) on the tensor-core
    convolution kernel, NHWC fp16 end to end:
      7x7/s2 first layer = im2col (csrc/update_glue.cu) + 1x1 GEMM; every other layer = conv_igemm mode 4;
      stride-2 layers are evaluated at stride 1 and store / count only the even pixels;
      norm_fn='instance': the convolutions accumulate the channel statistics in their epilogue, one fused apply
      pass does norm + ReLU (+ residual [+ its own norm] + ReLU); biases in front of a norm are dropped (they cancel);
      norm_fn='none' (context encoder): bias + ReLU in the conv epilogue, residual add + ReLU in the apply pass."""

    def __init__(self, enc, device):
        from . import networks as nw
        self.inorm = enc.norm is nw._inorm
        self.dev = device
        self.num_sms = _sm_budget(device, "NSLAM_SLAM_SMS")
        sd = {k: v.to(device).float() for k, v in enc.state_dict().items()}
        f32 = lambda t: t.float().contiguous()
        bias = (lambda k: None) if self.inorm else (lambda k: f32(sd[k + ".bias"]))
        P = {}
        w1 = torch.zeros(32, 152, 1, 1, device=device)
        w1[:, :147, 0, 0] = sd["conv1.weight"].permute(0, 2, 3, 1).reshape(32, 147)       # K index = (ky*7+kx)*3 + c
        P["conv1"] = (pack_weights(w1, [152]), bias("conv1"), 32)
        self.blocks = []
        for name, st in enc.blocks:
            cin = sd[name + ".conv1.weight"].shape[1]; cout = sd[name + ".conv1.weight"].shape[0]
            P[name + ".conv1"] = (pack_weights(sd[name + ".conv1.weight"], [cin]), bias(name + ".conv1"), cout)
            P[name + ".conv2"] = (pack_weights(sd[name + ".conv2.weight"], [cout]), bias(name + ".conv2"), cout)
            if st != 1:
                P[name + ".down"] = (pack_weights(sd[name + ".downsample.0.weight"], [cin]), bias(name + ".downsample.0"), cout)
            self.blocks.append((name, st, cin, cout))
        cout = sd["conv2.weight"].shape[0]
        P["conv2"] = (pack_weights(sd["conv2.weight"], [sd["conv2.weight"].shape[1]]), f32(sd["conv2.bias"]), cout)
        self.P = P

    def __call__(self, x):
        """x [B,3,H,W] fp32 normalised image -> [B,C,H/8,W/8] fp16 (NCHW view of NHWC storage)"""
        from . import networks as nw
        lib = _lib.load()
        B, _, H, W = x.shape
        dev = x.device
        h16 = dict(dtype=torch.float16, device=dev)
        x = x.float().contiguous()
        arena = torch.zeros(16, B * 128 * 2, dtype=torch.float32, device=dev) if self.inorm else None
        slot = [0]

        def st_buf(C):
            if arena is None:
                return None
            v = arena[slot[0]][:B * C * 2].view(B, C, 2)
            slot[0] += 1
            return v

        def nchw(t):                      # NHWC storage viewed as the NCHW-shaped channels-last tensor inorm_apply expects
            return t.permute(0, 3, 1, 2)
        act = 0 if self.inorm else 1
        h, w = H // 2, W // 2
        col = torch.empty(B, h, w, 152, **h16)
        _lib.check(lib.nslam_im2col7_s2(_lib.ptr(x), _lib.ptr(col), B, H, W, _lib.stream_ptr()), "im2col7")
        wp, b, n = self.P["conv1"]
        cur = torch.empty(B, h, w, n, **h16); s0 = st_buf(n)
        conv_enc([col], wp, b, B, h, w, 1, n, cur, act=act, stats=s0, num_sms=self.num_sms)
        if self.inorm:
            nw._inorm_apply(nchw(cur), s0)
        for name, st, cin, cout in self.blocks:
            ho, wo = (h + st - 1) // st, (w + st - 1) // st
            wp, b, _ = self.P[name + ".conv1"]
            y = torch.empty(B, ho, wo, cout, **h16); s1 = st_buf(cout)
            conv_enc([cur], wp, b, B, h, w, 3, cout, y, act=act, stats=s1, sub=st, num_sms=self.num_sms)
            if self.inorm:
                nw._inorm_apply(nchw(y), s1)
            wp, b, _ = self.P[name + ".conv2"]
            z = torch.empty(B, ho, wo, cout, **h16); s2 = st_buf(cout)
            conv_enc([y], wp, b, B, ho, wo, 3, cout, z, act=act, stats=s2, num_sms=self.num_sms)
            res, sr = cur, None
            if st != 1:
                wp, b, _ = self.P[name + ".down"]
                res = torch.empty(B, ho, wo, cout, **h16); sr = st_buf(cout)
                conv_enc([cur], wp, b, B, h, w, 1, cout, res, act=0, stats=sr, sub=st, num_sms=self.num_sms)
            # out = relu(res' + relu(norm?(z)));  z already carries its ReLU when there is no norm
            nw._inorm_apply(nchw(z), s2, relu=self.inorm, res=nchw(res), res_st=sr)
            cur, h, w = z, ho, wo
        wp, b, n = self.P["conv2"]
        out = torch.empty(B, h, w, n, **h16)
        conv_enc([cur], wp, b, B, h, w, 1, n, out, act=0, num_sms=self.num_sms)
        return out.permute(0, 3, 1, 2)
