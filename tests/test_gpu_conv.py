"""Tensor-core (wgmma) implicit-GEMM convolution (A5) vs a plain PyTorch fp32 reference of the same op, and the
fused update operator vs the module-by-module library path.  fp16 inputs/weights, fp32 accumulate:
tolerance 1e-2 abs + 1e-2 rel on O(1) activations (fp16 output rounding), stated per test."""
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
WEIGHTS = os.path.join(ROOT, "oracle", "_ref", "droid.pth")


def _ref_conv(srcs_nhwc, w, b, pad):
    x = torch.cat([s.float() for s in srcs_nhwc], -1).permute(0, 3, 1, 2)
    return F.conv2d(x, w.float(), b.float(), padding=pad).permute(0, 2, 3, 1)


@pytest.mark.parametrize("cfg", [
    dict(chs=[128], k=3, N=128, B=3, H=30, W=40),
    dict(chs=[128, 128, 128, 64], k=3, N=128, B=2, H=60, W=80),
    dict(chs=[200], k=1, N=128, B=2, H=30, W=40, real=[196]),
    dict(chs=[128], k=3, N=64, B=2, H=20, W=24),
    dict(chs=[256], k=3, N=16, B=2, H=30, W=40),
    dict(chs=[128], k=3, N=256, B=2, H=30, W=40),
    dict(chs=[128], k=1, N=256, B=1, H=43, W=77),
    dict(chs=[128, 64], k=3, N=128, B=1, H=20, W=40),          # 9 tiles: fewer tiles than SMs, odd count
    dict(chs=[128], k=3, N=256, B=1, H=8, W=16),               # a single tile
    dict(chs=[128, 128, 128, 64], k=3, N=128, B=5, H=60, W=80),    # 200 tiles: several tiles per persistent CTA
])
@pytest.mark.parametrize("act", [0, 1])
def test_conv_matches_torch(cfg, act):
    from nerf_slam_b200.conv import conv_tc, pack_weights
    g = torch.Generator().manual_seed(5)
    B, H, W, k, N = cfg["B"], cfg["H"], cfg["W"], cfg["k"], cfg["N"]
    real = cfg.get("real", cfg["chs"])
    srcs = []
    for C, Cr in zip(cfg["chs"], real):
        t = torch.randn(B, H, W, C, generator=g).half()
        t[..., Cr:] = 0
        srcs.append(t.to(DEV))
    cin = sum(real)
    w = (torch.randn(N, cin, k, k, generator=g) / (cin * k * k) ** 0.5).half().to(DEV)
    b = torch.randn(N, generator=g).to(DEV)
    out = torch.full((B, H, W, N), float("nan"), dtype=torch.float16, device=DEV)
    conv_tc(srcs, pack_weights(w, real), b, B, H, W, k, k // 2, N, mode=0, act=act, out0=out, out0_channels=N)
    torch.cuda.synchronize()
    ref = _ref_conv([s[..., :Cr] for s, Cr in zip(srcs, real)], w, b, k // 2)
    if act == 1:
        ref = torch.relu(ref)
    err = (out.float() - ref).abs()
    assert torch.isfinite(out).all()
    assert float((err - 1e-2 * ref.abs()).max()) < 1e-2, float(err.max())


def test_gru_fused_epilogues():
    """modes 3 (glo), 1 (z, r*net) and 2 (state update) against the ConvGRU equations (gru.py:19-32)"""
    from nerf_slam_b200.conv import conv_tc, pack_weights
    g = torch.Generator().manual_seed(9)
    B, H, W = 2, 30, 40
    rnd = lambda *s: torch.randn(*s, generator=g)
    net = (rnd(B, H, W, 128) * 0.5).half().to(DEV); inp = (rnd(B, H, W, 128) * 0.5).half().to(DEV)
    cor = (rnd(B, H, W, 128) * 0.5).half().to(DEV); flo = (rnd(B, H, W, 64) * 0.5).half().to(DEV)
    wz, wr, wq = [(rnd(128, 448, 3, 3) / 63).half().to(DEV) for _ in range(3)]
    bz, br, bq = [rnd(128).to(DEV) * 0.1 for _ in range(3)]
    ww = (rnd(128, 128, 1, 1) / 11).half().to(DEV); bw = rnd(128).to(DEV) * 0.1
    gz, gr, gq = [rnd(B, 128).to(DEV) * 0.1 for _ in range(3)]
    # glo
    gsum = torch.zeros(B, 128, device=DEV)
    conv_tc([net], pack_weights(ww, [128]), bw, B, H, W, 1, 0, 128, mode=3, net=net, gsum=gsum)
    ref_glo = (torch.sigmoid(_ref_conv([net], ww, bw, 0)) * net.float()).sum((1, 2))
    assert torch.allclose(gsum, ref_glo, rtol=2e-3, atol=2e-2), (gsum - ref_glo).abs().max()
    # z, r
    z = torch.empty(B, H, W, 128, dtype=torch.float16, device=DEV); rnet = torch.empty_like(z)
    srcs = [net, inp, cor, flo]
    conv_tc(srcs, pack_weights(torch.cat([wz, wr], 0), [128, 128, 128, 64]), torch.cat([bz, br]), B, H, W, 3, 1, 256,
            mode=1, gctx=torch.cat([gz, gr], 1).contiguous(), net=net, out0=z, out0_channels=128, out1=rnet)
    zr = torch.sigmoid(_ref_conv(srcs, wz, bz, 1) + gz[:, None, None])
    rr = torch.sigmoid(_ref_conv(srcs, wr, br, 1) + gr[:, None, None])
    assert torch.allclose(z.float(), zr, atol=6e-3), (z.float() - zr).abs().max()
    assert torch.allclose(rnet.float(), rr * net.float(), atol=8e-3), (rnet.float() - rr * net.float()).abs().max()
    # q + state update
    out = torch.empty_like(z)
    conv_tc([rnet, inp, cor, flo], pack_weights(wq, [128, 128, 128, 64]), bq, B, H, W, 3, 1, 128, mode=2, gctx=gq,
            net=net, zbuf=z, out0=out, out0_channels=128)
    q = torch.tanh(_ref_conv([rnet, inp, cor, flo], wq, bq, 1) + gq[:, None, None])
    ref = (1 - z.float()) * net.float() + z.float() * q
    torch.cuda.synchronize()
    assert torch.allclose(out.float(), ref, atol=1e-2), (out.float() - ref).abs().max()


@pytest.mark.parametrize("with_agg", [False, True])
def test_update_operator_tc_vs_library_path(with_agg):
    """full UpdateModule.forward: fused tensor-core operator vs the per-layer library path, same weights"""
    from nerf_slam_b200.conv import CORR_PAD, UpdateOperatorTC
    from nerf_slam_b200.networks import UpdateModule, load_droid_weights
    um = UpdateModule(torch.Generator().manual_seed(3))
    if os.path.exists(WEIGHTS):
        um.load_state_dict(load_droid_weights(WEIGHTS), "update_net.")
    um.to(device=DEV, dtype=torch.float16)
    op = UpdateOperatorTC(um, DEV)
    g = torch.Generator().manual_seed(4)
    E, H, W = 5, 30, 40
    net = torch.tanh(torch.randn(E, H, W, 128, generator=g)).half().to(DEV)
    inp = torch.relu(torch.randn(E, H, W, 128, generator=g)).half().to(DEV)
    corr = torch.zeros(E, H, W, CORR_PAD)
    corr[..., :196] = torch.randn(E, H, W, 196, generator=g) * 2
    corr = corr.half().to(DEV)
    motion = (torch.randn(E, 4, H, W, generator=g) * 3).to(DEV)
    ii = torch.tensor([0, 0, 1, 2, 2], device=DEV) if with_agg else None
    got = op.call_reference_convention(net, inp, corr, motion, ii)
    nchw = lambda t: t.permute(0, 3, 1, 2)
    ref = um(nchw(net)[None], nchw(inp)[None], nchw(corr[..., :196])[None], motion[None], ii, ii)
    torch.cuda.synchronize()
    close = lambda a, b, tol: float((a.float() - b.float()).abs().max()) < tol
    assert close(got[0], ref[0][0].permute(0, 2, 3, 1), 3e-2)           # hidden state
    assert close(got[1], ref[1][0], 6e-2), float((got[1] - ref[1][0].float()).abs().max())   # delta [px]
    assert close(got[2], ref[2][0], 2e-2)                               # weight in (0,1)
    if with_agg:
        assert close(got[3], ref[3][0], 2e-3)                           # eta
        assert close(got[4], ref[4][0].permute(0, 2, 3, 1), 8e-2)       # upmask logits


@pytest.mark.parametrize("norm,out_dim", [("instance", 128), ("none", 256)])
def test_encoder_tc_vs_library_path(norm, out_dim):
    """BasicEncoder on the tensor-core kernel (im2col first layer, statistics in the conv epilogue, stride-2
    stores) vs the same network through the library convolutions; two images, sizes that leave partial tiles"""
    from nerf_slam_b200.conv import EncoderTC
    from nerf_slam_b200.networks import BasicEncoder, load_droid_weights
    enc = BasicEncoder(out_dim, norm, torch.Generator().manual_seed(5))
    if os.path.exists(WEIGHTS):
        enc.load_state_dict(load_droid_weights(WEIGHTS), "feature_net." if norm == "instance" else "context_net.")
    enc.to(device=DEV, dtype=torch.float16)
    g = torch.Generator().manual_seed(6)
    x = torch.randn(1, 2, 3, 120, 152, generator=g).to(DEV)
    ref = enc(x)[0].float()
    got = EncoderTC(enc, DEV)(x[0]).float()
    torch.cuda.synchronize()
    assert got.shape == ref.shape == (2, out_dim, 15, 19)
    err = float((got - ref).abs().max())
    assert err < 5e-2 * max(1.0, float(ref.abs().max())), err


def test_update_op_step_matches_python_sequencing():
    """nslam_update_op_step (one C call, fixed workspace, in-place hidden state) vs UpdateOperatorTC.__call__
    (the same kernels issued one by one from Python).  Not bit-identical: the global-context column sums are
    fp32 atomics (order varies run to run) and the context GEMV is a different fp32 summation order than
    torch.addmm; everything downstream agrees to fp16 rounding."""
    from nerf_slam_b200 import _lib
    from nerf_slam_b200.conv import CORR_PAD, UpdateOperatorTC
    from nerf_slam_b200.networks import UpdateModule, load_droid_weights
    um = UpdateModule(torch.Generator().manual_seed(3))
    if os.path.exists(WEIGHTS):
        um.load_state_dict(load_droid_weights(WEIGHTS), "update_net.")
    um.to(device=DEV, dtype=torch.float16)
    op = UpdateOperatorTC(um, DEV)
    g = torch.Generator().manual_seed(14)
    E, H, W = 6, 30, 40
    net = torch.tanh(torch.randn(E, H, W, 128, generator=g)).half().to(DEV)
    inp = torch.relu(torch.randn(E, H, W, 128, generator=g)).half().to(DEV)
    corr = torch.zeros(E, H, W, CORR_PAD); corr[..., :196] = torch.randn(E, H, W, 196, generator=g) * 2
    corr = corr.half().to(DEV)
    yy, xx = torch.meshgrid(torch.arange(H).float(), torch.arange(W).float(), indexing="ij")
    coords0 = torch.stack([xx, yy], -1).contiguous().to(DEV)
    coords1 = (coords0[None] + torch.randn(E, H, W, 2, generator=g).to(DEV) * 3).contiguous()
    target = (coords1 + torch.randn(E, H, W, 2, generator=g).to(DEV) * 2).contiguous()
    ii = np.array([0, 0, 1, 2, 2, 2])
    ux, inv = np.unique(ii, return_inverse=True)
    order = np.argsort(inv, kind="stable").astype(np.int32)
    ptr = np.zeros(len(ux) + 1, np.int32); np.cumsum(np.bincount(inv), out=ptr[1:])
    seg_ptr, seg_edges, K = torch.as_tensor(ptr, device=DEV), torch.as_tensor(order, device=DEV), len(ux)
    ref = op(net, inp, corr, coords1, coords0, target=target, agg=(seg_ptr, seg_edges, K))
    ref = [t.clone() for t in ref]
    # one-call path
    ctx, ws = op.make_step(E, K, H, W, DEV)
    net2 = net.clone(); flow = target.clone(); conf = torch.empty_like(flow)
    bt = torch.empty(E, 2, H, W, device=DEV); bw = torch.empty_like(bt)
    upmask = torch.empty(K, H, W, 576, dtype=torch.float16, device=DEV)
    uxd = torch.as_tensor(ux, device=DEV); damping = torch.zeros(8, H, W, device=DEV); bad = torch.empty(K, H, W, device=DEV)
    ctx.net = ctx.net_out = net2.data_ptr(); ctx.inp = inp.data_ptr(); ctx.corr = corr.data_ptr()
    ctx.coords1, ctx.coords0 = coords1.data_ptr(), coords0.data_ptr()
    ctx.target = ctx.flow = flow.data_ptr(); ctx.conf = conf.data_ptr()
    ctx.ba_target, ctx.ba_weight = bt.data_ptr(), bw.data_ptr()
    ctx.seg_ptr, ctx.seg_edges = seg_ptr.data_ptr(), seg_edges.data_ptr()
    ctx.upmask = upmask.data_ptr()
    ctx.ux, ctx.damping, ctx.kx_ba, ctx.ba_damp, ctx.Kba, ctx.ep = uxd.data_ptr(), damping.data_ptr(), uxd.data_ptr(), bad.data_ptr(), K, 1e-7
    op.step(ctx)
    torch.cuda.synchronize()
    md = lambda a, b: float((a.float() - b.float()).abs().max())
    assert md(net2, ref[0]) < 4e-3 and md(flow, ref[1]) < 4e-2 and md(conf, ref[2]) < 2e-3, (md(net2, ref[0]), md(flow, ref[1]), md(conf, ref[2]))
    assert md(upmask, ref[4]) < 2e-2
    assert torch.equal(bt, flow.permute(0, 3, 1, 2)) and torch.equal(bw, conf.permute(0, 3, 1, 2))
    eta = 0.01 * torch.nn.functional.softplus(ref[3][..., 0].float())
    assert torch.allclose(damping[uxd], eta, rtol=2e-2, atol=1e-5)
    assert torch.allclose(bad, 0.2 * damping[uxd] + 1e-7, rtol=1e-5, atol=1e-9)
