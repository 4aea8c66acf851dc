"""CPU checks of the correlation backward passes: the oracle restatements (oracle/corr_grad.py) against torch fp64
autograd of the forwards, the derivation behind CorrBlock's gradient (dense volume route == on-the-fly route), and
the reference-composition golden (tests/golden/make_golden_corr_grad.py) reproduced by the product classes with the
oracle standing in for the kernels."""
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import corr as ocorr
from oracle import corr_grad as ograd

G = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _coords(rng, n, h1, w1, lo, hi, far=True):
    """[n,2,h1,w1] coordinates in [lo, hi) (windows straddle every border), some far outside the map"""
    c = rng.uniform(lo, hi, (n, 2, h1, w1)).astype(np.float32)
    if far:
        c[0, 0, 0, 0], c[0, 1, 0, 1], c[-1, 0, -1, -1], c[-1, 1, -1, -2] = 1e6, -1e6, -1e6, 1e6
    return c


def _lookup_t(volume, coords, r):
    """torch restatement of corr_index_forward (differentiable w.r.t. volume): [n,h1,w1,h2,w2] -> [n,rd,rd,h1,w1]"""
    n, h1, w1, h2, w2 = volume.shape
    rd = 2 * r + 1
    x0, y0 = coords[:, 0].double(), coords[:, 1].double()
    fx, fy = torch.floor(x0), torch.floor(y0)
    dx, dy = x0 - fx, y0 - fy
    xb, yb = fx.long() - r, fy.long() - r
    nn, yy, xx = torch.meshgrid(torch.arange(n), torch.arange(h1), torch.arange(w1), indexing="ij")
    taps = {}
    for i in range(rd + 1):
        for j in range(rd + 1):
            x1, y1 = xb + i, yb + j
            ok = (x1 >= 0) & (x1 < w2) & (y1 >= 0) & (y1 < h2)
            taps[i, j] = volume[nn, yy, xx, y1.clamp(0, h2 - 1), x1.clamp(0, w2 - 1)] * ok
    out = [[taps[i, j] * (1 - dx) * (1 - dy) + taps[i, j + 1] * (1 - dx) * dy + taps[i + 1, j] * dx * (1 - dy)
            + taps[i + 1, j + 1] * dx * dy for j in range(rd)] for i in range(rd)]
    return torch.stack([torch.stack(row, 1) for row in out], 1)


def _altcorr_t(f1, f2, coords, r):
    """torch restatement of altcorr_forward: f1 [B,H1,W1,C], f2 [B,H2,W2,C], coords [B,N,H1,W1,2] -> [B,N,rd^2,H1,W1]"""
    B, H1, W1, C = f1.shape
    _, H2, W2, _ = f2.shape
    N = coords.shape[1]
    rd = 2 * r + 1
    bb = torch.arange(B)[:, None, None]
    outs = []
    for n in range(N):
        x0, y0 = coords[:, n, ..., 0].double(), coords[:, n, ..., 1].double()
        fx, fy = torch.floor(x0), torch.floor(y0)
        dx, dy = x0 - fx, y0 - fy
        xb, yb = fx.long() - r, fy.long() - r
        dots = {}
        for iy in range(rd + 1):
            for ix in range(rd + 1):
                h2, w2 = yb + iy, xb + ix
                ok = (h2 >= 0) & (h2 < H2) & (w2 >= 0) & (w2 < W2)
                dots[iy, ix] = (f1 * f2[bb, h2.clamp(0, H2 - 1), w2.clamp(0, W2 - 1)]).sum(-1) * ok
        ch = [None] * (rd * rd)
        for ox in range(rd):
            for oy in range(rd):
                ch[oy + rd * ox] = (dots[oy, ox] * (1 - dy) * (1 - dx) + dots[oy, ox + 1] * (1 - dy) * dx
                                    + dots[oy + 1, ox] * dy * (1 - dx) + dots[oy + 1, ox + 1] * dy * dx)
        outs.append(torch.stack(ch, 1))
    return torch.stack(outs, 1)


def test_torch_restatements_match_the_forward_oracle():
    rng = np.random.default_rng(5)
    vol = rng.normal(0, 1, (2, 5, 6, 4, 7))
    c = _coords(rng, 2, 5, 6, -5, 11)
    got = _lookup_t(torch.from_numpy(vol), torch.from_numpy(c), 2).numpy()
    assert np.allclose(got, ocorr.corr_index_forward(vol.astype(np.float32), c, 2), atol=1e-5)
    f1, f2 = rng.normal(0, 1, (2, 5, 6, 8)), rng.normal(0, 1, (2, 4, 7, 8))
    ca = np.moveaxis(_coords(rng, 2 * 3, 5, 6, -5, 11), 1, -1).reshape(2, 3, 5, 6, 2).copy()
    got = _altcorr_t(torch.from_numpy(f1), torch.from_numpy(f2), torch.from_numpy(ca), 2).numpy()
    assert np.allclose(got, ocorr.altcorr_forward(f1.astype(np.float32), f2.astype(np.float32), ca, 2), atol=1e-4)


@pytest.mark.parametrize("r", [1, 2, 3])
def test_corr_index_backward_oracle_vs_fp64_autograd(r):
    rng = np.random.default_rng(10 + r)
    shape = (2, 5, 6, 4, 7)
    rd = 2 * r + 1
    c = _coords(rng, 2, 5, 6, -2 * r - 2, 9 + r)
    g = rng.normal(0, 1, (2, rd, rd, 5, 6))
    vol = torch.from_numpy(rng.normal(0, 1, shape)).requires_grad_()
    _lookup_t(vol, torch.from_numpy(c), r).backward(torch.from_numpy(g))
    ref = vol.grad.numpy()
    got = ograd.corr_index_backward(shape, c, g, r)
    assert got.dtype == np.float64
    assert np.allclose(got, ref, rtol=1e-12, atol=1e-12)
    assert np.count_nonzero(ref) > 0 and np.count_nonzero(got == 0) > 0
    # fp32 / fp16 restatements: the same values up to their rounding, +0 (never -0) where nothing is written
    g32 = ograd.corr_index_backward(shape, c, g.astype(np.float32), r)
    assert g32.dtype == np.float32 and np.abs(g32 - ref).max() <= 1e-5 * np.abs(ref).max()
    g16 = ograd.corr_index_backward(shape, c, g.astype(np.float16), r)
    assert g16.dtype == np.float16 and np.abs(g16.astype(np.float64) - ref).max() <= 1e-2 * np.abs(ref).max()
    assert not np.signbit(g16[g16 == 0]).any() and not np.signbit(g32[g32 == 0]).any()


@pytest.mark.parametrize("r,N", [(1, 1), (2, 3), (3, 2)])
def test_altcorr_backward_oracle_vs_fp64_autograd(r, N):
    rng = np.random.default_rng(20 + r)
    B, H1, W1, H2, W2, C = 2, 5, 6, 4, 7, 8
    rd = 2 * r + 1
    c = np.moveaxis(_coords(rng, B * N, H1, W1, -2 * r - 2, 9 + r), 1, -1).reshape(B, N, H1, W1, 2).copy()
    g = rng.normal(0, 1, (B, N, rd * rd, H1, W1))
    f1 = torch.from_numpy(rng.normal(0, 1, (B, H1, W1, C))).requires_grad_()
    f2 = torch.from_numpy(rng.normal(0, 1, (B, H2, W2, C))).requires_grad_()
    _altcorr_t(f1, f2, torch.from_numpy(c), r).backward(torch.from_numpy(g))
    g1, g2, gc = ograd.altcorr_backward(f1.detach().numpy(), f2.detach().numpy(), c, g, r)
    assert np.allclose(g1, f1.grad.numpy(), rtol=1e-12, atol=1e-12)
    assert np.allclose(g2, f2.grad.numpy(), rtol=1e-12, atol=1e-12)
    assert gc.shape == c.shape and not gc.any()


class _OracleSampler(torch.autograd.Function):
    """the reference's CorrSampler with the fp64 oracle as its two kernels"""

    @staticmethod
    def forward(ctx, volume, coords, r):
        ctx.save_for_backward(coords)
        ctx.r, ctx.shape = r, tuple(volume.shape)
        return _lookup_t(volume.detach(), coords, r)

    @staticmethod
    def backward(ctx, grad):
        coords, = ctx.saved_tensors
        return torch.from_numpy(ograd.corr_index_backward(ctx.shape, coords.numpy(), grad.numpy(), ctx.r)), None, None


def test_corrblock_gradient_dense_route_equals_on_the_fly_route(monkeypatch):
    """fp64: the reference's route (corr_index_backward on every level, then the gradients of avg_pool2d and of the
    all-pairs matmul) equals the route CorrBlock takes (altcorr_backward of (f1/4, pool^l(f2/4), coords/2^l), chained
    through the pooling by torch) — the derivation in nerf_slam_b200/corr.py::_CorrBlockLookup"""
    from nerf_slam_b200 import corr as pcorr
    rng = np.random.default_rng(31)
    E, C, H, W, r = 2, 8, 12, 18, 3                 # odd pooled sizes: 12x18 -> 6x9 -> 3x4 -> 1x2
    f1n, f2n = rng.normal(0, 1, (E, C, H, W)), rng.normal(0, 1, (E, C, H, W))
    yy, xx = np.meshgrid(np.arange(H), np.arange(W), indexing="ij")
    coords = (np.stack([xx, yy], 0)[None] + rng.uniform(-6, 6, (E, 2, H, W))).astype(np.float32)
    coords[0, :, 0, 0] = [1e6, 3.5]
    w = torch.from_numpy(rng.normal(0, 1, (E, 4 * 49, H, W)))
    c = torch.from_numpy(coords)

    # dense route: the reference's CorrBlock in fp64
    f1, f2 = torch.from_numpy(f1n).requires_grad_(), torch.from_numpy(f2n).requires_grad_()
    corr = torch.matmul((f1.reshape(E, C, H * W) / 4.0).transpose(1, 2), f2.reshape(E, C, H * W) / 4.0)
    corr = corr.reshape(E * H * W, 1, H, W)
    outs = []
    for l in range(4):
        outs.append(_OracleSampler.apply(corr.view(E, H, W, *corr.shape[2:]), c / 2 ** l, r).reshape(E, -1, H, W))
        if l < 3:
            corr = F.avg_pool2d(corr, 2, stride=2)
    (torch.cat(outs, 1) * w).sum().backward()
    dense1, dense2 = f1.grad.numpy(), f2.grad.numpy()

    # on-the-fly route: CorrBlock's autograd function with the fp64 oracle as altcorr_backward
    monkeypatch.setattr(pcorr.db, "corr_lookup_pyramid", lambda pyr, cc, rr: torch.zeros(E, 4 * 49, H, W, dtype=torch.float64))
    monkeypatch.setattr(pcorr.db, "altcorr_backward", lambda a, b, cc, g, rr: [
        torch.from_numpy(x) for x in ograd.altcorr_backward(a.detach().numpy(), b.detach().numpy(), cc.numpy(), g.numpy(), rr)])
    f1, f2 = torch.from_numpy(f1n).requires_grad_(), torch.from_numpy(f2n).requires_grad_()
    blk = pcorr.CorrBlock.__new__(pcorr.CorrBlock)
    blk.num_levels, blk.radius, blk.fmaps, blk.corr_pyramid = 4, r, (f1, f2), None
    a, b = (f / 4.0 for f in (f1, f2))            # _features() without its fp32 cast
    f2s = [b.permute(0, 2, 3, 1).contiguous()]
    for _ in range(3):
        b = F.avg_pool2d(b, 2, stride=2)
        f2s.append(b.permute(0, 2, 3, 1).contiguous())
    out = pcorr._CorrBlockLookup.apply(c, None, r, a.permute(0, 2, 3, 1).contiguous(), *f2s)
    (out * w).sum().backward()
    for got, ref in ((f1.grad.numpy(), dense1), (f2.grad.numpy(), dense2)):
        assert np.abs(got - ref).max() <= 1e-12 * np.abs(ref).max()


def _patch_oracle(monkeypatch, pcorr):
    T = torch.from_numpy

    def build(f_nhwc, ii, jj):
        f = f_nhwc.float().numpy().transpose(0, 3, 1, 2)
        return [T(p) for p in ocorr.corr_volume_pyramid(f[ii.numpy()], f[jj.numpy()])]
    monkeypatch.setattr(pcorr.db, "corr_volume_build", build)
    monkeypatch.setattr(pcorr.db, "corr_lookup_pyramid",
                        lambda pyr, c, r: T(ocorr.corr_lookup_pyramid([p.numpy() for p in pyr], c.numpy(), r)))
    monkeypatch.setattr(pcorr.db, "altcorr_forward", lambda f1, f2, c, r: (
        T(ocorr.altcorr_forward(f1.detach().numpy(), f2.detach().numpy(), c.numpy(), r)),))
    monkeypatch.setattr(pcorr.db, "altcorr_backward", lambda f1, f2, c, g, r: [
        T(x) for x in ograd.altcorr_backward(f1.detach().numpy(), f2.detach().numpy(), c.numpy(), g.numpy(), r)])


def test_golden_gradients_reproduced_by_the_oracle_backed_classes(monkeypatch):
    from nerf_slam_b200 import corr as pcorr
    _patch_oracle(monkeypatch, pcorr)
    g = np.load(os.path.join(G, "ref_corr_grad.npz"))
    fm = g["fmaps"].astype(np.float32)
    coords, w = torch.from_numpy(g["coords"]), torch.from_numpy(g["weights"].astype(np.float32))
    ii, jj = g["ii"], g["jj"]

    f = torch.from_numpy(fm).requires_grad_()
    out = pcorr.CorrBlock(f[:, ii], f[:, jj])(coords)
    assert out.dtype == torch.float16 and tuple(out.shape) == tuple(w.shape)
    (out.float() * w).sum().backward()
    ref = g["grad_corrblock"]
    assert np.abs(f.grad.numpy() - ref).max() <= 1e-4 * np.abs(ref).max()

    f = torch.from_numpy(fm).requires_grad_()
    out = pcorr.AltCorrBlock(f)(coords, torch.from_numpy(ii), torch.from_numpy(jj))
    (out * w).sum().backward()
    ref = g["grad_altcorrblock"]
    assert np.abs(f.grad.numpy() - ref).max() <= 1e-4 * np.abs(ref).max()


def test_corrblock_keeps_feature_maps_only_when_it_can_be_differentiated(monkeypatch):
    from nerf_slam_b200 import corr as pcorr
    _patch_oracle(monkeypatch, pcorr)
    f = torch.from_numpy(np.random.default_rng(3).normal(0, 1, (1, 2, 128, 16, 16)).astype(np.float32))
    assert pcorr.CorrBlock(f, f).fmaps is None                          # no input requires grad
    fg = f.clone().requires_grad_()
    with torch.no_grad():
        assert pcorr.CorrBlock(fg, fg).fmaps is None                    # built under no_grad
    blk = pcorr.CorrBlock(fg, f)
    assert blk.fmaps is not None and blk.fmaps[0].shape == (2, 128, 16, 16)
    other = pcorr.CorrBlock(fg[:, :1], f[:, :1])
    blk.cat(other)
    assert blk.fmaps[0].shape[0] == 3 and blk.corr_pyramid[0].shape[0] == 3
    blk[torch.tensor([True, False, True])]
    assert blk.fmaps[1].shape[0] == 2 and blk.corr_pyramid[3].shape[0] == 2
    blk.cat(pcorr.CorrBlock(f[:, :1], f[:, :1]))                        # a block without feature maps
    assert blk.fmaps is None and blk.corr_pyramid[0].shape[0] == 3
