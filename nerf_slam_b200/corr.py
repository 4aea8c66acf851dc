"""Correlation operators with the reference's class surface (networks/modules/corr.py):

  CorrBlock(fmap1, fmap2, num_levels=4, radius=3)  .__call__(coords) .cat(other) .__getitem__(mask)
  AltCorrBlock(fmaps, num_levels=4, radius=3)      .__call__(coords, ii, jj)

backed by the sm_90a kernels (wgmma volume build with fused pyramid, fused 4-level lookup,
on-the-fly alt-corr).  `CorrPool` is the arena the front-end uses instead of `CorrBlock.cat`:
pre-allocated pyramid slots, so adding/removing edges never re-copies volumes
(the reference's `torch.cat` re-copies the whole pool on every add, corr.py:52-55).
"""
import numpy as np
import torch
import torch.nn.functional as F

from . import _lib
from . import droid_backends as db


def coords_grid(ht, wd, device):
    """pixel coordinates [ht,wd,2] (x, y) fp32: the identity flow (networks/geom/projective_ops.py:14-19)"""
    y, x = torch.meshgrid(torch.arange(ht, device=device).float(), torch.arange(wd, device=device).float(), indexing="ij")
    return torch.stack([x, y], dim=-1)


def to_nhwc_half(fmap):
    """[..., C, H, W] -> [..., H, W, C] contiguous fp16"""
    return fmap.half().movedim(-3, -1).contiguous()


class _CorrBlockLookup(torch.autograd.Function):
    """CorrBlock's 4-level lookup with a gradient w.r.t. the feature maps, without a gradient volume.
    Level l of the volume is f1^T pool^l(f2) / 16 (average pooling over the target pixels is linear), so the lookup
    at coords / 2^l is the on-the-fly correlation of (f1/4, pool^l(f2/4), coords/2^l) and its gradient is
    altcorr_backward of those; torch chains it through the pooling and the /4.
    forward(coords [E,2,H,W], pyramid, radius, f1 [E,H,W,C], f2_0 .. f2_{L-1} [E,H>>l,W>>l,C]) -> [E,L*(2r+1)^2,H,W]
    with the values of the stored fp16 volume; no gradient for coords (the reference's CorrSampler returns None)."""

    @staticmethod
    def forward(ctx, coords, pyramid, radius, f1, *f2s):
        ctx.radius = radius
        ctx.save_for_backward(coords, f1, *f2s)
        return db.corr_lookup_pyramid(pyramid, coords, radius)

    @staticmethod
    def backward(ctx, grad):
        coords, f1, *f2s = ctx.saved_tensors
        E, _, H, W = coords.shape
        rd2 = (2 * ctx.radius + 1) ** 2
        grad = grad.to(f1.dtype)
        c = coords.permute(0, 2, 3, 1).reshape(E, 1, H, W, 2)
        g1, g2s = None, []
        for l, f2 in enumerate(f2s):
            gl = grad[:, l * rd2:(l + 1) * rd2].reshape(E, 1, rd2, H, W).contiguous()
            d1, d2, _ = db.altcorr_backward(f1, f2, (c / 2 ** l).contiguous(), gl, ctx.radius)
            g1 = d1 if g1 is None else g1 + d1
            g2s.append(d2)
        return (None, None, None, g1, *g2s)


class CorrBlock:
    """reference-compatible: fmap1/fmap2 [batch, num, C, ht, wd] (channels-first, as stored by the
    reference front-end).  The volume is built by the tensor-core kernel from channels-last copies.
    Differentiable w.r.t. fmap1 and fmap2 when built with grad enabled and a feature map that requires it: the block
    then also keeps the two feature maps and the lookup's gradient is computed by the on-the-fly route
    (_CorrBlockLookup).  Otherwise it keeps only the volume pyramid.  The pyramid tensors themselves carry no gradient."""

    def __init__(self, fmap1, fmap2, num_levels=4, radius=3):
        assert num_levels == 4
        self.num_levels, self.radius = num_levels, radius
        b, n, c, h, w = fmap1.shape
        E = b * n
        f = torch.cat([to_nhwc_half(fmap1.detach().reshape(E, c, h, w)),
                       to_nhwc_half(fmap2.detach().reshape(E, c, h, w))], 0)
        ii = torch.arange(E, dtype=torch.int32, device=f.device)
        self.corr_pyramid = db.corr_volume_build(f, ii, ii + E)
        self.fmaps = None
        if torch.is_grad_enabled() and (fmap1.requires_grad or fmap2.requires_grad):
            self.fmaps = (fmap1.reshape(E, c, h, w), fmap2.reshape(E, c, h, w))

    def _features(self):
        """(f1/4 channels-last, [pool^l(f2/4) channels-last for each level]) in fp32, with autograd history"""
        f1, f2 = (f.float() / 4.0 for f in self.fmaps)
        f2s = [f2.permute(0, 2, 3, 1).contiguous()]
        for _ in range(1, self.num_levels):
            f2 = F.avg_pool2d(f2, 2, stride=2)
            f2s.append(f2.permute(0, 2, 3, 1).contiguous())
        return f1.permute(0, 2, 3, 1).contiguous(), f2s

    def __call__(self, coords):
        batch, num, ht, wd, _ = coords.shape
        c = coords.permute(0, 1, 4, 2, 3).contiguous().view(batch * num, 2, ht, wd).float()
        if self.fmaps is not None and torch.is_grad_enabled():
            f1, f2s = self._features()
            out = _CorrBlockLookup.apply(c.detach(), self.corr_pyramid, self.radius, f1, *f2s)
        else:
            out = db.corr_lookup_pyramid(self.corr_pyramid, c, self.radius)
        return out.view(batch, num, -1, ht, wd)

    def cat(self, other):
        for i in range(self.num_levels):
            self.corr_pyramid[i] = torch.cat([self.corr_pyramid[i], other.corr_pyramid[i]], 0)
        if self.fmaps is not None and other.fmaps is not None:
            self.fmaps = tuple(torch.cat([a, o], 0) for a, o in zip(self.fmaps, other.fmaps))
        else:
            self.fmaps = None   # one side has no feature maps: the concatenated block has no gradient
        return self

    def __getitem__(self, index):
        for i in range(self.num_levels):
            self.corr_pyramid[i] = self.corr_pyramid[i][index]
        if self.fmaps is not None:
            self.fmaps = tuple(f[index] for f in self.fmaps)
        return self

    @staticmethod
    def corr(fmap1, fmap2):
        """level-0 volume only, reference layout [batch, num, ht, wd, ht, wd]"""
        blk = CorrBlock(fmap1, fmap2)
        b, n, _, h, w = fmap1.shape
        return blk.corr_pyramid[0].view(b, n, h, w, h, w)


class CorrPool:
    """Slot arena of correlation pyramids for the active edges of the factor graph."""

    def __init__(self, capacity, ht, wd, device, radius=3):
        self.capacity, self.ht, self.wd, self.radius = capacity, ht, wd, radius
        self.levels = [torch.empty(capacity, ht, wd, ht >> l, wd >> l, dtype=torch.float16, device=device)
                       for l in range(4)]
        self.free = list(range(capacity - 1, -1, -1))
        self.device = device

    def alloc(self, n):
        if n > len(self.free):
            raise RuntimeError(f"correlation pool exhausted ({self.capacity} slots)")
        return [self.free.pop() for _ in range(n)]

    def release(self, slots):
        self.free.extend(int(s) for s in slots)

    def build(self, fmaps_nhwc, fi, fj, slots):
        """fmaps_nhwc [NF,ht,wd,C] fp16; fi/fj flat frame indices (host lists) -> volumes into `slots`"""
        n = len(slots)
        if n == 0:
            return
        dev = self.device
        ii = _lib.h2d(np.asarray(fi, np.int32), dev)
        jj = _lib.h2d(np.asarray(fj, np.int32), dev)
        NF, H, W, C = fmaps_nhwc.shape
        if C == 128 and H % 2 == 0 and W in (64, 80):
            # one launch for all new edges, each into the slot it was given
            sl = _lib.h2d(np.asarray(slots, np.int32), dev)
            _lib.check(_lib.load().nslam_corr_volume_build_slots(
                _lib.ptr(fmaps_nhwc), NF, H, W, C, _lib.ptr(ii), _lib.ptr(jj), _lib.ptr(sl), n, self.capacity,
                *[_lib.ptr(lv) for lv in self.levels], _lib.stream_ptr()), "corr_volume_build_slots")
            return
        s = sorted(slots)
        contiguous = s == list(range(s[0], s[0] + n)) and list(slots) == s
        if contiguous:
            outs = [lv[s[0]:s[0] + n] for lv in self.levels]
            db.corr_volume_build_into(fmaps_nhwc, ii, jj, outs)
        else:
            for k, sl in enumerate(slots):
                outs = [lv[sl:sl + 1] for lv in self.levels]
                db.corr_volume_build_into(fmaps_nhwc, ii[k:k + 1], jj[k:k + 1], outs)

    def lookup(self, slots_dev, coords, nhwc=False, out=None):
        """slots_dev int32 [E] device.
        nhwc=False: coords [E,2,ht,wd] -> [E,196,ht,wd] fp16 (reference layout)
        nhwc=True : coords [E,ht,wd,2] (what reproject returns) -> [E,ht,wd,CORR_PAD] fp16, zero-padded
                    channels-last operand of the tensor-core update operator"""
        if nhwc:
            from .conv import CORR_PAD
            return db.corr_lookup_pyramid(self.levels, coords.contiguous(), self.radius, slots=slots_dev,
                                          nhwc_stride=CORR_PAD, coords_nhwc=True, out=out)
        return db.corr_lookup_pyramid(self.levels, coords, self.radius, slots=slots_dev)


class _AltCorrLayer(torch.autograd.Function):
    """the reference's CorrLayer (networks/modules/corr.py:75-89): altcorr_forward, with altcorr_backward as gradient
    (fmap1, fmap2, and an all-zero coordinate gradient, as the reference returns)"""

    @staticmethod
    def forward(ctx, fmap1, fmap2, coords, radius):
        ctx.radius = radius
        ctx.save_for_backward(fmap1, fmap2, coords)
        corr, = db.altcorr_forward(fmap1, fmap2, coords, radius)
        return corr

    @staticmethod
    def backward(ctx, grad):
        fmap1, fmap2, coords = ctx.saved_tensors
        g1, g2, gc = db.altcorr_backward(fmap1, fmap2, coords, grad.contiguous(), ctx.radius)
        return g1, g2, gc, None


class AltCorrBlock:
    """reference-compatible on-the-fly correlation (networks/modules/corr.py:92-140).  Differentiable w.r.t. the
    feature maps when called with grad enabled; the pyramid is built with torch ops, so gradients reach `fmaps`."""

    def __init__(self, fmaps, num_levels=4, radius=3):
        self.num_levels, self.radius = num_levels, radius
        B, N, C, H, W = fmaps.shape
        f = fmaps.view(B * N, C, H, W) / 4.0
        self.pyramid = []
        for i in range(num_levels):
            self.pyramid.append(f.permute(0, 2, 3, 1).contiguous().view(B, N, H // 2 ** i, W // 2 ** i, C))
            f = F.avg_pool2d(f, 2, stride=2)

    def corr_fn(self, coords, ii, jj):
        B, N, H, W, S, _ = coords.shape
        coords = coords.permute(0, 1, 4, 2, 3, 5)
        outs = []
        for i in range(self.num_levels):
            f1 = self.pyramid[0][:, ii]
            f2 = self.pyramid[i][:, jj]
            c = (coords / 2 ** i).reshape(B * N, S, H, W, 2).contiguous()
            f1 = f1.reshape((B * N,) + f1.shape[2:]).float().contiguous()
            f2 = f2.reshape((B * N,) + f2.shape[2:]).float().contiguous()
            if torch.is_grad_enabled() and (f1.requires_grad or f2.requires_grad or c.requires_grad):
                corr = _AltCorrLayer.apply(f1, f2, c, self.radius)
            else:
                corr, = db.altcorr_forward(f1, f2, c, self.radius)
            outs.append(corr.view(B, N, S, -1, H, W).permute(0, 1, 3, 4, 5, 2))
        return torch.cat(outs, dim=2)

    def __call__(self, coords, ii, jj):
        squeeze = False
        if coords.dim() == 5:
            coords = coords.unsqueeze(-2)
            squeeze = True
        corr = self.corr_fn(coords, ii, jj)
        if squeeze:
            corr = corr.squeeze(-1)
        return corr.contiguous()
