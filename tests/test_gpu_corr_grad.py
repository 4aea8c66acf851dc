"""GPU checks of the correlation backward operators (csrc/corr_backward.cu) and of the gradients of CorrBlock /
AltCorrBlock: against the reference's own backward kernels (oracle/build_ref_corr_grad.py, skipped when not built),
the CPU oracle (oracle/corr_grad.py), the golden of the reference's composition (tests/golden/ref_corr_grad.npz) and
each other."""
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import build_ref_corr_grad
from oracle import corr_grad as ograd

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
G = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


@pytest.fixture(scope="module")
def db():
    from nerf_slam_b200 import droid_backends
    return droid_backends


@pytest.fixture(scope="module")
def refgrad():
    m = build_ref_corr_grad.load()
    if m is None:
        pytest.skip("oracle/_ref/nslam_ref_corr_grad.so not built")
    return m


def _grid_coords(g, n, h1, w1, scale, jitter):
    """[n,2,h1,w1]: the pixel grid / scale plus uniform jitter, with a few coordinates far outside the map"""
    yy, xx = torch.meshgrid(torch.arange(h1), torch.arange(w1), indexing="ij")
    c = torch.stack([xx, yy], 0)[None].float() / scale + (torch.rand(n, 2, h1, w1, generator=g) * 2 - 1) * jitter
    c[0, 0, 0, 0], c[0, 1, 0, 1], c[-1, 0, -1, -1], c[-1, 1, 1, 2] = 1e6, -1e6, -1e6, 1e6
    return c.contiguous()


def _bits(t):
    return t.view(torch.int16 if t.dtype == torch.float16 else torch.int32)


CASES = [  # (n, h1, w1, h2, w2, r): the four pyramid levels at 60x80, an odd size, r = 1
    (1, 60, 80, 60, 80, 3), (2, 60, 80, 30, 40, 3), (2, 60, 80, 15, 20, 3), (2, 60, 80, 7, 10, 3),
    (3, 13, 17, 11, 19, 3), (2, 13, 17, 9, 7, 1),
]


@pytest.mark.parametrize("dtype", [torch.float16, torch.float32])
@pytest.mark.parametrize("case", CASES)
def test_corr_index_backward_bit_exact(db, refgrad, dtype, case):
    n, h1, w1, h2, w2, r = case
    g = torch.Generator().manual_seed(1200 + 2 * CASES.index(case) + (dtype == torch.float16))
    rd = 2 * r + 1
    coords = _grid_coords(g, n, h1, w1, h1 / h2, r + 3)
    cg = torch.randn(n, rd, rd, h1, w1, generator=g).to(dtype)
    vol = torch.empty(n, h1, w1, h2, w2, dtype=dtype, device=DEV)
    got, = db.corr_index_backward(vol, coords.to(DEV), cg.to(DEV), r)
    assert got.shape == vol.shape and got.dtype == dtype
    ref, = refgrad.corr_index_backward(vol, coords.to(DEV), cg.to(DEV), r)
    assert torch.equal(_bits(got), _bits(ref))                                   # bit-exact, +0 vs -0 included
    ora = ograd.corr_index_backward(tuple(vol.shape), coords.numpy(), cg.numpy(), r)
    assert np.array_equal(_bits(got).cpu().numpy(), ora.view(np.int16 if dtype == torch.float16 else np.int32))
    again, = db.corr_index_backward(vol, coords.to(DEV), cg.to(DEV), r)
    assert torch.equal(_bits(got), _bits(again))


def _rel(a, b):
    b = np.asarray(b, np.float64)
    return np.abs(np.asarray(a, np.float64) - b).max() / max(np.abs(b).max(), 1e-30)


@pytest.mark.parametrize("N,H2,W2", [(1, 60, 80), (3, 60, 80), (3, 30, 40)])
def test_altcorr_backward_vs_reference_and_oracle(db, refgrad, N, H2, W2):
    """1e-5 of each tensor's max magnitude.  The reference kernel is run only on H1 % 4 == 0, W1 % 8 == 0 (it reads
    coords out of bounds otherwise) and it reads other lanes' shared-memory entries without a barrier, so where it
    disagrees with the fp64 oracle, the oracle decides and the reference comparison is reported instead of asserted."""
    g = torch.Generator().manual_seed(1300 + N + H2)
    B, H1, W1, C, r = 2, 60, 80, 128, 3
    f1 = torch.randn(B, H1, W1, C, generator=g) / 4
    f2 = torch.randn(B, H2, W2, C, generator=g) / 4
    c = torch.stack([_grid_coords(g, B, H1, W1, H1 / H2, 6) for _ in range(N)], 1).permute(0, 1, 3, 4, 2).contiguous()
    cg = torch.randn(B, N, 49, H1, W1, generator=g)
    args = [t.to(DEV) for t in (f1, f2, c, cg)]
    g1, g2, gc = db.altcorr_backward(*args, r)
    o1, o2, _ = ograd.altcorr_backward(f1.double().numpy(), f2.double().numpy(), c.numpy(), cg.double().numpy(), r)
    assert _rel(g1.cpu(), o1) <= 1e-5 and _rel(g2.cpu(), o2) <= 1e-5
    assert gc.shape == c.shape and not gc.any()
    a1, a2, _ = db.altcorr_backward(*args, r)
    assert torch.equal(_bits(g1), _bits(a1)) and torch.equal(_bits(g2), _bits(a2))   # same bytes on every run
    r1, r2, rc = refgrad.altcorr_backward(*args, r)
    assert not rc.any()
    ref_ok = _rel(r1.cpu(), o1) <= 1e-5 and _rel(r2.cpu(), o2) <= 1e-5
    if ref_ok:
        assert _rel(g1.cpu(), r1.cpu()) <= 2e-5 and _rel(g2.cpu(), r2.cpu()) <= 2e-5
    else:
        print(f"reference altcorr_backward off the fp64 oracle: {_rel(r1.cpu(), o1):.2e} / {_rel(r2.cpu(), o2):.2e}")


def test_altcorr_backward_rejects_non_fp32(db):
    t = lambda *s: torch.zeros(*s, dtype=torch.float16, device=DEV)
    with pytest.raises(RuntimeError):
        db.altcorr_backward(t(1, 4, 8, 8), t(1, 4, 8, 8), torch.zeros(1, 1, 4, 8, 2, device=DEV), t(1, 1, 49, 4, 8), 3)


class _OracleAlt(torch.autograd.Function):
    """fp64 CorrLayer with the oracle's altcorr_backward (forward values are not needed for the gradient)"""

    @staticmethod
    def forward(ctx, f1, f2, coords, r):
        ctx.save_for_backward(f1, f2, coords)
        ctx.r = r
        return f1.new_zeros(f1.shape[0], coords.shape[1], (2 * r + 1) ** 2, *f1.shape[1:3])

    @staticmethod
    def backward(ctx, grad):
        f1, f2, coords = ctx.saved_tensors
        g1, g2, _ = ograd.altcorr_backward(f1.numpy(), f2.numpy(), coords.numpy(), grad.numpy(), ctx.r)
        return torch.from_numpy(g1), torch.from_numpy(g2), None, None


def _oracle_grad(fm, ii, jj, coords, w):
    """fp64 gradient of sum(out * w) w.r.t. fmaps for the AltCorrBlock composition (the function both blocks compute)"""
    f = torch.from_numpy(fm.astype(np.float64)).requires_grad_()
    B, N, C, H, W = f.shape
    x = f.view(B * N, C, H, W) / 4.0
    pyr = []
    for l in range(4):
        pyr.append(x.permute(0, 2, 3, 1).reshape(B, N, *x.shape[2:], C))
        if l < 3:
            x = F.avg_pool2d(x, 2, stride=2)
    c = torch.from_numpy(coords)
    outs = []
    for l in range(4):
        f1 = pyr[0][:, ii].reshape(-1, H, W, C).contiguous()
        f2 = pyr[l][:, jj].reshape(-1, *pyr[l].shape[2:]).contiguous()
        outs.append(_OracleAlt.apply(f1, f2, (c / 2 ** l).reshape(-1, 1, H, W, 2).contiguous(), 3))
    out = torch.cat([o.view(B, len(ii), 49, H, W) for o in outs], 2)
    (out * torch.from_numpy(w).double()).sum().backward()
    return f.grad.numpy()


def test_block_gradients_vs_golden_oracle_and_each_other():
    from nerf_slam_b200 import corr as pcorr
    g = np.load(os.path.join(G, "ref_corr_grad.npz"))
    fm, w = g["fmaps"].astype(np.float32), g["weights"].astype(np.float32)
    ii, jj = g["ii"], g["jj"]
    coords, wd = torch.from_numpy(g["coords"]).to(DEV), torch.from_numpy(w).to(DEV)

    f = torch.from_numpy(fm).to(DEV).requires_grad_()
    out = pcorr.CorrBlock(f[:, ii], f[:, jj])(coords)
    (out.float() * wd).sum().backward()
    grad_vol = f.grad.cpu().numpy()

    f = torch.from_numpy(fm).to(DEV).requires_grad_()
    out = pcorr.AltCorrBlock(f)(coords, torch.from_numpy(ii).to(DEV), torch.from_numpy(jj).to(DEV))
    (out * wd).sum().backward()
    grad_alt = f.grad.cpu().numpy()

    ora = _oracle_grad(fm, ii, jj, g["coords"], w)
    for got, gold in ((grad_vol, g["grad_corrblock"]), (grad_alt, g["grad_altcorrblock"])):
        assert _rel(got, gold) <= 1e-4
        assert _rel(got, ora) <= 1e-4
    assert _rel(grad_vol, grad_alt) <= 1e-4


def test_corrblock_under_no_grad_is_unchanged():
    from nerf_slam_b200 import corr as pcorr
    g = torch.Generator().manual_seed(77)
    f1 = torch.randn(1, 3, 128, 30, 40, generator=g).to(DEV)
    f2 = torch.randn(1, 3, 128, 30, 40, generator=g).to(DEV)
    coords = torch.stack([_grid_coords(g, 3, 30, 40, 1, 5).permute(0, 2, 3, 1)], 0).to(DEV).contiguous()
    plain = pcorr.CorrBlock(f1, f2)
    ref = plain(coords)
    fg1, fg2 = f1.clone().requires_grad_(), f2.clone().requires_grad_()
    with torch.no_grad():
        blk = pcorr.CorrBlock(fg1, fg2)
        out = blk(coords)
    assert blk.fmaps is None and plain.fmaps is None
    assert torch.equal(out, ref) and not out.requires_grad
    # with grad the forward values still come from the same fp16 volume
    blk = pcorr.CorrBlock(fg1, fg2)
    out = blk(coords)
    assert out.requires_grad and torch.equal(out.detach(), ref)
