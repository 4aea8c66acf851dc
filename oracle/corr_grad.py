"""ORACLE (test infrastructure only — never imported by the product path).

CPU restatements of the two backward operators of the reference's correlation layers, next to the forwards in
oracle/corr.py:
  corr_index_backward_kernel   src/correlation_kernels.cu:73-124 (host :157-185)
  altcorr_backward_kernel      src/altcorr_kernel.cu:152-286 (host :321-356)
Pinned against the reference's compiled kernels on the GPU (oracle/build_ref_corr_grad.py, tests/test_gpu_corr_grad.py)
and against torch fp64 autograd of the forwards (tests/test_cpu_corr_grad.py).
"""
import numpy as np
import scipy.sparse as sp

from .corr import F16, F32, _mac_half

F64 = np.float64


def _fma_f32(acc, s, w):
    # the reference's fp32 build contracts `g += cg * w` into one fused multiply-add: s*w is exact in fp64, so the
    # fused result is the fp64 sum rounded to fp32 (a double rounding, which differs from a single one only when the
    # fp64 sum lands exactly on an fp32 tie: about 2^-29 per operation)
    return (acc.astype(F64) + s.astype(F64) * w.astype(F64)).astype(F32)


def _mac_f64(acc, s, w):
    return acc + s * w


def corr_index_backward(volume_shape, coords, corr_grad, r):
    """volume_shape (n,h1,w1,h2,w2), coords [n,2,h1,w1], corr_grad [n,2r+1,2r+1,h1,w1] (fp16, fp32 or fp64)
    -> volume_grad [n,h1,w1,h2,w2] in corr_grad's dtype.
    Tap (i, j) sits at x1 = floor(x0) - r + i, y1 = floor(y0) - r + j; inside the map it receives
      g = 0 (+) cg[i-1][j-1]*w11 (+) cg[i-1][j]*w10 (+) cg[i][j-1]*w01 (+) cg[i][j]*w00     (terms with an index
    outside [0, 2r] skipped), stored as 0 + g.  fp16 rounds after every operation (c10::Half), fp32 fuses each
    multiply-add (see _fma_f32), fp64 is plain fp64 arithmetic with fp64 weights."""
    n, h1, w1, h2, w2 = volume_shape
    dt = corr_grad.dtype.type
    mac = {F16: _mac_half, F32: _fma_f32, F64: _mac_f64}[dt]
    cdt = F64 if dt == F64 else F32
    x0 = coords[:, 0].astype(cdt)
    y0 = coords[:, 1].astype(cdt)
    fx, fy = np.floor(x0), np.floor(y0)
    dx, dy = x0 - fx, y0 - fy
    one = cdt(1.0)
    w11 = (dx * dy).astype(dt)
    w10 = (dx * (one - dy)).astype(dt)
    w01 = ((one - dx) * dy).astype(dt)
    w00 = ((one - dx) * (one - dy)).astype(dt)
    rd = 2 * r + 1
    xb = fx.astype(np.int64) - r
    yb = fy.astype(np.int64) - r
    out = np.zeros(volume_shape, dtype=dt)
    nn, yy, xx = np.meshgrid(np.arange(n), np.arange(h1), np.arange(w1), indexing="ij")
    for i in range(rd + 1):
        for j in range(rd + 1):
            g = np.zeros((n, h1, w1), dtype=dt)
            if i > 0 and j > 0:
                g = mac(g, corr_grad[:, i - 1, j - 1], w11)
            if i > 0 and j < rd:
                g = mac(g, corr_grad[:, i - 1, j], w10)
            if i < rd and j > 0:
                g = mac(g, corr_grad[:, i, j - 1], w01)
            if i < rd and j < rd:
                g = mac(g, corr_grad[:, i, j], w00)
            g = (dt(0) + g).astype(dt)
            x1, y1 = xb + i, yb + j
            ok = (x1 >= 0) & (x1 < w2) & (y1 >= 0) & (y1 < h2)
            out[nn[ok], yy[ok], xx[ok], y1[ok], x1[ok]] = g[ok]
    return out


def altcorr_tap_matrix(coords, corr_grad, r, H2, W2, dtype=F64):
    """The linear map of altcorr: corr = taps of M, with M [B*H2*W2, B*H1*W1] (sparse) holding, for target q and
    source p, the sum over coordinate sets n and taps (iy, ix) landing on q of the weight
      g = cg[(iy-1)+rd(ix-1)]*dy*dx + cg[(iy-1)+rd*ix]*dy*(1-dx) + cg[iy+rd(ix-1)]*(1-dy)*dx + cg[iy+rd*ix]*(1-dy)*(1-dx)
    (src/altcorr_kernel.cu:237-252; channel = iy + (2r+1)*ix).  Taps outside fmap2 are dropped.
    fmap1_grad = M^T fmap2, fmap2_grad = M fmap1."""
    B, N, H1, W1, _ = coords.shape
    rd = 2 * r + 1
    hw = H1 * W1
    cg = corr_grad.astype(dtype)
    bsrc = np.broadcast_to(np.arange(B)[:, None, None] * hw + np.arange(hw).reshape(1, H1, W1), (B, H1, W1))
    rows, cols, vals = [], [], []
    for n in range(N):
        x0 = coords[:, n, :, :, 0].astype(dtype)
        y0 = coords[:, n, :, :, 1].astype(dtype)
        fx, fy = np.floor(x0), np.floor(y0)
        dx, dy = x0 - fx, y0 - fy
        xb, yb = fx.astype(np.int64) - r, fy.astype(np.int64) - r
        for iy in range(rd + 1):
            for ix in range(rd + 1):
                g = np.zeros((B, H1, W1), dtype=dtype)
                if iy > 0 and ix > 0:
                    g = g + cg[:, n, (iy - 1) + rd * (ix - 1)] * dy * dx
                if iy > 0 and ix < rd:
                    g = g + cg[:, n, (iy - 1) + rd * ix] * dy * (1 - dx)
                if iy < rd and ix > 0:
                    g = g + cg[:, n, iy + rd * (ix - 1)] * (1 - dy) * dx
                if iy < rd and ix < rd:
                    g = g + cg[:, n, iy + rd * ix] * (1 - dy) * (1 - dx)
                h2, w2 = yb + iy, xb + ix
                ok = (h2 >= 0) & (h2 < H2) & (w2 >= 0) & (w2 < W2)
                bq = np.arange(B)[:, None, None] * (H2 * W2) + h2 * W2 + w2
                rows.append(bq[ok]); cols.append(bsrc[ok]); vals.append(g[ok])
    rows, cols, vals = (np.concatenate(a) for a in (rows, cols, vals))
    return sp.coo_matrix((vals, (rows, cols)), shape=(B * H2 * W2, B * hw)).tocsr()


def altcorr_backward(fmap1, fmap2, coords, corr_grad, r):
    """fmap1 [B,H1,W1,C], fmap2 [B,H2,W2,C], coords [B,N,H1,W1,2], corr_grad [B,N,(2r+1)^2,H1,W1]
    -> (fmap1_grad, fmap2_grad, coords_grad), computed in fmap1's dtype (fp32 or fp64).
    coords_grad is zeros, as the reference returns it (its kernel never writes it)."""
    B, H1, W1, C = fmap1.shape
    _, H2, W2, _ = fmap2.shape
    dt = fmap1.dtype.type
    M = altcorr_tap_matrix(coords, corr_grad, r, H2, W2, dtype=dt)
    g1 = (M.T @ fmap2.reshape(-1, C).astype(dt)).reshape(B, H1, W1, C).astype(dt)
    g2 = (M @ fmap1.reshape(-1, C).astype(dt)).reshape(B, H2, W2, C).astype(dt)
    return g1, g2, np.zeros(coords.shape, dtype=dt)
