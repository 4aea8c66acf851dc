"""ORACLE (test infrastructure only — never imported by the product path).

CPU restatements of the correlation operators of the reference:
  A2  CorrBlock.__init__ / CorrBlock.corr         networks/modules/corr.py:23-38,63-72
  A3  corr_index_forward_kernel                    src/correlation_kernels.cu:19-70
  A4  altcorr_forward_kernel + AltCorrBlock        src/altcorr_kernel.cu:27-149, networks/modules/corr.py:92-126
Pinned by tests/golden/ (reference python modules imported on CPU, reference CUDA kernels run on
the GPU from oracle/_ref) — see tests/golden/README.md.
"""
import numpy as np

F16, F32 = np.float16, np.float32


def corr_volume_pyramid(fmap1, fmap2, num_levels=4):
    """fmap1, fmap2: [E, C, H, W] float16  ->  list of [E, H, W, H>>l, W>>l] float16.
    (f1/4)^T (f2/4) with fp32 accumulation rounded to fp16 (what the autocast HGEMM produces),
    then avg_pool2d(2,2) per level from the previous fp16 level (fp32 sum, fp16 round)."""
    E, C, H, W = fmap1.shape
    a = (fmap1.reshape(E, C, H * W) / F16(4.0)).astype(F32)
    b = (fmap2.reshape(E, C, H * W) / F16(4.0)).astype(F32)
    corr = np.einsum("ecm,ecn->emn", a, b, optimize=True).astype(F16)
    pyr = []
    cur = corr.reshape(E * H * W, H, W)
    for l in range(num_levels):
        pyr.append(cur.reshape(E, H, W, cur.shape[1], cur.shape[2]))
        h2, w2 = cur.shape[1] // 2, cur.shape[2] // 2
        c = cur[:, :2 * h2, :2 * w2].astype(F32)
        s = ((c[:, 0::2, 0::2] + c[:, 0::2, 1::2]) + c[:, 1::2, 0::2]) + c[:, 1::2, 1::2]
        cur = (s * F32(0.25)).astype(F16)
    return pyr


def _mac_half(acc, s, w):
    prod = (s.astype(F32) * w.astype(F32)).astype(F16)
    return (acc.astype(F32) + prod.astype(F32)).astype(F16)


def _mac_float(acc, s, w):
    return (acc + (s * w).astype(F32)).astype(F32)


def corr_index_forward(volume, coords, r):
    """volume [n,h1,w1,h2,w2] (fp16/fp32), coords [n,2,h1,w1] fp32 -> [n,2r+1,2r+1,h1,w1].
    Tap order and per-operator rounding of src/correlation_kernels.cu:46-68 (c10::Half arithmetic
    rounds after every multiply and add)."""
    n, h1, w1, h2, w2 = volume.shape
    half = volume.dtype == F16
    mac = _mac_half if half else _mac_float
    dt = F16 if half else F32
    x0 = coords[:, 0].astype(F32)
    y0 = coords[:, 1].astype(F32)
    fx, fy = np.floor(x0), np.floor(y0)
    dx, dy = (x0 - fx).astype(F32), (y0 - fy).astype(F32)
    rd = 2 * r + 1
    xb = fx.astype(np.int64) - r
    yb = fy.astype(np.int64) - r
    taps = np.zeros((rd + 1, rd + 1, n, h1, w1), dtype=dt)
    nn, yy, xx = np.meshgrid(np.arange(n), np.arange(h1), np.arange(w1), indexing="ij")
    for i in range(rd + 1):
        for j in range(rd + 1):
            x1, y1 = xb + i, yb + j
            ok = (x1 >= 0) & (x1 < w2) & (y1 >= 0) & (y1 < h2)
            v = volume[nn, yy, xx, np.clip(y1, 0, h2 - 1), np.clip(x1, 0, w2 - 1)]
            taps[i, j] = np.where(ok, v, dt(0))
    one = F32(1.0)
    w11 = (dx * dy).astype(dt)
    w10 = (dx * (one - dy)).astype(dt)
    w01 = ((one - dx) * dy).astype(dt)
    w00 = ((one - dx) * (one - dy)).astype(dt)
    out = np.zeros((n, rd, rd, h1, w1), dtype=dt)
    for i in range(rd):
        for j in range(rd):
            acc = np.zeros((n, h1, w1), dtype=dt)
            acc = mac(acc, taps[i, j], w00)
            acc = mac(acc, taps[i, j + 1], w01)
            acc = mac(acc, taps[i + 1, j], w10)
            acc = mac(acc, taps[i + 1, j + 1], w11)
            out[:, i, j] = acc
    return out


def corr_lookup_pyramid(pyramid, coords, r):
    """CorrBlock.__call__ (networks/modules/corr.py:40-50): level l sampled at coords/2^l,
    concatenated along channels -> [n, L*(2r+1)^2, h1, w1]"""
    outs = []
    for l, vol in enumerate(pyramid):
        o = corr_index_forward(vol, (coords / F32(2 ** l)).astype(F32), r)
        outs.append(o.reshape(o.shape[0], -1, o.shape[3], o.shape[4]))
    return np.concatenate(outs, axis=1)


def altcorr_forward(fmap1, fmap2, coords, r):
    """fmap1 [B,H1,W1,C], fmap2 [B,H2,W2,C], coords [B,N,H1,W1,2] -> [B,N,(2r+1)^2,H1,W1] (fp32 math).
    channel = iy + (2r+1)*ix (src/altcorr_kernel.cu:102-105)."""
    B, H1, W1, C = fmap1.shape
    _, H2, W2, _ = fmap2.shape
    N = coords.shape[1]
    rd = 2 * r + 1
    f1 = fmap1.astype(F32)
    f2 = fmap2.astype(F32)
    out = np.zeros((B, N, rd * rd, H1, W1), dtype=F32)
    bb = np.arange(B)[:, None, None]
    for n in range(N):
        x0 = coords[:, n, :, :, 0].astype(F32)
        y0 = coords[:, n, :, :, 1].astype(F32)
        fx, fy = np.floor(x0), np.floor(y0)
        dx, dy = x0 - fx, y0 - fy
        xb, yb = fx.astype(np.int64) - r, fy.astype(np.int64) - r
        dots = np.zeros((rd + 1, rd + 1, B, H1, W1), dtype=F32)  # [iy, ix]
        for iy in range(rd + 1):
            for ix in range(rd + 1):
                h2, w2 = yb + iy, xb + ix
                ok = (h2 >= 0) & (h2 < H2) & (w2 >= 0) & (w2 < W2)
                g = f2[bb, np.clip(h2, 0, H2 - 1), np.clip(w2, 0, W2 - 1)]
                dots[iy, ix] = np.where(ok, (f1 * g).sum(-1), 0.0)
        for ox in range(rd):
            for oy in range(rd):
                out[:, n, oy + rd * ox] = (dots[oy, ox] * (1 - dy) * (1 - dx) + dots[oy, ox + 1] * (1 - dy) * dx +
                                           dots[oy + 1, ox] * dy * (1 - dx) + dots[oy + 1, ox + 1] * dy * dx)
    return out.astype(fmap1.dtype)


def alt_pyramid(fmaps, num_levels=4):
    """AltCorrBlock.__init__ (networks/modules/corr.py:92-105): fmaps [N,C,H,W] (any float) ->
    list of channels-last levels [N, H>>l, W>>l, C] of fmaps/4 pooled with avg_pool2d(2,2)."""
    cur = (fmaps / fmaps.dtype.type(4.0))
    pyr = []
    for l in range(num_levels):
        pyr.append(np.ascontiguousarray(cur.transpose(0, 2, 3, 1)))
        h2, w2 = cur.shape[2] // 2, cur.shape[3] // 2
        c = cur[:, :, :2 * h2, :2 * w2].astype(F32)
        s = ((c[:, :, 0::2, 0::2] + c[:, :, 0::2, 1::2]) + c[:, :, 1::2, 0::2]) + c[:, :, 1::2, 1::2]
        cur = (s * F32(0.25)).astype(fmaps.dtype)
    return pyr
