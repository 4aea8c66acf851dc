"""host-side logic that needs no GPU: weight packing for the tensor-core convolution, hash-grid level table,
pose conversion of the NeRF hand-off"""
import math

import numpy as np
import torch

from oracle import ngp as ongp
from oracle import se3 as ose3


def test_pack_weights_layout():
    """packed image = [tap][source][64-channel block] blocks of [N_pad][64] fp16, 16-byte chunk j of row n stored at
    chunk position j ^ (n & 7)  (the 128-byte swizzle the wgmma shared-memory descriptor expects)"""
    from nerf_slam_b200.conv import pack_weights
    g = torch.Generator().manual_seed(0)
    for (N, srcs, k, npad) in ((16, [128], 3, None), (128, [128, 128, 128, 64], 3, None), (32, [152], 1, None),
                               (4, [256], 3, 16), (64, [32], 1, None)):
        cin = sum(srcs)
        w = torch.randn(N, cin, k, k, generator=g)
        img = pack_weights(w, srcs, n_pad=npad).float()
        Np = npad or N
        nblk = k * k * sum((c + 63) // 64 for c in srcs)
        assert img.numel() == nblk * Np * 64
        img = img.view(nblk, Np, 8, 8)
        b = 0
        for ky in range(k):
            for kx in range(k):
                off = 0
                for C in srcs:
                    for cb in range((C + 63) // 64):
                        blk = torch.zeros(Np, 64)
                        cs, ce = cb * 64, min(C, cb * 64 + 64)
                        blk[:N, :ce - cs] = w[:, off + cs:off + ce, ky, kx].half().float()
                        for n in range(0, Np, max(1, Np // 7)):           # sample rows
                            for j in range(8):
                                assert torch.equal(img[b, n, j ^ (n & 7)], blk[n, 8 * j:8 * j + 8]), (N, b, n, j)
                        b += 1
                    off += C


def test_level_table_matches_oracle():
    from nerf_slam_b200 import pyngp
    for aabb in (1.0, 4.0, 16.0):
        rows, total = pyngp.level_table(aabb)
        lv, tot = ongp.level_params(aabb)
        assert total == tot and len(rows) == len(lv) == 16
        for (sc, res, n, off, dense), o in zip(rows, lv):
            assert (sc, res, n, off) == (o[0], o[1], o[2], o[3])
            assert bool(dense) == (res ** 3 <= n)


def test_pose_tq_to_c2w_is_inverse_of_cam_T_world():
    from nerf_slam_b200.nerf_fusion import _pose_tq_to_c2w
    rng = np.random.default_rng(3)
    q = rng.normal(size=(5, 4)); q /= np.linalg.norm(q, axis=1, keepdims=True)
    t = rng.normal(size=(5, 3))
    tq = np.concatenate([t, q], 1)
    c2w = _pose_tq_to_c2w(tq)
    for k in range(5):
        T = ose3.matrix(tq[k].astype(np.float64)) if hasattr(ose3, "matrix") else None
        if T is None:
            x, y, z, w = q[k]
            R = np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                          [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                          [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])
            T = np.eye(4); T[:3, :3] = R; T[:3, 3] = t[k]
        assert np.allclose(c2w[k] @ T, np.eye(4), atol=1e-9)


def test_halo_tile_schedule_reproduces_the_convolution():
    """index emulation of csrc/conv_igemm.cu (HALO path): per (channel block, dx) one column-shifted tile with a
    1-pixel vertical halo, the three taps dy read it 16*dy rows further down, weights come from the packed image in
    (tap, source, block) order with the 128-byte swizzle undone — must equal F.conv2d on the concatenated input"""
    import torch.nn.functional as F
    from nerf_slam_b200.conv import pack_weights
    g = torch.Generator().manual_seed(5)
    B, H, W, N = 1, 11, 21, 16                                  # partial tiles in both directions
    chans = [128, 72]                                           # second source: 2 blocks, the last one 8 channels wide
    srcs = [torch.randn(B, H, W, c, generator=g) for c in chans]
    w = torch.randn(N, sum(chans), 3, 3, generator=g) * 0.1
    packed = pack_weights(w, chans).float().view(-1, N, 8, 8)   # [block][n][chunk position][8]
    rows = torch.arange(N)
    cbs = [(c + 63) // 64 for c in chans]
    cb_total = sum(cbs)

    def weight_block(tap, cbg):                                 # un-swizzled [N, 64]
        blk = packed[tap * cb_total + cbg]
        out = torch.empty(N, 8, 8)
        for j in range(8):
            out[rows, j] = blk[rows, j ^ (rows & 7)]
        return out.reshape(N, 64)

    ref = F.conv2d(torch.cat(srcs, -1).permute(0, 3, 1, 2).half().float(), w.half().float(), padding=1).permute(0, 2, 3, 1)
    got = torch.zeros(B, H, W, N)
    TH, TW = 8, 16
    for h0 in range(0, H, TH):
        for w0 in range(0, W, TW):
            acc = torch.zeros(TH * TW, N)
            cbg = 0
            for s, c in enumerate(chans):
                for cb in range(cbs[s]):
                    for dx in range(3):
                        # TMA box {64c, 16w, 10h} at (cb*64, w0+dx-1, h0-1): zero fill outside the image / channel range
                        tile = torch.zeros(TH + 2, TW, 64)
                        for hy in range(TH + 2):
                            for wx in range(TW):
                                y, x = h0 - 1 + hy, w0 + dx - 1 + wx
                                if 0 <= y < H and 0 <= x < W:
                                    ce = min(c, cb * 64 + 64)
                                    tile[hy, wx, :ce - cb * 64] = srcs[s][0, y, x, cb * 64:ce].half().float()
                        flat = tile.reshape(-1, 64)                              # smem rows: hy*16 + wx
                        for dy in range(3):
                            A = flat[dy * TW:dy * TW + TH * TW]                    # descriptor offset dy*16 rows
                            acc += A @ weight_block(dy * 3 + dx, cbg).T
                    cbg += 1
            for r in range(TH * TW):
                y, x = h0 + r // TW, w0 + r % TW
                if y < H and x < W:
                    got[0, y, x] = acc[r]
    assert float((got - ref).abs().max()) < 2e-3


def test_forward_placeholders_are_not_none():
    """RaftVisualFrontend.forward returns empty, non-None x0 / factors like the reference's empty gtsam containers
    (visual_frontend.py:248-249): the reference's VioSLAM._frontend stops the pipeline on `x0 is None`
    (slam/vio_slam.py:112-113)"""
    from nerf_slam_b200.frontend import EmptyFactorGraph, EmptyValues
    x0, f = EmptyValues(), EmptyFactorGraph()
    assert x0 is not None and f is not None and bool(x0) and x0.size() == 0 and len(f) == 0
