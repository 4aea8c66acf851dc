"""Record the feature-map gradients of the REFERENCE's correlation layers (networks/modules/corr.py): `CorrBlock`
(all-pairs volume by matmul, pyramid by avg_pool2d, `CorrSampler` per level at coords / 2^l, :6-72) and `AltCorrBlock`
(feature pyramid by pooling, `CorrLayer` per level, frame indexing, :75-140), run forward and backward on the CPU in
fp32 with the four CUDA entry points they call replaced by the CPU oracle's restatements (oracle/corr.py: the
forwards; oracle/corr_grad.py: corr_index_backward, altcorr_backward — pinned against the reference's compiled
kernels on the GPU by tests/test_gpu_corr_grad.py).  This pins the reference's composition: the /4 scalings, the
pooling, coords / 2^l per level, the channel order and the ii / jj indexing.  Build container only.

  python tests/golden/make_golden_corr_grad.py        ->  tests/golden/ref_corr_grad.npz

The loss is sum(out * w) with w exactly representable in fp16, so that a product path whose correlation output is
fp16 receives the same output gradient."""
import os
import sys
import types

import numpy as np
import torch

REF = os.environ.get("NSLAM_REFERENCE", "/root/reference")
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))


def inputs(seed=29):
    """fmaps [1,2,128,16,16] (fp16-representable), edges (0->1, 1->1), coords around the identity with windows that
    straddle every border, a few far outside the map, and loss weights w [1,2,196,16,16] (fp16-representable)"""
    rng = np.random.default_rng(seed)
    n, C, h, w = 2, 128, 16, 16
    fmaps = rng.normal(0, 1, (1, n, C, h, w)).astype(np.float16).astype(np.float32)
    ii = np.array([0, 1]); jj = np.array([1, 1])
    y, x = np.meshgrid(np.arange(h, dtype=np.float32), np.arange(w, dtype=np.float32), indexing="ij")
    coords = np.stack([x, y], -1)[None, None] + rng.uniform(-6, 6, (1, len(ii), h, w, 2)).astype(np.float32)
    coords[0, 0, 0, :3] = [[1e6, 2.5], [-1e6, 3.25], [4.5, -1e6]]
    weights = rng.normal(0, 1, (1, len(ii), 4 * 49, h, w)).astype(np.float16).astype(np.float32)
    return fmaps, ii, jj, coords, weights


def stand_in():
    """a `droid_backends` module whose four correlation entries are the oracle's restatements"""
    from oracle import corr as ocorr
    from oracle import corr_grad as ograd
    T = torch.from_numpy
    dbk = types.ModuleType("droid_backends")
    dbk.corr_index_forward = lambda vol, coords, r: (T(ocorr.corr_index_forward(vol.detach().numpy(), coords.numpy(), r)),)
    dbk.corr_index_backward = lambda vol, coords, g, r: (
        T(ograd.corr_index_backward(tuple(vol.shape), coords.numpy(), g.numpy(), r)),)
    dbk.altcorr_forward = lambda f1, f2, coords, r: (
        T(ocorr.altcorr_forward(f1.detach().numpy(), f2.detach().numpy(), coords.numpy(), r)),)
    dbk.altcorr_backward = lambda f1, f2, coords, g, r: tuple(
        T(a) for a in ograd.altcorr_backward(f1.detach().numpy(), f2.detach().numpy(), coords.numpy(), g.numpy(), r))
    return dbk


def main():
    sys.path.insert(0, ROOT)
    sys.modules["droid_backends"] = stand_in()
    sys.path.insert(0, REF)
    from networks.modules.corr import AltCorrBlock, CorrBlock
    fmaps, ii, jj, coords, weights = inputs()
    c, w = torch.from_numpy(coords), torch.from_numpy(weights)

    f = torch.from_numpy(fmaps).requires_grad_()
    out_vol = CorrBlock(f[:, ii], f[:, jj])(c)                                        # [1,E,196,h,w]
    (out_vol * w).sum().backward()
    grad_vol = f.grad.numpy().copy()

    f = torch.from_numpy(fmaps).requires_grad_()
    out_alt = AltCorrBlock(f)(c, torch.from_numpy(ii), torch.from_numpy(jj))          # [1,E,196,h,w]
    (out_alt * w).sum().backward()
    grad_alt = f.grad.numpy().copy()

    np.savez_compressed(os.path.join(HERE, "ref_corr_grad.npz"), fmaps=fmaps.astype(np.float16), ii=ii, jj=jj,
                        coords=coords, weights=weights.astype(np.float16), grad_corrblock=grad_vol,
                        grad_altcorrblock=grad_alt)
    print("grad shapes", grad_vol.shape, "max |grad|", float(np.abs(grad_vol).max()),
          "max |CorrBlock - AltCorrBlock|", float(np.abs(grad_vol - grad_alt).max()))


if __name__ == "__main__":
    main()
