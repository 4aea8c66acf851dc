"""ORACLE (test infrastructure only — never imported by the product path).

numpy / torch restatement of the NeRF mesh read-out (pyngp.Testbed.marching_cubes; kernels in csrc/ngp_tc.cu), rule for
rule: lattice points -> field = thresh - sigma -> visibility weights from the occupancy array -> marching cubes
(tests/tsdf_readout_oracle.py, min_weight 0, no colour volume) -> vertex colours from the network seen along -normal.
Positions are formed with the kernels' fp32 roundings (numpy rounds every elementwise operation), so the lattice points,
hash inputs and visibility weights match the device bit for bit."""
import numpy as np
import torch

from oracle import ngp as ongp
from tests import tsdf_readout_oracle as orc

F32 = np.float32
GRID = 128


def lattice_points(lo, h, dims):
    """-> [nz,ny,nx,3] fp32 points lo + h (i,j,k)"""
    nx, ny, nz = dims
    k, j, i = np.meshgrid(np.arange(nz, dtype=F32), np.arange(ny, dtype=F32), np.arange(nx, dtype=F32), indexing="ij")
    lo = np.asarray(lo, F32)
    h = F32(h)
    return np.stack([lo[0] + h * i, lo[1] + h * j, lo[2] + h * k], -1).astype(F32)


def hash_input(p, aabb_scale):
    """x01 = (p - aabb_lo) * inv_extent with the kernels' fp32 constants"""
    lo = F32(F32(0.5) - F32(0.5) * F32(aabb_scale))
    inv = F32(F32(1.0) / F32(aabb_scale))
    return ((np.asarray(p, F32) - lo).astype(F32) * inv).astype(F32)


def visibility(p, density, cascades):
    """weight 1 where the occupancy cell of cascade mip_from_pos(p) (the finest box holding p) has density >= 0, else 0;
    p [..., 3] fp32, density [cascades * 128^3]"""
    p = np.asarray(p, F32)
    m = np.abs(p - F32(0.5)).max(-1)
    _, e = np.frexp(m)
    e = np.where(m == 0, 0, e)
    mip = np.clip(e + 1, 0, cascades - 1)
    s = np.ldexp(F32(1.0), -mip).astype(F32)
    idx = np.floor((((p - F32(0.5)) * s[..., None]).astype(F32) + F32(0.5)) * F32(GRID)).astype(np.int64)
    inside = ((idx >= 0) & (idx < GRID)).all(-1)
    idx = np.clip(idx, 0, GRID - 1)
    cell = idx[..., 0] + GRID * (idx[..., 1] + GRID * idx[..., 2]) + mip.astype(np.int64) * GRID ** 3
    return (inside & (np.asarray(density)[cell] >= 0)).astype(F32)


def network_params(grid_half, mlp):
    """oracle/ngp.py parameters of a testbed's fp16 table and fp32 MLP blob (torch CPU tensors)"""
    P = {"grid": grid_half.float().cpu().view(-1, 2)}
    w = mlp.float().cpu()
    off = 0
    for name, (i, o) in dict(W1=(32, 64), W2=(64, 16), W3=(32, 64), W4=(64, 64), W5=(64, 16)).items():
        P[name] = w[off:off + i * o].view(i, o).clone()
        off += i * o
    return P


def network_sigma(P, aabb_scale):
    """sigma(p) of the oracle network, p [..., 3] fp32 numpy"""
    def f(p):
        x = torch.from_numpy(hash_input(p, aabb_scale).reshape(-1, 3))
        d = torch.zeros_like(x)
        d[:, 2] = 1.0
        with torch.no_grad():
            _, sigma = ongp.network(x, d, P, aabb_scale)
        return sigma.numpy().astype(F32).reshape(np.shape(p)[:-1])
    return f


def field(sigma, thresh):
    return (F32(thresh) - np.asarray(sigma, F32)).astype(F32)


def mesh(fld, weight, lo, h):
    """-> V, F, C (zeros), N of the marching cubes over the observed cubes (min_weight 0)"""
    return orc.marching_cubes(fld, weight, np.zeros(fld.shape + (3,), F32), np.asarray(lo, F32), F32(h), 0.0)


def color_records(V, N, aabb_scale):
    """forward_tc coordinate records [x01, 0, -n] (+z where the normal is 0) of the vertices"""
    V, N = np.asarray(V, F32), np.asarray(N, F32)
    d = -N
    none = (N == 0).all(-1)
    d[none] = (0.0, 0.0, 1.0)
    return np.concatenate([hash_input(V, aabb_scale), np.zeros((len(V), 1), F32), d], -1).astype(F32)


def linear_to_srgb(c):
    """inverse of the ingest's sRGB -> linear curve (0.04045 / 12.92 / 2.4)"""
    c = np.asarray(c, F32)
    hi = (F32(1.055) * np.power(c, F32(1.0 / 2.4), dtype=F32)).astype(F32) - F32(0.055)
    return np.where(c > F32(0.0031308), hi, (c * F32(12.92)).astype(F32)).astype(F32)


def network_colors(P, aabb_scale, V, N, srgb=False):
    rec = color_records(V, N, aabb_scale)
    with torch.no_grad():
        rgb, _ = ongp.network(torch.from_numpy(rec[:, :3]), torch.from_numpy(rec[:, 4:]), P, aabb_scale)
    rgb = rgb.numpy().astype(F32)
    return linear_to_srgb(rgb) if srgb else rgb


def read_ply(path):
    """binary PLY of TsdfMesh.write_ply -> V, N, C [V,3] fp32, F [T,3] int32"""
    with open(path, "rb") as f:
        data = f.read()
    end = data.index(b"end_header\n") + len(b"end_header\n")
    head = data[:end].decode("ascii").splitlines()
    nv = int([l for l in head if l.startswith("element vertex")][0].split()[-1])
    nf = int([l for l in head if l.startswith("element face")][0].split()[-1])
    vt = np.frombuffer(data, np.dtype([(k, "<f4") for k in ("x", "y", "z", "nx", "ny", "nz", "red", "green", "blue")]),
                       nv, end)
    ft = np.frombuffer(data, np.dtype([("n", "u1"), ("v", "<i4", (3,))]), nf, end + vt.nbytes)
    col = lambda *k: np.stack([vt[x] for x in k], 1).astype(F32)
    return col("x", "y", "z"), col("nx", "ny", "nz"), col("red", "green", "blue"), ft["v"].astype(np.int32)
