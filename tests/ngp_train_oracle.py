"""Restatement of the NeRF trainer's state-carrying kernels (csrc/ngp_train.cu, csrc/ngp_tc.cu) in numpy / torch.

Test infrastructure only.  Where the GPU must match bit for bit, a function replays the kernel's fp32 operations in
np.float32; everything else is fp64.  The rules, as the kernels define them:

- Refresh cells.  A refresh of n < 128^3 cells per cascade visits, in cascade `mip`, the cells
  density_cell(seed, mip, j) = (a j + b) mod 128^3 for j < n, with a odd: an affine permutation, so the cells of one
  refresh are distinct.  A full refresh (n = 128^3) visits cell j.  Thread i = mip n + j evaluates the jittered point
  p = ((ix + rnd01(seed, i, 11 + axis)) / 128 - 0.5) s + 0.5,  s = 2^mip,  and the network at x01 = (p - aabb_lo) / extent.
  In fp32, ix + jitter rounds up to ix + 1 when the jitter is within 2^-24 ix of 1, so a point can sit on the cell's
  upper face; it is still evaluated for its own cell.
- Visibility mark.  A cell at -1 becomes 0 when its centre, widened by the half diagonal h = 0.5 s / 128 sqrt(3), lies in
  front of (z + h > 1e-3) and inside the image of at least one ACTIVE camera: with z' = max(z, 1e-3),
  u +- fx h / z' and v +- fy h / z' overlap [0, w) x [0, h).  Cells at 0 or more are not touched.
- Refresh.  density = max(prev decay, exp(o0) MIN_STEP s) for every visited cell with prev >= 0; cells at -1 never change.
  A partial refresh decays only the cells it visits (published instant-ngp decays every visible cell on every update);
  the product keeps that rule, and the tests pin it.
- Mean and bits.  stats = (sum, count) of the cells >= 0; threshold = min(min_thickness, sum / count) (0 when count is 0);
  bit k of byte i is set when cell 8 i + k is above the threshold.
- Sparse Adam (tiny-cuda-nn semantics) on float4 groups: a group whose four gradients are all zero is not written at all;
  otherwise the gradient is zeroed and every element with a nonzero gradient (grid) or every element (MLP) takes
  grad = g + l2 w,  m = b1 m + (1 - b1) grad,  v = b2 v + (1 - b2) grad^2,  w -= lr (m bc1) / (sqrt(v bc2) + eps),
  bias corrections bc = 1 / (1 - beta^step) computed on the host in fp32 with powf; the fp16 copy of a written grid group
  is the fp32 master rounded to nearest.
- Table scatter.  dL/dtable[level l, corner c] += w_c(x) denc[s, l] / loss_scale over the samples s, with the corners,
  trilinear weights and grid_index of oracle.ngp.hash_encode: pos = x scale + 0.5 (the kernel rounds it once: fmaf),
  dense levels index (x + y res + z res^2) mod size (so x = 1 wraps), hashed levels x ^ y 2654435761 ^ z 805459861 mod T.
- Sample budget.  Ray i is kept iff n_i > 0 and its inclusive prefix sum is <= max_samples; R[12] = exclusive prefix sum
  of every ray, R[13] = n_i when kept else 0, counters = (inclusive sum of the last kept ray, number kept).
"""
import math

import numpy as np
import torch

from oracle import ngp as ongp

F32 = np.float32
GRID = 128
NC = GRID ** 3
SQRT3 = F32(1.73205080757)
MIN_STEP = ongp.MIN_STEP
M32 = np.uint64(0xFFFFFFFF)


# ------------------------------------------------------------------------------------------ refresh cells and points
def pcg(v):
    """ngp_common.cuh::pcg on uint64 arrays holding uint32 values"""
    v = np.asarray(v, np.uint64) & M32
    s = (v * np.uint64(747796405) + np.uint64(2891336453)) & M32
    w = (((s >> ((s >> np.uint64(28)) + np.uint64(4))) ^ s) * np.uint64(277803737)) & M32
    return ((w >> np.uint64(22)) ^ w) & M32


def rnd01(a, b, c):
    """ngp_common.cuh::rnd01 vectorised over b (np.float32; the conversion and the scale by 2^-24 are exact)"""
    h = pcg(pcg(pcg(np.uint64(a)) ^ (np.asarray(b, np.uint64) & M32)) ^ np.uint64(c))
    return (h >> np.uint64(8)).astype(F32) * F32(1.0 / 16777216.0)


def density_cell(seed, mip, j):
    """cell of cascade `mip` visited by thread j of a partial refresh"""
    ps = pcg(np.uint64(seed))
    a = pcg(ps ^ np.uint64(2 * mip)) | np.uint64(1)
    b = pcg(ps ^ np.uint64(2 * mip + 1))
    return ((a * np.asarray(j, np.uint64) + b) & np.uint64(NC - 1)).astype(np.int64)


def refresh_cells(seed, n_per_cascade, cascades, aabb_scale):
    """-> index [k] into the density array (mip NC + cell) and x01 [k,3] float32 (bit-exact to the kernels) of every
    thread of a refresh, in thread order"""
    idx, x01 = [], []
    lo, inv_ext = F32(F32(0.5) - F32(0.5) * F32(aabb_scale)), F32(F32(1.0) / F32(aabb_scale))
    for mip in range(cascades):
        j = np.arange(n_per_cascade, dtype=np.int64)
        cell = j if n_per_cascade >= NC else density_cell(seed, mip, j)
        i = mip * n_per_cascade + j
        ijk = np.stack([cell % GRID, (cell // GRID) % GRID, cell // (GRID * GRID)], -1).astype(F32)
        s = F32(2.0 ** mip)
        p = np.empty_like(ijk)
        for a in range(3):
            q = (ijk[:, a] + rnd01(seed, i, 11 + a)) / F32(GRID)           # a power-of-two divide: exact
            p[:, a] = (q - F32(0.5)) * s + F32(0.5)                        # * s exact, so fmaf gives the same value
        idx.append(mip * NC + cell)
        x01.append((p - lo) * inv_ext)
    return np.concatenate(idx), np.concatenate(x01).astype(F32)


def refresh(prev, idx, sigma, decay, s_of_idx):
    """density after a refresh of the cells idx with network densities sigma (float32, the kernel's exp(o0)):
    max(prev decay, sigma MIN_STEP s) in fp32 on the visited cells that are >= 0, everything else unchanged"""
    out = prev.copy()
    vis = prev[idx] >= 0
    i = idx[vis]
    thick = (sigma[vis].astype(F32) * MIN_STEP) * s_of_idx(i)
    out[i] = np.maximum(prev[i] * F32(decay), thick)
    return out


def cascade_scale(i):
    """s = 2^mip of density-array indices"""
    return (2.0 ** (np.asarray(i) // NC)).astype(F32)


# ------------------------------------------------------------------------------------------ visibility mark
def cell_centres(mip):
    c = np.arange(NC, dtype=np.int64)
    ijk = np.stack([c % GRID, (c // GRID) % GRID, c // (GRID * GRID)], -1).astype(np.float64)
    s = 2.0 ** mip
    return ((ijk + 0.5) / GRID - 0.5) * s + 0.5, 0.5 * s / GRID * float(SQRT3)


def mark_slack(cams18, active, mip):
    """fp64 visibility of the cells of cascade `mip` -> (visible [NC] bool, margin [NC] float64).

    margin: how far the decision is from flipping.  Per camera the five inequalities of the kernel (in front; the four
    image edges) give slacks in pixels (the depth test is scaled by fx / z' into pixels as well); a camera sees the cell
    robustly when its smallest slack is > margin, misses it robustly when its smallest slack is < -margin.  The cell's
    margin is the largest |smallest slack| over the cameras that see it, or the smallest |smallest slack| over all
    cameras when none does: cells with a small margin may go either way under fp32 rounding."""
    p, half = cell_centres(mip)
    best_in = np.full(NC, -np.inf)
    worst_out = np.full(NC, np.inf)
    for a in active:
        c = np.asarray(cams18[a], F32)
        M = c[:12].astype(np.float64).reshape(3, 4)
        fx, fy, cx, cy = (float(v) for v in c[12:16])
        w, h = (int(v) for v in c[16:18].view(np.int32))
        q = p - M[:, 3]
        xc, yc, zc = q @ M[:, 0], q @ M[:, 1], q @ M[:, 2]
        z = np.maximum(zc, 1e-3)
        u, v = fx * xc / z + cx, fy * yc / z + cy
        mu, mv = fx * half / z, fy * half / z
        sl = np.stack([(zc + half - 1e-3) * fx / z, u + mu, w - (u - mu), v + mv, h - (v - mv)], 0)
        m = sl.min(0)
        best_in = np.maximum(best_in, m)
        worst_out = np.minimum(worst_out, np.abs(m))
    vis = best_in > 0
    margin = np.where(vis, best_in, worst_out)
    return vis, margin


# ------------------------------------------------------------------------------------------ mean and bits
def threshold(stats, min_thickness):
    """density_bits_kernel's threshold from the kernel's own stats (fp32)"""
    s, c = F32(stats[0]), F32(stats[1])
    return min(F32(min_thickness), s / c if c > 0 else F32(0.0))


def pack_bits(density, thr):
    return np.packbits(density.reshape(-1, 8) > thr, axis=1, bitorder="little").reshape(-1)


# ------------------------------------------------------------------------------------------ sparse Adam
def adam_constants(step, beta1, beta2):
    """the host's fp32 constants: b1, b2, 1 - b1, 1 - b2 and bc1 = 1 / (1 - powf(b1, step)), bc2 likewise"""
    b1, b2 = F32(beta1), F32(beta2)
    bc1 = F32(1.0) / (F32(1.0) - np.power(b1, F32(step)))
    bc2 = F32(1.0) / (F32(1.0) - np.power(b2, F32(step)))
    return b1, b2, F32(1.0) - b1, F32(1.0) - b2, bc1, bc2


def adam(w, g, m, v, step, lr, beta1, beta2, eps, l2, sparse, m_new=None, v_new=None):
    """one Adam step over float4 groups in fp64 from fp32 state -> dict(w, m, v, written [n] bool, updated [n] bool,
    terms: magnitudes of the largest term of each update, for the error bounds).

    sparse: the hash-table rule (zero-gradient elements keep their state, all-zero groups are not written).
    m_new / v_new (optional, fp32): the kernel's own moments, used for the weight update so that the weight is checked
    from the moments the kernel actually holds."""
    b1, b2, omb1, omb2, bc1, bc2 = (float(c) for c in adam_constants(step, beta1, beta2))
    lr, eps, l2 = float(F32(lr)), float(F32(eps)), float(F32(l2))
    w64, g64, m64, v64 = (np.asarray(a, np.float64) for a in (w, g, m, v))
    group_nz = (g64.reshape(-1, 4) != 0).any(1).repeat(4)
    upd = (g64 != 0) if sparse else np.ones_like(group_nz)
    written = group_nz if sparse else np.ones_like(group_nz)
    grad = g64 + l2 * w64
    mo = np.where(upd, b1 * m64 + omb1 * grad, m64)
    vo = np.where(upd, b2 * v64 + omb2 * grad * grad, v64)
    mu = mo if m_new is None else np.asarray(m_new, np.float64)
    vu = vo if v_new is None else np.asarray(v_new, np.float64)
    stepv = lr * (mu * bc1) / (np.sqrt(vu * bc2) + eps)
    wo = np.where(upd, w64 - stepv, w64)
    return dict(w=wo, m=mo, v=vo, written=written, updated=upd,
                m_scale=np.maximum(np.abs(b1 * m64), np.abs(omb1 * grad)), v_scale=np.abs(vo),
                w_scale=np.maximum(np.abs(w64), np.abs(stepv)))


def ulp32(x):
    """spacing of float32 numbers at |x| (the smallest normal spacing below 2^-126)"""
    x = np.maximum(np.abs(np.asarray(x, np.float64)), 2.0 ** -126)
    return 2.0 ** (np.floor(np.log2(x)) - 23)


# ------------------------------------------------------------------------------------------ table scatter
def fma32(a, b, c):
    """fmaf(a, b, c) on float32 arrays: a b is exact in fp64; the fp64 sum is corrected to one rounding to fp32 by
    TwoSum (a double rounding can only go wrong when the fp64 sum sits exactly on a float32 midpoint)"""
    p = a.astype(np.float64) * b.astype(np.float64)
    c64 = np.asarray(c, np.float64)
    s = p + c64
    bb = s - p
    e = (p - (s - bb)) + (c64 - bb)                     # s + e == p + c exactly
    r = s.astype(F32)
    lo, hi = np.nextafter(r, F32(-np.inf)), np.nextafter(r, F32(np.inf))
    mid_lo, mid_hi = (r.astype(np.float64) + lo) / 2, (r.astype(np.float64) + hi) / 2
    r = np.where((s == mid_lo) & (e < 0), lo, r)        # ties that fp64 resolved without seeing e
    r = np.where((s == mid_hi) & (e > 0), hi, r)
    return r.astype(F32)


def corners(x01, aabb_scale, level, kernel_rounding=True):
    """-> table entry index [S,8] (within the level), trilinear weight [S,8] fp64, corner cells [S,8,3] of one level.
    kernel_rounding: pos = fmaf(x, scale, 0.5) as the kernels do; False: x scale + 0.5 with two fp32 roundings as
    oracle.ngp.hash_encode (torch) does"""
    lv, _ = ongp.level_params(aabb_scale)
    scale, res, n, _ = lv[level]
    x = np.asarray(x01, F32)
    sc = F32(scale)
    pos = fma32(x, np.full_like(x, sc), F32(0.5)) if kernel_rounding else (x * sc + F32(0.5)).astype(F32)
    f = np.floor(pos)
    wf = (pos - f).astype(np.float64)                  # exact
    base = f.astype(np.int64)
    idx, wt, cell = [], [], []
    for c in range(8):
        d = np.array([c & 1, (c >> 1) & 1, c >> 2])
        ijk = base + d
        w = np.prod(np.where(d == 1, wf, 1.0 - wf), axis=1)
        idx.append(np.asarray(ongp.grid_index(ijk[:, 0], ijk[:, 1], ijk[:, 2], res, n), np.int64))
        wt.append(w)
        cell.append(ijk)
    return np.stack(idx, 1), np.stack(wt, 1), np.stack(cell, 1)


def scatter(x01, g, aabb_scale, kernel_rounding=True):
    """table gradient [total,2] fp64 = sum over samples and levels of w_c(x) g[s, 2l:2l+2], plus the per-entry sum of
    |contributions| [total,2] and the number of contributing samples [total] (for error bounds).  g: [S,32] fp64"""
    lv, total = ongp.level_params(aabb_scale)
    g = np.asarray(g, np.float64)
    out, mag, cnt = np.zeros((total, 2)), np.zeros((total, 2)), np.zeros(total, np.int64)
    for l, (_, _, _, off) in enumerate(lv):
        idx, wt, _ = corners(x01, aabb_scale, l, kernel_rounding)
        c = wt[..., None] * g[:, None, 2 * l:2 * l + 2]                # [S,8,2]
        e = off + idx.reshape(-1)
        np.add.at(out, e, c.reshape(-1, 2))
        np.add.at(mag, e, np.abs(c).reshape(-1, 2))
        np.add.at(cnt, e, (np.abs(c).reshape(-1, 2).sum(1) > 0).astype(np.int64))
    return out, mag, cnt


def hashed_collision(aabb_scale, level=None, seed=0, tries=20000):
    """two distinct cells of a hashed level with the same table entry -> (level, cell_a [3], cell_b [3]); the cells and
    their +1 neighbours lie inside the lattice, so points in both cells are in [0,1]^3"""
    lv, _ = ongp.level_params(aabb_scale)
    levels = [l for l, (_, res, n, _) in enumerate(lv) if res ** 3 > n]
    l = levels[0] if level is None else level
    scale, res, n, _ = lv[l]
    rng = np.random.default_rng(seed)
    hi = int(math.floor(scale)) - 1
    ijk = rng.integers(1, hi, size=(tries, 3))
    h = np.asarray(ongp.grid_index(ijk[:, 0], ijk[:, 1], ijk[:, 2], res, n), np.int64)
    order = np.argsort(h, kind="stable")
    hs = h[order]
    dup = np.nonzero(hs[1:] == hs[:-1])[0]
    for k in dup:
        a, b = ijk[order[k]], ijk[order[k + 1]]
        if not np.array_equal(a, b):
            return l, a, b
    raise RuntimeError("no collision found")


def point_in_cell(cell, frac, aabb_scale, level):
    """float32 point whose level-`level` position fmaf(x, scale, 0.5) lies at cell + frac"""
    lv, _ = ongp.level_params(aabb_scale)
    scale = lv[level][0]
    return ((np.asarray(cell, np.float64) + frac - 0.5) / scale).astype(F32)


def edge_points(aabb_scale, kernel_rounding=True):
    """float32 points [K,3] at the edges of the lattice: on nodes (pos integral on every axis of some level, under the
    kernel's or hash_encode's rounding), on faces (one axis), at 0 and 1, and in the two cells of a hashed-level
    collision pair"""
    lv, _ = ongp.level_params(aabb_scale)
    pts = [np.zeros(3, F32), np.ones(3, F32), np.array([0, 1, 0.5], F32), np.array([1, 0, 1], F32)]
    for l in (0, 3, 7, 15):
        sc = F32(lv[l][0])
        for k in (1, 5, 9):
            x0 = F32((k - 0.5) / float(sc))
            for x in (x0, np.nextafter(x0, F32(1)), np.nextafter(x0, F32(0))):
                xa = np.array([x], F32)
                pos = fma32(xa, np.full_like(xa, sc), F32(0.5))[0] if kernel_rounding else F32(x * sc) + F32(0.5)
                if pos == F32(k):
                    pts.append(np.array([x, x, x], F32))                 # node
                    pts.append(np.array([x, 0.37, 0.61], F32))           # face
                    break
    l, ca, cb = hashed_collision(aabb_scale)
    for frac in (0.25, 0.75):
        pts.append(point_in_cell(ca, frac, aabb_scale, l))
        pts.append(point_in_cell(cb, frac, aabb_scale, l))
    return np.stack(pts).astype(F32)


def network_from_enc(enc, d, P):
    """oracle.ngp.network from a given encoding (so that autograd can report dL/denc)"""
    h = torch.relu(enc @ P["W1"])
    o = h @ P["W2"]
    sigma = torch.exp(o[:, 0])
    h = torch.relu(torch.cat([o, ongp.sh4(d)], -1) @ P["W3"])
    h = torch.relu(h @ P["W4"])
    return torch.sigmoid((h @ P["W5"])[:, :3]), sigma


# ------------------------------------------------------------------------------------------ sample budget
def sample_budget(counts, max_samples):
    """-> dict(offset [R] exclusive prefix sums, kept [R] bool, n [R] = counts where kept else 0, counters (used, kept))"""
    n = np.asarray(counts, np.int64)
    incl = np.cumsum(n)
    kept = (n > 0) & (incl <= max_samples)
    used = int(incl[kept][-1]) if kept.any() else 0
    return dict(offset=incl - n, kept=kept, n=np.where(kept, n, 0), counters=(used, int(kept.sum())))
