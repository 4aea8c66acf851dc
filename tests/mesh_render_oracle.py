"""ORACLE (test infrastructure only — never imported by the product path).

Restatement of nerf_slam_b200/csrc/mesh_render.cu's rules in fp64 by brute force over all triangles (no tree), chunked
over rays.  numpy rounds every elementwise operation and never fuses a multiply-add, as the kernel's explicit-rounding
intrinsics do.  The same code runs on torch fp64 tensors (`xp=torch`, on the GPU for the large cases): torch's
elementwise kernels round each operation the same way.

- `rays(...)`: origins and directions of the pixels of one view;
- `cast(...)`: the nearest watertight hit of each ray -> depth, triangle, normal, colour."""
import numpy as np

F32 = np.float32


def _rotation_f32(q):
    """tsdf_pose_rotation: the fp64 rotation of q_xyzw, each entry rounded to fp32 (no normalisation)"""
    x, y, z, w = (np.float64(v) for v in np.asarray(q, F32))
    r = np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                  [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                  [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])
    return r.astype(F32).astype(np.float64)


def rays(pose, intr, W, H, pixels=None):
    """-> origin [3] fp64, directions [P,3] fp64 of the pixels (flat indices v W + u; all when None)"""
    pose = np.asarray(pose, F32)
    R = _rotation_f32(pose[3:])
    t = pose[:3].astype(np.float64)
    o = np.array([-((R[0, c] * t[0] + R[1, c] * t[1]) + R[2, c] * t[2]) for c in range(3)])
    pix = np.arange(W * H) if pixels is None else np.asarray(pixels)
    u, v = (pix % W).astype(F32), (pix // W).astype(F32)
    fx, fy, cx, cy = (F32(x) for x in intr)
    dx = ((u - cx) / fx).astype(F32).astype(np.float64)
    dy = ((v - cy) / fy).astype(F32).astype(np.float64)
    d = np.stack([(R[0, c] * dx + R[1, c] * dy) + R[2, c] for c in range(3)], 1)
    return o, d


class _Np:
    where, minimum, sqrt, abs = staticmethod(np.where), staticmethod(np.minimum), staticmethod(np.sqrt), staticmethod(np.abs)

    @staticmethod
    def asarray(a, like):
        return np.asarray(a)

    @staticmethod
    def min1(a):
        return a.min(1)


class _Torch:
    def __init__(self):
        import torch
        self.t = torch

    def where(self, c, a, b):
        t = self.t
        like = a if t.is_tensor(a) else (b if t.is_tensor(b) else None)
        dtype = like.dtype if like is not None else t.float64
        a = a if t.is_tensor(a) else t.tensor(a, dtype=dtype, device=c.device)
        b = b if t.is_tensor(b) else t.tensor(b, dtype=dtype, device=c.device)
        return t.where(c, a, b)

    def minimum(self, a, b):
        return self.t.minimum(a, b)

    def sqrt(self, a):
        return self.t.sqrt(a)

    def abs(self, a):
        return self.t.abs(a)

    def asarray(self, a, like):
        return self.t.as_tensor(np.asarray(a), device=like.device)

    def min1(self, a):
        return a.min(1).values


def _sel(arrs, k, xp):
    """arrs [3] of [T] per axis, k [P] -> [P,T] = arrs[k[p]][t]"""
    a0, a1, a2 = (x[None, :] for x in arrs)
    k = k[:, None]
    return xp.where(k == 0, a0, xp.where(k == 1, a1, a2))


def cast(vertices, triangles, o, d, near=0.0, far=np.inf, cull=False, colors=None, chunk=1 << 22, xp=None):
    """the nearest hit of the rays (o [3], d [P,3] fp64) among all triangles -> depth [P] fp32 (0 on a miss), triangle
    [P] int64 (-1), normal [P,3] fp32, colour [P,3] fp32 (None without colours), numpy.  xp=None: numpy; "torch": torch
    tensors on the device of `vertices` if it is a tensor, else the CPU."""
    ops = _Np() if xp is None else _Torch()
    if xp is None:
        V = np.asarray(vertices, F32).astype(np.float64)
        T = np.asarray(triangles, np.int64)
        D = np.asarray(d, np.float64)
        tidx = np.arange(len(T))
    else:
        import torch
        dev = vertices.device if torch.is_tensor(vertices) else "cpu"
        V = torch.as_tensor(np.asarray(vertices.cpu() if torch.is_tensor(vertices) else vertices, F32)).to(dev, torch.float64)
        T = torch.as_tensor(np.asarray(triangles.cpu() if torch.is_tensor(triangles) else triangles, np.int64)).to(dev)
        D = torch.as_tensor(np.asarray(d, np.float64)).to(dev)
        tidx = torch.arange(len(T), device=dev)
    o = [float(x) for x in np.asarray(o, np.float64)]
    nearf, farf = float(np.float64(F32(near))), float(np.float64(F32(far)))
    P = D.shape[0]
    # per-ray shear
    absd = ops.abs(D)
    kz = (absd[:, 1] > absd[:, 0]) * 1
    kz = ops.where(absd[:, 2] > ops.where(kz == 1, absd[:, 1], absd[:, 0]), 2, kz)
    kx = ops.where(kz == 2, 0, kz + 1)
    ky = ops.where(kx == 2, 0, kx + 1)
    dz = ops.where(kz == 0, D[:, 0], ops.where(kz == 1, D[:, 1], D[:, 2]))
    swap = dz < 0
    kx, ky = ops.where(swap, ky, kx), ops.where(swap, kx, ky)
    dsel = lambda k: ops.where(k == 0, D[:, 0], ops.where(k == 1, D[:, 1], D[:, 2]))   # noqa: E731
    Sx, Sy, Sz = dsel(kx) / dz, dsel(ky) / dz, 1.0 / dz
    osel = lambda k: ops.where(k == 0, o[0], ops.where(k == 1, o[1], o[2]))           # noqa: E731
    ox, oy, oz = osel(kx), osel(ky), osel(kz)

    best_t = None
    best_i = None
    nt = T.shape[0]
    step = max(1, chunk // max(P, 1))
    for t0 in range(0, nt, step):
        Tc = T[t0:t0 + step]
        verts = [V[Tc[:, k]] for k in range(3)]                      # [Tc,3] each

        def shear(p):
            px = _sel([p[:, 0], p[:, 1], p[:, 2]], kx, ops) - ox[:, None]
            py = _sel([p[:, 0], p[:, 1], p[:, 2]], ky, ops) - oy[:, None]
            pz = _sel([p[:, 0], p[:, 1], p[:, 2]], kz, ops) - oz[:, None]
            return px - Sx[:, None] * pz, py - Sy[:, None] * pz, Sz[:, None] * pz

        (Ax, Ay, Az), (Bx, By, Bz), (Cx, Cy, Cz) = (shear(p) for p in verts)
        U = Cx * By - Cy * Bx
        Vv = Ax * Cy - Ay * Cx
        Wv = Bx * Ay - By * Ax
        mixed = ((U < 0) | (Vv < 0) | (Wv < 0)) & ((U > 0) | (Vv > 0) | (Wv > 0))
        det = (U + Vv) + Wv
        ok = ~mixed & (det != 0)
        if cull:
            ok = ok & (det > 0)
        Tn = (U * Az + Vv * Bz) + Wv * Cz
        t = Tn / ops.where(ok, det, 1.0)
        ok = ok & (t > nearf) & (t <= farf)
        inf = float("inf")
        tm = ops.where(ok, t, inf)
        cmin = ops.min1(tm)
        big = nt + 1
        cand = ops.where(ok & (tm == cmin[:, None]), tidx[t0:t0 + step][None, :], big)
        cidx = ops.min1(cand)
        if best_t is None:
            best_t, best_i = cmin, cidx
        else:
            better = (cmin < best_t) | ((cmin == best_t) & (cidx < best_i))
            best_t, best_i = ops.where(better, cmin, best_t), ops.where(better, cidx, best_i)
    hit = best_i < nt + 1
    if xp is not None:
        best_t, best_i, hit = best_t.cpu().numpy(), best_i.cpu().numpy(), hit.cpu().numpy()
        D = D.cpu().numpy()
        Sx, Sy, Sz = (x.cpu().numpy() for x in (Sx, Sy, Sz))
        kx, ky, kz = (x.cpu().numpy() for x in (kx, ky, kz))
    depth = np.where(hit, best_t, 0.0).astype(F32)
    tri = np.where(hit, best_i, -1).astype(np.int64)
    # normal and colour of the winners (numpy, per ray)
    Vn = np.asarray(vertices.cpu() if hasattr(vertices, "cpu") else vertices, F32).astype(np.float64)
    Tn_ = np.asarray(triangles.cpu() if hasattr(triangles, "cpu") else triangles, np.int64)
    normal = np.zeros((P, 3), F32)
    color = None if colors is None else np.zeros((P, 3), F32)
    h = np.flatnonzero(hit)
    if len(h):
        ids = Tn_[tri[h]]
        a, b, c = Vn[ids[:, 0]], Vn[ids[:, 1]], Vn[ids[:, 2]]
        e1, e2 = b - a, c - a
        x = np.stack([e1[:, 1] * e2[:, 2] - e1[:, 2] * e2[:, 1], e1[:, 2] * e2[:, 0] - e1[:, 0] * e2[:, 2],
                      e1[:, 0] * e2[:, 1] - e1[:, 1] * e2[:, 0]], 1)
        ln = np.sqrt((x[:, 0] * x[:, 0] + x[:, 1] * x[:, 1]) + x[:, 2] * x[:, 2])
        with np.errstate(invalid="ignore", divide="ignore"):
            normal[h] = np.where(ln[:, None] > 0, x / ln[:, None], 0.0).astype(F32)
        if colors is not None:
            C = np.asarray(colors.cpu() if hasattr(colors, "cpu") else colors, F32).astype(np.float64)
            r = np.arange(len(h))
            sx, sy, sz = Sx[h], Sy[h], Sz[h]
            okx, oky, okz = (np.asarray(o)[k[h]] for k in (kx, ky, kz))

            def shear1(p):
                px, py, pz = p[r, kx[h]] - okx, p[r, ky[h]] - oky, p[r, kz[h]] - okz
                return px - sx * pz, py - sy * pz

            (Ax, Ay), (Bx, By), (Cx, Cy) = shear1(a), shear1(b), shear1(c)
            U, Vv, Wv = Cx * By - Cy * Bx, Ax * Cy - Ay * Cx, Bx * Ay - By * Ax
            det = (U + Vv) + Wv
            ca, cb, cc = C[ids[:, 0]], C[ids[:, 1]], C[ids[:, 2]]
            color[h] = (((U[:, None] * ca + Vv[:, None] * cb) + Wv[:, None] * cc) / det[:, None]).astype(F32)
    return depth, tri, normal, color


def render(vertices, triangles, poses, intr, W, H, near=0.0, far=np.inf, cull=False, colors=None, pixels=None, xp=None):
    """cast() for every view of poses [n,7] -> depth [n,P], triangle [n,P], normal [n,P,3], colour [n,P,3] or None
    (P = W H, or the given flat pixel indices)"""
    out = [cast(vertices, triangles, *rays(p, intr, W, H, pixels), near, far, cull, colors, xp=xp) for p in np.asarray(poses)]
    depth, tri, normal = (np.stack([x[i] for x in out]) for i in range(3))
    color = None if colors is None else np.stack([x[3] for x in out])
    return depth, tri, normal, color
