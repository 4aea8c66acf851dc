"""ORACLE (test infrastructure only — never imported by the product path).

numpy restatements of the two read-outs of the dense TSDF volume in nerf_slam_b200/csrc/tsdf_mesh.cu, rule for rule and
fp32 operation for fp32 operation (no fused multiply-add anywhere: numpy rounds every elementwise operation), so that the
kernels can be compared element by element:

- `marching_cubes(...)`: vertices ordered by the linear index of the voxel that owns their lattice edge, then by axis
  x, y, z; triangles ordered by linear cube index, then by table order.
- `raycast(...)`: the z-parametrised ray march with the trilinear TSDF and the first + -> - transition as the hit.

The case table uses the Lorensen / Bourke corner and edge numbering.  It is derived here from one rule (below) and
`tests/test_cpu_tsdf_mesh.py` checks that the table compiled into the kernel is the same."""
import numpy as np

F32 = np.float32

# corner n of a cube -> (dx, dy, dz); edge e -> (corner a, corner b)
CORNERS = [(0, 0, 0), (1, 0, 0), (1, 1, 0), (0, 1, 0), (0, 0, 1), (1, 0, 1), (1, 1, 1), (0, 1, 1)]
EDGES = [(0, 1), (1, 2), (3, 2), (0, 3), (4, 5), (5, 6), (7, 6), (4, 7), (0, 4), (1, 5), (2, 6), (3, 7)]
# cube faces as cycles of corners
FACES = [(0, 1, 2, 3), (4, 5, 6, 7), (0, 1, 5, 4), (3, 2, 6, 7), (0, 3, 7, 4), (1, 2, 6, 5)]


def edge_owner_axis(e):
    """lattice edge e of a cube -> (owner corner offset (dx, dy, dz), axis 0/1/2): the owner is the lower endpoint"""
    a, b = EDGES[e]
    pa, pb = np.array(CORNERS[a]), np.array(CORNERS[b])
    return tuple(int(v) for v in np.minimum(pa, pb)), int(np.argmax(np.abs(pb - pa)))


def _edge_of(a, b):
    for e, (p, q) in enumerate(EDGES):
        if {p, q} == {a, b}:
            return e
    raise KeyError((a, b))


def make_tri_table():
    """256 cases x up to 5 triangles of edge indices; corner bit n set = tsdf < 0 at corner n (inside).

    Rule: on every cube face the iso-line separates the inside corners (marching squares; on an ambiguous face, whose
    inside corners are diagonal, each inside corner is cut off by its own segment).  The decision depends only on the
    face's four corners, so the two cubes sharing a face agree and the surface is closed.  The segments of the six faces
    join into loops; each loop is oriented so that (b - a) x (c - a) points from the inside corners to the outside ones
    (toward +tsdf), starts at its lowest edge index and is fanned from there."""
    mid = np.array([(np.array(CORNERS[a]) + np.array(CORNERS[b])) / 2.0 for a, b in EDGES])
    table = []
    for case in range(256):
        inside = [(case >> n) & 1 for n in range(8)]
        nbr = {}
        for f in FACES:
            es = [_edge_of(f[m], f[(m + 1) % 4]) for m in range(4)]
            cross = [m for m in range(4) if inside[f[m]] != inside[f[(m + 1) % 4]]]
            if len(cross) == 2:
                segs = [(es[cross[0]], es[cross[1]])]
            elif len(cross) == 4:
                segs = [(es[(m - 1) % 4], es[m]) for m in range(4) if inside[f[m]]]
            else:
                segs = []
            for a, b in segs:
                nbr.setdefault(a, []).append(b)
                nbr.setdefault(b, []).append(a)
        tris, seen = [], set()
        for start in sorted(nbr):
            if start in seen:
                continue
            loop, prev, cur = [start], None, start
            while True:
                seen.add(cur)
                nxt = [v for v in nbr[cur] if v != prev]
                nxt = nxt[0] if prev is not None else min(nbr[cur])
                if nxt == start:
                    break
                loop.append(nxt)
                prev, cur = cur, nxt
            P = mid[loop]
            newell = sum(np.cross(P[i], P[(i + 1) % len(P)]) for i in range(len(P)))
            out = sum((np.array(CORNERS[b]) - np.array(CORNERS[a])) * (1 if inside[a] else -1) for a, b in
                      (EDGES[e] for e in loop))
            if float(np.dot(newell, out)) < 0:
                loop = [loop[0]] + loop[1:][::-1]
            tris += [(loop[0], loop[i], loop[i + 1]) for i in range(1, len(loop) - 1)]
        table.append(tris)
    return table


TRI_TABLE = make_tri_table()


# ---------------------------------------------------------------------------------------------------------- marching cubes
def _gradient(t):
    """central differences of the TSDF per axis (one-sided at the border), fp32 -> [3, nz, ny, nx] as (gx, gy, gz)"""
    out = []
    for ax in (2, 1, 0):                                  # x, y, z axes of a [nz,ny,nx] array
        n = t.shape[ax]
        g = np.zeros_like(t)
        if n > 1:
            sl = lambda a, b: tuple(slice(a, b) if d == ax else slice(None) for d in range(3))
            g[sl(1, n - 1)] = (t[sl(2, n)] - t[sl(0, n - 2)]) * F32(0.5)
            g[sl(0, 1)] = t[sl(1, 2)] - t[sl(0, 1)]
            g[sl(n - 1, n)] = t[sl(n - 1, n)] - t[sl(n - 2, n - 1)]
        out.append(g)
    return out


def marching_cubes(tsdf, weight, color, origin, voxel_size, min_weight):
    """-> vertices [V,3], triangles [T,3] int32, vertex colours [V,3] in [0,1], vertex normals [V,3] (fp32 numpy)"""
    t = np.ascontiguousarray(tsdf, F32)
    w = np.ascontiguousarray(weight, F32)
    c = np.ascontiguousarray(color, F32)
    nz, ny, nx = t.shape
    neg = t < 0
    ok = w > F32(min_weight)
    # cube (k, j, i) spans voxels k..k+1, j..j+1, i..i+1; valid = 8 corners with weight > min_weight.  Padded by one on
    # both sides so that out-of-range cubes read as invalid: cvp[k+1, j+1, i+1] = cube (k, j, i)
    cvp = np.zeros((nz + 1, ny + 1, nx + 1), bool)
    if nx > 1 and ny > 1 and nz > 1:
        cv = np.ones((nz - 1, ny - 1, nx - 1), bool)
        case = np.zeros((nz - 1, ny - 1, nx - 1), np.int32)
        for n, (dx, dy, dz) in enumerate(CORNERS):
            sl = (slice(dz, nz - 1 + dz), slice(dy, ny - 1 + dy), slice(dx, nx - 1 + dx))
            cv &= ok[sl]
            case |= neg[sl].astype(np.int32) << n
        cvp[1:nz, 1:ny, 1:nx] = cv
    else:
        cv = np.zeros((max(nz - 1, 0), max(ny - 1, 0), max(nx - 1, 0)), bool)
        case = np.zeros(cv.shape, np.int32)
    # vertex on edge (owner voxel, axis): sign change and at least one of the <= 4 cubes sharing it is valid
    ex = np.zeros((nz, ny, nx, 3), bool)
    K, J, I = np.meshgrid(np.arange(nz), np.arange(ny), np.arange(nx), indexing="ij")
    ex[:, :, :-1, 0] = (neg[:, :, :-1] != neg[:, :, 1:]) & (
        cvp[1:, 1:, 1:nx] | cvp[1:, :-1, 1:nx] | cvp[:-1, 1:, 1:nx] | cvp[:-1, :-1, 1:nx])
    ex[:, :-1, :, 1] = (neg[:, :-1, :] != neg[:, 1:, :]) & (
        cvp[1:, 1:ny, 1:] | cvp[1:, 1:ny, :-1] | cvp[:-1, 1:ny, 1:] | cvp[:-1, 1:ny, :-1])
    ex[:-1, :, :, 2] = (neg[:-1] != neg[1:]) & (
        cvp[1:nz, 1:, 1:] | cvp[1:nz, 1:, :-1] | cvp[1:nz, :-1, 1:] | cvp[1:nz, :-1, :-1])
    flat = ex.reshape(-1)
    vid = np.cumsum(flat, dtype=np.int64) - 1
    vid = vid.reshape(nz, ny, nx, 3)
    sel = np.nonzero(flat)[0]
    vox, axis = sel // 3, sel % 3
    k, j, i = vox // (ny * nx), (vox // nx) % ny, vox % nx
    step = np.array([[1, 0, 0], [0, 1, 0], [0, 0, 1]])[axis]            # (di, dj, dk)
    k1, j1, i1 = k + step[:, 2], j + step[:, 1], i + step[:, 0]
    f0, f1 = t[k, j, i], t[k1, j1, i1]
    tt = f0 / (f0 - f1)
    org = np.asarray(origin, F32)
    vs = F32(voxel_size)
    idx = np.stack([i, j, k], 1).astype(F32)
    along = np.where(step.astype(bool), (idx + tt[:, None]).astype(F32), idx)
    verts = (org[None, :] + vs * along).astype(F32)
    c0, c1 = c[k, j, i], c[k1, j1, i1]
    cols = ((c0 + tt[:, None] * (c1 - c0)) / F32(255.0)).astype(F32)
    g = _gradient(t)
    g0 = np.stack([g[a][k, j, i] for a in range(3)], 1)
    g1 = np.stack([g[a][k1, j1, i1] for a in range(3)], 1)
    nrm = (g0 + tt[:, None] * (g1 - g0)).astype(F32)
    ln = np.sqrt(nrm[:, 0] * nrm[:, 0] + nrm[:, 1] * nrm[:, 1] + nrm[:, 2] * nrm[:, 2])
    with np.errstate(divide="ignore", invalid="ignore"):
        nrm = np.where(ln[:, None] > 0, nrm / ln[:, None], F32(0)).astype(F32)
    # triangles: valid cubes in linear order, then table order
    ntri_case = np.array([len(x) for x in TRI_TABLE], np.int64)
    tab = np.full((256, 5, 3), -1, np.int64)
    for cs, tl in enumerate(TRI_TABLE):
        for s, tri in enumerate(tl):
            tab[cs, s] = tri
    cubes = np.nonzero(cv.reshape(-1))[0]
    cc = case.reshape(-1)[cubes]
    nt = ntri_case[cc]
    keep = nt > 0
    cubes, cc, nt = cubes[keep], cc[keep], nt[keep]
    base = np.cumsum(nt) - nt
    T = int(nt.sum())
    tris = np.zeros((T, 3), np.int32)
    ck, cj, ci = cubes // ((ny - 1) * (nx - 1)), (cubes // (nx - 1)) % (ny - 1), cubes % (nx - 1)
    own = [edge_owner_axis(e) for e in range(12)]
    for s in range(5):
        m = nt > s
        for q in range(3):
            e = tab[cc[m], s, q]
            off = np.array([own[x][0] for x in e], np.int64).reshape(-1, 3)
            ax = np.array([own[x][1] for x in e], np.int64)
            tris[base[m] + s, q] = vid[ck[m] + off[:, 2], cj[m] + off[:, 1], ci[m] + off[:, 0], ax]
    return verts, tris, cols, nrm


# ---------------------------------------------------------------------------------------------------------------- ray cast
def _pose_rotation_center(tq):
    """cam_T_world (t, q_xyzw) -> rotation rounded to fp32 (as fp64) and the camera centre -R^T t rounded to fp32"""
    x, y, z, w = [float(v) for v in np.asarray(tq, F32)[3:]]
    R = np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                  [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                  [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]], np.float64)
    R = R.astype(F32).astype(np.float64)
    t = np.asarray(tq, F32)[:3].astype(np.float64)
    cw = np.array([-((R[0, a] * t[0] + R[1, a] * t[1]) + R[2, a] * t[2]) for a in range(3)]).astype(F32)
    return R, cw


def _corners(arr, iz, iy, ix):
    """8 cell corners [dz][dy][dx] of a [nz,ny,nx(,c)] array at integer cell origins"""
    return [[[arr[iz + dz, iy + dy, ix + dx] for dx in (0, 1)] for dy in (0, 1)] for dz in (0, 1)]


def _lerp(a, b, t):
    return (a + t * (b - a)).astype(F32)


def _trilinear(cn, fx, fy, fz):
    c0 = _lerp(_lerp(cn[0][0][0], cn[0][0][1], fx), _lerp(cn[0][1][0], cn[0][1][1], fx), fy)
    c1 = _lerp(_lerp(cn[1][0][0], cn[1][0][1], fx), _lerp(cn[1][1][0], cn[1][1][1], fx), fy)
    return _lerp(c0, c1, fz)


def raycast(tsdf, weight, color, origin, voxel_size, cam_T_world_tq, H, W, intr, min_depth, max_depth, sdf_trunc,
            min_weight):
    """one view -> depth [H,W] (0 = miss), colour [H,W,3] in [0,1], weight [H,W], normal [H,W,3]"""
    t = np.ascontiguousarray(tsdf, F32)
    wt = np.ascontiguousarray(weight, F32)
    col = np.ascontiguousarray(color, F32)
    nz, ny, nx = t.shape
    dims = np.array([nx, ny, nz])
    fx, fy, cx, cy = [F32(v) for v in intr]
    vs, zmin, zmax, trunc, wmin = F32(voxel_size), F32(min_depth), F32(max_depth), F32(sdf_trunc), F32(min_weight)
    R, cw = _pose_rotation_center(cam_T_world_tq)
    org = np.asarray(origin, F32)
    go = [((cw[a] - org[a]) / vs).astype(F32) for a in range(3)]
    v, u = np.meshgrid(np.arange(H), np.arange(W), indexing="ij")
    dxc = ((u.reshape(-1).astype(F32) - cx) / fx).astype(F32)
    dyc = ((v.reshape(-1).astype(F32) - cy) / fy).astype(F32)
    dw = [((R[0, a] * dxc.astype(np.float64) + R[1, a] * dyc.astype(np.float64)) + R[2, a] * 1.0).astype(F32)
          for a in range(3)]
    gd = [(dw[a] / vs).astype(F32) for a in range(3)]
    ln = np.sqrt((dxc * dxc + dyc * dyc) + F32(1.0)).astype(F32)
    max_steps = np.ceil(((zmax - zmin) * ln / vs).astype(F32)).astype(np.int64) + 2
    P = H * W

    def sample(rows, z):
        g = [(go[a] + z * gd[a][rows]).astype(F32) for a in range(3)]
        fl = [np.floor(g[a]) for a in range(3)]
        inb = np.ones(rows.shape, bool)
        for a in range(3):
            inb &= (fl[a] >= 0) & (fl[a] <= dims[a] - 2)
        ii = [np.where(inb, fl[a], 0).astype(np.int64) for a in range(3)]
        fr = [(g[a] - fl[a]).astype(F32) for a in range(3)]
        obs = inb.copy()
        wc = _corners(wt, ii[2], ii[1], ii[0])
        for dz in (0, 1):
            for dy in (0, 1):
                for dx in (0, 1):
                    obs &= wc[dz][dy][dx] > wmin
        f = _trilinear(_corners(t, ii[2], ii[1], ii[0]), fr[0], fr[1], fr[2])
        return obs, f

    z = np.full(P, zmin, F32)
    have_prev = np.zeros(P, bool)
    f_prev = np.zeros(P, F32)
    z_prev = np.zeros(P, F32)
    hit = np.zeros(P, bool)
    z_hit = np.zeros(P, F32)
    alive = np.arange(P)
    s = 0
    while alive.size:
        alive = alive[(z[alive] <= zmax) & (s < max_steps[alive])]
        if not alive.size:
            break
        za = z[alive]
        obs, f = sample(alive, za)
        h = obs & have_prev[alive] & (f_prev[alive] > 0) & (f <= 0)
        if h.any():
            r = alive[h]
            zp, fp = z_prev[r], f_prev[r]
            z_hit[r] = (zp + ((za[h] - zp) * fp) / (fp - f[h])).astype(F32)
            hit[r] = True
        step = np.where(obs & (f > 0), np.maximum((f * trunc).astype(F32), vs), vs).astype(F32)
        have_prev[alive] = obs
        f_prev[alive] = f
        z_prev[alive] = za
        z[alive] = (za + (step / ln[alive]).astype(F32)).astype(F32)
        alive = alive[~h]
        s += 1

    depth = np.zeros(P, F32)
    rgb = np.zeros((P, 3), F32)
    wout = np.zeros(P, F32)
    nrm = np.zeros((P, 3), F32)
    r = np.nonzero(hit)[0]
    if r.size:
        zh = z_hit[r]
        g = [(go[a] + zh * gd[a][r]).astype(F32) for a in range(3)]
        ii = [np.clip(np.floor(g[a]), 0, dims[a] - 2).astype(np.int64) for a in range(3)]
        fr = [(g[a] - ii[a].astype(F32)).astype(F32) for a in range(3)]
        depth[r] = zh
        wout[r] = _trilinear(_corners(wt, ii[2], ii[1], ii[0]), *fr)
        cc = _corners(col, ii[2], ii[1], ii[0])
        for ch in range(3):
            cn = [[[cc[dz][dy][dx][:, ch] for dx in (0, 1)] for dy in (0, 1)] for dz in (0, 1)]
            rgb[r, ch] = (_trilinear(cn, *fr) / F32(255.0)).astype(F32)
        tc = _corners(t, ii[2], ii[1], ii[0])
        d = lambda a, b: (a - b).astype(F32)
        gx = _lerp(_lerp(d(tc[0][0][1], tc[0][0][0]), d(tc[0][1][1], tc[0][1][0]), fr[1]),
                   _lerp(d(tc[1][0][1], tc[1][0][0]), d(tc[1][1][1], tc[1][1][0]), fr[1]), fr[2])
        gy = _lerp(_lerp(d(tc[0][1][0], tc[0][0][0]), d(tc[0][1][1], tc[0][0][1]), fr[0]),
                   _lerp(d(tc[1][1][0], tc[1][0][0]), d(tc[1][1][1], tc[1][0][1]), fr[0]), fr[2])
        gz = _lerp(_lerp(d(tc[1][0][0], tc[0][0][0]), d(tc[1][0][1], tc[0][0][1]), fr[0]),
                   _lerp(d(tc[1][1][0], tc[0][1][0]), d(tc[1][1][1], tc[0][1][1]), fr[0]), fr[1])
        gl = np.sqrt((gx * gx + gy * gy) + gz * gz).astype(F32)
        with np.errstate(divide="ignore", invalid="ignore"):
            for a, ga in enumerate((gx, gy, gz)):
                nrm[r, a] = np.where(gl > 0, ga / gl, F32(0)).astype(F32)
    return depth.reshape(H, W), rgb.reshape(H, W, 3), wout.reshape(H, W), nrm.reshape(H, W, 3)
