"""numpy fp64 restatement of the mesh operations (nerf_slam_b200/csrc/mesh_ops.cu, rules at its head).  Components come
from scipy.sparse.csgraph; every floating-point sum runs in the kernels' order (np.add.at applies its updates in index
order), so the results match the GPU bit for bit.  A refused input raises ValueError, as nerf_slam_b200.mesh_ops does."""
import numpy as np
from scipy.sparse import coo_matrix
from scipy.sparse.csgraph import connected_components as _csgraph_components

from tests.recon_eval_oracle import triangle_weights, visible

F32 = np.float32
BIAS = 1 << 20
EMPTY = np.uint64(0xFFFFFFFFFFFFFFFF)


def _check_indices(V, T):
    if len(T) and (np.any(T < 0) or np.any(T >= len(V))):
        raise ValueError("a triangle indexes a vertex outside the mesh")


def _check_finite(V, T):
    if len(T) and not np.isfinite(V[np.unique(T)]).all():
        raise ValueError("the mesh has non-finite vertex coordinates")


def _arrays(V, T):
    V = np.asarray(V, F32).reshape(-1, 3)
    T = np.asarray(T, np.int64).reshape(-1, 3)
    _check_indices(V, T)
    return V, T


def connected_components(V, T):
    """-> labels [T] int32, n_triangles [C] int64, area [C] float64"""
    V, T = _arrays(V, T)
    if len(T) == 0:
        return np.zeros(0, np.int32), np.zeros(0, np.int64), np.zeros(0, np.float64)
    w, flags = triangle_weights(V, T)
    if flags & 2:
        raise ValueError("the mesh has non-finite vertex coordinates")
    if flags & 4:
        raise ValueError("the mesh is too large for the 64-bit area sums")
    rows = np.concatenate([T[:, 0], T[:, 0]])
    cols = np.concatenate([T[:, 1], T[:, 2]])
    g = coo_matrix((np.ones(len(rows)), (rows, cols)), shape=(len(V), len(V)))
    _, vlab = _csgraph_components(g, directed=False)
    tlab = vlab[T[:, 0]]
    _, first = np.unique(tlab, return_index=True)             # lowest triangle of each component
    order = np.argsort(first, kind="stable")
    renum = np.empty(len(first), np.int64)
    renum[order] = np.arange(len(first))
    labels = renum[np.searchsorted(np.unique(tlab), tlab)]
    counts = np.bincount(labels, minlength=len(first)).astype(np.int64)
    fixed = np.zeros(len(first), np.uint64)
    np.add.at(fixed, labels, w)
    return labels.astype(np.int32), counts, fixed.astype(np.float64) / 2.0 ** 40


def vertex_normals(V, T):
    """-> [V,3] fp32"""
    V, T = _arrays(V, T)
    _check_finite(V, T)
    P = V.astype(np.float64)
    s = np.zeros((len(V), 3))
    if len(T):
        a, b, c = P[T[:, 0]], P[T[:, 1]], P[T[:, 2]]
        e1, e2 = b - a, c - a
        n = np.stack([e1[:, 1] * e2[:, 2] - e1[:, 2] * e2[:, 1], e1[:, 2] * e2[:, 0] - e1[:, 0] * e2[:, 2],
                      e1[:, 0] * e2[:, 1] - e1[:, 1] * e2[:, 0]], 1)
        np.add.at(s, T.reshape(-1), np.repeat(n, 3, axis=0))   # corners 3t + k: ascending triangle order per vertex
    l = np.sqrt((s[:, 0] * s[:, 0] + s[:, 1] * s[:, 1]) + s[:, 2] * s[:, 2])
    with np.errstate(invalid="ignore", divide="ignore"):
        out = np.where(l[:, None] > 0, s / l[:, None], 0.0)
    return out.astype(F32)


def submesh(V, T, keep, colors=None, normals=None):
    """-> (vertices, triangles, colors, normals) or None; colours 0 and vertex_normals of the output without colours"""
    V, T = _arrays(V, T)
    keep = np.asarray(keep, bool)
    if not keep.any():
        return None
    Tk = T[keep]
    used = np.zeros(len(V), bool)
    used[Tk.reshape(-1)] = True
    remap = np.cumsum(used) - 1
    Vo, To = V[used], remap[Tk].astype(np.int32)
    if colors is None:
        return Vo, To, np.zeros_like(Vo), vertex_normals(Vo, To)
    return Vo, To, np.asarray(colors, F32)[used], np.asarray(normals, F32)[used]


def remove_small_components(V, T, min_area, colors=None, normals=None):
    labels, _, area = connected_components(V, T)
    return submesh(V, T, area[labels] >= min_area, colors, normals)


def cull(V, T, poses, intr, W, H, depths=None, tol=0.05, near=0.0, far=np.inf, colors=None, normals=None):
    V, T = _arrays(V, T)
    _check_finite(V, T)
    seen = visible(V, poses, intr, W, H, depths, tol, near, far)
    return submesh(V, T, seen[T].any(1), colors, normals)


def cell_keys(V, voxel):
    """-> packed lattice keys [V] uint64 of floor(p / voxel) (EMPTY outside the key range)"""
    q = np.floor(np.asarray(V, F32).astype(np.float64) / np.float64(F32(voxel)))
    ok = np.all((q >= -BIAS) & (q < BIAS), axis=1)
    qi = np.where(ok[:, None], q, 0).astype(np.int64) + BIAS
    keys = (qi[:, 0].astype(np.uint64) | (qi[:, 1].astype(np.uint64) << np.uint64(21)) |
            (qi[:, 2].astype(np.uint64) << np.uint64(42)))
    return np.where(ok, keys, EMPTY)


def simplify_vertex_clustering(V, T, voxel, colors=None):
    """-> (vertices, triangles, colors, normals) or None"""
    with np.errstate(over="ignore"):
        v32 = F32(voxel)
    if not (np.isfinite(v32) and v32 > 0):
        raise ValueError("voxel_size must be positive and finite")
    V, T = _arrays(V, T)
    _check_finite(V, T)
    if len(T) == 0:
        return None
    used = np.zeros(len(V), bool)
    used[T.reshape(-1)] = True
    keys = np.full(len(V), EMPTY)
    keys[used] = cell_keys(V[used], v32)
    cells = np.unique(keys[keys != EMPTY])                     # ascending key order
    cell_of = np.full(len(V), -1, np.int64)
    has = keys != EMPTY
    cell_of[has] = np.searchsorted(cells, keys[has])
    tc = cell_of[T]
    valid = np.all(tc >= 0, axis=1) & (tc[:, 0] != tc[:, 1]) & (tc[:, 1] != tc[:, 2]) & (tc[:, 0] != tc[:, 2])
    keep = np.zeros(len(T), bool)
    idx = np.flatnonzero(valid)
    if len(idx):
        _, first = np.unique(np.sort(tc[idx], axis=1), axis=0, return_index=True)
        keep[idx[first]] = True
    if not keep.any():
        return None
    referenced = np.zeros(len(cells), bool)
    referenced[tc[keep].reshape(-1)] = True
    out_of = np.cumsum(referenced) - 1
    P = V.astype(np.float64)
    C = np.zeros_like(P) if colors is None else np.asarray(colors, F32).astype(np.float64)
    sp, sc = np.zeros((len(cells), 3)), np.zeros((len(cells), 3))
    order = np.flatnonzero(has)                                # vertex order
    np.add.at(sp, cell_of[order], P[order])
    np.add.at(sc, cell_of[order], C[order])
    n = np.bincount(cell_of[order], minlength=len(cells)).astype(np.float64)
    Vo = (sp / n[:, None])[referenced].astype(F32)
    Co = (sc / n[:, None])[referenced].astype(F32)
    To = out_of[tc[keep]].astype(np.int32)
    return Vo, To, Co, vertex_normals(Vo, To)
