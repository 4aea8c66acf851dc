"""Factor-graph management (SURVEY.md §8 row A18) shared by the live front end (frontend.RaftVisualFrontend) and
its reference-API twin (droid.FactorGraph): the edge list, the candidate edges of add_neighborhood_factors, the
order-sensitive proximity edge selection of add_proximity_factors (reference
slam/visual_frontends/visual_frontend.py:711-775) and the GraphAgg tables of an edge set.
Edge lists are control data and live on the host; per-edge tensors are gathered with integer indices built there
(boolean device masks would synchronise).  The proximity distances come from the device (`frame_distance` kernel);
the selection runs on the host copy, like the reference, but with the non-maximum suppression vectorised over edges
instead of three nested Python loops per edge."""
import numpy as np
import torch

from . import _lib


def _cat(a, b):
    return b if a is None else torch.cat([a, b], 0)


def _take(a, idx):
    return None if a is None else a.index_select(0, idx)


class EdgeList:
    """The edges of a factor graph (add_factors / rm_factors / rm_keyframe: networks/factor_graph.py:43-198,
    visual_frontend.py:530-574,807-907); a new EdgeList is an empty graph.

    Active edges: host int64 `ii`, `jj`, `age`, `slots` (correlation-pool slot; 0 where the owner keeps no volumes)
    and device tensors `net` (GRU hidden state [E,ht,wd,128] channels-last), `inp` (GRU input, same layout; only
    FactorGraph keeps it per edge), `flow`, `weight` ([E,ht,wd,2] fp32).  `net` / `inp` are None until the first
    edge arrives.  Stored inactive edges: `ii_inac`, `jj_inac` with the `flow_inac` / `weight_inac` they had when
    retired.  Bad edges `ii_bad`, `jj_bad` only suppress proximity candidates.  Device copies of the index lists are
    the owner's: the live front end uploads them eagerly, FactorGraph lazily.  Edge-set changes replace the host arrays
    with new ones, except the index shift of remove_keyframe; `slots` is never written in place."""

    def __init__(self, device, ht, wd):
        z = lambda: np.zeros(0, np.int64)
        e = lambda: torch.zeros(0, ht, wd, 2, device=device)
        self.device = device
        self.ii, self.jj, self.age, self.slots = z(), z(), z(), z()
        self.ii_inac, self.jj_inac, self.ii_bad, self.jj_bad = z(), z(), z(), z()
        self.net = self.inp = None
        self.flow, self.weight, self.flow_inac, self.weight_inac = e(), e(), e(), e()

    def filter_repeated(self, ii, jj):
        """drop candidates that are already active or stored as inactive (duplicates INSIDE the candidate list are
        kept, as in the reference: factor_graph.py:43-54, visual_frontend.py:896-907); membership on (i, j) packed
        into one integer"""
        have = np.concatenate([self.ii * 65536 + self.jj, self.ii_inac * 65536 + self.jj_inac])
        keep = ~np.isin(ii * 65536 + jj, have)
        return ii[keep], jj[keep]

    def retire_mask(self, n, max_factors):
        """active edges add_factors retires to make room for `n` new ones (all False when there is room).
        The cut is applied to argsort(age) (ties in index order, as torch's CPU sort yields) and the resulting mask
        POSITIONALLY to the edges — the reference's own quirk (factor_graph.py:107-108), kept."""
        if max_factors <= 0 or len(self.ii) + n <= max_factors:
            return np.zeros(len(self.ii), bool)
        return np.argsort(self.age, kind="stable") >= max_factors - n

    def append(self, ii, jj, slots, net, flow, weight, inp=None):
        """new active edges (age 0) with their slots and per-edge tensors"""
        self.ii, self.jj = np.concatenate([self.ii, ii]), np.concatenate([self.jj, jj])
        self.age = np.concatenate([self.age, np.zeros(len(ii), np.int64)])
        self.slots = np.concatenate([self.slots, slots])
        self.net, self.inp = _cat(self.net, net), _cat(self.inp, inp)
        self.flow, self.weight = torch.cat([self.flow, flow], 0), torch.cat([self.weight, weight], 0)

    def remove(self, mask, store=False):
        """drop the active edges under the host bool `mask`; with `store` they are kept as inactive edges together
        with their flow and weight.  -> the slots they held (for the owner to release)"""
        keep = ~mask
        kd = _lib.h2d(np.nonzero(keep)[0], self.device)
        if store:
            rd = _lib.h2d(np.nonzero(mask)[0], self.device)
            self.ii_inac = np.concatenate([self.ii_inac, self.ii[mask]])
            self.jj_inac = np.concatenate([self.jj_inac, self.jj[mask]])
            self.flow_inac = torch.cat([self.flow_inac, self.flow.index_select(0, rd)], 0)
            self.weight_inac = torch.cat([self.weight_inac, self.weight.index_select(0, rd)], 0)
        released = self.slots[mask]
        self.ii, self.jj, self.age, self.slots = self.ii[keep], self.jj[keep], self.age[keep], self.slots[keep]
        self.net, self.inp = _take(self.net, kd), _take(self.inp, kd)
        self.flow, self.weight = self.flow.index_select(0, kd), self.weight.index_select(0, kd)
        return released

    def remove_keyframe(self, kf):
        """keyframe `kf` leaves and the later ones move down one slot: inactive edges that touch it are dropped,
        indices above it shift in both lists (in place).  -> mask of the active edges that touch it, for remove()"""
        m = (self.ii_inac == kf) | (self.jj_inac == kf)
        self.ii_inac[self.ii_inac >= kf] -= 1
        self.jj_inac[self.jj_inac >= kf] -= 1
        if m.any():
            kd = _lib.h2d(np.nonzero(~m)[0], self.device)
            self.ii_inac, self.jj_inac = self.ii_inac[~m], self.jj_inac[~m]
            self.flow_inac = self.flow_inac.index_select(0, kd)
            self.weight_inac = self.weight_inac.index_select(0, kd)
        m = (self.ii == kf) | (self.jj == kf)
        self.ii[self.ii >= kf] -= 1
        self.jj[self.jj >= kf] -= 1
        return m

    def known(self):
        """(ii, jj) of the active, bad and stored inactive edges, in that order: the neighbourhoods the proximity
        selection suppresses first"""
        return (np.concatenate([self.ii, self.ii_bad, self.ii_inac]),
                np.concatenate([self.jj, self.jj_bad, self.jj_inac]))


def neighborhood_edges(t0, t1, radius, stereo):
    """candidate edges between the frames of [t0, t1) whose index distance is in (c, radius], c = 1 with a stereo
    rig (its (i, i) edges come from elsewhere) and 0 otherwise (factor_graph.py:305-320, visual_frontend.py:690-708)"""
    ii, jj = np.meshgrid(np.arange(t0, t1), np.arange(t0, t1), indexing="ij")
    ii, jj = ii.reshape(-1), jj.reshape(-1)
    d = np.abs(ii - jj)
    keep = (d > (1 if stereo else 0)) & (d <= radius)
    return ii[keep], jj[keep]


def agg_tables(ii_host, device):
    """GraphAgg tables of the edges with source frames `ii_host`: (ptr int32 [K+1], order int32 [E], K), the edges
    grouped by source frame (CSR over the K sorted unique sources).  Built on the host: no device sync."""
    ux, inv = np.unique(np.asarray(ii_host), return_inverse=True)
    order = np.argsort(inv, kind="stable").astype(np.int32)
    ptr = np.zeros(len(ux) + 1, np.int32)
    np.cumsum(np.bincount(inv, minlength=len(ux)), out=ptr[1:])
    return _lib.h2d(ptr, device), _lib.h2d(order, device), len(ux)


def _diamonds(nms):
    return [np.array([(di, dj) for di in range(-r, r + 1) for dj in range(-r, r + 1) if abs(di) + abs(dj) <= r],
                     dtype=np.int64).reshape(-1, 2) for r in range(nms + 1)]


def proximity_edges(d, ii, jj, ii1, jj1, kf0, kf1, t, rad, nms, thresh, max_factors, stereo):
    """The selection through the native host routine nslam_proximity_edges (csrc/ba_graph_host.cu); same arguments and
    results as proximity_edges_numpy below (the check in tests/test_cpu_graph.py)."""
    import ctypes
    lib = _lib.load(require_cuda=False)
    d = np.ascontiguousarray(d, dtype=np.float32)
    i1 = np.ascontiguousarray(ii1, dtype=np.int64).reshape(-1); j1 = np.ascontiguousarray(jj1, dtype=np.int64).reshape(-1)
    n_out = ctypes.c_int(0)
    # forced edges: <= 2 (rad + 1) + 1 per frame; the selection loop stops once the count exceeds max_factors
    cap = max(int(t) - int(kf0), 0) * (2 * int(rad) + 3) + max(int(max_factors), 0) + 8
    es = np.empty((cap, 2), np.int64)
    P = lambda a: a.ctypes.data_as(ctypes.c_void_p)
    rc = lib.nslam_proximity_edges(P(d), int(kf0), int(kf1), int(t), P(i1), P(j1), int(i1.shape[0]), int(rad), int(nms),
                                   float(thresh), int(max_factors), int(bool(stereo)), P(es), cap, ctypes.byref(n_out))
    if rc != 0:
        raise RuntimeError(f"nslam_proximity_edges failed ({rc}; {n_out.value} edges, capacity {cap})")
    return es[:n_out.value].copy()


def proximity_edges_numpy(d, ii, jj, ii1, jj1, kf0, kf1, t, rad, nms, thresh, max_factors, stereo):
    """d: fp32 distances over the meshgrid (ii, jj) = [kf0,t) x [kf1,t) (row-major), MODIFIED in place;
    ii1/jj1: existing (active + bad + inactive) edges whose neighbourhoods are suppressed first.
    Returns the selected directed edges [n,2] in the reference's order."""
    W = t - kf1
    d[(ii - rad) < jj] = np.inf
    d[d > 100] = np.inf
    dia = _diamonds(nms)

    def suppress_many(ia, ja):
        ia = np.asarray(ia, np.int64); ja = np.asarray(ja, np.int64)
        if ia.size == 0:
            return
        rr = np.clip(np.abs(ia - ja) - 2, 0, nms)
        for r in range(nms + 1):
            sel = rr == r
            if not sel.any():
                continue
            i1 = (ia[sel][:, None] + dia[r][None, :, 0]).reshape(-1)
            j1 = (ja[sel][:, None] + dia[r][None, :, 1]).reshape(-1)
            ok = (i1 >= kf0) & (i1 < t) & (j1 >= kf1) & (j1 < t)
            d[(i1[ok] - kf0) * W + (j1[ok] - kf1)] = np.inf

    suppress_many(ii1, jj1)
    es = []
    for i in range(kf0, t):
        if stereo:
            es.append((i, i))
            d[(i - kf0) * W + (i - kf1)] = np.inf
        for j in range(max(i - rad - 1, 0), i):
            es.append((i, j)); es.append((j, i))
            d[(i - kf0) * W + (j - kf1)] = np.inf          # may be a negative (wrapping) index, as in the reference
    # torch.argsort (unstable) on the reference side; ties are resolved by index order here (stable),
    # which is what torch's CPU sort yields for equal fp32 keys
    for k in np.argsort(d, kind="stable"):
        if d[k] > thresh:
            continue
        if len(es) > max_factors:
            break
        i, j = int(ii[k]), int(jj[k])
        es.append((i, j)); es.append((j, i))
        suppress_many([i], [j])
    return np.asarray(es, dtype=np.int64).reshape(-1, 2)
