"""The NeRF trainer's state-carrying kernels against tests/ngp_train_oracle.py: the occupancy refresh (mark, refresh on both
backends, partial refresh, mean and bits, two trainers on two streams), sparse Adam on the hash table and the MLP, the
table-gradient scatter of the tensor-core backward, and the sample budget of the ray sampler.

Nothing here depends on the tensor-core MLP's rounding: the refresh is compared with the forward kernel of the same
backend on the oracle's bit-exact points (the density head is shared), the scatter with an fp64 scatter of the kernel's
own encoding gradients, Adam with an fp64 step from the kernel's own state."""
import ctypes

import numpy as np
import pytest
import torch

from oracle import ngp as ongp
from tests import ngp_train_oracle as ot

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
F32 = np.float32
AABB = 4.0
H, W = 48, 64


def _L():
    from nerf_slam_b200 import _lib
    return _lib


def _testbed(seed, max_samples=1 << 16, max_rays=1 << 13):
    from nerf_slam_b200 import pyngp
    tb = pyngp.Testbed(seed=seed, max_samples=max_samples, max_rays=max_rays)
    tb.create_empty_nerf_dataset(6, 1.0, None, AABB, None)
    g = torch.Generator().manual_seed(seed)
    tb.grid_master.copy_(((torch.rand(tb.grid_master.shape, generator=g) * 2 - 1) * 0.5).to(DEV))
    tb.grid_half.copy_(tb.grid_master.half())
    tb.pack_weights()
    return tb


def _look(pos, z_axis, up=(0.0, 1.0, 0.0)):
    z = np.asarray(z_axis, np.float64); z /= np.linalg.norm(z)
    x = np.cross(np.asarray(up, np.float64), z); x /= np.linalg.norm(x)
    c2w = np.zeros((3, 4))
    c2w[:, 0], c2w[:, 1], c2w[:, 2], c2w[:, 3] = x, np.cross(z, x), z, pos
    return c2w


def _cameras(tb):
    """slots 0, 1, 3 active; slot 2 in `cams` but not active (it sees the top of the box alone); slot 3 stands outside
    the box and looks away from it"""
    tb._ensure_store(H, W)
    views = [_look((0.5, 0.5, -0.6), (0, 0, 1)), _look((1.6, 0.3, 0.5), (-1, 0, 0.2)),
             _look((0.5, 2.4, 0.5), (0, -1, 0), up=(0, 0, 1)), _look((3.5, 0.5, 0.5), (1, 0, 0))]
    for k, c2w in enumerate(views):
        tb._set_camera(k, c2w, (50.0, 50.0), (W / 2 - 0.5, H / 2 - 0.5), (W, H))
    tb._activate([0, 1, 3])
    return [0, 1, 3]


def _update(tb, n_per_cascade, seed, decay, min_thickness=0.01, backend="tcgen05"):
    L = _L()
    im = tb._images()
    L.check(L.load().nslam_ngp_update_density_grid(ctypes.byref(tb.model), ctypes.byref(im), n_per_cascade, seed, decay,
                                                   min_thickness, L.ptr(tb.packed) if backend == "tcgen05" else None,
                                                   tb.num_sms, L.stream_ptr()), "update_density_grid")


def _sigma(tb, x01, backend):
    """exp(o0) of the backend's forward kernel at x01 [n,3] float32"""
    L = _L()
    n = x01.shape[0]
    coords = torch.zeros(n, 7, device=DEV)
    coords[:, :3] = torch.from_numpy(x01).to(DEV)
    coords[:, 6] = 1.0
    out = torch.empty(n, 4, device=DEV)
    if backend == "tcgen05":
        L.check(L.load().nslam_ngp_forward_tc(ctypes.byref(tb.model), L.ptr(tb.packed), L.ptr(coords), None, n, n, L.ptr(out),
                                              None, tb.num_sms, L.stream_ptr()), "forward_tc")
    else:
        L.check(L.load().nslam_ngp_forward(ctypes.byref(tb.model), L.ptr(coords), n, L.ptr(out), L.stream_ptr()), "forward")
    return out[:, 3].cpu().numpy()


def _oracle_params(tb, dtype=torch.float64):
    P = {"grid": tb.grid_half.to(dtype).cpu().view(-1, 2)}
    w = tb.mlp.cpu().to(dtype)
    off = 0
    for name, (i, o) in dict(W1=(32, 64), W2=(64, 16), W3=(32, 64), W4=(64, 64), W5=(64, 16)).items():
        P[name] = w[off:off + i * o].view(i, o).clone(); off += i * o
    return P


@pytest.fixture(scope="module")
def occ():
    """a trainer with cameras, after a mark-only update from an all -1 grid with a few cells already >= 0"""
    tb = _testbed(21)
    active = _cameras(tb)
    g = torch.Generator().manual_seed(1)
    pre = torch.rand(tb.density.shape, generator=g)
    d0 = torch.where(pre < 0.01, pre, torch.full_like(pre, -1.0))        # 1 % of the cells start at a value >= 0
    tb.density.copy_(d0.to(DEV))
    _update(tb, 0, 7, 0.95)                                              # n = 0: mark, mean and bits only
    torch.cuda.synchronize()
    return dict(tb=tb, active=active, d0=d0.numpy(), marked=tb.density.cpu().numpy(), stats=tb.stats.cpu().numpy(),
                bits=tb.bits.cpu().numpy())


def test_mark_equals_the_visibility_rule(occ):
    """-1 -> 0 exactly where the fp64 rule says an active camera sees the cell, except cells within 1e-3 px of a
    decision boundary (140 of the 6.3 M cells of this camera set, by the oracle; allowed: 1e-4 of all cells); cells
    already >= 0 are bit-unchanged.  The inactive camera's own cells stay at -1; the camera outside the box sees none"""
    tb, d0, got = occ["tb"], occ["d0"], occ["marked"]
    pos = d0 >= 0
    assert np.array_equal(got[pos].view(np.int32), d0[pos].view(np.int32))
    assert set(np.unique(got[~pos]).tolist()) <= {-1.0, 0.0}
    cams = tb.cams_h
    excluded, newly = 0, 0
    for mip in range(tb.cascades):
        sl = slice(mip * ot.NC, (mip + 1) * ot.NC)
        vis, margin = ot.mark_slack(cams, occ["active"], mip)
        todo = ~pos[sl]
        sure = todo & (margin >= 1e-3)
        excluded += int((todo & ~sure).sum())
        assert np.array_equal(got[sl][sure] == 0.0, vis[sure]), mip
        newly += int((got[sl][todo] == 0.0).sum())
        # the camera in `cams` but not in `active` would add cells; the camera outside the box adds none
        vis2, _ = ot.mark_slack(cams, occ["active"] + [2], mip)
        extra = vis2 & ~vis & todo & (margin >= 1e-3)
        assert np.all(got[sl][extra] == -1.0)
        if mip == 0:
            assert extra.sum() > 1000
            assert not ot.mark_slack(cams, [3], mip)[0].any()
    assert excluded < 1e-4 * tb.density.numel(), excluded
    assert 0.05 * tb.density.numel() < newly < 0.9 * tb.density.numel()


@pytest.mark.parametrize("backend", ["tcgen05", "simt"])
def test_full_refresh_equals_the_rule_on_the_forward_kernels_density(occ, backend):
    """every visible cell == fmaxf(prev decay, sigma MIN_STEP s), bit for bit, with sigma from the same backend's forward
    kernel at the oracle's bit-exact points (the density head is shared); cells at -1 unchanged.  sigma within 3e-2 (tc,
    fp16 operands) / 5e-4 (simt) relative of the fp64 oracle network on 50k cells"""
    tb = occ["tb"]
    rng = np.random.default_rng(2)
    prev = occ["marked"].copy()
    vis = prev >= 0
    # half the visible cells hold a value the decay keeps above the new density, so both sides of the max are taken
    prev[vis & (rng.random(prev.size) < 0.5)] = F32(0.05)
    tb.density.copy_(torch.from_numpy(prev).to(DEV))
    seed = 1234
    _update(tb, ot.NC, seed, 0.95, backend=backend)
    idx, x01 = ot.refresh_cells(seed, ot.NC, tb.cascades, AABB)
    sigma = _sigma(tb, x01, backend)
    torch.cuda.synchronize()
    got = tb.density.cpu().numpy()
    want = ot.refresh(prev, idx, sigma, 0.95, ot.cascade_scale)
    diff = got.view(np.int32) != want.view(np.int32)
    assert not diff.any(), (int(diff.sum()), np.nonzero(diff)[0][:5], got[diff][:5], want[diff][:5])
    thick = (sigma[vis[idx]] * ot.MIN_STEP) * ot.cascade_scale(idx[vis[idx]])
    decayed = prev[idx[vis[idx]]] * F32(0.95)
    assert (thick > decayed).sum() > 1000 and (thick < decayed).sum() > 1000
    sub = np.random.default_rng(3).choice(idx.size, 50000, replace=False)
    P = _oracle_params(tb)
    d = torch.zeros(sub.size, 3, dtype=torch.float64); d[:, 2] = 1
    with torch.no_grad():
        _, ref = ongp.network(torch.from_numpy(x01[sub].astype(np.float64)), d, P, AABB)
    rel = np.abs(sigma[sub] - ref.numpy()) / ref.numpy()
    assert rel.max() < (3e-2 if backend == "tcgen05" else 5e-4), rel.max()


def test_partial_refresh_changes_exactly_the_visited_cells_and_stats_and_bits_follow(occ):
    """a quarter refresh (decay 0.95, new seed): the oracle's distinct cells take the rule's value, every other cell is
    bit-unchanged (no decay outside the visited cells: see the oracle).  Then stats[1] is the exact count of cells >= 0,
    stats[0] the fp64 sum of the kernel's own array within 1e-5 relative (fp32 partial sums of 592 fixed blocks), and the
    bits equal the threshold rule away from the threshold (1e-3 relative), for both sides of min(min_thickness, mean)"""
    tb = occ["tb"]
    tb.density.copy_(torch.from_numpy(occ["marked"]).to(DEV))
    _update(tb, ot.NC, 99, 0.95)
    torch.cuda.synchronize()
    prev = tb.density.cpu().numpy()
    seed = 4242
    _update(tb, ot.NC // 4, seed, 0.95)
    idx, x01 = ot.refresh_cells(seed, ot.NC // 4, tb.cascades, AABB)
    sigma = _sigma(tb, x01, "tcgen05")
    torch.cuda.synchronize()
    got = tb.density.cpu().numpy()
    want = ot.refresh(prev, idx, sigma, 0.95, ot.cascade_scale)
    assert np.array_equal(got.view(np.int32), want.view(np.int32))
    changed = np.nonzero(got.view(np.int32) != prev.view(np.int32))[0]
    visited = np.sort(idx[prev[idx] >= 0])
    # a visited cell keeps its bits only when its new density rounds to its old one (1 of 967 292 cells in the first
    # run on an H100); the values themselves were checked bit for bit above
    assert np.isin(changed, visited).all() and changed.size >= visited.size - 10
    mean = float(tb.stats[0] / tb.stats[1])
    for min_thick in (0.01, 0.5 * mean, 2.0 * mean):                    # both sides of min(min_thickness, mean)
        if min_thick != 0.01:
            _update(tb, 0, seed, 0.95, min_thickness=min_thick)          # n = 0: mark (a no-op now), mean and bits
        torch.cuda.synchronize()
        dens = tb.density.cpu().numpy()
        stats, bits = tb.stats.cpu().numpy(), tb.bits.cpu().numpy()
        assert stats[1] == float((dens >= 0).sum())
        s64 = dens[dens >= 0].astype(np.float64).sum()
        assert abs(float(stats[0]) - s64) <= 1e-5 * s64, (stats[0], s64)
        thr = ot.threshold(stats, min_thick)
        assert thr == (F32(min_thick) if min_thick < mean else F32(stats[0]) / F32(stats[1]))
        want_bits = np.unpackbits(ot.pack_bits(dens, thr), bitorder="little")
        got_bits = np.unpackbits(bits, bitorder="little")
        far = np.abs(dens.astype(np.float64) - float(thr)) > 1e-3 * float(thr)
        assert np.array_equal(got_bits[far], want_bits[far])
        assert 1e-3 < got_bits.mean() < 0.9


def test_two_trainers_refresh_on_two_streams_as_they_do_alone():
    """the refresh's mean reduction uses the trainer's own partials buffer: two trainers refreshing concurrently on two
    streams produce, each, the density, stats and bits of its solo run, bit for bit"""
    tbs = [_testbed(31), _testbed(32)]
    for tb in tbs:
        _cameras(tb)
    start = []
    for k, tb in enumerate(tbs):
        tb.density.fill_(-1.0)
        _update(tb, 0, 5 + k, 0.95)
        torch.cuda.synchronize()
        start.append(tb.density.clone())

    solo = []
    for k, tb in enumerate(tbs):
        tb.density.copy_(start[k])
        _update(tb, ot.NC, 50 + k, 0.95)
        _update(tb, ot.NC // 4, 60 + k, 0.95)
        torch.cuda.synchronize()
        solo.append((tb.density.clone(), tb.stats.clone(), tb.bits.clone()))
    for k, tb in enumerate(tbs):
        tb.density.copy_(start[k]); tb.stats.zero_(); tb.bits.zero_()
    torch.cuda.synchronize()
    streams = [torch.cuda.Stream(), torch.cuda.Stream()]
    for phase in range(2):                               # interleave the launches of the two trainers
        for k, tb in enumerate(tbs):
            with torch.cuda.stream(streams[k]):
                if phase == 0:
                    _update(tb, ot.NC, 50 + k, 0.95)
                else:
                    _update(tb, ot.NC // 4, 60 + k, 0.95)
    torch.cuda.synchronize()
    for k, tb in enumerate(tbs):
        for a, b in zip((tb.density, tb.stats, tb.bits), solo[k]):
            assert torch.equal(a, b), k
    assert not torch.equal(solo[0][1], solo[1][1])


def _adam_check(before, after, step, lr, b1, b2, eps, l2, sparse):
    """after == one Adam step of `before` to 4 ulp of each update's largest term; untouched state bit-unchanged"""
    w, g, m, v = (before[k] for k in ("w", "g", "m", "v"))
    o = ot.adam(w, g, m, v, step, lr, b1, b2, eps, l2, sparse)
    u = o["updated"]
    for k, scale in (("m", "m_scale"), ("v", "v_scale")):
        err = np.abs(after[k][u].astype(np.float64) - o[k][u])
        assert np.all(err <= 4 * ot.ulp32(o[scale][u])), (k, float((err / ot.ulp32(o[scale][u])).max()))
    # the weight from the moments the kernel holds (their own rounding is checked above)
    ow = ot.adam(w, g, m, v, step, lr, b1, b2, eps, l2, sparse, m_new=after["m"], v_new=after["v"])
    err = np.abs(after["w"][u].astype(np.float64) - ow["w"][u])
    assert np.all(err <= 4 * ot.ulp32(ow["w_scale"][u])), float((err / ot.ulp32(ow["w_scale"][u])).max())
    for k in ("w", "m", "v"):
        assert np.array_equal(after[k][~u].view(np.int32), before[k][~u].view(np.int32)), k
    assert not after["g"].any()
    if sparse:
        unwritten = ~o["written"]
        assert np.array_equal(after["g"][unwritten].view(np.int32), before["g"][unwritten].view(np.int32))
    return int(u.sum())


def test_sparse_grid_adam_and_mlp_adam_with_l2_match_the_oracle():
    """three steps of nslam_ngp_adam over the whole table (6.4 M slots) and the MLP (l2 = 1e-6, the product's value).
    The table gradient changes between steps and mixes all-zero, partially zero (some -0.0) and full float4 groups, on
    top of nonzero moments.  Bound: 4 ulp of the update's largest term (m: 1.5 roundings of the larger of b1 m and
    (1 - b1) grad; v: 3 roundings of the positive sum; w: 3.5 roundings of the larger of w and the step)"""
    L = _L()
    tb = _testbed(41)
    rng = np.random.default_rng(9)
    n = tb.grid_master.numel()
    tb.grid_m.copy_(torch.from_numpy((rng.standard_normal(n) * 1e-3).astype(F32)).to(DEV))
    tb.grid_v.copy_(torch.from_numpy((rng.random(n) * 1e-5).astype(F32)).to(DEV))
    tb.mlp_m.copy_(torch.from_numpy((rng.standard_normal(10240) * 1e-3).astype(F32)).to(DEV))
    tb.mlp_v.copy_(torch.from_numpy((rng.random(10240) * 1e-5).astype(F32)).to(DEV))
    lr, b1, b2, eps, l2 = 1e-2, 0.9, 0.99, 1e-15, 1e-6
    counts = []
    for step in range(1, 4):
        cls = rng.random(n // 4)
        g = (rng.standard_normal(n) * 10.0 ** rng.uniform(-4, -1, n)).astype(F32)
        mask = np.repeat(cls < 0.4, 4) | (np.repeat((cls >= 0.4) & (cls < 0.7), 4) & (rng.random(n) < 0.5))
        g[mask] = 0.0
        g[mask & (rng.random(n) < 0.1)] = -0.0
        gm = rng.standard_normal(10240).astype(F32) * F32(1e-2)
        gm[rng.random(10240) < 0.2] = 0.0
        tb.grid_grad.copy_(torch.from_numpy(g).to(DEV)); tb.mlp_grad.copy_(torch.from_numpy(gm).to(DEV))
        snap = lambda: dict(grid=dict(w=tb.grid_master.cpu().numpy(), g=tb.grid_grad.cpu().numpy(), m=tb.grid_m.cpu().numpy(),
                                      v=tb.grid_v.cpu().numpy(), half=tb.grid_half.cpu().numpy()),
                            mlp=dict(w=tb.mlp.cpu().numpy(), g=tb.mlp_grad.cpu().numpy(), m=tb.mlp_m.cpu().numpy(),
                                     v=tb.mlp_v.cpu().numpy()))
        before = snap()
        L.check(L.load().nslam_ngp_adam(ctypes.byref(tb.model), step, lr, b1, b2, eps, l2, L.stream_ptr()), "adam")
        torch.cuda.synchronize()
        after = snap()
        counts.append(_adam_check(before["grid"], after["grid"], step, lr, b1, b2, eps, 0.0, sparse=True))
        assert _adam_check(before["mlp"], after["mlp"], step, lr, b1, b2, eps, l2, sparse=False) == 10240
        half = after["grid"]["half"]
        assert np.array_equal(half.view(np.uint16), after["grid"]["w"].astype(np.float16).view(np.uint16))
    assert all(0.2 * n < c < 0.6 * n for c in counts), counts


# ------------------------------------------------------------------------------------------ table scatter
def _scatter_batches():
    """name -> (x [n,3] float32, per-ray counts).  The existing R = 24 / 300 batches, single rays of 1, 31, 33 samples,
    1000 samples on 8 rays in steps of 1e-4 (long runs in one cell on the coarse levels), alternating A, B, A, B cells,
    and the lattice's edges (nodes, faces, 0 and 1, a hashed collision pair) repeated into runs"""
    g = torch.Generator().manual_seed(1)
    out = {"R24": ((torch.rand(24 * 11, 3, generator=g) * 0.6 + 0.2).numpy(), [11] * 24),
           "R300": ((torch.rand(300 * 13, 3, generator=g) * 0.6 + 0.2).numpy(), [13] * 300)}
    rng = np.random.default_rng(2)
    for n in (1, 31, 33):
        out[f"n{n}"] = (rng.random((n, 3)) * 0.6 + 0.2, [n])
    o = rng.random((8, 1, 3)) * 0.4 + 0.3
    d = rng.standard_normal((8, 1, 3)); d /= np.linalg.norm(d, axis=-1, keepdims=True)
    out["runs1000"] = ((o + d * 1e-4 * np.arange(125)[None, :, None]).reshape(-1, 3), [125] * 8)
    a, b = np.array([0.31, 0.52, 0.47]), np.array([0.71, 0.22, 0.64])
    out["alternate"] = (np.where((np.arange(96) % 2 == 0)[:, None], a, b), [48, 48])
    e = ot.edge_points(AABB, kernel_rounding=True)
    out["edges"] = (np.repeat(e, 3, axis=0), [3 * len(e)])
    return {k: (np.asarray(x, F32), c) for k, (x, c) in out.items()}


def _run_backward(tb, x, counts, prefill, seed):
    L = _L()
    g = torch.Generator().manual_seed(seed)
    n, R = x.shape[0], len(counts)
    off = np.concatenate([[0], np.cumsum(counts)[:-1]])
    d = torch.nn.functional.normalize(torch.randn(R, 3, generator=g), dim=-1).repeat_interleave(torch.tensor(counts), 0)
    dt = torch.full((n,), 0.004)
    tdist = torch.cat([torch.arange(c).float() * 0.004 + 0.3 for c in counts])
    coords = torch.cat([torch.from_numpy(x), dt[:, None], d], -1).contiguous()
    rays = torch.zeros(R, 16)
    rays[:, 6] = 0.9
    tgt_rgb = torch.rand(R, 3, generator=g); tgt_dep = torch.rand(R, generator=g) * 0.5 + 0.2; cov = torch.rand(R, generator=g) * 0.5 + 0.1
    rays[:, 7], rays[:, 8], rays[:, 9:12] = tgt_dep, cov, tgt_rgb
    ri = rays.view(torch.int32)
    ri[:, 12] = torch.from_numpy(off.astype(np.int32)); ri[:, 13] = torch.tensor(counts, dtype=torch.int32)
    tb._bufs["rays"][:R].copy_(rays.to(DEV)); tb._bufs["coords"][:n].copy_(coords.to(DEV)); tb._bufs["tdist"][:n].copy_(tdist.to(DEV))
    bg = (0.2, 0.4, 0.6)
    results = []
    for _ in range(2):
        tb.grid_grad.copy_(prefill)
        L.check(L.load().nslam_ngp_loss_backward_tc(ctypes.byref(tb.model), ctypes.byref(tb.batch), L.ptr(tb.packed), R, n,
                                                    1.0, *bg, 1024.0, tb.num_sms, L.stream_ptr()), "loss_bwd_tc")
        torch.cuda.synchronize()
        results.append(tb.grid_grad.cpu().numpy())
        assert not tb.grid_grad_fx.any()
    assert np.array_equal(results[0].view(np.int32), results[1].view(np.int32))
    return results[0], tb._bufs["denc"][:n].cpu().numpy(), dict(d=d, dt=dt, tdist=tdist, off=off, tgt_rgb=tgt_rgb,
                                                                tgt_dep=tgt_dep, cov=cov, bg=bg)


def test_table_scatter_equals_the_fp64_scatter_of_the_kernels_encoding_gradients():
    """nslam_ngp_loss_backward_tc on a prefilled grid_grad == prefill + scatter(denc / loss_scale) in fp64 from the
    kernel's own denc, per entry within 1e-6 sum|contributions| (fp32 weights and run sums: < 6e-7) + 2^-23 |result|
    (the final fp32 add) + 2^-40 per contributing sample (the fixed-point rounding of each run); entries that receive
    nothing keep the prefill bit for bit; grid_grad_fx is zero on return; a second call gives the same bits.
    The direction of denc against autograd through oracle/ngp.py is the only check that touches the MLP's rounding:
    the smallest cosine measured over these batches on an H100 was 0.999929 (R300), so 1 - cos < 3e-4 keeps 4x headroom."""
    tb = _testbed(51)
    tb.mlp.mul_(0.5)
    tb.pack_weights()
    nt = tb.grid_grad.numel()
    prefill = ((torch.arange(nt, dtype=torch.int64) % 7 - 3).float() * 1e-4).to(DEV)
    pre = prefill.cpu().numpy()
    cos_min = 1.0
    for k, (name, (x, counts)) in enumerate(_scatter_batches().items()):
        got, denc, ctx = _run_backward(tb, x, counts, prefill, 100 + k)
        g = denc.astype(np.float64) / 1024.0
        ref, mag, cnt = ot.scatter(x, g, AABB, kernel_rounding=True)
        ref, mag = ref.reshape(-1), mag.reshape(-1)
        cnt2 = np.repeat(cnt, 2)
        want = pre.astype(np.float64) + ref
        err = np.abs(got.astype(np.float64) - want)
        bound = 1e-6 * mag + 2.0 ** -23 * np.abs(want) + cnt2 * 2.0 ** -40
        assert np.all(err <= bound), (name, float((err / bound).max()))
        none = mag == 0
        assert np.array_equal(got[none].view(np.int32), pre[none].view(np.int32)), name
        assert (~none).sum() >= 2 * 8 and np.abs(g).max() > 0, name
        # direction of the encoding gradients against autograd of the fp32 oracle
        P = _oracle_params(tb, torch.float32)
        enc = ongp.hash_encode(torch.from_numpy(x), P["grid"], AABB).detach().requires_grad_(True)
        rgb, sigma = ot.network_from_enc(enc, ctx["d"], P)
        ptr = list(ctx["off"]) + [len(x)]
        loss, _, _ = ongp.composite_loss(rgb, sigma, ctx["dt"], ctx["tdist"] * 0.9, ptr, ctx["tgt_rgb"], ctx["tgt_dep"],
                                         ctx["cov"], torch.tensor(ctx["bg"]).repeat(len(counts), 1), 1.0)
        loss.backward()
        a, b = enc.grad.double().numpy().reshape(-1), g.reshape(-1)
        cos = float(a @ b / (np.linalg.norm(a) * np.linalg.norm(b)))
        cos_min = min(cos_min, cos)
    assert cos_min > 1 - 3e-4, cos_min


# ------------------------------------------------------------------------------------------ sample budget
def _sample(tb, R, seed, cap=None):
    L = _L()
    tb.batch.max_samples = tb.max_samples if cap is None else cap
    tb._bufs["coords"].fill_(float("nan"))
    tb._bufs["rays"].zero_()
    im = tb._images()
    L.check(L.load().nslam_ngp_sample_phase(ctypes.byref(tb.model), ctypes.byref(im), ctypes.byref(tb.batch), R, seed,
                                            L.stream_ptr()), "sample")
    torch.cuda.synchronize()
    rays = tb._bufs["rays"][:R].cpu()
    ri = rays.view(torch.int32).numpy()
    return rays.numpy(), ri[:, 12].astype(np.int64), ri[:, 13].astype(np.int64), tb._bufs["counters"].cpu().numpy()[:2], \
        tb._bufs["coords"].cpu().numpy()


def _budget_tb(max_samples, bits):
    tb = _testbed(61, max_samples=max_samples, max_rays=2048)
    tb._ensure_store(H, W)
    c2w = np.eye(4)[:3].copy(); c2w[:, 3] = [0.5, 0.5, -0.4]
    tb._set_camera(0, c2w, (40.0, 40.0), (W / 2 - 0.5, H / 2 - 0.5), (W, H))
    tb._activate([0])
    tb.bits.copy_(bits)
    return tb


def _check_budget(R12, R13, ctr, coords, cap, last_count=None):
    """the kept set, offsets and counters follow the prefix rule; counts recovered from the exclusive offsets (the last
    ray's from R[13] when it is kept, else from `last_count`; unknown, the rule is checked on the other rays)"""
    counts = R12[1:] - R12[:-1]
    if R13[-1] > 0 or last_count is not None:
        counts = np.append(counts, R13[-1] if R13[-1] > 0 else last_count)
    b = ot.sample_budget(counts, cap)
    k = len(counts)
    assert np.array_equal(R12[:k], b["offset"]) and np.array_equal(R13[:k], b["n"])
    if k < len(R12):
        assert R13[-1] == 0 and R12[-1] == counts.sum()
    assert tuple(int(v) for v in ctr) == b["counters"]
    used = int(ctr[0])
    assert np.isfinite(coords[:used]).all() and np.isnan(coords[used:]).all()
    return counts


def test_sample_budget_follows_the_prefix_rule():
    """sample_rays / sample_scan with the batch over the budget (the trainer's steady state): Testbed(max_samples=4096),
    a 30 % occupied bitfield.  The kept rays, R[12] / R[13] and counters[0..1] follow the prefix rule of the oracle,
    per-ray counts equal oracle/ngp.py::march_lattice on 64 rays, rows past counters[0] keep their NaN sentinel.  Again
    with max_samples an exact prefix sum, and with R = 1500 (the scan carries across its 1024-ray chunks) cut inside
    the second chunk"""
    g = torch.Generator().manual_seed(7)
    ncell = 3 * ot.NC
    bits = torch.from_numpy(np.packbits((torch.rand(ncell, generator=g) < 0.3).numpy(), bitorder="little")).to(DEV)
    small, big = _budget_tb(4096, bits), _budget_tb(1 << 19, bits)
    seed, R = 777, 96
    # all 96 rays fit the big buffer: their records give the per-ray counts and rays to check against the march
    rays_b, R12b, R13b, ctr_b, _ = _sample(big, R, seed)
    assert ctr_b[1] == (R13b > 0).sum() and R13b.sum() > 4096 * 2
    lo, hi = 0.5 - 0.5 * AABB, 0.5 + 0.5 * AABB
    for i in np.nonzero(R13b > 0)[0][:64]:
        ref = ongp.march_lattice(rays_b[i, 0:3], rays_b[i, 3:6], lo, hi, big.nerf.training.near_distance, 1.0 / 256,
                                 big.cascades, bits.cpu().numpy(), float(ongp.rnd01(seed, int(i), 4)), 1024)
        assert len(ref) == R13b[i], i
    counts = R13b
    _, R12, R13, ctr, coords = _sample(small, R, seed)
    assert np.array_equal(_check_budget(R12, R13, ctr, coords, 4096, counts[-1]), counts)
    assert 0 < ctr[1] < (counts > 0).sum()
    # an exact fit: the budget equals the inclusive sum of a ray in the middle
    k = int(np.nonzero(counts > 0)[0][5])
    cap = int(np.cumsum(counts)[k])
    _, R12, R13, ctr, coords = _sample(small, R, seed, cap)
    _check_budget(R12, R13, ctr, coords, cap, counts[-1])
    assert ctr[0] == cap and R13[k] == counts[k]
    # R = 1500: first the counts (budget = the whole buffer), then a budget ending inside the second chunk
    R = 1500
    _, R12, R13, ctr, coords = _sample(big, R, seed + 1)
    counts = _check_budget(R12, R13, ctr, coords, big.max_samples)
    fits = np.nonzero((counts[1024:1400] > 0) & (np.cumsum(counts)[1024:1400] <= big.max_samples))[0]
    assert fits.size, np.cumsum(counts)[1024]
    k = 1024 + int(fits[len(fits) // 2])
    cap = int(np.cumsum(counts)[k])
    _, R12, R13, ctr, coords = _sample(big, R, seed + 1, cap)
    _check_budget(R12, R13, ctr, coords, cap)
    assert ctr[0] == cap and ctr[1] == (counts[:k + 1] > 0).sum()
