"""Self-checks of tests/ngp_train_oracle.py (no device): the refresh's cell permutation, the scatter rule against autograd
through oracle.ngp.hash_encode at the edges of the lattice, the Adam rule against torch.optim.Adam, the sample-budget
prefix rule on crafted counts."""
from fractions import Fraction

import numpy as np
import torch

from oracle import ngp as ongp
from tests import ngp_train_oracle as ot

F32 = np.float32
AABB = 4.0


def test_density_cell_is_a_bijection_and_a_quarter_refresh_hits_distinct_cells():
    j = np.arange(ot.NC)
    for seed in (0, 1, 1337 * 7919 + 16, 0xFFFFFFFF):
        for mip in range(3):
            cells = ot.density_cell(seed, mip, j)
            assert cells.min() == 0 and cells.max() == ot.NC - 1
            assert np.unique(cells).size == ot.NC, (seed, mip)
        idx, _ = ot.refresh_cells(seed, ot.NC // 4, 3, AABB)
        assert idx.size == 3 * ot.NC // 4 and np.unique(idx).size == idx.size
        assert np.array_equal(idx // ot.NC, np.repeat(np.arange(3), ot.NC // 4))
    # different seeds visit different quarters
    a, _ = ot.refresh_cells(5, ot.NC // 4, 1, AABB)
    b, _ = ot.refresh_cells(6, ot.NC // 4, 1, AABB)
    assert 0.1 < np.intersect1d(a, b).size / a.size < 0.4


def test_refresh_points_match_the_scalar_rng_and_lie_in_their_cells():
    seed = 91
    for i in (0, 1, 77, 2 ** 21 - 1, 3 * 2 ** 21 - 5):
        for c in (11, 12, 13):
            assert ot.rnd01(seed, np.array([i]), c)[0] == ongp.rnd01(seed, i, c)
    ps = ot.pcg(np.uint64(seed))
    for mip in range(3):
        a = ongp.pcg(int(ps) ^ (2 * mip)) | 1
        b = ongp.pcg(int(ps) ^ (2 * mip + 1))
        assert ot.density_cell(seed, mip, np.array([12345]))[0] == (a * 12345 + b) % ot.NC
    for n in (ot.NC, ot.NC // 4):
        idx, x01 = ot.refresh_cells(seed, n, 3, AABB)
        p = x01.astype(np.float64) * AABB + (0.5 - 0.5 * AABB)
        mip = idx // ot.NC
        s = 2.0 ** mip
        u = ((p - 0.5) / s[:, None] + 0.5) * ot.GRID                   # position in cells of the cascade
        c = idx % ot.NC
        ijk = np.stack([c % ot.GRID, (c // ot.GRID) % ot.GRID, c // (ot.GRID * ot.GRID)], -1)
        # inside the closed cell: ix + jitter rounds up to ix + 1 in fp32 for jitter within 2^-24 ix of 1 (190 of
        # the 6.3 M points of this full refresh sit on the upper face)
        assert np.all((u >= ijk) & (u <= ijk + 1))
        assert np.mean(np.floor(u) == ijk) > 1 - 1e-4


def test_fma32_rounds_once():
    rng = np.random.default_rng(0)
    a = rng.random(2000).astype(F32) * F32(3000)
    b = np.full_like(a, F32(1234.5677))
    c = np.full_like(a, F32(0.5))
    # ties: a b just off a float32 midpoint of the sum, which a two-step rounding would get wrong
    t = np.array([F32(1.0) + F32(2.0 ** -23)], F32)
    a = np.concatenate([a, t, np.array([F32(2.0 ** -30), F32(0.0), F32(1.0)], F32)])
    b = np.concatenate([b, np.array([F32(1.0) + F32(2.0 ** -23)], F32), np.array([F32(1.5), F32(7.0), F32(2.0 ** -24) * F32(1.5)], F32)])
    c = np.concatenate([c, np.array([F32(-1.0)], F32), np.array([F32(0.5), F32(0.5), F32(1.0)], F32)])
    got = ot.fma32(a, b, c)
    for x, y, z, r in zip(a, b, c, got):
        exact = Fraction(float(x)) * Fraction(float(y)) + Fraction(float(z))
        lo = F32(float(exact))
        cand = [np.nextafter(lo, F32(-np.inf)), lo, np.nextafter(lo, F32(np.inf))]
        err = [abs(Fraction(float(v)) - exact) for v in cand]
        best = min(err)
        assert abs(Fraction(float(r)) - exact) == best, (x, y, z, r)


def test_hashed_collision_pair_shares_an_entry():
    l, ca, cb = ot.hashed_collision(AABB)
    lv, _ = ongp.level_params(AABB)
    _, res, n, _ = lv[l]
    assert res ** 3 > n and not np.array_equal(ca, cb)
    assert ongp.grid_index(*[int(v) for v in ca], res, n) == ongp.grid_index(*[int(v) for v in cb], res, n)
    x = np.stack([ot.point_in_cell(ca, 0.25, AABB, l), ot.point_in_cell(cb, 0.25, AABB, l)])
    idx, _, cell = ot.corners(x, AABB, l)
    assert np.array_equal(cell[0, 0], ca) and np.array_equal(cell[1, 0], cb) and idx[0, 0] == idx[1, 0]


def test_scatter_oracle_equals_autograd_through_hash_encode():
    rng = np.random.default_rng(3)
    edge = ot.edge_points(AABB, kernel_rounding=False)
    x = np.concatenate([rng.random((300, 3)).astype(F32), edge]).astype(F32)
    assert x.min() >= 0 and x.max() <= 1
    G = rng.standard_normal((x.shape[0], 32))
    _, total = ongp.level_params(AABB)
    grid = torch.zeros(total, 2, dtype=torch.float64, requires_grad=True)
    enc = ongp.hash_encode(torch.from_numpy(x), grid, AABB)
    (enc * torch.from_numpy(G)).sum().backward()
    ref = grid.grad.numpy()
    got, mag, _ = ot.scatter(x, G, AABB, kernel_rounding=False)
    # hash_encode rounds the trilinear weights to fp32 (two products: < 2^-23 relative); the oracle keeps them in fp64
    err = np.abs(got - ref)
    assert np.all(err <= 1e-6 * mag), float((err / np.maximum(mag, 1e-300)).max())
    assert np.array_equal(got != 0, ref != 0)
    # the dense levels wrap at x = 1: the corner past the last lattice point lands on entry (res + ...) % size
    lv, _ = ongp.level_params(AABB)
    scale, res, n, _ = lv[0]
    idx, w, cell = ot.corners(np.ones((1, 3), F32), AABB, 0)
    assert cell.max() >= res - 1 and np.all(idx < n)
    # the kernel rounds pos = x scale + 0.5 once (fmaf), hash_encode twice: the weights differ by up to one fp32 ulp of
    # pos (5e-4 on the finest level), the corners only where pos is within that ulp of an integer -- not for these points
    for l in range(16):
        assert np.array_equal(ot.corners(x[:300], AABB, l, True)[0], ot.corners(x[:300], AABB, l, False)[0])


def test_adam_oracle_with_dense_gradient_equals_torch_adam():
    rng = np.random.default_rng(4)
    n = 4096
    lr, b1, b2, eps, l2 = (float(F32(v)) for v in (1e-2, 0.9, 0.99, 1e-15, 1e-6))
    w = rng.standard_normal(n) * 0.5
    p = torch.nn.Parameter(torch.from_numpy(w.copy()))
    opt = torch.optim.Adam([p], lr=lr, betas=(b1, b2), eps=eps, weight_decay=l2)
    m, v = np.zeros(n), np.zeros(n)
    for step in range(1, 4):
        g = rng.standard_normal(n) * 1e-2
        g[rng.random(n) < 0.2] = 0.0                     # dense rule: zero gradients still take the L2 term
        p.grad = torch.from_numpy(g.copy())
        opt.step()
        w_prev, m_prev, v_prev = w, m, v
        o = ot.adam(w, g, m, v, step, lr, b1, b2, eps, l2, sparse=False)
        w, m, v = o["w"], o["m"], o["v"]
        st = opt.state[p]
        # torch updates the moments by lerp (fp64 roundings apart, the same numbers); the oracle takes the bias
        # corrections in fp32 as the host does (2^-23 relative: 2e-9 on steps of 1e-2).  The L2 term alone moves the
        # steps by 5e-7, so 1e-8 still tells the rules apart
        assert np.allclose(m, st["exp_avg"].numpy(), rtol=1e-9, atol=1e-15)
        assert np.allclose(v, st["exp_avg_sq"].numpy(), rtol=1e-9, atol=1e-18)
        assert np.allclose(w, p.detach().numpy(), rtol=0, atol=1e-8)
        without_l2 = ot.adam(w_prev, g, m_prev, v_prev, step, lr, b1, b2, eps, 0.0, sparse=False)["w"]
        assert np.abs(without_l2 - w).max() > 1e-7


def test_sparse_adam_oracle_keeps_untouched_state():
    rng = np.random.default_rng(5)
    n = 64
    w, m, v = rng.standard_normal(n), rng.standard_normal(n) * 1e-3, rng.random(n) * 1e-5
    g = rng.standard_normal(n)
    g[0:4] = 0.0                                          # an all-zero group
    g[5] = 0.0; g[6] = -0.0                               # a partially zero group (-0 is zero)
    o = ot.adam(w, g, m, v, 2, 1e-2, 0.9, 0.99, 1e-15, 0.0, sparse=True)
    keep = np.zeros(n, bool); keep[[0, 1, 2, 3, 5, 6]] = True
    for k in ("w", "m", "v"):
        assert np.array_equal(o[k][keep], {"w": w, "m": m, "v": v}[k][keep])
        assert np.all(o[k][~keep] != {"w": w, "m": m, "v": v}[k][~keep])
    assert not o["written"][:4].any() and o["written"][4:].all()


def _naive_budget(counts, cap):
    used, kept, total, out = 0, 0, 0, []
    for c in counts:
        total += c
        ok = c > 0 and total <= cap
        out.append(ok)
        if ok:
            used, kept = total, kept + 1
    return np.array(out), (used, kept)


def test_sample_budget_prefix_rule():
    counts = [5, 0, 7, 3, 0, 9, 4]
    # exact fit: the budget equals the inclusive sum of ray 3
    b = ot.sample_budget(counts, 15)
    assert b["kept"].tolist() == [True, False, True, True, False, False, False]
    assert b["counters"] == (15, 3) and b["offset"].tolist() == [0, 5, 5, 12, 15, 15, 24]
    assert b["n"].tolist() == [5, 0, 7, 3, 0, 0, 0]
    # one sample short: ray 3 is dropped, and every ray after it
    assert ot.sample_budget(counts, 14)["counters"] == (12, 2)
    # a zero-length ray in the middle is never kept, but the rays after it are when they fit
    assert ot.sample_budget(counts, 1000)["kept"].tolist() == [True, False, True, True, False, True, True]
    assert ot.sample_budget(counts, 0)["counters"] == (0, 0)
    assert ot.sample_budget([0, 0], 10)["counters"] == (0, 0)
    # R = 2500 (three chunks of the kernel's 1024-thread scan), cut inside the third chunk
    rng = np.random.default_rng(6)
    c = rng.integers(0, 40, 2500)
    c[rng.random(2500) < 0.2] = 0
    cap = int(np.cumsum(c)[2200])
    b = ot.sample_budget(c, cap)
    kept, ctr = _naive_budget(c.tolist(), cap)
    assert np.array_equal(b["kept"], kept) and b["counters"] == ctr
    assert b["kept"][:2201].sum() == (c[:2201] > 0).sum() and not b["kept"][2201:].any()
    assert np.array_equal(b["offset"][1:] - b["offset"][:-1], c[:-1])
