"""Path B parity: sm_90a NeRF kernels vs the torch fp32 oracle (oracle/ngp.py), and convergence.
Tolerances: the hash table is read in fp16 by the kernels (oracle uses the same fp16-rounded
values), MLP math is fp32 -> rgb/sigma rel 1e-4; gradients rel 2e-3 (fp16 storage of the
recomputed activations in the backward tile)."""
import ctypes
import os

import numpy as np
import pytest
import torch

from oracle import ngp as ongp

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _testbed(seed=3, aabb=4):
    from nerf_slam_b200 import pyngp
    tb = pyngp.Testbed(seed=seed, max_samples=1 << 16, max_rays=1 << 13)
    tb.create_empty_nerf_dataset(8, 1.0, None, aabb, None)
    # non-trivial table values so that the encoding matters
    g = torch.Generator().manual_seed(seed)
    tb.grid_master.copy_(((torch.rand(tb.grid_master.shape, generator=g) * 2 - 1) * 0.5).to(DEV))
    tb.grid_half.copy_(tb.grid_master.half())
    return tb


def _oracle_params(tb):
    P = {"grid": tb.grid_half.float().cpu().view(-1, 2)}
    w = tb.mlp.cpu()
    off = 0
    for name, (i, o) in dict(W1=(32, 64), W2=(64, 16), W3=(32, 64), W4=(64, 64), W5=(64, 16)).items():
        P[name] = w[off:off + i * o].view(i, o).clone(); off += i * o
    return P


def test_level_table_matches_oracle():
    from nerf_slam_b200 import pyngp
    rows, total = pyngp.level_table(4.0)
    lv, tot = ongp.level_params(4.0)
    assert total == tot
    for a, b in zip(rows, lv):
        assert a[:4] == (b[0], b[1], b[2], b[3])


def test_forward_matches_oracle():
    from nerf_slam_b200 import _lib
    tb = _testbed()
    lib = _lib.load()
    g = torch.Generator().manual_seed(0)
    n = 1000
    x = torch.rand(n, 3, generator=g)
    d = torch.nn.functional.normalize(torch.randn(n, 3, generator=g), dim=-1)
    coords = torch.cat([x, torch.full((n, 1), 0.01), d], -1).contiguous().to(DEV)
    out = torch.zeros(n, 4, device=DEV)
    _lib.check(lib.nslam_ngp_forward(ctypes.byref(tb.model), _lib.ptr(coords), n, _lib.ptr(out), _lib.stream_ptr()), "fwd")
    rgb, sigma = ongp.network(x, d, _oracle_params(tb), 4.0)
    got = out.cpu()
    assert torch.allclose(got[:, :3], rgb, rtol=2e-4, atol=2e-5), (got[:, :3] - rgb).abs().max()
    assert torch.allclose(got[:, 3], sigma, rtol=5e-4, atol=1e-5), (got[:, 3] - sigma).abs().max()


def _grad_err(got, ref, backend):
    """simt (fp32 arithmetic): max-norm error relative to the largest entry.
    tcgen05 (fp16 operands with loss scaling, the mixed-precision recipe of instant-ngp): every term
    a_s * delta_s of a weight gradient carries ~2^-11 relative rounding, so the error floor scales with
    sum_s |a_s delta_s|, not with the (cancelling) sum itself: measured 3e-4 on single tiles and up to 5e-2
    of the layer's Frobenius norm where the true gradient nearly cancels.  Per-layer relative Frobenius
    error is bounded loosely here; the direction of the full gradient (cosine, checked by the caller)
    and the convergence test below are the sharp criteria."""
    if backend == "simt":
        return float((got - ref).abs().max() / (ref.abs().max() + 1e-12))
    return float((got - ref).norm() / (ref.norm() + 1e-20))


@pytest.mark.parametrize("backend,R,per,tol", [("simt", 24, 11, 3e-3), ("tcgen05", 24, 11, 1e-1), ("tcgen05", 300, 13, 1e-1),
                                               ("tcgen05", 8, 16, 1e-1)])
def test_loss_and_gradients_match_autograd(backend, R, per, tol):
    """simt: fp32 CUDA-core kernels, tight tolerance.  tcgen05: fp16 operands (weights, activations,
    loss-scaled deltas), fp32 accumulation -> gradients within 2 % of the largest entry."""
    from nerf_slam_b200 import _lib
    tb = _testbed(seed=5)
    lib = _lib.load()
    g = torch.Generator().manual_seed(1)
    n = R * per
    x = torch.rand(n, 3, generator=g) * 0.6 + 0.2
    d = torch.nn.functional.normalize(torch.randn(R, 3, generator=g), dim=-1).repeat_interleave(per, 0)
    dt = torch.rand(n, generator=g) * 0.05 + 0.01
    tdist = (torch.arange(per).float()[None] * 0.05 + 0.3).repeat(R, 1).reshape(-1)
    coords = torch.cat([x, dt[:, None], d], -1).contiguous()
    rays = torch.zeros(R, 16)
    rays[:, 3:6] = d[::per]
    rays[:, 6] = 0.9                                    # inv_len
    tgt_rgb = torch.rand(R, 3, generator=g)
    tgt_dep = torch.rand(R, generator=g) * 0.5 + 0.2
    tgt_dep[::5] = -1.0                                 # rays without depth
    cov = torch.rand(R, generator=g) * 0.5 + 0.1
    rays[:, 7], rays[:, 8], rays[:, 9:12] = tgt_dep, cov, tgt_rgb
    ri = rays.view(torch.int32)
    ri[:, 12] = torch.arange(R, dtype=torch.int32) * per
    ri[:, 13] = per
    tb._bufs["rays"][:R].copy_(rays.to(DEV)); tb._bufs["coords"][:n].copy_(coords.to(DEV)); tb._bufs["tdist"][:n].copy_(tdist.to(DEV))
    tb.mlp_grad.zero_(); tb.grid_grad.zero_()
    bg = (0.2, 0.4, 0.6)
    if backend == "simt":
        _lib.check(lib.nslam_ngp_loss_backward(ctypes.byref(tb.model), ctypes.byref(tb.batch), R, n, 1.0, *bg,
                                               tb.num_sms, _lib.stream_ptr()), "loss_bwd")
    else:
        tb.pack_weights()
        _lib.check(lib.nslam_ngp_loss_backward_tc(ctypes.byref(tb.model), ctypes.byref(tb.batch), _lib.ptr(tb.packed), R, n,
                                                  1.0, *bg, 1024.0, tb.num_sms, _lib.stream_ptr()), "loss_bwd_tc")
    torch.cuda.synchronize()
    # oracle with autograd
    P = _oracle_params(tb)
    for v in P.values():
        v.requires_grad_(True)
    rgb, sigma = ongp.network(x, d, P, 4.0)
    loss, _, _ = ongp.composite_loss(rgb, sigma, dt, tdist * 0.9, [i * per for i in range(R + 1)], tgt_rgb, tgt_dep, cov,
                                     torch.tensor(bg).repeat(R, 1), 1.0)
    loss.backward()
    assert abs(float(tb._bufs["loss"].item()) - float(loss)) < (1e-4 if backend == "simt" else 5e-3) * max(1.0, abs(float(loss)))
    gw = tb.mlp_grad.cpu()
    off = 0
    for name, (i, o) in dict(W1=(32, 64), W2=(64, 16), W3=(32, 64), W4=(64, 64), W5=(64, 16)).items():
        ref = P[name].grad
        got = gw[off:off + i * o].view(i, o); off += i * o
        if name == "W5":
            ref, got = ref[:, :3], got[:, :3]
        err = _grad_err(got, ref, backend)
        assert err < tol, f"{name}: rel err {err:.2e}"
    gg = tb.grid_grad.cpu().view(-1, 2)
    ref = P["grid"].grad
    err = _grad_err(gg, ref, backend)
    assert err < tol, f"grid: rel err {err:.2e}"
    full_got = torch.cat([gw[:off], gg.reshape(-1)]); full_ref = torch.cat([P[k].grad.reshape(-1) for k in ("W1", "W2", "W3", "W4")] +
                                                                         [torch.nn.functional.pad(P["W5"].grad[:, :3], (0, 13)).reshape(-1), ref.reshape(-1)])
    full_got = full_got.clone(); full_got[9216:10240].view(64, 16)[:, 3:] = 0     # W5 columns beyond rgb are unused
    cos = float(torch.dot(full_got, full_ref) / (full_got.norm() * full_ref.norm()))
    assert cos > (0.999999 if backend == "simt" else 0.9995), cos


def test_camera_pose_gradients_match_autograd():
    """optimize_extrinsics (fusion/nerf_fusion.py:99): nslam_ngp_cam_grad — dL/d(translation) and dL/d(rotation vector)
    per camera from the batch's encoding gradients — against autograd through the oracle network with the sample
    positions p = (o + dt_c) + t (d + w_c x d) (direction held fixed inside the spherical harmonics, as the published
    scheme does).  Then one Adam step moves the effective camera against the gradient and an ingest resets it."""
    from nerf_slam_b200 import _lib
    tb = _testbed(seed=8)
    lib = _lib.load()
    g = torch.Generator().manual_seed(4)
    R, per = 64, 12
    n = R * per
    img = (torch.arange(R) % 2).int()
    cam_o = torch.tensor([[0.1, -0.2, 0.0], [-0.3, 0.1, 0.2]])
    o = cam_o[img.long()]
    d = torch.nn.functional.normalize(torch.randn(R, 3, generator=g), dim=-1)
    tdist = (torch.arange(per).float()[None] * 0.06 + 0.25 + torch.rand(R, 1, generator=g) * 0.05).reshape(R, per)
    dt = torch.full((n,), 0.06)
    lo, ext = 0.5 - 0.5 * 4.0, 4.0
    xw = o[:, None] + tdist[..., None] * d[:, None]
    x01 = ((xw - lo) / ext).reshape(n, 3)
    coords = torch.cat([x01, dt[:, None], d.repeat_interleave(per, 0)], -1).contiguous()
    rays = torch.zeros(R, 16)
    rays[:, 0:3], rays[:, 3:6], rays[:, 6] = o, d, 0.9
    tgt_rgb = torch.rand(R, 3, generator=g); tgt_dep = torch.rand(R, generator=g) * 0.5 + 0.2; cov = torch.rand(R, generator=g) * 0.5 + 0.1
    rays[:, 7], rays[:, 8], rays[:, 9:12] = tgt_dep, cov, tgt_rgb
    ri = rays.view(torch.int32)
    ri[:, 12] = torch.arange(R, dtype=torch.int32) * per
    ri[:, 13] = per
    ri[:, 14] = img
    tb._bufs["rays"][:R].copy_(rays.to(DEV)); tb._bufs["coords"][:n].copy_(coords.to(DEV)); tb._bufs["tdist"][:n].copy_(tdist.reshape(-1).to(DEV))
    tb.mlp_grad.zero_(); tb.grid_grad.zero_(); tb.cam_grad.zero_()
    tb.pack_weights()
    bg = (0.2, 0.4, 0.6)
    _lib.check(lib.nslam_ngp_loss_backward_tc(ctypes.byref(tb.model), ctypes.byref(tb.batch), _lib.ptr(tb.packed), R, n,
                                              1.0, *bg, 1024.0, tb.num_sms, _lib.stream_ptr()), "loss_bwd_tc")
    lv = tb._lv
    _lib.check(lib.nslam_ngp_cam_grad(_lib.ptr(tb.grid_half), lv["scale"].ctypes.data, lv["res"].ctypes.data, lv["size"].ctypes.data,
                                      lv["offset"].ctypes.data, lv["dense"].ctypes.data, 4.0, _lib.ptr(tb._bufs["rays"]), R,
                                      _lib.ptr(tb._bufs["coords"]), _lib.ptr(tb._bufs["tdist"]), _lib.ptr(tb._bufs["denc"]), 1024.0,
                                      _lib.ptr(tb.cam_grad), int(tb.cam_grad.shape[0]), _lib.stream_ptr()), "cam_grad")
    torch.cuda.synchronize()
    # oracle
    P = _oracle_params(tb)
    dtc = torch.zeros(2, 3, requires_grad=True); wc = torch.zeros(2, 3, requires_grad=True)
    il = img.long()
    o2 = o + dtc[il]
    d2 = d + torch.cross(wc[il], d, dim=-1)
    x2 = ((o2[:, None] + tdist[..., None] * d2[:, None] - lo) / ext).reshape(n, 3)
    rgb, sigma = ongp.network(x2, d.repeat_interleave(per, 0), P, 4.0)
    loss, _, _ = ongp.composite_loss(rgb, sigma, dt, tdist.reshape(-1) * 0.9, [i * per for i in range(R + 1)], tgt_rgb, tgt_dep, cov,
                                     torch.tensor(bg).repeat(R, 1), 1.0)
    loss.backward()
    ref = torch.cat([dtc.grad, wc.grad], 1)                     # [2,6]
    got = tb.cam_grad[:2].cpu()
    assert float(tb.cam_grad[2:].abs().max()) == 0.0
    rel = float((got - ref).norm() / ref.norm())
    cos = float(torch.dot(got.reshape(-1), ref.reshape(-1)) / (got.norm() * ref.norm()))
    assert rel < 5e-2 and cos > 0.999, (rel, cos, got, ref)
    # Adam step + effective cameras; then an ingest of camera 0 resets its refinement
    base = torch.zeros(8, 18); base[:, [0, 5, 10]] = 1.0; base[:2, [3, 7, 11]] = cam_o
    tb.cams_base.copy_(base.to(DEV)); tb.cams.copy_(base.to(DEV))
    _lib.check(lib.nslam_ngp_cam_adam_apply(_lib.ptr(tb.cams_base), _lib.ptr(tb.cams), _lib.ptr(tb.cam_state[0]), _lib.ptr(tb.cam_grad),
                                            _lib.ptr(tb.cam_state[1]), _lib.ptr(tb.cam_state[2]), _lib.ptr(tb.cam_steps), 8, 1e-3, 0.9, 0.99,
                                            1e-10, 0.0, _lib.stream_ptr()), "cam_adam")
    torch.cuda.synchronize()
    off = tb.cam_state[0].cpu()
    assert torch.allclose(off[:2], -1e-3 * torch.sign(ref), atol=2e-5)           # first Adam step = -lr * sign(g)
    assert float(off[2:].abs().max()) == 0.0 and float(tb.cam_grad.abs().max()) == 0.0 and tb.cam_steps[:3].tolist() == [1, 1, 0]
    eff = tb.cams.cpu()
    assert torch.allclose(eff[:2, [3, 7, 11]], cam_o + off[:2, :3], atol=1e-7)
    w = off[0, 3:]
    Rw = torch.linalg.matrix_exp(torch.tensor([[0, -w[2], w[1]], [w[2], 0, -w[0]], [-w[1], w[0], 0]]))
    assert torch.allclose(eff[0, :12].view(3, 4)[:, :3], Rw, atol=1e-6)
    assert torch.equal(eff[2:], base[2:])


@pytest.mark.parametrize("backend", ["tcgen05", "simt"])
def test_render_matches_oracle(backend):
    """B4: Testbed.render (Shade and Depth) of a camera view against oracle/ngp.py::render_view — same pixel-centre rays,
    same jitter-free occupancy march, network, compositing over the background.  tcgen05 = the tensor-core forward the
    product renders with (fp16 operands: 1e-2 abs on colours); simt = fp32 CUDA-core forward (2e-4)."""
    from nerf_slam_b200 import pyngp
    tb = _testbed(seed=12)
    tb.mlp_backend = backend
    g = torch.Generator().manual_seed(6)
    tb.mlp.mul_(0.5)                                    # moderate densities: rays neither empty nor saturated at once
    tb.pack_weights()
    bits = (torch.rand(tb.bits.shape, generator=g) < 0.3).to(torch.uint8) * torch.randint(1, 256, tb.bits.shape, generator=g, dtype=torch.uint8)
    tb.bits.copy_(bits.to(DEV))
    W, H = 20, 12
    c2w = np.eye(4)[:3].copy(); c2w[:, 3] = [0.45, 0.55, 0.1]
    th = 0.2
    c2w[:3, :3] = np.array([[np.cos(th), 0, np.sin(th)], [0, 1, 0], [-np.sin(th), 0, np.cos(th)]])
    tb.camera_matrix = c2w.astype(np.float64)
    tb._view_intr = np.array([18.0, 18.0, W / 2 - 0.5, H / 2 - 0.5], np.float32)
    tb.background_color = [0.1, 0.3, 0.5, 1.0]
    tb.render_mode = pyngp.Shade
    rgb = tb.render(W, H, 1, True)[..., :3]
    tb.render_mode = pyngp.Depth
    dep = tb.render(W, H, 1, True)[..., 0]
    per_ray = max(8, min(1024, tb.max_samples // (min(32, tb.max_rays // W) * W)))      # Testbed.render's sample budget per ray
    ref_rgb, ref_dep = ongp.render_view(_oracle_params(tb), c2w, tb._view_intr, W, H, tb.aabb_scale, tb.cascades, bits.numpy(),
                                        tb.nerf.training.near_distance, tb.background_color[:3], max_per_ray=per_ray)
    tol = 1e-2 if backend == "tcgen05" else 2e-4
    assert np.abs(rgb - ref_rgb).max() < tol, np.abs(rgb - ref_rgb).max()
    assert np.abs(dep - ref_dep).max() < (3e-2 if backend == "tcgen05" else 1e-3) * max(1.0, ref_dep.max()), np.abs(dep - ref_dep).max()
    assert ref_dep.max() > 0.2 and np.ptp(ref_rgb) > 0.05          # the view is not trivial


def test_adam_step_matches_torch():
    from nerf_slam_b200 import _lib
    tb = _testbed(seed=6)
    lib = _lib.load()
    g = torch.Generator().manual_seed(2)
    grad = torch.randn(10240, generator=g)
    w0 = tb.mlp.cpu().clone()
    p = torch.nn.Parameter(w0.clone())
    opt = torch.optim.Adam([p], lr=1e-2, betas=(0.9, 0.99), eps=1e-15)
    for step in range(1, 4):
        tb.mlp_grad.copy_(grad.to(DEV))
        _lib.check(lib.nslam_ngp_adam(ctypes.byref(tb.model), step, 1e-2, 0.9, 0.99, 1e-15, 0.0, _lib.stream_ptr()), "adam")
        p.grad = grad.clone(); opt.step()
    assert torch.allclose(tb.mlp.cpu(), p.data, rtol=1e-5, atol=1e-7)
    assert float(tb.mlp_grad.abs().max()) == 0.0


@pytest.mark.parametrize("backend", ["tcgen05", "simt"])
def test_nerf_fits_synthetic_room(backend):
    """convergence: train on GT-posed views of the procedural room; PSNR must rise clearly"""
    from nerf_slam_b200.synthetic import SyntheticRoom
    import types
    from nerf_slam_b200.nerf_fusion import NerfFusion
    room = SyntheticRoom(160, 120, 12, seed=0, half_extent=(1.4, 1.0, 1.4), orbit_radius=0.3, step=0.25)
    args = types.SimpleNamespace(buffer=12, eval=False, mask_type="ours")
    nf = NerfFusion("nerf", args, DEV)
    nf.ngp.nerf.training.depth_supervision_lambda = 1.0
    nf.ngp.mlp_backend = backend
    nf.gt_fit_convention = "metric"           # metric poses + linear colours (the default mirrors the reference's GT tuples)
    pk = [room.packet(k) for k in range(12)]
    packet = {"k": np.arange(12), "poses": np.stack([p["poses"][0] for p in pk]), "images": np.stack([p["images"][0] for p in pk]),
              "depths": np.stack([p["depths"][0] for p in pk]), "calibs": pk[0]["calibs"]}
    # world is centred at the origin; shift into the trainer's box by using poses as they are (aabb_scale 4 covers [-1.5,2.5])
    nf.fuse({"data": packet})
    psnr0 = nf.eval_gt_traj(stride=4)["psnr"]
    for _ in range(300):
        nf.fit_volume_once()
    torch.cuda.synchronize()
    r = nf.eval_gt_traj(stride=4)
    assert np.isfinite(nf.ngp.sync_stats())
    assert r["psnr"] > psnr0 + 5.0 and r["psnr"] > 18.0, (psnr0, r)


def test_forward_tc_matches_oracle():
    """Tensor-core MLP forward (fp16 weights + fp16 inter-layer activations, fp32 accumulate) vs the fp32
    oracle: rgb in (0,1) abs 1e-2, sigma rel 3e-2."""
    from nerf_slam_b200 import _lib
    tb = _testbed(seed=8)
    lib = _lib.load()
    g = torch.Generator().manual_seed(3)
    n = 1000                                    # not a multiple of 128: exercises the partial tile
    x = torch.rand(n, 3, generator=g)
    d = torch.nn.functional.normalize(torch.randn(n, 3, generator=g), dim=-1)
    coords = torch.cat([x, torch.full((n, 1), 0.01), d], -1).contiguous().to(DEV)
    packed = torch.zeros(61440, dtype=torch.uint8, device=DEV)
    _lib.check(lib.nslam_ngp_pack_mlp(_lib.ptr(tb.mlp), _lib.ptr(packed), _lib.stream_ptr()), "pack")
    out = torch.zeros(n, 4, device=DEV)
    _lib.check(lib.nslam_ngp_forward_tc(ctypes.byref(tb.model), _lib.ptr(packed), _lib.ptr(coords), None, n, n,
                                        _lib.ptr(out), None, tb.num_sms, _lib.stream_ptr()), "fwd_tc")
    torch.cuda.synchronize()
    rgb, sigma = ongp.network(x, d, _oracle_params(tb), 4.0)
    got = out.cpu()
    assert torch.isfinite(got).all()
    assert float((got[:, :3] - rgb).abs().max()) < 1e-2
    assert float(((got[:, 3] - sigma).abs() / sigma).max()) < 3e-2
    # and against the SIMT forward kernel on the same inputs
    out2 = torch.zeros(n, 4, device=DEV)
    _lib.check(lib.nslam_ngp_forward(ctypes.byref(tb.model), _lib.ptr(coords), n, _lib.ptr(out2), _lib.stream_ptr()), "fwd")
    assert float((out[:, :3] - out2[:, :3]).abs().max()) < 1e-2


def test_sample_rays_matches_the_march_oracle():
    """every ray the sampler keeps must carry exactly the samples of oracle/ngp.py::march_lattice (bit-equal t and dt:
    the kernel rebuilds the lattice with the same serial fp32 recurrence), in ray order, with positions
    (o + t d - aabb_lo) / extent"""
    from nerf_slam_b200 import _lib
    tb = _testbed(seed=11)
    lib = _lib.load()
    g = torch.Generator().manual_seed(5)
    H, W = 48, 64
    tb._ensure_store(H, W)
    c2w = np.eye(4)[:3]; c2w[:, 3] = [0.5, 0.5, 0.5]
    tb._set_camera(0, c2w, (60.0, 60.0), (W / 2 - 0.5, H / 2 - 0.5), (W, H))
    tb._activate([0])
    bits = (torch.rand(tb.bits.shape, generator=g) < 0.25).to(torch.uint8) * torch.randint(1, 256, tb.bits.shape, generator=g, dtype=torch.uint8)
    tb.bits.copy_(bits.to(DEV))
    R, seed = 96, 1234
    im = tb._images()
    _lib.check(lib.nslam_ngp_sample_phase(ctypes.byref(tb.model), ctypes.byref(im), ctypes.byref(tb.batch), R, seed,
                                          _lib.stream_ptr()), "sample")
    torch.cuda.synchronize()
    rays = tb._bufs["rays"][:R].cpu(); ri = rays.view(torch.int32)
    coords = tb._bufs["coords"].cpu().numpy(); tdist = tb._bufs["tdist"].cpu().numpy()
    bits_h = bits.numpy()
    lo, hi = 0.5 - 0.5 * tb.aabb_scale, 0.5 + 0.5 * tb.aabb_scale
    checked = 0
    for i in range(R):
        n, base = int(ri[i, 13]), int(ri[i, 12])
        if n == 0:
            continue
        o = rays[i, 0:3].numpy(); d = rays[i, 3:6].numpy()
        jit = float(ongp.rnd01(seed, i, 4))                       # the kernel's per-ray jitter
        ref = ongp.march_lattice(o, d, lo, hi, tb.nerf.training.near_distance, 1.0 / 256, tb.cascades, bits_h, jit, 1024)
        assert len(ref) == n
        for k, (t, dt) in enumerate(ref):
            assert abs(float(t) - float(tdist[base + k])) <= 2e-6 and float(dt) == float(coords[base + k, 3])
            pos = (o + d * np.float32(t) - lo) / (hi - lo)
            assert np.allclose(coords[base + k, 0:3], pos, atol=2e-6)
        checked += 1
    assert checked > 0


@pytest.mark.parametrize("mask_type", ["ours", "raw", "ours_w_thresh", "no_depth"])
def test_process_slam_ingest_matches_reference_golden(mask_type):
    """B1/B2 end to end on the device: NerfFusion.process_slam (mask types, pose conversion on the host; sRGB->linear,
    alpha, 1/idepth in `ingest_image_kernel`) must leave in the trainer's slots what the REFERENCE's process_slam +
    send_data handed to pyngp (tests/golden/ref_process_slam.npz).  Images are stored in fp16 (2^-11 relative)."""
    import sys
    import types
    here = os.path.dirname(os.path.abspath(__file__))
    sys.path.insert(0, os.path.join(here, "golden"))
    import process_slam_scenario as sc
    from nerf_slam_b200.nerf_fusion import NerfFusion
    gold = np.load(os.path.join(here, "golden", "ref_process_slam.npz"))
    tb = _testbed()
    nf = object.__new__(NerfFusion)
    nf.mask_type, nf.ref_frames, nf.ngp = mask_type, {}, tb
    slam = sc.make_packet()
    for k in ("cam0_poses", "cam0_images", "cam0_idepths_up", "cam0_depths_cov_up", "gt_depths", "viz_idx"):
        slam[k] = slam[k].to(DEV)
    assert nf.process_slam([None, slam]) is False
    torch.cuda.synchronize()
    ids = gold[f"{mask_type}.ids"].tolist()
    assert tb.active_set == ids and tb.nerf.training.n_images_for_training == len(ids)
    for k, fid in enumerate(ids):
        img = tb.rgba[fid].float().cpu().numpy()
        ref = gold[f"{mask_type}.images"][k]
        assert np.abs(img - ref).max() <= 1e-3 * max(1.0, np.abs(ref).max()) and np.all(img[..., 3] == 1.0)
        assert np.allclose(tb.depth[fid].cpu().numpy()[..., None], gold[f"{mask_type}.depths"][k], rtol=2e-6, atol=0)
        assert np.array_equal(tb.depth_cov[fid].cpu().numpy()[..., None], gold[f"{mask_type}.covs"][k])
        cam = tb.cams_h[fid]
        assert np.allclose(cam[:12].reshape(3, 4), gold[f"{mask_type}.poses"][k], atol=2e-6)
        assert np.allclose(cam[12:14], gold[f"{mask_type}.fl"]) and np.allclose(cam[14:16], gold[f"{mask_type}.pp"])
        assert cam[16:18].view(np.int32).tolist() == gold[f"{mask_type}.res"].tolist()
