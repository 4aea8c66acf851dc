"""N-GPU equals 1-GPU (SURVEY.md §4(5), §8e): data-parallel NeRF training over NCCL — the all-reduced, averaged gradient of
two trainer ranks (each on its own ray batch) must equal the average of the two batches' gradients computed in one
process, and the asynchronous keyframe hand-off must deliver the sender's tensors bit for bit.  Needs >= 2 GPUs
(skipped otherwise; run with `gpurun --gpus 2`)."""
import os
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _testbed_with_images(dev):
    import ctypes  # noqa: F401
    from nerf_slam_b200 import pyngp
    from nerf_slam_b200.synthetic import SyntheticRoom
    torch.cuda.set_device(dev)
    tb = pyngp.Testbed(seed=21, max_samples=1 << 16, max_rays=1 << 12)
    tb.create_empty_nerf_dataset(4, 1.0, None, 4, None)
    g = torch.Generator().manual_seed(21)
    tb.grid_master.copy_(((torch.rand(tb.grid_master.shape, generator=g) * 2 - 1) * 0.3).to(tb.device))
    tb.grid_half.copy_(tb.grid_master.half())
    tb.pack_weights()
    room = SyntheticRoom(64, 48, 8, seed=0)
    ids, poses, imgs, deps = [], [], [], []
    for k in (0, 4):
        p = room.packet(k)
        ids.append(len(ids)); poses.append(np.linalg.inv(np.asarray(p["poses"][0], np.float64))[:3, :4])
        imgs.append(np.asarray(p["images"][0]).astype(np.float32) / 255.0); deps.append(np.asarray(p["depths"][0]).astype(np.float32))
    calib = room.calib
    intr = calib.camera_model.numpy()
    tb.nerf.training.update_training_images(ids, poses, imgs, deps, [np.ones_like(d) for d in deps], calib.resolution.numpy(),
                                            intr[2:], intr[:2], calib.depth_scale, 1.0)
    tb.update_density_grid(full=True)
    return tb


def _gradient(tb, seed):
    import ctypes
    from nerf_slam_b200 import _lib
    lib = _lib.load()
    tb.grid_grad.zero_(); tb.mlp_grad.zero_()
    im = tb._images()
    _lib.check(lib.nslam_ngp_train_step_tc(ctypes.byref(tb.model), ctypes.byref(im), ctypes.byref(tb.batch), _lib.ptr(tb.packed), 96,
                                           seed, 1.0, 0.0, 0.0, 0.0, float(tb.loss_scale), tb.num_sms, _lib.stream_ptr()), "train_step_tc")
    torch.cuda.synchronize()
    # the batch must fit the sample buffer: rays that find it full are dropped in arrival order, which would make the
    # gradient depend on the scheduling of the march (the trainer itself sizes its batches to ~fill the buffer)
    used, kept = [int(v) for v in tb._bufs["counters"][:2].tolist()]
    assert kept == 96 and used < tb.max_samples, (used, kept)
    return tb.grid_grad.clone(), tb.mlp_grad.clone()


def _worker_body(rank, world, port, q):
    os.environ["MASTER_ADDR"] = "127.0.0.1"; os.environ["MASTER_PORT"] = str(port)
    sys.path.insert(0, ROOT)
    import torch.distributed as dist
    from nerf_slam_b200 import dist as nd
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    torch.set_grad_enabled(False)
    tb = _testbed_with_images(rank)
    seeds = [1000 + 17 * r for r in range(world)]
    gg, gm = _gradient(tb, seeds[rank])
    tb.grid_grad.copy_(gg); tb.mlp_grad.copy_(gm); tb.cam_grad.zero_()
    nd.allreduce_grads(tb, None, world)
    torch.cuda.synchronize()
    got = tb.grid_grad.clone(), tb.mlp_grad.clone()        # _gradient() below reuses the gradient buffers
    ok = True
    if rank == 0:
        refs = [_gradient(tb, s) for s in seeds]           # both batches in ONE process
        rg = sum(r[0] for r in refs) / world; rm = sum(r[1] for r in refs) / world
    else:
        rg = rm = None
    # hand-off: 3 keyframes through a capacity-2 message ring
    H, W = 24, 32
    h = nd.Handoff(torch.device("cuda", rank), 2, H, W)
    g = torch.Generator().manual_seed(5)
    ref = (torch.tensor([3, 1, 7]), torch.randn(3, 7, generator=g), torch.randint(0, 255, (3, 3, H, W), dtype=torch.uint8, generator=g),
           torch.rand(3, H, W, generator=g), torch.rand(3, H, W, generator=g))
    if rank == 0:
        h.send(*[t.cuda(rank) for t in ref]); nd.send_sync(h); h.flush()
        # float atomics in the table scatter make two evaluations of the same batch differ in the last bits
        close = lambda a, b: bool(torch.allclose(a, b, rtol=1e-3, atol=1e-5 * float(b.abs().max())))
        ok &= close(got[0], rg) and close(got[1], rm) and float(rg.abs().max()) > 0 and float(rm.abs().max()) > 0
        if not ok:
            ok = (f"grid |d| {float((got[0] - rg).abs().max()):.3e} of {float(rg.abs().max()):.3e}, "
                  f"mlp |d| {float((got[1] - rm).abs().max()):.3e} of {float(rm.abs().max()):.3e}")
    else:
        msgs = []
        while True:
            n, flags, data = h.poll(block=True)
            if n:
                msgs.append([t.cpu() for t in data])
            if flags & nd.FLAG_SYNC:
                break
        cat = [torch.cat([m[k] for m in msgs]) for k in range(5)]
        ok &= all(torch.equal(a.to(b.dtype), b) for a, b in zip(cat, ref)) and len(msgs) == 2
    dist.barrier()
    q.put((rank, ok if isinstance(ok, str) else bool(ok)))
    dist.destroy_process_group()


def _worker(rank, world, port, q):
    try:
        _worker_body(rank, world, port, q)
    except Exception:                      # report instead of leaving the parent waiting for the queue
        import traceback
        q.put((rank, traceback.format_exc()))


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_two_rank_nccl_gradients_equal_single_process_and_handoff_is_exact():
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 29700 + (os.getpid() % 200)
    ps = [ctx.Process(target=_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in ps:
        p.start()
    try:
        res = [q.get(timeout=300) for _ in ps]
        for p in ps:
            p.join(timeout=60)
    finally:
        for p in ps:                       # a rank that died or hangs must not outlive the test
            if p.is_alive():
                p.terminate()
    assert all(ok is True for _, ok in res), res
