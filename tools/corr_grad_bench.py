"""Time the correlation backward operators at 640x480 (feature maps 60x80, C = 128, r = 3, 16 edges).

    python tools/corr_grad_bench.py [--edges 16] [--iters 20] [--warmup 5]

Prints one JSON line per figure, after a line with the card's name and power limit:
  corr_index_backward   4 levels, fp16: time per edge, bytes written per edge, bytes / time
  altcorr_backward      4 levels, fp32 (f1 = fmap/4, f2 = pooled fmap/4, coords / 2^l, one coordinate set)
  corrblock_backward    CorrBlock forward + backward of sum(out * w) w.r.t. both feature maps: backward time and the
                        peak memory the backward adds
  dense_route_backward  the reference's route for the same gradient: all-pairs volume by matmul (fp16), avg_pool2d
                        pyramid, corr_index_backward per level, then autograd of the pooling and of the matmul
For corr_index_backward, altcorr_backward and the dense route it also times the reference's kernels from
oracle/_ref/nslam_ref_corr_grad.so when that module exists.  Times are medians of `iters` CUDA-event-timed calls after
`warmup` calls.  Nothing is written to disk.
"""
import argparse
import json
import os
import subprocess
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from nerf_slam_b200 import corr as pcorr  # noqa: E402
from nerf_slam_b200 import droid_backends as db  # noqa: E402

H, W, C, R = 60, 80, 128, 3


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, plim = (s.strip() for s in q.split(","))
    except Exception:
        name, plim = torch.cuda.get_device_name(0), "unknown"
    return {"card": name, "power_limit": plim}


def timed(fn, iters, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(iters):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b))
    return sorted(ts)[len(ts) // 2]


def load_ref():
    try:
        from oracle import build_ref_corr_grad
        return build_ref_corr_grad.load()
    except Exception:
        return None


class _RefSampler(torch.autograd.Function):
    """CorrSampler (networks/modules/corr.py:6-20) on a given backend"""

    @staticmethod
    def forward(ctx, volume, coords, radius, backend):
        ctx.save_for_backward(volume, coords)
        ctx.radius, ctx.backend = radius, backend
        return db.corr_index_forward(volume, coords, radius)[0]

    @staticmethod
    def backward(ctx, grad):
        volume, coords = ctx.saved_tensors
        return ctx.backend.corr_index_backward(volume, coords, grad.contiguous(), ctx.radius)[0], None, None, None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--edges", type=int, default=16)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("corr_grad_bench needs a CUDA device")
    dev, E = "cuda:0", a.edges
    print(json.dumps(card()), flush=True)
    ref = load_ref()
    g = torch.Generator(device="cpu").manual_seed(0)
    yy, xx = torch.meshgrid(torch.arange(H), torch.arange(W), indexing="ij")
    base = torch.stack([xx, yy], 0)[None].float()
    coords = (base + torch.randn(E, 2, H, W, generator=g) * 4).to(dev).contiguous()           # [E,2,H,W] level-0 pixels
    sizes = [(H >> l, W >> l) for l in range(4)]

    # corr_index_backward, 4 levels, fp16
    vols = [torch.empty(E, H, W, h, w, dtype=torch.float16, device=dev) for h, w in sizes]
    cgs = [torch.randn(E, 7, 7, H, W, generator=g).half().to(dev) for _ in sizes]
    cls = [(coords / 2 ** l).contiguous() for l in range(4)]
    written = sum(v.numel() * 2 for v in vols)

    def run_cib(backend):
        return lambda: [backend.corr_index_backward(v, c, cg, R) for v, c, cg in zip(vols, cls, cgs)]
    for name, backend in (("ours", db), ("reference", ref)):
        if backend is None:
            continue
        ms = timed(run_cib(backend), a.iters, a.warmup)
        print(json.dumps({"op": "corr_index_backward", "impl": name, "levels": 4, "dtype": "fp16", "edges": E,
                          "ms_per_edge": round(ms / E, 4), "bytes_written_per_edge": written // E,
                          "write_GBps": round(written / (ms * 1e-3) / 1e9, 1)}), flush=True)
    del vols, cgs

    # altcorr_backward, 4 levels, fp32
    fm = torch.randn(E, C, H, W, generator=g).to(dev) / 4
    f1 = fm.permute(0, 2, 3, 1).contiguous()
    f2s, x = [], fm
    for l in range(4):
        f2s.append(x.permute(0, 2, 3, 1).contiguous())
        x = F.avg_pool2d(x, 2, stride=2)
    ca = [c.permute(0, 2, 3, 1).reshape(E, 1, H, W, 2).contiguous() for c in cls]
    ags = [torch.randn(E, 1, 49, H, W, generator=g).to(dev) for _ in range(4)]

    def run_acb(backend):
        return lambda: [backend.altcorr_backward(f1, f2, c, gg, R) for f2, c, gg in zip(f2s, ca, ags)]
    for name, backend in (("ours", db), ("reference", ref)):
        if backend is None:
            continue
        ms = timed(run_acb(backend), a.iters, a.warmup)
        print(json.dumps({"op": "altcorr_backward", "impl": name, "levels": 4, "dtype": "fp32", "edges": E,
                          "ms_per_edge": round(ms / E, 4)}), flush=True)
    del f2s, ags

    # CorrBlock backward (on-the-fly route) and the reference's dense route, same loss
    fa = torch.randn(1, E, C, H, W, generator=g).to(dev).requires_grad_()
    fb = torch.randn(1, E, C, H, W, generator=g).to(dev).requires_grad_()
    wgt = torch.randn(1, E, 196, H, W, generator=g).half().float().to(dev)
    c5 = coords.view(1, E, 2, H, W).permute(0, 1, 3, 4, 2).contiguous()

    def corrblock_step():
        out = pcorr.CorrBlock(fa, fb)(c5)
        loss = (out.float() * wgt).sum()
        return loss

    def dense_step(backend):
        def step():
            e, hw = E, H * W
            corr = torch.matmul((fa.view(e, C, hw).half() / 4).transpose(1, 2), fb.view(e, C, hw).half() / 4)
            corr = corr.view(e * hw, 1, H, W)
            outs = []
            for l in range(4):
                outs.append(_RefSampler.apply(corr.view(e, H, W, *corr.shape[2:]), cls[l], R, backend).view(1, e, -1, H, W))
                if l < 3:
                    corr = F.avg_pool2d(corr, 2, stride=2)
            return (torch.cat(outs, 2).float() * wgt).sum()
        return step

    routes = [("corrblock_backward", "ours", corrblock_step), ("dense_route_backward", "ours", dense_step(db))]
    if ref is not None:
        routes.append(("dense_route_backward", "reference", dense_step(ref)))
    for op, name, step in routes:
        def bwd():
            fa.grad = fb.grad = None
            loss = step()
            torch.cuda.synchronize()
            a_, b_ = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a_.record()
            loss.backward()
            b_.record()
            b_.synchronize()
            return a_.elapsed_time(b_)
        for _ in range(a.warmup):
            bwd()
        ts = sorted(bwd() for _ in range(a.iters))
        fa.grad = fb.grad = None
        loss = step()
        torch.cuda.synchronize()
        base_mem = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        loss.backward()
        torch.cuda.synchronize()
        peak = torch.cuda.max_memory_allocated() - base_mem
        print(json.dumps({"op": op, "impl": name, "edges": E, "backward_ms": round(ts[len(ts) // 2], 3),
                          "backward_ms_per_edge": round(ts[len(ts) // 2] / E, 4),
                          "backward_peak_extra_MB": round(peak / 2 ** 20, 1)}), flush=True)
        del loss


if __name__ == "__main__":
    main()
