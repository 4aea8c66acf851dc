"""Time the reconstruction evaluation (csrc/recon_eval.cu): the BVH build over 1 M reference points, exact nearest
neighbours of 1 M / 10 M / 30 M queries against it, sampling 1 M points from a mesh, with the peak device memory each
adds; scipy's cKDTree on the host CPU over the same sizes as context (build, and the same queries on all host
threads, one timing each).  Reference points are area-uniform samples of the synthetic
room's walls, queries the same surface perturbed by 1 cm noise plus 1 % uniform outliers in the room: what scoring a
reconstruction looks like.  GPU times: CUDA events, median of --reps after two warm-up calls.  Prints one JSON line
with the card's name and power limit.

    python tools/recon_eval_bench.py [--reps 5] [--no-cpu]

Needs a CUDA device: without one it stops with an error before timing."""
import argparse
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tools.tsdf_readout_bench import gpu_card  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--refs", type=int, default=1_000_000)
    ap.add_argument("--queries", type=str, default="1000000,10000000,30000000")
    ap.add_argument("--no-cpu", action="store_true")
    a = ap.parse_args()
    import torch
    from nerf_slam_b200 import _lib
    from nerf_slam_b200.evaluation import PointIndex, sample_surface
    from nerf_slam_b200.synthetic import SyntheticRoom
    _lib.load()                                            # raises NslamUnavailable without CUDA: no fallback
    dev = "cuda:0"
    mesh = SyntheticRoom(8, 6, 1).surface_mesh()
    sizes = [int(s) for s in a.queries.split(",")]

    def timed(fn):
        for _ in range(2):
            out = fn()
        torch.cuda.synchronize()
        ts = []
        for _ in range(a.reps):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            out = fn()
            e1.record()
            torch.cuda.synchronize()
            ts.append(e0.elapsed_time(e1))
        return out, round(float(np.median(ts)), 3), round(float(min(ts)), 3)

    def peak(fn):
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        out = fn()
        torch.cuda.synchronize()
        return out, int(torch.cuda.max_memory_allocated() - base)

    res = {}
    _, ms, mn = timed(lambda: sample_surface(mesh, 1_000_000, seed=0))
    _, pb = peak(lambda: sample_surface(mesh, 1_000_000, seed=0))
    res["sample_1M"] = {"ms": ms, "ms_min": mn, "peak_bytes": pb}

    ref = sample_surface(mesh, a.refs, seed=1)
    index, ms, mn = timed(lambda: PointIndex(ref))
    _, pb = peak(lambda: PointIndex(ref))
    res["bvh_build"] = {"points": a.refs, "ms": ms, "ms_min": mn, "peak_bytes": pb}

    g = torch.Generator(device=dev).manual_seed(0)
    queries = {}
    for n in sizes:
        q = sample_surface(mesh, n, seed=2)
        q += 0.01 * torch.randn(q.shape, device=dev, generator=g)
        k = n // 100
        q[:k] = (torch.rand(k, 3, device=dev, generator=g) * 2 - 1) * torch.tensor([3.0, 2.0, 3.0], device=dev)
        queries[n] = q
        (dist, _), ms, mn = timed(lambda: index.query(q, 1.0))
        _, pb = peak(lambda: index.query(q, 1.0))
        res[f"nearest_{n // 1_000_000}M"] = {"ms": ms, "ms_min": mn, "Mqueries_per_s": round(n / ms / 1e3, 1),
                                             "peak_bytes": pb, "matched": round(float(torch.isfinite(dist).float().mean()), 4)}
    if not a.no_cpu:
        from scipy.spatial import cKDTree
        r = ref.cpu().numpy().astype(np.float64)
        t0 = time.perf_counter()
        tree = cKDTree(r)
        res["cpu_ckdtree_build_ms"] = round((time.perf_counter() - t0) * 1e3, 1)
        for n in sizes:
            q = queries[n].cpu().numpy().astype(np.float64)
            t0 = time.perf_counter()
            tree.query(q, distance_upper_bound=1.0, workers=-1)
            res[f"cpu_ckdtree_query_{n // 1_000_000}M_ms"] = round((time.perf_counter() - t0) * 1e3, 1)
        res["cpu_threads"] = os.cpu_count()
    name, power = gpu_card()
    print(json.dumps({"bench": "recon_eval", "gpu": name or torch.cuda.get_device_name(0), "power_limit": power,
                      "reps": a.reps, **res}))


if __name__ == "__main__":
    main()
