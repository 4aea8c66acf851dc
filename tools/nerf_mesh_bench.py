"""Time the NeRF mesh read-out (pyngp.Testbed.marching_cubes) on the room of tests/test_gpu_nerf_mesh.py (half extent
1.4 x 1.0 x 1.4 m, 12 views at 160x120, 300 tensor-core steps): the lattice pass (density of every point), the marching
cubes (count, one host read, emission) and the colour pass, separately, at 256^3 and 512^3 over the training box.
Medians of CUDA-event timings after warm-up, vertex / triangle counts and the peak device memory of one whole read-out.
Prints one JSON line with the card's name and power limit.

    python tools/nerf_mesh_bench.py [--reps 5] [--thresh 10] [--res 256 512]

Needs a CUDA device: without one it stops with an error before training."""
import argparse
import json
import os
import sys
import types

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tools.tsdf_readout_bench import gpu_card  # noqa: E402


def train_room(dev="cuda:0", steps=300):
    import torch
    from nerf_slam_b200.nerf_fusion import NerfFusion
    from nerf_slam_b200.synthetic import SyntheticRoom
    room = SyntheticRoom(160, 120, 12, seed=0, half_extent=(1.4, 1.0, 1.4), orbit_radius=0.3, step=0.25)
    nf = NerfFusion("nerf", types.SimpleNamespace(buffer=12, eval=False, mask_type="ours"), dev)
    nf.ngp.nerf.training.depth_supervision_lambda = 1.0
    nf.gt_fit_convention = "metric"
    pk = [room.packet(k) for k in range(12)]
    nf.fuse({"data": {"k": np.arange(12), "poses": np.stack([p["poses"][0] for p in pk]),
                      "images": np.stack([p["images"][0] for p in pk]), "depths": np.stack([p["depths"][0] for p in pk]),
                      "calibs": pk[0]["calibs"]}})
    for _ in range(steps):
        nf.fit_volume_once()
    torch.cuda.synchronize()
    return nf


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--thresh", type=float, default=10.0)   # the room's wall level (tests/test_gpu_nerf_mesh.py)
    ap.add_argument("--res", type=int, nargs="+", default=[256, 512])
    a = ap.parse_args()
    import torch
    from nerf_slam_b200 import _lib
    from nerf_slam_b200.pyngp import mesh_lattice
    _lib.load()                                            # raises NslamUnavailable without CUDA: no fallback
    name, power = gpu_card()
    tb = train_room().ngp
    k = tb.mesh_kernels

    def timed(fn):
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
        ev[0].record()
        out = fn()
        ev[1].record()
        torch.cuda.synchronize()
        return out, ev[0].elapsed_time(ev[1])

    rows = []
    for res in a.res:
        lo, h, dims = mesh_lattice(res, None, tb.aabb_scale)
        t = {"lattice": [], "mesh": [], "colors": []}
        for rep in range(a.reps + 1):                      # the first repetition warms up
            (field, weight), tl = timed(lambda: k.lattice(tb, lo, h, dims, a.thresh))
            mesh, tm = timed(lambda: k.mesh(field, weight, lo, h))
            del field, weight
            _, tc = timed(lambda: k.colors(tb, mesh, False)) if mesh is not None else (None, 0.0)
            if rep:
                t["lattice"].append(tl); t["mesh"].append(tm); t["colors"].append(tc)
            nv = 0 if mesh is None else mesh.vertices.shape[0]
            nt = 0 if mesh is None else mesh.triangles.shape[0]
            del mesh
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        mesh = tb.marching_cubes(res, None, a.thresh)
        torch.cuda.synchronize()
        peak = torch.cuda.max_memory_allocated() - base
        del mesh
        rows.append({"res": res, "points": int(np.prod(dims)), "vertices": int(nv), "triangles": int(nt),
                     **{f"{key}_ms": round(float(np.median(v)), 3) for key, v in t.items()},
                     "peak_mem_mb": round(peak / 1e6, 1)})
    print(json.dumps({"card": name or torch.cuda.get_device_name(0), "power_limit": power, "thresh": a.thresh,
                      "reps": a.reps, "results": rows}))


if __name__ == "__main__":
    main()
