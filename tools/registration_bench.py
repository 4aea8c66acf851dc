"""Time ICP (csrc/registration.cu through nerf_slam_b200/registration.py) on the synthetic room: the BVH build over the
target samples, one iteration (transform, nearest, accumulate and the 38-integer read) at 0.1 M and 1 M source samples,
and whole coarse-to-fine Sim3 ICPs from the identity that bring two meshes back onto their room's true surface
from a known offset (7 degrees, 0.1 m, scale 0.9): the dense TSDF mesh of the room and the trained room's NeRF mesh,
built as tools/mesh_ops_bench.py builds them (the NeRF mesh without its components under 0.05 m^2).  Builds and
iterations: CUDA events, median of --reps after two warm-up calls; whole ICPs: host clock around a call that ends
in a device read, median of --reps.  Prints one JSON line with the card's name and power limit, read in the same run.

    python tools/registration_bench.py [--reps 5] [--res 512]

Needs a CUDA device: without one it stops with an error before timing."""
import argparse
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tools.mesh_ops_bench import room_meshes  # noqa: E402
from tools.tsdf_readout_bench import gpu_card  # noqa: E402

OFFSET = (0.9, 7.0, (0.1, -0.05, 0.08))          # scale, degrees about (0.3, 1, 0.2), translation (m)
DISTS = (0.5, 0.2, 0.1, 0.05)                    # the first stage reaches walls the 0.9 scale moved by up to 0.3 m


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--res", type=int, default=512)
    a = ap.parse_args()
    import torch
    from nerf_slam_b200 import _lib, mesh_ops, registration as reg
    from nerf_slam_b200.evaluation import PointIndex, sample_surface
    from nerf_slam_b200.synthetic import SyntheticRoom
    _lib.load()                                            # raises NslamUnavailable without CUDA: no fallback
    dev = "cuda:0"
    name, power = gpu_card()

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
        return out, float(np.median(ts))

    s, deg, t = OFFSET
    axis = np.array([0.3, 1.0, 0.2])
    offset = reg.compose(s, reg.rodrigues(np.deg2rad(deg) * axis / np.linalg.norm(axis)), t)
    nerf_mesh, _, _, _, tsdf_mesh, _, _ = room_meshes(a.res, dev)
    room_gt = tuple(torch.from_numpy(x).to(dev) for x in SyntheticRoom(64, 48, 2).surface_mesh())
    nerf_gt = tuple(torch.from_numpy(x).to(dev) for x in
                    SyntheticRoom(64, 48, 2, half_extent=(1.4, 1.0, 1.4)).surface_mesh())   # mesh_ops_bench's NeRF room
    res = {}
    with _lib.fixed_stream():
        tgt, nrm, _ = reg._target(room_gt, "point_to_plane", 200_000, 1)
        lo, hi = torch.aminmax(tgt, dim=0)
        frame = reg.target_frame(lo.tolist(), hi.tolist())
        _, ms = timed(lambda: PointIndex(tgt))
        res["bvh_build_200k_ms"] = round(ms, 3)
        for n in (100_000, 1_000_000):
            src = sample_surface(tsdf_mesh, n, 0)                  # aligned: the state of ICP's last iterations
            corr = reg._Correspondences(src, tgt, nrm, frame)
            for p2p in (False, True):
                _, ms = timed(lambda: corr.sums_at(1.0, np.eye(3), np.zeros(3), 0.1, p2p, True))
                res[f"iteration_{n // 1000}k_{'point' if p2p else 'plane'}_ms"] = round(ms, 3)
            del corr
    nerf_mesh = mesh_ops.remove_small_components(nerf_mesh, 0.05)      # floaters off first, as evaluations do
    for label, mesh, gt in (("tsdf_mesh", tsdf_mesh, room_gt), ("nerf_mesh", nerf_mesh, nerf_gt)):
        moved = reg.transform(mesh, offset)
        r = {"triangles": int(mesh.triangles.shape[0])}
        for metric in ("point_to_plane", "point_to_point"):
            ts = []
            for _ in range(a.reps):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                out = reg.icp(moved, gt, metric=metric, with_scale=True, max_corr_dist=DISTS)
                ts.append(time.perf_counter() - t0)
            E = out.transform @ offset
            r[metric] = {"ms": round(1e3 * float(np.median(ts)), 2), "iterations": out.iterations,
                         "converged": out.converged, "fitness": round(out.fitness, 4),
                         "inlier_rmse": round(out.inlier_rmse, 5),
                         "scale_error": abs(float(np.cbrt(np.linalg.det(E[:3, :3]))) - 1),
                         "translation_error": float(np.abs(E[:3, 3]).max())}
        res[label] = r
    print(json.dumps({"bench": "registration", "gpu": name or torch.cuda.get_device_name(0), "power_limit": power,
                      "reps": a.reps, "res": a.res, **res}))


if __name__ == "__main__":
    main()
