"""Time the SLAM point cloud (csrc/point_cloud.cu) on a full map: the synthetic room, 100 ground-truth keyframes at
640x480 with a synthetic depth variance (0.1 d^2)^2 and the uncertainty mask (the demo's default).  Three configurations
in one invocation: the cloud alone, the cloud with the multi-view filter (5 cm, 2 views), the cloud with 1 cm voxel
downsampling.  Each is timed end to end, host reads included, with CUDA events: median of --reps calls after warm-up.
Also reported: points in (candidate pixels) and out, peak device memory added by the call, the card's name and power
limit read in the same run.  Prints one JSON line.

    python tools/point_cloud_bench.py [--reps 7] [--keyframes 100]

Needs a CUDA device: without one it stops with an error before timing."""
import argparse
import json
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tools.tsdf_readout_bench import gpu_card  # noqa: E402


def room_keyframes(n, W=640, H=480, step=2):
    """ground-truth keyframes k = 0, step, 2 step, ... of the synthetic room -> cam_T_world [n,7], inverse depths,
    variances [n,H,W] fp32, images [n,3,H,W] u8, intrinsics fx, fy, cx, cy"""
    from nerf_slam_b200.frontend import matrix_to_tq
    from nerf_slam_b200.synthetic import SyntheticRoom
    room = SyntheticRoom(W, H, n * step, seed=0)
    poses = np.empty((n, 7), np.float32)
    idepth = np.empty((n, H, W), np.float32)
    images = np.empty((n, 3, H, W), np.uint8)
    for i in range(n):
        rgba, d16, w2c = room.render(i * step)
        poses[i] = matrix_to_tq(np.asarray(w2c, np.float64))
        idepth[i] = 1.0 / (d16[..., 0].astype(np.float32) * np.float32(room.calib.depth_scale))
        images[i] = rgba[..., :3].transpose(2, 0, 1)
    cov = ((0.1 / idepth ** 2) ** 2).astype(np.float32)
    return poses, idepth, cov, images, room.calib.camera_model.numpy().astype(np.float32)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--keyframes", type=int, default=100)
    a = ap.parse_args()
    import torch
    from nerf_slam_b200 import _lib
    from nerf_slam_b200.point_cloud import build_point_cloud
    _lib.load()                                            # raises NslamUnavailable without CUDA: no fallback
    dev = "cuda:0"
    poses, idepth, cov, images, intr = room_keyframes(a.keyframes)
    T = lambda x: torch.from_numpy(x).to(dev)
    packet = {"cam0_poses": T(poses), "cam0_idepths_up": T(idepth), "cam0_depths_cov_up": T(cov), "cam0_images": T(images)}
    K = T(intr)

    def run(cfg):
        return build_point_cloud(packet, K, **cfg)

    result = {}
    for name, cfg in (("cloud", {}), ("cloud_filter", {"filter_thresh": 0.05, "min_views": 2}),
                      ("cloud_voxel_1cm", {"voxel_size": 0.01})):
        for _ in range(2):
            run(cfg)
        torch.cuda.synchronize()
        ts = []
        for _ in range(a.reps):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            pc = run(cfg)
            e1.record()
            torch.cuda.synchronize()
            ts.append(e0.elapsed_time(e1))
        del pc
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        pc = run(cfg)
        torch.cuda.synchronize()
        result[name] = {"ms": round(float(np.median(ts)), 3), "ms_min": round(float(np.min(ts)), 3),
                        "points_out": len(pc), "peak_bytes": int(torch.cuda.max_memory_allocated() - base)}
        if pc.counts is not None:
            result[name]["points_merged"] = int(pc.counts.sum())
        del pc
    name, power = gpu_card()
    print(json.dumps({"bench": "point_cloud", "gpu": name or torch.cuda.get_device_name(0), "power_limit": power,
                      "keyframes": a.keyframes, "hw": list(idepth.shape[1:]), "points_in": int(idepth.size),
                      "mask": "uncertainty", "reps": a.reps, **result}))


if __name__ == "__main__":
    main()
