"""Time the TSDF read-outs on a 512^3 volume fused from the synthetic room: TsdfFusion.build_mesh and a 10-view 640x480
TsdfFusion.render_volume (CUDA events after warm-up).  Prints one JSON line with the card's name and power limit, the times,
the mesh size and the bytes the algorithm needs.

    python tools/tsdf_readout_bench.py [--res 512] [--reps 5]

Needs a CUDA device: without one it stops with an error once the volume would have to be fused."""
import argparse
import json
import os
import subprocess
import sys
import types

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def gpu_card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = [s.strip() for s in out.split(",")]
        return name, power
    except Exception as e:                                # the name still comes from torch below
        return None, f"unavailable ({e.__class__.__name__})"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--res", type=int, default=512)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--frames", type=int, default=40)
    a = ap.parse_args()
    import torch
    from nerf_slam_b200 import _lib
    from nerf_slam_b200.frontend import matrix_to_tq
    from nerf_slam_b200.synthetic import SyntheticRoom
    from nerf_slam_b200.tsdf_fusion import TsdfFusion
    H, W = 480, 640
    room = SyntheticRoom(W, H, a.frames, seed=0)
    p0 = room.packet(0)                                    # host-side scene set-up works without a device
    _lib.load()                                            # raises NslamUnavailable without CUDA: no fallback
    dev = "cuda:0"
    fus = TsdfFusion("sigma", types.SimpleNamespace(eval=False, tsdf_resolution=a.res, tsdf_center=(0.0, 0.0, 0.0)), dev)
    fus.voxel_size = 8.0 / a.res; fus.initialize()        # the room is 6 x 4 x 6 m
    step = max(1, a.frames // 10)
    for k in range(0, a.frames, step):
        p = p0 if k == 0 else room.packet(k)
        calib = p["calibs"][0]
        raw = torch.from_numpy(p["depths"][0, ..., 0].astype(np.float32)).to(dev)
        depth = raw * calib.depth_scale
        pkt = {"is_last_frame": False, "kf_idx": k, "viz_idx": torch.tensor([k], device=dev), "viz_idx_host": [k],
               "kf_idx_to_f_idx": {k: k}, "calibs": p["calibs"],
               "cam0_poses": torch.from_numpy(matrix_to_tq(np.asarray(p["poses"][0], np.float64))[None]).float().to(dev),
               "cam0_idepths_up": (1.0 / depth)[None], "cam0_depths_cov_up": torch.full((1, H, W), 0.04, device=dev),
               "cam0_images": torch.from_numpy(p["images"][..., :3]).permute(0, 3, 1, 2).contiguous().to(dev),
               "cam0_intrinsics": torch.from_numpy(calib.camera_model.numpy() / 8.0)[None].float().to(dev),
               "gt_depths": raw[None, None]}
        fus.fuse({"slam": [None, pkt]})
    packet = fus.get_history_packet()
    n_views = packet["cam0_poses"].shape[0]
    torch.cuda.synchronize()

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
        return out, float(np.median(ts)), float(min(ts))

    mesh, mesh_ms, mesh_min = timed(lambda: fus.build_mesh(0.5))
    args = (packet, fus.intrinsics, fus.min_weight_for_render, fus.max_depth_sigma_thresh)
    (depth, _), render_ms, render_min = timed(lambda: fus.render_volume(*args))
    nvox = a.res ** 3
    V, T = mesh.vertices.shape[0], mesh.triangles.shape[0]
    # bytes the mesh algorithm needs: the classify and compaction passes each read tsdf + weight (8 B/voxel), plus the
    # surface: vertex positions, colours, normals (36 B) and triangles (12 B)
    mesh_bytes = 2 * 8 * nvox + V * 36 + T * 12
    name, power = gpu_card()
    print(json.dumps({
        "bench": "tsdf_readout", "gpu": name or torch.cuda.get_device_name(0), "power_limit": power,
        "grid": [a.res] * 3, "voxel_m": fus.voxel_size, "fused_views": n_views,
        "mesh_ms": round(mesh_ms, 3), "mesh_ms_min": round(mesh_min, 3), "vertices": V, "triangles": T,
        "mesh_bytes_needed": mesh_bytes, "mesh_GBps": round(mesh_bytes / (mesh_ms * 1e6), 1),
        "render_views": n_views, "render_hw": [H, W], "render_ms": round(render_ms, 3), "render_ms_min": round(render_min, 3),
        "render_hit_fraction": round(float((depth > 0).float().mean()), 4)}))


if __name__ == "__main__":
    main()
