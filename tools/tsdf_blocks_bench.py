"""Time the voxel-block volume against the dense 512^3 grid on the standard synthetic room (6 x 4 x 6 m, 640x480 views,
the reference's 6/512 m voxel), in one invocation: per-keyframe integration (for blocks: activation, the one host read,
insertion and integration), build_mesh, a 10-view render_volume, peak device memory and the block count.  Medians of
CUDA-event timings after warm-up.  Prints one JSON line with the card's name and power limit.

    python tools/tsdf_blocks_bench.py [--reps 5] [--frames 40]

Needs a CUDA device: without one it stops with an error before fusing."""
import argparse
import json
import os
import sys
import types

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tools.tsdf_readout_bench import gpu_card  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
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
    _lib.load()                                            # raises NslamUnavailable without CUDA: no fallback
    dev = "cuda:0"
    packets = []
    for k in range(0, a.frames, max(1, a.frames // 10)):
        p = room.packet(k)
        calib = p["calibs"][0]
        raw = torch.from_numpy(p["depths"][0, ..., 0].astype(np.float32)).to(dev)
        depth = raw * calib.depth_scale
        packets.append({"is_last_frame": False, "kf_idx": k, "viz_idx": torch.tensor([k], device=dev), "viz_idx_host": [k],
                        "kf_idx_to_f_idx": {k: k}, "calibs": p["calibs"],
                        "cam0_poses": torch.from_numpy(matrix_to_tq(np.asarray(p["poses"][0], np.float64))[None]).float().to(dev),
                        "cam0_idepths_up": (1.0 / depth)[None], "cam0_depths_cov_up": torch.full((1, H, W), 0.04, device=dev),
                        "cam0_images": torch.from_numpy(p["images"][..., :3]).permute(0, 3, 1, 2).contiguous().to(dev),
                        "cam0_intrinsics": torch.from_numpy(calib.camera_model.numpy() / 8.0)[None].float().to(dev),
                        "gt_depths": raw[None, None]})

    def event_ms(fn):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        out = fn()
        e1.record()
        torch.cuda.synchronize()
        return out, e0.elapsed_time(e1)

    def timed(fn):
        for _ in range(2):
            fn()
        torch.cuda.synchronize()
        ts = [event_ms(fn)[1] for _ in range(a.reps)]
        return float(np.median(ts))

    result = {}
    for mode in ("dense", "blocks"):
        torch.cuda.empty_cache()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        args = types.SimpleNamespace(eval=False, tsdf_volume=mode, tsdf_resolution=512, tsdf_center=(0.0, 0.0, 0.0))
        fus = TsdfFusion("sigma", args, dev)
        fus.fuse({"slam": [None, packets[0]]})             # warm-up keyframe, then a fresh volume
        fus.initialize()
        torch.cuda.synchronize()
        ts = []
        for pkt in packets:
            ts.append(event_ms(lambda: fus.fuse({"slam": [None, pkt]}))[1])
        integrate_ms = float(np.median(ts))
        mesh_ms = timed(lambda: fus.build_mesh(0.5))
        mesh = fus.build_mesh(0.5)
        packet = fus.get_history_packet()
        render_ms = timed(lambda: fus.render_volume(packet, fus.intrinsics, fus.min_weight_for_render,
                                                    fus.max_depth_sigma_thresh))
        torch.cuda.synchronize()
        result[mode] = {"integrate_ms_per_keyframe": round(integrate_ms, 3), "mesh_ms": round(mesh_ms, 3),
                        "render_ms_10_views": round(render_ms, 3), "vertices": int(mesh.vertices.shape[0]),
                        "peak_bytes": int(torch.cuda.max_memory_allocated() - base)}
        if mode == "blocks":
            result[mode]["blocks"] = fus.volume.n_blocks
            result[mode]["capacity"] = fus.volume.capacity
        del fus, mesh
    name, power = gpu_card()
    print(json.dumps({"bench": "tsdf_blocks", "gpu": name or torch.cuda.get_device_name(0), "power_limit": power,
                      "room_m": [6, 4, 6], "hw": [H, W], "voxel_m": 6.0 / 512, "keyframes": len(packets), **result}))


if __name__ == "__main__":
    main()
