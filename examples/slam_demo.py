#!/usr/bin/env python3
"""The reference's entry point (examples/slam_demo.py) on the sm_90a implementation: same command line, e.g.

  python examples/slam_demo.py --dataset_dir=DIR --dataset_name=nerf --buffer=100 --slam --fusion=nerf [--eval]
  python examples/slam_demo.py --dataset_dir=synthetic --dataset_name=nerf --buffer=100 --slam --fusion=nerf

(`--dataset_dir=synthetic`: the procedural stream of nerf_slam_b200.synthetic instead of files; write it to disk in the
reference's format with nerf_slam_b200.datasets.write_transforms_dataset to feed the reference's own CLI.)

What differs from the reference (examples/slam_demo.py:57-191): one process per GPU instead of a process per module —
data, SLAM and fusion run in this process on streams of one GPU (the sequential branch, :160-181, without its queues);
with `--multi_gpu` launch it under torchrun with 2+ ranks (rank 0 = SLAM, other ranks = NeRF trainers, NCCL hand-off;
see bench.py / nerf_slam_b200.dist).  Out of scope, rejected with a message: euroc / real datasets, the Open3D GUI.
The reference's own examples/slam_demo.py also runs unchanged with `nerf_slam_b200/shim` first on PYTHONPATH
(tests/test_cpu_shim.py, tests/test_gpu_demo.py)."""
import argparse
import os
import sys
import time

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))


def parse_args(argv=None):
    """same options and defaults as the reference's parse_args (examples/slam_demo.py:20-55)"""
    p = argparse.ArgumentParser(description="Instant-SLAM")
    p.add_argument("--parallel_run", action="store_true", help="Whether to run in parallel")
    p.add_argument("--multi_gpu", action="store_true", help="Whether to run with multiple (two) GPUs")
    p.add_argument("--initial_k", type=int, help="Initial frame to parse in the dataset", default=0)
    p.add_argument("--final_k", type=int, help="Final frame to parse in the dataset, -1 is all.", default=-1)
    p.add_argument("--img_stride", type=int, help="Number of frames to skip when parsing the dataset", default=1)
    p.add_argument("--stereo", action="store_true", help="Use stereo images")
    p.add_argument("--weights", default="droid.pth", help="Path to the weights file")
    p.add_argument("--buffer", type=int, default=512, help="Number of keyframes to keep")
    p.add_argument("--dataset_dir", type=str, help="Path to the dataset directory", default="/home/tonirv/Datasets/euroc/V1_01_easy")
    p.add_argument("--dataset_name", type=str, default="euroc", choices=["euroc", "nerf", "replica", "real"], help="Dataset format to use.")
    p.add_argument("--mask_type", type=str, default="ours", choices=["no_depth", "raw", "ours", "ours_w_thresh"])
    p.add_argument("--slam", action="store_true", help="Run SLAM.")
    p.add_argument("--fusion", type=str, default="", choices=["tsdf", "sigma", "nerf", ""], help="Fusion approach ('' for none)")
    p.add_argument("--gui", action="store_true", help="Run O3D Gui, use when volume='tsdf'or'sigma'.")
    p.add_argument("--width", "--screenshot_w", type=int, default=0, help="Resolution width of GUI and screenshots.")
    p.add_argument("--height", "--screenshot_h", type=int, default=0, help="Resolution height of GUI and screenshots.")
    p.add_argument("--network", default="", help="Path to the network config. Uses the scene's default if unspecified.")
    p.add_argument("--eval", action="store_true", help="Evaluate method.")
    p.add_argument("--tsdf_volume", type=str, default="dense", choices=["dense", "blocks"],
                   help="--fusion=tsdf/sigma volume: a dense grid, or unbounded 16^3 voxel blocks allocated where depth reaches")
    p.add_argument("--tsdf_block_count", type=int, default=5000, help="initial block capacity of --tsdf_volume=blocks")
    # additions (not in the reference): bounds for a non-interactive run
    p.add_argument("--synthetic_frames", type=int, default=200, help="frames of the procedural stream (--dataset_dir=synthetic)")
    p.add_argument("--nerf_iters_per_frame", type=int, default=2, help="NeRF training steps interleaved per input frame")
    p.add_argument("--fit_iters_after", type=int, default=0, help="NeRF training steps after the stream has ended")
    return p.parse_args(argv)


def make_data(args):
    if args.dataset_name not in ("nerf", "replica"):
        raise NotImplementedError(f"dataset format '{args.dataset_name}' is outside the hot-path scope (DESIGN.md): use 'nerf'")
    if args.dataset_dir == "synthetic":
        from nerf_slam_b200.synthetic import SyntheticRoom
        import numpy as np
        room = SyntheticRoom(640, 480, args.synthetic_frames, seed=0)
        args.world_T_imu_t0 = np.asarray(room.packet(0)["poses"][0])
        return room
    from nerf_slam_b200.datasets import NeRFDataset
    # NB: like the reference, the default --final_k=-1 slices frames[initial_k:-1:stride] and so drops the last frame
    # (datasets/nerf_dataset.py:65); kept for identical streams
    return NeRFDataset(args, "cpu")


def run(args):
    import numpy as np
    import torch
    if args.gui:
        raise NotImplementedError("the Open3D GUI is outside the hot-path scope (DESIGN.md)")
    device = "cuda:0"
    data = make_data(args)
    if args.weights and not os.path.exists(args.weights):
        cand = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "oracle", "_ref", "droid.pth")
        args.weights = cand if os.path.exists(cand) else None
    slam = fusion = None
    if args.slam:
        from nerf_slam_b200.frontend import RaftVisualFrontend
        # first camera pose = prior and initial state (the commented-out intent of slam/vio_slam.py:92; the live code
        # hard-codes a Replica pose there)
        slam = RaftVisualFrontend(np.linalg.inv(np.asarray(args.world_T_imu_t0)), np.eye(4), args, device)
    if args.fusion == "nerf":
        from nerf_slam_b200.nerf_fusion import NerfFusion
        fusion = NerfFusion("nerf", args, device)
    elif args.fusion in ("tsdf", "sigma"):
        from nerf_slam_b200.tsdf_fusion import TsdfFusion
        fusion = TsdfFusion(args.fusion, args, device)
    t0 = time.perf_counter()
    frames = 0
    for packet in data.stream():
        frames += 1
        out = None
        if slam is not None:
            x0, factors, viz_out = slam(packet)
            out = [None, viz_out]
        if fusion is not None:
            fusion.fuse({"slam": out} if slam is not None else {"data": packet})
            if args.fusion == "nerf":
                for _ in range(max(args.nerf_iters_per_frame - 1, 0)):
                    fusion.fit_volume_once()
        if slam is not None and slam.stop_condition():
            break
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    print(f"{frames} frames in {dt:.2f} s ({frames / dt:.1f} frames/s)"
          + (f", {slam.kf_idx} keyframes, {slam.stats['updates']} update() calls" if slam is not None else "")
          + (f", {fusion.total_iters} NeRF iterations" if args.fusion == "nerf" else "")
          + (f", {fusion.integrated_frames} keyframe integrations into the {args.fusion} volume" if args.fusion in ("tsdf", "sigma") else ""))
    if args.fusion == "nerf":
        for _ in range(args.fit_iters_after):
            fusion.fit_volume_once()
        if args.eval:
            print("eval:", fusion.eval_gt_traj())
    return slam, fusion


if __name__ == "__main__":
    run(parse_args())
