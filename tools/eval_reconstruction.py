"""Score a reconstruction against ground truth on the GPU (nerf_slam_b200.evaluation.reconstruction_metrics) and print
one JSON line: accuracy, completion, chamfer_l1 (metres), precision, recall, f_score at the threshold, and the point
counts.  Either file may be a mesh (a PLY with faces: sampled uniformly by area) or a point cloud (used as it is).

    python tools/eval_reconstruction.py rec.ply gt.ply [--threshold 0.05] [--samples 200000] [--max_dist 1.0] [--seed 0]
                                        [--views transforms.json]

With --views, both meshes are also rendered at the frames of a NeRF-style transforms.json (poses and intrinsics parsed
as datasets.NeRFDataset does) and the line gains `mesh_depth_l1` (evaluation.mesh_depth_l1 with the same max_dist).

Needs a CUDA device."""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("reconstruction")
    ap.add_argument("ground_truth")
    ap.add_argument("--threshold", type=float, default=0.05, help="precision / recall threshold (m)")
    ap.add_argument("--samples", type=int, default=200_000, help="points sampled from each mesh")
    ap.add_argument("--max_dist", type=float, default=1.0, help="distances are clamped here in the means (m)")
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--views", default=None, help="transforms.json whose frames to render both meshes at")
    a = ap.parse_args(argv)
    from nerf_slam_b200.evaluation import read_ply, reconstruction_metrics

    def load(path):
        v, t = read_ply(path)
        return (v, t) if t is not None and len(t) else v

    m = reconstruction_metrics(load(a.reconstruction), load(a.ground_truth), threshold=a.threshold,
                               n_samples=a.samples, max_dist=a.max_dist, seed=a.seed)
    out = {"reconstruction": a.reconstruction, "ground_truth": a.ground_truth, **m}
    if a.views:
        out["mesh_depth_l1"] = depth_at_views(a.reconstruction, a.ground_truth, a.views, a.max_dist)
    print(json.dumps(out))


def depth_at_views(rec_path, gt_path, views, max_dist):
    """evaluation.mesh_depth_l1 of two PLY meshes at the frames of a transforms.json"""
    import numpy as np
    from nerf_slam_b200.datasets import NeRFDataset, dataset_args
    from nerf_slam_b200.evaluation import mesh_depth_l1, read_ply
    from nerf_slam_b200.frontend import matrix_to_tq
    ds = NeRFDataset(dataset_args(os.path.dirname(os.path.abspath(views)) or "."))
    cam, res = ds.calib.camera_model, ds.calib.resolution
    poses = np.asarray([matrix_to_tq(np.asarray(w2c, np.float64)) for w2c in ds.w2c], np.float32)
    meshes = []
    for path in (rec_path, gt_path):
        v, t = read_ply(path)
        if t is None or not len(t):
            raise SystemExit(f"--views renders meshes: {path} has no faces")
        meshes.append((v, t))
    return mesh_depth_l1(meshes[0], meshes[1], poses, cam.numpy(), res.width, res.height, max_dist=max_dist)


if __name__ == "__main__":
    main()
