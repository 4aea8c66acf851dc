"""Score a reconstruction against ground truth on the GPU (nerf_slam_b200.evaluation.reconstruction_metrics) and print
one JSON line: accuracy, completion, chamfer_l1 (metres), precision, recall, f_score at the threshold, and the point
counts.  Either file may be a mesh (a PLY with faces: sampled uniformly by area) or a point cloud (used as it is).

    python tools/eval_reconstruction.py rec.ply gt.ply [--threshold 0.05] [--samples 200000] [--max_dist 1.0] [--seed 0]

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
    a = ap.parse_args(argv)
    from nerf_slam_b200.evaluation import read_ply, reconstruction_metrics

    def load(path):
        v, t = read_ply(path)
        return (v, t) if t is not None and len(t) else v

    m = reconstruction_metrics(load(a.reconstruction), load(a.ground_truth), threshold=a.threshold,
                               n_samples=a.samples, max_dist=a.max_dist, seed=a.seed)
    print(json.dumps({"reconstruction": a.reconstruction, "ground_truth": a.ground_truth, **m}))


if __name__ == "__main__":
    main()
