"""Score a reconstruction against ground truth on the GPU (nerf_slam_b200.evaluation.reconstruction_metrics) and print
one JSON line: accuracy, completion, chamfer_l1 (metres), precision, recall, f_score at the threshold, and the point
counts.  Either file may be a mesh (a PLY with faces: sampled uniformly by area) or a point cloud (used as it is).

    python tools/eval_reconstruction.py rec.ply gt.ply [--threshold 0.05] [--samples 200000] [--max_dist 1.0] [--seed 0]
                                        [--views transforms.json] [--cull] [--min_component_area A]
                                        [--align icp|icp_sim3] [--align_metric point_to_plane|point_to_point]
                                        [--align_max_dist 0.2,0.1,0.05] [--init T.json]

With --views, both meshes are also rendered at the frames of a NeRF-style transforms.json (poses and intrinsics parsed
as datasets.NeRFDataset does) and the line gains `mesh_depth_l1` (evaluation.mesh_depth_l1 with the same max_dist).

--cull (needs --views and a ground-truth mesh) scores only what the cameras saw: the ground-truth mesh is rendered at
the views, the reconstruction mesh is culled with that depth (mesh_ops.cull, a face goes when none of its vertices is
seen) and the ground-truth samples are masked with it (evaluation.visible).  --min_component_area then drops the
reconstruction's connected components smaller than A m^2 (mesh_ops.remove_small_components).  Without these flags the
reconstruction is scored as it is.

--align first moves the reconstruction into the ground truth's frame (registration.icp from the reconstruction to the
ground truth, then registration.transform): "icp" fits a rigid transform, "icp_sim3" also the scale, as a monocular
SLAM map needs.  --align_metric picks point-to-plane (default; needs a ground-truth mesh) or point-to-point ICP,
--align_max_dist its coarse-to-fine correspondence distances (metres), --init a JSON 4x4 similarity to start from (e.g.
registration.trajectory_alignment of the SLAM and true poses).  Alignment runs before culling and scoring, with the same
--samples and --seed, and the line gains a `registration` object.  Without --align the output is unchanged.

Needs a CUDA device."""
import argparse
import json
import math
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
    ap.add_argument("--cull", action="store_true", help="score only what the --views cameras saw")
    ap.add_argument("--min_component_area", type=float, default=None,
                    help="drop the reconstruction's connected components smaller than this (m^2)")
    ap.add_argument("--align", choices=("icp", "icp_sim3"), default=None,
                    help="align the reconstruction to the ground truth first: rigid (icp) or with scale (icp_sim3)")
    ap.add_argument("--align_metric", choices=("point_to_plane", "point_to_point"), default=None,
                    help="ICP metric (default point_to_plane)")
    ap.add_argument("--align_max_dist", default=None, help="comma-separated correspondence distances, coarse to fine (m)")
    ap.add_argument("--init", default=None, help="JSON file with a 4x4 similarity to start the alignment from")
    a = ap.parse_args(argv)
    if a.cull and not a.views:
        ap.error("--cull needs --views")
    if not a.align and (a.align_metric or a.align_max_dist is not None or a.init):
        ap.error("--align_metric, --align_max_dist and --init need --align")
    if a.align_max_dist is not None:
        try:
            a.align_max_dist = [float(d) for d in a.align_max_dist.split(",")]
        except ValueError:
            ap.error(f"--align_max_dist must be comma-separated numbers, got {a.align_max_dist!r}")
        if not all(math.isfinite(d) and d > 0 for d in a.align_max_dist):
            ap.error(f"--align_max_dist must be positive and finite, got {a.align_max_dist}")
    if a.init:
        a.init = read_init(a.init, ap)
    if a.min_component_area is not None and not (math.isfinite(a.min_component_area) and a.min_component_area >= 0):
        ap.error(f"--min_component_area must be finite and >= 0, got {a.min_component_area}")
    from nerf_slam_b200.evaluation import read_ply, reconstruction_metrics

    def load(path):
        v, t = read_ply(path)
        return (v, t) if t is not None and len(t) else v

    rec, gt = load(a.reconstruction), load(a.ground_truth)
    registration = align(rec, gt, a) if a.align else None
    if registration is not None:
        rec = registration.pop("moved")
    gt_mask = None
    cleaned = a.cull or a.min_component_area is not None
    if cleaned:
        rec, gt_mask = clean_reconstruction(rec, gt, a)
    m = reconstruction_metrics(rec, gt, threshold=a.threshold, n_samples=a.samples, max_dist=a.max_dist, seed=a.seed,
                               gt_mask=gt_mask)
    out = {"reconstruction": a.reconstruction, "ground_truth": a.ground_truth, **m}
    if a.views and not cleaned and not a.align:
        out["mesh_depth_l1"] = depth_at_views(a.reconstruction, a.ground_truth, a.views, a.max_dist)
    elif a.views:
        from nerf_slam_b200.evaluation import mesh_depth_l1
        if not isinstance(gt, tuple):
            raise SystemExit(f"--views renders meshes: {a.ground_truth} has no faces")
        poses, intr, W, H = dataset_views(a.views)
        out["mesh_depth_l1"] = mesh_depth_l1(rec, gt, poses, intr, W, H, max_dist=a.max_dist)
    if registration is not None:
        out["registration"] = registration
    print(json.dumps(out))


def read_init(path, ap=None):
    """-> the 4x4 similarity in a JSON file (a list of 4 rows), refused when it is not one"""
    import numpy as np
    from nerf_slam_b200.registration import decompose
    fail = ap.error if ap is not None else SystemExit
    try:
        with open(path) as f:
            T = np.asarray(json.load(f), np.float64)
        decompose(T, "--init")
    except (OSError, ValueError, TypeError) as e:
        raise fail(f"--init {path}: {e}")
    return T


def align(rec, gt, a):
    """-> the registration object of the output line, with the moved reconstruction under "moved" """
    from nerf_slam_b200 import registration
    kw = {} if a.align_max_dist is None else {"max_corr_dist": a.align_max_dist}
    metric = a.align_metric or "point_to_plane"
    if metric == "point_to_plane" and not isinstance(gt, tuple):
        raise SystemExit(f"--align_metric point_to_plane needs a ground-truth mesh: {a.ground_truth} has no faces")
    r = registration.icp(rec, gt, init=a.init, metric=metric, with_scale=a.align == "icp_sim3", n_samples=a.samples,
                         seed=a.seed, **kw)
    return {"moved": registration.transform(rec, r.transform), "method": a.align, "metric": metric,
            "transform": r.transform.tolist(), "scale": r.scale, "fitness": r.fitness, "inlier_rmse": r.inlier_rmse,
            "iterations": r.iterations, "converged": r.converged, "degenerate": r.degenerate}


def clean_reconstruction(rec, gt, a):
    """-> (the reconstruction culled to the views by the ground truth's rendered depth and / or without its small
    components, the ground-truth mask under --cull or None)"""
    from nerf_slam_b200 import mesh_ops
    from nerf_slam_b200.evaluation import visible
    from nerf_slam_b200.mesh_render import MeshScene
    if not isinstance(rec, tuple):
        raise SystemExit(f"--cull and --min_component_area act on meshes: {a.reconstruction} has no faces")
    gt_mask = None
    if a.cull:
        if not isinstance(gt, tuple):
            raise SystemExit(f"--cull renders the ground truth: {a.ground_truth} has no faces")
        poses, intr, W, H = dataset_views(a.views)
        gt_depth = MeshScene(gt).render(poses, intr, W, H).depth
        rec = mesh_ops.cull(rec, poses, intr, W, H, depths=gt_depth)
        gt_mask = lambda p: visible(p, poses, intr, W, H, depths=gt_depth)  # noqa: E731
    if rec is not None and a.min_component_area is not None:
        rec = mesh_ops.remove_small_components(rec, a.min_component_area)
    if rec is None:
        raise SystemExit("no triangle of the reconstruction remains after cleaning")
    return rec, gt_mask


def dataset_views(views):
    """-> cam_T_world [n,7] fp32, intrinsics fx fy cx cy, width, height of the frames of a transforms.json"""
    import numpy as np
    from nerf_slam_b200.datasets import NeRFDataset, dataset_args
    from nerf_slam_b200.frontend import matrix_to_tq
    ds = NeRFDataset(dataset_args(os.path.dirname(os.path.abspath(views)) or "."))
    cam, res = ds.calib.camera_model, ds.calib.resolution
    poses = np.asarray([matrix_to_tq(np.asarray(w2c, np.float64)) for w2c in ds.w2c], np.float32)
    return poses, cam.numpy(), res.width, res.height


def depth_at_views(rec_path, gt_path, views, max_dist):
    """evaluation.mesh_depth_l1 of two PLY meshes at the frames of a transforms.json"""
    from nerf_slam_b200.evaluation import mesh_depth_l1, read_ply
    poses, intr, W, H = dataset_views(views)
    meshes = []
    for path in (rec_path, gt_path):
        v, t = read_ply(path)
        if t is None or not len(t):
            raise SystemExit(f"--views renders meshes: {path} has no faces")
        meshes.append((v, t))
    return mesh_depth_l1(meshes[0], meshes[1], poses, intr, W, H, max_dist=max_dist)


if __name__ == "__main__":
    main()
