"""Clean and simplify a triangle mesh on the GPU (nerf_slam_b200.mesh_ops) and write it as a PLY file.

    python tools/clean_mesh.py in.ply out.ply [--views transforms.json] [--min_component_area A] [--voxel V]

In order: with --views, the mesh is culled to the frames of a NeRF-style transforms.json, with occlusion taken from its
own depth rendered at those frames (mesh_ops.cull; a face goes when none of its vertices is seen); with
--min_component_area, connected components smaller than A m^2 are dropped; with --voxel, the mesh is simplified by
vertex clustering on cells of V metres.  Vertex colours are read when the file has them (0 otherwise); the normals
written are the area-weighted vertex normals (mesh_ops.vertex_normals) of the input, carried over by culling and
component removal and recomputed by clustering.  Prints one JSON line with the vertex and triangle counts.

Needs a CUDA device."""
import argparse
import json
import math
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))


def parse_args(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("input")
    ap.add_argument("output")
    ap.add_argument("--views", default=None, help="transforms.json whose frames to cull the mesh to")
    ap.add_argument("--min_component_area", type=float, default=None,
                    help="drop connected components smaller than this (m^2)")
    ap.add_argument("--voxel", type=float, default=None, help="vertex-clustering cell size (m)")
    a = ap.parse_args(argv)
    if a.min_component_area is not None and not (math.isfinite(a.min_component_area) and a.min_component_area >= 0):
        ap.error(f"--min_component_area must be finite and >= 0, got {a.min_component_area}")
    if a.voxel is not None and not (math.isfinite(a.voxel) and a.voxel > 0):
        ap.error(f"--voxel must be positive and finite, got {a.voxel}")
    return a


def main(argv=None):
    a = parse_args(argv)
    import torch
    from nerf_slam_b200 import mesh_ops
    from nerf_slam_b200.evaluation import read_ply
    from nerf_slam_b200.mesh_render import MeshScene
    from nerf_slam_b200.tsdf_fusion import TsdfMesh
    v, t, c = read_ply(a.input, return_colors=True)
    if t is None or not len(t):
        raise SystemExit(f"{a.input} has no faces")
    dev = torch.device("cuda", torch.cuda.current_device())
    V, T = torch.from_numpy(v).to(dev), torch.from_numpy(t).to(dev)
    C = torch.from_numpy(c).to(dev) if c is not None else torch.zeros_like(V)
    mesh = TsdfMesh(V, T, C, mesh_ops.vertex_normals((V, T)))
    counts = {"input_vertices": int(V.shape[0]), "input_triangles": int(T.shape[0])}
    if a.views:
        from eval_reconstruction import dataset_views
        poses, intr, W, H = dataset_views(a.views)
        depth = MeshScene(mesh).render(poses, intr, W, H).depth
        mesh = mesh_ops.cull(mesh, poses, intr, W, H, depths=depth)
        del depth
    if mesh is not None and a.min_component_area is not None:
        mesh = mesh_ops.remove_small_components(mesh, a.min_component_area)
    if mesh is not None and a.voxel is not None:
        mesh = mesh_ops.simplify_vertex_clustering(mesh, a.voxel)
    if mesh is None:
        raise SystemExit("no triangle remains: nothing written")
    mesh.write_ply(a.output)
    print(json.dumps({"input": a.input, "output": a.output, **counts, "vertices": int(mesh.vertices.shape[0]),
                      "triangles": int(mesh.triangles.shape[0])}))


if __name__ == "__main__":
    main()
