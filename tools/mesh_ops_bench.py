"""Time the mesh operations (csrc/mesh_ops.cu) on two meshes of the synthetic room at 512^3: the NeRF mesh of the room
trained as in tests/test_gpu_nerf_mesh.py (12 views, 300 steps, thresh 10; floaters included) and the dense TSDF mesh
fused from 10 of its 640x480 views.  Each operation: CUDA events, median of --reps after two warm-up calls, and the
bytes it must move at least (its inputs read once and its outputs written once, from the shapes below) over that time.
Prints one JSON line with the card's name and power limit, read in the same run.

    python tools/mesh_ops_bench.py [--reps 5] [--res 512]

Needs a CUDA device: without one it stops with an error before timing."""
import argparse
import json
import os
import sys
import types

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tools.tsdf_readout_bench import gpu_card  # noqa: E402

W, H = 640, 480


def min_bytes(op, nv, nt, out_v=0, out_t=0, n_views=0):
    """the least traffic of each operation: vertices 12 B, triangles 12 B, colours and normals 12 B each per vertex"""
    mesh_in = 12 * nv + 12 * nt
    mesh_out = 36 * out_v + 12 * out_t
    return {"components": mesh_in + 4 * nt,                          # + labels
            "submesh": 36 * nv + 12 * nt + nt + mesh_out,             # + the keep mask
            "remove_small_components": 36 * nv + 12 * nt + mesh_out,
            "cull": 36 * nv + 12 * nt + 4 * n_views * W * H + mesh_out,
            "vertex_normals": mesh_in + 12 * nv,
            "simplify_vertex_clustering": 24 * nv + 12 * nt + mesh_out}[op]


def room_meshes(res, dev):
    """-> the trained NeRF room's mesh with its 12 views (cam_T_world [12,7], intrinsics, (W, H)) and the dense TSDF mesh
    of 10 room views with its views (cam_T_world [10,7], intrinsics), both at res^3"""
    import torch
    from nerf_slam_b200.frontend import matrix_to_tq
    from nerf_slam_b200.nerf_fusion import NerfFusion
    from nerf_slam_b200.synthetic import SyntheticRoom
    from nerf_slam_b200.tsdf_fusion import TsdfFusion
    T = lambda x: torch.from_numpy(np.ascontiguousarray(x)).to(dev)  # noqa: E731

    # the trained NeRF room (tests/test_gpu_nerf_mesh.py's fixture)
    nroom = SyntheticRoom(160, 120, 12, seed=0, half_extent=(1.4, 1.0, 1.4), orbit_radius=0.3, step=0.25)
    nf = NerfFusion("nerf", types.SimpleNamespace(buffer=12, eval=False, mask_type="ours"), dev)
    nf.ngp.nerf.training.depth_supervision_lambda = 1.0
    nf.gt_fit_convention = "metric"
    pk = [nroom.packet(k) for k in range(12)]
    nf.fuse({"data": {"k": np.arange(12), "poses": np.stack([p["poses"][0] for p in pk]),
                      "images": np.stack([p["images"][0] for p in pk]), "depths": np.stack([p["depths"][0] for p in pk]),
                      "calibs": pk[0]["calibs"]}})
    for _ in range(300):
        nf.fit_volume_once()
    nerf_mesh = nf.ngp.marching_cubes(res, None, 10.0)
    nerf_poses = T(np.asarray([matrix_to_tq(np.asarray(nroom.render(k)[2], np.float64)) for k in range(12)], np.float32))
    nerf_intr, nerf_wh = nroom.calib.camera_model.numpy().astype(np.float32), (nroom.W, nroom.H)
    del nf
    torch.cuda.empty_cache()

    # the dense TSDF of 10 room views
    room = SyntheticRoom(W, H, 200, seed=0)
    intr = room.calib.camera_model.numpy().astype(np.float32)
    ks = list(range(0, 200, 20))
    poses = T(np.asarray([matrix_to_tq(np.asarray(room.render(k)[2], np.float64)) for k in ks], np.float32))
    fus = TsdfFusion("tsdf", types.SimpleNamespace(eval=False, tsdf_volume="dense", tsdf_resolution=res), dev)
    fus.voxel_size = 8.0 / res
    fus.initialize()
    depths = np.stack([room.render(k)[1][..., 0].astype(np.float32) * np.float32(room.calib.depth_scale) for k in ks])
    images = np.stack([room.render(k)[0][..., :3].transpose(2, 0, 1) for k in ks])
    fus.build_volume({"cam0_poses": poses, "cam0_idepths_up": T(1.0 / depths), "cam0_depths_cov_up": None,
                      "cam0_images": T(images)}, intr, None)
    tsdf_mesh = fus.build_mesh(0.5)
    fus.volume = None
    torch.cuda.empty_cache()
    return nerf_mesh, nerf_poses, nerf_intr, nerf_wh, tsdf_mesh, poses, intr


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--res", type=int, default=512)
    a = ap.parse_args()
    import torch
    from nerf_slam_b200 import _lib, mesh_ops
    from nerf_slam_b200.mesh_render import MeshScene
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

    nerf_mesh, nerf_poses, nerf_intr, nerf_wh, tsdf_mesh, poses, intr = room_meshes(a.res, dev)

    res = {}
    for label, mesh, p, K, (w, h) in (("nerf_mesh", nerf_mesh, nerf_poses, nerf_intr, nerf_wh),
                                      ("tsdf_mesh", tsdf_mesh, poses, intr, (W, H))):
        nv, nt = int(mesh.vertices.shape[0]), int(mesh.triangles.shape[0])
        depth = MeshScene(mesh).render(p, K, w, h).depth
        keep = torch.arange(nt, device=dev) % 2 == 0
        ops = {"components": lambda: mesh_ops.connected_components(mesh),
               "submesh": lambda: mesh_ops.submesh(mesh, keep),
               "remove_small_components": lambda: mesh_ops.remove_small_components(mesh, 0.01),
               "cull": lambda: mesh_ops.cull(mesh, p, K, w, h, depths=depth),
               "vertex_normals": lambda: mesh_ops.vertex_normals(mesh),
               "simplify_vertex_clustering": lambda: mesh_ops.simplify_vertex_clustering(mesh, 0.02)}
        r = {"vertices": nv, "triangles": nt}
        for op, fn in ops.items():
            out, ms = timed(fn)
            out_v = out_t = 0
            if hasattr(out, "vertices"):
                out_v, out_t = int(out.vertices.shape[0]), int(out.triangles.shape[0])
                r[f"{op}_out"] = [out_v, out_t]
            nb = min_bytes(op, nv, nt, out_v, out_t, int(p.shape[0]) if op == "cull" else 0)
            r[f"{op}_ms"] = round(ms, 3)
            r[f"{op}_min_GB_per_s"] = round(nb / ms / 1e6, 1)
        r["components"] = int(mesh_ops.connected_components(mesh)[1].shape[0])
        res[label] = r
        del depth
        torch.cuda.empty_cache()
    print(json.dumps({"bench": "mesh_ops", "gpu": name or torch.cuda.get_device_name(0), "power_limit": power,
                      "reps": a.reps, "res": a.res, **res}))


if __name__ == "__main__":
    main()
