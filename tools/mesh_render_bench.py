"""Time the triangle-mesh renderer (csrc/mesh_render.cu): the BVH build and depth rendering of 10 and 100 views at
640x480 for three meshes -- the synthetic room's exact surface (12 triangles), the dense TSDF mesh of the room fused from
10 of its views at 512^3, and the mesh of a NeRF (a random network's level set) at 512^3 -- with the TSDF ray cast of
the same 10 views (`render_volume`) beside it as context.  CUDA events, median of --reps after two warm-up calls; peak
device memory above what was allocated before each call.  Prints one JSON line with the card's name and power limit.

    python tools/mesh_render_bench.py [--reps 5] [--res 512]

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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--res", type=int, default=512)
    a = ap.parse_args()
    import torch
    from nerf_slam_b200 import _lib, pyngp
    from nerf_slam_b200.evaluation import _camera_centres
    from nerf_slam_b200.frontend import matrix_to_tq
    from nerf_slam_b200.mesh_render import MeshScene
    from nerf_slam_b200.pyngp import mesh_lattice
    from nerf_slam_b200.synthetic import SyntheticRoom
    from nerf_slam_b200.tsdf_fusion import TsdfFusion
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
        return out, round(float(np.median(ts)), 3)

    def peak(fn):
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        out = fn()
        torch.cuda.synchronize()
        return out, int(torch.cuda.max_memory_allocated() - base)

    room = SyntheticRoom(W, H, 200, seed=0)
    intr = room.calib.camera_model.numpy().astype(np.float32)
    views = lambda ks: torch.from_numpy(np.asarray(  # noqa: E731
        [matrix_to_tq(np.asarray(room.render(k)[2], np.float64)) for k in ks], np.float32)).to(dev)
    poses10, poses100 = views(range(0, 200, 20)), views(range(0, 200, 2))

    # the dense TSDF of 10 room views
    fus = TsdfFusion("tsdf", types.SimpleNamespace(eval=False, tsdf_volume="dense", tsdf_resolution=a.res), dev)
    fus.voxel_size = 8.0 / a.res
    fus.initialize()
    ks = list(range(0, 200, 20))
    depths = np.stack([room.render(k)[1][..., 0].astype(np.float32) * np.float32(room.calib.depth_scale) for k in ks])
    images = np.stack([room.render(k)[0][..., :3].transpose(2, 0, 1) for k in ks])
    T = lambda x: torch.from_numpy(np.ascontiguousarray(x)).to(dev)  # noqa: E731
    pk = {"cam0_poses": poses10, "cam0_idepths_up": T(1.0 / depths), "cam0_depths_cov_up": None, "cam0_images": T(images)}
    fus.build_volume(pk, intr, None)
    tsdf_mesh = fus.build_mesh(0.5)
    _, render_volume_ms = timed(lambda: fus.render_volume(pk, intr, fus.min_weight_for_render, fus.max_depth_sigma_thresh))
    fus.volume = None
    torch.cuda.empty_cache()

    # a NeRF mesh (a random network's level set) inside its own box; the room's views look at it from its centre
    tb = pyngp.Testbed(seed=4, max_samples=1 << 16, max_rays=1 << 13)
    tb.create_empty_nerf_dataset(8, 1.0, None, 4, None)
    g = torch.Generator().manual_seed(4)
    tb.grid_master.copy_(((torch.rand(tb.grid_master.shape, generator=g) * 2 - 1) * 0.5).to(dev))
    tb.grid_half.copy_(tb.grid_master.half())
    tb.pack_weights()
    tb.density.copy_(torch.where(torch.rand(tb.density.shape, generator=g) < 0.7, 0.0, -1.0).to(dev))
    lo, h, dims = mesh_lattice(64, None, tb.aabb_scale)
    field, weight = tb.mesh_kernels.lattice(tb, lo, h, dims, 0.0)
    thresh = float(torch.quantile(-field[weight > 0], 0.5))
    del field, weight
    nerf_mesh = tb.marching_cubes(a.res, None, thresh)
    del tb
    torch.cuda.empty_cache()
    V = nerf_mesh.vertices
    centre = ((V.min(0).values + V.max(0).values) / 2).cpu().numpy()
    nerf_poses = {}
    for n, p in ((10, poses10), (100, poses100)):
        q = p.clone()                                      # the room's rotations, camera centres moved by the mesh's
        cc = _camera_centres(p.cpu()) + centre             # t = -R c
        Rm = []
        for row in p.cpu().numpy():
            x, y, z, w = row[3:].astype(np.float64)
            Rm.append(np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                                [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                                [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]]))
        q[:, :3] = torch.from_numpy(np.stack([-R_ @ c for R_, c in zip(Rm, cc)]).astype(np.float32)).to(dev)
        nerf_poses[n] = q

    res = {}
    for label, mesh, pz in (("room_surface", room.surface_mesh(), {10: poses10, 100: poses100}),
                            ("tsdf_mesh", tsdf_mesh, {10: poses10, 100: poses100}),
                            ("nerf_mesh", nerf_mesh, nerf_poses)):
        scene, build_ms = timed(lambda: MeshScene(mesh))
        _, build_peak = peak(lambda: MeshScene(mesh))
        r = {"triangles": scene.n_tri, "bvh_build_ms": build_ms, "bvh_bytes": scene.bvh.numel(),
             "bvh_bytes_per_triangle": round(scene.bvh.numel() / scene.n_tri, 1), "build_peak_bytes": build_peak}
        for n, p in pz.items():
            out, ms = timed(lambda: scene.render(p, intr, W, H))
            _, pb = peak(lambda: scene.render(p, intr, W, H))
            r[f"render_{n}_ms"] = ms
            r[f"render_{n}_Mrays_per_s"] = round(n * W * H / ms / 1e3, 1)
            r[f"render_{n}_peak_bytes"] = pb
            r[f"render_{n}_hit_fraction"] = round(float((out.triangle >= 0).float().mean()), 4)
        res[label] = r
        del scene
        torch.cuda.empty_cache()
    print(json.dumps({"bench": "mesh_render", "gpu": name or torch.cuda.get_device_name(0), "power_limit": power,
                      "reps": a.reps, "hw": [H, W], "tsdf_res": a.res, "render_volume_10_ms": render_volume_ms, **res}))


if __name__ == "__main__":
    main()
