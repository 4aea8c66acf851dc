"""Golden for the SLAM point clouds: the reference GUI's own `get_depth_masks` and `build_pcls`
(gui/open3d_gui.py:289-299, 646-678), cut out of its source with `ast` and executed VERBATIM.  The GUI module imports
open3d, gtsam and lietorch, so only the two methods are compiled, into a class whose namespace supplies stand-ins:

- `SE3(poses).inv().matrix()`: lietorch's group inverse and matrix, restated in fp32 torch (lietorch is absent);
- `o3d.core.Tensor.from_dlpack`, `o3d.t.geometry.Image(...).to_legacy()`: pass the torch tensors through;
- `o3d.geometry.RGBDImage.create_from_color_and_depth(color, depth, depth_scale, depth_trunc, ...)`: depth / scale, kept
  where 0 < d < depth_trunc (csrc/point_cloud.cu's validity test);
- `draw_pcl(ix, rgbd, intrinsics, cam_pose)`: `PointCloud.create_from_rgbd_image(rgbd, K, project_valid_depth_only)` and
  `.transform(cam_pose)`: p_c = ((u - cx) d / fx, (v - cy) d / fy, d) in fp64, then cam_pose (fp32 matrix) applied in
  fp64, colours image / 255 in fp32, pixels row-major; the cloud of each keyframe is recorded.

What is pinned is what the reference does in its own code: which pixels survive the mask and the truncation, the pose
inversion, the colour layout and the keyframe order.

    python tests/golden/make_golden_point_cloud.py      (needs /root/reference; writes tests/golden/ref_point_cloud.npz)"""
import ast
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
REF = "/root/reference/gui/open3d_gui.py"


class SE3:
    """lietorch.SE3 on [..., 7] = (t, q_xyzw): inv() and matrix() in fp32"""

    def __init__(self, data):
        self.data = data.float()

    def inv(self):
        t, q = self.data[..., :3], self.data[..., 3:]
        R = _rot(q)
        return SE3(torch.cat([-(R.transpose(-1, -2) @ t[..., None])[..., 0], q * torch.tensor([-1.0, -1.0, -1.0, 1.0])], -1))

    def matrix(self):
        T = torch.zeros(self.data.shape[:-1] + (4, 4), dtype=torch.float32)
        T[..., :3, :3] = _rot(self.data[..., 3:])
        T[..., :3, 3] = self.data[..., :3]
        T[..., 3, 3] = 1.0
        return T


def _rot(q):
    x, y, z, w = q.unbind(-1)
    return torch.stack([torch.stack([1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)], -1),
                        torch.stack([2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)], -1),
                        torch.stack([2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)], -1)], -2)


class _Image:
    def __init__(self, t):
        self.t = t

    def to_legacy(self):
        return self.t.numpy()


class _RGBD:
    @staticmethod
    def create_from_color_and_depth(color, depth, depth_scale, depth_trunc, convert_rgb_to_intensity):
        assert not convert_rgb_to_intensity
        d = (depth / np.float32(depth_scale)).astype(np.float32)
        d = np.where((d > 0) & (d < np.float32(depth_trunc)), d, np.float32(0))
        return types.SimpleNamespace(color=color, depth=d)


class Intrinsics:
    def __init__(self, fx, fy, cx, cy):
        self.k = np.asarray([fx, fy, cx, cy], np.float32)

    def get_focal_length(self):
        return float(self.k[0]), float(self.k[1])

    def get_principal_point(self):
        return float(self.k[2]), float(self.k[3])


def _o3d():
    core = types.SimpleNamespace(Tensor=types.SimpleNamespace(from_dlpack=torch.utils.dlpack.from_dlpack))
    t = types.SimpleNamespace(geometry=types.SimpleNamespace(Image=_Image))
    return types.SimpleNamespace(core=core, t=t, geometry=types.SimpleNamespace(RGBDImage=_RGBD))


def gui_class():
    src = open(REF).read()
    cls = next(n for n in ast.parse(src).body if isinstance(n, ast.ClassDef) and n.name == "Open3dGui")
    body = "\n".join(ast.get_source_segment(src, f) for f in cls.body
                     if isinstance(f, ast.FunctionDef) and f.name in ("get_depth_masks", "build_pcls"))
    code = "class Open3dGui:\n" + "\n".join("    " + l if not l.startswith("    ") else l for l in body.split("\n"))
    ns = {"torch": torch, "np": np, "SE3": SE3, "o3d": _o3d()}
    exec(compile(code, REF, "exec"), ns)
    return ns["Open3dGui"]


def draw_pcl(self, ix, rgbd, intrinsics, cam_pose):
    (fx, fy), (cx, cy) = intrinsics.get_focal_length(), intrinsics.get_principal_point()
    d = rgbd.depth
    v, u = np.nonzero(d > 0)                                      # row-major
    z = d[v, u].astype(np.float64)
    pc = np.stack([(u - cx) * z / fx, (v - cy) * z / fy, z], -1)
    T = np.asarray(cam_pose, np.float32).astype(np.float64)
    pw = pc @ T[:3, :3].T + T[:3, 3]
    col = (np.asarray(rgbd.color)[v, u].astype(np.float32) / np.float32(255)).astype(np.float32)
    self.drawn.append((ix, v * d.shape[1] + u, pw, col))


def packet(n=4, H=12, W=16, seed=7):
    """n keyframes: kf 0 plain, kf 1 fully sigma-masked, kf 2 with depths >= max_depth, kf 3 with 0 / negative / NaN
    inverse depths and a few masked pixels"""
    g = torch.Generator().manual_seed(seed)
    t = torch.randn(n, 3, generator=g) * 0.5
    q = torch.nn.functional.normalize(torch.randn(n, 4, generator=g), dim=-1)
    idepth = torch.rand(n, H, W, generator=g) * 1.5 + 0.2           # depths 0.58 .. 5
    cov = torch.rand(n, H, W, generator=g) * 50.0                   # sigma up to 7 < 10
    cov[1] = 200.0                                                  # sigma 14: all masked
    idepth[2, :4] = 1.0 / 6.0                                       # exactly max_depth: dropped
    idepth[2, 4:6] = 1.0 / 7.5
    idepth[3, 0, :5] = 0.0
    idepth[3, 1, :5] = -0.7
    idepth[3, 2, :5] = float("nan")
    cov[3, 3, :7] = 100.0                                           # sigma exactly 10: masked
    cov[3, 4, :3] = float("nan")                                    # masked
    images = torch.randint(0, 256, (n, 3, H, W), dtype=torch.uint8, generator=g)
    return {"viz_idx": torch.arange(n), "cam0_poses": torch.cat([t, q], -1), "cam0_idepths_up": idepth,
            "cam0_depths_cov_up": cov, "cam0_images": images}


def main():
    Gui = gui_class()
    Gui.draw_pcl = draw_pcl
    pk = packet()
    intr = Intrinsics(14.5, 13.25, 7.75, 5.5)
    out = {"poses": pk["cam0_poses"].numpy(), "idepths": pk["cam0_idepths_up"].numpy(), "covs": pk["cam0_depths_cov_up"].numpy(),
           "images": pk["cam0_images"].numpy(), "intrinsics": intr.k, "max_depth": np.float32(6.0),
           "max_depth_sigma": np.float32(10.0)}
    for mode in ("uncertainty", "uniform"):
        gui = Gui.__new__(Gui)
        gui.depth_mask_type, gui.max_depth_sigma_thresh, gui.max_depth, gui.depth_scale = mode, 10.0, 6.0, 1.0
        gui.o3d_intrinsics, gui.drawn = intr, []
        gui.build_pcls({k: v.clone() for k, v in pk.items()})
        out[f"{mode}_kf"] = np.concatenate([np.full(len(p), ix) for ix, p, _, _ in gui.drawn]).astype(np.int32)
        out[f"{mode}_pix"] = np.concatenate([p for _, p, _, _ in gui.drawn]).astype(np.int64)
        out[f"{mode}_points"] = np.concatenate([p for _, _, p, _ in gui.drawn])
        out[f"{mode}_colors"] = np.concatenate([c for _, _, _, c in gui.drawn])
        print(mode, "points per keyframe", [len(p) for _, p, _, _ in gui.drawn])
    np.savez_compressed(os.path.join(HERE, "ref_point_cloud.npz"), **out)


if __name__ == "__main__":
    sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
    main()
