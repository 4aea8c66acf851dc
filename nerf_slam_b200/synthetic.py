"""Procedural "Replica-shaped" RGB-D stream (SURVEY.md §8d): an analytic textured box room ray-cast
in closed form, camera on a smooth Lissajous orbit.  No files, seeded, deterministic.

Packets follow the reference's dataset schema exactly (datasets/nerf_dataset.py:155-162):
  {"k", "t_cams", "poses" (w2c 4x4), "images" u8 [1,H,W,4] RGBA, "depths" int32 [1,H,W,1]
   (u16-scaled, depth_scale = 1/6553.5), "calibs" [CameraCalibration], "is_last_frame"}
"""
import numpy as np


class Resolution:
    def __init__(self, width, height):
        self.width, self.height = width, height

    def numpy(self):
        return np.array([self.width, self.height])

    def total(self):
        return self.width * self.height


class PinholeCameraModel:
    """same fields as datasets/dataset.py:72-102"""

    def __init__(self, fx, fy, cx, cy):
        self.fx, self.fy, self.cx, self.cy = fx, fy, cx, cy
        self.K = np.array([[fx, 0, cx], [0, fy, cy], [0, 0, 1.0]])

    def scale_intrinsics(self, scale_x, scale_y):
        """datasets/dataset.py:85-95"""
        self.fx *= scale_x; self.cx *= scale_x
        self.fy *= scale_y; self.cy *= scale_y
        self.K = np.array([[self.fx, 0, self.cx], [0, self.fy, self.cy], [0, 0, 1.0]])

    def numpy(self):
        return np.array([self.fx, self.fy, self.cx, self.cy])

    def matrix(self):
        return self.K


class CameraCalibration:
    """same fields as datasets/dataset.py:115-123"""

    def __init__(self, body_T_cam, camera_model, distortion_model, rate_hz, resolution, aabb, depth_scale):
        self.body_T_cam = body_T_cam
        self.camera_model = camera_model
        self.distortion_model = distortion_model
        self.rate_hz = rate_hz
        self.resolution = resolution
        self.aabb = aabb
        self.depth_scale = depth_scale


def _hash_noise(ix, iy, iz, seed):
    h = (ix * 374761393 + iy * 668265263 + iz * 2147483647 + seed * 1274126177) & 0xFFFFFFFF
    h = ((h ^ (h >> 13)) * 1274126177) & 0xFFFFFFFF
    h = h ^ (h >> 16)
    return (h & 0xFFFF).astype(np.float32) / 65535.0


def value_noise(p, freq, seed):
    """tri-linear value noise on world points p [...,3]"""
    q = p * freq
    i0 = np.floor(q).astype(np.int64)
    f = (q - i0).astype(np.float32)
    f = f * f * (3 - 2 * f)
    out = 0
    for dx in (0, 1):
        for dy in (0, 1):
            for dz in (0, 1):
                w = (f[..., 0] if dx else 1 - f[..., 0]) * (f[..., 1] if dy else 1 - f[..., 1]) * \
                    (f[..., 2] if dz else 1 - f[..., 2])
                out = out + w * _hash_noise(i0[..., 0] + dx, i0[..., 1] + dy, i0[..., 2] + dz, seed)
    return out


class SyntheticRoom:
    def __init__(self, width=640, height=480, n_frames=200, seed=0, half_extent=(3.0, 2.0, 3.0),
                 orbit_radius=0.7, step=0.012):
        self.W, self.H, self.n = width, height, n_frames
        self.seed = seed
        self.ext = np.asarray(half_extent, np.float64)
        fx = fy = width / 2.0                      # 90 deg HFOV
        self.calib = CameraCalibration(
            np.eye(4), PinholeCameraModel(fx, fy, width / 2.0 - 0.5, height / 2.0 - 0.5), None, 30.0,
            Resolution(width, height), np.array([[-2, -2, -2], [2, 2, 2]]), 1.0 / 6553.5)
        self.r, self.step = orbit_radius, step
        u, v = np.meshgrid(np.arange(width), np.arange(height))
        self.dirs_cam = np.stack([(u - self.calib.camera_model.cx) / fx, (v - self.calib.camera_model.cy) / fy,
                                  np.ones_like(u, dtype=np.float64)], -1)

    def __len__(self):
        return self.n

    def c2w(self, k):
        t = k * self.step
        pos = np.array([self.r * np.sin(2 * t), 0.25 * self.r * np.sin(3 * t + 0.5), self.r * np.sin(t) * np.cos(t)])
        yaw = 0.9 * t
        pitch = 0.12 * np.sin(1.7 * t)
        fwd = np.array([np.sin(yaw) * np.cos(pitch), np.sin(pitch), np.cos(yaw) * np.cos(pitch)])
        up0 = np.array([0, -1.0, 0])             # y down camera
        right = np.cross(fwd, up0); right /= np.linalg.norm(right)
        down = np.cross(fwd, right)
        T = np.eye(4)
        T[:3, 0], T[:3, 1], T[:3, 2], T[:3, 3] = right, down, fwd, pos
        return T

    def render(self, k):
        T = self.c2w(k)
        d = self.dirs_cam @ T[:3, :3].T
        o = T[:3, 3]
        with np.errstate(divide="ignore"):
            tpos = (self.ext - o) / d
            tneg = (-self.ext - o) / d
        tt = np.where(d > 0, tpos, tneg)
        t = tt.min(-1)
        face = tt.argmin(-1)
        hit = o + d * t[..., None]
        depth = t * 1.0                            # z-depth along the optical axis: dirs_cam z == 1
        base = np.array([[0.75, 0.55, 0.45], [0.45, 0.65, 0.75], [0.6, 0.7, 0.5]], np.float32)[face]
        n1 = value_noise(hit, 1.3, self.seed)[..., None]
        n2 = value_noise(hit, 5.1, self.seed + 1)[..., None]
        n3 = value_noise(hit, 17.0, self.seed + 2)[..., None]
        stripes = (0.5 + 0.5 * np.sin(hit.sum(-1) * 9.0))[..., None].astype(np.float32)
        alb = base * (0.45 + 0.55 * n1) + 0.25 * (n2 - 0.5) + 0.18 * (n3 - 0.5) + 0.08 * (stripes - 0.5)
        shade = np.clip(1.15 - 0.08 * t[..., None], 0.5, 1.1)
        rgb = np.clip(alb * shade, 0, 1)
        rgba = np.concatenate([(rgb * 255).astype(np.uint8), np.full(rgb.shape[:2] + (1,), 255, np.uint8)], -1)
        d16 = np.clip(depth / self.calib.depth_scale, 0, 65535).astype(np.uint16).astype(np.int32)[..., None]
        return rgba, d16, np.linalg.inv(T)

    def surface_mesh(self):
        """the exact surface `render` ray-casts: the room's six faces at +-half_extent as 12 triangles -> vertices [8,3]
        float32 (corner k at -ext / +ext per axis by bits 0, 1, 2 of k), triangles [12,3] int32 wound so that
        (b - a) x (c - a) points into the room, i.e. into free space (the convention of TsdfMesh)"""
        ext = self.ext.astype(np.float32)
        k = np.arange(8)
        vertices = np.stack([np.where((k >> a) & 1, ext[a], -ext[a]) for a in range(3)], 1).astype(np.float32)
        tris = []
        for a in range(3):
            b, c = (a + 1) % 3, (a + 2) % 3
            for side in (0, 1):
                # corners (b, c) = (0,0), (1,0), (1,1), (0,1) of the face: counter-clockwise about +e_a
                q = [side << a | i << b | j << c for i, j in ((0, 0), (1, 0), (1, 1), (0, 1))]
                if side:                                   # the +ext face looks toward -e_a
                    q = q[::-1]
                tris += [(q[0], q[1], q[2]), (q[0], q[2], q[3])]
        return vertices, np.asarray(tris, np.int32)

    def packet(self, k):
        rgba, d16, w2c = self.render(k)
        return {"k": np.arange(k, k + 1), "t_cams": np.array([k]), "poses": np.array([w2c]),
                "images": rgba[None], "depths": d16[None], "calibs": np.array([self.calib]),
                "is_last_frame": k >= self.n - 1}

    def stream(self):
        for k in range(self.n):
            yield self.packet(k)
