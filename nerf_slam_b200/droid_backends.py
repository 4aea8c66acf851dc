"""Drop-in replacement of the reference's `droid_backends` extension module.

Same 12 function names, argument order, tensor layouts, in-place semantics and error behaviour
as the pybind module defined at reference src/droid.cpp:347-363 — but every function forwards to
a hand-written sm_90a kernel through the C ABI of libnslam_sm90a.so (include/nslam.h).
`import nerf_slam_b200.droid_backends as droid_backends` (or put `nerf_slam_b200/shim` on
sys.path) and the reference's networks/modules/corr.py + visual_frontend.py run unchanged.

Error convention (src/droid.cpp:129-130): non-contiguous inputs raise RuntimeError; like the
reference there is no CPU path — CPU tensors raise.
"""
import ctypes

import numpy as np
import torch

from . import _lib
from .ba_graph import get_graph

_DT = {torch.float16: 0, torch.float32: 1}
# A14 covariance semantics (DESIGN.md §2): "kernel" (default) = what the reference's block really computes, in one CUDA
# kernel (csrc/ba_cov_ref.cu); "1" = the same values from nslam_ba_cov plus a fix-up of the depth maps of optimised
# frames in a handful of torch ops (kept as an independent cross-check in the tests); "0" = the intended formula.
# The live front end does not come through here: it uses nslam_ba_frontend_update (covariances written into the arenas).
_COV_MODE = "kernel"


def cov_reference_fixup(M, E, Q, disps_flat, z_cov, d_cov, win_k, win_q, win_f, P):
    """In place: rows `win_k` of z_cov / d_cov [K,HW] (depth maps whose frame win_f is optimised, pose index win_q) are
    replaced by the reference's value.  Its assignment `Ej[range(P), kf0-min:kf1-min] = Ei[range(P)]`
    (visual_frontend.py:1214) broadcasts Ei[q] into EVERY pose row, so for these maps
        x^T (L^-1 L^-T) x = Ei[q]^T (sum_{p,p'} M[p][p']) Ei[q]        with M = L^-1 L^-T  [6P,6P].
    M: flat [>= 36 P^2]; E [P+E,6,HW]; Q [K,HW]; disps_flat [N,HW]; index tensors int64 on the same device."""
    if win_k.numel() == 0:
        return
    n = 6 * P
    Msum = M[:n * n].view(P, 6, P, 6).sum(dim=(0, 2))
    Ei = E.index_select(0, win_q)
    acc = (Ei * torch.matmul(Msum, Ei)).sum(dim=1)              # e^T Msum e per pixel: [W,HW]
    q = Q.index_select(0, win_k)
    z = q + q * q * acc
    z_cov.index_copy_(0, win_k, z)
    d2 = disps_flat.index_select(0, win_f) ** 2
    d_cov.index_copy_(0, win_k, z / (d2 * d2))


def _chk(*ts):
    for t in ts:
        if not t.is_contiguous():
            raise RuntimeError("tensor must be contiguous")  # CHECK_CONTIGUOUS, src/droid.cpp:129
        if not t.is_cuda:
            raise RuntimeError("droid_backends (sm_90a) needs CUDA tensors; there is no CPU path")


def _i64(t):
    return t if t.dtype == torch.int64 else t.to(torch.int64)


# ------------------------------------------------------------------------------------------ corr
def corr_index_forward(volume, coords, radius):
    """src/droid.cpp:280-288 -> [corr[n, 2r+1, 2r+1, h1, w1]]"""
    _chk(volume, coords)
    lib = _lib.load()
    n, h1, w1, h2, w2 = volume.shape
    if volume.dtype not in _DT:
        raise RuntimeError("corr_index_forward: fp16/fp32 volumes only")
    coords = coords.float()
    rd = 2 * radius + 1
    out = torch.empty(n, rd, rd, h1, w1, dtype=volume.dtype, device=volume.device)
    _lib.check(lib.nslam_corr_index_forward(_lib.ptr(volume), _DT[volume.dtype], _lib.ptr(coords),
                                            _lib.ptr(out), n, h1, w1, h2, w2, radius,
                                            _lib.stream_ptr()), "corr_index_forward")
    return [out]


def corr_index_backward(volume, coords, corr_grad, radius):
    """src/droid.cpp:290-301. Training only; the inference path runs with autograd disabled
    (examples/slam_demo.py:198).  Symbol kept; out of scope of the hot path (SURVEY.md §2.2)."""
    raise NotImplementedError("corr_index_backward: training-only operator, not part of the "
                              "inference hot path (SURVEY.md §8, out of scope)")


def corr_lookup_pyramid(volumes, coords, radius, slots=None, nhwc_stride=0, coords_nhwc=False, out=None):
    """fused 4-level version of CorrBlock.__call__ (networks/modules/corr.py:40-50):
    volumes: list of [n,h1,w1,h2>>l,w2>>l]; coords [n,2,h1,w1] (level-0 pixels) ->
    [n, L*(2r+1)^2, h1, w1]"""
    lib = _lib.load()
    L = len(volumes)
    _chk(coords, *volumes)
    h1, w1 = volumes[0].shape[1:3]
    n = coords.shape[0]
    dt = volumes[0].dtype
    rd = 2 * radius + 1
    if out is not None:
        assert out.is_contiguous() and out.dtype == dt and out.numel() == n * h1 * w1 * (nhwc_stride or L * rd * rd)
    elif nhwc_stride:
        out = torch.empty(n, h1, w1, nhwc_stride, dtype=dt, device=coords.device)
    else:
        out = torch.empty(n, L * rd * rd, h1, w1, dtype=dt, device=coords.device)
    vptr = (ctypes.c_void_p * L)(*[v.data_ptr() for v in volumes])
    h2s = (ctypes.c_int * L)(*[v.shape[3] for v in volumes])
    w2s = (ctypes.c_int * L)(*[v.shape[4] for v in volumes])
    _lib.check(lib.nslam_corr_lookup_pyramid(ctypes.cast(vptr, ctypes.c_void_p),
                                             ctypes.cast(h2s, ctypes.c_void_p),
                                             ctypes.cast(w2s, ctypes.c_void_p), L, _DT[dt],
                                             _lib.ptr(coords), _lib.ptr(out), n, h1, w1, radius,
                                             _lib.ptr(slots), int(nhwc_stride), int(bool(coords_nhwc)),
                                             _lib.stream_ptr()), "corr_lookup_pyramid")
    return out


def _corrvol_entry(lib, H, W, C):
    """the row-pair kernel (csrc/corr_volume_rows.cu; bit-identical output, tests/test_gpu_parity.py) for the shapes it
    supports, the tiled kernel for everything else"""
    if C == 128 and H % 2 == 0 and W in (64, 80):
        return lib.nslam_corr_volume_build_rows
    return lib.nslam_corr_volume_build


def corr_volume_build(fmaps_nhwc, ii, jj, simt=False):
    """A2: fmaps [NF,H,W,C] fp16 channels-last, ii/jj int32 device frame indices ->
    4 pyramid levels [E,H,W,H>>l,W>>l] fp16 (CorrBlock.__init__, networks/modules/corr.py:23-38)"""
    lib = _lib.load()
    _chk(fmaps_nhwc, ii, jj)
    assert fmaps_nhwc.dtype == torch.float16 and ii.dtype == torch.int32 and jj.dtype == torch.int32
    NF, H, W, C = fmaps_nhwc.shape
    E = ii.shape[0]
    outs = [torch.empty(E, H, W, H >> l, W >> l, dtype=torch.float16, device=fmaps_nhwc.device)
            for l in range(4)]
    fn = lib.nslam_corr_volume_build_simt if simt else _corrvol_entry(lib, H, W, C)
    _lib.check(fn(_lib.ptr(fmaps_nhwc), NF, H, W, C, _lib.ptr(ii), _lib.ptr(jj), E,
                  *[_lib.ptr(o) for o in outs], _lib.stream_ptr()), "corr_volume_build")
    return outs


def corr_volume_build_into(fmaps_nhwc, ii, jj, outs):
    """as corr_volume_build but writes into caller-provided level tensors (arena slots)"""
    lib = _lib.load()
    NF, H, W, C = fmaps_nhwc.shape
    _lib.check(_corrvol_entry(lib, H, W, C)(_lib.ptr(fmaps_nhwc), NF, H, W, C, _lib.ptr(ii), _lib.ptr(jj),
                                            ii.shape[0], *[_lib.ptr(o) for o in outs], _lib.stream_ptr()),
               "corr_volume_build")


def altcorr_forward(fmap1, fmap2, coords, radius):
    """src/droid.cpp:303-313 -> [corr[b, n, (2r+1)^2, h, w]]"""
    _chk(fmap1, fmap2, coords)
    lib = _lib.load()
    if fmap1.dtype not in _DT or fmap2.dtype != fmap1.dtype:
        raise RuntimeError("altcorr_forward: fp16/fp32 feature maps only")
    B, H1, W1, C = fmap1.shape
    _, H2, W2, _ = fmap2.shape
    N = coords.shape[1]
    coords = coords.float()
    rd = 2 * radius + 1
    out = torch.empty(B, N, rd * rd, H1, W1, dtype=fmap1.dtype, device=fmap1.device)
    _lib.check(lib.nslam_altcorr_forward(_lib.ptr(fmap1), _lib.ptr(fmap2), _DT[fmap1.dtype],
                                         _lib.ptr(coords), _lib.ptr(out), B, N, H1, W1, H2, W2, C,
                                         radius, _lib.stream_ptr()), "altcorr_forward")
    return [out]


def altcorr_backward(fmap1, fmap2, coords, corr_grad, radius):
    """src/droid.cpp:315-327. Training only (see corr_index_backward)."""
    raise NotImplementedError("altcorr_backward: training-only operator, out of scope")


# ------------------------------------------------------------------------------------------ geometry
def frame_distance(poses, disps, intrinsics, ii, jj, beta):
    """src/droid.cpp:230-246"""
    ii, jj = _i64(ii).contiguous(), _i64(jj).contiguous()
    _chk(poses, disps, intrinsics, ii, jj)
    lib = _lib.load()
    n = ii.shape[0]
    ht, wd = disps.shape[1:]
    dist = torch.empty(n, dtype=torch.float32, device=poses.device)
    _lib.check(lib.nslam_frame_distance(_lib.ptr(poses), _lib.ptr(disps), _lib.ptr(intrinsics),
                                        _lib.ptr(ii), _lib.ptr(jj), n, ht, wd, float(beta),
                                        _lib.ptr(dist), _lib.stream_ptr()), "frame_distance")
    return dist


def projmap(poses, disps, intrinsics, ii, jj):
    """src/droid.cpp:249-264 -> [coords[n,h,w,3], valid[n,h,w,1]]"""
    ii, jj = _i64(ii).contiguous(), _i64(jj).contiguous()
    _chk(poses, disps, intrinsics, ii, jj)
    lib = _lib.load()
    n = ii.shape[0]
    ht, wd = disps.shape[1:]
    coords = torch.empty(n, ht, wd, 3, dtype=torch.float32, device=poses.device)
    valid = torch.empty(n, ht, wd, 1, dtype=torch.float32, device=poses.device)
    _lib.check(lib.nslam_projmap(_lib.ptr(poses), _lib.ptr(disps), _lib.ptr(intrinsics),
                                 _lib.ptr(ii), _lib.ptr(jj), n, ht, wd, _lib.ptr(coords),
                                 _lib.ptr(valid), _lib.stream_ptr()), "projmap")
    return [coords, valid]


def iproj(poses, disps, intrinsics):
    """src/droid.cpp:267-276 -> points[N,h,w,3]"""
    _chk(poses, disps, intrinsics)
    lib = _lib.load()
    n, ht, wd = disps.shape
    pts = torch.empty(n, ht, wd, 3, dtype=torch.float32, device=poses.device)
    _lib.check(lib.nslam_iproj(_lib.ptr(poses), _lib.ptr(disps), _lib.ptr(intrinsics), n, ht, wd,
                               _lib.ptr(pts), _lib.stream_ptr()), "iproj")
    return pts


def depth_filter(poses, disps, intrinsics, ix, thresh):
    """src/droid.cpp:330-344 -> counter[n,h,w]"""
    ix = _i64(ix).contiguous()
    _chk(poses, disps, intrinsics, ix, thresh)
    lib = _lib.load()
    num, ht, wd = disps.shape
    n = ix.shape[0]
    counter = torch.empty(n, ht, wd, dtype=torch.float32, device=poses.device)
    _lib.check(lib.nslam_depth_filter(_lib.ptr(poses), _lib.ptr(disps), _lib.ptr(intrinsics),
                                      _lib.ptr(ix), _lib.ptr(thresh), n, num, ht, wd,
                                      _lib.ptr(counter), _lib.stream_ptr()), "depth_filter")
    return counter


def reproject(poses, disps, intrinsics, ii, jj, want_valid=True, out=None):
    """A6 (pops.projective_transform, networks/geom/projective_ops.py:98-145, jacobian=False):
    poses [N,7], disps [N,h,w], intrinsics [N,4] or [4] -> coords [E,h,w,2], valid [E,h,w,1]"""
    ii, jj = _i64(ii).contiguous(), _i64(jj).contiguous()
    _chk(poses, disps, intrinsics, ii, jj)
    lib = _lib.load()
    E = ii.shape[0]
    ht, wd = disps.shape[1:]
    stride = 4 if intrinsics.dim() == 2 else 0
    coords = out if out is not None else torch.empty(E, ht, wd, 2, dtype=torch.float32, device=poses.device)
    assert coords.is_contiguous() and coords.numel() == E * ht * wd * 2
    valid = torch.empty(E, ht, wd, 1, dtype=torch.float32, device=poses.device) if want_valid else None
    _lib.check(lib.nslam_reproject(_lib.ptr(poses), _lib.ptr(disps), _lib.ptr(intrinsics), stride,
                                   _lib.ptr(ii), _lib.ptr(jj), E, ht, wd, _lib.ptr(coords),
                                   _lib.ptr(valid), _lib.stream_ptr()), "reproject")
    return coords, valid


def cvx_upsample(data, mask, pow=1.0, mask_nhwc=False):
    """A17 (utils/flow_viz.py:166-183): data [K,ht,wd,1] fp32, mask [K,576,ht,wd] (or channels-last
    [K,ht,wd,576] with mask_nhwc) -> [K,8ht,8wd,1].
    Does NOT write -inf into `mask` (the reference mutates its argument)."""
    lib = _lib.load()
    K, ht, wd = data.shape[:3]
    data = data.reshape(K, ht, wd).float().contiguous()
    mask = mask.reshape(K, ht, wd, 576) if mask_nhwc else mask.reshape(K, 576, ht, wd)
    if mask.dtype not in _DT:
        mask = mask.float()
    mask = mask.contiguous()
    out = torch.empty(K, 8 * ht, 8 * wd, dtype=torch.float32, device=data.device)
    _lib.check(lib.nslam_cvx_upsample(_lib.ptr(data), _lib.ptr(mask), _DT[mask.dtype],
                                      _lib.ptr(out), K, ht, wd, float(pow), int(bool(mask_nhwc)),
                                      _lib.stream_ptr()), "cvx_upsample")
    return out.unsqueeze(-1)


def cvx_upsample2(data, data2, mask, out, out2, pow=1.0, index=None):
    """two planes (inverse depth + depth covariance) through one softmax of a channels-last mask
    [K,ht,wd,576].  data*/out* are fp32 contiguous [*,ht,wd] / [*,8ht,8wd]; plane k of the mask is applied to
    row index[k] of data/out (int64 device tensor; identity when None).  Writes out/out2 in place."""
    lib = _lib.load()
    K, ht, wd = mask.shape[0], data.shape[-2], data.shape[-1]
    assert mask.is_contiguous() and mask.shape[-1] == 576
    for t in (data, data2, out, out2):
        assert t.is_contiguous() and t.dtype == torch.float32
    _lib.check(lib.nslam_cvx_upsample2(_lib.ptr(data), _lib.ptr(data2), _lib.ptr(mask), _DT[mask.dtype],
                                       _lib.ptr(out), _lib.ptr(out2), _lib.ptr(index), K, ht, wd, float(pow), 1,
                                       _lib.stream_ptr()), "cvx_upsample2")


# ------------------------------------------------------------------------------------------ BA
class BAProblem:
    """Device buffers + graph tables of one BA window; owns everything the kernels touch."""

    def __init__(self, poses, disps, intrinsics, extrinsics, disps_sens, targets, weights, eta,
                 ii_host, jj_host, kf0, kf1):
        dev = poses.device
        self.gh, self.g, self._gbuf = get_graph(ii_host, jj_host, kf0, kf1, dev)
        gh = self.gh
        ht, wd = disps.shape[1:]
        hw = ht * wd
        self.ht, self.wd, self.hw = ht, wd, hw
        tile = _lib.load().nslam_ba_tile_pixels()
        T = (hw + tile - 1) // tile
        f = dict(dtype=torch.float32, device=dev)
        n = 6 * gh.P
        self.H = torch.empty(n, n, **f)
        self.v = torch.empty(n, 1, **f)
        self.Q = torch.empty(gh.K, hw, **f)
        self.E = torch.empty(gh.P + gh.E, 6, hw, **f)
        self.w = torch.empty(gh.K, hw, **f)
        self.Hs = torch.empty(4, gh.E, 6, 6, **f)
        self.vs = torch.empty(2, gh.E, 6, **f)
        self._aux = torch.empty(max(gh.E, 1), 80, **f)
        self._part = torch.empty(max(gh.E, 1), T, 27, **f)
        nv = gh.NPAIR * 36 + gh.NR * 6
        self._spart = torch.empty(max(nv, 1), T, **f)
        self._sblk = torch.empty(max(nv, 1), **f)
        if eta.numel() != gh.K * hw:
            # same constraint as `eta.view({-1, ht*wd})` against ii_kf_ids (src/droid_kernels.cu:1751)
            raise RuntimeError(f"eta has {eta.numel() // hw} maps, graph needs {gh.K}")
        self._keep = (poses, disps, intrinsics, extrinsics, disps_sens, targets, weights, eta)
        b = _lib.BABuffers()
        b.poses = poses.data_ptr(); b.disps_sens = disps_sens.data_ptr() if disps_sens is not None else None
        b.intrinsics = intrinsics.data_ptr(); b.extrinsics = extrinsics.data_ptr()
        b.targets = targets.data_ptr(); b.weights = weights.data_ptr(); b.eta = eta.data_ptr()
        b.disps = disps.data_ptr()
        b.H = self.H.data_ptr(); b.v = self.v.data_ptr(); b.Q = self.Q.data_ptr()
        b.Emat = self.E.data_ptr(); b.w = self.w.data_ptr(); b.Hs = self.Hs.data_ptr()
        b.vs = self.vs.data_ptr(); b.edge_aux = self._aux.data_ptr(); b.part = self._part.data_ptr()
        b.spart = self._spart.data_ptr(); b.sblk = self._sblk.data_ptr()
        b.ht, b.wd, b.T = ht, wd, T
        self.b = b

    def linearize(self):
        lib = _lib.load()
        _lib.check(lib.nslam_ba_reduced_camera_matrix(ctypes.byref(self.g), ctypes.byref(self.b),
                                                      _lib.stream_ptr()), "reduced_camera_matrix")

    def solve(self, prior_idx=-1, prior_err=None, prior_info=0.0, lm=0.0, ep=0.0, want_linv=False):
        lib = _lib.load()
        P = self.gh.P
        n = 6 * P
        dev = self.H.device
        work = torch.empty(2 * n * n + 2 * n, dtype=torch.float64, device=dev)
        dx = torch.empty(P, 6, dtype=torch.float32, device=dev)
        linv = torch.empty(n, n, dtype=torch.float32, device=dev) if want_linv else None
        status = torch.zeros(1, dtype=torch.int32, device=dev)
        _lib.check(lib.nslam_ba_solve(_lib.ptr(self.H), _lib.ptr(self.v), P, prior_idx,
                                      _lib.ptr(prior_err), float(prior_info), float(lm), float(ep),
                                      _lib.ptr(work), _lib.ptr(dx), _lib.ptr(linv), _lib.ptr(status),
                                      _lib.stream_ptr()), "ba_solve")
        self._work = work
        return dx, linv, status

    def gauss_newton(self, iters, world_T_body, cam_T_world, cam_T_body, prior_idx=-1, prior_pose=None,
                     prior_info=0.0, want_linv=False, clamp_min=1e-3):
        """`iters` full BA iterations (linearise .. depth update) with ONE host call, no syncs.
        cam_T_world must be the `poses` tensor this problem was built on. Returns (dx, linv, status)."""
        lib = _lib.load()
        P = self.gh.P
        n = 6 * P
        dev = self.H.device
        work = torch.empty(2 * n * n + 2 * n, dtype=torch.float64, device=dev)
        dx = torch.empty(P, 6, dtype=torch.float32, device=dev)
        linv = torch.empty(n, n, dtype=torch.float32, device=dev) if want_linv else None
        status = torch.zeros(1, dtype=torch.int32, device=dev)
        perr = torch.zeros(6, dtype=torch.float32, device=dev)
        _lib.check(lib.nslam_ba_gn_iterations(ctypes.byref(self.g), ctypes.byref(self.b), int(iters),
                                              _lib.ptr(world_T_body), _lib.ptr(cam_T_world), _lib.ptr(cam_T_body),
                                              int(prior_idx), _lib.ptr(prior_pose), float(prior_info), _lib.ptr(work),
                                              _lib.ptr(dx), _lib.ptr(linv), _lib.ptr(perr), _lib.ptr(status),
                                              float(clamp_min), _lib.stream_ptr()), "ba_gn_iterations")
        self._work = (work, perr)
        return dx, linv, status

    def frontend_update(self, iters, world_T_body, cam_T_world, cam_T_body, status, prior_idx=-1, prior_pose=None,
                        prior_info=0.0, clamp_min=1e-3, cov_mode=None, idepths_cov=None, depths_cov=None, pose_cov=None,
                        lm=0.0, ep=0.0):
        """The live path's whole BA step (visual_frontend.py:1071-1232) as ONE host call on buffers owned by this
        problem: `iters` Gauss-Newton iterations, then the covariance block written in place into the keyframe arenas
        (idepths_cov / depths_cov [buffer,ht,wd], pose_cov [buffer,6,6]).  status: int32[2] device tensor owned by the
        caller ([0] last factorisation failed, [1] cumulative failures); a failed iteration changes nothing.
        cov_mode: None = no covariances, 1 = reference-exact, 0 = intended formula (DESIGN.md §2, A14)."""
        lib = _lib.load()
        P = self.gh.P
        n = 6 * P
        if getattr(self, "_fu", None) is None:
            dev = self.H.device
            self._fu = (torch.empty(2 * n * n + 2 * n, dtype=torch.float64, device=dev),
                        torch.empty(P, 6, dtype=torch.float32, device=dev),
                        torch.empty(n, n, dtype=torch.float32, device=dev),
                        torch.zeros(6, dtype=torch.float32, device=dev),
                        torch.empty(n * n + 36, dtype=torch.float32, device=dev))
        work, dx, linv, perr, M = self._fu
        assert status.dtype == torch.int32 and status.numel() >= 2
        if cov_mode is not None:
            for t in (idepths_cov, depths_cov, pose_cov):
                assert t.is_contiguous() and t.dtype == torch.float32
        _lib.check(lib.nslam_ba_frontend_update(
            ctypes.byref(self.g), ctypes.byref(self.b), int(iters), _lib.ptr(world_T_body), _lib.ptr(cam_T_world),
            _lib.ptr(cam_T_body), int(prior_idx), _lib.ptr(prior_pose), float(prior_info), float(lm), float(ep),
            _lib.ptr(work), _lib.ptr(dx),
            _lib.ptr(linv), _lib.ptr(perr), _lib.ptr(status), float(clamp_min), -1 if cov_mode is None else int(cov_mode),
            _lib.ptr(M), _lib.ptr(idepths_cov), _lib.ptr(depths_cov), _lib.ptr(pose_cov), _lib.stream_ptr()),
            "ba_frontend_update")
        return dx, linv

    def depth_update(self, dx, clamp_min=0.0):
        lib = _lib.load()
        _lib.check(lib.nslam_ba_depth(ctypes.byref(self.g), ctypes.byref(self.b), _lib.ptr(dx),
                                      float(clamp_min), _lib.stream_ptr()), "ba_depth")

    def covariances(self, linv, reference=None):
        """A14 -> (sigma_g [P,6,6], z_cov [K,ht,wd], depth_cov [K,ht,wd]).
        reference: None = "kernel"; "kernel" = the reference's block as it really behaves
        (its broadcast of Ei over the pose rows of optimised frames, visual_frontend.py:1214) in one CUDA kernel
        (csrc/ba_cov_ref.cu); True / "1" = the same from nslam_ba_cov + torch fix-up; False / "0" = the intended formula."""
        lib = _lib.load()
        gh = self.gh
        dev = self.H.device
        n = 6 * gh.P
        mode = _COV_MODE if reference is None else ({True: "1", False: "0"}.get(reference, reference))
        M = torch.empty(n * n + 36, dtype=torch.float32, device=dev)
        z_cov = torch.empty(gh.K, self.hw, dtype=torch.float32, device=dev)
        d_cov = torch.empty(gh.K, self.hw, dtype=torch.float32, device=dev)
        sg = torch.empty(gh.P, 6, 6, dtype=torch.float32, device=dev)
        fn = lib.nslam_ba_cov_reference if mode == "kernel" else lib.nslam_ba_cov
        _lib.check(fn(ctypes.byref(self.g), ctypes.byref(self.b), _lib.ptr(linv),
                      _lib.ptr(M), _lib.ptr(z_cov), _lib.ptr(d_cov),
                      _lib.stream_ptr()), "ba_cov")
        if mode == "1":
            if getattr(self, "_win", None) is None:
                kx = gh.tables["kx"].astype(np.int64)
                k = np.nonzero((kx >= gh.kf0) & (kx < gh.kf0 + gh.P))[0]
                self._win = (_lib.h2d(k, dev), _lib.h2d(kx[k] - gh.kf0, dev), _lib.h2d(kx[k], dev))
            disps = self._keep[1]
            cov_reference_fixup(M, self.E, self.Q, disps.reshape(disps.shape[0], -1), z_cov, d_cov, *self._win, gh.P)
        _lib.check(lib.nslam_ba_pose_cov(_lib.ptr(linv), gh.P, _lib.ptr(sg), _lib.stream_ptr()),
                   "ba_pose_cov")
        return sg, z_cov.view(gh.K, self.ht, self.wd), d_cov.view(gh.K, self.ht, self.wd)


def _host_edges(ii, jj):
    # one D2H copy of the (tiny) edge list; the reference does this ~8x per call
    return ii.detach().cpu().numpy().astype(np.int64), jj.detach().cpu().numpy().astype(np.int64)


def reduced_camera_matrix(poses, body_poses, disps, intrinsics, extrinsics, disps_sens, targets,
                          weights, eta, ii, jj, t0, t1):
    """src/droid.cpp:167-196 -> [H [6P,6P], v [6P,1], Q [K,HW], E [P+M,6,HW], w [K,HW]]"""
    _chk(poses, disps, intrinsics, extrinsics, disps_sens, targets, weights, eta, ii, jj)
    ih, jh = _host_edges(ii, jj)
    prob = BAProblem(poses, disps, intrinsics, extrinsics, disps_sens, targets, weights, eta,
                     ih, jh, t0, t1)
    prob.linearize()
    reduced_camera_matrix.last_problem = prob
    return [prob.H, prob.v, prob.Q, prob.E, prob.w]


def solve_depth(dx, disps, Q, E, w, ii, jj, t0, t1):
    """src/droid.cpp:198-218: dz = Q (w - E^T dx); disps[kx] += dz   (in place)"""
    _chk(dx, disps, Q, E, w, ii, jj)
    ih, jh = _host_edges(ii, jj)
    dev = disps.device
    gh, g, _ = get_graph(ih, jh, t0, t1, dev)
    ht, wd = disps.shape[1:]
    b = _lib.BABuffers()
    b.disps = disps.data_ptr(); b.Q = Q.data_ptr(); b.Emat = E.data_ptr(); b.w = w.data_ptr()
    tile = _lib.load().nslam_ba_tile_pixels()
    b.ht, b.wd, b.T = ht, wd, (ht * wd + tile - 1) // tile
    lib = _lib.load()
    dx = dx.float().contiguous()
    _lib.check(lib.nslam_ba_depth(ctypes.byref(g), ctypes.byref(b), _lib.ptr(dx), 0.0,
                                  _lib.stream_ptr()), "solve_depth")


def solve_poses(poses, dx, t0, t1):
    """src/droid.cpp:220-228: poses[k] <- exp(dx[k-t0]) * poses[k]  (in place, xi=[tau,phi])"""
    _chk(poses, dx)
    lib = _lib.load()
    _lib.check(lib.nslam_pose_retr(_lib.ptr(poses), _lib.ptr(dx), t0, t1, _lib.stream_ptr()),
               "solve_poses")


def ba(poses, body_poses, disps, intrinsics, extrinsics, disps_sens, targets, weights, eta, ii, jj,
       t0, t1, iterations, lm, ep, motion_only):
    """src/droid.cpp:133-165 (ba_cuda, src/droid_kernels.cu:1441-1568): the original DROID
    Gauss-Newton loop with LM damping `ep + lm*diag` and left pose retraction.  Mutates
    poses/disps in place, returns [dx, dz]."""
    _chk(poses, disps, intrinsics, disps_sens, targets, weights, ii, jj)
    ih, jh = _host_edges(ii, jj)
    return ba_host_edges(poses, disps, intrinsics, extrinsics, disps_sens, targets, weights, eta, ih, jh,
                         t0, t1, iterations, lm, ep, motion_only)


def ba_host_edges(poses, disps, intrinsics, extrinsics, disps_sens, targets, weights, eta, ih, jh,
                  t0, t1, iterations, lm, ep, motion_only):
    """`ba` with the edge list already on the host (int64 numpy): no device->host copy, no sync"""
    _chk(poses, disps, intrinsics, disps_sens, targets, weights)
    prob = BAProblem(poses, disps, intrinsics, extrinsics.contiguous(), disps_sens, targets, weights,
                     eta.contiguous(), ih, jh, t0, t1)
    lib = _lib.load()
    dx = dz = None
    for _ in range(iterations):
        prob.linearize()
        if motion_only:
            # A only: rebuild H,v without the Schur part
            H, v = _pose_only_system(prob)
            prob.H.copy_(H); prob.v.copy_(v)
        dx, _, _ = prob.solve(lm=lm, ep=ep)
        if not motion_only:
            before = disps[prob.gh.tables["kx"].astype(np.int64)].clone()
            prob.depth_update(dx)
            dz = (disps[prob.gh.tables["kx"].astype(np.int64)] - before).view(prob.gh.K, -1)
        _lib.check(lib.nslam_pose_retr(_lib.ptr(poses), _lib.ptr(dx), t0, t1, _lib.stream_ptr()),
                   "pose_retr")
    return [dx, dz]


def _pose_only_system(prob):
    """dense A and b from the per-edge blocks (motion_only branch of ba_cuda)"""
    gh = prob.gh
    P, E = gh.P, gh.E
    dev = prob.H.device
    ii = torch.as_tensor(gh.tables["ii"].astype(np.int64) - gh.kf0, device=dev)
    jj = torch.as_tensor(gh.tables["jj"].astype(np.int64) - gh.kf0, device=dev)
    H = torch.zeros(P, P, 6, 6, dtype=torch.float64, device=dev)
    v = torch.zeros(P, 6, dtype=torch.float64, device=dev)
    for w_, (a, b) in enumerate([(ii, ii), (ii, jj), (jj, ii), (jj, jj)]):
        ok = (a >= 0) & (a < P) & (b >= 0) & (b < P)
        H.index_put_((a[ok], b[ok]), prob.Hs[w_][ok].double(), accumulate=True)
    for w_, a in enumerate([ii, jj]):
        ok = (a >= 0) & (a < P)
        v.index_put_((a[ok],), prob.vs[w_][ok].double(), accumulate=True)
    return H.permute(0, 2, 1, 3).reshape(6 * P, 6 * P).float(), v.reshape(6 * P, 1).float()
