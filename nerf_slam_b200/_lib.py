"""ctypes binding of libnslam_sm90a.so — the only way the Python host code reaches the kernels.

There is deliberately no fallback: if the shared object is missing or a CUDA device is absent
the operators raise (`NslamUnavailable`), they never route through PyTorch/CPU code.
"""
import ctypes
import os

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, "libnslam_sm90a.so")

c_void_p, c_int, c_float = ctypes.c_void_p, ctypes.c_int, ctypes.c_float


class NslamUnavailable(RuntimeError):
    pass


class BAGraph(ctypes.Structure):
    """mirror of `nslam_ba_graph` (include/nslam_ba.h)"""
    _fields_ = [(n, c_int) for n in ("E", "P", "K", "kf0", "NR", "NPAIR", "RMAX", "NHC", "NVC")] + \
               [(n, c_void_p) for n in ("ii", "jj", "kx", "src_ptr", "src_edges", "row_ptr",
                                        "row_pose", "row_erow", "pair_off", "hc_ptr", "hc_idx",
                                        "vc_ptr", "vc_idx")]


class BABuffers(ctypes.Structure):
    """mirror of `nslam_ba_buffers` (include/nslam_ba.h)"""
    _fields_ = [(n, c_void_p) for n in ("poses", "disps_sens", "intrinsics", "extrinsics",
                                        "targets", "weights", "eta", "disps", "H", "v", "Q",
                                        "Emat", "w", "Hs", "vs", "edge_aux", "part", "spart",
                                        "sblk")] + \
               [(n, c_int) for n in ("ht", "wd", "T")]


N_UPDATE_WEIGHTS = 15      # NSLAM_W_COUNT (include/nslam_nn.h)


class UpdateCtx(ctypes.Structure):
    """mirror of `nslam_update_ctx` (include/nslam_nn.h)"""
    _fields_ = [(n, c_int) for n in ("E", "K", "H", "W", "num_sms", "corr_channels", "Kba")] + [("ep", c_float)] + \
               [(n, c_void_p) for n in ("net", "inp", "corr", "coords1", "coords0", "target", "seg_ptr", "seg_edges",
                                        "net_out", "flow", "conf", "ba_target", "ba_weight", "upmask",
                                        "ux", "damping", "kx_ba", "ba_damp")] + \
               [("wp", c_void_p * N_UPDATE_WEIGHTS), ("bias", c_void_p * N_UPDATE_WEIGHTS)] + \
               [(n, c_void_p) for n in ("glo_w", "glo_b", "c1", "c2", "mcol", "f1", "f2", "gsum", "gzr", "gq",
                                        "z", "rnet", "h0", "h2", "a1", "am", "a2", "e16")]


_P = c_void_p
_SIGNATURES = {
    # name: argtypes (all return int)
    "nslam_corr_index_forward": [_P, c_int, _P, _P, c_int, c_int, c_int, c_int, c_int, c_int, _P],
    "nslam_corr_lookup_pyramid": [_P, _P, _P, c_int, c_int, _P, _P, c_int, c_int, c_int, c_int, _P, c_int, c_int, _P],
    "nslam_corr_volume_build": [_P, c_int, c_int, c_int, c_int, _P, _P, c_int, _P, _P, _P, _P, _P],
    "nslam_corr_volume_build_rows": [_P, c_int, c_int, c_int, c_int, _P, _P, c_int, _P, _P, _P, _P, _P],
    "nslam_corr_volume_build_slots": [_P, c_int, c_int, c_int, c_int, _P, _P, _P, c_int, c_int, _P, _P, _P, _P, _P],
    "nslam_corr_volume_build_simt": [_P, c_int, c_int, c_int, c_int, _P, _P, c_int, _P, _P, _P, _P, _P],
    "nslam_altcorr_forward": [_P, _P, c_int, _P, _P, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_int, _P],
    "nslam_corr_index_backward": [_P, _P, c_int, _P, c_int, c_int, c_int, c_int, c_int, c_int, _P],
    "nslam_altcorr_backward_scratch": [c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_int, _P],
    "nslam_altcorr_backward": [_P, _P, _P, _P, _P, _P, _P, ctypes.c_ulonglong, c_int, c_int, c_int, c_int, c_int, c_int,
                               c_int, c_int, _P],
    "nslam_reproject": [_P, _P, _P, c_int, _P, _P, c_int, c_int, c_int, _P, _P, _P],
    "nslam_frame_distance": [_P, _P, _P, _P, _P, c_int, c_int, c_int, c_float, _P, _P],
    "nslam_projmap": [_P, _P, _P, _P, _P, c_int, c_int, c_int, _P, _P, _P],
    "nslam_iproj": [_P, _P, _P, c_int, c_int, c_int, _P, _P],
    "nslam_depth_filter": [_P, _P, _P, _P, _P, c_int, c_int, c_int, c_int, _P, _P],
    "nslam_cvx_upsample": [_P, _P, c_int, _P, c_int, c_int, c_int, c_float, c_int, _P],
    "nslam_cvx_upsample2": [_P, _P, _P, c_int, _P, _P, _P, c_int, c_int, c_int, c_float, c_int, _P],
    "nslam_motion_im2col": [_P, _P, _P, _P, c_int, c_int, c_int, _P],
    "nslam_flow_heads_post": [_P, _P, _P, _P, _P, _P, c_int, c_int, _P],
    "nslam_segment_mean": [_P, _P, _P, _P, c_int, c_int, _P],
    "nslam_eta_damping": [_P, _P, _P, c_int, _P, _P, c_int, c_int, c_float, _P],
    "nslam_conv_igemm_ex": [_P, _P, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_int, _P, _P, c_int, c_int,
                            _P, _P, _P, _P, _P, c_int, _P, _P, c_int, _P, c_int, _P],
    "nslam_im2col7_s2": [_P, _P, c_int, c_int, c_int, _P],
    "nslam_update_op_step": [ctypes.POINTER(UpdateCtx), _P],
    "nslam_inorm_stats": [_P, _P, c_int, c_int, c_int, c_int, _P],
    "nslam_inorm_apply": [_P, _P, _P, _P, _P, c_int, c_int, c_int, c_float, c_int, _P],
    "nslam_tsdf_integrate": [_P, _P, _P, c_int, c_int, c_int, _P, c_float, _P, _P, _P, c_int, c_int, _P, _P, c_float, c_float,
                             c_float, c_float, _P],
    "nslam_tsdf_mesh_plan": [c_int, c_int, c_int, _P],
    "nslam_tsdf_mesh_count": [_P, _P, c_int, c_int, c_int, c_float, _P, _P],
    "nslam_tsdf_mesh_emit": [_P, _P, _P, c_int, c_int, c_int, _P, c_float, c_float, _P, c_int, _P, _P, _P, _P, _P, _P],
    "nslam_tsdf_raycast": [_P, _P, _P, c_int, c_int, c_int, _P, c_float, _P, c_int, c_int, c_int, _P, c_float, c_float,
                           c_float, c_float, _P, _P, _P, _P, _P],
    "nslam_tsdf_blocks_scratch": [c_int, c_int, _P],
    "nslam_tsdf_blocks_activate": [_P, _P, c_int, c_int, _P, _P, c_float, c_float, c_float, _P, _P, c_int, c_int, _P,
                                   ctypes.c_longlong, _P, _P, _P, _P, _P],
    "nslam_tsdf_blocks_insert": [_P, c_int, c_int, _P, _P, _P, _P, _P, _P, _P, c_int, _P],
    "nslam_tsdf_blocks_rehash": [_P, c_int, _P, _P, c_int, _P],
    "nslam_tsdf_blocks_integrate": [_P, _P, _P, _P, _P, c_int, c_float, _P, _P, _P, c_int, c_int, _P, _P, c_float, c_float,
                                    c_float, c_float, _P],
    "nslam_tsdf_blocks_neighbours": [_P, c_int, _P, _P, c_int, _P, _P],
    "nslam_tsdf_blocks_mesh_plan": [c_int, _P],
    "nslam_tsdf_blocks_mesh_count": [_P, _P, _P, _P, c_int, c_float, _P, _P],
    "nslam_tsdf_blocks_mesh_emit": [_P, _P, _P, _P, _P, c_int, c_float, c_float, _P, c_int, _P, _P, _P, _P, _P, _P],
    "nslam_tsdf_blocks_raycast": [_P, _P, _P, _P, _P, _P, c_int, c_float, _P, c_int, c_int, c_int, _P, c_float, c_float,
                                  c_float, c_float, _P, _P, _P, _P, _P],
    "nslam_point_cloud_scratch": [c_int, c_int, c_int, _P],
    "nslam_point_cloud_count": [_P, _P, _P, c_int, c_int, c_int, c_int, c_float, c_float, _P, ctypes.c_longlong, _P, _P],
    "nslam_point_cloud_emit": [_P, _P, _P, _P, c_int, _P, _P, c_int, c_int, c_int, c_float, c_float, _P, ctypes.c_longlong,
                               _P, _P, _P],
    "nslam_point_cloud_voxel_scratch": [c_int, _P],
    "nslam_point_cloud_voxel_sort": [_P, c_int, c_float, _P, ctypes.c_longlong, _P, _P],
    "nslam_point_cloud_voxel_reduce": [_P, _P, c_int, _P, ctypes.c_longlong, c_int, _P, _P, _P, _P],
    # reconstruction evaluation (include/nslam_eval.h)
    "nslam_eval_surface_scratch": [c_int, _P],
    "nslam_eval_surface_area": [_P, c_int, _P, c_int, _P, ctypes.c_longlong, _P, _P],
    "nslam_eval_sample_surface": [_P, _P, c_int, c_int, ctypes.c_ulonglong, _P, ctypes.c_longlong, _P, _P, _P],
    "nslam_eval_bvh_scratch": [c_int, c_int, _P],
    "nslam_eval_bvh_build": [_P, c_int, c_int, _P, ctypes.c_longlong, _P],
    "nslam_eval_nearest_scratch": [c_int, _P],
    "nslam_eval_nearest": [_P, ctypes.c_longlong, c_int, c_int, _P, c_int, c_float, c_int, _P, ctypes.c_longlong, _P, _P,
                           _P],
    "nslam_eval_visible": [_P, c_int, _P, c_int, _P, c_int, c_int, _P, c_float, c_float, c_float, _P, _P],
    "nslam_eval_reduce": [_P, c_int, c_float, c_float, _P, _P],
    # registration (include/nslam_eval.h); the double arrays are HOST arrays
    "nslam_reg_transform": [_P, c_int, ctypes.POINTER(ctypes.c_double), c_int, _P, _P],
    "nslam_reg_face_normals": [_P, c_int, _P, c_int, _P, c_int, _P, _P, _P],
    "nslam_reg_accumulate": [_P, c_int, _P, _P, _P, c_int, ctypes.POINTER(ctypes.c_double), c_int, c_int, c_int, _P, _P],
    # triangle-mesh rendering (include/nslam_render.h)
    "nslam_render_bvh_scratch": [c_int, c_int, _P],
    "nslam_render_bvh_build": [_P, c_int, _P, c_int, c_int, _P, ctypes.c_longlong, _P, _P],
    "nslam_render_views": [_P, ctypes.c_longlong, c_int, c_int, _P, _P, c_int, _P, c_int, c_int, c_float, c_float, c_int,
                           c_int, _P, _P, _P, _P, _P],
    # triangle-mesh operations (include/nslam_mesh.h)
    "nslam_mesh_components_scratch": [c_int, c_int, _P],
    "nslam_mesh_components": [_P, c_int, _P, c_int, _P, ctypes.c_longlong, _P, _P, _P, _P, _P],
    "nslam_mesh_submesh_scratch": [c_int, c_int, _P],
    "nslam_mesh_submesh_count": [_P, c_int, c_int, _P, _P, ctypes.c_longlong, _P, _P],
    "nslam_mesh_submesh_emit": [_P, _P, _P, c_int, _P, c_int, _P, ctypes.c_longlong, _P, _P, _P, _P, _P],
    "nslam_mesh_any_vertex": [_P, _P, c_int, c_int, _P, _P, _P, _P],
    "nslam_mesh_vertex_normals_scratch": [c_int, c_int, _P],
    "nslam_mesh_vertex_normals": [_P, c_int, _P, c_int, _P, ctypes.c_longlong, _P, _P, _P],
    "nslam_mesh_cluster_scratch": [c_int, c_int, _P],
    "nslam_mesh_cluster_count": [_P, c_int, _P, c_int, c_float, _P, ctypes.c_longlong, _P, _P],
    "nslam_mesh_cluster_emit": [_P, _P, c_int, _P, c_int, _P, ctypes.c_longlong, _P, _P, _P, _P],
    "nslam_ba_reduced_camera_matrix": [ctypes.POINTER(BAGraph), ctypes.POINTER(BABuffers), _P],
    "nslam_ba_tile_pixels": [],
    "nslam_ba_solve": [_P, _P, c_int, c_int, _P, c_float, c_float, c_float, _P, _P, _P, _P, _P],
    "nslam_ba_retract": [_P, _P, _P, _P, c_int, c_int, _P],
    "nslam_pose_retr": [_P, _P, c_int, c_int, _P],
    "nslam_pose_prior_error": [_P, _P, _P, _P],
    "nslam_ba_depth": [ctypes.POINTER(BAGraph), ctypes.POINTER(BABuffers), _P, c_float, _P],
    "nslam_ba_cov": [ctypes.POINTER(BAGraph), ctypes.POINTER(BABuffers), _P, _P, _P, _P, _P],
    "nslam_proximity_edges": [_P, c_int, c_int, c_int, _P, _P, c_int, c_int, c_int, c_float, c_int, c_int, _P, c_int, _P],
    "nslam_ba_graph_build": [_P, _P, c_int, c_int, c_int, _P, c_int, _P],
    "nslam_ba_cov_reference": [ctypes.POINTER(BAGraph), ctypes.POINTER(BABuffers), _P, _P, _P, _P, _P],
    "nslam_ba_pose_cov": [_P, c_int, _P, _P],
    "nslam_ba_gn_iterations": [ctypes.POINTER(BAGraph), ctypes.POINTER(BABuffers), c_int, _P, _P, _P, c_int, _P,
                               c_float, _P, _P, _P, _P, _P, c_float, _P],
    "nslam_ba_cov_arena": [ctypes.POINTER(BAGraph), ctypes.POINTER(BABuffers), _P, _P, c_int, _P, _P, _P, _P, _P],
    "nslam_ba_frontend_update": [ctypes.POINTER(BAGraph), ctypes.POINTER(BABuffers), c_int, _P, _P, _P, c_int, _P,
                                 c_float, c_float, c_float, _P, _P, _P, _P, _P, c_float, c_int, _P, _P, _P, _P, _P],
    # Path B (include/nslam_ngp.h); struct pointers are passed with ctypes.byref
    "nslam_ngp_train_step": [_P, _P, _P, c_int, ctypes.c_uint, c_float, c_float, c_float, c_float, c_int, _P],
    "nslam_ngp_adam": [_P, c_int, c_float, c_float, c_float, c_float, c_float, _P],
    "nslam_ngp_forward": [_P, _P, c_int, _P, _P],
    "nslam_ngp_loss_backward": [_P, _P, c_int, c_int, c_float, c_float, c_float, c_float, c_int, _P],
    "nslam_ngp_update_density_grid": [_P, _P, c_int, ctypes.c_uint, c_float, c_float, _P, c_int, _P],
    "nslam_ngp_density_sample_tc": [_P, _P, c_int, ctypes.c_uint, c_float, c_int, _P],
    "nslam_ngp_render_tile": [_P, _P, _P, c_int, c_int, c_int, c_int, c_int, c_float, c_float, c_float, _P, _P, c_int, _P],
    "nslam_ngp_ingest_image": [_P, _P, _P, c_int, c_int, _P, _P, _P, _P],
    "nslam_ngp_ingest_batch": [_P, _P, _P, _P, c_int, c_int, c_int, _P, _P, _P, _P, c_float, c_float, c_float, c_float, _P, _P,
                               _P, _P, c_int, _P],
    "nslam_ngp_cam_grad": [_P, _P, _P, _P, _P, _P, c_float, _P, c_int, _P, _P, _P, c_float, _P, _P, c_int, _P],
    "nslam_ngp_cam_adam_apply": [_P, _P, _P, _P, _P, _P, _P, c_int, c_float, c_float, c_float, c_float, c_float, _P],
    "nslam_ngp_pack_mlp": [_P, _P, _P],
    "nslam_ngp_forward_tc": [_P, _P, _P, _P, c_int, c_int, _P, _P, c_int, _P],
    "nslam_ngp_backward_tc": [_P, _P, _P, _P, _P, c_float, _P, _P, c_int, c_int, _P],
    "nslam_ngp_train_step_tc": [_P, _P, _P, _P, c_int, ctypes.c_uint, c_float, c_float, c_float, c_float, c_float, c_int, _P],
    "nslam_ngp_loss_backward_tc": [_P, _P, _P, c_int, c_int, c_float, c_float, c_float, c_float, c_float, c_int, _P],
    "nslam_ngp_sample_phase": [_P, _P, _P, c_int, ctypes.c_uint, _P],
    "nslam_ngp_loss_phase": [_P, c_int, c_float, c_float, c_float, c_float, _P],
    "nslam_ngp_mesh_lattice": [_P, _P, _P, c_float, c_int, c_int, c_int, c_float, _P, _P, c_int, _P],
    "nslam_ngp_mesh_colors": [_P, _P, _P, _P, c_int, c_int, _P, _P, ctypes.c_longlong, c_int, _P],
    # tensor-core convolution (include/nslam_nn.h)
    "nslam_conv_igemm": [_P, _P, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_int, _P, _P, c_int, c_int,
                         _P, _P, _P, _P, _P, c_int, _P, _P, c_int, _P],
}

_lib = None
_cuda_ok = False


def exported_symbols():
    return sorted(_SIGNATURES)


def load(require_cuda=True):
    """dlopen the library (once) and attach prototypes. Raises NslamUnavailable, never falls back."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise NslamUnavailable(
                f"{LIB_PATH} not built — run `python -m nerf_slam_b200.build` (needs nvcc)")
        lib = ctypes.CDLL(LIB_PATH)
        for name, args in _SIGNATURES.items():
            fn = getattr(lib, name)
            fn.argtypes = args
            fn.restype = c_int
        _lib = lib
    global _cuda_ok
    if require_cuda and not _cuda_ok:
        import torch
        if not torch.cuda.is_available():
            raise NslamUnavailable("nerf_slam_b200 operators need a CUDA device (sm_90a); "
                                   "there is no CPU fallback")
        _cuda_ok = True          # checked once: the query costs ~4 us and every operator comes through here
    return _lib


def query_size(name, *args):
    """the size (bytes or an element count) that the C query `name(*args, long long* out)` writes; raises on an error"""
    out = ctypes.c_longlong(0)
    check(getattr(load(), name)(*args, ctypes.byref(out)), name)
    return out.value


def check(err, what):
    if err != 0:
        import torch
        msg = f"{what} failed with cudaError {err}"
        try:
            msg += f" ({torch.cuda.cudart().cudaGetErrorString(err)})"
        except Exception:
            pass
        raise RuntimeError(msg)


_fixed_stream = None


def stream_ptr():
    """cudaStream_t of torch's current stream.  The lookup costs ~14 us of host time; hot loops that issue
    dozens of launches on one stream wrap themselves in `fixed_stream()` so that it is done once."""
    if _fixed_stream is not None:
        return _fixed_stream
    import torch
    return c_void_p(torch.cuda.current_stream().cuda_stream)


class fixed_stream:
    """context manager: resolve the current stream once for all C-ABI calls inside (the caller guarantees
    that the current stream does not change within the block)"""

    def __enter__(self):
        global _fixed_stream
        import torch
        self._prev = _fixed_stream
        _fixed_stream = c_void_p(torch.cuda.current_stream().cuda_stream)
        return self

    def __exit__(self, *exc):
        global _fixed_stream
        _fixed_stream = self._prev
        return False


def ptr(t):
    """device pointer of a (contiguous) torch tensor, or NULL for None"""
    if t is None:
        return c_void_p(0)
    return c_void_p(t.data_ptr())


def h2d(a, device, dtype=None):
    """numpy array (or list) -> device tensor through PINNED memory with a non-blocking copy.
    `torch.as_tensor(ndarray, device=...)` copies from pageable memory, which makes the CUDA runtime
    synchronise the stream before every copy (one hidden device sync per small index upload).
    A CPU `device` gets the host tensor itself (no copy)."""
    import numpy as np
    import torch
    t = torch.from_numpy(np.ascontiguousarray(a))
    if dtype is not None and t.dtype != dtype:
        t = t.to(dtype)
    if torch.device(device).type == "cpu":
        return t
    if t.numel() == 0:
        return torch.empty(t.shape, dtype=t.dtype, device=device)
    return t.pin_memory().to(device, non_blocking=True)
