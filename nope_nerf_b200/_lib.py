"""ctypes binding of libnope_nerf_b200.so (include/nope_nerf_b200.h).

The product path has NO CPU fallback: importing this module loads the CUDA library and
raises immediately if it is missing; every call raises RuntimeError with nnb_last_error()
on a non-zero return code."""
import ctypes as C
import os

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("NNB_LIB_PATH") or os.path.join(HERE, "libnope_nerf_b200.so")   # NNB_LIB_PATH: instrumented debug builds

NUM_PARAMS = 595844              # hidden_dim 256; num_params(D) for the other widths
HIDDEN_DIMS = (64, 128, 256)     # model.hidden_dim values with a kernel instantiation
DIST_ALPHA, NDC, NORMALISE, USE_DIR, WHITE_BG, EVAL, SOFTPLUS, SHIFT_FIRST, STASH, RAW_DENSITY = 1, 2, 4, 8, 16, 32, 64, 128, 256, 2048
HVP = 16384                      # with STASH: workspace of nnb_field_hvp (second-order field backward)
OCC_ONLY = 32768                 # nnb_field_fwd on ENGINE_TC: density only, out = (0, 0, 0, a)
ENGINE_SIMT, ENGINE_TC = 0, 1
RS_SCALE_PCS, RS_DETACH_RGBS_SCALE, RS_SHIFT_FIRST, RS_WITH_SSIM, RS_GRAD_REF = 1, 2, 4, 8, 16   # nnb_refstage_args.flags

_f = C.c_void_p  # device pointers travel as integers


class RenderArgs(C.Structure):
    _fields_ = [("weights", _f), ("c2w", _f), ("cam", _f), ("ray_idx", _f), ("pixels", _f), ("depth", _f),
                ("depth_map", _f), ("scale", _f), ("shift", _f), ("noise", _f),
                ("N", C.c_int32), ("S", C.c_int32), ("H", C.c_int32), ("W", C.c_int32), ("h_d", C.c_int32), ("w_d", C.c_int32),
                ("near_", C.c_float), ("far_", C.c_float), ("flags", C.c_uint32), ("engine", C.c_int32),
                ("rgb", _f), ("depth_pred", _f), ("depth_gt", _f), ("mask", _f), ("z_vals", _f), ("alpha", _f),
                ("workspace", _f), ("workspace_bytes", C.c_size_t), ("pts", _f), ("dirs", _f), ("hidden_dim", C.c_int32)]


class RayMarchArgs(C.Structure):   # nnb_ray_march_args
    _fields_ = [("weights", _f), ("ray0", _f), ("ray_dir", _f), ("far_", _f), ("frac", _f),
                ("N", C.c_int32), ("n_steps", C.c_int32), ("n_secant", C.c_int32), ("hidden_dim", C.c_int32),
                ("near_", C.c_float), ("tau", C.c_float), ("flags", C.c_uint32), ("engine", C.c_int32),
                ("depth", _f), ("first", _f), ("bracket", _f), ("workspace", _f), ("workspace_bytes", C.c_size_t)]


class GeometryArgs(C.Structure):   # nnb_geometry_args
    _fields_ = [("weights", _f), ("T", _f), ("pixels", _f), ("frac", _f),
                ("N", C.c_int32), ("n_steps", C.c_int32), ("n_secant", C.c_int32), ("hidden_dim", C.c_int32),
                ("near_", C.c_float), ("tau", C.c_float), ("radius", C.c_float), ("flags", C.c_uint32), ("engine", C.c_int32),
                ("rgb", _f), ("rgb_surf", _f), ("ray0", _f), ("ray_dir", _f), ("far_", _f), ("depth", _f), ("grad", _f),
                ("workspace", _f), ("workspace_bytes", C.c_size_t)]


class FrameArgs(C.Structure):   # nnb_frame_args
    _fields_ = [("fwd", RenderArgs), ("t_min", C.c_float), ("n_eval", _f), ("t_final", _f)]


class RenderBwdArgs(C.Structure):
    _fields_ = [("fwd", RenderArgs), ("g_rgb", _f), ("g_depth_pred", _f), ("g_depth_gt", _f),
                ("g_weights", _f), ("g_c2w", _f), ("g_cam", _f), ("g_depth", _f), ("g_scale_shift", _f)]


class RefStageArgs(C.Structure):
    _fields_ = [("img_cur", _f), ("img_ref", _f), ("dpt_cur", _f), ("dpt_ref", _f), ("c2w_cur", _f), ("c2w_ref", _f), ("dist_cur", _f), ("dist_ref", _f),
                ("H", C.c_int32), ("W", C.c_int32), ("h_d", C.c_int32), ("w_d", C.c_int32), ("pc_ratio", C.c_int32), ("is_last", C.c_int32),
                ("flags", C.c_uint32), ("kx", C.c_float), ("ky", C.c_float), ("nearest_limit", C.c_float), ("w_pc", C.c_float), ("w_rgb_s", C.c_float),
                ("losses", _f), ("g_c2w", _f), ("g_dist", _f), ("workspace", _f), ("workspace_bytes", C.c_size_t),
                ("img_pp", _f), ("cam", _f), ("cam_idx_dev", _f), ("num_cams", C.c_int32), ("weights_dev", _f),
                ("g_kxy", _f), ("loss_total", _f), ("grad_scale", C.c_float), ("g_c2w_ref", _f), ("g_dist_ref", _f)]


MAX_RANKS = 8
FLAG_PAD_BYTES = 256


class AdamSeg(C.Structure):
    _fields_ = [("p", _f), ("m", _f), ("v", _f), ("offset", C.c_int64), ("count", C.c_int64), ("lr_dev", _f), ("step_dev", _f),
                ("beta1", C.c_float), ("beta2", C.c_float), ("eps", C.c_float)]


class AllreduceAdamArgs(C.Structure):
    _fields_ = [("peer_grads", _f * MAX_RANKS), ("peer_flags", _f * MAX_RANKS), ("world", C.c_int32), ("rank", C.c_int32),
                ("n_total", C.c_int64), ("reduced_out", _f), ("segs", AdamSeg * 8), ("nsegs", C.c_int32)]


def _load():
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(
            "nope_nerf_b200: CUDA library %s is missing. Build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            "(nvcc, sm_90a). There is no CPU fallback." % LIB_PATH)
    lib = C.CDLL(LIB_PATH)
    lib.nnb_last_error.restype = C.c_char_p
    lib.nnb_version.restype = C.c_int
    lib.nnb_workspace_bytes.restype = C.c_size_t
    lib.nnb_workspace_bytes.argtypes = [C.c_int32, C.c_int32, C.c_uint32, C.c_int32]
    lib.nnb_workspace_bytes_dim.restype = C.c_size_t
    lib.nnb_workspace_bytes_dim.argtypes = [C.c_int32, C.c_int32, C.c_uint32, C.c_int32, C.c_int32]
    lib.nnb_num_params.restype = C.c_size_t
    lib.nnb_num_params.argtypes = [C.c_int32]
    lib.nnb_render_fwd.argtypes = [C.POINTER(RenderArgs), C.c_void_p]
    lib.nnb_render_bwd.argtypes = [C.POINTER(RenderBwdArgs), C.c_void_p]
    lib.nnb_debug_wgrad.argtypes = [C.POINTER(RenderArgs), _f, C.c_void_p]   # test aid
    lib.nnb_field_fwd.argtypes = [C.POINTER(RenderArgs), _f, C.c_void_p]
    lib.nnb_ray_march.argtypes = [C.POINTER(RayMarchArgs), C.c_void_p]
    lib.nnb_ray_march_workspace_bytes.restype = C.c_size_t
    lib.nnb_ray_march_workspace_bytes.argtypes = [C.c_int32, C.c_int32, C.c_int32]
    lib.nnb_field_bwd.argtypes = [C.POINTER(RenderArgs), _f, _f, _f, _f, C.c_void_p]
    lib.nnb_field_hvp.argtypes = [C.POINTER(RenderArgs), _f, _f, _f, C.c_void_p]
    lib.nnb_field_vjp.argtypes = [C.POINTER(RenderArgs), _f, _f, _f, _f, C.c_void_p]
    lib.nnb_field_vjp_workspace_bytes.restype = C.c_size_t
    lib.nnb_field_vjp_workspace_bytes.argtypes = [C.c_int32, C.c_uint32, C.c_int32]
    lib.nnb_field_grad.argtypes = [C.POINTER(RenderArgs), _f, _f, _f, _f, _f, C.c_void_p]
    lib.nnb_field_grad_workspace_bytes.restype = C.c_size_t
    lib.nnb_field_grad_workspace_bytes.argtypes = [C.c_int32, C.c_uint32, C.c_int32]
    lib.nnb_field_hvp_tc.argtypes = [C.POINTER(RenderArgs), _f, _f, _f, C.c_void_p]
    lib.nnb_field_hvp_tc_workspace_bytes.restype = C.c_size_t
    lib.nnb_field_hvp_tc_workspace_bytes.argtypes = [C.c_int32, C.c_uint32, C.c_int32]
    lib.nnb_geometry_frame.argtypes = [C.POINTER(GeometryArgs), C.c_void_p]
    lib.nnb_geometry_frame_workspace_bytes.restype = C.c_size_t
    lib.nnb_geometry_frame_workspace_bytes.argtypes = [C.c_int32, C.c_int32, C.c_int32]
    lib.nnb_ray_march_engine.argtypes = [C.POINTER(RayMarchArgs), C.c_void_p]
    lib.nnb_geometry_frame_engine.argtypes = [C.POINTER(GeometryArgs), C.c_void_p]
    lib.nnb_ray_march_workspace_bytes_engine.restype = C.c_size_t
    lib.nnb_ray_march_workspace_bytes_engine.argtypes = [C.c_int32, C.c_int32, C.c_int32, C.c_int32]
    lib.nnb_geometry_frame_workspace_bytes_engine.restype = C.c_size_t
    lib.nnb_geometry_frame_workspace_bytes_engine.argtypes = [C.c_int32, C.c_int32, C.c_int32, C.c_int32]
    lib.nnb_render_frame.argtypes = [C.POINTER(FrameArgs), C.c_void_p]
    lib.nnb_render_frame_workspace_bytes.restype = C.c_size_t
    lib.nnb_render_frame_workspace_bytes.argtypes = [C.c_int32, C.c_int32, C.c_int32]
    lib.nnb_render_frame_engine.argtypes = [C.POINTER(FrameArgs), C.c_void_p]
    lib.nnb_render_frame_workspace_bytes_engine.restype = C.c_size_t
    lib.nnb_render_frame_workspace_bytes_engine.argtypes = [C.c_int32, C.c_int32, C.c_int32, C.c_int32]
    lib.nnb_render_frame_bwd.argtypes = [C.POINTER(RenderBwdArgs), C.c_void_p]
    lib.nnb_render_frame_bwd_workspace_bytes.restype = C.c_size_t
    lib.nnb_render_frame_bwd_workspace_bytes.argtypes = [C.c_int32, C.c_int32, C.c_int32]
    lib.nnb_render_frame_train_fwd.argtypes = [C.POINTER(RenderArgs), C.c_void_p]
    lib.nnb_render_frame_train_bwd.argtypes = [C.POINTER(RenderBwdArgs), C.c_void_p]
    lib.nnb_render_frame_bwd_workspace_bytes_engine.restype = C.c_size_t
    lib.nnb_render_frame_bwd_workspace_bytes_engine.argtypes = [C.c_int32, C.c_int32, C.c_int32, C.c_int32]
    lib.nnb_render_frame_bwd_engine.argtypes = [C.POINTER(RenderBwdArgs), C.c_void_p]
    lib.nnb_render_frame_train_fwd_engine.argtypes = [C.POINTER(RenderArgs), C.c_void_p]
    lib.nnb_render_frame_train_bwd_engine.argtypes = [C.POINTER(RenderBwdArgs), C.c_void_p]
    lib.nnb_render_frame_train_fwd_tmin.argtypes = [C.POINTER(FrameArgs), C.c_void_p]
    lib.nnb_render_frame_train_bwd_tmin.argtypes = [C.POINTER(RenderBwdArgs), C.c_void_p]
    lib.nnb_render_tmin_workspace_bytes.argtypes = [C.c_int32, C.c_int32, C.c_int32]
    lib.nnb_render_tmin_workspace_bytes.restype = C.c_size_t
    lib.nnb_render_fwd_tmin.argtypes = [C.POINTER(FrameArgs), C.c_void_p]
    lib.nnb_render_bwd_tmin.argtypes = [C.POINTER(RenderBwdArgs), C.c_void_p]
    lib.nnb_render_tmin_workspace_bytes_engine.argtypes = [C.c_int32, C.c_int32, C.c_int32, C.c_int32]
    lib.nnb_render_tmin_workspace_bytes_engine.restype = C.c_size_t
    lib.nnb_render_fwd_tmin_engine.argtypes = [C.POINTER(FrameArgs), C.c_void_p]
    lib.nnb_render_bwd_tmin_engine.argtypes = [C.POINTER(RenderBwdArgs), C.c_void_p]
    lib.nnb_pose_fwd.argtypes = [_f, _f, _f, C.c_int32, _f, C.c_void_p]
    lib.nnb_pose_bwd.argtypes = [_f, _f, _f, C.c_int32, _f, _f, _f, C.c_void_p]
    lib.nnb_loss_rgb_depth.argtypes = [_f, _f, _f, _f, C.c_int32, _f, _f, _f, C.c_int32, C.c_float, C.c_float, C.c_int32,
                                       C.c_float, _f, _f, _f, _f, C.c_void_p]
    lib.nnb_chamfer.argtypes = [_f, C.c_int32, _f, C.c_int32, _f, _f, _f, _f, C.c_float, _f, _f, C.c_void_p]
    lib.nnb_chamfer_workspace_bytes.restype = C.c_size_t
    lib.nnb_chamfer_workspace_bytes.argtypes = [C.c_int32, C.c_int32]
    lib.nnb_adam_step.argtypes = [_f, _f, _f, _f, C.c_int64, C.c_int32, C.c_float, C.c_float, C.c_float, C.c_float, C.c_void_p]
    lib.nnb_profile_events.argtypes = [C.c_void_p, C.c_int32]
    lib.nnb_pose_fwd_dev.argtypes = [_f, _f, _f, _f, _f, C.c_void_p]
    lib.nnb_pose_bwd_dev.argtypes = [_f, _f, _f, _f, _f, _f, _f, C.c_void_p]
    lib.nnb_distortion_fwd_dev.argtypes = [_f, _f, C.c_int32, _f, C.c_int32, _f, C.c_void_p]
    lib.nnb_distortion_bwd_dev.argtypes = [_f, C.c_int32, _f, C.c_int32, _f, _f, _f, C.c_void_p]
    lib.nnb_adam_step_dev.argtypes = [_f, _f, _f, _f, C.c_int64, _f, _f, C.c_float, C.c_float, C.c_float, C.c_void_p]
    lib.nnb_counter_incr.argtypes = [_f, C.c_int32, C.c_void_p]
    lib.nnb_sample_pixels.argtypes = [_f, C.c_int32, C.c_int32, _f, C.c_void_p]
    lib.nnb_loss_rgb_depth_indirect.argtypes = [_f, _f, _f, C.c_int32, _f, _f, _f, C.c_int32, C.c_float, C.c_float, C.c_int32, C.c_float, _f, _f,
                                                _f, _f, _f, C.c_void_p]
    lib.nnb_refstage_workspace_bytes.restype = C.c_size_t
    lib.nnb_refstage_workspace_bytes.argtypes = [C.c_int32, C.c_int32, C.c_int32]
    lib.nnb_refstage_workspace_bytes_flags.restype = C.c_size_t
    lib.nnb_refstage_workspace_bytes_flags.argtypes = [C.c_int32, C.c_int32, C.c_int32, C.c_uint32]
    lib.nnb_refstage.argtypes = [C.POINTER(RefStageArgs), C.c_void_p]
    lib.nnb_ipc_alloc.argtypes = [C.c_size_t, C.POINTER(C.c_void_p), C.POINTER(C.c_ubyte)]
    lib.nnb_ipc_open.argtypes = [C.POINTER(C.c_ubyte), C.POINTER(C.c_void_p)]
    lib.nnb_ipc_close.argtypes = [C.c_void_p]
    lib.nnb_ipc_free.argtypes = [C.c_void_p]
    lib.nnb_allreduce_adam.argtypes = [C.POINTER(AllreduceAdamArgs), C.c_void_p]
    lib.nnb_depth_invariant.argtypes = [_f, _f, _f, C.c_int32, _f, C.c_float, _f, _f, _f, C.c_void_p]
    lib.nnb_focal_fwd.argtypes = [_f, _f, C.c_int32, _f, C.c_void_p]
    lib.nnb_focal_bwd.argtypes = [_f, _f, C.c_int32, _f, _f, _f, _f, C.c_void_p]
    lib.nnb_pose_smooth.argtypes = [_f, C.c_int32, _f, C.c_float, _f, _f, _f, C.c_void_p]
    return lib


lib = _load()

EXPORTS = ["nnb_last_error", "nnb_version", "nnb_profile_events", "nnb_profile_cursor", "nnb_workspace_bytes", "nnb_render_fwd", "nnb_render_bwd", "nnb_pose_fwd",
           "nnb_pose_bwd", "nnb_loss_rgb_depth", "nnb_chamfer", "nnb_chamfer_workspace_bytes", "nnb_adam_step", "nnb_render_frame_engine",
           "nnb_render_frame_workspace_bytes_engine", "nnb_render_frame_bwd", "nnb_render_frame_bwd_workspace_bytes",
           "nnb_render_frame_train_fwd", "nnb_render_frame_train_bwd", "nnb_render_frame_bwd_workspace_bytes_engine",
           "nnb_render_frame_bwd_engine", "nnb_render_frame_train_fwd_engine", "nnb_render_frame_train_bwd_engine",
           "nnb_render_frame_train_fwd_tmin", "nnb_render_frame_train_bwd_tmin", "nnb_render_tmin_workspace_bytes", "nnb_render_fwd_tmin",
           "nnb_render_bwd_tmin", "nnb_render_tmin_workspace_bytes_engine", "nnb_render_fwd_tmin_engine", "nnb_render_bwd_tmin_engine"]


def check(rc, what):
    if rc != 0:
        raise RuntimeError("%s failed (%d): %s" % (what, rc, lib.nnb_last_error().decode()))


def num_params(hidden_dim=256):
    """floats in the flat MLP parameter vector of OfficialStaticNerf at width hidden_dim (ValueError for an unsupported width)"""
    n = lib.nnb_num_params(int(hidden_dim))
    if n == 0:
        raise ValueError("hidden_dim %s is not supported (supported: %s)" % (hidden_dim, ", ".join(map(str, HIDDEN_DIMS))))
    return int(n)


def ptr(t):
    """device pointer of a torch tensor (or None)"""
    return None if t is None else t.data_ptr()
