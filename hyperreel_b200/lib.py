"""ctypes binding of ``libhyperreel_b200.so`` (the C-ABI declared in ``include/hyperreel_b200.h``).

This file *is* the reference-side stub INTEGRATION.md describes: plain ``ctypes`` structures that mirror
the header one to one, no torch extension ABI.  There is no fallback: if the shared library is missing
or cannot be loaded, ``load_library()`` raises.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess
import threading

HR_ABI_VERSION = 26
HR_MAX_GROUPS = 4
HR_MAX_LAYERS = 10
HR_MAX_SAMPLES = 256
HR_MAX_PEERS = 8
HR_TC_MAX_PASSES = 40

ACT_IDENTITY, ACT_SIGMOID, ACT_TANH = 0, 1, 2
PARAM_IDENTITY, PARAM_TWO_PLANE, PARAM_PLUECKER = 0, 1, 2
ISECT_Z_PLANE, ISECT_SPHERE, ISECT_CYLINDER, ISECT_SPHERE_NEW, ISECT_DISTANCE, ISECT_VOXEL, ISECT_PLANE = 0, 1, 2, 3, 4, 5, 6
CONTRACT_NONE, CONTRACT_MIPNERF, CONTRACT_AFFINE = 0, 1, 2
SHADE_SH, SHADE_RGB = 0, 1
DENSE_RELU, DENSE_SOFTPLUS, DENSE_RELU_ABS = 0, 1, 2
MLP_FP32_SIMT, MLP_BF16X3_TC, MLP_ZERO, MLP_FP16_TC = 0, 1, 2, 3
SAMPLE_PERMUTE, SAMPLE_REPLACE = 0, 1  # hr_sample_train_rows modes
RESIZE_METHODS = {"pil_lanczos": 0, "pil_bicubic": 1, "pil_box": 2, "cv2_linear": 3, "cv2_area": 4}  # HR_RESIZE_*
RESIZE_BGR = 1
PIXEL_RGB8, PIXEL_RGBA8 = 0, 1  # HR_PIXEL_*: uint8 RGB, or RGBA composited over white where a colour is consumed
# extra fields of the colour net (hr_render_fields): key of the reference's dict `x` -> HR_FIELD_* id
FIELDS = {"points": 0, "distances": 1, "base_times": 2, "time_offset": 3, "times": 4, "viewdirs": 5, "weights": 6,
          "color_scale": 7, "color_shift": 8, "spatial_flow": 9, "sigma": 10, "point_sigma": 11, "point_offset": 12,
          "color_scale_global": 13, "color_shift_global": 14}
FIELD_CHANNELS = {k: 3 if k in ("points", "viewdirs", "color_scale", "color_shift", "spatial_flow", "point_offset",
                                 "color_scale_global", "color_shift_global") else 1 for k in FIELDS}
FIELD_OVER, FIELD_NO_OVER, FIELD_PRED_WEIGHTS = 0, 1, 2
PT_NONE, PT_POINT, PT_VIEW, PT_ORIGIN, PT_TIME = -1, 0, 3, 6, 9  # first channel of each source of the point net's input row

_PKG_DIR = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_PKG_DIR, "libhyperreel_b200.so")
CSRC_DIR = os.path.join(_PKG_DIR, "csrc")


class hr_act(C.Structure):
    _fields_ = [("kind", C.c_int32), ("inner_fac", C.c_float), ("shift", C.c_float), ("outer_fac", C.c_float),
                ("eased", C.c_int32), ("ease_mul", C.c_float), ("ease_add", C.c_float), ("ease_pad", C.c_int32)]


class hr_encode_group(C.Structure):
    _fields_ = [
        ("start", C.c_int32), ("end", C.c_int32), ("fn", C.c_int32), ("n_freqs", C.c_int32),
        ("exclude_identity", C.c_int32), ("freq_mult", C.c_float), ("base_mult", C.c_float),
        ("near", C.c_float), ("far", C.c_float), ("dir_mult", C.c_float), ("mom_mult", C.c_float),
    ]


class hr_config(C.Structure):
    _fields_ = [
        ("abi_version", C.c_int32), ("c_in", C.c_int32),
        ("n_groups", C.c_int32), ("groups", hr_encode_group * HR_MAX_GROUPS),
        ("mlp_in", C.c_int32), ("mlp_width", C.c_int32), ("mlp_layers", C.c_int32), ("mlp_skip", C.c_int32),
        ("mlp_out", C.c_int32), ("leaky_slope", C.c_float), ("mlp_mode", C.c_int32),
        ("n_samples", C.c_int32), ("head_stride", C.c_int32), ("off_z", C.c_int32), ("n_z", C.c_int32),
        ("off_flow", C.c_int32), ("off_sigma", C.c_int32), ("off_point_sigma", C.c_int32),
        ("off_offset", C.c_int32), ("off_cscale", C.c_int32), ("off_cshift", C.c_int32),
        ("act_z", hr_act), ("act_flow", hr_act), ("act_sigma", hr_act), ("act_point_sigma", hr_act),
        ("act_offset", hr_act), ("act_cscale", hr_act), ("act_cshift", hr_act),
        ("isect_type", C.c_int32), ("isect_act", hr_act), ("isect_use_sigma", C.c_int32),
        ("isect_density_off", C.c_int32), ("z_scale", C.c_float), ("isect_near", C.c_float),
        ("isect_far", C.c_float), ("isect_sort", C.c_int32), ("samples", C.c_float * HR_MAX_SAMPLES),
        ("contract_type", C.c_int32), ("contract_samples", C.c_int32),
        ("contract_start_radius", C.c_float), ("contract_end_radius", C.c_float),
        ("contract_start_distance", C.c_float), ("contract_end_distance", C.c_float),
        ("sphere_origin_initial", C.c_float * 3), ("sphere_origin_scale", C.c_float),
        ("use_flow", C.c_int32), ("num_keyframes", C.c_int32), ("num_frames", C.c_int32), ("flow_act", hr_act),
        ("use_offset", C.c_int32), ("offset_density_off", C.c_int32), ("offset_act", hr_act),
        ("dynamic", C.c_int32), ("aabb", C.c_float * 6), ("distance_scale", C.c_float),
        ("n_sigma", C.c_int32 * 3), ("n_app", C.c_int32 * 3), ("app_dim", C.c_int32), ("shading", C.c_int32),
        ("white_bg", C.c_int32), ("black_bg", C.c_int32), ("weight_thre", C.c_float),
        ("fea2dense", C.c_int32), ("density_shift", C.c_float), ("use_color_scale_shift", C.c_int32),
        ("clamp_output", C.c_int32),
        ("contract_affine_min", C.c_float * 3), ("contract_affine_den", C.c_float * 3), ("contract_dist_fac", C.c_float),
        ("off_cscale_global", C.c_int32), ("off_cshift_global", C.c_int32),
        ("act_cscale_global", hr_act), ("act_cshift_global", hr_act),
        ("sphere_resize_scale", C.c_float), ("sphere_resize_initial", C.c_float * 3),
        ("isect_axes", C.c_int32), ("z_scale3", C.c_float * 3), ("isect_outward", C.c_int32), ("isect_max_axis", C.c_int32),
        ("plane_normal", C.c_float * 9), ("plane_normal_scale", C.c_float),
        ("n_color_views", C.c_int32), ("act_ctransform", hr_act), ("act_ctshift", hr_act),
        ("cascade", C.c_int32), ("pre_samples", C.c_int32), ("pre_n_groups", C.c_int32),
        ("pre_groups", hr_encode_group * HR_MAX_GROUPS),
        ("pre_mlp_in", C.c_int32), ("pre_mlp_width", C.c_int32), ("pre_mlp_layers", C.c_int32), ("pre_mlp_skip", C.c_int32),
        ("pre_mlp_mode", C.c_int32), ("pre_head_stride", C.c_int32), ("pre_off_z", C.c_int32), ("pre_off_sigma", C.c_int32),
        ("pre_act_z", hr_act), ("pre_act_sigma", hr_act), ("pre_isect_act", hr_act),
        ("pre_use_sigma", C.c_int32), ("pre_sort", C.c_int32),
        ("pre_z_scale", C.c_float), ("pre_near", C.c_float), ("pre_far", C.c_float),
        ("pre_samples_tab", C.c_float * 32), ("pt_src", C.c_int32 * 8),
    ]


_FP = C.POINTER(C.c_float)


class hr_params(C.Structure):
    _fields_ = [
        ("on_device", C.c_int32),
        ("mlp_weight", C.c_void_p * HR_MAX_LAYERS), ("mlp_bias", C.c_void_p * HR_MAX_LAYERS),
        ("sigma_plane", C.c_void_p * 3), ("app_plane", C.c_void_p * 3),
        ("plane_h", C.c_int32 * 3), ("plane_w", C.c_int32 * 3),
        ("sigma_second", C.c_void_p * 3), ("app_second", C.c_void_p * 3),
        ("second_len", C.c_int32 * 3),
        ("basis_mat", C.c_void_p), ("color_embedding", C.c_void_p),
        ("pre_mlp_weight", C.c_void_p * HR_MAX_LAYERS), ("pre_mlp_bias", C.c_void_p * HR_MAX_LAYERS),
    ]


class hr_field_request(C.Structure):
    _fields_ = [("field", C.c_int32), ("mode", C.c_int32), ("out", C.c_void_p)]


class hr_visual_request(C.Structure):
    _fields_ = [("field", C.c_int32), ("mode", C.c_int32), ("channels", C.c_int32), ("use_abs", C.c_int32),
                ("bounded", C.c_int32), ("normalize", C.c_int32), ("lo", C.c_float), ("hi", C.c_float), ("out", C.c_void_p)]


class hr_train_opts(C.Structure):
    _fields_ = [("clamp_output", C.c_int32), ("white_bg", C.c_int32)]


class hr_grads(C.Structure):
    _fields_ = [("sigma_plane", C.c_void_p * 3), ("app_plane", C.c_void_p * 3), ("sigma_second", C.c_void_p * 3),
                ("app_second", C.c_void_p * 3), ("basis_mat", C.c_void_p), ("color_embedding", C.c_void_p)]


class hr_net_grads(C.Structure):
    _fields_ = [("weight", C.c_void_p * HR_MAX_LAYERS), ("bias", C.c_void_p * HR_MAX_LAYERS)]


class hr_camera(C.Structure):
    _fields_ = [
        ("c2w", C.c_float * 12), ("fx", C.c_float), ("fy", C.c_float), ("cx", C.c_float), ("cy", C.c_float),
        ("width", C.c_int32), ("height", C.c_int32), ("centered_pixels", C.c_int32), ("flipped", C.c_int32),
        ("normalize", C.c_int32), ("use_ndc", C.c_int32), ("ndc_near", C.c_float), ("cam_idx", C.c_float),
        ("time", C.c_float), ("fisheye", C.c_int32), ("k1", C.c_float), ("k2", C.c_float),
        ("two_plane", C.c_int32), ("lf_s", C.c_float), ("lf_t", C.c_float), ("lf_st_scale", C.c_float),
        ("lf_uv_scale", C.c_float), ("lf_near", C.c_float), ("lf_far", C.c_float), ("lf_aspect", C.c_float),
    ]


# entry points the header declares: name -> (restype, argtypes)
EXPORTS = {
    "hr_abi_version": (C.c_int, []),
    "hr_last_error": (C.c_char_p, []),
    "hr_create": (C.c_int, [C.POINTER(hr_config), C.c_int, C.POINTER(C.c_void_p)]),
    "hr_upload": (C.c_int, [C.c_void_p, C.POINTER(hr_params), C.c_void_p]),
    "hr_workspace_bytes": (C.c_int64, [C.c_void_p, C.c_int64]),
    "hr_train_workspace_bytes": (C.c_int64, [C.c_void_p, C.c_int64]),
    "hr_set_sub_batch": (C.c_int, [C.c_void_p, C.c_int64]),
    "hr_render": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p]),
    "hr_render_scatter": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.POINTER(C.c_void_p), C.c_int32, C.c_int64, C.c_void_p,
                                     C.c_int64, C.c_void_p]),
    "hr_render_stages": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p,
                                    C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p]),
    "hr_render_fields": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.POINTER(hr_field_request),
                                    C.c_int32, C.c_void_p, C.c_int64, C.c_void_p]),
    "hr_render_host": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_int64]),
    "hr_generate_rays": (C.c_int, [C.POINTER(hr_camera), C.c_int32, C.c_int64, C.c_int64, C.c_void_p, C.c_void_p]),
    "hr_sample_train_batch": (C.c_int, [C.c_void_p, C.c_int32, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32,
                                         C.c_uint64, C.c_int64, C.c_int64, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p,
                                         C.c_void_p, C.c_void_p, C.POINTER(C.c_int64), C.c_void_p]),
    "hr_sample_train_rows": (C.c_int, [C.c_void_p, C.c_int32, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32,
                                        C.c_void_p, C.c_void_p, C.c_int64, C.c_int32, C.c_uint64, C.c_int64, C.c_int64,
                                        C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                        C.POINTER(C.c_int64), C.c_void_p]),
    "hr_importance_workspace_bytes": (C.c_int64, [C.c_int32]),
    "hr_build_importance_table": (C.c_int, [C.c_void_p, C.c_int32, C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p,
                                             C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "hr_sample_train_mask_rows": (C.c_int, [C.c_void_p, C.c_int32, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_void_p,
                                             C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_int32, C.c_uint64, C.c_int64,
                                             C.c_int64, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                             C.c_void_p, C.POINTER(C.c_int64), C.c_void_p]),
    "hr_render_to8b": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p]),
    "hr_render_frame_to8b_host": (C.c_int, [C.c_void_p, C.POINTER(hr_camera), C.c_void_p, C.c_int64]),
    "hr_video_workspace_bytes": (C.c_int64, [C.c_void_p, C.c_int32, C.c_int32, C.c_int32]),
    "hr_render_video_to8b": (C.c_int, [C.c_void_p, C.POINTER(hr_camera), C.POINTER(C.c_float), C.c_int32, C.c_void_p, C.c_void_p,
                                        C.c_int64, C.c_void_p]),
    "hr_score_views_workspace_bytes": (C.c_int64, [C.c_void_p, C.c_int32, C.c_int32, C.c_int32]),
    "hr_score_views": (C.c_int, [C.c_void_p, C.POINTER(hr_camera), C.POINTER(C.c_float), C.c_int32, C.c_void_p, C.c_int32,
                                  C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p]),
    "hr_render_visuals_workspace_bytes": (C.c_int64, [C.c_void_p, C.POINTER(hr_visual_request), C.c_int32, C.c_int32, C.c_int32,
                                                       C.c_int32]),
    "hr_render_visuals": (C.c_int, [C.c_void_p, C.POINTER(hr_camera), C.POINTER(C.c_float), C.c_int32, C.c_void_p,
                                     C.POINTER(hr_visual_request), C.c_int32, C.c_void_p, C.c_int64, C.c_void_p]),
    "hr_encode_rays": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p]),
    "hr_render_heads": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.POINTER(hr_train_opts), C.c_void_p,
                                   C.c_int64, C.c_void_p]),
    "hr_render_backward": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.POINTER(hr_train_opts),
                                      C.c_void_p, C.c_int64, C.c_void_p]),
    "hr_grad_zero": (C.c_int, [C.c_void_p, C.c_void_p]),
    "hr_grad_read": (C.c_int, [C.c_void_p, C.POINTER(hr_grads), C.c_void_p]),
    "hr_train_net_workspace_bytes": (C.c_int64, [C.c_void_p, C.c_int64]),
    "hr_train_net_forward": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p]),
    "hr_train_net_backward": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.POINTER(hr_net_grads), C.c_void_p, C.c_int64,
                                         C.c_void_p]),
    "hr_set_activations": (C.c_int, [C.c_void_p, C.POINTER(hr_config)]),
    "hr_image_metrics_workspace_bytes": (C.c_int64, [C.c_int32, C.c_int32, C.c_int32]),
    "hr_image_metrics": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_int64,
                                    C.c_void_p]),
    "hr_resize_workspace_bytes": (C.c_int64, [C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32]),
    "hr_resize_frames": (C.c_int, [C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_int32, C.c_int32, C.c_int64,
                                    C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_int64, C.c_void_p]),
    "hr_launch_count": (C.c_int64, [C.c_void_p]),
    "hr_timing_enable": (C.c_int, [C.c_void_p, C.c_int]),
    "hr_timing_reset": (C.c_int, [C.c_void_p]),
    "hr_timing_read": (C.c_int, [C.c_void_p, C.POINTER(C.c_double), C.POINTER(C.c_double), C.POINTER(C.c_int64)]),
    "hr_timing_read_backward": (C.c_int, [C.c_void_p, C.POINTER(C.c_double), C.POINTER(C.c_int64)]),
    "hr_destroy": (C.c_int, [C.c_void_p]),
}

_lock = threading.Lock()
_lib = None


class HyperReelLibraryError(RuntimeError):
    pass


def build(verbose: bool = False) -> str:
    """Compile the CUDA sources for sm_90a into ``libhyperreel_b200.so`` (in-tree)."""
    cmd = ["make", "-C", CSRC_DIR, "-j", str(min(8, os.cpu_count() or 1))]
    res = subprocess.run(cmd, capture_output=True, text=True)
    if verbose or res.returncode != 0:
        print(res.stdout[-4000:])
        print(res.stderr[-4000:])
    if res.returncode != 0:
        raise HyperReelLibraryError("building libhyperreel_b200.so failed")
    return LIB_PATH


def load_library():
    """Load the C-ABI library.  Raises if it has not been built -- there is no other execution path."""
    global _lib
    with _lock:
        if _lib is not None:
            return _lib
        if not os.path.exists(LIB_PATH):
            raise HyperReelLibraryError(
                f"{LIB_PATH} not found: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                "(hyperreel_b200 has no CPU or PyTorch fallback)")
        lib = C.CDLL(LIB_PATH)
        for name, (res, args) in EXPORTS.items():
            fn = getattr(lib, name)  # AttributeError if the symbol is not exported
            fn.restype = res
            fn.argtypes = args
        if lib.hr_abi_version() != HR_ABI_VERSION:
            raise HyperReelLibraryError(f"ABI mismatch: library {lib.hr_abi_version()} vs binding {HR_ABI_VERSION}")
        _lib = lib
        return lib


def check(rc: int):
    if rc != 0:
        msg = load_library().hr_last_error().decode("utf-8", "replace")
        raise RuntimeError(f"hyperreel_b200: {msg}")
