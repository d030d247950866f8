"""ctypes binding of the C ABI declared in include/ivid_b200.h.

The product path has NO CPU fallback: if libivid_b200.so is missing or fails to load this module raises, and every
entry point converts a non-zero status into the Python exception type the reference would have raised
(AssertionError for `assert`s, NotImplementedError, RuntimeError).
"""
from __future__ import annotations

import ctypes
import os
from ctypes import POINTER, Structure, byref, c_char_p, c_double, c_float, c_int, c_int64, c_uint32, c_uint64, c_void_p

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libivid_b200.so")

IVID_OK = 0
IVID_ERR_INVALID_ARGUMENT = 1
IVID_ERR_NOT_IMPLEMENTED = 2
IVID_ERR_CUDA = 3
IVID_ERR_STATE = 4


class CondT(Structure):
    _fields_ = [
        ("kind", c_int),
        ("y_dev", c_void_p),
        ("mask_dev", c_void_p),
        ("mask_rgb_dev", c_void_p),
        ("noise_dev", c_void_p),
        ("seed", c_uint64),
        ("stream_id", c_uint32),
        ("sr_scale", c_int),          # kind 2: integer upsampling factor (0 = 2)
    ]


class StepArgsT(Structure):
    _fields_ = [
        ("kind", c_int),
        ("use_cfg", c_int),
        ("strength", c_float),
        ("clip_denoised", c_int),
        ("eta", c_float),
        ("classes_dev", c_void_p),
        ("cond", CondT),
        ("replace_rgb_dev", c_void_p),
        ("replace_rgb_mask_dev", c_void_p),
        ("replace_rgb_weight", c_double),
        ("replace_depth_dev", c_void_p),
        ("replace_depth_mask_dev", c_void_p),
        ("replace_depth_weight", c_double),
        ("constrain_depth_dev", c_void_p),
        ("constrain_depth_weight", c_double),
        ("step_noise_dev", c_void_p),
        ("seed", c_uint64),
        ("height", c_int),            # sample size; 0 = the backbone's image_size
        ("width", c_int),
        ("order", c_int),             # kind 2 (DPM-Solver++): 1 or 2 (0 = 2)
        ("prev_x0_dev", c_void_p),    # kind 2, single step: the previous step's pred_x0 (NULL = first order)
        ("t_last", c_int),            # kind 2, single step: the previous step's t
        ("sde", c_int),               # kind 2: 1 = the stochastic (SDE) update, which reads step noise
        ("guidance_interval", c_int), # 1: guide only steps whose model time is in [guidance_t_lo, guidance_t_hi]
        ("guidance_t_lo", c_int),
        ("guidance_t_hi", c_int),
        ("cache_interval", c_int),    # ivid_sampler_run: a full forward every cache_interval steps, reuse forwards between
        ("cache_branch", c_int),      # branch b of the reuse forwards, 0 <= b <= num_res_blocks
        ("cache_reuse", c_int),       # single step: 1 = this step's forward is a reuse forward
        ("unipc", c_int),             # kind 2: 1 = the UniPC predictor-corrector update (order 1..3)
        ("prev2_x0_dev", c_void_p),   # UniPC, single step: the older history D_{-2} / D_{-3} and their t
        ("t_last2", c_int),
        ("prev3_x0_dev", c_void_p),
        ("t_last3", c_int),
        ("prev_xt_dev", c_void_p),    # UniPC, single step: the corrector's base, the corrected x at t_last
        ("corrected_xt_dev", c_void_p),  # UniPC, optional output: this step's corrected x_t
        ("pag", c_int),               # 1: perturbed-attention guidance, eps += pag_scale * (eps_c - eps_perturbed)
        ("pag_scale", c_float),
        ("pag_layers", POINTER(c_int)),   # host array: attention-layer indices in state-dict order
        ("pag_num_layers", c_int),
        ("apg", c_int),               # 1: adaptive projected guidance replaces the classifier-free mix
        ("apg_eta", c_double),        # weight of the update's part parallel to D_c
        ("apg_norm", c_double),       # bound r on the update's norm; 0 = none
        ("apg_momentum", c_double),   # beta in (-1, 1)
        ("apg_state_dev", c_void_p),  # single step: [N,C,H,W] m_prev in, m out; NULL = zero history
        ("start_step", c_int),        # ivid_sampler_run: execute grid steps start_step .. steps-1 only (0 = all)
        ("dynamic_threshold", c_int), # 1: threshold x_0 at the threshold_ratio-quantile of |x_0| of each sample
        ("threshold_ratio", c_double),
        ("threshold_max", c_double),  # upper bound of the threshold; <= 0 = none
    ]


class OpConvT(Structure):
    _fields_ = [
        ("act0_dev", c_void_p), ("C0", c_int), ("ksize", c_int), ("w0_host", c_void_p), ("b0_host", c_void_p),
        ("e4m3", c_int), ("e_out", POINTER(c_int)),
        ("act1_dev", c_void_p), ("C1", c_int), ("act2_dev", c_void_p), ("C2", c_int), ("wskip_host", c_void_p),
        ("bskip_host", c_void_p),
        ("residual_dev", c_void_p), ("residual_up", c_int),
        ("N", c_int), ("H", c_int), ("W", c_int), ("Cout", c_int),
        ("out_dev", c_void_p), ("out_mode", c_int), ("out16_dev", c_void_p), ("stats_dev", c_void_p),
    ]


class OpGnT(Structure):
    _fields_ = [
        ("x0_dev", c_void_p), ("C0", c_int), ("x1_dev", c_void_p), ("C1", c_int), ("x_fp16", c_int),
        ("stats0_dev", c_void_p), ("stats1_dev", c_void_p),
        ("N", c_int), ("H", c_int), ("W", c_int), ("groups", c_int), ("eps", c_float),
        ("gamma_host", c_void_p), ("beta_host", c_void_p),
        ("film_dev", c_void_p), ("film_ld", c_int), ("film_off", c_int), ("film_add", c_int),
        ("silu", c_int), ("mode", c_int),
        ("out_dev", c_void_p), ("out_e4m3", c_int), ("out_lo_dev", c_void_p), ("out_raw16_dev", c_void_p),
        ("out_raw32_dev", c_void_p),
    ]


class OpResampleT(Structure):
    _fields_ = [
        ("mode", c_int), ("conv", c_int),
        ("x_dev", c_void_p), ("N", c_int), ("H", c_int), ("W", c_int), ("C", c_int),
        ("w_host", c_void_p), ("b_host", c_void_p),
        ("out_dev", c_void_p), ("out16_dev", c_void_p), ("stats_dev", c_void_p), ("operand_dev", c_void_p),
    ]


class WarpParamsT(Structure):
    _fields_ = [("fov_deg", c_double), ("near", c_double), ("far", c_double), ("atol", c_double), ("rtol", c_double),
                ("erode_rgb", c_int), ("padding", c_double)]


class FusionGridT(Structure):
    _fields_ = [("origin", c_float * 3), ("voxel", c_float), ("dims", c_int * 3)]


# name -> (restype, argtypes); also the list tests/test_abi.py checks against the header
SIGNATURES = {
    "ivid_last_error": (c_char_p, []),
    "ivid_version": (c_int, []),
    "ivid_device_info": (c_int, [c_int, POINTER(c_int), POINTER(c_int), POINTER(c_int)]),
    "ivid_unet_create": (c_int, [c_char_p, POINTER(c_void_p)]),
    "ivid_unet_destroy": (c_int, [c_void_p]),
    "ivid_unet_num_params": (c_int, [c_void_p, POINTER(c_int)]),
    "ivid_unet_param_info": (c_int, [c_void_p, c_int, POINTER(c_char_p), POINTER(c_int64), POINTER(c_int), POINTER(c_int)]),
    "ivid_unet_set_param": (c_int, [c_void_p, c_char_p, c_void_p, POINTER(c_int64), c_int]),
    "ivid_unet_finalize": (c_int, [c_void_p, c_int]),
    "ivid_unet_weight_arena": (c_int, [c_void_p, POINTER(c_void_p), POINTER(c_uint64)]),
    "ivid_unet_set_precision": (c_int, [c_void_p, c_int]),
    "ivid_fp8_e4m3_quantize": (c_int, [c_void_p, c_void_p, c_uint64]),
    "ivid_fp8_weight_exponent": (c_int, [c_void_p, c_uint64, POINTER(c_int)]),
    "ivid_unet_forward": (c_int, [c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_int, c_void_p]),
    "ivid_unet_forward_cond": (c_int, [c_void_p, c_void_p, c_int, POINTER(CondT), c_void_p, c_void_p, c_void_p, c_int, c_void_p]),
    "ivid_unet_forward_hw": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, POINTER(CondT), c_void_p, c_void_p, c_void_p, c_int,
                                     c_void_p]),
    "ivid_unet_forward_reuse": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, POINTER(CondT), c_void_p, c_void_p, c_void_p,
                                        c_int, c_int, c_void_p]),
    "ivid_unet_forward_perturbed": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, POINTER(CondT), c_void_p, c_void_p, c_void_p,
                                            c_int, c_int, POINTER(c_int), c_int, c_int, c_void_p]),
    "ivid_conv_tile": (c_int, [c_int, c_int, POINTER(c_int), POINTER(c_int), POINTER(c_int), POINTER(c_int)]),
    "ivid_unet_debug_tap": (c_int, [c_void_p, c_int, c_char_p, c_void_p, c_uint64, POINTER(c_int), POINTER(c_int), POINTER(c_int)]),
    "ivid_unet_profile_begin": (c_int, [c_void_p]),
    "ivid_unet_profile_end": (c_int, [c_void_p, c_char_p, c_int]),
    "ivid_sampler_create": (c_int, [POINTER(c_double), c_int, POINTER(c_void_p)]),
    "ivid_sampler_destroy": (c_int, [c_void_p]),
    "ivid_sampler_table": (c_int, [c_void_p, c_int, POINTER(c_double), c_int]),
    "ivid_sampler_step": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, POINTER(StepArgsT), c_void_p]),
    "ivid_sampler_step_dev": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_void_p, POINTER(StepArgsT), c_void_p]),
    "ivid_cfg_mix": (c_int, [c_void_p, c_float, c_void_p, c_uint64, c_void_p]),
    "ivid_guidance_mix": (c_int, [c_void_p, c_uint64, c_int, c_float, c_int, c_float, c_void_p, c_void_p]),
    "ivid_op_dynamic_threshold": (c_int, [c_void_p, c_int, c_int, c_double, c_double, c_void_p, c_void_p, c_void_p]),
    "ivid_op_apg": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_float, c_double, c_double, c_double, c_void_p, c_void_p]),
    "ivid_sampler_run": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, POINTER(StepArgsT), c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    "ivid_sampler_diffuse": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_uint64, c_int, c_uint64, c_void_p, c_void_p]),
    "ivid_op_conv2d": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_int, c_int, c_void_p, c_int,
                               c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_void_p]),
    "ivid_op_group_norm": (c_int, [c_void_p, c_int, c_void_p, c_int, c_int, c_int, c_int, c_int, c_float, c_void_p, c_void_p,
                                   c_void_p, c_int, c_int, c_void_p, c_void_p]),
    "ivid_op_conv2d_e4m3": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_int, c_int, c_void_p, c_int,
                                    c_void_p, c_void_p, c_void_p, c_void_p, c_int, POINTER(c_int), c_void_p]),
    "ivid_op_group_norm_e4m3": (c_int, [c_void_p, c_int, c_void_p, c_int, c_int, c_int, c_int, c_int, c_float, c_void_p,
                                        c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p]),
    "ivid_op_conv2d_ex": (c_int, [POINTER(OpConvT), c_void_p]),
    "ivid_op_group_norm_apply": (c_int, [POINTER(OpGnT), c_void_p]),
    "ivid_op_gn_stats": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p]),
    "ivid_op_resample": (c_int, [POINTER(OpResampleT), c_void_p]),
    "ivid_op_attention": (c_int, [c_void_p, c_int, c_int, c_int, c_void_p, c_void_p]),
    "ivid_op_attention_heads": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p]),
    "ivid_op_attention_perturbed": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p]),
    "ivid_warp_create": (c_int, [c_int, c_int, c_int, c_int, c_double, c_double, c_int, POINTER(c_void_p)]),
    "ivid_warp_destroy": (c_int, [c_void_p]),
    "ivid_warp_reset": (c_int, [c_void_p]),
    "ivid_warp_num_views": (c_int, [c_void_p, POINTER(c_int)]),
    "ivid_warp_add_view": (c_int, [c_void_p, c_void_p, c_void_p, c_int, POINTER(WarpParamsT), c_void_p]),
    "ivid_warp_mesh_from_depth": (c_int, [c_void_p, c_void_p, c_void_p, POINTER(WarpParamsT), c_void_p, c_void_p, c_void_p]),
    "ivid_warp_set_mesh": (c_int, [c_void_p, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p]),
    "ivid_warp_get_mesh": (c_int, [c_void_p, c_int, c_int, c_void_p, c_void_p, c_void_p]),
    "ivid_warp_render": (c_int, [c_void_p, c_void_p, c_int, c_double, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    "ivid_warp_aggregate": (c_int, [c_void_p, c_void_p, c_int, POINTER(WarpParamsT), c_void_p, c_void_p]),
    "ivid_warp_resolve_frame": (c_int, [c_void_p, c_double, c_double, c_void_p, c_void_p, c_void_p, c_void_p]),
    "ivid_warp_render_simple": (c_int, [c_void_p, c_void_p, c_int, c_void_p, c_int, c_void_p, c_void_p, c_double, c_void_p, c_void_p, c_void_p, c_void_p]),
    "ivid_warp_forward_backward": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, POINTER(WarpParamsT), c_void_p, c_void_p]),
    "ivid_warp_postfilter": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, POINTER(WarpParamsT), c_void_p, c_void_p]),
    "ivid_fusion_integrate": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_float, POINTER(FusionGridT), c_float,
                                      c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    "ivid_fusion_extract": (c_int, [POINTER(FusionGridT), c_void_p, c_void_p, c_void_p, c_void_p, c_int64, c_int64, c_void_p, c_void_p,
                                    c_void_p, POINTER(c_int64), POINTER(c_int64), c_void_p]),
}

_lib = None


def lib() -> ctypes.CDLL:
    """Load (once) and return the native library; raises if it is missing — there is no fallback."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise ImportError(
                f"{LIB_PATH} not found: build it with `python -m ivid_b200.build` (ivid_b200 has no CPU fallback)")
        l = ctypes.CDLL(LIB_PATH)
        for name, (res, args) in SIGNATURES.items():
            try:
                fn = getattr(l, name)
            except AttributeError:
                continue   # symbol check is done by tests/test_abi.py; optional groups may be absent in old builds
            fn.restype = res
            fn.argtypes = args
        _lib = l
    return _lib


def last_error() -> str:
    m = lib().ivid_last_error()
    return m.decode() if m else ""


def check(status: int) -> None:
    if status == IVID_OK:
        return
    msg = last_error()
    if status == IVID_ERR_INVALID_ARGUMENT:
        raise AssertionError(msg)
    if status == IVID_ERR_NOT_IMPLEMENTED:
        raise NotImplementedError(msg)
    raise RuntimeError(f"ivid_b200 native error {status}: {msg}")


def ptr(t) -> c_void_p:
    """Raw data pointer of a torch tensor (or None)."""
    if t is None:
        return c_void_p(None)
    return c_void_p(t.data_ptr())


def cur_stream(device=None) -> c_void_p:
    import torch
    return c_void_p(torch.cuda.current_stream(device).cuda_stream)
