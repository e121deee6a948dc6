"""ctypes binding of the C ABI declared in include/tensoir_b200.h.

The product path has NO fallback: if the shared library is missing or the tensors are not on a
CUDA device, calls raise.  Build the library with ``python -c "import __graft_entry__ as g; g.build()"``
(or ``python -m tensoir_b200.build``).
"""
from __future__ import annotations

import ctypes as C
import os

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("TIR_LIB") or os.path.join(_HERE, "lib", "libtensoir_b200.so")   # TIR_LIB: A/B builds

ABI_VERSION = 4
CNT_MASK, CNT_DENSITY, CNT_APP, CNT_RAYS, CNT_OVERFLOW, CNT_SLOTS = 0, 1, 2, 3, 4, 8
SAMPLE_STEP, SAMPLE_TABLE = 0, 1

f32p = C.c_void_p


class TirField(C.Structure):
    _fields_ = [
        ("dplane", C.c_void_p * 3), ("dline", C.c_void_p * 3), ("aplane", C.c_void_p * 3), ("aline", C.c_void_p * 3),
        ("dC", C.c_int32), ("aC", C.c_int32), ("grid", C.c_int32 * 3),
        ("aabb_lo", C.c_float * 3), ("aabb_hi", C.c_float * 3), ("inv_aabb", C.c_float * 3),
        ("amask", C.c_void_p), ("acell", C.c_void_p), ("agrid", C.c_int32 * 3),
        ("a_lo", C.c_float * 3), ("a_inv", C.c_float * 3), ("occ_lo", C.c_float * 3), ("occ_hi", C.c_float * 3),
        ("density_shift", C.c_float), ("distance_scale", C.c_float), ("weight_thres", C.c_float),
        ("softplus", C.c_int32),
    ]


class TirMlp(C.Structure):
    _fields_ = [
        ("w0", C.c_void_p), ("b0", C.c_void_p), ("w1", C.c_void_p), ("b1", C.c_void_p),
        ("w2", C.c_void_p), ("b2", C.c_void_p), ("basis", C.c_void_p), ("light_line", C.c_void_p),
        ("n_lights", C.c_int32), ("feat_dim", C.c_int32), ("hidden", C.c_int32), ("out_dim", C.c_int32),
        ("pe_feat", C.c_int32), ("pe_x", C.c_int32),
    ]


class TirMarchCfg(C.Structure):
    _fields_ = [
        ("sampling", C.c_int32), ("n_samples", C.c_int32), ("step", C.c_float), ("near", C.c_float),
        ("far", C.c_float), ("z_table", C.c_void_p), ("jitter", C.c_void_p), ("flags", C.c_int32),
    ]


class TirDensityVolume(C.Structure):
    _fields_ = [("data", C.c_void_p), ("lo", C.c_int32 * 3), ("n", C.c_int32 * 3)]


MARCH_NO_BBOX = 1
MARCH_LEAN_COUNTERS = 2
MARCH_CELL_BRICKS = 4


class TirAdamTensor(C.Structure):
    _fields_ = [("p", C.c_void_p), ("g", C.c_void_p), ("m", C.c_void_p), ("v", C.c_void_p), ("n", C.c_int64),
                ("lr_dev", C.c_void_p), ("lr", C.c_float), ("l1", C.c_float), ("step", C.c_void_p)]


class TirTvPlane(C.Structure):
    _fields_ = [("x", C.c_void_p), ("grad", C.c_void_p), ("H", C.c_int32), ("W", C.c_int32), ("C", C.c_int32),
                ("channel_last", C.c_int32), ("scale_h", C.c_float), ("scale_w", C.c_float)]


TV_MAX_PLANES = 3      # TIR_TV_MAX_PLANES


class TirRayMaps(C.Structure):
    _fields_ = [(k, C.c_void_p) for k in ("rgb", "depth", "normal", "albedo", "rough", "fresnel", "nd", "no")]


APP_SAMPLE_BYTES = 24  # sizeof(TirAppSample)
MAX_HEADS = 4          # TIR_MAX_HEADS


# ---- fused primary march (csrc/tir_primary.cu) ------------------------------------------------------------------------
class TirHeadJob(C.Structure):
    _fields_ = [("mlp", TirMlp), ("point_set", C.c_int32), ("x_in", C.c_int32), ("light_mode", C.c_int32),
                ("act", C.c_int32), ("role", C.c_int32)]


class TirPrimaryWork(C.Structure):
    _fields_ = ([("cap_valid", C.c_int64), ("cap_app", C.c_int64)]
                + [(k, C.c_void_p) for k in ("counts", "offsets", "t_last", "acc", "depth", "a_counts", "a_offsets",
                                             "packed", "v_ray", "v_sample", "v_xn", "v_z", "v_dist", "v_feat",
                                             "v_sigma", "v_weight", "v_trans", "a_src", "a_ray", "a_w", "a_xn", "a_xj",
                                             "noise")]
                + [("x0", C.c_void_p * 2), ("inp", C.c_void_p * MAX_HEADS), ("h1", C.c_void_p * MAX_HEADS),
                   ("h2", C.c_void_p * MAX_HEADS), ("out", C.c_void_p * MAX_HEADS), ("dn_feat", C.c_void_p),
                   ("dn_dfdx", C.c_void_p), ("status", C.c_void_p)])


class TirPrimaryBwdWork(C.Structure):
    _fields_ = ([(k, C.c_void_p) for k in ("g_packed", "g_acc", "g_depth", "g_weight", "g_feat")]
                + [("g_out", C.c_void_p * MAX_HEADS), ("gz1", C.c_void_p * MAX_HEADS), ("gz2", C.c_void_p * MAX_HEADS),
                   ("gfeat", C.c_void_p * MAX_HEADS), ("gx0", C.c_void_p * MAX_HEADS), ("g_dn_feat", C.c_void_p),
                   ("g_dn_dfdx", C.c_void_p)])


class TirPrimaryGrads(C.Structure):
    _fields_ = ([("dplane", C.c_void_p * 3), ("dline", C.c_void_p * 3), ("aplane", C.c_void_p * 3),
                 ("aline", C.c_void_p * 3), ("basis", C.c_void_p), ("light_line", C.c_void_p)]
                + [(k, C.c_void_p * MAX_HEADS) for k in ("w0", "b0", "w1", "b1", "w2", "b2")])


# ---- test-view metrics (csrc/tir_eval.cu) ------------------------------------------------------------------------------
class TirEvalView(C.Structure):
    _fields_ = ([("H", C.c_int32), ("W", C.c_int32), ("ssim", C.c_int32), ("reserved", C.c_int32)]
                + [(k, C.c_void_p) for k in ("rgb", "rgb_brdf", "gt_rgb", "albedo", "gt_albedo", "gt_mask", "ratio",
                                             "aligned_single", "aligned_three", "normal", "gt_normal")])


EVAL_N_OUT = 9         # TIR_EVAL_N_OUT


# ---- relighting (csrc/tir_relight.cu) ----------------------------------------------------------------------------------
class TirEnvMap(C.Structure):
    _fields_ = [("H", C.c_int32), ("W", C.c_int32)] + [(k, C.c_void_p) for k in ("rgb", "dir", "pdf_return", "cdf")]


RELIGHT_MAX_LIGHTS = 16   # TIR_RELIGHT_MAX_LIGHTS


# ---- material editing (csrc/tir_edit.cu) -------------------------------------------------------------------------------
class TirEditRule(C.Structure):
    _fields_ = [("flags", C.c_int32), ("albedo_op", C.c_int32), ("rough_op", C.c_int32), ("fresnel_op", C.c_int32),
                ("box_lo", C.c_float * 3), ("box_hi", C.c_float * 3), ("key", C.c_float * 3), ("key_tol", C.c_float),
                ("albedo", C.c_float * 3), ("rough", C.c_float), ("fresnel", C.c_float * 3)]


EDIT_MAX_RULES = 16       # TIR_EDIT_MAX_RULES
EDIT_NONE, EDIT_SET, EDIT_MUL = 0, 1, 2
EDIT_BOX, EDIT_KEY = 1, 2

# ---- analytic lights (csrc/tir_lights.cu) ------------------------------------------------------------------------------
class TirLight(C.Structure):
    _fields_ = [("type", C.c_int32), ("n_samples", C.c_int32), ("dir", C.c_float * 3), ("pos", C.c_float * 3),
                ("power", C.c_float * 3), ("extent", C.c_float), ("cos_inner", C.c_float), ("cos_outer", C.c_float)]


LIGHTS_MAX = 16           # TIR_LIGHTS_MAX
LIGHT_SAMPLES_MAX = 1024  # TIR_LIGHT_SAMPLES_MAX
LIGHT_DIRECTIONAL, LIGHT_POINT, LIGHT_SPOT = 0, 1, 2

PATH_SHADOW_NEAR = 0.05     # TIR_PATH_SHADOW_NEAR (csrc/tir_path.cu)

TRANSPORT_MAX_TEXELS = 2048  # TIR_TRANSPORT_MAX_TEXELS (csrc/tir_transport.cu)

EXPORTS = {
    "tir_abi_version": (C.c_int, []),
    "tir_pack_channels_last": (C.c_int, [f32p, f32p, C.c_int32, C.c_int32, C.c_int32, C.c_void_p]),
    "tir_unpack_channels_last_add": (C.c_int, [f32p, f32p, C.c_int32, C.c_int32, C.c_int32, C.c_void_p]),
    "tir_pack_alpha_mask": (C.c_int, [f32p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_void_p]),
    "tir_alpha_cells_bytes": (C.c_int, [C.c_int32, C.c_int32, C.c_int32, C.POINTER(C.c_int64)]),
    "tir_density_points": (C.c_int, [C.POINTER(TirField), f32p, C.c_int64, f32p, f32p, C.c_void_p]),
    "tir_alpha_mask_points": (C.c_int, [C.POINTER(TirField), f32p, C.c_int64, C.c_void_p, C.c_void_p]),
    "tir_march_density": (C.c_int, [C.POINTER(TirField), f32p, f32p, C.c_int64, C.POINTER(TirMarchCfg),
                                    f32p, f32p, f32p, C.c_void_p, C.c_void_p]),
    "tir_march_radiance": (C.c_int, [C.POINTER(TirField), C.POINTER(TirMlp), f32p, f32p, C.c_void_p, C.c_int64,
                                     C.POINTER(TirMarchCfg), f32p, f32p, f32p, f32p, C.c_void_p, C.c_void_p,
                                     C.c_int64, C.c_void_p, C.c_void_p]),
    "tir_secondary_radiance": (C.c_int, [C.POINTER(TirField), C.POINTER(TirMlp), f32p, f32p, C.c_void_p, C.c_int64,
                                         f32p, C.c_int32, C.POINTER(TirMarchCfg), f32p, f32p, C.c_void_p,
                                         C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p]),
    "tir_secondary_march": (C.c_int, [C.POINTER(TirField), f32p, f32p, C.c_int64, f32p, C.c_int32,
                                      C.POINTER(TirMarchCfg), f32p, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p,
                                      C.c_void_p]),
    "tir_density_volume_extent": (C.c_int, [C.POINTER(TirField), C.POINTER(C.c_int32), C.POINTER(C.c_int32)]),
    "tir_density_volume_build": (C.c_int, [C.POINTER(TirField), C.POINTER(TirDensityVolume), C.c_int64, C.c_void_p]),
    "tir_secondary_radiance_vol": (C.c_int, [C.POINTER(TirField), C.POINTER(TirMlp), f32p, f32p, C.c_void_p,
                                             C.c_int64, f32p, C.c_int32, C.POINTER(TirMarchCfg),
                                             C.POINTER(TirDensityVolume), f32p, f32p, C.c_void_p, C.c_void_p,
                                             C.c_int64, C.c_void_p, C.c_void_p]),
    "tir_secondary_march_vol": (C.c_int, [C.POINTER(TirField), f32p, f32p, C.c_int64, f32p, C.c_int32,
                                          C.POINTER(TirMarchCfg), C.POINTER(TirDensityVolume), f32p, C.c_void_p,
                                          C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p]),
    "tir_app_mlp": (C.c_int, [C.POINTER(TirField), C.POINTER(TirMlp), C.c_void_p, C.c_void_p, C.c_int64, f32p,
                              C.c_int32, C.c_void_p, f32p, C.c_void_p]),
    "tir_app_mlp_points_save": (C.c_int, [C.POINTER(TirField), C.POINTER(TirMlp), f32p, f32p, C.c_void_p, C.c_int64,
                                          C.c_int32, f32p, f32p, f32p, f32p, f32p, C.c_void_p]),
    "tir_shade_fwd": (C.c_int, [f32p, f32p, f32p, f32p, f32p, C.c_void_p, C.c_int64, f32p, f32p, C.c_int32, f32p,
                                C.c_int32, f32p, f32p, f32p, C.c_void_p]),
    "tir_shade_bwd": (C.c_int, [f32p, f32p, f32p, f32p, f32p, C.c_void_p, C.c_int64, f32p, f32p, C.c_int32, f32p,
                                C.c_int32, f32p, f32p, f32p, f32p, f32p, f32p, f32p, f32p, C.c_void_p]),
    "tir_generate_rays": (C.c_int, [f32p, C.c_void_p, C.c_void_p, C.c_int64, C.c_int32, C.c_int32, C.c_float, f32p,
                                    C.c_void_p]),
    "tir_tv_loss": (C.c_int, [C.c_void_p, C.c_int32, f32p, C.c_void_p]),
    "tir_tv_loss_bwd": (C.c_int, [C.c_void_p, C.c_int32, f32p, C.c_void_p]),
    "tir_adam_chunk_elems": (C.c_int, []),
    "tir_adam_step": (C.c_int, [C.c_void_p, C.c_int32, C.c_void_p, C.c_int64, C.c_void_p, C.c_float, C.c_float, C.c_float,
                                C.c_void_p, C.c_int32, C.c_void_p]),
    "tir_hits_prepare": (C.c_int, [f32p, f32p, f32p, C.c_void_p, C.c_int64, f32p, f32p, C.c_void_p]),
    "tir_shade_hits_fwd": (C.c_int, [f32p, C.c_void_p, f32p, f32p, f32p, f32p, C.c_void_p, C.c_int64, f32p, f32p,
                                     C.c_int32, f32p, C.c_int32, f32p, f32p, C.c_int32, f32p, f32p, C.c_void_p]),
    "tir_shade_hits_bwd": (C.c_int, [f32p, C.c_void_p, f32p, f32p, f32p, f32p, C.c_void_p, C.c_int64, f32p, f32p,
                                     C.c_int32, f32p, C.c_int32, f32p, f32p, C.c_int32, f32p, f32p, f32p, f32p, f32p,
                                     f32p, f32p, C.c_void_p]),
    "tir_vm_app_products": (C.c_int, [C.POINTER(TirField), f32p, C.c_int64, f32p, C.c_void_p]),
    "tir_vm_app_products_bwd": (C.c_int, [C.POINTER(TirField), f32p, C.c_int64, f32p, C.POINTER(C.c_void_p),
                                          C.POINTER(C.c_void_p), C.c_void_p]),
    "tir_vm_density_bwd": (C.c_int, [C.POINTER(TirField), f32p, C.c_int64, f32p, C.POINTER(C.c_void_p),
                                     C.POINTER(C.c_void_p), C.c_void_p]),
    "tir_vm_density_grad": (C.c_int, [C.POINTER(TirField), f32p, C.c_int64, f32p, f32p, C.c_void_p]),
    "tir_vm_density_grad_bwd": (C.c_int, [C.POINTER(TirField), f32p, C.c_int64, f32p, f32p, C.POINTER(C.c_void_p),
                                          C.POINTER(C.c_void_p), C.c_void_p]),
    "tir_valid_samples_count": (C.c_int, [C.POINTER(TirField), f32p, f32p, C.c_int64, C.POINTER(TirMarchCfg),
                                          C.c_void_p, C.c_void_p, C.c_void_p]),
    "tir_valid_samples_fill": (C.c_int, [C.POINTER(TirField), f32p, f32p, C.c_int64, C.POINTER(TirMarchCfg),
                                         C.c_void_p, C.c_void_p, C.c_void_p, f32p, f32p, f32p, C.c_int64, C.c_void_p]),
    "tir_composite_fwd": (C.c_int, [f32p, f32p, C.c_void_p, C.c_int64, C.c_float, f32p, f32p, f32p, C.c_int64,
                                    f32p, f32p, f32p, C.c_void_p]),
    "tir_composite_bwd": (C.c_int, [f32p, f32p, C.c_void_p, C.c_int64, C.c_float, f32p, f32p, f32p, f32p,
                                    C.c_int64, f32p, f32p, f32p, C.c_void_p]),
    "tir_primary_march": (C.c_int, [C.POINTER(TirField), C.c_void_p, C.c_int64, C.POINTER(TirMarchCfg),
                                    C.POINTER(TirPrimaryWork), C.c_void_p, C.c_void_p]),
    "tir_primary_app_list": (C.c_int, [C.POINTER(TirField), C.c_int64, C.POINTER(TirPrimaryWork), C.c_void_p]),
    "tir_primary_heads": (C.c_int, [C.POINTER(TirField), C.POINTER(TirHeadJob), C.c_int32, C.c_int32, C.c_void_p,
                                    C.c_void_p, C.c_int64, C.POINTER(TirPrimaryWork), C.c_float, C.c_int32,
                                    C.POINTER(TirRayMaps), C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "tir_primary_backward": (C.c_int, [C.POINTER(TirField), C.POINTER(TirHeadJob), C.c_int32, C.c_int32, C.c_void_p,
                                       C.c_void_p, C.c_int64, C.POINTER(TirPrimaryWork), C.POINTER(TirPrimaryBwdWork),
                                       C.c_float, C.c_int32, C.POINTER(TirRayMaps), C.c_void_p, C.c_void_p, C.c_void_p,
                                       C.POINTER(TirPrimaryGrads), C.c_void_p]),
    "tir_primary_radiance": (C.c_int, [C.POINTER(TirField), C.POINTER(TirHeadJob), C.c_void_p, C.c_void_p, C.c_int64,
                                       C.POINTER(TirPrimaryWork), C.c_int32, f32p, f32p, C.c_void_p]),
    "tir_primary_radiance_backward": (C.c_int, [C.POINTER(TirField), C.POINTER(TirHeadJob), C.c_void_p, C.c_void_p,
                                                C.c_int64, C.POINTER(TirPrimaryWork), C.POINTER(TirPrimaryBwdWork),
                                                C.c_int32, f32p, f32p, f32p, C.POINTER(TirPrimaryGrads),
                                                C.c_void_p]),
    "tir_tail_fwd": (C.c_int, [C.c_int64, f32p, C.c_void_p, f32p, f32p, f32p, f32p, f32p, f32p, f32p, C.c_void_p]),
    "tir_tail_bwd": (C.c_int, [C.c_int64, f32p, C.c_void_p, f32p, f32p, f32p, f32p, f32p, f32p, f32p, f32p, f32p, f32p,
                               f32p, f32p, f32p, C.c_void_p]),
    "tir_epilogue_fwd": (C.c_int, [C.c_int64, f32p, f32p, f32p, f32p, C.c_float, C.c_int32, C.POINTER(TirRayMaps),
                                   C.c_void_p, f32p, C.c_void_p]),
    "tir_epilogue_bwd": (C.c_int, [C.c_int64, f32p, f32p, f32p, f32p, C.c_float, C.c_int32, C.POINTER(TirRayMaps),
                                   f32p, f32p, f32p, f32p, f32p, C.c_void_p]),
    "tir_eval_work_size": (C.c_int, [C.c_int32, C.c_int32, C.POINTER(C.c_int64)]),
    "tir_eval_view": (C.c_int, [C.POINTER(TirEvalView), C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p]),
    "tir_eval_pairs_work_size": (C.c_int, [C.c_int32, C.c_int32, C.c_int32, C.POINTER(C.c_int64)]),
    "tir_eval_pairs": (C.c_int, [f32p, f32p, C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_int64, C.c_void_p,
                                 C.c_void_p]),
    "tir_relight_sample": (C.c_int, [C.POINTER(TirEnvMap), C.c_int32, f32p, f32p, f32p, f32p, C.c_int64, C.c_int32,
                                     C.c_float, C.c_void_p, C.c_void_p, C.c_void_p, f32p, f32p, C.c_int64, C.c_void_p,
                                     C.c_void_p]),
    "tir_relight_shade": (C.c_int, [C.POINTER(TirEnvMap), C.c_int32, f32p, f32p, f32p, f32p, C.c_int32, f32p, f32p,
                                    C.c_int64, C.c_int32, C.c_float, f32p, C.c_void_p, C.c_void_p, f32p, C.c_int32,
                                    f32p, f32p, C.c_int64, C.c_int64, C.c_void_p]),
    "tir_relight_mis_sample": (C.c_int, [C.POINTER(TirEnvMap), C.c_int32, f32p, f32p, f32p, f32p, f32p, C.c_int32,
                                         f32p, f32p, C.c_int64, C.c_int32, C.c_int32, C.c_float, C.c_void_p,
                                         C.c_void_p, f32p, C.c_void_p, f32p, f32p, C.c_int64, C.c_void_p, C.c_void_p]),
    "tir_relight_mis_shade": (C.c_int, [C.POINTER(TirEnvMap), C.c_int32, f32p, f32p, f32p, f32p, C.c_int32, f32p,
                                        f32p, C.c_int64, C.c_int32, C.c_int32, C.c_float, f32p, f32p, C.c_void_p, f32p,
                                        C.c_int32, f32p, f32p, f32p, C.c_int64, C.c_int64, C.c_void_p]),
    "tir_material_edit": (C.c_int, [C.POINTER(TirEditRule), C.c_int32, f32p, f32p, f32p, f32p, f32p, C.c_int32, f32p,
                                    f32p, C.c_int64, C.c_float, f32p, f32p, f32p, f32p, C.c_void_p, C.c_void_p]),
    "tir_lights_sample": (C.c_int, [C.POINTER(TirLight), C.c_int32, f32p, f32p, f32p, f32p, C.c_int64, C.c_float,
                                    C.c_void_p, f32p, f32p, C.c_void_p, f32p, f32p, C.c_int64, C.c_void_p, C.c_void_p]),
    "tir_lights_shade": (C.c_int, [C.POINTER(TirLight), C.c_int32, f32p, f32p, f32p, f32p, C.c_int32, f32p, f32p,
                                   C.c_int64, C.c_float, f32p, f32p, f32p, f32p, C.c_void_p, f32p, C.c_int32, f32p,
                                   f32p, f32p, C.c_int64, C.c_int64, C.c_void_p]),
    "tir_transport_sample": (C.c_int, [f32p, C.c_int32, f32p, f32p, f32p, f32p, C.c_int64, C.c_float, C.c_void_p,
                                       f32p, f32p, C.c_int64, C.c_void_p, C.c_void_p]),
    "tir_transport_build": (C.c_int, [f32p, f32p, C.c_int32, f32p, f32p, f32p, f32p, C.c_int32, f32p, f32p, C.c_int64,
                                      C.c_float, f32p, C.c_void_p, f32p, C.c_int32, f32p, C.c_void_p]),
    "tir_indirect_sample": (C.c_int, [f32p, f32p, f32p, f32p, f32p, C.c_int32, f32p, f32p, C.c_int64, C.c_int32,
                                      C.c_float, f32p, C.c_void_p, f32p, f32p, C.c_void_p, f32p, f32p, C.c_int64,
                                      C.c_void_p, C.c_void_p]),
    "tir_indirect_hits_work_size": (C.c_int, [C.c_int64, C.c_int32, C.POINTER(C.c_int64)]),
    "tir_indirect_hits": (C.c_int, [C.c_int64, C.c_int32, C.c_void_p, f32p, f32p, f32p, f32p, f32p, C.c_int32,
                                    C.POINTER(C.c_float), f32p, f32p, f32p, C.c_void_p, C.c_int64, C.c_void_p,
                                    C.c_void_p, C.c_int64, C.c_void_p]),
    "tir_indirect_radiance": (C.c_int, [C.POINTER(TirEnvMap), C.c_int32, f32p, f32p, f32p, f32p, C.c_int32, f32p,
                                        C.c_int64, C.c_int32, f32p, C.c_void_p, C.c_void_p, f32p, C.c_int32, f32p,
                                        C.c_int64, C.c_int64, C.c_void_p]),
    "tir_indirect_shade": (C.c_int, [C.POINTER(TirEnvMap), C.c_int32, f32p, f32p, f32p, f32p, C.c_int32, f32p, f32p,
                                     C.c_int64, C.c_int32, C.c_float, f32p, C.c_void_p, C.c_void_p, f32p, C.c_int32,
                                     C.c_int32, f32p, C.c_void_p, f32p, f32p, C.c_int64, f32p, f32p, f32p, C.c_int64,
                                     C.c_int64, C.c_void_p]),
    "tir_ground_sample": (C.c_int, [C.POINTER(TirEnvMap), C.c_int32, f32p, C.c_int64, C.c_float, C.POINTER(C.c_float),
                                    C.POINTER(C.c_float), C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, f32p, f32p,
                                    C.c_int64, C.c_void_p, C.c_void_p]),
    "tir_path_composite": (C.c_int, [C.POINTER(TirEnvMap), C.c_int32, f32p, f32p, C.c_int64, C.POINTER(C.c_float),
                                     C.c_float, C.c_void_p, C.c_void_p, f32p, C.c_int32, C.c_int32, f32p, f32p, f32p,
                                     C.c_int64, C.c_int64, C.c_void_p]),
    "tir_ground_lights_sample": (C.c_int, [C.POINTER(TirLight), C.c_int32, f32p, C.c_int64, C.c_float,
                                           C.POINTER(C.c_float), C.POINTER(C.c_float), C.c_void_p, f32p, C.c_void_p,
                                           f32p, f32p, C.c_int64, C.c_void_p, C.c_void_p]),
    "tir_path_lights_composite": (C.c_int, [C.POINTER(TirLight), C.c_int32, f32p, f32p, C.c_int64, C.c_float,
                                            C.POINTER(C.c_float), C.POINTER(C.c_float), f32p, C.c_void_p, f32p,
                                            C.c_int32, f32p, f32p, f32p, C.c_int64, C.c_int64, C.c_void_p]),
    "tir_marching_cubes_work_size": (C.c_int, [C.c_int32, C.c_int32, C.c_int32, C.POINTER(C.c_int64)]),
    "tir_marching_cubes_count": (C.c_int, [f32p, C.c_int32, C.c_int32, C.c_int32, C.c_float, C.c_void_p, C.c_int64,
                                           C.c_void_p, C.c_void_p]),
    "tir_marching_cubes_emit": (C.c_int, [f32p, C.c_int32, C.c_int32, C.c_int32, C.c_float, C.c_double, C.c_double,
                                          C.c_double, C.c_void_p, C.c_int64, C.c_int64, C.c_int64, f32p, C.c_void_p,
                                          C.c_void_p]),
    "tir_atlas_texels": (C.c_int, [C.c_void_p, C.c_int64, f32p, C.c_int32, C.c_int32, C.c_int64, C.c_int64, C.c_void_p,
                                   f32p, C.c_void_p]),
    "tir_atlas_encode": (C.c_int, [C.c_void_p, C.c_int64, f32p, C.c_int32, C.c_int32, C.c_int64, C.c_int64, f32p, f32p,
                                   f32p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "tir_atlas_corners": (C.c_int, [C.c_void_p, C.c_int64, f32p, C.c_int32, C.c_int32, f32p, f32p, f32p, f32p,
                                    C.c_void_p]),
}

# kernels launched per entry point (for bench.py's gpu_launches claim)
KERNELS_PER_CALL = {"tir_pack_channels_last": 1, "tir_unpack_channels_last_add": 1, "tir_pack_alpha_mask": 3,
                    "tir_density_points": 1, "tir_alpha_mask_points": 1, "tir_march_density": 1,
                    "tir_march_radiance": 2, "tir_secondary_march": 1, "tir_secondary_radiance": 2,
                    "tir_density_volume_build": 1, "tir_secondary_march_vol": 1, "tir_secondary_radiance_vol": 2, "tir_app_mlp": 1,
                    "tir_shade_fwd": 1, "tir_shade_bwd": 1, "tir_app_mlp_points_save": 1, "tir_vm_app_products": 1, "tir_vm_app_products_bwd": 1,
                    "tir_vm_density_bwd": 1, "tir_vm_density_grad": 1, "tir_vm_density_grad_bwd": 1,
                    "tir_valid_samples_count": 1, "tir_valid_samples_fill": 1, "tir_composite_fwd": 1,
                    "tir_adam_step": 2, "tir_tv_loss": 1, "tir_tv_loss_bwd": 1, "tir_generate_rays": 1, "tir_hits_prepare": 1, "tir_shade_hits_fwd": 1, "tir_shade_hits_bwd": 1,
                    "tir_primary_march": 6, "tir_primary_app_list": 1, "tir_primary_heads": 5,
                    "tir_primary_backward": 9, "tir_primary_radiance": 2, "tir_primary_radiance_backward": 6,
                    "tir_composite_bwd": 1, "tir_tail_fwd": 1, "tir_tail_bwd": 1, "tir_epilogue_fwd": 1,
                    "tir_epilogue_bwd": 1, "tir_eval_view": 3, "tir_relight_sample": 1, "tir_relight_shade": 1,
                    "tir_relight_mis_sample": 1, "tir_relight_mis_shade": 1, "tir_material_edit": 1, "tir_lights_sample": 1, "tir_lights_shade": 1,
                    "tir_transport_sample": 1, "tir_transport_build": 1,
                    "tir_indirect_sample": 1, "tir_indirect_hits": 3, "tir_indirect_radiance": 1,
                    "tir_indirect_shade": 1, "tir_marching_cubes_count": 7, "tir_marching_cubes_emit": 2,
                    "tir_atlas_texels": 1, "tir_atlas_encode": 1, "tir_atlas_corners": 1,
                    "tir_ground_sample": 1, "tir_path_composite": 1,
                    "tir_ground_lights_sample": 1, "tir_path_lights_composite": 1}
launch_count = 0

_lib = None


class _Counted:
    """Thin callable that counts kernel launches per C-ABI call."""

    def __init__(self, fn, k):
        self.fn, self.k = fn, k

    def __call__(self, *a):
        global launch_count
        launch_count += self.k
        return self.fn(*a)


class _LibProxy:
    def __init__(self, cdll):
        self._cdll = cdll
        for name in EXPORTS:
            fn = getattr(cdll, name)
            k = KERNELS_PER_CALL.get(name, 0)
            setattr(self, name, _Counted(fn, k) if k else fn)


class TirError(RuntimeError):
    pass


def load():
    """Load the shared library once; raise loudly if it has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise TirError(f"{LIB_PATH} not found: the CUDA extension is not built. Run "
                       f"`python -c 'import __graft_entry__ as g; g.build()'` from the repo root. "
                       f"tensoir_b200 has no CPU / PyTorch fallback.")
    lib = C.CDLL(LIB_PATH)
    for name, (res, args) in EXPORTS.items():
        fn = getattr(lib, name)
        fn.restype = res
        fn.argtypes = args
    v = lib.tir_abi_version()
    if v != ABI_VERSION:
        raise TirError(f"ABI version mismatch: library {v}, binding {ABI_VERSION}")
    _lib = _LibProxy(lib)
    return _lib


_STATUS = {-1: "TIR_ERR_NULL", -2: "TIR_ERR_SHAPE", -3: "TIR_ERR_CONFIG", -4: "TIR_ERR_CAPACITY"}


def check(rc, what):
    if rc == 0:
        return
    if rc < 0:
        raise TirError(f"{what}: {_STATUS.get(rc, rc)}")
    raise TirError(f"{what}: cudaError {rc}")


def dptr(t, dtype=torch.float32, allow_none=False):
    """Device pointer of a contiguous CUDA tensor (the ABI takes raw device pointers)."""
    if t is None:
        if allow_none:
            return None
        raise TirError("required tensor is None")
    if not t.is_cuda:
        raise TirError("tensoir_b200 kernels need CUDA tensors (no CPU fallback)")
    if dtype is not None and t.dtype != dtype:
        raise TirError(f"expected {dtype}, got {t.dtype}")
    if not t.is_contiguous():
        raise TirError("tensor must be contiguous")
    return C.c_void_p(t.data_ptr())


def stream_ptr():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)
