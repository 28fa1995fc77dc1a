"""ctypes binding of the C-ABI library (include/gf_b200.h).

The product path has NO fallback: if ``libgf_b200.so`` is missing or fails to load, importing an
op raises.  Build it with ``python -m gaussianformer_b200.csrc.build`` (or ``__graft_entry__.build()``).
"""
from __future__ import annotations

import ctypes
import os
from ctypes import POINTER, Structure, c_char_p, c_float, c_int, c_int32, c_size_t, c_uint32, c_void_p

_HERE = os.path.dirname(os.path.abspath(__file__))
# GF_B200_LIB: developer override to A/B an alternative build of the same library (tools/build_variant.py)
LIB_PATH = os.environ.get("GF_B200_LIB") or os.path.join(_HERE, "csrc", "libgf_b200.so")

GF_OK = 0
GF_SPLAT_BASE, GF_SPLAT_PROB = 0, 1
GF_FLAG_POINT_OUT_OF_GRID = 1
GF_FLAG_MEAN_OUT_OF_GRID = 2
GF_FLAG_RADIUS_LT_1 = 4
GF_FLAG_GENERIC_PATH = 256
GF_ERR_INVALID_ARG = 1
GF_ERR_WORKSPACE = 2
GF_ERR_UNSUPPORTED = 4
GF_DTYPE_F32, GF_DTYPE_F16, GF_DTYPE_BF16 = 0, 1, 2
GF_BWD_DETERMINISTIC = 1
GF_OCC_LOGITS, GF_OCC_PROBS = 0, 1
GF_OCC_VOXEL_MAJOR, GF_OCC_CLASS_MAJOR = 0, 1
GF_FLAG_LABEL_OUT_OF_RANGE = 8
GF_FLAG_INDEX_OUT_OF_RANGE = 16
GF_SUBM_DW_PIECES = 8
GF_REFINE_V1, GF_REFINE_V2 = 0, 1
GF_REFINE_IDENTITY, GF_REFINE_SOFTMAX, GF_REFINE_SOFTPLUS = 0, 1, 2
GF_REFINE_MAX_SEMANTICS = 32
# include/gf_b200_debug.h: route word of a deterministic backward
GF_DEBUG_ROUTE_BIN, GF_DEBUG_ROUTE_SLOT_OVERFLOW, GF_DEBUG_ROUTE_STRAY_POINTS, GF_DEBUG_ROUTE_GAUSSIAN = 0, 1, 2, 3

# include/gf_b200_debug.h: measurement hooks, not the drop-in boundary
DEBUG_EXPORTS = ("gf_debug_set_render_events", "gf_debug_gather_probe", "gf_debug_splat_backward_plan",
                 "gf_debug_splat_backward_route", "gf_debug_daf_plan", "gf_debug_occ_loss_order",
                 "gf_debug_subm_conv_neighbors")
EXPORTS = (
    "gf_abi_version", "gf_last_error", "gf_splat_supported_classes",
    "gf_splat_forward_workspace_bytes", "gf_splat_backward_workspace_bytes",
    "gf_splat_forward", "gf_splat_backward", "gf_splat_read_flags",
    "gf_daf_forward", "gf_daf_backward", "gf_daf_format", "gf_splat_ce_partials",
    "gf_daf_fused_supported", "gf_daf_fused_forward", "gf_daf_fused_backward",
    "gf_daf_forward_ex", "gf_daf_backward_ex", "gf_daf_fused_forward_ex", "gf_daf_fused_backward_ex",
    "gf_daf_format_ex", "gf_splat_backward_workspace_bytes_ex", "gf_splat_backward_ex",
    "gf_daf_backward_workspace_bytes", "gf_daf_backward_ex2", "gf_daf_fused_backward_workspace_bytes",
    "gf_daf_fused_backward_ex2", "gf_daf_project", "gf_daf_project_backward",
    "gf_daf_anchor_key_points", "gf_daf_anchor_key_points_backward",
    "gf_occ_loss_workspace_bytes", "gf_occ_loss",
    "gf_subm_conv_workspace_bytes", "gf_subm_conv_rulebook", "gf_subm_conv_forward", "gf_subm_conv_backward",
    "gf_gaussian_refine", "gf_gaussian_refine_backward",
)


class SplatDesc(Structure):
    _fields_ = [("G", c_int32), ("N", c_int32), ("C", c_int32), ("H", c_int32), ("W", c_int32), ("D", c_int32),
                ("variant", c_int32), ("radii_axes", c_int32), ("cov_stride", c_int32),
                ("pc_min", c_float * 3), ("grid_size", c_float), ("scale_multiplier", c_float),
                ("radii_min", c_int32), ("batch", c_int32), ("pts_shared", c_int32)]


class SplatInputs(Structure):
    _fields_ = [("pts", c_void_p), ("points_int", c_void_p), ("means", c_void_p), ("means_int", c_void_p),
                ("opacities", c_void_p), ("semantics", c_void_p), ("cov", c_void_p), ("radii", c_void_p),
                ("scales", c_void_p), ("rotations", c_void_p)]


class SplatOutputs(Structure):
    _fields_ = [("logits", c_void_p), ("bin_logits", c_void_p), ("density", c_void_p), ("probability", c_void_p),
                ("argmax", c_void_p), ("logits_cn", c_void_p), ("labels", c_void_p), ("class_weights", c_void_p),
                ("ce_partials", c_void_p)]


class SplatGrads(Structure):
    _fields_ = [("logits_grad", c_void_p), ("bin_logits_grad", c_void_p), ("density_grad", c_void_p),
                ("logits", c_void_p), ("bin_logits", c_void_p), ("probability", c_void_p),
                ("means_grad", c_void_p), ("opacity_grad", c_void_p), ("semantics_grad", c_void_p),
                ("cov_grad", c_void_p), ("scales_grad", c_void_p), ("rotations_grad", c_void_p)]


class DafDesc(Structure):
    _fields_ = [("batch", c_int32), ("num_cams", c_int32), ("num_feat", c_int32), ("num_embeds", c_int32),
                ("num_scale", c_int32), ("num_pts", c_int32), ("num_groups", c_int32)]


class DafFusedDesc(Structure):
    _fields_ = [("d", DafDesc), ("pts_per_anchor", c_int32)]


DAF_MAX_LEVELS = 8


class DafFormatDesc(Structure):
    _fields_ = [("batch_cams", c_int32), ("num_embeds", c_int32), ("num_scale", c_int32),
                ("hw", c_int32 * DAF_MAX_LEVELS)]


class DafKpsDesc(Structure):
    _fields_ = [("batch", c_int32), ("num_anchors", c_int32), ("anchor_dim", c_int32), ("num_fixed", c_int32),
                ("num_learnable", c_int32), ("lo", c_float * 3), ("extent", c_float * 3), ("scale_lo", c_float),
                ("scale_extent", c_float), ("learnable_fixed_scale", c_float)]


class OccLossDesc(Structure):
    _fields_ = [("batch", c_int32), ("N", c_int32), ("C", c_int32), ("branch", c_int32), ("layout", c_int32),
                ("ignore_index", c_int32), ("lovasz_ignore", c_int32), ("empty_label", c_int32),
                ("weight", c_float), ("ce_weight", c_float), ("lovasz_weight", c_float)]


class SubmConvDesc(Structure):
    _fields_ = [("batch", c_int32), ("num_rows", c_int32), ("X", c_int32), ("Y", c_int32), ("Z", c_int32),
                ("kernel_size", c_int32), ("c_in", c_int32), ("c_out", c_int32)]


class RefineDesc(Structure):
    _fields_ = [("variant", c_int32), ("batch", c_int32), ("num_anchors", c_int32), ("out_dim", c_int32),
                ("anchor_dim", c_int32), ("refine_prefix", c_int32), ("restrict_xyz", c_int32),
                ("include_opa", c_int32), ("semantic_dim", c_int32), ("semantics_act", c_int32),
                ("lo", c_float * 3), ("extent", c_float * 3), ("unit", c_float * 3), ("scale_lo", c_float),
                ("scale_extent", c_float)]


REFINE_OUTPUTS = ("new_anchor", "means", "scales", "rotations", "opacities", "semantics", "original_means",
                  "delta_means")


class RefineOutputs(Structure):
    _fields_ = [(n, c_void_p) for n in REFINE_OUTPUTS]


class RefineGrads(Structure):
    _fields_ = [(n, c_void_p) for n in REFINE_OUTPUTS]


class GfError(RuntimeError):
    pass


_lib = None


def lib():
    """The loaded library; raises (never falls back) when it is absent."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise ImportError(
                f"{LIB_PATH} is missing: the CUDA extension has not been built "
                "(run `python -m gaussianformer_b200.csrc.build`). There is no CPU fallback.")
        L = ctypes.CDLL(LIB_PATH)
        L.gf_abi_version.restype = c_int
        L.gf_last_error.restype = c_char_p
        L.gf_splat_supported_classes.argtypes = [POINTER(c_int32), c_int]
        L.gf_splat_forward_workspace_bytes.restype = c_size_t
        L.gf_splat_forward_workspace_bytes.argtypes = [POINTER(SplatDesc)]
        L.gf_splat_backward_workspace_bytes.restype = c_size_t
        L.gf_splat_backward_workspace_bytes.argtypes = [POINTER(SplatDesc)]
        L.gf_splat_forward.argtypes = [POINTER(SplatDesc), POINTER(SplatInputs), POINTER(SplatOutputs), c_void_p,
                                       c_size_t, c_void_p]
        L.gf_splat_backward.argtypes = [POINTER(SplatDesc), POINTER(SplatInputs), POINTER(SplatGrads), c_void_p,
                                        c_size_t, c_void_p]
        L.gf_splat_backward_workspace_bytes_ex.restype = c_size_t
        L.gf_splat_backward_workspace_bytes_ex.argtypes = [POINTER(SplatDesc), c_uint32]
        L.gf_splat_backward_ex.argtypes = [POINTER(SplatDesc), c_uint32, POINTER(SplatInputs), POINTER(SplatGrads),
                                           c_void_p, c_size_t, c_void_p]
        L.gf_debug_splat_backward_plan.argtypes = [ctypes.c_int64, c_int32]
        L.gf_debug_splat_backward_route.argtypes = [POINTER(SplatDesc), c_void_p, c_void_p, POINTER(c_uint32)]
        L.gf_splat_read_flags.argtypes = [c_void_p, c_void_p, POINTER(c_uint32)]
        L.gf_debug_set_render_events.argtypes = [c_void_p, c_void_p]
        L.gf_debug_gather_probe.argtypes = [c_void_p, c_void_p, ctypes.c_int64, c_int32, c_void_p, c_void_p]
        L.gf_splat_ce_partials.argtypes = [POINTER(SplatDesc)]
        L.gf_splat_ce_partials.restype = c_int
        L.gf_daf_forward.argtypes = [POINTER(DafDesc)] + [c_void_p] * 7
        L.gf_daf_backward.argtypes = [POINTER(DafDesc)] + [c_void_p] * 10
        L.gf_daf_fused_supported.argtypes = [POINTER(DafFusedDesc)]
        L.gf_daf_fused_forward.argtypes = [POINTER(DafFusedDesc)] + [c_void_p] * 10
        L.gf_daf_fused_backward.argtypes = [POINTER(DafFusedDesc)] + [c_void_p] * 14
        L.gf_daf_format.argtypes = [POINTER(DafFormatDesc), POINTER(c_void_p), c_void_p, c_int, c_void_p]
        L.gf_daf_forward_ex.argtypes = [POINTER(DafDesc), c_int32] + [c_void_p] * 7
        L.gf_daf_backward_ex.argtypes = [POINTER(DafDesc), c_int32] + [c_void_p] * 10
        L.gf_daf_fused_forward_ex.argtypes = [POINTER(DafFusedDesc), c_int32] + [c_void_p] * 10
        L.gf_daf_fused_backward_ex.argtypes = [POINTER(DafFusedDesc), c_int32] + [c_void_p] * 14
        L.gf_daf_format_ex.argtypes = [POINTER(DafFormatDesc), c_int32, POINTER(c_void_p), c_void_p, c_int, c_void_p]
        L.gf_daf_backward_workspace_bytes.restype = c_size_t
        L.gf_daf_backward_workspace_bytes.argtypes = [POINTER(DafDesc), c_uint32]
        L.gf_daf_backward_ex2.argtypes = [POINTER(DafDesc), c_int32, c_uint32] + [c_void_p] * 10 + [c_size_t, c_void_p]
        L.gf_daf_fused_backward_workspace_bytes.restype = c_size_t
        L.gf_daf_fused_backward_workspace_bytes.argtypes = [POINTER(DafFusedDesc), c_uint32]
        L.gf_daf_fused_backward_ex2.argtypes = ([POINTER(DafFusedDesc), c_int32, c_uint32] + [c_void_p] * 14 +
                                                [c_size_t, c_void_p])
        L.gf_debug_daf_plan.argtypes = [c_int32]
        L.gf_daf_project.argtypes = [c_int32, c_int32, c_int32] + [c_void_p] * 6
        L.gf_daf_project_backward.argtypes = [c_int32, c_int32, c_int32] + [c_void_p] * 6
        L.gf_daf_anchor_key_points.argtypes = [POINTER(DafKpsDesc)] + [c_void_p] * 5
        L.gf_daf_anchor_key_points_backward.argtypes = [POINTER(DafKpsDesc)] + [c_void_p] * 7
        L.gf_occ_loss_workspace_bytes.restype = c_size_t
        L.gf_occ_loss_workspace_bytes.argtypes = [POINTER(OccLossDesc)]
        L.gf_occ_loss.argtypes = [POINTER(OccLossDesc)] + [c_void_p] * 7 + [c_size_t, c_void_p]
        L.gf_debug_occ_loss_order.argtypes = [POINTER(OccLossDesc), c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]
        L.gf_subm_conv_workspace_bytes.restype = c_size_t
        L.gf_subm_conv_workspace_bytes.argtypes = [POINTER(SubmConvDesc)]
        L.gf_subm_conv_rulebook.argtypes = [POINTER(SubmConvDesc), c_void_p, c_void_p, c_size_t, c_void_p]
        L.gf_subm_conv_forward.argtypes = [POINTER(SubmConvDesc)] + [c_void_p] * 6
        L.gf_subm_conv_backward.argtypes = [POINTER(SubmConvDesc)] + [c_void_p] * 8
        L.gf_debug_subm_conv_neighbors.argtypes = [POINTER(SubmConvDesc)] + [c_void_p] * 6
        L.gf_gaussian_refine.argtypes = [POINTER(RefineDesc), c_void_p, c_void_p, POINTER(RefineOutputs), c_void_p]
        L.gf_gaussian_refine_backward.argtypes = [POINTER(RefineDesc), c_void_p, c_void_p, POINTER(RefineGrads),
                                                  c_void_p, c_void_p, c_void_p]
        if L.gf_abi_version() != 2:
            raise ImportError("libgf_b200.so: ABI version mismatch")
        _lib = L
    return _lib


def check(rc: int):
    if rc != GF_OK:
        raise GfError(f"gf_b200 error {rc}: {lib().gf_last_error().decode()}")


def supported_classes():
    buf = (c_int32 * 32)()
    n = lib().gf_splat_supported_classes(buf, 32)
    return [int(buf[i]) for i in range(n)]
