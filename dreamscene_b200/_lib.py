"""ctypes binding of libb200gsr.so (include/b200gsr.h, include/b200gsr_scene.h, include/b200gsr_step.h,
include/b200gsr_loss.h, include/b200gsr_frozen.h, include/b200gsr_stats.h,
include/b200gsr_reserve.h, include/b200gsr_frames.h, include/b200gsr_views_frozen.h, include/b200gsr_views_stats.h,
include/b200gsr_fields.h, include/b200gsr_mesh.h, include/b200gsr_mesh_colour.h, include/b200gsr_mesh_clean.h,
include/b200gsr_mesh_decimate.h).  Fails loudly if the library is missing: there is NO CPU or PyTorch fallback in the product path."""
from __future__ import annotations

import ctypes as C
import os
from typing import Optional

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("B200GSR_LIB", os.path.join(HERE, "libb200gsr.so"))   # override: A/B builds only


class Params(C.Structure):
    _fields_ = [("P", C.c_int32), ("M", C.c_int32), ("sh_degree", C.c_int32),
                ("image_height", C.c_int32), ("image_width", C.c_int32),
                ("tanfovx", C.c_float), ("tanfovy", C.c_float), ("scale_modifier", C.c_float),
                ("prefiltered", C.c_int32), ("score_flag", C.c_int32),
                ("bg", C.c_void_p), ("viewmatrix", C.c_void_p), ("projmatrix", C.c_void_p),
                ("campos", C.c_void_p)]


class Group(C.Structure):           # == b200gsr_group
    _fields_ = [(n, C.c_void_p) for n in ("xyz", "opacity", "scaling", "rotation", "f_dc", "f_rest")] + [("n", C.c_int32)]


class GroupGrad(C.Structure):       # == b200gsr_group_grad
    _fields_ = [(n, C.c_void_p) for n in ("xyz", "opacity", "scaling", "rotation", "f_dc", "f_rest")]


MAX_GROUPS = 24
MAX_VIEWS = 16
SCORE_DET_MAX_PIXELS = 1 << 26     # B200GSR_SCORE_DET_MAX_PIXELS: pixels of all views summed into one int64 score


class ViewInputs(C.Structure):      # == b200gsr_view_inputs
    _fields_ = [(n, C.c_void_p) for n in ("means3D", "shs", "colors_precomp", "opacities", "scales", "rotations", "cov3D_precomp")]


class ViewGrads(C.Structure):       # == b200gsr_view_grads
    _fields_ = [(n, C.c_void_p) for n in ("d_means3D", "d_means2D", "d_shs", "d_colors", "d_opacities", "d_scales",
                                          "d_rotations", "d_cov3D")] + [("accumulate", C.c_uint32)]


ADAM_MAX_TENSORS = 32               # B200GSR_ADAM_MAX_TENSORS: tensors per b200gsr_adam_step call


class AdamTensor(C.Structure):      # == b200gsr_adam_tensor
    _fields_ = [(n, C.c_void_p) for n in ("param", "grad", "exp_avg", "exp_avg_sq")] + [("n", C.c_int64)] + \
        [(n, C.c_float) for n in ("lerp_weight", "beta2", "one_minus_beta2", "eps", "step_size", "bc2_sqrt")]


class SavedLayout(C.Structure):
    _fields_ = [(n, C.c_size_t) for n in ("header", "tile_start", "work_order", "n_contrib",
                                          "keys", "geom", "dgeom", "bwd_items", "total")]


class ScratchLayout(C.Structure):
    _fields_ = [(n, C.c_size_t) for n in ("counters", "tile_count", "tile_cursor", "rectdepth",
                                          "ms_hist", "total")]


i32, u32, u64, sz, f32, vp, _P = C.c_int32, C.c_uint32, C.c_uint64, C.c_size_t, C.c_float, C.c_void_p, C.POINTER
# b200gsr_backward / _ex: the seven inputs, radii, depth_alpha, the two incoming gradients, saved, scratch, max_pairs and
# the eight gradient outputs
_BWD_ARGS = [vp] * 11 + [vp, sz, vp, sz, u64] + [vp] * 8

# Every entry point of include/b200gsr.h: name -> (restype, argtypes), in the header's order.
SIGNATURES = {
    "b200gsr_version": (C.c_int, []),
    "b200gsr_last_error": (C.c_char_p, []),
    "b200gsr_saved_layout_query": (C.c_int, [i32, i32, i32, u64, i32, _P(SavedLayout)]),
    "b200gsr_scratch_layout_query": (C.c_int, [i32, i32, i32, u64, _P(ScratchLayout)]),
    "b200gsr_forward": (C.c_int, [_P(Params)] + [vp] * 11 + [vp, sz, vp, sz, u64, u32, vp, u32, vp]),
    "b200gsr_backward": (C.c_int, [_P(Params)] + _BWD_ARGS + [vp]),
    "b200gsr_backward_ex": (C.c_int, [_P(Params)] + _BWD_ARGS + [u32, i32, i32, i32, vp]),
    "b200gsr_sh_grad_expand": (C.c_int, [i32, i32, i32, i32, vp, vp, sz, vp, vp]),
    "b200gsr_views_geometry": (C.c_int, [i32, i32, i32, _P(i32)]),
    "b200gsr_forward_views": (C.c_int, [i32, _P(Params), _P(ViewInputs)] + [vp] * 5 + [sz, vp, sz, u64, u32, vp, u32, vp]),
    "b200gsr_backward_views": (C.c_int, [i32, _P(Params), _P(ViewInputs)] + [vp] * 5 + [sz, u64, _P(ViewGrads), vp]),
    "b200gsr_backward_views_ex": (C.c_int, [i32, _P(Params), _P(ViewInputs)] + [vp] * 5 + [sz, u64, _P(ViewGrads), u32, vp]),
    "b200gsr_score_views": (C.c_int, [i32, _P(Params), _P(ViewInputs), vp, vp, sz, vp, sz, u64, u32, vp, u32, vp]),
    "b200gsr_score_finish": (C.c_int, [i32, vp, vp, u32, vp]),
    "b200gsr_mark_visible": (C.c_int, [i32, vp, vp, vp, vp, vp]),
    "b200gsr_assemble_forward": (C.c_int, [i32, _P(Group), i32, i32, f32, f32, vp, vp, u64] + [vp] * 5 + [vp]),
    "b200gsr_assemble_backward": (C.c_int, [i32, _P(Group), _P(GroupGrad), i32, i32, f32, f32, vp, vp, u64] + [vp] * 5 + [vp]),
    "b200gsr_disparity_forward": (C.c_int, [i32, i32, vp, vp, vp, vp, vp]),
    "b200gsr_disparity_backward": (C.c_int, [i32, i32, vp, vp, vp, vp, vp, vp, vp]),
    "b200gsr_disparity_backward_ex": (C.c_int, [i32, i32, vp, vp, vp, vp, vp, vp, u32, vp]),
    "b200gsr_densify_stats": (C.c_int, [i32, vp, vp, vp, vp, vp, vp]),
    "b200gsr_densify_scratch_bytes": (C.c_size_t, [i32]),
    "b200gsr_densify_plan": (C.c_int, [i32, vp, vp, vp, vp, f32, f32, f32, f32, f32, vp, vp, vp]),
    "b200gsr_densify_map": (C.c_int, [i32, i32, vp, vp, vp, vp, vp]),
    "b200gsr_compact_plan": (C.c_int, [i32, vp, vp, vp, vp, vp]),
    "b200gsr_gather_rows": (C.c_int, [i32, i32, vp, vp, vp, i32, vp]),
    "b200gsr_split_children": (C.c_int, [i32, i32, f32, vp, vp, vp, vp, vp, vp, vp, vp, vp]),
    "b200gsr_kth_smallest": (C.c_int, [i32, vp, u32, vp, vp, vp]),
    "b200gsr_adam_step": (C.c_int, [i32, _P(AdamTensor), vp]),
    "b200gsr_dist2_scratch_bytes": (C.c_size_t, [i32]),
    "b200gsr_dist2_knn3": (C.c_int, [i32, vp, vp, vp, sz, vp]),
    "b200gsr_profile_enable": (C.c_int, [i32]),
    "b200gsr_debug_counters": (C.c_int, [vp]),
    "b200gsr_profile_counts": (C.c_int, [_P(i32), _P(i32)]),
    "b200gsr_profile_read": (C.c_int, [i32, i32, _P(f32)]),
}
EXPORTS = list(SIGNATURES)

# The scene-render entry points of include/b200gsr_scene.h (same library), in that header's order.
SCENE_SIGNATURES = {
    "b200gsr_forward_scene": (C.c_int, [i32, _P(Params), i32, _P(Group), vp, vp, u64] + [vp] * 5 +
                              [sz, vp, sz, u64, u32, vp, u32, vp]),
    "b200gsr_backward_scene": (C.c_int, [i32, _P(Params), i32, _P(Group), _P(GroupGrad), vp, vp, u64] + [vp] * 6 +
                               [sz, u64, vp, u32, vp]),
}


class StepView(C.Structure):        # == b200gsr_step_view (include/b200gsr_step.h)
    _fields_ = [("tanfovx", C.c_float), ("tanfovy", C.c_float), ("shs_noise", C.c_float), ("scale_noise", C.c_float),
                ("sh_degree", C.c_int32), ("reserved", C.c_int32 * 3)]


# The graph-replay entry points of include/b200gsr_step.h (same library), in that header's order.
STEP_SIGNATURES = {
    "b200gsr_forward_scene_dyn": (C.c_int, [i32, _P(Params), i32, _P(Group), vp, vp] + [vp] * 5 +
                                  [sz, vp, sz, u64, u32, vp, u32, vp]),
    "b200gsr_backward_scene_dyn": (C.c_int, [i32, _P(Params), i32, _P(Group), _P(GroupGrad), vp, vp] + [vp] * 6 +
                                   [sz, u64, vp, u32, vp]),
    "b200gsr_adam_step_dyn": (C.c_int, [i32, _P(AdamTensor), vp, vp]),
    "b200gsr_pair_report": (C.c_int, [vp, vp, vp]),
}

# The loss entry points of include/b200gsr_loss.h (same library), in that header's order.
LOSS_SIGNATURES = {
    "b200gsr_recon_l2_scratch_bytes": (C.c_size_t, [i32, i32]),
    "b200gsr_recon_l2": (C.c_int, [i32, i32, vp, vp, i32, i32, vp, f32, vp, vp, vp, vp, sz, vp]),
    "b200gsr_tv_loss_scratch_bytes": (C.c_size_t, [i32, i32, i32, i32]),
    "b200gsr_tv_loss": (C.c_int, [i32, i32, i32, i32, vp, vp, vp, vp, i32, vp, sz, vp]),
    "b200gsr_scale_loss_scratch_bytes": (C.c_size_t, [i32]),
    "b200gsr_scale_loss": (C.c_int, [i32, vp, vp, vp, vp, i32, vp, sz, vp]),
}

# The frozen-group backwards of include/b200gsr_frozen.h (same library), in that header's order: the arguments of
# b200gsr_backward_scene / _dyn plus the uint32 frozen_groups mask before the stream.
FROZEN_SIGNATURES = {
    "b200gsr_backward_scene_frozen": (C.c_int, [i32, _P(Params), i32, _P(Group), _P(GroupGrad), vp, vp, u64] +
                                      [vp] * 6 + [sz, u64, vp, u32, u32, vp]),
    "b200gsr_backward_scene_dyn_frozen": (C.c_int, [i32, _P(Params), i32, _P(Group), _P(GroupGrad), vp, vp] +
                                          [vp] * 6 + [sz, u64, vp, u32, u32, vp]),
}


class GroupStats(C.Structure):      # == b200gsr_group_stats (include/b200gsr_stats.h)
    _fields_ = [(n, C.c_void_p) for n in ("xyz_gradient_accum", "denom", "max_radii2D")]


# The backwards with the densification statistics of include/b200gsr_stats.h (same library), in that header's order:
# the arguments of b200gsr_backward_scene[_dyn]_frozen up to frozen_groups, then the per-group statistics and the view
# (an int32 by value, a device pointer under _dyn) before the stream.
STATS_SIGNATURES = {
    "b200gsr_backward_scene_stats": (C.c_int, [i32, _P(Params), i32, _P(Group), _P(GroupGrad), vp, vp, u64] +
                                     [vp] * 6 + [sz, u64, vp, u32, u32, _P(GroupStats), i32, vp]),
    "b200gsr_backward_scene_dyn_stats": (C.c_int, [i32, _P(Params), i32, _P(Group), _P(GroupGrad), vp, vp] +
                                         [vp] * 6 + [sz, u64, vp, u32, u32, _P(GroupStats), vp, vp]),
}


class AdamLive(C.Structure):        # == b200gsr_adam_live (include/b200gsr_reserve.h)
    _fields_ = [("rows", C.c_void_p), ("row_floats", C.c_int32), ("reserved", C.c_int32)]


# The entry points over groups with reserved rows of include/b200gsr_reserve.h (same library), in that header's order:
# the arguments of b200gsr_forward_scene_dyn / b200gsr_backward_scene_dyn_stats plus the device live counts before the
# stream; the scale loss over the groups' table; the _dyn Adam step plus one live record per tensor.
RESERVE_SIGNATURES = {
    "b200gsr_forward_scene_dyn_live": (C.c_int, [i32, _P(Params), i32, _P(Group), vp, vp] + [vp] * 5 +
                                       [sz, vp, sz, u64, u32, vp, u32, vp, vp]),
    "b200gsr_backward_scene_dyn_live": (C.c_int, [i32, _P(Params), i32, _P(Group), _P(GroupGrad), vp, vp] +
                                        [vp] * 6 + [sz, u64, vp, u32, u32, _P(GroupStats), vp, vp, vp]),
    "b200gsr_scale_loss_live": (C.c_int, [i32, i32, _P(Group), vp, vp, vp, vp, vp, i32, vp, sz, vp]),
    "b200gsr_adam_step_dyn_live": (C.c_int, [i32, _P(AdamTensor), vp, _P(AdamLive), vp]),
}

# The video-frame entry point of include/b200gsr_frames.h (same library).
FRAMES_SIGNATURES = {
    "b200gsr_frames": (C.c_int, [i32, i32, i32, vp, vp, vp, vp, vp, vp, vp]),
}
FRAMES_STATS_BYTES = 32             # B200GSR_FRAMES_STATS_BYTES: scratch per view of b200gsr_frames


class RowRange(C.Structure):        # == b200gsr_row_range (include/b200gsr_views_frozen.h)
    _fields_ = [("lo", C.c_int32), ("len", C.c_int32)]


# The frozen-row backwards of include/b200gsr_views_frozen.h (same library), in that header's order: the arguments of
# b200gsr_backward_views_ex plus the host range array and its count before the stream; those of
# b200gsr_assemble_backward plus the uint32 frozen_groups mask before the stream.
VIEWS_FROZEN_SIGNATURES = {
    "b200gsr_backward_views_frozen": (C.c_int, [i32, _P(Params), _P(ViewInputs)] + [vp] * 5 +
                                      [sz, u64, _P(ViewGrads), u32, _P(RowRange), i32, vp]),
    "b200gsr_assemble_backward_frozen": (C.c_int, [i32, _P(Group), _P(GroupGrad), i32, i32, f32, f32, vp, vp, u64] +
                                         [vp] * 5 + [u32, vp]),
}
MAX_FROZEN_RANGES = 12              # B200GSR_MAX_FROZEN_RANGES


class RowStats(C.Structure):        # == b200gsr_row_stats (include/b200gsr_views_stats.h)
    _fields_ = [("lo", C.c_int32), ("len", C.c_int32)] + \
        [(n, C.c_void_p) for n in ("xyz_gradient_accum", "denom", "max_radii2D")]


# The statistics-gathering backward of include/b200gsr_views_stats.h (same library): the arguments of
# b200gsr_backward_views_frozen up to num_frozen, then the host record array, its count and the view before the stream.
VIEWS_STATS_SIGNATURES = {
    "b200gsr_backward_views_stats": (C.c_int, [i32, _P(Params), _P(ViewInputs)] + [vp] * 5 +
                                     [sz, u64, _P(ViewGrads), u32, _P(RowRange), i32, _P(RowStats), i32, i32, vp]),
}


class FieldsLayout(C.Structure):    # == b200gsr_fields_layout (include/b200gsr_fields.h)
    _fields_ = [("total", C.c_size_t), ("blocks_per_axis", C.c_int32), ("max_blocks_per_axis", C.c_int32),
                ("max_pairs", C.c_int64)]


class FieldsInfo(C.Structure):      # == b200gsr_fields_info (include/b200gsr_fields.h)
    _fields_ = [("scale", C.c_double), ("center", C.c_float * 3), ("extent", C.c_float), ("kept", C.c_int32),
                ("overflow", C.c_uint32), ("pairs", C.c_int64)]


# The opacity-field entry points of include/b200gsr_fields.h (same library), in that header's order.
FIELDS_SIGNATURES = {
    "b200gsr_fields_layout_query": (C.c_int, [i32, i32, i32, C.c_double, vp, _P(FieldsLayout)]),
    "b200gsr_fields": (C.c_int, [i32, vp, vp, vp, vp, i32, i32, C.c_double, vp, vp, vp, vp, sz, vp]),
}
FIELDS_MAX_R = 1024                 # B200GSR_FIELDS_MAX_R
FIELDS_MAX_CHUNKS = 32              # B200GSR_FIELDS_MAX_CHUNKS


class MeshLayout(C.Structure):      # == b200gsr_mesh_layout (include/b200gsr_mesh.h)
    _fields_ = [("total", C.c_size_t), ("points", C.c_int64), ("cells", C.c_int64)]


# The marching-cubes entry points of include/b200gsr_mesh.h (same library), in that header's order.
MESH_SIGNATURES = {
    "b200gsr_mesh_table": (C.c_int, [_P(C.c_uint8), _P(C.c_int8)]),
    "b200gsr_mesh_layout_query": (C.c_int, [i32, i32, i32, _P(MeshLayout)]),
    "b200gsr_mesh_count": (C.c_int, [i32, i32, i32, vp, f32, vp, vp, sz, vp]),
    "b200gsr_mesh_emit": (C.c_int, [i32, i32, i32, vp, f32, vp, sz, vp, i32, vp, i32, vp]),
}
MESH_MAX_TRIANGLES = 5              # B200GSR_MESH_MAX_TRIANGLES
MESH_TABLE_WIDTH = 15               # B200GSR_MESH_TABLE_WIDTH

# The colour-field and vertex-attribute entry points of include/b200gsr_mesh_colour.h (same library), in that header's
# order.
MESH_COLOUR_SIGNATURES = {
    "b200gsr_fields_rgb_layout_query": (C.c_int, [i32, i32, i32, C.c_double, vp, _P(FieldsLayout)]),
    "b200gsr_fields_rgb": (C.c_int, [i32, vp, vp, vp, vp, vp, i32, i32, C.c_double, vp, vp, vp, vp, vp, sz, vp]),
    "b200gsr_mesh_attributes": (C.c_int, [i32, i32, i32, vp, f32, vp, sz, vp, vp, i32, vp]),
}

# The mesh-component and cleaning entry points of include/b200gsr_mesh_clean.h (same library), in that header's order.
MESH_CLEAN_SIGNATURES = {
    "b200gsr_mesh_clean_layout_query": (C.c_int, [i32, i32, _P(sz)]),
    "b200gsr_mesh_components": (C.c_int, [i32, i32, vp, vp, vp, vp, sz, vp]),
    "b200gsr_mesh_clean_count": (C.c_int, [i32, i32, vp, vp, i32, C.c_double, i32, vp, vp, sz, vp]),
    "b200gsr_mesh_clean_emit": (C.c_int, [i32, i32, vp, vp, i32, C.c_double, i32, vp, sz, vp, vp, vp, i32, i32, vp]),
}

# The decimation entry points of include/b200gsr_mesh_decimate.h (same library), in that header's order.
MESH_DECIMATE_SIGNATURES = {
    "b200gsr_mesh_decimate_layout_query": (C.c_int, [i32, i32, _P(sz)]),
    "b200gsr_mesh_decimate_begin": (C.c_int, [i32, i32, vp, vp, i32, i32, vp, vp, sz, vp]),
    "b200gsr_mesh_decimate_rounds": (C.c_int, [i32, i32, i32, vp, vp, sz, vp]),
    "b200gsr_mesh_decimate_emit": (C.c_int, [i32, i32, vp, vp, sz, vp, vp, vp, i32, i32, vp]),
}
DECIMATE_MAX_VALENCE = 32           # B200GSR_DECIMATE_MAX_VALENCE
DECIMATE_STATUS_WORDS = 6           # B200GSR_DECIMATE_STATUS_WORDS

_lib = None
ABI_VERSION = 3
ERR_BAD_ARG = -1
FWD_NO_BACKWARD = 1
FWD_DETERMINISTIC = 2
BWD_COMPOSITE, BWD_PROJECT = 1, 2
BWD_DETERMINISTIC = 4
SAVED_DETERMINISTIC = 0x100


def load():
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        # Not a fallback: the only thing ever attempted is compiling the same sm_90a sources in-tree.
        err = None
        if "B200GSR_LIB" not in os.environ and not os.environ.get("B200GSR_NO_AUTOBUILD"):
            try:
                from . import _build
                _build.build()
            except Exception as e:   # noqa: BLE001 - reported below
                err = e
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(
                f"{LIB_PATH} is missing and could not be built ({err}). Build it with "
                "`python -m dreamscene_b200._build` (needs nvcc; sm_90a only). There is no CPU fallback.")
    lib = C.CDLL(LIB_PATH)
    for name, (restype, argtypes) in {**SIGNATURES, **SCENE_SIGNATURES, **STEP_SIGNATURES, **LOSS_SIGNATURES,
                                      **FROZEN_SIGNATURES, **STATS_SIGNATURES, **RESERVE_SIGNATURES,
                                      **FRAMES_SIGNATURES, **VIEWS_FROZEN_SIGNATURES, **VIEWS_STATS_SIGNATURES,
                                      **FIELDS_SIGNATURES, **MESH_SIGNATURES, **MESH_COLOUR_SIGNATURES,
                                      **MESH_CLEAN_SIGNATURES, **MESH_DECIMATE_SIGNATURES}.items():
        fn = getattr(lib, name)
        fn.restype, fn.argtypes = restype, argtypes
    if lib.b200gsr_version() != ABI_VERSION:
        raise RuntimeError(f"{LIB_PATH} has ABI version {lib.b200gsr_version()}, this package needs "
                           f"{ABI_VERSION}: rebuild with `python -m dreamscene_b200._build --force`")
    _lib = lib
    return lib


def last_error() -> str:
    return load().b200gsr_last_error().decode("utf-8", "replace")


def check(rc: int, what: str, bad_arg=None) -> None:
    """Raise for a non-zero return code of the entry point `what`: RuntimeError("<what> failed (<rc>): <message>").
    With `bad_arg`, B200GSR_ERR_BAD_ARG raises bad_arg(<message>) instead (the rasterizer raises a bare Exception for
    misused inputs, as the reference's own checks do)."""
    if rc:
        msg = last_error()
        if rc == ERR_BAD_ARG and bad_arg is not None:
            raise bad_arg(msg)
        raise RuntimeError(f"{what} failed ({rc}): {msg}")


def ptr(t: Optional[torch.Tensor]) -> Optional[C.c_void_p]:
    return None if t is None else C.c_void_p(t.data_ptr())


def stream(dev) -> C.c_void_p:
    """The current stream of `dev`, as the `void* stream` every entry point takes."""
    return C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)


def prepare(t: Optional[torch.Tensor]) -> Optional[torch.Tensor]:
    """An input as the kernels read it: float32, contiguous, and 16-byte aligned (they use 16-byte vector loads on
    rows).  `t` itself when it already is.  It does not detach: autograd saves the prepared tensors."""
    if t is None:
        return None
    if t.dtype != torch.float32:
        t = t.float()
    t = t.contiguous()
    if t.data_ptr() % 16:
        t = t.clone()
    return t


def saved_layout(P: int, H: int, W: int, max_pairs: int, with_backward: bool = True,
                 deterministic: bool = False) -> SavedLayout:
    """deterministic: `total` also covers the fixed-point accumulators of deterministic mode (appended; every
    offset is the same as without)."""
    out = SavedLayout()
    flag = int(bool(with_backward)) | (SAVED_DETERMINISTIC if deterministic else 0)
    check(load().b200gsr_saved_layout_query(P, H, W, max_pairs, flag, C.byref(out)), "b200gsr_saved_layout_query")
    return out


def scratch_layout(P: int, H: int, W: int, max_pairs: int) -> ScratchLayout:
    out = ScratchLayout()
    check(load().b200gsr_scratch_layout_query(P, H, W, max_pairs, C.byref(out)), "b200gsr_scratch_layout_query")
    return out


def stacked_height(B: int, H: int, W: int) -> int:
    """Height of the image that B stacked views of H x W occupy (b200gsr_forward_views, b200gsr_score_views)."""
    hs = C.c_int32(0)
    check(load().b200gsr_views_geometry(B, H, W, C.byref(hs)), "b200gsr_views_geometry")
    return int(hs.value)


FWD_STAGES = ("project_sh", "scan_order", "scatter", "tile_sort", "composite_fwd")
BWD_STAGES = ("composite_bwd", "project_bwd")


def profile_enable(max_calls: int) -> None:
    check(load().b200gsr_profile_enable(int(max_calls)), "b200gsr_profile_enable")


def profile_collect() -> dict:
    """-> {stage: [ms per recorded call]} for every call recorded since profile_enable."""
    lib = load()
    nf, nb = C.c_int32(0), C.c_int32(0)
    lib.b200gsr_profile_counts(C.byref(nf), C.byref(nb))
    out = {k: [] for k in FWD_STAGES + BWD_STAGES}
    buf = (C.c_float * 8)()
    for i in range(nf.value):
        if lib.b200gsr_profile_read(0, i, buf):
            raise RuntimeError(last_error())
        for k, name in enumerate(FWD_STAGES):
            out[name].append(float(buf[k]))
    for i in range(nb.value):
        if lib.b200gsr_profile_read(1, i, buf):
            raise RuntimeError(last_error())
        for k, name in enumerate(BWD_STAGES):
            out[name].append(float(buf[k]))
    return out


STAT_NAMES = ("bwd_pairs_evaluated", "bwd_pairs_contributing", "bwd_lane_contributions", "bwd_k1", "bwd_k2",
              "bwd_k3_4", "bwd_k5_8", "bwd_k9_16", "bwd_k17_32", "_9", "fwd_pairs_evaluated", "fwd_lane_blends",
              "_12", "_13", "_14", "_15",
              "fwd_busy_ns", "fwd_end_ns", "fwd_not_begin_ns", "fwd_workers", "fwd_max_item_ns",
              "bwd_busy_ns", "bwd_end_ns", "bwd_not_begin_ns", "bwd_workers", "bwd_max_item_evals", "bwd_max_item_ns")
STAT_WORDS = 32


def debug_counters(ptr) -> None:
    """ptr: device pointer to STAT_WORDS (32) zeroed uint64 (or None to switch the instrumented kernels off)."""
    rc = load().b200gsr_debug_counters(C.c_void_p(ptr) if ptr else None)
    if rc:
        raise RuntimeError(last_error())
