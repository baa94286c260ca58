"""ctypes binding of libnsb.so (C ABI declared in include/nsb.h).

The library is built in-tree (nersemble_b200/libnsb.so) by __graft_entry__.build() /
`make -C nersemble_b200/csrc`.  Loading fails loudly when it is missing.
"""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("NSB_LIB", os.path.join(_HERE, "libnsb.so"))   # NSB_LIB: kernel-variant A/B runs

MAX_LEVELS = 16
MEMBERS = 32


class Levels(C.Structure):
    _fields_ = [("n_levels", C.c_int32),
                ("scale", C.c_float * MAX_LEVELS),
                ("res", C.c_uint32 * MAX_LEVELS),
                ("entries", C.c_uint32 * MAX_LEVELS),
                ("offset", C.c_uint32 * MAX_LEVELS),
                ("hashed", C.c_uint32 * MAX_LEVELS)]


class FieldParams(C.Structure):
    _fields_ = [("tables", C.c_void_p), ("deform_bias", C.c_void_p),
                ("deform_packed_tb", C.c_void_p), ("deform_code_bias", C.c_void_p), ("deform_packed_umma", C.c_void_p), ("frame_table", C.c_void_p),
                ("frame_stride", C.c_int64), ("field_packed", C.c_void_p), ("warp_codes", C.c_void_p), ("blend_codes", C.c_void_p),
                ("n_timesteps", C.c_int32), ("aabb", C.c_float * 6), ("levels", Levels)]


class FieldOpts(C.Structure):
    _fields_ = [("cw_scale", C.c_float * MEMBERS), ("cw_bias", C.c_float * MEMBERS),
                ("pe_window", C.c_float * 8), ("use_deformation", C.c_int32), ("compute_rgb", C.c_int32)]


class Samples(C.Structure):
    _fields_ = [("n_samples", C.c_int64),
                ("origins", C.c_void_p), ("directions", C.c_void_p), ("ray_times", C.c_void_p),
                ("t_starts", C.c_void_p), ("t_ends", C.c_void_p), ("ray_indices", C.c_void_p),
                ("positions", C.c_void_p), ("sample_times", C.c_void_p), ("sample_directions", C.c_void_p),
                ("n_samples_dev", C.c_void_p), ("given_feat", C.c_void_p), ("sample_blend_codes", C.c_void_p),
                ("sample_code_bias", C.c_void_p)]


class FieldOut(C.Structure):
    _fields_ = [("sigma", C.c_void_p), ("rgb", C.c_void_p), ("offsets", C.c_void_p), ("feat", C.c_void_p),
                ("xs", C.c_void_p), ("deform_acts", C.c_void_p), ("deform_enc", C.c_void_p), ("corner_vals", C.c_void_p)]


class FieldBwdArgs(C.Structure):
    _fields_ = [("field_packed_t", C.c_void_p), ("feat", C.c_void_p), ("xs", C.c_void_p), ("sigma", C.c_void_p),
                ("rgb", C.c_void_p), ("d_sigma", C.c_void_p), ("d_rgb", C.c_void_p), ("loss_scale", C.c_float),
                ("d_feat", C.c_void_p), ("d_base_w", C.c_void_p), ("d_head_w", C.c_void_p), ("d_tables", C.c_void_p),
                ("d_blend_codes", C.c_void_p), ("d_xs", C.c_void_p), ("g_rank1", C.c_void_p), ("ts_slot", C.c_void_p),
                ("n_slots", C.c_int32), ("corner_vals", C.c_void_p), ("cw_slots_out", C.c_void_p),
                ("d_sample_blend_codes", C.c_void_p)]


class TableAdamArgs(C.Structure):
    _fields_ = [("total_entries", C.c_int64), ("tables", C.c_void_p), ("exp_avg", C.c_void_p), ("exp_avg_sq", C.c_void_p),
                ("tables_half", C.c_void_p), ("grad", C.c_void_p), ("g_rank1", C.c_void_p), ("cw_slots", C.c_void_p),
                ("n_slots", C.c_int32), ("grad_scale", C.c_float), ("lr", C.c_float), ("beta1", C.c_float),
                ("beta2", C.c_float), ("eps", C.c_float), ("weight_decay", C.c_float), ("bias_correction1", C.c_float),
                ("bias_correction2", C.c_float), ("step_size", C.c_float), ("bias_correction2_sqrt", C.c_float),
                ("one_minus_beta1", C.c_float), ("one_minus_beta2", C.c_float)]


class LossArgs(C.Structure):
    _fields_ = [("n_rays", C.c_int64), ("n_samples", C.c_int64), ("packed_info", C.c_void_p), ("t_starts", C.c_void_p),
                ("t_ends", C.c_void_p), ("weights", C.c_void_p), ("rgb", C.c_void_p), ("acc", C.c_void_p),
                ("depth", C.c_void_p), ("image", C.c_void_p), ("alpha", C.c_void_p), ("depth_target", C.c_void_p),
                ("use_masked_rgb", C.c_int32), ("alpha_mask_threshold", C.c_float), ("lambda_alpha", C.c_float),
                ("lambda_empty", C.c_float), ("lambda_near", C.c_float), ("lambda_depth", C.c_float),
                ("lambda_dist", C.c_float), ("eps_depth", C.c_float), ("dist_max_rays", C.c_int64),
                ("accum", C.c_void_p), ("values", C.c_void_p), ("coef", C.c_void_p), ("upstream", C.c_void_p),
                ("d_rgb", C.c_void_p), ("d_acc", C.c_void_p), ("d_depth", C.c_void_p), ("d_weights", C.c_void_p)]


class CompositeArgs(C.Structure):
    _fields_ = [("n_rays", C.c_int64), ("n_samples", C.c_int64), ("packed_info", C.c_void_p),
                ("t_starts", C.c_void_p), ("t_ends", C.c_void_p), ("sigma", C.c_void_p), ("rgb", C.c_void_p),
                ("offsets", C.c_void_p), ("training", C.c_int32),
                ("out_rgb", C.c_void_p), ("out_acc", C.c_void_p), ("out_depth", C.c_void_p),
                ("out_deform", C.c_void_p), ("out_weights", C.c_void_p), ("workspace", C.c_void_p)]


class DeformBwdArgs(C.Structure):
    _fields_ = [("deform_packed_t", C.c_void_p), ("deform_acts", C.c_void_p), ("deform_enc", C.c_void_p),
                ("d_xs", C.c_void_p), ("loss_scale", C.c_float), ("d_stem_w", C.c_void_p * 6), ("d_stem_b", C.c_void_p),
                ("d_r_w", C.c_void_p), ("d_r_b", C.c_void_p), ("d_v_w", C.c_void_p), ("d_v_b", C.c_void_p),
                ("d_warp_codes", C.c_void_p), ("dw_workspace", C.c_void_p), ("sample_warp_codes", C.c_void_p),
                ("d_sample_warp_codes", C.c_void_p)]


class CompositeBwdArgs(C.Structure):
    _fields_ = [("n_rays", C.c_int64), ("n_samples", C.c_int64), ("packed_info", C.c_void_p),
                ("t_starts", C.c_void_p), ("t_ends", C.c_void_p), ("sigma", C.c_void_p), ("rgb", C.c_void_p),
                ("d_out_rgb", C.c_void_p), ("d_out_acc", C.c_void_p), ("d_out_depth", C.c_void_p),
                ("d_weights", C.c_void_p), ("workspace", C.c_void_p), ("d_sigma", C.c_void_p), ("d_rgb", C.c_void_p)]


class MarchArgs(C.Structure):
    _fields_ = [("n_rays", C.c_int64), ("origins", C.c_void_p), ("directions", C.c_void_p),
                ("near_planes", C.c_void_p), ("far_planes", C.c_void_p), ("binaries", C.c_void_p),
                ("aabbs", C.c_void_p), ("levels", C.c_int32), ("res", C.c_int32),
                ("step", C.c_float), ("cone_angle", C.c_float), ("counts", C.c_void_p),
                ("offsets", C.c_void_p), ("t_starts", C.c_void_p), ("t_ends", C.c_void_p),
                ("ray_indices", C.c_void_p)]


class RenderArgs(C.Structure):
    _fields_ = [("n_rays", C.c_int64), ("origins", C.c_void_p), ("directions", C.c_void_p), ("ray_times", C.c_void_p),
                ("sampler", C.c_int32), ("n_per_ray", C.c_int32), ("near_plane", C.c_float),
                ("near_planes", C.c_void_p), ("far_planes", C.c_void_p), ("binaries", C.c_void_p), ("aabbs", C.c_void_p),
                ("levels", C.c_int32), ("res", C.c_int32), ("step", C.c_float), ("cone_angle", C.c_float),
                ("training", C.c_int32), ("capacity", C.c_int64), ("t_starts", C.c_void_p), ("t_ends", C.c_void_p),
                ("ray_indices", C.c_void_p), ("sigma", C.c_void_p), ("rgb", C.c_void_p), ("offsets", C.c_void_p),
                ("weights", C.c_void_p), ("packed_info", C.c_void_p), ("out_rgb", C.c_void_p), ("out_acc", C.c_void_p),
                ("out_depth", C.c_void_p), ("out_deform", C.c_void_p), ("workspace", C.c_void_p),
                ("march_scratch", C.c_void_p)]


class VisCompactArgs(C.Structure):
    _fields_ = [("n_rays", C.c_int64), ("capacity", C.c_int64), ("packed_info", C.c_void_p), ("t_starts", C.c_void_p),
                ("t_ends", C.c_void_p), ("sigma", C.c_void_p), ("ray_indices", C.c_void_p), ("early_stop_eps", C.c_float),
                ("alpha_thre", C.c_float), ("alpha_thre_cap", C.c_void_p), ("out_packed_info", C.c_void_p),
                ("out_t_starts", C.c_void_p), ("out_t_ends", C.c_void_p), ("out_ray_indices", C.c_void_p),
                ("feat", C.c_void_p), ("out_feat", C.c_void_p), ("xs", C.c_void_p), ("out_xs", C.c_void_p),
                ("corner_vals", C.c_void_p), ("out_corner_vals", C.c_void_p), ("workspace", C.c_void_p)]


class RayBatchArgs(C.Structure):
    _fields_ = [("n_rays", C.c_int64), ("indices", C.c_void_p), ("height", C.c_int64), ("width", C.c_int64),
                ("image_camera", C.c_void_p), ("image_times", C.c_void_p), ("intrinsics", C.c_void_p),
                ("camera_to_world", C.c_void_p), ("images", C.c_void_p), ("alpha_maps", C.c_void_p),
                ("depth_maps", C.c_void_p), ("origins", C.c_void_p), ("directions", C.c_void_p), ("pixel_area", C.c_void_p),
                ("directions_norm", C.c_void_p), ("times", C.c_void_p), ("camera_indices", C.c_void_p),
                ("out_image", C.c_void_p), ("out_alpha", C.c_void_p), ("out_depth", C.c_void_p)]


class NormalsArgs(C.Structure):     # nsb_normals_args
    _fields_ = [("offsets", C.c_void_p), ("grad_scale", C.c_float * 3), ("packed_info", C.c_void_p), ("n_rays", C.c_int64),
                ("weights", C.c_void_p), ("normals", C.c_void_p), ("out_normals", C.c_void_p),
                ("observation_space", C.c_int32), ("loss_scale", C.c_float), ("deform_packed_t", C.c_void_p),
                ("deform_packed_pe_t", C.c_void_p), ("vjp_scratch", C.c_void_p)]


class DeformVjpArgs(C.Structure):   # nsb_deform_vjp_args
    _fields_ = [("deform_packed_t", C.c_void_p), ("deform_packed_pe_t", C.c_void_p), ("u", C.c_void_p),
                ("loss_scale", C.c_float), ("d_pn", C.c_void_p)]


class DeformJacArgs(C.Structure):   # nsb_deform_jac_args
    _fields_ = [("tangent_scale", C.c_float), ("offsets", C.c_void_p), ("jacobian", C.c_void_p)]


class DeformInvArgs(C.Structure):   # nsb_deform_inv_args
    _fields_ = [("tangent_scale", C.c_float), ("init", C.c_void_p), ("max_iter", C.c_int32), ("tol", C.c_float),
                ("positions", C.c_void_p), ("residual", C.c_void_p), ("iterations", C.c_void_p), ("status", C.c_void_p)]


INV_CONVERGED, INV_NOT_CONVERGED, INV_SINGULAR = 0, 1, 2     # NSB_INV_*


class MeshArgs(C.Structure):       # nsb_mesh_args
    _fields_ = [("sigma", C.c_void_p), ("nx", C.c_int64), ("ny", C.c_int64), ("nz", C.c_int64), ("level", C.c_float),
                ("box_min", C.c_float * 3), ("h", C.c_float * 3), ("point_mask", C.c_void_p), ("vertex_base", C.c_void_p),
                ("tile_sums", C.c_void_p), ("n_vertices", C.c_int64), ("n_faces", C.c_int64), ("vertices", C.c_void_p),
                ("faces", C.c_void_p)]


MESH_TILE = 1024        # NSB_MESH_TILE


class FlowSelectArgs(C.Structure):  # nsb_flow_select_args
    _fields_ = [("n_rays", C.c_int64), ("capacity", C.c_int64), ("packed_info", C.c_void_p), ("t_starts", C.c_void_p),
                ("t_ends", C.c_void_p), ("weights", C.c_void_p), ("offsets", C.c_void_p), ("origins", C.c_void_p),
                ("directions", C.c_void_p), ("n_total", C.c_void_p), ("min_weight", C.c_float), ("ray_sel", C.c_void_p),
                ("sel_index", C.c_void_p), ("targets", C.c_void_p), ("init", C.c_void_p), ("n_selected", C.c_void_p),
                ("tile_sums", C.c_void_p)]


class FlowCompositeArgs(C.Structure):  # nsb_flow_composite_args
    _fields_ = [("n_rays", C.c_int64), ("capacity", C.c_int64), ("ray_sel", C.c_void_p), ("sel_index", C.c_void_p),
                ("init", C.c_void_p), ("positions", C.c_void_p), ("status", C.c_void_p), ("weights", C.c_void_p),
                ("intrinsics", C.c_float * 4), ("camera_to_world", C.c_float * 12), ("scene_flow", C.c_void_p),
                ("flow_weight", C.c_void_p), ("optical_flow", C.c_void_p)]


FLOW_TILE = 64          # NSB_FLOW_TILE


class RenderWsHeader(C.Structure):
    _fields_ = [("barrier", C.c_uint32), ("depth_range", C.c_uint32 * 2), ("status", C.c_int32), ("n_total", C.c_int64),
                ("reserved", C.c_int64 * 5)]


# every symbol include/nsb.h declares: (name, restype, argtypes)
SYMBOLS = {
    "nsb_version": (C.c_int, []),
    "nsb_last_error": (C.c_char_p, []),
    "nsb_deform_packed_bytes": (C.c_size_t, []),
    "nsb_field_packed_bytes": (C.c_size_t, []),
    "nsb_deform_packed_umma_bytes": (C.c_size_t, []),
    "nsb_blend_tables": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int64, C.c_void_p, C.c_void_p]),
    "nsb_field_forward": (C.c_int, [C.POINTER(FieldParams), C.POINTER(FieldOpts), C.POINTER(Samples),
                                    C.POINTER(FieldOut), C.c_void_p]),
    "nsb_field_backward": (C.c_int, [C.POINTER(FieldParams), C.POINTER(FieldOpts), C.POINTER(Samples),
                                     C.POINTER(FieldBwdArgs), C.c_void_p]),
    "nsb_deform_packed_t_bytes": (C.c_size_t, []),
    "nsb_deform_bwd_workspace_bytes": (C.c_size_t, []),
    "nsb_deform_backward": (C.c_int, [C.POINTER(FieldParams), C.POINTER(FieldOpts), C.POINTER(Samples),
                                      C.POINTER(DeformBwdArgs), C.c_void_p]),
    "nsb_deform_input_grad": (C.c_int, [C.POINTER(FieldParams), C.POINTER(FieldOpts), C.POINTER(Samples),
                                        C.POINTER(DeformVjpArgs), C.c_void_p]),
    "nsb_deform_jacobian": (C.c_int, [C.POINTER(FieldParams), C.POINTER(FieldOpts), C.POINTER(Samples),
                                      C.POINTER(DeformJacArgs), C.c_void_p]),
    "nsb_deform_inverse": (C.c_int, [C.POINTER(FieldParams), C.POINTER(FieldOpts), C.POINTER(Samples),
                                     C.POINTER(DeformInvArgs), C.c_void_p]),
    "nsb_losses_forward": (C.c_int, [C.POINTER(LossArgs), C.c_void_p]),
    "nsb_losses_backward": (C.c_int, [C.POINTER(LossArgs), C.c_void_p]),
    "nsb_table_adam_step": (C.c_int, [C.POINTER(TableAdamArgs), C.c_void_p]),
    "nsb_rank1_expand": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_int64, C.c_float, C.c_void_p, C.c_void_p]),
    "nsb_hash_blend_forward": (C.c_int, [C.POINTER(FieldParams), C.POINTER(FieldOpts), C.c_void_p, C.c_void_p,
                                         C.c_int64, C.c_void_p, C.c_int32, C.c_void_p]),
    "nsb_hash_blend_backward": (C.c_int, [C.POINTER(FieldParams), C.POINTER(FieldOpts), C.c_void_p, C.c_void_p,
                                          C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "nsb_composite_forward": (C.c_int, [C.POINTER(CompositeArgs), C.c_void_p]),
    "nsb_composite_backward": (C.c_int, [C.POINTER(CompositeBwdArgs), C.c_void_p]),
    "nsb_march_fixed": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_int32, C.c_float, C.c_float,
                                  C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "nsb_march_occupancy": (C.c_int, [C.POINTER(MarchArgs), C.c_void_p]),
    "nsb_visibility_mask": (C.c_int, [C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_float,
                                      C.c_float, C.c_void_p, C.c_void_p, C.c_void_p]),
    "nsb_occ_update": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_int64, C.c_float,
                                 C.c_float, C.c_void_p, C.c_void_p]),
    "nsb_occ_update_scratch_bytes": (C.c_size_t, [C.c_int64]),
    "nsb_render_workspace_bytes": (C.c_size_t, [C.c_int64]),
    "nsb_ray_batch": (C.c_int, [C.POINTER(RayBatchArgs), C.c_void_p]),
    "nsb_march_occupancy_packed": (C.c_int, [C.POINTER(MarchArgs), C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "nsb_visibility_compact": (C.c_int, [C.POINTER(VisCompactArgs), C.c_void_p]),
    "nsb_vis_compact_workspace_bytes": (C.c_size_t, [C.c_int64, C.c_int64]),
    "nsb_render_forward": (C.c_int, [C.POINTER(FieldParams), C.POINTER(FieldOpts), C.POINTER(RenderArgs), C.c_void_p]),
    "nsb_render_forward_interp": (C.c_int, [C.POINTER(FieldParams), C.POINTER(FieldOpts), C.POINTER(RenderArgs), C.c_void_p]),
    "nsb_normals_forward": (C.c_int, [C.POINTER(FieldParams), C.POINTER(FieldOpts), C.POINTER(Samples),
                                      C.POINTER(NormalsArgs), C.c_void_p]),
    "nsb_mesh_count": (C.c_int, [C.POINTER(MeshArgs), C.c_void_p]),
    "nsb_mesh_emit": (C.c_int, [C.POINTER(MeshArgs), C.c_void_p]),
    "nsb_flow_select": (C.c_int, [C.POINTER(FlowSelectArgs), C.c_void_p]),
    "nsb_flow_composite": (C.c_int, [C.POINTER(FlowCompositeArgs), C.c_void_p]),
}

_lib = None


def load() -> C.CDLL:
    """Load libnsb.so (once) and bind every declared symbol.  Raises if anything is missing."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(
            f"{LIB_PATH} not found: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            "or `make -C nersemble_b200/csrc`.  nersemble_b200 has no CPU fallback.")
    lib = C.CDLL(LIB_PATH)
    for name, (res, args) in SYMBOLS.items():
        fn = getattr(lib, name)          # AttributeError if the symbol is not exported
        fn.restype = res
        fn.argtypes = args
    if lib.nsb_version() != 200:
        raise RuntimeError(f"libnsb version mismatch: {lib.nsb_version()}")
    _lib = lib
    return lib


def check(rc: int, what: str) -> None:
    if rc != 0:
        msg = load().nsb_last_error().decode(errors="replace")
        raise RuntimeError(f"{what} failed (rc={rc}): {msg}")
