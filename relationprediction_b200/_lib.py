"""ctypes binding of librgcn_b200.so (the C-ABI declared in include/rgcn_b200.h).

There is NO CPU fallback: if the library cannot be loaded the import of the compute path fails
loudly.  (The oracle under /oracle is test infrastructure and is never imported from here.)
"""
import ctypes
import os
from ctypes import POINTER, c_char_p, c_double, c_float, c_int, c_int32, c_int64, c_void_p

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "lib", "librgcn_b200.so")

# every symbol include/rgcn_b200.h declares (tests check the .so exports all of them)
EXPORTED_SYMBOLS = [
    "rgcn_version", "rgcn_last_error", "rgcn_launch_count", "rgcn_profile_enable", "rgcn_profile_read",
    "rgcn_set_option", "rgcn_gemm_tf32x3", "rgcn_gemm_tn_tf32x3", "rgcn_graph_destroy_async", "rgcn_sample_edge_neighborhood", "rgcn_sampler_create", "rgcn_sampler_draw", "rgcn_sampler_draw_batch", "rgcn_sampler_destroy", "rgcn_sumsq_accumulate", "rgcn_adam_update",
    "rgcn_graph_create", "rgcn_graph_create_messages", "rgcn_graph_create_device", "rgcn_graph_create_messages_device",
    "rgcn_graph_destroy", "rgcn_graph_info",
    "rgcn_graph_export_bytes", "rgcn_graph_export",
    "rgcn_block_workspace_bytes", "rgcn_block_forward", "rgcn_block_backward",
    "rgcn_block_aggregate_workspace_bytes", "rgcn_block_aggregate", "rgcn_block_aggregate_backward", "rgcn_rows_add", "rgcn_rows_gather", "rgcn_relu_backward",
    "rgcn_basis_workspace_bytes", "rgcn_basis_forward", "rgcn_basis_backward",
    "rgcn_basis_onehot_workspace_bytes", "rgcn_basis_onehot_forward", "rgcn_basis_onehot_backward",
    "rgcn_basis_diagcoef_workspace_bytes", "rgcn_basis_diagcoef_forward", "rgcn_basis_diagcoef_backward",
    "rgcn_diag_workspace_bytes", "rgcn_diag_forward", "rgcn_diag_backward",
    "rgcn_compgcn_workspace_bytes", "rgcn_compgcn_forward", "rgcn_compgcn_backward",
    "rgcn_highway_workspace_bytes", "rgcn_highway_forward", "rgcn_highway_backward",
    "rgcn_variational_workspace_bytes", "rgcn_variational_forward", "rgcn_variational_backward",
    "distmult_forward", "distmult_backward", "distmult_rank_workspace_bytes", "distmult_rank",
    "distmult_backward_slices", "rgcn_block_slice_sumsq_workspace_bytes", "rgcn_block_slice_sumsq",
    "rgcn_complex_forward", "rgcn_complex_backward", "rgcn_complex_rank_workspace_bytes", "rgcn_complex_rank",
    "rgcn_topk_workspace_bytes", "distmult_topk", "rgcn_complex_topk",
    "rgcn_relation_rank_workspace_bytes", "distmult_relation_rank", "rgcn_complex_relation_rank",
    "rgcn_relation_topk_workspace_bytes", "distmult_relation_topk", "rgcn_complex_relation_topk",
    "rgcn_ensemble_rank_workspace_bytes", "rgcn_ensemble_rank",
    "rgcn_ensemble_topk_workspace_bytes", "rgcn_ensemble_topk",
    "rgcn_ensemble_relation_rank_workspace_bytes", "rgcn_ensemble_relation_rank",
    "rgcn_ensemble_relation_topk_workspace_bytes", "rgcn_ensemble_relation_topk",
    "rgcn_one_to_n_workspace_bytes", "distmult_one_to_n", "rgcn_complex_one_to_n",
    "rgcn_one_to_n_labels_workspace_bytes", "rgcn_one_to_n_labels",
    "rgcn_one_to_n_finish_workspace_bytes", "rgcn_one_to_n_finish",
    "rgcn_self_adversarial_workspace_bytes", "rgcn_self_adversarial_forward",
    "rgcn_rotate_forward", "rgcn_rotate_backward", "rgcn_rotate_self_adversarial_forward",
    "rgcn_rotate_rank_workspace_bytes", "rgcn_rotate_rank",
    "rgcn_transe_forward", "rgcn_transe_backward", "rgcn_transe_self_adversarial_forward",
    "rgcn_transe_rank_workspace_bytes", "rgcn_transe_rank", "rgcn_transe_topk_workspace_bytes", "rgcn_transe_topk",
    "rgcn_transe_relation_rank_workspace_bytes", "rgcn_transe_relation_rank",
    "rgcn_transe_relation_topk_workspace_bytes", "rgcn_transe_relation_topk",
    "rgcn_quate_forward", "rgcn_quate_backward", "rgcn_quate_self_adversarial_forward", "rgcn_quate_rank",
    "rgcn_quate_topk", "rgcn_quate_relation_rank_workspace_bytes", "rgcn_quate_relation_rank",
    "rgcn_quate_relation_topk_workspace_bytes", "rgcn_quate_relation_topk", "rgcn_quate_one_to_n",
    "rgcn_quate_query_rows",
    "rgcn_hole_transform_workspace_bytes", "rgcn_hole_transform", "rgcn_hole_forward", "rgcn_hole_backward",
    "rgcn_hole_self_adversarial_forward", "rgcn_hole_rank", "rgcn_hole_topk", "rgcn_hole_relation_rank",
    "rgcn_hole_relation_topk", "rgcn_hole_one_to_n", "rgcn_hole_query_rows",
    "rgcn_conve_one_to_n_workspace_bytes", "rgcn_conve_one_to_n", "rgcn_conve_one_to_n_finish_workspace_bytes",
    "rgcn_conve_one_to_n_finish", "rgcn_conve_query_rows_workspace_bytes", "rgcn_conve_query_rows",
    "rgcn_conve_rank_workspace_bytes", "rgcn_conve_rank", "rgcn_conve_topk_workspace_bytes", "rgcn_conve_topk",
]

RGCN_DECODER_DISTMULT, RGCN_DECODER_COMPLEX = 0, 1

RGCN_NORM_CANONICAL, RGCN_NORM_EXPLICIT, RGCN_NORM_NONE, RGCN_NORM_RELATION = 0, 1, 2, 3

(X_DST_ROWPTR, X_DST_SRC, X_DST_RELW, X_DST_NORM, X_DST_MID, X_SRC_ROWPTR, X_SRC_DST, X_SRC_RELW,
 X_SRC_NORM, X_SRC_MID, X_REL_PTR, X_REL_DST, X_REL_SRC, X_REL_NORM, X_REL_MID, X_MSG_NORM,
 X_REL2_PTR, X_REL2_SRC, X_REL2_DST, X_REL2_NORM, X_REL2_MID) = range(21)

_lib = None


class RgcnError(RuntimeError):
    pass


class ConvENet(ctypes.Structure):
    """rgcn_conve_net_t: the ConvE query network's shape, weights (device pointers) and dropout masks."""
    _fields_ = [("h", c_int32), ("C", c_int32), ("rel_inv", c_void_p), ("filters", c_void_p),
                ("conv_bias", c_void_p), ("W_fc", c_void_p), ("b_fc", c_void_p), ("input_mask", c_void_p),
                ("feature_mask", c_void_p), ("hidden_mask", c_void_p), ("input_keep", c_float),
                ("feature_keep", c_float), ("hidden_keep", c_float)]


class ConvEGrads(ctypes.Structure):
    """rgcn_conve_grads_t: the gradients of the ConvE decoder's own weights (device pointers)."""
    _fields_ = [("rel_inv", c_void_p), ("filters", c_void_p), ("conv_bias", c_void_p), ("W_fc", c_void_p),
                ("b_fc", c_void_p)]


def _declare(lib):
    vp = c_void_p
    lib.rgcn_version.restype = c_int
    lib.rgcn_last_error.restype = c_char_p
    lib.rgcn_launch_count.restype = c_int64
    lib.rgcn_gemm_tf32x3.restype = c_int
    lib.rgcn_gemm_tf32x3.argtypes = [vp, c_int64, vp, c_int64, c_int, vp, c_int64, c_int32, c_int32, c_int32,
                                     c_int, vp, c_int64, vp]
    lib.rgcn_gemm_tn_tf32x3.restype = c_int
    lib.rgcn_gemm_tn_tf32x3.argtypes = [vp, c_int64, vp, c_int64, vp, c_int64, c_int32, c_int32, c_int32, c_int, vp]
    lib.rgcn_sample_edge_neighborhood.restype = c_int
    lib.rgcn_sample_edge_neighborhood.argtypes = [vp, c_int64, c_int32, c_int64, ctypes.c_uint64, vp]
    lib.rgcn_sampler_create.restype = c_int
    lib.rgcn_sampler_create.argtypes = [vp, c_int64, c_int32, ctypes.POINTER(vp)]
    lib.rgcn_sampler_draw.restype = c_int
    lib.rgcn_sampler_draw.argtypes = [vp, c_int64, ctypes.c_uint64, vp]
    lib.rgcn_sampler_draw_batch.restype = c_int
    lib.rgcn_sampler_draw_batch.argtypes = [vp, c_int32, c_int32, c_int32, ctypes.c_uint64, vp, vp, vp]
    lib.rgcn_sampler_destroy.restype = None
    lib.rgcn_sampler_destroy.argtypes = [vp]
    lib.rgcn_sumsq_accumulate.restype = c_int
    lib.rgcn_sumsq_accumulate.argtypes = [vp, c_int64, vp, vp]
    lib.rgcn_adam_update.restype = c_int
    lib.rgcn_adam_update.argtypes = [vp, vp, vp, vp, c_int64, c_float, c_float, c_float, c_float, c_int64, vp,
                                     c_float, vp]
    lib.rgcn_set_option.restype = c_int
    lib.rgcn_set_option.argtypes = [c_char_p, c_int64]
    lib.rgcn_profile_enable.restype = c_int
    lib.rgcn_profile_enable.argtypes = [c_int]
    lib.rgcn_profile_read.restype = c_int
    lib.rgcn_profile_read.argtypes = [vp, c_int, vp, c_int]
    lib.rgcn_graph_create.restype = c_int
    lib.rgcn_graph_create.argtypes = [vp, c_int64, c_int32, c_int32, c_int, vp, vp, c_int, vp,
                                      POINTER(vp)]
    lib.rgcn_graph_create_messages.restype = c_int
    lib.rgcn_graph_create_messages.argtypes = [vp, vp, vp, vp, c_int64, c_int32, c_int32, c_int32,
                                               c_int, vp, POINTER(vp)]
    lib.rgcn_graph_create_device.restype = c_int
    lib.rgcn_graph_create_device.argtypes = [vp, c_int64, c_int32, c_int32, c_int, vp, vp, c_int, vp, POINTER(vp)]
    lib.rgcn_graph_create_messages_device.restype = c_int
    lib.rgcn_graph_create_messages_device.argtypes = [vp, vp, vp, vp, c_int64, c_int32, c_int32, c_int32,
                                                      c_int, vp, POINTER(vp)]
    lib.rgcn_graph_destroy.restype = c_int
    lib.rgcn_graph_destroy.argtypes = [vp]
    lib.rgcn_graph_destroy_async.restype = c_int
    lib.rgcn_graph_destroy_async.argtypes = [vp, vp]
    lib.rgcn_graph_info.restype = c_int
    lib.rgcn_graph_info.argtypes = [vp, POINTER(c_int64)]
    lib.rgcn_graph_export_bytes.restype = c_int64
    lib.rgcn_graph_export_bytes.argtypes = [vp, c_int]
    lib.rgcn_graph_export.restype = c_int
    lib.rgcn_graph_export.argtypes = [vp, c_int, vp, c_int64]
    lib.rgcn_block_workspace_bytes.restype = c_int64
    lib.rgcn_block_workspace_bytes.argtypes = [vp, c_int32, c_int32, c_int]
    lib.rgcn_block_forward.restype = c_int
    lib.rgcn_block_forward.argtypes = [vp, c_int32, c_int32, vp, vp, vp, vp, vp, c_float, c_int, vp,
                                       vp, c_int64, vp]
    lib.rgcn_block_backward.restype = c_int
    lib.rgcn_block_backward.argtypes = [vp, c_int32, c_int32, vp, vp, vp, vp, vp, c_float, c_int, vp,
                                        vp, vp, vp, vp, vp, vp, c_int64, vp]
    lib.rgcn_block_aggregate_workspace_bytes.restype = c_int64
    lib.rgcn_block_aggregate_workspace_bytes.argtypes = [vp, c_int32, c_int32, c_int]
    lib.rgcn_block_aggregate.restype = c_int
    lib.rgcn_block_aggregate.argtypes = [vp, c_int32, c_int32, vp, vp, vp, vp, vp, c_int64, vp]
    lib.rgcn_block_aggregate_backward.restype = c_int
    lib.rgcn_block_aggregate_backward.argtypes = [vp, c_int32, c_int32, vp, vp, vp, vp, vp, vp, vp, c_int, vp,
                                                  c_int64, vp]
    lib.rgcn_rows_add.restype = c_int
    lib.rgcn_rows_add.argtypes = [vp, vp, vp, c_int64, c_int32, vp]
    lib.rgcn_relu_backward.restype = c_int
    lib.rgcn_relu_backward.argtypes = [vp, vp, vp, c_int64, vp]
    lib.rgcn_rows_gather.restype = c_int
    lib.rgcn_rows_gather.argtypes = [vp, vp, vp, c_int64, c_int32, c_int32, vp]
    lib.rgcn_basis_workspace_bytes.restype = c_int64
    lib.rgcn_basis_workspace_bytes.argtypes = [vp, c_int32, c_int32, c_int]
    lib.rgcn_basis_forward.restype = c_int
    lib.rgcn_basis_forward.argtypes = [vp, c_int32, c_int32, vp, vp, vp, vp, vp, vp, vp, c_float,
                                       c_int, vp, vp, vp, c_int64, vp]
    lib.rgcn_basis_backward.restype = c_int
    lib.rgcn_basis_backward.argtypes = [vp, c_int32, c_int32, vp, vp, vp, vp, vp, vp, vp, c_float,
                                        c_int, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, c_int64, vp]
    lib.rgcn_basis_onehot_workspace_bytes.restype = c_int64
    lib.rgcn_basis_onehot_workspace_bytes.argtypes = [vp, c_int32, c_int32, c_int]
    lib.rgcn_basis_onehot_forward.restype = c_int
    lib.rgcn_basis_onehot_forward.argtypes = [vp, c_int32, c_int32, vp, vp, vp, vp, vp, vp, c_float, c_int, vp, vp,
                                              c_int64, vp]
    lib.rgcn_basis_onehot_backward.restype = c_int
    lib.rgcn_basis_onehot_backward.argtypes = [vp, c_int32, c_int32, vp, vp, vp, vp, vp, c_float, c_int, vp, vp, vp,
                                               vp, vp, vp, vp, vp, c_int64, vp]
    lib.rgcn_basis_diagcoef_workspace_bytes.restype = c_int64
    lib.rgcn_basis_diagcoef_workspace_bytes.argtypes = [vp, c_int32, c_int32, c_int]
    lib.rgcn_basis_diagcoef_forward.restype = c_int
    lib.rgcn_basis_diagcoef_forward.argtypes = [vp, c_int32, c_int32, vp, vp, vp, vp, vp, vp, vp, vp, c_float, c_int,
                                                vp, vp, vp, c_int64, vp]
    lib.rgcn_basis_diagcoef_backward.restype = c_int
    lib.rgcn_basis_diagcoef_backward.argtypes = [vp, c_int32, c_int32, vp, vp, vp, vp, vp, vp, vp, c_float, c_int,
                                                 vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, c_int64, vp]
    lib.rgcn_diag_workspace_bytes.restype = c_int64
    lib.rgcn_diag_workspace_bytes.argtypes = [vp, c_int32, c_int]
    lib.rgcn_diag_forward.restype = c_int
    lib.rgcn_diag_forward.argtypes = [vp, c_int32, vp, vp, vp, vp, vp, vp, c_float, c_int, vp, vp, c_int64, vp]
    lib.rgcn_diag_backward.restype = c_int
    lib.rgcn_diag_backward.argtypes = [vp, c_int32, vp, vp, vp, vp, vp, c_float, c_int, vp, vp, vp, vp, vp, vp, vp,
                                       vp, vp, c_int64, vp]
    lib.rgcn_compgcn_workspace_bytes.restype = c_int64
    lib.rgcn_compgcn_workspace_bytes.argtypes = [vp, c_int32, c_int32, c_int]
    lib.rgcn_compgcn_forward.restype = c_int
    lib.rgcn_compgcn_forward.argtypes = [vp, c_int32, c_int32, c_int, vp, vp, vp, vp, vp, vp, vp, c_float, c_int, vp,
                                         vp, vp, vp, c_int64, vp]
    lib.rgcn_compgcn_backward.restype = c_int
    lib.rgcn_compgcn_backward.argtypes = [vp, c_int32, c_int32, c_int, vp, vp, vp, vp, vp, vp, c_float, c_int, vp,
                                          vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, c_int64, vp]
    lib.rgcn_highway_workspace_bytes.restype = c_int64
    lib.rgcn_highway_workspace_bytes.argtypes = [c_int64, c_int32, c_int]
    lib.rgcn_highway_forward.restype = c_int
    lib.rgcn_highway_forward.argtypes = [vp, vp, vp, vp, c_int64, c_int32, vp, vp, vp, c_int64, vp]
    lib.rgcn_highway_backward.restype = c_int
    lib.rgcn_highway_backward.argtypes = [vp, vp, vp, vp, vp, c_int64, c_int32, vp, vp, vp, vp, vp, c_int64, vp]
    lib.rgcn_variational_workspace_bytes.restype = c_int64
    lib.rgcn_variational_workspace_bytes.argtypes = [c_int64, c_int32, c_int32, c_int]
    lib.rgcn_variational_forward.restype = c_int
    lib.rgcn_variational_forward.argtypes = [vp, c_int64, c_int32, c_int32, vp, vp, vp, vp, vp, vp, vp, vp, vp,
                                             c_int64, vp]
    lib.rgcn_variational_backward.restype = c_int
    lib.rgcn_variational_backward.argtypes = [vp, c_int64, c_int32, c_int32, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp,
                                              vp, vp, c_int64, vp]
    lib.distmult_forward.restype = c_int
    lib.distmult_forward.argtypes = [vp, vp, c_int32, c_int32, c_int32, vp, c_int64, vp, vp, vp, vp]
    lib.distmult_backward_slices.restype = c_int
    lib.distmult_backward_slices.argtypes = [vp, vp, c_int32, c_int32, c_int32, vp, c_int64, vp, vp,
                                             c_float, c_float, vp, vp, vp, vp, vp, vp]
    lib.rgcn_block_slice_sumsq_workspace_bytes.restype = c_int64
    lib.rgcn_block_slice_sumsq_workspace_bytes.argtypes = [vp, c_int32, c_int32]
    lib.rgcn_block_slice_sumsq.restype = c_int
    lib.rgcn_block_slice_sumsq.argtypes = [vp, c_int32, c_int32, vp, vp, vp, vp, c_int64, vp]
    lib.distmult_rank_workspace_bytes.restype = c_int64
    lib.distmult_rank_workspace_bytes.argtypes = [c_int32, c_int32, c_int64]
    lib.distmult_rank.restype = c_int
    lib.distmult_rank.argtypes = [vp, vp, c_int32, c_int32, c_int32, vp, c_int64, c_int, vp, c_int, vp, vp, vp, c_int64, vp]
    lib.distmult_backward.restype = c_int
    lib.distmult_backward.argtypes = [vp, vp, c_int32, c_int32, c_int32, vp, c_int64, vp, vp,
                                      c_float, c_float, vp, vp, vp, vp, vp]
    lib.rgcn_complex_forward.restype = c_int
    lib.rgcn_complex_forward.argtypes = [vp, vp, c_int32, c_int32, c_int32, vp, c_int64, vp, vp, vp, vp]
    lib.rgcn_complex_backward.restype = c_int
    lib.rgcn_complex_backward.argtypes = [vp, vp, c_int32, c_int32, c_int32, vp, c_int64, vp, vp,
                                          c_float, c_float, vp, vp, vp, vp, vp, vp]
    lib.rgcn_complex_rank_workspace_bytes.restype = c_int64
    lib.rgcn_complex_rank_workspace_bytes.argtypes = [c_int32, c_int32, c_int64]
    lib.rgcn_complex_rank.restype = c_int
    lib.rgcn_complex_rank.argtypes = [vp, vp, c_int32, c_int32, c_int32, vp, c_int64, c_int, vp, c_int, vp, vp, vp,
                                      c_int64, vp]
    lib.rgcn_topk_workspace_bytes.restype = c_int64
    lib.rgcn_topk_workspace_bytes.argtypes = [c_int32, c_int32, c_int64, c_int32]
    for name in ("distmult_topk", "rgcn_complex_topk"):
        getattr(lib, name).restype = c_int
        getattr(lib, name).argtypes = [vp, vp, c_int32, c_int32, c_int32, vp, c_int64, c_int, c_int32, vp, c_int, vp,
                                       vp, vp, c_int64, vp]
    lib.rgcn_relation_rank_workspace_bytes.restype = c_int64
    lib.rgcn_relation_rank_workspace_bytes.argtypes = [c_int32, c_int32, c_int64]
    lib.rgcn_relation_topk_workspace_bytes.restype = c_int64
    lib.rgcn_relation_topk_workspace_bytes.argtypes = [c_int32, c_int32, c_int64, c_int32]
    for name in ("distmult_relation_rank", "rgcn_complex_relation_rank"):
        getattr(lib, name).restype = c_int
        getattr(lib, name).argtypes = [vp, vp, c_int32, c_int32, c_int32, c_int32, vp, c_int64, vp, c_int, vp, vp, vp,
                                       c_int64, vp]
    for name in ("distmult_relation_topk", "rgcn_complex_relation_topk"):
        getattr(lib, name).restype = c_int
        getattr(lib, name).argtypes = [vp, vp, c_int32, c_int32, c_int32, c_int32, vp, c_int64, c_int32, vp, c_int,
                                       vp, vp, vp, c_int64, vp]
    lib.rgcn_ensemble_rank_workspace_bytes.restype = c_int64
    lib.rgcn_ensemble_rank_workspace_bytes.argtypes = [c_int32, c_int32, c_int32, c_int64]
    lib.rgcn_ensemble_rank.restype = c_int
    lib.rgcn_ensemble_rank.argtypes = [c_int32, vp, vp, c_int32, c_int32, c_int32, vp, vp, c_int32, c_int32, c_int32,
                                       c_double, vp, c_int64, c_int, vp, c_int, vp, vp, vp, c_int64, vp]
    lib.rgcn_ensemble_topk_workspace_bytes.restype = c_int64
    lib.rgcn_ensemble_topk_workspace_bytes.argtypes = [c_int32, c_int32, c_int32, c_int64, c_int32]
    lib.rgcn_ensemble_topk.restype = c_int
    lib.rgcn_ensemble_topk.argtypes = [c_int32, vp, vp, c_int32, c_int32, c_int32, vp, vp, c_int32, c_int32, c_int32,
                                       c_double, vp, c_int64, c_int, c_int32, vp, c_int, vp, vp, vp, vp, c_int64, vp]
    lib.rgcn_ensemble_relation_rank_workspace_bytes.restype = c_int64
    lib.rgcn_ensemble_relation_rank_workspace_bytes.argtypes = [c_int32, c_int32, c_int32, c_int64]
    lib.rgcn_ensemble_relation_rank.restype = c_int
    lib.rgcn_ensemble_relation_rank.argtypes = [c_int32, vp, vp, c_int32, c_int32, c_int32, vp, vp, c_int32, c_int32,
                                                c_int32, c_int32, c_double, vp, c_int64, vp, c_int, vp, vp, vp,
                                                c_int64, vp]
    lib.rgcn_ensemble_relation_topk_workspace_bytes.restype = c_int64
    lib.rgcn_ensemble_relation_topk_workspace_bytes.argtypes = [c_int32, c_int32, c_int32, c_int64, c_int32]
    lib.rgcn_ensemble_relation_topk.restype = c_int
    lib.rgcn_ensemble_relation_topk.argtypes = [c_int32, vp, vp, c_int32, c_int32, c_int32, vp, vp, c_int32, c_int32,
                                                c_int32, c_int32, c_double, vp, c_int64, c_int32, vp, c_int, vp, vp,
                                                vp, vp, c_int64, vp]
    lib.rgcn_one_to_n_workspace_bytes.restype = c_int64
    lib.rgcn_one_to_n_workspace_bytes.argtypes = [c_int32, c_int32, c_int64, c_int64]
    for name in ("distmult_one_to_n", "rgcn_complex_one_to_n"):
        getattr(lib, name).restype = c_int
        getattr(lib, name).argtypes = [vp, vp, c_int32, c_int32, c_int32, c_int32, vp, c_int64, vp, c_float, vp, vp,
                                       vp, vp, c_int64, vp, c_int64, vp]
    lib.rgcn_one_to_n_finish_workspace_bytes.restype = c_int64
    lib.rgcn_one_to_n_finish_workspace_bytes.argtypes = [c_int64]
    lib.rgcn_one_to_n_finish.restype = c_int
    lib.rgcn_one_to_n_finish.argtypes = [vp, vp, c_int32, c_int32, c_int32, c_int32, vp, c_int64, vp, vp, vp, vp, vp,
                                         vp, c_int64, vp]
    lib.rgcn_one_to_n_labels_workspace_bytes.restype = c_int64
    lib.rgcn_one_to_n_labels_workspace_bytes.argtypes = [c_int64]
    lib.rgcn_one_to_n_labels.restype = c_int
    lib.rgcn_one_to_n_labels.argtypes = [vp, vp, vp, c_int64, c_int32, c_int32, vp, c_int64, vp, vp, c_int64, vp]
    lib.rgcn_self_adversarial_workspace_bytes.restype = c_int64
    lib.rgcn_self_adversarial_workspace_bytes.argtypes = [c_int64, c_int32]
    lib.rgcn_self_adversarial_forward.restype = c_int
    lib.rgcn_self_adversarial_forward.argtypes = [c_int32, vp, vp, c_int32, c_int32, c_int32, vp, c_int64, c_int32,
                                                  c_float, vp, vp, vp, vp, c_int64, vp]
    lib.rgcn_rotate_forward.restype = c_int
    lib.rgcn_rotate_forward.argtypes = [vp, vp, c_int32, c_int32, c_int32, vp, c_int64, vp, c_float, vp, vp, vp]
    lib.rgcn_rotate_backward.restype = c_int
    lib.rgcn_rotate_backward.argtypes = [vp, vp, c_int32, c_int32, c_int32, vp, c_int64, vp, c_float, vp, c_float,
                                         c_float, vp, vp, vp, vp, vp, vp]
    lib.rgcn_rotate_self_adversarial_forward.restype = c_int
    lib.rgcn_rotate_self_adversarial_forward.argtypes = [vp, vp, c_int32, c_int32, c_int32, vp, c_int64, c_int32,
                                                         c_float, c_float, vp, vp, vp, vp, c_int64, vp]
    lib.rgcn_rotate_rank_workspace_bytes.restype = c_int64
    lib.rgcn_rotate_rank_workspace_bytes.argtypes = [c_int32, c_int32, c_int64]
    lib.rgcn_rotate_rank.restype = c_int
    lib.rgcn_rotate_rank.argtypes = [vp, vp, c_int32, c_int32, c_int32, vp, c_int64, c_int, vp, vp, vp, vp, c_int64,
                                     vp]
    # TransE: the RotatE argument lists; top-k as distmult_topk without reuse_split, plus gamma
    for fn in ("forward", "backward", "self_adversarial_forward"):
        getattr(lib, "rgcn_transe_" + fn).restype = c_int
        getattr(lib, "rgcn_transe_" + fn).argtypes = getattr(lib, "rgcn_rotate_" + fn).argtypes
    lib.rgcn_transe_rank_workspace_bytes.restype = c_int64
    lib.rgcn_transe_rank_workspace_bytes.argtypes = [c_int32, c_int32, c_int64]
    lib.rgcn_transe_rank.restype = c_int
    lib.rgcn_transe_rank.argtypes = [vp, vp, c_int32, c_int32, c_int32, vp, c_int64, c_int, vp, vp, vp, vp, c_int64,
                                     vp]
    lib.rgcn_transe_topk_workspace_bytes.restype = c_int64
    lib.rgcn_transe_topk_workspace_bytes.argtypes = [c_int32, c_int32, c_int64, c_int32]
    lib.rgcn_transe_topk.restype = c_int
    lib.rgcn_transe_topk.argtypes = [vp, vp, c_int32, c_int32, c_int32, vp, c_int64, c_int, c_int32, vp, c_float, vp,
                                     vp, vp, c_int64, vp]
    lib.rgcn_transe_relation_rank_workspace_bytes.restype = c_int64
    lib.rgcn_transe_relation_rank_workspace_bytes.argtypes = [c_int32, c_int32, c_int64]
    lib.rgcn_transe_relation_rank.restype = c_int
    lib.rgcn_transe_relation_rank.argtypes = [vp, vp, c_int32, c_int32, c_int32, c_int32, vp, c_int64, vp, vp, vp, vp,
                                              c_int64, vp]
    lib.rgcn_transe_relation_topk_workspace_bytes.restype = c_int64
    lib.rgcn_transe_relation_topk_workspace_bytes.argtypes = [c_int32, c_int32, c_int64, c_int32]
    lib.rgcn_transe_relation_topk.restype = c_int
    lib.rgcn_transe_relation_topk.argtypes = [vp, vp, c_int32, c_int32, c_int32, c_int32, vp, c_int64, c_int32, vp,
                                              c_float, vp, vp, vp, c_int64, vp]
    # QuatE: the DistMult argument lists; self-adversarial as rgcn_self_adversarial_forward without the decoder kind
    lib.rgcn_quate_forward.restype = c_int
    lib.rgcn_quate_forward.argtypes = lib.distmult_forward.argtypes
    lib.rgcn_quate_backward.restype = c_int
    lib.rgcn_quate_backward.argtypes = lib.distmult_backward_slices.argtypes
    lib.rgcn_quate_self_adversarial_forward.restype = c_int
    lib.rgcn_quate_self_adversarial_forward.argtypes = lib.rgcn_self_adversarial_forward.argtypes[1:]
    for name, like in (("rgcn_quate_rank", "distmult_rank"), ("rgcn_quate_topk", "distmult_topk"),
                       ("rgcn_quate_relation_rank", "distmult_relation_rank"),
                       ("rgcn_quate_relation_topk", "distmult_relation_topk"),
                       ("rgcn_quate_one_to_n", "distmult_one_to_n"),
                       ("rgcn_quate_relation_rank_workspace_bytes", "rgcn_relation_rank_workspace_bytes"),
                       ("rgcn_quate_relation_topk_workspace_bytes", "rgcn_relation_topk_workspace_bytes")):
        getattr(lib, name).restype = getattr(lib, like).restype
        getattr(lib, name).argtypes = getattr(lib, like).argtypes
    lib.rgcn_quate_query_rows.restype = c_int
    lib.rgcn_quate_query_rows.argtypes = [vp, vp, c_int32, c_int32, c_int32, vp, c_int64, c_int, vp, vp]
    # HolE: the QuatE argument lists (on transformed tables), plus the basis transform
    for name in ("forward", "backward", "self_adversarial_forward", "rank", "topk", "one_to_n", "query_rows"):
        getattr(lib, "rgcn_hole_" + name).restype = getattr(lib, "rgcn_quate_" + name).restype
        getattr(lib, "rgcn_hole_" + name).argtypes = getattr(lib, "rgcn_quate_" + name).argtypes
    for name, like in (("rgcn_hole_relation_rank", "distmult_relation_rank"),
                       ("rgcn_hole_relation_topk", "distmult_relation_topk")):
        getattr(lib, name).restype = getattr(lib, like).restype
        getattr(lib, name).argtypes = getattr(lib, like).argtypes
    lib.rgcn_hole_transform_workspace_bytes.restype = c_int64
    lib.rgcn_hole_transform_workspace_bytes.argtypes = [c_int32]
    lib.rgcn_hole_transform.restype = c_int
    lib.rgcn_hole_transform.argtypes = [vp, c_int64, c_int32, c_int, vp, c_int, vp, vp, c_int64, vp]
    net, grads = POINTER(ConvENet), POINTER(ConvEGrads)
    lib.rgcn_conve_one_to_n_workspace_bytes.restype = c_int64
    lib.rgcn_conve_one_to_n_workspace_bytes.argtypes = [c_int32, c_int32, c_int32, c_int32, c_int32, c_int64, c_int64]
    lib.rgcn_conve_one_to_n.restype = c_int
    lib.rgcn_conve_one_to_n.argtypes = [vp, vp, c_int32, c_int32, c_int32, c_int32, net, vp, c_int64, vp, c_float, vp,
                                        vp, vp, vp, grads, c_int64, vp, c_int64, vp]
    lib.rgcn_conve_one_to_n_finish_workspace_bytes.restype = c_int64
    lib.rgcn_conve_one_to_n_finish_workspace_bytes.argtypes = [c_int64]
    lib.rgcn_conve_one_to_n_finish.restype = c_int
    lib.rgcn_conve_one_to_n_finish.argtypes = [vp, vp, c_int32, c_int32, c_int32, c_int32, net, vp, c_int64, vp, vp,
                                               vp, grads, vp, vp, grads, vp, c_int64, vp]
    lib.rgcn_conve_query_rows_workspace_bytes.restype = c_int64
    lib.rgcn_conve_query_rows_workspace_bytes.argtypes = [c_int32, c_int32, c_int32, c_int64]
    lib.rgcn_conve_query_rows.restype = c_int
    lib.rgcn_conve_query_rows.argtypes = [vp, vp, c_int32, c_int32, c_int32, c_int32, net, vp, c_int64, c_int, vp, vp,
                                          c_int64, vp]
    lib.rgcn_conve_rank_workspace_bytes.restype = c_int64
    lib.rgcn_conve_rank_workspace_bytes.argtypes = [c_int32, c_int32, c_int32, c_int32, c_int64]
    lib.rgcn_conve_rank.restype = c_int
    lib.rgcn_conve_rank.argtypes = [vp, vp, c_int32, c_int32, c_int32, c_int32, net, vp, c_int64, c_int, vp, c_int, vp,
                                    vp, vp, c_int64, vp]
    lib.rgcn_conve_topk_workspace_bytes.restype = c_int64
    lib.rgcn_conve_topk_workspace_bytes.argtypes = [c_int32, c_int32, c_int32, c_int32, c_int64, c_int32]
    lib.rgcn_conve_topk.restype = c_int
    lib.rgcn_conve_topk.argtypes = [vp, vp, c_int32, c_int32, c_int32, c_int32, net, vp, c_int64, c_int, c_int32, vp,
                                    c_int, vp, vp, vp, c_int64, vp]


def load():
    """Load (building first if the .so is absent) and return the ctypes library handle."""
    global _lib
    if _lib is not None:
        return _lib
    # always go through build(): it is a fingerprint comparison when the .so is current, and it rebuilds a
    # stale library after csrc / header edits instead of loading it against the new ctypes signatures
    from . import build as _build
    try:
        _build.build()
    except Exception as e:  # no nvcc on this host: a library whose stamp matches the sources is still fine
        if not (os.path.exists(LIB_PATH) and _build.is_current()):
            raise RgcnError("librgcn_b200.so is missing or stale and could not be rebuilt: %s" % e) from e
    try:
        lib = ctypes.CDLL(LIB_PATH)
    except OSError as e:  # loud failure: the CUDA library IS the product path
        raise RgcnError("cannot load %s: %s (run `python -m relationprediction_b200.build`)"
                        % (LIB_PATH, e)) from e
    _declare(lib)
    _lib = lib
    return lib


def check(rc, what=""):
    if rc != 0:
        msg = load().rgcn_last_error()
        raise RgcnError("%s failed (rc=%d): %s" % (what, rc, (msg or b"").decode("utf-8", "replace")))


def set_option(name, value):
    check(load().rgcn_set_option(name.encode(), int(value)), "rgcn_set_option")


def profile_enable(on=True):
    load().rgcn_profile_enable(1 if on else 0)


def profile_read():
    """[(stage name, ms)] recorded since the last read (see rgcn_profile_enable)."""
    ms = (c_float * 96)()
    names = ctypes.create_string_buffer(4096)
    n = load().rgcn_profile_read(ms, 96, names, 4096)
    nm = names.value.decode().split("\n")
    return [(nm[i], float(ms[i])) for i in range(n)]


def launch_count():
    return int(load().rgcn_launch_count())
