"""ctypes binding of libb200rec.so (the C ABI declared in include/b200rec.h).

There is deliberately NO fallback: if the shared library is missing or an entry point fails, the caller
gets an exception -- never a silent PyTorch/CPU path.
"""
from __future__ import annotations

import ctypes as C
import os

_PKG = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_PKG, "libb200rec.so")

c_i64p = C.c_void_p      # device pointers travel as integers
c_f32p = C.c_void_p


class GradSource(C.Structure):
    """b2r_grad_source (include/b200rec.h)"""
    _fields_ = [("src", C.c_void_p), ("coef", C.c_void_p), ("src_id", C.c_void_p),
                ("n", C.c_int64), ("div", C.c_int32), ("ld", C.c_int32)]


class Optim(C.Structure):
    """b2r_optim (include/b200rec.h)"""
    _fields_ = [("kind", C.c_int32), ("lr", C.c_float), ("beta1", C.c_float), ("beta2", C.c_float),
                ("eps", C.c_float), ("weight_decay", C.c_float), ("bc1", C.c_float), ("bc2", C.c_float),
                ("state_ld", C.c_int32), ("clock", C.c_void_p)]


class BprmfTables(C.Structure):
    """b2r_bprmf_tables (include/b200rec.h)"""
    _fields_ = [("U", C.c_void_p), ("I", C.c_void_p), ("Um", C.c_void_p), ("Uv", C.c_void_p),
                ("Im", C.c_void_p), ("Iv", C.c_void_p), ("n_users", C.c_int64), ("n_items", C.c_int64),
                ("d", C.c_int32), ("_pad", C.c_int32)]


class Dropout(C.Structure):
    """b2r_dropout (include/b200rec.h)"""
    _fields_ = [("state", C.c_void_p), ("lengths", C.c_void_p), ("p", C.c_double), ("site", C.c_int32),
                ("L", C.c_int32)]


NEUMF_MAX_LAYERS = 4                        # B2R_NEUMF_MAX_LAYERS


class NeumfRows(C.Structure):
    """b2r_neumf_rows (include/b200rec.h)"""
    _fields_ = [("mf_u", C.c_void_p), ("mf_i", C.c_void_p), ("mlp_u", C.c_void_p), ("mlp_i", C.c_void_p),
                ("n_users", C.c_int64), ("n_items", C.c_int64), ("d", C.c_int32), ("n_layers", C.c_int32),
                ("widths", C.c_int32 * NEUMF_MAX_LAYERS), ("W", C.c_void_p * NEUMF_MAX_LAYERS),
                ("bias", C.c_void_p * NEUMF_MAX_LAYERS), ("w_out", C.c_void_p), ("users", C.c_void_p),
                ("targets", C.c_void_p), ("Bn", C.c_int32), ("b0", C.c_int32), ("b1", C.c_int32), ("_pad", C.c_int32),
                ("out", C.c_void_p), ("ld_out", C.c_int64)]


IMPRESSION_MAX_TOPK = 16                    # B2R_IMPRESSION_MAX_TOPK

OPT_SGD, OPT_ADAM, OPT_ADAGRAD = 0, 1, 2
SEQ_LAST_QUERY = 1                          # b2r_seq_train_check flag
PROF_SCORE_FWD, PROF_SCORE_BWDQ, PROF_SEGMENT_I, PROF_SEGMENT_U, PROF_PLAN_I, PROF_LOSS = range(6)

# name -> (restype, argtypes); must list every symbol include/b200rec.h declares (tests/test_abi.py checks)
SIGNATURES = {
    "b2r_version": (C.c_int, []),
    "b2r_last_error": (C.c_char_p, []),
    "b2r_launch_count": (C.c_longlong, []),
    "b2r_profile_arm": (C.c_int, [C.c_int, C.c_void_p, C.c_void_p]),
    "b2r_rowdot_fwd": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_int64,
                                 C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p]),
    "b2r_rowdot_bwd_query": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p,
                                       C.c_int, C.c_int, C.c_int, C.c_void_p]),
    "b2r_gather_rows": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_int,
                                  C.c_void_p, C.c_void_p]),
    "b2r_pairdot_fwd": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p,
                                  C.c_int64, C.c_int, C.c_void_p, C.c_void_p]),
    "b2r_pair_runs_sum": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_int64,
                                    C.c_int64, C.c_int, C.c_void_p]),
    "b2r_bpr_loss": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p]),
    "b2r_plan_workspace_bytes": (C.c_size_t, [C.c_int64, C.c_int64]),
    "b2r_plan_build_ex": (C.c_int, [C.c_void_p, C.c_int64, C.c_int64, C.c_int64, C.c_int64, C.c_void_p, C.c_void_p,
                                    C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p]),
    "b2r_gather_rows_strided": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_int, C.c_int64,
                                          C.c_int, C.c_int, C.c_void_p, C.c_void_p]),
    "b2r_segment_apply": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_int64, C.c_int,
                                    C.POINTER(GradSource), C.POINTER(GradSource), C.c_int, C.c_void_p,
                                    C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                    C.POINTER(Optim), C.c_void_p]),
    "b2r_direct_plan_workspace_bytes": (C.c_size_t, [C.c_int64, C.c_int64]),
    "b2r_direct_plan_init": (C.c_int, [C.c_void_p, C.c_size_t, C.c_int64, C.c_int64, C.c_void_p]),
    "b2r_direct_plan_build": (C.c_int, [C.c_void_p, C.c_int64, C.c_int64, C.c_int64, C.c_int64, C.c_void_p, C.c_size_t,
                                        C.c_void_p, C.c_void_p]),
    "b2r_direct_plan_apply": (C.c_int, [C.c_void_p, C.c_int64, C.c_int64, C.c_int, C.POINTER(GradSource),
                                        C.POINTER(GradSource), C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                        C.POINTER(Optim), C.c_void_p]),
    "b2r_optim_tick": (C.c_int, [C.c_void_p, C.c_float, C.c_double, C.c_double, C.c_void_p]),
    "b2r_dense_optim": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64,
                                  C.POINTER(Optim), C.c_void_p]),
    "b2r_linear_fwd": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int64,
                                 C.c_int, C.c_int, C.c_int, C.c_void_p]),
    "b2r_linear_fwd_tc": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int64,
                                    C.c_int, C.c_int, C.c_int, C.c_void_p]),
    "b2r_linear_fwd_uses_tc": (C.c_int, [C.c_int64, C.c_int, C.c_int]),
    "b2r_linear_tc": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int64,
                                C.c_int, C.c_int, C.c_int, C.c_void_p]),
    "b2r_linear_bwd_input": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int,
                                       C.c_int64, C.c_int, C.c_int, C.c_void_p]),
    "b2r_linear_bwd_weight_workspace_bytes": (C.c_size_t, [C.c_int64, C.c_int, C.c_int]),
    "b2r_linear_bwd_weight": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p,
                                        C.c_void_p, C.c_int64, C.c_int, C.c_int, C.c_void_p, C.c_size_t,
                                        C.c_void_p]),
    "b2r_linear_bwd_weight_tc_workspace_bytes": (C.c_size_t, [C.c_int64, C.c_int, C.c_int]),
    "b2r_linear_bwd_weight_tc": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p,
                                           C.c_void_p, C.c_int64, C.c_int, C.c_int, C.c_void_p, C.c_size_t,
                                           C.c_void_p]),
    "b2r_add_layernorm_fwd": (C.c_int, [C.c_void_p] * 7 + [C.c_int64, C.c_int, C.c_float, C.c_void_p]),
    "b2r_add_layernorm_bwd_workspace_bytes": (C.c_size_t, [C.c_int64, C.c_int]),
    "b2r_add_layernorm_bwd": (C.c_int, [C.c_void_p] * 9 + [C.c_int64, C.c_int, C.c_void_p, C.c_size_t, C.c_void_p]),
    "b2r_dropout_tick": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p]),
    "b2r_linear_fwd_dropout": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int64,
                                         C.c_int, C.c_int, C.c_int, C.POINTER(Dropout), C.c_void_p]),
    "b2r_linear_fwd_tc_dropout": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int64,
                                            C.c_int, C.c_int, C.c_int, C.POINTER(Dropout), C.c_void_p]),
    "b2r_linear_bwd_weight_dropout": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p,
                                                C.c_void_p, C.c_int64, C.c_int, C.c_int, C.POINTER(Dropout), C.c_void_p,
                                                C.c_size_t, C.c_void_p]),
    "b2r_linear_bwd_weight_tc_dropout": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p,
                                                   C.c_void_p, C.c_int64, C.c_int, C.c_int, C.POINTER(Dropout), C.c_void_p,
                                                   C.c_size_t, C.c_void_p]),
    "b2r_add_layernorm_fwd_dropout": (C.c_int, [C.c_void_p] * 7 + [C.c_int64, C.c_int, C.c_float, C.POINTER(Dropout),
                                                                   C.c_void_p]),
    "b2r_add_layernorm_bwd_dropout": (C.c_int, [C.c_void_p] * 10 + [C.c_int64, C.c_int, C.POINTER(Dropout), C.c_void_p,
                                                                    C.c_size_t, C.c_void_p]),
    "b2r_embed_history": (C.c_int, [C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p,
                                    C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p]),
    "b2r_attention_fwd_live": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_int,
                                         C.c_int, C.c_int, C.c_void_p]),
    "b2r_attention_bwd_live": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p,
                                         C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int,
                                         C.c_void_p]),
    "b2r_attention_fwd_rt": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p,
                                       C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p]),
    "b2r_attention_bwd_rt": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int] + [C.c_void_p] * 7 +
                             [C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p]),
    "b2r_select_last": (C.c_int, [C.c_void_p] * 4 + [C.c_int, C.c_int, C.c_int, C.c_void_p]),
    "b2r_select_last_bwd": (C.c_int, [C.c_void_p] * 4 + [C.c_int, C.c_int, C.c_int, C.c_void_p]),
    "b2r_small_table_grad_workspace_bytes": (C.c_size_t, [C.c_int64, C.c_int, C.c_int]),
    "b2r_small_table_grad": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_int64, C.c_int, C.c_int, C.c_void_p,
                                       C.c_void_p, C.c_size_t, C.c_void_p]),
    "b2r_seq_train_check": (C.c_int, [C.c_int, C.c_int, C.c_int, C.c_int, C.c_int]),
    "b2r_colscale": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_int, C.c_void_p]),
    "b2r_gt_rank": (C.c_int, [C.c_void_p, C.c_int64, C.c_int64, C.c_int64, C.c_void_p, C.c_void_p]),
    "b2r_rank_histogram": (C.c_int, [C.c_void_p, C.c_int64, C.c_int, C.c_void_p, C.c_void_p]),
    "b2r_rank_all_items": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_int64, C.c_int,
                                     C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "b2r_rank_all_items_clicked": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_int64, C.c_int, C.c_void_p,
                                             C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p,
                                             C.c_void_p, C.c_void_p, C.c_void_p]),
    "b2r_topk_rows_workspace_bytes": (C.c_size_t, [C.c_int64, C.c_int64, C.c_int]),
    "b2r_topk_rows": (C.c_int, [C.c_void_p, C.c_int64, C.c_int64, C.c_int64, C.c_int, C.c_void_p, C.c_void_p,
                                C.c_void_p, C.c_size_t, C.c_void_p]),
    "b2r_mask_clicked": (C.c_int, [C.c_void_p, C.c_int64, C.c_int64, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p,
                                   C.c_int64, C.c_void_p, C.c_void_p]),
    "b2r_topk_all_items_workspace_bytes": (C.c_size_t, [C.c_int, C.c_int64, C.c_int]),
    "b2r_topk_all_items": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_int64, C.c_int, C.c_void_p, C.c_void_p,
                                     C.c_int, C.c_void_p, C.c_void_p, C.c_int64, C.c_int, C.c_void_p, C.c_void_p,
                                     C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]),
    "b2r_collate_impression": (C.c_int, [C.c_void_p] * 5 + [C.c_int64, C.c_int64, C.c_int, C.c_int, C.c_int,
                                                            C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "b2r_collate_impression_train": (C.c_int, [C.c_void_p] * 8 + [C.c_int64, C.c_int64, C.c_int, C.c_int, C.c_int,
                                                                  C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                                                  C.c_void_p]),
    "b2r_impression_metrics_workspace_bytes": (C.c_size_t, [C.c_int, C.c_int, C.c_int]),
    "b2r_impression_metrics": (C.c_int, [C.c_void_p, C.c_int64, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p,
                                         C.POINTER(C.c_int), C.c_int, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]),
    "b2r_neumf_score_rows_check": (C.c_int, [C.c_int, C.c_int, C.c_void_p, C.c_int64, C.c_int64]),
    "b2r_neumf_window_rows": (C.c_int, [C.c_int64, C.c_int64]),
    "b2r_neumf_score_rows": (C.c_int, [C.POINTER(NeumfRows), C.c_void_p, C.c_void_p]),
    "b2r_adam_exact_advance": (C.c_int, [C.c_void_p, C.c_int64, C.c_int64, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p,
                                         C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]),
    "b2r_sample_negatives": (C.c_int, [C.c_void_p, C.c_int64, C.c_int, C.c_void_p, C.c_void_p, C.c_int64, C.c_int64,
                                       C.c_uint64, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p]),
    "b2r_collate_general": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_int, C.c_int,
                                      C.c_void_p, C.c_void_p, C.c_void_p]),
    "b2r_collate_history": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_int64,
                                      C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "b2r_attention_last_fwd": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p,
                                         C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p]),
    "b2r_attention_last_bwd": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p,
                                         C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int,
                                         C.c_void_p]),
    "b2r_pairdot_fwd_p2p": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p,
                                      C.c_int64, C.c_int64, C.c_int, C.c_void_p, C.c_void_p]),
    "b2r_listwise_workspace_bytes": (C.c_size_t, [C.c_int]),
    "b2r_listwise_loss": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p,
                                    C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]),
    "b2r_route_workspace_bytes": (C.c_size_t, [C.c_int, C.c_int]),
    "b2r_route_ids": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int64, C.c_int64, C.c_void_p, C.c_void_p,
                                C.c_int64, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t,
                                C.c_void_p, C.c_void_p]),
    "b2r_serve_rows": (C.c_int, [C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_int, C.c_int,
                                 C.c_void_p, C.c_void_p]),
    "b2r_scatter_f32_to_peers": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_int, C.c_int, C.c_float,
                                           C.c_void_p]),
    "b2r_scatter_rows_to_peers": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_int, C.c_int, C.c_int,
                                            C.c_void_p]),
    "b2r_sum_rows_from_peers": (C.c_int, [C.c_void_p, C.c_int, C.c_int64, C.c_void_p, C.c_int64, C.c_void_p]),
    "b2r_colsum_prod": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_int, C.c_void_p]),
    "b2r_bprmf_fused_fwd_bwd": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_int64,
                                          C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int,
                                          C.c_void_p, C.c_void_p]),
    "b2r_bprmf_step_workspace_bytes": (C.c_size_t, [C.c_int, C.c_int, C.c_int, C.c_int64, C.c_int64]),
    "b2r_bprmf_ctx_create": (C.c_int, [C.POINTER(C.c_void_p), C.c_int, C.c_int, C.c_int, C.c_int64, C.c_int64,
                                       C.c_void_p, C.c_size_t]),
    "b2r_bprmf_ctx_destroy": (C.c_int, [C.c_void_p]),
    "b2r_bprmf_ctx_reset": (C.c_int, [C.c_void_p]),
    "b2r_bprmf_ctx_plan_launch": (C.c_int, [C.c_void_p, C.c_int, C.c_int]),
    "b2r_bprmf_train_step": (C.c_int, [C.c_void_p, C.POINTER(BprmfTables), C.c_void_p, C.c_void_p, C.c_void_p,
                                       C.c_void_p, C.POINTER(Optim), C.c_void_p, C.c_void_p, C.c_void_p]),
}


class B200RecError(RuntimeError):
    pass


_lib = None


def load() -> C.CDLL:
    """Load libb200rec.so (built in-tree by `python -m rechorus_b200.build`); raises if absent."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise B200RecError(
            f"{LIB_PATH} not found: build it with `python -m rechorus_b200.build` "
            "(there is no PyTorch/CPU fallback for the hot path)")
    lib = C.CDLL(LIB_PATH)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)          # AttributeError if the .so lacks a declared symbol
        fn.restype = res
        fn.argtypes = args
    got = lib.b2r_version()
    if got // 100 != 1:
        raise B200RecError(f"libb200rec.so ABI version {got} does not match this package (expects 1xx)")
    _lib = lib
    return lib


def check(rc: int, what: str) -> None:
    if rc != 0:
        msg = load().b2r_last_error().decode("utf-8", "replace")
        raise B200RecError(f"{what} failed (code {rc}): {msg}")
