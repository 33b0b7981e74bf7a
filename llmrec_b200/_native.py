"""ctypes binding of libllmrec_b200.so (the C ABI declared in include/llmrec_b200.h).

There is NO fallback: if the library is missing or the device is not sm_90 every op raises.
"""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "lib", "libllmrec_b200.so")

MAX_SEG = 16
SPMM_SOFTMAX = 1

c_f32p = C.c_void_p
c_i32p = C.c_void_p
c_stream = C.c_void_p


class SpmmSeg(C.Structure):
    _fields_ = [("X", C.c_void_p), ("Y", C.c_void_p), ("Z", C.c_void_p), ("ldx", C.c_int64), ("ldy", C.c_int64),
                ("ldz", C.c_int64), ("flags", C.c_int32), ("_pad", C.c_int32)]


class SpmmTiling(C.Structure):
    _fields_ = [("tiles", C.c_void_p), ("split_row", C.c_void_p), ("split_first", C.c_void_p), ("scratch", C.c_void_p),
                ("n_tiles", C.c_int32), ("n_split", C.c_int32), ("n_split_tiles", C.c_int32), ("_pad", C.c_int32), ("split_tickets", C.c_void_p),
                ("src_mask", C.c_void_p)]


class ProjFwdProblem(C.Structure):
    _fields_ = [("X", C.c_void_p), ("W", C.c_void_p), ("bias", C.c_void_p), ("Y", C.c_void_p), ("wsplit", C.c_void_p),
                ("ldx", C.c_int64), ("ldy", C.c_int64), ("n", C.c_int64), ("k", C.c_int32), ("_reserved", C.c_int32)]


class ProjWgradProblem(C.Structure):
    _fields_ = [("X", C.c_void_p), ("dY", C.c_void_p), ("dW", C.c_void_p), ("db", C.c_void_p),
                ("ldx", C.c_int64), ("lddy", C.c_int64), ("n", C.c_int64), ("k", C.c_int32), ("accumulate", C.c_int32)]


class ProjFwdProblemBf16(C.Structure):      # X: raw bfloat16 bits
    _fields_ = ProjFwdProblem._fields_


class ProjWgradProblemBf16(C.Structure):    # X: raw bfloat16 bits
    _fields_ = ProjWgradProblem._fields_


class ProjFwdProblemI8(C.Structure):        # X: int8 table rows (llmrec_b200/feat_int8.py), ldx = row pitch in bytes
    _fields_ = ProjFwdProblem._fields_


class ProjWgradProblemI8(C.Structure):      # X: int8 table rows (llmrec_b200/feat_int8.py), ldx = row pitch in bytes
    _fields_ = ProjWgradProblem._fields_


class ProjRowMap(C.Structure):             # follows the problems of a grouped projection call that flags PROJ_ROW_MAP
    _fields_ = [("rows", C.c_void_p), ("n_dy", C.c_int64)]


PROJ_ROW_MAP = 2
WGRAD_ACCUMULATE = 1


class BprHead(C.Structure):
    _fields_ = [("XU", C.c_void_p), ("XI", C.c_void_p), ("GU", C.c_void_p), ("GI", C.c_void_p),
                ("ldxu", C.c_int64), ("ldxi", C.c_int64), ("ldgu", C.c_int64), ("ldgi", C.c_int64),
                ("w_mf", C.c_float), ("w_emb", C.c_float)]


class GradRegion(C.Structure):
    _fields_ = [("G", C.c_void_p), ("X", C.c_void_p), ("ldg", C.c_int64), ("ldx", C.c_int64), ("n", C.c_int64),
                ("width", C.c_int32), ("c", C.c_float)]


class Rank1Block(C.Structure):
    _fields_ = [("Y", C.c_void_p), ("scale", C.c_void_p), ("bias", C.c_void_p), ("ldy", C.c_int64), ("lds", C.c_int64), ("n", C.c_int64),
                ("width", C.c_int32), ("_pad", C.c_int32)]


class ColsumTerm(C.Structure):
    _fields_ = [("G", C.c_void_p), ("scale", C.c_void_p), ("ldg", C.c_int64), ("lds", C.c_int64), ("n", C.c_int64)]


# name -> (restype, argtypes); must list every symbol of include/llmrec_b200.h (checked by tests)
SIGNATURES = {
    "llmrec_abi_version": (C.c_int, []),
    "llmrec_last_error": (C.c_char_p, []),
    "llmrec_device_ok": (C.c_int, []),
    "llmrec_spmm_csr_f32": (C.c_int, [c_i32p, c_i32p, c_f32p, c_f32p, c_f32p, C.c_int32, C.c_int32, C.c_int32,
                                      C.POINTER(SpmmSeg), C.c_int32, C.POINTER(SpmmTiling), c_stream]),
    "llmrec_spmm_plan_tiles": (C.c_int, [C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "llmrec_spmm_rows_f32": (C.c_int, [c_i32p, c_i32p, c_f32p, c_f32p, c_f32p, C.c_int32, C.POINTER(SpmmSeg), c_i32p, c_i32p, C.c_int32, C.c_void_p, C.c_int32, c_stream]),
    "llmrec_row_softmax_bwd_rows_f32": (C.c_int, [c_f32p, C.c_int64, c_f32p, C.c_int64, c_f32p, C.c_int64, c_i32p, c_i32p, C.c_int32, C.c_int32, c_stream]),
    "llmrec_mark_neighbors": (C.c_int, [c_i32p, c_i32p, c_i32p, C.c_int32, C.c_void_p, c_stream]),
    "llmrec_mark_ids": (C.c_int, [c_i32p, C.c_int32, C.c_void_p, c_stream]),
    "llmrec_mark_ids_rows": (C.c_int, [c_i32p, c_i32p, C.c_int32, C.c_void_p, c_stream]),
    "llmrec_compact_mask": (C.c_int, [C.c_void_p, C.c_int32, c_i32p, c_i32p, c_stream]),
    "llmrec_zero_rows_f32": (C.c_int, [c_f32p, C.c_int64, c_i32p, C.c_int32, C.c_int32, c_stream]),
    "llmrec_assign_rows_f32": (C.c_int, [c_f32p, C.c_int64, c_i32p, C.c_int32, C.c_int32, c_f32p, C.c_int64, c_stream]),
    "llmrec_adamw_step_rows_f32": (C.c_int, [c_f32p, c_f32p, c_f32p, c_f32p, C.c_int64, C.c_int32, C.c_void_p, C.c_void_p, C.c_float, C.c_float, C.c_float, C.c_float, C.c_float, c_stream]),
    "llmrec_row_softmax_f32": (C.c_int, [c_f32p, C.c_int64, c_f32p, C.c_int64, C.c_int64, C.c_int32, c_stream]),
    "llmrec_row_softmax_bwd_f32": (C.c_int, [c_f32p, C.c_int64, c_f32p, C.c_int64, c_f32p, C.c_int64, C.c_int64, C.c_int32, c_stream]),
    "llmrec_proj_fwd_f32": (C.c_int, [c_f32p, C.c_int64, c_f32p, c_f32p, c_f32p, C.c_int64, C.c_int64, C.c_int32, C.c_int32, C.c_int32, c_f32p, c_stream]),
    "llmrec_proj_fwd_group_f32": (C.c_int, [C.POINTER(ProjFwdProblem), C.c_int32, C.c_int32, C.c_int32, c_stream]),
    "llmrec_proj_wgrad_group_f32": (C.c_int, [C.POINTER(ProjWgradProblem), C.c_int32, C.c_int32, C.c_int32, c_f32p, C.c_int64, c_stream]),
    "llmrec_proj_wgrad_group_scratch": (C.c_int64, [C.POINTER(ProjWgradProblem), C.c_int32, C.c_int32, C.c_int32]),
    "llmrec_proj_fwd_group_bf16": (C.c_int, [C.POINTER(ProjFwdProblemBf16), C.c_int32, C.c_int32, C.c_int32, c_stream]),
    "llmrec_proj_wgrad_group_bf16": (C.c_int, [C.POINTER(ProjWgradProblemBf16), C.c_int32, C.c_int32, C.c_int32, c_f32p, C.c_int64, c_stream]),
    "llmrec_proj_wgrad_group_bf16_scratch": (C.c_int64, [C.POINTER(ProjWgradProblemBf16), C.c_int32, C.c_int32, C.c_int32]),
    "llmrec_proj_fwd_group_i8": (C.c_int, [C.POINTER(ProjFwdProblemI8), C.c_int32, C.c_int32, C.c_int32, c_stream]),
    "llmrec_proj_wgrad_group_i8": (C.c_int, [C.POINTER(ProjWgradProblemI8), C.c_int32, C.c_int32, C.c_int32, c_f32p, C.c_int64, c_stream]),
    "llmrec_proj_wgrad_group_i8_scratch": (C.c_int64, [C.POINTER(ProjWgradProblemI8), C.c_int32, C.c_int32, C.c_int32]),
    "llmrec_proj_wgrad_f32": (C.c_int, [c_f32p, C.c_int64, c_f32p, C.c_int64, c_f32p, c_f32p, C.c_int64, C.c_int32, C.c_int32,
                                        C.c_int32, C.c_int32, c_f32p, C.c_int64, c_stream]),
    "llmrec_proj_wgrad_scratch": (C.c_int64, [C.c_int64, C.c_int32, C.c_int32, C.c_int32]),
    "llmrec_fuse_fwd_f32": (C.c_int, [C.POINTER(C.c_void_p), C.POINTER(C.c_int64), C.c_int32, C.POINTER(C.c_void_p), C.POINTER(C.c_int64),
                                      C.POINTER(C.c_float), C.c_int32, c_f32p, C.c_int64, c_i32p, C.c_int64, C.c_int32, c_stream]),
    "llmrec_fuse_bwd_f32": (C.c_int, [c_f32p, C.c_int64, C.c_int32, c_f32p, C.c_int64, C.POINTER(C.c_void_p), C.POINTER(C.c_int64),
                                      C.POINTER(C.c_float), C.POINTER(C.c_void_p), C.POINTER(C.c_int64), C.c_int32, C.c_int32,
                                      c_i32p, C.c_int64, C.c_int32, c_stream]),
    "llmrec_fuse_fwd_rows_f32": (C.c_int, [C.POINTER(C.c_void_p), C.POINTER(C.c_int64), C.c_int32, C.POINTER(C.c_void_p), C.POINTER(C.c_int64),
                                           C.POINTER(C.c_float), C.c_int32, c_f32p, C.c_int64, c_i32p, c_i32p, C.c_int32, C.c_int32, c_stream]),
    "llmrec_fuse_bwd_rows_f32": (C.c_int, [c_f32p, C.c_int64, C.c_int32, c_f32p, C.c_int64, C.POINTER(C.c_void_p), C.POINTER(C.c_int64),
                                           C.POINTER(C.c_float), C.POINTER(C.c_void_p), C.POINTER(C.c_int64), C.c_int32, C.c_int32,
                                           c_i32p, c_i32p, C.c_int32, C.c_int32, c_stream]),
    "llmrec_grad_init_f32": (C.c_int, [C.POINTER(GradRegion), C.c_int32, c_f32p, c_f32p, c_stream]),
    "llmrec_grad_init_scratch": (C.c_int64, []),
    "llmrec_bpr_heads_f32": (C.c_int, [C.POINTER(BprHead), C.c_int32, c_i32p, c_i32p, c_i32p, C.c_int32, C.c_int32, c_i32p, C.c_float,
                                       C.c_int32, c_f32p, c_f32p, c_f32p, c_stream]),
    "llmrec_bpr_work_elems": (C.c_int64, [C.c_int32, C.c_int32]),
    "llmrec_bpr_slot_plan_elems": (C.c_int64, [C.c_int32]),
    "llmrec_bpr_slot_plan": (C.c_int, [c_i32p, c_i32p, c_i32p, C.c_int32, c_i32p, c_i32p, c_stream]),
    "llmrec_bpr_heads_ordered_f32": (C.c_int, [C.POINTER(BprHead), C.c_int32, c_i32p, c_i32p, c_i32p, C.c_int32, C.c_int32, c_i32p, C.c_float,
                                               C.c_int32, c_f32p, c_f32p, c_f32p, c_i32p, c_stream]),
    "llmrec_sqnorm_grad_f32": (C.c_int, [c_f32p, C.c_int64, c_f32p, C.c_int64, C.c_int64, C.c_int32, C.c_float, C.c_int32,
                                         c_f32p, c_f32p, c_stream]),
    "llmrec_adamw_advance": (C.c_int, [C.c_void_p, C.c_double, C.c_double, C.c_double, c_stream]),
    "llmrec_adamw_step_f32": (C.c_int, [C.POINTER(C.c_void_p), C.POINTER(C.c_void_p), C.POINTER(C.c_void_p), C.POINTER(C.c_void_p),
                                        C.POINTER(C.c_int64), C.c_int32, C.c_void_p, C.c_float, C.c_float, C.c_float, C.c_float,
                                        C.c_float, c_stream]),
    "llmrec_score_topk_f32": (C.c_int, [c_f32p, C.c_int64, c_f32p, C.c_int64, c_i32p, C.c_int32, C.c_int32, C.c_int32, c_i32p, c_i32p,
                                        C.c_int32, c_i32p, c_f32p, C.c_int32, c_f32p, C.c_int64, c_stream]),
    "llmrec_score_topk_scratch": (C.c_int64, [C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32]),
    "llmrec_score_topk_among_f32": (C.c_int, [c_f32p, C.c_int64, c_f32p, C.c_int64, c_i32p, C.c_int32, c_i32p, C.c_int32, C.c_int32, c_i32p,
                                              c_i32p, C.c_int32, c_i32p, c_f32p, C.c_int32, c_f32p, C.c_int64, c_stream]),
    "llmrec_score_topk_among_scratch": (C.c_int64, [C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32]),
    "llmrec_score_topk_group_f32": (C.c_int, [c_f32p, C.c_int64, c_f32p, C.c_int64, c_i32p, c_i32p, C.c_int32, c_i32p, C.c_int32, C.c_int32,
                                              c_i32p, c_i32p, C.c_int32, C.c_int32, c_i32p, c_f32p, C.c_int32, c_f32p, C.c_int64, c_stream]),
    "llmrec_score_topk_group_scratch": (C.c_int64, [c_i32p, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32]),
    "llmrec_topk_hits": (C.c_int, [c_i32p, C.c_int32, C.c_int32, c_i32p, c_i32p, c_i32p, C.c_void_p, c_stream]),
    "llmrec_user_auc_f32": (C.c_int, [c_f32p, C.c_int64, c_f32p, C.c_int64, c_i32p, C.c_int32, C.c_int32, C.c_int32, c_i32p, c_i32p, c_i32p, c_i32p, c_f32p, c_stream]),
    "llmrec_score_pairs_f32": (C.c_int, [c_f32p, C.c_int64, c_f32p, C.c_int64, c_i32p, c_i32p, C.c_int32, C.c_int32, c_f32p, c_stream]),
    "llmrec_rerank_f32": (C.c_int, [c_f32p, C.c_int64, c_f32p, C.c_int64, c_i32p, C.c_int32, c_i32p, c_i32p, c_i32p, c_i32p, C.c_int32,
                                    C.c_int32, C.c_int32, c_i32p, c_f32p, c_stream]),
    "llmrec_explain_f32": (C.c_int, [c_f32p, C.c_int64, c_f32p, C.c_int64, C.POINTER(C.c_void_p), C.POINTER(C.c_int64), C.POINTER(C.c_void_p),
                                     C.POINTER(C.c_int64), C.POINTER(C.c_float), C.c_int32, C.POINTER(C.c_void_p), C.POINTER(C.c_int64), C.c_int32,
                                     c_f32p, C.c_int64, C.c_int32, C.c_int32, C.c_int32, c_i32p, c_f32p, C.c_int32, c_i32p, c_i32p, c_i32p,
                                     C.c_int32, c_f32p, c_f32p, c_f32p, C.c_int32, c_i32p, c_f32p, c_stream]),
    "llmrec_diversify_f32": (C.c_int, [c_f32p, C.c_int64, c_i32p, c_f32p, C.c_int64, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32,
                                       C.c_float, c_i32p, c_f32p, c_f32p, c_stream]),
    "llmrec_host_sample_items":(C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p]),
    "llmrec_host_sample_batch": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32,
                                           C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32,
                                           C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p]),
    "llmrec_device_sample_batch": (C.c_int, [c_i32p, C.c_int32, C.c_int32, c_i32p, c_i32p, C.c_int32, C.c_int32, c_i32p, c_i32p, C.c_int32, C.c_int32,
                                             c_i32p, C.c_int32, C.c_void_p, c_i32p, C.c_void_p, c_stream]),
    "llmrec_device_sample_batch_ref_work": (C.c_int64, [C.c_int32, C.c_int32, C.c_int32, C.c_int32]),
    "llmrec_device_sample_batch_ref": (C.c_int, [c_i32p, C.c_int32, C.c_int32, C.c_int32, c_i32p, c_i32p, c_i32p, C.c_int32, C.c_int32, C.c_int32,
                                                 c_i32p, c_i32p, C.c_int32, C.c_int32, c_i32p, C.c_int32, c_i32p, c_i32p, c_i32p, C.c_int64,
                                                 c_stream]),
    "llmrec_row_scale_softmax_f32": (C.c_int, [c_f32p, C.c_int64, c_f32p, c_f32p, C.c_int64, C.c_int64, C.c_int32, C.c_int32, c_stream]),
    "llmrec_gather_rows_f32": (C.c_int, [c_f32p, C.c_int64, c_i32p, C.c_int32, C.c_int32, c_f32p, C.c_int64, c_stream]),
    "llmrec_scatter_add_rows_f32": (C.c_int, [c_f32p, C.c_int64, c_i32p, C.c_int32, C.c_int32, c_f32p, C.c_int64, c_stream]),
    "llmrec_scatter_add_rows_ordered_f32": (C.c_int, [c_f32p, C.c_int64, c_i32p, C.c_int32, C.c_int32, c_f32p, C.c_int64, c_i32p, C.c_int64, c_stream]),
    "llmrec_scatter_add_rows_ordered_scratch": (C.c_int64, [C.c_int32]),
    "llmrec_row_normalize_f32": (C.c_int, [c_f32p, C.c_int64, c_f32p, C.c_int64, C.c_int64, C.c_int32, c_stream]),
    "llmrec_rank1_add_f32": (C.c_int, [C.POINTER(Rank1Block), C.c_int32, c_stream]),
    "llmrec_scaled_colsum_f32": (C.c_int, [C.POINTER(ColsumTerm), C.c_int32, C.c_int32, c_f32p, C.c_int32, c_f32p, c_stream]),
    "llmrec_scaled_colsum_scratch": (C.c_int64, [C.c_int32]),
    "llmrec_feat_reg_gram_f32": (C.c_int, [c_f32p, c_f32p, c_f32p, c_f32p, C.c_float, C.c_int32, C.c_int32, C.c_float, c_f32p, c_f32p, c_f32p, c_f32p, c_stream]),
    "llmrec_feat_reg_gram_scratch": (C.c_int64, [C.c_int32, C.c_int32]),
    "llmrec_fill_f32": (C.c_int, [c_f32p, C.c_int64, C.c_float, c_stream]),
}

_lib = None


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(
                f"{LIB_PATH} not found: build it with `python -m llmrec_b200.build` "
                "(llmrec_b200 has no CPU or PyTorch fallback for its kernels)")
        handle = C.CDLL(LIB_PATH)
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(handle, name)
            fn.restype = res
            fn.argtypes = args
        _lib = handle
    return _lib


def check(rc: int, what: str = ""):
    if rc != 0:
        msg = lib().llmrec_last_error().decode("utf-8", "replace")
        raise RuntimeError(f"llmrec_b200 {what} failed (rc={rc}): {msg}")
