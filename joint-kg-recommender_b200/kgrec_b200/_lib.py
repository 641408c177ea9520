"""ctypes binding of the C ABI declared in include/kgrec_b200.h.

The shared library is built in-tree by ``csrc/build.py`` (nvcc, sm_90a) into
``joint-kg-recommender_b200/lib/libkgrec_b200.so``.  There is no fallback: if the
library is missing, or a call fails, a RuntimeError is raised.
"""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(os.path.dirname(_HERE), "lib", "libkgrec_b200.so")

TRANSE, TRANSH, TRANSR, TUP, KTUP = range(5)
LOSS_MARGIN, LOSS_BPR = 0, 1
SIDE_HEAD, SIDE_TAIL, SIDE_REC = 0, 1, 2
ABI_VERSION = 2

c_f32p = C.c_void_p  # device pointers travel as integers


class Tables(C.Structure):
    _fields_ = [
        ("dim", C.c_int32), ("ld", C.c_int32), ("l1", C.c_int32), ("use_gumbel", C.c_int32),
        ("n_ent", C.c_int64), ("n_rel", C.c_int64), ("n_user", C.c_int64), ("n_item", C.c_int64),
        ("n_pref", C.c_int32), ("reserved", C.c_int32),
        ("ent", C.c_void_p), ("rel", C.c_void_p), ("norm", C.c_void_p), ("proj", C.c_void_p),
        ("user", C.c_void_p), ("item", C.c_void_p), ("pref", C.c_void_p), ("pref_norm", C.c_void_p),
        ("item2ent", C.c_void_p),
    ]


class Grads(C.Structure):
    _fields_ = [
        ("mode", C.c_int32), ("reserved", C.c_int32),
        ("ent", C.c_void_p), ("rel", C.c_void_p), ("norm", C.c_void_p), ("proj", C.c_void_p),
        ("user", C.c_void_p), ("item", C.c_void_p), ("pref", C.c_void_p), ("pref_norm", C.c_void_p),
    ]


class OptTable(C.Structure):          # struct kgrec_opt_table
    _fields_ = [
        ("table", C.c_void_p), ("acc", C.c_void_p), ("state1", C.c_void_p), ("state2", C.c_void_p),
        ("marks", C.c_void_p), ("rows", C.c_int64), ("dim", C.c_int32), ("keep_acc", C.c_int32),
        ("vec", C.c_int32), ("reserved", C.c_int32),
    ]


class MarkSeg(C.Structure):           # struct kgrec_mark_seg
    _fields_ = [
        ("ids", C.c_void_p), ("n", C.c_int64), ("idx_bytes", C.c_int32), ("compact", C.c_int32),
        ("remap", C.c_void_p), ("n_remap", C.c_int64), ("marks", C.c_void_p), ("rows", C.c_int64),
    ]


class OptParams(C.Structure):         # struct kgrec_opt_params
    _fields_ = [
        ("kind", C.c_int32), ("rows", C.c_int32), ("lr", C.c_float), ("eps", C.c_float), ("beta1", C.c_float),
        ("beta2", C.c_float), ("alpha", C.c_float), ("momentum", C.c_float), ("weight_decay", C.c_float),
        ("max_norm", C.c_float), ("step_counts", C.c_void_p),
    ]


ROWS_TOUCHED, ROWS_ALL = 0, 1


class StepState(C.Structure):         # struct kgrec_step_state (lives in device memory)
    _fields_ = [
        ("step", C.c_int64), ("gumbel_seed", C.c_uint64), ("sample_seed", C.c_uint64), ("epoch", C.c_int32),
        ("lr", C.c_float),
    ]


_SIGNATURES = {
    "kgrec_abi_version": (C.c_int, []),
    "kgrec_last_error": (C.c_char_p, []),
    "kgrec_sm_count": (C.c_int, []),
    "kgrec_score_fwd": (C.c_int, [C.POINTER(Tables), C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int,
                                  C.c_int64, C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p, C.c_void_p]),
    "kgrec_score_bwd": (C.c_int, [C.POINTER(Tables), C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int,
                                  C.c_int64, C.c_void_p, C.c_uint64, C.c_void_p, C.POINTER(Grads), C.c_void_p]),
    "kgrec_rank_loss_workspace_bytes": (C.c_int64, [C.c_int64]),
    "kgrec_corrupt_loss_step_workspace_bytes": (C.c_int64, [C.POINTER(Tables), C.c_int, C.c_int64]),
    "kgrec_rank_loss_fwd": (C.c_int, [C.POINTER(Tables), C.c_int, C.c_void_p, C.c_void_p, C.c_void_p,
                                      C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int64, C.c_int32,
                                      C.c_int64, C.c_int, C.c_float, C.c_void_p, C.c_uint64,
                                      C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "kgrec_rank_loss_bwd": (C.c_int, [C.POINTER(Tables), C.c_int, C.c_void_p, C.c_void_p, C.c_void_p,
                                      C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int64, C.c_int32,
                                      C.c_int64, C.c_int, C.c_float, C.c_void_p, C.c_uint64,
                                      C.c_void_p, C.c_void_p, C.c_float, C.c_void_p, C.POINTER(Grads), C.c_void_p]),
    "kgrec_rank_loss_step": (C.c_int, [C.POINTER(Tables), C.c_int, C.c_void_p, C.c_void_p, C.c_void_p,
                                       C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int64, C.c_int32,
                                       C.c_int64, C.c_int, C.c_float, C.c_float, C.c_void_p, C.c_uint64,
                                       C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(Grads), C.c_void_p, C.c_void_p,
                                       C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "kgrec_corrupt_loss_fwd": (C.c_int, [C.POINTER(Tables), C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int,
                                         C.c_int64, C.c_void_p, C.c_int32, C.c_int64, C.c_int, C.c_float,
                                         C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "kgrec_corrupt_loss_bwd": (C.c_int, [C.POINTER(Tables), C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int,
                                         C.c_int64, C.c_void_p, C.c_int32, C.c_int64, C.c_int, C.c_float,
                                         C.c_void_p, C.c_void_p, C.c_float, C.c_void_p, C.POINTER(Grads), C.c_void_p,
                                         C.c_void_p, C.c_void_p]),
    "kgrec_corrupt_loss_step": (C.c_int, [C.POINTER(Tables), C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int,
                                          C.c_int64, C.c_void_p, C.c_int32, C.c_int64, C.c_int, C.c_float, C.c_float, C.c_int32,
                                          C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(Grads), C.c_void_p, C.c_void_p,
                                          C.c_void_p, C.c_void_p, C.c_void_p]),
    "kgrec_hashset_capacity": (C.c_int64, [C.c_int64]),
    "kgrec_hashset_build": (C.c_int, [C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_void_p]),
    "kgrec_sample_corrupt": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int64, C.c_int32, C.c_int64,
                                       C.c_int64, C.c_void_p, C.c_int64, C.c_uint64, C.c_void_p, C.c_void_p, C.c_void_p]),
    "kgrec_sample_neg_items": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int64, C.c_int32, C.c_int64,
                                         C.c_void_p, C.c_int64, C.c_uint64, C.c_void_p, C.c_void_p, C.c_void_p]),
    "kgrec_rows_mark": (C.c_int, [C.POINTER(MarkSeg), C.c_int, C.c_int32, C.c_void_p, C.c_void_p]),
    "kgrec_rows_sqnorm": (C.c_int, [C.POINTER(OptTable), C.c_int, C.c_int32, C.c_void_p, C.c_void_p]),
    "kgrec_rows_update": (C.c_int, [C.POINTER(OptTable), C.c_int, C.c_int32, C.c_int, C.c_float, C.c_float, C.c_float,
                                    C.c_float, C.c_int64, C.c_float, C.c_void_p, C.c_float, C.c_void_p]),
    "kgrec_rec_rows_workspace_floats": (C.c_int64, [C.c_int64, C.c_int64, C.c_int32, C.c_int32, C.c_int]),
    "kgrec_rec_rows_step": (C.c_int, [C.POINTER(Tables), C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int64, C.c_int32,
                                      C.c_int64, C.c_int, C.c_float, C.c_float, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p,
                                      C.c_int32, C.POINTER(Grads), C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                      C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p]),
    "kgrec_step_advance": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p]),
    "kgrec_batch_gather": (C.c_int, [C.c_void_p, C.c_int64, C.c_void_p, C.POINTER(C.c_void_p), C.POINTER(C.c_void_p), C.c_int,
                                     C.c_int, C.c_int64, C.c_int64, C.c_void_p, C.c_void_p]),
    "kgrec_rows_mark_dev": (C.c_int, [C.POINTER(MarkSeg), C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]),
    "kgrec_rows_sqnorm_dev": (C.c_int, [C.POINTER(OptTable), C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]),
    "kgrec_rows_update_dev": (C.c_int, [C.POINTER(OptTable), C.c_int, C.c_void_p, C.c_int, C.c_float, C.c_float, C.c_float,
                                        C.c_float, C.c_void_p, C.c_float, C.c_void_p]),
    "kgrec_rows_update_ex": (C.c_int, [C.POINTER(OptTable), C.c_int, C.c_int32, C.POINTER(OptParams), C.c_void_p,
                                       C.c_void_p]),
    "kgrec_rows_update_ex_dev": (C.c_int, [C.POINTER(OptTable), C.c_int, C.c_void_p, C.POINTER(OptParams), C.c_void_p,
                                           C.c_void_p]),
    "kgrec_sample_corrupt_dev": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int64, C.c_int32, C.c_int64,
                                           C.c_int64, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "kgrec_sample_neg_items_dev": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int64, C.c_int32, C.c_int64,
                                             C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "kgrec_rank_loss_step_dev": (C.c_int, [C.POINTER(Tables), C.c_int, C.c_void_p, C.c_void_p, C.c_void_p,
                                           C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int64, C.c_int32,
                                           C.c_int64, C.c_int, C.c_float, C.c_float, C.c_void_p, C.c_void_p,
                                           C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(Grads), C.c_void_p, C.c_void_p,
                                           C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "kgrec_rec_rows_step_dev": (C.c_int, [C.POINTER(Tables), C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int64,
                                          C.c_int32, C.c_int64, C.c_int, C.c_float, C.c_float, C.c_void_p, C.c_void_p,
                                          C.c_void_p, C.c_void_p, C.c_int32, C.POINTER(Grads), C.c_void_p, C.c_void_p,
                                          C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "kgrec_reg_norm_rows": (C.c_int, [C.c_void_p, C.c_int64, C.c_int32, C.c_void_p, C.c_int, C.c_int64, C.c_float,
                                      C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "kgrec_reg_orth_tables": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_int32, C.c_float, C.c_void_p, C.c_void_p,
                                        C.c_void_p, C.c_void_p]),
    "kgrec_eval_scores": (C.c_int, [C.POINTER(Tables), C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_int,
                                    C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_int64, C.c_int64,
                                    C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p, C.c_int64, C.c_void_p]),
    "kgrec_eval_workspace_bytes": (C.c_int64, [C.c_int64, C.c_int32]),
    "kgrec_eval_topk": (C.c_int, [C.POINTER(Tables), C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_int,
                                  C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_int64, C.c_int64, C.c_int32,
                                  C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64,
                                  C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p]),
    "kgrec_merge_topk": (C.c_int, [C.c_void_p, C.c_int32, C.c_int64, C.c_int32, C.c_void_p, C.c_void_p]),
    "kgrec_eval_rank_count": (C.c_int, [C.POINTER(Tables), C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_int,
                                        C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_int64, C.c_int64,
                                        C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "kgrec_eval_rank_count_ex": (C.c_int, [C.POINTER(Tables), C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_int,
                                           C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_int64, C.c_int64,
                                           C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                           C.c_void_p]),
    "kgrec_eval_rank_count_dual": (C.c_int, [C.POINTER(Tables), C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_int,
                                             C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_int64, C.c_int64,
                                             C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                             C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "kgrec_rec_topk_metrics": (C.c_int, [C.c_void_p, C.c_int64, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p,
                                         C.c_void_p]),
    "kgrec_rec_gold_scores": (C.c_int, [C.POINTER(Tables), C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_int64, C.c_void_p,
                                        C.c_int64, C.c_int64, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64,
                                        C.c_void_p, C.c_void_p]),
    "kgrec_rec_rank_workspace_bytes": (C.c_int64, [C.c_int64, C.c_int64]),
    "kgrec_rec_rank_count": (C.c_int, [C.POINTER(Tables), C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_int64, C.c_void_p,
                                       C.c_int64, C.c_int64, C.c_int64, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p,
                                       C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p, C.c_int64,
                                       C.c_void_p]),
    "kgrec_transr_workspace_floats": (C.c_int64, [C.c_int64, C.c_int64, C.c_int32]),
    "kgrec_transr_eval_scores": (C.c_int, [C.POINTER(Tables), C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_int64,
                                           C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_int64, C.c_int64, C.c_int64,
                                           C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p]),
    "kgrec_transr_eval_topk": (C.c_int, [C.POINTER(Tables), C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_int64,
                                         C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_int64, C.c_int64, C.c_int64,
                                         C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64,
                                         C.c_void_p, C.c_void_p]),
    "kgrec_transr_eval_rank_count": (C.c_int, [C.POINTER(Tables), C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_int64,
                                               C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_int64, C.c_int64, C.c_int64,
                                               C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "kgrec_transr_eval_rank_count_ex": (C.c_int, [C.POINTER(Tables), C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_int64,
                                                  C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_int64, C.c_int64,
                                                  C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                                  C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "kgrec_transr_eval_rank_count_dual": (C.c_int, [C.POINTER(Tables), C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_int64,
                                                    C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_int64, C.c_int64,
                                                    C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                                    C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                                    C.c_void_p]),
    "kgrec_gumbel_aug_ld": (C.c_int32, [C.c_int32, C.c_int32]),
    "kgrec_gumbel_aug_supported": (C.c_int32, [C.c_int32, C.c_int32, C.c_int32]),
    "kgrec_gumbel_aug_rows": (C.c_int, [C.POINTER(Tables), C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_int64, C.c_int64,
                                        C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p]),
    "kgrec_pref_aug_ld": (C.c_int32, [C.c_int32]),
    "kgrec_pref_aug_supported": (C.c_int32, [C.c_int32, C.c_int32]),
    "kgrec_pref_eval_supported": (C.c_int32, [C.c_int32, C.c_int32, C.c_int32, C.c_int32]),
    "kgrec_pref_aug_rows": (C.c_int, [C.POINTER(Tables), C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_int64,
                                      C.c_int64, C.c_void_p, C.c_int64, C.c_void_p]),
    "kgrec_ktup_item_table": (C.c_int, [C.POINTER(Tables), C.c_int64, C.c_int64, C.c_void_p, C.c_int64,
                                        C.c_void_p]),
}

EXPORTS = tuple(sorted(_SIGNATURES))

_lib = None


def load():
    """Load (once) and return the ctypes handle.  Raises if the library is absent."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(
            "kgrec_b200: %s is missing -- build it with `python joint-kg-recommender_b200/csrc/build.py` "
            "(or __graft_entry__.build()).  There is no CPU or PyTorch fallback." % LIB_PATH)
    lib = C.CDLL(LIB_PATH)
    for name, (res, args) in _SIGNATURES.items():
        fn = getattr(lib, name)   # AttributeError here == header / library mismatch
        fn.restype = res
        fn.argtypes = args
    if lib.kgrec_abi_version() != ABI_VERSION:
        raise RuntimeError("kgrec_b200: ABI version mismatch (%d != %d)" % (lib.kgrec_abi_version(), ABI_VERSION))
    _lib = lib
    return lib


def check(rc):
    if rc != 0:
        msg = load().kgrec_last_error().decode("utf-8", "replace")
        raise RuntimeError("kgrec_b200 call failed (code %d): %s" % (rc, msg))
