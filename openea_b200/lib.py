"""ctypes binding of liboea.so (the C-ABI declared in include/oea.h).

There is deliberately NO fallback: if the shared library is missing or an entry point returns an
error, the call raises.  Loading does not create a CUDA context.
"""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
# OEA_LIB_PATH: kernel A/B experiments only (scripts/ab_score.sh builds variant libraries next to the default one)
LIB_PATH = os.environ.get("OEA_LIB_PATH") or os.path.join(_HERE, "_lib", "liboea.so")

SCORE_L1, SCORE_L2SQ = 0, 1
LOSS_MARGIN, LOSS_LIMITED, LOSS_LOGISTIC, LOSS_POSITIVE, LOSS_LOGSIGMOID = 0, 1, 2, 3, 4
OPT_SGD, OPT_ADAGRAD, OPT_ADAM, OPT_ADADELTA = 0, 1, 2, 3
WEIGHT_DIRECT, WEIGHT_RECIPROCAL = 0, 1
METRIC_INNER, METRIC_L1, METRIC_L2 = 0, 1, 2
P2P_MAX_WORLD = 16
MODEL_TRANSE, MODEL_TRANSH, MODEL_TRANSD, MODEL_DISTMULT, MODEL_SIMPLE = 0, 1, 2, 3, 4
MODEL_ROTATE, MODEL_HOLE, MODEL_TRANSR = 5, 6, 7


class OeaError(RuntimeError):
    pass


class Table(C.Structure):
    _fields_ = [("weight", C.c_void_p), ("grad", C.c_void_p), ("state1", C.c_void_p), ("state2", C.c_void_p),
                ("touched", C.c_void_p), ("rows", C.c_int32), ("dim", C.c_int32), ("pitch", C.c_int32),
                ("l2_norm", C.c_int32)]


class LossCfg(C.Structure):
    _fields_ = [("score_kind", C.c_int32), ("loss_kind", C.c_int32), ("margin", C.c_float),
                ("neg_margin", C.c_float), ("balance", C.c_float)]


class OptCfg(C.Structure):
    _fields_ = [("kind", C.c_int32), ("lr", C.c_float), ("beta1", C.c_float), ("beta2", C.c_float),
                ("eps", C.c_float), ("t", C.c_int32)]


class KgView(C.Structure):
    _fields_ = [("triples", C.c_void_p), ("n_triples", C.c_int32), ("entities", C.c_void_p),
                ("n_entities", C.c_int32), ("cand", C.c_void_p), ("ent2row", C.c_void_p), ("n_cand", C.c_int32)]


class TripleSet(C.Structure):
    _fields_ = [("slots", C.c_void_p), ("capacity", C.c_uint32), ("ent_bits", C.c_uint32), ("rel_bits", C.c_uint32),
                ("filter", C.c_void_p), ("filter_words", C.c_uint32)]


class SampleCfg(C.Structure):
    _fields_ = [("batch_size", C.c_int32), ("neg_per_pos", C.c_int32), ("step", C.c_int32), ("max_try", C.c_int32),
                ("epoch_seed", C.c_uint64), ("dev_seed", C.c_void_p), ("shard_rank", C.c_int32), ("shard_world", C.c_int32)]


class SimCfg(C.Structure):
    _fields_ = [("metric", C.c_int32), ("n1", C.c_int32), ("n2", C.c_int32), ("dim", C.c_int32),
                ("pitch1", C.c_int32), ("pitch2", C.c_int32), ("e1_t", C.c_void_p), ("e2_t", C.c_void_p),
                ("ld1_t", C.c_int64), ("ld2_t", C.c_int64)]


class SpmmHubs(C.Structure):
    _fields_ = [("long_rows", C.c_void_p), ("seg_ptr", C.c_void_p), ("seg_row", C.c_void_p), ("seg_start", C.c_void_p),
                ("n_long", C.c_int32), ("n_seg", C.c_int32)]


class Csr(C.Structure):
    _fields_ = [("rowptr", C.c_void_p), ("col", C.c_void_p), ("val", C.c_void_p), ("n_rows", C.c_int32),
                ("n_cols", C.c_int32), ("nnz", C.c_int64)]


_P, _I, _L = C.c_void_p, C.c_int32, C.c_int64
_TP = C.POINTER(Table)


class FedPipeline(C.Structure):
    _fields_ = [("copy_stream", C.c_void_p), ("compute_stream", C.c_void_p), ("ev_copied", C.c_void_p * 2),
                ("ev_computed", C.c_void_p * 2), ("dev_idx", C.c_void_p * 2), ("dev_loss", C.c_void_p * 2),
                ("host_loss", C.c_void_p * 2)]


class SeedXchg(C.Structure):
    _fields_ = [("rank", C.c_int32), ("world", C.c_int32), ("pitch", C.c_int32), ("max_rows", C.c_int32),
                ("window", C.c_void_p * 16), ("own_ids", C.c_void_p), ("n_own", C.c_int32), ("slot_ids", C.c_void_p),
                ("ticket", C.c_void_p)]


class Proje(C.Structure):
    # oea_proje: ent_embeds, rel_embeds, entity_w, entity_b ([E, 1]) and the [4, d] table of mlp_w, mlp_bias and the betas
    _fields_ = [("ent", _TP), ("rel", _TP), ("cls_w", _TP), ("cls_b", _TP), ("params", _TP)]


class Conve(C.Structure):
    # oea_conve: ProjE's four tables, then the tower's: conv [F, 12], bn_in [2, y], fc_w [2Fd, d], fc_out [3, d]
    _fields_ = [("ent", _TP), ("rel", _TP), ("cls_w", _TP), ("cls_b", _TP), ("conv", _TP), ("bn_in", _TP),
                ("fc_w", _TP), ("fc_out", _TP)]


class Nce(C.Structure):
    # oea_nce: the input table, the class table and the class biases ([C, 1])
    _fields_ = [("in_", _TP), ("cls_w", _TP), ("cls_b", _TP)]


class Model(C.Structure):
    # gamma / phase: RotatE's model constants (0 and ignored for the other kinds)
    _fields_ = [("kind", C.c_int32), ("ent", _TP), ("rel", _TP), ("ent_aux", _TP), ("rel_aux", _TP),
                ("gamma", C.c_float), ("phase", C.c_float)]


# name → (restype, argtypes).  Must list every symbol include/oea.h declares (tests check this).
SIGNATURES = {
    "oea_abi_version": (C.c_int, []),
    "oea_error_string": (C.c_char_p, [C.c_int]),
    "oea_triple_score_fed": (C.c_int, [_TP, _TP, _P, _P, _P, _I, _P, _P, _P, _I, C.POINTER(LossCfg), _P, _P]),
    "oea_triple_score_margin_weighted": (C.c_int, [_TP, _TP, _P, _P, _P, _P, _P, _P, _I, _P, _I, C.c_float,
                                                   C.POINTER(LossCfg), _P, _P]),
    "oea_pair_distance_loss": (C.c_int, [_TP, _P, _P, _I, _P, C.c_float, _P, _P]),
    "oea_triple_score_fed_grouped": (C.c_int, [_TP, _TP, _P, _P, _P, _I, _P, _P, _P, _I, C.POINTER(LossCfg), _P, _P]),
    "oea_triple_step_fed_grouped": (C.c_int, [_TP, _TP, _P, _P, _P, _I, _P, _P, _P, _I, C.POINTER(LossCfg),
                                              C.POINTER(OptCfg), _P, _P]),
    "oea_rowopt_apply": (C.c_int, [_TP, C.POINTER(OptCfg), _P]),
    "oea_rowopt_apply_pair": (C.c_int, [_TP, _TP, C.POINTER(OptCfg), _P]),
    "oea_rowopt_adadelta": (C.c_int, [_TP, C.POINTER(OptCfg), _P]),
    "oea_triple_step_sampled": (C.c_int, [_TP, _TP, C.POINTER(KgView), C.POINTER(KgView), C.POINTER(TripleSet),
                                          C.POINTER(SampleCfg), C.POINTER(LossCfg), C.POINTER(OptCfg), _P, _P, _P]),
    "oea_triple_score_sampled": (C.c_int, [_TP, _TP, C.POINTER(KgView), C.POINTER(KgView), C.POINTER(TripleSet),
                                           C.POINTER(SampleCfg), C.POINTER(LossCfg), _P, _P, _P, _P]),
    "oea_triple_step_fed_host": (C.c_int, [_TP, _TP, _P, _I, _P, _I, C.POINTER(LossCfg), C.POINTER(OptCfg),
                                           _P, _P, _P, C.POINTER(C.c_float), _P]),
    "oea_triple_step_fed_host_submit": (C.c_int, [_TP, _TP, C.POINTER(FedPipeline), _I, _P, _I, _P, _I,
                                                  C.POINTER(LossCfg), C.POINTER(OptCfg)]),
    "oea_triple_step_fed_host_collect": (C.c_int, [C.POINTER(FedPipeline), _I, C.POINTER(C.c_float)]),
    "oea_table_lookup": (C.c_int, [_TP, _P, _I, _P, _I, _P]),
    "oea_sim_transpose_ld": (C.c_int64, [_I]),
    "oea_sim_transpose_bytes": (C.c_size_t, [_I, _I]),
    "oea_sim_transpose": (C.c_int, [_P, _I, _I, _P, _P]),
    "oea_sim_topk_workspace_bytes": (C.c_size_t, [C.POINTER(SimCfg), _I]),
    "oea_sim_topk": (C.c_int, [C.POINTER(SimCfg), _P, _P, _P, _P, _I, _P, _P, _P, _P, C.c_size_t, _P]),
    "oea_sim_rank_workspace_bytes": (C.c_size_t, [C.POINTER(SimCfg)]),
    "oea_sim_rank": (C.c_int, [C.POINTER(SimCfg), _P, _P, _P, _P, _P, _P, _P, _P, C.c_size_t, _P]),
    "oea_sim_matrix": (C.c_int, [C.POINTER(SimCfg), _P, _P, _P, _P, _P, _L, _P]),
    "oea_sim_matrix_tc": (C.c_int, [C.POINTER(SimCfg), _P, _P, _P, _P, _P, _L, _P]),
    "oea_matrix_topk_mean_workspace_bytes": (C.c_size_t, [_I, _I, _I, _I]),
    "oea_matrix_topk_mean": (C.c_int, [_P, _L, _I, _I, _I, _I, _P, _P, C.c_size_t, _P]),
    "oea_rank_stats": (C.c_int, [_P, _I, _P, _I, _P, _P]),
    "oea_matrix_rank": (C.c_int, [_P, _L, _I, _I, _P, _P, _P, _P, _P, _P]),
    "oea_rows_normalize": (C.c_int, [_P, _I, _I, _I, _P, _I, _P]),
    "oea_rows_select_topk": (C.c_int, [_P, _L, _I, _I, _I, _P, _P, _P]),
    "oea_table_scatter_grad": (C.c_int, [_TP, _P, _I, _P, _I, _P]),
    "oea_loss_rows": (C.c_int, [_P, _P, _P, _I, _P, _P, _P, _I, _I, _I, C.POINTER(LossCfg), _P, _P, _P, _P, _P, _P, _P, _P]),
    "oea_mapping_workspace_bytes": (C.c_size_t, [_I]),
    "oea_mapping_fwd_bwd": (C.c_int, [_P, _P, _I, _I, _I, _P, _I, C.c_float, _P, _P, _P, _P, _P, C.c_size_t, _P]),
    "oea_spmm_long_row_threshold": (C.c_int, []),
    "oea_spmm_segment_nnz": (C.c_int, []),
    "oea_spmm_workspace_bytes": (C.c_size_t, [_I, _I]),
    "oea_spmm_csr": (C.c_int, [C.POINTER(Csr), C.POINTER(SpmmHubs), _P, _I, _P, _I, _I, _I, _P, C.c_float, _P, C.c_size_t, _P]),
    "oea_edge_softmax_fwd": (C.c_int, [C.POINTER(Csr), _P, _P, C.c_float, _P, _P]),
    "oea_sddmm": (C.c_int, [C.POINTER(Csr), _P, _I, _P, _I, _I, _P, _P]),
    "oea_edge_softmax_bwd": (C.c_int, [C.POINTER(Csr), _P, _P, C.c_float, _P, _P, _P, _P, _P]),
    "oea_align_loss_l1": (C.c_int, [_P, _I, _I, _P, _P, _I, _I, _P, _P, _P, _P, C.c_float, _P, _P, _P]),
    "oea_tripleset_build": (C.c_int, [_P, _I, _P, C.c_uint32, C.c_uint32, C.c_uint32, _P]),
    "oea_model_score_fed": (C.c_int, [C.POINTER(Model), _P, _P, _P, _I, _P, _P, _P, _I, C.POINTER(LossCfg), C.c_float,
                                      _P, _P]),
    "oea_transr_workspace_bytes": (C.c_size_t, [_I, _I, _I, _I]),
    "oea_transr_score_fed": (C.c_int, [C.POINTER(Model), _P, _P, _P, _I, _P, _P, _P, _I, C.POINTER(LossCfg), C.c_float,
                                       _P, C.c_size_t, _P, _P]),
    "oea_logu_sample_unique": (C.c_int, [_I, _I, C.c_uint64, _P, _P, _P, C.c_size_t, _P]),
    "oea_proje_workspace_bytes": (C.c_size_t, [_I, _I, _I, _I]),
    "oea_proje_score_fed": (C.c_int, [C.POINTER(Proje), _P, _P, _P, _I, _P, _P, _I, _P, C.c_size_t, _P, _P]),
    "oea_conve_workspace_bytes": (C.c_size_t, [_I, _I, _I, _I, _I]),
    "oea_conve_score_fed": (C.c_int, [C.POINTER(Conve), _P, _P, _P, _I, _P, _P, _I, C.c_float, C.c_uint64, _P,
                                      C.c_size_t, _P, _P]),
    "oea_nce_workspace_bytes": (C.c_size_t, [_I, _I, _I, _I]),
    "oea_nce_score_fed": (C.c_int, [C.POINTER(Nce), _P, _P, _I, _P, _P, _I, C.c_float, _P, C.c_size_t, _P, _P]),
    "oea_pairs_draw": (C.c_int, [_P, _I, _I, C.c_uint64, _I, _I, _P, _P, _P]),
    "oea_rows_gather_sort": (C.c_int, [_P, _L, _I, _I, _P, _P, _P]),
    "oea_gale_shapley_workspace_bytes": (C.c_size_t, [_I, _I]),
    "oea_gale_shapley": (C.c_int, [_P, _P, _I, _I, _I, _I, _P, _P, C.c_size_t, C.POINTER(C.c_int32), _P]),
    "oea_seed_xchg_window_bytes": (C.c_size_t, [_I, _I, _I]),
    "oea_p2p_window_create": (C.c_int, [C.c_size_t, C.POINTER(C.c_void_p), _P]),
    "oea_p2p_window_open": (C.c_int, [_P, C.POINTER(C.c_void_p)]),
    "oea_p2p_window_close": (C.c_int, [_P]),
    "oea_p2p_window_destroy": (C.c_int, [_P]),
    "oea_seed_push": (C.c_int, [C.POINTER(SeedXchg), _P, C.c_uint64, _P]),
    "oea_seed_pull": (C.c_int, [C.POINTER(SeedXchg), _P, C.c_uint64, C.c_uint64, _P]),
    "oea_seed_xchg_status": (C.c_int, [C.POINTER(SeedXchg), C.POINTER(C.c_int32)]),
    "oea_seed_pack": (C.c_int, [_P, _I, _P, _I, _P, _P]),
    "oea_seed_unpack": (C.c_int, [_P, _I, _P, _P, _I, _I, _I, _P]),
    "oea_triple_sample_batch": (C.c_int, [C.POINTER(KgView), C.POINTER(KgView), C.POINTER(TripleSet),
                                          C.POINTER(SampleCfg), _I, _TP, _P, _P, C.POINTER(C.c_int32), _P]),
}

_lib = None


def declared_symbols():
    """Entry-point names parsed from include/oea.h (used by the CPU export test)."""
    import re
    hdr = os.path.join(os.path.dirname(_HERE), "include", "oea.h")
    with open(hdr) as f:
        text = f.read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(oea_[a-z0-9_]+)\s*\(", text)))


def load():
    """dlopen liboea.so and attach signatures.  Raises OeaError when it is not built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise OeaError(
            "liboea.so is not built (%s). Run `python -m openea_b200.build`; there is no CPU fallback." % LIB_PATH)
    lib = C.CDLL(LIB_PATH)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)
        fn.restype = res
        fn.argtypes = args
    if lib.oea_abi_version() != 1:
        raise OeaError("liboea.so ABI version mismatch")
    _lib = lib
    return lib


def check(rc, what=""):
    if rc != 0:
        msg = load().oea_error_string(rc)
        raise OeaError("%s failed: rc=%d (%s)" % (what or "liboea call", rc, msg.decode() if msg else "?"))
