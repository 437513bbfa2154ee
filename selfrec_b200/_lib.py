"""ctypes binding of include/selfrec_b200.h (the C ABI of the CUDA library).

The structures below mirror the header field for field.  Loading fails loudly when the
library has not been built; device entry points fail loudly (SrbError) when no GPU is
usable -- there is no CPU fallback anywhere in the product path.
"""
import ctypes as C
import os

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, "libselfrec_b200.so")

c_i32p = C.POINTER(C.c_int32)
c_f32p = C.POINTER(C.c_float)
c_u32p = C.POINTER(C.c_uint32)
c_i64p = C.POINTER(C.c_int64)
VP = C.c_void_p


class SrbError(RuntimeError):
    pass


class HubSplit(C.Structure):
    _fields_ = [("n_rows", C.c_int32), ("n_work", C.c_int32), ("first", VP), ("work", VP), ("part", VP), ("seg", VP), ("seg_cnt", VP),
                ("order_cta", VP), ("order_warp", VP), ("n_cta", C.c_int32), ("n_warp", C.c_int32)]


HUB_CHUNK = 2048    # SRB_HUB_CHUNK
HUB_MIN_NNZ = 4096  # SRB_HUB_MIN_NNZ
HUB_WARP_SEG = 256  # SRB_HUB_WARP_SEG


class SpmmDesc(C.Structure):
    _fields_ = [
        ("rowptr", VP), ("colidx", VP), ("vals", VP),
        ("n_rows", C.c_int32), ("n_cols", C.c_int32), ("d", C.c_int32),
        ("row_order", VP), ("n_long_rows", C.c_int32), ("n_vlong_rows", C.c_int32), ("hub", HubSplit), ("n_vlong_dev", VP), ("col_mask", VP), ("X", VP), ("Y", VP), ("extra", VP), ("extra_scale", C.c_float),
        ("noise_mode", C.c_int32), ("noise", VP), ("eps", C.c_float),
        ("philox_seed", C.c_uint64), ("philox_offset", C.c_uint64), ("philox_step_dev", VP),
        ("sum_in", VP), ("sum_out", VP), ("sum_scale", C.c_float),
        ("adam_p", VP), ("adam_m", VP), ("adam_v", VP), ("adam_scalars", VP),
        ("beta1", C.c_double), ("beta2", C.c_double), ("adam_eps", C.c_float),
    ]


class EncoderDesc(C.Structure):
    _fields_ = [
        ("rowptr", VP), ("colidx", VP), ("vals", VP), ("row_order", VP), ("n_long_rows", C.c_int32),
        ("n_vlong_rows", C.c_int32), ("hub", HubSplit), ("n", C.c_int32), ("d", C.c_int32), ("n_layers", C.c_int32), ("include_ego", C.c_int32),
        ("layer_cl", C.c_int32), ("noise_mode", C.c_int32), ("noise", VP), ("eps", C.c_float),
        ("philox_seed", C.c_uint64), ("philox_offset", C.c_uint64), ("philox_step_dev", VP),
        ("last_rows", VP), ("n_last_rows", C.c_int32), ("last_rows_nv_dev", VP), ("last_rows_hub", HubSplit), ("last_rows_out", VP),
        ("E0", VP), ("final_out", VP), ("cl_out", VP), ("work0", VP), ("work1", VP), ("x1", VP),
    ]


class ScatterSeg(C.Structure):
    _fields_ = [("src", VP), ("rows", VP), ("n_dev", VP), ("n", C.c_int32), ("row_off", C.c_int32), ("scale", C.c_float)]


class BprDesc(C.Structure):
    _fields_ = [
        ("emb", VP), ("l2_emb", VP), ("n_users", C.c_int32), ("d", C.c_int32),
        ("u_idx", VP), ("i_idx", VP), ("j_idx", VP), ("b_dev", VP), ("b", C.c_int32),
        ("emb_scale", C.c_float), ("reg", C.c_float), ("l2_terms", C.c_int32), ("l2_div", C.c_float),
        ("grad_scale", C.c_float), ("losses", VP), ("g_emb", VP), ("g_l2", VP), ("scratch", VP),
    ]


class InfoNceProblem(C.Structure):
    _fields_ = [
        ("table1", VP), ("table2", VP), ("row_off1", C.c_int32), ("row_off2", C.c_int32),
        ("scale1", C.c_float), ("scale2", C.c_float), ("idx", VP), ("n_dev", VP), ("n", C.c_int32),
        ("weight", C.c_float), ("g1", VP), ("g2", VP), ("loss", VP),
    ]


class InfoNceDesc(C.Structure):
    _fields_ = [
        ("n_problems", C.c_int32), ("d", C.c_int32), ("b_cos", C.c_int32), ("temperature", C.c_float),
        ("prob", InfoNceProblem * 4), ("workspace", VP), ("workspace_bytes", C.c_int64),
    ]


class TopkDesc(C.Structure):
    _fields_ = [
        ("user_emb", VP), ("item_emb", VP), ("n_items", C.c_int32), ("d", C.c_int32),
        ("users", VP), ("n_q", C.c_int32), ("rated_ptr", VP), ("rated_idx", VP), ("k", C.c_int32),
        ("out_ids", VP), ("out_scores", VP), ("impl", C.c_int32), ("workspace", VP),
        ("workspace_bytes", C.c_int64),
    ]


class GraphCsr(C.Structure):
    _fields_ = [("rowptr", VP), ("colidx", VP), ("vals", VP), ("row_order", VP), ("n_long_rows", C.c_int32), ("n_vlong_rows", C.c_int32),
                ("hub", HubSplit)]


class GraphAssembleDesc(C.Structure):
    _fields_ = [
        ("n_users", C.c_int32), ("n_items", C.c_int32), ("nnz", C.c_int64), ("ui_ptr", VP), ("ui_col", VP), ("ui_val", VP),
        ("iu_ptr", VP), ("iu_col", VP), ("iu_perm", VP), ("keep_flags", VP), ("keep_idx", VP), ("n_keep", C.c_int64),
        ("reset_weights", C.c_int32), ("dinv_table", VP), ("dinv_table_n", C.c_int32), ("rowptr", VP), ("colidx", VP),
        ("vals", VP), ("dinv", VP), ("out_cap", C.c_int64), ("nnz_out", VP), ("workspace", VP), ("workspace_bytes", C.c_int64),
    ]


class StepDesc(C.Structure):
    _fields_ = [
        ("model", C.c_int32), ("n_users", C.c_int32), ("n_items", C.c_int32), ("d", C.c_int32),
        ("n_layers", C.c_int32), ("batch_cap", C.c_int32), ("layer_cl", C.c_int32),
        ("eps", C.c_float), ("tau", C.c_float), ("cl_rate", C.c_float), ("reg", C.c_float),
        ("lr", C.c_double), ("beta1", C.c_double), ("beta2", C.c_double), ("adam_eps", C.c_float),
        ("l2_div", C.c_float), ("noise_mode", C.c_int32), ("noise", VP), ("philox_seed", C.c_uint64),
        ("adj", GraphCsr), ("adj_view", GraphCsr * 2), ("batch", VP), ("params", VP), ("adam_m", VP),
        ("adam_v", VP), ("step_dev", VP), ("scalars", VP), ("losses", VP), ("workspace", VP),
        ("workspace_bytes", C.c_int64), ("fork_stream", VP), ("fork_event", VP), ("join_event", VP),
    ]


class ShardDesc(C.Structure):
    _fields_ = [
        ("model", C.c_int32), ("world", C.c_int32), ("rank", C.c_int32), ("n_users", C.c_int32), ("n_items", C.c_int32),
        ("d", C.c_int32), ("n_layers", C.c_int32), ("batch_cap", C.c_int32), ("layer_cl", C.c_int32),
        ("eps", C.c_float), ("tau", C.c_float), ("cl_rate", C.c_float), ("reg", C.c_float),
        ("lr", C.c_double), ("beta1", C.c_double), ("beta2", C.c_double), ("adam_eps", C.c_float), ("l2_div", C.c_float),
        ("noise_mode", C.c_int32), ("philox_seed", C.c_uint64),
        ("Ru", GraphCsr), ("Rt", GraphCsr), ("batch", VP), ("pu", VP), ("mu", VP), ("vu", VP), ("mi", VP), ("vi", VP),
        ("step_dev", VP), ("scalars", VP), ("losses", VP), ("sym", VP * 8), ("sym_mc", VP), ("sym_bytes", C.c_int64),
        ("workspace", VP), ("workspace_bytes", C.c_int64), ("fork_stream", VP), ("fork_event", VP), ("join_event", VP),
        ("nvls", C.c_int32), ("Ru_view", GraphCsr * 2), ("Rt_view", GraphCsr * 2),
    ]


class ShardLayout(C.Structure):
    _fields_ = [("sym_bytes", C.c_int64), ("workspace_bytes", C.c_int64), ("item_params", C.c_int64), ("item_final", C.c_int64),
                ("ctrl", C.c_int64)]


class KnnRows(C.Structure):
    _fields_ = [("row_ptr", VP), ("row_idx", VP), ("t_ptr", VP), ("t_idx", VP), ("rank", VP), ("n_rows", C.c_int32)]


KNN_MAX_TOPK = 1024  # SRB_KNN_MAX_TOPK

MODEL_IDS = {"MF": 0, "LightGCN": 1, "SimGCL": 2, "XSimGCL": 3, "SGL": 4}
BATCH_HEADER = 4

# name -> (restype, argtypes); every symbol include/selfrec_b200.h declares
SYMBOLS = {
    "srb_last_error": (C.c_char_p, []),
    "srb_version": (C.c_int, []),
    "srb_launch_count": (C.c_int64, []),
    "srb_device_ok": (C.c_int, []),
    "srb_spmm_csr": (C.c_int, [C.POINTER(SpmmDesc), VP]),
    "srb_spmm_epilogue_rows": (C.c_int, [C.POINTER(SpmmDesc), VP]),
    "srb_encoder_forward": (C.c_int, [C.POINTER(EncoderDesc), VP]),
    "srb_bpr_l2_fwd_bwd": (C.c_int, [C.POINTER(BprDesc), VP]),
    "srb_infonce_workspace_bytes": (C.c_int64, [C.c_int32, C.c_int32, C.c_int32]),
    "srb_infonce_fwd_bwd": (C.c_int, [C.POINTER(InfoNceDesc), VP]),
    "srb_batch_softmax_fwd_bwd": (C.c_int, [C.POINTER(InfoNceDesc), VP]),
    "srb_l2_reg_fwd": (C.c_int, [C.c_int32, C.POINTER(VP), c_i64p, c_i32p, C.c_float, VP, VP, VP]),
    "srb_l2_reg_bwd": (C.c_int, [C.c_int32, C.POINTER(VP), C.POINTER(VP), c_i64p, c_i32p, C.c_float, VP, VP, VP]),
    "srb_scatter_add_rows": (C.c_int, [VP, C.c_int32, VP, VP, C.c_int32, VP, C.c_int32, C.c_float, VP]),
    "srb_scatter_add_segments": (C.c_int, [VP, C.c_int32, C.c_int32, VP, VP]),
    "srb_rank_hit_masks": (C.c_int, [VP, C.c_int32, C.c_int32, VP, VP, VP, VP, VP]),
    "srb_random_sample_range": (C.c_int, [VP, C.c_int64, C.c_int64, C.c_int32, VP]),
    "srb_dataset_load": (VP, [C.c_char_p, C.c_char_p]),
    "srb_dataset_free": (None, [VP]),
    "srb_dataset_counts": (C.c_int, [VP, VP]),
    "srb_dataset_names": (C.c_int, [VP, C.c_int32, VP, VP]),
    "srb_dataset_pairs": (C.c_int, [VP, C.c_int32, VP, VP, VP]),
    "srb_dataset_interaction_csr": (C.c_int, [VP, VP, VP, VP]),
    "srb_dataset_adjacency_csr": (C.c_int, [VP, VP, VP, VP, VP, VP]),
    "srb_bipartite_adjacency_csr": (C.c_int, [VP, VP, C.c_int64, C.c_int32, C.c_int32, VP, VP, VP, VP, VP]),
    "srb_graph_assemble_workspace_bytes": (C.c_int64, [C.c_int32, C.c_int32, C.c_int64]),
    "srb_graph_assemble": (C.c_int, [C.POINTER(GraphAssembleDesc), VP]),
    "srb_adam_prepare": (C.c_int, [VP, VP, C.c_double, C.c_double, C.c_double, VP]),
    "srb_adam_step": (C.c_int, [VP, VP, VP, VP, C.c_int64, VP, C.c_double, C.c_double, C.c_float, VP]),
    "srb_topk_workspace_bytes": (C.c_int64, [C.c_int32, C.c_int32, C.c_int32, C.c_int32]),
    "srb_topk_fallback_count_offset": (C.c_int64, [C.c_int32, C.c_int32]),
    "srb_topk_tc_error_bound": (C.c_float, [C.c_int32]),
    "srb_score_topk": (C.c_int, [C.POINTER(TopkDesc), VP]),
    "srb_score_rows": (C.c_int, [VP, VP, C.c_int32, VP, C.c_int32, C.c_int32, VP, VP]),
    "srb_topk_rows": (C.c_int, [VP, C.c_int32, C.c_int32, C.c_int32, VP, VP, VP]),
    "srb_step_workspace_bytes": (C.c_int64, [C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32]),
    "srb_train_step": (C.c_int, [C.POINTER(StepDesc), VP]),
    "srb_sampler_create": (VP, [c_i32p, c_i32p, C.c_int64, C.c_int32, C.c_int32]),
    "srb_sampler_destroy": (None, [VP]),
    "srb_sampler_set_state": (C.c_int, [VP, c_u32p]),
    "srb_sampler_get_state": (C.c_int, [VP, c_u32p]),
    "srb_sampler_begin_epoch": (C.c_int, [VP, c_i64p]),
    "srb_sampler_next_batch": (C.c_int, [VP, C.c_int32, C.c_int32, c_i32p]),
    "srb_sampler_next_batch_negs": (C.c_int, [VP, C.c_int32, C.c_int32, c_i32p, c_i32p, c_i32p]),
    "srb_sampler_epoch": (C.c_int64, [VP, C.c_int32, C.c_int32, c_i32p, C.c_int64]),
    "srb_sampler_pairs": (C.c_int64, [VP]),
    "srb_sampler_ring_start": (C.c_int, [VP, C.c_int32, C.c_int32, C.c_int32]),
    "srb_sampler_ring_pop": (C.c_int, [VP, c_i32p]),
    "srb_sampler_ring_stop": (C.c_int, [VP]),
    "srb_sampler_get_order": (C.c_int, [VP, c_i32p, c_i32p]),
    "srb_sampler_set_order": (C.c_int, [VP, c_i32p, c_i32p, C.c_int64]),
    "srb_sampler_cursor": (C.c_int, [VP, c_i64p]),
    "srb_sampler_seek": (C.c_int, [VP, C.c_int64]),
    "srb_shard_plan": (C.c_int, [C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32,
                                 C.POINTER(ShardLayout)]),
    "srb_shard_step": (C.c_int, [C.POINTER(ShardDesc), VP]),
    "srb_shard_forward": (C.c_int, [C.POINTER(ShardDesc), VP, VP]),
    "srb_knn_neighbors_workspace_bytes": (C.c_int64, [C.c_int32]),
    "srb_knn_neighbors": (C.c_int, [C.POINTER(KnnRows), C.c_int32, C.c_int64, VP, VP, VP, VP, C.c_int64, VP]),
    "srb_knn_score_rows": (C.c_int, [C.c_int32, VP, C.c_int32, C.c_int32, VP, VP, VP, C.c_int32, VP, VP, VP, VP, VP, VP]),
    "srb_topk_f64_workspace_bytes": (C.c_int64, [C.c_int32, C.c_int32]),
    "srb_topk_rows_f64": (C.c_int, [VP, C.c_int32, C.c_int32, C.c_int32, VP, VP, VP, C.c_int64, VP]),
}

_lib = None


def load():
    """Load libselfrec_b200.so (once).  Raises SrbError if it was never built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise SrbError(
            f"{LIB_PATH} is missing: build it with `python -m selfrec_b200.build` "
            "(or __graft_entry__.build()).  There is no CPU fallback."
        )
    lib = C.CDLL(LIB_PATH)
    for name, (res, args) in SYMBOLS.items():
        fn = getattr(lib, name)  # AttributeError if the library lacks a declared symbol
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


def last_error():
    return load().srb_last_error().decode("utf-8", "replace")


def check(rc, what=""):
    if rc != 0:
        raise SrbError(f"{what or 'selfrec_b200'} failed (rc={rc}): {last_error()}")


def require_device():
    """Raise unless a CUDA device is usable (no CPU fallback)."""
    lib = load()
    if lib.srb_device_ok() != 0:
        raise SrbError("selfrec_b200 needs a CUDA device (sm_90a): " + last_error())
    return lib


def launch_count():
    return int(load().srb_launch_count())
