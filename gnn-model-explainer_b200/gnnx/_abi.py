"""ctypes binding of libgnnx.so (include/gnnx.h).  No fallback: importing this module without
the built library raises, and creating an engine without a CUDA device raises."""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("GNNX_LIB_PATH") or os.path.join(_HERE, "lib", "libgnnx.so")   # GNNX_LIB_PATH: tools/ A-B builds of the same ABI

GX_OK = 0
GX_ERR_UNSUPPORTED = -3    # gx_status: valid in the reference but not built here
GX_HOST, GX_DEVICE = 0, 1
GX_INIT_M0, GX_INIT_PHILOX, GX_INIT_STATE = 0, 1, 2
GX_VERSION = 211
GX_TRACE_COLS = 8
TR_LOSS_EDGES, TR_PRED, TR_SIZE, TR_ENT, TR_LAP, TR_FEAT, TR_DENSITY, TR_PGT = range(8)
GX_MODEL_BN = 1
GX_MODEL_ATT = 2
GX_MAX_HEAD_LAYERS = 4

EXPORTS = [
    "gx_default_hparams", "gx_last_error", "gx_version", "gx_create", "gx_destroy", "gx_set_stream",
    "gx_sync", "gx_set_model", "gx_set_graph_csr", "gx_neighborhood_rows", "gx_plan_nodes",
    "gx_plan_fetch", "gx_explain_nodes", "gx_densify", "gx_launch_count", "gx_last_explain_ms",
    "gx_set_graph_batch_csr", "gx_plan_graphs", "gx_explain_graphs", "gx_grad_nodes", "gx_grad_graphs",
    "gx_explain_nodes_ex", "gx_explain_graphs_ex", "gx_offedge_regularisers", "gx_offedge_regularisers_graphs",
    "gx_debug_force_stream", "gx_debug_ieee_edge", "gx_debug_set_dump", "gx_debug_set_gang", "gx_debug_set_cluster", "gx_denoise_topk",
    "gx_model_forward", "gx_comm_unique_id", "gx_comm_init", "gx_comm_destroy", "gx_count_nodes", "gx_allgather_masks", "gx_unshard_masks",
    "gx_plan_class_counts", "gx_last_class_ms", "gx_explain_nodes_unconstrained", "gx_explain_graphs_unconstrained",
    "gx_set_model_att", "gx_set_model_head", "gx_count_graphs", "gx_densify_graphs", "gx_denoise_topk_edges",
]


class GxModelDims(C.Structure):
    _fields_ = [("input_dim", C.c_int32), ("hidden_dim", C.c_int32), ("embed_dim", C.c_int32),
                ("num_classes", C.c_int32), ("num_layers", C.c_int32), ("flags", C.c_int32)]


class GxHparams(C.Structure):
    _fields_ = [("num_epochs", C.c_int32), ("lr", C.c_float), ("beta1", C.c_float), ("beta2", C.c_float),
                ("eps", C.c_float), ("coef_size", C.c_float), ("coef_feat_size", C.c_float),
                ("coef_ent", C.c_float), ("coef_lap", C.c_float), ("mask_act", C.c_int32),
                ("mask_bias", C.c_int32), ("init", C.c_int32), ("seed", C.c_uint64),
                ("start_step", C.c_int32), ("opt", C.c_int32), ("opt_scheduler", C.c_int32), ("opt_decay_step", C.c_int32),
                ("opt_decay_rate", C.c_float), ("opt_restart", C.c_int32)]


GX_OPT = {"adam": 0, "sgd": 1, "rmsprop": 2, "adagrad": 3}
GX_SCHED = {"none": 0, "step": 1, "cos": 2}


class GxExplainIo(C.Structure):
    """include/gnnx.h gx_explain_io: optional trace / optimiser-state buffers (all void* here; 0 = unused)."""
    _fields_ = [(n, C.c_void_p) for n in (
        "m0_edges", "edge_mask", "feat_mask", "trace", "trace_pred", "adam_m_in", "adam_v_in", "feat_state_in",
        "mask_param_out", "adam_m_out", "adam_v_out", "feat_state_out")]


class GnnxError(RuntimeError):
    def __init__(self, status, message):
        super().__init__("libgnnx status %d: %s" % (status, message))
        self.status = status


_lib = None


def lib():
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise ImportError(
            "libgnnx.so not found at %s -- build it with `python __graft_entry__.py` "
            "(or gnn-model-explainer_b200/csrc/build.sh); there is no CPU fallback" % LIB_PATH)
    L = C.CDLL(LIB_PATH)
    vp, i32p, i64p, f32p = C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p
    L.gx_last_error.restype = C.c_char_p
    L.gx_version.restype = C.c_int
    L.gx_default_hparams.argtypes = [C.POINTER(GxHparams)]
    L.gx_default_hparams.restype = None
    L.gx_create.argtypes = [C.c_int, C.POINTER(vp)]
    L.gx_destroy.argtypes = [vp]
    L.gx_set_stream.argtypes = [vp, vp]
    L.gx_sync.argtypes = [vp]
    L.gx_set_model.argtypes = [vp, C.POINTER(GxModelDims), C.POINTER(vp), C.POINTER(vp), f32p, f32p]
    L.gx_set_model_att.argtypes = [vp, C.POINTER(GxModelDims), C.POINTER(vp), C.POINTER(vp), C.POINTER(vp), f32p, f32p]
    L.gx_set_model_head.argtypes = [vp, C.POINTER(GxModelDims), C.POINTER(vp), C.POINTER(vp), C.POINTER(vp), C.c_int32, i32p, C.POINTER(vp),
                                    C.POINTER(vp)]
    L.gx_set_graph_csr.argtypes = [vp, C.c_int64, i32p, i32p, f32p, C.c_int32, i32p, i32p]
    L.gx_neighborhood_rows.argtypes = [vp, i32p, C.c_int32, C.c_int32, vp]
    L.gx_plan_nodes.argtypes = [vp, i32p, C.c_int32, C.c_int32, C.POINTER(C.c_int64), C.POINTER(C.c_int64)]
    L.gx_plan_fetch.argtypes = [vp, i64p, i64p, i32p, i32p, i32p, i32p]
    L.gx_explain_nodes.argtypes = [vp, C.POINTER(GxHparams), C.c_int, f32p, f32p, f32p]
    L.gx_densify.argtypes = [vp, C.c_int, f32p, vp]
    L.gx_set_graph_batch_csr.argtypes = [vp, C.c_int32, C.c_int32, i32p, i32p, f32p, C.c_int32, i32p]
    L.gx_plan_graphs.argtypes = [vp, i32p, C.c_int32, i64p, C.POINTER(C.c_int64)]
    L.gx_explain_graphs.argtypes = [vp, C.POINTER(GxHparams), C.c_int, f32p, f32p, f32p]
    L.gx_explain_nodes_ex.argtypes = [vp, C.POINTER(GxHparams), C.c_int, C.POINTER(GxExplainIo)]
    L.gx_explain_graphs_ex.argtypes = [vp, C.POINTER(GxHparams), C.c_int, C.POINTER(GxExplainIo)]
    L.gx_explain_nodes_unconstrained.argtypes = [vp, C.POINTER(GxHparams), C.c_int, f32p, f32p, f32p, f32p, f32p]
    L.gx_explain_graphs_unconstrained.argtypes = [vp, C.POINTER(GxHparams), C.c_int, f32p, f32p, f32p, f32p, f32p]
    L.gx_offedge_regularisers.argtypes = [vp, C.POINTER(GxHparams), C.c_int, f32p, vp]
    L.gx_offedge_regularisers_graphs.argtypes = [vp, C.POINTER(GxHparams), C.c_int, f32p, vp]
    L.gx_grad_nodes.argtypes = [vp, C.c_int, f32p]
    L.gx_grad_graphs.argtypes = [vp, C.c_int, i32p, f32p]
    L.gx_denoise_topk.argtypes = [vp, C.c_int, f32p, C.c_int32, C.c_int32, f32p, i32p, i32p, f32p]
    L.gx_denoise_topk_edges.argtypes = [vp, C.c_int, f32p, C.c_int32, C.c_int32, f32p, i32p, i32p, f32p]
    L.gx_comm_unique_id.argtypes = [C.c_char_p]
    L.gx_comm_init.argtypes = [vp, C.c_int32, C.c_int32, C.c_char_p]
    L.gx_comm_destroy.argtypes = [vp]
    L.gx_count_nodes.argtypes = [vp, i32p, C.c_int32, C.c_int32, i32p, i32p]
    L.gx_allgather_masks.argtypes = [vp, f32p, C.c_int64, C.c_int64, f32p]
    L.gx_unshard_masks.argtypes = [vp, f32p, C.c_int32, i64p, i64p, i32p, f32p]
    L.gx_count_graphs.argtypes = [vp, i32p, C.c_int32, i32p, i32p]
    L.gx_densify_graphs.argtypes = [vp, C.c_int, i32p, C.c_int32, f32p, vp]
    L.gx_debug_force_stream.argtypes = [vp, C.c_int]
    L.gx_debug_ieee_edge.argtypes = [vp, C.c_int]
    L.gx_debug_set_dump.argtypes = [vp, vp]
    L.gx_model_forward.argtypes = [vp, C.c_int, f32p]
    L.gx_debug_set_gang.argtypes = [vp, C.c_int]
    L.gx_debug_set_cluster.argtypes = [vp, C.c_int, C.c_int64]
    L.gx_launch_count.argtypes = [vp]
    L.gx_plan_class_counts.argtypes = [vp, i32p, i32p, i32p]
    L.gx_last_class_ms.argtypes = [vp, f32p, f32p]
    L.gx_launch_count.restype = C.c_int64
    L.gx_last_explain_ms.argtypes = [vp, C.POINTER(C.c_float)]
    for name in EXPORTS:
        getattr(L, name)  # AttributeError here means the library does not match include/gnnx.h
    if L.gx_version() != GX_VERSION:
        raise ImportError("libgnnx.so is version %d, this binding expects %d -- rebuild (python __graft_entry__.py)" % (L.gx_version(), GX_VERSION))
    _lib = L
    return L


def check(status):
    if status != GX_OK:
        raise GnnxError(status, lib().gx_last_error().decode("utf-8", "replace"))
