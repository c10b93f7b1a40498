"""ctypes binding of libadaptive_b200.so (the C ABI declared in include/adaptive_b200.h).

This is the binding a maintainer of the reference would add (INTEGRATION.md).  PyTorch is used only for
device memory and streams: every call passes raw device pointers + the current CUDA stream.
There is NO CPU fallback: a missing library raises ImportError-like RuntimeError, a missing sm_90 (H100) device
makes every compute call raise AdaptiveB200Error.
"""
from __future__ import annotations

import ctypes
import math
import threading
import os
from ctypes import POINTER, Structure, c_char_p, c_float, c_int, c_int64, c_size_t, c_uint64, c_void_p
from typing import Optional, Tuple

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libadaptive_b200.so")

AC_KNN_AUTO, AC_KNN_EXACT, AC_KNN_TENSOR = 0, 1, 2
AC_KNN_MAX_K = 2048
AC_KNN_TENSOR_MAX_K = 1024
AC_ACT_LOGITS, AC_ACT_SOFTMAX, AC_ACT_SIGMOID = 0, 1, 2
AC_LOSS_CE, AC_LOSS_BCE, AC_LOSS_CE_STRATEGIC = 0, 1, 2
AC_COST_LINEAR, AC_COST_SEPARABLE = 0, 1
AC_STRATEGIC_CANDIDATES = 50
AC_ARCH_BERT, AC_ARCH_ROBERTA, AC_ARCH_MODERNBERT, AC_ARCH_MPNET, AC_ARCH_DEBERTA, AC_ARCH_ROTARY = 0, 1, 2, 3, 4, 5
AC_ARCH_EUROBERT = 6
AC_ENCODER_MAX_S = 512
AC_MODERNBERT_MAX_S = 8192
AC_PREC_TF32, AC_PREC_F16 = 0, 1
AC_FFN_GELU_ERF, AC_FFN_GELU_TANH, AC_FFN_SWIGLU = 0, 1, 2
AC_PROJ_EMB, AC_PROJ_QKV, AC_PROJ_WO, AC_PROJ_FFN1, AC_PROJ_W2, AC_PROJ_FFN1_ROWS = 0, 1, 2, 3, 4, 5
_PROJ_ROLES = {0: "AC_PROJ_EMB", 1: "AC_PROJ_QKV", 2: "AC_PROJ_WO", 3: "AC_PROJ_FFN1", 4: "AC_PROJ_W2",
               5: "AC_PROJ_FFN1_ROWS"}
# hidden_act of a post-LN (BERT-family) config -> ac_encoder_config.ffn_act (SwiGLU is NomicBERT's alone: nomic_bert_settings)
FFN_ACTS = {"gelu": AC_FFN_GELU_ERF, "gelu_new": AC_FFN_GELU_TANH, "gelu_pytorch_tanh": AC_FFN_GELU_TANH}

EXPORTS = [
    "ac_version", "ac_last_error", "ac_device_check",
    "ac_knn_workspace_bytes", "ac_knn_l2_topk", "ac_knn_make_shadow", "ac_row_sqnorm", "ac_topk_merge", "ac_proto_scores",
    "ac_segment_mean", "ac_memory_append_prune",
    "ac_head_forward", "ac_head_train_workspace_bytes", "ac_head_train_step", "ac_head_train_epoch", "ac_head_phase_timing", "ac_head_train_plan", "ac_head_grad", "ac_ewc_penalty",
    "ac_strategic_workspace_bytes", "ac_strategic_best_response", "ac_head_train_strategic_workspace_bytes", "ac_head_train_strategic",
    "ac_encoder_create", "ac_encoder_destroy", "ac_encoder_forward_cls", "ac_encoder_last_hidden", "ac_encoder_attention",
    "ac_encoder_projection",
    "ac_linear_tc",
    "ac_proto_class_scores", "ac_proto_class_scores_n", "ac_blend_dense", "ac_topk_desc_workspace_bytes", "ac_topk_desc", "ac_blend_topk",
    "ac_pipeline_create", "ac_pipeline_destroy", "ac_pipeline_predict_device", "ac_pipeline_predict_host",
    "ac_pipeline_encode", "ac_pipeline_embeddings", "ac_pipeline_search_shard", "ac_pipeline_finish_sharded",
    "ac_pipeline_debug_copy", "ac_pipeline_knn_stats", "ac_launch_count", "ac_profile_enable", "ac_profile_read",
    "ac_tokenizer_create", "ac_tokenizer_destroy", "ac_tokenize_workspace_bytes", "ac_tokenize", "ac_tokenize_pack",
    "ac_tokenizer_create_bpe", "ac_tokenize_workspace_bytes_text", "ac_tokenizer_create_unigram",
]


class AdaptiveB200Error(RuntimeError):
    pass


class HeadParams(Structure):
    _fields_ = [("D", c_int), ("H0", c_int), ("H1", c_int), ("C", c_int),
                ("W0", c_void_p), ("b0", c_void_p), ("W1", c_void_p), ("b1", c_void_p),
                ("W2", c_void_p), ("b2", c_void_p)]


class TrainCfg(Structure):
    _fields_ = [("lr", c_float), ("beta1", c_float), ("beta2", c_float), ("eps", c_float),
                ("weight_decay", c_float), ("max_norm", c_float),
                ("step", c_int), ("loss_kind", c_int), ("dropout_p", c_float),
                ("mask0", c_void_p), ("mask1", c_void_p), ("seed", c_uint64),
                ("ewc_fisher", POINTER(HeadParams)), ("ewc_star", POINTER(HeadParams)),
                ("ewc_lambda", c_float), ("ewc_C_old", c_int),
                ("n_regular", c_int), ("strategic_lambda", c_float)]


class StrategicCfg(Structure):
    _fields_ = [("cost_kind", c_int), ("c1", c_void_p), ("c2", c_void_p), ("delta", c_float * 10),
                ("dropout_p", c_float), ("seed", c_uint64), ("step", c_int)]


class EncoderConfig(Structure):
    _fields_ = [("arch", c_int), ("layers", c_int), ("hidden", c_int), ("heads", c_int), ("intermediate", c_int),
                ("vocab", c_int), ("max_pos", c_int), ("type_vocab", c_int), ("pad_idx", c_int),
                ("ln_eps", c_float), ("precision", c_int), ("max_tokens", c_int), ("cls_only", c_int),
                ("sliding_window", c_int), ("layer_sliding", POINTER(ctypes.c_int32)),
                ("rope_full", c_void_p), ("rope_sliding", c_void_p), ("rel_bias", c_void_p),
                ("pos_key", c_void_p), ("pos_query", c_void_p), ("pos_span", c_int), ("rel_index", c_void_p),
                ("embedding_size", c_int), ("ffn_act", c_int), ("rel_radius", c_int)]


_PP = POINTER(c_void_p)


class TokenizerSpec(Structure):
    _fields_ = [("norm", c_void_p), ("cls", c_void_p), ("pool", c_void_p), ("pool_len", c_int64),
                ("vocab_bytes", c_void_p), ("vocab_offsets", c_void_p), ("vocab_ids", c_void_p), ("n_vocab", c_int),
                ("added_bytes", c_void_p), ("added_offsets", c_void_p), ("added_ids", c_void_p), ("n_added", c_int),
                ("prefix", c_char_p), ("prefix_len", c_int),
                ("cls_id", c_int), ("sep_id", c_int), ("pad_id", c_int), ("unk_id", c_int), ("max_input_chars", c_int)]


class BPETokenizerSpec(Structure):
    _fields_ = [("cls", c_void_p), ("split", c_int), ("add_prefix_space", c_int), ("ignore_merges", c_int),
                ("vocab_bytes", c_void_p), ("vocab_offsets", c_void_p), ("vocab_ids", c_void_p), ("n_vocab", c_int),
                ("byte_ids", c_void_p), ("merges", c_void_p), ("n_merges", c_int),
                ("added_bytes", c_void_p), ("added_offsets", c_void_p), ("added_ids", c_void_p), ("added_flags", c_void_p),
                ("n_added", c_int), ("cls_id", c_int), ("sep_id", c_int), ("pad_id", c_int)]


class UnigramTokenizerSpec(Structure):
    _fields_ = [("cls", c_void_p), ("map_keys", c_void_p), ("map_key_offsets", c_void_p), ("map_values", c_void_p),
                ("map_value_offsets", c_void_p), ("n_map", c_int), ("grow", c_int),
                ("piece_bytes", c_void_p), ("piece_offsets", c_void_p), ("piece_scores", c_void_p), ("n_pieces", c_int),
                ("unk_id", c_int),
                ("added_bytes", c_void_p), ("added_offsets", c_void_p), ("added_ids", c_void_p), ("added_flags", c_void_p),
                ("n_added", c_int), ("cls_id", c_int), ("sep_id", c_int), ("pad_id", c_int)]


class EncoderWeights(Structure):
    _fields_ = [("word_emb", c_void_p), ("pos_emb", c_void_p), ("type_emb", c_void_p),
                ("emb_ln_w", c_void_p), ("emb_ln_b", c_void_p),
                ("q_w", _PP), ("q_b", _PP), ("k_w", _PP), ("k_b", _PP), ("v_w", _PP), ("v_b", _PP),
                ("ao_w", _PP), ("ao_b", _PP), ("ao_ln_w", _PP), ("ao_ln_b", _PP),
                ("ff1_w", _PP), ("ff1_b", _PP), ("ff2_w", _PP), ("ff2_b", _PP),
                ("out_ln_w", _PP), ("out_ln_b", _PP),
                ("attn_norm_w", _PP), ("final_norm_w", c_void_p), ("wqkv", _PP), ("wi", _PP),
                ("emb_proj_w", c_void_p), ("emb_proj_b", c_void_p)]


_lib = None


def load_library() -> ctypes.CDLL:
    """Load the shared library and declare signatures.  Needs no GPU (symbol check only)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise AdaptiveB200Error(
            f"{LIB_PATH} is missing: build it with `python -m adaptive_classifier_b200.build` "
            "(adaptive_classifier_b200 has no CPU or PyTorch fallback)")
    L = ctypes.CDLL(LIB_PATH)
    L.ac_version.restype = c_int
    L.ac_last_error.restype = c_char_p
    L.ac_device_check.restype = c_int
    L.ac_knn_workspace_bytes.argtypes = [c_int, c_int64, c_int, c_int, c_int, POINTER(c_size_t)]
    L.ac_knn_l2_topk.argtypes = [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int64, c_int, c_int, c_void_p, c_void_p,
                                 c_int64, c_void_p, c_size_t, c_int, c_void_p, c_void_p]
    L.ac_knn_make_shadow.argtypes = [c_void_p, c_int64, c_int, c_void_p, c_void_p]
    L.ac_row_sqnorm.argtypes = [c_void_p, c_int64, c_int, c_void_p, c_void_p]
    L.ac_topk_merge.argtypes = [c_void_p, c_void_p, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p]
    L.ac_proto_scores.argtypes = [c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p]
    L.ac_segment_mean.argtypes = [c_void_p, c_void_p, c_int64, c_int, c_int, c_void_p, c_void_p, c_void_p]
    L.ac_memory_append_prune.argtypes = [c_void_p, c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_int,
                                         c_void_p, c_void_p, c_void_p, c_size_t, c_void_p]
    L.ac_head_forward.argtypes = [c_void_p, c_int, POINTER(HeadParams), c_int, c_void_p, c_void_p, c_size_t, c_void_p]
    L.ac_head_train_workspace_bytes.argtypes = [c_int, c_int, POINTER(HeadParams), POINTER(c_size_t)]
    L.ac_head_train_step.argtypes = [c_void_p, c_void_p, c_int, POINTER(HeadParams), POINTER(HeadParams),
                                     POINTER(HeadParams), POINTER(TrainCfg), c_void_p, c_void_p, c_size_t, c_void_p]
    L.ac_head_train_epoch.argtypes = [c_void_p, c_void_p, c_void_p, c_int, c_int, POINTER(HeadParams), POINTER(HeadParams),
                                      POINTER(HeadParams), POINTER(TrainCfg), c_void_p, c_void_p, c_void_p, c_size_t, c_void_p]
    L.ac_head_grad.argtypes = [c_void_p, c_void_p, c_int, POINTER(HeadParams), c_int, POINTER(HeadParams),
                               POINTER(HeadParams), c_float, c_void_p, c_void_p, c_size_t, c_void_p]
    L.ac_ewc_penalty.argtypes = [POINTER(HeadParams), POINTER(HeadParams), POINTER(HeadParams), c_float, c_float,
                                 c_int, c_void_p, c_void_p]
    L.ac_strategic_workspace_bytes.argtypes = [c_int, POINTER(HeadParams), POINTER(c_size_t)]
    L.ac_strategic_best_response.argtypes = [c_void_p, c_int, POINTER(HeadParams), POINTER(StrategicCfg), c_void_p, c_void_p,
                                             c_void_p, c_void_p, c_size_t, c_void_p]
    L.ac_head_train_strategic_workspace_bytes.argtypes = [c_int, POINTER(HeadParams), POINTER(c_size_t)]
    L.ac_head_train_strategic.argtypes = [c_void_p, c_void_p, c_void_p, c_int, c_int, POINTER(HeadParams), POINTER(HeadParams),
                                          POINTER(HeadParams), POINTER(TrainCfg), POINTER(StrategicCfg), c_void_p, c_void_p,
                                          c_size_t, c_void_p]
    L.ac_encoder_create.argtypes = [POINTER(EncoderConfig), POINTER(EncoderWeights), POINTER(c_void_p)]
    L.ac_encoder_destroy.argtypes = [c_void_p]
    L.ac_encoder_forward_cls.argtypes = [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p]
    L.ac_encoder_last_hidden.argtypes = [c_void_p, c_void_p, c_int64, c_void_p]
    L.ac_encoder_attention.argtypes = [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p]
    L.ac_encoder_projection.argtypes = [c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p,
                                        c_void_p, c_void_p, c_void_p]
    L.ac_linear_tc.argtypes = [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int,
                               c_int, c_int, c_void_p]
    L.ac_proto_class_scores.argtypes = [c_void_p, c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p, c_void_p]
    L.ac_proto_class_scores_n.argtypes = [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p]
    L.ac_blend_dense.argtypes = [c_void_p, c_void_p, c_int, c_void_p, c_int, c_int, c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_void_p]
    L.ac_topk_desc_workspace_bytes.argtypes = [c_int, c_int, c_int, POINTER(c_size_t)]
    L.ac_topk_desc.argtypes = [c_void_p, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p, c_size_t, c_void_p]
    L.ac_blend_topk.argtypes = [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_float, c_float,
                                c_void_p, c_void_p, c_void_p]
    L.ac_pipeline_create.argtypes = [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int64, c_int, POINTER(HeadParams),
                                     c_int, c_int, c_int, c_int64, c_int, POINTER(c_void_p)]
    L.ac_pipeline_encode.argtypes = [c_void_p, c_void_p, c_void_p, c_int, c_void_p]
    L.ac_pipeline_embeddings.argtypes = [c_void_p, POINTER(c_void_p)]
    L.ac_pipeline_search_shard.argtypes = [c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p]
    L.ac_pipeline_finish_sharded.argtypes = [c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p, c_void_p]
    L.ac_pipeline_destroy.argtypes = [c_void_p]
    L.ac_pipeline_predict_device.argtypes = [c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_void_p]
    L.ac_pipeline_predict_host.argtypes = [c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_void_p]
    L.ac_pipeline_debug_copy.argtypes = [c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_void_p]
    L.ac_profile_enable.argtypes = [c_int]
    L.ac_tokenizer_create.argtypes = [POINTER(TokenizerSpec), POINTER(c_void_p)]
    L.ac_tokenizer_destroy.argtypes = [c_void_p]
    L.ac_tokenize_workspace_bytes.argtypes = [c_void_p, c_int, POINTER(c_size_t)]
    L.ac_tokenize.argtypes = [c_void_p, c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_size_t,
                              c_void_p]
    L.ac_tokenize_pack.argtypes = [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p]
    L.ac_tokenizer_create_bpe.argtypes = [POINTER(BPETokenizerSpec), POINTER(c_void_p)]
    L.ac_tokenize_workspace_bytes_text.argtypes = [c_void_p, c_int, c_int64, c_int, POINTER(c_size_t)]
    L.ac_tokenizer_create_unigram.argtypes = [POINTER(UnigramTokenizerSpec), POINTER(c_void_p)]
    L.ac_pipeline_knn_stats.argtypes = [c_void_p, c_void_p, c_int, c_void_p]
    L.ac_profile_read.argtypes = [c_int, POINTER(ctypes.c_double), POINTER(ctypes.c_double), POINTER(ctypes.c_double),
                                  POINTER(ctypes.c_longlong)]
    for name in EXPORTS:
        fn = getattr(L, name)
        if name == "ac_launch_count":
            fn.restype = ctypes.c_longlong
        elif name not in ("ac_last_error",):
            fn.restype = c_int
    _lib = L
    return L


def check(rc: int, what: str = ""):
    if rc != 0:
        msg = load_library().ac_last_error()
        raise AdaptiveB200Error(f"{what} failed (rc={rc}): {msg.decode() if msg else ''}")


def stream_ptr() -> int:
    return torch.cuda.current_stream().cuda_stream


def ptr(t: Optional[torch.Tensor]) -> Optional[int]:
    return None if t is None else t.data_ptr()


def _f32c(t: torch.Tensor) -> torch.Tensor:
    assert t.is_cuda and t.dtype == torch.float32, "expected a CUDA fp32 tensor"
    return t.contiguous()


# ------------------------------------------------------------------------------------------------
# thin Python wrappers (tensor in / tensor out) used by the drop-in classes, the tests and bench.py
# ------------------------------------------------------------------------------------------------
_ws_tls = threading.local()


def _workspace(nbytes: int, device) -> torch.Tensor:
    """Scratch for one C call, cached per (thread, device).  Per THREAD because ctypes releases the GIL: two host threads (e.g. one
    inside PrototypeMemory's lock running a search, one inside a classifier's device lock running the head) enqueue on the same
    stream, and a scratch buffer shared between them would be rewritten between two kernels of the other thread's call."""
    cache = getattr(_ws_tls, "ws", None)
    if cache is None:
        cache = _ws_tls.ws = {}
    key = (device.index if device.index is not None else torch.cuda.current_device())
    ws = cache.get(key)
    if ws is None or ws.numel() < nbytes:
        ws = torch.empty(int(nbytes * 1.25) + 1024, dtype=torch.uint8, device=device)
        cache[key] = ws
    return ws


def knn_make_shadow(P: torch.Tensor) -> torch.Tensor:
    """fp16 (RNE) shadow of the prototype matrix for the tensor path's coarse pass"""
    L = load_library()
    P = _f32c(P)
    out = torch.empty(P.shape, dtype=torch.float16, device=P.device)
    check(L.ac_knn_make_shadow(P.data_ptr(), P.shape[0], P.shape[1], out.data_ptr(), stream_ptr()), "ac_knn_make_shadow")
    return out


def knn_l2_topk(Q: torch.Tensor, P: torch.Tensor, k: int, *, p_sqnorm: Optional[torch.Tensor] = None,
                p_half: Optional[torch.Tensor] = None, row_offset: int = 0, algo: int = AC_KNN_AUTO,
                stats: Optional[torch.Tensor] = None):
    """stats: optional CUDA int32[4] accumulator (see ac_knn_l2_topk): with it the call never synchronises and the CALLER must
    check stats[1] (buffer overflow -> redo those queries with AC_KNN_EXACT); without it the library does both itself."""
    L = load_library()
    Q = _f32c(Q)
    P = _f32c(P)
    B, D = Q.shape
    N = P.shape[0]
    assert P.shape[1] == D
    nbytes = c_size_t(0)
    check(L.ac_knn_workspace_bytes(B, N, D, k, algo, ctypes.byref(nbytes)), "ac_knn_workspace_bytes")
    ws = _workspace(nbytes.value, Q.device)
    out_d = torch.empty((B, k), dtype=torch.float32, device=Q.device)
    out_i = torch.empty((B, k), dtype=torch.int64, device=Q.device)
    check(L.ac_knn_l2_topk(Q.data_ptr(), P.data_ptr(), ptr(p_sqnorm), ptr(p_half), B, N, D, k, out_d.data_ptr(),
                           out_i.data_ptr(), row_offset, ws.data_ptr(), ws.numel(), algo, ptr(stats), stream_ptr()), "ac_knn_l2_topk")
    return out_d, out_i


def row_sqnorm(P: torch.Tensor) -> torch.Tensor:
    L = load_library()
    P = _f32c(P)
    out = torch.empty((P.shape[0],), dtype=torch.float32, device=P.device)
    check(L.ac_row_sqnorm(P.data_ptr(), P.shape[0], P.shape[1], out.data_ptr(), stream_ptr()), "ac_row_sqnorm")
    return out


def topk_merge(d: torch.Tensor, i: torch.Tensor):
    L = load_library()
    d = _f32c(d)
    i = i.contiguous()
    G, B, k = d.shape
    od = torch.empty((B, k), dtype=torch.float32, device=d.device)
    oi = torch.empty((B, k), dtype=torch.int64, device=d.device)
    check(L.ac_topk_merge(d.data_ptr(), i.data_ptr(), G, B, k, od.data_ptr(), oi.data_ptr(), stream_ptr()), "ac_topk_merge")
    return od, oi


def proto_scores(d: torch.Tensor, idx: Optional[torch.Tensor]) -> torch.Tensor:
    L = load_library()
    d = _f32c(d)
    B, k = d.shape
    out = torch.empty_like(d)
    check(L.ac_proto_scores(d.data_ptr(), ptr(idx.contiguous() if idx is not None else None), B, k, out.data_ptr(),
                            stream_ptr()), "ac_proto_scores")
    return out


def segment_mean(X: torch.Tensor, cls: torch.Tensor, C: int):
    L = load_library()
    X = _f32c(X)
    cls = cls.to(torch.int32).contiguous()
    n, D = X.shape
    mean = torch.zeros((C, D), dtype=torch.float32, device=X.device)
    cnt = torch.zeros((C,), dtype=torch.int32, device=X.device)
    check(L.ac_segment_mean(X.data_ptr(), cls.data_ptr(), n, D, C, mean.data_ptr(), cnt.data_ptr(), stream_ptr()),
          "ac_segment_mean")
    return mean, cnt


def memory_append_prune(rows, order, count, new_rows, new_index, cls_start, touched):
    """rows [n_slots, cap+1, D], order [n_slots, cap+1] int32, count [n_slots] int32 (updated in place) ->
    (src [n_touched, cap] int32, proto [n_touched, D] fp32): see ac_memory_append_prune"""
    L = load_library()
    n_slots, cap1, D = rows.shape
    nt = touched.numel()
    src = torch.empty((nt, cap1 - 1), dtype=torch.int32, device=rows.device)
    proto = torch.empty((nt, D), dtype=torch.float32, device=rows.device)
    ws = _workspace(nt * D * 8 + 256, rows.device)
    check(L.ac_memory_append_prune(rows.data_ptr(), order.data_ptr(), count.data_ptr(), cap1 - 1, D, _f32c(new_rows).data_ptr(),
                                   new_index.data_ptr(), cls_start.data_ptr(), touched.data_ptr(), nt, src.data_ptr(), proto.data_ptr(),
                                   ws.data_ptr(), ws.numel(), stream_ptr()), "ac_memory_append_prune")
    return src, proto


def head_params_struct(p: dict) -> HeadParams:
    """p: {'W0','b0','W1','b1','W2','b2'} CUDA fp32 contiguous tensors (nn.Linear layout)."""
    hp = HeadParams()
    hp.D = p["W0"].shape[1]
    hp.H0 = p["W0"].shape[0]
    hp.H1 = p["W1"].shape[0]
    hp.C = p["W2"].shape[0]
    for n in ("W0", "b0", "W1", "b1", "W2", "b2"):
        t = p[n]
        assert t.is_cuda and t.dtype == torch.float32 and t.is_contiguous(), n
        setattr(hp, n, t.data_ptr())
    return hp


def head_forward(X: torch.Tensor, p: dict, act: int = AC_ACT_LOGITS) -> torch.Tensor:
    L = load_library()
    X = _f32c(X)
    hp = head_params_struct(p)
    B = X.shape[0]
    out = torch.empty((B, hp.C), dtype=torch.float32, device=X.device)
    scratch = torch.empty((B * (hp.H0 + hp.H1),), dtype=torch.float32, device=X.device)
    check(L.ac_head_forward(X.data_ptr(), B, ctypes.byref(hp), act, out.data_ptr(), scratch.data_ptr(),
                            scratch.numel(), stream_ptr()), "ac_head_forward")
    return out


def head_train_step(X, targets, p, m, v, *, step, loss_kind=AC_LOSS_CE, lr=1e-3, betas=(0.9, 0.999), eps=1e-8,
                    weight_decay=0.01, max_norm=1.0, dropout_p=0.1, masks=None, seed=0,
                    ewc=None, out_stats=None, n_regular=0, strategic_lambda=0.0):
    """One optimizer step in place on p/m/v.  ewc = (fisher_dict, star_dict, lambda, C_old) or None.
    loss_kind=AC_LOSS_CE_STRATEGIC: X = [x ; br] with n_regular rows each, targets repeated.
    Returns the device tensor [task_loss, ewc_penalty, grad_norm]."""
    L = load_library()
    X = _f32c(X)
    B = X.shape[0]
    hp, hm, hv = head_params_struct(p), head_params_struct(m), head_params_struct(v)
    cfg = TrainCfg()
    cfg.lr, cfg.beta1, cfg.beta2, cfg.eps = lr, betas[0], betas[1], eps
    cfg.weight_decay, cfg.max_norm = weight_decay, max_norm
    cfg.step, cfg.loss_kind, cfg.dropout_p, cfg.seed = step, loss_kind, dropout_p, seed
    cfg.n_regular, cfg.strategic_lambda = int(n_regular), float(strategic_lambda)
    keep = []
    if masks is not None:
        m0, m1 = _f32c(masks[0]), _f32c(masks[1])
        keep += [m0, m1]
        cfg.mask0, cfg.mask1 = m0.data_ptr(), m1.data_ptr()
    if ewc is not None:
        fs, ss = head_params_struct(ewc[0]), head_params_struct(ewc[1])
        keep += [fs, ss]
        cfg.ewc_fisher, cfg.ewc_star = ctypes.pointer(fs), ctypes.pointer(ss)
        cfg.ewc_lambda, cfg.ewc_C_old = float(ewc[2]), int(ewc[3])
    nbytes = c_size_t(0)
    check(L.ac_head_train_workspace_bytes(B, 1, ctypes.byref(hp), ctypes.byref(nbytes)), "ac_head_train_workspace_bytes")
    ws = _workspace(nbytes.value, X.device)
    if out_stats is None:
        out_stats = torch.zeros((4,), dtype=torch.float32, device=X.device)
    targets = targets.contiguous()
    check(L.ac_head_train_step(X.data_ptr(), targets.data_ptr(), B, ctypes.byref(hp), ctypes.byref(hm),
                               ctypes.byref(hv), ctypes.byref(cfg), out_stats.data_ptr(), ws.data_ptr(), ws.numel(),
                               stream_ptr()), "ac_head_train_step")
    return out_stats


def head_train_epoch(X, targets, perm, p, m, v, *, first_step, batch, loss_kind=AC_LOSS_CE, lr=1e-3, betas=(0.9, 0.999),
                     eps=1e-8, weight_decay=0.01, max_norm=1.0, dropout_p=0.1, seed=0, ewc=None, loss_accum=None,
                     step_stats=None):
    """All optimizer steps of one epoch in ONE kernel launch (batches gathered on the device from `perm`).
    step_stats: optional CUDA fp32 [steps, 3] receiving (task loss, EWC penalty, grad norm) of every step.
    Returns (loss_accum tensor, steps)."""
    L = load_library()
    X = _f32c(X)
    n = X.shape[0]
    hp, hm, hv = head_params_struct(p), head_params_struct(m), head_params_struct(v)
    cfg = TrainCfg()
    cfg.lr, cfg.beta1, cfg.beta2, cfg.eps = lr, betas[0], betas[1], eps
    cfg.weight_decay, cfg.max_norm = weight_decay, max_norm
    cfg.step, cfg.loss_kind, cfg.dropout_p, cfg.seed = first_step, loss_kind, dropout_p, seed
    keep = []
    if ewc is not None:
        fs, ss = head_params_struct(ewc[0]), head_params_struct(ewc[1])
        keep += [fs, ss]
        cfg.ewc_fisher, cfg.ewc_star = ctypes.pointer(fs), ctypes.pointer(ss)
        cfg.ewc_lambda, cfg.ewc_C_old = float(ewc[2]), int(ewc[3])
    nbytes = c_size_t(0)
    steps = (n + batch - 1) // batch
    check(L.ac_head_train_workspace_bytes(batch, steps, ctypes.byref(hp), ctypes.byref(nbytes)), "ac_head_train_workspace_bytes")
    ws = _workspace(nbytes.value, X.device)
    if step_stats is not None:
        assert step_stats.is_cuda and step_stats.dtype == torch.float32 and step_stats.is_contiguous() and step_stats.numel() >= 3 * steps
    if loss_accum is None:
        loss_accum = torch.zeros((1,), dtype=torch.float32, device=X.device)
    targets = targets.contiguous()
    perm = perm.to(device=X.device, dtype=torch.int64).contiguous()
    check(L.ac_head_train_epoch(X.data_ptr(), targets.data_ptr(), perm.data_ptr(), n, batch, ctypes.byref(hp),
                                ctypes.byref(hm), ctypes.byref(hv), ctypes.byref(cfg), loss_accum.data_ptr(), ptr(step_stats),
                                ws.data_ptr(), ws.numel(), stream_ptr()), "ac_head_train_epoch")
    return loss_accum, steps


def head_phase_timing(enable: bool = True):
    """diagnostic: nanoseconds three observed CTAs of the training kernel (holders of a layer-0 / layer-1 / layer-2 block) spent per
    phase / grid barrier (13 counters) and inside the product routines (7 counters from index 14) since enabled: 3 lists of 24"""
    out = (ctypes.c_ulonglong * 72)()
    check(load_library().ac_head_phase_timing(1 if enable else 0, out), "ac_head_phase_timing")
    v = [int(x) for x in out]
    return [v[0:24], v[24:48], v[48:72]]


def head_train_plan(p, batch: int = 32):
    """diagnostic: {ctas, stages, moments_resident, smem_bytes} of the training kernel for this head"""
    hp = head_params_struct(p)
    out = (ctypes.c_int * 5)()
    check(load_library().ac_head_train_plan(batch, ctypes.byref(hp), out), "ac_head_train_plan")
    return dict(zip(("ctas", "stages", "moments_resident", "smem_bytes"), [int(x) for x in out][:4]))


def head_grad(X, targets, p, *, loss_kind=AC_LOSS_CE, grad_out=None, fisher=None, inv_n_batches=1.0):
    L = load_library()
    X = _f32c(X)
    B = X.shape[0]
    hp = head_params_struct(p)
    g = head_params_struct(grad_out) if grad_out is not None else None
    f = head_params_struct(fisher) if fisher is not None else None
    nbytes = c_size_t(0)
    check(L.ac_head_train_workspace_bytes(B, 1, ctypes.byref(hp), ctypes.byref(nbytes)), "ac_head_train_workspace_bytes")
    ws = _workspace(nbytes.value, X.device)
    loss = torch.zeros((1,), dtype=torch.float32, device=X.device)
    targets = targets.contiguous()
    check(L.ac_head_grad(X.data_ptr(), targets.data_ptr(), B, ctypes.byref(hp), loss_kind,
                         ctypes.byref(g) if g is not None else None, ctypes.byref(f) if f is not None else None,
                         float(inv_n_batches), loss.data_ptr(), ws.data_ptr(), ws.numel(), stream_ptr()), "ac_head_grad")
    return loss


_DELTAS = None


def strategic_deltas() -> list:
    """The 10 feature moves of the reference's candidate set (strategic.py:110), with its fp32 bits."""
    global _DELTAS
    if _DELTAS is None:
        _DELTAS = torch.linspace(-2.0, 2.0, 10).tolist()
    return _DELTAS


def _strategic_cfg(cost_kind, c1, c2, dropout_p, seed, step):
    sc = StrategicCfg()
    sc.cost_kind = int(cost_kind)
    sc.c1 = c1.data_ptr()
    sc.c2 = c2.data_ptr() if c2 is not None else None
    for j, d in enumerate(strategic_deltas()):
        sc.delta[j] = d
    sc.dropout_p, sc.seed, sc.step = float(dropout_p), int(seed), int(step)
    return sc


def strategic_best_response(X, p, cost_kind, c1, c2=None, *, dropout_p=0.0, seed=0, step=0, want_rows=True):
    """Best response of every row of X [B, D] against the head p: (choice int32 [B], utility fp32 [B], Y [B, D] or None).
    c1, c2: CUDA fp32 [D] cost coefficients (c2 only for AC_COST_SEPARABLE)."""
    L = load_library()
    X = _f32c(X)
    B = X.shape[0]
    hp = head_params_struct(p)
    c1 = _f32c(c1)
    c2 = _f32c(c2) if c2 is not None else None
    sc = _strategic_cfg(cost_kind, c1, c2, dropout_p, seed, step)
    nbytes = c_size_t(0)
    check(L.ac_strategic_workspace_bytes(B, ctypes.byref(hp), ctypes.byref(nbytes)), "ac_strategic_workspace_bytes")
    ws = _workspace(nbytes.value, X.device)
    choice = torch.empty((B,), dtype=torch.int32, device=X.device)
    util = torch.empty((B,), dtype=torch.float32, device=X.device)
    Y = torch.empty_like(X) if want_rows else None
    check(L.ac_strategic_best_response(X.data_ptr(), B, ctypes.byref(hp), ctypes.byref(sc), choice.data_ptr(), util.data_ptr(),
                                       ptr(Y), ws.data_ptr(), ws.numel(), stream_ptr()), "ac_strategic_best_response")
    return choice, util, Y


def head_train_strategic(X, targets, perms, p, m, v, *, cost_kind, c1, c2=None, lr, strategic_lambda, dropout_p=0.1, seed=0,
                         betas=(0.9, 0.999), eps=1e-8, weight_decay=0.01, max_norm=1.0):
    """classifier.py:1602-1647 in one call: perms int64 [epochs * n] (the DataLoader orders), fresh moments m / v (step 1 first).
    Returns the device step statistics [steps, 3] = (strategic loss, 0, grad norm before clipping)."""
    L = load_library()
    X = _f32c(X)
    n = X.shape[0]
    epochs = perms.numel() // n
    hp, hm, hv = head_params_struct(p), head_params_struct(m), head_params_struct(v)
    cfg = TrainCfg()
    cfg.lr, cfg.beta1, cfg.beta2, cfg.eps = lr, betas[0], betas[1], eps
    cfg.weight_decay, cfg.max_norm = weight_decay, max_norm
    cfg.step, cfg.loss_kind, cfg.dropout_p, cfg.seed = 1, AC_LOSS_CE_STRATEGIC, dropout_p, seed
    cfg.strategic_lambda = float(strategic_lambda)
    c1 = _f32c(c1)
    c2 = _f32c(c2) if c2 is not None else None
    sc = _strategic_cfg(cost_kind, c1, c2, dropout_p, seed, 0)
    nbytes = c_size_t(0)
    check(L.ac_head_train_strategic_workspace_bytes(n, ctypes.byref(hp), ctypes.byref(nbytes)), "ac_head_train_strategic_workspace_bytes")
    ws = _workspace(nbytes.value, X.device)
    batch = min(16, n)
    stats = torch.zeros((epochs * ((n + batch - 1) // batch), 3), dtype=torch.float32, device=X.device)
    targets = targets.to(device=X.device, dtype=torch.int64).contiguous()
    perms = perms.to(device=X.device, dtype=torch.int64).contiguous()
    check(L.ac_head_train_strategic(X.data_ptr(), targets.data_ptr(), perms.data_ptr(), n, epochs, ctypes.byref(hp), ctypes.byref(hm),
                                    ctypes.byref(hv), ctypes.byref(cfg), ctypes.byref(sc), stats.data_ptr(), ws.data_ptr(), ws.numel(),
                                    stream_ptr()), "ac_head_train_strategic")
    return stats


def ewc_penalty(p, fisher, star, lam: float, batch_size: Optional[int], C_old: int = 0) -> torch.Tensor:
    L = load_library()
    hp, hf, hs = head_params_struct(p), head_params_struct(fisher), head_params_struct(star)
    out = torch.zeros((1,), dtype=torch.float32, device=p["W0"].device)
    inv = 1.0 / batch_size if batch_size else 1.0
    check(L.ac_ewc_penalty(ctypes.byref(hp), ctypes.byref(hf), ctypes.byref(hs), float(lam), float(inv), C_old,
                           out.data_ptr(), stream_ptr()), "ac_ewc_penalty")
    return out


def linear_tc(X, W, bias, residual=None, epi: int = 0, round_out: bool = False, out_half: bool = False) -> torch.Tensor:
    """X, W fp32 -> tf32 path; X, W fp16 -> fp16 path (the encoder's); Y fp32 unless out_half.  epi 4 (SwiGLU) takes W's
    rows interleaved in 32-row groups (activated, multiplier) and returns Y [M, N / 2]."""
    L = load_library()
    assert X.is_cuda and W.is_cuda and X.dtype == W.dtype and X.dtype in (torch.float32, torch.float16)
    X, W = X.contiguous(), W.contiguous()
    prec = AC_PREC_F16 if X.dtype == torch.float16 else AC_PREC_TF32
    M, K = X.shape
    N = W.shape[0]
    Y = torch.empty((M, N // 2 if epi == 4 else N), dtype=torch.float16 if out_half else torch.float32, device=X.device)
    check(L.ac_linear_tc(X.data_ptr(), W.data_ptr(), ptr(bias), ptr(residual), Y.data_ptr(), M, N, K, epi,
                         1 if round_out else 0, prec, 1 if out_half else 0, stream_ptr()), "ac_linear_tc")
    return Y


def distilbert_to_bert_state_dict(sd: dict, c):
    """DistilBERT (HF models/distilbert/modeling_distilbert.py) is the BERT post-LN block without token-type embeddings:
    rename its parameters to the BERT names the encoder consumes and supply an all-zero single-row type table."""
    if getattr(c, "activation", "gelu") != "gelu" or getattr(c, "sinusoidal_pos_embds", False):
        raise AdaptiveB200Error("DistilBERT variant with non-GELU activation / sinusoidal positions is not implemented")
    out = {
        "embeddings.word_embeddings.weight": sd["embeddings.word_embeddings.weight"],
        "embeddings.position_embeddings.weight": sd["embeddings.position_embeddings.weight"],
        "embeddings.token_type_embeddings.weight": torch.zeros((1, c.dim), dtype=torch.float32),
        "embeddings.LayerNorm.weight": sd["embeddings.LayerNorm.weight"],
        "embeddings.LayerNorm.bias": sd["embeddings.LayerNorm.bias"],
    }
    ren = {"attention.q_lin": "attention.self.query", "attention.k_lin": "attention.self.key",
           "attention.v_lin": "attention.self.value", "attention.out_lin": "attention.output.dense",
           "sa_layer_norm": "attention.output.LayerNorm", "ffn.lin1": "intermediate.dense", "ffn.lin2": "output.dense",
           "output_layer_norm": "output.LayerNorm"}
    for l in range(c.n_layers):
        for src, dst in ren.items():
            for wb in ("weight", "bias"):
                out[f"encoder.layer.{l}.{dst}.{wb}"] = sd[f"transformer.layer.{l}.{src}.{wb}"]
    dims = dict(layers=c.n_layers, hidden=c.dim, heads=c.n_heads, intermediate=c.hidden_dim, vocab=c.vocab_size,
                max_pos=c.max_position_embeddings, type_vocab=1, ln_eps=1e-12, pad_idx=0)
    return out, dims


def mpnet_relative_bias_table(weight: torch.Tensor, heads: int) -> torch.Tensor:
    """[heads, 2 AC_ENCODER_MAX_S - 1] fp32 table of ac_encoder_config.rel_bias: entry (h, AC_ENCODER_MAX_S - 1 + key - query)
    = weight[bucket(key - query), h], with HF MPNetEncoder.relative_position_bucket's formula and fp32 arithmetic (32 buckets:
    16 per direction, exact below distance 8, log-spaced up to 128, saturated beyond)."""
    weight = weight.detach().to(device="cpu", dtype=torch.float32)
    assert weight.shape == (32, heads), weight.shape
    n = -torch.arange(-(AC_ENCODER_MAX_S - 1), AC_ENCODER_MAX_S, dtype=torch.long)     # query - key
    num_buckets, max_exact, max_distance = 16, 8, 128
    ret = (n < 0).to(torch.long) * num_buckets
    n = torch.abs(n)
    large = max_exact + (torch.log(n.float() / max_exact) / math.log(max_distance / max_exact)
                         * (num_buckets - max_exact)).to(torch.long)
    large = torch.min(large, torch.full_like(large, num_buckets - 1))
    bucket = ret + torch.where(n < max_exact, n, large)
    return weight[bucket].t().contiguous()


def mpnet_to_bert_state_dict(sd: dict, c):
    """MPNet (HF models/mpnet/modeling_mpnet.py) is the post-LN BERT block with RoBERTa's position rule (padding_idx 1), no
    token-type embeddings and a relative position bias on the attention scores: rename its parameters to the BERT names the
    encoder consumes, supply an all-zero single-row type table and turn encoder.relative_attention_bias into the rel_bias
    table.  pooler.* is not used.  Raises AdaptiveB200Error naming any setting the CUDA path does not implement."""
    if c.hidden_act != "gelu":
        raise AdaptiveB200Error(f"MPNet hidden_act={c.hidden_act!r}: only exact-erf 'gelu' is implemented")
    heads = c.num_attention_heads
    if heads <= 0 or c.hidden_size != 64 * heads:
        raise AdaptiveB200Error(f"MPNet head_dim={c.hidden_size / heads:g} (hidden={c.hidden_size}, heads={heads}): only "
                                "head_dim 64 is implemented")
    if c.relative_attention_num_buckets != 32:
        raise AdaptiveB200Error(f"MPNet relative_attention_num_buckets={c.relative_attention_num_buckets}: only 32 is "
                                "implemented (the bucket count HF's forward uses)")
    out = {k: sd[k] for k in ("embeddings.word_embeddings.weight", "embeddings.position_embeddings.weight",
                              "embeddings.LayerNorm.weight", "embeddings.LayerNorm.bias")}
    out["embeddings.token_type_embeddings.weight"] = torch.zeros((1, c.hidden_size), dtype=torch.float32)
    ren = {"attention.attn.q": "attention.self.query", "attention.attn.k": "attention.self.key",
           "attention.attn.v": "attention.self.value", "attention.attn.o": "attention.output.dense",
           "attention.LayerNorm": "attention.output.LayerNorm", "intermediate.dense": "intermediate.dense",
           "output.dense": "output.dense", "output.LayerNorm": "output.LayerNorm"}
    for l in range(c.num_hidden_layers):
        for src, dst in ren.items():
            for wb in ("weight", "bias"):
                out[f"encoder.layer.{l}.{dst}.{wb}"] = sd[f"encoder.layer.{l}.{src}.{wb}"]
    dims = dict(layers=c.num_hidden_layers, hidden=c.hidden_size, heads=heads, intermediate=c.intermediate_size,
                vocab=c.vocab_size, max_pos=c.max_position_embeddings, type_vocab=1, ln_eps=c.layer_norm_eps, pad_idx=1,
                rel_bias=mpnet_relative_bias_table(sd["encoder.relative_attention_bias.weight"], heads))
    return out, dims


def deberta_rel_index(position_buckets: int, max_relative_positions: int,
                      radius: int = AC_ENCODER_MAX_S) -> Tuple[torch.Tensor, int]:
    """(rel_index, span) of ac_encoder_config: int32 [2 radius - 1] with entry radius - 1 + r =
    c(r) = clamp(bucket(r) + span, 0, 2 span - 1) for r = query - key, with HF build_relative_position's arithmetic
    (make_log_bucket_position: identity below span / 2, log-spaced up to max_relative_positions; no buckets when either
    setting is < 1), span = position_buckets, or max_relative_positions without buckets.  radius is the table's
    ac_encoder_config.rel_radius (AC_ENCODER_MAX_S: rel_radius 0)."""
    r = torch.arange(-(radius - 1), radius, dtype=torch.long)
    if position_buckets > 0 and max_relative_positions > 0:
        sign = torch.sign(r)
        mid = position_buckets // 2
        abs_pos = torch.where((r < mid) & (r > -mid), torch.tensor(mid - 1).type_as(r), torch.abs(r))
        log_pos = torch.ceil(torch.log(abs_pos / mid) / torch.log(torch.tensor((max_relative_positions - 1) / mid))
                             * (mid - 1)) + mid
        r = torch.where(abs_pos <= mid, r.type_as(log_pos), log_pos * sign).to(torch.long)
    span = position_buckets if position_buckets > 0 else max_relative_positions
    return torch.clamp(r + span, 0, 2 * span - 1).to(torch.int32), span


def deberta_settings(c) -> None:
    """Raises AdaptiveB200Error naming any DebertaV2Config setting the CUDA path does not implement (no device call)."""
    heads = c.num_attention_heads
    head_dim = getattr(c, "attention_head_size", None) or (c.hidden_size // heads if heads > 0 else 0)
    pat = c.pos_att_type if c.pos_att_type is not None else []
    pat = [x.strip() for x in pat.lower().split("|")] if isinstance(pat, str) else list(pat)
    refusals = [
        (getattr(c, "conv_kernel_size", 0) > 0,
         f"conv_kernel_size={getattr(c, 'conv_kernel_size', 0)}: the ConvLayer of deberta-v2-xlarge/xxlarge"),
        (getattr(c, "embedding_size", c.hidden_size) != c.hidden_size,
         f"embedding_size={getattr(c, 'embedding_size', None)} != hidden_size={c.hidden_size}: the embed_proj"),
        (not getattr(c, "relative_attention", False), "relative_attention=False"),
        (len(pat) != 2 or set(pat) != {"c2p", "p2c"}, f"pos_att_type={pat!r}: only exactly ['c2p', 'p2c']"),
        (c.hidden_act != "gelu", f"hidden_act={c.hidden_act!r}: only exact-erf 'gelu'"),
        (head_dim != 64 or c.hidden_size != 64 * heads,
         f"head_dim={head_dim} (hidden={c.hidden_size}, heads={heads}, attention_head_size="
         f"{getattr(c, 'attention_head_size', None)}): only head_dim 64"),
        (c.max_position_embeddings > AC_ENCODER_MAX_S,
         f"max_position_embeddings={c.max_position_embeddings}: at most {AC_ENCODER_MAX_S}"),
    ]
    for bad, what in refusals:
        if bad:
            raise AdaptiveB200Error(f"DeBERTa {what} is not implemented in the CUDA path")


def deberta_to_bert_state_dict(sd: dict, c):
    """DeBERTa-v2 / v3 (HF models/deberta_v2/modeling_deberta_v2.py) is the post-LN BERT block with disentangled attention:
    rename its parameters to the BERT names the encoder consumes, supply all-zero position (BERT ids) and single-row type
    tables where the checkpoint has none (position_biased_input off, type_vocab_size 0), and build the per-layer fp32
    position tables pos_key / pos_query [layers, 2 span, H] (from the encoder's rel_embeddings, LayerNorm-ed under
    norm_rel_ebd = layer_norm, through key_proj / query_proj or pos_key_proj / pos_query_proj) and rel_index
    (deberta_rel_index).  Without absolute positions (position_biased_input False: deberta-v3-*, mdeberta-v3-base) dims
    also carry rel_index_long, the radius-AC_MODERNBERT_MAX_S index, with which the encoder takes sequences up to
    AC_MODERNBERT_MAX_S tokens.  Raises AdaptiveB200Error naming any setting the CUDA path does not implement."""
    deberta_settings(c)
    H, L = c.hidden_size, c.num_hidden_layers
    f32 = lambda t: t.detach().to(device="cpu", dtype=torch.float32)
    out = {k: sd[k] for k in ("embeddings.word_embeddings.weight", "embeddings.LayerNorm.weight",
                              "embeddings.LayerNorm.bias")}
    out["embeddings.position_embeddings.weight"] = (
        sd["embeddings.position_embeddings.weight"] if getattr(c, "position_biased_input", True)
        else torch.zeros((c.max_position_embeddings, H), dtype=torch.float32))
    out["embeddings.token_type_embeddings.weight"] = (
        sd["embeddings.token_type_embeddings.weight"] if c.type_vocab_size > 0 else torch.zeros((1, H), dtype=torch.float32))
    ren = {"attention.self.query_proj": "attention.self.query", "attention.self.key_proj": "attention.self.key",
           "attention.self.value_proj": "attention.self.value", "attention.output.dense": "attention.output.dense",
           "attention.output.LayerNorm": "attention.output.LayerNorm", "intermediate.dense": "intermediate.dense",
           "output.dense": "output.dense", "output.LayerNorm": "output.LayerNorm"}
    for l in range(L):
        for src, dst in ren.items():
            for wb in ("weight", "bias"):
                out[f"encoder.layer.{l}.{dst}.{wb}"] = sd[f"encoder.layer.{l}.{src}.{wb}"]
    buckets = getattr(c, "position_buckets", -1)
    max_rel = getattr(c, "max_relative_positions", -1)
    if max_rel < 1:
        max_rel = c.max_position_embeddings
    rel_index, span = deberta_rel_index(buckets, max_rel)
    # without absolute positions nothing in the model depends on the length: the long index lets S run to
    # AC_MODERNBERT_MAX_S (Encoder's rel_index_long); with them, max_position_embeddings <= 512 bounds S
    extra = {}
    if not getattr(c, "position_biased_input", True):
        extra["rel_index_long"] = deberta_rel_index(buckets, max_rel, AC_MODERNBERT_MAX_S)[0]
    rel = f32(sd["encoder.rel_embeddings.weight"])
    norm = [x.strip() for x in getattr(c, "norm_rel_ebd", "none").lower().split("|")]
    if "layer_norm" in norm:
        rel = torch.nn.functional.layer_norm(rel, (H,), f32(sd["encoder.LayerNorm.weight"]),
                                             f32(sd["encoder.LayerNorm.bias"]), c.layer_norm_eps)
    rel = rel[:2 * span]
    share = getattr(c, "share_att_key", False)
    pk, pq = [], []
    for l in range(L):
        p = f"encoder.layer.{l}.attention.self."
        kname, qname = ("key_proj", "query_proj") if share else ("pos_key_proj", "pos_query_proj")
        pk.append(torch.nn.functional.linear(rel, f32(sd[p + kname + ".weight"]), f32(sd[p + kname + ".bias"])))
        pq.append(torch.nn.functional.linear(rel, f32(sd[p + qname + ".weight"]), f32(sd[p + qname + ".bias"])))
    dims = dict(layers=L, hidden=H, heads=c.num_attention_heads, intermediate=c.intermediate_size, vocab=c.vocab_size,
                max_pos=c.max_position_embeddings, type_vocab=max(c.type_vocab_size, 1), ln_eps=c.layer_norm_eps,
                pad_idx=0, pos_key=torch.stack(pk), pos_query=torch.stack(pq), pos_span=span, rel_index=rel_index, **extra)
    return out, dims


def _factorized_settings(c, family: str) -> None:
    """Refusals shared by ALBERT and ELECTRA (post-LN BERT blocks behind factorized embeddings), raised before any device call
    with the setting's name."""
    H, E = c.hidden_size, getattr(c, "embedding_size", c.hidden_size)
    if H % 128 != 0 or H > 1024:
        raise AdaptiveB200Error(f"{family} hidden_size={H} is not implemented in the CUDA path: the encoder takes hidden "
                                "<= 1024 in multiples of 128")
    check_head_dim(H, c.num_attention_heads, family)
    if E % 128 != 0 or E <= 0 or E > H:
        raise AdaptiveB200Error(f"{family} embedding_size={E} (hidden_size={H}) is not implemented in the CUDA path: it must "
                                "be a multiple of 128 and <= hidden_size")
    if c.hidden_act not in FFN_ACTS:
        raise AdaptiveB200Error(f"{family} hidden_act={c.hidden_act!r} is not implemented in the CUDA path (only "
                                f"{', '.join(repr(a) for a in FFN_ACTS)})")
    pet = getattr(c, "position_embedding_type", "absolute")
    if pet != "absolute":
        raise AdaptiveB200Error(f"{family} position_embedding_type={pet!r} is not implemented in the CUDA path (only "
                                "'absolute')")


def albert_settings(c) -> None:
    """Raises AdaptiveB200Error naming any AlbertConfig setting the CUDA path does not implement (no device call):
    albert-xlarge / xxlarge (hidden 2048 / 4096), head_dim other than 64 / 32, embedding_size not a multiple of 128 or
    larger than hidden, hidden_act other than gelu / gelu_new / gelu_pytorch_tanh, non-absolute positions, and a layer walk
    HF itself cannot run (num_hidden_groups outside 1 .. num_hidden_layers, inner_group_num < 1)."""
    _factorized_settings(c, "ALBERT")
    if not 1 <= c.num_hidden_groups <= c.num_hidden_layers or c.inner_group_num < 1:
        raise AdaptiveB200Error(f"ALBERT num_hidden_groups={c.num_hidden_groups}, inner_group_num={c.inner_group_num} "
                                f"(num_hidden_layers={c.num_hidden_layers}) is not a valid layer walk")


def electra_settings(c) -> None:
    """Raises AdaptiveB200Error naming any ElectraConfig setting the CUDA path does not implement (no device call)."""
    _factorized_settings(c, "ELECTRA")


def albert_layer_sources(c) -> list:
    """(group, inner layer) of every effective layer of an ALBERT encoder, in order: HF AlbertTransformer runs group
    int(i / (num_hidden_layers / num_hidden_groups)) for i < num_hidden_layers, each group its inner_group_num layers."""
    return [(int(i / (c.num_hidden_layers / c.num_hidden_groups)), j)
            for i in range(c.num_hidden_layers) for j in range(c.inner_group_num)]


def albert_to_bert_state_dict(sd: dict, c):
    """ALBERT (HF models/albert/modeling_albert.py) is the post-LN BERT block behind factorized embeddings (tables and
    LayerNorm at width embedding_size, then encoder.embedding_hidden_mapping_in to hidden) with cross-layer parameter
    sharing.  Returns the BERT names per effective layer -- layers that share parameters map to the SAME source tensor, which
    Encoder packs once -- plus the projection as embeddings_project.*, and the Encoder dims.  pooler.* is not used."""
    albert_settings(c)
    out = {k: sd[k] for k in ("embeddings.word_embeddings.weight", "embeddings.position_embeddings.weight",
                              "embeddings.token_type_embeddings.weight", "embeddings.LayerNorm.weight",
                              "embeddings.LayerNorm.bias")}
    for wb in ("weight", "bias"):
        out[f"embeddings_project.{wb}"] = sd[f"encoder.embedding_hidden_mapping_in.{wb}"]
    ren = {"attention.query": "attention.self.query", "attention.key": "attention.self.key",
           "attention.value": "attention.self.value", "attention.dense": "attention.output.dense",
           "attention.LayerNorm": "attention.output.LayerNorm", "ffn": "intermediate.dense", "ffn_output": "output.dense",
           "full_layer_layer_norm": "output.LayerNorm"}
    walk = albert_layer_sources(c)
    for l, (g, j) in enumerate(walk):
        for src, dst in ren.items():
            for wb in ("weight", "bias"):
                out[f"encoder.layer.{l}.{dst}.{wb}"] = sd[f"encoder.albert_layer_groups.{g}.albert_layers.{j}.{src}.{wb}"]
    dims = dict(layers=len(walk), hidden=c.hidden_size, heads=c.num_attention_heads, intermediate=c.intermediate_size,
                vocab=c.vocab_size, max_pos=c.max_position_embeddings, type_vocab=c.type_vocab_size, ln_eps=c.layer_norm_eps,
                pad_idx=0, embedding_size=c.embedding_size, ffn_act=FFN_ACTS[c.hidden_act])
    return out, dims


def electra_to_bert_state_dict(sd: dict, c):
    """ELECTRA (HF models/electra/modeling_electra.py) is BERT with embedding tables at width embedding_size and, when that
    differs from hidden, embeddings_project to hidden after the embedding LayerNorm.  The layer names are BERT's already;
    returns them plus embeddings_project.* when present, and the Encoder dims."""
    electra_settings(c)
    out = {k: v for k, v in sd.items() if k.startswith(("embeddings.", "embeddings_project.", "encoder.layer."))}
    out.pop("embeddings.position_ids", None)
    out.pop("embeddings.token_type_ids", None)
    E = c.embedding_size
    dims = dict(layers=c.num_hidden_layers, hidden=c.hidden_size, heads=c.num_attention_heads,
                intermediate=c.intermediate_size, vocab=c.vocab_size, max_pos=c.max_position_embeddings,
                type_vocab=c.type_vocab_size, ln_eps=c.layer_norm_eps, pad_idx=0,
                embedding_size=E if E != c.hidden_size else 0, ffn_act=FFN_ACTS[c.hidden_act])
    return out, dims


def check_head_dim(hidden: int, heads: int, what: str = "encoder") -> None:
    """The attention kernels of the BERT-family encoder take head_dim = hidden / heads of 64 (bert-base, RoBERTa, DistilBERT)
    or 32 (all-MiniLM, BGE-small, E5-small, GTE-small); raises AdaptiveB200Error naming anything else (no device call)."""
    if heads <= 0 or hidden % heads != 0:
        raise AdaptiveB200Error(f"{what} hidden={hidden} is not divisible by heads={heads}: head_dim must be 64 or 32")
    head_dim = hidden // heads
    if head_dim not in (64, 32):
        raise AdaptiveB200Error(f"{what} head_dim={head_dim} (hidden={hidden}, heads={heads}): only head_dim 64 and 32 are "
                                "implemented")


def modernbert_rope_table(theta: float, n_pos: int = AC_ENCODER_MAX_S, head_dim: int = 64) -> torch.Tensor:
    """[n_pos, head_dim] fp32 table the encoder's RoPE epilogue reads: row p = cos | sin of the head_dim / 2 frequencies at
    position p, computed with HF ModernBertRotaryEmbedding's own formula (default rope type, attention scaling 1)."""
    inv_freq = 1.0 / (theta ** (torch.arange(0, head_dim, 2, dtype=torch.int64).to(dtype=torch.float) / head_dim))
    pos = torch.arange(n_pos).float()
    freqs = (inv_freq[None, :, None].float() @ pos[None, None, :]).transpose(1, 2)[0]      # [n_pos, head_dim / 2]
    return torch.cat((freqs.cos(), freqs.sin()), dim=-1).contiguous()


def modernbert_settings(c) -> dict:
    """Encoder arguments of a ModernBertConfig; raises AdaptiveB200Error naming any setting the CUDA path does not implement
    (checked before any device call)."""
    if getattr(c, "hidden_activation", "gelu") != "gelu":
        raise AdaptiveB200Error(f"ModernBERT hidden_activation={c.hidden_activation!r}: only exact-erf 'gelu' is implemented")
    for flag in ("norm_bias", "attention_bias", "mlp_bias"):
        if getattr(c, flag, False):
            raise AdaptiveB200Error(f"ModernBERT {flag}=True is not implemented (the published checkpoints have no biases)")
    heads = c.num_attention_heads
    head_dim = getattr(c, "head_dim", None) or c.hidden_size // heads
    if head_dim != 64 or c.hidden_size != heads * 64:
        raise AdaptiveB200Error(f"ModernBERT head_dim={head_dim}: only head_dim 64 is implemented")
    types = list(c.layer_types)
    if len(types) != c.num_hidden_layers or not set(types) <= {"full_attention", "sliding_attention"}:
        raise AdaptiveB200Error(f"ModernBERT layer_types={types!r}: only full_attention / sliding_attention are implemented")
    theta = {}
    for lt in ("full_attention", "sliding_attention"):
        rp = c.rope_parameters[lt]
        if rp.get("rope_type", "default") != "default":
            raise AdaptiveB200Error(f"ModernBERT rope_type={rp.get('rope_type')!r} ({lt}): only 'default' RoPE is implemented")
        theta[lt] = float(rp["rope_theta"])
    window = int(c.sliding_window)
    if "sliding_attention" in types and window < 1:
        raise AdaptiveB200Error(f"ModernBERT sliding_window={window}: the half-window must be >= 1")
    # the longest sequence the encoder accepts and the rows of its RoPE tables; never fewer than the BERT-family limit
    max_pos = max(AC_ENCODER_MAX_S, int(c.max_position_embeddings))
    if max_pos > AC_MODERNBERT_MAX_S:
        raise AdaptiveB200Error(f"ModernBERT max_position_embeddings={c.max_position_embeddings}: at most "
                                f"{AC_MODERNBERT_MAX_S} is implemented")
    return dict(layers=c.num_hidden_layers, hidden=c.hidden_size, heads=heads, intermediate=c.intermediate_size,
                vocab=c.vocab_size, max_pos=max_pos, ln_eps=c.norm_eps,
                pad_idx=(c.pad_token_id if c.pad_token_id is not None else 0),
                sliding_window=window, layer_sliding=[1 if t == "sliding_attention" else 0 for t in types],
                rope_theta=(theta["full_attention"], theta["sliding_attention"]))


def _rotary_settings(c, family: str, acts) -> None:
    """Refusals shared by NomicBERT and jina-embeddings-v3 (post-LN BERT blocks with RoPE on q and k), raised before any
    device call with the setting's name."""
    rp = getattr(c, "rope_parameters", None) or {}
    if rp.get("rope_type", "default") != "default":
        raise AdaptiveB200Error(f"{family} rope_type={rp.get('rope_type')!r} is not implemented in the CUDA path (only "
                                "'default' RoPE; dynamic NTK, YaRN and linear scaling need a table per sequence length)")
    H, heads = c.hidden_size, c.num_attention_heads
    if H % 128 != 0 or H > 1024:
        raise AdaptiveB200Error(f"{family} hidden_size={H} is not implemented in the CUDA path: the encoder takes hidden "
                                "<= 1024 in multiples of 128")
    head_dim = getattr(c, "head_dim", None) or (H // heads if heads > 0 else 0)
    if heads <= 0 or head_dim != 64 or H != 64 * heads:
        raise AdaptiveB200Error(f"{family} head_dim={head_dim} (hidden={H}, heads={heads}) is not implemented in the CUDA "
                                "path: only head_dim 64")
    if c.hidden_act not in acts:
        raise AdaptiveB200Error(f"{family} hidden_act={c.hidden_act!r} is not implemented in the CUDA path (only "
                                f"{', '.join(repr(a) for a in acts)})")


def nomic_bert_settings(c) -> None:
    """Raises AdaptiveB200Error naming any NomicBertConfig setting the CUDA path does not implement (no device call)."""
    _rotary_settings(c, "NomicBERT", ("silu", "swish"))


def jina_v3_settings(c) -> None:
    """Raises AdaptiveB200Error naming any JinaEmbeddingsV3Config setting the CUDA path does not implement (no device
    call)."""
    _rotary_settings(c, "jina-embeddings-v3", tuple(FFN_ACTS))


def _rotary_dims(c, ffn_act: int) -> dict:
    """Encoder dims of a rotary config: max_pos = the RoPE table's rows and the longest S, max(512, min(max_position_embeddings,
    AC_MODERNBERT_MAX_S)) (HF itself fails past max_position_embeddings when no token_type_ids are passed)"""
    rp = getattr(c, "rope_parameters", None) or {}
    return dict(layers=c.num_hidden_layers, hidden=c.hidden_size, heads=c.num_attention_heads,
                intermediate=c.intermediate_size, vocab=c.vocab_size,
                max_pos=max(AC_ENCODER_MAX_S, min(int(c.max_position_embeddings), AC_MODERNBERT_MAX_S)),
                type_vocab=max(int(c.type_vocab_size), 1), ln_eps=c.layer_norm_eps, pad_idx=0, ffn_act=ffn_act,
                rope_theta=float(rp.get("rope_theta", getattr(c, "default_theta", 10000.0))))


def _rotary_to_bert_state_dict(sd: dict, c, ffn, ffn_act: int):
    """the native names of a NomicBertModel / JinaEmbeddingsV3Model (layers.l.self_attn.*, post_*_layernorm, mlp.*) as the
    BERT names Encoder consumes; ffn(sd, layer prefix) gives the FFN's BERT names -> (weight, bias or None).  Biases the checkpoint does
    not have become zeros, so that ac_encoder_create never sees a NULL bias.  pooler.* is not used."""
    out = {k: sd[k] for k in ("embeddings.word_embeddings.weight", "embeddings.token_type_embeddings.weight",
                              "embeddings.LayerNorm.weight", "embeddings.LayerNorm.bias")}
    ren = {"self_attn.q_proj": "attention.self.query", "self_attn.k_proj": "attention.self.key",
           "self_attn.v_proj": "attention.self.value", "self_attn.o_proj": "attention.output.dense",
           "post_attention_layernorm": "attention.output.LayerNorm", "post_mlp_layernorm": "output.LayerNorm"}
    for l in range(c.num_hidden_layers):
        src, dst = f"layers.{l}.", f"encoder.layer.{l}."
        for a, b in ren.items():
            w = sd[src + a + ".weight"]
            out[dst + b + ".weight"] = w
            out[dst + b + ".bias"] = sd.get(src + a + ".bias", torch.zeros(w.shape[0], dtype=torch.float32))
        for b, (w, bias) in ffn(sd, src).items():
            out[dst + b + ".weight"] = w
            out[dst + b + ".bias"] = bias if bias is not None else torch.zeros(w.shape[0], dtype=torch.float32)
    return out, _rotary_dims(c, ffn_act)


def nomic_bert_to_bert_state_dict(sd: dict, c):
    """NomicBERT (HF models/nomic_bert): RoPE (theta 1000 by default), no q/k/v/o biases, SwiGLU FFN
    down(silu(gate_proj x) * up_proj x) without biases.  FFN1 is cat([gate_proj, up_proj]) [2I, H] (AC_FFN_SWIGLU's row
    order).  Returns the BERT names and the Encoder dims (arch "rotary")."""
    nomic_bert_settings(c)
    ffn = lambda sd, p: {
        "intermediate.dense": (torch.cat([sd[p + "mlp.gate_proj.weight"], sd[p + "mlp.up_proj.weight"]]), None),
        "output.dense": (sd[p + "mlp.down_proj.weight"], None)}
    return _rotary_to_bert_state_dict(sd, c, ffn, AC_FFN_SWIGLU)


def jina_v3_to_bert_state_dict(sd: dict, c):
    """jina-embeddings-v3 (HF models/jina_embeddings_v3): RoPE (theta 20000 by default) with q/k/v/o biases, FFN
    fc2(GELU(fc1 x)) with biases.  Returns the BERT names and the Encoder dims (arch "rotary")."""
    jina_v3_settings(c)
    ffn = lambda sd, p: {"intermediate.dense": (sd[p + "mlp.fc1.weight"], sd[p + "mlp.fc1.bias"]),
                         "output.dense": (sd[p + "mlp.fc2.weight"], sd[p + "mlp.fc2.bias"])}
    return _rotary_to_bert_state_dict(sd, c, ffn, FFN_ACTS[c.hidden_act])


def eurobert_settings(c) -> dict:
    """Encoder dims of a EuroBertConfig; raises AdaptiveB200Error naming any setting the CUDA path does not implement (checked
    before any device call).  The sequence limit and the RoPE table's rows are max(512, min(max_position_embeddings,
    AC_MODERNBERT_MAX_S))."""
    rp = getattr(c, "rope_parameters", None) or {}
    if rp.get("rope_type", "default") != "default":
        raise AdaptiveB200Error(f"EuroBERT rope_type={rp.get('rope_type')!r} is not implemented in the CUDA path (only "
                                "'default' RoPE; llama3, YaRN, dynamic NTK and linear scaling change the table)")
    for flag in ("attention_bias", "mlp_bias"):
        if getattr(c, flag, False):
            raise AdaptiveB200Error(f"EuroBERT {flag}=True is not implemented in the CUDA path (the published checkpoints "
                                    "have no biases)")
    H, heads = c.hidden_size, c.num_attention_heads
    if H % 128 != 0 or H > 1024:
        raise AdaptiveB200Error(f"EuroBERT hidden_size={H} is not implemented in the CUDA path: the encoder takes hidden "
                                "<= 1024 in multiples of 128")
    head_dim = getattr(c, "head_dim", None) or (H // heads if heads > 0 else 0)
    if heads <= 0 or head_dim != 64 or H != 64 * heads:
        raise AdaptiveB200Error(f"EuroBERT head_dim={head_dim} (hidden={H}, heads={heads}) is not implemented in the CUDA "
                                "path: only head_dim 64")
    if c.hidden_act not in ("silu", "swish"):
        raise AdaptiveB200Error(f"EuroBERT hidden_act={c.hidden_act!r} is not implemented in the CUDA path (only 'silu', "
                                "'swish')")
    kv = c.num_key_value_heads if c.num_key_value_heads is not None else heads
    if kv <= 0 or heads % kv != 0:
        raise AdaptiveB200Error(f"EuroBERT num_key_value_heads={kv} does not divide num_attention_heads={heads}")
    return dict(layers=c.num_hidden_layers, hidden=H, heads=heads, intermediate=c.intermediate_size, vocab=c.vocab_size,
                max_pos=max(AC_ENCODER_MAX_S, min(int(c.max_position_embeddings), AC_MODERNBERT_MAX_S)),
                ln_eps=c.rms_norm_eps, pad_idx=(c.pad_token_id if c.pad_token_id is not None else 0),
                rope_theta=float(rp.get("rope_theta", 10000.0)))


def eurobert_to_modernbert_names(sd: dict, c):
    """EuroBertModel's parameters under the ModernBERT names the "eurobert" Encoder reads (include/adaptive_b200.h,
    AC_ARCH_EUROBERT): input_layernorm -> attn_norm (layer 0's too), post_attention_layernorm -> mlp_norm, o_proj -> attn.Wo,
    cat(q, k, v) -> attn.Wqkv, cat(gate_proj, up_proj) -> mlp.Wi, down_proj -> mlp.Wo, norm -> final_norm.  Grouped-query
    attention: k_proj / v_proj rows are expanded to every query head in HF repeat_kv's order (query head h reads kv head
    h // (heads / num_key_value_heads)) before the concatenation, so no kernel sees kv heads.  Returns the names and the
    Encoder dims (eurobert_settings)."""
    dims = eurobert_settings(c)
    heads, L = dims["heads"], dims["layers"]
    kv = c.num_key_value_heads if c.num_key_value_heads is not None else heads

    def expand(w):            # [kv 64, H] -> [heads 64, H]
        return w.view(kv, 1, 64, -1).expand(kv, heads // kv, 64, w.shape[-1]).reshape(heads * 64, -1)

    out = {"embeddings.tok_embeddings.weight": sd["embed_tokens.weight"], "final_norm.weight": sd["norm.weight"]}
    for l in range(L):
        p = f"layers.{l}."
        out[p + "attn_norm.weight"] = sd[p + "input_layernorm.weight"]
        out[p + "mlp_norm.weight"] = sd[p + "post_attention_layernorm.weight"]
        out[p + "attn.Wqkv.weight"] = torch.cat([sd[p + "self_attn.q_proj.weight"], expand(sd[p + "self_attn.k_proj.weight"]),
                                                 expand(sd[p + "self_attn.v_proj.weight"])])
        out[p + "attn.Wo.weight"] = sd[p + "self_attn.o_proj.weight"]
        out[p + "mlp.Wi.weight"] = torch.cat([sd[p + "mlp.gate_proj.weight"], sd[p + "mlp.up_proj.weight"]])
        out[p + "mlp.Wo.weight"] = sd[p + "mlp.down_proj.weight"]
    return out, dims


class Encoder:
    """Owner of an ac_encoder handle built from an HF BERT/RoBERTa/ModernBERT state_dict (CUDA fp32 tensors).  arch "mpnet"
    takes the BERT names (mpnet_to_bert_state_dict) and rel_bias, the [heads, 2 AC_ENCODER_MAX_S - 1] table of
    mpnet_relative_bias_table; arch "deberta" the BERT names and the pos_key / pos_query / pos_span / rel_index of
    deberta_to_bert_state_dict, and with rel_index_long (position-free configs) that index in place of rel_index, passed
    with rel_radius AC_MODERNBERT_MAX_S so that sequences run up to that length.  embedding_size (0 = hidden) and the
    "embeddings_project.*" tensors give factorized embeddings (albert_to_bert_state_dict, electra_to_bert_state_dict);
    ffn_act is AC_FFN_GELU_ERF or AC_FFN_GELU_TANH.
    arch "rotary" takes the BERT names without a position table, RoPE with base rope_theta on q and k, and ffn_act
    AC_FFN_SWIGLU too (nomic_bert_to_bert_state_dict, jina_v3_to_bert_state_dict).  arch "eurobert" takes the ModernBERT
    names of eurobert_to_modernbert_names (RMSNorms, layer 0's attn_norm used, no embedding norm) and one rope_theta.
    Names that refer to the same source tensor (ALBERT's shared layers) are copied and packed once."""

    def __init__(self, sd: dict, *, arch: str, layers: int, hidden: int, heads: int, intermediate: int, vocab: int,
                 max_pos: int = AC_ENCODER_MAX_S, type_vocab: int = 1, ln_eps: float, pad_idx: int = 0,
                 max_tokens: int = 65536, device="cuda", cls_only: bool = True, sliding_window: int = 0,
                 layer_sliding=None, rope_theta=None, rel_bias: Optional[torch.Tensor] = None,
                 pos_key: Optional[torch.Tensor] = None, pos_query: Optional[torch.Tensor] = None, pos_span: int = 0,
                 rel_index: Optional[torch.Tensor] = None, rel_index_long: Optional[torch.Tensor] = None,
                 embedding_size: int = 0, ffn_act: int = AC_FFN_GELU_ERF):
        L = load_library()
        self._L = L
        self.hidden = hidden
        self.heads = heads
        self.intermediate = intermediate
        self.embedding_size = embedding_size or hidden
        self.max_tokens = max_tokens
        dev = torch.device(device)
        keep = {}
        copies = {}

        def g(name):
            # one device copy per source tensor: names that share a tensor (ALBERT's shared layers) pass the same pointer,
            # which ac_encoder_create packs once
            src = sd[name]
            key = (src.data_ptr(), tuple(src.shape), tuple(src.stride()), src.dtype, src.device)
            if key not in copies:
                copies[key] = (src, src.detach().to(device=dev, dtype=torch.float32).contiguous())
            return copies[key][1].data_ptr()

        def arr(fmt):
            a = (c_void_p * layers)(*[g(fmt.format(l)) for l in range(layers)])
            keep[fmt] = a
            return ctypes.cast(a, _PP)

        w = EncoderWeights()
        if arch in ("modernbert", "eurobert"):
            # HF ModernBertModel names; mlp_norm travels in ao_ln_w, attn.Wo in ao_w, mlp.Wo in ff2_w (include/adaptive_b200.h)
            eb = arch == "eurobert"
            w.word_emb = g("embeddings.tok_embeddings.weight")
            if not eb:                          # EuroBERT has no embedding norm
                w.emb_ln_w = g("embeddings.norm.weight")
            w.final_norm_w = g("final_norm.weight")
            p = "layers.{}."
            w.ao_w, w.ao_ln_w, w.ff2_w = arr(p + "attn.Wo.weight"), arr(p + "mlp_norm.weight"), arr(p + "mlp.Wo.weight")
            w.wqkv, w.wi = arr(p + "attn.Wqkv.weight"), arr(p + "mlp.Wi.weight")
            # ModernBERT's layer-0 attn_norm is Identity; EuroBERT's input_layernorm of layer 0 is a real RMSNorm
            an = (c_void_p * layers)(*[g(f"layers.{l}.attn_norm.weight") if (l or eb) else None for l in range(layers)])
            ls = (ctypes.c_int32 * layers)(*(layer_sliding or [0] * layers))
            rope = [modernbert_rope_table(t, max_pos).to(dev) for t in ((rope_theta,) if eb else rope_theta)]
            keep.update(an=an, ls=ls, rope=rope)
            w.attn_norm_w = ctypes.cast(an, _PP)
            cfg = EncoderConfig(AC_ARCH_EUROBERT if eb else AC_ARCH_MODERNBERT, layers, hidden, heads, intermediate, vocab,
                                max_pos, 1, pad_idx, ln_eps, AC_PREC_F16, max_tokens, 1 if cls_only else 0, sliding_window,
                                ctypes.cast(ls, POINTER(ctypes.c_int32)), rope[0].data_ptr(), rope[-1].data_ptr())
            if eb:
                cfg.rope_sliding, cfg.ffn_act = None, AC_FFN_SWIGLU
        else:
            w.word_emb = g("embeddings.word_embeddings.weight")
            if arch != "rotary":
                w.pos_emb = g("embeddings.position_embeddings.weight")
            w.type_emb = g("embeddings.token_type_embeddings.weight")
            w.emb_ln_w = g("embeddings.LayerNorm.weight")
            w.emb_ln_b = g("embeddings.LayerNorm.bias")
            p = "encoder.layer.{}."
            w.q_w, w.q_b = arr(p + "attention.self.query.weight"), arr(p + "attention.self.query.bias")
            w.k_w, w.k_b = arr(p + "attention.self.key.weight"), arr(p + "attention.self.key.bias")
            w.v_w, w.v_b = arr(p + "attention.self.value.weight"), arr(p + "attention.self.value.bias")
            w.ao_w, w.ao_b = arr(p + "attention.output.dense.weight"), arr(p + "attention.output.dense.bias")
            w.ao_ln_w, w.ao_ln_b = arr(p + "attention.output.LayerNorm.weight"), arr(p + "attention.output.LayerNorm.bias")
            w.ff1_w, w.ff1_b = arr(p + "intermediate.dense.weight"), arr(p + "intermediate.dense.bias")
            w.ff2_w, w.ff2_b = arr(p + "output.dense.weight"), arr(p + "output.dense.bias")
            w.out_ln_w, w.out_ln_b = arr(p + "output.LayerNorm.weight"), arr(p + "output.LayerNorm.bias")
            if "embeddings_project.weight" in sd:      # factorized embeddings (ALBERT, ELECTRA)
                w.emb_proj_w, w.emb_proj_b = g("embeddings_project.weight"), g("embeddings_project.bias")
            code = {"bert": AC_ARCH_BERT, "roberta": AC_ARCH_ROBERTA, "mpnet": AC_ARCH_MPNET, "deberta": AC_ARCH_DEBERTA,
                    "rotary": AC_ARCH_ROTARY}[arch]
            cfg = EncoderConfig(code, layers, hidden, heads, intermediate, vocab, max_pos, type_vocab, pad_idx, ln_eps,
                                AC_PREC_F16, max_tokens, 1 if cls_only else 0)
            cfg.embedding_size, cfg.ffn_act = embedding_size, ffn_act
            if arch == "rotary":          # ac_encoder_create refuses a rotary encoder without its table
                rope = modernbert_rope_table(float(rope_theta), max_pos).to(dev)
                keep["rope"] = rope
                cfg.rope_full = rope.data_ptr()
            if rel_bias is not None:      # ac_encoder_create refuses an MPNet encoder without it
                rb = rel_bias.detach().to(device=dev, dtype=torch.float32).contiguous()
                keep["rel_bias"] = rb
                cfg.rel_bias = rb.data_ptr()
            if arch == "deberta":         # ac_encoder_create refuses a DeBERTa encoder without its tables
                if rel_index_long is not None:
                    rel_index = rel_index_long
                    cfg.rel_radius = (rel_index.numel() + 1) // 2
                pos = [t.detach().to(device=dev, dtype=dt).contiguous() if t is not None else None
                       for t, dt in ((pos_key, torch.float32), (pos_query, torch.float32), (rel_index, torch.int32))]
                keep["pos"] = pos
                cfg.pos_key, cfg.pos_query, cfg.rel_index = (ptr(t) for t in pos)
                cfg.pos_span = pos_span
        h = c_void_p()
        with torch.cuda.device(dev):
            check(L.ac_encoder_create(ctypes.byref(cfg), ctypes.byref(w), ctypes.byref(h)), "ac_encoder_create")
        self.handle = h
        del keep, copies  # the handle holds its own packed copies

    @classmethod
    def from_hf(cls, model, max_tokens: int = 65536, device="cuda", cls_only: bool = True):
        """Build from an in-memory HF BertModel / RobertaModel / DistilBertModel / MPNetModel / DebertaV2Model / AlbertModel /
        ElectraModel / NomicBertModel / JinaEmbeddingsV3Model (post-LN blocks; the last two with RoPE, Nomic's FFN SwiGLU),
        ModernBertModel (pre-LN, RoPE, GeGLU, sliding-window layers) or EuroBertModel (pre-norm with RMSNorm, RoPE, SwiGLU,
        grouped-query attention expanded to every head; sequences up to max(512, min(max_position_embeddings,
        AC_MODERNBERT_MAX_S))).  NomicBERT and jina-embeddings-v3 take sequences up
        to max(512, min(max_position_embeddings, AC_MODERNBERT_MAX_S)), RoPE positions 0..S-1 whatever the padding; their
        remote-code modules (trust_remote_code=True), whose parameter names differ, are refused.  head_dim 64 or 32 for BERT / RoBERTa /
        DistilBERT, 64 for MPNet, DeBERTa and ModernBERT.  Sequences up to 512 tokens, or for ModernBERT up to max(512, max_position_embeddings) <=
        AC_MODERNBERT_MAX_S.  DeBERTa-v2 / v3 without absolute positions (position_biased_input False: deberta-v3-*,
        mdeberta-v3-base) takes sequences up to AC_MODERNBERT_MAX_S, as HF does; with absolute positions the 512 limit
        stays.  A RoBERTa / XLM-RoBERTa model with head_dim 64 whose position table has more than
        512 + pad_token_id + 1 rows (bge-m3, snowflake-arctic-embed-l-v2.0: 8194) takes sequences up to
        min(AC_MODERNBERT_MAX_S, max_position_embeddings - pad_token_id - 1), which run the long full-attention kernel
        past 512 tokens; BERT-arch models keep the 512 limit."""
        c = model.config
        mt = getattr(c, "model_type", "bert")
        if mt == "modernbert":
            dims = modernbert_settings(c)
            return cls(dict(model.state_dict()), arch="modernbert", max_tokens=max_tokens, device=device, cls_only=cls_only,
                       **dims)
        if mt == "mpnet":
            sd, dims = mpnet_to_bert_state_dict(dict(model.state_dict()), c)
            return cls(sd, arch="mpnet", max_tokens=max_tokens, device=device, cls_only=cls_only, **dims)
        if mt == "deberta":
            raise AdaptiveB200Error("encoder architecture model_type='deberta' (DeBERTa v1) is not implemented in the CUDA "
                                    "path (DeBERTa-v2 / v3, model_type 'deberta-v2', is)")
        if mt == "deberta-v2":
            sd, dims = deberta_to_bert_state_dict(dict(model.state_dict()), c)
            return cls(sd, arch="deberta", max_tokens=max_tokens, device=device, cls_only=cls_only, **dims)
        if mt == "distilbert":
            check_head_dim(c.dim, c.n_heads, "DistilBERT")
            sd, dims = distilbert_to_bert_state_dict(dict(model.state_dict()), c)
            return cls(sd, arch="bert", max_tokens=max_tokens, device=device, cls_only=cls_only, **dims)
        if mt == "albert":
            # state_dict() lists every shared parameter once; the renaming maps the shared layers onto those tensors
            sd, dims = albert_to_bert_state_dict(dict(model.state_dict()), c)
            return cls(sd, arch="bert", max_tokens=max_tokens, device=device, cls_only=cls_only, **dims)
        if mt == "electra":
            sd, dims = electra_to_bert_state_dict(dict(model.state_dict()), c)
            return cls(sd, arch="bert", max_tokens=max_tokens, device=device, cls_only=cls_only, **dims)
        if mt == "eurobert":
            from transformers import EuroBertModel
            if not isinstance(model, EuroBertModel):
                raise AdaptiveB200Error(f"model_type 'eurobert' from {type(model).__module__}.{type(model).__name__} is not the "
                                        "native transformers EuroBertModel: remote-code modules (trust_remote_code=True) are "
                                        "not implemented in the CUDA path; load the model without trust_remote_code")
            sd, dims = eurobert_to_modernbert_names(dict(model.state_dict()), c)
            return cls(sd, arch="eurobert", max_tokens=max_tokens, device=device, cls_only=cls_only, **dims)
        if mt in ("nomic_bert", "jina_embeddings_v3"):
            from transformers import JinaEmbeddingsV3Model, NomicBertModel
            native = NomicBertModel if mt == "nomic_bert" else JinaEmbeddingsV3Model
            if not isinstance(model, native):
                raise AdaptiveB200Error(f"model_type '{mt}' from {type(model).__module__}.{type(model).__name__} is not the "
                                        f"native transformers {native.__name__}: remote-code modules (trust_remote_code=True) "
                                        "are not implemented in the CUDA path; load the model without trust_remote_code")
            to_bert = nomic_bert_to_bert_state_dict if mt == "nomic_bert" else jina_v3_to_bert_state_dict
            sd, dims = to_bert(dict(model.state_dict()), c)
            return cls(sd, arch="rotary", max_tokens=max_tokens, device=device, cls_only=cls_only, **dims)
        if mt not in ("bert", "roberta", "xlm-roberta"):
            raise AdaptiveB200Error(f"encoder architecture '{mt}' is not implemented in the CUDA path yet")
        if getattr(c, "hidden_act", "gelu") not in FFN_ACTS or getattr(c, "position_embedding_type", "absolute") != "absolute":
            raise AdaptiveB200Error(f"hidden_act={getattr(c, 'hidden_act', None)!r}: only GELU (exact erf 'gelu', tanh "
                                    "'gelu_new' / 'gelu_pytorch_tanh') and absolute position embeddings are implemented")
        check_head_dim(c.hidden_size, c.num_attention_heads, mt)
        sd = {k: v for k, v in model.state_dict().items()}
        return cls(sd, arch="bert" if mt == "bert" else "roberta", layers=c.num_hidden_layers, hidden=c.hidden_size,
                   heads=c.num_attention_heads, intermediate=c.intermediate_size, vocab=c.vocab_size,
                   max_pos=c.max_position_embeddings, type_vocab=c.type_vocab_size, ln_eps=c.layer_norm_eps,
                   pad_idx=(c.pad_token_id if c.pad_token_id is not None else 0), max_tokens=max_tokens, device=device,
                   cls_only=cls_only, ffn_act=FFN_ACTS[getattr(c, "hidden_act", "gelu")])

    def forward_cls(self, ids: torch.Tensor, mask: Optional[torch.Tensor] = None,
                    type_ids: Optional[torch.Tensor] = None, out: Optional[torch.Tensor] = None) -> torch.Tensor:
        assert ids.is_cuda and ids.dtype == torch.int32 and ids.is_contiguous()
        B, S = ids.shape
        if out is None:
            out = torch.empty((B, self.hidden), dtype=torch.float32, device=ids.device)
        if mask is not None:
            mask = mask.to(torch.int32).contiguous()
        if type_ids is not None:
            type_ids = type_ids.to(torch.int32).contiguous()
        check(self._L.ac_encoder_forward_cls(self.handle, ids.data_ptr(), ptr(mask), ptr(type_ids), B, S,
                                             out.data_ptr(), stream_ptr()), "ac_encoder_forward_cls")
        return out

    def last_hidden(self, B: int, S: int) -> torch.Tensor:
        out = torch.empty((B * S, self.hidden), dtype=torch.float32, device="cuda")
        check(self._L.ac_encoder_last_hidden(self.handle, out.data_ptr(), out.numel(), stream_ptr()),
              "ac_encoder_last_hidden")
        return out

    def attention(self, q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, mask: Optional[torch.Tensor] = None, *,
                  window: int = 0, cls_rows: bool = False, pad_fill: float = 0.0) -> torch.Tensor:
        """Parity entry: this encoder's attention stage alone (ac_encoder_attention).  q, k, v [B, S, heads, head_dim] are
        rounded to fp16 and laid out as the QKV epilogue leaves them (q | k rows; V transposed per (sequence, feature) with
        the keys padded to a multiple of 8, the pad keys holding pad_fill, which a correct kernel never lets through).
        Returns the context [B, S, heads, head_dim] fp16; with cls_rows only rows 0..127 of every sequence are computed."""
        B, S, heads, dh = q.shape
        assert heads == self.heads and heads * dh == self.hidden and k.shape == q.shape and v.shape == q.shape and q.is_cuda
        qk = torch.cat([q.reshape(B * S, self.hidden), k.reshape(B * S, self.hidden)], dim=1).to(torch.float16).contiguous()
        S_pad = (S + 7) // 8 * 8
        vT = torch.full((B, self.hidden, S_pad), pad_fill, dtype=torch.float16, device=q.device)
        vT[:, :, :S] = v.reshape(B, S, self.hidden).transpose(1, 2)
        if mask is not None:
            mask = mask.to(torch.int32).contiguous()
        ctx = torch.empty((B * S, self.hidden), dtype=torch.float16, device=q.device)
        check(self._L.ac_encoder_attention(self.handle, qk.data_ptr(), vT.data_ptr(), ptr(mask), B, S, window,
                                           1 if cls_rows else 0, ctx.data_ptr(), stream_ptr()), "ac_encoder_attention")
        return ctx.view(B, S, heads, dh)

    def projection(self, role: int, layer: int, B: int, S: int, a: torch.Tensor, y: Optional[torch.Tensor] = None,
                   stats: Optional[torch.Tensor] = None) -> tuple:
        """Parity entry: one projection role of layer `layer` alone (ac_encoder_projection, AC_PROJ_*), as the forward runs it.
        a [B*S, K] fp16 (K = E, H or I by role), y [B*S, H] fp32 residual sums, stats [B*S, 2] fp32 (mu, r) rows; all CUDA.
        Returns, by role: EMB (y, fp16 y); QKV (q | k [B*S, 2H], V^T [B*H, S_pad]); WO / W2 (y_new, fp16 y_new, stats of
        y_new [B*S, 2]); FFN1 / FFN1_ROWS (activations [B*S, I],)."""
        M, H, dev = B * S, self.hidden, a.device
        # the C entry copies M rows of each input: a tensor of another shape would be read out of bounds
        name = _PROJ_ROLES.get(role, f"role {role}")
        width = {AC_PROJ_EMB: self.embedding_size, AC_PROJ_W2: self.intermediate}.get(role, H)
        need = {"a": (a, (M, width))}
        if role in (AC_PROJ_QKV, AC_PROJ_WO, AC_PROJ_FFN1, AC_PROJ_W2):
            need["stats"] = (stats, (M, 2))
        if role in (AC_PROJ_WO, AC_PROJ_W2):
            need["y"] = (y, (M, H))
        for arg, (t, shape) in need.items():
            if t is None or tuple(t.shape) != shape:
                got = "None" if t is None else f"shape {tuple(t.shape)}"
                raise AdaptiveB200Error(f"Encoder.projection: {arg} is {got}; {name} needs {shape} (B={B} S={S})")
        for arg, (t, _) in need.items():
            if not t.is_cuda:
                raise AdaptiveB200Error(f"Encoder.projection: {arg} is on {t.device}; {name} needs CUDA tensors")
        a = a.to(torch.float16).contiguous()
        if y is not None:
            y = y.to(torch.float32).contiguous()
        if stats is not None:
            stats = stats.to(torch.float32).contiguous()
        new = lambda *shape, dt=torch.float16: torch.empty(shape, dtype=dt, device=dev)
        stats_out = None
        if role == AC_PROJ_EMB:
            outs = (new(M, H, dt=torch.float32), new(M, H))
        elif role == AC_PROJ_QKV:
            outs = (new(M, 2 * H), new(B * H, (S + 7) // 8 * 8))
        elif role in (AC_PROJ_WO, AC_PROJ_W2):
            stats_out = new(M, 2, dt=torch.float32)
            outs = (new(M, H, dt=torch.float32), new(M, H), stats_out)
        else:
            outs = (new(M, self.intermediate),)
        check(self._L.ac_encoder_projection(self.handle, layer, role, B, S, a.data_ptr(), ptr(y), ptr(stats),
                                            outs[0].data_ptr(), ptr(outs[1] if len(outs) > 1 else None), ptr(stats_out),
                                            stream_ptr()), "ac_encoder_projection")
        return outs

    def close(self):
        if getattr(self, "handle", None):
            self._L.ac_encoder_destroy(self.handle)
            self.handle = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def tokenizer_spec_struct(spec: dict):
    """(TokenizerSpec, arrays it points into) from tokenizer.wordpiece_spec's dict and the Unicode tables of its flags"""
    import numpy as np
    from .tokenizer import pack_strings, unicode_tables
    norm, cls, pool = unicode_tables(*spec["flags"])
    pool = pool if pool.size else np.zeros(1, dtype=np.uint32)
    words = list(spec["vocab"])
    vb, vo = pack_strings(words)
    vi = np.asarray([spec["vocab"][w] for w in words], dtype=np.int32)
    ab, ao = pack_strings([a for a, _ in spec["added"]])
    ai = np.asarray([i for _, i in spec["added"]] or [0], dtype=np.int32)
    keep = [norm, cls, pool, vb, vo, vi, ab, ao, ai]
    p = [a.ctypes.data for a in keep]
    st = TokenizerSpec(p[0], p[1], p[2], len(pool), p[3], p[4], p[5], len(words), p[6], p[7], p[8], len(spec["added"]),
                       spec["prefix"], len(spec["prefix"]), spec["cls_id"], spec["sep_id"], spec["pad_id"], spec["unk_id"],
                       spec["max_input_chars"])
    return st, keep


def bpe_spec_struct(spec: dict):
    """(BPETokenizerSpec, arrays it points into) from tokenizer.bpe_spec's dict and the codepoint classes"""
    import numpy as np
    from .tokenizer import bpe_classes, bpe_vocab_bytes, pack_strings
    cls = bpe_classes()
    words, wids = bpe_vocab_bytes(spec["vocab"])
    vo = np.zeros(len(words) + 1, dtype=np.int64)
    np.cumsum([len(w) for w in words], out=vo[1:])
    vb = np.frombuffer(b"".join(words) or b"\0", dtype=np.uint8)
    vi = np.asarray(wids, dtype=np.int32)
    bi = np.asarray(spec["byte_ids"], dtype=np.int32)
    mg = np.asarray(spec["merges"] or [(0, 0, 0)], dtype=np.int32).reshape(-1, 3)
    added = spec["added"]
    ab, ao = pack_strings([a[0] for a in added])
    ai = np.asarray([a[1] for a in added] or [0], dtype=np.int32)
    af = np.asarray([a[2] | a[3] << 1 | a[4] << 2 for a in added] or [0], dtype=np.uint8)
    keep = [cls, vb, vo, vi, bi, mg, ab, ao, ai, af]
    p = [a.ctypes.data for a in keep]
    st = BPETokenizerSpec(p[0], spec["split"], int(spec["prefix_space"]), int(spec["ignore_merges"]), p[1], p[2], p[3],
                          len(words), p[4], p[5], len(spec["merges"]), p[6], p[7], p[8], p[9], len(added),
                          spec["cls_id"], spec["sep_id"], spec["pad_id"])
    return st, keep


def unigram_spec_struct(spec: dict):
    """(UnigramTokenizerSpec, arrays it points into) from tokenizer.unigram_spec's dict and the codepoint classes"""
    import numpy as np
    from .tokenizer import pack_strings, unigram_classes
    cls = unigram_classes()
    def packed(blobs):
        off = np.zeros(len(blobs) + 1, dtype=np.int64)
        np.cumsum([len(x) for x in blobs], out=off[1:])
        return np.frombuffer(b"".join(blobs) or b"\0", dtype=np.uint8), off
    mk, mko = packed([k for k, _ in spec["charsmap"]])
    mv, mvo = packed([v for _, v in spec["charsmap"]])
    pb, po = packed([p for p, _ in spec["pieces"]])
    ps = np.asarray([sc for _, sc in spec["pieces"]], dtype=np.float64)
    added = spec["added"]
    ab, ao = pack_strings([a[0] for a in added])
    ai = np.asarray([a[1] for a in added] or [0], dtype=np.int32)
    af = np.asarray([a[2] | a[3] << 1 | a[4] << 2 for a in added] or [0], dtype=np.uint8)
    keep = [cls, mk, mko, mv, mvo, pb, po, ps, ab, ao, ai, af]
    p = [a.ctypes.data for a in keep]
    st = UnigramTokenizerSpec(p[0], p[1], p[2], p[3], p[4], len(spec["charsmap"]), spec["grow"], p[5], p[6], p[7],
                              len(spec["pieces"]), spec["unk_id"], p[8], p[9], p[10], p[11], len(added),
                              spec["cls_id"], spec["sep_id"], spec["pad_id"])
    return st, keep


class _DeviceTokenizer:
    """What every device tokenizer (WordPiece, BPE, Unigram) shares: the handle, one pinned H2D copy of the texts' offsets and
    bytes, the one readback of the batch's longest row, and the pack into [B, S] tensors."""
    _readback = 1                                   # int32 the call reads back: the longest row (BPE, Unigram: and the texts left)

    def _create(self, create, st, type_ids: bool, device):
        self._L = load_library()
        self.device = torch.device(device)
        self.type_ids = type_ids
        h = c_void_p()
        with torch.cuda.device(self.device):
            check(create(ctypes.byref(st), ctypes.byref(h)), create.__name__)
        self.handle = h
        self._host = torch.empty(0, dtype=torch.uint8).pin_memory()
        self._dev = torch.empty(0, dtype=torch.uint8, device=self.device)
        self._max_len_host = torch.zeros(self._readback, dtype=torch.int32).pin_memory()

    def _workspace_bytes(self, B: int, n_text: int, max_length: int) -> int:
        raise NotImplementedError

    def _left_rows(self, texts, max_length, tokens, lengths) -> int:
        """rows of the texts the kernels left to the host (BPE, Unigram); returns their longest length"""
        return 0

    def __call__(self, texts, max_length: int):
        """ids, mask, type_ids (None when the tokenizer emits none) [B, S] int32 on the device, S = the batch's longest; None
        when a text has no UTF-8 form (a lone surrogate), which the caller leaves to the host tokenizer."""
        try:
            enc = [t.encode("utf-8") for t in texts]
        except UnicodeEncodeError:
            return None
        B = len(enc)
        lens = [len(e) for e in enc]
        n_text = sum(lens)
        head = (8 * (B + 1) + 255) // 256 * 256            # int64 offsets, then the bytes, in one pinned buffer / one H2D copy
        total = head + n_text
        if self._host.numel() < total:
            self._host = torch.empty(int(total * 1.25) + 4096, dtype=torch.uint8).pin_memory()
            self._dev = torch.empty(self._host.numel(), dtype=torch.uint8, device=self.device)
        off = self._host[: 8 * (B + 1)].view(torch.int64)
        off[0] = 0
        torch.cumsum(torch.tensor(lens, dtype=torch.int64), 0, out=off[1:])
        mv = memoryview(self._host.numpy())
        mv[head:total] = b"".join(enc)
        with torch.cuda.device(self.device):
            self._dev[:total].copy_(self._host[:total], non_blocking=True)
            tokens = torch.empty((B, max_length), dtype=torch.int32, device=self.device)
            lengths = torch.empty(B + self._readback, dtype=torch.int32, device=self.device)
            ws = _workspace(self._workspace_bytes(B, n_text, max_length), self.device)
            check(self._L.ac_tokenize(self.handle, self._dev.data_ptr() + head, self._dev.data_ptr(), B, max_length,
                                      tokens.data_ptr(), lengths.data_ptr(), lengths.data_ptr() + 4 * B, ws.data_ptr(),
                                      ws.numel(), stream_ptr()), "ac_tokenize")
            self._max_len_host.copy_(lengths[B:], non_blocking=False)     # the one readback: the encoder needs S at launch
            S = int(self._max_len_host[0])
            if self._readback > 1 and int(self._max_len_host[1]):
                S = max(S, self._left_rows(texts, max_length, tokens, lengths))
            ids = torch.empty((B, S), dtype=torch.int32, device=self.device)
            mask = torch.empty_like(ids)
            tt = torch.empty_like(ids) if self.type_ids else None
            check(self._L.ac_tokenize_pack(self.handle, tokens.data_ptr(), lengths.data_ptr(), B, max_length, S, ids.data_ptr(),
                                           mask.data_ptr(), ptr(tt), stream_ptr()), "ac_tokenize_pack")
        return ids, mask, tt

    def close(self):
        if getattr(self, "handle", None):
            self._L.ac_tokenizer_destroy(self.handle)
            self.handle = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class WordPieceTokenizer(_DeviceTokenizer):
    """Owner of an ac_tokenizer handle: `tokenizer(texts, max_length=..., truncation=True, padding=True)` of a WordPiece
    tokenizer of the BERT shape (tokenizer.wordpiece_spec), computed on the device with identical ids."""

    def __init__(self, spec: dict, device="cuda"):
        st, keep = tokenizer_spec_struct(spec)
        self._create(load_library().ac_tokenizer_create, st, spec["type_ids"], device)
        del keep

    @classmethod
    def from_hf(cls, tokenizer, device="cuda"):
        """(WordPieceTokenizer, "") for a supported tokenizer, else (None, the reason)"""
        from .tokenizer import wordpiece_spec
        spec, why = wordpiece_spec(tokenizer)
        if spec is None:
            return None, why
        return cls(spec, device), ""

    def _workspace_bytes(self, B: int, n_text: int, max_length: int) -> int:
        nb = c_size_t()
        check(self._L.ac_tokenize_workspace_bytes(self.handle, B, ctypes.byref(nb)), "ac_tokenize_workspace_bytes")
        return nb.value


class _HandBackTokenizer(_DeviceTokenizer):
    """A device tokenizer whose kernels leave some texts (lengths = -1, max_len[1] = 1) to the host tokenizer: the handle's
    workspace depends on the text bytes, and the rows of the texts left are written before the pack."""
    _readback = 2

    def __init__(self, spec: dict, tokenizer, device="cuda"):
        st, keep = self._spec_struct(spec)
        self._create(self._create_fn(load_library()), st, spec["type_ids"], device)
        del keep
        self._hf = tokenizer

    @classmethod
    def from_hf(cls, tokenizer, device="cuda"):
        """(tokenizer, "") for a supported tokenizer, else (None, the reason)"""
        spec, why = cls._spec(tokenizer)
        if spec is None:
            return None, why
        return cls(spec, tokenizer, device), ""

    def _workspace_bytes(self, B: int, n_text: int, max_length: int) -> int:
        nb = c_size_t()
        check(self._L.ac_tokenize_workspace_bytes_text(self.handle, B, n_text, max_length, ctypes.byref(nb)),
              "ac_tokenize_workspace_bytes_text")
        return nb.value

    def _left_rows(self, texts, max_length, tokens, lengths) -> int:
        left = torch.nonzero(lengths[: len(texts)].cpu() < 0).flatten().tolist()
        rows = self._hf([texts[i] for i in left], max_length=max_length, truncation=True)["input_ids"]
        host = torch.zeros((len(left), max_length), dtype=torch.int32)
        for r, ids in enumerate(rows):
            host[r, : len(ids)] = torch.tensor(ids, dtype=torch.int32)
        idx = torch.tensor(left, dtype=torch.int64, device=self.device)
        tokens[idx] = host.to(self.device)
        lengths[idx] = torch.tensor([len(r) for r in rows], dtype=torch.int32).to(self.device)
        return max(len(r) for r in rows)


class BPETokenizer(_HandBackTokenizer):
    """Owner of an ac_tokenizer handle of a byte-level BPE tokenizer (RoBERTa, ModernBERT, EuroBERT; tokenizer.bpe_spec):
    `tokenizer(texts, max_length=..., truncation=True, padding=True)` computed on the device with identical ids.  A text with
    a kept word longer than AC_BPE_MAX_WORD bytes is tokenized by `tokenizer` itself, on the host."""
    _spec_struct = staticmethod(bpe_spec_struct)

    @staticmethod
    def _create_fn(L):
        return L.ac_tokenizer_create_bpe

    @staticmethod
    def _spec(tokenizer):
        from .tokenizer import bpe_spec
        return bpe_spec(tokenizer)


class UnigramTokenizer(_HandBackTokenizer):
    """Owner of an ac_tokenizer handle of a SentencePiece Unigram tokenizer of the XLM-RoBERTa shape (xlm-roberta-*, bge-m3,
    multilingual-e5-*, jina-embeddings-v3; tokenizer.unigram_spec): `tokenizer(texts, max_length=..., truncation=True,
    padding=True)` computed on the device with identical ids.  A text with a kept word longer than AC_UNIGRAM_MAX_WORD bytes
    is tokenized by `tokenizer` itself, on the host."""
    _spec_struct = staticmethod(unigram_spec_struct)

    @staticmethod
    def _create_fn(L):
        return L.ac_tokenizer_create_unigram

    @staticmethod
    def _spec(tokenizer):
        from .tokenizer import unigram_spec
        return unigram_spec(tokenizer)


def proto_class_scores(d, idx, row_class=None, n_classes: Optional[int] = None):
    """k <= 32: one thread per query; larger k (predict(): k = num_classes): one CTA per query, needs n_classes"""
    L = load_library()
    d = _f32c(d)
    idx = idx.contiguous()
    B, k = d.shape
    cls = torch.empty((B, k), dtype=torch.int32, device=d.device)
    sc = torch.empty((B, k), dtype=torch.float32, device=d.device)
    if k <= 32 and n_classes is None:
        check(L.ac_proto_class_scores(d.data_ptr(), idx.data_ptr(), ptr(row_class), B, k, cls.data_ptr(), sc.data_ptr(),
                                      stream_ptr()), "ac_proto_class_scores")
    else:
        assert n_classes is not None, "k > 32 needs the number of classes"
        check(L.ac_proto_class_scores_n(d.data_ptr(), idx.data_ptr(), ptr(row_class), B, k, int(n_classes), cls.data_ptr(),
                                        sc.data_ptr(), stream_ptr()), "ac_proto_class_scores_n")
    return cls, sc


def blend_dense(p_cls, p_score, head_probs, w_proto, w_head, kout: int):
    """predict() blend over all classes (classifier.py:446-480) -> (cls [B,kout] int32, score [B,kout])"""
    L = load_library()
    B, kp = p_cls.shape
    C = w_proto.numel()
    out_cls = torch.empty((B, kout), dtype=torch.int32, device=p_cls.device)
    out_sc = torch.empty((B, kout), dtype=torch.float32, device=p_cls.device)
    check(L.ac_blend_dense(p_cls.data_ptr(), _f32c(p_score).data_ptr(), kp, ptr(head_probs), B, C, _f32c(w_proto).data_ptr(),
                           ptr(w_head), kout, out_cls.data_ptr(), out_sc.data_ptr(), stream_ptr()), "ac_blend_dense")
    return out_cls, out_sc


def topk_desc(values: torch.Tensor, k: int):
    """-> (vals [B,k] descending, idx [B,k] int64); ties -> lower index."""
    L = load_library()
    values = _f32c(values)
    B, C = values.shape
    nbytes = c_size_t(0)
    check(L.ac_topk_desc_workspace_bytes(B, C, k, ctypes.byref(nbytes)), "ac_topk_desc_workspace_bytes")
    ws = _workspace(nbytes.value, values.device)
    neg = torch.empty((B, k), dtype=torch.float32, device=values.device)
    idx = torch.empty((B, k), dtype=torch.int64, device=values.device)
    check(L.ac_topk_desc(values.data_ptr(), B, C, k, neg.data_ptr(), idx.data_ptr(), ws.data_ptr(), ws.numel(),
                         stream_ptr()), "ac_topk_desc")
    return -neg, idx


def blend_topk(p_cls, p_score, h_idx, h_val, k: int, w_proto: float = 0.7, w_head: float = 0.3):
    """h_val: head probabilities (descending) for h_idx, or None for prototype-only."""
    L = load_library()
    B = p_cls.shape[0]
    kh = 0 if h_idx is None else h_idx.shape[1]
    neg = (-h_val).contiguous() if h_val is not None else None
    out_cls = torch.empty((B, k), dtype=torch.int32, device=p_cls.device)
    out_sc = torch.empty((B, k), dtype=torch.float32, device=p_cls.device)
    check(L.ac_blend_topk(p_cls.data_ptr(), p_score.data_ptr(), ptr(h_idx), ptr(neg), B, k, kh, w_proto, w_head,
                          out_cls.data_ptr(), out_sc.data_ptr(), stream_ptr()), "ac_blend_topk")
    return out_cls, out_sc


def launch_count() -> int:
    return int(load_library().ac_launch_count())


def profile_enable(on: bool):
    check(load_library().ac_profile_enable(1 if on else 0), "ac_profile_enable")


def profile_read(cls: int):
    ms, fl, by = ctypes.c_double(0), ctypes.c_double(0), ctypes.c_double(0)
    n = ctypes.c_longlong(0)
    check(load_library().ac_profile_read(cls, ctypes.byref(ms), ctypes.byref(fl), ctypes.byref(by), ctypes.byref(n)),
          "ac_profile_read")
    return {"ms": ms.value, "flops": fl.value, "bytes": by.value, "launches": n.value}


class _ExternalCudaBuffer:
    """__cuda_array_interface__ view of a device buffer owned by a C handle (fp32, row-major)"""

    def __init__(self, ptr_value: int, shape, device):
        self.__cuda_array_interface__ = {"shape": tuple(shape), "typestr": "<f4", "data": (int(ptr_value), False), "version": 3,
                                         "strides": None}


class Pipeline:
    """ids -> E -> K -> class scores -> H -> blend, device or host (pinned) buffers at the boundary."""

    def __init__(self, enc: Encoder, P: torch.Tensor, max_B: int, S: int, k: int, *, head: Optional[dict] = None,
                 row_class: Optional[torch.Tensor] = None, p_sqnorm: Optional[torch.Tensor] = None,
                 p_half: Optional[torch.Tensor] = None, row_offset: int = 0, shards: int = 1):
        L = load_library()
        self._L = L
        self.enc, self.P, self.p_sqnorm, self.row_class, self.p_half = enc, _f32c(P), p_sqnorm, row_class, p_half
        self.head = head
        self.max_B, self.S, self.k = max_B, S, k
        hp = head_params_struct(head) if head is not None else None
        h = c_void_p()
        check(L.ac_pipeline_create(enc.handle, self.P.data_ptr(), ptr(p_sqnorm), ptr(p_half), ptr(row_class), self.P.shape[0],
                                   self.P.shape[1], ctypes.byref(hp) if hp is not None else None, max_B, S, k,
                                   row_offset, shards, ctypes.byref(h)), "ac_pipeline_create")
        self.handle = h
        self.shards = shards
        self.out_cls_host = torch.empty((max_B, k), dtype=torch.int32).pin_memory()
        self.out_score_host = torch.empty((max_B, k), dtype=torch.float32).pin_memory()
        self.out_cls = torch.empty((max_B, k), dtype=torch.int32, device=self.P.device)
        self.out_score = torch.empty((max_B, k), dtype=torch.float32, device=self.P.device)

    def predict_device(self, ids_dev: torch.Tensor, mask_dev: Optional[torch.Tensor] = None):
        B = ids_dev.shape[0]
        check(self._L.ac_pipeline_predict_device(self.handle, ids_dev.data_ptr(), ptr(mask_dev), B,
                                                 self.out_cls.data_ptr(), self.out_score.data_ptr(), stream_ptr()),
              "ac_pipeline_predict_device")
        return self.out_cls[:B], self.out_score[:B]

    def predict_host(self, ids_host: torch.Tensor):
        assert (not ids_host.is_cuda) and ids_host.dtype == torch.int32 and ids_host.is_contiguous()
        B = ids_host.shape[0]
        check(self._L.ac_pipeline_predict_host(self.handle, ids_host.data_ptr(), B, self.out_cls_host.data_ptr(),
                                               self.out_score_host.data_ptr(), stream_ptr()), "ac_pipeline_predict_host")
        return self.out_cls_host[:B], self.out_score_host[:B]

    # ---- phases of the row-sharded multi-GPU step (parallel.ShardedPipeline runs the collectives between them)
    def encode(self, ids_dev: torch.Tensor, mask_dev: Optional[torch.Tensor] = None) -> torch.Tensor:
        """E (+ the head forked onto the side stream); returns a [B, D] view of the pipeline's embedding buffer"""
        B = ids_dev.shape[0]
        check(self._L.ac_pipeline_encode(self.handle, ids_dev.data_ptr(), ptr(mask_dev), B, stream_ptr()), "ac_pipeline_encode")
        if getattr(self, "_emb_view", None) is None:
            p = c_void_p()
            check(self._L.ac_pipeline_embeddings(self.handle, ctypes.byref(p)), "ac_pipeline_embeddings")
            D = self.P.shape[1]
            # wrap the handle-owned device buffer without copying (lifetime = the pipeline's)
            self._emb_store = _ExternalCudaBuffer(p.value, (self.max_B, D), self.P.device)
            self._emb_view = torch.as_tensor(self._emb_store, device=self.P.device)
        return self._emb_view[:B]

    def search_shard(self, q_all: torch.Tensor, G: int, B: int, packed: torch.Tensor) -> None:
        check(self._L.ac_pipeline_search_shard(self.handle, _f32c(q_all).data_ptr(), G, B, packed.data_ptr(), stream_ptr()),
              "ac_pipeline_search_shard")

    def finish_sharded(self, received: torch.Tensor, G: int, B: int):
        check(self._L.ac_pipeline_finish_sharded(self.handle, received.data_ptr(), G, B, self.out_cls.data_ptr(),
                                                 self.out_score.data_ptr(), stream_ptr()), "ac_pipeline_finish_sharded")
        return self.out_cls[:B], self.out_score[:B]

    def knn_stats(self, reset: bool = True) -> dict:
        """search statistics since the last reset (synchronises): queries that took the second tensor pass, queries whose
        candidate buffer overflowed (results not exact -> redo with AC_KNN_EXACT), max rows collected, searches"""
        out = (ctypes.c_int32 * 4)()
        check(self._L.ac_pipeline_knn_stats(self.handle, out, 1 if reset else 0, stream_ptr()), "ac_pipeline_knn_stats")
        return {"second_pass_queries": int(out[0]), "overflow_queries": int(out[1]), "max_collected": int(out[2]), "searches": int(out[3])}

    def debug_views(self, B: int):
        """(emb [B,D], knn_d [B,k], knn_i [B,k]) of the last call."""
        D = self.P.shape[1]
        emb = torch.empty((B, D), dtype=torch.float32, device=self.P.device)
        kd = torch.empty((B, self.k), dtype=torch.float32, device=self.P.device)
        ki = torch.empty((B, self.k), dtype=torch.int64, device=self.P.device)
        check(self._L.ac_pipeline_debug_copy(self.handle, B, emb.data_ptr(), kd.data_ptr(), ki.data_ptr(), stream_ptr()),
              "ac_pipeline_debug_copy")
        return emb, kd, ki

    def close(self):
        if getattr(self, "handle", None):
            self._L.ac_pipeline_destroy(self.handle)
            self.handle = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
