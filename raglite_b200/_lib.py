"""ctypes binding of the C-ABI in include/raglite_b200.h.

There is no CPU fallback: if the shared library cannot be loaded (or built), every entry point
raises.  Device pointers are passed as integers (``tensor.data_ptr()``), the stream as the raw
``cudaStream_t`` of ``torch.cuda.current_stream()``.
"""

from __future__ import annotations

import ctypes as C
import threading

from . import _build

RL_METRIC = {"cosine": 0, "dot": 1, "l2": 2, "l1": 3}
RL_ALGO = {"auto": 0, "fp32": 1, "tcgen05": 2}
RL_FLAG_REUSE_THRESHOLDS = 1
RL_FLAG_TIME_KERNELS = 2
RL_FLAG_COUNT_UNFILTERED = 4
RL_STATUS_CAND_OVERFLOW = 1
RL_STATUS_TIE_OVERFLOW = 2
RL_STATUS_QUERY_NONFINITE = 4
RL_MAX_SURVIVORS = 4096   # finalize window (include/raglite_b200.h)

EXPORTS = [
    "rl_version", "rl_last_error", "rl_device_info", "rl_row_stats", "rl_row_stats_f16", "rl_chunk_row_map", "rl_adapter_apply",
    "rl_maxsim_workspace_bytes", "rl_maxsim_topk", "rl_maxsim_count_at_least", "rl_maxsim_unfiltered_bound", "rl_maxsim_stats", "rl_maxsim_kernel_times", "rl_maxsim_release", "rl_maxsim_copy_dump", "rl_maxsim_copy_eps", "rl_maxsim_copy_candidates", "rl_topk_merge", "rl_topk_merge_packed", "rl_hits_packed_bytes", "rl_row_mask", "rl_rrf_fuse", "rl_span_collate", "rl_best_vectors", "rl_adapter_targets",
    "rl_segment_mean_pool", "rl_xenc_linear_image_bytes", "rl_xenc_pack_linear", "rl_xenc_linear",
    "rl_xenc_workspace_bytes", "rl_xenc_score", "rl_xenc_attention", "rl_xenc_encode", "rl_xenc_encode_attention",
    "rl_xenc_embed_ln", "rl_xenc_add_ln", "rl_xenc_cls_head", "rl_bm25_stats", "rl_bm25_workspace_bytes",
    "rl_bm25_packed_bytes", "rl_bm25_topk_global", "rl_bm25_merge_packed", "rl_tsrank_topk_global",
    "rl_sat_token_logits", "rl_sat_workspace_bytes", "rl_sat_char_probas", "rl_sentence_partition_workspace_bytes",
    "rl_sentence_partition", "rl_chunklet_partition_workspace_bytes", "rl_chunklet_partition",
    "rl_chunk_similarities_workspace_bytes", "rl_chunk_similarities", "rl_chunk_partition_workspace_bytes",
    "rl_chunk_partition", "rl_fts_workspace_bytes", "rl_fts_mark", "rl_fts_stem", "rl_fts_verify", "rl_fts_stem_bytes",
    "rl_fts_term_keys", "rl_dequant_rows_f16", "rl_xenc_qlinear_image_bytes", "rl_xenc_pack_qlinear",
    "rl_xenc_concat_qlinear", "rl_xenc_linear_q", "rl_chunk_embedding_blend", "rl_llm_workspace_bytes", "rl_llm_forward",
    "rl_llm_qgemv_workspace_bytes", "rl_llm_qgemv", "rl_llm_embed", "rl_llm_qk_norm_rope", "rl_llm_attention_workspace_bytes",
    "rl_llm_attention", "rl_llm_sample_workspace_bytes", "rl_llm_sample", "rl_grammar_token_index",
    "rl_llm_sample_masked",
]
_SIZE_T_RESULTS = ("rl_maxsim_workspace_bytes", "rl_xenc_linear_image_bytes", "rl_xenc_workspace_bytes",
                   "rl_hits_packed_bytes", "rl_bm25_workspace_bytes", "rl_bm25_packed_bytes", "rl_sat_workspace_bytes",
                   "rl_sentence_partition_workspace_bytes", "rl_chunklet_partition_workspace_bytes",
                   "rl_chunk_similarities_workspace_bytes", "rl_chunk_partition_workspace_bytes", "rl_fts_workspace_bytes",
                   "rl_xenc_qlinear_image_bytes", "rl_llm_workspace_bytes", "rl_llm_qgemv_workspace_bytes",
                   "rl_llm_attention_workspace_bytes", "rl_llm_sample_workspace_bytes")
RL_LLM_MAX_EOG = 8
RL_LLM_NO_TOKEN = -1
RL_XENC_IMAGE_F16 = 0
RL_XENC_IMAGE_QUANT = 1


class ScanParams(C.Structure):
    _fields_ = [
        ("E", C.c_void_p), ("inv_norm", C.c_void_p), ("sq_norm", C.c_void_p), ("row_chunk", C.c_void_p),
        ("row_stats", C.c_void_p), ("row_allowed", C.c_void_p),
        ("n_rows", C.c_int64), ("ld", C.c_int64), ("chunk_base", C.c_int64),
        ("d", C.c_int32), ("max_vecs_per_chunk", C.c_int32),
        ("Q", C.c_void_p),
        ("B", C.c_int32), ("metric", C.c_int32), ("k", C.c_int32), ("num_hits", C.c_int32), ("algo", C.c_int32),
        ("flags", C.c_uint32), ("sample_stride", C.c_int32), ("cand_cap", C.c_int32), ("e_dtype", C.c_int32),
        ("rows_unit_scale", C.c_int32), ("row_alive", C.c_void_p),
    ]


class ScanStats(C.Structure):
    _fields_ = [
        ("launches", C.c_int32), ("sample_stride", C.c_int32), ("cand_cap", C.c_int32), ("algo", C.c_int32),
        ("n_sample_rows", C.c_int64), ("cand_total", C.c_int64), ("cand_max", C.c_int64),
        ("survivors_total", C.c_int64), ("survivors_max", C.c_int64),
    ]


class XencLayer(C.Structure):
    _fields_ = [(n, C.c_void_p) for n in ("qkv_img", "qkv_bias", "o_img", "o_bias", "ln1_g", "ln1_b", "up_img", "up_bias",
                                           "down_img", "down_bias", "ln2_g", "ln2_b")] + [
        (n, C.c_int32) for n in ("qkv_type", "o_type", "up_type", "down_type")]


class XencWeights(C.Structure):
    _fields_ = [
        ("n_layers", C.c_int32), ("hidden", C.c_int32), ("n_heads", C.c_int32), ("ffn", C.c_int32), ("vocab", C.c_int32),
        ("max_pos", C.c_int32), ("type_vocab", C.c_int32), ("ln_eps", C.c_float),
        ("word_emb", C.c_void_p), ("pos_emb", C.c_void_p), ("type_emb", C.c_void_p), ("emb_ln_g", C.c_void_p),
        ("emb_ln_b", C.c_void_p), ("layers", C.POINTER(XencLayer)), ("pooler_w", C.c_void_p), ("pooler_b", C.c_void_p),
        ("cls_w", C.c_void_p), ("cls_b", C.c_void_p), ("n_labels", C.c_int32),
    ]


RL_LLM_MAX_PARTS = 32


class LlmLinear(C.Structure):   # rl_llm_linear
    _fields_ = [("parts", C.c_void_p * RL_LLM_MAX_PARTS), ("n_parts", C.c_int32), ("N", C.c_int32), ("K", C.c_int32)]


class LlmLayer(C.Structure):   # rl_llm_layer
    _fields_ = [(n, LlmLinear) for n in ("q", "k", "v", "o", "gate", "up", "down")] + [
        (n, C.c_void_p) for n in ("attn_norm", "q_norm", "k_norm", "ffn_norm")]


class LlmWeights(C.Structure):   # rl_llm_weights
    _fields_ = [(n, C.c_int32) for n in ("n_layers", "hidden", "n_head", "n_kv", "ffn", "vocab", "n_ctx")] + [
        ("eps", C.c_float), ("rope_base", C.c_float), ("token_embd", LlmLinear), ("output", LlmLinear),
        ("output_norm", C.c_void_p), ("layers", C.POINTER(LlmLayer))]


_lock = threading.Lock()
_lib: C.CDLL | None = None


def _declare(lib: C.CDLL) -> None:
    vp, i32, i64 = C.c_void_p, C.c_int32, C.c_int64
    lib.rl_version.restype = C.c_int
    lib.rl_last_error.restype = C.c_char_p
    lib.rl_device_info.argtypes = [C.POINTER(C.c_int), C.POINTER(C.c_int), C.POINTER(C.c_int), C.POINTER(C.c_size_t)]
    lib.rl_row_stats.argtypes = [vp, i64, i32, i64, vp, vp, vp, vp]
    lib.rl_row_stats_f16.argtypes = [vp, i64, i32, i64, vp, vp, vp, vp]
    lib.rl_chunk_row_map.argtypes = [vp, i64, vp, vp]
    lib.rl_adapter_apply.argtypes = [vp, vp, vp, i32, i32, i32, vp]
    lib.rl_maxsim_workspace_bytes.argtypes = [C.POINTER(ScanParams)]
    lib.rl_maxsim_workspace_bytes.restype = C.c_size_t
    lib.rl_maxsim_topk.argtypes = [C.POINTER(ScanParams), vp, vp, vp, vp, vp, C.c_size_t, vp]
    lib.rl_maxsim_count_at_least.argtypes = [C.POINTER(ScanParams), vp, C.c_int, vp, vp, C.c_size_t, vp]
    lib.rl_maxsim_unfiltered_bound.argtypes = [C.POINTER(ScanParams), vp, vp, vp]
    lib.rl_maxsim_stats.argtypes = [C.POINTER(ScanParams), vp, C.POINTER(ScanStats), vp]
    lib.rl_maxsim_kernel_times.argtypes = [vp, C.POINTER(C.c_float)]
    lib.rl_maxsim_release.argtypes = [vp]
    lib.rl_row_mask.argtypes = [vp, vp, vp, i64, vp, vp]
    lib.rl_maxsim_copy_dump.argtypes = [C.POINTER(ScanParams), vp, vp, C.POINTER(C.c_int64), vp]
    lib.rl_maxsim_copy_eps.argtypes = [C.POINTER(ScanParams), vp, vp, vp]
    lib.rl_maxsim_copy_candidates.argtypes = [C.POINTER(ScanParams), vp, vp, vp, vp, vp, vp, vp]
    lib.rl_topk_merge.argtypes = [vp, vp, vp, i32, i32, i32, i32, i32, vp, vp, vp, vp]
    lib.rl_hits_packed_bytes.argtypes = [i32, i32, i32]
    lib.rl_hits_packed_bytes.restype = C.c_size_t
    lib.rl_topk_merge_packed.argtypes = [vp, i64, i32, i32, i32, i32, i32, vp, vp, vp, vp]
    lib.rl_best_vectors.argtypes = [vp, i32, i64, i32, vp, vp, i32, i32, vp, vp, vp, vp]
    lib.rl_adapter_targets.argtypes = [vp, vp, i32, i32, i32, vp, C.c_double, vp, vp, vp, vp]
    lib.rl_rrf_fuse.argtypes = [vp, vp, i32, i32, i32, C.c_double, i32, vp, vp, vp, vp]
    lib.rl_span_collate.argtypes = [vp, i32, i32, vp, vp, vp, vp, vp, i64, vp, i32, vp, vp, vp, vp, vp, vp, vp]
    lib.rl_segment_mean_pool.argtypes = [vp, i64, i32, vp, vp, i32, i32, vp, vp]
    lib.rl_chunk_embedding_blend.argtypes = [vp, i64, vp, vp, i64, i64, i32, C.c_uint16, C.c_uint16, vp, vp]
    lib.rl_xenc_linear_image_bytes.argtypes = [i32, i32]
    lib.rl_xenc_linear_image_bytes.restype = C.c_size_t
    lib.rl_xenc_pack_linear.argtypes = [vp, i32, i32, vp, vp]
    lib.rl_xenc_linear.argtypes = [vp, vp, vp, vp, i32, i32, i32, i32, vp]
    lib.rl_xenc_workspace_bytes.argtypes = [C.POINTER(XencWeights), i32]
    lib.rl_xenc_workspace_bytes.restype = C.c_size_t
    lib.rl_xenc_score.argtypes = [C.POINTER(XencWeights), vp, vp, vp, vp, i32, i32, i32, vp, vp, vp, C.c_size_t, vp]
    lib.rl_xenc_attention.argtypes = [vp, vp, i32, i32, i32, i32, i32, vp, vp, C.c_size_t, vp]
    lib.rl_xenc_encode.argtypes = [C.POINTER(XencWeights), vp, vp, vp, vp, i32, i32, i32, vp, vp, C.c_size_t, vp]
    lib.rl_xenc_encode_attention.argtypes = [vp, vp, i32, i32, i32, i32, i32, vp, vp, C.c_size_t, vp]
    lib.rl_xenc_embed_ln.argtypes = [C.POINTER(XencWeights), vp, vp, vp, i32, vp, vp]
    lib.rl_xenc_add_ln.argtypes = [vp, vp, vp, vp, C.c_float, i32, i32, i32, vp, vp]
    lib.rl_xenc_cls_head.argtypes = [C.POINTER(XencWeights), vp, vp, i32, vp, vp, vp]
    lib.rl_bm25_stats.argtypes = [vp, vp, vp, vp, i64, i64, vp, vp, vp]
    lib.rl_bm25_workspace_bytes.argtypes = [i64, i32]
    lib.rl_bm25_workspace_bytes.restype = C.c_size_t
    lib.rl_bm25_packed_bytes.argtypes = [i32, i32]
    lib.rl_bm25_packed_bytes.restype = C.c_size_t
    lib.rl_bm25_topk_global.argtypes = [vp, vp, vp, vp, vp, i64, i64, vp, vp, vp, i32, i32, C.c_double, C.c_double, i64, vp,
                                        vp, C.c_size_t, vp]
    lib.rl_bm25_merge_packed.argtypes = [vp, i32, i32, i32, vp, vp, vp, vp]
    lib.rl_tsrank_topk_global.argtypes = [vp, vp, vp, i64, i64, vp, vp, vp, i32, i32, i64, vp, vp, C.c_size_t, vp]
    lib.rl_sat_token_logits.argtypes = [vp, i64, i32, vp, vp, i32, vp, vp]
    lib.rl_sat_workspace_bytes.argtypes = [i64, i32, i32]
    lib.rl_sat_workspace_bytes.restype = C.c_size_t
    lib.rl_sat_char_probas.argtypes = [vp, i32, vp, vp, vp, i32, i64, i64, vp, vp, vp, vp, vp, vp, vp, vp, vp, C.c_size_t,
                                       vp]
    lib.rl_sentence_partition_workspace_bytes.argtypes = [i64]
    lib.rl_sentence_partition_workspace_bytes.restype = C.c_size_t
    lib.rl_sentence_partition.argtypes = [vp, vp, vp, vp, vp, i32, i64, vp, vp, vp, vp, C.c_size_t, vp]
    lib.rl_chunklet_partition_workspace_bytes.argtypes = [i64, i32]
    lib.rl_chunklet_partition.argtypes = [vp, vp, vp, vp, vp, i32, i64, vp, vp, vp, vp, C.c_size_t, vp]
    lib.rl_chunk_similarities_workspace_bytes.argtypes = [i64]
    lib.rl_chunk_similarities.argtypes = [vp, i32, i64, i32, vp, i32, i64, vp, vp, vp, vp, vp, C.c_size_t, vp]
    lib.rl_chunk_partition_workspace_bytes.argtypes = [i64, i32]
    lib.rl_chunk_partition.argtypes = [vp, vp, vp, vp, i32, i64, vp, vp, vp, vp, C.c_size_t, vp]
    lib.rl_fts_workspace_bytes.argtypes = [i64]
    lib.rl_fts_mark.argtypes = [vp, i64, vp, vp, vp, C.c_size_t, vp]
    lib.rl_fts_stem.argtypes = [vp, vp, i64, vp, i32, i32, vp, vp, vp, vp]
    lib.rl_fts_verify.argtypes = [vp, vp, vp, vp, vp, vp, i64, vp, vp]
    lib.rl_fts_stem_bytes.argtypes = [vp, vp, vp, vp, vp, i64, vp, vp, vp]
    lib.rl_fts_term_keys.argtypes = [vp, vp, i64, vp, i64, vp, vp]
    lib.rl_dequant_rows_f16.argtypes = [i32, vp, i64, i32, vp, vp]
    lib.rl_xenc_qlinear_image_bytes.argtypes = [i32, i32, i32]
    lib.rl_xenc_pack_qlinear.argtypes = [i32, vp, i32, i32, vp, vp]
    lib.rl_xenc_concat_qlinear.argtypes = [C.POINTER(C.c_void_p), i32, vp, vp]
    lib.rl_xenc_linear_q.argtypes = [vp, vp, vp, vp, i32, i32, i32, i32, vp]
    vp, i32, f32 = C.c_void_p, C.c_int32, C.c_float
    lib.rl_llm_workspace_bytes.argtypes = [C.POINTER(LlmWeights), i32]
    lib.rl_llm_forward.argtypes = [C.POINTER(LlmWeights), vp, i32, i32, vp, vp, vp, vp, C.c_size_t, vp]
    lib.rl_llm_qgemv_workspace_bytes.argtypes = [i32, i32]
    lib.rl_llm_qgemv.argtypes = [C.POINTER(LlmLinear), vp, vp, i32, vp, C.c_size_t, vp]
    lib.rl_llm_embed.argtypes = [C.POINTER(LlmLinear), vp, i32, vp, vp]
    lib.rl_llm_qk_norm_rope.argtypes = [vp, i32, i32, i32, i32, vp, vp, f32, f32, i32, vp, vp, vp, vp]
    lib.rl_llm_attention_workspace_bytes.argtypes = [i32, i32, i32, i32, i32]
    lib.rl_llm_attention.argtypes = [vp, vp, vp, i32, i32, i32, i32, i32, vp, vp, C.c_size_t, vp]
    lib.rl_llm_sample_workspace_bytes.argtypes = [i32]
    lib.rl_llm_sample.argtypes = [vp, i32, vp, i32, f32, i32, f32, f32, f32, f32, vp, vp, C.c_size_t, vp]
    lib.rl_grammar_token_index.argtypes = [vp, i32, vp, vp, i32, vp, vp]
    lib.rl_llm_sample_masked.argtypes = [vp, i32, vp, i32, f32, i32, f32, f32, f32, f32, vp, i32, vp,
                                         C.POINTER(C.c_int32), i32, vp, vp, vp, C.c_size_t, vp]
    for name in EXPORTS:
        if name != "rl_last_error":
            getattr(lib, name).restype = C.c_size_t if name in _SIZE_T_RESULTS else C.c_int


def load(*, build_if_missing: bool = True) -> C.CDLL:
    """Load (building first if needed) the CUDA library.  Raises if that is impossible."""
    global _lib  # noqa: PLW0603
    with _lock:
        if _lib is None:
            path = _build.LIB_PATH
            if build_if_missing and _build.is_stale():
                path = _build.build()
            if not path.exists():
                raise RuntimeError(f"{path} is missing and could not be built; raglite_b200 has no CPU fallback")
            lib = C.CDLL(str(path))
            _declare(lib)
            _lib = lib
        return _lib


class RagliteB200Error(RuntimeError):
    pass


def check(rc: int, what: str) -> None:
    if rc != 0:
        msg = load().rl_last_error().decode(errors="replace")
        if rc == -1:
            raise ValueError(f"{what}: {msg}")
        raise RagliteB200Error(f"{what} failed ({rc}): {msg}")
