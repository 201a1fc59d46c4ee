"""ctypes binding of libpkv.so (include/pkv.h). Fails loudly: there is no CPU or PyTorch fallback."""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libpkv.so")

PKV_OK, PKV_ERR_INVALID_ARG, PKV_ERR_UNSUPPORTED_DTYPE, PKV_ERR_UNSUPPORTED_ARCH = 0, 1, 2, 3
PKV_ERR_CUDA, PKV_ERR_WORKSPACE, PKV_ERR_UNSUPPORTED, PKV_ERR_POOLING = 4, 5, 6, 7

METHODS = {"pyramidkv": 0, "snapkv": 1, "h2o": 2, "streamingllm": 3, "l2norm": 4}
POOLING = {"avgpool": 0, "maxpool": 1}
SCORE_KERNELS = {"auto": 0, "mma": 1, "tcgen05": 2}

# every symbol include/pkv.h declares (checked by tests/test_abi.py without a GPU)
EXPORTS = [
    "pkv_version", "pkv_last_error", "pkv_launch_count", "pkv_layer_budget", "pkv_evict_workspace_layout",
    "pkv_evict_workspace_bytes", "pkv_evict_prefill", "pkv_stage_scores", "pkv_stage_pool", "pkv_stage_topk",
    "pkv_stage_gather", "pkv_decode_workspace_bytes", "pkv_decode_attn", "pkv_decode_attn_graph", "pkv_cache_append", "pkv_host_pick_rows", "pkv_debug_read_stamps", "pkv_rope_inplace", "pkv_update_flatten_view", "pkv_adakv_scratch_bytes", "pkv_adakv_counts",
    "pkv_ragged_place_window", "pkv_decode_attn_ragged", "pkv_evict_single_launch", "pkv_stage_scan_pool",
    "pkv_evict_prefill_batch", "pkv_evict_batch_supported", "pkv_stage_batch", "pkv_decode_attn_batch",
    "pkv_decode_attn_batch_fp8", "pkv_cache_quantize_fp8", "pkv_decode_attn_batch_gqa", "pkv_decode_attn_batch_gqa_fp8",
    "pkv_evict_pooled_kv_offset", "pkv_cache_install", "pkv_sample_tokens", "pkv_decode_attn_window",
    "pkv_decode_attn_heavy", "pkv_decode_heavy_workspace_bytes",
    "pkv_token_logprobs", "pkv_sample_tokens_penalized", "pkv_token_rules", "pkv_sample_tokens_constrained",
    "pkv_beam_candidates", "pkv_beam_step", "pkv_cache_reorder",
]
RULE_BIAS, RULE_BAN, RULE_BAD, RULE_STOP = 1, 2, 4, 8     # pkv_token_rules_desc.flags[b]
SEQ_BIAS, SEQ_BAD, SEQ_STOP = 0, 1, 2                     # pkv_token_rules_desc.seq_kind
FLAG_GQA_SHARED = 128          # pkv_evict_desc.flags: one compacted cache per KV head


class EvictDesc(C.Structure):
    _fields_ = [
        ("struct_bytes", C.c_uint32), ("method", C.c_int32), ("dtype", C.c_int32), ("pooling", C.c_int32),
        ("kernel_size", C.c_int32), ("num_q_heads", C.c_int32), ("num_kv_heads", C.c_int32), ("head_dim", C.c_int32),
        ("window", C.c_int32), ("device", C.c_int32), ("seq_len", C.c_int64), ("top_k", C.c_int64),
        ("q", C.c_void_p), ("q_stride_h", C.c_int64), ("q_stride_s", C.c_int64),
        ("k", C.c_void_p), ("k_stride_h", C.c_int64), ("k_stride_s", C.c_int64),
        ("v", C.c_void_p), ("v_stride_h", C.c_int64), ("v_stride_s", C.c_int64),
        ("k_cache", C.c_void_p), ("v_cache", C.c_void_p), ("cache_stride_h", C.c_int64),
        ("idx_out", C.c_void_p), ("workspace", C.c_void_p), ("workspace_bytes", C.c_uint64),
        ("flags", C.c_uint32), ("reserved", C.c_uint32),
    ]


class WsLayout(C.Structure):
    _fields_ = [
        ("total_bytes", C.c_uint64), ("logits_off", C.c_uint64), ("partial_off", C.c_uint64),
        ("pooled_off", C.c_uint64), ("idx32_off", C.c_uint64), ("h2o_stats_off", C.c_uint64),
        ("h2o_acc_off", C.c_uint64), ("s_pad", C.c_int64), ("n_slots", C.c_int64), ("nw", C.c_int64),
        ("pooled_pitch", C.c_int64), ("fused_off", C.c_uint64),
    ]


class DecodeDesc(C.Structure):
    _fields_ = [
        ("struct_bytes", C.c_uint32), ("dtype", C.c_int32), ("num_q_heads", C.c_int32), ("num_kv_heads", C.c_int32),
        ("head_dim", C.c_int32), ("device", C.c_int32), ("length", C.c_int64),
        ("q", C.c_void_p), ("k_new", C.c_void_p), ("v_new", C.c_void_p),
        ("k_cache", C.c_void_p), ("v_cache", C.c_void_p), ("cache_stride_h", C.c_int64),
        ("out", C.c_void_p), ("workspace", C.c_void_p), ("workspace_bytes", C.c_uint64),
        ("softmax_scale", C.c_float), ("reserved", C.c_uint32),
    ]


class DecodeWindow(C.Structure):
    _fields_ = [
        ("struct_bytes", C.c_uint32), ("num_seqs", C.c_int32), ("cache_stride_b", C.c_int64),
        ("gqa_shared", C.c_int32), ("reserved", C.c_int32),
        ("rows", C.c_void_p), ("prompt_rows", C.c_void_p), ("step_dev", C.c_void_p), ("max_length", C.c_int64),
        ("k_scale", C.c_void_p), ("v_scale", C.c_void_p), ("scale_stride_h", C.c_int64), ("scale_stride_b", C.c_int64),
        ("window", C.c_int64),
    ]


class DecodeHeavy(C.Structure):
    _fields_ = [
        ("struct_bytes", C.c_uint32), ("reserved", C.c_int32), ("heavy", C.c_int64),
        ("scores", C.c_void_p), ("gen", C.c_void_p), ("victim", C.c_void_p), ("scratch", C.c_void_p), ("scratch_bytes", C.c_uint64),
    ]


class RopeDesc(C.Structure):
    _fields_ = [
        ("struct_bytes", C.c_uint32), ("dtype", C.c_int32), ("num_q_heads", C.c_int32), ("num_kv_heads", C.c_int32),
        ("head_dim", C.c_int32), ("device", C.c_int32), ("seq_len", C.c_int64),
        ("q", C.c_void_p), ("q_stride_h", C.c_int64), ("q_stride_s", C.c_int64),
        ("k", C.c_void_p), ("k_stride_h", C.c_int64), ("k_stride_s", C.c_int64),
        ("cos", C.c_void_p), ("sin", C.c_void_p), ("cs_stride_s", C.c_int64),
    ]


SAMPLE_ADVANCE = 1            # pkv_sample_desc.flags: token_index[b] += 1 after the draw


class SampleDesc(C.Structure):
    _fields_ = [
        ("struct_bytes", C.c_uint32), ("dtype", C.c_int32), ("device", C.c_int32), ("batch", C.c_int32),
        ("vocab", C.c_int64), ("logits", C.c_void_p), ("logits_stride", C.c_int64),
        ("temperature", C.c_void_p), ("top_k", C.c_void_p), ("top_p", C.c_void_p), ("seed", C.c_void_p),
        ("token_index", C.c_void_p), ("tokens", C.c_void_p), ("tokens_stride", C.c_int64), ("column", C.c_int64),
        ("flags", C.c_uint32), ("reserved", C.c_uint32),
    ]


class SamplePenalty(C.Structure):
    _fields_ = [
        ("struct_bytes", C.c_uint32), ("reserved", C.c_uint32),
        ("repetition_penalty", C.c_void_p), ("presence_penalty", C.c_void_p), ("frequency_penalty", C.c_void_p),
        ("min_p", C.c_void_p), ("prompt_mask", C.c_void_p), ("counts", C.c_void_p), ("stride", C.c_int64),
    ]


class TokenRulesDesc(C.Structure):
    _fields_ = [
        ("struct_bytes", C.c_uint32), ("device", C.c_int32), ("batch", C.c_int32), ("vocab", C.c_int32),
        ("history", C.c_void_p), ("history_stride", C.c_int64), ("history_len", C.c_void_p), ("prompt_len", C.c_void_p),
        ("flags", C.c_void_p), ("ngram", C.c_void_p), ("min_new_tokens", C.c_void_p), ("n_seq", C.c_void_p),
        ("seq_off", C.c_void_p), ("seq_kind", C.c_void_p), ("seq_bias", C.c_void_p), ("seq_stride", C.c_int64),
        ("seq_tokens", C.c_void_p), ("tokens_stride", C.c_int64), ("eos", C.c_void_p), ("n_eos", C.c_int32),
        ("reserved", C.c_int32), ("append", C.c_void_p), ("append_stride", C.c_int64), ("append_column", C.c_int64),
        ("bias", C.c_void_p), ("bias_stride", C.c_int64), ("ban", C.c_void_p), ("ban_stride", C.c_int64),
        ("stop", C.c_void_p),
    ]


class SampleRules(C.Structure):
    _fields_ = [
        ("struct_bytes", C.c_uint32), ("reserved", C.c_uint32), ("flags", C.c_void_p),
        ("bias", C.c_void_p), ("bias_stride", C.c_int64), ("ban", C.c_void_p), ("ban_stride", C.c_int64),
    ]


class LogprobsDesc(C.Structure):
    _fields_ = [
        ("struct_bytes", C.c_uint32), ("dtype", C.c_int32), ("device", C.c_int32), ("batch", C.c_int32),
        ("vocab", C.c_int64), ("logits", C.c_void_p), ("logits_stride", C.c_int64),
        ("tokens", C.c_void_p), ("tokens_stride", C.c_int64), ("tokens_column", C.c_int64),
        ("top_n", C.c_int32), ("flags", C.c_uint32), ("cursor", C.c_void_p), ("column", C.c_int64),
        ("logprob", C.c_void_p), ("logprob_stride", C.c_int64),
        ("top_ids", C.c_void_p), ("top_logprobs", C.c_void_p), ("top_stride", C.c_int64),
    ]


MAX_TOP_LOGPROBS = 20         # pkv_logprobs_desc.top_n


class BeamStepDesc(C.Structure):
    _fields_ = [
        ("struct_bytes", C.c_uint32), ("device", C.c_int32), ("num_prompts", C.c_int32), ("num_beams", C.c_int32),
        ("top_k", C.c_int32), ("cand_rows_per_prompt", C.c_int32), ("n_eos", C.c_int32), ("early_stopping", C.c_int32),
        ("max_steps", C.c_int32), ("step_offset", C.c_int32), ("step", C.c_void_p), ("cand_lp", C.c_void_p),
        ("cand_id", C.c_void_p), ("eos", C.c_void_p), ("scale", C.c_void_p), ("running", C.c_void_p),
        ("pool_score", C.c_void_p), ("pool_step", C.c_void_p), ("pool_parent", C.c_void_p), ("pool_token", C.c_void_p),
        ("pool_done", C.c_void_p), ("heuristic", C.c_void_p), ("done", C.c_void_p), ("bp_token", C.c_void_p),
        ("bp_parent", C.c_void_p), ("cp", C.c_void_p), ("next_token", C.c_void_p), ("parent", C.c_void_p),
        ("diverge", C.c_void_p),
    ]


MAX_BEAMS, MAX_BEAM_CANDIDATES = 16, 80   # PKV_MAX_BEAMS, PKV_MAX_BEAM_CANDIDATES


class PkvError(RuntimeError):
    def __init__(self, code: int, msg: str):
        super().__init__(f"libpkv error {code}: {msg}")
        self.code = code


_lib = None


def lib() -> C.CDLL:
    """Load libpkv.so. Raises if it has not been built — the eviction path has no other implementation."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(
            f"{LIB_PATH} is missing. Build it with `python -m pyramidkv_b200.build` (needs nvcc; targets sm_90a). "
            "pyramidkv_b200 has no CPU/PyTorch fallback for the eviction path.")
    L = C.CDLL(LIB_PATH)
    i32, i64, u64, p = C.c_int, C.c_int64, C.c_uint64, C.c_void_p
    L.pkv_version.restype = i32
    L.pkv_last_error.restype = C.c_char_p
    L.pkv_launch_count.restype = u64
    L.pkv_host_pick_rows.argtypes = [p, i64, i64, i64, C.c_int32, C.c_int32, i64, p, i64, p]
    L.pkv_host_pick_rows.restype = i32
    L.pkv_debug_read_stamps.argtypes = [C.POINTER(u64), i32]
    L.pkv_debug_read_stamps.restype = i32
    L.pkv_layer_budget.argtypes = [i32, i64, i64, i32, i32, i64, i32, C.POINTER(i64), C.POINTER(i32)]
    L.pkv_layer_budget.restype = i32
    L.pkv_evict_workspace_layout.argtypes = [C.POINTER(EvictDesc), C.POINTER(WsLayout)]
    L.pkv_evict_workspace_layout.restype = i32
    L.pkv_evict_workspace_bytes.argtypes = [C.POINTER(EvictDesc)]
    L.pkv_evict_workspace_bytes.restype = u64
    L.pkv_evict_pooled_kv_offset.argtypes = [C.POINTER(EvictDesc), C.POINTER(u64)]
    L.pkv_evict_pooled_kv_offset.restype = i32
    for name in ("pkv_evict_prefill", "pkv_stage_scores", "pkv_stage_pool", "pkv_stage_topk", "pkv_stage_gather", "pkv_stage_scan_pool"):
        fn = getattr(L, name)
        fn.argtypes = [C.POINTER(EvictDesc), p]
        fn.restype = i32
    L.pkv_evict_single_launch.argtypes = [C.POINTER(EvictDesc)]
    L.pkv_evict_single_launch.restype = i32
    L.pkv_evict_prefill_batch.argtypes = [C.POINTER(EvictDesc), i32, p]      # contiguous array of descriptors
    L.pkv_evict_prefill_batch.restype = i32
    L.pkv_stage_batch.argtypes = [C.POINTER(EvictDesc), i32, i32, p]
    L.pkv_stage_batch.restype = i32
    L.pkv_evict_batch_supported.argtypes = [C.POINTER(EvictDesc), i32]
    L.pkv_evict_batch_supported.restype = i32
    L.pkv_decode_workspace_bytes.argtypes = [C.POINTER(DecodeDesc)]
    L.pkv_decode_workspace_bytes.restype = u64
    for name in ("pkv_decode_attn", "pkv_cache_append"):
        fn = getattr(L, name)
        fn.argtypes = [C.POINTER(DecodeDesc), p]
        fn.restype = i32
    L.pkv_adakv_scratch_bytes.argtypes = [C.c_int32]
    L.pkv_adakv_scratch_bytes.restype = u64
    L.pkv_adakv_counts.argtypes = [C.POINTER(EvictDesc), i64, C.c_int32, p, u64, p, p]
    L.pkv_adakv_counts.restype = i32
    L.pkv_ragged_place_window.argtypes = [C.POINTER(EvictDesc), p, p]
    L.pkv_ragged_place_window.restype = i32
    L.pkv_decode_attn_ragged.argtypes = [C.POINTER(DecodeDesc), p, p, i64, p]
    L.pkv_decode_attn_ragged.restype = i32
    L.pkv_update_flatten_view.argtypes = [p, p, p, p, p, C.c_int32, C.c_int32, C.c_int32, p]
    L.pkv_update_flatten_view.restype = i32
    L.pkv_rope_inplace.argtypes = [C.POINTER(RopeDesc), p]
    L.pkv_rope_inplace.restype = i32
    L.pkv_decode_attn_graph.argtypes = [C.POINTER(DecodeDesc), p, i64, p]
    L.pkv_decode_attn_graph.restype = i32
    L.pkv_decode_attn_batch.argtypes = [C.POINTER(DecodeDesc), C.c_int32, i64, p, p, i64, p]
    L.pkv_decode_attn_batch.restype = i32
    L.pkv_decode_attn_batch_fp8.argtypes = [C.POINTER(DecodeDesc), C.c_int32, i64, p, p, i64, p, p, i64, i64, p]
    L.pkv_decode_attn_batch_fp8.restype = i32
    L.pkv_decode_attn_batch_gqa.argtypes = [C.POINTER(DecodeDesc), C.c_int32, i64, p, p, i64, p]
    L.pkv_decode_attn_batch_gqa.restype = i32
    L.pkv_decode_attn_batch_gqa_fp8.argtypes = [C.POINTER(DecodeDesc), C.c_int32, i64, p, p, i64, p, p, i64, i64, p]
    L.pkv_decode_attn_batch_gqa_fp8.restype = i32
    L.pkv_decode_attn_window.argtypes = [C.POINTER(DecodeDesc), C.POINTER(DecodeWindow), p]
    L.pkv_decode_attn_window.restype = i32
    L.pkv_decode_attn_heavy.argtypes = [C.POINTER(DecodeDesc), C.POINTER(DecodeWindow), C.POINTER(DecodeHeavy), p]
    L.pkv_decode_attn_heavy.restype = i32
    L.pkv_decode_heavy_workspace_bytes.argtypes = [C.c_int32, C.c_int32, i64]
    L.pkv_decode_heavy_workspace_bytes.restype = u64
    # tables: src / dst / scales [2*layers] pointers, capacities and rows [layers] int64, rows_dev [layers] pointers or NULL
    L.pkv_cache_quantize_fp8.argtypes = [C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32, p, p, p, p, p, p, p, p]
    L.pkv_cache_quantize_fp8.restype = i32
    # elem_bytes, num_seqs, num_heads, head_dim, device, num_layers, slot, then the tables (src, dst, src_scales, dst_scales
    # [2*layers] pointers; capacities and rows [layers] int64; rows_dev, dst_rows [layers] pointers), step_dev, stream
    L.pkv_cache_install.argtypes = [C.c_int32] * 7 + [p] * 11
    L.pkv_cache_install.restype = i32
    L.pkv_sample_tokens.argtypes = [C.POINTER(SampleDesc), p]
    L.pkv_sample_tokens.restype = i32
    L.pkv_sample_tokens_penalized.argtypes = [C.POINTER(SampleDesc), C.POINTER(SamplePenalty), p]
    L.pkv_sample_tokens_penalized.restype = i32
    L.pkv_token_rules.argtypes = [C.POINTER(TokenRulesDesc), p]
    L.pkv_token_rules.restype = i32
    L.pkv_sample_tokens_constrained.argtypes = [C.POINTER(SampleDesc), C.POINTER(SamplePenalty), C.POINTER(SampleRules), p]
    L.pkv_sample_tokens_constrained.restype = i32
    L.pkv_token_logprobs.argtypes = [C.POINTER(LogprobsDesc), p]
    L.pkv_token_logprobs.restype = i32
    L.pkv_beam_candidates.argtypes = [C.c_int32, C.c_int32, C.c_int32, C.c_int64, p, C.c_int64, C.c_int32] + [p] * 5
    L.pkv_beam_candidates.restype = i32
    L.pkv_beam_step.argtypes = [C.POINTER(BeamStepDesc), p]
    L.pkv_beam_step.restype = i32
    L.pkv_cache_reorder.argtypes = [C.c_int32] * 8 + [p] * 9 + [C.c_int32, p]
    L.pkv_cache_reorder.restype = i32
    if L.pkv_version() != 3:
        raise RuntimeError(f"libpkv ABI version {L.pkv_version()} != 3; rebuild with `python -m pyramidkv_b200.build --force`")
    _lib = L
    return L


def last_error() -> str:
    return lib().pkv_last_error().decode(errors="replace")


def check(rc: int) -> None:
    """Map a pkv_status to the exception the reference would raise for the same condition."""
    if rc == PKV_OK:
        return
    msg = last_error()
    if rc == PKV_ERR_POOLING:
        raise ValueError("Pooling method not supported")          # pyramidkv_utils.py:237
    if rc == PKV_ERR_INVALID_ARG:
        raise ValueError(msg)
    if rc in (PKV_ERR_UNSUPPORTED, PKV_ERR_UNSUPPORTED_DTYPE):
        raise NotImplementedError(msg)
    raise PkvError(rc, msg)


def launch_count() -> int:
    return int(lib().pkv_launch_count())
