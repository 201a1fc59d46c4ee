"""Patched `LlamaAttention.forward` / `MistralAttention.forward` for HF transformers 5.x.

Restates what the reference's 36 patched forwards do around the eviction call (they differ only in which
`init_*` they call): q/k/v projection, RoPE, [prefill] attention over the FULL K/V + `kv_cluster.update_kv` +
cache update, [decode] append + attention over the compacted cache.
  reference: pyramidkv/llama_model.py:87-205 (eager), :208-320 (sdpa), :323-453 (flash);
             pyramidkv/mistral_model.py:1772-1878, :1881-2023, :2026-2188.

Differences by design (H100-first):
  * K/V are never `repeat_kv`-expanded in HBM (llama_model.py:158-159): the eviction kernels read each kv head
    once and write the per-query-head compacted cache directly.
  * The decode step is one fused launch (in-place append + attention) instead of torch.cat + transposes + attention.
  * Prefill is detected by "this layer's cache is empty" instead of the per-module kv_seq_len counter
    (llama_model.py:165) — same behaviour, no dependence on prepare_inputs_for_generation having run.
The dense prefill attention itself is not on the eviction hot path: it goes through HF's own attention
interface (sdpa / flash_attention_2 / eager), exactly like the reference calls flash_attn_func on the full K/V.
"""
from __future__ import annotations

from typing import Callable, Optional

import torch
from transformers.modeling_utils import ALL_ATTENTION_FUNCTIONS

from .cache import (PkvBatchCacheLayer, PkvCacheLayer, PkvRaggedCacheLayer, decode_heavy, decode_window, gqa_shared,
                    install_layer, kv_cache_dtype, layer_is_empty, quantize_caches_fp8)
from .kv_cluster import INIT_BY_METHOD, flush_pending

DEFAULT_DECODE_RESERVE = 256   # rows of head-room behind the compacted prompt (grows by doubling)


def _dense_attention(module, modeling, query_states, key_states, value_states, attention_mask, **kwargs):
    """Full-sequence attention through HF's interface (library code; handles GQA without materialising repeats)."""
    interface: Callable = ALL_ATTENTION_FUNCTIONS.get_interface(module.config._attn_implementation, modeling.eager_attention_forward)
    extra = {}
    if "mistral" in modeling.__name__:
        extra["sliding_window"] = getattr(module.config, "sliding_window", None)
    out, weights = interface(module, query_states, key_states, value_states, attention_mask,
                             dropout=0.0 if not module.training else module.attention_dropout,
                             scaling=module.scaling, **extra, **kwargs)
    return out, weights


def last_layer_idx(module) -> int:
    """The layer whose prefill forward evicts the parked layers: the model's last one. (A runner that holds only a slice of the
    layers - pipeline.PipelineRunner - flushes explicitly after its own last layer.)"""
    return int(getattr(module.config, "num_hidden_layers", 0)) - 1


def _has_padding(attention_mask) -> bool:
    """True when a prepared attention mask ([b, 1, q, kv], bool or additive) hides a key from the LAST query row of some
    sample, i.e. the batch is padded. The eviction (like the reference's: its clusters ignore attention_mask,
    pyramidkv_utils.py:197) scores every row, so padded batches would keep and attend pad tokens."""
    if attention_mask is None or not torch.is_tensor(attention_mask) or attention_mask.dim() != 4:
        return False
    row = attention_mask[:, 0, -1, :]
    return bool((~row).any()) if row.dtype == torch.bool else bool((row < 0).any())


def _maybe_quantize(module, past_key_values, cluster) -> None:
    """Knob pkv_kv_cache_dtype = "fp8_e4m3": once the LAST layer's prefill has filled its cache (and the parked evictions
    are flushed), every layer's compacted cache becomes a PkvFp8CacheLayer in one launch. The conversion runs after the
    eviction, so it covers every compacting method."""
    if kv_cache_dtype(module.config) is None or module.layer_idx != last_layer_idx(module):
        return
    if getattr(past_key_values, "_pkv_pending", None):
        flush_pending(past_key_values._pkv_pending, cluster.backend)
    quantize_caches_fp8(past_key_values, cluster.backend)


def make_forward(method: str, modeling, original_forward):
    init_cluster = INIT_BY_METHOD[method]

    def forward(self, hidden_states: torch.Tensor, position_embeddings=None, attention_mask: Optional[torch.Tensor] = None,
                past_key_values=None, **kwargs):
        if past_key_values is None:      # no cache => nothing to evict; the stock forward is exact
            return original_forward(self, hidden_states, position_embeddings, attention_mask, None, **kwargs)

        init_cluster(self)               # llama_model.py:101 — knobs are re-read from self.config on every call
        cluster = self.kv_cluster

        input_shape = hidden_states.shape[:-1]
        bsz, q_len = input_shape
        hidden_shape = (*input_shape, -1, self.head_dim)
        query_states = self.q_proj(hidden_states).view(hidden_shape).transpose(1, 2)   # [b, Hq, q, D], physically [b, q, Hq, D]
        key_states = self.k_proj(hidden_states).view(hidden_shape).transpose(1, 2)     # [b, Hkv, q, D]
        value_states = self.v_proj(hidden_states).view(hidden_shape).transpose(1, 2)
        cos, sin = position_embeddings
        if getattr(self.config, "pkv_fused_rope", False) and not torch.is_grad_enabled():
            # SURVEY.md §8 f2: one in-place launch (pkv_rope_inplace) instead of HF's ten elementwise launches and four
            # full-size temporaries; bit-identical results. Opt-in knob on the shared config, like the reference's knobs.
            static = getattr(past_key_values, "_pkv_static", None)
            if q_len > 1 and getattr(static, "spec", False):
                # the verify step of speculative decoding: one launch over the B*Q token rows (q [Hq, B*Q, D], cos / sin
                # [B*Q, D]: per-sequence positions)
                cluster.backend.rope_inplace(query_states.transpose(1, 2).view(bsz * q_len, -1, self.head_dim).transpose(0, 1),
                                             key_states.transpose(1, 2).view(bsz * q_len, -1, self.head_dim).transpose(0, 1),
                                             cos.expand(bsz, -1, -1).reshape(bsz * q_len, -1),
                                             sin.expand(bsz, -1, -1).reshape(bsz * q_len, -1))
            elif q_len == 1 and bsz > 1:
                # a batched decode step: one launch with the batch axis as the token axis (q [Hq, B, D], cos / sin [B, D])
                cs = (cos, sin) if cos.shape[0] == bsz else (cos.expand(bsz, -1, -1).contiguous(), sin.expand(bsz, -1, -1).contiguous())
                cluster.backend.rope_inplace(query_states[:, :, 0, :].transpose(0, 1), key_states[:, :, 0, :].transpose(0, 1),
                                             cs[0][:, 0, :], cs[1][:, 0, :])
            else:
                for b in range(bsz):
                    cluster.backend.rope_inplace(query_states[b], key_states[b], cos[b if cos.shape[0] > 1 else 0], sin[b if sin.shape[0] > 1 else 0])
        else:
            query_states, key_states = modeling.apply_rotary_pos_emb(query_states, key_states, cos, sin)
        num_q_heads = query_states.shape[1]

        if layer_is_empty(past_key_values, self.layer_idx):
            # ---------------- prefill (llama_model.py:165-168) ----------------
            if bsz > 1 and _has_padding(attention_mask):
                raise NotImplementedError("pyramidkv_b200: padded batches are not supported (the eviction ignores attention_mask like "
                                          "the reference, whose README lists batch inference as unsupported); run prompts one by one")
            self.kv_seq_len = q_len
            attn_output, attn_weights = _dense_attention(self, modeling, query_states, key_states, value_states,
                                                         attention_mask, **kwargs)
            cluster.inputs_ready = True      # the launch in front of the eviction is the dense attention: it only reads q / k / v
            reserve = int(getattr(self.config, "pkv_decode_reserve", DEFAULT_DECODE_RESERVE))
            window = decode_window(self.config)
            heavy = decode_heavy(self.config)   # knob pkv_decode_heavy: heavy hitters in that window
            if window is not None:       # knob pkv_decode_window: at most R decoded rows behind the prompt
                reserve = min(reserve, window)
            group = num_q_heads // key_states.shape[1] if gqa_shared(self.config) else 1
            if group > 1 and getattr(cluster, "ragged", False):
                raise NotImplementedError(f"pkv_gqa_shared: {method} sets a budget per QUERY head, which one cache per KV head "
                                          "cannot hold (AdaKV / HeadKV with per-KV-head budgets are not built)")
            if getattr(cluster, "ragged", False) and cluster.compressed(q_len):
                # AdaKV / HeadKV (llama_model.py:2317-2320): per-head budgets -> padded buffers + per-head row counts
                if bsz != 1:
                    raise NotImplementedError("AdaKV / HeadKV are batch size 1 (pyramidkv_utils.py:723)")
                k_buf, v_buf, head_rows = cluster.evict_ragged(query_states[0], key_states[0], value_states[0], reserve=reserve)
                if window is not None:   # the per-(sequence, head) row-count form carries the window
                    layer = PkvBatchCacheLayer(k_buf[None], v_buf[None], [[int(r) for r in head_rows]], [q_len], window=window,
                                               heavy=heavy)
                else:
                    layer = PkvRaggedCacheLayer(k_buf[None], v_buf[None], head_rows, seen_tokens=q_len)
                install_layer(past_key_values, self.layer_idx, layer)
                _maybe_quantize(self, past_key_values, cluster)
                attn_output = attn_output.reshape(*input_shape, -1).contiguous()
                return self.o_proj(attn_output), attn_weights
            # Deferred eviction (knob pkv_defer_eviction, default on): a layer's eviction reads only this layer's q / k / v and
            # nothing reads the compacted cache before the first decode step, so the window methods park their evictions and the
            # LAST layer evicts all of them in one pass (pkv_evict_prefill_batch: four launches per 32 layers instead of three
            # per layer; K / V of the parked layers stay alive until then: 134 MB per layer for Llama-3-8B at 32K).
            pending = None
            if bsz == 1 and getattr(self.config, "pkv_defer_eviction", True):
                pending = getattr(past_key_values, "_pkv_pending", None)
                if pending is None:
                    pending = past_key_values._pkv_pending = []
            bufs = [cluster.evict_into(query_states[b], key_states[b], value_states[b], reserve=reserve, pending=pending,
                                       **({"gqa_shared": True} if group > 1 else {})) for b in range(bsz)]
            if pending and self.layer_idx == last_layer_idx(self):
                flush_pending(pending, cluster.backend)
            rows = bufs[0][2]
            if bsz == 1:
                k_buf, v_buf = bufs[0][0][None], bufs[0][1][None]
            else:
                k_buf, v_buf = torch.stack([t[0] for t in bufs]), torch.stack([t[1] for t in bufs])
            if group > 1 or window is not None:
                # knob pkv_gqa_shared: one cache per KV head; knob pkv_decode_window: a ring of decoded rows. Both are held in
                # the per-(sequence, head) row-count form
                layer = PkvBatchCacheLayer(k_buf, v_buf, [[rows] * k_buf.shape[1]] * bsz, [q_len] * bsz, group=group, window=window,
                                           heavy=heavy)
            else:
                layer = PkvCacheLayer(k_buf, v_buf, rows, seen_tokens=q_len)
            install_layer(past_key_values, self.layer_idx, layer)
            _maybe_quantize(self, past_key_values, cluster)
        else:
            # ---------------- decode (llama_model.py:169-170) ----------------
            if getattr(past_key_values, "_pkv_pending", None):      # a prefill that stopped before its last layer (never with generate())
                flush_pending(past_key_values._pkv_pending, cluster.backend)
            layer = past_key_values.layers[self.layer_idx]
            if not isinstance(layer, PkvCacheLayer):
                raise RuntimeError("pyramidkv_b200: the cache of this layer was not created by the patched prefill "
                                   "(mixing a stock DynamicCache prefill with the patched decode is unsupported)")
            self.kv_seq_len = getattr(self, "kv_seq_len", layer.seen_tokens) + q_len
            attn_weights = None
            static = getattr(past_key_values, "_pkv_static", None)
            if q_len == 1:
                # one launch per layer: the new row is appended in place and attended (the cache form picks the kernel).
                # In the static loop (generate.StaticDecoder) the buffers were reserved up front, the row count includes the
                # device step counter and StaticDecoder.finish() settles the Python bookkeeping.
                if static is None:
                    layer.reserve(1)
                out = layer.decode(cluster.backend, query_states[:, :, 0, :], key_states[:, :, 0, :], value_states[:, :, 0, :],
                                   static, self.scaling)
                if static is None:
                    layer.advance(1)
                attn_output = out[:, None]
            elif static is not None and getattr(static, "spec", False):
                # the verify step of speculative decoding (generate.SpeculativeDecoder): the Q new rows of every sequence
                # stored and attended causally in one launch per layer, q / k / v read in their [b, q, H, D] layout
                attn_output = layer.decode_multi(cluster.backend, query_states.transpose(1, 2), key_states.transpose(1, 2),
                                                 value_states.transpose(1, 2), static, self.scaling)
            else:
                # several new tokens after the prefill (not produced by generate()): generic append + library attention
                keys, values = layer.update(key_states, value_states)
                T = keys.shape[2]
                mask = torch.ones(q_len, T, dtype=torch.bool, device=keys.device).tril(diagonal=T - q_len)
                attn_output = torch.nn.functional.scaled_dot_product_attention(
                    query_states, keys, values, attn_mask=mask, scale=self.scaling).transpose(1, 2)

        attn_output = attn_output.reshape(*input_shape, -1).contiguous()
        attn_output = self.o_proj(attn_output)
        return attn_output, attn_weights

    forward._pkv_method = method
    forward._pkv_original = original_forward
    return forward
