"""Layer-sharded WHOLE-MODEL runner: BASELINE.json configs[4] (Llama-3-70B, PyramidKV budget 2048, 32K ctx, "HF device_map
layer-sharded across 2/4/8 x GPUs") through the real plugin.

The reference reaches several GPUs only through accelerate's `device_map="auto"` (run_longbench.py:390): consecutive decoder
layers on consecutive GPUs inside ONE process, hooks moving the hidden state with `.to(device)`, one GPU busy at a time.
The form of the same split here: one process per GPU (torchrun), rank r owns the contiguous layers
`sharding.layer_ranges(L, world)[r]` (embedding on rank 0, final norm + lm_head on the last rank), the hidden state crosses
each stage boundary with ONE point-to-point transfer (NCCL send/recv over NVLink / NVSwitch; gloo in the CPU tests) and the
sampled token comes back with one broadcast. Eviction, the compacted cache and decode attention stay local to the layer's
GPU — the eviction path needs no collective (SURVEY.md §8e). Weights are random-init (no checkpoints offline), seeded PER
COMPONENT so that every world size builds the same model and a 140 GB model never has to exist in one process.
"""
from __future__ import annotations

import time
from dataclasses import dataclass, field
from typing import List, Optional

import torch
import torch.distributed as dist

from .runner import ARCHS
from .sharding import layer_ranges


@dataclass
class Stage:
    config: object
    family: str
    first_layer: int
    layers: List[torch.nn.Module]
    rotary: torch.nn.Module
    embed: Optional[torch.nn.Module] = None          # rank 0
    norm: Optional[torch.nn.Module] = None           # last rank
    lm_head: Optional[torch.nn.Module] = None        # last rank
    extras: dict = field(default_factory=dict)


def _init_like_hf(module: torch.nn.Module, seed: int, std: float) -> None:
    """HF `_init_weights`: Linear / Embedding weights ~ N(0, initializer_range), norm weights 1 — from a per-component seed."""
    torch.manual_seed(seed)
    for m in module.modules():
        if isinstance(m, (torch.nn.Linear, torch.nn.Embedding)):
            m.weight.data.normal_(mean=0.0, std=std)
            if getattr(m, "bias", None) is not None:
                m.bias.data.zero_()


def make_config(arch: str, attn_implementation: str, device: torch.device, max_positions: int = 65536):
    import transformers
    family, hidden, inter, layers, heads, kv, hd, vocab, theta = ARCHS[arch]
    kw = dict(hidden_size=hidden, intermediate_size=inter, num_hidden_layers=layers, num_attention_heads=heads,
              num_key_value_heads=kv, head_dim=hd, vocab_size=vocab, rope_theta=theta, max_position_embeddings=max_positions)
    cfg = transformers.LlamaConfig(**kw) if family == "llama" else transformers.MistralConfig(sliding_window=None, **kw)
    cfg._attn_implementation = "eager" if attn_implementation in ("eager", "None") or device.type == "cpu" else "sdpa"
    return family, cfg


def build_stage(arch: str, rank: int, world: int, device: torch.device, dtype: torch.dtype = torch.bfloat16,
                attn_implementation: str = "sdpa", seed: int = 42) -> Stage:
    """Materialise only this rank's share of the model directly on its device."""
    family, cfg = make_config(arch, attn_implementation, device)
    if family == "llama":
        import transformers.models.llama.modeling_llama as M
        Layer, Norm, Rot = M.LlamaDecoderLayer, M.LlamaRMSNorm, M.LlamaRotaryEmbedding
    else:
        import transformers.models.mistral.modeling_mistral as M
        Layer, Norm, Rot = M.MistralDecoderLayer, M.MistralRMSNorm, M.MistralRotaryEmbedding
    a, b = layer_ranges(cfg.num_hidden_layers, world)[rank]
    old = torch.get_default_dtype()
    torch.set_default_dtype(dtype)
    try:
        with torch.device(device):
            layers = []
            for l in range(a, b):
                layer = Layer(cfg, l).eval()
                _init_like_hf(layer, seed + 1 + l, cfg.initializer_range)
                layers.append(layer)
            stage = Stage(cfg, family, a, layers, Rot(config=cfg))
            if rank == 0:
                stage.embed = torch.nn.Embedding(cfg.vocab_size, cfg.hidden_size).eval()
                _init_like_hf(stage.embed, seed + 100_003, cfg.initializer_range)
            if rank == world - 1:
                stage.norm = Norm(cfg.hidden_size, eps=cfg.rms_norm_eps).eval()
                stage.lm_head = torch.nn.Linear(cfg.hidden_size, cfg.vocab_size, bias=False).eval()
                _init_like_hf(stage.lm_head, seed + 100_019, cfg.initializer_range)
    finally:
        torch.set_default_dtype(old)
    return stage


class PipelineRunner:
    """Greedy generation over the layer-sharded model. Every rank calls the same methods in the same order."""

    def __init__(self, stage: Stage, group=None):
        from transformers import DynamicCache
        if getattr(stage.config, "pkv_kv_cache_dtype", None) not in (None, "auto"):
            raise NotImplementedError("the FP8 compacted cache (pkv_kv_cache_dtype) is converted by the model's last layer in one "
                                      "launch; the layer-sliced pipeline flushes per rank and keeps the 16-bit cache")
        if getattr(stage.config, "pkv_gqa_shared", False):
            raise NotImplementedError("the GQA-shared cache (pkv_gqa_shared) is installed in the batched row-count form that the "
                                      "layer-sliced pipeline does not decode; it keeps the per-query-head cache")
        if getattr(stage.config, "pkv_decode_window", None) is not None or getattr(stage.config, "pkv_decode_heavy", None) is not None:
            raise NotImplementedError("the decode window (pkv_decode_window) holds every layer in the batched row-count form "
                                      "that the layer-sliced pipeline does not decode")
        self.stage, self.group = stage, group
        self.rank = dist.get_rank(group) if dist.is_initialized() else 0
        self.world = dist.get_world_size(group) if dist.is_initialized() else 1
        p = next(iter(stage.layers[0].parameters())) if stage.layers else (stage.embed or stage.lm_head).weight
        self.device, self.dtype = p.device, p.dtype
        self.cache = DynamicCache(config=stage.config)
        self.seen = 0

    def reset(self) -> None:
        from transformers import DynamicCache
        self.cache = DynamicCache(config=self.stage.config)
        self.seen = 0

    def _mask(self, q_len: int):
        # sdpa takes the causal flag itself (attention_mask None); HF's eager attention needs the additive mask tensor
        if q_len == 1 or self.stage.config._attn_implementation != "eager":
            return None
        m = torch.full((q_len, q_len), torch.finfo(self.dtype).min, dtype=self.dtype, device=self.device).triu(1)
        return m[None, None]

    @torch.no_grad()
    def step(self, ids: Optional[torch.Tensor], q_len: int) -> torch.Tensor:
        """One forward over q_len new tokens (`ids` [1, q_len] is read on rank 0 only). Returns the next token [1, 1] on every rank."""
        st, cfg = self.stage, self.stage.config
        pos = torch.arange(self.seen, self.seen + q_len, device=self.device)[None]
        if self.rank == 0:
            h = st.embed(ids.to(self.device))
        else:
            h = torch.empty(1, q_len, cfg.hidden_size, dtype=self.dtype, device=self.device)
            dist.recv(h, src=self.rank - 1, group=self.group)
        pos_emb = st.rotary(h, position_ids=pos)
        mask = self._mask(q_len)
        for layer in st.layers:
            h = layer(h, attention_mask=mask, position_embeddings=pos_emb, position_ids=pos, past_key_values=self.cache, use_cache=True)
        if getattr(self.cache, "_pkv_pending", None):        # this stage's parked evictions: all of its layers in one pass
            from .kv_cluster import flush_pending
            flush_pending(self.cache._pkv_pending)
        self.seen += q_len
        tok = torch.empty(1, 1, dtype=torch.long, device=self.device)
        if self.rank + 1 < self.world:
            dist.send(h.contiguous(), dst=self.rank + 1, group=self.group)
        else:
            tok = st.lm_head(st.norm(h[:, -1:, :]))[:, -1, :].argmax(dim=-1, keepdim=True)
        if self.world > 1:
            dist.broadcast(tok, src=self.world - 1, group=self.group)
        return tok

    def _sync(self):
        if self.device.type == "cuda":
            torch.cuda.synchronize(self.device)
        if self.world > 1:
            dist.barrier(group=self.group)

    def generate(self, ids: torch.Tensor, max_new_tokens: int) -> dict:
        """Prefill + greedy decode. `ids` must be the same tensor on every rank (only rank 0 reads it). Returns the tokens and
        wall-clock timings bracketed by barriers (device-side max-over-ranks timing is bench.py's job)."""
        self.reset()
        self._sync()
        t0 = time.perf_counter()
        tok = self.step(ids, ids.shape[1])
        self._sync()
        t1 = time.perf_counter()
        toks = [tok]
        for _ in range(max_new_tokens - 1):
            tok = self.step(tok, 1)
            toks.append(tok)
        self._sync()
        t2 = time.perf_counter()
        rows = [int(l.keys.shape[-2]) for l in self.cache.layers if getattr(l, "keys", None) is not None and l.keys.numel()]
        return {"tokens": torch.cat(toks, dim=1)[0].tolist(), "prefill_ms": (t1 - t0) * 1e3,
                "decode_tok_per_s": (max_new_tokens - 1) / max(t2 - t1, 1e-9) if max_new_tokens > 1 else 0.0,
                "cache_rows_local_first_last": [rows[0], rows[-1]] if rows else []}
