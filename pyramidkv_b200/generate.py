"""The generate loop on the far side of the eviction path (SURVEY.md §8 row f3).

The reference decodes through HF `generate`: per token and layer a `torch.cat` of the whole layer cache
(cache_utils_think.py:383-384), two transposes, one attention launch (llama_model.py:401-445), `position_ids` rebuilt
from the attention mask (llama_model.py:2617-2631) and ~1 000 host-launched kernels — launch-bound by a wide margin.
Here the compacted cache is pre-reserved for the whole generation, the number of rows is a DEVICE counter
(`pkv_decode_attn_graph`), and one greedy step (embedding -> every decoder layer through the patched attention forward
-> norm -> lm_head -> argmax -> token/position/step bookkeeping) is a fixed sequence of launches with fixed arguments:
it is captured once in a CUDA graph and replayed per token. The host only reads the tokens back at the end.

`greedy_generate` is the drop-in for `model.generate(ids, max_new_tokens=N, num_beams=1, do_sample=False)`
(run_longbench.py:264-275): same tokens as HF's greedy loop through the same patched forward (tests/test_generate.py,
CPU, eager mode with the test backend; `-m gpu`: graph vs eager vs HF generate).

`greedy_generate_batch` decodes several prompts of any lengths together: each is prefilled alone (the same prefill as
`greedy_generate`), their compacted caches are joined (`cache.join_caches`) and one step decodes all of them - one graph
replay per token, one attention launch per layer (`pkv_decode_attn_batch`) - so the weights are streamed once per step for
the whole batch instead of once per sequence.

With `model.config.pkv_kv_cache_dtype = "fp8_e4m3"` the prefill leaves FP8 caches (`cache.PkvFp8CacheLayer`); all three loops
take them as they are (the knob is the single source: no parameter here), one `pkv_decode_attn_batch_fp8` launch per layer.
Likewise with `model.config.pkv_gqa_shared = True` (one cache per KV head, `group` > 1): one `pkv_decode_attn_batch_gqa(_fp8)`
launch per layer.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Optional

import torch

from .cache import PkvBatchCacheLayer, PkvCacheLayer, PkvRaggedCacheLayer, join_caches


@dataclass
class _StaticState:
    step: torch.Tensor        # int32 [1]: decode steps already taken in this static run (read by the decode kernel)
    workspace: torch.Tensor   # split-T partials, shared by all layers (launches are stream-ordered)


class StaticDecoder:
    """Greedy decode over an already prefilled (and evicted) cache with a fixed per-step launch sequence.

    model: a patched LlamaForCausalLM / MistralForCausalLM; cache: the DynamicCache the patched prefill filled with
    PkvCacheLayer entries - one prompt, an equal-length batch prefilled as one forward, or prompts joined by
    `cache.join_caches`; first_token: the token the prefill produced per sequence ([B] or [B, 1] int64).
    eos_token_id (int or list): a sequence that produced one is done - it keeps decoding in lock-step, but its tokens are
    `pad_token_id` from then on (on the device: `done` [B]); None masks nothing."""

    def __init__(self, model, cache, first_token: torch.Tensor, max_steps: int, use_graph: Optional[bool] = None,
                 eos_token_id=None, pad_token_id: int = 0):
        self.model, self.cache, self.max_steps = model, cache, int(max_steps)
        layers = [l for l in cache.layers if isinstance(l, PkvCacheLayer)]
        if len(layers) != model.config.num_hidden_layers:
            raise RuntimeError("StaticDecoder needs a cache prefilled by the patched forward on every layer "
                               "(method 'fullkv' and stock caches go through model.generate)")
        self.layers = layers
        dev = layers[0].device
        bsz = layers[0].k_buf.shape[0]
        if isinstance(layers[0], PkvRaggedCacheLayer) and bsz != 1:
            raise NotImplementedError("ragged caches are batch size 1; join them (cache.join_caches) to decode them together")
        for l in layers:
            l.reserve(self.max_steps)                      # off the per-token path: no reallocation while the graph lives
        backend = model.model.layers[0].self_attn.kv_cluster.backend
        hq, d = layers[0].k_buf.shape[1] * getattr(layers[0], "group", 1), layers[0].k_buf.shape[3]   # query heads
        self.state = _StaticState(step=torch.zeros(1, dtype=torch.int32, device=dev),
                                  workspace=backend.decode_workspace(bsz * hq, d, dev))
        self.ids = first_token.reshape(bsz, 1).to(device=dev, dtype=torch.long).clone()
        seen = layers[0].seq_seen if isinstance(layers[0], PkvBatchCacheLayer) else [layers[0].seen_tokens] * bsz
        self.pos = torch.tensor(seen, dtype=torch.long, device=dev).reshape(bsz, 1)
        self.cursor = torch.zeros(1, dtype=torch.long, device=dev)
        self.tokens = torch.zeros(bsz, self.max_steps, dtype=torch.long, device=dev)
        self.eos = self.done = None
        if eos_token_id is not None:
            eos = eos_token_id if isinstance(eos_token_id, (list, tuple)) else [eos_token_id]
            self.eos = torch.tensor([int(e) for e in eos], dtype=torch.long, device=dev)
            self.done = (self.ids == self.eos[None, :]).any(dim=1, keepdim=True)      # [B, 1]
        self.pad_token_id = int(pad_token_id)
        self.taken = 0
        self.graph = None
        self.use_graph = (dev.type == "cuda") if use_graph is None else bool(use_graph)
        cache._pkv_static = self.state

    # one greedy step; every tensor it touches is static, every launch argument constant
    def _step(self) -> None:
        m = self.model.model
        h = m.embed_tokens(self.ids)
        pos_emb = m.rotary_emb(h, position_ids=self.pos)
        for layer in m.layers[: self.model.config.num_hidden_layers]:
            h = layer(h, attention_mask=None, position_embeddings=pos_emb, position_ids=self.pos,
                      past_key_values=self.cache, use_cache=True)
        h = m.norm(h)
        logits = self.model.lm_head(h[:, -1, :])
        nxt = logits.argmax(dim=-1, keepdim=True)                       # [B, 1]
        if self.done is not None:
            nxt = torch.where(self.done, self.pad_token_id, nxt)
            self.done.logical_or_((nxt == self.eos[None, :]).any(dim=1, keepdim=True))
        self.tokens.index_copy_(1, self.cursor, nxt)
        self.ids.copy_(nxt)
        self.pos.add_(1)
        self.cursor.add_(1)
        self.state.step.add_(1)

    def _capture(self) -> None:
        # warm up on a side stream (lazy initialisation, cuBLAS workspaces), restore the counters, then capture
        state = [t for t in (self.ids, self.pos, self.cursor, self.state.step, self.tokens, self.done) if t is not None]
        snap = [t.clone() for t in state]
        s = torch.cuda.Stream(device=self.ids.device)
        s.wait_stream(torch.cuda.current_stream(self.ids.device))
        with torch.cuda.stream(s):
            self._step()
        torch.cuda.current_stream(self.ids.device).wait_stream(s)
        # the warm-up step appended row length+1+0 of every layer; the captured run rewrites the same row first
        for t, v in zip(state, snap):
            t.copy_(v)
        self.graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(self.graph):
            self._step()
        for t, v in zip(state, snap):
            t.copy_(v)                                   # capture does not execute, but keep the invariant explicit

    @torch.no_grad()
    def run(self, steps: int) -> torch.Tensor:
        """Take `steps` more greedy steps; returns all tokens produced so far by this decoder, [B, taken] (device)."""
        if self.taken + steps > self.max_steps:
            raise ValueError(f"{self.taken} + {steps} steps exceed the {self.max_steps} reserved")
        if self.use_graph and self.graph is None and steps > 0:
            self._capture()
        for _ in range(steps):
            if self.graph is not None:
                self.graph.replay()
            else:
                self._step()
        self.taken += steps
        return self.tokens[:, : self.taken]

    def finish(self, kept=None) -> None:
        """Settle the host bookkeeping (rows / tokens seen per layer) and leave static mode; the cache is then a normal
        compacted cache again (further `model.generate`/forward calls continue from it). `kept[b]`: the rows sequence b keeps
        (joined caches only; default: every step taken) - rows appended after a sequence's EOS stay in the buffers uncounted."""
        if getattr(self.cache, "_pkv_static", None) is self.state:
            del self.cache._pkv_static
        for l in self.layers:
            if kept is not None and isinstance(l, PkvBatchCacheLayer):
                l.settle(kept)
            else:
                l.advance(self.taken)
        self.graph = None
        self.taken = 0


def _prefill(model, input_ids: torch.Tensor):
    """Prefill (+ eviction in every patched layer) of one prompt: (first token [1, 1], cache)."""
    from transformers import DynamicCache
    if hasattr(model, "prepare_inputs_for_generation"):
        for layer in model.model.layers:                 # what the patched prepare_inputs does on an empty cache (llama_model.py:2609-2612)
            layer.self_attn.kv_seq_len = 0
    cache = DynamicCache(config=model.config)
    out = model(input_ids=input_ids, past_key_values=cache, use_cache=True, logits_to_keep=1)
    return out.logits[:, -1, :].argmax(dim=-1, keepdim=True), cache


def _eos_set(eos_token_id) -> set:
    if eos_token_id is None:
        return set()
    return set(int(e) for e in (eos_token_id if isinstance(eos_token_id, (list, tuple)) else [eos_token_id]))


@torch.no_grad()
def greedy_generate(model, input_ids: torch.Tensor, max_new_tokens: int, use_graph: Optional[bool] = None,
                    return_cache: bool = False, eos_token_id=None, check_every: int = 16):
    """Prefill (+ eviction in every patched layer) then up to `max_new_tokens - 1` static decode steps.
    Returns sequences [1, prompt + generated] like `generate(...).sequences` (and the cache on request).
    `eos_token_id` (int or list, as the reference runner passes it: run_longbench.py:270-272) ends the generation with the first
    such token (kept, like HF); the device never waits for the host, so the tokens are inspected every `check_every` steps
    and the surplus steps are dropped."""
    if input_ids.dim() != 2 or input_ids.shape[0] != 1:
        raise NotImplementedError("batch size 1 (as in the reference: README.md:47); greedy_generate_batch decodes several prompts together")
    eos = _eos_set(eos_token_id)
    first, cache = _prefill(model, input_ids)
    toks = [first]
    if max_new_tokens > 1 and not (eos and int(first) in eos):
        dec = StaticDecoder(model, cache, first, max_new_tokens - 1, use_graph=use_graph)
        if not eos:
            toks.append(dec.run(max_new_tokens - 1).clone())
        else:
            done, keep = 0, max_new_tokens - 1
            while done < max_new_tokens - 1:
                n = min(max(1, check_every), max_new_tokens - 1 - done)
                got = dec.run(n)[0, done:done + n].tolist()              # one device-to-host read per chunk
                hit = next((i for i, t in enumerate(got) if t in eos), None)
                done += n
                if hit is not None:
                    keep = done - n + hit + 1
                    break
            toks.append(dec.tokens[:, :keep].clone())
            # rows appended after the EOS stay in the buffers but are not counted: the cache ends with the EOS token
            dec.taken = keep
        dec.finish()
    seq = torch.cat([input_ids, *toks], dim=1)
    return (seq, cache) if return_cache else seq


@torch.no_grad()
def greedy_generate_batch(model, prompts, max_new_tokens: int, eos_token_id=None, pad_token_id: int = 0,
                          use_graph: Optional[bool] = None, check_every: int = 16, return_cache: bool = False):
    """Greedy generation for several prompts of any lengths (1-D or [1, S] id tensors): each prompt is prefilled alone
    exactly as `greedy_generate` does, the compacted caches are joined, and up to `max_new_tokens - 1` steps decode all of
    them together (`StaticDecoder` over the joined cache). Each sequence stops at its first `eos_token_id` (kept, like HF);
    the loop ends once all are done, which the host checks every `check_every` steps. Returns one 1-D tensor per prompt,
    prompt + generated (and the joined cache on request, its per-sequence rows ending at each EOS)."""
    ids = [p.reshape(1, -1) for p in prompts]
    if not ids:
        raise ValueError("greedy_generate_batch: no prompts")
    eos = _eos_set(eos_token_id)
    firsts, caches = [], []
    for p in ids:
        f, c = _prefill(model, p)
        firsts.append(f)
        caches.append(c)
    first = torch.cat(firsts)                                            # [B, 1]
    steps = max(0, max_new_tokens - 1)
    cache = join_caches(caches, reserve=steps)
    del caches
    first_host = first[:, 0].tolist()
    kept = [0] * len(ids)
    gen = torch.empty(len(ids), 0, dtype=torch.long)
    if steps and not all(t in eos for t in first_host):
        dec = StaticDecoder(model, cache, first, steps, use_graph=use_graph, eos_token_id=sorted(eos) if eos else None,
                            pad_token_id=pad_token_id)
        while dec.taken < steps:
            dec.run(min(max(1, check_every) if eos else steps, steps - dec.taken))
            if eos and bool(dec.done.all()):                            # one device-to-host read per chunk
                break
        gen = dec.tokens[:, : dec.taken].cpu()
        for b in range(len(ids)):
            if first_host[b] in eos:
                continue
            row = gen[b].tolist()
            hit = next((i for i, t in enumerate(row) if t in eos), None)
            kept[b] = len(row) if hit is None else hit + 1
        dec.finish(kept)
    seqs = [torch.cat([p[0].cpu(), first[b].cpu(), gen[b, : kept[b]]]).to(p.device) for b, p in enumerate(ids)]
    return (seqs, cache) if return_cache else seqs
