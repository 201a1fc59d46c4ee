"""Host-side mirror of the reference's eviction-policy interface (pyramidkv/pyramidkv_utils.py).

Same class names, constructor arguments, `update_kv` signature, defaults and error behaviour as
`PyramidKVCluster` (:173-283), `SnapKVCluster` (:285-347), `H2OKVCluster` (:516-575),
`StreamingLLMKVCluster` (:578-620) and the `init_*` factories (:880-1031) — but `update_kv` is ONE call into
libpkv.so (hand-written sm_90a kernels) instead of a ~16-op PyTorch chain, and it accepts the un-repeated
K/V ([bsz, H_kv, S, D]) as well as the reference's post-`repeat_kv` tensors ([bsz, H_q, S, D]).

There is no CPU implementation here. Host (CPU) tensors are staged to the GPU, evicted there, and the
compacted K/V copied back — that is the end-to-end path bench.py times.
"""
from __future__ import annotations

from typing import Optional, Tuple

import torch

from . import ops

SELECT_MAX_K = 16384          # largest top_k of the select kernels (pkv_topk.cu: topk_supported)


class CudaBackend:
    """The product backend: every call lands in libpkv.so."""
    name = "libpkv-sm100a"

    def layer_budget(self, *a, **kw):
        return ops.layer_budget(*a, **kw)

    accepts_inputs_ready = True

    def evict(self, method, q, k, v, window_size, top_k, k_cache, v_cache, kernel_size, pooling, idx_out=None, inputs_ready=False,
              gqa_shared=False):
        ops.evict_prefill(method, q, k, v, window_size, top_k, k_cache, v_cache, kernel_size, pooling, idx_out, inputs_ready=inputs_ready,
                          gqa_shared=gqa_shared)

    accepts_layer_batch = True

    def evict_batch(self, items) -> int:
        """Deferred eviction: `items` = the parked evictions of the layers of one prompt (dicts with the arguments of `evict`).
        One pass over all layers of a device (pkv_evict_prefill_batch: four launches per 32 layers) when they can share launches,
        else layer by layer. Layers placed on several GPUs of one process (accelerate's device_map) are batched per device, each
        on that device's current stream. Returns the number of layers that went through a batch."""
        def plan(it, ws=None):
            return ops.plan_evict(it["method"], it["q"], it["k"], it["v"], it["W"], it["top_k"], it["k_cache"], it["v_cache"],
                                  it["kernel_size"], it["pooling"], it["idx_out"], inputs_ready=True, workspace=ws)
        by_device = {}
        for it in items:
            by_device.setdefault(it["k"].device, []).append(it)
        batched = 0
        for dev, group in by_device.items():
            with torch.cuda.device(dev):
                done = False
                if len(group) >= 2 and all(it["method"] in ("pyramidkv", "snapkv") for it in group):
                    first = plan(group[0])
                    wss = ops.batch_workspaces(first, len(group), max(it["top_k"] for it in group))
                    plans = [plan(it, ws) for it, ws in zip(group, wss)]
                    if ops.batch_supported(plans):
                        ops.EvictBatch(plans).run()
                        batched += len(group)
                        done = True
                if not done:
                    for it in group:
                        self.evict(it["method"], it["q"], it["k"], it["v"], it["W"], it["top_k"], it["k_cache"], it["v_cache"],
                                   it["kernel_size"], it["pooling"], it["idx_out"], inputs_ready=True)
        return batched

    def decode_attn(self, q, k_cache, v_cache, length, k_new, v_new, out=None, softmax_scale=0.0, step=None,
                    max_length=0, workspace=None, head_rows=None):
        return ops.decode_attn(q, k_cache, v_cache, length, k_new, v_new, out, softmax_scale, step, max_length, workspace, head_rows)

    def decode_attn_batch(self, q, k_buf, v_buf, length, k_new, v_new, rows=None, step=None, max_length=0, workspace=None,
                          out=None, softmax_scale=0.0):
        return ops.decode_attn_batch(q, k_buf, v_buf, length, k_new, v_new, rows, step, max_length, workspace, out, softmax_scale)

    # -- the opt-in FP8 cache (model.config.pkv_kv_cache_dtype = "fp8_e4m3") --
    def cache_quantize_fp8(self, layers):
        ops.cache_quantize_fp8(layers)

    def decode_attn_batch_fp8(self, q, k_q, v_q, k_scale, v_scale, length, k_new, v_new, rows=None, step=None, max_length=0,
                              workspace=None, out=None, softmax_scale=0.0):
        return ops.decode_attn_batch_fp8(q, k_q, v_q, k_scale, v_scale, length, k_new, v_new, rows, step, max_length, workspace,
                                         out, softmax_scale)

    # -- GQA-shared caches (model.config.pkv_gqa_shared = True): one cache per KV head --
    def decode_attn_batch_gqa(self, q, k_buf, v_buf, length, k_new, v_new, rows=None, step=None, max_length=0, workspace=None,
                              out=None, softmax_scale=0.0):
        return ops.decode_attn_batch_gqa(q, k_buf, v_buf, length, k_new, v_new, rows, step, max_length, workspace, out, softmax_scale)

    def decode_attn_batch_gqa_fp8(self, q, k_q, v_q, k_scale, v_scale, length, k_new, v_new, rows=None, step=None, max_length=0,
                                  workspace=None, out=None, softmax_scale=0.0):
        return ops.decode_attn_batch_gqa_fp8(q, k_q, v_q, k_scale, v_scale, length, k_new, v_new, rows, step, max_length, workspace,
                                             out, softmax_scale)

    # -- the decode window (model.config.pkv_decode_window = R): prompt rows plus a ring of the last R appended rows --
    def decode_attn_window(self, q, k_buf, v_buf, length, k_new, v_new, prompt_rows, window, rows=None, step=None, max_length=0,
                           workspace=None, out=None, softmax_scale=0.0, scales=None, gqa=False):
        return ops.decode_attn_window(q, k_buf, v_buf, length, k_new, v_new, prompt_rows, window, rows, step, max_length,
                                      workspace, out, softmax_scale, scales, gqa)

    # -- heavy hitters in the decode window (model.config.pkv_decode_heavy = H): the least-attended generated row leaves --
    def decode_attn_heavy(self, q, k_buf, v_buf, length, k_new, v_new, prompt_rows, window, heavy, scores, gen, victim, rows=None,
                          step=None, max_length=0, workspace=None, scratch=None, out=None, softmax_scale=0.0, scales=None,
                          gqa=False):
        return ops.decode_attn_heavy(q, k_buf, v_buf, length, k_new, v_new, prompt_rows, window, heavy, scores, gen, victim, rows,
                                     step, max_length, workspace, scratch, out, softmax_scale, scales, gqa)

    def decode_heavy_workspace(self, num_seqs, num_q_heads, window, device):
        return torch.empty(ops.decode_heavy_workspace_bytes(num_seqs, num_q_heads, window), dtype=torch.uint8, device=device)

    # -- continuous batching: one prompt's compacted cache into one slot of a batched cache --
    def cache_install(self, layers, slot, step):
        ops.cache_install(layers, slot, step)

    def rope_inplace(self, q, k, cos, sin):
        ops.rope_inplace(q, k, cos, sin)

    # -- sampled decoding: one token per row of logits, per-row parameters in device memory --
    def sample_tokens(self, logits, params, out, col, advance=True):
        ops.sample_tokens(logits, params, out, col, advance)

    def sample_tokens_penalized(self, logits, params, out, col, advance=True):
        ops.sample_tokens_penalized(logits, params, out, col, advance)

    def sample_tokens_constrained(self, logits, params, out, col, advance=True):
        ops.sample_tokens_constrained(logits, params, out, col, advance)

    def token_rules(self, params, vocab, append=None, col=0):
        ops.token_rules(params, vocab, append, col)

    # -- token log-probabilities: the raw log-softmax at a token and at the row's top N --
    def token_logprobs(self, logits, tokens, out_lp, out_ids, out_top, col=0, tokens_col=0, cursor=None):
        ops.token_logprobs(logits, tokens, out_lp, out_ids, out_top, col, tokens_col, cursor)

    # -- beam search: candidates per beam row, one step per prompt, the cache reorder of every layer --
    def beam_candidates(self, logits, st):
        R = logits.shape[0]
        ops.beam_candidates(logits, st.m[:R], st.log_z[:R], st.cand_lp[:R], st.cand_id[:R])

    def beam_step(self, st, rows_per_prompt, step, step_offset):
        ops.beam_step(st, rows_per_prompt, step, step_offset)

    def cache_reorder(self, items, P, k, parent, diverge, step, step_offset):
        ops.cache_reorder(items, P, k, parent, diverge, step, step_offset)

    # -- ragged per-head budgets (AdaKV / HeadKV): scores first, budgets from the host, then select + gather --
    def ragged_begin(self, q, k, v, window_size, kernel_size, pooling):
        """Stages 1-2 (window logits, softmax + pool) into a workspace that stays alive until ragged_finish."""
        Hq, D = q.shape[0], q.shape[-1]
        n = k.shape[-2] - window_size
        kc, vc = (torch.empty(Hq, window_size, D, dtype=k.dtype, device=k.device) for _ in range(2))   # stages 1-2 write no cache rows
        probe = ops.plan_evict("snapkv", q, k, v, window_size, 0, kc, vc, kernel_size, pooling, window_mean=True)
        # ONE workspace sized for the largest possible selection, so that the pooled scores survive the re-plan in ragged_finish
        ws = torch.empty(ops.workspace_bytes_for(probe, n), dtype=torch.uint8, device=k.device)
        plan = ops.plan_evict("snapkv", q, k, v, window_size, 0, kc, vc, kernel_size, pooling, workspace=ws, window_mean=True)
        ops.run_stage(plan, "scores")
        ops.run_stage(plan, "pool")
        return dict(plan=plan, ws=ws, q=q, k=k, v=v, W=window_size, kernel=kernel_size, pooling=pooling)

    def adakv_counts(self, handle, base_capacity, normalize):
        return ops.adakv_counts(handle["plan"], base_capacity, normalize)

    def ragged_finish(self, handle, caps, reserve):
        """Uniform select of min(max(caps), 16384) rows per head + gather; every head whose budget is above the select
        kernels' limit then takes its cap_h rows from a stable descending sort of its pooled row (the same (score desc,
        index asc) order); last, the window rows move to [cap_h, cap_h + W)."""
        q, k, v, W = handle["q"], handle["k"], handle["v"], handle["W"]
        Hq, D = q.shape[0], q.shape[-1]
        kmax = max(caps)
        k_buf = torch.empty(Hq, kmax + W + reserve, D, dtype=k.dtype, device=k.device)
        v_buf = torch.empty_like(k_buf)
        ksel = min(kmax, SELECT_MAX_K)
        plan = ops.plan_evict("snapkv", q, k, v, W, ksel, k_buf, v_buf, handle["kernel"], handle["pooling"], workspace=handle["ws"],
                              window_mean=True)
        # AdaKV can hand one head most of the layer's Hq * base slots, and HeadKV's budgets come from a file: either can pass
        # the select kernels' limit although max_capacity_prompt - W does not
        pooled = ops.ws_pooled(plan)
        big = {h: torch.sort(pooled[h].float(), descending=True, stable=True).indices[:c] for h, c in enumerate(caps) if c > SELECT_MAX_K}
        if ksel > 0:
            ops.run_stage(plan, "topk")
        ops.run_stage(plan, "gather")
        G = Hq // k.shape[-3]
        for h, order in big.items():
            k_buf[h, :order.numel()] = k[h // G].index_select(0, order)
            v_buf[h, :order.numel()] = v[h // G].index_select(0, order)
        caps_dev = torch.tensor(caps, dtype=torch.int32, device=k.device)
        ops.ragged_place_window(plan, caps_dev)
        return k_buf, v_buf

    def decode_workspace(self, num_q_heads, head_dim, device):
        return torch.empty(ops.decode_workspace_bytes(num_q_heads, head_dim), dtype=torch.uint8, device=device)

    # prompt-lookup speculative decoding (generate.SpeculativeDecoder)
    def decode_attn_multi(self, q, k_buf, v_buf, k_new, v_new, rows=None, length=0, step=None, max_length=0, scales=None,
                          gqa=False, workspace=None, out=None, softmax_scale=0.0):
        return ops.decode_attn_multi(q, k_buf, v_buf, k_new, v_new, rows, length, step, max_length, scales, gqa, workspace, out,
                                     softmax_scale)

    def prompt_lookup(self, st):
        ops.prompt_lookup(st)

    def spec_step(self, st, rows):
        ops.spec_step(st, rows)

    # prompt-lookup speculation in the continuous loop (generate.ContinuousSpecDecoder)
    def decode_attn_packed(self, q, k_buf, v_buf, k_new, v_new, row_start, row_count, num_queries, rows=None, max_length=0,
                           scales=None, gqa=False, workspace=None, out=None, softmax_scale=0.0):
        return ops.decode_attn_packed(q, k_buf, v_buf, k_new, v_new, row_start, row_count, num_queries, rows, max_length,
                                      scales, gqa, workspace, out, softmax_scale)

    def spec_pack(self, st, pk):
        ops.spec_pack(st, pk)

    @staticmethod
    def check_knobs(method: str, window_size: int, max_capacity_prompt=None) -> None:
        """What the sm_90a scoring kernels take, checked when the cluster is built (the reference accepts any window_size;
        here an unsupported one fails at construction with the supported set named, not in the middle of generate())."""
        if method in ("pyramidkv", "snapkv", "adakv", "headkv"):
            if window_size % 8 != 0 or not 8 <= window_size <= 64:
                raise NotImplementedError(f"window_size={window_size}: the {method} scoring kernels of libpkv take window sizes "
                                          "8, 16, 24, ..., 64 (StreamingLLM and H2O take any window)")
            if method in ("adakv", "headkv") and window_size & (window_size - 1):
                raise NotImplementedError(f"window_size={window_size}: AdaKV / HeadKV average the window rows and need a power of two (8, 16, 32, 64)")
        if max_capacity_prompt is not None and method != "l2norm" and max_capacity_prompt - window_size > 16384:
            raise NotImplementedError(f"max_capacity_prompt - window_size = {max_capacity_prompt - window_size}: libpkv selects at most "
                                      "16384 tokens per head and layer (top_k limit of the select kernels, INTEGRATION.md)")


_default_backend = CudaBackend()


def default_device() -> torch.device:
    if not torch.cuda.is_available():
        raise RuntimeError("pyramidkv_b200 needs a CUDA device (H100, sm_90a); there is no CPU fallback")
    return torch.device("cuda", torch.cuda.current_device())


class _KVCluster:
    method = ""
    # rows of head-room allocated behind the compacted prompt so decode can append in place
    decode_reserve = 0

    def __init__(self, window_size=64, max_capacity_prompt=256 + 64, kernel_size=5, pooling="avgpool", merge=None,
                 backend=None, **_ignored):
        self.window_size = window_size
        self.max_capacity_prompt = max_capacity_prompt
        assert self.max_capacity_prompt - self.window_size > 0     # pyramidkv_utils.py:184 / :290 / :521 / :583
        self.kernel_size = kernel_size
        self.pooling = pooling
        self.merge = merge
        self.backend = backend or _default_backend
        self.last_indices: Optional[torch.Tensor] = None
        self.return_indices = False
        self.last_h2d_bytes = self.last_d2h_bytes = 0       # bytes the last host-buffer update_kv moved over the bus
        self._check_knobs()

    def _check_knobs(self):
        check = getattr(self.backend, "check_knobs", None)   # (the CPU test backend takes anything the oracle takes)
        if check is not None:
            check(self.method, self.window_size, self.max_capacity_prompt)

    def reset(self, window_size=64, max_capacity_prompt=256 + 64, kernel_size=5, pooling="avgpool", merge=None):
        self.window_size = window_size
        self.max_capacity_prompt = max_capacity_prompt
        assert self.max_capacity_prompt - self.window_size > 0
        self._check_knobs()
        self.kernel_size = kernel_size
        self.pooling = pooling
        self.merge = merge

    # -- per-layer budget (overridden by PyramidKV) --
    def budget(self, q_len: int) -> Tuple[int, int]:
        return self.backend.layer_budget(self.method, self.max_capacity_prompt, self.window_size, 2, 0, q_len)

    def evict_into(self, query_states, key_states, value_states, reserve: int = 0, pending: Optional[list] = None,
                   gqa_shared: bool = False):
        """Evict one prompt (bsz == 1 slice, [H,S,D] tensors on the GPU) into freshly allocated cache buffers.
        Returns (k_buf, v_buf, rows): buffers [Hq, rows + reserve, D]; rows = S when nothing is evicted.
        `pending`: a list to PARK this eviction on instead of launching it (window methods only): the buffers are returned
        unfilled and `flush_pending(pending, backend)` later evicts all parked layers in one pass (CudaBackend.evict_batch).
        `gqa_shared` (knob pkv_gqa_shared, Hq > Hkv): one selection per KV head (PKV_FLAG_GQA_SHARED), buffers
        [Hkv, rows + reserve, D]; never parked (the layer batch is not built for it)."""
        Hq, D = query_states.shape[-3], query_states.shape[-1]
        gqa_shared = gqa_shared and key_states.shape[-3] != Hq
        if gqa_shared:
            Hq, pending = key_states.shape[-3], None          # the heads of the cache
        S = key_states.shape[-2]          # query_states may hold only the last window_size rows
        mode, top_k = self.budget(S)
        method, W = self.method, self.window_size
        if mode == 0:
            # q_len < max_capacity_prompt: the reference returns K/V untouched (:218 / :314 / :541 / :603).
            # The cache is still per query head, so this is the identity gather of all S rows.
            method, W, top_k = "streamingllm", 1, S - 1
        else:
            if self.merge is not None:
                if self.merge == "pivot":
                    raise NotImplementedError("merge='pivot' (LOOK-M, pyramidkv_utils.py:119-170) is outside the hot path built here")
                raise ValueError("Merge method not supported")          # pyramidkv_utils.py:164
            if method in ("pyramidkv", "snapkv") and self.pooling not in ("avgpool", "maxpool"):
                raise ValueError("Pooling method not supported")        # pyramidkv_utils.py:237
        rows = top_k + W
        k_buf = torch.empty(Hq, rows + reserve, D, dtype=key_states.dtype, device=key_states.device)
        v_buf = torch.empty_like(k_buf)
        idx = None
        if self.return_indices and mode == 1:
            idx = torch.empty(Hq, top_k, dtype=torch.int64, device=key_states.device)
        # PKV_FLAG_INPUTS_READY: the patched forward sets `inputs_ready` when the kernel just before this call (its dense
        # attention) only READ q/k/v — the K scan may then start while that kernel drains
        extra = {"inputs_ready": True} if getattr(self, "inputs_ready", False) and getattr(self.backend, "accepts_inputs_ready", False) else {}
        self.last_indices = idx
        if pending is not None and mode == 1 and method in ("pyramidkv", "snapkv") and getattr(self.backend, "accepts_layer_batch", False):
            # the window methods read only the last W query rows: a copy of those (64 KB), so that parking the layer keeps K and V
            # alive but not the whole Q projection (4x the size of K with GQA)
            q_win = query_states[..., query_states.shape[-2] - W:, :].contiguous()
            pending.append(dict(method=method, q=q_win, k=key_states, v=value_states, W=W, top_k=top_k, k_cache=k_buf, v_cache=v_buf,
                                kernel_size=self.kernel_size, pooling=self.pooling, idx_out=idx))
            return k_buf, v_buf, rows
        if gqa_shared:
            extra["gqa_shared"] = True
        self.backend.evict(method, query_states, key_states, value_states, W, top_k, k_buf, v_buf,
                           self.kernel_size, self.pooling, idx, **extra)
        return k_buf, v_buf, rows

    def update_kv(self, key_states, query_states, value_states, attention_mask, num_key_value_groups):
        """Reference signature (pyramidkv_utils.py:197). `attention_mask` and `num_key_value_groups` are ignored,
        as in the reference. Returns (key_states, value_states) of shape [bsz, H_q, rows, D]."""
        assert key_states.shape[-2] == query_states.shape[-2]       # pyramidkv_utils.py:200
        bsz, num_heads, q_len, head_dim = query_states.shape
        if q_len < self.max_capacity_prompt and key_states.shape[1] == num_heads:
            return key_states, value_states                          # same objects, like the reference
        src_device = key_states.device
        W = self.window_size
        outs_k, outs_v = [], []
        for b in range(bsz):
            q, k, v = query_states[b], key_states[b], value_states[b]
            if self.method == "l2norm":
                q = q[:, q_len - 1:, :]          # L2Norm reads no queries: one row travels along to carry the head count
            elif self.method != "h2o":
                q = q[:, q_len - W:, :]          # the window methods read only the last W query rows
            if not k.is_cuda:                    # host buffers: stage in, evict on the GPU, copy back
                kb, vb = self._evict_host(q, k, v)
                outs_k.append(kb)
                outs_v.append(vb)
                continue
            kb, vb, rows = self.evict_into(q, k, v, reserve=self.decode_reserve)
            outs_k.append(kb[:, :rows])
            outs_v.append(vb[:, :rows])
        K = torch.stack(outs_k) if bsz > 1 else outs_k[0][None]
        V = torch.stack(outs_v) if bsz > 1 else outs_v[0][None]
        return K, V

    def _evict_host(self, q, k, v):
        """K/Q/V in host memory (pinned for full PCIe speed), results back in host memory. Only what the GPU needs
        crosses the bus: K and the query rows go up, the compacted K rows and the selected indices come down; the V rows
        are picked up on the host with those indices — V itself (half of the input bytes) never moves. StreamingLLM and
        the nothing-to-evict branch keep no scores, so they take the plain staged path."""
        dev = default_device()
        S = k.shape[-2]
        nbytes = lambda *ts: sum(t.numel() * t.element_size() for t in ts)
        mode, top_k = self.budget(S)
        if mode == 0 or self.method == "streamingllm":
            qd, kd, vd = (t.to(dev, non_blocking=True) for t in (q, k, v))
            kb, vb, rows = self.evict_into(qd, kd, vd)
            self.last_h2d_bytes, self.last_d2h_bytes = nbytes(q, k, v), 2 * nbytes(kb[:, :rows])
            return kb[:, :rows].to(k.device), vb[:, :rows].to(k.device)
        want_idx = self.return_indices
        self.return_indices = True
        try:
            qd, kd = q.to(dev, non_blocking=True), k.to(dev, non_blocking=True)
            kb, _, rows = self.evict_into(qd, kd, kd)            # the V source is aliased to K: its gathered rows are discarded
        finally:
            self.return_indices = want_idx
        idx = self.last_indices.to(k.device)                     # [Hq, top_k] (synchronises the stream)
        Hq, W = idx.shape[0], self.window_size
        rows_idx = torch.cat([idx, torch.arange(S - W, S).expand(Hq, W)], dim=1)                      # :271-282 row order
        vb = ops.host_pick_rows(v, rows_idx)                                                           # [Hq, rows, D], host memory only
        if not want_idx:
            self.last_indices = None
        self.last_h2d_bytes, self.last_d2h_bytes = nbytes(q, k), nbytes(kb[:, :rows], idx)
        return kb[:, :rows].to(k.device), vb


def flush_pending(pending: Optional[list], backend=None) -> int:
    """Evict every parked layer (see _KVCluster.evict_into(pending=...)) on the current stream and empty the list."""
    if not pending:
        return 0
    items = list(pending)
    pending.clear()                      # the K / V / Q references die with `items` once the launches are queued
    return (backend or _default_backend).evict_batch(items)


class PyramidKVCluster(_KVCluster):
    """pyramidkv_utils.py:173-283. Per-layer pyramidal budget :205-215; beta fixed at 20 (:174)."""
    method = "pyramidkv"

    def __init__(self, num_hidden_layers=32, window_size=64, max_capacity_prompt=256 + 64, kernel_size=5,
                 pooling="avgpool", beta=20, num_layers=80, layer_idx=None, merge=None, backend=None):
        super().__init__(window_size, max_capacity_prompt, kernel_size, pooling, merge, backend)
        self.layer_idx = layer_idx
        self.num_hidden_layers = num_hidden_layers
        self.steps = -1
        self.beta = beta

    def budget(self, q_len: int):
        return self.backend.layer_budget("pyramidkv", self.max_capacity_prompt, self.window_size,
                                         self.num_hidden_layers, self.layer_idx, q_len, self.beta)


class SnapKVCluster(_KVCluster):
    """pyramidkv_utils.py:285-347."""
    method = "snapkv"

    def __init__(self, window_size=64, max_capacity_prompt=256 + 64, kernel_size=5, pooling="avgpool", merge=None,
                 recent_size=32, ratio=0.4, backend=None):
        super().__init__(window_size, max_capacity_prompt, kernel_size, pooling, merge, backend)
        self.recent_size = recent_size
        self.ratio = ratio


class H2OKVCluster(_KVCluster):
    """pyramidkv_utils.py:516-575 (full-matrix scores, mask on the last WxW block only, no pooling)."""
    method = "h2o"


class StreamingLLMKVCluster(_KVCluster):
    """pyramidkv_utils.py:578-620 (first max_capacity_prompt - window_size tokens + last window_size)."""
    method = "streamingllm"


class L2NormCluster(_KVCluster):
    """pyramidkv_utils.py:394-431: keeps the `max_capacity_prompt` tokens of SMALLEST key L2 norm (no observation window,
    no queries), rows in ascending-norm order; layers listed in `skip_layers` keep everything (:416-417). The reference's
    `argsort` is not stable, so its order among equal norms is implementation-defined; here it is (norm, index) ascending
    — the order of a stable sort."""
    method = "l2norm"

    def __init__(self, max_capacity_prompt: int = 256 + 64, layer_idx: int = 0, skip_layers=(), backend=None):
        # (the reference constructor has no window / kernel / pooling / merge knobs: pyramidkv_utils.py:395-398)
        self.max_capacity_prompt = max_capacity_prompt
        self.layer_idx = layer_idx
        self.skip_layers = list(skip_layers)
        self.window_size, self.kernel_size, self.pooling, self.merge = 0, 1, "avgpool", None
        self.backend = backend or _default_backend
        self.last_indices = None
        self.return_indices = False
        self.last_h2d_bytes = self.last_d2h_bytes = 0

    def reset(self, max_capacity_prompt: int = 256 + 64, layer_idx: int = 0, skip_layers=()):
        self.max_capacity_prompt, self.layer_idx, self.skip_layers = max_capacity_prompt, layer_idx, list(skip_layers)

    def budget(self, q_len: int):
        if self.layer_idx in self.skip_layers:
            return 0, q_len                                            # :416-417
        return self.backend.layer_budget("l2norm", self.max_capacity_prompt, 0, 2, 0, q_len)

    def update_kv(self, key_states, query_states, value_states, attention_mask, num_key_value_groups):
        if self.layer_idx in self.skip_layers and key_states.shape[1] == query_states.shape[1]:
            assert key_states.shape[-2] == query_states.shape[-2]
            return key_states, value_states                            # same objects, like the reference
        return super().update_kv(key_states, query_states, value_states, attention_mask, num_key_value_groups)


def _round_half_even_f32(counts, one_minus_floor: float, floor_capacity: int):
    """`torch.round(head_adaptive_capacity * (1 - floor_ratio) + floor_capacity).int()` (pyramidkv_utils.py:715): the int64
    counts are multiplied in float32 by the float32 value of (1 - floor), the int is added in float32, round half to even."""
    t = torch.tensor(counts, dtype=torch.int64)
    return torch.round(t * one_minus_floor + floor_capacity).int().tolist()


class _RaggedCluster:
    """Shared machinery of AdaKV and HeadKV: per-head budgets cap_h, head h keeps its cap_h best tokens + the last W.
    The reference builds one flat [sum_h len_h, D] tensor and re-allocates it on every decoded token
    (DynamicCacheSplitHeadFlatten + update_flatten_view); here the cache stays a padded [Hq, capacity, D] buffer with per-head
    row counts, appended to in place by the decode kernel."""
    ragged = True
    method = ""

    def _init_common(self, window_size, kernel_size, pooling, max_capacity_prompt, layer_idx, num_hidden_layers, backend):
        self.window_size, self.kernel_size, self.pooling = window_size, kernel_size, pooling
        self.max_capacity_prompt = max_capacity_prompt
        self.base_capacity = max_capacity_prompt - window_size
        self.num_hidden_layers, self.layer_idx = num_hidden_layers, layer_idx
        self.backend = backend or _default_backend
        self.head_lens = None                     # metadata names of the reference (:640-645)
        self.max_seqlen_k = 0
        self.klen_sum = 0
        self.cu_klen = 0
        self.cu_offset = None
        self.cu_headlens = None
        self.last_capacities = None

    def _capacities(self, handle, num_heads: int):
        raise NotImplementedError

    def _init_metadata(self, k_lens, device):
        """`init_metadata` (pyramidkv_utils.py:682-696): what the reference's varlen attention and update_flatten_view read."""
        n = len(k_lens)
        self.head_lens = torch.tensor(k_lens, dtype=torch.int32, device=device)
        self.klen_sum, self.max_seqlen_k = int(sum(k_lens)), int(max(k_lens))
        self.cu_headlens = torch.cumsum(self.head_lens, dim=0, dtype=torch.int32)
        self.cu_klen = torch.cat([self.cu_headlens - self.head_lens, torch.tensor([self.klen_sum], dtype=torch.int32, device=device)])
        self.layer_qlens = torch.ones(n, dtype=torch.int32, device=device)
        self.qlen_sum = n
        self.cu_qlen = torch.cat([torch.cumsum(self.layer_qlens, 0, dtype=torch.int32) - self.layer_qlens,
                                  torch.tensor([n], dtype=torch.int32, device=device)])
        self.cu_offset = torch.arange(0, n + 1, dtype=torch.int32, device=device)
        self.cu_head_offset = torch.arange(1, n + 1, dtype=torch.int32, device=device)

    def compressed(self, q_len: int) -> bool:
        return not (self.base_capacity > q_len - self.window_size)          # :698 / :832

    def evict_into(self, query_states, key_states, value_states, reserve: int = 0, pending: Optional[list] = None):
        """(`pending` is accepted and ignored: AdaKV / HeadKV are evicted layer by layer.) The not-compressed branch (:698-701 / :832-835): every head keeps all S rows — the identity gather into per-query-head
        buffers, exactly like the other policies' short-prompt branch. Returns (k_buf, v_buf, rows)."""
        Hq, D = query_states.shape[-3], query_states.shape[-1]
        S = key_states.shape[-2]
        assert not self.compressed(S)
        k_buf = torch.empty(Hq, S + reserve, D, dtype=key_states.dtype, device=key_states.device)
        v_buf = torch.empty_like(k_buf)
        self.backend.evict("streamingllm", query_states, key_states, value_states, 1, S - 1, k_buf, v_buf, self.kernel_size, self.pooling, None)
        return k_buf, v_buf, S

    def evict_ragged(self, query_states, key_states, value_states, reserve: int = 0):
        """One prompt ([H,S,D] tensors, bsz == 1 slice). Returns (k_buf, v_buf, head_rows): buffers [Hq, max_h rows + reserve, D]
        and the per-head row counts cap_h + W (host list)."""
        if self.pooling not in ("avgpool", "maxpool"):
            raise ValueError("Pooling method not supported")                # :671
        W = self.window_size
        q = query_states[:, query_states.shape[-2] - W:, :] if query_states.shape[-2] != W else query_states
        handle = self.backend.ragged_begin(q, key_states, value_states, W, self.kernel_size, self.pooling)
        caps = [int(c) for c in self._capacities(handle, query_states.shape[0])]
        n = key_states.shape[-2] - W
        # the reference slices `sorted_indices[..., :cap]` (pyramidkv_utils.py:738-744 / :866-872): a budget above the n
        # candidates keeps all n of them, a negative one keeps none
        caps = [min(max(c, 0), n) for c in caps]
        self.last_capacities = caps
        k_buf, v_buf = self.backend.ragged_finish(handle, caps, reserve)
        return k_buf, v_buf, [c + W for c in caps]

    def update_kv(self, key_states, query_states, value_states):
        """Reference signature (pyramidkv_utils.py:674 / :808): K/V [1, H, S, D] (repeat_kv-expanded or not) -> the FLAT
        [sum_h len_h, D] tensors the reference returns, with its metadata attributes set."""
        bsz, num_heads, q_len, head_dim = query_states.shape
        assert bsz == 1                                                     # :723
        if not self.compressed(q_len):
            self._init_metadata([q_len] * num_heads, key_states.device)
            rep = num_heads // key_states.shape[1]
            K = key_states.repeat_interleave(rep, dim=1) if rep > 1 else key_states
            V = value_states.repeat_interleave(rep, dim=1) if rep > 1 else value_states
            return K.reshape(-1, head_dim), V.reshape(-1, head_dim)
        k_buf, v_buf, rows = self.evict_ragged(query_states[0], key_states[0], value_states[0])
        self._init_metadata(rows, key_states.device)
        return (torch.cat([k_buf[h, :rows[h]] for h in range(num_heads)], dim=0),
                torch.cat([v_buf[h, :rows[h]] for h in range(num_heads)], dim=0))


class AdaKVCluster(_RaggedCluster):
    """pyramidkv_utils.py:622-757 (adapted there from FFY0/AdaKV): the heads of a layer share num_heads * base_capacity slots
    in proportion to how many of the globally largest (optionally normalised) pooled scores they own, mixed with a floor."""
    method = "adakv"

    def __init__(self, window_size=32, kernel_size=7, pooling="maxpool", max_capacity_prompt=None, floor=None, normalize=None,
                 layer_idx=None, num_hidden_layers=None, backend=None):
        self._init_common(window_size, kernel_size, pooling, max_capacity_prompt, layer_idx, num_hidden_layers, backend)
        self.floor_ratio = floor
        self.floor_capacity = int(self.base_capacity * self.floor_ratio)
        self.adaptive_capacity = self.base_capacity - self.floor_capacity
        self.normalize = normalize

    def _capacities(self, handle, num_heads):
        gt, eq = self.backend.adakv_counts(handle, self.base_capacity, bool(self.normalize))
        need = num_heads * self.base_capacity - sum(gt)
        counts = []
        for h in range(num_heads):          # ties at the threshold: lower flat index first (torch.topk on CUDA) = lower heads first
            take = min(need, eq[h])
            need -= take
            counts.append(gt[h] + take)
        assert need == 0 and sum(counts) == num_heads * self.base_capacity   # :714
        return _round_half_even_f32(counts, 1 - self.floor_ratio, self.floor_capacity)


class HeadKVCluster(_RaggedCluster):
    """pyramidkv_utils.py:760-878: budgets per (layer, head) given by the runner (`head_capacity[layer_idx][head]`)."""
    method = "headkv"

    def __init__(self, window_size=32, kernel_size=7, pooling="maxpool", max_capacity_prompt=None, layer_idx=None,
                 num_hidden_layers=None, head_capacity=None, backend=None):
        self._init_common(window_size, kernel_size, pooling, max_capacity_prompt, layer_idx, num_hidden_layers, backend)
        self.head_adaptive_capacity = head_capacity

    def _capacities(self, handle, num_heads):
        row = self.head_adaptive_capacity[self.layer_idx]
        return [int(row[h]) for h in range(num_heads)]


# ---- init_* factories: read knobs off `self.config`, default them, (re)build the cluster ----
def _default_knobs(module, capacity_default: int) -> None:
    cfg = module.config
    if not hasattr(module, "kv_cluster"):                      # defaults are only filled on first use (:881-891)
        if not hasattr(cfg, "window_size"):
            cfg.window_size = 32
        if not hasattr(cfg, "max_capacity_prompt"):
            cfg.max_capacity_prompt = capacity_default
        if not hasattr(cfg, "kernel_size"):
            cfg.kernel_size = 5
        if not hasattr(cfg, "pooling"):
            cfg.pooling = "avgpool"
        if not hasattr(cfg, "merge"):
            cfg.merge = None


def _knobs(module) -> dict:
    cfg = module.config
    return dict(window_size=cfg.window_size, max_capacity_prompt=cfg.max_capacity_prompt,
                kernel_size=cfg.kernel_size, pooling=cfg.pooling, merge=cfg.merge)


def init_pyramidkv(self, num_hidden_layers):
    """pyramidkv_utils.py:880-902 (default capacity 2048)."""
    _default_knobs(self, 2048)
    self.kv_cluster = PyramidKVCluster(num_hidden_layers=num_hidden_layers, layer_idx=self.layer_idx,
                                       backend=getattr(self, "_pkv_backend", None), **_knobs(self))


def init_snapkv(self):
    """pyramidkv_utils.py:904-924 (default capacity 4096)."""
    _default_knobs(self, 4096)
    self.kv_cluster = SnapKVCluster(backend=getattr(self, "_pkv_backend", None), **_knobs(self))


def init_H2O(self):
    """pyramidkv_utils.py:990-1009."""
    _default_knobs(self, 2048)
    self.kv_cluster = H2OKVCluster(backend=getattr(self, "_pkv_backend", None), **_knobs(self))


def init_StreamingLLM(self):
    """pyramidkv_utils.py:1011-1031."""
    _default_knobs(self, 2048)
    self.kv_cluster = StreamingLLMKVCluster(backend=getattr(self, "_pkv_backend", None), **_knobs(self))


def init_l2norm(self):
    """pyramidkv_utils.py:954-968 (defaults: capacity 4096, skip_layers [0, 1])."""
    cfg = self.config
    if not hasattr(self, "kv_cluster"):
        if not hasattr(cfg, "max_capacity_prompt"):
            cfg.max_capacity_prompt = 4096
        if not hasattr(cfg, "layer_idx"):
            cfg.layer_idx = 0
        if not hasattr(cfg, "skip_layers"):
            cfg.skip_layers = [0, 1]
    self.kv_cluster = L2NormCluster(max_capacity_prompt=cfg.max_capacity_prompt, layer_idx=self.layer_idx,
                                    skip_layers=cfg.skip_layers, backend=getattr(self, "_pkv_backend", None))


def _default_ragged_knobs(cfg):
    if not hasattr(cfg, "window_size"):
        cfg.window_size = 32
    if not hasattr(cfg, "max_capacity_prompt"):
        cfg.max_capacity_prompt = 2048
    if not hasattr(cfg, "kernel_size"):
        cfg.kernel_size = 5
    if not hasattr(cfg, "pooling"):
        cfg.pooling = "maxpool"


def init_adakv(self):
    """pyramidkv_utils.py:1033-1059. The cluster is built once per module (`hasattr` guard :1049); the floor is read from
    `config.floor` (the runner sets it, run_longbench.py:259) although the default is filled into `config.floor_ratio` (:1043)."""
    cfg = self.config
    if not hasattr(self, "kv_cluster"):
        _default_ragged_knobs(cfg)
        if not hasattr(cfg, "floor_ratio"):
            cfg.floor_ratio = 0.2
        if not hasattr(cfg, "normalize"):
            cfg.normalize = True
        self.kv_cluster = AdaKVCluster(num_hidden_layers=cfg.num_hidden_layers, layer_idx=self.layer_idx, window_size=cfg.window_size,
                                       max_capacity_prompt=cfg.max_capacity_prompt, kernel_size=cfg.kernel_size, pooling=cfg.pooling,
                                       floor=cfg.floor, normalize=cfg.normalize, backend=getattr(self, "_pkv_backend", None))


def init_headkv(self):
    """pyramidkv_utils.py:1062-1086 (`config.head_capacity` is mandatory: ValueError("Must have head_capacity") :1073)."""
    cfg = self.config
    if not hasattr(self, "kv_cluster"):
        _default_ragged_knobs(cfg)
        if not hasattr(cfg, "head_capacity"):
            raise ValueError("Must have head_capacity")
        self.kv_cluster = HeadKVCluster(num_hidden_layers=cfg.num_hidden_layers, layer_idx=self.layer_idx, window_size=cfg.window_size,
                                        max_capacity_prompt=cfg.max_capacity_prompt, kernel_size=cfg.kernel_size, pooling=cfg.pooling,
                                        head_capacity=cfg.head_capacity, backend=getattr(self, "_pkv_backend", None))


INIT_BY_METHOD = {
    "pyramidkv": lambda m: init_pyramidkv(m, num_hidden_layers=m.config.num_hidden_layers),
    "snapkv": init_snapkv,
    "h2o": init_H2O,
    "streamingllm": init_StreamingLLM,
    "l2norm": init_l2norm,
    "adakv": init_adakv,
    "headkv": init_headkv,
}
