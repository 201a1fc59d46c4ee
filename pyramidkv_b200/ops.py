"""Tensor-level wrappers over the C ABI (include/pkv.h). PyTorch here is plumbing only: it owns device
memory (caching allocator) and the current stream; all arithmetic of the eviction path runs in libpkv.so.
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass
from typing import Dict, Optional, Tuple

import torch

from . import _lib
from ._lib import METHODS, POOLING, SCORE_KERNELS, DecodeDesc, DecodeHeavy, DecodeMulti, DecodeWindow, EvictDesc, RopeDesc, SpecDesc, WsLayout

_DTYPES = {torch.bfloat16: 0, torch.float16: 1}


def _dtype_code(t: torch.Tensor) -> int:
    try:
        return _DTYPES[t.dtype]
    except KeyError:
        raise NotImplementedError(f"pyramidkv_b200 supports bf16 and fp16 caches, got {t.dtype}") from None


def _require_cuda(*ts: torch.Tensor) -> None:
    for t in ts:
        if t is not None and not t.is_cuda:
            raise RuntimeError("pyramidkv_b200: tensors must live on a CUDA (sm_90a) device — there is no CPU fallback. "
                               "Host buffers go through KVCluster.update_kv, which stages them to the GPU.")


def _hsd(t: torch.Tensor, name: str) -> torch.Tensor:
    """[H, S, D] view (accepts [1, H, S, D]) with a contiguous last dim; strides are taken as they are."""
    if t.dim() == 4:
        if t.shape[0] != 1:
            raise ValueError(f"{name}: batch size must be 1 per call (got {t.shape[0]})")
        t = t[0]
    if t.dim() != 3:
        raise ValueError(f"{name}: expected [H, S, D], got {tuple(t.shape)}")
    if t.stride(-1) != 1 or t.stride(0) % 8 or t.stride(1) % 8 or t.data_ptr() % 16:
        t = t.contiguous()
    return t


def layer_budget(method: str, max_capacity_prompt: int, window_size: int, num_layers: int, layer_idx: int,
                 q_len: int, beta: int = 20) -> Tuple[int, int]:
    """(mode, top_k) exactly as the reference computes it (pyramidkv_utils.py:205-220, :334, :562, :607).
    mode 0: q_len < max_capacity_prompt -> nothing is evicted. Pure host arithmetic in libpkv."""
    assert max_capacity_prompt - window_size > 0           # pyramidkv_utils.py:184
    k, mode = C.c_int64(0), C.c_int(0)
    _lib.check(_lib.lib().pkv_layer_budget(METHODS[method], max_capacity_prompt, window_size, num_layers,
                                           layer_idx if layer_idx is not None else 0, q_len, beta,
                                           C.byref(k), C.byref(mode)))
    return mode.value, k.value


# ---- workspace: one growing uint8 tensor per (device, stream); torch owns the memory ----
_workspaces: Dict[Tuple[int, int], torch.Tensor] = {}


def _workspace(device: torch.device, nbytes: int) -> torch.Tensor:
    key = (device.index if device.index is not None else torch.cuda.current_device(),
           torch.cuda.current_stream(device).cuda_stream)
    ws = _workspaces.get(key)
    if ws is None or ws.numel() < nbytes:
        ws = torch.empty(max(nbytes, 1 << 20), dtype=torch.uint8, device=device)
        _workspaces[key] = ws
    return ws


@dataclass
class EvictPlan:
    """A filled descriptor plus the tensors that keep its pointers alive."""
    desc: EvictDesc
    layout: WsLayout
    workspace: torch.Tensor
    keep: tuple

    def stream_ptr(self) -> int:
        return torch.cuda.current_stream(self.workspace.device).cuda_stream


def plan_evict(method: str, q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, window_size: int, top_k: int,
               k_cache: torch.Tensor, v_cache: torch.Tensor, kernel_size: int = 5, pooling: str = "avgpool",
               idx_out: Optional[torch.Tensor] = None, score_kernel: str = "auto",
               workspace: Optional[torch.Tensor] = None, window_mean: bool = False, staged: bool = False,
               inputs_ready: bool = False, single_launch: bool = False, fused: bool = False,
               gqa_shared: bool = False) -> EvictPlan:
    """`staged`: PKV_FLAG_STAGED (stages 1-4 as separate launches even where the fused kernel applies). `single_launch`:
    PKV_FLAG_SINGLE_LAUNCH (stages 1-4 in ONE launch instead of the default fused stages 1-2 + select kernel). `fused`:
    PKV_FLAG_FUSED (the fused stages 1-2 kernel for every supported shape, not only where it is measured faster).
    `inputs_ready`: PKV_FLAG_INPUTS_READY (q/k/v were not written by the kernel just before this call: K streaming may
    start early). `gqa_shared`: PKV_FLAG_GQA_SHARED (one selection and one cache per KV head: k_cache / v_cache are
    [Hkv, capacity, D] and idx_out [Hkv, top_k]; include/pkv.h gives the group reduction)."""
    if method not in METHODS:
        raise ValueError(f"unknown method {method!r}")
    if pooling not in POOLING:
        if method in ("pyramidkv", "snapkv"):
            raise ValueError("Pooling method not supported")   # pyramidkv_utils.py:237
        pooling = "avgpool"
    _require_cuda(q, k, v, k_cache, v_cache, idx_out)
    k, v = _hsd(k, "key_states"), _hsd(v, "value_states")
    kc, vc = k_cache, v_cache
    if kc.dim() == 4:
        kc, vc = kc[0], vc[0]
    Hkv, S = k.shape[0], k.shape[1]
    if method == "l2norm":
        # L2NormCluster reads no queries (pyramidkv_utils.py:406-431): q is ignored (may be None); heads come from the cache
        if window_size != 0:
            raise ValueError("l2norm keeps no observation window: window_size must be 0")
        q = None
        Hq, Sq, D = kc.shape[0], S, k.shape[2]
        q_tail = False
    else:
        q = _hsd(q, "query_states")
        Hq, Sq, D = q.shape
        # q is either the whole [Hq, S, D] tensor or just its last `window_size` rows (all the window methods read)
        # (StreamingLLM never reads q at all.)
        q_tail = Sq != S and method != "h2o" and (Sq == window_size or method == "streamingllm")
        assert Sq == S or q_tail                                   # pyramidkv_utils.py:200
    Hc = Hkv if gqa_shared else Hq            # heads of the cache
    if not (kc.is_contiguous() and vc.is_contiguous()) or kc.shape != vc.shape or kc.shape[0] != Hc or kc.shape[2] != D:
        raise ValueError(f"k_cache/v_cache must be contiguous [{'Hkv' if gqa_shared else 'Hq'}, capacity, D] tensors of equal shape")
    d = EvictDesc()
    d.struct_bytes = C.sizeof(EvictDesc)
    d.method, d.dtype, d.pooling, d.kernel_size = METHODS[method], _dtype_code(k), POOLING[pooling], int(kernel_size)
    d.num_q_heads, d.num_kv_heads, d.head_dim, d.window = Hq, Hkv, D, int(window_size)
    d.device = k.device.index if k.device.index is not None else torch.cuda.current_device()
    d.seq_len, d.top_k = S, int(top_k)
    if q is not None:
        # for a tail-only q the base pointer is shifted so that row S-W+w of the logical tensor is q[:, w]
        d.q = q.data_ptr() - ((S - Sq) * q.stride(1) * 2 if (q_tail and method != "streamingllm") else 0)
        d.q_stride_h, d.q_stride_s = q.stride(0), q.stride(1)
    else:
        d.q, d.q_stride_h, d.q_stride_s = None, 0, D
    d.k, d.k_stride_h, d.k_stride_s = k.data_ptr(), k.stride(0), k.stride(1)
    d.v, d.v_stride_h, d.v_stride_s = v.data_ptr(), v.stride(0), v.stride(1)
    d.k_cache, d.v_cache, d.cache_stride_h = kc.data_ptr(), vc.data_ptr(), kc.stride(0)
    if idx_out is not None:
        if idx_out.dtype != torch.int64 or not idx_out.is_contiguous() or idx_out.numel() != Hc * top_k:
            raise ValueError("idx_out must be a contiguous int64 [heads of the cache, top_k] tensor")
        d.idx_out = idx_out.data_ptr()
    d.flags = SCORE_KERNELS[score_kernel] | (4 if window_mean else 0) | (8 if inputs_ready else 0) | (16 if staged else 0) | (32 if single_launch else 0) | (64 if fused else 0)
    d.flags |= _lib.FLAG_GQA_SHARED if gqa_shared else 0
    L = WsLayout()
    _lib.check(_lib.lib().pkv_evict_workspace_layout(C.byref(d), C.byref(L)))
    ws = workspace if workspace is not None else _workspace(k.device, int(L.total_bytes))
    d.workspace, d.workspace_bytes = ws.data_ptr(), ws.numel()
    return EvictPlan(d, L, ws, (q, k, v, kc, vc, idx_out))


def workspace_bytes_for(plan: EvictPlan, top_k: int) -> int:
    """Workspace size of the same eviction with another top_k (the segments in front of idx32 do not move)."""
    d = EvictDesc.from_buffer_copy(plan.desc)
    d.top_k = int(top_k)
    return int(_lib.lib().pkv_evict_workspace_bytes(C.byref(d)))


def evict_prefill(method: str, q, k, v, window_size: int, top_k: int, k_cache, v_cache, kernel_size: int = 5,
                  pooling: str = "avgpool", idx_out=None, score_kernel: str = "auto", inputs_ready: bool = False,
                  gqa_shared: bool = False) -> None:
    """One layer's prefill eviction on the current CUDA stream (asynchronous).

    q [Hq,S,D]; k, v [Hkv,S,D] un-repeated (or Hkv == Hq after repeat_kv); writes rows 0..top_k+W-1 of
    k_cache/v_cache [Hq, capacity, D] ([Hkv, capacity, D] with `gqa_shared`). Replaces *KVCluster.update_kv
    (pyramidkv_utils.py:197-620)."""
    plan = plan_evict(method, q, k, v, window_size, top_k, k_cache, v_cache, kernel_size, pooling, idx_out, score_kernel,
                      inputs_ready=inputs_ready, gqa_shared=gqa_shared)
    _lib.check(_lib.lib().pkv_evict_prefill(C.byref(plan.desc), plan.stream_ptr()))


def batch_workspaces(plan: EvictPlan, n_layers: int, max_top_k: Optional[int] = None) -> list:
    """`n_layers` disjoint workspaces (256-byte aligned slices of ONE allocation) for a layer batch: unlike the per-layer
    calls, which reuse one workspace in stream order, the layers of a batch are in flight together. `plan` is any layer's
    plan; `max_top_k` the largest budget among the layers (the index segments grow with top_k)."""
    nbytes = workspace_bytes_for(plan, max_top_k) if max_top_k is not None else int(plan.layout.total_bytes)
    nbytes = (nbytes + 255) // 256 * 256
    big = torch.empty(nbytes * n_layers, dtype=torch.uint8, device=plan.workspace.device)
    return [big[i * nbytes:(i + 1) * nbytes] for i in range(n_layers)]


def _desc_array(plans):
    arr = (EvictDesc * len(plans))()
    for i, p in enumerate(plans):
        C.memmove(C.byref(arr, i * C.sizeof(EvictDesc)), C.byref(p.desc), C.sizeof(EvictDesc))
    return arr


def batch_supported(plans) -> bool:
    """Can these layers' evictions run as ONE layer batch (pkv_evict_prefill_batch)? Window methods, identical geometry."""
    if len(plans) < 2 or len({p.workspace.data_ptr() for p in plans}) != len(plans):
        return False
    return bool(_lib.lib().pkv_evict_batch_supported(_desc_array(plans), len(plans)))


class EvictBatch:
    """The descriptors of several layers as one contiguous array (built once, launched many times)."""
    STAGES = {"all": 0, "scores": 1, "pool": 2, "select": 3}

    def __init__(self, plans):
        if len({p.workspace.data_ptr() for p in plans}) != len(plans):
            raise ValueError("evict_prefill_batch: every layer needs its own workspace (ops.batch_workspaces)")
        self.plans = list(plans)
        self.descs = _desc_array(self.plans)

    def run(self, stage: str = "all") -> None:
        _lib.check(_lib.lib().pkv_stage_batch(self.descs, len(self.plans), self.STAGES[stage], self.plans[0].stream_ptr()))


def evict_prefill_batch(plans) -> None:
    """The evictions of several layers of one prompt in one pass (four launches per 32 layers) on the current stream.
    Every plan needs its OWN workspace (`batch_workspaces`). Raises NotImplementedError when the layers cannot share
    a launch (`batch_supported` asks first)."""
    EvictBatch(plans).run()


def host_pick_rows(src: torch.Tensor, rows: torch.Tensor) -> torch.Tensor:
    """src: HOST tensor [Hkv, S, D] (any strides with a contiguous last dim); rows: int64 [Hq, n_rows] on the host.
    Returns a dense host tensor [Hq, n_rows, D], head h reading kv head h // (Hq // Hkv). No device work
    (`pkv_host_pick_rows`): the host half of the compaction when V is host-resident."""
    if src.is_cuda or rows.is_cuda or rows.dtype != torch.int64 or src.dim() != 3 or rows.dim() != 2 or src.stride(2) != 1:
        raise ValueError("host_pick_rows: src must be a host [Hkv, S, D] tensor with a contiguous last dim, rows a host int64 [Hq, n]")
    rows = rows.contiguous()
    Hkv, S, D = src.shape
    Hq, n = rows.shape
    out = torch.empty(Hq, n, D, dtype=src.dtype)
    if n == 0:
        return out
    e = src.element_size()
    _lib.check(_lib.lib().pkv_host_pick_rows(src.data_ptr(), src.stride(0) * e, src.stride(1) * e, S, Hkv, Hq, D * e,
                                              rows.data_ptr(), n, out.data_ptr()))
    return out


def run_stage(plan: EvictPlan, stage: str) -> None:
    fn = getattr(_lib.lib(), {"scores": "pkv_stage_scores", "pool": "pkv_stage_pool", "topk": "pkv_stage_topk",
                              "gather": "pkv_stage_gather", "all": "pkv_evict_prefill", "scan_pool": "pkv_stage_scan_pool"}[stage])
    _lib.check(fn(C.byref(plan.desc), plan.stream_ptr()))


# ---- workspace views for stage-injection tests / debugging ----
def ws_logits(plan: EvictPlan) -> torch.Tensor:
    """[Hkv, s_pad, nw] view of the masked logits (model dtype); column = head_in_group*W + w."""
    d, L = plan.desc, plan.layout
    dt = torch.bfloat16 if d.dtype == 0 else torch.float16
    n = d.num_kv_heads * L.s_pad * L.nw
    return plan.workspace[L.logits_off:L.logits_off + 2 * n].view(dt).view(d.num_kv_heads, L.s_pad, L.nw)


def ws_logits_as_reference(plan: EvictPlan) -> torch.Tensor:
    """The same logits permuted to the reference layout [Hq, W, S]."""
    d = plan.desc
    G = d.num_q_heads // d.num_kv_heads
    x = ws_logits(plan)[:, :d.seq_len, :].reshape(d.num_kv_heads, d.seq_len, G, d.window)
    return x.permute(0, 2, 3, 1).reshape(d.num_q_heads, d.window, d.seq_len).contiguous()


def ws_partials(plan: EvictPlan) -> torch.Tensor:
    """[Hkv, n_slots, nw, 2] float32 (max, sumexp) per 128-token tile."""
    d, L = plan.desc, plan.layout
    n = d.num_kv_heads * L.n_slots * L.nw * 2
    return plan.workspace[L.partial_off:L.partial_off + 4 * n].view(torch.float32).view(d.num_kv_heads, L.n_slots, L.nw, 2)


def ws_pooled(plan: EvictPlan) -> torch.Tensor:
    """[Hq, S-W] view of the top-k input (pooled scores)."""
    d, L = plan.desc, plan.layout
    dt = torch.bfloat16 if d.dtype == 0 else torch.float16
    n = d.num_q_heads * L.pooled_pitch
    return plan.workspace[L.pooled_off:L.pooled_off + 2 * n].view(dt).view(d.num_q_heads, L.pooled_pitch)[:, :d.seq_len - d.window]


def ws_pooled_kv(plan: EvictPlan) -> torch.Tensor:
    """[Hkv, S-W] view of the per-KV-head top-k input of a `gqa_shared` plan (the group reduction of `ws_pooled`)."""
    d, L = plan.desc, plan.layout
    off = C.c_uint64(0)
    _lib.check(_lib.lib().pkv_evict_pooled_kv_offset(C.byref(d), C.byref(off)))
    off = int(off.value)
    dt = torch.bfloat16 if d.dtype == 0 else torch.float16
    n = d.num_kv_heads * L.pooled_pitch
    return plan.workspace[off:off + 2 * n].view(dt).view(d.num_kv_heads, L.pooled_pitch)[:, :d.seq_len - d.window]


def single_launch(plan: EvictPlan) -> int:
    """How `pkv_evict_prefill` runs this plan: 0 staged launches, 1 fused stages 1-2 (pkv_evict_fused.cu) + select kernel,
    2 everything in one launch."""
    return int(_lib.lib().pkv_evict_single_launch(C.byref(plan.desc)))


def ws_fused_status(plan: EvictPlan) -> int:
    """Status word of the single-launch kernel's exchange area: 0, or 1 + the exchange whose wait timed out."""
    off = int(plan.layout.fused_off) + 8
    return int(plan.workspace[off:off + 4].view(torch.int32).item())


def ws_idx32(plan: EvictPlan) -> torch.Tensor:
    d, L = plan.desc, plan.layout
    n = d.num_q_heads * d.top_k
    return plan.workspace[L.idx32_off:L.idx32_off + 4 * n].view(torch.int32).view(d.num_q_heads, d.top_k)


# ---- ragged per-head budgets (AdaKV / HeadKV) ----
def adakv_counts(plan: EvictPlan, base_capacity: int, normalize: bool):
    """After stages 1-2 of `plan` (method snapkv): per head, the (normalised) pooled scores above / equal to the value of rank
    Hq * base_capacity over all heads (`pkv_adakv_counts`; pyramidkv_utils.py:702-712). Returns host lists (gt, eq) — one
    small device-to-host copy, like the reference's own `.item()` at :714."""
    Hq = plan.desc.num_q_heads
    dev = plan.workspace.device
    scratch = torch.empty(int(_lib.lib().pkv_adakv_scratch_bytes(Hq)), dtype=torch.uint8, device=dev)
    counts = torch.empty(2 * Hq + 2, dtype=torch.int32, device=dev)
    _lib.check(_lib.lib().pkv_adakv_counts(C.byref(plan.desc), int(base_capacity), int(bool(normalize)), scratch.data_ptr(),
                                           scratch.numel(), counts.data_ptr(), plan.stream_ptr()))
    host = counts.cpu().tolist()
    return host[:Hq], host[Hq:2 * Hq]


def ragged_place_window(plan: EvictPlan, caps: torch.Tensor) -> None:
    """Rows [caps[h], caps[h] + W) of head h <- the last W source rows (`pkv_ragged_place_window`); caps int32 [Hq] on the device."""
    _require_cuda(caps)
    if caps.dtype != torch.int32 or caps.numel() != plan.desc.num_q_heads or not caps.is_contiguous():
        raise ValueError("caps must be a contiguous int32 [Hq] device tensor")
    _lib.check(_lib.lib().pkv_ragged_place_window(C.byref(plan.desc), caps.data_ptr(), plan.stream_ptr()))


# ---- the step in front of the path ----
def rope_inplace(q: torch.Tensor, k: torch.Tensor, cos: torch.Tensor, sin: torch.Tensor) -> None:
    """Rotary embedding of q [Hq, S, D] and k [Hkv, S, D] IN PLACE (any 16-byte-aligned strides, e.g. HF's transposed views of
    the projection outputs); cos/sin [S, D] in the model dtype. One launch; bit-identical to HF `apply_rotary_pos_emb`
    (llama_model.py:157 / :276 / :378)."""
    _require_cuda(q, k, cos, sin)
    if q.dim() != 3 or k.dim() != 3 or cos.dim() != 2 or cos.shape != sin.shape or cos.shape != (q.shape[1], q.shape[2]) \
            or k.shape[1:] != q.shape[1:] or q.dtype != k.dtype or cos.dtype != q.dtype or sin.dtype != q.dtype:
        raise ValueError("rope_inplace: q [Hq,S,D], k [Hkv,S,D], cos/sin [S,D], one dtype")
    for t in (q, k, cos, sin):
        if t.stride(-1) != 1 or any(s % 8 for s in t.stride()[:-1]) or t.data_ptr() % 16:
            raise ValueError("rope_inplace: tensors need a contiguous last dim, strides that are multiples of 8 elements and "
                             "16-byte-aligned storage (in-place operation: no staging copy is made)")
    if sin.stride(0) != cos.stride(0):
        sin = sin.contiguous()
        cos = cos.contiguous()
    d = RopeDesc()
    d.struct_bytes = C.sizeof(RopeDesc)
    d.dtype, d.num_q_heads, d.num_kv_heads, d.head_dim = _dtype_code(q), q.shape[0], k.shape[0], q.shape[2]
    d.device = q.device.index if q.device.index is not None else torch.cuda.current_device()
    d.seq_len = q.shape[1]
    d.q, d.q_stride_h, d.q_stride_s = q.data_ptr(), q.stride(0), q.stride(1)
    d.k, d.k_stride_h, d.k_stride_s = k.data_ptr(), k.stride(0), k.stride(1)
    d.cos, d.sin, d.cs_stride_s = cos.data_ptr(), sin.data_ptr(), cos.stride(0)
    _lib.check(_lib.lib().pkv_rope_inplace(C.byref(d), torch.cuda.current_stream(q.device).cuda_stream))


# ---- decode ----
def decode_attn(q: torch.Tensor, k_cache: torch.Tensor, v_cache: torch.Tensor, length: int,
                k_new: Optional[torch.Tensor] = None, v_new: Optional[torch.Tensor] = None,
                out: Optional[torch.Tensor] = None, softmax_scale: float = 0.0,
                step: Optional[torch.Tensor] = None, max_length: int = 0,
                workspace: Optional[torch.Tensor] = None, head_rows: Optional[torch.Tensor] = None) -> torch.Tensor:
    """q [Hq, D]; caches [Hq, capacity, D]; `length` = valid rows AFTER appending k_new/v_new [Hkv, D] (if given).
    Returns out [Hq, D]. Replaces torch.cat + attention of the decode step (llama_model.py:170-183 / :403-445).

    Graph-replayable form (`pkv_decode_attn_graph`): `step` is an int32 device scalar the kernel adds to `length`
    (which is then the row count at step 0), `max_length` the row count the launch is sized for (default: the cache
    capacity); pass a `workspace` that outlives the captured graph.

    Ragged caches (AdaKV / HeadKV, `pkv_decode_attn_ragged`): `head_rows` int32 [Hq] on the device holds every head's own
    row count after the prefill; `length` then counts only the rows appended since (including this step's)."""
    _require_cuda(q, k_cache, v_cache, k_new, v_new, out, step, workspace, head_rows)
    if k_cache.dim() == 4:
        k_cache, v_cache = k_cache[0], v_cache[0]
    Hq, cap, D = k_cache.shape
    q = q.reshape(Hq, D)
    if not q.is_contiguous():
        q = q.contiguous()
    if out is None:
        out = torch.empty(Hq, D, dtype=q.dtype, device=q.device)
    d = DecodeDesc()
    d.struct_bytes = C.sizeof(DecodeDesc)
    d.dtype, d.num_q_heads, d.head_dim = _dtype_code(q), Hq, D
    d.device = q.device.index if q.device.index is not None else torch.cuda.current_device()
    d.length = int(length)
    d.q, d.k_cache, d.v_cache, d.cache_stride_h, d.out = q.data_ptr(), k_cache.data_ptr(), v_cache.data_ptr(), k_cache.stride(0), out.data_ptr()
    keep = [q, out]
    if k_new is not None:
        k_new = k_new.reshape(-1, D)
        v_new = v_new.reshape(-1, D)
        if not k_new.is_contiguous():
            k_new = k_new.contiguous()
        if not v_new.is_contiguous():
            v_new = v_new.contiguous()
        d.num_kv_heads = k_new.shape[0]
        d.k_new, d.v_new = k_new.data_ptr(), v_new.data_ptr()
        keep += [k_new, v_new]
    else:
        d.num_kv_heads = Hq
    if length > cap:
        raise ValueError(f"cache capacity {cap} exceeded (length {length})")
    if head_rows is not None and (head_rows.dtype != torch.int32 or head_rows.numel() != Hq or not head_rows.is_contiguous()):
        raise ValueError("head_rows must be a contiguous int32 [Hq] device tensor")
    nbytes = int(_lib.lib().pkv_decode_workspace_bytes(C.byref(d)))
    ws = workspace if workspace is not None else _workspace(q.device, nbytes)
    d.workspace, d.workspace_bytes = ws.data_ptr(), ws.numel() * ws.element_size()
    d.softmax_scale = float(softmax_scale)
    stream = torch.cuda.current_stream(q.device).cuda_stream
    if head_rows is not None:
        if step is not None and (step.dtype != torch.int32 or step.numel() != 1):
            raise ValueError("step must be an int32 device tensor with one element")
        _lib.check(_lib.lib().pkv_decode_attn_ragged(C.byref(d), head_rows.data_ptr(), step.data_ptr() if step is not None else None,
                                                     int(max_length) or cap, stream))
    elif step is None:
        _lib.check(_lib.lib().pkv_decode_attn(C.byref(d), stream))
    else:
        if step.dtype != torch.int32 or step.numel() != 1:
            raise ValueError("step must be an int32 device tensor with one element")
        _lib.check(_lib.lib().pkv_decode_attn_graph(C.byref(d), step.data_ptr(), int(max_length) or cap, stream))
    return out


def decode_attn_batch(q: torch.Tensor, k_buf: torch.Tensor, v_buf: torch.Tensor, length: int,
                      k_new: Optional[torch.Tensor] = None, v_new: Optional[torch.Tensor] = None,
                      rows: Optional[torch.Tensor] = None, step: Optional[torch.Tensor] = None, max_length: int = 0,
                      workspace: Optional[torch.Tensor] = None, out: Optional[torch.Tensor] = None,
                      softmax_scale: float = 0.0) -> torch.Tensor:
    """The decode step of B sequences in ONE launch (`pkv_decode_attn_batch`). q [B, Hq, D] (e.g. HF's
    `query_states[:, :, 0, :]`); buffers [B, Hq, capacity, D]; k_new / v_new [B, Hkv, D] appended as each sequence's last
    row. Sequence b, head h attends `length` (+ `*step`) (+ `rows[b*Hq + h]`) rows: `rows` is an int32 device tensor
    [B*Hq] (or [B, Hq]) or None (every sequence holds `length` rows). The launch is sized for `max_length` rows (default:
    the capacity) and is graph-replayable; every sequence's output and appended row are bit-identical to `decode_attn` in
    the graph form (or the ragged form, for per-head rows) on that sequence alone. Returns out [B, Hq, D]."""
    return _decode_batch("pkv_decode_attn_batch", "decode_attn_batch", q, k_buf, v_buf, None, length, k_new, v_new,
                         rows, step, max_length, workspace, out, softmax_scale)


def _decode_batch(entry, what, q, k_buf, v_buf, scales, length, k_new, v_new, rows, step, max_length, workspace, out,
                  softmax_scale, gqa: bool = False, window: int = 0, prompt_rows: Optional[torch.Tensor] = None,
                  heavy=None) -> torch.Tensor:
    """The checks and the descriptor of the batched decode launches, then the launch of the C entry point `entry`.
    `scales`: (k_scale, v_scale) of an FP8 cache, or None. `gqa`: a GQA-shared cache (k_buf / v_buf [B, Hkv, capacity, D],
    q [B, Hq, D]). `window` > 0: the decode window over `prompt_rows` (`pkv_decode_attn_window`); with `heavy` = (H, scores,
    gen, victim, scratch) its heavy hitters (`pkv_decode_attn_heavy`)."""
    _require_cuda(q, k_buf, v_buf, k_new, v_new, rows, step, workspace, out, prompt_rows, *(scales or ()), *(heavy or ())[1:])
    if scales is not None:
        _check_fp8_buffers(k_buf, v_buf, scales[0], scales[1], what)
    elif k_buf.dim() != 4 or k_buf.shape != v_buf.shape or k_buf.stride() != v_buf.stride() or k_buf.stride(3) != 1 \
            or k_buf.stride(2) != k_buf.shape[3]:
        raise ValueError(f"{what}: k_buf / v_buf must be [B, H, capacity, D] tensors of equal shape and strides, rows contiguous")
    B, H, cap, D = k_buf.shape
    heads = "Hkv" if gqa else "Hq"        # the heads of the cache
    if q.dim() != 3 or q.shape[0] != B or q.shape[2] != D or (q.shape[1] % H if gqa else q.shape[1] != H):
        raise ValueError(f"{what}: q must be [B, Hq, D] with B = {B}, D = {D} and Hq "
                         f"{'a multiple of Hkv = ' if gqa else '= '}{H}, got {tuple(q.shape)}")
    Hq = q.shape[1]
    q = q.contiguous()
    if out is None:
        out = torch.empty(B, Hq, D, dtype=q.dtype, device=q.device)
    elif out.shape != (B, Hq, D) or not out.is_contiguous() or out.dtype != q.dtype:
        raise ValueError(f"{what}: out must be a contiguous [B, Hq, D] tensor of q's dtype")
    max_length = int(max_length) or cap
    if not 1 <= length <= max_length <= cap:
        raise ValueError(f"{what}: cache capacity {cap} exceeded or bad row counts (length {length}, max_length {max_length})")
    if step is not None and (step.dtype != torch.int32 or step.numel() != 1):
        raise ValueError("step must be an int32 device tensor with one element")
    if window:
        if prompt_rows is None or prompt_rows.dtype != torch.int32 or prompt_rows.numel() != B * H or not prompt_rows.is_contiguous():
            raise ValueError(f"{what}: prompt_rows must be a contiguous int32 device tensor of B*{heads} = {B * H} elements")
        if not torch.cuda.is_current_stream_capturing():
            # the rows attended: min(n, P + R) per (sequence, cache head) (one device read; a captured launch relies on the caller)
            n = (rows.reshape(-1).long() if rows is not None else 0) + int(length) + (int(step) if step is not None else 0)
            most = int(torch.minimum(prompt_rows.reshape(-1).long() + int(window),
                                     n if torch.is_tensor(n) else torch.full_like(prompt_rows.reshape(-1).long(), n)).max())
            if most > max_length:
                raise ValueError(f"{what}: cache capacity exceeded: {most} rows for max_length {max_length} (capacity {cap})")
    if rows is not None:
        if rows.dtype != torch.int32 or rows.numel() != B * H or not rows.is_contiguous():
            raise ValueError(f"{what}: rows must be a contiguous int32 device tensor of B*{heads} = {B * H} elements")
        if not window and not torch.cuda.is_current_stream_capturing():
            # (one device read; a captured launch relies on the caller, and the kernel reads and writes no row of a
            # (sequence, head) whose count exceeds max_length)
            most = int(rows.max()) + int(length) + (int(step) if step is not None else 0)
            if most > max_length:
                raise ValueError(f"{what}: cache capacity exceeded: {most} rows for max_length {max_length} (capacity {cap})")
    d = DecodeDesc()
    d.struct_bytes = C.sizeof(DecodeDesc)
    d.dtype, d.num_q_heads, d.num_kv_heads, d.head_dim = _dtype_code(q), B * Hq, H, D
    d.device = q.device.index if q.device.index is not None else torch.cuda.current_device()
    d.length = int(length)
    d.q, d.k_cache, d.v_cache, d.cache_stride_h, d.out = q.data_ptr(), k_buf.data_ptr(), v_buf.data_ptr(), k_buf.stride(1), out.data_ptr()
    keep = [q, out]
    if k_new is not None:
        if k_new.dim() != 3 or k_new.shape[0] != B or k_new.shape[2] != D or (gqa and k_new.shape[1] != H) or v_new is None \
                or v_new.shape != k_new.shape or k_new.dtype != q.dtype or v_new.dtype != q.dtype:
            raise ValueError(f"{what}: k_new / v_new must be [B, Hkv, D] tensors of q's dtype"
                             + (f", Hkv = {H}" if gqa else ""))
        k_new, v_new = k_new.contiguous(), v_new.contiguous()
        d.num_kv_heads = k_new.shape[1]
        d.k_new, d.v_new = k_new.data_ptr(), v_new.data_ptr()
        keep += [k_new, v_new]
    nbytes = int(_lib.lib().pkv_decode_workspace_bytes(C.byref(d)))      # one set of split partials per (sequence, query head)
    d.num_q_heads = Hq
    ws = workspace if workspace is not None else _workspace(q.device, nbytes)
    d.workspace, d.workspace_bytes = ws.data_ptr(), ws.numel() * ws.element_size()
    d.softmax_scale = float(softmax_scale)
    if window:
        w = DecodeWindow()
        w.struct_bytes = C.sizeof(DecodeWindow)
        w.num_seqs, w.cache_stride_b, w.gqa_shared, w.window = B, k_buf.stride(0), int(gqa), int(window)
        w.rows = rows.data_ptr() if rows is not None else None
        w.prompt_rows = prompt_rows.data_ptr()
        w.step_dev = step.data_ptr() if step is not None else None
        w.max_length = max_length
        if scales is not None:
            w.k_scale, w.v_scale = scales[0].data_ptr(), scales[1].data_ptr()
            w.scale_stride_h, w.scale_stride_b = scales[0].stride(1), scales[0].stride(0)
        stream = torch.cuda.current_stream(q.device).cuda_stream
        if heavy is not None:
            H_, scores, gen, victim, scratch = heavy
            for t, dt, n in ((scores, torch.float32, B * H * window), (gen, torch.int32, B * H * window), (victim, torch.int32, B * H)):
                if t.dtype != dt or t.numel() != n or not t.is_contiguous():
                    raise ValueError(f"{what}: scores / gen / victim must be contiguous {dt} device tensors of {n} elements")
            if scratch is None:
                scratch = _heavy_scratch(q.device, decode_heavy_workspace_bytes(B, Hq, window))
            hv = DecodeHeavy()
            hv.struct_bytes = C.sizeof(DecodeHeavy)
            hv.heavy = int(H_)
            hv.scores, hv.gen, hv.victim = scores.data_ptr(), gen.data_ptr(), victim.data_ptr()
            hv.scratch, hv.scratch_bytes = scratch.data_ptr(), scratch.numel() * scratch.element_size()
            _lib.check(_lib.lib().pkv_decode_attn_heavy(C.byref(d), C.byref(w), C.byref(hv), stream))
        else:
            _lib.check(_lib.lib().pkv_decode_attn_window(C.byref(d), C.byref(w), stream))
        return out
    args = (C.byref(d), B, k_buf.stride(0), rows.data_ptr() if rows is not None else None,
            step.data_ptr() if step is not None else None, max_length)
    if scales is not None:
        ks, vs = scales
        args += (ks.data_ptr(), vs.data_ptr(), ks.stride(1), ks.stride(0))
    _lib.check(getattr(_lib.lib(), entry)(*args, torch.cuda.current_stream(q.device).cuda_stream))
    return out


# ---- the opt-in FP8 (E4M3) compacted cache (include/pkv.h: pkv_cache_quantize_fp8, pkv_decode_attn_batch_fp8) ----
FP8_DTYPE = torch.float8_e4m3fn


def _check_fp8_buffers(kq: torch.Tensor, vq: torch.Tensor, ks: torch.Tensor, vs: torch.Tensor, what: str):
    if kq.dtype != FP8_DTYPE or vq.dtype != FP8_DTYPE:
        raise ValueError(f"{what}: the FP8 buffers must be torch.float8_e4m3fn, got {kq.dtype} / {vq.dtype}")
    if kq.dim() != 4 or kq.shape != vq.shape or not kq.is_contiguous() or not vq.is_contiguous():
        raise ValueError(f"{what}: the FP8 buffers must be contiguous [B, Hq, capacity, D] tensors of equal shape")
    if ks.dtype != torch.float32 or vs.dtype != torch.float32 or ks.shape != kq.shape[:3] or vs.shape != ks.shape \
            or not ks.is_contiguous() or not vs.is_contiguous():
        raise ValueError(f"{what}: the scales must be contiguous float32 [B, Hq, capacity] = {tuple(kq.shape[:3])} tensors")
    if kq.data_ptr() % 16 or vq.data_ptr() % 16:
        raise ValueError(f"{what}: the FP8 buffers must be 16-byte aligned")


def cache_quantize_fp8(layers) -> None:
    """Convert the compacted 16-bit caches of several layers to FP8 on the current stream: one launch per 32 layers
    (`pkv_cache_quantize_fp8`). `layers`: (k, v, k_q, v_q, k_scale, v_scale, rows, rows_dev) per layer, with k / v the
    16-bit [B, Hq, capacity, D] buffers the eviction wrote, k_q / v_q float8_e4m3fn [B, Hq, capacity', D] and k_scale /
    v_scale float32 [B, Hq, capacity'] to fill; every (sequence, head) converts `rows` rows, or, when `rows_dev` (int32
    [B*Hq] on the device) is given, its own count from it (at most `rows`). Rows past the count are not written."""
    layers = list(layers)
    if not layers:
        return
    k0 = layers[0][0]
    B, Hq, _, D = k0.shape
    n = len(layers)
    src, dst, scl = (C.c_void_p * (2 * n))(), (C.c_void_p * (2 * n))(), (C.c_void_p * (2 * n))()
    scap, dcap, rows_t = (C.c_int64 * n)(), (C.c_int64 * n)(), (C.c_int64 * n)()
    rdev = (C.c_void_p * n)()
    for i, (k, v, kq, vq, ks, vs, rows, rows_dev) in enumerate(layers):
        _require_cuda(k, v, kq, vq, ks, vs, rows_dev)
        if k.dim() != 4 or k.shape != v.shape or not k.is_contiguous() or not v.is_contiguous() or k.dtype != v.dtype:
            raise ValueError(f"cache_quantize_fp8: layer {i}: the 16-bit buffers must be contiguous [B, Hq, capacity, D] tensors of equal shape")
        if k.dtype != k0.dtype or k.device != k0.device or (k.shape[0], k.shape[1], k.shape[3]) != (B, Hq, D):
            raise ValueError(f"cache_quantize_fp8: layer {i}: batch, heads, head_dim, dtype and device must match layer 0")
        _check_fp8_buffers(kq, vq, ks, vs, f"cache_quantize_fp8: layer {i}")
        if (kq.shape[0], kq.shape[1], kq.shape[3]) != (B, Hq, D) or kq.device != k.device:
            raise ValueError(f"cache_quantize_fp8: layer {i}: the FP8 buffers must be [B, Hq, capacity, D] = [{B}, {Hq}, *, {D}] on {k.device}")
        if not 0 <= int(rows) <= min(k.shape[2], kq.shape[2]):
            raise ValueError(f"cache_quantize_fp8: layer {i}: rows={rows} exceeds a capacity ({k.shape[2]}, {kq.shape[2]})")
        if rows_dev is not None and (rows_dev.dtype != torch.int32 or rows_dev.numel() != B * Hq or not rows_dev.is_contiguous()):
            raise ValueError(f"cache_quantize_fp8: layer {i}: rows_dev must be a contiguous int32 device tensor of B*Hq = {B * Hq} elements")
        src[2 * i], src[2 * i + 1] = k.data_ptr(), v.data_ptr()
        dst[2 * i], dst[2 * i + 1] = kq.data_ptr(), vq.data_ptr()
        scl[2 * i], scl[2 * i + 1] = ks.data_ptr(), vs.data_ptr()
        scap[i], dcap[i], rows_t[i] = k.shape[2], kq.shape[2], int(rows)
        rdev[i] = rows_dev.data_ptr() if rows_dev is not None else None
    dev = k0.device.index if k0.device.index is not None else torch.cuda.current_device()
    _lib.check(_lib.lib().pkv_cache_quantize_fp8(_dtype_code(k0), B, Hq, D, dev, n, src, dst, scl, scap, dcap, rows_t,
                                                 rdev if any(l[7] is not None for l in layers) else None,
                                                 torch.cuda.current_stream(k0.device).cuda_stream))


def decode_attn_batch_fp8(q: torch.Tensor, k_q: torch.Tensor, v_q: torch.Tensor, k_scale: torch.Tensor, v_scale: torch.Tensor,
                          length: int, k_new: Optional[torch.Tensor] = None, v_new: Optional[torch.Tensor] = None,
                          rows: Optional[torch.Tensor] = None, step: Optional[torch.Tensor] = None, max_length: int = 0,
                          workspace: Optional[torch.Tensor] = None, out: Optional[torch.Tensor] = None,
                          softmax_scale: float = 0.0) -> torch.Tensor:
    """`decode_attn_batch` over an FP8 cache (`pkv_decode_attn_batch_fp8`): k_q / v_q float8_e4m3fn [B, Hq, capacity, D],
    k_scale / v_scale float32 [B, Hq, capacity]; q [B, Hq, D] and k_new / v_new [B, Hkv, D] in bf16 / fp16. The new row
    is quantised, stored (bytes and scale) and attended as stored. The same row counts, launch sizing and graph
    replayability as `decode_attn_batch`; one sequence is B = 1 (step None for a host launch). Returns out [B, Hq, D]."""
    return _decode_batch("pkv_decode_attn_batch_fp8", "decode_attn_batch_fp8", q, k_q, v_q, (k_scale, v_scale), length,
                         k_new, v_new, rows, step, max_length, workspace, out, softmax_scale)


# ---- GQA-shared caches (PKV_FLAG_GQA_SHARED): one cache per KV head, decoded once per group ----
def decode_attn_batch_gqa(q: torch.Tensor, k_buf: torch.Tensor, v_buf: torch.Tensor, length: int,
                          k_new: Optional[torch.Tensor] = None, v_new: Optional[torch.Tensor] = None,
                          rows: Optional[torch.Tensor] = None, step: Optional[torch.Tensor] = None, max_length: int = 0,
                          workspace: Optional[torch.Tensor] = None, out: Optional[torch.Tensor] = None,
                          softmax_scale: float = 0.0) -> torch.Tensor:
    """`decode_attn_batch` over GQA-shared caches (`pkv_decode_attn_batch_gqa`): buffers [B, Hkv, capacity, D], one per KV
    head, read once for the Hq / Hkv query heads of its group; q / out [B, Hq, D]; k_new / v_new [B, Hkv, D]; `rows` int32
    [B*Hkv]. Query head h's output and the appended row are bit-identical to `decode_attn_batch` over the cache
    repeat-interleaved along the heads. Workspace: `decode_workspace_bytes(B*Hq, D)`."""
    return _decode_batch("pkv_decode_attn_batch_gqa", "decode_attn_batch_gqa", q, k_buf, v_buf, None, length, k_new,
                         v_new, rows, step, max_length, workspace, out, softmax_scale, gqa=True)


def decode_attn_batch_gqa_fp8(q: torch.Tensor, k_q: torch.Tensor, v_q: torch.Tensor, k_scale: torch.Tensor, v_scale: torch.Tensor,
                              length: int, k_new: Optional[torch.Tensor] = None, v_new: Optional[torch.Tensor] = None,
                              rows: Optional[torch.Tensor] = None, step: Optional[torch.Tensor] = None, max_length: int = 0,
                              workspace: Optional[torch.Tensor] = None, out: Optional[torch.Tensor] = None,
                              softmax_scale: float = 0.0) -> torch.Tensor:
    """`decode_attn_batch_fp8` over GQA-shared FP8 caches (`pkv_decode_attn_batch_gqa_fp8`): k_q / v_q float8_e4m3fn
    [B, Hkv, capacity, D], k_scale / v_scale float32 [B, Hkv, capacity]; otherwise as `decode_attn_batch_gqa`."""
    return _decode_batch("pkv_decode_attn_batch_gqa_fp8", "decode_attn_batch_gqa_fp8", q, k_q, v_q, (k_scale, v_scale),
                         length, k_new, v_new, rows, step, max_length, workspace, out, softmax_scale, gqa=True)


# ---- the decode window (include/pkv.h: pkv_decode_attn_window) ----
def decode_attn_window(q: torch.Tensor, k_buf: torch.Tensor, v_buf: torch.Tensor, length: int,
                       k_new: Optional[torch.Tensor], v_new: Optional[torch.Tensor], prompt_rows: torch.Tensor, window: int,
                       rows: Optional[torch.Tensor] = None, step: Optional[torch.Tensor] = None, max_length: int = 0,
                       workspace: Optional[torch.Tensor] = None, out: Optional[torch.Tensor] = None,
                       softmax_scale: float = 0.0, scales=None, gqa: bool = False) -> torch.Tensor:
    """The decode step of `decode_attn_batch` / `_gqa` / `_fp8` / `_gqa_fp8` (picked by `scales` = (k_scale, v_scale) of an
    FP8 cache and `gqa`) with a decode window of `window` = R >= 1 rows (`pkv_decode_attn_window`): (sequence b, cache head c)
    keeps its P = prompt_rows[b*H + c] prompt rows (int32 device tensor [B*H]) and its last R appended rows, the j-th
    appended row at P + j mod R. The logical row count n = `length` (+ `*step`) (+ `rows[b*H + c]`) is that of the
    unwindowed launch; P + min(n - P, R) rows are attended. The launch is sized for `max_length` rows (default: the
    capacity), which must hold P + R, and is graph-replayable. Returns out [B, Hq, D]."""
    if int(window) < 1:
        raise ValueError(f"decode_attn_window: window={window} must be >= 1")
    return _decode_batch("pkv_decode_attn_window", "decode_attn_window", q, k_buf, v_buf, scales, length, k_new, v_new, rows, step, max_length, workspace, out,
                         softmax_scale, gqa=gqa, window=int(window), prompt_rows=prompt_rows)


# ---- the heavy-hitter decode window (include/pkv.h: pkv_decode_attn_heavy) ----
_heavy_scratches: Dict[Tuple[int, int], torch.Tensor] = {}


def _heavy_scratch(device: torch.device, nbytes: int) -> torch.Tensor:
    """The per-step logit and (m, l) scratch of a host-launched heavy step: one growing buffer per (device, stream), like
    `_workspace` (the static loops pass their own, which a captured graph keeps)."""
    key = (device.index if device.index is not None else torch.cuda.current_device(),
           torch.cuda.current_stream(device).cuda_stream)
    t = _heavy_scratches.get(key)
    if t is None or t.numel() < nbytes:
        t = torch.empty(max(nbytes, 1 << 16), dtype=torch.uint8, device=device)
        _heavy_scratches[key] = t
    return t


def decode_heavy_workspace_bytes(num_seqs: int, num_q_heads: int, window: int) -> int:
    """Bytes of the per-step scratch of `decode_attn_heavy` (`pkv_decode_heavy_workspace_bytes`)."""
    return int(_lib.lib().pkv_decode_heavy_workspace_bytes(int(num_seqs), int(num_q_heads), int(window)))


def decode_attn_heavy(q: torch.Tensor, k_buf: torch.Tensor, v_buf: torch.Tensor, length: int, k_new: torch.Tensor,
                      v_new: torch.Tensor, prompt_rows: torch.Tensor, window: int, heavy: int, scores: torch.Tensor,
                      gen: torch.Tensor, victim: torch.Tensor, rows: Optional[torch.Tensor] = None,
                      step: Optional[torch.Tensor] = None, max_length: int = 0, workspace: Optional[torch.Tensor] = None,
                      scratch: Optional[torch.Tensor] = None, out: Optional[torch.Tensor] = None, softmax_scale: float = 0.0,
                      scales=None, gqa: bool = False) -> torch.Tensor:
    """`decode_attn_window` whose full window replaces the generated row with the least accumulated attention instead of
    the oldest, keeping the R - H most recent rows (`pkv_decode_attn_heavy`, include/pkv.h). `heavy` = H in [0, R - 1];
    `scores` fp32, `gen` int32 (each [B, H_cache, R]) and `victim` int32 [B*H_cache] are the layer's state, updated in
    place; `scratch` (uint8, `decode_heavy_workspace_bytes(B, Hq, R)` bytes; default: a buffer per stream) holds the
    per-step logits, shared by every layer. Graph-replayable. Returns out [B, Hq, D]."""
    if int(window) < 1 or not 0 <= int(heavy) < int(window):
        raise ValueError(f"decode_attn_heavy: window={window}, heavy={heavy}: expected window >= 1 and 0 <= heavy < window")
    if k_new is None or v_new is None:
        raise ValueError("decode_attn_heavy: the step appends a row: k_new and v_new are required")
    return _decode_batch("pkv_decode_attn_heavy", "decode_attn_heavy", q, k_buf, v_buf, scales, length, k_new, v_new, rows, step,
                         max_length, workspace, out, softmax_scale, gqa=gqa, window=int(window), prompt_rows=prompt_rows,
                         heavy=(int(heavy), scores, gen, victim, scratch))


# ---- continuous batching: admission into one slot of a batched cache (include/pkv.h: pkv_cache_install) ----
def cache_install(layers, slot: int, step: torch.Tensor) -> None:
    """Copy one prompt's compacted cache into slot `slot` of batched caches, every layer in one launch per 32 layers
    (`pkv_cache_install`), and set the slot's decode row counts to `rows - *step` on the device. `layers`: per layer
    (src_k, src_v, src_scales, rows, rows_dev, dst_k, dst_v, dst_scales, dst_rows) with src_k / src_v the prompt's
    contiguous [1, H, capacity, D] buffers (None when rows == 0: parking), dst_k / dst_v the batched [B, H, capacity', D]
    buffers of the same dtype (bf16 / fp16, or float8_e4m3fn with (k_scale, v_scale) float32 scales of shape [.., capacity]
    as src_scales / dst_scales), `rows` the rows per head, `rows_dev` an optional int32 [H] device count per head (at most
    `rows`) and dst_rows the int32 [B*H] row counts the decode kernels read. `step`: the int32 [1] device step counter."""
    layers = list(layers)
    if not layers:
        return
    k0 = layers[0][5]
    B, H, _, D = k0.shape
    fp8 = k0.dtype == FP8_DTYPE
    if not fp8 and k0.dtype not in (torch.bfloat16, torch.float16):
        raise ValueError(f"cache_install: unsupported cache dtype {k0.dtype}")
    if step.dtype != torch.int32 or step.numel() != 1:
        raise ValueError("cache_install: step must be an int32 device tensor with one element")
    _require_cuda(step)
    n = len(layers)
    src, dst = (C.c_void_p * (2 * n))(), (C.c_void_p * (2 * n))()
    sscl, dscl = (C.c_void_p * (2 * n))(), (C.c_void_p * (2 * n))()
    scap, dcap, rows_t = (C.c_int64 * n)(), (C.c_int64 * n)(), (C.c_int64 * n)()
    rdev, drows = (C.c_void_p * n)(), (C.c_void_p * n)()
    for i, (sk, sv, ss, rows, rows_dev, dk, dv, ds, dr) in enumerate(layers):
        what = f"cache_install: layer {i}"
        _require_cuda(sk, sv, rows_dev, dk, dv, dr, *(ss or ()), *(ds or ()))
        if dk.dim() != 4 or dk.shape != dv.shape or not dk.is_contiguous() or not dv.is_contiguous():
            raise ValueError(f"{what}: the batched buffers must be contiguous [B, H, capacity, D] tensors of equal shape")
        if dk.dtype != k0.dtype or dv.dtype != k0.dtype or (dk.shape[0], dk.shape[1], dk.shape[3]) != (B, H, D) or dk.device != k0.device:
            raise ValueError(f"{what}: batch, heads, head_dim, dtype and device must match layer 0")
        if fp8:
            if ds is None:
                raise ValueError(f"{what}: an FP8 cache needs its scales")
            _check_fp8_buffers(dk, dv, ds[0], ds[1], what)
        elif ds is not None or ss is not None:
            raise ValueError(f"{what}: scales go with FP8 caches only")
        if dr.dtype != torch.int32 or dr.numel() != B * H or not dr.is_contiguous():
            raise ValueError(f"{what}: dst_rows must be a contiguous int32 device tensor of B*H = {B * H} elements")
        rows = int(rows)
        if rows > 0:
            if sk is None or sv is None or sk.shape != sv.shape or sk.dim() != 4 or sk.shape[0] != 1 \
                    or not sk.is_contiguous() or not sv.is_contiguous():
                raise ValueError(f"{what}: the source must be contiguous [1, H, capacity, D] buffers of equal shape")
            if sk.dtype != dk.dtype or sv.dtype != dk.dtype:
                raise ValueError(f"{what}: source dtype {sk.dtype} differs from the batched cache's {dk.dtype}")
            if sk.shape[1] != H or sk.shape[3] != D:
                raise ValueError(f"{what}: source heads / head_dim {tuple(sk.shape[1::2])} differ from the batched cache's ({H}, {D})")
            if fp8:
                if ss is None:
                    raise ValueError(f"{what}: an FP8 source needs its scales")
                _check_fp8_buffers(sk, sv, ss[0], ss[1], what)
            if rows_dev is not None and (rows_dev.dtype != torch.int32 or rows_dev.numel() != H or not rows_dev.is_contiguous()):
                raise ValueError(f"{what}: rows_dev must be a contiguous int32 device tensor of H = {H} elements")
            src[2 * i], src[2 * i + 1] = sk.data_ptr(), sv.data_ptr()
            scap[i] = sk.shape[2]
            if fp8:
                sscl[2 * i], sscl[2 * i + 1] = ss[0].data_ptr(), ss[1].data_ptr()
            rdev[i] = rows_dev.data_ptr() if rows_dev is not None else None
        dst[2 * i], dst[2 * i + 1] = dk.data_ptr(), dv.data_ptr()
        if fp8:
            dscl[2 * i], dscl[2 * i + 1] = ds[0].data_ptr(), ds[1].data_ptr()
        dcap[i], rows_t[i], drows[i] = dk.shape[2], rows, dr.data_ptr()
    dev = k0.device.index if k0.device.index is not None else torch.cuda.current_device()
    _lib.check(_lib.lib().pkv_cache_install(1 if fp8 else 2, B, H, D, dev, n, int(slot), src, dst, sscl if fp8 else None,
                                            dscl if fp8 else None, scap, dcap, rows_t,
                                            rdev if any(r is not None for r in rdev) else None, drows, step.data_ptr(),
                                            torch.cuda.current_stream(k0.device).cuda_stream))


def decode_workspace_bytes(num_q_heads: int, head_dim: int) -> int:
    """Upper bound of the decode workspace for any cache length (`pkv_decode_workspace_bytes`)."""
    d = DecodeDesc()
    d.struct_bytes = C.sizeof(DecodeDesc)
    d.num_q_heads, d.num_kv_heads, d.head_dim = num_q_heads, num_q_heads, head_dim
    return int(_lib.lib().pkv_decode_workspace_bytes(C.byref(d)))


def cache_append(k_cache: torch.Tensor, v_cache: torch.Tensor, k_new: torch.Tensor, v_new: torch.Tensor, length: int) -> None:
    """Write k_new/v_new [Hkv, D] as row length-1 of every query head's cache (repeat_kv semantics)."""
    _require_cuda(k_cache, v_cache, k_new, v_new)
    if k_cache.dim() == 4:
        k_cache, v_cache = k_cache[0], v_cache[0]
    Hq, cap, D = k_cache.shape
    k_new, v_new = k_new.reshape(-1, D).contiguous(), v_new.reshape(-1, D).contiguous()
    d = DecodeDesc()
    d.struct_bytes = C.sizeof(DecodeDesc)
    d.dtype, d.num_q_heads, d.num_kv_heads, d.head_dim = _dtype_code(k_cache), Hq, k_new.shape[0], D
    d.device = k_cache.device.index if k_cache.device.index is not None else torch.cuda.current_device()
    d.length = int(length)
    d.k_new, d.v_new = k_new.data_ptr(), v_new.data_ptr()
    d.k_cache, d.v_cache, d.cache_stride_h = k_cache.data_ptr(), v_cache.data_ptr(), k_cache.stride(0)
    _lib.check(_lib.lib().pkv_cache_append(C.byref(d), torch.cuda.current_stream(k_cache.device).cuda_stream))


# ---- sampled decoding (include/pkv.h: pkv_sample_tokens, DESIGN.md §4.6) ----
def sample_tokens(logits: torch.Tensor, params, out: torch.Tensor, col: int, advance: bool = True) -> None:
    """One token per row of `logits` [B, V] (bf16 / fp16, rows may be strided) into out[:, col] (int64 [B, *]), in ONE
    launch: temperature, top-k, top-p and a Gumbel-max draw keyed by Philox4x32-10 (seed, token index), each row with its
    own parameters. `params` holds the per-row DEVICE tensors `temperature` (float32 [B]), `top_k` (int32), `top_p`
    (float32), `seed` (int64, the 64 seed bits) and `index` (int64, the row's token index t; incremented in place when
    `advance`) - generate.SamplingState. Nothing is read back: the launch replays in a CUDA graph."""
    d = _sample_desc("sample_tokens", logits, params, out, col, advance)
    _lib.check(_lib.lib().pkv_sample_tokens(C.byref(d), torch.cuda.current_stream(logits.device).cuda_stream))


def _check_row_params(fn, logits, params, fields):
    B = logits.shape[0]
    for name, dt in fields:
        t = getattr(params, name)
        if t.dtype != dt or t.numel() != B or not t.is_contiguous() or t.device != logits.device:
            raise ValueError(f"{fn}: params.{name} must be a contiguous {dt} tensor of B = {B} elements on {logits.device}")


def _sample_desc(fn, logits, params, out, col, advance):
    _require_cuda(logits, out, params.temperature, params.top_k, params.top_p, params.seed, params.index)
    if logits.dim() != 2 or logits.stride(1) != 1:
        raise ValueError(f"{fn}: logits must be [B, V] with contiguous rows, got {tuple(logits.shape)}")
    B, V = logits.shape
    if out.dim() != 2 or out.dtype != torch.long or out.shape[0] != B or out.stride(1) != 1:
        raise ValueError(f"{fn}: out must be an int64 [B={B}, n] tensor with contiguous rows")
    _check_row_params(fn, logits, params, (("temperature", torch.float32), ("top_k", torch.int32), ("top_p", torch.float32),
                                           ("seed", torch.int64), ("index", torch.int64)))
    d = _lib.SampleDesc()
    d.struct_bytes = C.sizeof(_lib.SampleDesc)
    d.dtype = _dtype_code(logits)
    d.device = logits.device.index if logits.device.index is not None else torch.cuda.current_device()
    d.batch, d.vocab = B, V
    d.logits, d.logits_stride = logits.data_ptr(), logits.stride(0) if B > 1 else V
    d.temperature, d.top_k, d.top_p = params.temperature.data_ptr(), params.top_k.data_ptr(), params.top_p.data_ptr()
    d.seed, d.token_index = params.seed.data_ptr(), params.index.data_ptr()
    d.tokens, d.tokens_stride, d.column = out.data_ptr(), out.stride(0) if B > 1 else out.shape[1], int(col)
    d.flags = _lib.SAMPLE_ADVANCE if advance else 0
    return d


def sample_tokens_penalized(logits: torch.Tensor, params, out: torch.Tensor, col: int, advance: bool = True) -> None:
    """`sample_tokens` with repetition, presence and frequency penalties and min-p (include/pkv.h:
    pkv_sample_tokens_penalized, DESIGN.md §4.10), in ONE launch. `params` also holds the per-row DEVICE tensors
    `repetition_penalty`, `presence_penalty`, `frequency_penalty`, `min_p` (float32 [B]), `prompt_mask` (uint8 [B, S],
    nonzero for the row's prompt tokens) and `counts` (int32 [B, S], the row's generated-token counts; with `advance` the
    drawn token's count is incremented in place), S >= V with contiguous rows. A row whose new parameters are at their
    defaults (1, 0, 0, 0) gets `sample_tokens`' token."""
    fn = "sample_tokens_penalized"
    d = _sample_desc(fn, logits, params, out, col, advance)
    B, V = logits.shape
    _check_row_params(fn, logits, params, [(n, torch.float32) for n in ("repetition_penalty", "presence_penalty",
                                                                        "frequency_penalty", "min_p")])
    mask, counts = params.prompt_mask, params.counts
    _require_cuda(mask, counts)
    if (mask.dim() != 2 or mask.dtype != torch.uint8 or counts.dtype != torch.int32 or mask.shape != counts.shape
            or mask.shape[0] != B or mask.shape[1] < V or not mask.is_contiguous() or not counts.is_contiguous()
            or mask.device != logits.device or counts.device != logits.device):
        raise ValueError(f"{fn}: params.prompt_mask / params.counts must be contiguous uint8 / int32 [B={B}, S >= V={V}] "
                         f"tensors on {logits.device}")
    p = _lib.SamplePenalty()
    p.struct_bytes = C.sizeof(_lib.SamplePenalty)
    p.repetition_penalty, p.presence_penalty = params.repetition_penalty.data_ptr(), params.presence_penalty.data_ptr()
    p.frequency_penalty, p.min_p = params.frequency_penalty.data_ptr(), params.min_p.data_ptr()
    p.prompt_mask, p.counts, p.stride = mask.data_ptr(), counts.data_ptr(), mask.shape[1]
    _lib.check(_lib.lib().pkv_sample_tokens_penalized(C.byref(d), C.byref(p),
                                                      torch.cuda.current_stream(logits.device).cuda_stream))


def _penalty_struct(fn, logits, params):
    B, V = logits.shape
    _check_row_params(fn, logits, params, [(n, torch.float32) for n in ("repetition_penalty", "presence_penalty",
                                                                        "frequency_penalty", "min_p")])
    mask, counts = params.prompt_mask, params.counts
    _require_cuda(mask, counts)
    if (mask.dim() != 2 or mask.dtype != torch.uint8 or counts.dtype != torch.int32 or mask.shape != counts.shape
            or mask.shape[0] != B or mask.shape[1] < V or not mask.is_contiguous() or not counts.is_contiguous()
            or mask.device != logits.device or counts.device != logits.device):
        raise ValueError(f"{fn}: params.prompt_mask / params.counts must be contiguous uint8 / int32 [B={B}, S >= V={V}] "
                         f"tensors on {logits.device}")
    p = _lib.SamplePenalty()
    p.struct_bytes = C.sizeof(_lib.SamplePenalty)
    p.repetition_penalty, p.presence_penalty = params.repetition_penalty.data_ptr(), params.presence_penalty.data_ptr()
    p.frequency_penalty, p.min_p = params.frequency_penalty.data_ptr(), params.min_p.data_ptr()
    p.prompt_mask, p.counts, p.stride = mask.data_ptr(), counts.data_ptr(), mask.shape[1]
    return p


def _check_rule_tensor(fn, name, t, dtype, rows, min_cols=None):
    ok = t.dtype == dtype and t.is_cuda and t.is_contiguous() and t.shape[0] == rows
    if min_cols is not None:
        ok = ok and t.dim() == 2 and t.shape[1] >= min_cols
    if not ok:
        raise ValueError(f"{fn}: {name} must be a contiguous CUDA {dtype} tensor of {rows} rows"
                         + ("" if min_cols is None else f" and >= {min_cols} columns") + f", got {t.dtype} {tuple(t.shape)}")


def sample_tokens_constrained(logits: torch.Tensor, params, out: torch.Tensor, col: int, advance: bool = True) -> None:
    """`sample_tokens_penalized` with the rule terms `token_rules` wrote (include/pkv.h: pkv_sample_tokens_constrained,
    DESIGN.md §4.11), in ONE launch: per row, x = f32(logit) + the sequence-bias sum, the penalties, then the bans (set to
    -inf; bad words add -inf), then the draw. `params` (generate.SamplingState) also holds `rule_flags` (int32 [B]),
    `bias` (float32 [B, >= V]) and `ban` (int32 [B, >= 2 * ceil(V / 32)]). A row with no rule flag reads none of them and
    gets `sample_tokens_penalized`' token."""
    fn = "sample_tokens_constrained"
    d = _sample_desc(fn, logits, params, out, col, advance)
    p = _penalty_struct(fn, logits, params)
    B, V = logits.shape
    _check_rule_tensor(fn, "params.rule_flags", params.rule_flags, torch.int32, B)
    _check_rule_tensor(fn, "params.bias", params.bias, torch.float32, B, V)
    _check_rule_tensor(fn, "params.ban", params.ban, torch.int32, B, 2 * ((V + 31) // 32))
    r = _lib.SampleRules()
    r.struct_bytes = C.sizeof(_lib.SampleRules)
    r.flags = params.rule_flags.data_ptr()
    r.bias, r.bias_stride = params.bias.data_ptr(), params.bias.shape[1]
    r.ban, r.ban_stride = params.ban.data_ptr(), params.ban.shape[1]
    _lib.check(_lib.lib().pkv_sample_tokens_constrained(C.byref(d), C.byref(p), C.byref(r),
                                                        torch.cuda.current_stream(logits.device).cuda_stream))


def token_rules(params, vocab: int, append: Optional[torch.Tensor] = None, col: int = 0) -> None:
    """One `pkv_token_rules` launch (include/pkv.h, DESIGN.md §4.11) over the per-row DEVICE state of
    generate.SamplingState: with `append` (int64 [B, n]), first append append[:, col] to each row's history; then write
    each row's sequence-bias sums (`params.bias`), ban bitmaps (`params.ban`) and stop flag (`params.stop`, bool [B, 1])
    from its history (`history` int32 [B, cap], `history_len` / `prompt_len` int32 [B]) and rules (`rule_flags`, `ngram`,
    `min_new` int32 [B]; `n_seq` int32 [B], `seq_off` / `seq_kind` int32 and `seq_bias` float32 [B, S], `seq_tokens` int32
    [B, T]; `eos` int32 [E], `n_eos`). Nothing is read back: the launch replays in a CUDA graph."""
    fn = "token_rules"
    B = params.history.shape[0]
    V = int(vocab)
    for name, dt, cols in (("history", torch.int32, 1), ("history_len", torch.int32, None), ("prompt_len", torch.int32, None),
                           ("rule_flags", torch.int32, None), ("ngram", torch.int32, None), ("min_new", torch.int32, None),
                           ("n_seq", torch.int32, None), ("seq_off", torch.int32, 2), ("seq_kind", torch.int32, 2),
                           ("seq_bias", torch.float32, 2), ("seq_tokens", torch.int32, 1), ("bias", torch.float32, V),
                           ("ban", torch.int32, 2 * ((V + 31) // 32)), ("stop", torch.bool, None)):
        _check_rule_tensor(fn, f"params.{name}", getattr(params, name), dt, B, cols)
    if params.seq_off.shape != params.seq_kind.shape or params.seq_off.shape != params.seq_bias.shape:
        raise ValueError(f"{fn}: params.seq_off, seq_kind and seq_bias must have one shape")
    d = _lib.TokenRulesDesc()
    d.struct_bytes = C.sizeof(_lib.TokenRulesDesc)
    d.device = params.history.device.index if params.history.device.index is not None else torch.cuda.current_device()
    d.batch, d.vocab = B, V
    d.history, d.history_stride = params.history.data_ptr(), params.history.shape[1]
    d.history_len, d.prompt_len = params.history_len.data_ptr(), params.prompt_len.data_ptr()
    d.flags, d.ngram, d.min_new_tokens, d.n_seq = (params.rule_flags.data_ptr(), params.ngram.data_ptr(),
                                                   params.min_new.data_ptr(), params.n_seq.data_ptr())
    d.seq_off, d.seq_kind, d.seq_bias = params.seq_off.data_ptr(), params.seq_kind.data_ptr(), params.seq_bias.data_ptr()
    d.seq_stride = params.seq_off.shape[1]
    d.seq_tokens, d.tokens_stride = params.seq_tokens.data_ptr(), params.seq_tokens.shape[1]
    d.eos, d.n_eos = params.eos.data_ptr(), int(params.n_eos)
    if append is not None:
        if append.dtype != torch.long or append.dim() != 2 or append.shape[0] != B or append.stride(1) != 1 or not append.is_cuda:
            raise ValueError(f"{fn}: append must be an int64 CUDA [B={B}, n] tensor with contiguous rows")
        if not 0 <= int(col) < append.shape[1]:
            raise ValueError(f"{fn}: col={col} outside [0, {append.shape[1]}) of append")
        d.append, d.append_stride, d.append_column = append.data_ptr(), append.stride(0) if B > 1 else append.shape[1], int(col)
    d.bias, d.bias_stride = params.bias.data_ptr(), params.bias.shape[1]
    d.ban, d.ban_stride = params.ban.data_ptr(), params.ban.shape[1]
    d.stop = params.stop.data_ptr()
    _lib.check(_lib.lib().pkv_token_rules(C.byref(d), torch.cuda.current_stream(params.history.device).cuda_stream))


# ---- token log-probabilities (include/pkv.h: pkv_token_logprobs, DESIGN.md §4.8) ----
def token_logprobs(logits: torch.Tensor, tokens: torch.Tensor, out_lp: torch.Tensor, out_ids: torch.Tensor,
                   out_top: torch.Tensor, col: int = 0, tokens_col: int = 0, cursor: Optional[torch.Tensor] = None) -> None:
    """log_softmax(f32(logits)) of each row of `logits` [B, V] (bf16 / fp16, rows may be strided), the model's raw
    distribution, in ONE launch: out_lp[b, c] (float32 [B, n]) at the token tokens[b, tokens_col] (int64 [B, *]), and the
    row's top N = out_ids.shape[2] tokens (logit descending, index ascending) with their log-probabilities into
    out_ids[b, c] (int64 [B, n, N]) and out_top[b, c] (float32 [B, n, N]). c = col, plus the DEVICE int64 `cursor` [1]
    when given (not bounds-checked: the caller keeps it inside n). Nothing is read back: the launch replays in a CUDA graph."""
    _require_cuda(logits, tokens, out_lp, out_ids, out_top, *(() if cursor is None else (cursor,)))
    if logits.dim() != 2 or logits.stride(1) != 1:
        raise ValueError(f"token_logprobs: logits must be [B, V] with contiguous rows, got {tuple(logits.shape)}")
    B, V = logits.shape
    if tokens.dim() != 2 or tokens.dtype != torch.long or tokens.shape[0] != B or tokens.stride(1) != 1:
        raise ValueError(f"token_logprobs: tokens must be an int64 [B={B}, n] tensor with contiguous rows")
    if out_lp.dim() != 2 or out_lp.dtype != torch.float32 or out_lp.shape[0] != B or not out_lp.is_contiguous():
        raise ValueError(f"token_logprobs: out_lp must be a contiguous float32 [B={B}, n] tensor")
    n = out_lp.shape[1]
    if (out_ids.dim() != 3 or out_ids.dtype != torch.long or tuple(out_ids.shape[:2]) != (B, n) or not out_ids.is_contiguous()
            or out_top.dtype != torch.float32 or out_top.shape != out_ids.shape or not out_top.is_contiguous()):
        raise ValueError(f"token_logprobs: out_ids / out_top must be contiguous int64 / float32 [B={B}, n={n}, N] tensors")
    if cursor is not None and (cursor.dtype != torch.long or cursor.numel() != 1):
        raise ValueError("token_logprobs: cursor must be a one-element int64 tensor")
    N = out_ids.shape[2]
    d = _lib.LogprobsDesc()
    d.struct_bytes = C.sizeof(_lib.LogprobsDesc)
    d.dtype = _dtype_code(logits)
    d.device = logits.device.index if logits.device.index is not None else torch.cuda.current_device()
    d.batch, d.vocab, d.top_n = B, V, N
    d.logits, d.logits_stride = logits.data_ptr(), logits.stride(0) if B > 1 else V
    d.tokens, d.tokens_stride, d.tokens_column = tokens.data_ptr(), tokens.stride(0) if B > 1 else tokens.shape[1], int(tokens_col)
    d.cursor = None if cursor is None else cursor.data_ptr()
    d.column = int(col)
    d.logprob, d.logprob_stride = out_lp.data_ptr(), n
    if N > 0:
        d.top_ids, d.top_logprobs, d.top_stride = out_ids.data_ptr(), out_top.data_ptr(), n * N
    _lib.check(_lib.lib().pkv_token_logprobs(C.byref(d), torch.cuda.current_stream(logits.device).cuda_stream))


# ---- beam search (include/pkv.h: pkv_beam_candidates, pkv_beam_step, pkv_cache_reorder; DESIGN.md §4.12) ----
def beam_candidates(logits: torch.Tensor, m: torch.Tensor, log_z: torch.Tensor, cand_lp: torch.Tensor,
                    cand_id: torch.Tensor) -> None:
    """Per row of `logits` [R, V] (bf16 / fp16, contiguous rows): m [R], log_z [R] (float32) and the row's top K =
    cand_lp.shape[1] tokens (logit descending, index ascending) into cand_id (int32 [R, K]) with their log-probabilities
    into cand_lp (float32 [R, K]). One launch; it replays in a CUDA graph."""
    _require_cuda(logits, m, log_z, cand_lp, cand_id)
    if logits.dim() != 2 or logits.stride(1) != 1:
        raise ValueError(f"beam_candidates: logits must be [R, V] with contiguous rows, got {tuple(logits.shape)}")
    R, V = logits.shape
    K = cand_lp.shape[1] if cand_lp.dim() == 2 else -1
    if (cand_lp.shape != (R, K) or cand_id.shape != (R, K) or cand_lp.dtype != torch.float32 or cand_id.dtype != torch.int32
            or not cand_lp.is_contiguous() or not cand_id.is_contiguous()):
        raise ValueError(f"beam_candidates: cand_lp / cand_id must be contiguous float32 / int32 [R={R}, K] tensors")
    if m.shape != (R,) or log_z.shape != (R,) or m.dtype != torch.float32 or log_z.dtype != torch.float32:
        raise ValueError(f"beam_candidates: m / log_z must be float32 [R={R}] tensors")
    dev = logits.device.index if logits.device.index is not None else torch.cuda.current_device()
    _lib.check(_lib.lib().pkv_beam_candidates(_dtype_code(logits), dev, R, V, logits.data_ptr(),
                                              logits.stride(0) if R > 1 else V, K, m.data_ptr(), log_z.data_ptr(),
                                              cand_lp.data_ptr(), cand_id.data_ptr(),
                                              torch.cuda.current_stream(logits.device).cuda_stream))


_BEAM_FIELDS = ("running", "pool_score", "pool_step", "pool_parent", "pool_token", "pool_done", "heuristic", "done",
                "bp_token", "bp_parent", "cp", "next_token", "parent", "diverge")


def beam_step(st, rows_per_prompt: int, step: torch.Tensor, step_offset: int) -> None:
    """One `pkv_beam_step` launch over the state `st` (generate.BeamState): its candidates (`rows_per_prompt` rows per
    prompt: k, or 1 for the prefill's row), iteration *step + step_offset read on the device."""
    _require_cuda(st.cand_lp, step, *(getattr(st, f) for f in _BEAM_FIELDS))
    if step.dtype != torch.int32 or step.numel() != 1:
        raise ValueError("beam_step: step must be a one-element int32 tensor")
    d = _lib.BeamStepDesc()
    d.struct_bytes = C.sizeof(_lib.BeamStepDesc)
    d.device = st.running.device.index if st.running.device.index is not None else torch.cuda.current_device()
    d.num_prompts, d.num_beams, d.top_k, d.cand_rows_per_prompt = st.P, st.k, st.K, int(rows_per_prompt)
    d.n_eos, d.early_stopping, d.max_steps, d.step_offset = st.n_eos, st.early_stopping, st.max_steps, int(step_offset)
    d.step, d.cand_lp, d.cand_id = step.data_ptr(), st.cand_lp.data_ptr(), st.cand_id.data_ptr()
    d.eos, d.scale = st.eos_dev.data_ptr(), st.scale.data_ptr()
    for f in _BEAM_FIELDS:
        setattr(d, f, getattr(st, f).data_ptr())
    _lib.check(_lib.lib().pkv_beam_step(C.byref(d), torch.cuda.current_stream(st.running.device).cuda_stream))


def cache_reorder(items, P: int, k: int, parent: torch.Tensor, diverge: torch.Tensor, step: torch.Tensor,
                  step_offset: int) -> None:
    """Every layer's beam reorder in one launch per 32 layers (`pkv_cache_reorder`). items: per layer (k_buf, v_buf,
    k_scale, v_scale, base, window, heavy_state) as `cache.PkvBatchCacheLayer._reorder_item` gives them: rows [P*k, H,
    cap, D] (16-bit, or E4M3 with fp32 scales [P*k, H, cap]), base int32 [P*k*H] the row of generated slot 0, window R
    or None, heavy_state (scores, gen, victim) or None."""
    if not items:
        raise ValueError("cache_reorder: no layers")
    k0 = items[0][0]
    B, H, _, D = k0.shape
    fp8 = k0.dtype == torch.float8_e4m3fn
    if B != P * k:
        raise ValueError(f"cache_reorder: {B} sequences, expected {P} prompts x {k} beams")
    window, heavy = items[0][5], items[0][6] is not None
    _require_cuda(parent, diverge, step)
    if parent.dtype != torch.int32 or diverge.dtype != torch.int32 or parent.numel() != B or diverge.numel() != B:
        raise ValueError(f"cache_reorder: parent / diverge must be int32 [{B}]")
    n = len(items)
    planes, caps, base, hs, hg, vic = (C.c_void_p * (4 * n))(), (C.c_int64 * n)(), (C.c_void_p * n)(), \
        (C.c_void_p * n)(), (C.c_void_p * n)(), (C.c_void_p * n)()
    for i, (kb, vb, ks, vs, rows, win, hstate) in enumerate(items):
        if kb.shape[:2] != (B, H) or kb.shape[3] != D or vb.shape != kb.shape or kb.dtype != k0.dtype or not kb.is_contiguous() \
                or not vb.is_contiguous() or win != window or (hstate is not None) != heavy:
            raise ValueError(f"cache_reorder: layer {i}: every layer must hold the same form and shape")
        if (ks is not None) != fp8 or rows.dtype != torch.int32 or rows.numel() != B * H:
            raise ValueError(f"cache_reorder: layer {i}: scales go with E4M3 rows; base must be int32 [{B * H}]")
        planes[4 * i], planes[4 * i + 1] = kb.data_ptr(), vb.data_ptr()
        if fp8:
            planes[4 * i + 2], planes[4 * i + 3] = ks.data_ptr(), vs.data_ptr()
        caps[i], base[i] = kb.shape[2], rows.data_ptr()
        if heavy:
            hs[i], hg[i], vic[i] = (t.data_ptr() for t in hstate)
    dev = k0.device.index if k0.device.index is not None else torch.cuda.current_device()
    _lib.check(_lib.lib().pkv_cache_reorder(int(P), int(k), H, D * (1 if fp8 else 2), dev, n, int(window or 0), int(heavy),
                                            planes, caps, base, hs if heavy else None, hg if heavy else None,
                                            vic if heavy else None, parent.data_ptr(), diverge.data_ptr(), step.data_ptr(),
                                            int(step_offset), torch.cuda.current_stream(k0.device).cuda_stream))


# ---- prompt-lookup speculative decoding (include/pkv.h: pkv_decode_attn_multi, pkv_prompt_lookup, pkv_spec_step) ----
def _token_rows(t: torch.Tensor) -> torch.Tensor:
    """t [B, Q, H, D] as the kernel reads it: rows contiguous, token s*Q + j at one stride, strides multiples of 8
    elements and a 16-byte aligned base (HF's [b, q, H, D] projections are, as they are); otherwise a contiguous copy."""
    ok = t.stride(3) == 1 and t.stride(0) == t.shape[1] * t.stride(1) and t.stride(1) % 8 == 0 and t.stride(2) % 8 == 0 \
        and t.data_ptr() % 16 == 0
    return t if ok else t.contiguous()


def decode_attn_multi(q: torch.Tensor, k_buf: torch.Tensor, v_buf: torch.Tensor, k_new: torch.Tensor, v_new: torch.Tensor,
                      rows: Optional[torch.Tensor] = None, length: int = 0, step: Optional[torch.Tensor] = None,
                      max_length: int = 0, scales=None, gqa: bool = False, workspace: Optional[torch.Tensor] = None,
                      out: Optional[torch.Tensor] = None, softmax_scale: float = 0.0) -> torch.Tensor:
    """The verify attention of speculative decoding (`pkv_decode_attn_multi`): q [B, Q, Hq, D] and k_new / v_new
    [B, Q, Hkv, D] (HF's projections, read in place), buffers [B, H, capacity, D] (H = Hq, or Hkv with `gqa`; float8_e4m3fn
    with `scales` = (k_scale, v_scale) [B, H, capacity]). Sequence b, cache head c holds n0 = `length` (+ `*step`) (+
    `rows[b*H + c]`) rows: the Q new rows are stored at n0 .. n0 + Q - 1 and query j attends rows [0, n0 + j + 1). The
    launch is sized for `max_length` rows (default: the capacity) and replays in a CUDA graph. Returns out [B, Q, Hq, D]."""
    what = "decode_attn_multi"
    _require_cuda(q, k_buf, v_buf, k_new, v_new, rows, step, workspace, out, *(scales or ()))
    if scales is not None:
        _check_fp8_buffers(k_buf, v_buf, scales[0], scales[1], what)
    elif k_buf.dim() != 4 or k_buf.shape != v_buf.shape or k_buf.stride() != v_buf.stride() or k_buf.stride(3) != 1 \
            or k_buf.stride(2) != k_buf.shape[3]:
        raise ValueError(f"{what}: k_buf / v_buf must be [B, H, capacity, D] tensors of equal shape and strides, rows contiguous")
    B, H, cap, D = k_buf.shape
    if q.dim() != 4 or q.shape[0] != B or q.shape[3] != D or not 1 <= q.shape[1] <= _lib.MAX_SPEC_QUERIES:
        raise ValueError(f"{what}: q must be [B={B}, Q <= {_lib.MAX_SPEC_QUERIES}, Hq, D={D}], got {tuple(q.shape)}")
    Q, Hq = q.shape[1], q.shape[2]
    Hkv = k_new.shape[2] if k_new.dim() == 4 else -1
    if k_new.shape != (B, Q, Hkv, D) or v_new.shape != k_new.shape or Hkv < 1 or Hq % Hkv \
            or k_new.dtype != q.dtype or v_new.dtype != q.dtype or (H != (Hkv if gqa else Hq)):
        raise ValueError(f"{what}: k_new / v_new must be [B, Q, Hkv, D] of q's dtype, and the cache hold "
                         f"{'Hkv' if gqa else 'Hq'} heads; got {tuple(k_new.shape)}, {tuple(v_new.shape)}, cache heads {H}")
    q, k_new, v_new = _token_rows(q), _token_rows(k_new), _token_rows(v_new)
    if k_new.stride() != v_new.stride():
        k_new, v_new = k_new.contiguous(), v_new.contiguous()
    if out is None:
        out = torch.empty(B, Q, Hq, D, dtype=q.dtype, device=q.device)
    elif out.shape != (B, Q, Hq, D) or not out.is_contiguous() or out.dtype != q.dtype:
        raise ValueError(f"{what}: out must be a contiguous [B, Q, Hq, D] tensor of q's dtype")
    max_length = int(max_length) or cap
    if not Q <= max_length <= cap or int(length) < 0:
        raise ValueError(f"{what}: cache capacity {cap} exceeded or bad row counts (length {length}, max_length {max_length})")
    if step is not None and (step.dtype != torch.int32 or step.numel() != 1):
        raise ValueError("step must be an int32 device tensor with one element")
    if rows is not None:
        if rows.dtype != torch.int32 or rows.numel() != B * H or not rows.is_contiguous():
            raise ValueError(f"{what}: rows must be a contiguous int32 device tensor of B*H = {B * H} elements")
        if not torch.cuda.is_current_stream_capturing():
            # (one device read; a captured launch relies on the caller, and the kernel writes no row of a count out of range)
            most = int(rows.max()) + int(length) + (int(step) if step is not None else 0) + Q
            if most > max_length:
                raise ValueError(f"{what}: cache capacity exceeded: {most} rows for max_length {max_length} (capacity {cap})")
    d = DecodeDesc()
    d.struct_bytes = C.sizeof(DecodeDesc)
    d.dtype, d.num_q_heads, d.num_kv_heads, d.head_dim = _dtype_code(q), Hq, Hkv, D
    d.device = q.device.index if q.device.index is not None else torch.cuda.current_device()
    d.length = int(length)
    d.q, d.k_new, d.v_new, d.out = q.data_ptr(), k_new.data_ptr(), v_new.data_ptr(), out.data_ptr()
    d.k_cache, d.v_cache, d.cache_stride_h = k_buf.data_ptr(), v_buf.data_ptr(), k_buf.stride(1)
    if workspace is None:
        workspace = _workspace(q.device, decode_workspace_bytes(B * Hq * Q, D))
    d.workspace, d.workspace_bytes = workspace.data_ptr(), workspace.numel() * workspace.element_size()
    d.softmax_scale = float(softmax_scale)
    m = DecodeMulti()
    m.struct_bytes = C.sizeof(DecodeMulti)
    m.num_seqs, m.num_queries, m.gqa_shared, m.cache_stride_b = B, Q, int(gqa), k_buf.stride(0)
    m.rows = rows.data_ptr() if rows is not None else None
    m.step_dev = step.data_ptr() if step is not None else None
    m.max_length = max_length
    if scales is not None:
        m.k_scale, m.v_scale = scales[0].data_ptr(), scales[1].data_ptr()
        m.scale_stride_h, m.scale_stride_b = scales[0].stride(1), scales[0].stride(0)
    m.q_stride_t, m.q_stride_h = q.stride(1), q.stride(2)
    m.kv_stride_t, m.kv_stride_h = k_new.stride(1), k_new.stride(2)
    m.out_stride_t, m.out_stride_h = out.stride(1), out.stride(2)
    _lib.check(_lib.lib().pkv_decode_attn_multi(C.byref(d), C.byref(m), torch.cuda.current_stream(q.device).cuda_stream))
    return out


_SPEC_FIELDS = (("hist", torch.int64, 2), ("hist_len", torch.int32, 1), ("budget", torch.int32, 1), ("done", torch.bool, 1),
                ("out", torch.int64, 2), ("out_len", torch.int32, 1), ("ids", torch.int64, 2), ("pos", torch.int64, 2),
                ("draft_len", torch.int32, 1), ("emitted", torch.int32, 1), ("tokens", torch.int64, 2))


def _spec_desc(fn: str, st, rows=None):
    """The pkv_spec_desc of a `generate.SpecState` (its device tensors, checked) and the row-count tensors of `rows`."""
    B, Q = st.ids.shape
    for name, dt, dim in _SPEC_FIELDS:
        t = getattr(st, name)
        _require_cuda(t)
        if t.dtype != dt or t.dim() != dim or t.shape[0] != B or not t.is_contiguous() or (name in ("pos", "tokens") and t.shape[1] != Q):
            raise ValueError(f"{fn}: {name} must be a contiguous {dt} device tensor of {B} rows" + (f" x {Q}" if dim == 2 else ""))
    d = SpecDesc()
    d.struct_bytes = C.sizeof(SpecDesc)
    d.device = st.ids.device.index if st.ids.device.index is not None else torch.cuda.current_device()
    d.num_seqs, d.num_queries, d.max_ngram, d.n_eos = B, Q, int(st.max_ngram), int(st.eos.numel())
    d.pad_token_id, d.hist_cap, d.out_cap = int(st.pad_token_id), st.hist.shape[1], st.out.shape[1]
    for name, _, _ in _SPEC_FIELDS:
        setattr(d, name, getattr(st, name).data_ptr())
    if st.eos.numel():
        _require_cuda(st.eos)
        if st.eos.dtype != torch.int64 or not st.eos.is_contiguous():
            raise ValueError(f"{fn}: eos must be a contiguous int64 device tensor")
        d.eos = st.eos.data_ptr()
    table = None
    if rows:
        for r in rows:
            _require_cuda(r)
            if r.dtype != torch.int32 or not r.is_contiguous() or r.numel() != rows[0].numel() or r.numel() % B:
                raise ValueError(f"{fn}: every row-count tensor must be a contiguous int32 device tensor of B*H elements")
        table = (C.c_void_p * len(rows))(*[r.data_ptr() for r in rows])
        d.num_layers, d.num_heads, d.rows = len(rows), rows[0].numel() // B, C.cast(table, C.c_void_p)
    return d, table


def prompt_lookup(st) -> None:
    """Rule 1 of include/pkv.h for every sequence of `st` (`pkv_prompt_lookup`): its next verify ids, positions and draft
    length from its history."""
    d, _ = _spec_desc("prompt_lookup", st)
    _lib.check(_lib.lib().pkv_prompt_lookup(C.byref(d), torch.cuda.current_stream(st.ids.device).cuda_stream))


def spec_step(st, rows) -> None:
    """Rule 3 then rule 1 for every sequence of `st` (`pkv_spec_step`) from its verify argmaxes `st.tokens`; `rows`: the
    int32 [B*H] row counts of every layer, advanced by each sequence's emitted tokens (one launch per 32 layers)."""
    d, table = _spec_desc("spec_step", st, list(rows))
    _lib.check(_lib.lib().pkv_spec_step(C.byref(d), torch.cuda.current_stream(st.ids.device).cuda_stream))
    del table
