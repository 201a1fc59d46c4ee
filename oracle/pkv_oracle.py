"""ctypes binding of the CPU oracle (oracle/pkv_oracle.cpp).

TEST INFRASTRUCTURE ONLY: imported by tests/, __graft_entry__.smoke() and bench.py's
cpu_baseline / --impl reference legs. Nothing under pyramidkv_b200/ imports this module.

All functions take CPU torch tensors in the model dtype (bf16 / fp16) and return CPU tensors.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess
from dataclasses import dataclass
from typing import Optional

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "libpkv_oracle.so")

METHODS = {"pyramidkv": 0, "snapkv": 1, "h2o": 2, "streamingllm": 3, "l2norm": 4}
POOLING = {"avgpool": 0, "maxpool": 1}
TIE_LOWEST_INDEX, TIE_TORCH_CPU = 0, 1

_lib = None


def build(force: bool = False) -> str:
    """Compile the oracle with the committed Makefile (g++ only; no GPU needed)."""
    src = os.path.join(_HERE, "pkv_oracle.cpp")
    if force or not os.path.exists(_SO) or os.path.getmtime(_SO) < os.path.getmtime(src):
        subprocess.run(["make", "-C", _HERE, "-B", "libpkv_oracle.so"], check=True, capture_output=True)
    return _SO


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(_SO):
            build()
        L = C.CDLL(_SO)
        i32, i64, p = C.c_int, C.c_int64, C.c_void_p
        L.pkvo_version.restype = i32
        L.pkvo_num_threads.restype = i32
        L.pkvo_layer_budget.argtypes = [i32, i64, i64, i32, i32, i64, i32, C.POINTER(i64), C.POINTER(i32)]
        L.pkvo_layer_budget.restype = i32
        L.pkvo_window_logits.argtypes = [p, p, i32, i32, i32, i64, i32, i32, i64, i64, i64, i64, p]
        L.pkvo_window_logits.restype = None
        L.pkvo_softmax_rows.argtypes = [p, i32, i64, i64, p]
        L.pkvo_softmax_rows.restype = None
        L.pkvo_window_sum.argtypes = [p, i32, i32, i32, i64, p]
        L.pkvo_window_sum.restype = None
        L.pkvo_pool.argtypes = [p, i32, i32, i64, i32, i32, p]
        L.pkvo_pool.restype = i32
        L.pkvo_topk.argtypes = [p, i32, i32, i64, i64, i32, p]
        L.pkvo_topk.restype = i32
        L.pkvo_gather.argtypes = [p, i32, i32, i64, i32, i32, i64, i64, p, i64, p, i64]
        L.pkvo_gather.restype = None
        L.pkvo_h2o_scores.argtypes = [p, p, i32, i32, i32, i64, i32, i32, i64, i64, i64, i64, p]
        L.pkvo_h2o_scores.restype = None
        L.pkvo_key_norms.argtypes = [p, i32, i32, i64, i32, i64, i64, p]
        L.pkvo_key_norms.restype = None
        L.pkvo_window_mean.argtypes = [p, i32, i32, i32, i64, p]
        L.pkvo_window_mean.restype = None
        L.pkvo_adakv_capacities.argtypes = [p, i32, i32, i64, i64, C.c_float, i64, i32, p, p, p, p, p, p]
        L.pkvo_adakv_capacities.restype = i32
        L.pkvo_rope_inplace.argtypes = [p, i32, i32, i64, i32, i64, i64, p, p, i64]
        L.pkvo_rope_inplace.restype = None
        L.pkvo_evict.argtypes = [i32, i32, i32, i32, i32, i32, i32, i64, i32, i32, i64,
                                 p, i64, i64, p, i64, i64, p, i64, i64, p, p, i64, p, p, p, p, p]
        L.pkvo_evict.restype = i32
        L.pkvo_decode_attn.argtypes = [p, p, p, i32, i32, i32, i64, i64, p]
        L.pkvo_decode_attn.restype = None
        L.pkvo_decode_attn_exact.argtypes = [p, p, p, i32, i32, i32, i64, i64, p]
        L.pkvo_decode_attn_exact.restype = None
        _lib = L
    return _lib


def num_threads() -> int:
    return int(lib().pkvo_num_threads())


def _dt(t: torch.Tensor) -> int:
    if t.dtype == torch.bfloat16:
        return 0
    if t.dtype == torch.float16:
        return 1
    raise TypeError(f"oracle supports bf16/fp16 only, got {t.dtype}")


def _chk3(t: torch.Tensor, name: str) -> torch.Tensor:
    """[H, S, D] view with a contiguous last dim; accepts [1, H, S, D]."""
    if t.dim() == 4:
        assert t.shape[0] == 1, f"{name}: batch size must be 1"
        t = t[0]
    assert t.dim() == 3 and t.device.type == "cpu", name
    if t.stride(-1) != 1:
        t = t.contiguous()
    return t


def layer_budget(method: str, max_capacity_prompt: int, window_size: int, num_layers: int, layer_idx: int,
                 q_len: int, beta: int = 20):
    """-> (mode, k): mode 0 = passthrough (q_len < capacity), 1 = evict keeping k + window rows."""
    k, mode = C.c_int64(0), C.c_int(0)
    rc = lib().pkvo_layer_budget(METHODS[method], max_capacity_prompt, window_size, num_layers, layer_idx, q_len,
                                 beta, C.byref(k), C.byref(mode))
    if rc:
        raise AssertionError("max_capacity_prompt - window_size must be > 0")
    return mode.value, k.value


@dataclass
class EvictResult:
    k_cache: torch.Tensor            # [Hq, k+W, D]
    v_cache: torch.Tensor
    idx: Optional[torch.Tensor]      # [Hq, k] int64
    logits: Optional[torch.Tensor]   # [Hq, W, S]
    probs: Optional[torch.Tensor]    # [Hq, W, S]
    wsum: Optional[torch.Tensor]     # [Hq, S-W]
    pooled: Optional[torch.Tensor]   # [Hq, S-W]


def evict(method: str, q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, window_size: int, top_k: int,
          kernel_size: int = 5, pooling: str = "avgpool", tie_mode: int = TIE_LOWEST_INDEX,
          stages: bool = True) -> EvictResult:
    """One layer's prefill eviction. q [Hq,S,D] (or [1,Hq,S,D]); k, v [Hkv,S,D] (un-repeated or repeated).
    method "l2norm": window_size must be 0, top_k = max_capacity_prompt; `pooled` holds the negated key norms."""
    q, k, v = _chk3(q, "q"), _chk3(k, "k"), _chk3(v, "v")
    Hq, S, D = q.shape
    Hkv = k.shape[0]
    W, dt = window_size, _dt(q)
    if pooling not in POOLING:
        raise ValueError("Pooling method not supported")
    n = S - W
    cap = top_k + W
    kc = torch.empty(Hq, cap, D, dtype=q.dtype)
    vc = torch.empty(Hq, cap, D, dtype=q.dtype)
    scoring = method in ("pyramidkv", "snapkv")
    logits = torch.empty(Hq, W, S, dtype=q.dtype) if (stages and scoring) else None
    probs = torch.empty(Hq, W, S, dtype=q.dtype) if (stages and scoring) else None
    wsum = torch.empty(Hq, n, dtype=q.dtype) if (stages and method != "streamingllm") else None
    pooled = torch.empty(Hq, n, dtype=q.dtype) if (stages and method != "streamingllm") else None
    idx = torch.empty(Hq, top_k, dtype=torch.int64)
    ptr = lambda t: t.data_ptr() if t is not None else None
    rc = lib().pkvo_evict(METHODS[method], dt, POOLING[pooling], kernel_size, tie_mode, Hq, Hkv, S, D, W, top_k,
                          q.data_ptr(), q.stride(0), q.stride(1), k.data_ptr(), k.stride(0), k.stride(1),
                          v.data_ptr(), v.stride(0), v.stride(1), kc.data_ptr(), vc.data_ptr(), cap,
                          ptr(logits), ptr(probs), ptr(wsum), ptr(pooled), idx.data_ptr())
    if rc == 2:
        raise ValueError("Pooling method not supported")
    if rc:
        raise ValueError("oracle: bad argument")
    return EvictResult(kc, vc, idx, logits, probs, wsum, pooled)


def key_norms(k):
    """[Hkv, S] L2 norms of the key rows in the model dtype (torch.norm(key_states, p=2, dim=-1), pyramidkv_utils.py:420)."""
    k = _chk3(k, "k")
    Hkv, S, D = k.shape
    out = torch.empty(Hkv, S, dtype=k.dtype)
    lib().pkvo_key_norms(k.data_ptr(), _dt(k), Hkv, S, D, k.stride(0), k.stride(1), out.data_ptr())
    return out


def adakv_scores(q, k, window_size, kernel_size=7, pooling="maxpool"):
    """`calcul_attn_sore` of AdaKV / HeadKV (pyramidkv_utils.py:647-672): window logits -> softmax -> MEAN over the window
    rows -> 1-D pool. q [Hq,S,D], k [Hkv,S,D] -> [Hq, S-W] model dtype."""
    q, k = _chk3(q, "q"), _chk3(k, "k")
    Hq, S, D = q.shape
    W = window_size
    probs = softmax_rows(window_logits(q, k, W))
    out = torch.empty(Hq, S - W, dtype=q.dtype)
    lib().pkvo_window_mean(probs.data_ptr(), _dt(q), Hq, W, S, out.data_ptr())
    return pool(out, kernel_size, pooling)


def adakv_capacities(score, base_capacity, floor_ratio=0.2, normalize=True, details=False, ratio_out=None):
    """Per-head budgets (pyramidkv_utils.py:702-717) under the CUDA path's tie rule. score [H, n] -> int32 [H]
    (details=True: also counts above / equal to the global threshold and the threshold itself). A head whose scores are
    all zero has ratio 0 / 0 = NaN under `normalize`; its scaled scores rank above every value, as in torch.
    `ratio_out`: a float32 [H] tensor that receives every head's ratio (1 without `normalize`)."""
    import numpy as np
    x = score.contiguous()
    H, n = x.shape
    caps = torch.empty(H, dtype=torch.int32)
    gt, eq = torch.empty(H, dtype=torch.int64), torch.empty(H, dtype=torch.int64)
    thr = torch.zeros(1, dtype=x.dtype)
    scaled = torch.empty_like(x) if details else None
    rc = lib().pkvo_adakv_capacities(x.data_ptr(), _dt(x), H, n, base_capacity, float(np.float32(1 - floor_ratio)),
                                     int(base_capacity * floor_ratio), int(bool(normalize)), caps.data_ptr(), gt.data_ptr(),
                                     eq.data_ptr(), thr.data_ptr(), scaled.data_ptr() if details else None,
                                     ratio_out.data_ptr() if ratio_out is not None else None)
    if rc:
        raise ValueError("oracle: base_capacity out of range")
    return (caps, gt, eq, thr, scaled) if details else caps


def ragged_evict(k, v, score, capacities, window_size):
    """Head h keeps its capacities[h] best-scored tokens ((score desc, index asc) order) + the last `window_size` tokens
    (pyramidkv_utils.py:731-757 / :852-878). k, v [Hkv,S,D]; score [Hq, S-W]. Returns (k_rows, v_rows, idx): lists of
    per-head tensors [c_h + W, D] and the per-head index tensors."""
    k, v = _chk3(k, "k"), _chk3(v, "v")
    Hq = score.shape[0]
    kmax = int(max(int(c) for c in capacities)) if len(capacities) else 0
    idx = topk(score, kmax, TIE_LOWEST_INDEX)
    G = Hq // k.shape[0]
    ks, vs, ids = [], [], []
    for h in range(Hq):
        c = int(capacities[h])
        ih = idx[h:h + 1, :c].contiguous()
        ks.append(gather(k[h // G:h // G + 1], ih, window_size, 1)[0])
        vs.append(gather(v[h // G:h // G + 1], ih, window_size, 1)[0])
        ids.append(ih[0])
    return ks, vs, ids


def rope_inplace(x, cos, sin):
    """x [H, S, D] (any strides, contiguous last dim) rotated IN PLACE; cos/sin [S, D] model dtype
    (HF apply_rotary_pos_emb, llama_model.py:157)."""
    assert x.dim() == 3 and x.stride(-1) == 1 and x.shape[-1] <= 512 and cos.shape == sin.shape == (x.shape[1], x.shape[2])
    cos, sin = cos.contiguous(), sin.contiguous()
    lib().pkvo_rope_inplace(x.data_ptr(), _dt(x), x.shape[0], x.shape[1], x.shape[2], x.stride(0), x.stride(1),
                            cos.data_ptr(), sin.data_ptr(), cos.stride(0))
    return x


def window_logits(q, k, window_size):
    q, k = _chk3(q, "q"), _chk3(k, "k")
    Hq, S, D = q.shape
    out = torch.empty(Hq, window_size, S, dtype=q.dtype)
    lib().pkvo_window_logits(q.data_ptr(), k.data_ptr(), _dt(q), Hq, k.shape[0], S, D, window_size,
                             q.stride(0), q.stride(1), k.stride(0), k.stride(1), out.data_ptr())
    return out


def softmax_rows(logits):
    x = logits.contiguous()
    out = torch.empty_like(x)
    S = x.shape[-1]
    lib().pkvo_softmax_rows(x.data_ptr(), _dt(x), x.numel() // S, S, out.data_ptr())
    return out


def window_sum(probs):
    p = probs.contiguous()
    Hq, W, S = p.shape
    out = torch.empty(Hq, S - W, dtype=p.dtype)
    lib().pkvo_window_sum(p.data_ptr(), _dt(p), Hq, W, S, out.data_ptr())
    return out


def pool(wsum, kernel_size, pooling):
    if pooling not in POOLING:
        raise ValueError("Pooling method not supported")
    x = wsum.contiguous()
    out = torch.empty_like(x)
    rc = lib().pkvo_pool(x.data_ptr(), _dt(x), x.shape[0], x.shape[1], kernel_size, POOLING[pooling], out.data_ptr())
    if rc:
        raise ValueError("oracle: kernel_size must be odd and >= 1")
    return out


def topk(scores, k, tie_mode=TIE_LOWEST_INDEX):
    x = scores.contiguous()
    out = torch.empty(x.shape[0], k, dtype=torch.int64)
    rc = lib().pkvo_topk(x.data_ptr(), _dt(x), x.shape[0], x.shape[1], k, tie_mode, out.data_ptr())
    if rc:
        raise ValueError("oracle: k out of range")
    return out


def gather(src, idx, window_size, num_q_heads):
    src = _chk3(src, "src")
    Hkv, S, D = src.shape
    k = idx.shape[1] if idx is not None else 0
    out = torch.empty(num_q_heads, k + window_size, D, dtype=src.dtype)
    ip = idx.contiguous().data_ptr() if idx is not None else None
    lib().pkvo_gather(src.data_ptr(), num_q_heads, Hkv, S, D, window_size, src.stride(0), src.stride(1), ip, k,
                      out.data_ptr(), k + window_size)
    return out


def h2o_scores(q, k, window_size):
    q, k = _chk3(q, "q"), _chk3(k, "k")
    Hq, S, D = q.shape
    out = torch.empty(Hq, S - window_size, dtype=q.dtype)
    lib().pkvo_h2o_scores(q.data_ptr(), k.data_ptr(), _dt(q), Hq, k.shape[0], S, D, window_size,
                          q.stride(0), q.stride(1), k.stride(0), k.stride(1), out.data_ptr())
    return out


def decode_attn(q, k_cache, v_cache, length):
    """q [Hq, D]; caches [Hq, cap, D] contiguous; first `length` rows valid -> [Hq, D] model dtype."""
    q, kc, vc = q.contiguous(), k_cache.contiguous(), v_cache.contiguous()
    Hq, cap, D = kc.shape
    out = torch.empty(Hq, D, dtype=q.dtype)
    lib().pkvo_decode_attn(q.data_ptr(), kc.data_ptr(), vc.data_ptr(), _dt(q), Hq, D, length, cap, out.data_ptr())
    return out


def decode_attn_exact(q, k_cache, v_cache, length):
    q, kc, vc = q.contiguous(), k_cache.contiguous(), v_cache.contiguous()
    Hq, cap, D = kc.shape
    out = torch.empty(Hq, D, dtype=torch.float32)
    lib().pkvo_decode_attn_exact(q.data_ptr(), kc.data_ptr(), vc.data_ptr(), _dt(q), Hq, D, length, cap,
                                 out.data_ptr())
    return out
