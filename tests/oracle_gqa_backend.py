"""TEST-ONLY backend for GQA-shared caches (knob pkv_gqa_shared): the FP8 oracle backend plus the torch twin of the group
reduction of include/pkv.h (PKV_FLAG_GQA_SHARED), an eviction that selects per KV head, and grouped decodes that
repeat-interleave the per-KV-head cache into the existing oracle decodes. Never importable from product code."""
import torch

from oracle import pkv_oracle as O
from oracle_fp8_backend import OracleFp8Backend


def group_reduce(pooled: torch.Tensor, G: int) -> torch.Tensor:
    """pooled [Hq, n] (bf16 / fp16) -> [Hq / G, n]: rn_dtype((sum over g ascending, in fp32, of pooled[j*G+g]) / f32(G)).
    Tensor-by-tensor additions and one tensor division: IEEE fp32 operations, each correctly rounded."""
    x = pooled.detach().cpu().float()
    Hq, n = x.shape
    xs = x.reshape(Hq // G, G, n)
    s = xs[:, 0].clone()
    for g in range(1, G):
        s = s + xs[:, g]
    return (s / torch.full_like(s, float(G))).to(pooled.dtype)


def _full_q(q, S):
    if q.shape[-2] == S:
        return q
    full = torch.zeros(q.shape[0], S, q.shape[-1], dtype=q.dtype)
    full[:, S - q.shape[-2]:] = q
    return full


def evict_gqa(method, q, k, v, window_size, top_k, kernel_size=5, pooling="avgpool", tie_mode=O.TIE_LOWEST_INDEX):
    """The GQA-shared eviction of one layer on the CPU: (k_cache [Hkv, top_k+W, D], v_cache, idx [Hkv, top_k], s_kv or None)."""
    Hkv, S, _ = k.shape
    q = _full_q(q, S)
    G = q.shape[0] // Hkv
    pooling = pooling if pooling in O.POOLING else "avgpool"
    if method in ("streamingllm", "l2norm"):
        # the selection does not depend on the query head: the per-query-head result with the duplicates removed
        r = O.evict(method, q, k, v, window_size, top_k, kernel_size, pooling, tie_mode=tie_mode, stages=False)
        return r.k_cache[::G].contiguous(), r.v_cache[::G].contiguous(), r.idx[::G].contiguous(), None
    r = O.evict(method, q, k, v, window_size, top_k, kernel_size, pooling, tie_mode=tie_mode, stages=True)
    s_kv = group_reduce(r.pooled, G)
    idx = O.topk(s_kv, top_k, tie_mode)
    return O.gather(k, idx, window_size, Hkv), O.gather(v, idx, window_size, Hkv), idx, s_kv


class OracleGqaBackend(OracleFp8Backend):
    name = "oracle-cpu gqa-shared (tests only)"

    def evict(self, method, q, k, v, window_size, top_k, k_cache, v_cache, kernel_size, pooling, idx_out=None, gqa_shared=False):
        if not gqa_shared:
            return super().evict(method, q, k, v, window_size, top_k, k_cache, v_cache, kernel_size, pooling, idx_out)
        kc, vc, idx, _ = evict_gqa(method, q, k, v, window_size, top_k, kernel_size, pooling, self.tie_mode)
        rows = top_k + window_size
        k_cache[:, :rows] = kc
        v_cache[:, :rows] = vc
        if idx_out is not None:
            idx_out.copy_(idx)

    @staticmethod
    def _expand(G, *ts):
        return [t.repeat_interleave(G, dim=1).contiguous() for t in ts]

    def decode_attn_batch_gqa(self, q, k_buf, v_buf, length, k_new, v_new, rows=None, step=None, max_length=0, workspace=None,
                              out=None, softmax_scale=0.0):
        B, Hkv = k_buf.shape[:2]
        G = q.shape[1] // Hkv
        kx, vx = self._expand(G, k_buf, v_buf)
        rx = rows.reshape(B, Hkv).repeat_interleave(G, dim=1).reshape(-1).contiguous() if rows is not None else None
        res = self.decode_attn_batch(q, kx, vx, length, k_new, v_new, rx, step, max_length, None, None, softmax_scale)
        k_buf.copy_(kx[:, ::G])
        v_buf.copy_(vx[:, ::G])
        if out is not None:
            out.copy_(res)
            return out
        return res

    def decode_attn_batch_gqa_fp8(self, q, k_q, v_q, k_scale, v_scale, length, k_new, v_new, rows=None, step=None, max_length=0,
                                  workspace=None, out=None, softmax_scale=0.0):
        B, Hkv = k_q.shape[:2]
        G = q.shape[1] // Hkv
        kx, vx = (t.view(torch.uint8).repeat_interleave(G, dim=1).view(torch.float8_e4m3fn) for t in (k_q, v_q))
        ksx, vsx = self._expand(G, k_scale, v_scale)
        rx = rows.reshape(B, Hkv).repeat_interleave(G, dim=1).reshape(-1).contiguous() if rows is not None else None
        res = self.decode_attn_batch_fp8(q, kx, vx, ksx, vsx, length, k_new, v_new, rx, step, max_length, None, None, softmax_scale)
        k_q.view(torch.uint8).copy_(kx.view(torch.uint8)[:, ::G])
        v_q.view(torch.uint8).copy_(vx.view(torch.uint8)[:, ::G])
        k_scale.copy_(ksx[:, ::G])
        v_scale.copy_(vsx[:, ::G])
        if out is not None:
            out.copy_(res)
            return out
        return res
