"""TEST-ONLY backend for the decode window (knob pkv_decode_window): the sampling oracle backend (every cache form) plus
`decode_attn_window`, the CPU twin of `pkv_decode_attn_window` (include/pkv.h). Never importable from product code."""
import torch

from oracle import pkv_oracle as O
from oracle_fp8_backend import dequantize, quantize_rows
from oracle_sampling_backend import OracleSamplingBackend


def window_slot(n: int, P: int, R: int):
    """(row the n-th row is stored at, rows attended) of a (sequence, cache head) with P prompt rows and window R."""
    if n > P + R:
        return P + (n - 1 - P) % R, P + R
    return n - 1, n


def decode_window_twin(q, k_buf, v_buf, scales, length, k_new, v_new, prompt_rows, window, rows=None, step=None, max_length=0,
                       softmax_scale=0.0, gqa=False):
    """The semantics restated per (sequence b, cache head c): n = length (+ *step) (+ rows[b*H + c]), P = prompt_rows[b*H + c];
    the new row (FP8: quantised by the rule of include/pkv.h) goes to its ring slot, and every query head reading cache head c
    attends the rows [0, attended). A count n < 1, P < 0 or an attended count above the capacity reads and writes nothing and
    gives a NaN output. 16-bit rows go through the oracle's decode (the rounding the unwindowed backends use);
    E4M3 rows through the fp64 attention over the dequantised rows of the FP8 backend."""
    B, H, cap, D = k_buf.shape
    Hq = q.shape[1]
    G = Hq // H if gqa else 1                    # query heads per cache head
    Gq = Hq // k_new.shape[1]                    # query heads per KV head (the source of the new row)
    extra = int(length) + (int(step.item()) if step is not None else 0)
    scale = softmax_scale or D ** -0.5
    if scales is not None:
        kq_new, ks_new = quantize_rows(k_new)
        vq_new, vs_new = quantize_rows(v_new)
    res = torch.empty(B, Hq, D, dtype=q.dtype)
    for b in range(B):
        for c in range(H):
            n = extra + (int(rows.reshape(-1)[b * H + c]) if rows is not None else 0)
            P = int(prompt_rows.reshape(-1)[b * H + c])
            slot, T = window_slot(n, P, int(window))
            assert (max_length or cap) <= cap
            if n < 1 or P < 0 or T > (max_length or cap):     # out of range: nothing read or written, a NaN output
                res[b, c * G:c * G + G] = float("nan")
                continue
            kv = (c * G) // Gq                   # the KV head of the query heads reading this cache head
            if scales is None:
                k_buf[b, c, slot], v_buf[b, c, slot] = k_new[b, kv], v_new[b, kv]
            else:
                k_buf.view(torch.uint8)[b, c, slot] = kq_new.view(torch.uint8)[b, kv].to(k_buf.device)
                v_buf.view(torch.uint8)[b, c, slot] = vq_new.view(torch.uint8)[b, kv].to(v_buf.device)
                scales[0][b, c, slot] = ks_new[b, kv]
                scales[1][b, c, slot] = vs_new[b, kv]
            for h in range(c * G, c * G + G):
                if scales is None:
                    res[b, h] = O.decode_attn(q[b, h:h + 1].contiguous(), k_buf[b, c:c + 1], v_buf[b, c:c + 1], T)[0]
                else:
                    K = dequantize(k_buf[b, c, :T], scales[0][b, c, :T]).double()
                    V = dequantize(v_buf[b, c, :T], scales[1][b, c, :T]).double()
                    p = torch.softmax((K @ q[b, h].cpu().double()) * scale, dim=0)
                    res[b, h] = (p @ V).to(q.dtype)
    return res


class OracleWindowBackend(OracleSamplingBackend):
    name = "oracle-cpu decode window (tests only)"

    def decode_attn_window(self, q, k_buf, v_buf, length, k_new, v_new, prompt_rows, window, rows=None, step=None, max_length=0,
                           workspace=None, out=None, softmax_scale=0.0, scales=None, gqa=False):
        res = decode_window_twin(q, k_buf, v_buf, scales, length, k_new, v_new, prompt_rows, window, rows, step, max_length,
                                 softmax_scale, gqa).to(q.device)
        if out is not None:
            out.copy_(res)
            return out
        return res
