"""TEST-ONLY backend for heavy hitters in the decode window (knob pkv_decode_heavy): the window oracle backend plus
`decode_attn_heavy`, the CPU twin of `pkv_decode_attn_heavy` (include/pkv.h) with the probabilities and scores in fp64.
Never importable from product code."""
import torch

from oracle import pkv_oracle as O
from oracle_fp8_backend import dequantize, quantize_rows
from oracle_window_backend import OracleWindowBackend, window_slot


def pick_victim(A, gen, held: int, j: int, R: int, H: int) -> int:
    """The slot (index past P) of the next victim after the step that appended generation j: among the `held` slots whose
    row has generation index <= j + 1 - (R - H), the smallest A, ties to the smallest generation index. None when no row
    qualifies (a count that repeats, as a finished slot's does, appends generation j again)."""
    last = j + 1 - (R - H)
    cands = [(float(A[k]), int(gen[k]), k) for k in range(held) if int(gen[k]) <= last]
    return min(cands)[2] if cands else None


def decode_heavy_twin(q, k_buf, v_buf, scales, length, k_new, v_new, prompt_rows, window, heavy, scores, gen, victim, rows=None,
                      step=None, max_length=0, softmax_scale=0.0, gqa=False):
    """The semantics restated per (sequence b, cache head c): the window's step, with the new row at victim[b*H + c] once
    n > P + R, then the bookkeeping (the new row's A from 0, every held generated row adding its fp64 probabilities summed
    over the query heads of the cache head, and the next victim) in `scores` / `gen` / `victim` (updated in place, in their
    own dtype). Out-of-range counts and victims outside [P, P + R) read and write nothing and give a NaN output."""
    B, H, cap, D = k_buf.shape
    Hq = q.shape[1]
    G = Hq // H if gqa else 1
    Gq = Hq // k_new.shape[1]
    R = int(window)
    extra = int(length) + (int(step.item()) if step is not None else 0)
    scale = softmax_scale or D ** -0.5
    if scales is not None:
        kq_new, ks_new = quantize_rows(k_new)
        vq_new, vs_new = quantize_rows(v_new)
    res = torch.empty(B, Hq, D, dtype=q.dtype)
    A, GEN, VIC = scores.reshape(B * H, R), gen.reshape(B * H, R), victim.reshape(-1)
    for b in range(B):
        for c in range(H):
            bc = b * H + c
            n = extra + (int(rows.reshape(-1)[bc]) if rows is not None else 0)
            P = int(prompt_rows.reshape(-1)[bc])
            slot, T = window_slot(n, P, R)
            if n > P + R and n >= 1 and P >= 0:
                slot = int(VIC[bc])
            if n < 1 or P < 0 or T > (max_length or cap) or (n > P + R and not P <= slot < P + R):
                res[b, c * G:c * G + G] = float("nan")
                continue
            kv = (c * G) // Gq
            if scales is None:
                k_buf[b, c, slot], v_buf[b, c, slot] = k_new[b, kv], v_new[b, kv]
                K, V = k_buf[b, c, :T].cpu().double(), v_buf[b, c, :T].cpu().double()
            else:
                k_buf.view(torch.uint8)[b, c, slot] = kq_new.view(torch.uint8)[b, kv].to(k_buf.device)
                v_buf.view(torch.uint8)[b, c, slot] = vq_new.view(torch.uint8)[b, kv].to(v_buf.device)
                scales[0][b, c, slot] = ks_new[b, kv]
                scales[1][b, c, slot] = vs_new[b, kv]
                K = dequantize(k_buf[b, c, :T], scales[0][b, c, :T]).double().cpu()
                V = dequantize(v_buf[b, c, :T], scales[1][b, c, :T]).double().cpu()
            probs = torch.zeros(T, dtype=torch.float64)
            for h in range(c * G, c * G + G):
                p = torch.softmax((K @ q[b, h].cpu().double()) * scale, dim=0)
                probs += p
                if scales is None:
                    res[b, h] = O.decode_attn(q[b, h:h + 1].contiguous(), k_buf[b, c:c + 1], v_buf[b, c:c + 1], T)[0]
                else:
                    res[b, h] = (p @ V).to(q.dtype)
            if n <= P:              # an append inside the prompt: nothing is scored
                continue
            j = n - 1 - P
            held, k_new_slot = min(j + 1, R), slot - P
            for k in range(held):
                a = 0.0 if k == k_new_slot else float(A[bc, k])
                if k == k_new_slot:
                    GEN[bc, k] = j
                A[bc, k] = a + float(probs[P + k])
            if j + 1 >= R:
                k = pick_victim(A[bc], GEN[bc], held, j, R, int(heavy))
                VIC[bc] = -1 if k is None else P + k          # -1: the following steps are out of range
    return res


class OracleHeavyBackend(OracleWindowBackend):
    name = "oracle-cpu heavy-hitter decode window (tests only)"
    heavy_override = None      # tests: run every heavy layer with this H (H = 0, which the knob refuses, is the ring)

    def decode_heavy_workspace(self, num_seqs, num_q_heads, window, device):
        return None

    def decode_attn_heavy(self, q, k_buf, v_buf, length, k_new, v_new, prompt_rows, window, heavy, scores, gen, victim, rows=None,
                          step=None, max_length=0, workspace=None, scratch=None, out=None, softmax_scale=0.0, scales=None,
                          gqa=False):
        if self.heavy_override is not None:
            heavy = self.heavy_override
        res = decode_heavy_twin(q, k_buf, v_buf, scales, length, k_new, v_new, prompt_rows, window, heavy, scores, gen, victim,
                                rows, step, max_length, softmax_scale, gqa).to(q.device)
        if out is not None:
            out.copy_(res)
            return out
        return res
