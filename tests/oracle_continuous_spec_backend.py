"""TEST-ONLY backend for prompt-lookup speculation in the continuous loop: the speculative oracle backend plus CPU twins of
`pkv_spec_pack` (rule 2' of include/pkv.h, restated in `pack`) and `pkv_decode_attn_packed` (the dense verify twin of
tests/oracle_spec_backend.py, run per sequence over its packed rows). Never importable from product code."""
import torch

import oracle_spec_backend as OSB
from oracle_spec_backend import OracleSpecBackend


def pack(done, draft_len, budget, D: int, step: int):
    """Rule 2': slots take draft tokens in turn from slot step mod B; a done slot gets no row, a live slot b 1 + d' rows
    with d' = min(d_b, m_b - 1, the budget left); rows contiguous in slot order. Returns (d' per slot, row counts, row
    starts) as lists."""
    B = len(done)
    left = int(D)
    granted, count = [0] * B, [0] * B
    for k in range(B):
        b = (step % B + k) % B
        if done[b]:
            continue
        g = max(0, min(int(draft_len[b]), int(budget[b]) - 1, left))
        left -= g
        granted[b], count[b] = g, 1 + g
    start = [sum(count[:b]) for b in range(B)]
    return granted, count, start


def pack_twin(st, pk) -> None:
    """pkv_spec_pack on a SpecState and a PackState (host or device tensors)."""
    B, Q = st.ids.shape
    granted, count, start = pack([bool(x) for x in st.done.tolist()], st.draft_len.tolist(), st.budget.tolist(),
                                 pk.max_draft_tokens, int(pk.step.reshape(-1)[0]))
    M = pk.ids.numel()
    ids, pos = [st.pad_token_id] * M, [0] * M
    for b in range(B):
        for j in range(count[b]):
            ids[start[b] + j] = int(st.ids[b, j])
            pos[start[b] + j] = int(st.pos[b, j])
    st.draft_len.copy_(torch.tensor(granted, dtype=torch.int32))
    pk.row_count.copy_(torch.tensor(count, dtype=torch.int32))
    pk.row_start.copy_(torch.tensor(start, dtype=torch.int32))
    pk.ids.view(-1).copy_(torch.tensor(ids, dtype=torch.long))
    pk.pos.view(-1).copy_(torch.tensor(pos, dtype=torch.long))
    pk.totals[0] += sum(granted)
    pk.totals[1] += sum(c > 0 for c in count)


def packed_twin(q, k_buf, v_buf, k_new, v_new, row_start, row_count, num_queries, rows=None, max_length=0, scales=None,
                gqa=False, softmax_scale=0.0):
    """The packed verify attention on the CPU: q [1, M, Hq, D], k_new / v_new [1, M, Hkv, D]; sequence b's rows
    [row_start[b], row_start[b] + row_count[b]) go through the dense twin; rows no sequence owns are 0."""
    M, Hq, D = q.shape[1], q.shape[2], q.shape[3]
    B, H = k_buf.shape[:2]
    out = torch.zeros(1, M, Hq, D, dtype=q.dtype)
    for b in range(B):
        s0, c = int(row_start[b]), int(row_count[b])
        if c == 0 or c > num_queries or s0 < 0 or s0 + c > M:
            continue
        sc = None if scales is None else (scales[0][b:b + 1], scales[1][b:b + 1])
        r = None if rows is None else rows.reshape(-1)[b * H:(b + 1) * H]
        res = OSB.multi_twin(q[:, s0:s0 + c], k_buf[b:b + 1], v_buf[b:b + 1], k_new[:, s0:s0 + c], v_new[:, s0:s0 + c],
                             rows=r, max_length=max_length, scales=sc, gqa=gqa, softmax_scale=softmax_scale)
        out[0, s0:s0 + c] = res[0]
    return out


class OracleContinuousSpecBackend(OracleSpecBackend):
    name = "oracle-cpu continuous speculative (tests only)"

    def decode_attn_packed(self, q, k_buf, v_buf, k_new, v_new, row_start, row_count, num_queries, rows=None, max_length=0,
                           scales=None, gqa=False, workspace=None, out=None, softmax_scale=0.0):
        res = packed_twin(q, k_buf, v_buf, k_new, v_new, row_start, row_count, num_queries, rows, max_length, scales, gqa,
                          softmax_scale)
        if out is not None:
            out.copy_(res)
            return out
        return res

    def spec_pack(self, st, pk):
        pack_twin(st, pk)
