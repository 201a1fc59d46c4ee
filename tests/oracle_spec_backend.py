"""TEST-ONLY backend for prompt-lookup speculative decoding: the beam-search oracle backend plus CPU twins of
`pkv_decode_attn_multi` (fp64 attention over the rows each query sees, after storing the Q new rows as the cache form holds
them), `pkv_prompt_lookup` and `pkv_spec_step` (oracle/spec.py, sequence by sequence). Never importable from product code."""
import torch

from oracle import spec as OS
from oracle_beam_backend import OracleBeamBackend
from oracle_fp8_backend import dequantize, quantize_rows


def multi_twin(q, k_buf, v_buf, k_new, v_new, rows=None, length=0, step=None, max_length=0, scales=None, gqa=False,
               softmax_scale=0.0):
    """The verify attention on the CPU: q [B, Q, Hq, D], k_new / v_new [B, Q, Hkv, D]; writes the new rows in place and
    returns out [B, Q, Hq, D] (NaN for a (sequence, cache head) whose count is out of range)."""
    B, Q, Hq, D = q.shape
    H, cap = k_buf.shape[1], k_buf.shape[2]
    Hkv = k_new.shape[2]
    G = Hq // Hkv
    GH = G if gqa else 1
    max_length = int(max_length) or cap
    scale = softmax_scale or D ** -0.5
    extra = int(length) + (int(step.reshape(-1)[0]) if step is not None else 0)
    out = torch.full((B, Q, Hq, D), float("nan"), dtype=torch.float64)
    for b in range(B):
        for c in range(H):
            n0 = extra + (int(rows.reshape(-1)[b * H + c]) if rows is not None else 0)
            if n0 < 0 or n0 + Q > max_length:
                continue
            g = c if gqa else c // G
            if scales is None:
                k_buf[b, c, n0:n0 + Q] = k_new[b, :, g].to(k_buf.device)
                v_buf[b, c, n0:n0 + Q] = v_new[b, :, g].to(v_buf.device)
                K = k_buf[b, c, :n0 + Q].double().cpu()
                V = v_buf[b, c, :n0 + Q].double().cpu()
            else:
                for buf, sc, new in ((k_buf, scales[0], k_new), (v_buf, scales[1], v_new)):
                    qb, s = quantize_rows(new[b, :, g])
                    buf.view(torch.uint8)[b, c, n0:n0 + Q] = qb.view(torch.uint8).to(buf.device)
                    sc[b, c, n0:n0 + Q] = s.to(sc.device)
                K = dequantize(k_buf[b, c, :n0 + Q], scales[0][b, c, :n0 + Q]).double()
                V = dequantize(v_buf[b, c, :n0 + Q], scales[1][b, c, :n0 + Q]).double()
            heads = range(c * GH, c * GH + GH) if gqa else [c]
            mask = torch.arange(n0 + Q)[None, :] > (n0 + torch.arange(Q))[:, None]      # [Q, rows]: not visible
            for h in heads:
                s = (q[b, :, h].double().cpu() @ K.T) * scale
                p = torch.softmax(s.masked_fill(mask, float("-inf")), dim=-1)
                out[b, :, h] = p @ V
    return out.to(q.dtype)


def lookup_twin(st) -> None:
    """pkv_prompt_lookup on a SpecState (host or device tensors), sequence by sequence through oracle/spec.draft."""
    B, Q = st.ids.shape
    eos = st.eos.tolist()
    for b in range(B):
        L = int(st.hist_len[b])
        h = st.hist[b, :L].tolist()
        live = not bool(st.done[b])
        d = OS.draft(h, Q - 1, st.max_ngram, eos, int(st.budget[b])) if live else []
        st.ids[b] = torch.tensor([h[-1]] + d + [st.pad_token_id] * (Q - 1 - len(d)), dtype=torch.long)
        st.pos[b] = torch.arange(L - 1, L - 1 + Q)
        st.draft_len[b] = len(d)


def step_twin(st, rows) -> None:
    """pkv_spec_step: rule 3 through oracle/spec.accept, the cursors and every layer's row counts, then rule 1."""
    B, Q = st.ids.shape
    eos = st.eos.tolist()
    for b in range(B):
        n = 0
        if not bool(st.done[b]):
            d = int(st.draft_len[b])
            m = int(st.budget[b])
            toks = OS.accept(st.ids[b, 1:1 + d].tolist(), st.tokens[b].tolist(), m, eos)
            n = len(toks)
            L, o = int(st.hist_len[b]), int(st.out_len[b])
            st.hist[b, L:L + n] = torch.tensor(toks, dtype=torch.long)
            st.out[b, o:o + n] = torch.tensor(toks, dtype=torch.long)
            st.hist_len[b] = L + n
            st.out_len[b] = o + n
            st.budget[b] = m - n
            if toks[-1] in eos or m - n <= 0:
                st.done[b] = True
        st.emitted[b] = n
        for r in rows:
            H = r.numel() // B
            r.view(B, H)[b] += n
    lookup_twin(st)


class OracleSpecBackend(OracleBeamBackend):
    name = "oracle-cpu speculative (tests only)"

    def decode_attn_multi(self, q, k_buf, v_buf, k_new, v_new, rows=None, length=0, step=None, max_length=0, scales=None,
                          gqa=False, workspace=None, out=None, softmax_scale=0.0):
        res = multi_twin(q, k_buf, v_buf, k_new, v_new, rows, length, step, max_length, scales, gqa, softmax_scale)
        if out is not None:
            out.copy_(res)
            return out
        return res

    def prompt_lookup(self, st):
        lookup_twin(st)

    def spec_step(self, st, rows):
        step_twin(st, rows)
