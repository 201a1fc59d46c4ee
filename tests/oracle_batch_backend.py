"""TEST-ONLY backend for batched decoding: the CPU oracle backend plus `decode_attn_batch` (pkv_decode_attn_batch), answered
sequence by sequence through the oracle's single-sequence decode. Never importable from product code."""
import torch

from oracle_backend import OracleBackend


class OracleBatchBackend(OracleBackend):
    name = "oracle-cpu batched (tests only)"

    def decode_attn_batch(self, q, k_buf, v_buf, length, k_new, v_new, rows=None, step=None, max_length=0, workspace=None,
                          out=None, softmax_scale=0.0):
        """rows [B*Hq] -> each sequence's head_rows (the ragged form); rows None -> `length` (+ *step) rows everywhere."""
        B, Hq = k_buf.shape[0], k_buf.shape[1]
        assert q.shape == (B, Hq, q.shape[-1]) and (rows is None or (rows.dtype == torch.int32 and rows.numel() == B * Hq))
        res = torch.empty(B, Hq, q.shape[-1], dtype=q.dtype)
        for b in range(B):
            hr = rows.reshape(B, Hq)[b] if rows is not None else None
            res[b] = self.decode_attn(q[b], k_buf[b], v_buf[b], length, k_new[b], v_new[b], step=step,
                                      max_length=max_length or k_buf.shape[2], head_rows=hr)
        if out is not None:
            out.copy_(res)
            return out
        return res
