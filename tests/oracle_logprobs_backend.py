"""TEST-ONLY backend for token log-probabilities: the sampling oracle backend with the decode window (every cache form:
16-bit, FP8, GQA-shared, AdaKV / HeadKV, decode window) plus `token_logprobs`, the CPU twin of `pkv_token_logprobs`
(include/pkv.h) from oracle/logprobs.py. Never importable from product code."""
import torch

from oracle import logprobs as LP
from oracle_window_backend import OracleWindowBackend


def logprobs_twin(logits, tokens, out_lp, out_ids, out_top, col=0, tokens_col=0, cursor=None):
    if logits.dtype not in (torch.bfloat16, torch.float16):
        raise NotImplementedError(f"token_logprobs: bf16 / fp16 logits, got {logits.dtype}")
    c = int(col) + (int(cursor.reshape(-1)[0]) if cursor is not None else 0)
    rows = logits.detach().float().cpu().numpy()
    N = out_ids.shape[2]
    for b in range(rows.shape[0]):
        lp, ids, top = LP.logprobs_row(rows[b], int(tokens[b, tokens_col]), N)
        out_lp[b, c] = lp
        out_ids[b, c] = torch.from_numpy(ids)
        out_top[b, c] = torch.from_numpy(top).float()


class OracleLogprobsBackend(OracleWindowBackend):
    name = "oracle-cpu logprobs (tests only)"

    def token_logprobs(self, logits, tokens, out_lp, out_ids, out_top, col=0, tokens_col=0, cursor=None):
        logprobs_twin(logits, tokens, out_lp, out_ids, out_top, col, tokens_col, cursor)
