"""TEST-ONLY backend for sampled decoding: the continuous-batching oracle backend (every cache form: 16-bit, FP8, GQA-shared,
AdaKV / HeadKV) plus `sample_tokens`, the CPU twin of `pkv_sample_tokens` (include/pkv.h) from oracle/sampling.py. Never
importable from product code."""
import torch

from oracle import sampling as S
from oracle_continuous_backend import OracleContinuousBackend


def sample_twin(logits, params, out, col, advance=True):
    if logits.dtype not in (torch.bfloat16, torch.float16):
        raise NotImplementedError(f"sample_tokens: bf16 / fp16 logits, got {logits.dtype}")
    rows = logits.detach().float().cpu().numpy()
    for b in range(rows.shape[0]):
        seed = int(params.seed[b]) % 2 ** 64
        d = S.sample_row(rows[b], float(params.temperature[b]), int(params.top_k[b]), float(params.top_p[b]), seed,
                         int(params.index[b]))
        out[b, col] = d.token
    if advance:
        params.index.add_(1)


class OracleSamplingBackend(OracleContinuousBackend):
    name = "oracle-cpu sampling (tests only)"

    def sample_tokens(self, logits, params, out, col, advance=True):
        sample_twin(logits, params, out, col, advance)
