"""TEST-ONLY backend for the penalized sampler: the log-probability oracle backend (every cache form, the decode window
included) plus `sample_tokens_penalized`, the CPU twin of `pkv_sample_tokens_penalized` (include/pkv.h, DESIGN.md §4.10).
The rules are restated here: penalties in fp32 numpy (steps 1-3), then the kept set of oracle/sampling.py in fp64 and
min-p. Never importable from product code."""
from dataclasses import replace

import numpy as np
import torch

from oracle import sampling as S
from oracle_logprobs_backend import OracleLogprobsBackend

MIN_P_TOLERANCE = 1e-6        # relative: the kernel's expf may decide min-p differently only this close to min_p


def penalize(logits, repetition, presence, frequency, mask, counts) -> np.ndarray:
    """Steps 1-3: x = f32(logit); the repetition penalty over the prompt (mask) and generated (counts > 0) tokens; then
    x - frequency * count, then - presence, over the generated ones. Each operation rounded to fp32 once."""
    x = np.asarray(logits, dtype=np.float32).copy()
    c = np.asarray(counts).astype(np.int64)
    seen = c > 0
    rho = np.float32(repetition)
    with np.errstate(over="ignore", invalid="ignore"):
        if rho != 1:
            hit = seen | (np.asarray(mask) != 0)
            x = np.where(hit, np.where(x < 0, x * rho, x / rho), x).astype(np.float32)
        fq, pr = np.float32(frequency), np.float32(presence)
        sub = (fq * c[seen].astype(np.float32)).astype(np.float32)
        x[seen] = ((x[seen] - sub).astype(np.float32) - pr).astype(np.float32)
    return x


def params_valid(repetition, presence, frequency, min_p) -> bool:
    r, p, f, m = (np.float32(v) for v in (repetition, presence, frequency, min_p))
    return bool(0 < r < np.inf and np.isfinite(p) and np.isfinite(f) and 0 <= m <= 1)


def sample_row_penalized(logits, temperature, top_k, top_p, seed, t, repetition=1.0, presence=0.0, frequency=0.0,
                         min_p=0.0, mask=None, counts=None) -> S.Draw:
    """Rules 1-5 of pkv_sample_tokens_penalized for one row. `near_top_p` also marks a token that depends on a min-p
    comparison within a relative MIN_P_TOLERANCE of min_p."""
    V = np.asarray(logits).shape[0]
    mask = np.zeros(V, np.uint8) if mask is None else mask
    counts = np.zeros(V, np.int32) if counts is None else counts
    if not params_valid(repetition, presence, frequency, min_p):
        return S.Draw(-1, None, False, np.inf, 0.0)
    x = penalize(logits, repetition, presence, frequency, mask, counts)
    d = S.sample_row(x, temperature, top_k, top_p, seed, t)
    mp = np.float64(np.float32(min_p))
    if d.kept is None or mp == 0:
        return d
    y = (x / np.float32(temperature)).astype(np.float32)
    e = np.exp(y.astype(np.float64) - np.float64(y.max()))
    kept = d.kept & (e >= mp)
    # y == max: expf(0) = 1 exactly on both sides, so only the others can fall on either side of min_p
    near = d.near_top_p or bool((d.kept & (y != y.max()) & (np.abs(e - mp) <= MIN_P_TOLERANCE * mp)).any())
    g = -np.log(-np.log(S.uniforms(V, seed, t)))
    s = np.where(kept, y.astype(np.float64) + g, -np.inf)
    ks = np.sort(s[kept])[::-1]
    gap = float(ks[0] - ks[1]) if ks.size > 1 else np.inf
    scale = float(max(abs(ks[0]), np.abs(y[kept].astype(np.float64)).max(), np.abs(g[kept]).max()))
    return replace(d, token=int(np.argmax(s)), kept=kept, near_top_p=near, gap=gap, scale=scale)


def sample_penalized_twin(logits, params, out, col, advance=True):
    if logits.dtype not in (torch.bfloat16, torch.float16):
        raise NotImplementedError(f"sample_tokens_penalized: bf16 / fp16 logits, got {logits.dtype}")
    rows = logits.detach().float().cpu().numpy()
    V = rows.shape[1]
    mask = params.prompt_mask.cpu().numpy()
    counts = params.counts.cpu().numpy()
    for b in range(rows.shape[0]):
        d = sample_row_penalized(rows[b], float(params.temperature[b]), int(params.top_k[b]), float(params.top_p[b]),
                                 int(params.seed[b]) % 2 ** 64, int(params.index[b]), float(params.repetition_penalty[b]),
                                 float(params.presence_penalty[b]), float(params.frequency_penalty[b]),
                                 float(params.min_p[b]), mask[b, :V], counts[b, :V])
        out[b, col] = d.token
        if advance and d.token >= 0:
            params.counts[b, d.token] += 1
    if advance:
        params.index.add_(1)


class OraclePenaltyBackend(OracleLogprobsBackend):
    name = "oracle-cpu penalized sampling (tests only)"

    def sample_tokens_penalized(self, logits, params, out, col, advance=True):
        sample_penalized_twin(logits, params, out, col, advance)
