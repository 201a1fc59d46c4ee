"""fp64 restatement of eviction stages 1-2 in torch, for the device or the host.

The rounding chain is the CPU oracle's (oracle/pkv_oracle.cpp: score_elem, add_mask, pkvo_window_logits,
pkvo_softmax_rows, pkvo_window_sum, pkvo_window_mean, pkvo_pool, pkvo_h2o_scores, pkvo_key_norms):
  - the dot product in fp64, rounded to fp32, then to the model dtype;
  - the divide by sqrt(D) in fp32 (sqrt(D) as an fp32 scalar), rounded to the dtype;
  - the mask add on the last W x W block: fp32 add of finfo(dtype).min, rounded to the dtype (fp16: may give -inf);
  - the softmax in fp64 (max, exp, sum, divide), rounded to fp32, then to the dtype;
  - the window sum / mean: fp32 running sum over the W rows in row order (divide by W in fp32), one rounding;
  - the pool: max exact; avg an fp32 running sum in ascending token order with zero padding, fp32 divide, one rounding.
These match the oracle bit for bit except where the oracle's fp32 `expf` and the fp64 exp round to different fp32
values; the rounding to the dtype hides most of those.

One deliberate difference: H2O's column sums are accumulated in fp64 and rounded once (to fp32, then to the dtype), the
exact sum of the rounded probabilities. The oracle accumulates them in an fp32 running sum in row order, whose own error
grows with S (up to (S - 1) * 2^-24 relative); `h2o_scores` is therefore the better yardstick at long prompts, and the
oracle may differ from it by that summation error only.

Everything is chunked (over kv heads, and for H2O over query rows) so that no [Hq, S, S] tensor is ever held.
"""
from __future__ import annotations

import math

import torch

F64 = torch.float64


def finfo_min(dt) -> float:
    return float(torch.finfo(dt).min)


def rnd(x: torch.Tensor, dt) -> torch.Tensor:
    """fp64 / fp32 -> fp32 (round to nearest even) -> dtype (round to nearest even), returned as fp32."""
    return x.float().to(dt).float()


def sqrt_d32(D: int) -> torch.Tensor:
    return torch.tensor(math.sqrt(D), dtype=torch.float32)


def logits_block(qrows: torch.Tensor, keys: torch.Tensor, dt) -> torch.Tensor:
    """Unmasked logits of query rows [..., R, D] against keys [S, D] (dtype tensors): fp32 tensor [..., R, S] holding dtype
    values. fp64 GEMM (products of 16-bit values are exact in fp64), rounded to fp32, to the dtype, / sqrt(D) in fp32, to the
    dtype."""
    dot = torch.matmul(qrows.to(F64), keys.to(F64).transpose(-1, -2))
    r1 = rnd(dot, dt)
    return rnd(r1 / sqrt_d32(keys.shape[-1]).to(r1.device), dt)


def mask_block(x: torch.Tensor, rows: torch.Tensor, cols: torch.Tensor, n: int, dt) -> torch.Tensor:
    """Causal mask on the last W x W block: element (row i, col j) with i, j >= n and j > i gets round(x + finfo.min)."""
    m = (rows[:, None] >= n) & (cols[None, :] >= n) & (cols[None, :] > rows[:, None])
    if not bool(m.any()):
        return x
    masked = rnd(x + torch.tensor(finfo_min(dt), dtype=torch.float32, device=x.device), dt)
    return torch.where(m, masked, x)


def window_logits(q: torch.Tensor, k: torch.Tensor, W: int) -> torch.Tensor:
    """Observation-window logits after the mask add, [Hq, W, S] in the dtype (pkvo_window_logits). q is [Hq, S, D] or just
    its last W rows [Hq, W, D]; k is [Hkv, S, D]."""
    Hq, Hkv, S = q.shape[0], k.shape[0], k.shape[1]
    G, dt, n = Hq // Hkv, k.dtype, S - W
    qw = q[:, -W:]
    out = torch.empty(Hq, W, S, dtype=dt, device=k.device)
    rows = torch.arange(n, S, device=k.device)
    cols = torch.arange(S, device=k.device)
    for g in range(Hkv):
        x = logits_block(qw[g * G:(g + 1) * G], k[g], dt)                 # [G, W, S]
        x = mask_block(x.reshape(G * W, S), rows.repeat(G), cols, n, dt).reshape(G, W, S)
        out[g * G:(g + 1) * G] = x.to(dt)
    return out


def window_masked(W: int, S: int, device=None) -> torch.Tensor:
    """[1, W, S] bool: True where the causal mask of the last W x W block applies to window row w (token j >= S - W and
    j - (S - W) > w). Taken from the geometry, not from the values: in fp16 a masked logit is finfo.min = -65504, finite."""
    w = torch.arange(W, device=device)[:, None]
    jw = torch.arange(S, device=device)[None, :] - (S - W)
    return (jw > w)[None]


def softmax_stats(x: torch.Tensor):
    """fp64 (max, sum exp(x - max)) over the last dim of dtype logits."""
    xd = x.to(F64)
    m = xd.max(dim=-1, keepdim=True).values
    return m.squeeze(-1), torch.exp(xd - m).sum(dim=-1)


def softmax_rows(logits: torch.Tensor) -> torch.Tensor:
    """softmax(dim=-1) in fp64, rounded to fp32, then to the dtype (pkvo_softmax_rows)."""
    out = torch.empty_like(logits)
    for h in range(logits.shape[0]):                     # one head at a time: fp64 temporaries of [W, S] only
        xd = logits[h].to(F64)
        e = torch.exp(xd - xd.max(dim=-1, keepdim=True).values)
        out[h] = (e / e.sum(dim=-1, keepdim=True)).float().to(logits.dtype)
    return out


def _window_acc(probs: torch.Tensor) -> torch.Tensor:
    W, S = probs.shape[1], probs.shape[2]
    acc = torch.zeros(probs.shape[0], S - W, dtype=torch.float32, device=probs.device)
    for w in range(W):
        acc = acc + probs[:, w, :S - W].float()
    return acc


def window_sum(probs: torch.Tensor) -> torch.Tensor:
    """[Hq, W, S] -> [Hq, S-W]: fp32 running sum over the W rows, one rounding (pkvo_window_sum)."""
    return _window_acc(probs).to(probs.dtype)


def window_mean(probs: torch.Tensor) -> torch.Tensor:
    """AdaKV / HeadKV: the window sum divided by W in fp32, one rounding (pkvo_window_mean)."""
    W = probs.shape[1]
    return (_window_acc(probs) / torch.tensor(float(W), dtype=torch.float32)).to(probs.dtype)


def pool(wsum: torch.Tensor, kernel: int, pooling: str) -> torch.Tensor:
    """max_pool1d / avg_pool1d(kernel, padding=kernel // 2, stride=1, count_include_pad=True) (pkvo_pool)."""
    pad = kernel // 2
    H, n = wsum.shape
    x = wsum.float()
    if pooling == "maxpool":
        xp = torch.nn.functional.pad(x, (pad, pad), value=float("-inf"))
        r = xp[:, 0:n]
        for d in range(1, kernel):
            r = torch.maximum(r, xp[:, d:d + n])
        return r.to(wsum.dtype)
    xp = torch.nn.functional.pad(x, (pad, pad), value=0.0)
    s = torch.zeros(H, n, dtype=torch.float32, device=wsum.device)
    for d in range(kernel):                              # ascending token order, fp32
        s = s + xp[:, d:d + n]
    return (s / torch.tensor(float(kernel), dtype=torch.float32)).to(wsum.dtype)


def window_scores(logits: torch.Tensor, kernel: int, pooling: str, mean: bool = False) -> torch.Tensor:
    """Stage 2 on given logits [Hq, W, S]: softmax, window sum (or mean), pool."""
    probs = softmax_rows(logits)
    return pool(window_mean(probs) if mean else window_sum(probs), kernel, pooling)


def tile_partials(logits: torch.Tensor, G: int, tile: int = 128):
    """Per 128-token tile and logit column, the fp64 (max, sum exp(x - max)) of the valid tokens: [Hkv, tiles, G*W] each.
    Column order is the workspace's: head_in_group * W + w."""
    Hq, W, S = logits.shape
    Hkv, tiles = Hq // G, (S + tile - 1) // tile
    ms, ls = [], []
    for g in range(Hkv):                                 # one kv head at a time: fp64 temporaries of [G*W, S] only
        x = logits[g * G:(g + 1) * G].to(F64).reshape(G * W, S)
        x = torch.nn.functional.pad(x, (0, tiles * tile - S), value=float("-inf")).reshape(G * W, tiles, tile)
        m = x.max(dim=-1).values
        ms.append(m.t())
        ls.append(torch.exp(x - m[..., None]).nan_to_num(0.0).sum(dim=-1).t())
        del x
    return torch.stack(ms), torch.stack(ls)


def h2o_scores(q: torch.Tensor, k: torch.Tensor, W: int, rows_per_chunk: int = 512):
    """H2O scores (pkvo_h2o_scores): full softmax over all S keys with the causal mask on the last W x W block only; the
    column sums over all S rows of the probabilities rounded to the dtype, for keys j < S - W.
    Returns (colsum [Hq, S-W] dtype, row max [Hq, S] fp64, row sum-exp [Hq, S] fp64, flip share [Hq, S] fp64). The column
    sums are accumulated in fp64 and rounded once (see the module docstring). The flip share of a row is
    sum_j p_j * (e^(2 ulp(x_j)) - 1): the most its sum-exp can move relative to L when logits move by up to 2 dtype ulps."""
    Hq, S, D = q.shape
    Hkv = k.shape[0]
    G, dt, n = Hq // Hkv, k.dtype, S - W
    dev = k.device
    acc = torch.zeros(Hq, n, dtype=F64, device=dev)
    M = torch.empty(Hq, S, dtype=F64, device=dev)
    L = torch.empty(Hq, S, dtype=F64, device=dev)
    Fs = torch.empty(Hq, S, dtype=F64, device=dev)
    mant = 8 if dt == torch.bfloat16 else 11
    cols = torch.arange(S, device=dev)
    for g in range(Hkv):
        for r0 in range(0, S, rows_per_chunk):
            r1 = min(S, r0 + rows_per_chunk)
            x = logits_block(q[g * G:(g + 1) * G, r0:r1], k[g], dt)           # [G, R, S]
            rows = torch.arange(r0, r1, device=dev)
            if r1 > n:
                x = mask_block(x.reshape(G * (r1 - r0), S), rows.repeat(G), cols, n, dt).reshape(G, r1 - r0, S)
            xd = x.to(F64)
            m = xd.max(dim=-1, keepdim=True).values
            e = torch.exp(xd - m)
            s = e.sum(dim=-1, keepdim=True)
            M[g * G:(g + 1) * G, r0:r1] = m.squeeze(-1)
            L[g * G:(g + 1) * G, r0:r1] = s.squeeze(-1)
            u = torch.exp2(torch.floor(torch.log2(xd.abs().clamp(min=2.0 ** -24))) - (mant - 1))
            Fs[g * G:(g + 1) * G, r0:r1] = (e * torch.expm1(2 * u)).nan_to_num(nan=0.0).sum(dim=-1) / s.squeeze(-1)
            del u
            p = rnd(e[..., :n] / s, dt)
            acc[g * G:(g + 1) * G] += p.to(F64).sum(dim=1)
            del x, xd, e, p
    return acc.float().to(dt), M, L, Fs


def key_norms(k: torch.Tensor) -> torch.Tensor:
    """torch.norm(k, p=2, dim=-1) as pkvo_key_norms: squares summed in fp64, rounded to fp32, fp32 sqrt, one rounding."""
    return torch.sqrt(k.to(F64).pow(2).sum(dim=-1).float()).to(k.dtype)
