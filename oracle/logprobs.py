"""CPU restatement of the log-probability rules of include/pkv.h (pkv_token_logprobs, DESIGN.md §4.8) in fp64: the raw
log-softmax of a row of 16-bit logits at a token and at the row's top N. Test infrastructure; the product never imports it."""
from __future__ import annotations

import numpy as np


def logprobs_row(logits, token: int, top_n: int):
    """(lp of `token`, top ids [top_n] int64, top lps [top_n] fp64) for one row (any float array holding the 16-bit values
    exactly). Top order: logit descending, then index ascending. A row with a NaN or +-inf logit gives NaN log-probabilities
    and top ids -1; so do the top entries past the vocabulary. A token outside [0, V) gives NaN."""
    x = np.asarray(logits, dtype=np.float32).astype(np.float64)
    V = x.shape[0]
    ids = np.full(top_n, -1, dtype=np.int64)
    top = np.full(top_n, np.nan)
    if not np.isfinite(x).all():
        return float("nan"), ids, top
    m = x.max()
    lp = (x - m) - np.log(np.exp(x - m).sum())
    n = min(top_n, V)
    order = np.lexsort((np.arange(V), -x))[:n]           # logit descending, index ascending
    ids[:n] = order
    top[:n] = lp[order]
    t = int(token)
    return (float(lp[t]) if 0 <= t < V else float("nan")), ids, top
