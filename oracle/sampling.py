"""CPU restatement of the sampling rules of include/pkv.h (pkv_sample_tokens, DESIGN.md §4.6): numpy Philox4x32-10, the
kept set of temperature / top-k / top-p in fp64, and the Gumbel-max draw. Test infrastructure; the product never imports it."""
from __future__ import annotations

from dataclasses import dataclass

import numpy as np

M0, M1 = 0xD2511F53, 0xCD9E8D57
W0, W1 = 0x9E3779B9, 0xBB67AE85
MASK = 0xFFFFFFFF
TOP_P_TOLERANCE = 1e-5        # relative: the kernel's prefix mass may decide differently only this close to top_p


def philox4x32_10(ctr, key):
    """ctr: 4 arrays (or ints) of uint32 words, key: 2. Returns the 4 output words as uint64 arrays holding uint32 values."""
    c = [np.asarray(w, dtype=np.uint64) & MASK for w in ctr]
    c = np.broadcast_arrays(*c)
    c = [w.copy() for w in c]
    k0, k1 = int(key[0]) & MASK, int(key[1]) & MASK
    for r in range(10):
        if r:
            k0, k1 = (k0 + W0) & MASK, (k1 + W1) & MASK
        p0 = np.uint64(M0) * c[0]
        p1 = np.uint64(M1) * c[2]
        hi0, lo0 = p0 >> np.uint64(32), p0 & np.uint64(MASK)
        hi1, lo1 = p1 >> np.uint64(32), p1 & np.uint64(MASK)
        c = [hi1 ^ c[1] ^ np.uint64(k0), lo1, hi0 ^ c[3] ^ np.uint64(k1), lo0]
    return c


def uniforms(V: int, seed: int, t: int) -> np.ndarray:
    """u_i for i < V: word (i & 3) of Philox(counter = {i >> 2, 0, lo32(t), hi32(t)}, key = {lo32(seed), hi32(seed)}),
    u = (2 * (r >> 9) + 1) * 2^-24 (fp64, exact)."""
    seed, t = int(seed) % 2 ** 64, int(t) % 2 ** 64
    g = np.arange((V + 3) // 4, dtype=np.uint64)
    words = philox4x32_10([g, 0, t & MASK, t >> 32], [seed & MASK, seed >> 32])
    r = np.stack(words, axis=1).reshape(-1)[:V]
    return ((r >> np.uint64(9)) * 2 + 1).astype(np.float64) * 2.0 ** -24


@dataclass
class Draw:
    token: int
    kept: np.ndarray | None      # bool [V]; None when the token is the argmax of rule 1 / 6
    near_top_p: bool             # the token depends on prefix masses within a relative TOP_P_TOLERANCE of top_p
    gap: float                   # best minus second-best perturbed score over the kept set (inf with one kept token)
    scale: float                 # magnitude of the perturbed scores compared (for an ulp-relative tolerance)


def sample_row(logits, temperature: float, top_k: int, top_p: float, seed: int, t: int) -> Draw:
    """Rules 1-6 for one row of logits (any float array holding the 16-bit values exactly)."""
    l = np.asarray(logits, dtype=np.float32)
    V = l.shape[0]
    T = np.float32(temperature)
    top_p = np.float32(top_p)
    if not (T >= 0 and top_k >= 0 and 0 < top_p <= 1):
        return Draw(-1, None, False, np.inf, 0.0)
    amax = int(np.argmax(l))                              # first index; NaN counts as the largest (as torch.argmax)
    if T == 0 or top_k == 1 or np.isnan(l[amax]):
        return Draw(amax, None, False, np.inf, 0.0)
    with np.errstate(over="ignore", divide="ignore", invalid="ignore"):
        x = (l / T).astype(np.float32)                    # IEEE fp32 division
    m = x.max()
    if not np.isfinite(m):
        return Draw(amax, None, False, np.inf, 0.0)
    kept = np.ones(V, dtype=bool)
    if 1 < top_k < V:
        kappa = np.sort(x)[::-1][top_k - 1]
        kept = x >= kappa
    near = False
    g = -np.log(-np.log(uniforms(V, seed, t)))
    if top_p < 1:
        idx = np.nonzero(kept)[0]
        order = idx[np.lexsort((idx, -x[idx].astype(np.float64)))]     # x descending, index ascending
        e = np.exp(x[order].astype(np.float64) - np.float64(m))
        cum = np.cumsum(e) / e.sum()
        p = np.float64(top_p)
        hit = np.nonzero(cum >= p)[0]
        n = int(hit[0]) + 1 if hit.size else len(order)
        # every prefix length a mass error of TOP_P_TOLERANCE could pick; the row is "near" when they draw different tokens
        lo = np.nonzero(cum >= p * (1 - TOP_P_TOLERANCE))[0]
        hi = np.nonzero(cum >= p * (1 + TOP_P_TOLERANCE))[0]
        n_lo = int(lo[0]) + 1 if lo.size else len(order)
        n_hi = int(hi[0]) + 1 if hi.size else len(order)
        if n_hi > n_lo:
            so = x[order].astype(np.float64) + g[order]
            best = np.maximum.accumulate(so)
            near = bool(best[n_hi - 1] != best[n_lo - 1])
        kept = np.zeros(V, dtype=bool)
        kept[order[:n]] = True
    s = np.where(kept, x.astype(np.float64) + g, -np.inf)
    tok = int(np.argmax(s))                               # lowest index among ties
    ks = np.sort(s[kept])[::-1]
    gap = float(ks[0] - ks[1]) if ks.size > 1 else np.inf
    scale = float(max(abs(ks[0]), np.abs(x[kept].astype(np.float64)).max(), np.abs(g[kept]).max()))
    return Draw(tok, kept, near, gap, scale)


def kept_probabilities(logits, temperature: float, top_k: int, top_p: float) -> np.ndarray:
    """softmax(x) over the kept set (fp64, zero elsewhere): the distribution the draw follows."""
    d = sample_row(logits, temperature, top_k, top_p, 0, 0)
    l = np.asarray(logits, dtype=np.float32)
    if d.kept is None:
        p = np.zeros(l.shape[0])
        p[d.token] = 1.0
        return p
    x = (l / np.float32(temperature)).astype(np.float32).astype(np.float64)
    e = np.where(d.kept, np.exp(x - x[d.kept].max()), 0.0)
    return e / e.sum()
