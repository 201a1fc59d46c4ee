"""Beam search rules (include/pkv.h: pkv_beam_candidates, pkv_beam_step, pkv_cache_reorder; DESIGN.md §4.12), restated
in numpy fp32 as the reference of the kernels and of the test-only CPU backend.

They are steps c-g of transformers' `GenerationMixin._beam_search` (5.5.0, do_sample=False) for one prompt, with every
tie cut by (value descending, index ascending) where `torch.topk` leaves the order unspecified:
  c. score(r, v) = running[r] + lp_v; the candidates are the top K = max(2, 1 + n_eos) * k of the k rows' entries by
     (score descending, flat index r * V + v ascending);
  d. hit_c: token v_c is an EOS id, or t + 1 = max_steps (the maximum length);
  e. running: the top k of score_c + (hit_c ? -1e9 : -0);
  f. pool: x_c = score_c / (t + 1)^length_penalty, then + -1e9 when every pool entry is finished and early_stopping is True,
     + -1e9 when the early-stop heuristic already failed, + -1e9 unless hit_c and c < k; the new pool is the top k of the
     old k entries followed by the K x_c; a new entry is finished when hit_c and c < k;
  g. heuristic' = heuristic and any_j(running[0] / L^length_penalty > (finished_j ? min pool : -1e9)) with L = max_steps
     when early_stopping is "never" and length_penalty > 0, else t + 1; done = not heuristic' or (every pool entry
     finished and early_stopping is True) or t + 1 = max_steps.
The two divisions are torch's division of an fp32 tensor by a Python float d: on CUDA a multiply by f32(1 / d), the
reciprocal taken in double (form "cuda", what the kernel does; tests/test_gpu_beam.py probes it), on the CPU an IEEE
division by f32(d) (form "cpu", what HF computes on the CPU).
"""
from __future__ import annotations

import numpy as np

NEG = np.float32(-1.0e9)
NEG0 = np.float32(-0.0)


def scale(x: np.float32, d: float, form: str) -> np.float32:
    if form == "cuda":
        return np.float32(np.float32(x) * np.float32(1.0 / d))
    return np.float32(np.float32(x) / np.float32(d))


def _key(s):
    s = np.float32(s)
    return -np.inf if s != s else float(s)


def step(S, lp, ids, rows_per_prompt: int, t: int, form: str = "cuda") -> None:
    """One iteration of every prompt on S (numpy arrays, updated in place; the fields of generate.BeamState): lp / ids
    [rows, K] the candidates of each row (rows_per_prompt rows per prompt: k, or 1 at iteration 0)."""
    k, K, T = S.k, S.K, S.max_steps
    es = S.early_stopping
    for p in range(S.done.shape[0]):
        bk = p * k
        if S.done[p] or t >= T:
            S.next_token[bk:bk + k] = 0
            S.parent[bk:bk + k] = np.arange(k)
            S.diverge[bk:bk + k] = t
            continue
        ent = []
        for r in range(k):
            row = p if rows_per_prompt == 1 else bk + r
            for j in range(K):
                v = int(ids[row, j])
                ent.append((np.float32(S.running[bk + r] + np.float32(lp[row, j])), r, v))
        # an id of -1 (no entry: a non-finite row) after every token of its row, such entries by position; its token is 0
        order_e = sorted(range(len(ent)), key=lambda i: (-_key(ent[i][0]), ent[i][1], ent[i][2] if ent[i][2] >= 0 else 2 ** 32, i))
        cand = [(ent[i][0], ent[i][1], max(ent[i][2], 0)) for i in order_e[:K]]
        last = t + 1 >= T
        hit = [last or c[2] in S.eos for c in cand]
        run = [np.float32(c[0] + (NEG if h else NEG0)) for c, h in zip(cand, hit)]
        order = sorted(range(K), key=lambda c: (-_key(run[c]), c))[:k]
        d_pool, d_heur = S.divisors[t]
        all_fin = bool(S.pool_done[bk:bk + k].all())
        heur = bool(S.heuristic[p])
        xs = []
        for c in range(K):
            x = scale(cand[c][0], d_pool, form)
            x = np.float32(x + (NEG if all_fin and es == 1 else NEG0))
            x = np.float32(x + (NEG0 if heur else NEG))
            x = np.float32(x + (NEG0 if hit[c] and c < k else NEG))
            xs.append(x)
        merged = [(np.float32(S.pool_score[bk + j]), (int(S.pool_step[bk + j]), int(S.pool_parent[bk + j]),
                   int(S.pool_token[bk + j]), bool(S.pool_done[bk + j]))) for j in range(k)]
        merged += [(xs[c], (t, cand[c][1], cand[c][2], hit[c] and c < k)) for c in range(K)]
        pool = sorted(range(k + K), key=lambda i: (-_key(merged[i][0]), i))[:k]
        par = [cand[c][1] for c in order]
        cp = S.cp[p].copy()
        for a in range(k):
            S.diverge[bk + a] = t if par[a] == a else cp[a, par[a]]
            for b in range(k):
                S.cp[p, a, b] = t if par[a] == par[b] else cp[par[a], par[b]]
        for a in range(k):
            c = order[a]
            S.running[bk + a] = run[c]
            S.bp_token[bk + a, t] = cand[c][2]
            S.bp_parent[bk + a, t] = cand[c][1]
            S.next_token[bk + a] = cand[c][2]
            S.parent[bk + a] = cand[c][1]
            s, (st, pa, tk, fin) = merged[pool[a]]
            S.pool_score[bk + a] = s
            S.pool_step[bk + a], S.pool_parent[bk + a], S.pool_token[bk + a], S.pool_done[bk + a] = st, pa, tk, fin
        best = scale(S.running[bk], d_heur, form)
        ps = S.pool_score[bk:bk + k].astype(np.float32)
        worst = np.float32(ps.min())
        fins = S.pool_done[bk:bk + k].astype(bool)
        any_ = any(best > (worst if f else NEG) for f in fins)
        h = heur and any_
        S.heuristic[p] = h
        S.done[p] = (not h) or (bool(fins.all()) and es == 1) or last


def reorder_rows(n: int, parent, diverge, window=None, heavy=False):
    """Per beam slot a: the generated slots it copies from parent[a] (rule 3 of include/pkv.h)."""
    out = []
    for a, (pa, d) in enumerate(zip(parent, diverge)):
        if pa == a:
            out.append([])
        elif window is None:
            out.append(list(range(int(d), n)))
        elif heavy:
            out.append(list(range(min(n, window))))
        else:
            out.append(sorted(j % window for j in range(max(int(d), n - window), n)))
    return out
