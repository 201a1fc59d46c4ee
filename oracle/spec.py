"""The rules of prompt-lookup speculative decoding (include/pkv.h: pkv_prompt_lookup, pkv_spec_step; DESIGN.md §4.13),
restated in plain Python: the reference the CPU twins of the kernels (tests/oracle_spec_backend.py) and the GPU tests
compare against.

HF's `generate(prompt_lookup_num_tokens=K, max_matching_ngram_size=N, do_sample=False)` without logits processors, per
sequence, with history h = prompt + tokens emitted so far (length L) and remaining budget m:
  1. draft: for n = min(N, L - 1) down to 1 the lowest start i with h[i:i+n] == h[L-n:L] and i + n < L; the draft is
     h[i+n : min(i+n+K, L)] cut before its first EOS id; no match: empty. No draft when m <= 1.
  2. verify: one forward over [last emitted, draft..., padding] gives the argmaxes t_0 .. t_K.
  3. accept: a = the number of leading j < d with draft[j] == t_j, a = min(a, m - 1); emit t_0 .. t_a, stopping after the
     first EOS id among them; done after an EOS or when m reaches 0.
"""
from __future__ import annotations


def draft(h, K: int, N: int, eos=(), m: int = 2) -> list:
    """Rule 1: the draft (a list of at most K ids) for history `h` (a sequence of ids) and budget `m`."""
    h = [int(t) for t in h]
    L = len(h)
    if m <= 1:
        return []
    eos = set(int(e) for e in eos)
    for n in range(min(N, L - 1), 0, -1):
        tail = h[L - n:]
        for i in range(0, L - n):
            if h[i:i + n] == tail:
                out = []
                for t in h[i + n:min(i + n + K, L)]:
                    if t in eos:
                        break
                    out.append(t)
                return out
    return []


def accept(draft_ids, t, m: int, eos=()) -> list:
    """Rule 3: the tokens emitted for draft `draft_ids` (d ids), verify argmaxes `t` (at least d + 1 ids) and budget m >= 1."""
    d = len(draft_ids)
    a = 0
    while a < d and int(draft_ids[a]) == int(t[a]):
        a += 1
    a = min(a, m - 1)
    out = []
    eos = set(int(e) for e in eos)
    for k in range(a + 1):
        out.append(int(t[k]))
        if int(t[k]) in eos:
            break
    return out
