"""TEST-ONLY backend for beam search: the heavy-hitter oracle backend (every cache form: 16-bit, FP8, GQA-shared, AdaKV /
HeadKV, decode window, heavy hitters) plus the CPU twins of `pkv_beam_candidates` (torch.log_softmax, as HF computes it),
`pkv_beam_step` (oracle/beam.py with HF's CPU division) and `pkv_cache_reorder` (the rows of rule 3 of include/pkv.h,
copied with torch indexing). `gather_reorder` is the reference those are held to: it replaces `cache.reorder_caches` and
gathers whole beam slots, with no divergence rows and no per-form tables. Never importable from product code."""
from types import SimpleNamespace

import numpy as np
import torch

from oracle import beam as OB
from oracle_heavy_backend import OracleHeavyBackend


def candidates_twin(logits, st):
    lp = torch.log_softmax(logits.float(), dim=-1)
    srt, idx = torch.sort(lp, dim=-1, descending=True, stable=True)        # ties: the lower index first
    R = logits.shape[0]
    st.cand_lp[:R] = srt[:, : st.K]
    st.cand_id[:R] = idx[:, : st.K].to(torch.int32)
    st.m[:R] = logits.float().max(dim=-1).values
    st.log_z[:R] = torch.logsumexp(logits.float() - st.m[:R, None], dim=-1)


def state_view(st):
    """The fields of a BeamState as numpy views (in place), with the parameters oracle/beam.step reads."""
    ns = SimpleNamespace(k=st.k, K=st.K, max_steps=st.max_steps, early_stopping=st.early_stopping, eos=list(st.eos),
                         divisors=st.divisors)
    for f in ("running", "pool_score", "pool_step", "pool_parent", "pool_token", "pool_done", "heuristic", "done",
              "bp_token", "bp_parent", "cp", "next_token", "parent", "diverge"):
        setattr(ns, f, getattr(st, f).numpy())
    return ns


def step_twin(st, rows_per_prompt, step, step_offset):
    S = state_view(st)
    OB.step(S, st.cand_lp.numpy(), st.cand_id.numpy(), rows_per_prompt, int(step.reshape(-1)[0]) + int(step_offset), "cpu")


def reorder_twin(items, P, k, parent, diverge, step, step_offset):
    """Every copy of pkv_cache_reorder, from a snapshot of the buffers taken before any write."""
    n = int(step.reshape(-1)[0]) + int(step_offset)
    par, div = parent.cpu().tolist(), diverge.cpu().tolist()
    par = [pa + (a // k) * k for a, pa in enumerate(par)]            # parent slots as sequence indices
    for kb, vb, ks, vs, base, window, heavy in items:
        B, H = kb.shape[:2]
        rows = OB.reorder_rows(n, par, div, window, heavy is not None)
        planes = [t for t in (kb, vb, ks, vs) if t is not None]
        snap = [t.clone() for t in planes]
        bs = base.reshape(B, H).cpu()
        for a in range(B):
            if not rows[a]:
                continue
            src = par[a]
            for h in range(H):
                dst_rows = [int(bs[a, h]) + s for s in rows[a]]
                src_rows = [int(bs[src, h]) + s for s in rows[a]]
                for t, c in zip(planes, snap):
                    t[a, h, dst_rows] = c[src, h, src_rows]
        if heavy is not None:
            hsnap = [t.clone() for t in heavy]
            for a in range(B):
                if par[a] != a:
                    src = par[a]
                    heavy[0][a] = hsnap[0][src]
                    heavy[1][a] = hsnap[1][src]
                    heavy[2].view(B, H)[a] = hsnap[2].view(B, H)[src]


class OracleBeamBackend(OracleHeavyBackend):
    name = "oracle-cpu beam search (tests only)"

    def beam_candidates(self, logits, st):
        candidates_twin(logits, st)

    def beam_step(self, st, rows_per_prompt, step, step_offset):
        step_twin(st, rows_per_prompt, step, step_offset)

    def cache_reorder(self, items, P, k, parent, diverge, step, step_offset):
        reorder_twin(items, P, k, parent, diverge, step, step_offset)


def gather_reorder(batch, num_prompts, num_beams, parent, diverge, step, step_offset, backend=None):
    """The reference reorder: every beam slot whose parent is another slot takes all of that slot's generated rows (every
    row past its prompt; under a decode window the whole ring), their scales, and with heavy hitters the slot's whole
    heavy-hitter state, by torch indexing from a snapshot. Rows are found from the host counts of each layer (the prompt
    rows, which the static loop does not advance), not from the tables the kernel reads."""
    n = int(step.reshape(-1)[0]) + int(step_offset)
    k = int(num_beams)
    src = [p + (a // k) * k for a, p in enumerate(parent.cpu().tolist())]
    for l in batch.layers:
        B, H = l.k_buf.shape[:2]
        prompt = l.prompt_rows_host if l.window is not None else l.rows_host
        m = n if l.window is None else min(n, l.window)
        bufs = [getattr(l, name) for name in l._BUFFERS]
        snap = [t.clone() for t in bufs]
        for b in range(B):
            if src[b] == b:
                continue
            for h in range(H):
                p0 = int(prompt[b][h])
                assert int(prompt[src[b]][h]) == p0      # the beams of a prompt share its prompt rows
                for t, c in zip(bufs, snap):
                    t[b, h, p0:p0 + m] = c[src[b], h, p0:p0 + m]
        if l.heavy is not None:
            hs = [l.heavy_scores, l.heavy_gen, l.victim.view(B, H)]
            hsnap = [t.clone() for t in hs]
            for b in range(B):
                if src[b] != b:
                    for t, c in zip(hs, hsnap):
                        t[b] = c[src[b]]
