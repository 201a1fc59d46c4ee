"""TEST-ONLY backend for the generation constraints: the penalized-sampling oracle backend (every cache form, the decode
window included) plus `token_rules` and `sample_tokens_constrained`, the CPU twins of `pkv_token_rules` and
`pkv_sample_tokens_constrained` (include/pkv.h, DESIGN.md §4.11). The twins unpack generate.SamplingState's device tables
and apply oracle/constraints.py, so the packing is checked along with the rules. Never importable from product code."""
import numpy as np
import torch

import oracle_penalty_backend as OP
from oracle import constraints as OC
from oracle_penalty_backend import OraclePenaltyBackend
from pyramidkv_b200 import _lib


def unpack_row(params, b):
    """Row b of the state: (history, prompt_len, flags, ngram, min_new, [(tokens, kind, bias)], eos)."""
    n = int(params.history_len[b])
    hist = params.history[b, :n].tolist()
    off = params.seq_off[b].tolist()
    tok = params.seq_tokens[b].tolist()
    seqs = [(tuple(tok[off[j]:off[j + 1]]), int(params.seq_kind[b, j]), float(params.seq_bias[b, j]))
            for j in range(int(params.n_seq[b]))]
    eos = params.eos[: int(params.n_eos)].tolist()
    return hist, int(params.prompt_len[b]), int(params.rule_flags[b]), int(params.ngram[b]), int(params.min_new[b]), seqs, eos


def row_terms(hist, prompt_len, flags, ngram, min_new, seqs, eos, vocab):
    """pkv_token_rules' outputs for one row: bias (fp32 [V]), set-ban and add-ban (bool [V]), stop."""
    bias = np.zeros(vocab, np.float32)
    if flags & _lib.RULE_BIAS:
        bias = OC.sequence_bias(hist, [(s, w) for s, k, w in seqs if k == _lib.SEQ_BIAS], vocab)
    set_ban = np.zeros(vocab, bool)
    if flags & _lib.RULE_BAN:
        set_ban = OC.ngram_bans(hist, ngram, vocab) | OC.min_new_bans(hist, prompt_len, min_new, eos, vocab)
    add_ban = np.zeros(vocab, bool)
    if flags & _lib.RULE_BAD:
        add_ban = OC.bad_word_bans(hist, [s for s, k, _ in seqs if k == _lib.SEQ_BAD], (), vocab)
    stop = bool(flags & _lib.RULE_STOP) and OC.stopped(hist, [s for s, k, _ in seqs if k == _lib.SEQ_STOP])
    return bias, set_ban, add_ban, stop


def pack_bits(ban) -> np.ndarray:
    """bool [V] -> the int32 words of pkv_token_rules (bit v of word v >> 5)."""
    V = ban.shape[0]
    W = (V + 31) // 32
    b = np.zeros(W * 32, np.uint64)
    b[:V] = ban
    words = (b.reshape(W, 32) << np.arange(32, dtype=np.uint64)).sum(axis=1).astype(np.uint32)
    return words.view(np.int32)


def token_rules_twin(params, vocab, append=None, col=0):
    B = params.history.shape[0]
    W = (vocab + 31) // 32
    for b in range(B):
        if append is not None:
            n = int(params.history_len[b])
            if n < params.history.shape[1]:
                params.history[b, n] = int(append[b, col])
                params.history_len[b] = n + 1
        hist, plen, flags, ngram, min_new, seqs, eos = unpack_row(params, b)
        bias, set_ban, add_ban, stop = row_terms(hist, plen, flags, ngram, min_new, seqs, eos, vocab)
        if flags & _lib.RULE_BIAS:
            params.bias[b, :vocab] = torch.from_numpy(bias)
        if flags & (_lib.RULE_BAN | _lib.RULE_BAD):
            params.ban[b, :W] = torch.from_numpy(pack_bits(set_ban))
            params.ban[b, W:2 * W] = torch.from_numpy(pack_bits(add_ban))
        params.stop[b, 0] = stop


def _bits(words, vocab) -> np.ndarray:
    w = np.asarray(words).view(np.uint32).astype(np.uint64)
    return ((w[:, None] >> np.arange(32, dtype=np.uint64)) & 1).reshape(-1)[:vocab].astype(bool)


def constrained_x(logits_row, flags, bias, ban_words, repetition, presence, frequency, mask, counts) -> np.ndarray:
    """x of pkv_sample_tokens_constrained for one row: bias, penalties, bans."""
    V = logits_row.shape[0]
    W = (V + 31) // 32
    x = np.asarray(logits_row, np.float32)
    if flags & _lib.RULE_BIAS:
        x = OC.add_bias(x, np.asarray(bias[:V], np.float32))
    x = OP.penalize(x, repetition, presence, frequency, mask, counts)
    set_ban = _bits(ban_words[:W], V) if flags & _lib.RULE_BAN else np.zeros(V, bool)
    add_ban = _bits(ban_words[W:2 * W], V) if flags & _lib.RULE_BAD else None
    return OC.apply_bans(x, set_ban, add_ban)


def sample_constrained_twin(logits, params, out, col, advance=True):
    if logits.dtype not in (torch.bfloat16, torch.float16):
        raise NotImplementedError(f"sample_tokens_constrained: bf16 / fp16 logits, got {logits.dtype}")
    rows = logits.detach().float().cpu().numpy()
    V = rows.shape[1]
    mask = params.prompt_mask.cpu().numpy()
    counts = params.counts.cpu().numpy()
    bias = params.bias.cpu().numpy()
    ban = params.ban.cpu().numpy()
    for b in range(rows.shape[0]):
        rho, pres, freq, mp = (float(params.repetition_penalty[b]), float(params.presence_penalty[b]),
                               float(params.frequency_penalty[b]), float(params.min_p[b]))
        if not OP.params_valid(rho, pres, freq, mp):
            tok = -1
        else:
            x = constrained_x(rows[b], int(params.rule_flags[b]) & 7, bias[b], ban[b], rho, pres, freq, mask[b, :V],
                              counts[b, :V])
            tok = OP.sample_row_penalized(x, float(params.temperature[b]), int(params.top_k[b]), float(params.top_p[b]),
                                          int(params.seed[b]) % 2 ** 64, int(params.index[b]), 1.0, 0.0, 0.0, mp).token
        out[b, col] = tok
        if advance and tok >= 0:
            params.counts[b, tok] += 1
    if advance:
        params.index.add_(1)


class OracleConstraintBackend(OraclePenaltyBackend):
    name = "oracle-cpu constrained sampling (tests only)"

    def token_rules(self, params, vocab, append=None, col=0):
        token_rules_twin(params, vocab, append, col)

    def sample_tokens_constrained(self, logits, params, out, col, advance=True):
        sample_constrained_twin(logits, params, out, col, advance)

