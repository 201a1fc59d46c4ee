"""The generate loop on the far side of the eviction path (SURVEY.md §8 row f3).

The reference decodes through HF `generate`: per token and layer a `torch.cat` of the whole layer cache
(cache_utils_think.py:383-384), two transposes, one attention launch (llama_model.py:401-445), `position_ids` rebuilt
from the attention mask (llama_model.py:2617-2631) and ~1 000 host-launched kernels — launch-bound by a wide margin.
Here the compacted cache is pre-reserved for the whole generation, the number of rows is a DEVICE counter
(`pkv_decode_attn_graph`), and one greedy step (embedding -> every decoder layer through the patched attention forward
-> norm -> lm_head -> argmax -> token/position/step bookkeeping) is a fixed sequence of launches with fixed arguments:
it is captured once in a CUDA graph and replayed per token. The host only reads the tokens back at the end.

`greedy_generate` is the drop-in for `model.generate(ids, max_new_tokens=N, num_beams=1, do_sample=False)`
(run_longbench.py:264-275): same tokens as HF's greedy loop through the same patched forward (tests/test_generate.py,
CPU, eager mode with the test backend; `-m gpu`: graph vs eager vs HF generate).

`greedy_generate_batch` decodes several prompts of any lengths together: each is prefilled alone (the same prefill as
`greedy_generate`), their compacted caches are joined (`cache.join_caches`) and one step decodes all of them - one graph
replay per token, one attention launch per layer (`pkv_decode_attn_batch`) - so the weights are streamed once per step for
the whole batch instead of once per sequence.

With `model.config.pkv_kv_cache_dtype = "fp8_e4m3"` the prefill leaves FP8 caches (`cache.PkvFp8CacheLayer`); all three loops
take them as they are (the knob is the single source: no parameter here), one `pkv_decode_attn_batch_fp8` launch per layer.
Likewise with `model.config.pkv_gqa_shared = True` (one cache per KV head, `group` > 1): one `pkv_decode_attn_batch_gqa(_fp8)`
launch per layer.

`greedy_generate_continuous` keeps a fixed number of slots busy: when a sequence stops (EOS or its own `max_new_tokens`),
the next waiting prompt is prefilled and copied into its slot in place (`pkv_cache_install`, one launch for every layer),
while the captured step graph keeps replaying unchanged.

All three loops are greedy by default. `sampling=SamplingParams(...)` (or one per prompt) draws each token instead - the
prefill's with token index t = 0, decode step n's with t = n - with temperature, top-k, top-p and a per-request seed, one
`pkv_sample_tokens` launch per step for the whole batch in place of the argmax (DESIGN.md §4.6). A request's tokens depend
only on its logits, its parameters and its seed, not on its batch position, slot or the graph. Its repetition, presence and
frequency penalties and min-p (HF's RepetitionPenaltyLogitsProcessor and MinPLogitsWarper, vLLM's presence / frequency
penalties) are applied on the device from a per-row prompt mask and generated-token count table, in one
`pkv_sample_tokens_penalized` launch per step instead (DESIGN.md §4.10); `SamplingParams(temperature=0,
repetition_penalty=r)` is HF's `generate(do_sample=False, repetition_penalty=r)`. Its generation constraints (sequence
bias, no-repeat n-grams, bad words, min_new_tokens and stop sequences: HF's SequenceBias, NoRepeatNGram, NoBadWords and
MinNewTokensLength processors and a stopping criterion over the ids) read each row's token history on the device - its
whole prompt, however much of it the compacted cache keeps, then every generated token - through one `pkv_token_rules`
launch after each draw and one `pkv_sample_tokens_constrained` launch in place of the penalized one (DESIGN.md §4.11). A
sequence that completes a stop sequence ends there like one that emitted EOS.

`logprobs=N` (0 to 20) in any of the three loops also returns one `TokenLogprobs` per prompt: the log-probability of every
generated token and the N most likely tokens at each position, under the model's raw distribution (log_softmax of the
logits, whatever the sampling parameters), from one `pkv_token_logprobs` launch per step after the argmax or the draw
(DESIGN.md §4.8). `score_continuations` forces given continuations through the same step and returns their
log-probabilities over the compacted cache: the likelihood a cache form gives a fixed text.

`beam_search_generate` is HF's `generate(num_beams=k, do_sample=False)`: each prompt is prefilled once, its cache joined k
times, and every beam of every prompt decodes in lock-step in `StaticDecoder`, whose beam mode replaces the argmax by three
launches (`pkv_beam_candidates`, `pkv_beam_step`, `pkv_cache_reorder`: DESIGN.md §4.12).
"""
from __future__ import annotations

import math
import operator
import time
from dataclasses import dataclass
from typing import List, Optional

import torch

from .cache import PkvBatchCacheLayer, PkvCacheLayer, admit_cache, join_caches, park_cache, reorder_caches


@dataclass(frozen=True)
class SamplingParams:
    """One request's sampling settings, applied in HF's order: repetition penalty, temperature, top-k, top-p, min-p, then
    the draw. temperature 0 or top_k 1: the greedy token (of the penalized logits). top_k 0 and top_p 1 switch those filters
    off. The temperature is used as an fp32 value; the 64-bit seed and the token index key the Philox stream of the
    Gumbel-max draw (DESIGN.md §4.6). repetition_penalty (> 0; 1: off) divides the positive and multiplies the negative
    logits of the prompt's and the generated tokens; presence_penalty and frequency_penalty (0: off) subtract, from each
    generated token's logit, the penalty and the penalty times its count (vLLM's order, after the repetition penalty); min_p
    (in [0, 1]; 0: off) drops the tokens whose probability is below min_p times the largest (DESIGN.md §4.10).
    The constraints (DESIGN.md §4.11; every default leaves its rule off) come first, in HF's order around the penalties:
    sequence_bias ((token-id tuple, bias) pairs), no_repeat_ngram_size, bad_words_ids (token-id tuples), min_new_tokens
    (EOS is banned until that many tokens are generated), and stop_sequences (token-id tuples: the sequence ends with the
    token that completes one, kept). Lists are frozen to tuples."""
    temperature: float = 1.0
    top_k: int = 0
    top_p: float = 1.0
    seed: int = 0
    repetition_penalty: float = 1.0
    presence_penalty: float = 0.0
    frequency_penalty: float = 0.0
    min_p: float = 0.0
    sequence_bias: tuple = ()
    no_repeat_ngram_size: int = 0
    bad_words_ids: tuple = ()
    min_new_tokens: int = 0
    stop_sequences: tuple = ()

    def __post_init__(self):
        if not float(self.temperature) >= 0.0:
            raise ValueError(f"SamplingParams: temperature must be >= 0, got {self.temperature}")
        if int(self.top_k) != self.top_k or int(self.top_k) < 0:
            raise ValueError(f"SamplingParams: top_k must be an integer >= 0, got {self.top_k}")
        if not 0.0 < float(self.top_p) <= 1.0:
            raise ValueError(f"SamplingParams: top_p must be in (0, 1], got {self.top_p}")
        if int(self.seed) != self.seed or not 0 <= int(self.seed) < 2 ** 64:
            raise ValueError(f"SamplingParams: seed must be an integer in [0, 2^64), got {self.seed}")
        if not 0.0 < float(self.repetition_penalty) < math.inf:
            raise ValueError(f"SamplingParams: repetition_penalty must be finite and > 0, got {self.repetition_penalty}")
        for name in ("presence_penalty", "frequency_penalty"):
            if not math.isfinite(float(getattr(self, name))):
                raise ValueError(f"SamplingParams: {name} must be finite, got {getattr(self, name)}")
        if not 0.0 <= float(self.min_p) <= 1.0:
            raise ValueError(f"SamplingParams: min_p must be in [0, 1], got {self.min_p}")
        bias = []
        for pair in self.sequence_bias:
            if len(pair) != 2:
                raise ValueError(f"SamplingParams: sequence_bias takes (token ids, bias) pairs, got {pair!r}")
            ids, w = _token_ids(pair[0], "sequence_bias"), _finite(pair[1])
            if w is None:
                raise ValueError(f"SamplingParams: sequence_bias values must be finite numbers, got {pair[1]!r}")
            if any(ids == b[0] for b in bias):
                raise ValueError(f"SamplingParams: sequence_bias repeats the sequence {ids}")
            bias.append((ids, w))
        object.__setattr__(self, "sequence_bias", tuple(bias))
        for name in ("bad_words_ids", "stop_sequences"):
            object.__setattr__(self, name, tuple(_token_ids(s, name) for s in getattr(self, name)))
        for name in ("no_repeat_ngram_size", "min_new_tokens"):
            v = getattr(self, name)
            if isinstance(v, bool) or int(v) != v or int(v) < 0:
                raise ValueError(f"SamplingParams: {name} must be an integer >= 0, got {v!r}")
            object.__setattr__(self, name, int(v))

    @property
    def penalized(self) -> bool:
        """Some penalty or min-p is on: the draw needs the request's prompt and generated tokens."""
        return (float(self.repetition_penalty) != 1.0 or float(self.presence_penalty) != 0.0
                or float(self.frequency_penalty) != 0.0 or float(self.min_p) != 0.0)

    @property
    def constrained(self) -> bool:
        """Some generation constraint is on: the draw needs the request's token history."""
        return bool(self.sequence_bias or self.no_repeat_ngram_size or self.bad_words_ids or self.min_new_tokens
                    or self.stop_sequences)


def _finite(w) -> Optional[float]:
    """A bias value as a Python float (numpy scalars and 0-d tensors included), or None when it is not a finite number."""
    if isinstance(w, (bool, str, bytes)):
        return None
    try:
        v = float(w)
    except (TypeError, ValueError):
        return None
    return v if math.isfinite(v) else None


def _token_ids(seq, what: str) -> tuple:
    """A sequence of token ids (Python or numpy integers, integer tensors) as a tuple of Python ints."""
    err = ValueError(f"SamplingParams: every {what} sequence must be a non-empty sequence of token ids >= 0, got {seq!r}")
    if isinstance(seq, (str, bytes)):
        raise err
    try:
        items = list(seq)
    except TypeError:
        raise err from None
    ids = []
    for t in items:
        if isinstance(t, bool):
            raise err
        try:
            v = operator.index(t)
        except TypeError:
            raise err from None
        if v < 0:
            raise err
        ids.append(v)
    if not ids:
        raise err
    return tuple(ids)


class _StopTail:
    """The host's stop check of one sequence: `push` each generated token (the prefill's first) and it tells whether the
    sequence ends there, at an EOS id or at the last token of one of `p`'s stop sequences. It keeps the sequence's last
    tokens, prompt included, as many as its longest stop sequence: a stop sequence may start inside the prompt."""

    def __init__(self, prompt: torch.Tensor, eos: set, p: Optional[SamplingParams]):
        self.eos = eos
        self.stops = () if p is None else p.stop_sequences
        self.k = max((len(q) for q in self.stops), default=0)
        self.tail = prompt.reshape(-1)[-self.k:].tolist() if self.k else []

    def push(self, token) -> bool:
        t = int(token)
        if self.k:
            self.tail.append(t)
            del self.tail[: -self.k]
        return t in self.eos or any(tuple(self.tail[len(self.tail) - len(q):]) == q for q in self.stops
                                    if len(q) <= len(self.tail))


def _rule_tables(p: SamplingParams, eos: set):
    """One request's rules as pkv_token_rules reads them: (flags, n-gram size, min_new_tokens, [(tokens, kind, bias)]).
    Bias sequences are grouped by their last token (the single-token one first, then in the request's order: the order of
    HF's sums); single-token bad words equal to an EOS id are dropped, and min_new_tokens needs an EOS id, as in HF."""
    from . import _lib
    bias = sorted(((s, w) for s, w in p.sequence_bias), key=lambda sw: (sw[0][-1], len(sw[0]) != 1))
    bad = [s for s in p.bad_words_ids if not (len(s) == 1 and s[0] in eos)]
    min_new = p.min_new_tokens if eos else 0
    seqs = ([(s, _lib.SEQ_BIAS, w) for s, w in bias] + [(s, _lib.SEQ_BAD, 0.0) for s in bad]
            + [(s, _lib.SEQ_STOP, 0.0) for s in p.stop_sequences])
    flags = ((_lib.RULE_BIAS if bias else 0) | (_lib.RULE_BAN if p.no_repeat_ngram_size or min_new else 0)
             | (_lib.RULE_BAD if bad else 0) | (_lib.RULE_STOP if p.stop_sequences else 0))
    return flags, p.no_repeat_ngram_size, min_new, seqs


def _seed_i64(seed: int) -> int:
    seed = int(seed)
    return seed - 2 ** 64 if seed >= 2 ** 63 else seed      # the same 64 bits in an int64 tensor


EARLY_STOPPING = {False: 0, True: 1, "never": 2}   # pkv_beam_step_desc.early_stopping
MAX_BEAMS = 16


def beam_divisors(max_steps: int, length_penalty: float, early_stopping) -> list:
    """HF's length-penalty divisors per iteration t, as the Python floats it divides by: the pool's (t + 1)^lp and the
    heuristic's L^lp (L = max_steps when early_stopping is "never" and lp > 0, else t + 1)."""
    return [((t + 1) ** length_penalty,
             (max_steps if early_stopping == "never" and length_penalty > 0.0 else t + 1) ** length_penalty)
            for t in range(max_steps)]


_PENALTY_FIELDS = ("repetition_penalty", "presence_penalty", "frequency_penalty", "min_p")


class SamplingState:
    """The per-row device state `sample_tokens` reads: parameters and the token index of each row (sequence or slot).
    Rows are rewritten in place (`set_row`), so a captured graph keeps its pointers.

    With penalties (some request sets one, or `penalties=True` for rows that may later take such a request), also the
    state `sample_tokens_penalized` reads: the four penalty parameters per row, the prompt mask (uint8 [B, vocab]) and the
    generated-token counts (int32 [B, vocab]), built from `prompts` (one id tensor per row) and `first` (each row's token
    drawn so far, counted once; None: nothing generated yet). B * vocab * 5 bytes, allocated only then.

    With constraints (some request sets one, or `constraints=True`), also the state of `token_rules` and
    `sample_tokens_constrained` (it implies the penalty state): each row's token history (int32 [B, cap]: the prompt, then
    `first`, then one token per `rules(append=...)`; `history` reserves cap >= the longest prompt + `history` tokens), its
    rules packed into flat tables, the `eos` ids the rules use, and their per-step outputs: bias (float32 [B, vocab]), the
    two ban bitmaps (int32 [B, 2 * ceil(vocab / 32)]) and the stop flags (bool [B, 1]). `rules` must run once before the
    first constrained draw (the decoders and the prefill do)."""

    def __init__(self, params: List[SamplingParams], device, index: int = 0, vocab: Optional[int] = None, prompts=None,
                 first: Optional[torch.Tensor] = None, penalties: bool = False, constraints: bool = False, eos=None,
                 history: int = 0):
        self.temperature = torch.tensor([float(p.temperature) for p in params], dtype=torch.float32, device=device)
        self.top_k = torch.tensor([min(int(p.top_k), 2 ** 31 - 1) for p in params], dtype=torch.int32, device=device)
        self.top_p = torch.tensor([float(p.top_p) for p in params], dtype=torch.float32, device=device)
        self.seed = torch.tensor([_seed_i64(p.seed) for p in params], dtype=torch.int64, device=device)
        self.index = torch.full((len(params),), int(index), dtype=torch.int64, device=device)
        self.constrained = bool(constraints) or any(p.constrained for p in params)
        self.penalized = bool(penalties) or self.constrained or any(p.penalized for p in params)
        if not self.penalized:
            return
        if vocab is None or prompts is None or len(prompts) != len(params):
            raise ValueError("SamplingState: penalties need the vocabulary size and one prompt per row")
        for name in _PENALTY_FIELDS:
            setattr(self, name, torch.tensor([float(getattr(p, name)) for p in params], dtype=torch.float32, device=device))
        self.prompt_mask = torch.zeros(len(params), int(vocab), dtype=torch.uint8, device=device)
        self.counts = torch.zeros(len(params), int(vocab), dtype=torch.int32, device=device)
        for row, ids in enumerate(prompts):
            self._set_history(row, ids, None if first is None else first.reshape(-1)[row])
        if not self.constrained:
            return
        B, V = len(params), int(vocab)
        self.vocab = V
        self.rule_eos = _eos_set(eos)
        self.eos = torch.tensor(sorted(self.rule_eos) or [0], dtype=torch.int32, device=device)
        self.n_eos = len(self.rule_eos)
        cap = max(int(torch.as_tensor(ids).numel()) for ids in prompts) + (first is not None) + int(history)
        self.history = torch.zeros(B, max(1, cap), dtype=torch.int32, device=device)
        for name in ("history_len", "prompt_len", "rule_flags", "ngram", "min_new", "n_seq"):
            setattr(self, name, torch.zeros(B, dtype=torch.int32, device=device))
        self.seq_off = torch.zeros(B, 2, dtype=torch.int32, device=device)
        self.seq_kind = torch.zeros(B, 2, dtype=torch.int32, device=device)
        self.seq_bias = torch.zeros(B, 2, dtype=torch.float32, device=device)
        self.seq_tokens = torch.zeros(B, 1, dtype=torch.int32, device=device)
        self.bias = torch.zeros(B, V, dtype=torch.float32, device=device)
        self.ban = torch.zeros(B, 2 * ((V + 31) // 32), dtype=torch.int32, device=device)
        self.stop = torch.zeros(B, 1, dtype=torch.bool, device=device)
        for row, (p, ids) in enumerate(zip(params, prompts)):
            self._set_rules(row, p, ids, None if first is None else first.reshape(-1)[row])

    def _check_ids(self, p: SamplingParams, prompt) -> None:
        """Every id of `prompt` and of `p`'s rule sequences is in [0, vocab)."""
        V = self.counts.shape[1]
        ids = torch.as_tensor(prompt).reshape(-1)
        if ids.numel() and (int(ids.min()) < 0 or int(ids.max()) >= V):
            raise ValueError(f"SamplingState: prompt ids outside [0, {V})")
        rules = [s for s, _ in p.sequence_bias] + list(p.bad_words_ids) + list(p.stop_sequences)
        if any(max(s) >= V for s in rules):
            raise ValueError(f"SamplingState: rule token ids outside [0, {V})")

    def _grow(self, name: str, cols: int) -> bool:
        t = getattr(self, name)
        if t.shape[1] >= cols:
            return False
        new = torch.zeros(t.shape[0], max(cols, 2 * t.shape[1]), dtype=t.dtype, device=t.device)
        new[:, : t.shape[1]] = t
        setattr(self, name, new)
        return True

    def _set_rules(self, row: int, p: SamplingParams, prompt, first) -> bool:
        """Row `row`'s history (prompt, then `first`) and packed rules; True when a table was reallocated."""
        flags, ngram, min_new, seqs = _rule_tables(p, self.rule_eos)
        self._check_ids(p, prompt)
        hist = torch.as_tensor(prompt).reshape(-1).to(torch.int32)
        n_prompt = hist.numel()
        if first is not None:
            hist = torch.cat([hist, torch.as_tensor(first).reshape(1).to(device=hist.device, dtype=torch.int32)])
        toks = [t for s, _, _ in seqs for t in s]
        off = [0]
        for s, _, _ in seqs:
            off.append(off[-1] + len(s))
        grew = self._grow("history", hist.numel())
        grew |= self._grow("seq_tokens", max(1, len(toks)))
        for name in ("seq_off", "seq_kind", "seq_bias"):
            grew |= self._grow(name, len(seqs) + 1)
        dev = self.history.device
        self.history[row].zero_()
        self.history[row, : hist.numel()] = hist.to(dev)
        self.history_len[row] = hist.numel()
        self.prompt_len[row] = n_prompt
        self.rule_flags[row] = flags
        self.ngram[row] = ngram
        self.min_new[row] = min_new
        self.n_seq[row] = len(seqs)
        self.seq_off[row, : len(off)] = torch.tensor(off, dtype=torch.int32, device=dev)
        if seqs:
            self.seq_kind[row, : len(seqs)] = torch.tensor([k for _, k, _ in seqs], dtype=torch.int32, device=dev)
            self.seq_bias[row, : len(seqs)] = torch.tensor([w for _, _, w in seqs], dtype=torch.float32, device=dev)
            self.seq_tokens[row, : len(toks)] = torch.tensor(toks, dtype=torch.int32, device=dev)
        return grew

    def rules(self, backend, append: Optional[torch.Tensor] = None) -> None:
        """One `token_rules` launch for every row: with `append` ([B, 1] int64), each row's history takes its token
        first; then the bias, bans and stop flags of the next draw."""
        backend.token_rules(self, self.vocab, append, 0)

    def rule_state(self) -> list:
        """The device tensors `rules(append=...)` advances (restored after the warm-up step of a graph capture)."""
        return [self.history_len, self.bias, self.ban, self.stop] if self.constrained else []

    def _set_history(self, row: int, prompt: torch.Tensor, first: Optional[torch.Tensor]) -> None:
        ids = torch.as_tensor(prompt).reshape(-1).to(device=self.counts.device, dtype=torch.long)
        V = self.counts.shape[1]
        if ids.numel() and (int(ids.min()) < 0 or int(ids.max()) >= V):
            raise ValueError(f"SamplingState: prompt ids outside [0, {V})")
        self.prompt_mask[row].zero_()
        self.prompt_mask[row].index_fill_(0, ids, 1)
        self.counts[row].zero_()
        if first is not None:
            self.counts[row].index_fill_(0, torch.as_tensor(first).reshape(1).to(device=self.counts.device, dtype=torch.long), 1)

    def set_row(self, row: int, p: SamplingParams, index: int, prompt=None, first: Optional[torch.Tensor] = None,
                history: int = 0) -> bool:
        """Row `row` takes the parameters `p` at token index `index`; with penalties, its prompt mask becomes `prompt`'s
        ids and its counts count `first` (the token drawn so far) once; with constraints, its history becomes `prompt` +
        `first` with room for `history` more tokens, and its rules `p`'s. True when a constraint table was reallocated
        (a captured graph then holds stale pointers); `rules` must run before the row's next draw."""
        if p.penalized and not self.penalized:
            raise ValueError("SamplingState.set_row: a request with penalties or min-p needs a state built with penalties")
        if p.constrained and not self.constrained:
            raise ValueError("SamplingState.set_row: a request with constraints needs a state built with constraints")
        if self.penalized and prompt is None:
            raise ValueError("SamplingState.set_row: a state with penalties needs the row's prompt ids")
        if self.penalized:
            self._check_ids(p, prompt)                 # before any of the row's state changes
        self.temperature[row] = float(p.temperature)
        self.top_k[row] = min(int(p.top_k), 2 ** 31 - 1)
        self.top_p[row] = float(p.top_p)
        self.seed[row] = _seed_i64(p.seed)
        self.index[row] = int(index)
        grew = False
        if self.penalized:
            for name in _PENALTY_FIELDS:
                getattr(self, name)[row] = float(getattr(p, name))
            self._set_history(row, prompt, first)
        if self.constrained:
            grew = self._grow("history", torch.as_tensor(prompt).numel() + (first is not None) + int(history))
            grew |= self._set_rules(row, p, prompt, first)
        return grew

    def draw(self, backend, logits, out, col, advance=True) -> None:
        """One launch for every row: `sample_tokens`, or `sample_tokens_penalized` when the state has penalties, or
        `sample_tokens_constrained` when it has constraints."""
        if self.constrained:
            backend.sample_tokens_constrained(logits, self, out, col, advance)
        elif self.penalized:
            backend.sample_tokens_penalized(logits, self, out, col, advance)
        else:
            backend.sample_tokens(logits, self, out, col, advance)


def _sampling_list(sampling, n: int, what: str):
    """None, one SamplingParams for every prompt, or one per prompt -> None or a list of n."""
    if sampling is None:
        return None
    if isinstance(sampling, SamplingParams):
        return [sampling] * n
    out = list(sampling)
    if len(out) != n or not all(isinstance(p, SamplingParams) for p in out):
        raise ValueError(f"{what}: sampling must be a SamplingParams or one per prompt ({n})")
    return out


class BeamState:
    """The device state of beam search over P prompts of k beams (include/pkv.h: pkv_beam_step; DESIGN.md §4.12): each
    beam row's candidates (m, log Z, top K ids and log-probabilities, K = max(2, 1 + n_eos) * k), the running scores,
    the finished pool (score, (step, parent, token) handle, finished flag), the early-stop heuristic and done flag of each
    prompt, the backpointers [P*k, max_steps] the host rebuilds hypotheses from, the common-prefix matrix [P, k, k] and
    the step's outputs: next token, parent slot and divergence row of each beam. Every tensor is written in place, so a
    captured decode graph keeps its pointers. `scale` [max_steps, 2] holds f32(1 / d) of HF's length-penalty divisors d:
    torch's CUDA division of an fp32 tensor by a Python float d multiplies by that; `divisors` the Python floats d."""

    def __init__(self, P: int, k: int, max_steps: int, eos, length_penalty: float, early_stopping, device):
        self.P, self.k, self.max_steps = int(P), int(k), int(max_steps)
        self.eos = sorted(_eos_set(eos))
        self.n_eos = len(self.eos)
        self.K = max(2, 1 + self.n_eos) * self.k
        self.early_stopping = EARLY_STOPPING[early_stopping]
        self.divisors = beam_divisors(self.max_steps, float(length_penalty), early_stopping)
        B, dev = self.P * self.k, device
        i32 = dict(dtype=torch.int32, device=dev)
        self.scale = torch.tensor([[1.0 / d for d in row] for row in self.divisors], dtype=torch.float32, device=dev)
        self.eos_dev = torch.tensor(self.eos or [0], **i32)
        self.m = torch.zeros(B, dtype=torch.float32, device=dev)
        self.log_z = torch.zeros(B, dtype=torch.float32, device=dev)
        self.cand_lp = torch.zeros(B, self.K, dtype=torch.float32, device=dev)
        self.cand_id = torch.zeros(B, self.K, **i32)
        self.running = torch.full((self.P, self.k), -1e9, dtype=torch.float32, device=dev)
        self.running[:, 0] = 0.0
        self.running = self.running.reshape(B)
        self.pool_score = torch.full((B,), -1e9, dtype=torch.float32, device=dev)
        self.pool_step = torch.full((B,), -1, **i32)
        self.pool_parent = torch.zeros(B, **i32)
        self.pool_token = torch.zeros(B, **i32)
        self.pool_done = torch.zeros(B, dtype=torch.uint8, device=dev)
        self.heuristic = torch.ones(self.P, dtype=torch.uint8, device=dev)
        self.done = torch.zeros(self.P, dtype=torch.uint8, device=dev)
        self.bp_token = torch.zeros(B, self.max_steps, **i32)
        self.bp_parent = torch.zeros(B, self.max_steps, **i32)
        self.cp = torch.zeros(self.P, self.k, self.k, **i32)
        self.next_token = torch.zeros(B, dtype=torch.long, device=dev)
        self.parent = torch.arange(B, **i32) % self.k
        self.diverge = torch.zeros(B, **i32)

    def state(self) -> list:
        """The tensors a step reads and advances (restored after the warm-up step of a graph capture)."""
        return [self.running, self.pool_score, self.pool_step, self.pool_parent, self.pool_token, self.pool_done,
                self.heuristic, self.done, self.bp_token, self.bp_parent, self.cp]

    def step(self, backend, logits, rows_per_prompt: int, step: torch.Tensor, step_offset: int) -> None:
        """Candidates of `logits` (one row per beam, or with rows_per_prompt = 1 one per prompt) and one beam step at
        iteration *step + step_offset: two launches."""
        backend.beam_candidates(logits, self)
        backend.beam_step(self, rows_per_prompt, step, step_offset)

    def hypotheses(self, n: int) -> list:
        """Per prompt, its best n pool entries (best first): (generated tokens, fp32 score)."""
        tok, par = self.bp_token.cpu().numpy(), self.bp_parent.cpu().numpy()
        score = self.pool_score.cpu()
        handles = torch.stack([self.pool_step, self.pool_parent, self.pool_token]).cpu().T.tolist()
        out = []
        for p in range(self.P):
            bk = p * self.k
            hyps = []
            for j in range(n):
                t, r, v = handles[bk + j]
                seq = [int(v)]
                for s in range(t - 1, -1, -1):     # back through the slots' backpointers
                    seq.append(int(tok[bk + r, s]))
                    r = int(par[bk + r, s])
                hyps.append((seq[::-1] if t >= 0 else [], score[bk + j].clone()))
            out.append(hyps)
        return out


@dataclass
class TokenLogprobs:
    """Log-probabilities of one sequence's tokens (host tensors, n tokens, N = the `logprobs` / `top_n` asked for), under
    the model's raw distribution log_softmax(f32(logits)): temperature 1, no filters. token_ids [n] int64 (the generated or
    scored tokens), logprobs [n] float32, top_ids [n, N] int64 (logit descending, index ascending) and top_logprobs [n, N]
    float32. A position whose logits hold a NaN or +-inf has NaN log-probabilities and top ids -1."""
    token_ids: torch.Tensor
    logprobs: torch.Tensor
    top_ids: torch.Tensor
    top_logprobs: torch.Tensor


MAX_LOGPROBS = 20


def _check_logprobs(n, what: str) -> Optional[int]:
    if n is None:
        return None
    if isinstance(n, bool) or int(n) != n or not 0 <= int(n) <= MAX_LOGPROBS:
        raise ValueError(f"{what}: logprobs must be None or an integer in [0, {MAX_LOGPROBS}], got {n!r}")
    return int(n)


class _LogprobBuffers:
    """Static [B, n] / [B, n, N] buffers `token_logprobs` writes at a column (a device cursor in the decode step)."""

    def __init__(self, B: int, n: int, N: int, device):
        self.lp = torch.zeros(B, n, dtype=torch.float32, device=device)
        self.ids = torch.zeros(B, n, N, dtype=torch.long, device=device)
        self.top = torch.zeros(B, n, N, dtype=torch.float32, device=device)

    def write(self, backend, logits, tokens, cursor=None) -> None:
        backend.token_logprobs(logits, tokens, self.lp, self.ids, self.top, 0, 0, cursor)

    def host(self, steps: int):
        """Copies of the first `steps` columns on the host (the buffers are rewritten by the next chunk)."""
        return tuple(t[:, :steps].to("cpu", copy=True) for t in (self.lp, self.ids, self.top))


def _join_entries(tokens, parts) -> TokenLogprobs:
    """tokens: ids [n]; parts: (lp [k], ids [k, N], top [k, N]) host pieces in order, k summing to n."""
    return TokenLogprobs(torch.as_tensor(tokens, dtype=torch.long).reshape(-1), torch.cat([p[0] for p in parts]),
                         torch.cat([p[1] for p in parts]), torch.cat([p[2] for p in parts]))


def _backend(model):
    return model.model.layers[0].self_attn.kv_cluster.backend


@dataclass
class _StaticState:
    step: torch.Tensor        # int32 [1]: decode steps already taken in this static run (read by the decode kernel)
    workspace: torch.Tensor   # split-T partials, shared by all layers (launches are stream-ordered)
    heavy_scratch: Optional[torch.Tensor] = None   # knob pkv_decode_heavy: the per-step logits, shared by all layers
    spec: bool = False        # the verify step of speculative decoding: q_len > 1 goes through `decode_multi`
    pack: Optional["PackState"] = None   # ... or, in the continuous loop, over packed rows through `decode_packed`


class StaticDecoder:
    """Greedy decode over an already prefilled (and evicted) cache with a fixed per-step launch sequence.

    model: a patched LlamaForCausalLM / MistralForCausalLM; cache: the DynamicCache the patched prefill filled with
    PkvCacheLayer entries - one prompt, an equal-length batch prefilled as one forward, or prompts joined by
    `cache.join_caches`; first_token: the token the prefill produced per sequence ([B] or [B, 1] int64).
    eos_token_id (int or list): a sequence that produced one is done - it keeps decoding in lock-step, but its tokens are
    `pad_token_id` from then on (on the device: `done` [B]); None masks nothing. sampling: None (greedy: the argmax) or one
    SamplingParams per sequence, whose first decode step draws with token index 1 (the prefill's token is t = 0); with
    penalties or min-p, `prompts` gives each sequence's prompt ids (the first token counts as generated).
    logprobs: None, or N: each step also writes the log-probability of its token and the top N into `self.logprobs`
    (`_LogprobBuffers`, column = the step). forced: None, or int64 [B, max_steps]: step n takes forced[:, n] as its token
    instead of the argmax (teacher forcing; it is then the next step's input, and with `logprobs` the token scored). beam: None, or the
    `BeamState` of a cache joined num_beams times per prompt: each step's beam step (`pkv_beam_candidates`,
    `pkv_beam_step`) picks every beam's next token and parent in place of the argmax, and `pkv_cache_reorder` moves each
    beam's generated rows to its parent's (DESIGN.md §4.12)."""

    def __init__(self, model, cache, first_token: torch.Tensor, max_steps: int, use_graph: Optional[bool] = None,
                 eos_token_id=None, pad_token_id: int = 0, sampling: Optional[List[SamplingParams]] = None,
                 logprobs: Optional[int] = None, forced: Optional[torch.Tensor] = None, prompts=None,
                 beam: Optional["BeamState"] = None):
        layers = [l for l in cache.layers if isinstance(l, PkvCacheLayer)]
        if len(layers) != model.config.num_hidden_layers:
            raise RuntimeError("StaticDecoder needs a cache prefilled by the patched forward on every layer "
                               "(method 'fullkv' and stock caches go through model.generate)")
        for l in layers:
            l.reserve(int(max_steps))                      # off the per-token path: no reallocation while the graph lives
        self._setup(model, cache, layers, first_token, max_steps, use_graph, eos_token_id, pad_token_id, sampling, logprobs,
                    prompts)
        if forced is not None:
            if sampling is not None:
                raise ValueError("StaticDecoder: forced tokens and sampling exclude each other")
            if tuple(forced.shape) != (self.ids.shape[0], self.max_steps):
                raise ValueError(f"StaticDecoder: forced must be [B={self.ids.shape[0]}, {self.max_steps}], got {tuple(forced.shape)}")
            self.forced = forced.to(device=self.ids.device, dtype=torch.long).contiguous()
        self.beam = beam
        if beam is not None and (sampling is not None or forced is not None or logprobs is not None or eos_token_id is not None):
            raise ValueError("StaticDecoder: beam search excludes sampling, forced tokens, logprobs and eos_token_id")
        self.done = None if self.eos is None else (self.ids == self.eos[None, :]).any(dim=1, keepdim=True)   # [B, 1]
        if self.constrained:
            # a stop sequence completed by the first token; from then on each step ORs in its stop flags
            self.done = self.sampling.stop.clone() if self.done is None else self.done.logical_or_(self.sampling.stop)
        if layers[0].window is not None and self.done is not None:
            # decode window: a finished sequence's later rows would overwrite ring rows its cache keeps, so its row counts
            # leave the range the kernel attends (it reads and writes nothing; its tokens are pad_token_id anyway)
            self.window_rows = torch.stack([l.rows for l in layers])
            for i, l in enumerate(layers):
                l.rows = self.window_rows[i]
            self._stop_finished()

    def _setup(self, model, cache, layers, first_token, max_steps, use_graph, eos_token_id, pad_token_id, sampling,
               logprobs=None, prompts=None, penalties=False, constraints=False, history=None) -> None:
        """The state both decoders hold: the step counter and workspace the decode launches read, the per-sequence input
        ids and positions, the token buffer [B, max_steps] and its cursor, the EOS ids, when sampling, the per-sequence
        sampling state with the buffer the sampled tokens land in, and with `logprobs` the buffers of the log-probabilities."""
        self.model, self.cache, self.layers, self.max_steps = model, cache, layers, int(max_steps)
        dev = layers[0].device
        bsz = layers[0].k_buf.shape[0]
        self.backend = model.model.layers[0].self_attn.kv_cluster.backend
        self.state = _StaticState(step=torch.zeros(1, dtype=torch.int32, device=dev),
                                  workspace=self.backend.decode_workspace(bsz * layers[0].num_q_heads, layers[0].k_buf.shape[3], dev))
        if layers[0].heavy is not None:
            self.state.heavy_scratch = self.backend.decode_heavy_workspace(bsz, layers[0].num_q_heads, layers[0].window, dev)
        self.ids = first_token.reshape(bsz, 1).to(device=dev, dtype=torch.long).clone()
        self.pos = torch.tensor(layers[0].seq_seen, dtype=torch.long, device=dev).reshape(bsz, 1)
        self.cursor = torch.zeros(1, dtype=torch.long, device=dev)
        self.tokens = torch.zeros(bsz, self.max_steps, dtype=torch.long, device=dev)
        self.eos = None
        if eos_token_id is not None:
            eos = eos_token_id if isinstance(eos_token_id, (list, tuple)) else [eos_token_id]
            self.eos = torch.tensor([int(e) for e in eos], dtype=torch.long, device=dev)
        self.pad_token_id = int(pad_token_id)
        self.taken = 0
        self.graph = None
        self.window_rows = None   # [layers, B * heads] decode-window row counts, when finished sequences must stop writing
        self.use_graph = (dev.type == "cuda") if use_graph is None else bool(use_graph)
        self.sampling = None
        if sampling is not None:
            if len(sampling) != bsz:
                raise ValueError(f"{len(sampling)} SamplingParams for {bsz} sequences")
            self.sampling = SamplingState(sampling, dev, index=1, vocab=model.lm_head.weight.shape[0], prompts=prompts,
                                          first=self.ids, penalties=penalties, constraints=constraints,
                                          eos=eos_token_id, history=self.max_steps if history is None else history)
            self.sampled = torch.zeros(bsz, 1, dtype=torch.long, device=dev)
            if self.sampling.constrained:
                self.sampling.rules(self.backend)                         # the first step's rule terms and stop flags
        self.constrained = self.sampling is not None and self.sampling.constrained
        self.forced = None
        self.beam = None
        self.logprobs = None if logprobs is None else _LogprobBuffers(bsz, self.max_steps, int(logprobs), dev)
        cache._pkv_static = self.state

    def _greedy_token(self) -> torch.Tensor:
        """The forward of one token per sequence through every layer (appending to the cache); the argmax [B, 1], with
        sampling the drawn tokens (one `sample_tokens` launch for every sequence; each token index advances by one), or the
        forced tokens at the cursor. With `logprobs`, one `token_logprobs` launch then scores the token at the cursor."""
        m = self.model.model
        h = m.embed_tokens(self.ids)
        pos_emb = m.rotary_emb(h, position_ids=self.pos)
        for layer in m.layers[: self.model.config.num_hidden_layers]:
            h = layer(h, attention_mask=None, position_embeddings=pos_emb, position_ids=self.pos,
                      past_key_values=self.cache, use_cache=True)
        h = m.norm(h)
        logits = self.model.lm_head(h[:, -1, :])
        if self.beam is not None:
            # this step's row is iteration step + 1 of the beam search (iteration 0 read the prefill's logits)
            self.beam.step(self.backend, logits, self.beam.k, self.state.step, 1)
            reorder_caches(self.cache, self.beam.P, self.beam.k, self.beam.parent, self.beam.diverge, self.state.step, 1,
                           self.backend)
            tok = self.beam.next_token.view(-1, 1)
        elif self.forced is not None:
            tok = self.forced.index_select(1, self.cursor)                # [B, 1]
        elif self.sampling is not None:
            self.sampling.draw(self.backend, logits, self.sampled, 0)
            tok = self.sampled
        else:
            tok = logits.argmax(dim=-1, keepdim=True)                     # [B, 1]
        if self.logprobs is not None:
            self.logprobs.write(self.backend, logits, tok, self.cursor)
        return tok

    _STOPPED = -(2 ** 30)   # a row count no step counter brings back into range

    def _stop_finished(self) -> None:
        B = self.done.shape[0]
        self.window_rows.view(len(self.layers), B, -1).masked_fill_(self.done.view(1, B, 1), self._STOPPED)

    # one greedy step; every tensor it touches is static, every launch argument constant
    def _step(self) -> None:
        nxt = self._greedy_token()
        if self.done is not None:
            nxt = torch.where(self.done, self.pad_token_id, nxt)
            if self.eos is not None:
                self.done.logical_or_((nxt == self.eos[None, :]).any(dim=1, keepdim=True))
            if self.constrained:
                self.sampling.rules(self.backend, self.sampled)           # append the token; the next step's rules
                self.done.logical_or_(self.sampling.stop)
            if self.window_rows is not None:
                self._stop_finished()
        self.tokens.index_copy_(1, self.cursor, nxt)
        self.ids.copy_(nxt)
        self.pos.add_(1)
        self.cursor.add_(1)
        self.state.step.add_(1)

    def _counters(self) -> list:
        """The device tensors a step advances (restored after the warm-up step of a capture)."""
        idx = self.sampling.index if self.sampling is not None else None
        counts = self.sampling.counts if self.sampling is not None and self.sampling.penalized else None
        # the heavy-hitter state a step updates (knob pkv_decode_heavy): restored so that the captured step starts from it
        heavy = [t for l in self.layers if l.heavy is not None for t in (l.heavy_scores, l.heavy_gen, l.victim)]
        rules = self.sampling.rule_state() if self.sampling is not None else []
        # beam search: the warm-up step of a capture runs at step 0, where the reorder only touches the row the captured
        # step rewrites, so restoring the beam state restores everything
        rules += self.beam.state() if self.beam is not None else []
        return [t for t in (self.ids, self.pos, self.cursor, self.state.step, self.tokens, self.done, idx, counts,
                            self.window_rows) if t is not None] + heavy + rules

    def _capture(self) -> None:
        # warm up on a side stream (lazy initialisation, cuBLAS workspaces), restore the counters, then capture
        if self.beam is not None and self.taken:
            raise RuntimeError("StaticDecoder: a beam search graph is captured before its first step")
        state = self._counters()
        snap = [t.clone() for t in state]
        s = torch.cuda.Stream(device=self.ids.device)
        s.wait_stream(torch.cuda.current_stream(self.ids.device))
        with torch.cuda.stream(s):
            self._step()
        torch.cuda.current_stream(self.ids.device).wait_stream(s)
        # the warm-up step appended row length+1+0 of every layer; the captured run rewrites the same row first
        for t, v in zip(state, snap):
            t.copy_(v)
        self.graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(self.graph):
            self._step()
        for t, v in zip(state, snap):
            t.copy_(v)                                   # capture does not execute, but keep the invariant explicit

    @torch.no_grad()
    def run(self, steps: int) -> torch.Tensor:
        """Take `steps` more greedy steps; returns all tokens produced so far by this decoder, [B, taken] (device)."""
        if self.taken + steps > self.max_steps:
            raise ValueError(f"{self.taken} + {steps} steps exceed the {self.max_steps} reserved")
        if self.use_graph and self.graph is None and steps > 0:
            self._capture()
        for _ in range(steps):
            if self.graph is not None:
                self.graph.replay()
            else:
                self._step()
        self.taken += steps
        return self.tokens[:, : self.taken]

    def finish(self, kept=None) -> None:
        """Settle the host bookkeeping (rows / tokens seen per layer) and leave static mode; the cache is then a normal
        compacted cache again (further `model.generate`/forward calls continue from it). `kept[b]`: the rows sequence b keeps
        (joined caches only; default: every step taken) - rows appended after a sequence's EOS stay in the buffers uncounted."""
        if getattr(self.cache, "_pkv_static", None) is self.state:
            del self.cache._pkv_static
        for l in self.layers:
            if kept is not None:
                l.settle(kept)
            else:
                l.advance(self.taken)
        self.graph = None
        self.taken = 0


def _prefill_logits(model, input_ids: torch.Tensor):
    """Prefill (+ eviction in every patched layer) of one prompt: (logits of its last position [1, V], cache)."""
    from transformers import DynamicCache
    if hasattr(model, "prepare_inputs_for_generation"):
        for layer in model.model.layers:                 # what the patched prepare_inputs does on an empty cache (llama_model.py:2609-2612)
            layer.self_attn.kv_seq_len = 0
    cache = DynamicCache(config=model.config)
    out = model(input_ids=input_ids, past_key_values=cache, use_cache=True, logits_to_keep=1)
    return out.logits[:, -1, :], cache


def _score(model, logits: torch.Tensor, token: torch.Tensor, top_n: int):
    """The log-probability entry of `token` [1, 1] under `logits` [1, V]: host (lp [1], ids [1, N], top [1, N])."""
    buf = _LogprobBuffers(1, 1, top_n, logits.device)
    buf.write(_backend(model), logits, token)
    lp, ids, top = buf.host(1)
    return lp[0], ids[0], top[0]


def _prefill(model, input_ids: torch.Tensor, sampling: Optional[SamplingParams] = None, logprobs: Optional[int] = None,
             eos=None):
    """Prefill (+ eviction in every patched layer) of one prompt: (first token [1, 1], cache), and with `logprobs` the
    first token's log-probability entry (`_score`). The token is the argmax, or with `sampling` drawn with token index 0
    (with constraints, under the rules of the prompt as history; `eos`: the EOS ids they use)."""
    logits, cache = _prefill_logits(model, input_ids)
    if sampling is None:
        first = logits.argmax(dim=-1, keepdim=True)
    else:
        first = torch.zeros(1, 1, dtype=torch.long, device=logits.device)
        st = SamplingState([sampling], logits.device, index=0, vocab=logits.shape[1], prompts=[input_ids], eos=eos)
        if st.constrained:
            st.rules(_backend(model))
        st.draw(_backend(model), logits, first, 0, advance=False)
    if logprobs is None:
        return first, cache
    return first, cache, _score(model, logits, first, logprobs)


def _eos_set(eos_token_id) -> set:
    if eos_token_id is None:
        return set()
    return set(int(e) for e in (eos_token_id if isinstance(eos_token_id, (list, tuple)) else [eos_token_id]))


@torch.no_grad()
def greedy_generate(model, input_ids: torch.Tensor, max_new_tokens: int, use_graph: Optional[bool] = None,
                    return_cache: bool = False, eos_token_id=None, check_every: int = 16,
                    sampling: Optional[SamplingParams] = None, logprobs: Optional[int] = None,
                    prompt_lookup_num_tokens: Optional[int] = None, max_matching_ngram_size: Optional[int] = None):
    """Prefill (+ eviction in every patched layer) then up to `max_new_tokens - 1` static decode steps. Greedy unless
    `sampling` (a SamplingParams) is given: every token is then drawn with it (DESIGN.md §4.6).
    Returns sequences [1, prompt + generated] like `generate(...).sequences` (and the cache on request).
    `eos_token_id` (int or list, as the reference runner passes it: run_longbench.py:270-272) ends the generation with the first
    such token (kept, like HF); the device never waits for the host, so the tokens are inspected every `check_every` steps
    and the surplus steps are dropped. With `logprobs` = N (0 to 20) the return value gains, as its last element, a list of
    one `TokenLogprobs` for the generated tokens (DESIGN.md §4.8).
    `prompt_lookup_num_tokens` = K (1 to 15) decodes by greedy prompt-lookup speculation (HF's argument of that name, with
    `max_matching_ngram_size` N, 1 to 8, default 2): each step drafts up to K tokens by matching the last N-gram of the
    prompt and the tokens so far, verifies them in one forward and keeps the accepted ones (`SpeculativeDecoder`, DESIGN.md
    §4.13). The cache is joined (`cache.join_caches`) first; every cache form but the decode window runs. Greedy only."""
    if input_ids.dim() != 2 or input_ids.shape[0] != 1:
        raise NotImplementedError("batch size 1 (as in the reference: README.md:47); greedy_generate_batch decodes several prompts together")
    eos = _eos_set(eos_token_id)
    spec = _check_spec(prompt_lookup_num_tokens, max_matching_ngram_size, sampling, logprobs, "greedy_generate")
    if spec is not None:
        first, gen, cache = _speculative(model, [input_ids], max_new_tokens, *spec, eos, 0, use_graph, check_every)
        seq = torch.cat([input_ids, first.to(input_ids.device),
                         torch.tensor([gen[0]], dtype=torch.long, device=input_ids.device).reshape(1, -1)], dim=1)
        return (seq, cache) if return_cache else seq
    if sampling is not None and not isinstance(sampling, SamplingParams):
        raise ValueError("greedy_generate: sampling must be a SamplingParams")
    logprobs = _check_logprobs(logprobs, "greedy_generate")
    first, cache, *entry = _prefill(model, input_ids, sampling, logprobs, sorted(eos))
    toks, parts = [first], entry
    tail = _StopTail(input_ids, eos, sampling)
    if max_new_tokens > 1 and not tail.push(first):
        # with a decode window the device stops the sequence at its EOS, so that no later row replaces a kept one; the
        # constraints' rules use the EOS ids too
        windowed = eos and getattr(cache.layers[0], "window", None) is not None
        constrained = sampling is not None and sampling.constrained
        dec = StaticDecoder(model, cache, first, max_new_tokens - 1, use_graph=use_graph,
                            eos_token_id=sorted(eos) if eos and (windowed or constrained) else None,
                            sampling=None if sampling is None else [sampling], logprobs=logprobs, prompts=[input_ids])
        keep = max_new_tokens - 1
        if not eos and not tail.stops:
            toks.append(dec.run(max_new_tokens - 1).clone())
        else:
            done, keep = 0, max_new_tokens - 1
            while done < max_new_tokens - 1:
                n = min(max(1, check_every), max_new_tokens - 1 - done)
                got = dec.run(n)[0, done:done + n].tolist()              # one device-to-host read per chunk
                hit = next((i for i, t in enumerate(got) if tail.push(t)), None)
                done += n
                if hit is not None:
                    keep = done - n + hit + 1
                    break
            toks.append(dec.tokens[:, :keep].clone())
            # rows appended after the EOS stay in the buffers but are not counted: the cache ends with the EOS token
            dec.taken = keep
        if logprobs is not None:
            parts.append(tuple(t[0] for t in dec.logprobs.host(keep)))
        dec.finish()
    seq = torch.cat([input_ids, *toks], dim=1)
    out = (seq, cache) if return_cache else (seq,)
    if logprobs is not None:
        out += ([_join_entries(seq[0, input_ids.shape[1]:].cpu(), parts)],)
    return out if len(out) > 1 else seq


@torch.no_grad()
def greedy_generate_batch(model, prompts, max_new_tokens: int, eos_token_id=None, pad_token_id: int = 0,
                          use_graph: Optional[bool] = None, check_every: int = 16, return_cache: bool = False, sampling=None,
                          logprobs: Optional[int] = None, prompt_lookup_num_tokens: Optional[int] = None,
                          max_matching_ngram_size: Optional[int] = None):
    """Greedy generation for several prompts of any lengths (1-D or [1, S] id tensors): each prompt is prefilled alone
    exactly as `greedy_generate` does, the compacted caches are joined, and up to `max_new_tokens - 1` steps decode all of
    them together (`StaticDecoder` over the joined cache). Each sequence stops at its first `eos_token_id` (kept, like HF);
    the loop ends once all are done, which the host checks every `check_every` steps. Returns one 1-D tensor per prompt,
    prompt + generated (and the joined cache on request, its per-sequence rows ending at each EOS). Greedy unless `sampling`
    (one SamplingParams for all prompts, or one per prompt) is given: each prompt's tokens are then drawn with its own.
    With `logprobs` = N (0 to 20) the return value gains, as its last element, one `TokenLogprobs` per prompt for its
    generated tokens (DESIGN.md §4.8). `prompt_lookup_num_tokens` / `max_matching_ngram_size`: greedy prompt-lookup
    speculation as in `greedy_generate`, every prompt drafting from its own history."""
    ids = [p.reshape(1, -1) for p in prompts]
    if not ids:
        raise ValueError("greedy_generate_batch: no prompts")
    eos = _eos_set(eos_token_id)
    spec = _check_spec(prompt_lookup_num_tokens, max_matching_ngram_size, sampling, logprobs, "greedy_generate_batch")
    if spec is not None:
        first, gen, cache = _speculative(model, ids, max_new_tokens, *spec, eos, pad_token_id, use_graph, check_every)
        seqs = [torch.cat([p[0].cpu(), first[b].cpu(), torch.tensor(gen[b], dtype=torch.long)]).to(p.device)
                for b, p in enumerate(ids)]
        return (seqs, cache) if return_cache else seqs
    samp = _sampling_list(sampling, len(ids), "greedy_generate_batch")
    logprobs = _check_logprobs(logprobs, "greedy_generate_batch")
    firsts, caches, entries = [], [], []
    for i, p in enumerate(ids):
        f, c, *e = _prefill(model, p, None if samp is None else samp[i], logprobs, sorted(eos))
        firsts.append(f)
        caches.append(c)
        entries.append(e)
    first = torch.cat(firsts)                                            # [B, 1]
    steps = max(0, max_new_tokens - 1)
    cache = join_caches(caches, reserve=steps)
    del caches
    first_host = first[:, 0].tolist()
    kept = [0] * len(ids)
    gen = torch.empty(len(ids), 0, dtype=torch.long)
    tails = [_StopTail(p, eos, None if samp is None else samp[b]) for b, p in enumerate(ids)]
    stops = any(t.stops for t in tails)
    ended = [t.push(f) for t, f in zip(tails, first_host)]
    if steps and not all(ended):
        dec = StaticDecoder(model, cache, first, steps, use_graph=use_graph, eos_token_id=sorted(eos) if eos else None,
                            pad_token_id=pad_token_id, sampling=samp, logprobs=logprobs, prompts=ids)
        while dec.taken < steps:
            dec.run(min(max(1, check_every) if eos or stops else steps, steps - dec.taken))
            if dec.done is not None and bool(dec.done.all()):           # one device-to-host read per chunk
                break
        gen = dec.tokens[:, : dec.taken].cpu()
        for b in range(len(ids)):
            if ended[b]:
                continue
            row = gen[b].tolist()
            hit = next((i for i, t in enumerate(row) if tails[b].push(t)), None)
            kept[b] = len(row) if hit is None else hit + 1
        if logprobs is not None:
            lp, lp_ids, lp_top = dec.logprobs.host(dec.taken)
            for b in range(len(ids)):
                entries[b].append((lp[b, : kept[b]], lp_ids[b, : kept[b]], lp_top[b, : kept[b]]))
        dec.finish(kept)
    seqs = [torch.cat([p[0].cpu(), first[b].cpu(), gen[b, : kept[b]]]).to(p.device) for b, p in enumerate(ids)]
    out = (seqs, cache) if return_cache else (seqs,)
    if logprobs is not None:
        out += ([_join_entries(s[p.shape[1]:].cpu(), e) for s, p, e in zip(seqs, ids, entries)],)
    return out if len(out) > 1 else seqs


MAX_PROMPT_LOOKUP_TOKENS, MAX_MATCHING_NGRAM = 15, 8


def _check_spec(num_tokens, ngram, sampling, logprobs, what: str):
    """(K, N) of prompt-lookup speculative decoding, or None when it is off; ValueError for what it excludes."""
    if num_tokens is None:
        if ngram is not None:
            raise ValueError(f"{what}: max_matching_ngram_size goes with prompt_lookup_num_tokens")
        return None
    ngram = 2 if ngram is None else ngram
    for name, v, hi in (("prompt_lookup_num_tokens", num_tokens, MAX_PROMPT_LOOKUP_TOKENS),
                        ("max_matching_ngram_size", ngram, MAX_MATCHING_NGRAM)):
        if isinstance(v, bool) or not isinstance(v, int) or not 1 <= v <= hi:
            raise ValueError(f"{what}: {name} must be an integer in [1, {hi}], got {v!r}")
    if sampling is not None or logprobs is not None:
        raise ValueError(f"{what}: prompt_lookup_num_tokens is greedy only: it excludes sampling and logprobs")
    return int(num_tokens), int(ngram)


def _check_spec_cache_form(model) -> None:
    from .cache import decode_heavy, decode_window
    for knob, v in (("pkv_decode_heavy", decode_heavy(model.config)), ("pkv_decode_window", decode_window(model.config))):
        if v is not None:
            raise NotImplementedError(f"prompt_lookup_num_tokens with {knob} = {v} is not built: the rows a verify step "
                                      "writes for rejected drafts would already have replaced rows the decode window keeps")


class SpecState:
    """The device state of prompt-lookup speculative decoding (include/pkv.h: pkv_prompt_lookup, pkv_spec_step) over B
    sequences with Q = K + 1 verify rows: each sequence's history (prompt, then every emitted token; int64 [B, cap] and its
    length), remaining budget, done flag, the tokens the steps emitted (int64 [B, max_new_tokens - 1], pad_token_id past
    each sequence's cursor `out_len`), the next verify step's input ids and positions [B, Q], the draft length, the tokens
    the last step emitted and the verify argmaxes `tokens` [B, Q]. Every tensor is written in place, so a captured step
    keeps its pointers. `budgets` (one per sequence, in place of max_new_tokens - 1 for all) and `out_cap` (the width of
    `out`) serve the continuous loop, whose slots come and go."""

    def __init__(self, prompts, first: torch.Tensor, max_new_tokens: int, K: int, N: int, eos, pad_token_id: int, device,
                 budgets=None, out_cap: Optional[int] = None):
        B, Q, steps = len(prompts), K + 1, max(0, int(max_new_tokens) - 1)
        lens = [int(p.numel()) for p in prompts]
        i32, i64 = dict(dtype=torch.int32, device=device), dict(dtype=torch.long, device=device)
        self.hist = torch.zeros(B, max(lens) + max(1, int(max_new_tokens)), **i64)
        for b, p in enumerate(prompts):
            self.hist[b, : lens[b]] = p.reshape(-1).to(device)
            self.hist[b, lens[b]] = first.reshape(-1)[b]
        self.prompt_len = torch.tensor(lens, **i32)
        self.hist_len = self.prompt_len + 1
        self.budget = torch.full((B,), steps, **i32) if budgets is None else torch.tensor([int(n) for n in budgets], **i32)
        self.eos = torch.tensor(sorted(_eos_set(eos)), **i64)
        if self.eos.numel() > 4:
            raise ValueError("prompt_lookup_num_tokens: at most 4 EOS ids")
        self.done = torch.isin(first.reshape(-1).to(device), self.eos) | (self.budget <= 0)
        self.out = torch.full((B, max(1, steps) if out_cap is None else int(out_cap)), int(pad_token_id), **i64)
        self.out_len = torch.zeros(B, **i32)
        self.ids = torch.zeros(B, Q, **i64)
        self.pos = torch.zeros(B, Q, **i64)
        self.draft_len = torch.zeros(B, **i32)
        self.emitted = torch.zeros(B, **i32)
        self.tokens = torch.zeros(B, Q, **i64)
        self.max_ngram, self.pad_token_id = int(N), int(pad_token_id)

    def state(self) -> list:
        """The tensors a step advances (restored after the warm-up step of a graph capture; the history and output rows
        past the restored cursors are rewritten by the next step)."""
        return [self.hist_len, self.budget, self.done, self.out_len, self.ids, self.pos, self.draft_len, self.emitted,
                self.tokens]

    def set_row(self, b: int, prompt: torch.Tensor, first: torch.Tensor, budget: int) -> bool:
        """Sequence b starts over with `prompt` (1-D ids), its first token and `budget` tokens to emit, in place. True when
        the history had to grow (a new tensor: a captured step must be captured again)."""
        prompt = prompt.reshape(-1)
        n = int(prompt.numel())
        grew = n + 1 + max(0, int(budget)) > self.hist.shape[1]
        if grew:
            hist = torch.zeros(self.hist.shape[0], n + 1 + int(budget), dtype=self.hist.dtype, device=self.hist.device)
            hist[:, : self.hist.shape[1]] = self.hist
            self.hist = hist
        first = first.reshape(-1)[:1].to(self.hist.device)
        self.hist[b, :n] = prompt.to(self.hist.device)
        self.hist[b, n] = first[0]
        self.prompt_len[b] = n
        self.hist_len[b] = n + 1
        self.budget[b] = int(budget)
        self.done[b] = bool(torch.isin(first, self.eos).any()) or int(budget) <= 0
        self.out_len[b] = 0
        return grew


class PackState:
    """The packed verify rows of a continuous speculative step (include/pkv.h: pkv_spec_pack, pkv_decode_attn_packed):
    M = B + max_draft_tokens token rows, their ids and positions (int64 [1, M]), each slot's first row and row count (int32
    [B]), the step counter `step` the budget rotation starts from, and `totals` int64 [2]: the draft tokens granted and
    the live slot-steps, summed over the steps."""

    def __init__(self, B: int, K: int, max_draft_tokens: int, step: torch.Tensor, device):
        M = B + int(max_draft_tokens)
        self.num_queries, self.max_draft_tokens = K + 1, int(max_draft_tokens)
        self.ids = torch.zeros(1, M, dtype=torch.long, device=device)
        self.pos = torch.zeros(1, M, dtype=torch.long, device=device)
        self.row_start = torch.zeros(B, dtype=torch.int32, device=device)
        self.row_count = torch.zeros(B, dtype=torch.int32, device=device)
        self.step = step
        self.totals = torch.zeros(2, dtype=torch.long, device=device)


class SpeculativeDecoder(StaticDecoder):
    """Greedy prompt-lookup speculative decoding (HF's `generate(prompt_lookup_num_tokens=K, max_matching_ngram_size=N)`)
    over a joined cache (`cache.join_caches`, any form but the decode window) of the prompts `prompts` whose prefill
    produced `first_token` [B] or [B, 1]. One step, captured once in a CUDA graph: the embedding of the [B, Q] verify ids
    (the last emitted token and up to K draft tokens), every layer (the attention stores the Q new rows and attends them
    causally: `decode_multi`), the LM head on all B*Q rows, their argmax and one `pkv_spec_step` launch that accepts, emits,
    advances every layer's row counts and drafts the next step's ids by prompt lookup (DESIGN.md §4.13). Each step emits
    1 .. K + 1 tokens per live sequence, so max_new_tokens - 1 steps finish every sequence. `forced_drafts` (tests and
    measurements): None, or int64 [B, F] - after every step sequence b drafts forced_drafts[b, E : E + K], E its tokens
    generated so far (the prefill's included), in place of the lookup."""

    def __init__(self, model, cache, first_token: torch.Tensor, prompts, max_new_tokens: int, num_tokens: int,
                 max_ngram: int = 2, use_graph: Optional[bool] = None, eos_token_id=None, pad_token_id: int = 0,
                 forced_drafts: Optional[torch.Tensor] = None):
        layers = [l for l in cache.layers if isinstance(l, PkvBatchCacheLayer)]
        if len(layers) != model.config.num_hidden_layers or len(layers) != len(cache.layers):
            raise RuntimeError("SpeculativeDecoder needs a joined cache (cache.join_caches) on every layer")
        if layers[0].window is not None:
            raise NotImplementedError("speculative decoding under the decode window (pkv_decode_window / pkv_decode_heavy) "
                                      "is not built")
        K, steps = int(num_tokens), max(0, int(max_new_tokens) - 1)
        for l in layers:
            # the rows, the decoded tokens and one verify step's K + 1: a sequence that spent its budget still verifies (and
            # writes, uncounted) Q rows behind its last one while the others run
            l.reserve(steps + K + 1)
        self._setup(model, cache, layers, first_token, max(1, steps), use_graph, None, pad_token_id, None)
        dev, B = self.ids.device, len(prompts)
        self.state.workspace = self.backend.decode_workspace(B * layers[0].num_q_heads * (K + 1), layers[0].k_buf.shape[3], dev)
        self.state.spec = True
        self.spec = SpecState(prompts, self.ids, max_new_tokens, K, max_ngram, eos_token_id, pad_token_id, dev)
        self.ids, self.pos, self.done = self.spec.ids, self.spec.pos, self.spec.done
        self.forced_drafts = None
        if forced_drafts is not None:
            self.forced_drafts = forced_drafts.to(device=dev, dtype=torch.long).contiguous()
            self._offsets = torch.arange(K, device=dev)
        self.backend.prompt_lookup(self.spec)
        if self.forced_drafts is not None:
            self._force_drafts()

    def _force_drafts(self) -> None:
        st, K = self.spec, self.spec.ids.shape[1] - 1
        idx = ((st.hist_len - st.prompt_len).long()[:, None] + self._offsets).clamp_(max=self.forced_drafts.shape[1] - 1)
        st.ids[:, 1:].copy_(self.forced_drafts.gather(1, idx))
        st.draft_len.copy_(torch.where(st.done | (st.budget <= 1), 0, K))

    def _verify_logits(self) -> torch.Tensor:
        """The forward of the [B, Q] verify ids at their positions through every layer: logits [B, Q, V]."""
        return _forward_rows(self.model, self.cache, self.ids, self.pos)

    def _step(self) -> None:
        self.spec.tokens.copy_(self._verify_logits().argmax(dim=-1))
        self.backend.spec_step(self.spec, [l.rows for l in self.layers])
        if self.forced_drafts is not None:
            self._force_drafts()

    def _counters(self) -> list:
        return self.spec.state() + [l.rows for l in self.layers]

    def generated(self) -> list:
        """Per sequence, the tokens the steps emitted (host lists; the prefill's first token not included)."""
        out, n = self.spec.out.cpu(), self.spec.out_len.cpu().tolist()
        return [out[b, : n[b]].tolist() for b in range(out.shape[0])]

    def run_to_end(self, check_every: int = 16) -> int:
        """Replay until every sequence is done (the host reads the done flags every `check_every` replays) or
        max_new_tokens - 1 replays; returns the replays taken."""
        while self.taken < self.max_steps and not bool(self.done.all()):
            self.run(min(max(1, int(check_every)), self.max_steps - self.taken))
        return self.taken


def _forward_rows(model, cache, ids: torch.Tensor, pos: torch.Tensor) -> torch.Tensor:
    """The forward of token rows `ids` at positions `pos` (both [b, q]) through every layer over `cache`: logits [b, q, V]."""
    m = model.model
    h = m.embed_tokens(ids)
    pos_emb = m.rotary_emb(h, position_ids=pos)
    for layer in m.layers[: model.config.num_hidden_layers]:
        h = layer(h, attention_mask=None, position_embeddings=pos_emb, position_ids=pos, past_key_values=cache, use_cache=True)
    return model.lm_head(m.norm(h))


def _speculative(model, ids, max_new_tokens: int, K: int, N: int, eos: set, pad_token_id: int, use_graph, check_every: int):
    """Prefill each prompt alone, join the caches and decode them by prompt lookup: (first tokens [B, 1], generated host
    lists per prompt, the joined cache with each sequence's rows ending at its last token)."""
    _check_spec_cache_form(model)
    firsts, caches = [], []
    for p in ids:
        f, c = _prefill(model, p, None, None, sorted(eos))
        firsts.append(f)
        caches.append(c)
    first = torch.cat(firsts)
    steps = max(0, max_new_tokens - 1)
    cache = join_caches(caches, reserve=steps + K + 1)
    del caches
    gen = [[] for _ in ids]
    if steps and not all(int(f) in eos for f in first[:, 0].tolist()):
        dec = SpeculativeDecoder(model, cache, first, ids, max_new_tokens, K, N, use_graph=use_graph,
                                 eos_token_id=sorted(eos) if eos else None, pad_token_id=pad_token_id)
        dec.run_to_end(check_every)
        gen = dec.generated()
        dec.finish([len(g) for g in gen])
    return first, gen, cache


class ContinuousDecoder(StaticDecoder):
    """The step of `StaticDecoder` over a fixed set of slots whose sequences come and go (continuous batching).

    cache: a batched cache (`join_caches`) of B slots; first_token [B] the next input per slot; left[b] the decode steps slot b
    may still take. Per step, on the device: a slot becomes `done` when its `left` reaches 0 or it emits an EOS; a done slot
    emits `pad_token_id`, and its row counts stop growing (each later step attends and overwrites the same row). The token
    buffer holds one chunk, [B, chunk]; `run_chunk` replays `steps` steps, reads them with one device-to-host copy and
    resets the cursor in place. Between chunks `admit` copies a prefilled prompt into a slot and `park` empties one; both
    write the buffers and row counts in place, so the captured graph keeps replaying. `grow_for` reallocates the buffers
    when an admission needs more rows; the graph is then captured again. `prompts` (each slot's prompt ids) and `penalties`
    (keep the penalty state even when no starting request needs it, for later admissions) as in `SamplingState`."""

    def __init__(self, model, cache, first_token: torch.Tensor, left, chunk: int, use_graph: Optional[bool] = None,
                 eos_token_id=None, pad_token_id: int = 0, sampling: Optional[List[SamplingParams]] = None,
                 logprobs: Optional[int] = None, prompts=None, penalties: bool = False, constraints: bool = False,
                 history: int = 0):
        layers = [l for l in cache.layers if isinstance(l, PkvBatchCacheLayer)]
        if len(layers) != model.config.num_hidden_layers or len(layers) != len(cache.layers):
            raise RuntimeError("ContinuousDecoder needs a batched cache (cache.join_caches) on every layer")
        self._setup(model, cache, layers, first_token, max(1, int(chunk)), use_graph, eos_token_id, pad_token_id, sampling,
                    logprobs, prompts, penalties, constraints, max([int(n) for n in left] + [int(history)]))
        # every layer's row counts are rows of one tensor, so one op per step stops them growing for the done slots
        self.rows_all = torch.stack([l.rows for l in layers])
        for i, l in enumerate(layers):
            l.rows = self.rows_all[i]
        self.left = torch.tensor([int(n) for n in left], dtype=torch.long, device=self.ids.device).reshape(self.ids.shape[0], 1)
        self.done = self.left <= 0
        self.captures = 0
        self.parked = set()

    def _step(self) -> None:
        nxt = torch.where(self.done, self.pad_token_id, self._greedy_token())
        self.left.sub_(1)
        stop = self.left <= 0
        if self.eos is not None:
            stop.logical_or_((nxt == self.eos[None, :]).any(dim=1, keepdim=True))
        if self.constrained:
            self.sampling.rules(self.backend, self.sampled)
            stop.logical_or_(self.sampling.stop)
        self.done.logical_or_(stop)
        self.rows_all.view(len(self.layers), self.done.shape[0], -1).sub_(self.done.view(1, -1, 1).to(torch.int32))
        self.tokens.index_copy_(1, self.cursor, nxt)
        self.ids.copy_(nxt)
        self.pos.add_(1)
        self.cursor.add_(1)
        self.state.step.add_(1)

    def _counters(self) -> list:
        return super()._counters() + [self.left, self.rows_all]

    def _capture(self) -> None:
        super()._capture()
        self.captures += 1

    def run_chunk(self, steps: int) -> torch.Tensor:
        """Take `steps` (<= chunk) steps; their tokens [B, steps] on the host (with `logprobs`, their log-probabilities in
        `chunk_logprobs`: host [B, steps], [B, steps, N], [B, steps, N])."""
        self.run(steps)
        toks = self.tokens[:, :steps].cpu()
        if self.logprobs is not None:
            self.chunk_logprobs = self.logprobs.host(steps)
        self.cursor.zero_()
        self.taken = 0
        return toks

    def grow_for(self, src_cache, new_tokens: int) -> bool:
        """Make every layer hold the rows of the single-prompt cache `src_cache` plus `new_tokens` (amortised doubling, like
        `reserve`). True when a buffer was reallocated (the graph is then captured again on the next chunk)."""
        grew = False
        for l, s in zip(self.layers, src_cache.layers):
            # with a decode window at most R decoded rows: the capacity depends only on the prompt and R
            grew |= l.fit(max(s.rows_host[0]) + (int(new_tokens) if l.window is None else min(int(new_tokens), l.window)))
        if grew:
            self.graph = None
        return grew

    def admit(self, slot: int, src_cache, first_token: torch.Tensor, left: int, sampling: Optional[SamplingParams] = None,
              prompt=None) -> None:
        """Slot `slot` continues the prefilled prompt `src_cache` (first token `first_token`, `left` decode steps); a sampling
        decoder takes the request's `sampling` parameters, its next token drawn with token index 1, and with penalties its
        prompt mask (`prompt`: the prompt ids) and counts (the first token once) are rebuilt in place."""
        if (sampling is None) != (self.sampling is None):
            raise ValueError("admit: pass sampling parameters exactly when the decoder samples")
        if sampling is not None:
            # checks the request before the slot changes; a reallocated constraint table needs a new graph
            if self.sampling.set_row(slot, sampling, 1, prompt, first_token, history=max(0, int(left))):
                self.graph = None
            if self.constrained:
                self.sampling.rules(self.backend)      # every row's history is unchanged but this slot's
        admit_cache(self.cache, slot, src_cache, self.state.step, self.backend)
        self.ids[slot] = first_token.reshape(-1)[:1].to(self.ids.device)
        self.pos[slot] = self.layers[0].seq_seen[slot]
        self.left[slot] = int(left)
        self.done[slot] = int(left) <= 0
        self.parked.discard(slot)

    def park(self, slot: int) -> None:
        if slot in self.parked:
            return
        park_cache(self.cache, slot, self.state.step, self.backend)
        self.ids[slot] = self.pad_token_id
        self.done[slot] = True
        self.parked.add(slot)

    def finish(self, kept=None) -> None:
        """Leave static mode. The slots' host row counts are those of their admissions (the decoded rows are not booked)."""
        if getattr(self.cache, "_pkv_static", None) is self.state:
            del self.cache._pkv_static
        self.graph = None
        self.taken = 0


class ContinuousSpecDecoder(SpeculativeDecoder, ContinuousDecoder):
    """Greedy prompt-lookup speculation in the continuous loop (DESIGN.md §4.14): the slots of `ContinuousDecoder`, each
    step a verify step of `SpeculativeDecoder` over M = B + max_draft_tokens packed token rows instead of a dense [B, K + 1]
    block. One step, captured once in a CUDA graph: `pkv_spec_pack` (rule 2': every live slot gets its last token and a
    share of the max_draft_tokens draft tokens, in turn from slot step mod B; a done slot gets no row), the forward of the
    [1, M] rows (the attention stores and attends each slot's rows: `decode_packed`), the LM head and argmax on the M rows,
    a gather of each slot's argmaxes into `spec.tokens` and `pkv_spec_step`. `prompts` and `first_token` [B] as in
    `SpeculativeDecoder`; left[b] the tokens slot b may still emit; `chunk` the steps between host reads (`run_chunk`).
    Between chunks `admit` rewrites a slot in place and `park` leaves one done. `history`: the longest budget a later
    admission brings (the history is sized for it). `forced_drafts` (tests and measurements): None, or int64 [B, F] per
    slot, as in `SpeculativeDecoder`; `admit` takes the new request's row."""

    def __init__(self, model, cache, first_token: torch.Tensor, prompts, left, chunk: int, num_tokens: int, max_ngram: int = 2,
                 max_draft_tokens: Optional[int] = None, use_graph: Optional[bool] = None, eos_token_id=None,
                 pad_token_id: int = 0, history: int = 0, forced_drafts: Optional[torch.Tensor] = None):
        layers = [l for l in cache.layers if isinstance(l, PkvBatchCacheLayer)]
        if len(layers) != model.config.num_hidden_layers or len(layers) != len(cache.layers):
            raise RuntimeError("ContinuousSpecDecoder needs a batched cache (cache.join_caches) on every layer")
        if layers[0].window is not None:
            raise NotImplementedError("speculative decoding under the decode window (pkv_decode_window / pkv_decode_heavy) "
                                      "is not built")
        B, K, chunk = len(prompts), int(num_tokens), max(1, int(chunk))
        D = B * K if max_draft_tokens is None else int(max_draft_tokens)
        if not 1 <= D <= B * K:
            raise ValueError(f"max_draft_tokens must be in [1, {B * K}], got {D}")
        left = [int(n) for n in left]
        self._setup(model, cache, layers, first_token, chunk, use_graph, None, pad_token_id, None)
        dev = self.ids.device
        self.state.workspace = self.backend.decode_workspace(B * layers[0].num_q_heads * (K + 1), layers[0].k_buf.shape[3], dev)
        self.state.spec = True
        self.spec = SpecState(prompts, self.ids, max(left + [int(history)]) + 1, K, max_ngram, eos_token_id, pad_token_id, dev,
                              budgets=left, out_cap=chunk * (K + 1))
        self.state.pack = PackState(B, K, D, self.state.step, dev)
        self.ids, self.pos, self.done = self.spec.ids, self.spec.pos, self.spec.done
        self._cols = torch.arange(K + 1, device=dev)
        self._no_offset = torch.zeros(1, dtype=torch.int32, device=dev)   # admissions install absolute row counts
        self.captures = 0
        self.parked = set()
        self.forced_drafts = None
        if forced_drafts is not None:
            self.forced_drafts = forced_drafts.to(device=dev, dtype=torch.long).contiguous()
            self._offsets = torch.arange(K, device=dev)
        self.backend.prompt_lookup(self.spec)
        if self.forced_drafts is not None:
            self._force_drafts()

    def _verify_logits(self) -> torch.Tensor:
        """The forward of the packed rows: logits [1, M, V]."""
        return _forward_rows(self.model, self.cache, self.state.pack.ids, self.state.pack.pos)

    def _step(self) -> None:
        st, pk = self.spec, self.state.pack
        self.backend.spec_pack(st, pk)
        am = self._verify_logits().argmax(dim=-1)[0]                           # [M]
        # slot b's argmaxes t_j sit at rows row_start[b] + j, j < row_count[b]; the rest are never read by the step
        st.tokens.copy_(am[(pk.row_start.long()[:, None] + self._cols).clamp_(max=am.numel() - 1)])
        self.backend.spec_step(st, [l.rows for l in self.layers])
        if self.forced_drafts is not None:
            self._force_drafts()
        self.state.step.add_(1)

    def _counters(self) -> list:
        return super()._counters() + [self.state.step, self.state.pack.totals]

    def run_chunk(self, steps: int) -> list:
        """Take `steps` (<= chunk) steps; per slot, the tokens they emitted (host lists, one device-to-host read)."""
        self.run(steps)
        st = self.spec
        host = torch.cat([st.out, st.out_len.long()[:, None]], dim=1).cpu()
        st.out_len.zero_()
        self.taken = 0
        return [host[b, : int(host[b, -1])].tolist() for b in range(host.shape[0])]

    def admit(self, slot: int, src_cache, first_token: torch.Tensor, left: int, sampling: Optional[SamplingParams] = None,
              prompt=None, forced: Optional[torch.Tensor] = None) -> None:
        """Slot `slot` continues the prefilled prompt `prompt` (its cache `src_cache`, first token `first_token`, `left`
        tokens to emit): its history row and cache rows are rewritten in place (the rows at their absolute counts), and
        the lookup drafts again (unchanged for the other slots). `forced`: the request's forced drafts, with
        `forced_drafts`."""
        if sampling is not None:
            raise ValueError("admit: prompt-lookup speculation is greedy only")
        if self.spec.set_row(slot, prompt, first_token, left):
            self.graph = None
        admit_cache(self.cache, slot, src_cache, self._no_offset, self.backend)
        if self.forced_drafts is not None:
            self.forced_drafts[slot].fill_(self.pad_token_id)
            f = forced.reshape(-1)[: self.forced_drafts.shape[1]]
            self.forced_drafts[slot, : f.numel()] = f.to(self.forced_drafts.device)
        self.backend.prompt_lookup(self.spec)
        if self.forced_drafts is not None:
            self._force_drafts()
        self.parked.discard(slot)

    def park(self, slot: int) -> None:
        self.done[slot] = True
        self.parked.add(slot)


def _sync(device: torch.device) -> None:
    if device.type == "cuda":
        torch.cuda.synchronize(device)


@torch.no_grad()
def greedy_generate_continuous(model, prompts, max_new_tokens, num_slots: int, eos_token_id=None, pad_token_id: int = 0,
                               use_graph: Optional[bool] = None, check_every: int = 16, return_stats: bool = False,
                               sampling=None, logprobs: Optional[int] = None, prompt_lookup_num_tokens: Optional[int] = None,
                               max_matching_ngram_size: Optional[int] = None, max_draft_tokens: Optional[int] = None,
                               _forced_drafts=None):
    """Greedy generation for any number of prompts (1-D or [1, S] id tensors) through `num_slots` sequences decoded together
    (continuous batching). `max_new_tokens`: an int, or one per prompt. The first `num_slots` prompts are prefilled one at a
    time and joined exactly as in `greedy_generate_batch`; decoding then runs in chunks of `check_every` steps. After each
    chunk the host reads its tokens once, retires every sequence that emitted an EOS (kept) or reached its own
    `max_new_tokens`, and prefills the next waiting prompts in order, each into a free slot (`ContinuousDecoder.admit`); a
    slot with nothing left to admit is parked. Returns one 1-D tensor per prompt, in prompt order, prompt + generated (the
    format of `greedy_generate_batch`), and with `return_stats` a dict: decode_steps, live_slot_steps (the sum over steps
    of the slots holding an unfinished sequence), admissions (prompts admitted after the start), regrowths, graph_captures,
    prefill_s / decode_s (host wall time of the prefills and of the rest of the loop) and per prompt `prefill_ms` and
    `cache_rows_first_last` (rows of its first and last layer after the prefill). Greedy unless `sampling` (one
    SamplingParams for all prompts, or one per prompt) is given: each request's tokens are then drawn with its own, and
    equal those it gets from `greedy_generate_batch` with the same parameters wherever its logits are equal there. With
    `logprobs` = N (0 to 20) the return value gains, as its last element, one `TokenLogprobs` per prompt for its generated
    tokens, read with the tokens once per chunk (DESIGN.md §4.8).
    `prompt_lookup_num_tokens` = K / `max_matching_ngram_size` = N: greedy prompt-lookup speculation as in
    `greedy_generate` (`ContinuousSpecDecoder`, DESIGN.md §4.14): each step verifies one token per live slot plus at most
    `max_draft_tokens` = D draft tokens shared by the slots (1 to num_slots * K, default num_slots * K), packed into
    num_slots + D rows. The stats then gain `granted_drafts` and `accepted_drafts` (run totals), and live_slot_steps counts
    verify steps of live slots. Every cache form but the decode window runs; greedy only. `_forced_drafts` (tests and
    measurements): one 1-D id tensor per prompt; after every step its slot drafts from it at the index of its tokens so far
    (the first included), in place of the lookup."""
    ids = [p.reshape(1, -1) for p in prompts]
    if not ids:
        raise ValueError("greedy_generate_continuous: no prompts")
    caps = [int(n) for n in max_new_tokens] if isinstance(max_new_tokens, (list, tuple)) else [int(max_new_tokens)] * len(ids)
    if len(caps) != len(ids):
        raise ValueError(f"greedy_generate_continuous: {len(caps)} max_new_tokens for {len(ids)} prompts")
    if int(num_slots) < 1:
        raise ValueError(f"greedy_generate_continuous: num_slots must be >= 1, got {num_slots}")
    eos = _eos_set(eos_token_id)
    spec = _check_spec(prompt_lookup_num_tokens, max_matching_ngram_size, sampling, logprobs, "greedy_generate_continuous")
    if spec is None and max_draft_tokens is not None:
        raise ValueError("greedy_generate_continuous: max_draft_tokens goes with prompt_lookup_num_tokens")
    if spec is not None:
        _check_spec_cache_form(model)
        hi = int(num_slots) * spec[0]
        if max_draft_tokens is not None and (isinstance(max_draft_tokens, bool) or not isinstance(max_draft_tokens, int)
                                             or not 1 <= max_draft_tokens <= hi):
            raise ValueError(f"greedy_generate_continuous: max_draft_tokens must be an integer in [1, {hi}] "
                             f"(num_slots * prompt_lookup_num_tokens), got {max_draft_tokens!r}")
    samp = _sampling_list(sampling, len(ids), "greedy_generate_continuous")
    logprobs = _check_logprobs(logprobs, "greedy_generate_continuous")
    chunk = max(1, int(check_every))
    dev = ids[0].device
    gen = [[] for _ in ids]                        # generated tokens per prompt, the prefill's first token included
    lps = [[] for _ in ids]                        # with logprobs: their entries, host (lp [k], ids [k, N], top [k, N])
    stats = dict(decode_steps=0, live_slot_steps=0, admissions=0, regrowths=0, graph_captures=0, prefill_s=0.0, decode_s=0.0,
                 prefill_ms=[0.0] * len(ids), cache_rows_first_last=[[] for _ in ids])
    t_start = time.perf_counter()

    tails = [_StopTail(p, eos, None if samp is None else samp[i]) for i, p in enumerate(ids)]
    ended = [False] * len(ids)                     # the last token pushed ended the sequence (EOS or stop sequence)

    def push(i, t):
        gen[i].append(t)
        ended[i] = tails[i].push(t)

    def finished(i):
        return len(gen[i]) >= max(1, caps[i]) or ended[i]

    def prefill(i):
        _sync(dev)
        t0 = time.perf_counter()
        first, cache, *entry = _prefill(model, ids[i], None if samp is None else samp[i], logprobs, sorted(eos))
        push(i, int(first))                        # waits for the prefill
        lps[i].extend(entry)
        ms = (time.perf_counter() - t0) * 1e3
        stats["prefill_ms"][i] = ms
        stats["prefill_s"] += ms / 1e3
        stats["cache_rows_first_last"][i] = [max(cache.layers[0].rows_host[0]), max(cache.layers[-1].rows_host[0])]
        return first, cache

    B = min(int(num_slots), len(ids))
    firsts, caches = zip(*[prefill(i) for i in range(B)])
    cache = join_caches(list(caches), reserve=max(caps))
    del caches
    slot_req = list(range(B))
    left = [0 if finished(b) else caps[b] - 1 for b in range(B)]
    forced = None
    if spec is None:
        dec = ContinuousDecoder(model, cache, torch.cat(firsts), left, chunk,
                                use_graph=use_graph, eos_token_id=sorted(eos) if eos else None, pad_token_id=pad_token_id,
                                sampling=None if samp is None else samp[:B], logprobs=logprobs, prompts=ids[:B],
                                penalties=samp is not None and any(p.penalized for p in samp),
                                constraints=samp is not None and any(p.constrained for p in samp), history=max(caps))
    else:
        K, N = spec
        if _forced_drafts is not None:
            width = max(caps) + K
            forced = [torch.full((width,), int(pad_token_id), dtype=torch.long) for _ in ids]
            for f, src in zip(forced, _forced_drafts):
                src = torch.as_tensor(src, dtype=torch.long).reshape(-1)[:width].cpu()
                f[: src.numel()] = src
        D = min(B * K, max_draft_tokens if max_draft_tokens is not None else int(num_slots) * K)
        dec = ContinuousSpecDecoder(model, cache, torch.cat(firsts), [p.reshape(-1) for p in ids[:B]], left, chunk, K, N, D,
                                    use_graph=use_graph, eos_token_id=sorted(eos) if eos else None,
                                    pad_token_id=pad_token_id, history=max(caps),
                                    forced_drafts=None if forced is None else torch.stack(forced[:B]))
    decoded = 0                                    # tokens the decode steps emitted
    waiting = B
    while True:
        for s in range(B):
            if slot_req[s] is not None and not finished(slot_req[s]):
                continue
            slot_req[s] = None
            while waiting < len(ids) and slot_req[s] is None:
                i = waiting
                waiting += 1
                first, single = prefill(i)
                if finished(i):
                    continue
                stats["regrowths"] += int(dec.grow_for(single, caps[i]))
                dec.admit(s, single, first, caps[i] - 1, None if samp is None else samp[i], ids[i],
                          **({} if forced is None else {"forced": forced[i]}))
                stats["admissions"] += 1
                slot_req[s] = i
            if slot_req[s] is None:
                dec.park(s)
        live = [s for s in range(B) if slot_req[s] is not None]
        if not live:
            break
        n = min(chunk, max(caps[slot_req[s]] - len(gen[slot_req[s]]) for s in live))
        toks = dec.run_chunk(n)                    # one device-to-host read per chunk
        stats["decode_steps"] += n
        for s in live:
            r = slot_req[s]
            for j, t in enumerate(toks[s] if spec is not None else toks[s].tolist()):
                push(r, t)
                decoded += 1
                if finished(r):
                    break
            if logprobs is not None:
                lps[r].append(tuple(x[s, : j + 1] for x in dec.chunk_logprobs))
    stats["live_slot_steps"] = decoded
    if spec is not None:
        granted, live_steps = dec.state.pack.totals.tolist()
        stats.update(live_slot_steps=live_steps, granted_drafts=granted, accepted_drafts=decoded - live_steps)
    dec.finish()
    stats["graph_captures"] = dec.captures
    stats["decode_s"] = time.perf_counter() - t_start - stats["prefill_s"]
    seqs = [torch.cat([p[0].cpu(), torch.tensor(g, dtype=torch.long)]).to(p.device) for p, g in zip(ids, gen)]
    out = (seqs, stats) if return_stats else (seqs,)
    if logprobs is not None:
        out += ([_join_entries(g, e) for g, e in zip(gen, lps)],)
    return out if len(out) > 1 else seqs


@torch.no_grad()
def score_continuations(model, prompts, continuations, top_n: int = 0, use_graph: Optional[bool] = None) -> List[TokenLogprobs]:
    """Teacher-forced log-probabilities of given continuations over the compacted cache: one `TokenLogprobs` per (prompt,
    continuation) pair (1-D or [1, S] id tensors, or lists of ids; every continuation holds at least one token), for the
    continuation's tokens, with the top `top_n` (0 to 20) at each position. Each prompt is prefilled alone with its
    eviction, exactly as in `greedy_generate_batch`, whose logits score continuation[0]; the caches are joined and a
    `StaticDecoder` in forced mode takes max(len) - 1 steps, step n feeding continuation[n] through the one-token decode step
    (every cache form, the decode window included) and scoring continuation[n + 1]. Shorter continuations are padded on the
    device and trimmed here. On the greedy continuations of `greedy_generate_batch` it returns the log-probabilities that
    `greedy_generate_batch(logprobs=...)` reports: both join the caches and run the same step."""
    ids = [p.reshape(1, -1) for p in prompts]
    conts = [torch.as_tensor(c, dtype=torch.long).reshape(-1).cpu() for c in continuations]
    if not ids or len(conts) != len(ids):
        raise ValueError(f"score_continuations: {len(ids)} prompts and {len(conts)} continuations; one per prompt, at least one")
    if any(c.numel() == 0 for c in conts):
        raise ValueError("score_continuations: every continuation needs at least one token")
    top_n = _check_logprobs(top_n, "score_continuations")
    if top_n is None:
        raise ValueError("score_continuations: top_n must be an integer in [0, 20]")
    firsts, caches, entries = [], [], []
    for p, c in zip(ids, conts):
        logits, cache = _prefill_logits(model, p)
        if not all(isinstance(l, PkvCacheLayer) for l in cache.layers):
            raise RuntimeError("score_continuations needs a cache prefilled by the patched forward on every layer "
                               "(method 'fullkv' and stock caches go through model.generate)")
        first = c[:1].reshape(1, 1).to(logits.device)
        firsts.append(first)
        caches.append(cache)
        entries.append([_score(model, logits, first, top_n)])
    steps = max(c.numel() for c in conts) - 1
    cache = join_caches(caches, reserve=steps)
    del caches
    if steps:
        forced = torch.zeros(len(ids), steps, dtype=torch.long)
        for b, c in enumerate(conts):
            forced[b, : c.numel() - 1] = c[1:]
        dec = StaticDecoder(model, cache, torch.cat(firsts), steps, use_graph=use_graph, logprobs=top_n, forced=forced)
        dec.run(steps)
        lp, lp_ids, lp_top = dec.logprobs.host(steps)
        kept = [c.numel() - 1 for c in conts]
        for b, k in enumerate(kept):
            entries[b].append((lp[b, :k], lp_ids[b, :k], lp_top[b, :k]))
        dec.finish(kept)
    return [_join_entries(c, e) for c, e in zip(conts, entries)]


@torch.no_grad()
def beam_search_generate(model, prompts, max_new_tokens: int, num_beams: int, *, length_penalty: float = 1.0,
                         early_stopping=False, num_return_sequences: int = 1, eos_token_id=None,
                         use_graph: Optional[bool] = None, check_every: int = 16):
    """HF's `generate(num_beams=num_beams, do_sample=False, length_penalty=..., early_stopping=...,
    num_return_sequences=..., max_new_tokens=...)` over the compacted caches (DESIGN.md §4.12). `prompts`: one 1-D (or
    [1, S]) id tensor, or a list of them of any lengths. Each prompt is prefilled once at batch 1 (its deferred layer batch
    and FP8 conversion included); its prefill logits row gives the first step's candidates, read for each of its beams;
    its cache is joined num_beams times and all beams of all prompts decode in lock-step in `StaticDecoder`, one graph
    replay per step. A prompt is done when HF's loop would stop for it alone; its state is then frozen. The host reads the
    done flags once per `check_every` steps.

    Returns, per prompt, `num_return_sequences` hypotheses, best first: (1-D tensor of the prompt and its generated ids,
    ending in the EOS when it ended on one; its fp32 score, HF's `sequences_scores`)."""
    single = torch.is_tensor(prompts)
    ids = [p.reshape(1, -1) for p in ([prompts] if single else list(prompts))]
    if not ids:
        raise ValueError("beam_search_generate: no prompts")
    if isinstance(num_beams, bool) or int(num_beams) != num_beams or not 2 <= int(num_beams) <= MAX_BEAMS:
        raise ValueError(f"beam_search_generate: num_beams must be an integer in [2, {MAX_BEAMS}], got {num_beams!r}")
    k = int(num_beams)
    if isinstance(max_new_tokens, bool) or int(max_new_tokens) != max_new_tokens or int(max_new_tokens) < 1:
        raise ValueError(f"beam_search_generate: max_new_tokens must be an integer >= 1, got {max_new_tokens!r}")
    T = int(max_new_tokens)
    if not (early_stopping is True or early_stopping is False or early_stopping == "never"):
        raise ValueError(f"beam_search_generate: early_stopping must be True, False or 'never', got {early_stopping!r}")
    if isinstance(num_return_sequences, bool) or int(num_return_sequences) != num_return_sequences \
            or not 1 <= int(num_return_sequences) <= k:
        raise ValueError(f"beam_search_generate: num_return_sequences must be in [1, num_beams={k}], got {num_return_sequences!r}")
    if isinstance(length_penalty, bool) or not math.isfinite(float(length_penalty)):
        raise ValueError(f"beam_search_generate: length_penalty must be a finite number, got {length_penalty!r}")
    eos = eos_token_id if isinstance(eos_token_id, (list, tuple)) else ([] if eos_token_id is None else [eos_token_id])
    V = model.lm_head.weight.shape[0]
    if len(eos) > 4 or any(isinstance(e, bool) or int(e) != e or not 0 <= int(e) < V for e in eos):
        raise ValueError(f"beam_search_generate: eos_token_id must be an id in [0, {V}) or a list of at most 4, got {eos_token_id!r}")
    if len(set(int(e) for e in eos)) != len(eos):
        raise ValueError(f"beam_search_generate: eos_token_id repeats an id: {eos_token_id!r}")
    rows, caches = [], []
    for p in ids:
        logits, cache = _prefill_logits(model, p)
        if not all(isinstance(l, PkvCacheLayer) for l in cache.layers):
            raise RuntimeError("beam_search_generate needs a cache prefilled by the patched forward on every layer "
                               "(method 'fullkv' and stock caches go through model.generate)")
        rows.append(logits)
        caches.append(cache)
    backend = _backend(model)
    dev = rows[0].device
    st = BeamState(len(ids), k, T, [int(e) for e in eos], float(length_penalty), early_stopping, dev)
    st.step(backend, torch.cat(rows).contiguous(), 1, torch.zeros(1, dtype=torch.int32, device=dev), 0)   # iteration 0
    del rows
    if T > 1 and not bool(st.done.all()):
        cache = join_caches([c for c in caches for _ in range(k)], reserve=T - 1)
        del caches
        dec = StaticDecoder(model, cache, st.next_token.clone(), T - 1, use_graph=use_graph, beam=st)
        while dec.taken < T - 1:
            dec.run(min(max(1, int(check_every)), T - 1 - dec.taken))
            if bool(st.done.all()):                                  # one device-to-host read per chunk
                break
        dec.finish()
    out = []
    for p, hyps in zip(ids, st.hypotheses(int(num_return_sequences))):
        out.append([(torch.cat([p[0].cpu(), torch.tensor(g, dtype=torch.long)]).to(p.device), score) for g, score in hyps])
    return out[0] if single else out
