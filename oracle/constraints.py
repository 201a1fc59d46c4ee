"""The generation constraints of DESIGN.md §4.11 restated in numpy, one row at a time: HF's SequenceBiasLogitsProcessor,
NoRepeatNGramLogitsProcessor, NoBadWordsLogitsProcessor and MinNewTokensLengthLogitsProcessor (transformers 5.5) and a
stop-sequence criterion, each as the fp32 operation the processor performs. `history` is the row's ids: its prompt, then
every token generated so far; `prompt_len` its prompt's length."""
import numpy as np


def _applies(history, seq) -> bool:
    """HF's SequenceBias test: a single-token sequence always applies; a longer one when it is no longer than the history
    and its first L - 1 tokens are the last L - 1 of the history."""
    L = len(seq)
    if L == 1:
        return True
    return L <= len(history) and list(history[len(history) - (L - 1):]) == list(seq[:-1])


def sequence_bias(history, pairs, vocab: int) -> np.ndarray:
    """The fp32 bias row: zeros, plus the single-token biases, plus, in the pairs' order, b (when the sequence applies)
    or 0.0 at each longer sequence's last token."""
    bias = np.zeros(vocab, np.float32)
    for seq, b in pairs:
        if len(seq) == 1:
            bias[seq[0]] = np.float32(bias[seq[0]] + np.float32(b))
    for seq, b in pairs:
        if len(seq) == 1 or len(seq) > len(history):
            continue
        bias[seq[-1]] = np.float32(bias[seq[-1]] + (np.float32(b) if _applies(history, seq) else np.float32(0.0)))
    return bias


def ngram_bans(history, n: int, vocab: int) -> np.ndarray:
    """The tokens no_repeat_ngram_size = n bans: the last token of every n-gram of the history whose first n - 1 tokens
    are the history's last n - 1 (nothing while len(history) + 1 < n)."""
    ban = np.zeros(vocab, bool)
    h = np.asarray(history, np.int64)
    if n <= 0 or h.size < n:
        return ban
    win = np.lib.stride_tricks.sliding_window_view(h, n)
    hit = (win[:, : n - 1] == h[h.size - n + 1:]).all(axis=1)
    ban[win[hit, n - 1]] = True
    return ban


def bad_word_bans(history, bad_words, eos, vocab: int) -> np.ndarray:
    """The tokens the bad words add -inf to: the last token of each that applies, single-token EOS ids dropped."""
    eos = set(eos or ())
    ban = np.zeros(vocab, bool)
    for seq in bad_words:
        if len(seq) == 1 and seq[0] in eos:
            continue
        if _applies(history, seq):
            ban[seq[-1]] = True
    return ban


def min_new_bans(history, prompt_len: int, min_new: int, eos, vocab: int) -> np.ndarray:
    ban = np.zeros(vocab, bool)
    if eos and len(history) - prompt_len < min_new:
        ban[[e for e in eos if 0 <= e < vocab]] = True
    return ban


def stopped(history, stop_sequences) -> bool:
    """A stop sequence equals the history's last tokens."""
    h = list(history)
    return any(len(s) <= len(h) and h[len(h) - len(s):] == list(s) for s in stop_sequences)


def add_bias(x, bias) -> np.ndarray:
    return (np.asarray(x, np.float32) + bias).astype(np.float32)


def apply_bans(x, set_ban, add_ban=None) -> np.ndarray:
    """Set the `set_ban` tokens to -inf; with `add_ban` (bad words on), add -inf there and 0 elsewhere."""
    x = np.asarray(x, np.float32).copy()
    if add_ban is not None:
        with np.errstate(invalid="ignore"):
            x = (x + np.where(add_ban, np.float32(-np.inf), np.float32(0.0))).astype(np.float32)
    x[set_ban] = -np.inf
    return x

