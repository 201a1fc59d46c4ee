"""Compacted per-layer KV cache for HF transformers 5.x `DynamicCache`.

The reference stores the evicted K/V by calling `DynamicCache.update` (HF 4.44: list append on the first
call, `torch.cat` of the WHOLE layer cache on every decode step — cache_utils_think.py:379-384) and overwrites
`past_key_value._seen_tokens` with the true sequence length (llama_model.py:172). Here the layer owns
pre-allocated buffers [bsz, H_q, capacity, D]; decode appends in place (libpkv `pkv_decode_attn`), and
`get_seq_length()` reports the number of tokens SEEN (so HF derives correct RoPE positions) while the stored
length is the compacted one.
"""
from __future__ import annotations

from typing import Optional, Tuple

import torch
from transformers.cache_utils import DynamicLayer


def _devlen_args(layer, static) -> dict:
    """The arguments of a device-length decode launch: sized for the capacity; in the static loop (generate.StaticDecoder)
    the rows also count the device step counter and the launch uses the loop's workspace."""
    return dict(step=static.step if static is not None else None, max_length=layer.capacity,
                workspace=static.workspace if static is not None else None)


class PkvCacheLayer(DynamicLayer):
    """One layer's compacted cache. keys/values are views of the valid rows of the underlying buffers."""

    is_sliding = False
    group = 1                        # query heads per cache head (> 1: a GQA-shared cache, `PkvBatchCacheLayer`)
    window = None                    # decode window R (knob `pkv_decode_window`; `PkvBatchCacheLayer` only)
    heavy = None                     # heavy hitters H in the decode window (knob `pkv_decode_heavy`; `PkvBatchCacheLayer` only)
    _BUFFERS = ("k_buf", "v_buf")    # the [B, H, capacity, ...] tensors a resize or a join copies

    def __init__(self, k_buf: torch.Tensor, v_buf: torch.Tensor, length: int, seen_tokens: int):
        super().__init__()
        assert k_buf.dim() == 4 and k_buf.shape == v_buf.shape   # [bsz, Hq, capacity, D]
        self.k_buf, self.v_buf = k_buf, v_buf
        self.length = int(length)          # valid rows per head
        self.seen_tokens = int(seen_tokens)
        self.dtype, self.device = k_buf.dtype, k_buf.device
        self.is_initialized = True
        self._refresh_views()

    # -- bookkeeping --
    @property
    def capacity(self) -> int:
        return self.k_buf.shape[2]

    @property
    def num_q_heads(self) -> int:
        return self.k_buf.shape[1] * self.group

    # -- row counts, the same view over every form --
    @property
    def rows_host(self) -> list:
        """[B][H]: the rows sequence b keeps for cache head h."""
        return [[self.length] * self.k_buf.shape[1] for _ in range(self.k_buf.shape[0])]

    @property
    def rows_dev(self) -> Optional[torch.Tensor]:
        """The same counts on the device (int32, B*H) for a kernel to read; None when every count is `length`."""
        return None

    @property
    def seq_seen(self) -> list:
        """[B]: the tokens sequence b has seen."""
        return [self.seen_tokens] * self.k_buf.shape[0]

    def _refresh_views(self) -> None:
        self.keys = self.k_buf[:, :, : self.length]
        self.values = self.v_buf[:, :, : self.length]

    def _resize(self, capacity: int) -> None:
        """New buffers of `capacity` rows per (sequence, head) holding every row of the old ones (rows the decode kernel
        appended past the host counts included)."""
        old = self.capacity
        for name in self._BUFFERS:
            t = getattr(self, name)
            nt = torch.empty((t.shape[0], t.shape[1], capacity) + tuple(t.shape[3:]), dtype=t.dtype, device=t.device)
            nt[:, :, :old] = t
            setattr(self, name, nt)
        self._refresh_views()

    def fit(self, rows: int) -> bool:
        """Make room for `rows` rows per (sequence, head) by amortised doubling (the copy happens off the per-token path).
        True when the buffers were reallocated."""
        if rows <= self.capacity:
            return False
        self._resize(max(rows, self.capacity + max(64, self.capacity // 2)))
        return True

    def reserve(self, extra_rows: int) -> None:
        """Make room for `extra_rows` more rows."""
        self.fit(self.length + extra_rows)

    def _scales(self):
        """(k_scale, v_scale) of an FP8 cache; None for 16-bit ones."""
        return None

    def decode(self, backend, q: torch.Tensor, k_new: torch.Tensor, v_new: torch.Tensor, static=None,
               softmax_scale: float = 0.0) -> torch.Tensor:
        """One decode step of every sequence: q [B, Hq, D], k_new / v_new [B, Hkv, D] (appended in place as each sequence's
        next row). Returns the attention output [B, Hq, D]. `static`: the step counter and workspace of a graph-replayable
        loop (generate.StaticDecoder), whose rows the buffers already hold; None for a host-launched step."""
        if q.shape[0] > 1:       # an equal-length batch prefilled as one forward: one launch
            return backend.decode_attn_batch(q, self.k_buf, self.v_buf, self.length + 1, k_new, v_new, rows=None,
                                             **_devlen_args(self, static), softmax_scale=softmax_scale)
        out = torch.empty(q.shape, dtype=q.dtype, device=q.device)
        # one sequence: the host-length launch (pkv_decode_attn), or the device-length one inside the static loop
        backend.decode_attn(q[0], self.k_buf[0], self.v_buf[0], self.length + 1, k_new[0], v_new[0], out[0],
                            softmax_scale=softmax_scale, **(_devlen_args(self, static) if static is not None else {}))
        return out

    def advance(self, rows: int) -> None:
        """Rows were appended in place by the decode kernel."""
        self.length += rows
        self.seen_tokens += rows
        self._refresh_views()

    # -- DynamicLayer interface --
    def lazy_initialization(self, key_states: torch.Tensor, value_states: torch.Tensor) -> None:  # pragma: no cover
        self.is_initialized = True

    def update(self, key_states: torch.Tensor, value_states: torch.Tensor, *args, **kwargs) -> Tuple[torch.Tensor, torch.Tensor]:
        """Generic append of [bsz, H, q, D] states (H == H_q, or H_kv which is repeat-expanded like
        llama_model.py:158-159). Used only off the fast path (q_len > 1 after prefill)."""
        q = key_states.shape[2]
        hq = self.k_buf.shape[1]
        if key_states.shape[1] != hq:
            rep = hq // key_states.shape[1]
            key_states = key_states.repeat_interleave(rep, dim=1)
            value_states = value_states.repeat_interleave(rep, dim=1)
        self.reserve(q)
        self.k_buf[:, :, self.length: self.length + q] = key_states
        self.v_buf[:, :, self.length: self.length + q] = value_states
        self.advance(q)
        return self.keys, self.values

    def get_seq_length(self) -> int:
        # tokens seen, not rows stored: the reference sets past_key_value._seen_tokens = self.kv_seq_len (llama_model.py:172)
        return self.seen_tokens

    def get_mask_sizes(self, query_length: int) -> Tuple[int, int]:
        return self.length + query_length, 0

    def get_max_cache_shape(self) -> int:
        return -1

    def crop(self, max_length: int) -> None:
        raise NotImplementedError("cropping a compacted cache is undefined (rows are in score order, not position order)")

    def batch_repeat_interleave(self, repeats: int) -> None:
        self.k_buf = self.k_buf.repeat_interleave(repeats, dim=0)
        self.v_buf = self.v_buf.repeat_interleave(repeats, dim=0)
        self._refresh_views()

    def batch_select_indices(self, indices: torch.Tensor) -> None:
        self.k_buf = self.k_buf[indices, ...]
        self.v_buf = self.v_buf[indices, ...]
        self._refresh_views()


class PkvRaggedCacheLayer(PkvCacheLayer):
    """AdaKV / HeadKV: every head keeps its own number of rows. The reference stores ONE flat [sum_h len_h, D] tensor per
    layer and rebuilds it on every decoded token (DynamicCacheSplitHeadFlatten.update + update_flatten_view,
    pyramidkv_utils.py:52-74); here the buffers stay padded [1, Hq, capacity, D], `head_rows` (int32 [Hq], device) holds the
    rows of each head after the prefill, and decode appends row head_rows[h] + t of every head in place. `length` is the
    LONGEST head's row count (what the buffers must hold); `appended` the tokens decoded so far."""

    def __init__(self, k_buf: torch.Tensor, v_buf: torch.Tensor, head_rows_host, seen_tokens: int):
        if k_buf.shape[0] != 1:
            raise NotImplementedError("ragged caches are batch size 1; join them (cache.join_caches) to decode them together")
        self.head_rows_host = [int(r) for r in head_rows_host]
        self.base_rows = max(self.head_rows_host)
        self.head_rows = torch.tensor(self.head_rows_host, dtype=torch.int32, device=k_buf.device)
        super().__init__(k_buf, v_buf, self.base_rows, seen_tokens)

    @property
    def appended(self) -> int:
        return self.length - self.base_rows

    @property
    def rows_host(self) -> list:
        return [[r + self.appended for r in self.head_rows_host]]

    @property
    def rows_dev(self) -> torch.Tensor:
        return self.head_rows + self.appended if self.appended else self.head_rows

    def decode(self, backend, q, k_new, v_new, static=None, softmax_scale: float = 0.0) -> torch.Tensor:
        # pkv_decode_attn_ragged: row head_rows[h] + appended + 1 (+ the step counter in the static loop)
        out = torch.empty(q.shape, dtype=q.dtype, device=q.device)
        backend.decode_attn(q[0], self.k_buf[0], self.v_buf[0], self.appended + 1, k_new[0], v_new[0], out[0],
                            softmax_scale=softmax_scale, head_rows=self.head_rows, **_devlen_args(self, static))
        return out

    def head_view(self, h: int):
        """Valid rows of head h: ([rows_h, D] keys, values) of batch 0."""
        r = self.head_rows_host[h] + self.appended
        return self.k_buf[0, h, :r], self.v_buf[0, h, :r]

    def update(self, key_states, value_states, *args, **kwargs):
        raise NotImplementedError("multi-token append to a ragged (AdaKV / HeadKV) cache is not defined by the reference "
                                  "(its decode path asserts seqlen == 1, pyramidkv_utils.py:58-59)")

    def batch_repeat_interleave(self, repeats: int) -> None:
        raise NotImplementedError("ragged caches are batch size 1 (pyramidkv_utils.py:723)")

    def batch_select_indices(self, indices: torch.Tensor) -> None:
        raise NotImplementedError("ragged caches are batch size 1 (pyramidkv_utils.py:723)")


class PkvBatchCacheLayer(PkvCacheLayer):
    """The compacted caches of B prompts, prefilled one at a time and joined (`join_caches`), decoded together: buffers
    [B, Hq, capacity, D], `rows_host[b][h]` the rows sequence b keeps for head h (prompts shorter than the budget keep
    every row; AdaKV / HeadKV heads differ) and `rows` the same counts on the device (int32 [B*Hq], what
    `pkv_decode_attn_batch` adds to its row count). Decode appends one row to every sequence per step; `settle` books the
    rows each sequence really kept (a sequence that stopped at its EOS keeps fewer). `length` is the longest (sequence,
    head)'s row count (what the buffers must hold); `seq_seen[b]` the tokens sequence b has seen.

    `group` G > 1: a GQA-shared cache (knob `pkv_gqa_shared`): one cache per KV head, [B, Hkv, capacity, D], read once for
    the G query heads of its group (`pkv_decode_attn_batch_gqa`); `rows_host[b][j]` counts KV head j's rows. G = 1 (the
    default) is the per-query-head cache.

    `window` R (knob `pkv_decode_window`): (sequence b, head h) keeps its `prompt_rows_host[b][h]` = P prompt rows and a ring
    of its last R appended rows, the j-th at row P + j mod R (`pkv_decode_attn_window`). `generated[b]` counts the rows
    sequence b appended; `rows_host[b][h]` = P + min(generated[b], R) are the rows the buffers hold, in ring order (not
    token order) past P, while the device `rows` hold the logical counts P + generated[b] the kernel derives the ring slot
    from. `prompt_rows` is the device copy of P (int32 [B*H]). None: no window.

    `heavy` H (knob `pkv_decode_heavy`, with a window): once the window is full the new row replaces the generated row with
    the least accumulated attention among all but the R - H - 1 most recent (`pkv_decode_attn_heavy`). The layer's state,
    updated on the device by every step: `heavy_scores` fp32 [B, H, R] and `heavy_gen` int32 [B, H, R] (the accumulated
    attention and the generation index of the row in each slot past P) and `victim` int32 [B*H] (the row the next step
    replaces). Slots still fill in order and are then replaced in place, so `rows_host` is the window's. None: the ring."""

    rows_host = seq_seen = None    # held per sequence here (set in __init__), not derived from `length` as in the base class

    def __init__(self, k_buf: torch.Tensor, v_buf: torch.Tensor, rows_host, seq_seen, group: int = 1, window: Optional[int] = None,
                 prompt_rows=None, generated=None, heavy: Optional[int] = None, heavy_state=None):
        self.group = int(group)
        self.rows_host = [[int(r) for r in row] for row in rows_host]
        self.seq_seen = [int(s) for s in seq_seen]
        assert len(self.rows_host) == len(self.seq_seen) == k_buf.shape[0] and all(len(r) == k_buf.shape[1] for r in self.rows_host)
        self.window = None if window is None else int(window)
        if self.window is not None:
            # a cache that enters the window with rows of its own (the prefill's, or a joined cache's) counts them as its prompt
            self.prompt_rows_host = [list(r) for r in (prompt_rows if prompt_rows is not None else self.rows_host)]
            self.generated = [int(g) for g in generated] if generated is not None else [0] * len(self.rows_host)
            self.prompt_rows = self._device_counts(self.prompt_rows_host, k_buf.device)
        self.heavy = None if heavy is None else int(heavy)
        if self.heavy is not None:
            assert self.window is not None and 0 <= self.heavy < self.window
            B, H = k_buf.shape[:2]
            if heavy_state is None:    # a new cache: nothing generated yet, so no slot is read before the step that fills it
                heavy_state = (torch.zeros(B, H, self.window, dtype=torch.float32, device=k_buf.device),
                               torch.full((B, H, self.window), -1, dtype=torch.int32, device=k_buf.device),
                               torch.full((B * H,), -1, dtype=torch.int32, device=k_buf.device))
            self.heavy_scores, self.heavy_gen, self.victim = heavy_state
        self.rows = self._device_rows(k_buf.device)
        super().__init__(k_buf, v_buf, max(max(r) for r in self.rows_host), max(self.seq_seen))

    @property
    def rows_dev(self) -> Optional[torch.Tensor]:
        if self.window is not None:      # the rows the buffers hold (the device `rows` are the logical counts)
            return self._device_counts(self.rows_host, self.device)
        return None if all(r == self.length for row in self.rows_host for r in row) else self.rows

    @staticmethod
    def _device_counts(rows, device) -> torch.Tensor:
        return torch.tensor([r for row in rows for r in row], dtype=torch.int32, device=device)

    def _device_rows(self, device) -> torch.Tensor:
        if self.window is None:
            return self._device_counts(self.rows_host, device)
        return self._device_counts([[p + g for p in row] for row, g in zip(self.prompt_rows_host, self.generated)], device)

    def settle(self, appended) -> None:
        """Sequence b appended `appended[b]` rows to every head (in place, by the decode kernel). With a window the buffers
        hold P + min(generated, R) of them."""
        assert len(appended) == len(self.rows_host)
        for b, n in enumerate(appended):
            if self.window is None:
                self.rows_host[b] = [r + int(n) for r in self.rows_host[b]]
            else:
                self.generated[b] += int(n)
                self.rows_host[b] = [p + min(self.generated[b], self.window) for p in self.prompt_rows_host[b]]
            self.seq_seen[b] += int(n)
        self.rows = self._device_rows(self.device)     # a new tensor: launches already queued keep reading the old one
        self.length = max(max(r) for r in self.rows_host)
        self.seen_tokens = max(self.seq_seen)
        self._refresh_views()

    def reserve(self, extra_rows: int) -> None:
        """Make room for `extra_rows` more appended rows; with a window never more than P + R rows per (sequence, head)."""
        if self.window is None:
            return super().reserve(extra_rows)
        self.fit(max(p + min(g + int(extra_rows), self.window)
                     for row, g in zip(self.prompt_rows_host, self.generated) for p in row))

    def advance(self, rows: int) -> None:
        self.settle([rows] * len(self.rows_host))

    def head_view(self, b: int, h: int):
        """Valid rows of sequence b, head h: ([rows, D] keys, values)."""
        r = self.rows_host[b][h]
        return self.k_buf[b, h, :r], self.v_buf[b, h, :r]

    def decode(self, backend, q, k_new, v_new, static=None, softmax_scale: float = 0.0) -> torch.Tensor:
        # rows = layer.rows[b, h] + 1 (+ the step counter in the static loop); G > 1: each KV head read once for its group
        if self.heavy is not None:
            return backend.decode_attn_heavy(q, self.k_buf, self.v_buf, 1, k_new, v_new, self.prompt_rows, self.window, self.heavy,
                                             self.heavy_scores, self.heavy_gen, self.victim, rows=self.rows,
                                             **_devlen_args(self, static), scratch=getattr(static, "heavy_scratch", None),
                                             softmax_scale=softmax_scale, scales=self._scales(), gqa=self.group > 1)
        if self.window is not None:
            return backend.decode_attn_window(q, self.k_buf, self.v_buf, 1, k_new, v_new, self.prompt_rows, self.window,
                                              rows=self.rows, **_devlen_args(self, static), softmax_scale=softmax_scale,
                                              scales=self._scales(), gqa=self.group > 1)
        fn = backend.decode_attn_batch_gqa if self.group > 1 else backend.decode_attn_batch
        return fn(q, self.k_buf, self.v_buf, 1, k_new, v_new, rows=self.rows, **_devlen_args(self, static),
                  softmax_scale=softmax_scale)

    # -- continuous batching (generate.ContinuousDecoder): one slot rewritten in place while a decode graph holds the buffers --
    def admit(self, slot: int, src_layer, step: torch.Tensor, backend=None) -> None:
        """Copy the single-prompt layer `src_layer` (the form this batch holds: `PkvCacheLayer` / `PkvRaggedCacheLayer`, or,
        for a GQA-shared or FP8 batch, a batch-1 layer of the same group and dtype) into slot `slot`, and set the slot's
        device row counts to src rows - *step, so that the next decode step appends after them (`pkv_cache_install`). Every
        write is in place; `rows_host[slot]` and `seq_seen[slot]` follow."""
        _install([self], slot, [src_layer], step, backend)

    def park(self, slot: int, step: torch.Tensor, backend=None) -> None:
        """Leave slot `slot` empty: its device row counts become -*step, so a decode step attends and overwrites one row."""
        _install([self], slot, None, step, backend)

    def grow(self, capacity: int) -> None:
        """New buffers of `capacity` rows per (sequence, head) holding every row of the old ones (the rows the decode kernel
        appended included). `rows` stays the same tensor; a decode graph over the old buffers must be captured again."""
        if capacity > self.capacity:
            self._resize(capacity)

    def _install_item(self, slot: int, src):
        """(the `cache_install` tuple of this layer, the slot's host row counts, its tokens seen)."""
        B, H, _, D = self.k_buf.shape
        if not 0 <= int(slot) < B:
            raise ValueError(f"slot {slot} outside [0, {B})")
        dst = (self.k_buf, self.v_buf, self._scales(), self.rows)
        if src is None:
            return (None, None, None, 0, None, *dst), [0] * H, 0
        if not isinstance(src, PkvCacheLayer) or _form(src) != _form(self):
            raise ValueError(f"admit: a {type(src).__name__} (group {getattr(src, 'group', 1)}, decode window "
                             f"{getattr(src, 'window', None)}, heavy hitters {getattr(src, 'heavy', None)}) cannot enter a "
                             f"{type(self).__name__} of group {self.group}, decode window {self.window}, heavy hitters "
                             f"{self.heavy}: FP8 and 16-bit caches, and caches of different groups, decode windows or heavy "
                             "hitters (pkv_decode_heavy), do not mix")
        if src.k_buf.shape[0] != 1 or src.k_buf.shape[1] != H or src.k_buf.shape[3] != D or src.dtype != self.dtype \
                or src.device != self.device:
            raise ValueError(f"admit: the source must be one prompt of {H} heads, head_dim {D}, {self.dtype} on {self.device}; "
                             f"got {tuple(src.k_buf.shape)} {src.dtype} on {src.device}")
        rows_host = src.rows_host[0]
        n = max(rows_host)
        if n > self.capacity:
            raise ValueError(f"admit: {n} rows exceed the capacity {self.capacity} (grow the batch first)")
        return (src.k_buf, src.v_buf, src._scales(), n, src.rows_dev, *dst), rows_host, src.seq_seen[0]

    def _reorder_item(self):
        """(the `cache_reorder` tuple of this layer): the rows and their scales, the row of each (sequence, head)'s
        generated slot 0 (its prompt rows), the decode window and the heavy-hitter state."""
        ks, vs = self._scales() or (None, None)
        base = self.prompt_rows if self.window is not None else self.rows
        heavy = None if self.heavy is None else (self.heavy_scores, self.heavy_gen, self.victim)
        return self.k_buf, self.v_buf, ks, vs, base, self.window, heavy

    def _book(self, slot: int, rows_host, seen: int) -> None:
        self.rows_host[slot] = list(rows_host)
        self.seq_seen[slot] = int(seen)
        if self.window is not None:
            # the admitted rows are the slot's prompt (a parked slot: none); written in place for a captured decode graph
            H = len(rows_host)
            self.prompt_rows_host[slot] = list(rows_host)
            self.generated[slot] = 0
            self.prompt_rows[slot * H:(slot + 1) * H].copy_(torch.tensor(rows_host, dtype=torch.int32))
        if self.heavy is not None:
            # a new sequence starts with no generated rows; reset in place, where a captured decode graph reads the state
            self.heavy_scores[slot].zero_()
            self.heavy_gen[slot].fill_(-1)
            self.victim[slot * len(rows_host):(slot + 1) * len(rows_host)].fill_(-1)
        self.length = max(max(r) for r in self.rows_host)
        self.seen_tokens = max(self.seq_seen)
        self._refresh_views()

    def update(self, key_states, value_states, *args, **kwargs):
        if self.window is not None:
            raise NotImplementedError("multi-token append under the decode window (pkv_decode_window) is not built: decode one "
                                      "token per step")
        raise NotImplementedError("multi-token append to a joined batch is not defined: its sequences hold different row counts "
                                  "(decode it one token per step: generate.StaticDecoder / greedy_generate_batch)")

    def batch_repeat_interleave(self, repeats: int) -> None:
        raise NotImplementedError("a joined batch holds one row count per sequence and head; repeat the prompts before joining")

    def batch_select_indices(self, indices: torch.Tensor) -> None:
        raise NotImplementedError("a joined batch holds one row count per sequence and head; join the selected prompts instead")


KV_CACHE_DTYPES = (None, "fp8_e4m3")   # model.config.pkv_kv_cache_dtype


def kv_cache_dtype(config) -> Optional[str]:
    """The knob `pkv_kv_cache_dtype` of a model config: None (the default: the 16-bit cache) or "fp8_e4m3"."""
    v = getattr(config, "pkv_kv_cache_dtype", None)
    v = None if v == "auto" else v
    if v not in KV_CACHE_DTYPES:
        raise ValueError(f"pkv_kv_cache_dtype={v!r}: expected None or 'fp8_e4m3'")
    return v


def decode_window(config) -> Optional[int]:
    """The knob `pkv_decode_window` of a model config: None (the default: every decoded row stays) or R >= 1, the decoded rows
    each sequence keeps behind its compacted prompt (the oldest is overwritten first)."""
    v = getattr(config, "pkv_decode_window", None)
    if v is None:
        return None
    if isinstance(v, bool) or not isinstance(v, int) or v < 1:
        raise ValueError(f"pkv_decode_window={v!r}: expected None or an int >= 1")
    return int(v)


def decode_heavy(config) -> Optional[int]:
    """The knob `pkv_decode_heavy` of a model config: None (the default: the decode window replaces its oldest row) or H, an
    int with 1 <= H <= R - 1 under `pkv_decode_window` = R: the window keeps its R - H most recent generated rows, and each
    new row replaces the one with the least accumulated attention among the others (H2O's heavy hitters, DESIGN.md §4.9)."""
    v = getattr(config, "pkv_decode_heavy", None)
    if v is None:
        return None
    window = decode_window(config)
    if window is None:
        raise ValueError(f"pkv_decode_heavy={v!r} needs the decode window (pkv_decode_window = R)")
    if isinstance(v, bool) or not isinstance(v, int) or not 1 <= v <= window - 1:
        raise ValueError(f"pkv_decode_heavy={v!r}: expected None or an int in [1, R - 1] = [1, {window - 1}]")
    return int(v)


def gqa_shared(config) -> bool:
    """The knob `pkv_gqa_shared` of a model config (default False): one selection and one compacted cache per KV head."""
    v = getattr(config, "pkv_gqa_shared", False)
    if v not in (False, True, None, 0, 1):
        raise ValueError(f"pkv_gqa_shared={v!r}: expected True or False")
    return bool(v)


class PkvFp8CacheLayer(PkvBatchCacheLayer):
    """The compacted cache in FP8 (knob `pkv_kv_cache_dtype = "fp8_e4m3"`): `k_buf` / `v_buf` hold E4M3 bytes
    (torch.float8_e4m3fn [B, Hq, capacity, D]) and `k_scale` / `v_scale` one fp32 scale per (sequence, head, row)
    ([B, Hq, capacity]); row x of the 16-bit cache is stored as round(x * 448 / max|x|) and stands for its bytes times
    the scale max|x| / 448 (include/pkv.h, pkv_cache_quantize_fp8). Half the bytes of the 16-bit cache plus 8 bytes per
    row and head. Always in the per-(sequence, head) row-count form of `PkvBatchCacheLayer`, so one class holds a single
    prompt, an equal-length batch, AdaKV / HeadKV heads of different lengths and joined prompts. Decode appends one
    quantised row per sequence and step (`pkv_decode_attn_batch_fp8`)."""

    _BUFFERS = ("k_buf", "v_buf", "k_scale", "v_scale")

    def __init__(self, k_q: torch.Tensor, v_q: torch.Tensor, k_scale: torch.Tensor, v_scale: torch.Tensor, rows_host, seq_seen,
                 group: int = 1, **window):
        assert k_q.dtype == torch.float8_e4m3fn and k_scale.shape == k_q.shape[:3] and v_scale.shape == k_scale.shape
        self.k_scale, self.v_scale = k_scale, v_scale
        super().__init__(k_q, v_q, rows_host, seq_seen, group, **window)

    def _scales(self):
        return self.k_scale, self.v_scale

    def decode(self, backend, q, k_new, v_new, static=None, softmax_scale: float = 0.0) -> torch.Tensor:
        # the kernel quantises the new K / V row and attends it as stored
        if self.window is not None:
            return super().decode(backend, q, k_new, v_new, static, softmax_scale)
        fn = backend.decode_attn_batch_gqa_fp8 if self.group > 1 else backend.decode_attn_batch_fp8
        return fn(q, self.k_buf, self.v_buf, self.k_scale, self.v_scale, 1, k_new, v_new, rows=self.rows,
                  **_devlen_args(self, static), softmax_scale=softmax_scale)

    @staticmethod
    def dequantize(q: torch.Tensor, scale: torch.Tensor) -> torch.Tensor:
        """float32 rows: bytes times the row scale."""
        return q.float() * scale[..., None]

    def head_view(self, b: int, h: int):
        """Dequantised valid rows of sequence b, head h: ([rows, D] float32 keys, values)."""
        r = self.rows_host[b][h]
        return (self.dequantize(self.k_buf[b, h, :r], self.k_scale[b, h, :r]),
                self.dequantize(self.v_buf[b, h, :r], self.v_scale[b, h, :r]))

    def update(self, key_states, value_states, *args, **kwargs):
        raise NotImplementedError("multi-token append to an FP8 cache is not built: decode it one token per step (the FP8 "
                                  "cache covers the decode path; prefill and the multi-token path stay 16-bit)")

    def batch_repeat_interleave(self, repeats: int) -> None:
        raise NotImplementedError("an FP8 cache holds one row count per sequence and head (beam search over FP8 caches is "
                                  "not built); repeat the prompts before joining")

    def batch_select_indices(self, indices: torch.Tensor) -> None:
        raise NotImplementedError("an FP8 cache holds one row count per sequence and head; join the selected prompts instead")


def quantize_caches_fp8(past_key_values, backend) -> int:
    """Convert every compacted layer of `past_key_values` (`PkvCacheLayer` / `PkvRaggedCacheLayer`, or a GQA-shared
    `PkvBatchCacheLayer`, filled by the patched prefill) to a `PkvFp8CacheLayer` with ONE backend call
    (`pkv_cache_quantize_fp8`: one launch per 32 layers; a GQA-shared cache converts its Hkv heads) and drop the 16-bit
    buffers. The FP8 buffers keep each layer's capacity (the decode head-room included). Returns the number of layers
    converted."""
    idx, items, metas = [], [], []
    for i, l in enumerate(past_key_values.layers):
        if not isinstance(l, PkvCacheLayer) or isinstance(l, PkvFp8CacheLayer):
            continue
        B, H, cap, D = l.k_buf.shape
        kq = torch.empty(B, H, cap, D, dtype=torch.float8_e4m3fn, device=l.device)
        vq = torch.empty_like(kq)
        ks = torch.empty(B, H, cap, dtype=torch.float32, device=l.device)
        vs = torch.empty_like(ks)
        items.append((l.k_buf, l.v_buf, kq, vq, ks, vs, l.length, l.rows_dev))
        metas.append(((kq, vq, ks, vs, l.rows_host, l.seq_seen, l.group), _window_args(l)))
        idx.append(i)
    if items:
        backend.cache_quantize_fp8(items)
    for i, (m, w) in zip(idx, metas):
        past_key_values.layers[i] = PkvFp8CacheLayer(*m, **w)
    return len(idx)


def _form(layer) -> tuple:
    """What decides whether two compacted layers may share a batch: FP8 or 16-bit, the group (GQA-shared caches) and the
    decode window with its heavy hitters."""
    return isinstance(layer, PkvFp8CacheLayer), layer.group, layer.window, layer.heavy


def _window_args(layer) -> dict:
    """The decode-window state of a layer (with its heavy-hitter state) as `PkvBatchCacheLayer` keyword arguments."""
    if layer.window is None:
        return {}
    heavy = {} if layer.heavy is None else dict(heavy=layer.heavy, heavy_state=(layer.heavy_scores, layer.heavy_gen, layer.victim))
    return dict(window=layer.window, prompt_rows=layer.prompt_rows_host, generated=layer.generated, **heavy)


def join_caches(caches, reserve: int = 0):
    """One batched cache from B single-prompt caches filled by the patched prefill (every layer a batch-1 `PkvCacheLayer` or
    `PkvRaggedCacheLayer`): layer by layer the valid rows are copied once into [B, Hq, longest + reserve, D] buffers
    (`PkvBatchCacheLayer`). A cache may be passed several times. Stock / FullKV caches raise. Single-prompt FP8 caches
    (`PkvFp8CacheLayer`) join the same way, bytes and scales copied once, into a `PkvFp8CacheLayer`; FP8 and 16-bit
    caches do not mix. GQA-shared caches (knob `pkv_gqa_shared`, `group` > 1) join into a layer of the same group; caches of
    different groups do not mix either."""
    from transformers import DynamicCache
    if not caches:
        raise ValueError("join_caches: no caches")
    n_layers = len(caches[0].layers)
    layers = [l for c in caches for l in c.layers]
    if any(len(c.layers) != n_layers for c in caches) or not all(isinstance(l, PkvCacheLayer) for l in layers):
        raise RuntimeError("join_caches needs caches prefilled by the patched forward on every layer "
                           "(method 'fullkv' and stock caches are not compacted)")
    forms = {_form(l) for l in layers}
    if len({form[2:] for form in forms}) > 1:
        raise ValueError("join_caches: caches of different decode windows cannot be joined together (set pkv_decode_window and "
                         "pkv_decode_heavy the same for every prompt)")
    if len({form[1] for form in forms}) > 1:
        raise ValueError("join_caches: GQA-shared and per-query-head caches (or caches of different groups) cannot be joined "
                         "together (set pkv_gqa_shared the same for every prompt)")
    if len(forms) > 1:
        raise ValueError("join_caches: FP8 and 16-bit caches cannot be joined together (set pkv_kv_cache_dtype the same "
                         "for every prompt)")
    if any(l.k_buf.shape[0] != 1 for l in layers):
        raise ValueError("join_caches joins single-prompt (batch 1) caches")
    out = DynamicCache()
    out.layers = []
    for i in range(n_layers):
        src = [c.layers[i] for c in caches]
        l0 = src[0]
        _, h, _, d = l0.k_buf.shape
        if any(l.k_buf.shape[1] != h or l.k_buf.shape[3] != d or l.dtype != l0.dtype or l.device != l0.device for l in src):
            raise ValueError(f"join_caches: layer {i}: head counts, head_dim, dtype or device differ between the caches")
        rows = [l.rows_host[0] for l in src]
        cap = max(max(r) for r in rows) + int(reserve)
        if l0.window is not None:    # at most P + R rows per (sequence, head)
            cap = max(p + min(l.generated[0] + int(reserve), l.window) for l in src for p in l.prompt_rows_host[0])
        bufs = []
        for name in l0._BUFFERS:
            t0 = getattr(l0, name)
            t = torch.empty((len(src), h, cap) + tuple(t0.shape[3:]), dtype=t0.dtype, device=t0.device)
            for b, l in enumerate(src):
                t[b, :, : l.length] = getattr(l, name)[0, :, : l.length]
            bufs.append(t)
        cls = type(l0) if isinstance(l0, PkvBatchCacheLayer) else PkvBatchCacheLayer
        win = {}
        if l0.window is not None:
            win = dict(window=l0.window, prompt_rows=[l.prompt_rows_host[0] for l in src], generated=[l.generated[0] for l in src])
            if l0.heavy is not None:
                win.update(heavy=l0.heavy, heavy_state=(torch.cat([l.heavy_scores for l in src]), torch.cat([l.heavy_gen for l in src]),
                                                        torch.cat([l.victim for l in src])))
        out.layers.append(cls(*bufs, rows, [l.seq_seen[0] for l in src], l0.group, **win))
    return out


def _install(layers, slot: int, sources, step: torch.Tensor, backend=None) -> None:
    """Admit `sources[i]` (None: park) into slot `slot` of `layers[i]`, all layers in ONE backend call (`pkv_cache_install`:
    one launch per 32 layers), then update the host mirrors."""
    if backend is None:
        from .kv_cluster import _default_backend as backend
    items, books = [], []
    for i, l in enumerate(layers):
        if not isinstance(l, PkvBatchCacheLayer):
            raise ValueError(f"layer {i}: slots are admitted into batched caches (join_caches), not into a {type(l).__name__}")
        item, rows_host, seen = l._install_item(slot, None if sources is None else sources[i])
        items.append(item)
        books.append((rows_host, seen))
    backend.cache_install(items, int(slot), step)
    for l, (rows_host, seen) in zip(layers, books):
        l._book(int(slot), rows_host, seen)


def admit_cache(batch, slot: int, src, step: torch.Tensor, backend=None) -> None:
    """`PkvBatchCacheLayer.admit` for every layer of the batched cache `batch` from the single-prompt cache `src` (both
    DynamicCaches), in one launch."""
    if len(src.layers) != len(batch.layers):
        raise ValueError(f"admit: the source has {len(src.layers)} layers, the batch {len(batch.layers)}")
    _install(batch.layers, slot, list(src.layers), step, backend)


def park_cache(batch, slot: int, step: torch.Tensor, backend=None) -> None:
    """`PkvBatchCacheLayer.park` for every layer of the batched cache `batch`, in one launch."""
    _install(batch.layers, slot, None, step, backend)


def reorder_caches(batch, num_prompts: int, num_beams: int, parent: torch.Tensor, diverge: torch.Tensor, step: torch.Tensor,
                   step_offset: int, backend=None) -> None:
    """Beam search: sequence p * num_beams + a of the batched cache `batch` (`join_caches` of each prompt's cache
    num_beams times) takes the generated rows of sequence p * num_beams + parent[..] from row diverge[..] on, in every
    layer, in one launch per 32 layers (`pkv_cache_reorder`; n = *step + step_offset generated rows, read on the device)."""
    if backend is None:
        from .kv_cluster import _default_backend as backend
    for i, l in enumerate(batch.layers):
        if not isinstance(l, PkvBatchCacheLayer):
            raise ValueError(f"layer {i}: beams are reordered in batched caches (join_caches), not in a {type(l).__name__}")
    backend.cache_reorder([l._reorder_item() for l in batch.layers], num_prompts, num_beams, parent, diverge, step,
                          step_offset)


def layer_is_empty(past_key_values, layer_idx: int) -> bool:
    """Prefill detection = "this layer's cache is empty" (the reference compares key length with the
    per-module `kv_seq_len` counter that `prepare_inputs_for_generation` resets — llama_model.py:165, :2609-2612)."""
    layers = getattr(past_key_values, "layers", None)
    if layers is None or layer_idx >= len(layers):
        return True
    layer = layers[layer_idx]
    if isinstance(layer, PkvCacheLayer):
        return layer.length == 0
    return layer.get_seq_length() == 0


def install_layer(past_key_values, layer_idx: int, layer: PkvCacheLayer) -> None:
    layers = past_key_values.layers
    cls = getattr(past_key_values, "layer_class_to_replicate", None)
    while len(layers) <= layer_idx:
        layers.append(cls() if cls is not None else DynamicLayer())
    layers[layer_idx] = layer
