"""Runner layer: the callers that sit on either side of the eviction path (SURVEY.md §8 row f1).

`run_longbench.py` and `run_needle_in_haystack.py` at the repo root expose the reference's command lines
(run_longbench.py:321-366, run_needle_in_haystack.py:498-529, scripts/scripts_needle/eval.sh:18-26) on top of this
module. There is no network in the build/test boxes, so checkpoints, tokenizers and the LongBench / needle corpora are
replaced by what the reference's own flow reduces to for timing purposes: a random-init model of the named
architecture (seed 42, the runners' seed) and synthetic token-id prompts of the dataset's typical length. What is kept
exactly is the plugin sequence of the reference runners:

    replace_llama(method); replace_mistral(method)            # run_longbench.py:382-384
    per layer: self_attn.config.{window_size, max_capacity_prompt, kernel_size, pooling, merge}   # :253-261
    model.generate(..., max_new_tokens=N, num_beams=1, do_sample=False)                            # :264-275

Every prompt yields one record: prompt length, tokens generated, prefill ms (generate with one new token), decode
tok/s over the remaining tokens, compacted cache rows of the first / last layer.
"""
from __future__ import annotations

import contextlib
import io
import sys
import json
import os
import time
from dataclasses import dataclass
from typing import Callable, Dict, Iterable, List, Optional

import torch

# name -> (family, hidden, intermediate, layers, q heads, kv heads, head_dim, vocab, rope_theta)
ARCHS: Dict[str, tuple] = {
    "llama3-8b": ("llama", 4096, 14336, 32, 32, 8, 128, 128256, 5e5),
    "llama3-70b": ("llama", 8192, 28672, 80, 64, 8, 128, 128256, 5e5),
    "mistral-7b-v0.2": ("mistral", 4096, 14336, 32, 32, 8, 128, 32000, 1e6),
    "tiny-llama": ("llama", 512, 1024, 4, 8, 2, 64, 1024, 5e5),
    "tiny-mistral": ("mistral", 512, 1024, 4, 8, 2, 64, 1024, 1e6),
}

# LongBench task -> (typical prompt tokens, max_new_tokens). Lengths are round figures of the corpus statistics; the
# generation lengths are the per-task caps the reference applies (run_longbench.py dataset2maxlen).
LONGBENCH_SHAPES: Dict[str, tuple] = {
    "narrativeqa": (18000, 128), "qasper": (3600, 128), "multifieldqa_en": (4600, 64), "hotpotqa": (9200, 32),
    "2wikimqa": (4900, 32), "musique": (11200, 32), "gov_report": (8700, 512), "qmsum": (10600, 512),
    "multi_news": (2100, 512), "trec": (5200, 64), "triviaqa": (8200, 32), "samsum": (6300, 128),
    "passage_count": (11100, 32), "passage_retrieval_en": (9300, 32), "lcc": (1200, 64), "repobench-p": (4200, 64),
}

METHOD_ALIASES = {"full": "fullkv", "fullkv": "fullkv"}
WINDOW_METHODS = ("snapkv", "pyramidkv", "h2o")


def canonical_method(name: str) -> str:
    n = name.lower()
    return METHOD_ALIASES.get(n, n)


def resolve_arch(model_path: Optional[str], model_provider: Optional[str] = None) -> str:
    """The reference takes a checkpoint path; offline we accept an architecture name, or pick one from the path / provider."""
    for cand in (model_path or "", model_provider or ""):
        c = cand.lower()
        if c in ARCHS:
            return c
        if "70b" in c:
            return "llama3-70b"
        if "mistral" in c:
            return "mistral-7b-v0.2"
        if "llama" in c:
            return "llama3-8b"
    return "llama3-8b"


def _resolve_attn(attn_implementation: str, device: torch.device, dtype: torch.dtype) -> str:
    """HF attention backend for the dense prefill: what the caller asked for (run_longbench.py:349 choices), checked once with
    a tiny call where the backend is a separate library — a backend that cannot run here is reported, never silently swapped."""
    if attn_implementation in ("eager", "None") or device.type == "cpu":
        return "eager"
    if attn_implementation != "flash_attention_2":
        return "sdpa"
    try:
        from flash_attn import flash_attn_func
        x = torch.zeros(1, 16, 2, 64, dtype=dtype if dtype in (torch.float16, torch.bfloat16) else torch.float16, device=device)
        flash_attn_func(x, x, x, causal=True)
        torch.cuda.synchronize(device)
        return "flash_attention_2"
    except Exception as e:   # noqa: BLE001 - any import / arch / launch failure of the external library
        print(f"pyramidkv_b200.runner: flash_attention_2 requested but the flash_attn library does not run on this device "
              f"({type(e).__name__}: {str(e)[:120]}); using sdpa for the dense prefill attention", file=sys.stderr)
        return "sdpa"


def build_model(arch: str, device: torch.device, dtype: torch.dtype = torch.float16, attn_implementation: str = "sdpa",
                max_positions: int = 65536):
    """Random-init model of the named architecture (no checkpoints offline). The reference loads fp16
    (run_longbench.py:388); north_star asks for bf16 as well — `dtype` selects."""
    import transformers
    family, hidden, inter, layers, heads, kv, hd, vocab, theta = ARCHS[arch]
    kw = dict(hidden_size=hidden, intermediate_size=inter, num_hidden_layers=layers, num_attention_heads=heads,
              num_key_value_heads=kv, head_dim=hd, vocab_size=vocab, rope_theta=theta, max_position_embeddings=max_positions)
    if family == "llama":
        cfg, cls = transformers.LlamaConfig(**kw), transformers.LlamaForCausalLM
    else:
        cfg, cls = transformers.MistralConfig(sliding_window=None, **kw), transformers.MistralForCausalLM
    # the reference's flash_attention_2 / sdpa choice only affects the dense prefill attention (library code, not this path)
    cfg._attn_implementation = _resolve_attn(attn_implementation, device, dtype)
    torch.manual_seed(42)
    old = torch.get_default_dtype()
    torch.set_default_dtype(dtype)
    try:
        with torch.device(device):
            model = cls(cfg)
    finally:
        torch.set_default_dtype(old)
    return model.eval()


def patch(method: str) -> None:
    from pyramidkv.monkeypatch import replace_llama, replace_mistral
    with contextlib.redirect_stdout(io.StringIO()):
        replace_llama(method)
        replace_mistral(method)


def head_capacities(model, max_capacity_prompts: int, head_beta: float = 1.01, head_path: str = "", seed: int = 42) -> torch.Tensor:
    """HeadKV budgets exactly as the reference runner derives them (run_longbench.py:225-234): per-head scores (mean of the
    head's list in the JSON at `head_path`, one line `{"layer-head": [scores...]}`), normalised, times the pool
    (B // beta) * L * H, plus the per-head minimum B - B // beta, rounded. The score files of the reference snapshot are empty
    (SURVEY.md appendix A.13), so without a readable file the scores are synthetic (seeded uniform(0.5, 1.5))."""
    import numpy as np
    L, H = model.config.num_hidden_layers, model.config.num_attention_heads
    scores = None
    if head_path and os.path.exists(head_path) and os.path.getsize(head_path) > 0:
        with open(head_path, "r") as f:
            head_list = json.loads(f.readline())
        scores = [np.mean(l[1]) for l in head_list.items()]
    if scores is None or len(scores) != L * H:
        scores = list(np.random.default_rng(seed).uniform(0.5, 1.5, L * H))
    t = torch.tensor(np.asarray(scores) / sum(scores))
    total_attention = t.reshape(L, H)
    total_pool_capacity = (max_capacity_prompts // head_beta) * L * H
    min_num = max_capacity_prompts - max_capacity_prompts // head_beta
    return torch.round(total_attention * total_pool_capacity + min_num).int()


def set_knobs(model, method: str, max_capacity_prompt: int, merge=None, backend_factory: Optional[Callable] = None,
              floor: float = 0.2, head_beta: float = 1.01, head_path: str = "") -> int:
    """run_longbench.py:219-261: window 8 (StreamingLLM: capacity - 4), kernel 7, maxpool, same capacity on every layer, `floor`
    for AdaKV, `head_capacity` for HeadKV. Returns the window size. `backend_factory` is the tests' injection point (oracle
    backend on a CPU box)."""
    window = max_capacity_prompt - 4 if method == "streamingllm" else 8
    if method == "headkv":
        model.model.config.head_capacity = head_capacities(model, max_capacity_prompt, head_beta, head_path)
    for layer in model.model.layers:
        c = layer.self_attn.config
        c.window_size, c.max_capacity_prompt, c.kernel_size, c.pooling, c.merge = window, max_capacity_prompt, 7, "maxpool", merge
        c.floor = floor
        if backend_factory is not None:
            layer.self_attn._pkv_backend = backend_factory()
    return window


@dataclass
class PromptResult:
    prompt_tokens: int
    new_tokens: int
    prefill_ms: float
    decode_tok_per_s: float
    cache_rows_first_last: List[int]
    pred_ids: List[int]


def _sync(device: torch.device) -> None:
    if device.type == "cuda":
        torch.cuda.synchronize(device)


def _run_prompt_static(model, ids: torch.Tensor, max_new_tokens: int, use_graph: Optional[bool],
                       prompt_lookup_num_tokens: Optional[int] = None) -> PromptResult:
    """Same record through the static loop (pyramidkv_b200.generate: pre-reserved cache, device-side row counter, one CUDA
    graph replay per token). Prefill and decode are timed separately — no subtraction of two generate calls is needed.
    prompt_lookup_num_tokens K: the cache is joined and decoded by greedy prompt-lookup speculation (SpeculativeDecoder,
    one graph replay per verify step, K draft tokens)."""
    from transformers import DynamicCache
    from .cache import join_caches
    from .generate import SpeculativeDecoder, StaticDecoder
    dev = ids.device

    def prefill():
        for layer in model.model.layers:
            layer.self_attn.kv_seq_len = 0
        cache = DynamicCache(config=model.config)
        out = model(input_ids=ids, past_key_values=cache, use_cache=True, logits_to_keep=1)
        return out.logits[:, -1, :].argmax(dim=-1, keepdim=True), cache

    with torch.no_grad():
        prefill()
        _sync(dev)
        t0 = time.perf_counter()
        first, cache = prefill()
        _sync(dev)
        t1 = time.perf_counter()
        toks, decode_s = [first], 0.0
        if max_new_tokens > 1 and prompt_lookup_num_tokens:
            K = int(prompt_lookup_num_tokens)
            cache = join_caches([cache], reserve=max_new_tokens + K)
            dec = SpeculativeDecoder(model, cache, first, [ids[0]], max_new_tokens, K, use_graph=use_graph)
            if dec.use_graph:
                dec._capture()
            _sync(dev)
            t2 = time.perf_counter()
            dec.run_to_end(max_new_tokens)
            gen = dec.generated()
            _sync(dev)
            decode_s = time.perf_counter() - t2
            toks.append(torch.tensor([gen[0]], dtype=torch.long, device=dev).reshape(1, -1))
            dec.finish([len(gen[0])])
        elif max_new_tokens > 1:
            dec = StaticDecoder(model, cache, first, max_new_tokens - 1, use_graph=use_graph)
            if dec.use_graph:
                dec._capture()                       # graph capture is a one-off cost per prompt shape, not decode time
            _sync(dev)
            t2 = time.perf_counter()
            toks.append(dec.run(max_new_tokens - 1).clone())
            _sync(dev)
            decode_s = time.perf_counter() - t2
            dec.finish()
    rows = [int(l.keys.shape[-2]) for l in cache.layers if getattr(l, "keys", None) is not None]
    return PromptResult(int(ids.shape[1]), max_new_tokens, (t1 - t0) * 1e3,
                        (max_new_tokens - 1) / max(decode_s, 1e-9) if max_new_tokens > 1 else 0.0,
                        [rows[0], rows[-1]] if rows else [], torch.cat(toks, dim=1)[0].tolist())


def _run_batch_static(model, prompts: List[torch.Tensor], max_new_tokens: int, use_graph: Optional[bool]):
    """Several prompts through greedy_generate_batch's flow: each prefilled alone (timed alone, after an untimed warm-up at
    its length), the caches joined, then one static decode of all of them. Returns (one PromptResult per prompt, the
    batch's aggregate decode tok/s = sequences * steps / decode time)."""
    from .cache import join_caches
    from .generate import StaticDecoder, _prefill
    dev = prompts[0].device
    firsts, caches, prefill_ms = [], [], []
    with torch.no_grad():
        for ids in prompts:
            _prefill(model, ids)
            _sync(dev)
            t0 = time.perf_counter()
            f, c = _prefill(model, ids)
            _sync(dev)
            prefill_ms.append((time.perf_counter() - t0) * 1e3)
            firsts.append(f)
            caches.append(c)
        first = torch.cat(firsts)
        cache = join_caches(caches, reserve=max(0, max_new_tokens - 1))
        del caches
        gen, decode_s = torch.empty(len(prompts), 0, dtype=torch.long, device=dev), 0.0
        if max_new_tokens > 1:
            dec = StaticDecoder(model, cache, first, max_new_tokens - 1, use_graph=use_graph)
            if dec.use_graph:
                dec._capture()                       # graph capture is a one-off cost per batch shape, not decode time
            _sync(dev)
            t0 = time.perf_counter()
            gen = dec.run(max_new_tokens - 1).clone()
            _sync(dev)
            decode_s = time.perf_counter() - t0
            dec.finish()
    steps = max_new_tokens - 1
    per_seq = steps / max(decode_s, 1e-9) if steps > 0 else 0.0
    res = []
    for b, ids in enumerate(prompts):
        rows = [max(l.rows_host[b]) for l in cache.layers]
        res.append(PromptResult(int(ids.shape[1]), max_new_tokens, prefill_ms[b], per_seq, [rows[0], rows[-1]],
                                torch.cat([first[b], gen[b]]).tolist()))
    return res, per_seq * len(prompts)


def _run_continuous(model, prompts: List[torch.Tensor], max_new_tokens: List[int], slots: int):
    """All prompts through one greedy_generate_continuous with `slots` slots (graph replay), after an untimed warm-up prefill
    per prompt length. Returns (one PromptResult per prompt, the run's `continuous` record block)."""
    from .generate import _prefill, greedy_generate_continuous
    dev = prompts[0].device
    with torch.no_grad():
        for n in sorted({int(p.shape[1]) for p in prompts}):
            _prefill(model, next(p for p in prompts if p.shape[1] == n))
        _sync(dev)
        seqs, st = greedy_generate_continuous(model, prompts, max_new_tokens, slots, return_stats=True)
    steps = st["decode_steps"]
    block = {"slots": min(slots, len(prompts)), "decode_steps": steps,
             "occupancy": st["live_slot_steps"] / max(1, min(slots, len(prompts)) * steps),
             "aggregate_tok_per_s": st["live_slot_steps"] / max(st["decode_s"], 1e-9),
             "admissions": st["admissions"], "regrowths": st["regrowths"], "graph_captures": st["graph_captures"]}
    res = []
    for i, (p, n, s) in enumerate(zip(prompts, max_new_tokens, seqs)):
        pred = s[p.shape[1]:].tolist()
        rows = [r + len(pred) - 1 for r in st["cache_rows_first_last"][i]]      # the decoded tokens' rows, as the other loops book them
        res.append(PromptResult(int(p.shape[1]), n, st["prefill_ms"][i], 0.0, rows, pred))
    return res, block


def run_prompt(model, ids: torch.Tensor, max_new_tokens: int, decode_loop: str = "hf",
               prompt_lookup_num_tokens: Optional[int] = None) -> PromptResult:
    """Greedy generate exactly as the reference runner does. One untimed warm-up call at this prompt length (allocator,
    cuBLAS heuristics, lazy module init), then two timed calls: one new token (prefill + eviction of all layers) and the
    full length; decode tok/s is taken over the difference. decode_loop = "static" / "static-eager" replaces HF's loop by
    the static one (SURVEY.md §8 f3); with it, prompt_lookup_num_tokens K decodes by prompt-lookup speculation."""
    if decode_loop != "hf":
        if decode_loop not in ("static", "static-eager"):
            raise ValueError(f"decode_loop must be hf, static or static-eager, got {decode_loop!r}")
        return _run_prompt_static(model, ids, max_new_tokens, None if decode_loop == "static" else False,
                                  prompt_lookup_num_tokens)
    if prompt_lookup_num_tokens:
        raise NotImplementedError("prompt_lookup_num_tokens runs in the static loop (decode_loop static or static-eager)")
    dev = ids.device
    kw = dict(attention_mask=torch.ones_like(ids), num_beams=1, do_sample=False, pad_token_id=0, return_dict_in_generate=True)
    with torch.no_grad():
        model.generate(ids, max_new_tokens=1, min_new_tokens=1, **kw)
        _sync(dev)
        t0 = time.perf_counter()
        first = model.generate(ids, max_new_tokens=1, min_new_tokens=1, **kw)
        _sync(dev)
        t1 = time.perf_counter()
        out = model.generate(ids, max_new_tokens=max_new_tokens, min_new_tokens=max_new_tokens, **kw)
        _sync(dev)
        t2 = time.perf_counter()
    prefill_ms = (t1 - t0) * 1e3
    decode_s = max((t2 - t1) - (t1 - t0), 1e-9)
    rows = [int(l.keys.shape[-2]) for l in out.past_key_values.layers if getattr(l, "keys", None) is not None]
    del first
    return PromptResult(int(ids.shape[1]), max_new_tokens, prefill_ms,
                        (max_new_tokens - 1) / decode_s if max_new_tokens > 1 else 0.0,
                        [rows[0], rows[-1]] if rows else [], out.sequences[0, ids.shape[1]:].tolist())


def synthetic_prompt(vocab: int, length: int, seed: int, device: torch.device) -> torch.Tensor:
    g = torch.Generator().manual_seed(seed)
    return torch.randint(1, vocab, (1, length), generator=g).to(device)      # id 0 is the pad id


def run_suite(arch: str, method: str, max_capacity_prompt: int, prompts: Iterable[tuple], device: Optional[torch.device] = None,
              dtype: torch.dtype = torch.float16, attn_implementation: str = "sdpa", merge=None, seed: int = 42,
              backend_factory: Optional[Callable] = None, out_path: Optional[str] = None, tag: Optional[dict] = None,
              decode_loop: str = "hf", floor: float = 0.2, head_beta: float = 1.01, head_path: str = "",
              capacity_ratio: float = -1, eval_batch_size: int = 1, kv_cache_dtype: str = "auto",
              gqa_shared: bool = False, decode_window: Optional[int] = None, decode_heavy: Optional[int] = None,
              prompt_lookup_num_tokens: Optional[int] = None) -> List[dict]:
    """prompts: iterable of (name, prompt_tokens, max_new_tokens). One JSON record per prompt (also appended to out_path).
    eval_batch_size N > 1: consecutive prompts with the same max_new_tokens are decoded N at a time (static loops only;
    each prompt is still prefilled alone, so its prefill_ms, cache rows and tokens are its own).
    kv_cache_dtype "fp8_e4m3": the compacted caches are converted to FP8 after the prefill (model.config.pkv_kv_cache_dtype);
    the records then carry "kv_cache_dtype". "auto" (the default) changes nothing.
    gqa_shared: one selection and one compacted cache per KV head (model.config.pkv_gqa_shared); the records then carry
    "gqa_shared". FullKV, AdaKV and HeadKV refuse it.
    decode_window R: each sequence keeps its compacted prompt plus its last R decoded tokens (model.config.pkv_decode_window);
    the records then carry "decode_window". FullKV refuses it.
    decode_heavy H (with decode_window R): the window keeps its R - H most recent decoded tokens and, of the others, those
    with the most accumulated attention (model.config.pkv_decode_heavy); the records then carry "decode_heavy".
    decode_loop "continuous": every prompt goes through one greedy_generate_continuous with eval_batch_size slots, whatever
    its max_new_tokens; each record keeps its own prefill_ms, cache rows and tokens and carries the run's "continuous" block
    (slots, decode_steps, occupancy, aggregate_tok_per_s) instead of a per-prompt decode rate.
    prompt_lookup_num_tokens K (static loops, eval_batch_size 1, an eviction method): greedy prompt-lookup speculative
    decoding with K draft tokens per step; the records then carry "prompt_lookup_num_tokens"."""
    if kv_cache_dtype not in ("auto", "fp8_e4m3"):
        raise ValueError(f"kv_cache_dtype must be auto or fp8_e4m3, got {kv_cache_dtype!r}")
    if kv_cache_dtype != "auto" and canonical_method(method) == "fullkv":
        raise NotImplementedError("--kv_cache_dtype fp8_e4m3 converts the compacted cache of an eviction method; FullKV keeps "
                                  "HF's own cache (the reference's --quant_method caches are not built)")
    if gqa_shared and canonical_method(method) in ("fullkv", "adakv", "headkv"):
        raise NotImplementedError(f"--gqa_shared selects one compacted cache per KV head; {canonical_method(method)} "
                                  + ("keeps HF's own cache" if canonical_method(method) == "fullkv" else "sets budgets per query head"))
    if decode_window is not None and canonical_method(method) == "fullkv":
        raise NotImplementedError("--decode_window bounds the compacted cache of an eviction method; FullKV keeps HF's own cache")
    if decode_heavy is not None and canonical_method(method) == "fullkv":
        raise NotImplementedError("--decode_heavy chooses the rows of the decode window; FullKV keeps HF's own cache")
    if eval_batch_size < 1:
        raise ValueError(f"eval_batch_size must be >= 1, got {eval_batch_size}")
    continuous = decode_loop == "continuous"
    if (eval_batch_size > 1 or continuous) and (decode_loop == "hf" or canonical_method(method) == "fullkv"):
        raise NotImplementedError("eval_batch_size > 1 decodes the joined compacted caches of the prompts with the static loop: "
                                  "use --decode_loop static or static-eager with an eviction method (padded HF batches are not supported)")
    if decode_loop not in ("hf", "static", "static-eager", "continuous"):
        raise ValueError(f"decode_loop must be hf, static, static-eager or continuous, got {decode_loop!r}")
    if prompt_lookup_num_tokens is not None and (decode_loop not in ("static", "static-eager") or eval_batch_size > 1
                                                 or canonical_method(method) == "fullkv"):
        raise NotImplementedError("--prompt_lookup_num_tokens runs in the static loop with eval_batch_size 1 and an eviction "
                                  "method")
    if device is None:
        if not torch.cuda.is_available():
            raise RuntimeError("the runners need a CUDA device (H100, sm_90a); there is no CPU fallback")
        device = torch.device("cuda", torch.cuda.current_device())
    method = canonical_method(method)
    patch(method)
    try:
        model = build_model(arch, device, dtype, attn_implementation)
        window = 0
        if method != "fullkv" and max_capacity_prompt != -1:
            window = set_knobs(model, method, max_capacity_prompt, merge, backend_factory, floor, head_beta, head_path)
        elif method != "fullkv" and capacity_ratio == -1:
            raise ValueError("either max_capacity_prompts or max_capacity_prompts_ratio must be given")
        if kv_cache_dtype != "auto":
            model.config.pkv_kv_cache_dtype = kv_cache_dtype
        if gqa_shared:
            model.config.pkv_gqa_shared = True
        if decode_window is not None:
            from .cache import decode_window as decode_window_knob
            model.config.pkv_decode_window = decode_window
            decode_window_knob(model.config)           # rejects a bad value before any prompt runs
        if decode_heavy is not None:
            from .cache import decode_heavy as decode_heavy_knob
            model.config.pkv_decode_heavy = decode_heavy
            decode_heavy_knob(model.config)            # rejects a bad value (or a missing window) before any prompt runs
        records = []
        prompts = list(prompts)
        if (eval_batch_size > 1 or continuous) and max_capacity_prompt == -1 and capacity_ratio != -1 and len({p[1] for p in prompts}) > 1:
            raise NotImplementedError("--max_capacity_prompts_ratio sets a budget per prompt length; batch prompts of one length")

        def emit(group, rs, extra):
            for j, r in zip(group, rs):
                rec = {"task": prompts[j][0], "arch": arch, "method": method,
                       "max_capacity_prompt": model.config.max_capacity_prompt if method != "fullkv" else max_capacity_prompt, "window": window,
                       "decode_loop": decode_loop if method != "fullkv" else "hf",
                       **({"kv_cache_dtype": kv_cache_dtype} if kv_cache_dtype != "auto" else {}),
                       **({"gqa_shared": True} if gqa_shared else {}),
                       **({"decode_window": int(decode_window)} if decode_window is not None else {}),
                       **({"decode_heavy": int(decode_heavy)} if decode_heavy is not None else {}),
                       **({"prompt_lookup_num_tokens": int(prompt_lookup_num_tokens)} if prompt_lookup_num_tokens else {}),
                       "dtype": str(dtype).replace("torch.", ""), "data": "synthetic token ids, random-init weights", **(tag or {}),
                       "prompt_tokens": r.prompt_tokens, "new_tokens": r.new_tokens, "prefill_ms": r.prefill_ms,
                       **({} if continuous else {"decode_tok_per_s": r.decode_tok_per_s}), **extra,
                       "cache_rows_first_last": r.cache_rows_first_last, "pred_ids": r.pred_ids}
                records.append(rec)
                print(json.dumps({k: v for k, v in rec.items() if k != "pred_ids"}), flush=True)
                if out_path:
                    os.makedirs(os.path.dirname(os.path.abspath(out_path)), exist_ok=True)
                    with open(out_path, "a") as f:
                        f.write(json.dumps(rec) + "\n")

        if continuous:
            if prompts and max_capacity_prompt == -1 and capacity_ratio != -1:
                window = set_knobs(model, method, round(prompts[0][1] * capacity_ratio), merge, backend_factory, floor, head_beta, head_path)
            ids = [synthetic_prompt(model.config.vocab_size, p[1], seed + j, device) for j, p in enumerate(prompts)]
            if ids:
                rs, block = _run_continuous(model, ids, [p[2] for p in prompts], eval_batch_size)
                emit(range(len(prompts)), rs, {"continuous": block})
            return records
        i = 0
        while i < len(prompts):
            group = [i]                                   # consecutive prompts decoded together: same max_new_tokens
            while len(group) < eval_batch_size and group[-1] + 1 < len(prompts) and prompts[group[-1] + 1][2] == prompts[i][2]:
                group.append(group[-1] + 1)
            if method != "fullkv" and max_capacity_prompt == -1 and capacity_ratio != -1:
                # run_longbench.py:213-216: with --max_capacity_prompts -1 the budget is a fraction of EACH prompt's length
                cap_i = round(prompts[i][1] * capacity_ratio)
                window = set_knobs(model, method, cap_i, merge, backend_factory, floor, head_beta, head_path)
            ids = [synthetic_prompt(model.config.vocab_size, prompts[j][1], seed + j, device) for j in group]
            batch = {}
            if eval_batch_size > 1:
                rs, agg = _run_batch_static(model, ids, prompts[i][2], None if decode_loop == "static" else False)
                batch = {"eval_batch_size": eval_batch_size, "batch_size": len(group), "batch_decode_tok_per_s_aggregate": agg}
            else:
                rs = [run_prompt(model, ids[0], prompts[i][2], decode_loop if method != "fullkv" else "hf", prompt_lookup_num_tokens)]
            emit(group, rs, batch)
            i = group[-1] + 1
        return records
    finally:
        from pyramidkv.monkeypatch import restore
        restore()
