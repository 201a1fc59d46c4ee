#!/usr/bin/env python
"""LongBench-shaped runner with the reference's command line (run_longbench.py:321-366) over the GPU eviction path.

    python run_longbench.py --method pyramidkv --model_path llama3-8b --max_capacity_prompts 128 \
        --attn_implementation sdpa --dataset narrativeqa --save_dir results/ --max_num_examples 4

No network: `--model_path` names an architecture (llama3-8b, llama3-70b, mistral-7b-v0.2, tiny-llama, tiny-mistral; a
checkpoint path is mapped to the architecture it names) that is random-initialised with the runners' seed 42, and each
example is a synthetic token-id prompt of the task's typical length. The per-layer knobs (window 8, kernel 7, maxpool;
StreamingLLM window = capacity - 4) and the greedy `generate` call are the reference's (:219-275). Flags of methods
outside the hot path (quantisation, AdaKV/HeadKV/ThinK knobs) are accepted and rejected with a clear error when used."""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
from pyramidkv_b200 import runner  # noqa: E402


def build_parser() -> argparse.ArgumentParser:
    p = argparse.ArgumentParser()
    p.add_argument("--seed", type=int, default=42)
    p.add_argument("--base_dir", type=str, default="")
    p.add_argument("--dataset", type=str, default="narrativeqa", help="LongBench task name or 'all' (sets prompt length and max_new_tokens)")
    p.add_argument("--data_file", type=str, default="", help="ignored: prompts are synthetic (no corpora offline)")
    p.add_argument("--save_dir", type=str, default="")
    p.add_argument("--model_name", type=str, default=None)
    p.add_argument("--model_path", type=str, default="llama3-8b")
    p.add_argument("--max_num_examples", type=int, default=2)
    p.add_argument("--sample_method", type=str, default="topk", choices=["random", "topk"])
    p.add_argument("--max_new_tokens", type=int, default=None)
    p.add_argument("--eval_batch_size", type=int, default=1,
                   help="N > 1 (static decode loops): prompts are prefilled one at a time and decoded N at a time")
    p.add_argument("--use_cache", type=bool, default=True)
    p.add_argument("--attn_implementation", type=str, default="flash_attention_2", choices=["flash_attention_2", "sdpa", "eager"])
    p.add_argument("--method", type=str, default=None)
    p.add_argument("--quant_method", type=str, default=None, choices=["kivi", "kvquant"])
    p.add_argument("--nbits", type=int, default=8)
    p.add_argument("--max_capacity_prompts", type=int, default=512)
    p.add_argument("--max_capacity_prompts_ratio", type=float, default=-1)
    p.add_argument("--steps", type=int, default=-1)
    p.add_argument("--merge", type=str, default=None)
    p.add_argument("--floor", type=float, default=0.2)
    p.add_argument("--head_path", type=str, default="")
    p.add_argument("--head_beta", type=float, default=1.01)
    p.add_argument("--recent_size", type=int, default=32)
    p.add_argument("--pruning_ratio", type=float, default=0.4)
    p.add_argument("--use_chat_format", action="store_true")
    p.add_argument("--chat_formatting_function", type=str, default="")
    p.add_argument("--dtype", type=str, default="float16", choices=["float16", "bfloat16"], help="the reference loads fp16 (:388)")
    p.add_argument("--prompt_tokens", type=int, default=0, help="override the task's typical prompt length")
    p.add_argument("--decode_loop", type=str, default="hf", choices=["hf", "static", "static-eager", "continuous"],
                   help="hf: model.generate as in the reference; static: pyramidkv_b200.generate (CUDA-graph replay per token); "
                        "continuous: every prompt through --eval_batch_size slots, a finished sequence's slot taking the next prompt")
    p.add_argument("--prompt_lookup_num_tokens", type=int, default=None,
                   help="--decode_loop static or continuous: greedy prompt-lookup speculative decoding with K (1..15) draft "
                        "tokens per step (HF's generate argument of that name; DESIGN.md §4.13, §4.14)")
    p.add_argument("--kv_cache_dtype", type=str, default="auto", choices=["auto", "fp8_e4m3"],
                   help="auto: the compacted cache in the model dtype; fp8_e4m3: FP8 bytes + one fp32 scale per row (half the KV bytes)")
    p.add_argument("--gqa_shared", action="store_true",
                   help="one selection and one compacted cache per KV head (the score averaged over each GQA group): "
                        "Hq/Hkv times fewer cache bytes; not for fullkv / adakv / headkv")
    p.add_argument("--decode_window", type=int, default=None,
                   help="keep each sequence's cache at its compacted prompt plus its last R decoded tokens (fixed memory for "
                        "any generation length); default: every decoded token stays")
    p.add_argument("--decode_heavy", type=int, default=None,
                   help="with --decode_window R: keep the R - H most recent decoded tokens and, in the other H slots, the "
                        "tokens with the most accumulated attention (H2O heavy hitters, 1 <= H <= R - 1); default: the "
                        "oldest token leaves")
    return p


def main(argv=None, backend_factory=None, device=None):
    args = build_parser().parse_args(argv)
    if args.method is None:
        raise SystemExit("--method is required (FullKV, PyramidKV, SnapKV, H2O, StreamingLLM)")
    if args.quant_method is not None:
        raise NotImplementedError("quantised caches (--quant_method) are outside the eviction hot path built here")
    if args.eval_batch_size != 1 and args.decode_loop == "hf":
        raise NotImplementedError("--eval_batch_size > 1 needs --decode_loop static or static-eager (the prompts are prefilled one at "
                                  "a time and their compacted caches decoded together); padded HF batches are not supported")
    method = runner.canonical_method(args.method)
    arch = runner.resolve_arch(args.model_path, args.model_name)
    tasks = sorted(runner.LONGBENCH_SHAPES) if args.dataset in ("all", "") else [args.dataset]
    prompts = []
    for t in tasks:
        if t not in runner.LONGBENCH_SHAPES:
            raise SystemExit(f"unknown LongBench task {t!r}; known: {sorted(runner.LONGBENCH_SHAPES)}")
        length, new = runner.LONGBENCH_SHAPES[t]
        length = args.prompt_tokens or length
        for _ in range(max(1, args.max_num_examples or 1)):
            prompts.append((t, length, args.max_new_tokens or new))
    capacity = args.max_capacity_prompts                                  # -1 + --max_capacity_prompts_ratio: per prompt (run_longbench.py:213-216)
    out = None
    if args.save_dir:
        tag = capacity if capacity != -1 else f"ratio{args.max_capacity_prompts_ratio}"
        out = os.path.join(args.save_dir, f"{arch}_{tag}", args.dataset, f"{method}.jsonl")
    recs = runner.run_suite(arch, method, capacity, prompts, device=device, dtype=getattr(torch, args.dtype),
                            attn_implementation=args.attn_implementation, merge=args.merge, seed=args.seed,
                            backend_factory=backend_factory, out_path=out, decode_loop=args.decode_loop,
                            floor=args.floor, head_beta=args.head_beta, head_path=args.head_path,
                            capacity_ratio=args.max_capacity_prompts_ratio, eval_batch_size=args.eval_batch_size,
                            kv_cache_dtype=args.kv_cache_dtype, gqa_shared=args.gqa_shared,
                            decode_window=args.decode_window, decode_heavy=args.decode_heavy,
                            prompt_lookup_num_tokens=args.prompt_lookup_num_tokens)
    n = len(recs)
    print(json.dumps({"summary": True, "arch": arch, "method": method, "max_capacity_prompts": capacity, "examples": n,
                      "mean_prefill_ms": sum(r["prefill_ms"] for r in recs) / n,
                      **({"continuous": recs[0]["continuous"]} if "continuous" in recs[0] else
                         {"mean_decode_tok_per_s": sum(r["decode_tok_per_s"] for r in recs) / n})}))
    return recs


if __name__ == "__main__":
    main()
