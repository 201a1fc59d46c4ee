#!/usr/bin/env python
"""Needle-style context sweep with the reference's command line (run_needle_in_haystack.py:498-529,
scripts/scripts_needle/eval.sh:18-26) over the GPU eviction path.

    python run_needle_in_haystack.py --s_len 1000 --e_len 8001 --step 1000 --model_provider Mistral \
        --model_name mistral-7b-v0.2 --method pyramidkv --max_capacity_prompt 96 --attn_implementation sdpa

No network: the haystack / needle texts, the tokenizer and the checkpoint are replaced by synthetic token-id prompts of
each context length and a random-init model of the named architecture (seed 42); retrieval accuracy is therefore not
scored — the sweep reports prefill ms, decode tok/s and the compacted cache size per context length, with the knobs the
reference sets for this runner (window 8, kernel 7, maxpool; StreamingLLM window = capacity - 4)."""
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
    p.add_argument("-s", "--s_len", metavar="N", type=int, default=1000)
    p.add_argument("-e", "--e_len", metavar="N", type=int, default=8001)
    p.add_argument("--model_name", type=str, default=None)
    p.add_argument("--attn_implementation", type=str, default="flash_attention_2", choices=["flash_attention_2", "sdpa", "None"])
    p.add_argument("--model_version", type=str, default=None)
    p.add_argument("--model_name_suffix", type=str, default=None)
    p.add_argument("--model_provider", type=str, default="LLaMA")
    p.add_argument("--api_key", type=str, default="")
    p.add_argument("--step", type=int, default=1000)
    p.add_argument("--method", type=str, default="full", choices=["full", "pyramidkv", "snapkv", "streamingllm", "h2o", "cam"])
    p.add_argument("--max_capacity_prompt", type=int, default=128)
    p.add_argument("--max_new_tokens", type=int, default=32)
    p.add_argument("--dtype", type=str, default="float16", choices=["float16", "bfloat16"])
    p.add_argument("--save_dir", type=str, default="")
    p.add_argument("--decode_loop", type=str, default="hf", choices=["hf", "static", "static-eager"],
                   help="hf: model.generate as in the reference; static: pyramidkv_b200.generate (CUDA-graph replay per token)")
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
    if args.method == "cam":
        raise NotImplementedError("CAM is outside the eviction hot path built here (SURVEY.md §8)")
    arch = runner.resolve_arch(args.model_name, args.model_provider)
    prompts = [(f"ctx{n}", n, args.max_new_tokens) for n in range(args.s_len, args.e_len, args.step)]
    if not prompts:
        raise SystemExit("empty context sweep: need s_len < e_len")
    out = None
    if args.save_dir:
        out = os.path.join(args.save_dir, f"{args.model_version or arch}_{args.method}_{args.max_capacity_prompt}.jsonl")
    recs = runner.run_suite(arch, args.method, args.max_capacity_prompt, prompts, device=device, dtype=getattr(torch, args.dtype),
                            attn_implementation=args.attn_implementation, backend_factory=backend_factory, out_path=out,
                            tag={"runner": "needle"}, decode_loop=args.decode_loop, kv_cache_dtype=args.kv_cache_dtype, gqa_shared=args.gqa_shared,
                            decode_window=args.decode_window, decode_heavy=args.decode_heavy)
    print(json.dumps({"summary": True, "arch": arch, "method": runner.canonical_method(args.method),
                      "max_capacity_prompt": args.max_capacity_prompt, "contexts": [r["prompt_tokens"] for r in recs],
                      "prefill_ms": [round(r["prefill_ms"], 3) for r in recs],
                      "decode_tok_per_s": [round(r["decode_tok_per_s"], 2) for r in recs]}))
    return recs


if __name__ == "__main__":
    main()
