#!/usr/bin/env python
"""Sampled decoding on the H100: python tools/sampling_bench.py [--batch 1,8,32,64] [--loop_batch 1,32] [--prompt 1024]

1. Kernel: one pkv_sample_tokens launch (V = 128256, bf16 logits, T = 0.7, top_p = 0.9, top_k 0 and 50) per batch size,
   next to HF's warper chain on the same logits (fp32 upcast as HF's generate does, TemperatureLogitsWarper, TopKLogitsWarper,
   TopPLogitsWarper, softmax, torch.multinomial), both timed with CUDA events in the same run.
2. Loops: the per-step time of the static loop (StaticDecoder over joined caches) and of the continuous loop
   (ContinuousDecoder.run_chunk, every slot live) on a random-init Llama-3-8B, PyramidKV at budget 128 (the reference
   runners' knobs), greedy against sampling (T = 0.7, top_p = 0.9), graph replay, CUDA events around the timed steps.
Prints one JSON line with the card's name and power limit; writes nothing else.
"""
import argparse
import contextlib
import io
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from decode_batch_bench import gpu_card  # noqa: E402
from full_model_bench import build_model  # noqa: E402

V = 128256


def _events_ms(fn, reps):
    fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


def kernel_numbers(dev, batches, reps=200):
    from transformers.generation.logits_process import TemperatureLogitsWarper, TopKLogitsWarper, TopPLogitsWarper
    from pyramidkv_b200 import ops
    from pyramidkv_b200.generate import SamplingParams, SamplingState
    out = []
    for B in batches:
        g = torch.Generator(device=dev).manual_seed(B)
        logits = (torch.randn(B, V, device=dev, generator=g) * 2.5).bfloat16()
        toks = torch.empty(B, 1, dtype=torch.long, device=dev)
        ids = torch.zeros(B, 1, dtype=torch.long, device=dev)
        row = {"batch": B, "vocab": V, "logit_bytes": B * V * 2}
        for k in (0, 50):
            st = SamplingState([SamplingParams(0.7, k, 0.9, seed=b) for b in range(B)], dev)
            row[f"pkv_sample_tokens_top_k{k}_us"] = 1e3 * _events_ms(lambda: ops.sample_tokens(logits, st, toks, 0), reps)
            warpers = [TemperatureLogitsWarper(0.7)] + ([TopKLogitsWarper(k)] if k else []) + [TopPLogitsWarper(0.9)]

            def hf():
                s = logits.float()
                for w in warpers:
                    s = w(ids, s)
                return torch.multinomial(torch.softmax(s, dim=-1), num_samples=1)
            row[f"hf_warpers_multinomial_top_k{k}_us"] = 1e3 * _events_ms(hf, max(20, reps // 4))
        row["one_pass_over_logits_at_3.35TB/s_us"] = row["logit_bytes"] / 3.35e12 * 1e6
        out.append(row)
    return out


@torch.no_grad()
def loop_numbers(model, dev, batches, prompt_len, steps=64):
    from pyramidkv_b200 import runner
    from pyramidkv_b200.cache import join_caches
    from pyramidkv_b200.generate import ContinuousDecoder, SamplingParams, StaticDecoder, _prefill
    out = []
    for B in batches:
        prompts = [runner.synthetic_prompt(model.config.vocab_size, prompt_len, 100 + i, dev) for i in range(B)]
        row = {"batch": B, "prompt_tokens": prompt_len, "timed_steps": steps}
        for loop in ("static", "continuous"):
            for mode in ("greedy", "sampling"):
                samp = None if mode == "greedy" else [SamplingParams(0.7, 0, 0.9, seed=7 + b) for b in range(B)]
                firsts, caches = zip(*[_prefill(model, p) for p in prompts])
                cache = join_caches(list(caches), reserve=2 * steps + 16)
                del caches
                first = torch.cat(firsts)
                if loop == "static":
                    dec = StaticDecoder(model, cache, first, 2 * steps + 8, sampling=samp)
                    dec.run(4)                                      # capture + warm-up
                    fn = lambda: dec.run(steps)                     # noqa: E731
                else:
                    dec = ContinuousDecoder(model, cache, first, [10 ** 6] * B, chunk=steps, sampling=samp)
                    dec.run_chunk(4)
                    fn = lambda: dec.run_chunk(steps)               # noqa: E731
                torch.cuda.synchronize()
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                fn()
                b.record()
                torch.cuda.synchronize()
                row[f"{loop}_{mode}_step_ms"] = a.elapsed_time(b) / steps
                dec.finish()
                del dec, cache
                torch.cuda.empty_cache()
            row[f"{loop}_sampling_overhead_pct"] = 100 * (row[f"{loop}_sampling_step_ms"] / row[f"{loop}_greedy_step_ms"] - 1)
        out.append(row)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", default="1,8,32,64", help="kernel batch sizes")
    ap.add_argument("--loop_batch", default="1,32", help="batch sizes of the loop measurements ('' skips them)")
    ap.add_argument("--prompt", type=int, default=1024)
    ap.add_argument("--budget", type=int, default=128)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("tools/sampling_bench.py measures on a CUDA device (H100); there is none here")
    dev = torch.device("cuda", 0)
    res = {"gpu": gpu_card(dev), "kernel": kernel_numbers(dev, [int(x) for x in args.batch.split(",") if x.strip()])}
    loop_batch = [int(x) for x in args.loop_batch.split(",") if x.strip()]
    if loop_batch:
        from pyramidkv.monkeypatch import replace_llama, restore
        model = build_model("llama3-8b", dev)
        with contextlib.redirect_stdout(io.StringIO()):
            replace_llama("pyramidkv")
        try:
            for layer in model.model.layers:                         # run_longbench.py:253-261
                c = layer.self_attn.config
                c.window_size, c.max_capacity_prompt, c.kernel_size, c.pooling = 8, args.budget, 7, "maxpool"
            model.config.pkv_fused_rope = True
            res["loops"] = {"model": "llama3-8b (random init)", "method": "pyramidkv", "budget": args.budget,
                            "rows": loop_numbers(model, dev, loop_batch, args.prompt)}
        finally:
            restore()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
