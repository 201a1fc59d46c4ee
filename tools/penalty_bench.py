#!/usr/bin/env python
"""Penalized sampling on the H100: python tools/penalty_bench.py [--batch 1,8,32,64] [--loop_batch 1,32] [--prompt 1024]

1. Kernel: one pkv_sample_tokens_penalized launch next to one pkv_sample_tokens launch on the same logits (V = 128256, bf16,
   T = 0.7, top_p = 0.9, top_k 0 and 50; and T = 0, the greedy token of the penalized logits), per batch size, with a
   realistic history per row: a prompt mask of 4096 ids and counts over 512 generated ids (repetition_penalty 1.1, presence
   and frequency 0.3, min_p 0.05). CUDA events around many launches.
2. Loops: the per-step time of the static loop at each --loop_batch and of the continuous loop at the largest, on a
   random-init Llama-3-8B, PyramidKV at budget 128, graph replay: sampling (T = 0.7, top_p = 0.9) without and with the
   penalties above. HF's own generate loop at B = 1, greedy, with and without repetition_penalty = 1.1 (per new token,
   from the difference of 33 and 1 new tokens): the alternative a user of the penalty has without this path.
Prints one JSON line with the card's name and power limit; writes nothing else.
"""
import argparse
import contextlib
import io
import json
import os
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from decode_batch_bench import gpu_card  # noqa: E402
from full_model_bench import build_model  # noqa: E402
from sampling_bench import _events_ms  # noqa: E402

V = 128256
PEN = dict(repetition_penalty=1.1, presence_penalty=0.3, frequency_penalty=0.3, min_p=0.05)


def _history(st, B, dev, seed):
    g = torch.Generator(device=dev).manual_seed(seed)
    for b in range(B):
        st.prompt_mask[b, torch.randint(0, V, (4096,), device=dev, generator=g)] = 1
        st.counts[b, torch.randint(0, V, (512,), device=dev, generator=g)] = torch.randint(
            1, 8, (512,), device=dev, generator=g, dtype=torch.int32)


def kernel_numbers(dev, batches, reps=200):
    from pyramidkv_b200 import ops
    from pyramidkv_b200.generate import SamplingParams, SamplingState
    out = []
    for B in batches:
        g = torch.Generator(device=dev).manual_seed(B)
        logits = (torch.randn(B, V, device=dev, generator=g) * 2.5).bfloat16()
        toks = torch.empty(B, 1, dtype=torch.long, device=dev)
        prompts = [torch.zeros(1, dtype=torch.long, device=dev)] * B
        row = {"batch": B, "vocab": V}
        for name, T, k in (("top_k0", 0.7, 0), ("top_k50", 0.7, 50), ("greedy", 0.0, 0)):
            plain = SamplingState([SamplingParams(T, k, 0.9 if T else 1.0, seed=b) for b in range(B)], dev)
            pen = SamplingState([SamplingParams(T, k, 0.9 if T else 1.0, seed=b, **PEN) for b in range(B)], dev, vocab=V,
                                prompts=prompts)
            _history(pen, B, dev, B)
            # advance off: every timed launch sees the same history
            row[f"sample_tokens_{name}_us"] = 1e3 * _events_ms(lambda: ops.sample_tokens(logits, plain, toks, 0, False), reps)
            row[f"penalized_{name}_us"] = 1e3 * _events_ms(
                lambda: ops.sample_tokens_penalized(logits, pen, toks, 0, False), reps)
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
        loops = ("static", "continuous") if B == max(batches) else ("static",)
        for loop in loops:
            for mode in ("greedy", "sampling", "penalized"):
                samp = None if mode == "greedy" else [
                    SamplingParams(0.7, 0, 0.9, seed=7 + b, **(PEN if mode == "penalized" else {})) for b in range(B)]
                firsts, caches = zip(*[_prefill(model, p) for p in prompts])
                cache = join_caches(list(caches), reserve=2 * steps + 16)
                del caches
                first = torch.cat(firsts)
                if loop == "static":
                    dec = StaticDecoder(model, cache, first, 2 * steps + 8, sampling=samp, prompts=prompts)
                    dec.run(4)                                      # capture + warm-up
                    fn = lambda: dec.run(steps)                     # noqa: E731
                else:
                    dec = ContinuousDecoder(model, cache, first, [10 ** 6] * B, chunk=steps, sampling=samp, prompts=prompts)
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
            row[f"{loop}_penalized_over_sampling_pct"] = 100 * (row[f"{loop}_penalized_step_ms"] / row[f"{loop}_sampling_step_ms"] - 1)
            row[f"{loop}_penalized_over_greedy_pct"] = 100 * (row[f"{loop}_penalized_step_ms"] / row[f"{loop}_greedy_step_ms"] - 1)
        out.append(row)
    return out


@torch.no_grad()
def hf_numbers(model, dev, prompt_len, new=33):
    from pyramidkv_b200 import runner
    ids = runner.synthetic_prompt(model.config.vocab_size, prompt_len, 100, dev).reshape(1, -1)
    res = {"batch": 1, "prompt_tokens": prompt_len, "new_tokens": new - 1}

    def run(n, rho):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        model.generate(ids, attention_mask=torch.ones_like(ids), max_new_tokens=n, min_new_tokens=n, num_beams=1,
                       do_sample=False, repetition_penalty=rho, pad_token_id=0)
        torch.cuda.synchronize()
        return time.perf_counter() - t0
    for rho in (1.0, 1.1):
        run(new, rho)                                               # warm-up
        per = (min(run(new, rho) for _ in range(3)) - min(run(1, rho) for _ in range(3))) / (new - 1)
        res[f"hf_generate_rho{rho}_step_ms"] = 1e3 * per
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", default="1,8,32,64", help="kernel batch sizes")
    ap.add_argument("--loop_batch", default="1,32", help="batch sizes of the loop measurements ('' skips them)")
    ap.add_argument("--prompt", type=int, default=1024)
    ap.add_argument("--budget", type=int, default=128)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("tools/penalty_bench.py measures on a CUDA device (H100); there is none here")
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
            res["loops"] = {"model": "llama3-8b (random init)", "method": "pyramidkv", "budget": args.budget, "penalties": PEN,
                            "rows": loop_numbers(model, dev, loop_batch, args.prompt)}
            res["hf_loop"] = hf_numbers(model, dev, args.prompt)
        finally:
            restore()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
