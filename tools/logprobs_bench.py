#!/usr/bin/env python
"""Token log-probabilities on the H100: python tools/logprobs_bench.py [--batch 1,8,32,64] [--skip_loops] [--skip_fidelity]

1. Kernel: one pkv_token_logprobs launch (V = 128256, bf16 logits) per batch size and top N in {0, 5, 20}, next to the torch
   chain log_softmax(float) + gather + topk on the same logits, both timed with CUDA events in the same run.
2. Step overhead: the per-step time of the static loop (B = 1 and 32) and of the continuous loop (16 slots, every slot
   live) with and without logprobs=5, on a random-init Llama-3-8B, PyramidKV at budget 128, graph replay.
3. Fidelity: seeded prompts and one fixed seeded continuation scored by `score_continuations` under each cache form, against
   the bf16 per-query-head cache at the same budget and against the uncompressed model (one plain forward over prompt +
   continuation under replace_llama("fullkv"), log_softmax over the continuation positions): mean and max |delta log-prob|
   per token and top-1 agreement. Random-init weights: this measures how far each form moves the model's distribution,
   not task accuracy.
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
    from pyramidkv_b200 import ops
    out = []
    for B in batches:
        g = torch.Generator(device=dev).manual_seed(B)
        logits = (torch.randn(B, V, device=dev, generator=g) * 2.5).bfloat16()
        toks = torch.randint(0, V, (B, 1), device=dev, generator=g)
        row = {"batch": B, "vocab": V, "logit_bytes": B * V * 2}
        for N in (0, 5, 20):
            lp = torch.empty(B, 1, device=dev)
            ids = torch.empty(B, 1, N, dtype=torch.long, device=dev)
            top = torch.empty(B, 1, N, device=dev)
            row[f"pkv_token_logprobs_n{N}_us"] = 1e3 * _events_ms(lambda: ops.token_logprobs(logits, toks, lp, ids, top), reps)

            def chain():
                ls = torch.log_softmax(logits.float(), dim=-1)
                r = ls.gather(1, toks)
                return (r, torch.topk(ls, N, dim=-1)) if N else r
            row[f"torch_log_softmax_gather_topk_n{N}_us"] = 1e3 * _events_ms(chain, reps)
        row["one_pass_over_logits_at_3.35TB/s_us"] = row["logit_bytes"] / 3.35e12 * 1e6
        out.append(row)
    return out


def _timed_ms(fn, steps):
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / steps


@torch.no_grad()
def loop_numbers(model, dev, prompt_len, steps=64):
    from pyramidkv_b200 import runner
    from pyramidkv_b200.cache import join_caches
    from pyramidkv_b200.generate import ContinuousDecoder, StaticDecoder, _prefill
    out = []
    for loop, B in (("static", 1), ("static", 32), ("continuous", 16)):
        prompts = [runner.synthetic_prompt(model.config.vocab_size, prompt_len, 100 + i, dev) for i in range(B)]
        row = {"loop": loop, "batch": B, "prompt_tokens": prompt_len, "timed_steps": steps}
        # alternate off / on twice: the spread of the same setting is part of the number
        for rep in range(2):
            for lp in (None, 5):
                firsts, caches = zip(*[_prefill(model, p) for p in prompts])
                cache = join_caches(list(caches), reserve=2 * steps + 16)
                del caches
                first = torch.cat(firsts)
                if loop == "static":
                    dec = StaticDecoder(model, cache, first, 2 * steps + 8, logprobs=lp)
                    dec.run(4)                                      # capture + warm-up
                    ms = _timed_ms(lambda: dec.run(steps), steps)
                else:
                    dec = ContinuousDecoder(model, cache, first, [10 ** 6] * B, chunk=steps, logprobs=lp)
                    dec.run_chunk(4)
                    ms = _timed_ms(lambda: dec.run_chunk(steps), steps)
                row.setdefault("off_step_ms" if lp is None else "logprobs5_step_ms", []).append(ms)
                dec.finish()
                del dec, cache
                torch.cuda.empty_cache()
        off, on = min(row["off_step_ms"]), min(row["logprobs5_step_ms"])
        row["overhead_pct_of_best"] = 100 * (on / off - 1)
        out.append(row)
    return out


def _knobs(model, budget, fp8=False, gqa=False, window=None, heavy=None):
    for layer in model.model.layers:                               # run_longbench.py:253-261
        c = layer.self_attn.config
        c.window_size, c.max_capacity_prompt, c.kernel_size, c.pooling = 8, budget, 7, "maxpool"
    model.config.pkv_kv_cache_dtype = "fp8_e4m3" if fp8 else None
    model.config.pkv_gqa_shared = bool(gqa)
    model.config.pkv_decode_window = window
    model.config.pkv_decode_heavy = heavy


def _diff(e, ref_lp, ref_top1):
    d = (e.logprobs.double() - ref_lp).abs()
    return {"mean_abs_dlogprob": float(d.mean()), "max_abs_dlogprob": float(d.max()),
            "top1_agreement": float((e.top_ids[:, 0] == ref_top1).double().mean())}


@torch.no_grad()
def fidelity(model, dev, n_prompts, prompt_len, cont_len, budgets):
    from pyramidkv.monkeypatch import replace_llama
    from pyramidkv_b200 import runner
    from pyramidkv_b200.generate import score_continuations
    prompts = [runner.synthetic_prompt(model.config.vocab_size, prompt_len, 500 + i, dev) for i in range(n_prompts)]
    cont = runner.synthetic_prompt(model.config.vocab_size, cont_len, 999, dev)[0]
    conts = [cont] * n_prompts
    with contextlib.redirect_stdout(io.StringIO()):
        replace_llama("fullkv")
    _knobs(model, budgets[0])
    full_lp, full_top1 = [], []
    for p in prompts:
        ids = torch.cat([p[0], cont]).reshape(1, -1)
        logits = model(input_ids=ids, use_cache=False, logits_to_keep=cont_len + 1).logits[0, :-1].float()
        ls = torch.log_softmax(logits, dim=-1)
        full_lp.append(ls.gather(1, cont.reshape(-1, 1))[:, 0].double().cpu())
        full_top1.append(ls.argmax(dim=-1).cpu())
        del logits, ls
    with contextlib.redirect_stdout(io.StringIO()):
        replace_llama("pyramidkv")
    forms = [("bf16", {}), ("fp8", dict(fp8=True)), ("gqa_shared", dict(gqa=True)), ("gqa_shared_fp8", dict(fp8=True, gqa=True)),
             ("window_256", dict(window=256)), ("window_1024", dict(window=1024)),
             ("heavy_256_128", dict(window=256, heavy=128)), ("heavy_1024_512", dict(window=1024, heavy=512))]
    rows = []
    for budget in budgets:
        base = None
        for name, kw in forms:
            _knobs(model, budget, **kw)
            got = score_continuations(model, prompts, conts, top_n=1)
            torch.cuda.empty_cache()
            if base is None:
                base = got
            vs_full = [_diff(e, f, t) for e, f, t in zip(got, full_lp, full_top1)]
            vs_bf16 = [_diff(e, b.logprobs.double(), b.top_ids[:, 0]) for e, b in zip(got, base)]
            avg = lambda rs, k: sum(r[k] for r in rs) / len(rs)                 # noqa: E731
            mx = lambda rs, k: max(r[k] for r in rs)                            # noqa: E731
            rows.append({"budget": budget, "form": name,
                         "vs_fullkv": {"mean_abs_dlogprob": avg(vs_full, "mean_abs_dlogprob"),
                                       "max_abs_dlogprob": mx(vs_full, "max_abs_dlogprob"),
                                       "top1_agreement": avg(vs_full, "top1_agreement")},
                         "vs_bf16_cache": {"mean_abs_dlogprob": avg(vs_bf16, "mean_abs_dlogprob"),
                                           "max_abs_dlogprob": mx(vs_bf16, "max_abs_dlogprob"),
                                           "top1_agreement": avg(vs_bf16, "top1_agreement")},
                         "mean_logprob": float(torch.cat([e.logprobs for e in got]).double().mean())})
    _knobs(model, budgets[0])
    return {"prompts": n_prompts, "prompt_tokens": prompt_len, "continuation_tokens": cont_len,
            "fullkv_mean_logprob": float(torch.cat(full_lp).mean()), "rows": rows}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", default="1,8,32,64", help="kernel batch sizes")
    ap.add_argument("--skip_loops", action="store_true")
    ap.add_argument("--skip_fidelity", action="store_true")
    ap.add_argument("--prompt", type=int, default=1024, help="prompt tokens of the step-overhead loops")
    ap.add_argument("--fid_prompts", type=int, default=4)
    ap.add_argument("--fid_prompt", type=int, default=3000)
    ap.add_argument("--fid_cont", type=int, default=1100, help="forced continuation tokens (above the largest window R)")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("tools/logprobs_bench.py measures on a CUDA device (H100); there is none here")
    dev = torch.device("cuda", 0)
    res = {"gpu": gpu_card(dev), "kernel": kernel_numbers(dev, [int(x) for x in args.batch.split(",") if x.strip()])}
    if not (args.skip_loops and args.skip_fidelity):
        from pyramidkv.monkeypatch import replace_llama, restore
        model = build_model("llama3-8b", dev)
        with contextlib.redirect_stdout(io.StringIO()):
            replace_llama("pyramidkv")
        try:
            _knobs(model, 128)
            model.config.pkv_fused_rope = True
            if not args.skip_loops:
                res["loops"] = {"model": "llama3-8b (random init)", "method": "pyramidkv", "budget": 128,
                                "rows": loop_numbers(model, dev, args.prompt)}
            if not args.skip_fidelity:
                res["fidelity"] = {"model": "llama3-8b (random init)", "method": "pyramidkv",
                                   **fidelity(model, dev, args.fid_prompts, args.fid_prompt, args.fid_cont, (128, 2048))}
        finally:
            restore()
    res["gpu_after"] = gpu_card(dev)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
