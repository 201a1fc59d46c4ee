#!/usr/bin/env python
"""Generation constraints on the H100: python tools/constraint_bench.py [--batch 1,8,32,64] [--history 1024,32768,131072]
[--loop_batch 1,32] [--prompt 1024]

1. Kernels (V = 128256, bf16): one pkv_token_rules launch (with its append) and one pkv_sample_tokens_constrained launch
   (T = 0.7, top_p = 0.9, the penalties of tools/penalty_bench.py) next to one pkv_sample_tokens_penalized launch, per
   batch size and history length. Every row has every rule: 20 bias sequences, no_repeat_ngram_size 3 over a history of
   a 512-token alphabet (its n-grams recur), 10 bad words, min_new_tokens 4 and 4 stop sequences. CUDA events around many
   launches.
2. HF's processor chain for the same rules (SequenceBias, NoRepeatNGram, NoBadWords, MinNewTokensLength and a
   stop-sequence criterion over the ids) at B = 1 on the GPU, per history length: what a user of these rules pays per token
   without this path.
3. Loops: the per-step time of the static loop at each --loop_batch and of the continuous loop at the largest, on a
   random-init Llama-3-8B, PyramidKV at budget 128, graph replay: greedy, penalized sampling, and penalized sampling with
   the constraints above.
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
from penalty_bench import PEN  # noqa: E402
from sampling_bench import _events_ms  # noqa: E402

V = 128256


def rules(seed):
    g = torch.Generator().manual_seed(seed)
    ids = lambda n: tuple(torch.randint(0, V, (n,), generator=g).tolist())   # noqa: E731
    return dict(sequence_bias=[(ids(1 + i % 3), 0.5 - (i % 5)) for i in range(20)], no_repeat_ngram_size=3,
                bad_words_ids=[ids(1 + i % 2) for i in range(10)], min_new_tokens=4, stop_sequences=[ids(3) for _ in range(4)])


def kernel_numbers(dev, batches, histories, reps=100):
    from pyramidkv_b200 import ops
    from pyramidkv_b200.generate import SamplingParams, SamplingState
    out = []
    for L in histories:
        for B in batches:
            g = torch.Generator(device=dev).manual_seed(B)
            logits = (torch.randn(B, V, device=dev, generator=g) * 2.5).bfloat16()
            alpha = torch.randint(0, V, (512,), device=dev, generator=g)
            prompts = [alpha[torch.randint(0, 512, (L,), device=dev, generator=g)] for _ in range(B)]
            toks = torch.randint(0, V, (B, 1), device=dev, generator=g)
            pen = SamplingState([SamplingParams(0.7, 0, 0.9, seed=b, **PEN) for b in range(B)], dev, vocab=V, prompts=prompts)
            con = SamplingState([SamplingParams(0.7, 0, 0.9, seed=b, **PEN, **rules(b)) for b in range(B)], dev, vocab=V,
                                prompts=prompts, eos=[2], history=reps + 16)
            ops.token_rules(con, V)
            lens = con.history_len.clone()
            row = {"batch": B, "history": L, "vocab": V}
            row["penalized_us"] = 1e3 * _events_ms(lambda: ops.sample_tokens_penalized(logits, pen, toks, 0, False), reps)
            row["constrained_us"] = 1e3 * _events_ms(lambda: ops.sample_tokens_constrained(logits, con, toks, 0, False), reps)
            row["token_rules_us"] = 1e3 * _events_ms(lambda: ops.token_rules(con, V, toks, 0), reps)
            con.history_len.copy_(lens)
            out.append(row)
            del pen, con
            torch.cuda.empty_cache()
    return out


@torch.no_grad()
def hf_numbers(dev, histories, reps=5):
    from transformers import LogitsProcessorList, StoppingCriteria
    from transformers.generation import logits_process as LP
    r = rules(0)

    class Stop(StoppingCriteria):
        def __call__(self, input_ids, scores, **kw):
            h = input_ids[0].tolist()
            return torch.tensor([any(h[len(h) - len(s):] == list(s) for s in r["stop_sequences"])], device=input_ids.device)
    out = []
    for L in histories:
        g = torch.Generator(device=dev).manual_seed(L)
        alpha = torch.randint(0, V, (512,), device=dev, generator=g)
        ids = alpha[torch.randint(0, 512, (1, L), device=dev, generator=g)]
        scores = torch.randn(1, V, device=dev, generator=g)
        chain = LogitsProcessorList([LP.SequenceBiasLogitsProcessor({s: w for s, w in r["sequence_bias"]}),
                                     LP.NoRepeatNGramLogitsProcessor(3), LP.NoBadWordsLogitsProcessor([list(s) for s in r["bad_words_ids"]], [2]),
                                     LP.MinNewTokensLengthLogitsProcessor(L - 2, 4, [2], device=dev)])
        stop = Stop()

        def step():
            chain(ids, scores)
            stop(ids, scores)
        step()
        out.append({"batch": 1, "history": L, "hf_processors_ms": _events_ms(step, reps)})
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
        for loop in (("static", "continuous") if B == max(batches) else ("static",)):
            for mode in ("greedy", "penalized", "constrained"):
                samp = None if mode == "greedy" else [
                    SamplingParams(0.7, 0, 0.9, seed=7 + b, **PEN, **(rules(b) if mode == "constrained" else {})) for b in range(B)]
                firsts, caches = zip(*[_prefill(model, p) for p in prompts])
                cache = join_caches(list(caches), reserve=2 * steps + 16)
                del caches
                first = torch.cat(firsts)
                if loop == "static":
                    dec = StaticDecoder(model, cache, first, 2 * steps + 8, sampling=samp, prompts=prompts)
                    dec.run(4)                                      # capture + warm-up
                    fn = lambda: dec.run(steps)                     # noqa: E731
                else:
                    dec = ContinuousDecoder(model, cache, first, [10 ** 6] * B, chunk=steps, sampling=samp, prompts=prompts,
                                            history=2 * steps + 8)
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
            row[f"{loop}_constrained_over_penalized_pct"] = 100 * (row[f"{loop}_constrained_step_ms"] / row[f"{loop}_penalized_step_ms"] - 1)
        out.append(row)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", default="1,8,32,64", help="kernel batch sizes")
    ap.add_argument("--history", default="1024,32768,131072", help="history lengths of the kernel measurements")
    ap.add_argument("--loop_batch", default="1,32", help="batch sizes of the loop measurements ('' skips them)")
    ap.add_argument("--prompt", type=int, default=1024)
    ap.add_argument("--budget", type=int, default=128)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("tools/constraint_bench.py measures on a CUDA device (H100); there is none here")
    dev = torch.device("cuda", 0)
    hist = [int(x) for x in args.history.split(",") if x.strip()]
    res = {"gpu": gpu_card(dev), "kernel": kernel_numbers(dev, [int(x) for x in args.batch.split(",") if x.strip()], hist),
           "hf_processors": hf_numbers(dev, hist)}
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
