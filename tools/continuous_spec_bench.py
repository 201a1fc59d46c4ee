"""Prompt-lookup speculation in the continuous loop on the H100 (DESIGN.md §4.14): Llama-3-8B random-init, PyramidKV
budgets, prompts of S tokens that repeat spans of themselves, B slots, K draft tokens, D draft tokens per step. Per
configuration, CUDA events around graph replays of one decoder over the same joined cache (row counts restored between
runs; no slot finishes inside the timed window):
  - plain: the ContinuousDecoder step (one token per slot);
  - natural: the ContinuousSpecDecoder step with the lookup's own drafts - its acceptance on random-init weights says
    nothing about a trained model;
  - accepted: the same step with drafts forced to the greedy continuation (every granted draft is accepted).
Each reports ms per step, tokens/s and the granted / accepted draft totals. And the attention alone: pkv_decode_attn_packed
against pkv_decode_attn_multi at equal shapes, and with half of the counts at 0. The card's name and power limit are read
in the same run. Writes one JSON file (--out) and prints it."""
from __future__ import annotations

import argparse
import json
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)

from spec_bench import card, timed  # noqa: E402


@torch.no_grad()
def kernel_bench(B=64, Q=5, rows=2048, Hq=32, Hkv=8, D=128, iters=50) -> dict:
    from pyramidkv_b200 import ops
    dev = torch.device("cuda", 0)
    g = torch.Generator(device=dev).manual_seed(0)
    cap = rows + Q + 64
    k = torch.randn(B, Hq, cap, D, device=dev, generator=g).bfloat16()
    v = torch.randn_like(k)
    q = torch.randn(B, Q, Hq, D, device=dev, generator=g).bfloat16()
    kn = torch.randn(B, Q, Hkv, D, device=dev, generator=g).bfloat16()
    vn = torch.randn_like(kn)
    r = torch.full((B * Hq,), rows, dtype=torch.int32, device=dev)
    ws = torch.empty(ops.decode_workspace_bytes(B * Hq * Q, D), dtype=torch.uint8, device=dev)
    out = torch.empty(B, Q, Hq, D, dtype=torch.bfloat16, device=dev)
    multi = timed(lambda: ops.decode_attn_multi(q, k, v, kn, vn, rows=r, workspace=ws, out=out), iters)
    M = B * Q
    qp, kp, vp, op = q.view(1, M, Hq, D), kn.view(1, M, Hkv, D), vn.view(1, M, Hkv, D), out.view(1, M, Hq, D)
    start = torch.arange(B, dtype=torch.int32, device=dev) * Q
    full = torch.full((B,), Q, dtype=torch.int32, device=dev)
    half = full.clone()
    half[1::2] = 0
    res = {"B": B, "Q": Q, "rows": rows, "Hq": Hq, "Hkv": Hkv, "D": D, "multi_ms": round(multi, 4)}
    for name, count in (("packed_ms", full), ("packed_half_zero_ms", half)):
        ms = timed(lambda: ops.decode_attn_packed(qp, k, v, kp, vp, start, count, Q, rows=r, workspace=ws, out=op), iters)
        res[name] = round(ms, 4)
    return res


def _time(dec, steps: int):
    """(ms per step, tokens emitted) over `steps` graph replays after the capture."""
    if dec.graph is None:
        dec._capture()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    dec.run(steps)
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / steps


@torch.no_grad()
def e2e(model, caches, firsts, prompts, B: int, ks, steps: int) -> dict:
    from pyramidkv_b200 import generate as G
    T = (max(ks) + 1) * (steps + 1) + max(ks) + 1
    cache = G.join_caches(caches[:B], reserve=T + 2)
    first = torch.cat(firsts[:B])
    rows0 = [l.rows.clone() for l in cache.layers]

    def restore():
        for l, r in zip(cache.layers, rows0):
            l.rows.copy_(r)

    res = {"B": B}
    plain = G.ContinuousDecoder(model, cache, first, [T] * B, T)
    plain.run(1)
    plain_ms = _time(plain, steps)
    plain.run(T - 1 - steps)
    table = torch.cat([first, plain.tokens[:, :T]], dim=1)                # the greedy continuation of every slot
    plain.finish()
    restore()
    res["plain"] = {"step_ms": round(plain_ms, 3), "tok_s": round(B * 1000.0 / plain_ms, 1)}
    left = [(max(ks) + 1) * (steps + 1)] * B
    for K in ks:
        for D in sorted({B * K, B, max(1, B // 2)}, reverse=True):
            row = {}
            for mode, forced in (("natural", None), ("accepted", table)):
                dec = G.ContinuousSpecDecoder(model, cache, first, [p.reshape(-1) for p in prompts[:B]], left, steps, K, 2, D,
                                              forced_drafts=forced)
                ms = _time(dec, steps)
                n = int(dec.spec.out_len.sum())
                granted, live = dec.state.pack.totals.tolist()
                row[mode] = {"step_ms": round(ms, 3), "tok_s": round(n * 1000.0 / (ms * steps), 1),
                             "granted_drafts": granted, "accepted_drafts": n - live,
                             "step_over_plain": round(ms / plain_ms, 3)}
                dec.finish()
                restore()
            row["natural"]["note"] = "random-init weights: acceptance says nothing about a trained model"
            res[f"K{K}_D{D}"] = row
    del cache
    torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--budgets", type=int, nargs="+", default=[128, 2048])
    ap.add_argument("--prompt", type=int, default=2048, help="prompt tokens")
    ap.add_argument("--slots", type=int, nargs="+", default=[1, 8, 32, 64])
    ap.add_argument("--ks", type=int, nargs="+", default=[2, 4, 8])
    ap.add_argument("--steps", type=int, default=12)
    ap.add_argument("--per-query-head", action="store_true",
                    help="one cache per query head; the default holds one per KV head (pkv_gqa_shared), so that 64 slots "
                         "of 2048 rows fit in 80 GB next to their prefills")
    ap.add_argument("--skip-e2e", action="store_true")
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("continuous_spec_bench measures on a CUDA device; none is visible")
    from pyramidkv_b200 import generate as G
    from pyramidkv_b200 import runner
    res = {"card": card(), "kernel": [kernel_bench(), kernel_bench(Q=9)], "e2e": []}
    print(json.dumps({"card": res["card"], "kernel": res["kernel"]}), flush=True)
    if not args.skip_e2e:
        runner.patch("pyramidkv")
        dev = torch.device("cuda", 0)
        model = runner.build_model("llama3-8b", dev, torch.bfloat16, "sdpa")
        model.config.pkv_fused_rope = True
        model.config.pkv_gqa_shared = not args.per_query_head
        res["gqa_shared"] = not args.per_query_head
        prompts = []
        for b in range(max(args.slots)):
            base = runner.synthetic_prompt(model.config.vocab_size, 256, 100 + b, dev)[0]
            prompts.append(base.repeat(-(-args.prompt // 256))[: args.prompt].reshape(1, -1))
        for budget in args.budgets:
            runner.set_knobs(model, "pyramidkv", budget)
            firsts, caches = [], []
            with torch.no_grad():
                for p in prompts:
                    f, c = G._prefill(model, p)
                    firsts.append(f)
                    caches.append(c)
            for B in args.slots:
                r = e2e(model, caches, firsts, prompts, B, args.ks, args.steps)
                r.update(budget=budget, prompt=args.prompt)
                res["e2e"].append(r)
                print(json.dumps(r), flush=True)
            del caches
            torch.cuda.empty_cache()
    text = json.dumps(res, indent=1)
    print(text)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(text)


if __name__ == "__main__":
    main()
