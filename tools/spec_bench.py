"""Prompt-lookup speculative decoding on the H100 (DESIGN.md §4.13): Llama-3-8B random-init, PyramidKV budgets, prompts of
S tokens, B sequences, K draft tokens. Per configuration, CUDA events around graph replays:
  - plain: the greedy step of StaticDecoder (one token per sequence);
  - verify: one SpeculativeDecoder step (Q = K + 1 rows per sequence), its drafts forced to be all rejected (one token per
    sequence per step) and all accepted (K + 1 tokens per step), as tokens/s - the two bound what real drafts give;
  - natural: the lookup's own drafts; its acceptance on random-init weights says nothing about a trained model.
And the verify attention alone: pkv_decode_attn_multi against Q launches of pkv_decode_attn_batch over the same rows.
The card's name and power limit are read in the same run. Writes one JSON file (--out) and prints it."""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card() -> dict:
    out = {"name": torch.cuda.get_device_name(0)}
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        out["power_limit_and_max_sm_clock"] = r.stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        out["power_limit_and_max_sm_clock"] = f"not read ({type(e).__name__})"
    return out


def timed(fn, n: int) -> float:
    """ms per call of fn over n calls (after one warm-up call), CUDA events."""
    fn()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    for _ in range(n):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / n


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
    q1 = [q[:, j].contiguous() for j in range(Q)]
    k1 = [kn[:, j].contiguous() for j in range(Q)]
    v1 = [vn[:, j].contiguous() for j in range(Q)]
    out1 = torch.empty(B, Hq, D, dtype=torch.bfloat16, device=dev)

    def singles():
        for j in range(Q):
            ops.decode_attn_batch(q1[j], k, v, 1 + j, k1[j], v1[j], rows=r, workspace=ws, out=out1)
    single = timed(singles, iters)
    return {"B": B, "Q": Q, "rows": rows, "Hq": Hq, "Hkv": Hkv, "D": D, "multi_ms": round(multi, 4),
            "q_single_launches_ms": round(single, 4), "speedup": round(single / multi, 3)}


@torch.no_grad()
def e2e(model, S: int, B: int, ks, steps: int) -> dict:
    from pyramidkv_b200 import generate as G
    from pyramidkv_b200 import runner
    dev = torch.device("cuda", 0)
    prompts = []
    for b in range(B):
        # LongBench-like: a prompt that repeats spans of itself
        base = runner.synthetic_prompt(model.config.vocab_size, 512, 100 + b, dev)[0]
        prompts.append(base.repeat(-(-S // 512))[:S])
    firsts, caches = [], []
    for p in prompts:
        f, c = G._prefill(model, p.reshape(1, -1))
        firsts.append(f)
        caches.append(c)
    first = torch.cat(firsts)
    T = steps + 1
    res = {"S": S, "B": B}
    dec = G.StaticDecoder(model, G.join_caches(caches, reserve=T), first, steps)
    dec.run(1)
    torch.cuda.synchronize()
    a, b_ = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    dec.run(steps - 1)
    b_.record()
    torch.cuda.synchronize()
    plain_ms = a.elapsed_time(b_) / (steps - 1)
    table = torch.cat([first, dec.tokens], dim=1)
    res["plain_step_ms"] = round(plain_ms, 3)
    res["plain_tok_s"] = round(B * 1000.0 / plain_ms, 1)
    V = model.config.vocab_size
    for K in ks:
        row = {}
        for mode, forced in (("all_rejected", (table + 1) % V), ("all_accepted", table), ("natural", None)):
            sd = G.SpeculativeDecoder(model, G.join_caches(caches, reserve=T + K + 1), first, prompts, T, K,
                                      forced_drafts=forced)
            sd.run(1)
            torch.cuda.synchronize()
            e0 = int(sd.spec.out_len.sum())
            n = max(1, min(steps - 1, -(-steps // (K + 1)) if mode == "all_accepted" else steps - 1) - 1)
            a.record()
            sd.run(n)
            b_.record()
            torch.cuda.synchronize()
            ms = a.elapsed_time(b_)
            emitted = int(sd.spec.out_len.sum()) - e0
            row[mode] = {"step_ms": round(ms / n, 3), "tok_s": round(emitted * 1000.0 / ms, 1),
                         "tokens_per_step_per_seq": round(emitted / (n * B), 3)}
            sd.finish([0] * B)
        row["verify_over_plain_step"] = round(row["all_rejected"]["step_ms"] / plain_ms, 3)
        row["natural"]["note"] = "random-init weights: acceptance says nothing about a trained model"
        res[f"K{K}"] = row
    return res


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--budgets", type=int, nargs="+", default=[128, 2048])
    ap.add_argument("--prompts", type=int, nargs="+", default=[4096, 32768])
    ap.add_argument("--batches", type=int, nargs="+", default=[1, 8])
    ap.add_argument("--ks", type=int, nargs="+", default=[2, 4, 8])
    ap.add_argument("--steps", type=int, default=48)
    ap.add_argument("--skip-e2e", action="store_true")
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("spec_bench measures on a CUDA device; none is visible")
    from pyramidkv_b200 import runner
    res = {"card": card(), "kernel": kernel_bench(), "e2e": []}
    print(json.dumps({"card": res["card"], "kernel": res["kernel"]}), flush=True)
    if not args.skip_e2e:
        runner.patch("pyramidkv")
        model = runner.build_model("llama3-8b", torch.device("cuda", 0), torch.bfloat16, "sdpa")
        model.config.pkv_fused_rope = True
        for budget in args.budgets:
            runner.set_knobs(model, "pyramidkv", budget)
            for S in args.prompts:
                for B in args.batches:
                    if S * B > 65536:
                        continue   # 32K prompts at B = 1 only: eight of them would spend minutes in prefill
                    r = e2e(model, S, B, args.ks, args.steps)
                    r["budget"] = budget
                    res["e2e"].append(r)
                    print(json.dumps(r), flush=True)
    text = json.dumps(res, indent=1)
    print(text)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(text)


if __name__ == "__main__":
    main()
