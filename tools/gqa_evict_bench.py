#!/usr/bin/env python
"""Per-prompt eviction time with and without GQA-shared selection: python tools/gqa_evict_bench.py [--ctx 32768] [--budget 128,2048]

Llama-3-8B geometry (32 layers, 32 query heads, 8 KV heads, head_dim 128, bf16), PyramidKV with the reference runners' knobs
(window 8, kernel 7, maxpool) and its per-layer budgets. For one prompt of --ctx tokens it times the eviction of all 32 layers
as the patched prefill runs it:
  off  the per-query-head caches: the deferred layer batch (pkv_evict_prefill_batch, four launches per 32 layers)
  on   PKV_FLAG_GQA_SHARED: per layer scores, pool, group reduction, select + gather into one cache per KV head (the layer
       batch is not built for the flag)
The two modes alternate in the same process, CUDA events around --reps repetitions of the 32 layers. Random inputs; two sets of
layer inputs alternate so that consecutive layers do not read the same K from L2. Prints one JSON line with the card's name and
power limit. Writes nothing but stdout.
"""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from decode_batch_bench import gpu_card  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ctx", type=int, default=32768)
    ap.add_argument("--budget", default="128,2048")
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("tools/gqa_evict_bench.py measures on a CUDA device (H100); there is none here")
    from pyramidkv_b200 import ops
    dev = torch.device("cuda", 0)
    L, Hq, Hkv, D, W, S = 32, 32, 8, 128, 8, args.ctx
    g = torch.Generator(device=dev).manual_seed(0)
    sets = [(torch.randn(Hq, W, D, generator=g, device=dev).bfloat16(), torch.randn(Hkv, S, D, generator=g, device=dev).bfloat16(),
             torch.randn(Hkv, S, D, generator=g, device=dev).bfloat16()) for _ in range(2)]
    results = []
    for budget in [int(x) for x in args.budget.split(",") if x.strip()]:
        ks = [ops.layer_budget("pyramidkv", budget, W, L, l, S)[1] for l in range(L)]
        runs = {}
        for gqa in (False, True):
            H = Hkv if gqa else Hq
            caches = [tuple(torch.empty(H, k + W, D, dtype=torch.bfloat16, device=dev) for _ in range(2)) for k in ks]
            if gqa:
                plans = [ops.plan_evict("pyramidkv", *sets[l % 2], W, ks[l], *caches[l], 7, "maxpool", inputs_ready=True, gqa_shared=True)
                         for l in range(L)]
                run = lambda plans=plans: [ops.run_stage(p, "all") for p in plans]
            else:
                probe = ops.plan_evict("pyramidkv", *sets[0], W, ks[0], *caches[0], 7, "maxpool", inputs_ready=True)
                wss = ops.batch_workspaces(probe, L, max(ks))
                batch = ops.EvictBatch([ops.plan_evict("pyramidkv", *sets[l % 2], W, ks[l], *caches[l], 7, "maxpool", inputs_ready=True,
                                                       workspace=wss[l]) for l in range(L)])
                run = batch.run
            runs[gqa] = (run, caches)
        times = {False: [], True: []}
        for gqa in (False, True):
            runs[gqa][0]()                                        # warm-up
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        for _ in range(args.reps):
            for gqa in (False, True):
                e0.record()
                runs[gqa][0]()
                e1.record()
                torch.cuda.synchronize()
                times[gqa].append(e0.elapsed_time(e1))
        results.append({"budget": budget, "top_k_first_last": [ks[0], ks[-1]],
                        "evict_ms_off": min(times[False]), "evict_ms_on": min(times[True]),
                        "evict_ms_off_all": times[False], "evict_ms_on_all": times[True],
                        "cache_bytes_off": sum(2 * c[0].numel() * 2 for c in runs[False][1]),
                        "cache_bytes_on": sum(2 * c[0].numel() * 2 for c in runs[True][1])})
        del runs
        torch.cuda.empty_cache()
    print(json.dumps({"model": "llama3-8b geometry", "method": "pyramidkv", "ctx": S, "layers": L, "gpu": gpu_card(dev),
                      "reps": args.reps, "results": results}))


if __name__ == "__main__":
    main()
