"""Decode window (knob pkv_decode_window) on the H100: continuous batching over a random-init Llama-3-8B, PyramidKV, knob off
against R in --windows, the arms alternating in one process. Per arm: decode and wall tok/s, the mean decode step, the KV
bytes one decode step reads and one slot holds at the end of generation (computed from shapes), the largest slot count whose
caches fit next to the weights (computed from bytes, before allocating, as tools/decode_batch_bench.py does), regrowths and
graph captures. Prints one JSON line per arm and one with the card it ran on.

  python tools/decode_window_bench.py --prompt 4096 --new 4096 --slots 8 --windows 256,1024 --budget 128
  python tools/decode_window_bench.py --budget 2048 --fp8 --gqa_shared
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402

from pyramidkv_b200 import generate as G  # noqa: E402
from pyramidkv_b200 import runner  # noqa: E402

HBM_BYTES = 80 * 2 ** 30


def card() -> dict:
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    name, power = (r.stdout.strip().split(", ") + ["?", "?"])[:2]
    return {"gpu": name, "power_limit": power}


def cache_bytes(cfg, rows_per_layer, fp8: bool, gqa: bool) -> int:
    """Bytes of one sequence's K and V over all layers with rows_per_layer[l] rows per cache head (FP8: + two fp32 scales)."""
    heads = cfg.num_key_value_heads if gqa else cfg.num_attention_heads
    D = cfg.hidden_size // cfg.num_attention_heads
    per_row = 2 * (D * (1 if fp8 else 2) + (4 if fp8 else 0))
    return sum(r * heads * per_row for r in rows_per_layer)


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--prompt", type=int, default=4096)
    ap.add_argument("--new", type=int, default=4096, help="max_new_tokens of every request")
    ap.add_argument("--slots", type=int, default=8)
    ap.add_argument("--requests", type=int, default=0, help="prompts (default: the slot count)")
    ap.add_argument("--budget", type=int, default=128)
    ap.add_argument("--windows", default="256,1024", help="comma-separated R; the knob off always runs too")
    ap.add_argument("--fp8", action="store_true")
    ap.add_argument("--gqa_shared", action="store_true")
    ap.add_argument("--repeats", type=int, default=1, help="rounds of the alternating arms")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("decode_window_bench needs a CUDA device (H100)")
    dev = torch.device("cuda", 0)
    runner.patch("pyramidkv")
    model = runner.build_model("llama3-8b", dev, torch.bfloat16, "sdpa")
    runner.set_knobs(model, "pyramidkv", a.budget)
    if a.fp8:
        model.config.pkv_kv_cache_dtype = "fp8_e4m3"
    if a.gqa_shared:
        model.config.pkv_gqa_shared = True
    cfg = model.config
    weights = sum(p.numel() * p.element_size() for p in model.parameters())
    prompts = [runner.synthetic_prompt(cfg.vocab_size, a.prompt, 100 + i, dev) for i in range(a.requests or a.slots)]
    print(json.dumps({"card": card(), "prompt": a.prompt, "new": a.new, "slots": a.slots, "budget": a.budget, "fp8": a.fp8,
                      "gqa_shared": a.gqa_shared}), flush=True)
    arms = [None] + [int(w) for w in a.windows.split(",") if w]
    G.greedy_generate_continuous(model, prompts[:1], 4, 1)                       # warm-up: modules, cuBLAS, allocator
    for rep in range(a.repeats):
        for R in arms:
            cfg.pkv_decode_window = R
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            seqs, st = G.greedy_generate_continuous(model, prompts, a.new, a.slots, check_every=64, return_stats=True)
            torch.cuda.synchronize()
            wall = time.perf_counter() - t0
            prompt_rows = st["cache_rows_first_last"][0]
            # rows per cache head at the end of generation: the prompt's (first / last layer, pyramidal in between) + decoded
            P = [round(prompt_rows[0] + (prompt_rows[1] - prompt_rows[0]) * l / (cfg.num_hidden_layers - 1))
                 for l in range(cfg.num_hidden_layers)]
            kept = a.new - 1 if R is None else min(a.new - 1, R)
            slot_bytes = cache_bytes(cfg, [p + kept for p in P], a.fp8, a.gqa_shared)
            generated = sum(len(s) for s in seqs) - a.prompt * len(seqs)
            print(json.dumps({
                "repeat": rep, "decode_window": R, "decode_steps": st["decode_steps"],
                "decode_ms_per_step": 1e3 * st["decode_s"] / max(1, st["decode_steps"]),
                "decode_tok_per_s": st["live_slot_steps"] / st["decode_s"], "wall_tok_per_s": generated / wall,
                # the last step reads every live slot's rows once (K and V)
                "kv_bytes_per_step_last": slot_bytes * a.slots, "bytes_per_slot_end": slot_bytes,
                "max_slots_that_fit": int((HBM_BYTES - weights - 4 * 2 ** 30) // slot_bytes),
                "regrowths": st["regrowths"], "graph_captures": st["graph_captures"],
                "ms_per_step_at_1_1k_2k_4k": "not measured"}), flush=True)
    cfg.pkv_decode_window = None


if __name__ == "__main__":
    main()
