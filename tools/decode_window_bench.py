"""Decode window (knob pkv_decode_window) on the H100: continuous batching over a random-init Llama-3-8B, PyramidKV, knob off
against R in --windows, the arms alternating in one process. Per arm: decode and wall tok/s, the mean decode step, the KV
bytes one decode step reads and one slot holds at the end of generation (computed from shapes), the largest slot count whose
caches fit next to the weights (computed from bytes, before allocating, as tools/decode_batch_bench.py does), regrowths and
graph captures. Prints one JSON line per arm and one with the card it ran on. --heavy adds, for every R, the heavy-hitter arm
H = R / 2 (knob pkv_decode_heavy) next to the ring, and one line per R with the device time of each kernel of one layer's
decode attention (torch.profiler, ring against heavy, at the slot count, with the budget as every cache head's prompt rows
and a full window). --skip_off leaves out the knob-off arm, which the ring-against-heavy comparison does not use and which
§4.7 already measures; it is the longest arm of a run.

  python tools/decode_window_bench.py --prompt 4096 --new 4096 --slots 8 --windows 256,1024 --budget 128
  python tools/decode_window_bench.py --budget 2048 --fp8 --gqa_shared
  python tools/decode_window_bench.py --windows 256,1024 --heavy --skip_off --repeats 2
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


def _kernel_us(fn, iters: int) -> dict:
    """Mean device time per launch of each decode kernel `fn` launches, in microseconds, from torch.profiler's CUDA activity
    over `iters` calls (after a warm-up): the kernels alone, without the host wrapper or the gaps between launches."""
    from torch.profiler import ProfilerActivity, profile
    for _ in range(20):
        fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(iters):
            fn()
        torch.cuda.synchronize()
    out = {}
    for e in prof.key_averages():
        for name in ("decode_heavy_kernel", "decode_combine_kernel", "decode_kernel"):
            if name in e.key:
                total = getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0.0)
                t, n = out.get(name, (0.0, 0))
                out[name] = (t + total, n + e.count)
                break
    return {k: t / n for k, (t, n) in out.items()}


def layer_kernels_us(cfg, slots: int, P: int, R: int, fp8: bool, gqa: bool, iters: int = 300) -> dict:
    """One layer's decode attention with a full window over `slots` sequences of P prompt rows: the device time of each kernel
    of a ring step (`decode_attn_window`) and of a heavy step, H = R / 2 (`decode_attn_heavy`: the decode kernel with the
    logit stores, the combine with its (m, l) stores when the rows are split, and `decode_heavy_kernel`)."""
    from pyramidkv_b200 import ops
    dev = torch.device("cuda", 0)
    Hq, Hkv = cfg.num_attention_heads, cfg.num_key_value_heads
    D = cfg.hidden_size // Hq
    H = Hkv if gqa else Hq
    cap = P + R
    g = torch.Generator(device=dev).manual_seed(0)
    k = torch.randn(slots, H, cap, D, generator=g, device=dev).bfloat16()
    v = torch.randn(slots, H, cap, D, generator=g, device=dev).bfloat16()
    scales = None
    if fp8:
        amax = k.float().abs().amax(-1).clamp_min(1e-6)
        scales = (amax / 448, v.float().abs().amax(-1).clamp_min(1e-6) / 448)
        k = (k.float() / scales[0][..., None]).to(torch.float8_e4m3fn)
        v = (v.float() / scales[1][..., None]).to(torch.float8_e4m3fn)
    q = torch.randn(slots, Hq, D, generator=g, device=dev).bfloat16()
    kn = torch.randn(slots, Hkv, D, generator=g, device=dev).bfloat16()
    vn = torch.randn(slots, Hkv, D, generator=g, device=dev).bfloat16()
    prompt_rows = torch.full((slots * H,), P, dtype=torch.int32, device=dev)
    rows = prompt_rows.clone()
    ws = torch.empty(ops.decode_workspace_bytes(slots * Hq, D), dtype=torch.uint8, device=dev)
    scratch = torch.empty(ops.decode_heavy_workspace_bytes(slots, Hq, R), dtype=torch.uint8, device=dev)
    state = (torch.zeros(slots, H, R, device=dev), torch.full((slots, H, R), -1, dtype=torch.int32, device=dev),
             torch.full((slots * H,), -1, dtype=torch.int32, device=dev))
    out = torch.empty_like(q)
    # the step counter advances with every launch, as in a decode loop: each launch appends the next generated row (a count
    # that repeats would append the same generation again, which is not a decode step)
    step = torch.zeros(1, dtype=torch.int32, device=dev)

    def ring():
        ops.decode_attn_window(q, k, v, 1, kn, vn, prompt_rows, R, rows=rows, step=step, max_length=cap, workspace=ws, out=out,
                               scales=scales, gqa=gqa)
        step.add_(1)

    def heavy():
        ops.decode_attn_heavy(q, k, v, 1, kn, vn, prompt_rows, R, R // 2, *state, rows=rows, step=step, max_length=cap,
                              workspace=ws, scratch=scratch, out=out, scales=scales, gqa=gqa)
        step.add_(1)

    for _ in range(2 * R):                            # fill the window: every timed launch replaces a row
        heavy()
    runs = {"ring": [], "heavy": []}
    for _ in range(2):                                # alternating, to show the spread
        runs["ring"].append(_kernel_us(ring, iters))
        runs["heavy"].append(_kernel_us(heavy, iters))
    ring_total = min(sum(r.values()) for r in runs["ring"])
    heavy_total = min(sum(r.values()) for r in runs["heavy"])
    return {"window": R, "heavy": R // 2, "slots": slots, "prompt_rows": P, "ring_kernels_us": ring_total,
            "heavy_kernels_us": heavy_total, "heavy_extra_us": heavy_total - ring_total, "runs": runs}


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--prompt", type=int, default=4096)
    ap.add_argument("--new", type=int, default=4096, help="max_new_tokens of every request")
    ap.add_argument("--slots", type=int, default=8)
    ap.add_argument("--requests", type=int, default=0, help="prompts (default: the slot count)")
    ap.add_argument("--budget", type=int, default=128)
    ap.add_argument("--windows", default="256,1024", help="comma-separated R; the knob off runs too unless --skip_off")
    ap.add_argument("--fp8", action="store_true")
    ap.add_argument("--gqa_shared", action="store_true")
    ap.add_argument("--repeats", type=int, default=1, help="rounds of the alternating arms")
    ap.add_argument("--heavy", action="store_true", help="add the heavy-hitter arm H = R / 2 for every R")
    ap.add_argument("--skip_off", action="store_true", help="leave out the knob-off arm")
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
    windows = [int(w) for w in a.windows.split(",") if w]
    arms = ([] if a.skip_off else [(None, None)]) + [x for R in windows for x in [(R, None)] + ([(R, R // 2)] if a.heavy else [])]
    if a.heavy:
        for R in windows:
            print(json.dumps({"layer_kernels": layer_kernels_us(cfg, a.slots, a.budget, R, a.fp8, a.gqa_shared)}), flush=True)
    G.greedy_generate_continuous(model, prompts[:1], 4, 1)                       # warm-up: modules, cuBLAS, allocator
    for rep in range(a.repeats):
        for R, H in arms:
            cfg.pkv_decode_window, cfg.pkv_decode_heavy = R, H
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
                "repeat": rep, "decode_window": R, "decode_heavy": H, "decode_steps": st["decode_steps"],
                "decode_ms_per_step": 1e3 * st["decode_s"] / max(1, st["decode_steps"]),
                "decode_tok_per_s": st["live_slot_steps"] / st["decode_s"], "wall_tok_per_s": generated / wall,
                # the last step reads every live slot's rows once (K and V)
                "kv_bytes_per_step_last": slot_bytes * a.slots, "bytes_per_slot_end": slot_bytes,
                "max_slots_that_fit": int((HBM_BYTES - weights - 4 * 2 ** 30) // slot_bytes),
                "regrowths": st["regrowths"], "graph_captures": st["graph_captures"],
                "ms_per_step_at_1_1k_2k_4k": "not measured"}), flush=True)
    cfg.pkv_decode_window = cfg.pkv_decode_heavy = None


if __name__ == "__main__":
    main()
