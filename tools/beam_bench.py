#!/usr/bin/env python
"""Beam search on the H100: python tools/beam_bench.py [--prompt 32768] [--budgets 128,2048] [--beams 2,4,8] [--new 256]
[--kernels_only] [--skip_hf]

1. Kernels: CUDA-event µs of one pkv_beam_candidates launch (k rows of V = 128256 bf16 logits), one pkv_beam_step
   launch (one prompt) and one pkv_cache_reorder launch over the Llama-3-8B geometry (32 layers, 32 heads, D 128, bf16) at
   n generated rows, in its worst case (every slot takes another slot's rows and shares none of them), with the bytes
   that launch moves.
2. Loop: a random-init Llama-3-8B, PyramidKV at each budget, one `prompt`-token prompt. Greedy `greedy_generate` is the
   k = 1 row; `beam_search_generate` for each k (graph replay): end-to-end time, prefill time, ms per step and tokens / s
   (k beams per step). A separate eager run of the same search counts the reorder bytes of every step (the rows each slot
   copies, K and V over every layer). The same request through HF's `generate(num_beams=k)` on the patched model, end to
   end (its k prefills included), unless --skip_hf.
Prints one JSON line with the card's name and power limit, read in the same run; writes nothing else.
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

V = 128256
L8B, H8B, D8B = 32, 32, 128


def _events_us(fn, reps=100):
    fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return 1e3 * a.elapsed_time(b) / reps


def kernel_numbers(dev, beams, n):
    from pyramidkv_b200 import ops
    from pyramidkv_b200.generate import BeamState
    out = []
    for k in beams:
        st = BeamState(1, k, n + 2, [2], 1.0, False, dev)
        logits = (torch.randn(k, V, device=dev) * 2.5).bfloat16()
        row = {"k": k, "K": st.K, "vocab": V}
        row["pkv_beam_candidates_us"] = _events_us(lambda: ops.beam_candidates(logits, st.m, st.log_z, st.cand_lp, st.cand_id))
        step = torch.full((1,), 1, dtype=torch.int32, device=dev)
        snap = [t.clone() for t in st.state()]

        def one_step():
            for t, s in zip(st.state(), snap):
                t.copy_(s)
            ops.beam_step(st, k, step, 0)
        restore_us = _events_us(lambda: [t.copy_(s) for t, s in zip(st.state(), snap)])
        row["pkv_beam_step_us"] = _events_us(one_step) - restore_us
        cap = n + 8                   # prompt rows are never touched: none are allocated
        layers = []
        for _ in range(L8B):
            kb = torch.zeros(k, H8B, cap, D8B, dtype=torch.bfloat16, device=dev)
            base = torch.zeros(k * H8B, dtype=torch.int32, device=dev)
            layers.append((kb, torch.zeros_like(kb), None, None, base, None, None))
        parent = torch.tensor([(a + 1) % k for a in range(k)], dtype=torch.int32, device=dev)   # a cycle
        diverge = torch.zeros(k, dtype=torch.int32, device=dev)
        rstep = torch.full((1,), n - 1, dtype=torch.int32, device=dev)
        row["reorder_rows"] = n
        row["pkv_cache_reorder_worst_us"] = _events_us(lambda: ops.cache_reorder(layers, 1, k, parent, diverge, rstep, 1), 20)
        row["reorder_worst_bytes_each_way"] = k * n * L8B * H8B * D8B * 2 * 2
        row["reorder_worst_gbps"] = 2 * row["reorder_worst_bytes_each_way"] / (row["pkv_cache_reorder_worst_us"] * 1e3)
        del layers
        torch.cuda.empty_cache()
        out.append(row)
    return out


def _knobs(model, budget):
    for layer in model.model.layers:                               # run_longbench.py:253-261
        c = layer.self_attn.config
        c.window_size, c.max_capacity_prompt, c.kernel_size, c.pooling = 8, budget, 7, "maxpool"


def _wall(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    r = fn()
    torch.cuda.synchronize()
    return r, 1e3 * (time.perf_counter() - t0)


@torch.no_grad()
def loop_numbers(model, dev, prompt_len, budgets, beams, new, skip_hf):
    from pyramidkv_b200 import generate as G
    from pyramidkv_b200 import runner
    prompt = runner.synthetic_prompt(model.config.vocab_size, prompt_len, 7, dev)
    rows = []
    for budget in budgets:
        _knobs(model, budget)
        _, prefill_ms = _wall(lambda: G._prefill_logits(model, prompt))
        _, prefill_ms = _wall(lambda: G._prefill_logits(model, prompt))          # warm
        G.greedy_generate(model, prompt, 8)
        _, ms = _wall(lambda: G.greedy_generate(model, prompt, new))
        rows.append({"budget": budget, "k": 1, "loop": "greedy_generate", "end_to_end_ms": ms, "prefill_ms": prefill_ms,
                     "ms_per_step": (ms - prefill_ms) / (new - 1), "tokens_per_s": (new - 1) / ((ms - prefill_ms) / 1e3)})
        for k in beams:
            G.beam_search_generate(model, prompt, 8, k)
            _, ms = _wall(lambda: G.beam_search_generate(model, prompt, new, k))
            row = {"budget": budget, "k": k, "loop": "beam_search_generate", "end_to_end_ms": ms, "prefill_ms": prefill_ms,
                   "ms_per_step": (ms - prefill_ms) / (new - 1),
                   "beam_tokens_per_s": k * (new - 1) / ((ms - prefill_ms) / 1e3)}
            counted = []
            real = G.reorder_caches

            def counting(batch, P, kk, parent, diverge, step, off, backend=None):
                n = int(step) + off
                par, div = parent.tolist(), diverge.tolist()
                rows_moved = sum(n - d for a, (p, d) in enumerate(zip(par, div)) if p != a % kk)
                l0 = batch.layers
                counted.append(sum(rows_moved * l.k_buf.shape[1] * l.k_buf.shape[3] * l.k_buf.element_size() * 2 for l in l0))
                real(batch, P, kk, parent, diverge, step, off, backend)
            G.reorder_caches = counting
            try:
                G.beam_search_generate(model, prompt, new, k, use_graph=False)
            finally:
                G.reorder_caches = real
            row["reorder_bytes_per_step_mean"] = sum(counted) / max(1, len(counted))
            row["reorder_bytes_per_step_max"] = max(counted, default=0)
            if not skip_hf:
                try:
                    _, hf_ms = _wall(lambda: model.generate(prompt, num_beams=k, do_sample=False, max_new_tokens=new,
                                                            pad_token_id=0))
                    row["hf_generate_num_beams_end_to_end_ms"] = hf_ms
                except torch.cuda.OutOfMemoryError as e:
                    row["hf_generate_num_beams_end_to_end_ms"] = f"out of memory: {str(e).splitlines()[0]}"
                torch.cuda.empty_cache()
            rows.append(row)
            torch.cuda.empty_cache()
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--prompt", type=int, default=32768)
    ap.add_argument("--budgets", default="128,2048")
    ap.add_argument("--beams", default="2,4,8")
    ap.add_argument("--new", type=int, default=256)
    ap.add_argument("--kernels_only", action="store_true")
    ap.add_argument("--skip_hf", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("tools/beam_bench.py measures on a CUDA device (H100); there is none here")
    dev = torch.device("cuda", 0)
    beams = [int(x) for x in args.beams.split(",") if x.strip()]
    res = {"gpu": gpu_card(dev), "kernel": kernel_numbers(dev, beams, args.new)}
    if not args.kernels_only:
        from pyramidkv.monkeypatch import replace_llama
        model = build_model("llama3-8b", dev)
        with contextlib.redirect_stdout(io.StringIO()):
            replace_llama("pyramidkv")
        model.config.pkv_fused_rope = True
        res["loop"] = loop_numbers(model, dev, args.prompt, [int(x) for x in args.budgets.split(",")], beams, args.new,
                                   args.skip_hf)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
