#!/usr/bin/env python
"""Batched greedy decode on the whole model: python tools/decode_batch_bench.py [--batch 1,8,32,64] [--ctx 32768] [--budget 128]

Random-init Llama-3-8B (no checkpoints offline), PyramidKV through pyramidkv.monkeypatch.replace_llama with fused RoPE, the
reference runners' knobs (window 8, kernel 7, maxpool). Prints one JSON line with the card's name and power limit and:
  single          the single-sequence static loop (StaticDecoder over one prompt's cache, CUDA graph) for comparison
  decode_batched  generate.greedy_generate_batch's loop (joined caches, one graph replay per step, one pkv_decode_attn_batch
                  launch per layer) per batch size B: aggregate tok/s, ms per step, and the bound
                  (weight bytes + algorithmic KV bytes) / HBM bandwidth
  decode_batched_attn  the attention launches of one step alone, KV bytes read over their time as a fraction of the bandwidth
--kv_cache_dtype bf16,fp8_e4m3 measures both caches, alternating them per batch size in the same process: the FP8 caches are
the bf16 caches of the same prompts converted exactly as the knob pkv_kv_cache_dtype = "fp8_e4m3" converts them after the
prefill; their KV bytes count one byte per element plus the two 4-byte scales of every row and head. --batch max picks, per
dtype, the largest batch whose joined caches fit the free device memory, computed from bytes before allocating.
--gqa_shared off,on measures the per-query-head caches and the GQA-shared ones (knob pkv_gqa_shared: one cache per KV head,
decoded by pkv_decode_attn_batch_gqa(_fp8)) of the same prompts, alternating them per batch size like the dtypes; the KV bytes
of a shared cache count its Hkv heads.
Writes nothing but stdout.
"""
import argparse
import contextlib
import io
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from bench import peaks  # noqa: E402
from full_model_bench import build_model  # noqa: E402


def gpu_card(device):
    """Name and power limit of the card the numbers come from (a power-limited H100 clocks lower under sustained load)."""
    idx = device.index if device.index is not None else torch.cuda.current_device()
    info = {"name": torch.cuda.get_device_name(idx), "power_limit_w": None}
    try:
        r = subprocess.run(["nvidia-smi", f"--id={idx}", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits"],
                           capture_output=True, text=True, timeout=30)
        name, limit = [x.strip() for x in r.stdout.strip().split(",")[:2]]
        info = {"name": name, "power_limit_w": float(limit)}
    except Exception as e:   # noqa: BLE001 - the numbers stand without it; say why it is missing
        info["power_limit_error"] = repr(e)[:120]
    return info


def _kv_row_bytes(D, kv_dtype):
    """Bytes one (sequence, head) reads per cached row for K and V: bf16 elements, or E4M3 bytes plus two fp32 scales."""
    return 2 * D * 2 if kv_dtype == "bf16" else 2 * D + 8


def _cache_bytes_per_seq(model, caches, reserve, kv_dtype):
    """Bytes one sequence's joined cache allocates (the buffers are [H, longest + reserve, D] per layer, H the cache's heads:
    Hq, or Hkv for a GQA-shared cache)."""
    D = model.config.head_dim
    return sum(ls[0].k_buf.shape[1] * (max(l.length for l in ls) + reserve) * _kv_row_bytes(D, kv_dtype)
               for ls in zip(*[c.layers for c in caches]))


def decode_batched_numbers(model, device, ctx, batch_sizes, weight_bytes, new_tokens=32, distinct=2, attn_steps=50,
                           kv_dtypes=("bf16",), headroom_bytes=4 << 30, gqa_modes=(False,)):
    """Batched greedy decode (pyramidkv_b200.generate: joined compacted caches, one CUDA-graph replay per step, one attention
    launch per layer whatever the batch). `distinct` prompts are prefilled and joined repeated up to each batch size B: the
    cost of a decode step does not depend on the cache contents, and this avoids B prefills of the long prompt.
    decode_batched: aggregate tok/s and ms per step next to the bound (weight bytes + KV bytes) / HBM bandwidth.
    decode_batched_attn: the attention launches of one step alone (all layers, CUDA events over attn_steps steps); KV bytes
    read per step over their time as a fraction of the bandwidth. For each B the cache dtypes are measured one after the
    other. batch_sizes may hold "max": the largest B whose joined caches fit the free memory less `headroom_bytes`."""
    from transformers import DynamicCache
    from pyramidkv_b200 import ops
    from pyramidkv_b200.cache import PkvFp8CacheLayer, join_caches, quantize_caches_fp8
    from pyramidkv_b200.generate import StaticDecoder, _prefill
    bw_gbs, bw_src = peaks()
    firsts, caches = [], {}
    for gqa in gqa_modes:
        model.config.pkv_gqa_shared = gqa
        caches[gqa, "bf16"] = []
        for i in range(distinct):
            ids = torch.randint(1, model.config.vocab_size, (1, ctx), generator=torch.Generator().manual_seed(100 + i)).to(device)
            f, c = _prefill(model, ids)
            if gqa == gqa_modes[0]:
                firsts.append(f)
            caches[gqa, "bf16"].append(c)
        if "fp8_e4m3" in kv_dtypes:
            backend = model.model.layers[0].self_attn.kv_cluster.backend
            caches[gqa, "fp8_e4m3"] = []
            for c in caches[gqa, "bf16"]:                # the conversion the knob runs after the prefill, on a copy of the list
                c8 = DynamicCache()
                c8.layers = list(c.layers)
                quantize_caches_fp8(c8, backend)
                caches[gqa, "fp8_e4m3"].append(c8)
    model.config.pkv_gqa_shared = False
    reserve = new_tokens + 3
    points, attn, fits = [], [], {}
    torch.cuda.synchronize()
    for Bspec in batch_sizes:
        for gqa, kv_dtype in [(g, k) for g in gqa_modes for k in kv_dtypes]:
            tag = {"kv_cache_dtype": kv_dtype, **({"gqa_shared": gqa} if len(gqa_modes) > 1 or gqa else {})}
            per_seq = _cache_bytes_per_seq(model, caches[gqa, kv_dtype], reserve, kv_dtype)
            if Bspec == "max":
                free, total = torch.cuda.mem_get_info(device)
                B = max(1, int((free - headroom_bytes) // per_seq))
                fits[kv_dtype + ("+gqa_shared" if gqa else "")] = {"batch": B, "cache_bytes_per_seq": per_seq, "free_bytes": free,
                                                                   "total_bytes": total, "headroom_bytes": headroom_bytes}
            else:
                B = int(Bspec)
            pick = [i % distinct for i in range(B)]
            cache = join_caches([caches[gqa, kv_dtype][i] for i in pick], reserve=reserve)
            first = torch.cat([firsts[i] for i in pick])
            fp8 = isinstance(cache.layers[0], PkvFp8CacheLayer)
            D = cache.layers[0].k_buf.shape[3]
            # algorithmic KV bytes of one step: every (sequence, head) reads its K and V rows (+ the appended one)
            kv_bytes = sum((r + 1) * _kv_row_bytes(D, kv_dtype) for l in cache.layers for row in l.rows_host for r in row)
            # attention alone: the per-layer batched launches of one step at the first step's row counts (fixed step counter)
            Hq, Hkv = model.config.num_attention_heads, model.config.num_key_value_heads
            g = torch.Generator(device=device).manual_seed(B)
            q = torch.randn(B, Hq, D, generator=g, device=device).bfloat16()
            kn = torch.randn(B, Hkv, D, generator=g, device=device).bfloat16()
            step = torch.zeros(1, dtype=torch.int32, device=device)
            ws = torch.empty(ops.decode_workspace_bytes(B * Hq, D), dtype=torch.uint8, device=device)
            out = torch.empty(B, Hq, D, dtype=torch.bfloat16, device=device)

            def attn_step():
                for l in cache.layers:
                    if l.group > 1 and fp8:
                        ops.decode_attn_batch_gqa_fp8(q, l.k_buf, l.v_buf, l.k_scale, l.v_scale, 1, kn, kn, rows=l.rows, step=step,
                                                      max_length=l.capacity, workspace=ws, out=out)
                    elif l.group > 1:
                        ops.decode_attn_batch_gqa(q, l.k_buf, l.v_buf, 1, kn, kn, rows=l.rows, step=step, max_length=l.capacity,
                                                  workspace=ws, out=out)
                    elif fp8:
                        ops.decode_attn_batch_fp8(q, l.k_buf, l.v_buf, l.k_scale, l.v_scale, 1, kn, kn, rows=l.rows, step=step,
                                                  max_length=l.capacity, workspace=ws, out=out)
                    else:
                        ops.decode_attn_batch(q, l.k_buf, l.v_buf, 1, kn, kn, rows=l.rows, step=step, max_length=l.capacity,
                                              workspace=ws, out=out)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            for _ in range(3):
                attn_step()
            graph = torch.cuda.CUDAGraph()                   # replayed: the host-side argument checks are not kernel time
            with torch.cuda.graph(graph):
                attn_step()
            graph.replay()
            torch.cuda.synchronize()
            e0.record()
            for _ in range(attn_steps):
                graph.replay()
            e1.record()
            torch.cuda.synchronize()
            attn_ms = e0.elapsed_time(e1) / attn_steps
            attn.append({"batch": B, **tag, "attn_ms_per_step": attn_ms, "launches_per_step": len(cache.layers),
                         "kv_bytes_per_step": kv_bytes, "kv_gbs": kv_bytes / (attn_ms * 1e-3) / 1e9,
                         "frac_of_hbm": kv_bytes / (attn_ms * 1e-3) / (bw_gbs * 1e9)})
            del graph
            dec = StaticDecoder(model, cache, first, new_tokens + 3, use_graph=True)
            dec.run(3)
            torch.cuda.synchronize()
            e0.record()
            dec.run(new_tokens)
            e1.record()
            torch.cuda.synchronize()
            ms = e0.elapsed_time(e1) / new_tokens
            bound_ms = (weight_bytes + kv_bytes) / (bw_gbs * 1e9) * 1e3
            points.append({"batch": B, **tag, "ms_per_step": ms, "aggregate_tok_s": B * 1e3 / ms,
                           "kv_bytes_per_step": kv_bytes, "weight_bytes": weight_bytes,
                           "weight_floor_ms": weight_bytes / (bw_gbs * 1e9) * 1e3, "bound_ms": bound_ms, "step_over_bound": ms / bound_ms})
            dec.finish()
            del dec, cache, first
            torch.cuda.empty_cache()
    note = f"bandwidth {bw_gbs:.0f} GB/s: {bw_src}"
    return ({"ctx": ctx, "new_tokens": new_tokens, "distinct_prompts": distinct, "bandwidth": note, "points": points, "fits": fits},
            {"steps": attn_steps, "bandwidth": note, "points": attn})


def single_sequence(model, device, ctx, new_tokens=128):
    """The single-sequence static loop over one prompt's cache (what bench.py reports as whole_model.decode_tok_s)."""
    from pyramidkv_b200.generate import StaticDecoder, _prefill
    ids = torch.randint(1, model.config.vocab_size, (1, ctx), generator=torch.Generator().manual_seed(0)).to(device)
    tok, cache = _prefill(model, ids)
    dec = StaticDecoder(model, cache, tok, max_steps=new_tokens + 3, use_graph=True)
    dec.run(3)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    dec.run(new_tokens)
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / new_tokens
    dec.finish()
    return {"new_tokens": new_tokens, "ms_per_tok": ms, "tok_s": 1e3 / ms}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", default="1,8,32,64", help="batch sizes")
    ap.add_argument("--ctx", type=int, default=32768)
    ap.add_argument("--budget", type=int, default=128)
    ap.add_argument("--new", type=int, default=32, help="timed decode steps per batch size")
    ap.add_argument("--kv_cache_dtype", default="bf16", help="comma-separated cache dtypes: bf16, fp8_e4m3")
    ap.add_argument("--gqa_shared", default="off", help="comma-separated: off, on (knob pkv_gqa_shared)")
    ap.add_argument("--no_single", action="store_true", help="skip the single-sequence loop")
    args = ap.parse_args()
    kv_dtypes = [x.strip() for x in args.kv_cache_dtype.split(",") if x.strip()]
    if not kv_dtypes or any(x not in ("bf16", "fp8_e4m3") for x in kv_dtypes):
        raise SystemExit(f"--kv_cache_dtype takes bf16 and / or fp8_e4m3, got {args.kv_cache_dtype!r}")
    gqa_modes = [x.strip() for x in args.gqa_shared.split(",") if x.strip()]
    if not gqa_modes or any(x not in ("off", "on") for x in gqa_modes):
        raise SystemExit(f"--gqa_shared takes off and / or on, got {args.gqa_shared!r}")
    gqa_modes = tuple(x == "on" for x in gqa_modes)
    if not torch.cuda.is_available():
        raise SystemExit("tools/decode_batch_bench.py measures on a CUDA device (H100); there is none here")
    device = torch.device("cuda", 0)
    from pyramidkv.monkeypatch import replace_llama, restore
    model = build_model("llama3-8b", device)
    with contextlib.redirect_stdout(io.StringIO()):
        replace_llama("pyramidkv")
    try:
        for layer in model.model.layers:                         # run_longbench.py:253-261
            c = layer.self_attn.config
            c.window_size, c.max_capacity_prompt, c.kernel_size, c.pooling = 8, args.budget, 7, "maxpool"
        model.config.pkv_fused_rope = True
        weight_bytes = sum(p.numel() * p.element_size() for p in model.parameters())
        with torch.no_grad():
            single = None if args.no_single else single_sequence(model, device, args.ctx)
            torch.cuda.empty_cache()
            batch = [x.strip() if x.strip() == "max" else int(x) for x in args.batch.split(",") if x.strip()]
            batched, attn = decode_batched_numbers(model, device, args.ctx, batch, weight_bytes, new_tokens=args.new,
                                                   kv_dtypes=kv_dtypes, gqa_modes=gqa_modes)
    finally:
        restore()
    print(json.dumps({"model": "llama3-8b (random init)", "method": "pyramidkv", "ctx": args.ctx, "budget": args.budget,
                      "dtype": "bf16", "kv_cache_dtypes": kv_dtypes, "gqa_shared": list(gqa_modes), "fused_rope": True, "gpu": gpu_card(device), "weight_bytes": weight_bytes,
                      "single": single, "decode_batched": batched, "decode_batched_attn": attn}))


if __name__ == "__main__":
    main()
