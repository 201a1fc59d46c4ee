#!/usr/bin/env python
"""Continuous against lock-step batched decoding on the whole model: python tools/continuous_batch_bench.py

Random-init Llama-3-8B (no checkpoints offline), PyramidKV with the reference runners' knobs, seeded synthetic prompts, no EOS:
random-init weights almost never emit one, so each request's own max_new_tokens stands in for an EOS-driven length. For each
configuration the same request list goes through
  lockstep    consecutive groups of N requests, each prefilled alone and joined, then decoded together for the group's
              largest max_new_tokens (greedy_generate_batch's flow); each request keeps its own first max_new_tokens tokens
  continuous  greedy_generate_continuous with N slots: a finished request's slot takes the next waiting prompt
in one process, one after the other, and their tokens are compared. Request mixes:
  decode_heavy  prompts of 1-2K tokens, max_new_tokens drawn (seeded) from LongBench's caps {32, 64, 128, 512}
  longbench     the tasks of runner.LONGBENCH_SHAPES in seeded order, prompt lengths times --lb_scale, the task's cap
Configurations: budget 128 in bf16 with --slots_128 slots, and budget 2048 with GQA-shared + FP8 caches and N the largest
batch whose caches fit the free memory twice (the prompts' own caches and their join are alive together once; at most
--max_slots). Per configuration and mode: wall time split into prefill and
decode, decode steps, occupancy (live slot-steps / (N * steps)), aggregate generated tok/s (decode-step tokens over decode
time, and every generated token over the wall time), admissions, regrowths, graph captures, whether both modes gave the same
tokens; the cost of one admission through pkv_cache_install against torch slice copies; the card's name and power limit.
The request count is a multiple of N so that every lock-step group runs its GEMMs on N rows like the continuous loop (a
smaller last group may round differently), and every prompt is prefilled once, untimed, before the two timed runs.
Prints one JSON line per configuration and a markdown table; writes nothing else.
"""
import argparse
import contextlib
import io
import json
import os
import random
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from decode_batch_bench import gpu_card  # noqa: E402
from full_model_bench import build_model  # noqa: E402

CAPS = (32, 64, 128, 512)


def requests(mix, n, lb_scale, seed):
    """[(prompt length, max_new_tokens)] of one mix, seeded."""
    rng = random.Random(seed)
    if mix == "decode_heavy":
        return [(rng.randint(1024, 2048), rng.choice(CAPS)) for _ in range(n)]
    from pyramidkv_b200.runner import LONGBENCH_SHAPES
    tasks = sorted(LONGBENCH_SHAPES)
    out = []
    while len(out) < n:
        rng.shuffle(tasks)
        out += [(max(64, int(LONGBENCH_SHAPES[t][0] * lb_scale)), LONGBENCH_SHAPES[t][1]) for t in tasks]
    return out[:n]


def _sync():
    torch.cuda.synchronize()


@torch.no_grad()
def lockstep(model, prompts, caps, N):
    from pyramidkv_b200.cache import join_caches
    from pyramidkv_b200.generate import StaticDecoder, _prefill
    out, pre_s, steps, live = [], 0.0, 0, 0
    t_all = time.perf_counter()
    for g0 in range(0, len(prompts), N):
        group, gcaps = prompts[g0:g0 + N], caps[g0:g0 + N]
        _sync()
        t0 = time.perf_counter()
        firsts, caches = zip(*[_prefill(model, p) for p in group])
        _sync()
        pre_s += time.perf_counter() - t0
        n = max(gcaps) - 1
        cache = join_caches(list(caches), reserve=n)
        del caches
        first = torch.cat(firsts)
        gen = torch.empty(len(group), 0, dtype=torch.long)
        if n > 0:
            dec = StaticDecoder(model, cache, first, n)
            gen = dec.run(n).cpu()
            dec.finish()
            del dec                                # the next group's caches need the memory of this one
        steps += n
        live += sum(c - 1 for c in gcaps)
        out += [[int(first[b])] + gen[b, : c - 1].tolist() for b, c in enumerate(gcaps)]
        del cache
    wall = time.perf_counter() - t_all
    return out, {"prefill_s": pre_s, "decode_s": wall - pre_s, "wall_s": wall, "decode_steps": steps, "live_slot_steps": live,
                 "admissions": 0, "regrowths": 0, "graph_captures": (len(prompts) + N - 1) // N}


@torch.no_grad()
def continuous(model, prompts, caps, N):
    from pyramidkv_b200.generate import greedy_generate_continuous
    _sync()
    t0 = time.perf_counter()
    seqs, st = greedy_generate_continuous(model, prompts, caps, N, return_stats=True)
    _sync()
    wall = time.perf_counter() - t0
    keep = ("prefill_s", "decode_s", "decode_steps", "live_slot_steps", "admissions", "regrowths", "graph_captures")
    return [s[p.shape[1]:].tolist() for s, p in zip(seqs, prompts)], {**{k: st[k] for k in keep}, "wall_s": wall}


def _finish(r, N, generated):
    r["occupancy"] = r["live_slot_steps"] / max(1, N * r["decode_steps"])
    r["decode_tok_per_s"] = r["live_slot_steps"] / max(r["decode_s"], 1e-9)
    r["wall_tok_per_s"] = generated / max(r["wall_s"], 1e-9)
    return r


@torch.no_grad()
def admission_cost(model, N, dev, reps=20):
    """One admission of a 1.5K-token prompt into a batch of N slots: pkv_cache_install (admit_cache: one launch) against the
    same copies as torch slice copies plus the row-count update (a few launches per layer). Device time per admission
    (CUDA events over `reps`), host time per admission (to a synchronise) and launches."""
    from pyramidkv_b200.cache import admit_cache, join_caches
    from pyramidkv_b200.generate import _prefill
    ids = torch.randint(1, model.config.vocab_size, (1, 1536), generator=torch.Generator().manual_seed(5)).to(dev)
    _, c = _prefill(model, ids)
    batch = join_caches([c] * N, reserve=64)
    step = torch.full((1,), 3, dtype=torch.int32, device=dev)
    backend = model.model.layers[0].self_attn.kv_cluster.backend

    def kernel():
        admit_cache(batch, 1, c, step, backend)

    def torch_copies():
        for l, s in zip(batch.layers, c.layers):
            n, H = s.length, l.k_buf.shape[1]
            for name in l._BUFFERS:
                getattr(l, name)[1, :, :n].copy_(getattr(s, name)[0, :, :n])
            l.rows[H:2 * H] = n - step

    out = {}
    for name, fn in (("pkv_cache_install", kernel), ("torch_copies", torch_copies)):
        fn()
        _sync()
        t0 = time.perf_counter()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(reps):
            fn()
        b.record()
        _sync()
        out[name] = {"device_ms": a.elapsed_time(b) / reps, "host_ms": (time.perf_counter() - t0) * 1e3 / reps}
    del batch
    return out


def cache_bytes_per_seq(model, budget, reserve, dev):
    """Bytes one slot's GQA-shared FP8 cache allocates at this budget (from one prefilled prompt longer than the budget)."""
    from pyramidkv_b200.generate import _prefill
    ids = torch.randint(1, model.config.vocab_size, (1, budget + 512), generator=torch.Generator().manual_seed(7)).to(dev)
    _, c = _prefill(model, ids)
    return sum(l.k_buf.shape[1] * (l.length + reserve) * (2 * l.k_buf.shape[3] + 8) for l in c.layers)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--model", default="llama3-8b", choices=["llama3-8b", "tiny"])
    ap.add_argument("--mixes", default="decode_heavy,longbench")
    ap.add_argument("--configs", default="128,2048", help="128: bf16 caches; 2048: GQA-shared + FP8 caches")
    ap.add_argument("--slots_128", type=int, default=32)
    ap.add_argument("--max_slots", type=int, default=256)
    ap.add_argument("--requests_per_slot", type=int, default=2)
    ap.add_argument("--lb_scale", type=float, default=0.125, help="LongBench prompt lengths are scaled by this to fit the run time")
    ap.add_argument("--headroom_gb", type=float, default=10.0)
    ap.add_argument("--seed", type=int, default=1)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("continuous_batch_bench measures on the GPU (H100, sm_90a); no CUDA device found")
    from pyramidkv.monkeypatch import replace_llama
    from pyramidkv_b200 import runner
    dev = torch.device("cuda", torch.cuda.current_device())
    with contextlib.redirect_stdout(io.StringIO()):
        replace_llama("pyramidkv")
    model = build_model(args.model, dev)
    model.config.pkv_fused_rope = True
    from pyramidkv_b200.generate import _prefill
    card = gpu_card(dev)
    rows = []
    for cfg in [int(c) for c in args.configs.split(",")]:
        runner.set_knobs(model, "pyramidkv", cfg)
        model.config.pkv_kv_cache_dtype = "fp8_e4m3" if cfg == 2048 else None
        model.config.pkv_gqa_shared = cfg == 2048
        if cfg == 2048:
            free = torch.cuda.mem_get_info(dev)[0]
            per_seq = cache_bytes_per_seq(model, cfg, max(CAPS), dev)
            # the N single-prompt caches and their join are alive together once: count each slot twice
            N = max(1, min(args.max_slots, int((free - args.headroom_gb * 2 ** 30) // (2 * per_seq))))
        else:
            N = args.slots_128
        for mix in args.mixes.split(","):
            # a multiple of N: every lock-step group then runs its GEMMs on N rows, as the continuous loop always does
            reqs = requests(mix, N * max(1, round(args.requests_per_slot)), args.lb_scale, args.seed)
            prompts = [runner.synthetic_prompt(model.config.vocab_size, n, args.seed * 1000 + i, dev) for i, (n, _) in enumerate(reqs)]
            caps = [c for _, c in reqs]
            generated = sum(caps)
            with torch.no_grad():                  # untimed: first prefills at each prompt length (kernel choices, allocator)
                for p in prompts:
                    _prefill(model, p)
            _sync()
            lock_toks, lock = lockstep(model, prompts, caps, N)
            cont_toks, cont = continuous(model, prompts, caps, N)
            res = {"config": f"budget {cfg}" + (", GQA-shared + FP8" if cfg == 2048 else ", bf16"), "mix": mix, "slots": N,
                   "requests": len(reqs), "generated_tokens": generated, "prompt_tokens": sum(n for n, _ in reqs),
                   "lockstep": _finish(lock, N, generated), "continuous": _finish(cont, N, generated),
                   "tokens_equal": lock_toks == cont_toks,
                   "differing_requests": [i for i, (a, b) in enumerate(zip(lock_toks, cont_toks)) if a != b][:20], "card": card}
            print(json.dumps(res), flush=True)
            rows.append(res)
        adm = admission_cost(model, N, dev)
        print(json.dumps({"config": f"budget {cfg}", "slots": N, "admission": adm, "card": card}), flush=True)
        rows[-1]["admission"] = adm
        torch.cuda.empty_cache()
    print(f"\n{card['name']}, power limit {card.get('power_limit_w')} W\n")
    print("| config | mix | N | requests | mode | wall s | prefill s | decode s | decode steps | occupancy | decode tok/s | "
          "wall tok/s | admissions | regrowths | graph captures |")
    print("|---|---|---|---|---|---|---|---|---|---|---|---|---|---|---|")
    for r in rows:
        for mode in ("lockstep", "continuous"):
            m = r[mode]
            print(f"| {r['config']} | {r['mix']} | {r['slots']} | {r['requests']} | {mode} | {m['wall_s']:.1f} | {m['prefill_s']:.1f} | "
                  f"{m['decode_s']:.1f} | {m['decode_steps']} | {m['occupancy']:.2f} | {m['decode_tok_per_s']:,.0f} | "
                  f"{m['wall_tok_per_s']:,.0f} | {m['admissions']} | {m['regrowths']} | {m['graph_captures']} |")
    print("\n| config | N | admission | device ms | host ms |\n|---|---|---|---|---|")
    for r in rows:
        for k, v in r.get("admission", {}).items():
            print(f"| {r['config']} | {r['slots']} | {k} | {v['device_ms']:.3f} | {v['host_ms']:.3f} |")


if __name__ == "__main__":
    main()
