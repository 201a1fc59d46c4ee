"""Phase timeline of the score and select kernels from in-kernel clock64 stamps (PKV_STAMPS=1, PKV_BUILD_STAMPS=1 build).

    python tools/stamps.py [LAYERS]             per-layer calls of the default workload (layers 0..LAYERS-1, pyramid budgets)
    python tools/stamps.py batch [WORKLOAD]     the layer batch of WORKLOAD (default: the headline), all its layers

Runs a few steps, then prints the stamps the LAST launches left: deltas in microseconds from each kernel's entry stamp. In the
layer batch the select stamps come from the CTA of layer 0 (the largest budget), head 0.
"""
import ctypes as C
import os
import sys

os.environ["PKV_STAMPS"] = "1"
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

import bench  # noqa: E402
from pyramidkv_b200 import _lib  # noqa: E402

SELECT = {0: "entry", 1: "first cluster barrier", 2: "predecessor complete", 3: "keys loaded", 4: "min/max exchanged",
          5: "histogram pass 1", 6: "histogram pass 2", 7: "bases", 8: "winners broadcast", 9: "ranked, idx written", 10: "gather done",
          32: "  (hist 1 built)", 33: "  (hist 1 exchanged)", 34: "  (hist 2 built)", 35: "  (hist 2 exchanged)", 36: "  (winners staged)", 37: "  (flat list built)", 38: "  (ranks counted)", 46: "  (last CTA: hist 2 exchanged)", 47: "  (last CTA: bases)", 44: "  (last CTA: winners staged)", 45: "  (last CTA: broadcast done)"}
# k above the rank limit: the leader sorts; stamps 8-10 then mean something else
SELECT_LEADER = {**{i: n for i, n in SELECT.items() if i < 8 or i in (32, 33, 34, 35, 46, 47)},
                 8: "leader sorted, idx written", 9: "cluster barrier", 10: "gather done"}
SCORE = {0: "entry", 1: "prologue done", 2: "predecessor complete", 3: "first TMA issued", 4: "ring filled", 5: "last TMA issued",
         6: "first tile landed", 7: "second tile landed", 8: "last tile landed", 9: "first accumulator ready",
         10: "last accumulator ready", 11: "last tile stored", 12: "partials flushed", 13: "exit"}


MHZ = float(os.environ.get("PKV_SM_MHZ", "1980"))   # stamps are SM cycles (clock64); cycles / MHz = microseconds


def read_stamps():
    torch.cuda.synchronize()
    buf = (C.c_uint64 * 128)()
    n = _lib.lib().pkv_debug_read_stamps(buf, 128)
    assert n == 128, "stamps disabled?"
    return list(buf)


def print_select(v, names, k):
    print(f"== select kernel (one CTA of head 0), k = {k}")
    t0 = v[0]
    rel = lambda i: (v[i] - (v[43] if "last CTA" in names[i] else t0)) / MHZ   # each CTA's stamps against its own entry
    for i in sorted((i for i in names if v[i]), key=rel):
        print(f"  {names[i]:40s} {rel(i):8.2f} us")
    for r in range(8):
        if v[48 + r]:
            print(f"  rank {r}: keys above thr {v[56 + r] >> 32}, ties {v[56 + r] & 0xffffffff}")


def batch_main(workload):
    dev = torch.device("cuda:0")
    wl = bench.Workload(workload, dev)
    assert wl.batch is not None, "the layer batch does not take this workload"
    for _ in range(5):
        wl.batch.run()
    for _ in range(3):   # the select launch alone: its CTAs start together, as in the batch after the pool launch
        wl.batch.run("select")
    v = read_stamps()
    k = wl.k_l[0]
    leader = k > int(os.environ.get("PKV_RANK_MAX", "512"))
    print(f"layer batch {workload}: {wl.L} layers x {wl.Hq} heads, S = {wl.S}, budgets {wl.k_l[0]}..{wl.k_l[-1]}")
    print_select(v, SELECT_LEADER if leader else SELECT, k)


def main():
    if len(sys.argv) > 1 and sys.argv[1] == "batch":
        return batch_main(sys.argv[2] if len(sys.argv) > 2 else bench.DEFAULT_WORKLOAD)
    dev = torch.device("cuda:0")
    layers = int(sys.argv[1]) if len(sys.argv) > 1 else 4
    wl = bench.Workload("llama3-8b-32k-b128", dev, layers=layers)
    for _ in range(5):
        wl.step()
    v = read_stamps()
    print_select(v, SELECT, wl.k_l[-1])
    for base, tag in ((64, "CTA 0"), (96, "last CTA")):
        print(f"== score kernel ({tag})")
        t0 = v[base]
        for i in sorted(SCORE):
            if v[base + i]:
                print(f"  {SCORE[i]:40s} {(v[base + i] - t0) / MHZ:8.2f} us")


if __name__ == "__main__":
    main()
