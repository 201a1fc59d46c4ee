"""Every form of the score and pool stages (stages 1-2) at the prompt lengths it runs at, against an fp64 reference.

Stage 1 writes the masked observation-window logits (or, for H2O, the per-row softmax statistics) and stage 2 turns them
into the pooled scores the select ranks. The library picks the kernels from the shape: the TMA + wgmma window scorer
(`pkv_score_tc5.cu`) with its ring depth and per-CTA tile ranges, or the mma.sync scorer (`pkv_score.cu`); the fused
stages 1-2 kernel (`pkv_evict_fused.cu`) where a CTA's logits fit in shared memory; the layer batch's contiguous or
layer-major walk with the merged or per-CTA partial merge; the pool kernel's instantiations by window and kernel size;
H2O's wgmma or mma.sync passes (`pkv_h2o_tc5.cu`, `pkv_h2o.cu`); the key norms of L2Norm and the window mean of
AdaKV / HeadKV.

The CPU oracle's scalar loops cannot reach the lengths the benchmark runs (32K-token H2O, 131K-token window methods), so
every case here is compared with `gpu_reference`, an fp64 torch restatement of the oracle's rounding chain that runs on the
device. `test_reference_matches_oracle` pins that restatement to the oracle first, on the CPU at small shapes and on the
GPU at shapes the oracle still handles.

The library has no query for most of these choices, so this file restates them (line references below) and labels each
case. `test_case_list_reaches_every_form` (no GPU) checks that the cases reach every form on a 132-SM H100; where the
library does report a form (`pkv_evict_single_launch`, the wgmma scorer refusing a shape) the label is checked against it.
"""
from __future__ import annotations

import math
import os
import subprocess
import sys
import time
from typing import NamedTuple

import pytest
import torch

import gpu_reference as R
from attention_landscapes import assert_stage2, ulp_own
from gpu_util import ulp_diff

H100_SMS = 132
BF, FP = torch.bfloat16, torch.float16
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# ---------------------------------------------------------------------------------------------------------------------------
# Restatement of the stage 1-2 form choice.
# ---------------------------------------------------------------------------------------------------------------------------
TILE = 128                           # pkv_common.cuh:15 kTileTokens
TC5_SMEM_BUDGET = 220 * 1024         # pkv_score_tc5.cu:404 kSmemBudget
SUB_BYTES = 128 * 128                # pkv_score_tc5.cu:30 kSubBytes
FUSED_SMEM_BUDGET = 224 * 1024       # pkv_evict_fused.cu:896
FUSED_FIXED = 24576                  # pkv_internal.h:83 kFusedFixedSmem
FUSED_MAX_PAD, FUSED_MAX_GRID = 32, 160   # pkv_internal.h:81-82
FUSED_EPI_THREADS, FUSED_EPI_WARPS = 512, 16   # pkv_evict_fused.cu:43-44
FUSED_BINS = 256                     # pkv_evict_fused.cu:49
BATCH_STAGES = 4                     # pkv_api.cu:517 (PKV_BATCH_STAGES unset)
MAX_LAYER_BATCH = 32                 # pkv_internal.h:43


def tiles_of(S: int) -> int:
    return (S + TILE - 1) // TILE


def score_tc5_supported(Hq: int, Hkv: int, W: int, S: int, sms: int) -> bool:     # pkv_score_tc5.cu:513-521
    G = Hq // Hkv
    return G * W in (32, 64) and G <= 256 and W <= 256 and Hkv <= sms and S < 2 ** 31   # (torch allocations are 16-byte aligned)


def tc5_grid(Hkv: int, S: int, sms: int) -> int:                                   # pkv_score_tc5.cu:508-511
    return min(tiles_of(S) * Hkv, sms)


def tc5_ring_depth(D: int, NW: int, q_bufs: int = 2, max_stages: int = 0) -> int:  # pkv_score_tc5.cu:406, :445-449
    fixed = 1024 + q_bufs * (D // 64) * NW * 128 + 8 * NW * 8 + 256
    ns = min(6, (TC5_SMEM_BUDGET - fixed) // ((D // 64) * SUB_BYTES))
    return min(ns, max_stages) if 2 <= max_stages < ns else ns


def tc5_ranges(Hkv: int, S: int, grid: int):
    """Per CTA its contiguous [begin, end) of the (kv head, tile) list (pkv_score_tc5.cu:150-151)."""
    T = tiles_of(S) * Hkv
    return [((c * T) // grid, ((c + 1) * T) // grid) for c in range(grid)]


def tc5_walk(Hkv: int, S: int, sms: int):
    """(longest per-CTA range in tiles, whether some CTA's range spans two kv heads) of the per-layer launch."""
    tpg = tiles_of(S)
    rs = tc5_ranges(Hkv, S, tc5_grid(Hkv, S, sms))
    return max(e - b for b, e in rs), any(b // tpg != (e - 1) // tpg for b, e in rs if e > b)


def tc5_first_cta(g: int, tpg: int, total: int, grid: int) -> int:               # pkv_common.cuh:207-209
    return (g * tpg * grid + grid + total - 1) // total - 1


def fused_plan(Hq: int, Hkv: int, S: int, D: int, W: int, k: int, kernel: int, sms: int):
    """make_plan (pkv_evict_fused.cu:915-970), flag form: tiles per CTA (tmax), or None where the fused kernel refuses."""
    G, n = Hq // Hkv, S - W
    nw = G * W
    if nw not in (32, 64) or W not in (8, 16) or (nw // 4) % W:
        return None
    if G > 8 or FUSED_EPI_THREADS % G or FUSED_EPI_WARPS % G or D not in (64, 128):
        return None
    if k < 1 or n < 1 or S >= 2 ** 30 or kernel // 2 > FUSED_MAX_PAD:
        return None
    sm = min(sms, FUSED_MAX_GRID)
    if Hkv > sm:
        return None
    tpg = tiles_of(S)
    cpg = min(sm // Hkv, tpg)
    tmax = (tpg + cpg - 1) // cpg
    store = tmax * TILE * nw * 2
    stage = (D // 64) * SUB_BYTES
    if store + FUSED_FIXED + 1024 + stage > FUSED_SMEM_BUDGET:
        return None
    kcap, mine_cap = (k + 1) & ~1, k // cpg + 2
    post_a = G * (tmax * TILE + 2 * FUSED_MAX_PAD) * 4 + G * tmax * TILE * 2 + G * FUSED_BINS * 4 + cpg * nw * 8
    avail = FUSED_SMEM_BUDGET - FUSED_FIXED - 1024 - store
    if kcap * 8 + mine_cap * 8 > avail or post_a > avail:
        return None
    if min(6, avail // stage, tmax) < 1:
        return None
    return tmax


def h2o_tc5_supported(S: int) -> bool:                                             # pkv_h2o_tc5.cu:403-408
    return tiles_of(S) >= 4 and S < 2 ** 31


def layer_major_ok(Hkv: int, S: int, sms: int) -> bool:                            # pkv_score_tc5.cu:535-538
    return (tiles_of(S) * Hkv) // tc5_grid(Hkv, S, sms) >= 8


def pool_inst(W: int, kernel: int, mean: bool = False) -> str:                     # pkv_score.cu:439, :478-488
    if mean:
        return "pool:mean"
    if W != 8:
        return "pool:generic"
    return f"pool:w8k{kernel}" if kernel in (5, 7) else "pool:w8k0"


class Case(NamedTuple):
    name: str
    kind: str        # "window" (per-layer staged), "fused", "batch", "h2o", "l2norm", "mean"
    Hq: int
    Hkv: int
    S: int
    D: int
    W: int
    dtype: torch.dtype
    kernel: int = 7
    pooling: str = "maxpool"
    scorer: str = "tcgen05"      # window: tcgen05 / mma; h2o: tc5 / mma
    inputs: str = "gauss"        # gauss, or a landscape built on the device: heavy (exact-dot), sink
    layers: int = 1
    merge: bool = True           # layer batch: merged partials (default) or PKV_BATCH_MERGE=0


def forms(c: Case, sms: int = H100_SMS) -> set:
    """The forms a case reaches at `sms` SMs."""
    out = set()
    if c.kind == "h2o":
        out.add(f"h2o:{c.scorer}" if c.scorer == "mma" or h2o_tc5_supported(c.S) else "h2o:mma")
        return out
    if c.kind == "l2norm":
        return {"l2norm"}
    G = c.Hq // c.Hkv
    tc5 = c.scorer == "tcgen05" and score_tc5_supported(c.Hq, c.Hkv, c.W, c.S, sms)
    if c.kind == "batch":
        out.add("batch:layer-major" if layer_major_ok(c.Hkv, c.S, sms) else "batch:contiguous")
        out.add("batch:merged" if c.merge else "batch:self-merge")
        if c.layers > MAX_LAYER_BATCH:
            out.add("batch:two-launches")
        out.add(pool_inst(c.W, c.kernel))
        return out
    if c.kind == "fused":
        tm = fused_plan(c.Hq, c.Hkv, c.S, c.D, c.W, 120, c.kernel, sms)
        out.add("fused:takes" if tm else "fused:refuses")
        if tm:
            return out
    if tc5:
        out.add(f"tc5:ns{tc5_ring_depth(c.D, G * c.W)}")
        if tc5_walk(c.Hkv, c.S, sms)[1]:
            out.add("tc5:span2")
    else:
        out.add("mma")
    out.add(pool_inst(c.W, c.kernel, c.kind == "mean"))
    return out


def reachable_forms(sms: int = H100_SMS) -> set:
    out = {"h2o:tc5", "h2o:mma", "l2norm", "pool:mean", "batch:layer-major", "batch:contiguous", "batch:merged",
           "batch:self-merge", "batch:two-launches", "fused:takes", "fused:refuses", "mma", "tc5:span2"}
    for D in (64, 128):
        for NW in (32, 64):
            out.add(f"tc5:ns{tc5_ring_depth(D, NW)}")
    for W in (8, 16, 32, 64):
        for kernel in (1, 3, 5, 7, 9):
            out.add(pool_inst(W, kernel))
    return out


# ---------------------------------------------------------------------------------------------------------------------------
# The cases.
# ---------------------------------------------------------------------------------------------------------------------------
def _fused_edge(Hq, Hkv, D, W, sms=H100_SMS):
    """(last length the fused kernel takes, first it refuses), scanning up in whole tiles then tokens."""
    S = 1024
    while fused_plan(Hq, Hkv, S + TILE, D, W, 120, 7, sms):
        S += TILE
    while fused_plan(Hq, Hkv, S + 1, D, W, 120, 7, sms):
        S += 1
    return S, S + 1


FUSED_LAST, FUSED_FIRST_REFUSED = _fused_edge(32, 8, 128, 8)

H2O_CASES = [
    Case("h2o_8b_32k", "h2o", 32, 8, 32768, 128, 8, BF, scorer="tc5"),
    Case("h2o_8b_32k_mma", "h2o", 32, 8, 32768, 128, 8, BF, scorer="mma"),
    Case("h2o_20000_heavy", "h2o", 8, 2, 20000, 128, 32, BF, scorer="tc5", inputs="heavy"),
    Case("h2o_20000_heavy_mma", "h2o", 8, 2, 20000, 128, 32, BF, scorer="mma", inputs="heavy"),
    Case("h2o_16k_fp16_d64", "h2o", 8, 2, 16384, 64, 8, FP, scorer="tc5"),
    Case("h2o_16k_fp16_d64_mma", "h2o", 8, 2, 16384, 64, 8, FP, scorer="mma"),
    Case("h2o_8k_sink_w32", "h2o", 8, 2, 8192, 128, 32, BF, scorer="tc5", inputs="sink"),
    Case("h2o_8k_sink_w32_mma", "h2o", 8, 2, 8192, 128, 32, BF, scorer="mma", inputs="sink"),
]

WINDOW_CASES = [
    Case("tc5_8b_40960", "window", 32, 8, 40960, 128, 8, BF),
    Case("tc5_8b_65536_fp16_avg5", "window", 32, 8, 65536, 128, 8, FP, kernel=5, pooling="avgpool"),
    Case("tc5_8b_131072", "window", 32, 8, 131072, 128, 8, BF),
    Case("tc5_8b_131072_heavy", "window", 32, 8, 131072, 128, 8, BF, inputs="heavy"),
    Case("tc5_70b_g8_262144", "window", 64, 8, 262144, 128, 8, BF, kernel=3),
    Case("tc5_8b_fused_edge_fp16", "window", 32, 8, FUSED_FIRST_REFUSED, 128, 8, FP),
    Case("tc5_d64_w16_131072", "window", 8, 2, 131072, 64, 16, BF, kernel=9, pooling="avgpool"),
    Case("mma_mha_w8_65536", "window", 8, 8, 65536, 128, 8, BF, scorer="mma"),
    Case("mma_g4_w64_65536_fp16", "window", 16, 4, 65536, 128, 64, FP, kernel=5, pooling="avgpool", scorer="mma"),
    Case("mma_mha_d64_65536", "window", 8, 8, 65536, 64, 8, BF, kernel=5, scorer="mma"),
]

FUSED_CASES = [
    Case("fused_last_taken", "fused", 32, 8, FUSED_LAST, 128, 8, BF),
    Case("fused_first_refused", "fused", 32, 8, FUSED_FIRST_REFUSED, 128, 8, BF),
]

BATCH_CASES = [
    Case("batch_8b_131072_x8", "batch", 32, 8, 131072, 128, 8, BF, layers=8),
    Case("batch_8b_131072_x8_self_merge", "batch", 32, 8, 131072, 128, 8, BF, layers=8, merge=False),
    Case("batch_short_contiguous", "batch", 32, 8, 4096, 128, 8, BF, kernel=5, pooling="avgpool", layers=4),
    Case("batch_33_layers", "batch", 4, 1, 16384, 64, 8, BF, layers=33),
]

OTHER_CASES = [
    Case("l2norm_8b_131072", "l2norm", 32, 8, 131072, 128, 0, BF),
    Case("mean_8b_131072", "mean", 32, 8, 131072, 128, 8, BF),
]

ALL_CASES = H2O_CASES + WINDOW_CASES + FUSED_CASES + BATCH_CASES + OTHER_CASES


def test_case_list_reaches_every_form():
    """No GPU: the cases reach every stage 1-2 form on a 132-SM H100, the window cases the longest per-CTA tile ranges
    of the benchmark's lengths, and the fused edge is where the restatement puts it."""
    reached = set().union(*(forms(c) for c in ALL_CASES))
    missing = reachable_forms() - reached
    assert not missing, f"forms no case reaches: {sorted(missing)}"
    longest = max(tc5_walk(c.Hkv, c.S, H100_SMS)[0] for c in WINDOW_CASES if "mma" not in forms(c))
    assert longest >= tc5_walk(8, 262144, H100_SMS)[0]
    assert fused_plan(32, 8, FUSED_LAST, 128, 8, 120, 7, H100_SMS) and not fused_plan(32, 8, FUSED_FIRST_REFUSED, 128, 8, 120, 7, H100_SMS)
    assert FUSED_LAST < 40960 < 131072, "the fused kernel's tile limit moved: revisit the window cases' lengths"
    for c in ALL_CASES:
        if c.kind in ("window", "batch") and c.scorer == "tcgen05":
            assert score_tc5_supported(c.Hq, c.Hkv, c.W, c.S, H100_SMS), c.name


# ---------------------------------------------------------------------------------------------------------------------------
# The reference against the oracle.
# ---------------------------------------------------------------------------------------------------------------------------
def _mant(dt):
    return 8 if dt == BF else 11


def _exact_x(Hkv, S, seed, gap=60.0, device="cpu"):
    """Exact-dot key values: integers in [-8, 8], one token per kv head `gap` above them in the last third (past tile 0)."""
    g = torch.Generator(device=device).manual_seed(seed)
    x = torch.randint(-8, 9, (Hkv, S), generator=g, device=device).float()
    n = S - 64
    pos = torch.randint(max(2 * n // 3, 129), n, (Hkv,), generator=g, device=device)
    x[torch.arange(Hkv, device=device), pos] = 8 + gap
    return x


def make(c: Case, seed: int, device, q_rows=None):
    """Inputs of a case on `device`: q [Hq, q_rows or S, D], k and v [Hkv, S, D]. `heavy`: exact-dot (q = c in dim 0, k = x
    in dim 0; every logit is exact in every path), with one key > kRefSlack = 40 above every earlier one. `sink`: Gaussian
    with tokens 0-3 about 30 above the background."""
    rows = q_rows or c.S
    g = torch.Generator(device=device).manual_seed(seed)
    if c.inputs == "heavy":
        cq = float(torch.tensor(math.sqrt(c.D)).to(c.dtype).float())
        q = torch.zeros(c.Hq, rows, c.D, device=device)
        q[:, :, 0] = cq
        k = torch.zeros(c.Hkv, c.S, c.D, device=device)
        k[:, :, 0] = _exact_x(c.Hkv, c.S, seed, device=device)
    else:
        q = torch.randn(c.Hq, rows, c.D, generator=g, device=device)
        k = torch.randn(c.Hkv, c.S, c.D, generator=g, device=device)
        if c.inputs == "sink":
            q[:, :, -1] = 4.0
            k[:, :, -1] = 0.0
            k[:, :4, -1] = 30.0 * math.sqrt(c.D) / 4.0
    v = torch.randn(c.Hkv, c.S, c.D, generator=g, device=device)
    return q.to(c.dtype), k.to(c.dtype), v.to(c.dtype)


def _check_ref_vs_oracle(oracle, c: Case, device):
    q, k, v = make(c, 11, "cpu")
    n = c.S - c.W
    nb = lambda t: max(4, t.numel() >> 8)                                   # noqa: E731
    if c.kind == "h2o":
        ref, M, L, _ = R.h2o_scores(q.to(device), k.to(device), c.W)
        ref = ref.cpu()
        o = oracle.h2o_scores(q, k, c.W)
        # oracle: fp32 running sum in row order, |sum - exact| <= (S - 1) 2^-24 * sum; + the two roundings to the dtype
        bound = ref.double().abs() * (c.S - 1) * 2.0 ** -24 + 2.0 ** -(_mant(c.dtype) - 1) * ref.double().abs().clamp(min=2.0 ** -133)
        over = (o.double() - ref.double()).abs() > bound
        bad = int(over.sum())
        print(f"PKV_MEASURED ref_vs_oracle {c.name} h2o colsum: {mismatch_count(o, ref)}/{ref.numel()} differ, {bad} beyond the summation bound")
        assert bad <= nb(ref), f"{bad} column sums beyond the oracle's fp32 summation error"
        assert float(ulp_own(o, ref, c.dtype).max()) <= 2
        return
    lg = R.window_logits(q.to(device), k.to(device), c.W).cpu()
    olg = oracle.window_logits(q, k, c.W)
    bad_l = mismatch_count(lg, olg)
    probs, oprobs = R.softmax_rows(lg.to(device)).cpu(), oracle.softmax_rows(olg)
    ws, ows = R.window_sum(probs.to(device)).cpu(), oracle.window_sum(oprobs)
    pooled, opooled = R.pool(ws.to(device), c.kernel, c.pooling).cpu(), oracle.pool(ows, c.kernel, c.pooling)
    # the window sum and pool are restated exactly: on the ORACLE's probabilities they must be bit-identical
    assert torch.equal(R.window_sum(oprobs.to(device)).cpu().view(torch.int16), ows.view(torch.int16))
    assert torch.equal(R.pool(ows.to(device), c.kernel, c.pooling).cpu().view(torch.int16), opooled.view(torch.int16))
    bad_p, bad_w, bad_o = mismatch_count(probs, oprobs), mismatch_count(ws, ows), mismatch_count(pooled, opooled)
    print(f"PKV_MEASURED ref_vs_oracle {c.name} logits {bad_l}/{lg.numel()} probs {bad_p}/{probs.numel()} "
          f"wsum {bad_w}/{ws.numel()} pooled {bad_o}/{pooled.numel()} differ")
    assert bad_l <= max(2, lg.numel() >> 18), "logits: the rounding chain is not the oracle's"
    for a, b, what in ((probs, oprobs, "probabilities"), (ws, ows, "window sums"), (pooled, opooled, "pooled")):
        d = mismatch_count(a, b)
        assert d <= nb(a), f"{what}: {d} differ (expf / fp64 exp rounding differences are rare)"
        if d:
            assert float(ulp_own(a, b, c.dtype).max()) <= 1, what
    if c.inputs == "heavy":
        assert bad_l == 0, "exact-dot logits must be bit-identical"


def mismatch_count(a, b) -> int:
    return int((a.contiguous().view(torch.int16) != b.contiguous().view(torch.int16)).sum())


REF_CPU = [Case("cpu_h2o", "h2o", 4, 2, 700, 64, 8, BF), Case("cpu_h2o_fp16_heavy", "h2o", 2, 1, 900, 64, 16, FP, inputs="heavy"),
           Case("cpu_snap", "window", 8, 2, 1500, 64, 8, BF, kernel=7), Case("cpu_snap_fp16_avg", "window", 4, 4, 999, 128, 16, FP, kernel=5, pooling="avgpool"),
           Case("cpu_heavy", "window", 8, 2, 2000, 64, 8, BF, inputs="heavy"), Case("cpu_sink", "window", 4, 1, 1300, 64, 32, BF, inputs="sink", kernel=3, pooling="avgpool")]
REF_GPU = [Case("gpu_h2o_4096", "h2o", 8, 2, 4096, 128, 8, BF), Case("gpu_h2o_8192_fp16", "h2o", 2, 1, 8192, 64, 32, FP),
           Case("gpu_h2o_3000_heavy", "h2o", 4, 1, 3000, 128, 8, BF, inputs="heavy"),
           Case("gpu_snap_32768", "window", 32, 8, 32768, 128, 8, BF), Case("gpu_snap_20000_fp16", "window", 16, 2, 20000, 64, 8, FP, kernel=5, pooling="avgpool"),
           Case("gpu_snap_32768_heavy", "window", 8, 2, 32768, 128, 8, BF, inputs="heavy")]


@pytest.mark.parametrize("c", REF_CPU, ids=lambda c: c.name)
def test_reference_matches_oracle(oracle, c):
    """The fp64 reference reproduces the oracle's rounding chain: logits bit-identical, probabilities / window sums / pooled
    scores identical up to rare 1-ulp fp32-exp differences, H2O column sums within the oracle's own fp32 summation error."""
    _check_ref_vs_oracle(oracle, c, "cpu")


@pytest.mark.gpu
@pytest.mark.parametrize("c", REF_GPU, ids=lambda c: c.name)
def test_reference_matches_oracle_on_gpu(oracle, c):
    _check_ref_vs_oracle(oracle, c, torch.device("cuda", 0))


# ---------------------------------------------------------------------------------------------------------------------------
# GPU cases.
# ---------------------------------------------------------------------------------------------------------------------------
def _dev():
    return torch.device("cuda", 0)


def _sms() -> int:
    return torch.cuda.get_device_properties(0).multi_processor_count


def _plan(c: Case, q, k, v, top_k, score_kernel=None, **kw):
    from pyramidkv_b200 import ops
    kc = torch.empty(c.Hq, top_k + max(c.W, 1), c.D, dtype=c.dtype, device=_dev())
    idx = torch.empty(c.Hq, top_k, dtype=torch.int64, device=_dev())
    method = {"h2o": "h2o", "l2norm": "l2norm"}.get(c.kind, "snapkv")
    return ops.plan_evict(method, q, k, v, c.W, top_k, kc, torch.empty_like(kc), c.kernel, c.pooling, idx_out=idx,
                          score_kernel=score_kernel or ("mma" if c.scorer == "mma" else "tcgen05" if c.kind != "h2o" else "auto"), **kw), idx


def _h2o_stats(plan) -> torch.Tensor:
    d, L = plan.desc, plan.layout
    n = d.num_q_heads * L.s_pad * 2
    return plan.workspace[L.h2o_stats_off:L.h2o_stats_off + 4 * n].view(torch.float32).view(d.num_q_heads, L.s_pad, 2)[:, :d.seq_len]


def _h2o_run(c: Case):
    q, k, v = make(c, c.S, _dev())
    plan, idx = _plan(c, q, k, v, 64)
    from pyramidkv_b200 import ops
    for st in ("scores", "pool", "topk"):
        ops.run_stage(plan, st)
    torch.cuda.synchronize()
    return q, k, ops.ws_pooled(plan).clone(), _h2o_stats(plan).clone(), idx


def _h2o_check(oracle, c: Case, pooled, stats, idx, q, k):
    """Bars (per element, derived, not fitted):
      - column sums: each kernel probability is the reference's rounded probability or a neighbour (one dtype ulp, from the
        fp32 exp / 1/L error, <= 2^-(mant-1) relative), so the sum moves by <= 2 ulp. The kernel's own fp32 summation
        error is gamma_n relative for a chain of n sequential adds: tc5 pass 1 adds 8 terms per tile into each of two
        accumulators, then those two and 8 slices (n = S/16 + 9: 2^-14 at 16K, 2^-13 at 32K); mma pass 1 adds 2 terms per
        8 query rows per thread, then a 2-level shuffle tree (n = S/4 + 2: 2^-12 at 16K, 2^-11 at 32K). That is <= 0.5
        fp16 ulp (ulp >= 2^-11 relative) and <= 0.125 bf16 ulp. Both results are rounded once more (1 ulp): <= 3.5, bar 4
        ulp (assert_stage2);
      - row statistics: on exact-dot inputs every logit is exact, so M equals the fp64 row max and L is within the fp32
        summation error of pass 0, rel = (8 tiles + 16) 2^-24 (8 adds per tile into each of two running sums, 8 slices)
        + 2^-16 (exp2 approximation, fma rounding of x log2 e, one rescale per kRefSlack move). Elsewhere a logit the kernel
        rounds differently moves by <= 2 dtype ulps (a 1-ulp change of round(q.k) moves the quotient by <= 1 ulp before its
        own rounding), so M is within 2 ulp and L within rel + the row's flip share (gpu_reference.h2o_scores); and since
        flips are rare (<= 2e-3 of logits) and move L beyond rel only when the flipped logit carries >= 1% of the row's
        mass, at most 1e-3 of the rows may exceed rel;
      - the selection is exact on the kernel's own scores."""
    ref, M, L, Fs = R.h2o_scores(q, k, c.W)
    assert_stage2(pooled.cpu(), ref.cpu(), f"{c.name}: column sums vs the fp64 reference", max_ulp=4)
    bad = mismatch_count(pooled, ref)
    tol = 2e-2 if c.inputs == "gauss" else 2e-3
    assert bad <= max(4, int(tol * ref.numel())), f"{c.name}: {bad}/{ref.numel()} column sums differ"
    m, l = stats[..., 0].double(), stats[..., 1].double()
    mulp = torch.exp2(torch.floor(torch.log2(M.abs().clamp(min=2.0 ** -100))) - (_mant(c.dtype) - 1))
    dm = (m - M).abs() / mulp
    exact = c.inputs == "heavy"
    assert bool((dm <= (0 if exact else 2)).all()), f"{c.name}: row max off by {float(dm.max())} ulp at {int((dm > 0).sum())} rows"
    rel = (8 * tiles_of(c.S) + 16) * 2.0 ** -24 + 2.0 ** -16
    err = (l * torch.exp(m - M) - L).abs() / L
    lim = rel if exact else rel + Fs
    assert bool((err <= lim).all()), f"{c.name}: row sum-exp off by {float(err.max()):.3g} (bar {float(torch.as_tensor(lim).max()):.3g})"
    beyond = int((err > rel).sum())
    assert beyond <= max(4, err.numel() // 1000), f"{c.name}: {beyond} rows beyond the fp32 summation bound {rel:.3g}"
    assert torch.equal(oracle.topk(pooled.cpu().contiguous(), idx.shape[1], oracle.TIE_LOWEST_INDEX), idx.cpu())
    print(f"PKV_MEASURED {c.name}: colsum {bad}/{ref.numel()} differ from fp64 (max {float(ulp_own(pooled, ref, c.dtype).max()):.2f} ulp), "
          f"row-sum rel err {float(err.max()):.2e}, {beyond}/{err.numel()} rows beyond {rel:.2e}")
    return ref


_H2O_CHILD = r"""
import sys, torch
sys.path.insert(0, "tests")
import test_gpu_score_forms as T
from oracle import pkv_oracle as O
O.build()
out = {}
for c in T.H2O_CASES:
    if c.scorer == "mma":
        q, k, pooled, stats, idx = T._h2o_run(c)
        T._h2o_check(O, c, pooled, stats, idx, q, k)
        out[c.name.replace("_mma", "")] = pooled.cpu()
        del q, k
        torch.cuda.empty_cache()
torch.save(out, sys.argv[1])
print(f"PKV_MEASURED h2o mma child peak {torch.cuda.max_memory_allocated() / 2**30:.2f} GiB")
"""


@pytest.mark.gpu
def test_h2o_both_kernels_at_length(oracle, libpkv, tmp_path):
    """H2O at 8K-32K tokens: the wgmma kernel here, the mma.sync kernel in a child with PKV_H2O=mma (the knob is read once
    per process), both against the fp64 reference; then each other at the H2O class bar."""
    t0 = time.time()
    mine = {}
    for c in H2O_CASES:
        if c.scorer != "tc5":
            continue
        assert forms(c) == {"h2o:tc5"}
        q, k, pooled, stats, idx = _h2o_run(c)
        _h2o_check(oracle, c, pooled, stats, idx, q, k)
        mine[c.name] = pooled.cpu()
        del q, k
        torch.cuda.empty_cache()
    path = tmp_path / "mma.pt"
    r = subprocess.run([sys.executable, "-c", _H2O_CHILD, str(path)], timeout=400, env={**os.environ, "PKV_H2O": "mma"}, cwd=ROOT,
                       capture_output=True, text=True)
    print(r.stdout[-4000:])
    assert r.returncode == 0, r.stderr[-4000:]
    mma = torch.load(path)
    for name, pooled in mine.items():
        other = mma[name]
        bad = mismatch_count(pooled, other)
        assert bad <= max(4, int(2e-2 * pooled.numel())), f"{name}: {bad} scores differ between the kernels"
        assert ulp_diff(pooled, other) <= 4
    print(f"PKV_MEASURED h2o both kernels: {time.time() - t0:.1f} s")


def _partials_check(c: Case, plan, logits):
    """Each CTA's softmax partial (m, l) of a logit column against the fp64 (max, sum exp) of the tiles the CTA covered:
    m is a logit of the range within kRefSlack = 40 below its maximum; l * e^(m - max) is within (2 t + 16) 2^-24 (t tiles of
    two rows per thread in fp32 running sums, 8-lane and 8-group merges) + 2^-16 (fast exp, reference moves) of the fp64 sum,
    relative."""
    from pyramidkv_b200 import ops
    G = c.Hq // c.Hkv
    pm, pl = R.tile_partials(logits, G)                                     # [Hkv, tiles, NW]
    part = ops.ws_partials(plan).double()
    tpg = tiles_of(c.S)
    worst = 0.0
    if c.scorer == "mma":
        slots = [(g, t, t, t + 1) for g in range(c.Hkv) for t in range(tpg)]
    else:
        grid = tc5_grid(c.Hkv, c.S, torch.cuda.get_device_properties(0).multi_processor_count)
        T = tpg * c.Hkv
        slots = []
        for g in range(c.Hkv):
            first = tc5_first_cta(g, tpg, T, grid)
            for cta, (b, e) in enumerate(tc5_ranges(c.Hkv, c.S, grid)):
                lo, hi = max(b, g * tpg), min(e, (g + 1) * tpg)
                if lo < hi:
                    slots.append((g, cta - first, lo - g * tpg, hi - g * tpg))
    for g, slot, t0, t1 in slots:
        M = pm[g, t0:t1].max(dim=0).values
        Ls = (pl[g, t0:t1] * torch.exp(pm[g, t0:t1] - M)).nan_to_num(0.0).sum(dim=0)
        m, l = part[g, slot, :, 0], part[g, slot, :, 1]
        assert bool(((m <= M) & (m >= M - 40)).all()), f"{c.name}: partial reference outside [max - 40, max] (kv head {g}, slot {slot})"
        err = float(((l * torch.exp(m - M) - Ls).abs() / Ls).max())
        worst = max(worst, err)
        assert err <= (2 * (t1 - t0) + 16) * 2.0 ** -24 + 2.0 ** -16, f"{c.name}: partial sum-exp rel err {err:.3g} (kv head {g}, slot {slot})"
    return worst


def flip_ulps(ref_logits: torch.Tensor) -> float:
    """Per-element bar (ulps of each element's own magnitude) of stage 2 against the reference run on the INPUTS. A logit the
    kernel rounds to the neighbouring dtype value (fp32 accumulation order; <= 2e-3 of them) scales its probability by
    e^(+-ulp(x)), so a window sum or pooled score moves by at most e^ulp(max |x|) - 1 relative, i.e.
    (e^ulp(max |x|) - 1) * 2^mant ulps of the dtype; plus the 2 ulp of the comparison on the kernel's own logits. The
    maximum is over the logits the mask leaves alone (taken from the geometry: fp16's masked value -65504 is finite).
    (The older 4-ulp class bar holds for logits below 2 in magnitude; at 131K tokens the largest Gaussian logits exceed 4.)"""
    dt = ref_logits.dtype
    live = ~R.window_masked(ref_logits.shape[1], ref_logits.shape[2], ref_logits.device)
    xm = float(ref_logits.float().masked_fill(~live, 0.0).abs().max())
    u = 2.0 ** (math.floor(math.log2(max(xm, 2.0 ** -14))) - (_mant(dt) - 1))
    return 2 + math.ceil(math.expm1(u) * 2 ** _mant(dt))


def _live_logit_ulps(a: torch.Tensor, b: torch.Tensor, live: torch.Tensor) -> float:
    """gpu_util.ulp_diff over the live (unmasked) logits, one head at a time (fp64 temporaries of [W, S] only): |a - b| in
    ulps of the larger operand, magnitudes floored at 2^-6 of the largest live logit."""
    mant = _mant(b.dtype)
    floor = max(float(b.float().masked_fill(~live, 0.0).abs().max()) * 2.0 ** -6, 1e-30)
    worst = 0.0
    for h in range(b.shape[0]):
        fa, fb = a[h].double(), b[h].double()
        mag = torch.clamp(torch.maximum(fa.abs(), fb.abs()), min=floor)
        u = ((fa - fb).abs() / torch.exp2(torch.floor(torch.log2(mag)) - (mant - 1)))[live[h]]
        worst = max(worst, float(u.max()))
    return worst


def _check_vs_inputs(c: Case, pooled, ref, ref_lg):
    """Stage 2 against the reference on the inputs: <= 2e-3 of the elements (fp16: x3) differ, each by <= flip_ulps of its
    own magnitude; on exact-dot inputs every logit is exact and the bar is assert_stage2's 2 ulp."""
    bad = mismatch_count(pooled, ref)
    if c.inputs == "heavy":
        assert_stage2(pooled.cpu(), ref.cpu(), f"{c.name}: pooled vs the reference (exact-dot)")
        return bad, 2
    tol = 2e-3 * (3 if c.dtype == FP else 1)
    assert bad <= max(4, int(tol * ref.numel())), f"{c.name}: {bad}/{ref.numel()} pooled scores differ from the reference"
    fu, u = flip_ulps(ref_lg), float(ulp_own(pooled, ref, c.dtype).max())
    assert u <= fu, f"{c.name}: pooled {u} ulp from the reference (bar {fu})"
    return bad, fu


def _window_check(oracle, c: Case, logits, pooled, idx, q, k, mean=False):
    """Stage 1: logits vs the reference on the inputs: masked exactly where the geometry says (finfo.min or -inf there,
    above finfo.min / 2 everywhere else); <= 2e-3 of them differ, the live ones by <= 2 ulp with magnitudes floored at
    2^-6 of the largest live logit (q.k cancels: fp32 accumulation order vs fp64); exact on exact-dot inputs. Stage 2:
    against the reference on the kernel's OWN logits, every element within 2 ulp (assert_stage2); against the reference on
    the inputs, _check_vs_inputs. Stage 3: the selection is exact on the kernel's pooled scores."""
    ref_lg = R.window_logits(q, k, c.W)
    masked = R.window_masked(c.W, c.S, logits.device).expand_as(logits)
    half_min = R.finfo_min(c.dtype) / 2
    for t, who in ((logits, "kernel"), (ref_lg, "reference")):
        low = t.float() < half_min
        assert torch.equal(low, masked), f"{c.name}: {who} mask pattern differs from the geometry at {int((low != masked).sum())} logits"
    bad_l = mismatch_count(logits, ref_lg)
    live = ~masked
    if c.inputs == "heavy":
        assert bad_l == 0, f"{c.name}: exact-dot logits differ at {bad_l}"
    else:
        assert bad_l <= max(4, int(2e-3 * ref_lg.numel())), f"{c.name}: {bad_l} logits differ"
        assert _live_logit_ulps(logits, ref_lg, live) <= 2
    own = R.window_scores(logits, c.kernel, c.pooling, mean)
    assert_stage2(pooled.cpu(), own.cpu(), f"{c.name}: pooled vs the reference on the kernel's logits")
    ref = R.window_scores(ref_lg, c.kernel, c.pooling, mean)
    bad, fu = _check_vs_inputs(c, pooled, ref, ref_lg)
    if idx is not None:
        assert torch.equal(oracle.topk(pooled.cpu().contiguous(), idx.shape[1], oracle.TIE_LOWEST_INDEX), idx.cpu())
    return bad_l, bad, fu


def _window_inputs(c: Case, seed):
    """K and V [Hkv, S, D] in HF's strided layout, Q as only the last W rows of a strided [Hq, S, D] view (the rows the
    window scorers read)."""
    q, k, v = make(c, seed, _dev(), q_rows=c.W)
    k = k.permute(1, 0, 2).contiguous().permute(1, 0, 2)
    return q.permute(1, 0, 2).contiguous().permute(1, 0, 2), k, v


@pytest.mark.gpu
@pytest.mark.parametrize("c", WINDOW_CASES, ids=lambda c: c.name)
def test_window_scores_at_length(oracle, libpkv, c):
    """Per-layer staged stages 1-2 at 40K-262K tokens, on the scorer the case names (stage by stage, logits readable)."""
    from pyramidkv_b200 import ops
    q, k, v = _window_inputs(c, c.S + c.Hq)
    if c.scorer == "mma" and not score_tc5_supported(c.Hq, c.Hkv, c.W, c.S, _sms()):
        with pytest.raises(NotImplementedError):
            ops.run_stage(_plan(c, q, k, v, 64, score_kernel="tcgen05")[0], "scores")
    plan, idx = _plan(c, q, k, v, 120)
    assert ops.single_launch(plan) == 0
    t0 = time.time()
    ops.run_stage(plan, "scores")
    logits = ops.ws_logits_as_reference(plan).clone()
    ops.run_stage(plan, "pool")
    ops.run_stage(plan, "topk")
    torch.cuda.synchronize()
    pooled = ops.ws_pooled(plan).clone()
    worst = _partials_check(c, plan, logits)
    bad_l, bad, fu = _window_check(oracle, c, logits, pooled, idx, q, k)
    print(f"PKV_MEASURED {c.name} {sorted(forms(c, _sms()))}: logits {bad_l}/{logits.numel()} pooled {bad}/{pooled.numel()} differ from fp64 "
          f"(flip_ulps {fu}); "
          f"partials rel err {worst:.2e}; {time.time() - t0:.1f} s")


@pytest.mark.gpu
@pytest.mark.parametrize("c", FUSED_CASES, ids=lambda c: c.name)
def test_fused_stages_at_the_tile_limit(oracle, libpkv, c):
    """PKV_FLAG_FUSED and pkv_stage_scan_pool at the last length the fused kernel takes and the first it refuses; the
    refused shape runs as staged launches with the same bars."""
    from pyramidkv_b200 import ops
    if _sms() != H100_SMS:
        pytest.skip(f"the fused kernel's tile limit is restated for {H100_SMS} SMs; this device has {_sms()}")
    q, k, v = _window_inputs(c, c.S)
    takes = "fused:takes" in forms(c)
    plan, idx = _plan(c, q, k, v, 120, fused=True)
    assert ops.single_launch(plan) == (1 if takes else 0), "pkv_evict_single_launch disagrees with the restated plan"
    if takes:
        ops.run_stage(plan, "scan_pool")
    else:
        with pytest.raises(NotImplementedError):
            ops.run_stage(plan, "scan_pool")
        ops.run_stage(plan, "scores")
        ops.run_stage(plan, "pool")
    torch.cuda.synchronize()
    pooled = ops.ws_pooled(plan).clone()
    ref_lg = R.window_logits(q, k, c.W)
    ref = R.window_scores(ref_lg, c.kernel, c.pooling)
    bad, fu = _check_vs_inputs(c, pooled, ref, ref_lg)
    if not takes:
        _window_check(oracle, c, ops.ws_logits_as_reference(plan), pooled, None, q, k)
    plan2, idx2 = _plan(c, q, k, v, 120, fused=True)
    ops.run_stage(plan2, "all")
    torch.cuda.synchronize()
    p2 = ops.ws_pooled(plan2).clone()
    assert mismatch_count(p2, ref) <= max(4, int(2e-3 * ref.numel()))
    assert torch.equal(oracle.topk(p2.cpu().contiguous(), 120, oracle.TIE_LOWEST_INDEX), idx2.cpu())
    print(f"PKV_MEASURED {c.name} S={c.S} {sorted(forms(c))}: pooled {bad}/{ref.numel()} differ from fp64 (flip_ulps {fu})")


def _batch_run(c: Case):
    """Stage 1 then stage 2 of a layer batch (stage 0 where a left-over layer needs the per-layer launches), each layer
    checked against the reference: logits where the batch keeps them, pooled scores always."""
    from pyramidkv_b200 import ops
    v = None
    layers = []
    for l in range(c.layers):
        q, k, vv = _window_inputs(c, 1000 * l + c.S)
        v = vv if v is None else v                           # V is not read by stages 1-2: one tensor for every layer
        layers.append((q, k))
    budgets = [120 + 8 * (l % 5) for l in range(c.layers)]
    plan0, _ = _plan(c, layers[0][0], layers[0][1], v, max(budgets))
    wss = ops.batch_workspaces(plan0, c.layers, max(budgets))
    plans = []
    for (q, k), b, ws in zip(layers, budgets, wss):
        plans.append(_plan(c, q, k, v, b, workspace=ws)[0])
    assert ops.batch_supported(plans)
    batch = ops.EvictBatch(plans)
    staged = c.layers <= MAX_LAYER_BATCH
    if staged:
        batch.run("scores")
        torch.cuda.synchronize()
        logits = [ops.ws_logits_as_reference(p).clone() for p in plans]
        batch.run("pool")
    else:
        batch.run("all")
        logits = [None] * c.layers
    torch.cuda.synchronize()
    worst = 0
    for l, ((q, k), p) in enumerate(zip(layers, plans)):
        pooled = ops.ws_pooled(p)
        if logits[l] is not None:
            bl, bp, _ = _window_check(None, c, logits[l], pooled, None, q, k)
            worst = max(worst, bl, bp)
        else:
            ref_lg = R.window_logits(q, k, c.W)
            ref = R.window_scores(ref_lg, c.kernel, c.pooling)
            bad, _ = _check_vs_inputs(c, pooled, ref, ref_lg)
            worst = max(worst, bad)
    print(f"PKV_MEASURED {c.name} {sorted(forms(c, _sms()))}: worst layer {worst} mismatches; "
          f"peak {torch.cuda.max_memory_allocated() / 2**30:.2f} GiB")


_BATCH_CHILD = r"""
import sys
sys.path.insert(0, "tests")
import test_gpu_score_forms as T
T._batch_run([c for c in T.BATCH_CASES if c.name == sys.argv[1]][0])
"""


@pytest.mark.gpu
@pytest.mark.parametrize("c", BATCH_CASES, ids=lambda c: c.name)
def test_layer_batch_stage_by_stage(libpkv, c):
    """The layer batch's score launch (layer-major walk at 131 072 tokens, contiguous ranges when short, two launches for 33
    layers), then its pool launch with the merged partials or, in a child with PKV_BATCH_MERGE=0, every pool CTA merging
    them itself."""
    if c.merge:
        _batch_run(c)
        return
    torch.cuda.empty_cache()
    r = subprocess.run([sys.executable, "-c", _BATCH_CHILD, c.name], timeout=400, env={**os.environ, "PKV_BATCH_MERGE": "0"},
                       cwd=ROOT, capture_output=True, text=True)
    print(r.stdout[-4000:])
    assert r.returncode == 0, r.stderr[-4000:]


@pytest.mark.gpu
def test_l2norm_and_window_mean_at_131k(oracle, libpkv):
    """L2Norm's negated key norms (bit-exact up to fp32-summation boundary cases, <= 2e-3 of them by 1 ulp) and the AdaKV /
    HeadKV window mean (<= 2e-3 of the scores, <= flip_ulps) at 131 072 tokens."""
    from pyramidkv_b200 import kv_cluster as kcl, ops
    c = OTHER_CASES[0]
    q, k, v = _window_inputs(c._replace(W=8), c.S)
    B = 512
    plan, idx = _plan(c, None, k, v, B)
    ops.run_stage(plan, "scores")
    ops.run_stage(plan, "pool")
    ops.run_stage(plan, "topk")
    torch.cuda.synchronize()
    keys = ops.ws_pooled(plan)
    want = (-R.key_norms(k)).repeat_interleave(c.Hq // c.Hkv, dim=0)
    bad = mismatch_count(keys, want)
    assert bad <= max(2, keys.numel() // 500), f"{bad} norms differ"
    assert float(ulp_own(keys, want, c.dtype).max()) <= 1
    assert torch.equal(oracle.topk(keys.cpu().contiguous(), B, oracle.TIE_LOWEST_INDEX), idx.cpu())
    print(f"PKV_MEASURED l2norm_131072: {bad}/{keys.numel()} norms differ")
    del k, v
    for m in OTHER_CASES[1:]:
        q, k, v = _window_inputs(m, m.S + 1)
        h = kcl.CudaBackend().ragged_begin(q, k, v, m.W, m.kernel, m.pooling)
        torch.cuda.synchronize()
        mine = ops.ws_pooled(h["plan"])
        own = ops.ws_logits_as_reference(h["plan"])
        bl, bm, fu = _window_check(None, m, own, mine, None, q, k, mean=True)
        print(f"PKV_MEASURED {m.name}: logits {bl}/{own.numel()} window-mean scores {bm}/{mine.numel()} differ from fp64 (flip_ulps {fu})")
        del q, k, v, h, mine, own
        torch.cuda.empty_cache()
