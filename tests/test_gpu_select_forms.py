"""Every form of the top-k select (stage 3) and its K / V gather (stage 4), at the budgets and prompt lengths it launches for.

The library picks the select kernel's form from the shape: the per-layer thread-block cluster (2, 4 or 8 CTAs per head, with a
rank, radix or bitonic sort, as a stage of its own, fused with the gather, or with the pool inside it), the single-CTA
fallback (keys in shared memory or re-read, survivor list or full key set), and the layer batch (one CTA per head or a
cluster of 2, 4 or 8, three register builds). A wrong index still yields a cache of the right shape, so every case here is held
to the CPU oracle's selection exactly (value descending, lowest index among equal values), and every cache row to a byte copy
of the K / V row it names.

The library has no query for the form it picked, so this file restates the choice (pkv_topk_cluster.cu, pkv_topk.cu,
pkv_api.cu) and labels each case with it. `test_case_list_reaches_every_form` (no GPU) checks that the cases reach every
reachable combination on a 132-SM H100; `test_restatement_matches_the_library` pins the restatement to
`pkv_evict_batch_supported` on the device.
"""
from __future__ import annotations

import time
from typing import NamedTuple

import pytest
import torch

from gpu_util import dev, mismatch

H100_SMS = 132

# ---------------------------------------------------------------------------------------------------------------------------
# Restatement of the form choice. Line numbers are those of pkv_topk_cluster.cu unless noted.
# ---------------------------------------------------------------------------------------------------------------------------
K_THREADS = 512                 # :29
K_MAX_CLUSTER = 8               # :32
K_MAX_PAD = 32                  # :33
K_MAX_W = 64                    # :34
K_BINS = 256                    # :35
K_RANK_MAX_K = 1024             # :36
K_SMEM_BUDGET = 200 * 1024      # :801
K_RADIX_MAX_K = 8192            # :822
K_TOPK_SMEM_BUDGET = 200 * 1024  # pkv_topk.cu:307
K_COARSE_BITS = 4               # pkv_topk.cu:21
K_MAX_LAYER_BATCH = 32          # pkv_internal.h:43
K_TILE_TOKENS = 128             # pkv_common.cuh:15
K_POOL_IN_SELECT_MAX_S = 12288  # pkv_api.cu:349
MAX_K, MAX_N = 1 << 14, 1 << 20  # :979, :984, :990


def next_pow2(v: int) -> int:                     # :804
    p = 2
    while p < v:
        p <<= 1
    return p


def pick_cluster(Hq: int, sms: int) -> int:       # :806-810
    c = K_MAX_CLUSTER
    while c > 1 and Hq * c > sms:
        c >>= 1
    return c


def rank_limit(batch: bool) -> int:               # :815-818 (PKV_RANK_MAX unset)
    return 512 if batch else K_RANK_MAX_K


def blk_entries(k: int) -> int:                   # :820
    return (k + 2) & ~1


def select_smem(n: int, k: int, c: int, pool: bool = False, batch: bool = False) -> int:   # :824-861
    n8 = (n + 7) // 8
    words = (n8 + c - 1) // c
    rank = k <= rank_limit(batch)
    if batch and c == 1:                          # :828-841 (SOLO)
        b = (blk_entries(k) if rank else next_pow2(max(k, 1))) * 8
        keys = words * 16
        if not rank and k <= K_RADIX_MAX_K:
            keys = max(keys, ((k * 8 + 15) & ~15) + 16 * K_THREADS * 2)
        b = (b + keys + 15) & ~15
        if rank:
            b += (k + 2) * 8
        return b
    b = (blk_entries(k) if rank else next_pow2(max(k, 1))) * 8 + words * 16
    if pool:
        b += (words * 8 + 2 * K_MAX_PAD) * 4
    b = (b + 15) & ~15
    b += 2 * K_MAX_CLUSTER * K_BINS * 4
    b += (k // c + 2) * 8
    b = (b + 15) & ~15
    if rank:
        b += K_MAX_CLUSTER * blk_entries(k) * 8 + ((k + 1) & ~1) * 8 + (k // c + 2) * 4
    elif k <= K_RADIX_MAX_K:
        b = (b + 15) & ~15
        b += ((k + 1) & ~1) * 8
    return b


def batch_cluster(n: int, k: int) -> int:         # :865-869
    c = 1
    while c < K_MAX_CLUSTER and select_smem(n, k, c, batch=True) > K_SMEM_BUDGET:
        c <<= 1
    return c


def topk_cluster_supported(Hq: int, n: int, k: int, sms: int) -> bool:   # :977-981
    c = pick_cluster(Hq, sms)
    if c < 2 or k < 1 or k > MAX_K or n >= MAX_N:
        return False
    return select_smem(n, k, c) <= K_SMEM_BUDGET


def select_fused_supported(Hq: int, n: int, k: int, D: int, W: int, kernel: int, pool: bool, sms: int) -> bool:   # :988-994
    c = pick_cluster(Hq, sms)
    if c < 2 or k < 1 or k > MAX_K or n >= MAX_N or D not in (64, 128):
        return False
    if pool and (W > K_MAX_W or kernel // 2 > K_MAX_PAD):
        return False
    return select_smem(n, k, c, pool) <= K_SMEM_BUDGET


def select_batch_supported(n: int, k: int, D: int = 64) -> bool:      # :983-987
    if k < 1 or k > MAX_K or n >= MAX_N or D not in (64, 128):
        return False
    return select_smem(n, k, batch_cluster(n, k), batch=True) <= K_SMEM_BUDGET


def single_cta(n: int, k: int):                   # pkv_topk.cu:336-345: (keys_in_smem, surv_cap)
    n8 = (n + 7) // 8
    sort_bytes, key_bytes = next_pow2(k) * 8, n8 * 16
    keys_in_smem = sort_bytes + key_bytes + 4096 <= K_TOPK_SMEM_BUDGET
    used = sort_bytes + (key_bytes if keys_in_smem else 0)
    surv_bytes = min(K_TOPK_SMEM_BUDGET - used, key_bytes) & ~15
    return keys_in_smem, surv_bytes // 2


def s_pad(S: int) -> int:                         # pkv_api.cu:113
    return (S + K_TILE_TOKENS - 1) // K_TILE_TOKENS * K_TILE_TOKENS


class Form(NamedTuple):
    kind: str    # "layer" (per-layer cluster), "single" (one CTA per head, pkv_topk.cu), "batch" (layer batch)
    ctas: int    # CTAs per head
    sort: str    # rank / radix / bitonic (the single-CTA kernel always sorts bitonic)
    inst: str    # layer: stage / gather / pool; single: keys smem / global; batch: register build occ1 / occ2 / occ3


def sort_path(k: int, batch: bool) -> str:       # :911 (rank_path), :842-859 / :831-836 (radix_off set up to kRadixMaxK)
    return "rank" if k <= rank_limit(batch) else "radix" if k <= K_RADIX_MAX_K else "bitonic"


def _single(n: int, k: int) -> Form:
    return Form("single", 1, "bitonic", "smem" if single_cta(n, k)[0] else "global")


def stage_form(Hq: int, n: int, k: int, sms: int) -> Form:
    """pkv_stage_topk: launch_topk (pkv_topk.cu:319-323) -> the cluster kernel's stage-only instantiation, else one CTA per head."""
    if topk_cluster_supported(Hq, n, k, sms):
        return Form("layer", pick_cluster(Hq, sms), sort_path(k, False), "stage")
    return _single(n, k)


def prefill_form(Hq: int, S: int, W: int, k: int, D: int, kernel: int, sms: int) -> Form:
    """pkv_evict_prefill with the default flags and knobs (pkv_api.cu:375-388): pool inside the select cluster up to
    s_pad = 12288, else the pool launch and the select + gather cluster; where neither fits, the single-CTA select and the
    gather launch."""
    n = S - W
    pool = s_pad(S) <= K_POOL_IN_SELECT_MAX_S
    if pool and not select_fused_supported(Hq, n, k, D, W, kernel, True, sms):
        pool = False
    if select_fused_supported(Hq, n, k, D, W, kernel, pool, sms):
        return Form("layer", pick_cluster(Hq, sms), sort_path(k, False), "pool" if pool else "gather")
    return _single(n, k)


def batch_forms(n: int, ks) -> list:
    """launch_select_layers (:1005-1014): one CTA count for the launch (the largest any layer needs), the register build from
    the largest k, the sort path per layer."""
    c = max(batch_cluster(n, k) for k in ks)
    kmax = max(ks)
    if c == 1:
        occ = 2 if kmax > rank_limit(True) else 3
    else:
        occ = 1 if kmax > K_RANK_MAX_K else 3
    return [Form("batch", c, sort_path(k, True), f"occ{occ}") for k in ks]


# every combination the library can launch, found by walking a grid of shapes (with two-layer launches for the batch, where
# one layer's CTA count serves the other's budget)
_N_GRID = [1000, 4000, 8000, 12000, 12280, 16000, 20000, 23000, 24000, 32760, 40000, 50000, 65536, 80000, 100000, 131064,
           160000, 200000, 262136, 400000, 524288, 800000, MAX_N - 1, MAX_N + 8]
_K_GRID = [1, 64, 512, 513, 1000, 1024, 1025, 2048, 4000, 8192, 8193, 9000, 12000, 16384]


def reachable_forms(sms: int = H100_SMS) -> set:
    out = set()
    for n in _N_GRID:
        for k in _K_GRID:
            if k > n:
                continue
            for Hq in (8, 32, 64, 72):
                out.add(stage_form(Hq, n, k, sms))
                out.add(prefill_form(Hq, n + 8, 8, k, 128, 7, sms))
        ks = [k for k in _K_GRID if k <= n and select_batch_supported(n, k)]
        for i, a in enumerate(ks):
            for b in ks[i:]:
                out.update(batch_forms(n, [a, b]))
    return out


# ---------------------------------------------------------------------------------------------------------------------------
# The cases. Each is labelled by the restatement at the device's SM count.
# ---------------------------------------------------------------------------------------------------------------------------
# per-layer stage injection: (Hq, n, k)
STAGE_CASES = [
    (8, 40003, 1024), (8, 40003, 1025), (8, 99997, 8192), (8, 99997, 8193), (8, 99997, 12000), (8, 99997, 16384),
    (8, 5003, 5003), (8, 12000, 12000),                                    # k = n: radix, bitonic
    (32, 32763, 1000), (32, 32763, 4000), (32, 32763, 8193), (32, 40000, 16384),
    (64, 32763, 1024), (64, 32763, 3000), (64, 20001, 8200),
    (64, 20001, 16384), (72, 80000, 1000),                                 # single CTA, keys in shared memory (+ overflow)
    (32, 131064, 12000),                                                   # single CTA, keys re-read
    (4, MAX_N - 9, 16384), (4, MAX_N - 1, 1), (4, MAX_N + 5, 16384), (4, MAX_N + 5, 4000),   # around 2^20 tokens
]

# layer-batch stage injection: (n, budgets of the layers)
MIXED = [1, 64, 512, 513, 1025, 8192, 8193, 16384]
BATCH_CASES = [
    (30001, [64, 512]),                                   # SOLO, rank, 40-register build
    (30001, MIXED),                                       # SOLO, every sort path, 64-register build
    (30001, [512, 513]),                                  # SOLO, the batch's rank limit
    (131064, [64, 512]),                                  # 2 CTAs, rank
    (131064, [513, 1024]),                                # 2 CTAs, leader radix sort in the 40-register build
    (131064, [1, 64, 512, 513, 1024, 1025, 2048]),        # 2 CTAs, rank and radix in the 56-register build
    (40003, MIXED),                                       # 4 CTAs, every sort path
    (262136, [1, 512, 513, 1024]),                        # 4 CTAs, 40-register build
    (99997, MIXED),                                       # 8 CTAs, every sort path
    (400000, [1, 512, 513, 1025, 4000]),                  # 8 CTAs at 400K tokens
    (400000, [1, 512, 513, 1024]),                        # 8 CTAs, 40-register build
    (131064, [1, 64, 512, 513, 1024, 1025, 2048, 100] * 4),   # 32 layers in one launch
]


# end to end, layer batch against per-layer pkv_evict_prefill:
# (name, Hq, Hkv, S, D, W, kernel, pooling, dtype, layers, budget (max_capacity_prompt))
E2E_BATCH = [
    ("llama3_8b_128k", 32, 8, 131072, 128, 8, 7, "maxpool", torch.bfloat16, 3, 128),
    ("solo_edge_g8_fp16", 64, 8, 100003, 128, 8, 5, "avgpool", torch.float16, 3, 512),
    ("quarter_m_cluster4", 8, 2, 262144, 128, 8, 7, "maxpool", torch.bfloat16, 3, 1024),
    ("33_layers", 4, 1, 131072, 64, 8, 7, "maxpool", torch.bfloat16, 33, 1024),
]

# end to end, per-layer pkv_evict_prefill: (Hq, Hkv, S, D, k, dtype)
E2E_LAYER = [
    (32, 8, 32768, 128, 12000, torch.bfloat16),           # cluster select + gather, bitonic (k > 8192)
    (32, 8, 12008, 128, 12000, torch.bfloat16),           # pool inside the select, bitonic
    (32, 8, 131072, 128, 12000, torch.bfloat16),          # single-CTA fallback (keys re-read), then the gather
    (8, 2, 12008, 128, 1000, torch.float16), (8, 2, 12008, 128, 4000, torch.bfloat16), (8, 2, 12008, 128, 12000, torch.float16),
    (32, 8, 12008, 128, 1000, torch.bfloat16), (32, 8, 12008, 128, 4000, torch.float16),
    (64, 8, 12008, 128, 1000, torch.bfloat16), (64, 8, 12008, 128, 4000, torch.float16),
    (8, 2, 32768, 128, 1000, torch.bfloat16), (8, 2, 32768, 128, 4000, torch.float16), (8, 2, 65536, 128, 16384, torch.bfloat16),
    (32, 8, 32768, 128, 1000, torch.float16), (32, 8, 32768, 128, 4000, torch.bfloat16),
    (64, 8, 32768, 128, 1000, torch.bfloat16), (64, 8, 32768, 128, 4000, torch.float16), (64, 8, 16392, 128, 8200, torch.bfloat16),
    (64, 8, 24008, 128, 16384, torch.float16),            # single-CTA fallback, keys in shared memory
    (128, 16, 4104, 128, 1000, torch.bfloat16),           # Hq > 66: no cluster fits on 132 SMs
]


def _e2e_batch_forms(case, sms=H100_SMS):
    _, Hq, Hkv, S, D, W, kernel, pooling, dtype, L, budget = case
    ks = _budgets(L, budget, W, S)
    n = S - W
    forms = []
    for l0 in range(0, L, K_MAX_LAYER_BATCH):
        chunk = ks[l0:l0 + K_MAX_LAYER_BATCH]
        if len(chunk) == 1:                        # pkv_api.cu:499-503: a left-over layer runs the per-layer launches
            forms.append(prefill_form(Hq, S, W, chunk[0], D, kernel, sms))
        else:
            forms += batch_forms(n, chunk)
    return forms


def _budgets(L, budget, W, S):
    """PyramidKV's per-layer budgets (pkv_layer_budget: host arithmetic, no device needed)."""
    from pyramidkv_b200 import ops
    return [ops.layer_budget("pyramidkv", budget, W, L, l, S)[1] for l in range(L)]


def case_forms(sms: int = H100_SMS) -> dict:
    """{form: [case ids]} over every case of this file."""
    hit = {}
    for Hq, n, k in STAGE_CASES:
        hit.setdefault(stage_form(Hq, n, k, sms), []).append(f"stage Hq{Hq} n{n} k{k}")
    for n, ks in BATCH_CASES:
        for f in batch_forms(n, ks):
            hit.setdefault(f, []).append(f"batch n{n} ks{ks[:8]}")
    for case in E2E_BATCH:
        for f in _e2e_batch_forms(case, sms):
            hit.setdefault(f, []).append(f"e2e {case[0]}")
    for Hq, Hkv, S, D, k, dtype in E2E_LAYER:
        hit.setdefault(prefill_form(Hq, S, 8, k, D, 7, sms), []).append(f"prefill Hq{Hq} S{S} k{k}")
    return hit


def test_case_list_reaches_every_form():
    """(CTA count x sort path x instantiation) and (CTA count x sort path x register build): every combination the
    restatement can reach on a 132-SM H100 has a case, and every case is a shape the library accepts."""
    reach = reachable_forms()
    hit = case_forms()
    missing = sorted(reach - set(hit))
    assert not missing, f"forms no case reaches: {missing}"
    assert set(hit) <= reach, f"cases label forms the grid never reaches: {sorted(set(hit) - reach)}"
    # combinations that cannot launch (each found by hand from select_smem)
    assert Form("batch", 2, "bitonic", "occ1") not in reach                   # 2 CTAs never hold a k > 8192 sort buffer
    assert Form("layer", 2, "bitonic", "pool") not in reach
    for n, ks in BATCH_CASES:
        assert 2 <= len(ks) <= K_MAX_LAYER_BATCH and all(k <= n and select_batch_supported(n, k) for k in ks), (n, ks)
    for Hq, n, k in STAGE_CASES:
        assert 1 <= k <= min(n, MAX_K)
    # where the single-CTA fallback runs: Hq 32 at 128K with k >= 8192, Hq 64 at 32K with k >= 8192, every prompt >= 2^20
    assert stage_form(32, 131072 - 8, 8192, H100_SMS).kind == "single"
    assert stage_form(64, 32768 - 8, 8192, H100_SMS).kind == "single"
    assert stage_form(8, MAX_N, 64, H100_SMS).kind == "single"
    # the layer batch: one CTA per head up to about 100K tokens, bench.py's 128K workload on 2-CTA clusters
    assert batch_cluster(99000, 234) == 1 and batch_cluster(102400, 234) == 2
    assert {f.ctas for f in _e2e_batch_forms(E2E_BATCH[0])} == {2}
    assert {f.ctas for f in _e2e_batch_forms(E2E_BATCH[2])} == {4}
    print("forms:", len(hit), "reachable:", len(reach))
    for f in sorted(hit):
        print(f, len(hit[f]), hit[f][0])


# ---------------------------------------------------------------------------------------------------------------------------
# GPU: helpers
# ---------------------------------------------------------------------------------------------------------------------------
SENTINEL = 0x7777        # bits of every cache row past k + W: the kernels must leave them alone
PAD_SCORE = 0x7bff       # bits written past n in each pooled row: a large finite score in bf16 and fp16 that no select may see


@pytest.fixture(scope="module", autouse=True)
def _runtime_and_peak_memory(request):
    t0 = time.perf_counter()
    if torch.cuda.is_available():
        torch.cuda.reset_peak_memory_stats()
    yield
    if torch.cuda.is_available() and torch.cuda.is_initialized():
        msg = (f"test_gpu_select_forms: {time.perf_counter() - t0:.1f} s, "
               f"peak device memory {torch.cuda.max_memory_allocated() / 2**30:.2f} GiB")
        tr = request.config.pluginmanager.get_plugin("terminalreporter")
        tr.write_line(msg) if tr else print(msg)


def _sms() -> int:
    return torch.cuda.get_device_properties(0).multi_processor_count


def _encoded_kv(Hkv, S, D, dtype, layer=0):
    """K and V [Hkv, S, D] whose rows spell out (layer, kv head, token) in their first two elements and a hash of them in the
    rest: a row copied from the wrong token, head or layer cannot match by chance."""
    t = torch.arange(S, device=dev(), dtype=torch.int32)[None, :, None]
    h = torch.arange(Hkv, device=dev(), dtype=torch.int32)[:, None, None]
    d = torch.arange(D, device=dev(), dtype=torch.int32)[None, None, :]
    x = (t * 40503 + d * 2531 + h * 977 + layer * 7919 + (t >> 12) * 131) & 0xffff
    x[..., 0] = (t[..., 0] & 0xffff).expand(Hkv, S)
    x[..., 1] = ((t[..., 0] >> 16) | (h[..., 0] << 5) | (layer << 10)).expand(Hkv, S)
    k = x.to(torch.int16).view(dtype)
    v = (x ^ 0x5a5a).to(torch.int16).view(dtype)
    return k, v


def _cache(Hq, k, W, D, dtype):
    kc = torch.full((Hq, k + W + 2, D), SENTINEL, dtype=torch.int16, device=dev()).view(dtype)
    idx = torch.full((Hq, k), -1, dtype=torch.int64, device=dev())
    return kc, kc.clone(), idx


def _inject(plan, scores):
    """Write `scores` [Hq, n] into the plan's pooled rows, with PAD_SCORE in each row's padding past n."""
    from pyramidkv_b200 import ops
    d, L = plan.desc, plan.layout
    full = plan.workspace[L.pooled_off:L.pooled_off + 2 * d.num_q_heads * L.pooled_pitch].view(torch.int16)
    full.view(d.num_q_heads, L.pooled_pitch).fill_(PAD_SCORE)
    ops.ws_pooled(plan).copy_(scores.to(dev()))


def _check(oracle, plan, scores, idx, kc, vc, k_src, v_src, k, W, what):
    """The bars of every case: indices == the oracle's top-k of `scores`, idx_out == idx32, cache rows [0, k + W) byte copies
    of the selected rows and the window, rows past k + W untouched."""
    from pyramidkv_b200 import ops
    Hq = idx.shape[0]
    want = oracle.topk(scores.contiguous(), k, oracle.TIE_LOWEST_INDEX)
    got = idx.cpu()
    if not torch.equal(got, want):
        heads = (got != want).any(1).nonzero().flatten().tolist()
        h = heads[0]
        j = int((got[h] != want[h]).nonzero()[0])
        raise AssertionError(f"{what}: indices differ from the oracle in heads {heads[:8]} of {Hq}; head {h} first at rank {j}: "
                             f"got token {int(got[h, j])}, want {int(want[h, j])}")
    assert torch.equal(ops.ws_idx32(plan).cpu().long(), got), f"{what}: idx_out differs from idx32"
    Hkv, S = k_src.shape[0], k_src.shape[1]
    rows = torch.cat([idx, torch.arange(S - W, S, device=dev()).expand(Hq, W)], 1)
    heads = (torch.arange(Hq, device=dev()) // (Hq // Hkv))[:, None]
    for name, c, src in (("K", kc, k_src), ("V", vc, v_src)):
        same = (c[:, :k + W].view(torch.int16) == src[heads, rows].view(torch.int16)).all(-1)
        if not bool(same.all()):
            h, r = (int(x) for x in (~same).nonzero()[0])
            raise AssertionError(f"{what}: {name} cache head {h} row {r} is not a copy of token {int(rows[h, r])}")
        assert bool((c[:, k + W:].view(torch.int16) == SENTINEL).all()), f"{what}: {name} rows past k + W were written"


# ---- crafted pooled rows ----
PATTERNS = ("equal", "levels2", "levels5", "zeros", "subnormal", "run", "normal", "levels34")


def _levels(n, count, dtype, g):
    vals = (torch.rand(count, generator=g) * 0.9 + 0.05).to(dtype)
    return vals[torch.randint(0, count, (n,), generator=g)]


def _run_row(n, k, dtype, start, end, g):
    """Low scores, a run of equal scores over [start, end) holding the k-th value (about half of the run is taken, lowest
    index first), and the k - (taken) best scores scattered outside it. None when k leaves no room for such a run."""
    L = end - start
    m = max(1, L // 2)
    top = k - m
    if top < 0:
        top, m = 0, k
    if top > n - L:
        top = n - L
        m = k - top
    if not 1 <= m < L:
        return None
    row = (torch.rand(n, generator=g) * 0.25).to(dtype)
    row[start:end] = 0.5
    outside = torch.cat([torch.arange(0, start), torch.arange(end, n)])
    row[outside[torch.randperm(outside.numel(), generator=g)[:top]]] = (1 + torch.rand(top, generator=g)).to(dtype)
    return row


def _row(pattern, h, n, k, dtype, span, ctas, run_len, g):
    if pattern == "equal":
        return torch.full((n,), 0.375).to(dtype)
    if pattern.startswith("levels"):
        return _levels(n, {"levels2": 2, "levels5": 5}.get(pattern, 3 + h % 2), dtype, g)
    if pattern == "zeros":                       # thousands of exact zeros, the k-th value among them
        row = torch.zeros(n, dtype=dtype)
        pos = torch.randperm(n, generator=g)[:k // 2]
        row[pos] = (torch.rand(pos.numel(), generator=g) + 0.01).to(dtype)
        return row
    if pattern == "subnormal":                   # subnormals, zeros and a few normal values
        top = 0x7f if dtype == torch.bfloat16 else 0x3ff
        bits = torch.randint(1, top + 1, (n,), generator=g, dtype=torch.int16)
        bits[torch.randperm(n, generator=g)[:n // 8]] = 0
        row = bits.view(dtype).clone()
        row[torch.randperm(n, generator=g)[:k // 4]] = 0.5
        return row
    if pattern == "run":                         # ties across the per-CTA key ranges (or the overflow run)
        bounds = [r * span for r in range(1, ctas) if r * span < n] or [n // 2]
        start, end = max(0, bounds[0] - 200), min(n, bounds[-1] + 200)
        if run_len and run_len < n:
            start = max(0, min(n - run_len, start))
            end = start + run_len
        row = _run_row(n, k, dtype, start, end, g)
        return row if row is not None else _levels(n, 2, dtype, g)
    return torch.randn(n, generator=g).to(dtype)  # "normal": negative values too


def _craft(Hq, n, k, dtype, span, ctas, seed, run_len=0):
    g = torch.Generator().manual_seed(seed)
    return torch.stack([_row(PATTERNS[h % len(PATTERNS)], h, n, k, dtype, span, ctas, run_len, g) for h in range(Hq)])


def _span(n, ctas):                              # tokens per CTA key range: words_per_cta * 8 (:882)
    return ((n + 7) // 8 + ctas - 1) // ctas * 8


def _key(bits: torch.Tensor) -> torch.Tensor:     # order-preserving 16-bit key (:127-130, pkv_topk.cu:40-43)
    b = bits.to(torch.int32) & 0xffff
    return torch.where(b >= 0x8000, b ^ 0xffff, b ^ 0x8000)


def _overflows(scores, k, surv_cap):
    """Heads whose single-CTA survivor list overflows: the survivors hold every key equal to the k-th (pkv_topk.cu:140-170),
    and the list is built only when more than kCoarseBits bits differ between the smallest and largest key."""
    out = []
    for h in range(scores.shape[0]):
        row = scores[h]
        kth = row.float().sort(descending=True).values[k - 1]
        keys = _key(row.view(torch.int16))
        nbits = int(keys.min() ^ keys.max()).bit_length()
        if nbits > K_COARSE_BITS and int((row.float() == kth).sum()) > surv_cap:
            out.append(h)
    return out


# ---------------------------------------------------------------------------------------------------------------------------
# GPU: the restatement against the library
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_restatement_matches_the_library(libpkv):
    """pkv_evict_batch_supported against select_batch_supported on both sides of the layer batch's support edge, and the
    device's SM count against the one the case labels assume."""
    from pyramidkv_b200 import ops
    Hq, Hkv, W, D = 4, 1, 8, 64
    Smax = MAX_N + 16
    kk = torch.zeros(Hkv, Smax, D, dtype=torch.bfloat16, device=dev())
    q = torch.zeros(Hq, W, D, dtype=torch.bfloat16, device=dev())
    probes = []
    for S in (30008, 40008, 100000, 100008, 102408, 131072, 160008, 200000, 262144, 400000, 524296, 800000, 800008,
              MAX_N - 16, MAX_N + 8):
        for ks in ([1, 1], [512, 512], [513, 513], [1024, 1024], [1025, 1025], [4000, 4000], [8000, 8000], [8192, 8192],
                   [8193, 8193], [16000, 16000], [16384, 16384], [16385, 16385], [1, 16384], [512, 8000]):
            if max(ks) > S - W:
                continue
            plans = []
            for k in ks:
                kc = torch.empty(Hq, k + W, D, dtype=torch.bfloat16, device=dev())
                plans.append(ops.plan_evict("snapkv", q, kk[:, :S], kk[:, :S], W, k, kc, kc, 1, "maxpool"))
            wss = ops.batch_workspaces(plans[0], len(ks), max(ks))
            plans = [ops.plan_evict("snapkv", q, kk[:, :S], kk[:, :S], W, k, p.keep[3], p.keep[4], 1, "maxpool", workspace=ws)
                     for k, p, ws in zip(ks, plans, wss)]
            lib = ops.batch_supported(plans)
            mine = all(select_batch_supported(S - W, k, D) for k in ks)
            probes.append((S, ks, lib, mine))
    wrong = [p for p in probes if p[2] != p[3]]
    assert not wrong, f"restatement disagrees with pkv_evict_batch_supported at (S, budgets, library, restatement): {wrong}"
    by = {(S, ks[0], ks[1]): lib for S, ks, lib, _ in probes}
    assert by[(200000, 8000, 8000)] and not by[(200000, 16000, 16000)]          # the support edge at 200 000 tokens
    assert any(p[2] for p in probes) and any(not p[2] for p in probes)
    print(f"{len(probes)} probes agree; supported at {sum(p[2] for p in probes)}")
    if _sms() != H100_SMS:
        pytest.skip(f"{_sms()} SMs: the per-layer cluster sizes of the case labels assume {H100_SMS}")


# ---------------------------------------------------------------------------------------------------------------------------
# GPU: per-layer stage injection (pkv_stage_topk, then pkv_stage_gather)
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16], ids=["bf16", "fp16"])
@pytest.mark.parametrize("Hq,n,k", STAGE_CASES)
def test_stage_injection(oracle, libpkv, Hq, n, k, dtype):
    from pyramidkv_b200 import ops
    W, D, Hkv = 8, 64, 1
    S = n + W
    form = stage_form(Hq, n, k, _sms())
    if form.kind == "single":        # ties across the emit loop's 8192-token passes, and enough to overflow the survivor list
        span, ctas = 8192, 4
        surv_cap = single_cta(n, k)[1]
        run_len = surv_cap + 2048 if surv_cap + 2048 < n else 0
    else:
        span, ctas, surv_cap, run_len = _span(n, form.ctas), form.ctas, 0, 0
    k_src, v_src = _encoded_kv(Hkv, S, D, dtype)
    q = torch.zeros(Hq, W, D, dtype=dtype, device=dev())
    kc, vc, idx = _cache(Hq, k, W, D, dtype)
    plan = ops.plan_evict("snapkv", q, k_src, v_src, W, k, kc, vc, 1, "maxpool", idx_out=idx)
    scores = _craft(Hq, n, k, dtype, span, ctas, seed=n * 7 + k + Hq, run_len=run_len)
    _inject(plan, scores)
    ops.run_stage(plan, "topk")
    ops.run_stage(plan, "gather")
    torch.cuda.synchronize()
    _check(oracle, plan, scores, idx, kc, vc, k_src, v_src, k, W, f"{form} Hq {Hq} n {n} k {k}")
    if run_len:
        assert _overflows(scores, k, surv_cap), "no head overflowed the survivor list"


# ---------------------------------------------------------------------------------------------------------------------------
# GPU: layer-batch stage injection (stage 3 of pkv_stage_batch: select + gather)
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16], ids=["bf16", "fp16"])
@pytest.mark.parametrize("n,ks", BATCH_CASES, ids=[f"n{n}-L{len(ks)}-kmax{max(ks)}-{i}" for i, (n, ks) in enumerate(BATCH_CASES)])
def test_batch_select_injection(oracle, libpkv, n, ks, dtype):
    from pyramidkv_b200 import ops
    Hq, Hkv, W, D = 8, 1, 8, 64
    S = n + W
    forms = batch_forms(n, ks)
    c = forms[0].ctas
    span, ctas = (_span(n, c), c) if c > 1 else (_span(n, 4), 4)
    q = torch.zeros(Hq, W, D, dtype=dtype, device=dev())
    layers = []
    for l, k in enumerate(ks):
        k_src, v_src = _encoded_kv(Hkv, S, D, dtype, layer=l)
        kc, vc, idx = _cache(Hq, k, W, D, dtype)
        layers.append((k_src, v_src, kc, vc, idx))
    first = ops.plan_evict("snapkv", q, layers[0][0], layers[0][1], W, ks[0], layers[0][2], layers[0][3], 1, "maxpool")
    wss = ops.batch_workspaces(first, len(ks), max(ks))
    plans = [ops.plan_evict("snapkv", q, k_src, v_src, W, k, kc, vc, 1, "maxpool", idx_out=idx, workspace=ws)
             for k, (k_src, v_src, kc, vc, idx), ws in zip(ks, layers, wss)]
    assert ops.batch_supported(plans)
    scores = [_craft(Hq, n, k, dtype, span, ctas, seed=1000 * l + n + k) for l, k in enumerate(ks)]
    for p, s in zip(plans, scores):
        _inject(p, s)
    ops.EvictBatch(plans).run("select")
    torch.cuda.synchronize()
    for l, (k, p, s, f) in enumerate(zip(ks, plans, scores, forms)):
        k_src, v_src, kc, vc, idx = layers[l]
        _check(oracle, p, s, idx, kc, vc, k_src, v_src, k, W, f"{f} layer {l} of {len(ks)} n {n} k {k}")


# ---------------------------------------------------------------------------------------------------------------------------
# GPU: end to end at long prompts
# ---------------------------------------------------------------------------------------------------------------------------
def _inputs(Hq, Hkv, S, D, dtype, g):
    """q's window rows [Hq, W, D] and K / V in HF's [S, H, D] memory layout, drawn on the device."""
    k = torch.randn(S, Hkv, D, device=dev(), dtype=dtype, generator=g).permute(1, 0, 2)
    v = torch.randn(S, Hkv, D, device=dev(), dtype=dtype, generator=g).permute(1, 0, 2)
    q = torch.randn(Hq, 8, D, device=dev(), dtype=dtype, generator=g)
    return q, k, v


def _oracle_pooled(oracle, q, k, v, W, top_k, kernel, pooling):
    S = k.shape[1]
    q_full = torch.empty(q.shape[0], S, q.shape[2], dtype=q.dtype)    # the oracle reads only the window rows
    q_full[:, S - W:] = q.cpu()
    return oracle.evict("pyramidkv", q_full, k.cpu(), v.cpu(), W, top_k, kernel, pooling, tie_mode=oracle.TIE_LOWEST_INDEX).pooled


@pytest.mark.gpu
@pytest.mark.parametrize("case", E2E_BATCH, ids=[c[0] for c in E2E_BATCH])
def test_layer_batch_end_to_end(oracle, libpkv, case):
    """The layer batch against per-layer pkv_evict_prefill on the same inputs (test_gpu_batch's bars), every head of every
    layer against the oracle's top-k of the pooled rows the batch wrote, one layer's pooled rows against oracle.evict."""
    from pyramidkv_b200 import ops
    name, Hq, Hkv, S, D, W, kernel, pooling, dtype, L, budget = case
    ks = _budgets(L, budget, W, S)
    forms = _e2e_batch_forms(case, _sms())
    g = torch.Generator(device=dev()).manual_seed(L * 1000 + Hq)
    layers = [_inputs(Hq, Hkv, S, D, dtype, g) for _ in range(L)]
    ref = []
    for (q, k, v), top_k in zip(layers, ks):
        kc, vc, idx = _cache(Hq, top_k, W, D, dtype)
        plan = ops.plan_evict("pyramidkv", q, k, v, W, top_k, kc, vc, kernel, pooling, idx_out=idx)
        ops.run_stage(plan, "all")
        ref.append((ops.ws_pooled(plan).cpu(), idx, kc, vc))
    plans = []
    for l, ((q, k, v), top_k) in enumerate(zip(layers, ks)):
        kc, vc, idx = _cache(Hq, top_k, W, D, dtype)
        if l == 0:
            wss = ops.batch_workspaces(ops.plan_evict("pyramidkv", q, k, v, W, top_k, kc, vc, kernel, pooling), L, max(ks))
        plans.append(ops.plan_evict("pyramidkv", q, k, v, W, top_k, kc, vc, kernel, pooling, idx_out=idx, workspace=wss[l]))
    assert ops.batch_supported(plans)
    ops.evict_prefill_batch(plans)
    torch.cuda.synchronize()
    identical = 0
    for l, (p, top_k) in enumerate(zip(plans, ks)):
        (q, k, v), f = layers[l], forms[l]
        pr, ir, kr, vr = ref[l]
        pg = ops.ws_pooled(p).cpu()
        ig, kg, vg = p.keep[5], p.keep[3], p.keep[4]
        what = f"{name} layer {l} ({f}, k {top_k})"
        _check(oracle, p, pg, ig, kg, vg, k, v, top_k, W, what)
        # the score CTAs cut the token range at other places in a batch, so a merged (max, sumexp) may differ in the last ulp;
        # over 100K-token rows that leaves few rows identical, so the bar is test_gpu_batch's element count
        bad = mismatch(pg, pr)
        assert bad <= max(4, int(2e-3 * pr.numel())), f"{what}: pooled differs from the per-layer call at {bad}/{pr.numel()}"
        same = [h for h in range(Hq) if torch.equal(pg[h], pr[h])]
        identical += len(same)
        for h in same:
            assert torch.equal(ig[h], ir[h]), f"{what} head {h}: indices differ for equal scores"
            assert torch.equal(kg[h].view(torch.int16), kr[h].view(torch.int16)) and torch.equal(vg[h].view(torch.int16), vr[h].view(torch.int16)), \
                f"{what} head {h}: cache differs for equal scores"
    l = L // 2
    o = _oracle_pooled(oracle, *layers[l], W, ks[l], kernel, pooling)
    bad = mismatch(ops.ws_pooled(plans[l]).cpu(), o)
    print(f"PKV_MEASURED select_forms {name}: identical pooled rows {identical}/{L * Hq}, layer {l} vs oracle {bad}/{o.numel()}")
    assert bad <= int(1e-3 * o.numel()), f"{name} layer {l}: pooled differs from the oracle at {bad}/{o.numel()}"


@pytest.mark.gpu
@pytest.mark.parametrize("Hq,Hkv,S,D,k,dtype", E2E_LAYER)
def test_prefill_end_to_end(oracle, libpkv, Hq, Hkv, S, D, k, dtype):
    """Per-layer pkv_evict_prefill through each cluster size x sort path x (pool inside the select / select + gather), and
    the single-CTA fallback: the indices are the oracle's top-k of the pooled rows the GPU wrote, the rows their copies, the
    pooled rows those of oracle.evict."""
    from pyramidkv_b200 import ops
    W, kernel, pooling = 8, 7, "maxpool"
    form = prefill_form(Hq, S, W, k, D, kernel, _sms())
    g = torch.Generator(device=dev()).manual_seed(S + k + Hq)
    q, kk, vv = _inputs(Hq, Hkv, S, D, dtype, g)
    kc, vc, idx = _cache(Hq, k, W, D, dtype)
    plan = ops.plan_evict("pyramidkv", q, kk, vv, W, k, kc, vc, kernel, pooling, idx_out=idx)
    ops.run_stage(plan, "all")
    torch.cuda.synchronize()
    pooled = ops.ws_pooled(plan).cpu()
    _check(oracle, plan, pooled, idx, kc, vc, kk, vv, k, W, f"{form} Hq {Hq} S {S} k {k}")
    o = _oracle_pooled(oracle, q, kk, vv, W, k, kernel, pooling)
    bad = mismatch(pooled, o)
    print(f"PKV_MEASURED select_forms prefill {form} Hq {Hq} S {S} k {k}: pooled vs oracle {bad}/{o.numel()}")
    assert bad <= max(4, int(2e-3 * o.numel())), f"{form}: pooled differs from the oracle at {bad}/{o.numel()}"
