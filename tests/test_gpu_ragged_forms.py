"""AdaKV and HeadKV at the prompt lengths and head skews they run at: the budget kernels, the host's tie split and rounding,
the ragged select + gather (with per-head budgets above the select kernels' 16 384), the window placement, and decode and
the E4M3 conversion over very uneven per-head row counts.

Skew is the point of AdaKV: a head whose attention is spread over the whole prompt can win most of the layer's Hq * base
slots while sink and local heads keep a few hundred, and HeadKV's budgets come from a head-score file. Gaussian inputs keep
every budget near base, so every case here is built to reach a named regime, and asserts through the oracle that it does:

- a budget above 16 384 (the largest top_k of the select kernels; such heads take the sort path of `ragged_finish`);
- a head that takes all n of its candidates;
- threshold ties shared by two or more heads, of which the lower heads take the tied slots;
- a threshold of exactly 0 with -0.0 (0x8000) among the zeros;
- subnormal scores at the threshold;
- a NaN ratio (normalize, a head whose scores are all zero: 0 / 0), whose scaled scores rank above every value;
- base == n and base == 1.

Bars. The budget kernels (`pkv_adakv_counts`, called through `_lib` so that the threshold and the ratios can be read) must
equal the oracle exactly: counts above / equal to the threshold, the threshold's bit pattern, every ratio and the host's
budgets. Both sides round the same double-precision multiset sums, so there is no tolerance. Against torch_chain (torch's
fp32-accumulated `.sum()`), a ratio may differ by 1 ulp; differing heads are reported. Every cache row is a byte copy of
`oracle.ragged_evict` on the GPU's own pooled scores.
"""
from __future__ import annotations

import ctypes as C
import math
from typing import NamedTuple

import pytest
import torch

from gpu_util import dev

BF, FP = torch.bfloat16, torch.float16
SELECT_MAX_K = 16384
ADAKV_BINS = 32768                       # pkv_adakv.cu: kBins; scratch = [kBins] u32 histogram | 4 u32 | [Hq] float ratios
REGIMES = ("cap_over_16384", "count_eq_n", "shared_ties", "zero_thr_negzero", "subnormal_thr", "nan_ratio", "base_eq_n",
           "base_eq_1")


# ---------------------------------------------------------------------------------------------------------------------------
# Injected pooled rows
# ---------------------------------------------------------------------------------------------------------------------------
class Case(NamedTuple):
    name: str
    Hq: int
    Hkv: int
    D: int
    dtype: torch.dtype
    n: int
    base: int
    normalize: bool
    kinds: str            # one letter per head, repeated to Hq: s sink, b broad, z all zero, p sparse, u subnormal


def _row(kind: str, n: int, dtype, g) -> torch.Tensor:
    """One pooled row [n] in `dtype`. Sink rows are identical across heads (same ratio, so their background ties)."""
    if kind == "s":                      # 0.9 on token 0, a decaying local band at the end, a flat background of 2^-20
        x = torch.full((n,), 2.0 ** -20)
        d = torch.arange(299, -1, -1, dtype=torch.float64)
        band = torch.exp(-d / 60.0)
        x[n - 300:] = (0.1 * band / band.sum()).float()
        x[0] = 0.9
    elif kind == "b":                    # attention spread over the whole prompt
        x = (1.0 + 0.3 * torch.randn(n, generator=g)).clamp(min=0.05) / n
    elif kind == "z":                    # all zero, every third one -0.0
        x = torch.zeros(n)
        x[::3] = -0.0
    elif kind == "p":                    # 1% non-zero, the rest +0.0 / -0.0
        x = torch.zeros(n)
        x[1::2] = -0.0
        nz = torch.randperm(n, generator=g)[: max(1, n // 100)]
        x[nz] = torch.rand(nz.numel(), generator=g) * 1e-3 + 1e-5
    elif kind == "u":                    # subnormal multiples of the dtype's smallest subnormal, half of them zero
        tiny, top = (2.0 ** -133, 127) if dtype == BF else (2.0 ** -24, 1023)
        x = torch.randint(1, top + 1, (n,), generator=g).double() * tiny
        x[torch.rand(n, generator=g) < 0.5] = 0.0
        return x.to(dtype)
    else:
        raise ValueError(kind)
    return x.to(dtype)


def inject_rows(c: Case) -> torch.Tensor:
    g = torch.Generator().manual_seed(c.n + c.base + c.Hq)
    kinds = (c.kinds * c.Hq)[: c.Hq]
    return torch.stack([_row(k, c.n, c.dtype, g) for k in kinds])


CASES = [
    Case("broad_8b_32k_norm", 32, 8, 128, BF, 32736, 2016, True, "sssssbssssssssssssssssssssssssss"),
    Case("broad_8b_32k_raw_fp16", 32, 8, 128, FP, 32736, 2016, False, "sssssbssssssssssssssssssssssssss"),
    Case("broad_g8_100k_raw", 64, 8, 128, BF, 100003, 2016, False, "sb" + "s" * 62),
    Case("broad_8b_131k_16352_raw", 32, 8, 128, BF, 131040, 16352, False, "bs"),
    Case("nan_mha_131k_16352", 8, 8, 64, FP, 131040, 16352, True, "zsssbsss"),
    Case("nan_mha_32k_16352_all_n", 8, 8, 64, FP, 32736, 16352, True, "szsbssss"),
    Case("nan_mha_32k_96", 8, 8, 64, BF, 32736, 96, True, "sssz"),
    Case("zero_thr_8b_32k_raw", 32, 8, 128, BF, 32736, 2016, False, "p"),
    Case("zero_thr_8b_32k_norm_fp16", 32, 8, 128, FP, 32736, 2016, True, "p"),
    Case("subnormal_8b_32k_96", 32, 8, 128, BF, 32736, 96, False, "u"),
    Case("subnormal_g8_100k_96_fp16", 64, 8, 128, FP, 100003, 96, True, "uup"),
    Case("base_n_mha_32k", 8, 8, 64, BF, 32736, 32736, True, "sb"),
    Case("base_n_mha_100k_raw_fp16", 8, 8, 64, FP, 100003, 100003, False, "bsu"),
    Case("base_1_8b_131k_norm", 32, 8, 128, BF, 131040, 1, True, "sssbs"),
    Case("base_1_g8_32k_raw_fp16", 64, 8, 128, FP, 32736, 1, False, "s"),
]


def _is_nan16(bits: int, dtype) -> bool:
    e = bits & 0x7fff
    return e > 0x7f80 if dtype == BF else e > 0x7c00


def _key(bits: int, dtype) -> int:
    """A 16-bit score as the budget kernels key it: negatives (only -0.0 occurs) are 0, NaN is the top bin 0x7fff."""
    bits &= 0xffff
    if _is_nan16(bits, dtype):
        return 0x7fff
    return 0 if bits & 0x8000 else bits


class OracleResult(NamedTuple):
    caps: list
    gt: list
    eq: list
    thr_key: int
    ratio: torch.Tensor
    total_above: int


def oracle_counts(oracle, rows: torch.Tensor, base: int, normalize: bool) -> OracleResult:
    ratio = torch.empty(rows.shape[0], dtype=torch.float32)
    caps, gt, eq, thr, _ = oracle.adakv_capacities(rows, base, 0.2, normalize, details=True, ratio_out=ratio)
    thr_bits = int(thr.view(torch.int16)[0]) & 0xffff
    return OracleResult(caps.tolist(), gt.tolist(), eq.tolist(), _key(thr_bits, rows.dtype), ratio, int(sum(gt.tolist())))


def regimes(rows: torch.Tensor, base: int, normalize: bool, r: OracleResult) -> set:
    """The regimes an injected case reaches, read off the oracle's result."""
    H, n = rows.shape
    dtype = rows.dtype
    out = set()
    if max(r.caps) > SELECT_MAX_K:
        out.add("cap_over_16384")
    need = H * base - r.total_above
    counts, left = [], need
    for h in range(H):
        take = min(left, r.eq[h])
        left -= take
        counts.append(r.gt[h] + take)
    if n in counts:
        out.add("count_eq_n")
    if sum(1 for e in r.eq if e > 0) >= 2 and 0 < need < sum(r.eq):
        out.add("shared_ties")
    bits = rows.view(torch.int16).int() & 0xffff
    if r.thr_key == 0 and bool((bits == 0x8000).any()):
        out.add("zero_thr_negzero")
    min_normal = 0x0080 if dtype == BF else 0x0400
    if 0 < r.thr_key < min_normal:
        out.add("subnormal_thr")
    if normalize and bool(torch.isnan(r.ratio).any()):
        out.add("nan_ratio")
    if base == n:
        out.add("base_eq_n")
    if base == 1:
        out.add("base_eq_1")
    return out


_oracle_cache: dict = {}


def _oracle_case(oracle, c: Case):
    if c.name not in _oracle_cache:
        rows = inject_rows(c)
        r = oracle_counts(oracle, rows, c.base, c.normalize)
        _oracle_cache.clear()
        _oracle_cache[c.name] = (rows, r, regimes(rows, c.base, c.normalize, r))
    return _oracle_cache[c.name]


def test_injected_cases_reach_every_regime(oracle):
    """No GPU: every regime of the module docstring is reached by at least one injected case."""
    reached = {}
    for c in CASES:
        _, r, got = _oracle_case(oracle, c)
        print(f"{c.name}: max budget {max(r.caps)}, {sorted(got)}")
        for g in got:
            reached.setdefault(g, []).append(c.name)
    missing = [x for x in REGIMES if x not in reached]
    assert not missing, f"no case reaches {missing}"


def test_oracle_ranks_nan_ratio_like_torch(oracle):
    """A head whose scores are all zero gets ratio 0 / 0 = NaN under normalize; torch ranks NaN above every value, and so
    must the oracle (before, its nth_element ran over NaNs with a `>` comparator: undefined behaviour)."""
    from oracle import torch_chain as tc
    for dtype in (BF, FP):
        H, n = 4, 16
        score = (torch.arange(H * n, dtype=torch.float32).reshape(H, n) % 7 + 1) / 64
        score[1] = 0.0
        score[1, ::2] = -0.0
        score = score.to(dtype)
        for base in (3, 8, 16):
            ratio = torch.empty(H, dtype=torch.float32)
            caps, gt, eq, _, _ = oracle.adakv_capacities(score, base, 0.2, True, details=True, ratio_out=ratio)
            assert bool(torch.isnan(ratio[1])) and not bool(torch.isnan(ratio[[0, 2, 3]]).any())
            want, _ = tc.adakv_capacities(score[None], base, 0.2, True, tie_rule="lowest_index")
            assert caps.tolist() == want.tolist(), (dtype, base, caps.tolist(), want.tolist())
            assert gt[1] + min(eq[1], H * base) == min(n, H * base)        # the NaN head comes first


# ---------------------------------------------------------------------------------------------------------------------------
# GPU: the budget kernels at length, by stage injection
# ---------------------------------------------------------------------------------------------------------------------------
_ratio_report: list = []


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=[c.name for c in CASES])
def test_budget_kernels_injected(oracle, libpkv, case):
    from oracle import torch_chain as tc
    from pyramidkv_b200 import _lib, kv_cluster as kc, ops
    c = case
    rows, r, _ = _oracle_case(oracle, c)
    W = 8
    S = c.n + W
    q = torch.zeros(c.Hq, W, c.D, dtype=c.dtype, device=dev())
    k = torch.zeros(c.Hkv, S, c.D, dtype=c.dtype, device=dev())
    be = kc.CudaBackend()
    handle = be.ragged_begin(q, k, k, W, 7, "maxpool")
    plan = handle["plan"]
    pooled = ops.ws_pooled(plan)
    pooled.copy_(rows.to(dev()))
    scratch = torch.zeros(int(_lib.lib().pkv_adakv_scratch_bytes(c.Hq)), dtype=torch.uint8, device=dev())
    counts = torch.empty(2 * c.Hq + 2, dtype=torch.int32, device=dev())
    _lib.check(_lib.lib().pkv_adakv_counts(C.byref(plan.desc), c.base, int(c.normalize), scratch.data_ptr(), scratch.numel(),
                                           counts.data_ptr(), plan.stream_ptr()))
    torch.cuda.synchronize()
    got = counts.cpu().tolist()
    ratio = scratch[ADAKV_BINS * 4 + 16: ADAKV_BINS * 4 + 16 + 4 * c.Hq].view(torch.float32).cpu()
    assert got[: c.Hq] == r.gt, "values above the threshold"
    assert got[c.Hq: 2 * c.Hq] == r.eq, "values equal to the threshold"
    assert got[2 * c.Hq] == r.thr_key, f"threshold bits {got[2 * c.Hq]:#06x} vs {r.thr_key:#06x}"
    assert got[2 * c.Hq + 1] == r.total_above
    nan_k, nan_o = torch.isnan(ratio), torch.isnan(r.ratio)
    assert torch.equal(nan_k, nan_o) and torch.equal(ratio[~nan_k].view(torch.int32), r.ratio[~nan_o].view(torch.int32)), "ratios"
    cl = kc.AdaKVCluster(window_size=W, kernel_size=7, pooling="maxpool", max_capacity_prompt=c.base + W, floor=0.2,
                         normalize=c.normalize, layer_idx=0, num_hidden_layers=1)
    assert [int(x) for x in cl._capacities(handle, c.Hq)] == r.caps
    # torch_chain on the device: its ratio is torch's fp32-accumulated .sum(), rounded to the model dtype
    pd = pooled.contiguous()
    diff = 0
    if c.normalize:
        srt = torch.sort(pd.float(), dim=-1, descending=True, stable=True).values.to(c.dtype)
        tr = tc.adakv_ratio(srt, c.base)[:, 0].float().cpu()
        assert torch.equal(torch.isnan(tr), nan_k)
        fin = ~nan_k
        a, b = tr[fin].to(c.dtype).view(torch.int16).int(), ratio[fin].to(c.dtype).view(torch.int16).int()
        diff = int((a != b).sum())
        assert int((a - b).abs().max()) <= 1 if a.numel() else True, "a ratio more than 1 ulp from torch's"
        _ratio_report.append((c.name, diff, c.Hq))
        print(f"PKV_MEASURED ratio_vs_torch_chain {c.name}: {diff}/{c.Hq} heads differ by 1 ulp")
    if diff == 0:
        # -0.0 goes in as +0.0: torch's radix sort orders -0.0 below +0.0, while the library keys both as 0 (the scores it
        # sees are sums of probabilities, never -0.0)
        caps_t, _ = tc.adakv_capacities((pd + 0.0)[None], c.base, 0.2, c.normalize, tie_rule="lowest_index")
        assert caps_t.cpu().tolist() == r.caps, "budgets differ from torch_chain"


# ---------------------------------------------------------------------------------------------------------------------------
# GPU: the ragged eviction end to end
# ---------------------------------------------------------------------------------------------------------------------------
def build_heads(kinds: str, Hq: int, Hkv: int, S: int, D: int, W: int, dtype, seed: int):
    """Exact-dot inputs with one logit row per QUERY head: query head h has c = sqrt(D) in dim h % G and KV head h // G holds
    head h's logits x in that dim, so every logit is one exact product. q [Hq, W, D] (the window rows; every query row is
    the same), k / v [Hkv, S, D] on the CPU.
    Kinds: s sink (16 on token 0, a band 8 - d/64 over the last 512 tokens, 0 elsewhere); b broad (0.5 N(0,1)); w the
    window attends to itself (30 on the window keys, 0 elsewhere: every non-window probability underflows in fp16);
    p sparse (0.5 N(0,1) on the first 20 000 tokens, -120 on the rest, whose probabilities underflow in bf16 and fp16)."""
    G = Hq // Hkv
    assert G <= D
    g = torch.Generator().manual_seed(seed)
    cval = float(torch.tensor(math.sqrt(D)).to(dtype).float())
    q = torch.zeros(Hq, W, D)
    k = torch.zeros(Hkv, S, D)
    d = torch.arange(S - 1, -1, -1).float()
    for h in range(Hq):
        kind = kinds[h % len(kinds)]
        if kind == "s":
            x = torch.where(d < 512, 8.0 - d / 64.0, torch.zeros(S))
            x[0] = 16.0
        elif kind == "b":
            x = 0.5 * torch.randn(S, generator=g)
        elif kind == "w":
            x = torch.zeros(S)
            x[S - W:] = 30.0
        elif kind == "p":
            x = torch.full((S,), -120.0)
            x[:20000] = 0.5 * torch.randn(20000, generator=g)
            x[S - W:] = 0.0
        else:
            raise ValueError(kind)
        q[h, :, h % G] = cval
        k[h // G, :, h % G] = x
    v = torch.randn(Hkv, S, D, generator=g)
    return q.to(dtype), k.to(dtype), v.to(dtype)


def _check_rows(oracle, k_buf, v_buf, rows, k, v, pooled, caps, W):
    ks, vs, _ = oracle.ragged_evict(k, v, pooled, caps, W)
    kb, vb = k_buf.cpu(), v_buf.cpu()
    for h in range(len(caps)):
        assert rows[h] == caps[h] + W
        assert torch.equal(kb[h, :rows[h]].view(torch.int16), ks[h].view(torch.int16)), f"K rows of head {h} (cap {caps[h]})"
        assert torch.equal(vb[h, :rows[h]].view(torch.int16), vs[h].view(torch.int16)), f"V rows of head {h} (cap {caps[h]})"


ADAKV_E2E = [  # (name, Hq, Hkv, D, dtype, S, B, W, normalize, kinds)
    ("8b_32k_w8_norm", 32, 8, 128, BF, 32768, 2048, 8, True, "sssssbssssssssssssssssssssssssss"),
    ("8b_32k_w8_raw", 32, 8, 128, BF, 32768, 2048, 8, False, "sssssbssssssssssssssssssssssssss"),
    ("8b_32k_w32_norm", 32, 8, 128, BF, 32768, 2048, 32, True, "ssssssssssssssssssssssssssssssb"),
    ("8b_32k_w32_raw", 32, 8, 128, BF, 32768, 2048, 32, False, "ssssssssssssssssssssssssssssssb"),
    ("8b_131k_fp16_nan", 32, 8, 128, FP, 131072, 8192, 32, True, "swssssbsssssssssssssssssssssssss"),
]


@pytest.mark.gpu
@pytest.mark.parametrize("name,Hq,Hkv,D,dtype,S,B,W,normalize,kinds", ADAKV_E2E, ids=[x[0] for x in ADAKV_E2E])
def test_adakv_end_to_end(oracle, libpkv, name, Hq, Hkv, D, dtype, S, B, W, normalize, kinds):
    from oracle import torch_chain as tc
    from pyramidkv_b200 import kv_cluster as kc, ops
    q, k, v = build_heads(kinds, Hq, Hkv, S, D, W, dtype, seed=S + W)
    qd, kd, vd = q.to(dev()), k.to(dev()), v.to(dev())
    base = B - W
    cl = kc.AdaKVCluster(window_size=W, kernel_size=7, pooling="maxpool", max_capacity_prompt=B, floor=0.2, normalize=normalize,
                         layer_idx=0, num_hidden_layers=1)
    handle = cl.backend.ragged_begin(qd, kd, vd, W, 7, "maxpool")
    pooled_dev = ops.ws_pooled(handle["plan"]).contiguous()
    pooled = pooled_dev.cpu()
    r = oracle_counts(oracle, pooled, base, normalize)
    got = regimes(pooled, base, normalize, r)
    assert "cap_over_16384" in got, f"{name}: largest budget {max(r.caps)}"
    if dtype == FP:
        assert "nan_ratio" in got and "count_eq_n" in got, f"{name}: {sorted(got)}"
    k_buf, v_buf, rows = cl.evict_ragged(qd, kd, vd, reserve=3)
    torch.cuda.synchronize()
    assert cl.last_capacities == r.caps
    print(f"PKV_MEASURED {name}: largest budget {max(r.caps)}, smallest {min(r.caps)}, regimes {sorted(got)}")
    _check_rows(oracle, k_buf, v_buf, rows, k, v, pooled, r.caps, W)
    assert k_buf.shape[1] == max(rows) + 3
    del k_buf, v_buf
    # update_kv against torch_chain on the same device, on the GPU's own pooled scores (the chain's ratio may differ by 1 ulp:
    # then its budgets are not the library's, and the gather is checked with the library's budgets)
    G = Hq // Hkv
    K, V = tc.repeat_kv(kd[None], G), tc.repeat_kv(vd[None], G)
    caps_t, idx_t = tc.adakv_capacities(pooled_dev[None], base, 0.2, normalize, tie_rule="lowest_index")
    if caps_t.tolist() != r.caps:
        print(f"PKV_MEASURED {name}: torch_chain budgets differ on heads "
              f"{[h for h in range(Hq) if int(caps_t[h]) != r.caps[h]]} (its ratio is torch's .sum())")
    kf_t, vf_t, lens_t = tc.ragged_gather(K, V, idx_t, r.caps, W)
    kf, vf = cl.update_kv(kd[None], qd[:, :1].expand(Hq, S, D).contiguous()[None], vd[None])
    assert cl.head_lens.tolist() == lens_t
    assert cl.cu_klen.tolist() == [0] + torch.tensor(lens_t).cumsum(0).tolist()
    assert torch.equal(kf.view(torch.int16), kf_t.view(torch.int16)) and torch.equal(vf.view(torch.int16), vf_t.view(torch.int16))


@pytest.mark.gpu
def test_headkv_end_to_end_and_launches(oracle, libpkv):
    """HeadKV at 100 003 tokens with budgets 0, 1, 16 384, 16 385, 26 000 (6 000 of them tied zeros, taken in index order)
    and one above n (clamped to n). With every budget at most 16 384 the select + gather path launches exactly what the
    select, the gather and the window placement launch; above it, the sort path adds no library launch."""
    from pyramidkv_b200 import _lib, kv_cluster as kc, ops
    Hq, Hkv, D, W, S, dtype = 32, 8, 128, 32, 100003, BF
    n = S - W
    row = [0, 1, 16384, 16385, 26000, 200000] + [100 + 37 * h for h in range(6, Hq)]
    q, k, v = build_heads("sssbpb" + "s" * 26, Hq, Hkv, S, D, W, dtype, seed=3)
    qd, kd, vd = q.to(dev()), k.to(dev()), v.to(dev())
    cl = kc.HeadKVCluster(window_size=W, kernel_size=7, pooling="maxpool", max_capacity_prompt=2048, layer_idx=0,
                          num_hidden_layers=1, head_capacity=[row])
    k_buf, v_buf, rows = cl.evict_ragged(qd, kd, vd, reserve=3)
    torch.cuda.synchronize()
    caps = [min(c, n) for c in row]
    assert cl.last_capacities == caps
    handle = cl.backend.ragged_begin(qd, kd, vd, W, 7, "maxpool")
    pooled = ops.ws_pooled(handle["plan"]).cpu().contiguous()
    nz = int((pooled[4].float() != 0).sum())
    assert nz < 26000 < n, f"head 4: {nz} non-zero scores, the zero ties are not reached"
    _check_rows(oracle, k_buf, v_buf, rows, k, v, pooled, caps, W)
    del k_buf, v_buf
    # launches: budgets at most 16 384
    small = [min(c, SELECT_MAX_K) for c in caps]
    kmax = max(small)
    kb = torch.empty(Hq, kmax + W, D, dtype=dtype, device=dev())
    plan = ops.plan_evict("snapkv", qd, kd, vd, W, kmax, kb, torch.empty_like(kb), 7, "maxpool",
                          workspace=handle["ws"], window_mean=True)
    n0 = _lib.launch_count()
    ops.run_stage(plan, "topk")
    ops.run_stage(plan, "gather")
    expect = _lib.launch_count() - n0 + 1
    for cs in (small, caps):
        n0 = _lib.launch_count()
        kb2, _ = cl.backend.ragged_finish(handle, cs, 0)
        assert _lib.launch_count() - n0 == expect, f"{_lib.launch_count() - n0} library launches, expected {expect}"
        assert kb2.shape == (Hq, max(cs) + W, D)
        del kb2
    torch.cuda.synchronize()


# ---------------------------------------------------------------------------------------------------------------------------
# GPU: decode and the E4M3 conversion over the skewed cache
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_decode_and_fp8_on_skewed_cache(oracle, libpkv):
    """Per-head rows from 1 040 to 26 040 in one launch: decode steps in the host-length and the graph-replayed form, each
    head's output within the fp64 bound of test_gpu_landscapes and its new row appended at its own position; then
    `cache_quantize_fp8` with device row counts, bit-equal to the rule per head and nothing written past a head's rows."""
    from oracle_fp8_backend import quantize_rows
    from test_gpu_landscapes import _bound, _exact_attn
    from pyramidkv_b200 import ops
    Hq, Hkv, D, dtype, steps = 32, 8, 128, BF, 4
    G = Hq // Hkv
    head_rows = [1040 + 806 * ((h * 7) % Hq) for h in range(Hq)]
    assert min(head_rows) == 1040 and max(head_rows) == 1040 + 806 * 31
    cap = max(head_rows) + 2 * steps + 1
    g = torch.Generator().manual_seed(11)
    k0 = (torch.randn(Hq, cap, D, generator=g) * 0.8).to(dtype)
    v0 = torch.randn(Hq, cap, D, generator=g).to(dtype)
    hr = torch.tensor(head_rows, dtype=torch.int32, device=dev())
    news = [((torch.randn(Hq, D, generator=g) * 0.8).to(dtype), (torch.randn(Hkv, D, generator=g) * 0.8).to(dtype),
             torch.randn(Hkv, D, generator=g).to(dtype)) for _ in range(steps)]
    ke, ve = k0.to(dev()), v0.to(dev())
    kg, vg = k0.to(dev()), v0.to(dev())
    sq, skn, svn = (torch.zeros_like(t.to(dev())) for t in news[0])
    step = torch.zeros(1, dtype=torch.int32, device=dev())
    ws = torch.empty(ops.decode_workspace_bytes(Hq, D), dtype=torch.uint8, device=dev())
    out_g = torch.empty(Hq, D, dtype=dtype, device=dev())
    ops.decode_attn(sq, kg.clone(), vg.clone(), 1, skn, svn, out=out_g, head_rows=hr, step=step, max_length=cap, workspace=ws)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        ops.decode_attn(sq, kg, vg, 1, skn, svn, out=out_g, head_rows=hr, step=step, max_length=cap, workspace=ws)
    worst = 0.0
    for t, (qh, kn, vn) in enumerate(news):
        oe = ops.decode_attn(qh.to(dev()), ke, ve, t + 1, kn.to(dev()), vn.to(dev()), head_rows=hr, max_length=cap)
        sq.copy_(qh.to(dev()))
        skn.copy_(kn.to(dev()))
        svn.copy_(vn.to(dev()))
        step.fill_(t)
        graph.replay()
        torch.cuda.synchronize()
        oe, og = oe.cpu(), out_g.cpu()
        for h in range(Hq):
            T = head_rows[h] + t + 1
            for kc_, vc_ in ((ke, ve), (kg, vg)):
                assert torch.equal(kc_[h, T - 1].cpu(), kn[h // G]) and torch.equal(vc_[h, T - 1].cpu(), vn[h // G]), (t, h)
                assert bool((kc_[h, T].cpu() == k0[h, T]).all()), f"step {t} head {h}: wrote past its row"
            kk, vv = ke[h:h + 1, :T].float(), ve[h:h + 1, :T].float()
            ref, s_max, A = _exact_attn(qh[h:h + 1].to(dev()).float(), kk, vv)
            ref = ref.cpu()
            vmax = float(vv.abs().max())
            bound, eps = _bound(ref, dtype, D, cap, Hq, s_max, A, False, vmax)
            for o, form in ((oe, "host length"), (og, "graph")):
                err = (o[h:h + 1].double() - ref).abs()
                worst = max(worst, float((err / bound).max()))
                assert bool((err <= bound).all()), f"{form} step {t} head {h} ({T} rows): error beyond the bound"
    print(f"PKV_MEASURED skewed decode: largest error / bound {worst:.3g}")
    # E4M3 conversion with device row counts (the rows the prompt left, before the appended ones)
    sentinel_b, sentinel_s = 0x55, -1.0
    kq = torch.full((1, Hq, cap, D), sentinel_b, dtype=torch.uint8, device=dev()).view(torch.float8_e4m3fn)
    vq = torch.full_like(kq.view(torch.uint8), sentinel_b).view(torch.float8_e4m3fn)
    ks = torch.full((1, Hq, cap), sentinel_s, device=dev())
    vs = torch.full_like(ks, sentinel_s)
    ops.cache_quantize_fp8([(ke[None].contiguous(), ve[None].contiguous(), kq, vq, ks, vs, max(head_rows), hr)])
    torch.cuda.synchronize()
    kqc, vqc, ksc, vsc = kq.view(torch.uint8).cpu()[0], vq.view(torch.uint8).cpu()[0], ks.cpu()[0], vs.cpu()[0]
    kec, vec = ke.cpu(), ve.cpu()
    for h in range(Hq):
        nrow = head_rows[h]
        for src, qq, ss in ((kec, kqc, ksc), (vec, vqc, vsc)):
            wq, wsc = quantize_rows(src[h, :nrow])
            assert torch.equal(qq[h, :nrow], wq.view(torch.uint8)) and torch.equal(ss[h, :nrow], wsc), f"head {h}"
            assert bool((qq[h, nrow:] == sentinel_b).all()) and bool((ss[h, nrow:] == sentinel_s).all()), f"head {h}: wrote past"
