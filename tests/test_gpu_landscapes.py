"""-m gpu: the eviction and decode kernels on the attention landscapes of tests/attention_landscapes.py (sinks, late heavy
hitters, near one-hot rows, bf16-subnormal probabilities, outlier channels, repeated keys, fp16 masks that round to -inf).

Eviction bars, on every path (staged mma.sync and wgmma scorers, PKV_FLAG_FUSED (fused stages 1-2 + select kernel),
PKV_FLAG_SINGLE_LAUNCH, the layer batch, PKV_FLAG_GQA_SHARED, H2O on both kernels, AdaKV window mean, L2Norm). The two fused
paths skip the shapes the fused kernels do not take:
- Stage 1 (staged runs): the mask pattern and the masked values equal the oracle's, -inf versus finfo.min included. On
  exact-dot landscapes every logit is bit-identical; elsewhere the existing 2-ulp class (gpu_util.ulp_diff).
- Stage 2: against the oracle run on the GPU's own logits (softmax_rows -> window_sum -> pool), which takes stage-1 rounding
  flips out of the comparison. Every element within 2 ulp of its own magnitude (subnormal ulps below the smallest normal;
  no floor relative to the row's maximum, so a subnormal compared with 0 is a miss), and zero exactly where the oracle's is
  zero, except where the oracle's value is below 4x the dtype's smallest subnormal. Paths that keep no logits (fused,
  single launch, batch, GQA-shared, H2O) meet the same bars against the oracle on exact-dot inputs, and their pooled scores
  meet them against the staged path's.
- Stage 3: the indices equal oracle.topk(GPU pooled, lowest index); on exact-dot landscapes also oracle.evict's indices,
  set and order, on every head.
- Stage 4: the gathered rows are byte copies; the slack rows are untouched (gpu_evict), the fused status word reads 0.

Decode bar. The reference is fp64 softmax attention over the rows the cache holds (dequantised for E4M3). With u = 2^-24,
the kernel's fp32 arithmetic gives, per output element,
    |out - exact| <= ulp_out(|exact|) + eps * max|v|,
    eps = u * (2 (D + 2) A + 4 s_max + 2 (n_lane + n_split + 16)),
where
- A = scale * max_j sum_e |q_e k_je| bounds the dot product's fp32 error, (D + 2) u A. It is 0 for exact-dot keys, whose
  single non-zero product is exact.
- 4 u s_max covers the rounding of s = dot * scale and of s - m before expf (2 ulp), through which every weight's relative
  error enters the output twice (numerator and denominator).
- 2 u (n_lane + n_split + 16) covers the fp32 accumulation: each lane folds n_lane rows with one rounding each, then
  log2 of the row groups, 8 warps and n_split split partials are merged.
The sink, heavy-hitter and outlier-channel K and V (V outliers up to 100) run through every decode entry point at
T in {1, 256, 257, 2056, 32768, 131072}, with the large row in the first split, the last split and on a split boundary.
"""
import math
import os
import subprocess
import sys

import pytest
import torch

from attention_landscapes import assert_stage2, build, ulp_own
from gpu_util import dev, gpu_evict, hf_layout, ulp_diff

pytestmark = pytest.mark.gpu

BF, FP = torch.bfloat16, torch.float16
# (landscape, Hq, Hkv, S, D, W, dtype, kernel, pooling, budget): budget None = n // 8
EVICT = [
    ("sink", 32, 8, 4096, 128, 8, BF, 7, "maxpool", None),
    ("heavy", 32, 8, 4096, 128, 8, BF, 7, "maxpool", None),
    ("peaked", 32, 8, 4096, 128, 8, BF, 7, "maxpool", 64),           # below the non-zero count
    ("peaked", 32, 8, 4096, 128, 8, BF, 7, "maxpool", 1024),         # above it: thousands of zeros tie
    ("subnormal", 32, 8, 4096, 128, 8, BF, 7, "maxpool", "band"),
    ("repeated", 32, 8, 4096, 128, 8, BF, 5, "avgpool", None),
    ("outlier", 32, 8, 4096, 128, 8, BF, 7, "maxpool", None),
    ("heavy", 16, 2, 3000, 128, 8, BF, 5, "avgpool", None),          # G = 8 (the wgmma scorer takes G * W in {32, 64})
    ("subnormal", 16, 2, 3000, 128, 8, BF, 7, "maxpool", "band"),
    ("repeated", 16, 2, 3000, 128, 8, BF, 7, "maxpool", None),
    ("peaked", 16, 2, 3000, 128, 8, BF, 7, "maxpool", 512),
    ("subnormal", 16, 4, 3000, 128, 16, BF, 7, "maxpool", "band"),   # W = 16
    ("subnormal", 8, 4, 1500, 128, 32, BF, 7, "maxpool", "band"),    # W = 32
    ("fp16mask", 8, 4, 2000, 64, 32, FP, 7, "maxpool", None),        # D = 64, fp16
    ("fp16mask", 8, 2, 2000, 64, 8, FP, 5, "avgpool", None),
    ("outlier", 8, 2, 2000, 64, 16, FP, 7, "maxpool", None),
    ("sink", 8, 2, 2000, 64, 16, FP, 7, "maxpool", None),
    ("peaked", 8, 4, 2000, 64, 32, FP, 5, "avgpool", 600),
    ("repeated", 8, 2, 2000, 64, 8, FP, 7, "maxpool", None),
]
BIG = [("repeated", 8, 2, 32760, 128, 8, BF, 7, "maxpool", 2048),   # the cluster forms of the select
       ("repeated", 4, 1, 72000, 128, 8, BF, 7, "maxpool", 2048)]
PATHS = ["mma", "tc5", "fused", "single"]


def _top_k(L, budget):
    n = L.q.shape[1] - L.W
    if budget == "band":
        return min(n, L.info["normal"] + 64)
    return min(n, budget if budget is not None else n // 8)


_cache = {}


def _landscape(oracle, name, Hq, Hkv, S, D, W, dtype, kernel, pooling):
    key = (name, Hq, Hkv, S, D, W, dtype, kernel, pooling)
    if key not in _cache:
        _cache.clear()
        L = build(name, Hq, Hkv, S, D, W, dtype, seed=S + Hq + W)
        L.check(oracle) if name != "subnormal" else L.check(oracle, kernel=kernel, pooling=pooling)
        _cache[key] = L
    return _cache[key]


def _oracle_ref(oracle, L, top_k, kernel, pooling):
    k = ("ref", top_k, kernel, pooling)
    if k not in L.info:
        L.info[k] = oracle.evict("snapkv", L.q, L.k, L.v, L.W, top_k, kernel, pooling)
    return L.info[k]


def _check_logits(gl, ol, exact, dtype):
    gf, of = gl.float(), ol.float()
    assert torch.equal(torch.isneginf(gf), torch.isneginf(of)), "-inf pattern differs"
    fmin = torch.finfo(dtype).min
    assert torch.equal(gf == fmin, of == fmin), "finfo.min pattern differs"
    if exact:
        assert torch.equal(gl.view(torch.int16), ol.view(torch.int16)), "exact-dot logits differ from the oracle"
    else:
        fin = torch.isfinite(of) & (of > -1e30)
        assert ulp_diff(gl[fin], ol[fin]) <= 2      # the existing class: a dot product that cancels carries absolute error


def _run_path(oracle, L, path, top_k, kernel, pooling):
    q, k, v, W = L.q, L.k, L.v, L.W
    dtype = q.dtype
    if path in ("mma", "tc5"):
        r = gpu_evict("snapkv", q, k, v, W, top_k, kernel, pooling, score_kernel="mma" if path == "mma" else "tcgen05")
        _check_logits(r.logits, oracle.window_logits(q, k, W), L.exact, dtype)
        own = oracle.pool(oracle.window_sum(oracle.softmax_rows(r.logits.contiguous())), kernel, pooling)
        assert_stage2(r.pooled, own, f"{path}: pooled vs the oracle on the GPU's logits")
    else:
        r = gpu_evict("snapkv", q, k, v, W, top_k, kernel, pooling, score_kernel="tcgen05", staged=False,
                      single_launch=(path == "single"), fused=(path == "fused"))
        if r.single_launch == 0:
            pytest.skip("the fused kernels do not take this shape (it runs as staged launches)")
        assert r.single_launch == (2 if path == "single" else 1)
        st = gpu_evict("snapkv", q, k, v, W, top_k, kernel, pooling, score_kernel="tcgen05")
        assert_stage2(r.pooled, st.pooled, f"{path}: pooled vs the staged path's")
    if L.exact:
        ref = _oracle_ref(oracle, L, top_k, kernel, pooling)
        assert_stage2(r.pooled, ref.pooled, f"{path}: pooled vs the oracle (exact-dot)")
    return r


def _check_select_gather(oracle, L, r, top_k, kernel, pooling):
    assert torch.equal(r.idx, oracle.topk(r.pooled, top_k, oracle.TIE_LOWEST_INDEX)), "indices differ from topk(own pooled)"
    if L.exact:
        ref = _oracle_ref(oracle, L, top_k, kernel, pooling)
        bad = [h for h in range(r.idx.shape[0]) if not torch.equal(r.idx[h], ref.idx[h])]
        assert not bad, f"indices differ from oracle.evict on heads {bad[:8]}"
    Hq = L.q.shape[0]
    assert torch.equal(r.k_cache.view(torch.int16), oracle.gather(L.k, r.idx, L.W, Hq).view(torch.int16))
    assert torch.equal(r.v_cache.view(torch.int16), oracle.gather(L.v, r.idx, L.W, Hq).view(torch.int16))


@pytest.mark.parametrize("path", PATHS)
@pytest.mark.parametrize("name,Hq,Hkv,S,D,W,dtype,kernel,pooling,budget", EVICT)
def test_evict_paths(oracle, libpkv, name, Hq, Hkv, S, D, W, dtype, kernel, pooling, budget, path):
    L = _landscape(oracle, name, Hq, Hkv, S, D, W, dtype, kernel, pooling)
    top_k = _top_k(L, budget)
    r = _run_path(oracle, L, path, top_k, kernel, pooling)
    _check_select_gather(oracle, L, r, top_k, kernel, pooling)


@pytest.mark.parametrize("path", ["tc5", "fused"])
@pytest.mark.parametrize("name,Hq,Hkv,S,D,W,dtype,kernel,pooling,budget", BIG)
def test_evict_long_repeated_keys(oracle, libpkv, name, Hq, Hkv, S, D, W, dtype, kernel, pooling, budget, path):
    """Runs of identical keys across the per-CTA ranges and the cluster ranks of the select, at 32760 and 72000 tokens."""
    L = _landscape(oracle, name, Hq, Hkv, S, D, W, dtype, kernel, pooling)
    top_k = min(budget, L.info["tied"] // 2)          # the threshold falls inside the runs
    r = _run_path(oracle, L, path, top_k, kernel, pooling)
    _check_select_gather(oracle, L, r, top_k, kernel, pooling)


# ---------------- the layer batch ----------------
@pytest.mark.parametrize("names,Hq,Hkv,S,D,W,budget", [
    (("subnormal", "peaked", "repeated"), 32, 8, 4096, 128, 8, 256),
    (("heavy", "peaked"), 16, 2, 3000, 128, 8, 512),
    (("subnormal", "peaked", "repeated") * 11, 8, 2, 1000, 128, 8, 128),     # 33 layers: the left-over layer
])
def test_layer_batch(oracle, libpkv, names, Hq, Hkv, S, D, W, budget):
    from pyramidkv_b200 import ops
    layers = [build(nm, Hq, Hkv, S, D, W, BF, seed=100 + i) for i, nm in enumerate(names)]
    Lc = len(layers)
    ks = [ops.layer_budget("pyramidkv", budget, W, Lc, l, S)[1] for l in range(Lc)]
    plans, bufs, wss = [], [], None
    for l, L in enumerate(layers):
        qd, kd, vd = hf_layout(L.q[:, S - W:].contiguous()), hf_layout(L.k), hf_layout(L.v)
        kc = torch.full((Hq, ks[l] + W + 2, D), 7.0, dtype=BF, device=dev())
        vc = torch.full_like(kc, 7.0)
        idx = torch.full((Hq, ks[l]), -1, dtype=torch.int64, device=dev())
        if wss is None:
            wss = ops.batch_workspaces(ops.plan_evict("pyramidkv", qd, kd, vd, W, ks[l], kc, vc, 7, "maxpool", idx_out=idx), Lc, max(ks))
        plans.append(ops.plan_evict("pyramidkv", qd, kd, vd, W, ks[l], kc, vc, 7, "maxpool", idx_out=idx, workspace=wss[l]))
        bufs.append((kc, vc, idx))
    assert ops.batch_supported(plans)
    ops.evict_prefill_batch(plans)
    torch.cuda.synchronize()
    for l, (L, p, (kc, vc, idx)) in enumerate(zip(layers, plans, bufs)):
        pooled = ops.ws_pooled(p).cpu().contiguous()
        ref = oracle.evict("snapkv", L.q, L.k, L.v, W, ks[l], 7, "maxpool")
        assert_stage2(pooled, ref.pooled, f"layer {l} ({L.name}): pooled vs the oracle")
        ic = idx.cpu()
        assert torch.equal(ic, oracle.topk(pooled, ks[l])), f"layer {l}: indices vs topk(own pooled)"
        assert torch.equal(ic, ref.idx), f"layer {l}: indices vs oracle.evict"
        assert torch.equal(kc[:, :ks[l] + W].cpu().view(torch.int16), oracle.gather(L.k, ic, W, Hq).view(torch.int16))
        assert bool((kc[:, ks[l] + W:] == 7.0).all()) and bool((vc[:, ks[l] + W:] == 7.0).all())


# ---------------- GQA-shared selection ----------------
@pytest.mark.parametrize("name,Hq,Hkv,S,D,W,dtype,budget", [
    ("subnormal", 32, 8, 4096, 128, 8, BF, 256), ("peaked", 32, 8, 4096, 128, 8, BF, 1024),
    ("repeated", 16, 2, 3000, 128, 16, BF, 128), ("fp16mask", 8, 2, 2000, 64, 32, FP, 200)])
def test_gqa_shared(oracle, libpkv, name, Hq, Hkv, S, D, W, dtype, budget):
    from oracle_gqa_backend import group_reduce
    from pyramidkv_b200 import ops
    L = build(name, Hq, Hkv, S, D, W, dtype, seed=S + 1)
    G = Hq // Hkv
    kc = torch.full((Hkv, budget + W + 3, D), 7.0, dtype=dtype, device=dev())
    vc = torch.full_like(kc, 7.0)
    idx = torch.full((Hkv, budget), -1, dtype=torch.int64, device=dev())
    plan = ops.plan_evict("snapkv", hf_layout(L.q), hf_layout(L.k), hf_layout(L.v), W, budget, kc, vc, 7, "maxpool",
                          idx_out=idx, gqa_shared=True)
    ops.run_stage(plan, "all")
    torch.cuda.synchronize()
    pooled = ops.ws_pooled(plan).cpu().contiguous()
    s_kv = ops.ws_pooled_kv(plan).cpu().contiguous()
    ref = oracle.evict("snapkv", L.q, L.k, L.v, W, budget, 7, "maxpool")
    assert_stage2(pooled, ref.pooled, "pooled vs the oracle")
    assert torch.equal(s_kv.view(torch.int16), group_reduce(pooled, G).view(torch.int16))
    ic = idx.cpu()
    assert torch.equal(ic, oracle.topk(s_kv, budget))
    assert torch.equal(ic, oracle.topk(group_reduce(ref.pooled, G), budget))
    assert torch.equal(kc[:, :budget + W].cpu().view(torch.int16), oracle.gather(L.k, ic, W, Hkv).view(torch.int16))
    assert bool((kc[:, budget + W:] == 7.0).all())


# ---------------- H2O on both kernels ----------------
_H2O_CHILD = r"""
import sys, torch
sys.path.insert(0, "tests")
from attention_landscapes import build
from gpu_util import gpu_evict
out = {}
for (name, Hq, Hkv, S, D, W, k, dt) in [("subnormal", 8, 2, 2000, 128, 8, 200, torch.bfloat16),
                                        ("peaked", 32, 8, 2048, 128, 8, 300, torch.bfloat16),
                                        ("fp16mask", 4, 2, 1030, 64, 16, 64, torch.float16)]:
    L = build(name, Hq, Hkv, S, D, W, dt, seed=S)
    r = gpu_evict("h2o", L.q, L.k, L.v, W, k)
    out[(name, Hq, Hkv, S, D, W, k, str(dt))] = (r.pooled, r.idx, r.k_cache)
torch.save(out, sys.argv[1])
"""


def test_h2o_both_kernels(oracle, libpkv, tmp_path):
    """Exact-dot logits: both kernels' column sums within 4 ulp of their own magnitude of the oracle's (S terms summed in
    another order), zero exactly where the oracle's is, and the selection exact on each kernel's own scores."""
    res = {}
    for name in ("mma", "tc5"):
        path = tmp_path / f"{name}.pt"
        subprocess.run([sys.executable, "-c", _H2O_CHILD, str(path)], check=True, timeout=300,
                       env={**os.environ, "PKV_H2O": name}, cwd=os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
        res[name] = torch.load(path, weights_only=False)
    for kern, out in res.items():
        for key, (pooled, idx, kc) in out.items():
            name, Hq, Hkv, S, D, W, k, dts = key
            dt = BF if "bfloat16" in dts else FP
            L = build(name, Hq, Hkv, S, D, W, dt, seed=S)
            ref = oracle.h2o_scores(L.q, L.k, W)
            assert_stage2(pooled, ref, f"h2o {kern} {key}", max_ulp=4)
            assert torch.equal(oracle.topk(pooled.contiguous(), k, oracle.TIE_LOWEST_INDEX), idx), f"h2o {kern} {key}"


# ---------------- AdaKV / HeadKV window mean ----------------
@pytest.mark.parametrize("name,Hq,Hkv,S,D,W,B", [("peaked", 8, 2, 1024, 128, 8, 128), ("peaked", 32, 8, 4096, 128, 32, 512),
                                                 ("subnormal", 8, 2, 2000, 128, 8, 256)])
def test_adakv_window_mean_and_counts(oracle, libpkv, name, Hq, Hkv, S, D, W, B):
    """Mean-pooled scores vs the oracle's (exact-dot); threshold counts at zero ties across heads; the ragged rows."""
    from pyramidkv_b200 import kv_cluster as kc
    L = build(name, Hq, Hkv, S, D, W, BF, seed=S + B)
    qd, kd, vd = hf_layout(L.q), hf_layout(L.k), hf_layout(L.v)
    be = kc.CudaBackend()
    handle = be.ragged_begin(qd[:, S - W:, :], kd, vd, W, 7, "maxpool")
    from pyramidkv_b200 import ops
    pooled = ops.ws_pooled(handle["plan"]).cpu().contiguous()
    assert_stage2(pooled, oracle.adakv_scores(L.q, L.k, W, 7, "maxpool"), "window-mean pooled vs the oracle")
    base = B - W
    for normalize in (True, False):
        gt, eq = be.adakv_counts(handle, base, normalize)
        caps_o, gt_o, eq_o, thr, _ = oracle.adakv_capacities(pooled, base, 0.2, normalize, details=True)
        assert gt == gt_o.tolist() and eq == eq_o.tolist()
    c = kc.AdaKVCluster(window_size=W, kernel_size=7, pooling="maxpool", max_capacity_prompt=B, floor=0.2, normalize=True,
                        layer_idx=0, num_hidden_layers=4)
    k_buf, v_buf, rows = c.evict_ragged(qd, kd, vd, reserve=3)
    torch.cuda.synchronize()
    ks, vs, _ = oracle.ragged_evict(L.k, L.v, pooled, c.last_capacities, W)
    for h in range(Hq):
        assert torch.equal(k_buf[h, :rows[h]].cpu(), ks[h]) and torch.equal(v_buf[h, :rows[h]].cpu(), vs[h]), f"head {h}"


# ---------------- L2Norm on outlier keys ----------------
@pytest.mark.parametrize("dtype", [BF, FP])
def test_l2norm_outlier_keys(oracle, libpkv, dtype):
    from pyramidkv_b200 import ops
    Hq, Hkv, S, D, B = 32, 8, 4096, 128, 512
    if dtype == FP:
        Hq, Hkv, D = 8, 2, 64
    L = build("outlier", Hq, Hkv, S, D, 8, dtype, seed=9)
    kc = torch.full((Hq, B + 3, D), 7.0, dtype=dtype, device=dev())
    vc = torch.full_like(kc, 7.0)
    idx = torch.full((Hq, B), -1, dtype=torch.int64, device=dev())
    plan = ops.plan_evict("l2norm", None, hf_layout(L.k), hf_layout(L.v), 0, B, kc, vc, idx_out=idx)
    ops.run_stage(plan, "all")
    torch.cuda.synchronize()
    keys = ops.ws_pooled(plan).cpu().contiguous()
    want = (-oracle.key_norms(L.k).float()).to(dtype).repeat_interleave(Hq // Hkv, dim=0)
    assert float(ulp_own(keys, want, dtype).max()) <= 1, "key norms beyond 1 ulp"
    ic = idx.cpu()
    assert torch.equal(ic, oracle.topk(keys, B))
    assert torch.equal(kc[:, :B].cpu().view(torch.int16), oracle.gather(L.k, ic, 0, Hq).view(torch.int16))


# ---------------- decode ----------------
U = 2.0 ** -24


def _splits(Hq, T):
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    ns = min(max((T + 255) // 256, 1), (sms * 4 + Hq - 1) // Hq, 64)
    return max(ns, 1)


def _decode_rows(kind, H, T, D, dtype, pos, seed):
    """K [H, T, D], V [H, T, D] and q [H, D]: 'sink' / 'heavy' are exact-dot keys (one non-zero dim) with one row
    `gap` above the rest at `pos`; 'outlier' has 4 massive channels in K. V carries outliers up to 100."""
    g = torch.Generator().manual_seed(seed)
    q = (torch.randn(H, D, generator=g) * 0.8)
    v = torch.randn(H, T, D, generator=g)
    v[:, torch.randperm(T, generator=g)[:max(1, T // 64)], 3] = 100.0
    v[:, pos, :8] = -100.0
    if kind == "outlier":
        k = torch.randn(H, T, D, generator=g) * 0.8
        dims = [5, 17, 64, D - 1]
        for d in dims:
            q[:, d] = 2.0
            k[:, :, d] = 30 + 70 * torch.rand(H, T, generator=g)
        exact = False
    else:
        q[:, 0] = 4.0
        k = torch.zeros(H, T, D)
        k[:, :, 0] = torch.randint(-4, 5, (H, T), generator=g).float()
        k[:, pos, 0] = 4.0 + (30.0 if kind == "sink" else 60.0) * math.sqrt(D) / 4.0
        exact = True
    return q.to(dtype), k.to(dtype), v.to(dtype), exact


def _exact_attn(q, k, v):
    """fp64 softmax attention: q [H, D], k / v [H, T, D] (float) -> [H, D]; also s_max and A."""
    D = q.shape[-1]
    s = torch.einsum("hd,htd->ht", q.double(), k.double()) / math.sqrt(D)
    A = (torch.einsum("hd,htd->ht", q.double().abs(), k.double().abs()) / math.sqrt(D)).max()
    p = torch.softmax(s, dim=-1)
    return torch.einsum("ht,htd->hd", p, v.double()), float(s.abs().max()), float(A)


def _bound(exact_out, dtype, D, T, Hq, s_max, A, exact, vmax, E=8):
    ns = _splits(Hq, T)
    chunk = -(-T // ns)
    rpw = 32 // (D // E)
    n_lane = -(-chunk // (rpw * 8))
    eps = U * ((0 if exact else 2 * (D + 2) * A) + 4 * s_max + 2 * (n_lane + ns + 16))
    mant = 8 if dtype == BF else 11
    ulp = torch.exp2(torch.floor(torch.log2(exact_out.abs().clamp(min=1e-30))) - (mant - 1))
    return ulp + eps * vmax, eps


_measured = []


def _check_decode(out, ref, dtype, D, T, Hq, s_max, A, exact, vmax, what, E=8):
    bound, eps = _bound(ref, dtype, D, T, Hq, s_max, A, exact, vmax, E)
    err = (out.double().cpu() - ref).abs()
    worst = float(((err - (bound - eps * vmax)).clamp(min=0)).max() / vmax)
    _measured.append((what, worst, eps))
    print(f"decode {what}: max (|err| - 1 ulp) / max|v| = {worst:.3g}, derived eps = {eps:.3g}")
    assert bool((err <= bound).all()), f"{what}: error beyond 1 ulp + {eps:.3g} * max|v| (measured {worst:.3g})"


def _positions(Hq, T):
    ns = _splits(Hq, T)
    chunk = -(-T // ns)
    return sorted({0, min(T - 1, (ns - 1) * chunk + 1), min(T - 1, chunk)})      # first split, last split, on a boundary


DECODE_T = [1, 256, 257, 2056, 32768, 131072]


@pytest.mark.parametrize("kind", ["sink", "heavy", "outlier"])
@pytest.mark.parametrize("T", DECODE_T)
def test_decode_attn_landscapes(oracle, libpkv, kind, T):
    """pkv_decode_attn, the batched launch with ragged rows, the GQA-shared launch (G = 2, 4, 8) and the E4M3 forms."""
    from oracle_fp8_backend import dequantize, quantize_rows
    from pyramidkv_b200 import ops
    Hkv, D, dtype = 2, 128, BF
    for G in ((2, 4, 8) if T <= 2056 else (4,)):
        Hq = Hkv * G
        positions = _positions(Hq, T)
        if T >= 32768:
            positions = positions[-1:] if kind != "sink" else positions[:1]     # a few cases at the largest shapes
        for pos in positions:
            qh, kk, vv, exact = _decode_rows(kind, Hkv, T, D, dtype, pos, seed=T + pos + G)
            q = qh.repeat_interleave(G, dim=0)
            k_rep, v_rep = kk.repeat_interleave(G, dim=0), vv.repeat_interleave(G, dim=0)
            ref, s_max, A = _exact_attn(q, k_rep.float(), v_rep.float())
            vmax = float(vv.float().abs().max())
            tag = f"{kind} T={T} pos={pos} G={G}"
            # pkv_decode_attn (T rows, nothing appended)
            out = ops.decode_attn(q.to(dev()), k_rep.to(dev()), v_rep.to(dev()), T)
            _check_decode(out, ref, dtype, D, T, Hq, s_max, A, exact, vmax, "decode_attn " + tag)
            # batched: two sequences, the second with ragged rows (T // 2 + 1 rows on odd heads)
            kb = torch.stack([k_rep, k_rep]).to(dev())
            vb = torch.stack([v_rep, v_rep]).to(dev())
            rows = torch.full((2, Hq), T, dtype=torch.int32)
            rows[1, 1::2] = T // 2 + 1
            qb = torch.stack([q, q]).to(dev())
            ob = ops.decode_attn_batch(qb, kb, vb, 1, rows=(rows - 1).reshape(-1).contiguous().to(dev())).cpu()
            for b in range(2):
                for h in range(Hq):
                    n = int(rows[b, h])
                    if n == T:
                        r1, sm1, a1 = ref[h:h + 1], s_max, A
                    else:
                        r1, sm1, a1 = _exact_attn(q[h:h + 1], k_rep[h:h + 1, :n].float(), v_rep[h:h + 1, :n].float())
                    _check_decode(ob[b, h:h + 1], r1, dtype, D, n, Hq, sm1, a1, exact, vmax, f"batch b={b} h={h} " + tag)
            # GQA-shared: one cache per KV head
            og = ops.decode_attn_batch_gqa(q[None].to(dev()), kk[None].to(dev()), vv[None].to(dev()), T).cpu()[0]
            _check_decode(og, ref, dtype, D, T, Hq, s_max, A, exact, vmax, "gqa " + tag)
            # E4M3 rows: the reference attends the dequantised rows
            (kq, ks), (vq, vs) = quantize_rows(kk), quantize_rows(vv)
            kd_, vd_ = dequantize(kq, ks), dequantize(vq, vs)
            ref8, s8, A8 = _exact_attn(q, kd_.repeat_interleave(G, 0), vd_.repeat_interleave(G, 0))
            vmax8 = float(vd_.abs().max())
            rep8 = lambda t: t.view(torch.uint8).repeat_interleave(G, 0).view(torch.float8_e4m3fn)[None].to(dev())
            o8 = ops.decode_attn_batch_fp8(q[None].to(dev()), rep8(kq), rep8(vq), ks.repeat_interleave(G, 0)[None].to(dev()),
                                           vs.repeat_interleave(G, 0)[None].to(dev()), T).cpu()[0]
            _check_decode(o8, ref8, dtype, D, T, Hq, s8, A8, exact, vmax8, "fp8 " + tag, E=16)
            og8 = ops.decode_attn_batch_gqa_fp8(q[None].to(dev()), kq[None].to(dev()), vq[None].to(dev()), ks[None].to(dev()),
                                                vs[None].to(dev()), T).cpu()[0]
            _check_decode(og8, ref8, dtype, D, T, Hq, s8, A8, exact, vmax8, "gqa fp8 " + tag, E=16)


@pytest.mark.parametrize("kind", ["sink", "heavy", "outlier"])
def test_decode_window_after_wrap(oracle, libpkv, kind):
    """pkv_decode_attn_window: the prompt rows hold the large row; appended rows wrap the ring of R rows twice."""
    from pyramidkv_b200 import ops
    Hq, Hkv, D, P, R, steps, dtype = 8, 2, 128, 600, 5, 13, BF
    G = Hq // Hkv
    qh, kk, vv, exact = _decode_rows(kind, Hkv, P + steps, D, dtype, 300, seed=7)
    kr, vr = kk.repeat_interleave(G, 0), vv.repeat_interleave(G, 0)
    cap = P + R + 2
    kb = torch.zeros(1, Hq, cap, D, dtype=dtype)
    vb = torch.zeros_like(kb)
    kb[0, :, :P], vb[0, :, :P] = kr[:, :P], vr[:, :P]
    kb, vb = kb.to(dev()), vb.to(dev())
    prompt_rows = torch.full((Hq,), P, dtype=torch.int32, device=dev())
    step = torch.zeros(1, dtype=torch.int32, device=dev())
    q = qh.repeat_interleave(G, 0)
    vmax = float(vv.float().abs().max())
    for t in range(steps):
        step.fill_(t)
        out = ops.decode_attn_window(q[None].to(dev()), kb, vb, 1, kk[None, :, P + t].to(dev()), vv[None, :, P + t].to(dev()),
                                     prompt_rows, R, rows=prompt_rows, step=step, max_length=cap).cpu()[0]
        keep = list(range(P)) + list(range(P + max(0, t + 1 - R), P + t + 1))
        ref, s_max, A = _exact_attn(q, kr[:, keep].float(), vr[:, keep].float())
        _check_decode(out, ref, dtype, D, len(keep), Hq, s_max, A, exact, vmax, f"window {kind} t={t}")
