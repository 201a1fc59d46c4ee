"""Seeded prefill inputs shaped like real attention: sinks, late heavy hitters, near one-hot rows, bf16-subnormal
probabilities, massive-activation channels, runs of identical keys and fp16 masks that round to -inf.

`make_inputs` draws iid Gaussians, whose window logits are close to N(0, 1): a flat softmax in which no probability
underflows, no pooled row is mostly zeros, no tile's maximum stands out and no two scores tie. These builders reach the
code written for the other cases (the score kernels' moving reference, the clamps of the fast exp, the empty and -inf
softmax partials, the lowest-index tie rule across tiles, CTAs and cluster ranks).

`build(name, Hq, Hkv, S, D, W, dtype, seed)` returns a `Landscape`: CPU q [Hq, S, D] and k, v [Hkv, S, D], whether it is
exact-dot, and `check(oracle)`, which asserts through the oracle's own logits / probabilities / pooled scores that the
regime is really present (so that a later edit cannot quietly turn a landscape back into a Gaussian test).

Exact-dot landscapes: q has one non-zero dim (the same value c on every row), k one non-zero value x_j in the same dim.
The matmul then sums one exact product and zeros, so the fp32 accumulator holds c * x_j exactly in every kernel and in
the oracle, and every path's logits must equal the oracle's bit for bit. c ~ sqrt(D) makes the logit ~ x_j.
"""
from __future__ import annotations

import math
from dataclasses import dataclass
from typing import Callable

import torch

EXACT = ("heavy", "peaked", "subnormal", "repeated", "fp16mask")
NAMES = ("sink",) + EXACT + ("outlier",)
BF16_TINY = 2.0 ** -126        # smallest normal of bf16 (= fp32)


@dataclass
class Landscape:
    name: str
    q: torch.Tensor
    k: torch.Tensor
    v: torch.Tensor
    W: int
    exact: bool
    check: Callable
    info: dict


def _c(D, dtype):
    """The query value of the exact-dot landscapes: sqrt(D) rounded to the model dtype (D = 64: exactly 8)."""
    return float(torch.tensor(math.sqrt(D)).to(dtype).float())


def _exact(Hq, Hkv, S, D, dtype, x, seed):
    """q [Hq,S,D] = c in dim 0; k [Hkv,S,D] = x [Hkv,S] in dim 0; v Gaussian."""
    g = torch.Generator().manual_seed(seed + 7)
    q = torch.zeros(Hq, S, D)
    q[:, :, 0] = _c(D, dtype)
    k = torch.zeros(Hkv, S, D)
    k[:, :, 0] = x
    v = torch.randn(Hkv, S, D, generator=g)
    return q.to(dtype), k.to(dtype), v.to(dtype)


def _rows(oracle, L):
    """Oracle window logits [Hq, W, S] as fp32."""
    return oracle.window_logits(L.q, L.k, L.W).float()


def build(name, Hq, Hkv, S, D, W, dtype, seed=0, **kw) -> Landscape:
    g = torch.Generator().manual_seed(seed)
    n = S - W
    info = {}

    if name == "sink":
        # Gaussian q / k; tokens 0-3 sit `delta` above the background: one sink dim, q = 4 there, k = delta*sqrt(D)/4
        delta = kw.get("delta", 30.0)
        q = torch.randn(Hq, S, D, generator=g)
        k = torch.randn(Hkv, S, D, generator=g)
        v = torch.randn(Hkv, S, D, generator=g)
        q[:, :, D - 1] = 4.0
        k[:, :, D - 1] = 0.0
        k[:, :4, D - 1] = delta * math.sqrt(D) / 4.0
        q, k, v = q.to(dtype), k.to(dtype), v.to(dtype)
        info["delta"] = delta

        def check(oracle, L=None):
            lg = _rows(oracle, L)[:, :, :n]
            gap = lg[:, :, :4].min(-1).values - lg[:, :, 4:].median(-1).values
            assert float(gap.min()) >= delta - 8, "sink tokens do not stand out"
        exact = False

    elif name == "heavy":
        # integer background in [-8, 8]; one token in the last third of the prompt, past the first tile, sits `gap` above
        # everything before it: tiles scored earlier set the running reference, this one moves it (> kRefSlack = 40)
        gap = kw.get("gap", 60.0)
        x = torch.randint(-8, 9, (Hkv, S), generator=g).float()
        pos = torch.randint(max(2 * n // 3, 129), n, (Hkv,), generator=g)
        for h in range(Hkv):
            x[h, pos[h]] = 8 + gap
        q, k, v = _exact(Hq, Hkv, S, D, dtype, x, seed)
        info["pos"] = pos.tolist()

        def check(oracle, L=None):
            lg = _rows(oracle, L)
            G = Hq // Hkv
            for h in range(Hq):
                p = info["pos"][h // G]
                assert p >= 128 and p >= 2 * n // 3
                assert float(lg[h, :, p].min() - lg[h, :, :p].max()) >= 40, "heavy hitter within kRefSlack of the earlier tiles"
        exact = True

    elif name == "peaked":
        # a sink 100 above a background spread over [-100, -60] (exp < e^-150: exactly 0) and `live` tokens 0..25 below the
        # sink: most probabilities are exactly 0 and most pooled scores tie at 0
        live = kw.get("live", 40)
        x = torch.randint(-100, -59, (Hkv, S), generator=g).float()
        for h in range(Hkv):
            sel = torch.randperm(n - 1, generator=g)[:live] + 1
            x[h, sel] = 100 - torch.randint(0, 26, (live,), generator=g).float()
        x[:, 0] = 100
        q, k, v = _exact(Hq, Hkv, S, D, dtype, x, seed)

        def check(oracle, L=None):
            pr = oracle.softmax_rows(oracle.window_logits(L.q, L.k, L.W)).float()
            assert float((pr == 0).float().mean()) > 0.9, "rows are not mostly exact zeros"
            spread = _rows(oracle, L)
            spread = spread[torch.isfinite(spread) & (spread > -1e30)]
            assert float(spread.max() - spread.min()) > 150
        exact = True

    elif name == "subnormal":
        # bf16 subnormal band: a sink at token 0, background ~200 below it, band tokens 88-94 below it, where
        # softmax(fp32).to(bfloat16) keeps subnormal probabilities that a flush-to-zero exp would drop
        assert dtype == torch.bfloat16
        per = kw.get("band", 16)
        x = torch.full((Hkv, S), -100.0)
        x[:, 0] = 100
        shift = math.ceil(math.log(W / 8))          # a sum of W equal probabilities must stay subnormal
        for h in range(Hkv):
            sel = torch.randperm(n - 1, generator=g)[:per] + 1
            x[h, sel] = 100 - shift - torch.tensor([88.0, 89.0, 90.0, 91.0, 92.0])[torch.randint(0, 5, (per,), generator=g)]
        q, k, v = _exact(Hq, Hkv, S, D, dtype, x, seed)

        def check(oracle, L=None, kernel=7, pooling="maxpool"):
            r = oracle.evict("snapkv", L.q, L.k, L.v, L.W, 1, kernel, pooling)
            p = r.pooled.float()
            sub = (p > 0) & (p < BF16_TINY)
            assert int(sub.sum(-1).min()) >= 4, "no subnormal pooled scores"
            info["normal"] = int((p >= BF16_TINY).sum(-1).max())
        exact = True

    elif name == "repeated":
        # runs of identical K rows (pad / repeated tokens) 6 above an integer background, straddling 128-token tile
        # boundaries and the 1/8 .. 7/8 points of the scored range (per-CTA ranges, cluster ranks): many exact ties at the
        # selection threshold
        run = kw.get("run", 24)
        x = torch.randint(-4, 5, (Hkv, S), generator=g).float()
        centers = sorted({c for c in [128 * t for t in range(1, n // 128)][:6] + [n * f // 8 for f in range(1, 8)]
                          if run // 2 <= c <= n - run // 2})
        for c in centers:
            x[:, c - run // 2:c + run // 2] = 6
        q, k, v = _exact(Hq, Hkv, S, D, dtype, x, seed)
        info["tied"] = len(centers) * run

        def check(oracle, L=None):
            kk = L.k[:, :n, 0].float()
            assert int((kk == 6).sum(-1).min()) >= run * 2
            assert any(bool((kk[:, 128 * t - 1] == 6).all() and (kk[:, 128 * t] == 6).all()) for t in range(1, n // 128 + 1))
        exact = True

    elif name == "fp16mask":
        # fp16: window keys whose logits are <= -16 (some exactly -16), so finfo.min + x rounds to -inf in the masked block
        assert dtype == torch.float16
        c = _c(D, dtype)
        x = torch.randint(-4, 5, (Hkv, S), generator=g).float()
        m16 = float(torch.tensor(-16.0 * math.sqrt(D) / c).to(dtype))     # c * m16 / sqrt(D) rounds to -16
        x[:, n:] = torch.tensor([m16, -20.0, m16, -40.0])[torch.arange(W) % 4]
        x[:, n] = 0.0                                                       # never masked (window row 0's own key)
        q, k, v = _exact(Hq, Hkv, S, D, dtype, x, seed)

        def check(oracle, L=None):
            lg = _rows(oracle, L)
            assert bool(torch.isneginf(lg[:, :, n:]).any()), "no -inf in the masked block"
            assert bool((lg[:, W - 1, n:] == -16).any()), "no logit at exactly -16"
        exact = True

    elif name == "outlier":
        # massive activations: 2-4 dims of q and k at 30-100 (same sign per channel, magnitude per token), the rest randn.
        # fp16 keeps |q.k| < 65504 (q's outliers at most 30, 3 dims)
        q = torch.randn(Hq, S, D, generator=g)
        k = torch.randn(Hkv, S, D, generator=g)
        v = torch.randn(Hkv, S, D, generator=g)
        nd = 3 if dtype == torch.float16 else 4
        dims = torch.randperm(D, generator=g)[:nd]
        qmax = 30.0 if dtype == torch.float16 else 60.0
        for d in dims.tolist():
            q[:, :, d] = qmax * (0.5 + 0.5 * torch.rand(Hq, S, generator=g))
            k[:, :, d] = 30 + 70 * torch.rand(Hkv, S, generator=g)
        v[:, :, dims[0]] = 100 * torch.sign(torch.randn(Hkv, S, generator=g))          # V outliers too
        q, k, v = q.to(dtype), k.to(dtype), v.to(dtype)
        info["dims"] = dims.tolist()

        def check(oracle, L=None):
            assert float(L.q.float().abs().max()) >= 30 and float(L.k.float().abs().max()) >= 30
            raw = torch.einsum("hsd,gtd->hgst", L.q[:, -1:].double(), L.k.double())
            assert float(raw.abs().max()) < 65504
            lg = _rows(oracle, L)
            fin = lg[torch.isfinite(lg) & (lg > -1e30)]
            assert float(fin.max() - fin.min()) > 100
        exact = False
    else:
        raise ValueError(name)

    L = Landscape(name, q, k, v, W, exact, None, info)
    L.check = lambda oracle, **a: check(oracle, L, **a)
    return L


def ulp_own(a: torch.Tensor, b: torch.Tensor, dtype) -> torch.Tensor:
    """|a - b| in ulps of each element's own magnitude max(|a|, |b|) in `dtype` (subnormal ulps below the smallest
    normal), elementwise; no floor relative to the tensor's maximum."""
    mant = 8 if dtype == torch.bfloat16 else 11
    emin = -126 if dtype == torch.bfloat16 else -14
    fa, fb = a.double(), b.double()
    mag = torch.maximum(fa.abs(), fb.abs())
    e = torch.floor(torch.log2(torch.clamp(mag, min=2.0 ** emin)))
    ulp = torch.exp2(e - (mant - 1))
    return (fa - fb).abs() / ulp


def smallest_subnormal(dtype) -> float:
    return 2.0 ** -133 if dtype == torch.bfloat16 else 2.0 ** -24


def assert_stage2(got: torch.Tensor, ref: torch.Tensor, what: str, max_ulp: float = 2.0):
    """Every element within `max_ulp` ulps of its own magnitude; zero exactly where the reference is zero, except where
    the reference is below 4x the dtype's smallest subnormal."""
    dt = ref.dtype
    assert got.shape == ref.shape
    u = ulp_own(got, ref, dt)
    bad = u > max_ulp
    assert not bool(bad.any()), f"{what}: {int(bad.sum())} elements beyond {max_ulp} ulp (max {float(u.max()):.1f})"
    gz, rz = got.float() == 0, ref.float() == 0
    tiny = ref.double().abs() < 4 * smallest_subnormal(dt)
    zbad = (gz != rz) & ~tiny
    assert not bool(zbad.any()), f"{what}: zero pattern differs at {int(zbad.sum())} elements"
