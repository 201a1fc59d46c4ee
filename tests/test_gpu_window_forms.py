"""The decode window (`pkv_decode_attn_window`, DESIGN.md §4.7), its heavy hitters (`pkv_decode_attn_heavy`, §4.9) and the
beam reorder of both windows (`pkv_cache_reorder`) at the windows they run at: R = 256 ... 4096 over ragged prompts of up to
2048 rows per (sequence, cache head), B = 8 and 64, and heads above 16 384 rows.

These sizes reach code paths the small-window tests never run: several slots per thread in `decode_heavy_kernel` (R > 512),
heavy steps whose (m, l) come from `decode_combine_kernel` over up to 64 splits, single-split sequences inside a launch sized
for many, and the new ring row in a middle split or exactly on a split's first or last row. `test_cases_reach_every_regime`
(no GPU) restates the split rule and asserts that the cases below reach every one of these regimes on a 132-SM H100; the GPU
tests print the labels of the device they run on.

Bound of the ring's output (test_ring_at_scale, check (b)). u = 2^-24. Per (sequence, query head), with the fp64 softmax p
and scores s over exactly the attended rows: the fp32 score of a row differs from s by at most
ds = D * u * max_r sum_i |q_i k_ri| * scale + 4u * max|s| (the D-term fma dot product; the roundings of the scale, of the
score product and of s - m). The kernel sums a sequence's rows in a fixed tree: each lane group of a CTA adds
ceil(chunk / (8 * RPW)) rows in turn (chunk = ceil(T / ns) rows per split, RPW rows per warp step: 2 for 16-bit D = 128,
4 otherwise), then log2(RPW) shuffle levels, 8 warps in turn and the ns split partials in turn: depth
d = ceil(chunk / (8 RPW)) + log2 RPW + 8 + ns. Every level rescales by an expf (at most 2 ulp, 2^-22 relative) and
rounds once (u). So every weight w_i = expf(s_i - m) as it enters l and acc carries a relative error of at most
eps = 2 ds + 2^-22 + d (2^-22 + u) + 2u (its own expf, the products pe * v_scale and pv * v), and the fp32 output
sum w_i v_i / sum w_i is within 2 eps / (1 - eps) * sum_i p_i |v_i| + 2u |out| of the fp64 one, before the rounding to
bf16 / fp16 (one ulp of the exact output covers it). At T = 18 000 rows, ns = 64 and D = 128 this is ~1e-4 * sum p|v|:
the sum is over the split tree, not over T, so the bound stays below the 1e-3 + 1 ulp the small-window test applies.

Bound of the heavy scores (checks (b) and (d)). A GPU probability is expf(s - m) / l with the fp32 score s and state (m, l)
of the step: relative to the fp64 one it errs by at most eps_p = 4 ds + 2 * 2^-22 + d (2^-22 + u) + 2u (ds in s and in m,
the expf, the sum l as above, the subtraction and the division), taken over the query heads of the cache head. A slot adds
the sum of its G heads' probabilities in ascending head order and then adds that to A: G roundings of at most u * A each.
So every slot carries a budget, reset when a row is appended and grown at every step by eps_p * add + G u A, and
|A - A64| <= budget + ABS. A crafted window seeds the fp64 twin with the crafted fp32 A, so only the additions made here
count. ABS = 1e-10 keeps the comparison from being purely relative at A = 0; no A here comes near it.
"""
from __future__ import annotations

import math
from typing import NamedTuple, Optional

import pytest
import torch

from gpu_util import dev
from oracle_beam_backend import reorder_twin
from oracle_heavy_backend import pick_victim
from oracle_window_backend import window_slot
from test_gpu_beam import BK, _cache
from test_gpu_decode_heavy import _argmin
from test_gpu_decode_window import _launch_existing, _prewrite, _same, _ulp

H100_SMS = 132
HEAVY_THREADS = 512          # pkv_decode.cu: kHeavyThreads, the slots of one pass of decode_heavy_kernel
U = 2.0 ** -24
ABS = 1e-10
SENTINEL = 7.0
needs_cuda = pytest.mark.skipif(not torch.cuda.is_available(), reason="needs a CUDA device")

# (dtype, D, Hq, Hkv)
GEOMS = {"8b": (torch.bfloat16, 128, 32, 8), "70b": (torch.bfloat16, 128, 64, 8), "d64": (torch.float16, 64, 16, 8),
         "hq8": (torch.bfloat16, 128, 8, 4)}
FORMS = [(False, False), (True, False), (False, True), (True, True)]          # (fp8, shared)
SHARED = [(False, True), (True, True)]


def splits_for(Hq: int, T: int, sms: int) -> int:
    """decode_splits_for (pyramidkv_b200/csrc/pkv_internal.h): the split count of T rows for Hq query heads per sequence."""
    ns = (T + 255) // 256
    ns = min(ns, (sms * 4 + Hq - 1) // Hq)
    return min(max(ns, 1), 64)


def split_cap(Hq: int, sms: int) -> int:
    return min(64, (sms * 4 + Hq - 1) // Hq)


class Spec(NamedTuple):
    name: str
    geom: str
    B: int
    R: int
    fp8: bool
    shared: bool
    heavy: Optional[int]     # H of the heavy-hitter rule; None: the ring
    long: bool = False       # heads above 16 384 rows
    empty: bool = False      # heavy: driven from an empty window instead of a crafted full one

    @property
    def dims(self):
        dtype, D, Hq, Hkv = GEOMS[self.geom]
        return dtype, D, Hq, Hkv, (Hkv if self.shared else Hq)

    @property
    def seed(self) -> int:
        return sum(ord(ch) * (i + 1) for i, ch in enumerate(self.name)) % 100003

    def prompt_rows(self) -> torch.Tensor:
        """Ragged P per (sequence, cache head) in [1, 2048], with both ends present; `long`: two heads above 16 384."""
        H = self.dims[4]
        g = torch.Generator().manual_seed(self.seed)
        P = torch.randint(1, 2049, (self.B, H), generator=g, dtype=torch.int64)
        P[0, 0], P[-1, -1] = 1, 2048
        if self.long:
            P[0, 1 % H], P[-1, 0] = 16422, 16390
        return P

    def cap(self, P) -> int:
        return int(P.max()) + self.R + 3

    def bytes(self) -> int:
        """Device bytes of a case: two copies of K, V (and scales), and the fp64 twin's per-chunk temporaries."""
        dtype, D, Hq, Hkv, H = self.dims
        row = D * (1 if self.fp8 else 2) + (4 if self.fp8 else 0)
        return 4 * self.B * H * self.cap(self.prompt_rows()) * row + (1 << 29)


def _fmt(fp8, shared):
    return ("e4m3" if fp8 else "16bit") + ("_shared" if shared else "_perq")


RING = []
for _g, _B, _R, _forms, _long in [("8b", 8, 1024, FORMS, False), ("8b", 64, 256, SHARED, False), ("8b", 8, 4096, FORMS, False),
                                  ("70b", 8, 1024, FORMS, False), ("70b", 8, 4096, SHARED, False),
                                  ("d64", 64, 1024, FORMS, False), ("d64", 64, 4096, SHARED, False),
                                  ("hq8", 8, 1024, FORMS, True), ("hq8", 64, 256, FORMS, False)]:
    for _f8, _sh in _forms:
        RING.append(Spec(f"ring_{_g}_B{_B}_R{_R}_{_fmt(_f8, _sh)}{'_long' if _long else ''}", _g, _B, _R, _f8, _sh, None, _long))


def _heavy_specs():
    out, i = [], 0
    names = list(GEOMS)
    for R in (256, 512, 513, 1024, 4096):
        for H in (1, R // 2, R - 1):
            for f, (f8, sh) in enumerate(FORMS):
                geom, B = names[(i + i // 4) % 4], (8, 64)[(i // 4) % 2]
                s = Spec("", geom, B, R, f8, sh, H)
                if s.bytes() > 1 << 32:
                    s = s._replace(B=8)
                if s.bytes() > 1 << 32:
                    s = s._replace(geom="d64")
                out.append(s._replace(name=f"heavy_{s.geom}_B{s.B}_R{R}_H{H}_{_fmt(f8, sh)}"))
                i += 1
    out.append(Spec("heavy_hq8_B8_R1024_H512_16bit_perq_long", "hq8", 8, 1024, False, False, 512, True))
    return out


HEAVY = _heavy_specs()
EMPTY = Spec("heavy_8b_B8_R1024_H512_16bit_perq_from_empty", "8b", 8, 1024, False, False, 512, empty=True)
CRAFT_STEPS = 64


# ---------------------------------------------------------------------------------------------------------------------------
# The plan of the ring steps and the regime of every step (no GPU)
# ---------------------------------------------------------------------------------------------------------------------------
def _chunk(Hq, T, nsplit, sms):
    ns = min(nsplit, splits_for(Hq, T, sms))
    return ns, -(-T // ns)


def slot_label(Hq, T, nsplit, slot, sms):
    """(split count of the sequence, split of the slot: first / middle / last / only, edge: r_begin / r_end-1 / None)."""
    ns, chunk = _chunk(Hq, T, nsplit, sms)
    last = -(-T // chunk) - 1
    s = slot // chunk
    pos = "only" if last == 0 else "first" if s == 0 else "last" if s == last else "middle"
    edge = "r_begin" if slot == s * chunk else "r_end-1" if slot == min(T, (s + 1) * chunk) - 1 else None
    return ns, pos, edge


EDGE_KINDS = [("first", "r_end-1"), ("middle", "r_begin"), ("middle", "r_end-1"), ("last", "r_begin"), ("last", "r_end-1")]


def _edge_target(Hq, P, R, nsplit, sms, want):
    """A ring row of (P, R) on a split edge, of the kind `want` where one exists."""
    T = P + R
    ns, chunk = _chunk(Hq, T, nsplit, sms)
    cands = []
    for i in range(-(-T // chunk)):
        for row in (i * chunk, min(T, (i + 1) * chunk) - 1):
            if P <= row < T:
                cands.append((slot_label(Hq, T, nsplit, row, sms)[1:], row))
    hit = [row for kind, row in cands if kind == want]
    return hit[0] if hit else cands[0][1]


def ring_plan(spec: Spec, sms: int):
    """The ring steps of a case: (step, per-head row offset off [B, H]); the count of (b, c) is n = 1 + step + P + off.
    Episodes of consecutive steps: the first two appends (n = P + 1, P + 2), the first wrap (n = P + R + 1 ...), two with each
    head's new row on a split edge (kinds rotating over the heads), and one after many wraps (n > 2^20)."""
    _, _, Hq, _, H = spec.dims
    P, R = spec.prompt_rows(), spec.R
    nsplit = splits_for(Hq, spec.cap(P), sms)
    zero = torch.zeros_like(P)
    steps = [(0, zero), (1, zero), (R, zero), (R + 1, zero), (R + 2, zero)]
    for e in range(2):
        s = 3 * R + 11 + e * R
        off = torch.empty_like(P)
        for b in range(spec.B):
            for c in range(H):
                want = EDGE_KINDS[(b * H + c + 2 * e) % len(EDGE_KINDS)]
                target = _edge_target(Hq, int(P[b, c]), R, nsplit, sms, want)
                off[b, c] = (target - int(P[b, c]) - s) % R
        steps += [(s, off), (s + 1, off)]
    g = torch.Generator().manual_seed(spec.seed + 1)
    off = torch.randint(0, R, tuple(P.shape), generator=g, dtype=torch.int64)
    steps += [(1 << 20, off), ((1 << 20) + 1, off)]
    return steps


def labels(spec: Spec, sms: int) -> set:
    """The regimes a case reaches on a device with `sms` SMs."""
    _, _, Hq, _, H = spec.dims
    P, R = spec.prompt_rows(), spec.R
    nsplit = splits_for(Hq, spec.cap(P), sms)
    got = {f"launch_splits={nsplit}"}
    if int((P + R).max()) > 16384:
        got.add("P+R>16384")
    capv = split_cap(Hq, sms)
    if spec.heavy is None:
        for s, off in ring_plan(spec, sms):
            n = 1 + s + P + off
            for b in range(spec.B):
                for c in range(H):
                    slot, T = window_slot(int(n[b, c]), int(P[b, c]), R)
                    ns, pos, edge = slot_label(Hq, T, nsplit, slot, sms)
                    got.add(f"slot_{pos}")
                    if edge:
                        got.add(f"slot_on_{edge}")
                    if ns == 1 and nsplit > 1:
                        got.add("single_split_in_multi_split_launch")
                    if ns == capv:
                        got.add(f"split_cap_Hq{Hq}={capv}")
    else:
        full = [splits_for(Hq, int(t), sms) for t in (P + R).reshape(-1)]
        if max(full) == capv or nsplit == capv:
            got.add(f"split_cap_Hq{Hq}={capv}")
        if spec.empty and int(P.min()) + 1 <= 256 and nsplit > 1:
            got.add("single_split_in_multi_split_launch")        # step 0: n = P + 1 rows
        if nsplit > 1 and spec.B >= 8:
            got.add("heavy_combine_B>=8")
        got.add(f"heavy_R{R}_slots_per_thread{-(-R // HEAVY_THREADS)}")
    return got


REQUIRED = {"single_split_in_multi_split_launch", "slot_first", "slot_middle", "slot_last", "slot_on_r_begin",
            "slot_on_r_end-1", "split_cap_Hq32=17", "split_cap_Hq64=9", "split_cap_Hq8=64", "heavy_combine_B>=8",
            "heavy_R512_slots_per_thread1", "heavy_R513_slots_per_thread2", "heavy_R4096_slots_per_thread8", "P+R>16384"}


def test_cases_reach_every_regime():
    """No GPU: on a 132-SM H100 the cases reach every regime of REQUIRED, and every case fits in about 4 GB."""
    assert (splits_for(32, 10 ** 6, H100_SMS), splits_for(64, 10 ** 6, H100_SMS), splits_for(8, 10 ** 6, H100_SMS)) == (17, 9, 64)
    got = set()
    for spec in RING + HEAVY + [EMPTY]:
        got |= labels(spec, H100_SMS)
        assert spec.bytes() <= 1 << 32, spec.name
    assert REQUIRED <= got, sorted(REQUIRED - got)
    # heavy covers every R and H of the matrix in every form, at both batch sizes
    assert {(s.R, s.heavy, s.fp8, s.shared) for s in HEAVY} >= {(R, H, f, sh) for R in (256, 512, 513, 1024, 4096)
                                                                 for H in (1, R // 2, R - 1) for f, sh in FORMS}
    assert {s.B for s in HEAVY} == {8, 64} and {s.B for s in RING} == {8, 64}
    assert {(s.R, s.fp8, s.shared) for s in RING} >= {(R, f, sh) for R in (256, 1024, 4096) for f, sh in SHARED}
    # the plan lands where it says: the first wrap at n = P + R + 1 and a count above 2^20
    spec = RING[0]
    P, plan = spec.prompt_rows(), ring_plan(spec, H100_SMS)
    assert any(bool((1 + s + P + off == P + spec.R + 1).all()) for s, off in plan)
    assert int(max(int((1 + s + P + off).min()) for s, off in plan)) >= 1 << 20


# ---------------------------------------------------------------------------------------------------------------------------
# Device cases
# ---------------------------------------------------------------------------------------------------------------------------
def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


class Form:
    """The buffers of one case on the device, in the attribute layout the imported helpers read, with the step inputs drawn
    on demand (q / kn / vn keyed by step). Rows past P + R hold SENTINEL."""

    def __init__(self, spec: Spec):
        self.spec = spec
        self.dtype, self.D, self.Hq, self.Hkv, self.H = spec.dims
        self.fp8, self.shared, self.B, self.R = spec.fp8, spec.shared, spec.B, spec.R
        self.P = spec.prompt_rows()
        self.cap = spec.cap(self.P)
        self.G = self.Hq // self.H
        self.kv_of = torch.arange(self.H) if self.shared else torch.arange(self.Hq) // (self.Hq // self.Hkv)
        self.g = torch.Generator(device=dev()).manual_seed(spec.seed)
        shape = (self.B, self.H, self.cap, self.D)
        past = (torch.arange(self.cap, device=dev()) >= (self.P + self.R).to(dev())[..., None])[..., None]

        def plane(dtype, scale):   # one sequence at a time: no fp32 copy of a whole plane
            out = torch.empty(shape, dtype=dtype, device=dev())
            for b in range(self.B):
                x = (torch.randn(shape[1:], generator=self.g, device=dev()) * scale).clamp(-440, 440)
                out[b] = torch.where(past[b], SENTINEL, x).to(dtype)
            return out
        if self.fp8:   # E4M3 bytes of N(0, 100^2) and per-row scales around 0.8 / 100 (K) and 1 / 100 (V)
            self.bufs = [plane(torch.float8_e4m3fn, 100), plane(torch.float8_e4m3fn, 100)]
            for width in (0.8, 1.0):
                self.bufs.append((torch.rand(shape[:3], generator=self.g, device=dev()) + 0.5) * (width / 100))
        else:
            self.bufs = [plane(self.dtype, 0.8), plane(self.dtype, 1.0)]
        self.q, self.kn, self.vn = {}, {}, {}
        self.ws = torch.empty(_ops().decode_workspace_bytes(self.B * self.Hq, self.D), dtype=torch.uint8, device=dev())
        self.prompt_dev = self.P.to(dev()).reshape(-1).int().contiguous()

    def draw(self, t):
        self.q[t] = (torch.randn(self.B, self.Hq, self.D, generator=self.g, device=dev()) * 0.8).to(self.dtype)
        self.kn[t] = torch.randn(self.B, self.Hkv, self.D, generator=self.g, device=dev()).to(self.dtype)
        self.vn[t] = torch.randn(self.B, self.Hkv, self.D, generator=self.g, device=dev()).to(self.dtype)
        return self.q[t], self.kn[t], self.vn[t]

    def scales(self, bufs):
        return (bufs[2], bufs[3]) if self.fp8 else None

    def nsplit(self, sms):
        return splits_for(self.Hq, self.cap, sms)

    def depth(self, T, sms):
        """d of the docstring per (sequence, cache head): the levels of the kernel's summation tree over T rows."""
        rpw = 32 // (self.D // (16 if self.fp8 else 8))
        ns = torch.minimum(torch.full_like(T, self.nsplit(sms)), torch.clamp((T + 255) // 256, 1, split_cap(self.Hq, sms)))
        chunk = (T + ns - 1) // ns
        return (chunk + 8 * rpw - 1) // (8 * rpw) + int(math.log2(rpw)) + 8 + ns


def _ops():
    from pyramidkv_b200 import ops
    return ops


def _attend64(f: Form, bufs, q, attended, with_v=True):
    """fp64 attention of every (sequence, query head) over rows [0, attended[b, c]) of its cache head, as an einsum over
    [B, H, G, D] x [B, H, cap, D] a few sequences at a time. Returns the probabilities summed over each cache head's query
    heads [B, H, cap], the score error ds of the docstring [B, Hq], and with V the output and sum_i p_i |v_i| [B, Hq, D]."""
    B, H, G, D, cap = f.B, f.H, f.G, f.D, f.cap
    scale = D ** -0.5
    per = max(1, (1 << 28) // (H * cap * D * 8))
    att = attended.to(dev())
    probs = torch.empty(B, H, cap, dtype=torch.float64, device=dev())
    ds = torch.empty(B, f.Hq, dtype=torch.float64, device=dev())
    out = torch.empty(B, f.Hq, D, dtype=torch.float64, device=dev()) if with_v else None
    mass = torch.empty_like(out) if with_v else None
    rows = torch.arange(cap, device=dev())
    for s0 in range(0, B, per):
        s1 = min(B, s0 + per)
        K = bufs[0][s0:s1].double()
        if f.fp8:
            K = K * bufs[2][s0:s1].double()[..., None]
        qg = q[s0:s1].double().reshape(s1 - s0, H, G, D)
        masked = (rows[None, None, :] >= att[s0:s1][..., None])[:, :, None, :]
        s = (torch.einsum("bhgd,bhrd->bhgr", qg, K) * scale).masked_fill(masked, float("-inf"))
        qk = torch.einsum("bhgd,bhrd->bhgr", qg.abs(), K.abs()).masked_fill(masked, 0.0).amax(-1)
        sabs = s.abs().masked_fill(masked, 0.0).amax(-1)
        ds[s0:s1] = (D * U * qk * scale + 4 * U * sabs).reshape(s1 - s0, f.Hq)
        p = torch.softmax(s, dim=-1)
        probs[s0:s1] = p.sum(2)
        del K, qk
        if with_v:
            V = bufs[1][s0:s1].double()
            if f.fp8:
                V = V * bufs[3][s0:s1].double()[..., None]
            out[s0:s1] = torch.einsum("bhgr,bhrd->bhgd", p, V).reshape(s1 - s0, f.Hq, D)
            mass[s0:s1] = torch.einsum("bhgr,bhrd->bhgd", p, V.abs()).reshape(s1 - s0, f.Hq, D)
    return probs, ds, out, mass


@pytest.mark.gpu
@needs_cuda
# ---------------------------------------------------------------------------------------------------------------------------
# The ring
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("spec", RING, ids=[s.name for s in RING])
def test_ring_at_scale(libpkv, spec):
    """At every step of the plan: (a) the output and every buffer byte equal the existing batch entry point run without
    k_new over the same buffers with the new row pre-written at its ring slot; (b) the output is within the derived bound of
    the fp64 attention over exactly min(n, P + R) rows."""
    ops = _ops()
    torch.cuda.reset_peak_memory_stats()
    sms = _sms()
    f = Form(spec)
    print(f"PKV_MEASURED {spec.name} labels on {sms} SMs: {sorted(labels(spec, sms))}")
    win, ref = f.bufs, [t.clone() for t in f.bufs]
    step = torch.zeros(1, dtype=torch.int32, device=dev())
    nsplit = f.nsplit(sms)
    worst = 0.0
    for s, off in ring_plan(spec, sms):
        q, kn, vn = f.draw(s)
        step.fill_(s)
        rows = (f.P + off).to(dev()).reshape(-1).int().contiguous()
        out = ops.decode_attn_window(q, win[0], win[1], 1, kn, vn, f.prompt_dev, f.R, rows=rows, step=step,
                                     max_length=f.cap, workspace=f.ws, scales=f.scales(win), gqa=f.shared)
        n = 1 + s + f.P + off
        slot = torch.where(n > f.P + f.R, f.P + (n - 1 - f.P) % f.R, n - 1)
        attended = torch.minimum(n, f.P + f.R)
        _prewrite(f, ref, s, slot)
        want = _launch_existing(f, ref, q, (attended - 1).to(dev()).reshape(-1).int().contiguous(), f.ws)
        assert torch.equal(out, want), s                                                  # (a) the output bits
        assert _same(win, ref), s                                                         # (a) every buffer byte
        _, ds, exact, mass = _attend64(f, win, q, attended)                               # (b)
        d = f.depth(attended, sms).to(dev()).repeat_interleave(f.G, dim=1).double()       # [B, Hq]
        eps = 2 * ds + 2.0 ** -22 + d * (2.0 ** -22 + U) + 2 * U
        bar = (2 * eps / (1 - eps))[..., None] * mass + 2 * U * exact.abs() + _ulp(exact.to(f.dtype)).double()
        err = (out.double() - exact).abs()
        assert bool((err <= bar).all()), (s, float((err - bar).max()))
        worst = max(worst, float((err / bar).max()))
    print(f"PKV_MEASURED {spec.name}: largest output error / bound {worst:.3g}; "
          f"peak {torch.cuda.max_memory_allocated() / 2 ** 30:.2f} GiB")


# ---------------------------------------------------------------------------------------------------------------------------
# Heavy hitters
# ---------------------------------------------------------------------------------------------------------------------------
def _craft(f: Form, j0: int):
    """A full window the rule reaches after the step that appended generation j0 - 1: distinct generation indices, every
    generation in (j0 - (R - H), j0 - 1] held, H + 1 older ones, A log-uniform over 1e-4 .. 10 so that the candidates
    separate, except a group of up to four candidates that share one K row and the smallest A (exact ties, broken by the
    generation index) and victim = the rule's pick. Returns (scores, gen, victim)."""
    B, H, R, Hh, g = f.B, f.H, f.R, f.spec.heavy, f.g
    last = j0 - (R - Hh)
    protected = torch.arange(last + 1, j0, device=dev()).expand(B, H, R - Hh - 1)
    old = torch.argsort(torch.rand(B, H, last + 1, generator=g, device=dev()), dim=-1)[..., :Hh + 1]
    gens = torch.cat([protected, old], dim=-1)
    gen = torch.gather(gens, -1, torch.argsort(torch.rand(B, H, R, generator=g, device=dev()), dim=-1)).int().contiguous()
    A = torch.pow(10.0, torch.rand(B, H, R, generator=g, device=dev()) * 5 - 4)
    m = min(4, Hh + 1)
    cand = torch.where(gen <= last, torch.arange(R, device=dev()), 2 * R)
    tie = torch.sort(cand, dim=-1).values[..., :m]                                     # m candidate slots per head
    A.scatter_(-1, tie, (A.amin(-1, keepdim=True) / 2).expand(B, H, m))
    bi = torch.arange(B, device=dev())[:, None, None]
    ci = torch.arange(H, device=dev())[None, :, None]
    rows = f.P.to(dev())[..., None] + tie
    src = rows[..., :1].expand_as(rows)
    kb = f.bufs[0].view(torch.uint8) if f.fp8 else f.bufs[0]
    kb[bi, ci, rows] = kb[bi, ci, src]
    if f.fp8:
        f.bufs[2][bi, ci, rows] = f.bufs[2][bi, ci, src]
    k, _ = _argmin(A, gen, R, last)
    for b, c in ((0, 0), (B - 1, H - 1)):
        assert pick_victim(A[b, c].cpu(), gen[b, c].cpu(), R, j0 - 1, R, Hh) == int(k[b, c])
    victim = (f.P.to(dev()) + k).int().reshape(-1).contiguous()
    return A.float().contiguous(), gen, victim


def _drive_heavy(f: Form, steps, state, sms):
    """Runs `steps` heavy steps (rows = P, so generation j = step) from `state` and checks (a) to (d) of the heavy test
    at each. Returns (near ties, choices)."""
    ops = _ops()
    B, H, R, G, Hh = f.B, f.H, f.R, f.G, f.spec.heavy
    scores, gen, victim = state
    hv, ref = f.bufs, [t.clone() for t in f.bufs]
    A64, gen64 = scores.double().clone(), gen.long().clone()
    budget = torch.zeros_like(A64)
    P = f.P.to(dev())
    step = torch.zeros(1, dtype=torch.int32, device=dev())
    ar = torch.arange(R, device=dev())
    d = None
    near = choices = 0
    for t in steps:
        q, kn, vn = f.draw(t)
        step.fill_(t)
        v_before = victim.clone().reshape(B, H).long()
        out = ops.decode_attn_heavy(q, hv[0], hv[1], 1, kn, vn, f.prompt_dev, R, Hh, scores, gen, victim, rows=f.prompt_dev,
                                    step=step, max_length=f.cap, workspace=f.ws, scales=f.scales(hv), gqa=f.shared)
        slot = v_before if t + 1 > R else P + t
        attended = torch.minimum(P + t + 1, P + R)
        _prewrite(f, ref, t, slot.cpu())
        want = _launch_existing(f, ref, q, (attended - 1).reshape(-1).int().contiguous(), f.ws)
        assert torch.equal(out, want), t                                                  # (a)
        assert _same(hv, ref), t
        probs, ds, _, _ = _attend64(f, hv, q, attended.cpu(), with_v=False)
        if d is None or t < R:
            d = f.depth(attended.cpu(), sms).to(dev()).double()
        eps = (4 * ds + 2 * 2.0 ** -22 + 2 * U).reshape(B, H, G).amax(-1) + d * (2.0 ** -22 + U)      # [B, H]
        held = min(t + 1, R)
        is_new = ar[None, None, :] == (slot - P)[..., None]
        A64 = torch.where(is_new, 0.0, A64)
        budget = torch.where(is_new, 0.0, budget)
        gen64 = torch.where(is_new, t, gen64)
        add = torch.gather(probs, 2, (P[..., None] + ar).clamp_max(f.cap - 1))
        live = ar[None, None, :] < held
        A64 = torch.where(live, A64 + add, A64)
        budget = torch.where(live, budget + eps[..., None] * add + G * U * A64, budget)
        assert torch.equal(gen.long(), gen64), t                                          # (d) slot by slot
        err = (scores.double() - A64).abs()[..., :held]
        bar = budget[..., :held] + ABS
        assert bool((err <= bar).all()), (t, float((err - bar).max()))                    # (b)
        if t + 1 >= R:
            last = t + 1 - (R - Hh)
            k_gpu, _ = _argmin(scores, gen, held, last)
            assert torch.equal(victim.reshape(B, H).long(), P + k_gpu), t               # (c)
            k64, a = _argmin(A64, gen64, held, last)
            two = a.topk(2, dim=-1, largest=False)                                      # H + 1 >= 2 candidates
            slack = torch.gather(budget, 2, two.indices).sum(-1) + 2 * ABS
            tie = (two.values[..., 1] - two.values[..., 0]) <= slack
            assert not bool(((k64 != k_gpu) & ~tie).any()), t                           # (d) the twin's own choice
            # near ties, not counting the crafted exact ties (equal fp32 scores on the GPU, decided by the generation index
            # and checked exactly by (c); fp64 einsum rounding can set their twin values a few ulp apart)
            exact_tie = torch.gather(scores, 2, two.indices).diff(dim=-1).squeeze(-1) == 0
            near += int((tie & ~exact_tie).sum())
            choices += B * H
    return near, choices


@pytest.mark.gpu
@needs_cuda
@pytest.mark.parametrize("spec", HEAVY, ids=[s.name for s in HEAVY])
def test_heavy_from_crafted_window(libpkv, spec):
    """From a crafted full window, CRAFT_STEPS steps with checks (a) to (d) (see test_gpu_decode_heavy.py) at each."""
    torch.cuda.reset_peak_memory_stats()
    sms = _sms()
    f = Form(spec)
    print(f"PKV_MEASURED {spec.name} labels on {sms} SMs: {sorted(labels(spec, sms))}")
    j0 = 3 * spec.R + 5
    state = _craft(f, j0)
    near, choices = _drive_heavy(f, range(j0, j0 + CRAFT_STEPS), state, sms)
    print(f"PKV_MEASURED {spec.name}: near ties {near} of {choices} choices; "
          f"peak {torch.cuda.max_memory_allocated() / 2 ** 30:.2f} GiB")
    # Near ties: choices where the twin's two smallest candidates lie within their bounds (the bound is the worst case, so
    # it cannot certify such a choice), not counting the crafted exact ties. On an H100 (700 W): with H = 1 or R - 1 at
    # most 18 of 131 072 choices; with H = R / 2, where hundreds of candidates accumulate nearly the same attention, up to
    # 3509 of 32 768 (R = 4096, E4M3 GQA-shared) and 428 of 4096 (R = 1024, E4M3 GQA-shared).
    assert near <= max(2, choices // (6 if spec.heavy == spec.R // 2 else 1000)), near


@pytest.mark.gpu
@needs_cuda
def test_heavy_from_empty(libpkv):
    """8B bf16, a cache per query head, B = 8, R = 1024, H = 512: from an empty window through the fill and R / 2
    replacements, checks (a) to (d) at every step."""
    torch.cuda.reset_peak_memory_stats()
    sms = _sms()
    f = Form(EMPTY)
    print(f"PKV_MEASURED {EMPTY.name} labels on {sms} SMs: {sorted(labels(EMPTY, sms))}")
    state = (torch.zeros(f.B, f.H, f.R, dtype=torch.float32, device=dev()),
             torch.full((f.B, f.H, f.R), -1, dtype=torch.int32, device=dev()),
             torch.full((f.B * f.H,), -1, dtype=torch.int32, device=dev()))
    near, choices = _drive_heavy(f, range(f.R + f.R // 2), state, sms)
    print(f"PKV_MEASURED {EMPTY.name}: near ties {near} of {choices} choices; "
          f"peak {torch.cuda.max_memory_allocated() / 2 ** 30:.2f} GiB")
    # on an H100 (700 W): 384 of 131 328 choices
    assert near <= choices // 200, near


@pytest.mark.gpu
@needs_cuda
def test_heavy_graph_replay_across_the_fill(libpkv):
    """One captured heavy step (8B bf16, B = 8, R = 1024, H = 512; prompts up to 2048 rows: a 12-split launch with the
    combine) replayed across the fill and the first replacements equals host launches bit for bit: outputs, buffers and
    scores / gen / victim."""
    ops = _ops()
    spec = EMPTY._replace(name="heavy_graph")
    host = Form(spec)
    graph_bufs = [t.clone() for t in host.bufs]
    B, H, R, Hh = host.B, host.H, host.R, spec.heavy

    def state():
        return (torch.zeros(B, H, R, dtype=torch.float32, device=dev()), torch.full((B, H, R), -1, dtype=torch.int32, device=dev()),
                torch.full((B * H,), -1, dtype=torch.int32, device=dev()))
    hstate, gstate = state(), state()
    step = torch.zeros(1, dtype=torch.int32, device=dev())
    ws2 = torch.empty_like(host.ws)
    scratch = torch.empty(ops.decode_heavy_workspace_bytes(B, host.Hq, R), dtype=torch.uint8, device=dev())
    q_s, kn_s, vn_s = (x.clone() for x in host.draw(-1))
    out_s = torch.empty(B, host.Hq, host.D, dtype=host.dtype, device=dev())

    def launch(bufs, st):
        ops.decode_attn_heavy(q_s, bufs[0], bufs[1], 1, kn_s, vn_s, host.prompt_dev, R, Hh, *st, rows=host.prompt_dev, step=step,
                              max_length=host.cap, workspace=ws2, scratch=scratch, out=out_s, gqa=False)
    warm = [t.clone() for t in graph_bufs]
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        launch(warm, state())
    torch.cuda.current_stream().wait_stream(s)
    del warm
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        launch(graph_bufs, gstate)
    assert host.nsplit(_sms()) > 1
    for t in range(R + 64):
        q, kn, vn = host.draw(t)
        step.fill_(t)
        q_s.copy_(q)
        kn_s.copy_(kn)
        vn_s.copy_(vn)
        g.replay()
        want = ops.decode_attn_heavy(q, host.bufs[0], host.bufs[1], 1, kn, vn, host.prompt_dev, R, Hh, *hstate,
                                     rows=host.prompt_dev, step=step, max_length=host.cap, workspace=host.ws, gqa=False)
        assert torch.equal(out_s, want) and _same(graph_bufs, host.bufs), t
        assert all(torch.equal(x, y) for x, y in zip(gstate, hstate)), t


# ---------------------------------------------------------------------------------------------------------------------------
# Beam reorder over full windows
# ---------------------------------------------------------------------------------------------------------------------------
REORDER = [(kind, R, n) for kind in ("ring", "heavy") for R in (256, 1024) for n in (R + 37, 3 * R + 5)]


@pytest.mark.gpu
@needs_cuda
@pytest.mark.parametrize("kind,R,n", REORDER)
@pytest.mark.parametrize("k", [16, 4])
@pytest.mark.parametrize("D,fp8", [(64, False), (128, False), (64, True), (128, True)])
def test_reorder_full_windows(libpkv, kind, R, n, k, D, fp8):
    """`pkv_cache_reorder` over full ring and heavy windows: every plane, scale and scores / gen / victim byte-equal to
    the twin for the swap, cycle, many-to-one and random parent maps; rows past the window and other prompts untouched."""
    P, H = 2, 2
    g = torch.Generator().manual_seed(R + n + k + D + fp8)
    layers = [_cache((fp8, R, kind == "heavy"), P, k, H, 8 + R + 3, D, dev(), g) for _ in range(2)]
    pats = {"swap": [j ^ 1 for j in range(k)], "cycle": [(j + 1) % k for j in range(k)], "one": [k // 2] * k,
            "random": torch.randint(0, k, (k,), generator=g).tolist()}
    step = torch.tensor([n - 1], dtype=torch.int32, device=dev())
    cl = lambda t: None if t is None else t.clone()   # noqa: E731
    for pattern, row in pats.items():
        items = [(cl(a), cl(b), cl(c), cl(d), e, w, None if h is None else tuple(cl(x) for x in h)) for a, b, c, d, e, w, h in layers]
        parent = torch.tensor(row * P, dtype=torch.int32, device=dev())
        diverge = torch.randint(0, n + 1, (P * k,), generator=g, dtype=torch.int32).to(dev())
        diverge = torch.where(parent == torch.arange(P * k, device=dev(), dtype=torch.int32) % k, n, diverge)
        ref = [(*(None if t is None else t.cpu() for t in it[:5]), it[5], None if it[6] is None else tuple(x.cpu() for x in it[6]))
               for it in items]
        reorder_twin(ref, P, k, parent.cpu(), diverge.cpu(), step.cpu(), 1)
        BK.cache_reorder(items, P, k, parent, diverge, step, 1)
        torch.cuda.synchronize()
        for got, want in zip(items, ref):
            for a, b in zip(got[:4], want[:4]):
                if a is not None:
                    assert torch.equal(a.cpu().view(torch.uint8), b.view(torch.uint8)), pattern
            if got[6] is not None:
                for a, b in zip(got[6], want[6]):
                    assert torch.equal(a.cpu(), b), pattern

