"""-m gpu: heavy hitters in the decode window (`pkv_decode_attn_heavy`, ops.decode_attn_heavy) over every cache form: 16-bit
and E4M3 rows, a cache per query head and GQA-shared, bf16 / fp16, D = 64 / 128, G = 1, 2, 4, 8, B = 1, 3, 64, ragged
prompt rows P, driven across the wrap. At every step:
(a) the output and every byte of the buffers equal the existing batch entry point run without k_new over the same buffer with
    the new row already at its slot (n - 1 before the window is full, the victim after);
(b) `scores` agree with an fp64 restatement of the rule over the same rows within REL * A + ABS (derived below);
(c) `victim` is exactly the argmin of the rule (ties to the smallest generation index) applied to the GPU's own scores;
(d) the held generation indices equal the fp64 twin's, except at steps where the twin's two smallest candidate scores lie
    within the bound of (b): those are counted (and must stay rare), and the twin then follows the GPU's choice.
Also: H = 0 equals `pkv_decode_attn_window` bit for bit (outputs, caches, and gen holds the ring's rows), a captured launch
replayed across the wrap equals host launches in outputs and state, out-of-range counts write nothing and give NaN, and each
argument error returns its code.

Bound of (b). A GPU probability is expf(s - m) / l with s the fp32 score and (m, l) the fp32 softmax state. Relative to the
fp64 probability its error collects: the fp32 dot product of D terms (|err s| <= D * 2^-24 * sum|q_i k_i| * scale, at most
about 5e-5 for these inputs, also in m), the subtraction and expf (|s - m| * 2^-24 plus 2 ulp), the online sum l (at most
T * 2^-24 relative, T <= 700 here: 4.2e-5) and the division (0.5 ulp): under 2e-4 of p. A adds at most 3R such terms
and as many fp32 additions (2^-24 each, relative to A), so |A - A64| <= 2e-4 * A + 3R * 2^-24 * A. REL = 5e-4 covers it for
R <= 40, ABS = 1e-6 the fp32 resolution of tiny scores."""
import ctypes as C

import pytest
import torch

from gpu_util import dev
from oracle_fp8_backend import quantize_rows

pytestmark = pytest.mark.gpu

REL, ABS = 5e-4, 1e-6
SENTINEL = 7.0
# (dtype, D, Hq, Hkv): G = 4, 8, 2, 1, 8
GEOMS = [(torch.bfloat16, 128, 32, 8), (torch.float16, 64, 16, 2), (torch.bfloat16, 64, 8, 4), (torch.float16, 128, 8, 8),
         (torch.bfloat16, 128, 16, 2)]
# (B, R): one long window over prompts long enough for several splits, small windows over larger batches
RUNS = [(1, 40), (3, 8), (64, 5)]
FORMS = [(False, False), (True, False), (False, True), (True, True)]


class Case:
    """Buffers of one cache form, the inputs of `steps` steps and the heavy state."""

    def __init__(self, dtype, D, Hq, Hkv, fp8, shared, B, R, steps, seed=0, pmax=None):
        g = torch.Generator().manual_seed(seed + 7 * D + Hq + B + R)
        self.dtype, self.D, self.Hq, self.Hkv, self.fp8, self.shared, self.B, self.R = dtype, D, Hq, Hkv, fp8, shared, B, R
        self.H = Hkv if shared else Hq
        pmax = pmax or (600 if B <= 3 else 40)
        self.P = torch.randint(1, pmax + 1, (B, self.H), generator=g, dtype=torch.int32)
        self.cap = int(self.P.max()) + R + 3
        x16 = torch.full((B, self.H, self.cap, D), SENTINEL, dtype=dtype)
        k16, v16 = x16.clone(), x16.clone()
        for b in range(B):
            for c in range(self.H):
                n = int(self.P[b, c])
                k16[b, c, :n] = (torch.randn(n, D, generator=g) * 0.8).to(dtype)
                v16[b, c, :n] = torch.randn(n, D, generator=g).to(dtype)
        if fp8:
            kq, ks = quantize_rows(k16)
            vq, vs = quantize_rows(v16)
            self.bufs = [kq, vq, ks, vs]
        else:
            self.bufs = [k16, v16]
        self.q = (torch.randn(steps, B, Hq, D, generator=g) * 0.8).to(dtype)
        self.kn = torch.randn(steps, B, Hkv, D, generator=g).to(dtype)
        self.vn = torch.randn(steps, B, Hkv, D, generator=g).to(dtype)
        self.kv_of = torch.arange(self.H) if shared else torch.arange(Hq) // (Hq // Hkv)

    def device_bufs(self):
        return [t.to(dev()) for t in self.bufs]

    def state(self):
        return (torch.zeros(self.B, self.H, self.R, dtype=torch.float32, device=dev()),
                torch.full((self.B, self.H, self.R), -1, dtype=torch.int32, device=dev()),
                torch.full((self.B * self.H,), -1, dtype=torch.int32, device=dev()))


def _launch_heavy(case, bufs, t, prompt_rows, rows, step, ws, heavy, state, scratch=None, out=None):
    from pyramidkv_b200 import ops
    scales = (bufs[2], bufs[3]) if case.fp8 else None
    return ops.decode_attn_heavy(case.q[t].to(dev()), bufs[0], bufs[1], 1, case.kn[t].to(dev()), case.vn[t].to(dev()), prompt_rows,
                                 case.R, heavy, *state, rows=rows, step=step, max_length=case.cap, workspace=ws, scratch=scratch,
                                 out=out, scales=scales, gqa=case.shared)


def _launch_existing(case, bufs, q, rows, ws):
    """The existing batch entry point of the form without k_new: `1 + rows` rows."""
    from pyramidkv_b200 import ops
    if case.fp8:
        fn = ops.decode_attn_batch_gqa_fp8 if case.shared else ops.decode_attn_batch_fp8
        return fn(q, bufs[0], bufs[1], bufs[2], bufs[3], 1, None, None, rows=rows, max_length=case.cap, workspace=ws)
    fn = ops.decode_attn_batch_gqa if case.shared else ops.decode_attn_batch
    return fn(q, bufs[0], bufs[1], 1, None, None, rows=rows, max_length=case.cap, workspace=ws)


def _prewrite(case, bufs, t, slot):
    bi = torch.arange(case.B)[:, None].expand(case.B, case.H)
    ci = torch.arange(case.H)[None, :].expand(case.B, case.H)
    kn, vn = case.kn[t][:, case.kv_of], case.vn[t][:, case.kv_of]
    slot = slot.cpu()
    if case.fp8:
        kq, ks = quantize_rows(kn)
        vq, vs = quantize_rows(vn)
        bufs[0].view(torch.uint8)[bi, ci, slot] = kq.view(torch.uint8).to(dev())
        bufs[1].view(torch.uint8)[bi, ci, slot] = vq.view(torch.uint8).to(dev())
        bufs[2][bi, ci, slot] = ks.to(dev())
        bufs[3][bi, ci, slot] = vs.to(dev())
    else:
        bufs[0][bi, ci, slot] = kn.to(dev())
        bufs[1][bi, ci, slot] = vn.to(dev())


def _probs64(case, bufs, q, attended):
    """fp64 softmax of every (sequence, query head) over rows [0, attended) of its cache head, summed over the query heads of
    each cache head: [B, H, cap]."""
    if case.fp8:
        K = bufs[0].double() * bufs[2].double()[..., None]
    else:
        K = bufs[0].double()
    G = case.Hq // case.H
    Kq = K.repeat_interleave(G, dim=1)
    A = attended.to(dev()).repeat_interleave(G, dim=1)
    s = torch.einsum("bhd,bhrd->bhr", q.double(), Kq) * case.D ** -0.5
    s = s.masked_fill(torch.arange(case.cap, device=dev())[None, None, :] >= A[..., None], float("-inf"))
    return torch.softmax(s, dim=-1).reshape(case.B, case.H, G, case.cap).sum(2)


def _argmin(A, gen, held, last):
    """Slot index of the smallest (A, gen) among slots [0, held) with gen <= last, per (sequence, cache head)."""
    R = A.shape[-1]
    ok = (torch.arange(R, device=A.device) < held) & (gen <= last)
    a = torch.where(ok, A.double(), float("inf"))
    amin = a.min(-1, keepdim=True).values
    g = torch.where(ok & (a == amin), gen.long(), 2 ** 40)
    return g.argmin(-1), a


def _same(a, b):
    return all(torch.equal(x.view(torch.uint8) if x.dtype == torch.float8_e4m3fn else x,
                           y.view(torch.uint8) if y.dtype == torch.float8_e4m3fn else y) for x, y in zip(a, b))


@pytest.mark.parametrize("B,R", RUNS)
@pytest.mark.parametrize("fp8,shared", FORMS)
@pytest.mark.parametrize("dtype,D,Hq,Hkv", GEOMS)
def test_heavy_steps(oracle, libpkv, dtype, D, Hq, Hkv, fp8, shared, B, R):
    from pyramidkv_b200 import ops
    if shared and Hq == Hkv:
        pytest.skip("G = 1 has no GQA-shared form")
    Hh = R // 2
    steps = 2 * R + 10
    case = Case(dtype, D, Hq, Hkv, fp8, shared, B, R, steps)
    hv, ref = case.device_bufs(), case.device_bufs()
    scores, gen, victim = state = case.state()
    A64 = torch.zeros(B, case.H, R, dtype=torch.float64, device=dev())
    gen64 = torch.full((B, case.H, R), -1, dtype=torch.long, device=dev())
    prompt_rows = case.P.to(dev()).reshape(-1).contiguous()
    rows = prompt_rows.clone()                                   # logical count n = 1 + step + P: generation j = step
    step = torch.zeros(1, dtype=torch.int32, device=dev())
    ws = torch.empty(ops.decode_workspace_bytes(B * Hq, D), dtype=torch.uint8, device=dev())
    P = case.P.to(dev()).long()
    near = 0
    for t in range(steps):
        step.fill_(t)
        v_before = victim.clone().reshape(B, case.H).long()
        out = _launch_heavy(case, hv, t, prompt_rows, rows, step, ws, Hh, state)
        full = t + 1 > R
        slot = v_before if full else P + t
        attended = torch.minimum(P + t + 1, P + R)
        _prewrite(case, ref, t, slot)
        want = _launch_existing(case, ref, case.q[t].to(dev()), (attended - 1).reshape(-1).contiguous().int(), ws)
        assert torch.equal(out, want), t                                          # (a)
        assert _same(hv, ref), t
        # (b) the fp64 twin over the same rows, from its own state
        probs = _probs64(case, hv, case.q[t].to(dev()), attended)
        held = min(t + 1, R)
        k_new = slot - P                                                           # [B, H]
        ar = torch.arange(R, device=dev())
        is_new = ar[None, None, :] == k_new[..., None]
        A64 = torch.where(is_new, 0.0, A64)
        gen64 = torch.where(is_new, t, gen64)
        idx = (P[..., None] + ar[None, None, :]).clamp_max(case.cap - 1)
        add = torch.gather(probs, 2, idx)
        A64 = torch.where(ar[None, None, :] < held, A64 + add, A64)
        assert torch.equal(gen.long(), gen64), t                                  # (d) the held set (slot by slot)
        err = (scores.double() - A64).abs()[..., :held]
        bar = REL * A64[..., :held] + ABS
        assert bool((err <= bar).all()), (t, float((err - bar).max()))
        if t + 1 >= R:
            last = t + 1 - (R - Hh)
            # (c) the GPU's victim is the rule's argmin over its own scores, exactly
            k_gpu, _ = _argmin(scores, gen, held, last)
            assert torch.equal(victim.reshape(B, case.H).long(), P + k_gpu), t
            # (d) the twin's own choice; near ties (two smallest candidates within the bound) follow the GPU's
            k64, a = _argmin(A64, gen64, held, last)
            two = a.topk(2, dim=-1, largest=False).values              # H + 1 >= 3 candidates
            tie = (two[..., 1] - two[..., 0]) <= 2 * (REL * two[..., 1] + ABS)
            differ = k64 != k_gpu
            assert not bool((differ & ~tie).any()), t
            near += int(tie.sum())
    # near ties are rare: on an H100, 55 of 217 344 choices over this whole matrix (DESIGN.md §4.9)
    assert near <= max(2, B * case.H * (steps - R + 1) // 50), near


@pytest.mark.parametrize("fp8,shared", FORMS)
def test_heavy_zero_is_the_window(oracle, libpkv, fp8, shared):
    from pyramidkv_b200 import ops
    dtype, D, Hq, Hkv, B, R = torch.bfloat16, 128, 32, 8, 3, 7
    steps = 3 * R
    case = Case(dtype, D, Hq, Hkv, fp8, shared, B, R, steps, seed=2)
    hv, win = case.device_bufs(), case.device_bufs()
    state = case.state()
    prompt_rows = case.P.to(dev()).reshape(-1).contiguous()
    step = torch.zeros(1, dtype=torch.int32, device=dev())
    ws = torch.empty(ops.decode_workspace_bytes(B * Hq, D), dtype=torch.uint8, device=dev())
    scales = (win[2], win[3]) if fp8 else None
    for t in range(steps):
        step.fill_(t)
        out = _launch_heavy(case, hv, t, prompt_rows, prompt_rows, step, ws, 0, state)
        want = ops.decode_attn_window(case.q[t].to(dev()), win[0], win[1], 1, case.kn[t].to(dev()), case.vn[t].to(dev()),
                                      prompt_rows, R, rows=prompt_rows, step=step, max_length=case.cap, workspace=ws,
                                      scales=scales, gqa=shared)
        assert torch.equal(out, want) and _same(hv, win), t
        ring = torch.tensor([max(j for j in range(t + 1) if j % R == k) if k <= t else -1 for k in range(R)], dtype=torch.int32)
        assert torch.equal(state[1].cpu(), ring.expand(B, case.H, R)), t


@pytest.mark.parametrize("fp8,shared", [(False, False), (True, True), (False, True)])
def test_graph_replay_across_the_wrap(oracle, libpkv, fp8, shared):
    from pyramidkv_b200 import ops
    dtype, D, Hq, Hkv, B, R = torch.bfloat16, 128, 32, 8, 3, 7
    steps = 4 * R
    case = Case(dtype, D, Hq, Hkv, fp8, shared, B, R, steps, seed=5)
    host, graph = case.device_bufs(), case.device_bufs()
    hstate, gstate = case.state(), case.state()
    prompt_rows = case.P.to(dev()).reshape(-1).contiguous()
    step = torch.zeros(1, dtype=torch.int32, device=dev())
    ws = torch.empty(ops.decode_workspace_bytes(B * Hq, D), dtype=torch.uint8, device=dev())
    ws2 = torch.empty_like(ws)
    scratch = torch.empty(ops.decode_heavy_workspace_bytes(B, Hq, R), dtype=torch.uint8, device=dev())
    q_s = case.q[0].to(dev())
    kn_s, vn_s = case.kn[0].to(dev()), case.vn[0].to(dev())
    out_s = torch.empty(B, Hq, D, dtype=dtype, device=dev())

    def launch(bufs, state):
        scales = (bufs[2], bufs[3]) if fp8 else None
        ops.decode_attn_heavy(q_s, bufs[0], bufs[1], 1, kn_s, vn_s, prompt_rows, R, R // 2, *state, rows=prompt_rows, step=step,
                              max_length=case.cap, workspace=ws2, scratch=scratch, out=out_s, scales=scales, gqa=shared)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        launch(graph, gstate)                   # warm-up; buffers and state are rebuilt below
    torch.cuda.current_stream().wait_stream(s)
    graph, gstate = case.device_bufs(), case.state()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        launch(graph, gstate)
    for t in range(steps):
        step.fill_(t)
        q_s.copy_(case.q[t].to(dev()))
        kn_s.copy_(case.kn[t].to(dev()))
        vn_s.copy_(case.vn[t].to(dev()))
        g.replay()
        want = _launch_heavy(case, host, t, prompt_rows, prompt_rows, step, ws, R // 2, hstate)
        assert torch.equal(out_s, want) and _same(graph, host), t
        assert all(torch.equal(x, y) for x, y in zip(gstate, hstate)), t


def test_out_of_range_and_argument_errors(oracle, libpkv):
    from pyramidkv_b200 import _lib, ops
    dtype, D, Hq, Hkv, B, R = torch.bfloat16, 64, 8, 4, 3, 5
    case = Case(dtype, D, Hq, Hkv, False, False, B, R, 2, seed=9, pmax=20)
    bufs = case.device_bufs()
    P = case.P.clone()
    rows = P.clone() + 2 * R                                    # n = P + 2R + 1: the window is full
    rows[0, 1] = -50                                            # n < 1
    P[1, 2] = -1                                                # P < 0
    P[2, 3] = case.cap - R + 1                                  # P + R above max_length
    rows[2, 3] = P[2, 3] + 2 * R
    bad = torch.zeros(B, Hq, dtype=torch.bool)
    bad[0, 1] = bad[1, 2] = bad[2, 3] = bad[0, 5] = True
    step = torch.zeros(1, dtype=torch.int32, device=dev())
    scores = torch.rand(B, Hq, R, device=dev())
    gen = torch.arange(R, dtype=torch.int32, device=dev()).repeat(B, Hq, 1)        # every held row is a candidate
    victim = (P.to(dev()).reshape(-1) + 1).int()
    victim[5] = int(P[0, 5]) + R                                # a victim outside [P, P + R)
    state = [scores, gen, victim]
    before = [x.clone() for x in bufs] + [x.clone() for x in state]
    d, w, h, keep = _descs(case, bufs, P, rows, step, state)
    rc = _lib.lib().pkv_decode_attn_heavy(C.byref(d), C.byref(w), C.byref(h), torch.cuda.current_stream().cuda_stream)
    assert rc == 0, _lib.last_error()
    torch.cuda.synchronize()
    out = keep["out"].cpu()
    assert bool(torch.isnan(out[bad]).all()) and not bool(torch.isnan(out[~bad]).any())
    for x, y in zip(bufs + state, before):
        xb, yb = x.cpu(), y.cpu()
        if xb.dim() == 1:
            xb, yb = xb.reshape(B, Hq), yb.reshape(B, Hq)
        assert torch.equal(xb[bad], yb[bad])                    # nothing written for the out-of-range heads
        assert not torch.equal(xb[~bad], yb[~bad])              # (the others did write)
    # argument errors
    cases = [("h", None, _lib.PKV_ERR_INVALID_ARG), ("struct_bytes", 8, _lib.PKV_ERR_INVALID_ARG),
             ("heavy", -1, _lib.PKV_ERR_INVALID_ARG), ("heavy", R, _lib.PKV_ERR_INVALID_ARG),
             ("scores", None, _lib.PKV_ERR_INVALID_ARG), ("gen", "misaligned", _lib.PKV_ERR_INVALID_ARG),
             ("victim", None, _lib.PKV_ERR_INVALID_ARG), ("scratch", None, _lib.PKV_ERR_INVALID_ARG),
             ("scratch_bytes", 16, _lib.PKV_ERR_WORKSPACE), ("k_new", None, _lib.PKV_ERR_INVALID_ARG),
             ("window", 0, _lib.PKV_ERR_INVALID_ARG)]
    for field, value, code in cases:
        d, w, h, keep = _descs(case, bufs, case.P, case.P, step, case.state())
        hp = C.byref(h)
        if field == "h":
            hp = None
        elif field == "k_new":
            d.k_new = d.v_new = None
        elif field == "window":
            w.window = value
        else:
            setattr(h, field, keep["gen"].data_ptr() + 2 if value == "misaligned" else value)
        rc = _lib.lib().pkv_decode_attn_heavy(C.byref(d), C.byref(w), hp, torch.cuda.current_stream().cuda_stream)
        assert rc == code, (field, value, rc)
    with pytest.raises(ValueError):
        ops.decode_attn_heavy(case.q[0].to(dev()), bufs[0], bufs[1], 1, case.kn[0].to(dev()), case.vn[0].to(dev()),
                              case.P.to(dev()).reshape(-1).contiguous(), R, R, *case.state())


def _descs(case, bufs, P, rows, step, state):
    from pyramidkv_b200 import _lib, ops
    keep = dict(q=case.q[0].to(dev()).contiguous(), kn=case.kn[0].to(dev()).contiguous(), vn=case.vn[0].to(dev()).contiguous(),
                out=torch.empty(case.B, case.Hq, case.D, dtype=case.dtype, device=dev()),
                prompt_rows=P.to(dev()).reshape(-1).contiguous().int(), rows=rows.to(dev()).reshape(-1).contiguous().int(),
                ws=torch.empty(ops.decode_workspace_bytes(case.B * case.Hq, case.D), dtype=torch.uint8, device=dev()),
                scratch=torch.empty(ops.decode_heavy_workspace_bytes(case.B, case.Hq, case.R), dtype=torch.uint8, device=dev()),
                gen=state[1])
    d = _lib.DecodeDesc()
    d.struct_bytes = C.sizeof(_lib.DecodeDesc)
    d.dtype, d.num_q_heads, d.num_kv_heads, d.head_dim = 0 if case.dtype == torch.bfloat16 else 1, case.Hq, case.Hkv, case.D
    d.device = dev().index or 0
    d.length = 1
    d.q, d.k_new, d.v_new = keep["q"].data_ptr(), keep["kn"].data_ptr(), keep["vn"].data_ptr()
    d.k_cache, d.v_cache, d.cache_stride_h, d.out = bufs[0].data_ptr(), bufs[1].data_ptr(), bufs[0].stride(1), keep["out"].data_ptr()
    d.workspace, d.workspace_bytes = keep["ws"].data_ptr(), keep["ws"].numel()
    w = _lib.DecodeWindow()
    w.struct_bytes = C.sizeof(_lib.DecodeWindow)
    w.num_seqs, w.cache_stride_b, w.gqa_shared, w.window = case.B, bufs[0].stride(0), int(case.shared), case.R
    w.rows, w.prompt_rows, w.step_dev, w.max_length = keep["rows"].data_ptr(), keep["prompt_rows"].data_ptr(), step.data_ptr(), case.cap
    h = _lib.DecodeHeavy()
    h.struct_bytes = C.sizeof(_lib.DecodeHeavy)
    h.heavy = case.R // 2
    h.scores, h.gen, h.victim = state[0].data_ptr(), state[1].data_ptr(), state[2].data_ptr()
    h.scratch, h.scratch_bytes = keep["scratch"].data_ptr(), keep["scratch"].numel()
    return d, w, h, keep
