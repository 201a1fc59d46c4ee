"""-m gpu: the decode window (`pkv_decode_attn_window`, ops.decode_attn_window) over every cache form: 16-bit and E4M3 rows,
a cache per query head and GQA-shared (G = 2, 4, 8), ragged prompt rows P per (sequence, cache head), windows R = 1 ... 300
driven for 3R steps. At every step (a) the output and every byte of the buffers equal the existing batch entry point run
without k_new over the same buffer with the new row already at its ring slot and P + min(g, R) rows, and (b) the output is
within 1e-3 + 1 ulp of the fp64 attention over exactly the rows the semantics name. (c) R >= the steps taken is bit-identical
to the unwindowed launch, (d) one captured launch replayed across the wrap equals host launches, and (e) counts out of range
give NaN outputs and write nothing, bad arguments PKV_ERR_INVALID_ARG."""
import ctypes as C

import pytest
import torch

from gpu_util import dev
from oracle_fp8_backend import quantize_rows
from oracle_window_backend import window_slot

pytestmark = pytest.mark.gpu

ATOL = 1e-3
SENTINEL = 7.0
# (dtype, D, Hq, Hkv): G = 4, 8, 2
GEOMS = [(torch.bfloat16, 128, 32, 8), (torch.float16, 64, 16, 2), (torch.bfloat16, 64, 8, 4)]
# (B, R): one long window over prompts long enough for several splits, small windows over large batches
RUNS = [(1, 300), (3, 7), (3, 64), (64, 1), (64, 7)]


def _ulp(t):
    mant = 8 if t.dtype == torch.bfloat16 else 11
    return torch.exp2(torch.floor(torch.log2(t.float().abs().clamp_min(1e-8))) - (mant - 1))


class Case:
    """Buffers of one cache form, two copies (window launch / reference), and the inputs of `steps` steps."""

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
        # the KV head whose new row cache head c stores
        self.kv_of = torch.arange(self.H) if shared else torch.arange(Hq) // (Hq // Hkv)

    def device_bufs(self):
        return [t.to(dev()) for t in self.bufs]


def _launch_window(case, bufs, t, prompt_rows, rows, step, ws, window=None):
    from pyramidkv_b200 import ops
    k, v = bufs[0], bufs[1]
    scales = (bufs[2], bufs[3]) if case.fp8 else None
    return ops.decode_attn_window(case.q[t].to(dev()), k, v, 1, case.kn[t].to(dev()), case.vn[t].to(dev()), prompt_rows,
                                  window or case.R, rows=rows, step=step, max_length=case.cap, workspace=ws, scales=scales,
                                  gqa=case.shared)


def _launch_existing(case, bufs, q, rows, ws, k_new=None, v_new=None, step=None):
    """The existing batch entry point of the form: `1 + rows (+ *step)` rows, appending k_new / v_new when given."""
    from pyramidkv_b200 import ops
    if case.fp8:
        fn = ops.decode_attn_batch_gqa_fp8 if case.shared else ops.decode_attn_batch_fp8
        return fn(q, bufs[0], bufs[1], bufs[2], bufs[3], 1, k_new, v_new, rows=rows, step=step, max_length=case.cap, workspace=ws)
    fn = ops.decode_attn_batch_gqa if case.shared else ops.decode_attn_batch
    return fn(q, bufs[0], bufs[1], 1, k_new, v_new, rows=rows, step=step, max_length=case.cap, workspace=ws)


def _prewrite(case, bufs, t, slot):
    """Store step t's new row of every (sequence, cache head) at its ring slot, as the kernel stores it."""
    bi = torch.arange(case.B)[:, None].expand(case.B, case.H)
    ci = torch.arange(case.H)[None, :].expand(case.B, case.H)
    kn, vn = case.kn[t][:, case.kv_of], case.vn[t][:, case.kv_of]            # [B, H, D]
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


def _exact(case, bufs, q, attended):
    """fp64 attention of every (sequence, query head) over rows [0, attended[b, c]) of its cache head."""
    if case.fp8:
        K = bufs[0].double() * bufs[2].double()[..., None]
        V = bufs[1].double() * bufs[3].double()[..., None]
    else:
        K, V = bufs[0].double(), bufs[1].double()
    G = case.Hq // case.H
    K, V = K.repeat_interleave(G, dim=1), V.repeat_interleave(G, dim=1)
    A = attended.to(dev()).repeat_interleave(G, dim=1)                         # [B, Hq]
    s = torch.einsum("bhd,bhrd->bhr", q.double(), K) * case.D ** -0.5
    s = s.masked_fill(torch.arange(case.cap, device=dev())[None, None, :] >= A[..., None], float("-inf"))
    return torch.einsum("bhr,bhrd->bhd", torch.softmax(s, dim=-1), V)


def _same(a, b):
    return all(torch.equal(x.view(torch.uint8) if x.dtype == torch.float8_e4m3fn else x,
                           y.view(torch.uint8) if y.dtype == torch.float8_e4m3fn else y) for x, y in zip(a, b))


@pytest.mark.parametrize("B,R", RUNS)
@pytest.mark.parametrize("fp8,shared", [(False, False), (True, False), (False, True), (True, True)])
@pytest.mark.parametrize("dtype,D,Hq,Hkv", GEOMS)
def test_window_steps_equal_existing_entry_and_oracle(oracle, libpkv, dtype, D, Hq, Hkv, fp8, shared, B, R):
    from pyramidkv_b200 import ops
    steps = 3 * R
    case = Case(dtype, D, Hq, Hkv, fp8, shared, B, R, steps)
    win, ref = case.device_bufs(), case.device_bufs()
    prompt_rows = case.P.to(dev()).reshape(-1).contiguous()
    rows = prompt_rows.clone()                                   # logical count n = 1 + step + P
    step = torch.zeros(1, dtype=torch.int32, device=dev())
    ws = torch.empty(ops.decode_workspace_bytes(B * Hq, D), dtype=torch.uint8, device=dev())
    for t in range(steps):
        step.fill_(t)
        out = _launch_window(case, win, t, prompt_rows, rows, step, ws)
        n = case.P + 1 + t
        slot = torch.where(n > case.P + R, case.P + (n - 1 - case.P) % R, n - 1).long()
        attended = torch.minimum(n, case.P + R)
        assert (int(slot[0, 0]), int(attended[0, 0])) == window_slot(int(n[0, 0]), int(case.P[0, 0]), R)
        _prewrite(case, ref, t, slot)
        want = _launch_existing(case, ref, case.q[t].to(dev()), (attended - 1).to(dev()).reshape(-1).contiguous().int(), ws)
        assert torch.equal(out, want), t                                          # (a) the output bits
        assert _same(win, ref), t                                                 # (a) every byte of the buffers
        exact = _exact(case, win, case.q[t].to(dev()), attended)                   # (b)
        err = (out.double() - exact).abs()
        bar = ATOL + _ulp(exact.to(dtype)).double()
        assert bool((err <= bar).all()), (t, float((err - bar).max()))


@pytest.mark.parametrize("fp8,shared", [(False, False), (True, False), (False, True), (True, True)])
@pytest.mark.parametrize("dtype,D,Hq,Hkv", GEOMS)
def test_window_at_least_the_steps_is_the_unwindowed_launch(oracle, libpkv, dtype, D, Hq, Hkv, fp8, shared):
    from pyramidkv_b200 import ops
    B, steps = 3, 40
    case = Case(dtype, D, Hq, Hkv, fp8, shared, B, steps, steps, seed=3)
    win, ref = case.device_bufs(), case.device_bufs()
    prompt_rows = case.P.to(dev()).reshape(-1).contiguous()
    step = torch.zeros(1, dtype=torch.int32, device=dev())
    ws = torch.empty(ops.decode_workspace_bytes(B * Hq, D), dtype=torch.uint8, device=dev())
    for t in range(steps):
        step.fill_(t)
        for R in (steps, steps + 1000):
            w = [x.clone() for x in win]
            out = _launch_window(case, w, t, prompt_rows, prompt_rows, step, ws, window=R)
        want = _launch_existing(case, ref, case.q[t].to(dev()), prompt_rows, ws, case.kn[t].to(dev()), case.vn[t].to(dev()), step)
        win = w
        assert torch.equal(out, want) and _same(win, ref), t


@pytest.mark.parametrize("fp8,shared", [(False, False), (True, True)])
def test_graph_replay_across_the_wrap(oracle, libpkv, fp8, shared):
    from pyramidkv_b200 import ops
    dtype, D, Hq, Hkv, B, R = torch.bfloat16, 128, 32, 8, 3, 7
    steps = 3 * R
    case = Case(dtype, D, Hq, Hkv, fp8, shared, B, R, steps, seed=5)
    host, graph = case.device_bufs(), case.device_bufs()
    prompt_rows = case.P.to(dev()).reshape(-1).contiguous()
    step = torch.zeros(1, dtype=torch.int32, device=dev())
    ws = torch.empty(ops.decode_workspace_bytes(B * Hq, D), dtype=torch.uint8, device=dev())
    ws2 = torch.empty_like(ws)
    q_s = case.q[0].to(dev())
    kn_s, vn_s = case.kn[0].to(dev()), case.vn[0].to(dev())
    out_s = torch.empty(B, Hq, D, dtype=dtype, device=dev())
    scales = (graph[2], graph[3]) if fp8 else None
    # warm up on the side stream, then capture one launch; the warm-up's row is rewritten by the first replay
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        ops.decode_attn_window(q_s, graph[0], graph[1], 1, kn_s, vn_s, prompt_rows, R, rows=prompt_rows, step=step,
                               max_length=case.cap, workspace=ws2, out=out_s, scales=scales, gqa=shared)
    torch.cuda.current_stream().wait_stream(s)
    graph = case.device_bufs()
    scales = (graph[2], graph[3]) if fp8 else None
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        ops.decode_attn_window(q_s, graph[0], graph[1], 1, kn_s, vn_s, prompt_rows, R, rows=prompt_rows, step=step,
                               max_length=case.cap, workspace=ws2, out=out_s, scales=scales, gqa=shared)
    for t in range(steps):
        step.fill_(t)
        q_s.copy_(case.q[t].to(dev()))
        kn_s.copy_(case.kn[t].to(dev()))
        vn_s.copy_(case.vn[t].to(dev()))
        g.replay()
        want = _launch_window(case, host, t, prompt_rows, prompt_rows, step, ws)
        assert torch.equal(out_s, want) and _same(graph, host), t


def test_out_of_range_and_argument_errors(oracle, libpkv):
    from pyramidkv_b200 import _lib, ops
    dtype, D, Hq, Hkv, B, R = torch.bfloat16, 64, 8, 4, 3, 5
    case = Case(dtype, D, Hq, Hkv, False, False, B, R, 2, seed=9, pmax=20)
    bufs = case.device_bufs()
    before = [x.clone() for x in bufs]
    P = case.P.clone()
    rows = P.clone() + 2 * R                                    # n = P + 2R + 1: the ring is full
    rows[0, 1] = -50                                            # n < 1
    P[1, 2] = -1                                                # P < 0
    P[2, 3] = case.cap - R + 1                                  # P + R above max_length
    rows[2, 3] = P[2, 3] + 2 * R
    bad = torch.zeros(B, Hq, dtype=torch.bool)
    bad[0, 1] = bad[1, 2] = bad[2, 3] = True
    step = torch.zeros(1, dtype=torch.int32, device=dev())
    # the host check refuses counts above max_length, so launch through the C entry point directly
    d, w, keep = _descs(case, bufs, P, rows, step)
    rc = _lib.lib().pkv_decode_attn_window(C.byref(d), C.byref(w), torch.cuda.current_stream().cuda_stream)
    assert rc == 0, _lib.last_error()
    torch.cuda.synchronize()
    out = keep["out"].cpu()
    assert bool(torch.isnan(out[bad]).all()) and not bool(torch.isnan(out[~bad]).any())
    for x, y in zip(bufs, before):
        xb = x.cpu()
        yb = y.cpu()
        assert torch.equal(xb[bad], yb[bad])                    # nothing written for the out-of-range heads
    # argument errors
    for field, value in (("window", 0), ("window", -3), ("prompt_rows", None), ("prompt_rows", "misaligned"), ("struct_bytes", 8)):
        d, w, keep = _descs(case, bufs, case.P, case.P, step)
        if value == "misaligned":
            value = keep["prompt_rows"].data_ptr() + 2
        setattr(w, field, value)
        rc = _lib.lib().pkv_decode_attn_window(C.byref(d), C.byref(w), torch.cuda.current_stream().cuda_stream)
        assert rc == _lib.PKV_ERR_INVALID_ARG, (field, value, rc)
    with pytest.raises(ValueError):
        ops.decode_attn_window(case.q[0].to(dev()), bufs[0], bufs[1], 1, case.kn[0].to(dev()), case.vn[0].to(dev()),
                               case.P.to(dev()).reshape(-1).contiguous(), 0)


def _descs(case, bufs, P, rows, step):
    from pyramidkv_b200 import _lib, ops
    keep = dict(q=case.q[0].to(dev()).contiguous(), kn=case.kn[0].to(dev()).contiguous(), vn=case.vn[0].to(dev()).contiguous(),
                out=torch.empty(case.B, case.Hq, case.D, dtype=case.dtype, device=dev()),
                prompt_rows=P.to(dev()).reshape(-1).contiguous().int(), rows=rows.to(dev()).reshape(-1).contiguous().int(),
                ws=torch.empty(ops.decode_workspace_bytes(case.B * case.Hq, case.D), dtype=torch.uint8, device=dev()))
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
    return d, w, keep
