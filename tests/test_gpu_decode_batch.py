"""-m gpu: one decode launch for several sequences (`pkv_decode_attn_batch`, ops.decode_attn_batch). Every sequence's output
and appended row are byte-equal to the one-sequence graph (or ragged) launch at the same step, within 1e-3 + 1 ulp of the
exact attention, and nothing past each (sequence, head)'s rows is written."""
import pytest
import torch

from gpu_util import dev

pytestmark = pytest.mark.gpu

ATOL = 1e-3
BASE = [0, 16, 255, 256, 2055]             # rows before the append: {1, 17, 256, 257, 2056} attended at step 0
STEPS = 10
SENTINEL = 7.0


def _ulp(t):
    mant = 8 if t.dtype == torch.bfloat16 else 11
    return torch.exp2(torch.floor(torch.log2(t.float().abs().clamp_min(1e-8))) - (mant - 1))


def _case(dtype, D, Hq, Hkv, ragged, seed=0):
    g = torch.Generator().manual_seed(seed + D + Hq)
    B, cap = len(BASE), max(BASE) + STEPS + 2
    rows = torch.tensor([[max(0, r - (7 * h) % 40) if ragged else r for h in range(Hq)] for r in BASE], dtype=torch.int32)
    k = torch.full((B, Hq, cap, D), SENTINEL, dtype=dtype)
    v = torch.full((B, Hq, cap, D), SENTINEL, dtype=dtype)
    for b in range(B):
        for h in range(Hq):
            n = int(rows[b, h])
            k[b, h, :n] = (torch.randn(n, D, generator=g) * 0.8).to(dtype)
            v[b, h, :n] = torch.randn(n, D, generator=g).to(dtype)
    q = (torch.randn(STEPS, B, Hq, D, generator=g) * 0.8).to(dtype)
    kn = torch.randn(STEPS, B, Hkv, D, generator=g).to(dtype)
    vn = torch.randn(STEPS, B, Hkv, D, generator=g).to(dtype)
    return rows, k, v, q, kn, vn


GEOMS = [(torch.bfloat16, 128, 32, 8), (torch.float16, 128, 8, 8), (torch.bfloat16, 64, 16, 2)]


@pytest.mark.parametrize("ragged", [False, True])
@pytest.mark.parametrize("dtype,D,Hq,Hkv", GEOMS)
def test_batch_bit_identical_to_single_sequence(oracle, libpkv, dtype, D, Hq, Hkv, ragged):
    from pyramidkv_b200 import ops
    rows, k, v, q, kn, vn = _case(dtype, D, Hq, Hkv, ragged)
    B, cap = k.shape[0], k.shape[2]
    kb, vb = k.to(dev()), v.to(dev())
    ks, vs = k.to(dev()), v.to(dev())
    rows_d = rows.to(dev()).reshape(-1)
    step = torch.zeros(1, dtype=torch.int32, device=dev())
    ws = torch.empty(ops.decode_workspace_bytes(B * Hq, D), dtype=torch.uint8, device=dev())
    for t in range(3):                                                   # three steps: the row counts grow by one each
        step.fill_(t)
        out = ops.decode_attn_batch(q[t].to(dev()), kb, vb, 1, kn[t].to(dev()), vn[t].to(dev()), rows=rows_d, step=step,
                                    max_length=cap, workspace=ws)
        for b in range(B):
            if ragged:
                one = ops.decode_attn(q[t, b].to(dev()), ks[b], vs[b], 1, kn[t, b].to(dev()), vn[t, b].to(dev()), step=step,
                                      max_length=cap, head_rows=rows_d[b * Hq:(b + 1) * Hq].contiguous())
            else:
                one = ops.decode_attn(q[t, b].to(dev()), ks[b], vs[b], int(rows[b, 0]) + 1, kn[t, b].to(dev()), vn[t, b].to(dev()),
                                      step=step, max_length=cap)
            assert torch.equal(out[b].view(torch.int16), one.view(torch.int16)), (t, b)
        assert torch.equal(kb.view(torch.int16), ks.view(torch.int16)) and torch.equal(vb.view(torch.int16), vs.view(torch.int16))
        # accuracy against the exact attention, head by head over that head's rows
        kc, vc, o = kb.cpu(), vb.cpu(), out.cpu()
        for b in range(B):
            for h in range(Hq):
                T = int(rows[b, h]) + t + 1
                exact = oracle.decode_attn_exact(q[t, b, h:h + 1], kc[b, h:h + 1], vc[b, h:h + 1], T)
                assert torch.all((o[b, h].float() - exact[0]).abs() <= ATOL + _ulp(o[b, h])), (b, h)
    # the appended rows are k_new / v_new of the sequence's kv head, and nothing else was written
    kc = kb.cpu()
    G = Hq // Hkv
    for b in range(B):
        for h in range(Hq):
            n = int(rows[b, h])
            for t in range(3):
                assert torch.equal(kc[b, h, n + t], kn[t, b, h // G])
            assert torch.equal(kc[b, h, :n], k[b, h, :n]) and bool((kc[b, h, n + 3:] == SENTINEL).all())


def test_graph_replay_equals_host_launches(libpkv):
    from pyramidkv_b200 import ops
    dtype, D, Hq, Hkv = torch.bfloat16, 128, 32, 8
    rows, k, v, q, kn, vn = _case(dtype, D, Hq, Hkv, ragged=True, seed=5)
    B, cap = k.shape[0], k.shape[2]
    rows_d = rows.to(dev()).reshape(-1)
    qd, knd, vnd = q[0].to(dev()), kn[0].to(dev()), vn[0].to(dev())
    ws = torch.empty(ops.decode_workspace_bytes(B * Hq, D), dtype=torch.uint8, device=dev())
    # host launches, step 0..9
    kh, vh = k.to(dev()), v.to(dev())
    step = torch.zeros(1, dtype=torch.int32, device=dev())
    host = []
    for t in range(STEPS):
        step.fill_(t)
        host.append(ops.decode_attn_batch(qd, kh, vh, 1, knd, vnd, rows=rows_d, step=step, max_length=cap, workspace=ws).clone())
    # one captured launch (+ the step increment), replayed ten times
    kg, vg = k.to(dev()), v.to(dev())
    gstep = torch.zeros(1, dtype=torch.int32, device=dev())
    out = torch.empty(B, Hq, D, dtype=dtype, device=dev())
    ops.decode_attn_batch(qd, kg.clone(), vg.clone(), 1, knd, vnd, rows=rows_d, step=gstep, max_length=cap, workspace=ws, out=out)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        ops.decode_attn_batch(qd, kg, vg, 1, knd, vnd, rows=rows_d, step=gstep, max_length=cap, workspace=ws, out=out)
        gstep.add_(1)
    replayed = []
    for _ in range(STEPS):
        graph.replay()
        replayed.append(out.clone())
    torch.cuda.synchronize()
    for a, b in zip(host, replayed):
        assert torch.equal(a.view(torch.int16), b.view(torch.int16))
    assert torch.equal(kh.view(torch.int16), kg.view(torch.int16)) and torch.equal(vh.view(torch.int16), vg.view(torch.int16))


def test_one_launch_whatever_the_batch_size(libpkv):
    from pyramidkv_b200 import _lib, ops
    D, Hq, Hkv, cap = 128, 32, 8, 400
    counts = []
    for B in (1, 8):
        kb = torch.randn(B, Hq, cap, D, device=dev()).bfloat16()
        q = torch.randn(B, Hq, D, device=dev()).bfloat16()
        kn = torch.randn(B, Hkv, D, device=dev()).bfloat16()
        rows = torch.full((B * Hq,), 299, dtype=torch.int32, device=dev())
        step = torch.zeros(1, dtype=torch.int32, device=dev())
        ops.decode_attn_batch(q, kb, kb.clone(), 1, kn, kn, rows=rows, step=step)
        n0 = _lib.launch_count()
        ops.decode_attn_batch(q, kb, kb.clone(), 1, kn, kn, rows=rows, step=step)
        counts.append(_lib.launch_count() - n0)
    torch.cuda.synchronize()
    assert counts[0] == counts[1] >= 1


def test_argument_errors(libpkv):
    from pyramidkv_b200 import ops
    B, Hq, D, cap = 2, 4, 128, 16
    kb = torch.zeros(B, Hq, cap, D, dtype=torch.bfloat16, device=dev())
    q = torch.zeros(B, Hq, D, dtype=torch.bfloat16, device=dev())
    ok = torch.full((B * Hq,), 3, dtype=torch.int32, device=dev())
    ops.decode_attn_batch(q, kb, kb.clone(), 1, rows=ok)
    with pytest.raises(ValueError, match="int32"):
        ops.decode_attn_batch(q, kb, kb.clone(), 1, rows=ok.long())
    with pytest.raises(ValueError, match="B\\*Hq"):
        ops.decode_attn_batch(q, kb, kb.clone(), 1, rows=ok[:Hq].contiguous())
    with pytest.raises(ValueError, match="capacity"):
        ops.decode_attn_batch(q, kb, kb.clone(), 1, rows=torch.tensor([3] * 7 + [cap], dtype=torch.int32, device=dev()))
    with pytest.raises(ValueError, match="capacity"):
        ops.decode_attn_batch(q, kb, kb.clone(), cap + 1)
    with pytest.raises(ValueError, match="num_seqs"):
        ops.decode_attn_batch(q[:0], kb[:0], kb[:0].clone(), 1)
