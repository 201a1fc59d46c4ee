"""Prompt-lookup speculation in the continuous loop on the H100 (-m gpu): `pkv_decode_attn_packed` against fp64 attention
(the bound of tests/test_gpu_spec.py) with ragged counts 0 .. Q at random starts, its stored rows, the rows it must not
touch and its zero rows; the dense layout through the packed entry bit for bit against `pkv_decode_attn_multi`;
`pkv_spec_pack` bit for bit against its CPU twin; graph replay against host launches; and the loop end to end at the
Llama-3-8B attention geometry, graph on against graph off."""
import pytest
import torch

import oracle_continuous_spec_backend as OCSB
import test_gpu_spec as TGS
from oracle_fp8_backend import quantize_rows

pytestmark = pytest.mark.gpu


def _dev():
    return torch.device("cuda", 0)


def _layout(B, Q, g, gaps=True):
    """Random counts in [0, Q] (some 0) and ascending starts with random gaps; returns (start, count, M)."""
    count = torch.randint(0, Q + 1, (B,), generator=g, dtype=torch.int32)
    count[torch.rand(B, generator=g) < 0.25] = 0
    count[0] = Q
    start, r = [], int(torch.randint(0, 3, (1,), generator=g)) if gaps else 0
    for b in range(B):
        start.append(r)
        r += int(count[b]) + (int(torch.randint(0, 3, (1,), generator=g)) if gaps else 0)
    return torch.tensor(start, dtype=torch.int32), count, r + (2 if gaps else 0)


def _packed_inputs(q, kn, vn, start, count, M):
    B, Q, Hq, D = q.shape
    qp = torch.full((1, M, Hq, D), float("nan"), dtype=q.dtype)
    kp = torch.full((1, M, kn.shape[2], D), float("nan"), dtype=q.dtype)
    vp = kp.clone()
    for b in range(B):
        s0, c = int(start[b]), int(count[b])
        qp[0, s0:s0 + c], kp[0, s0:s0 + c], vp[0, s0:s0 + c] = q[b, :c], kn[b, :c], vn[b, :c]
    return qp, kp, vp


@pytest.mark.parametrize("dtype, D, Hq, Hkv, fp8, gqa, Q, B, n_max", TGS.CASES + [(torch.bfloat16, 128, 32, 8, False, False, 9, 12, 2000)])
def test_packed_attention(libpkv, dtype, D, Hq, Hkv, fp8, gqa, Q, B, n_max):
    from pyramidkv_b200 import ops
    q, kn, vn, rows, (kb, vb, sc), cap = TGS._setup(dtype, D, Hq, Hkv, fp8, gqa, Q, B, n_max, seed=7)
    g = torch.Generator().manual_seed(11)
    start, count, M = _layout(B, Q, g)
    qp, kp, vp = _packed_inputs(q, kn, vn, start, count, M)
    H = kb.shape[1]
    before = [t.clone() for t in (kb, vb) + (() if sc is None else sc)]
    out = ops.decode_attn_packed(qp.to(_dev()), kb, vb, kp.to(_dev()), vp.to(_dev()), start.to(_dev()), count.to(_dev()), Q,
                                 rows=rows.reshape(-1).to(_dev()), scales=sc, gqa=gqa)
    torch.cuda.synchronize()
    out = out.cpu()
    owned = torch.zeros(M, dtype=torch.bool)
    G = Hq // Hkv
    for b in range(B):
        s0, c = int(start[b]), int(count[b])
        owned[s0:s0 + c] = True
        for ch in range(H):
            n0 = int(rows[b, ch])
            gk = ch if gqa else ch // G
            if sc is None:
                assert torch.equal(kb[b, ch, n0:n0 + c].cpu(), kn[b, :c, gk]) and torch.equal(vb[b, ch, n0:n0 + c].cpu(), vn[b, :c, gk])
            else:
                for buf, s_, new in ((kb, sc[0], kn), (vb, sc[1], vn)):
                    qb, s = quantize_rows(new[b, :c, gk])
                    assert torch.equal(buf.view(torch.uint8)[b, ch, n0:n0 + c].cpu(), qb.view(torch.uint8))
                    assert torch.equal(s_[b, ch, n0:n0 + c].cpu(), s)
            for now, old in zip((kb, vb) + (() if sc is None else sc), before):
                # nothing outside the slot's new rows (all of its rows when its count is 0)
                assert torch.equal(now[b, ch, :n0].cpu().view(torch.uint8), old[b, ch, :n0].cpu().view(torch.uint8))
                assert torch.equal(now[b, ch, n0 + c:].cpu().view(torch.uint8), old[b, ch, n0 + c:].cpu().view(torch.uint8))
            if c == 0:
                continue
            K = TGS._rows_of(kb, None if sc is None else sc[0], b, ch, n0 + c)
            V = TGS._rows_of(vb, None if sc is None else sc[1], b, ch, n0 + c)
            for h in (range(ch * G, ch * G + G) if gqa else [ch]):
                ref, s_max, A = TGS._ref(q[b, :c, h], K, V, n0, D ** -0.5)
                bound = TGS._bound(ref, dtype, D, n0 + c, s_max, A, float(V.abs().max()), TGS._splits(Hq, n0 + c))
                err = (out[0, s0:s0 + c, h].double() - ref).abs()
                assert bool((err <= bound).all()), f"(b={b}, h={h}, n0={n0}, count={c}): error {float(err.max()):.3g}"
    assert not out[0, ~owned].view(torch.int16).any(), "rows no sequence owns must be zero"
    print(f"counts {count.tolist()}, M {M}")


def test_dense_layout_bit_equal(libpkv):
    from pyramidkv_b200 import ops
    for case in (TGS.CASES[0], TGS.CASES[3], TGS.CASES[6], TGS.CASES[9]):
        dtype, D, Hq, Hkv, fp8, gqa, Q, B, n_max = case
        q, kn, vn, rows, (kb, vb, sc), cap = TGS._setup(dtype, D, Hq, Hkv, fp8, gqa, Q, B, n_max, seed=3)
        kb2, vb2 = kb.clone(), vb.clone()
        sc2 = None if sc is None else (sc[0].clone(), sc[1].clone())
        r = rows.reshape(-1).to(_dev())
        dense = ops.decode_attn_multi(q.to(_dev()), kb, vb, kn.to(_dev()), vn.to(_dev()), rows=r, scales=sc, gqa=gqa)
        start = torch.arange(B, dtype=torch.int32) * Q
        count = torch.full((B,), Q, dtype=torch.int32)
        packed = ops.decode_attn_packed(q.reshape(1, B * Q, Hq, D).to(_dev()), kb2, vb2, kn.reshape(1, B * Q, Hkv, D).to(_dev()),
                                        vn.reshape(1, B * Q, Hkv, D).to(_dev()), start.to(_dev()), count.to(_dev()), Q, rows=r,
                                        scales=sc2, gqa=gqa)
        torch.cuda.synchronize()
        assert torch.equal(dense.reshape(1, B * Q, Hq, D).view(torch.int16), packed.view(torch.int16)), f"{case}: outputs"
        assert torch.equal(kb.view(torch.uint8), kb2.view(torch.uint8)) and torch.equal(vb.view(torch.uint8), vb2.view(torch.uint8))
        if sc is not None:
            assert torch.equal(sc[0], sc2[0]) and torch.equal(sc[1], sc2[1])


def _pack_states(B, K, D, device, seed):
    from pyramidkv_b200.generate import PackState, SpecState
    g = torch.Generator().manual_seed(seed)
    lengths = [int(x) for x in torch.randint(2, 300, (B,), generator=g)]
    prompts = [torch.randint(0, 5, (n,), generator=g).to(device) for n in lengths]
    first = torch.randint(0, 5, (B,), generator=g).to(device)
    budgets = [int(x) for x in torch.randint(0, 12, (B,), generator=g)]
    st = SpecState(prompts, first, 40, K, 2, [4], 0, device, budgets=budgets)
    step = torch.zeros(1, dtype=torch.int32, device=device)
    return st, PackState(B, K, D, step, device)


@pytest.mark.parametrize("B", [1, 8, 64, 165])
def test_pack_matches_twin(libpkv, B):
    from pyramidkv_b200 import ops
    K = 6
    for D in sorted({1, K, B, max(1, B // 2), B * K}):
        gpu, gpk = _pack_states(B, K, D, _dev(), B + D)
        cpu, cpk = _pack_states(B, K, D, torch.device("cpu"), B + D)
        ops.prompt_lookup(gpu)
        OCSB.OSB.lookup_twin(cpu)
        for step in (0, 1, B - 1, B + 3, 12345):
            for st, pk in ((gpu, gpk), (cpu, cpk)):
                pk.step.fill_(step)
            ops.spec_pack(gpu, gpk)
            OCSB.pack_twin(cpu, cpk)
            for name in ("ids", "pos", "row_start", "row_count", "totals"):
                assert torch.equal(getattr(gpk, name).cpu(), getattr(cpk, name)), f"D={D} step {step}: {name}"
            assert torch.equal(gpu.draft_len.cpu(), cpu.draft_len), f"D={D} step {step}: draft_len"
            ops.prompt_lookup(gpu)                    # the lookup's drafts again for the next step
            OCSB.OSB.lookup_twin(cpu)


def test_graph_replay_equals_host_launch(libpkv):
    from pyramidkv_b200 import ops
    dtype, D, Hq, Hkv, Q, B = torch.bfloat16, 128, 32, 8, 5, 6
    q, kn, vn, rows, (kb, vb, _), cap = TGS._setup(dtype, D, Hq, Hkv, False, False, Q, B, 3000, seed=5)
    st, pk = _pack_states(B, Q - 1, 7, _dev(), 9)
    ops.prompt_lookup(st)
    M = pk.ids.numel()
    g = torch.Generator().manual_seed(1)
    qp = torch.randn(1, M, Hq, D, generator=g).to(dtype).to(_dev())
    kp = torch.randn(1, M, Hkv, D, generator=g).to(dtype).to(_dev())
    vp = torch.randn(1, M, Hkv, D, generator=g).to(dtype).to(_dev())
    r = rows.reshape(-1).to(_dev())
    ws = torch.empty(ops.decode_workspace_bytes(B * Hq * Q, D), dtype=torch.uint8, device=_dev())
    out = torch.empty(1, M, Hq, D, dtype=dtype, device=_dev())
    snap = [t.clone() for t in (st.draft_len,)]

    def step():
        ops.spec_pack(st, pk)
        ops.decode_attn_packed(qp, kb, vb, kp, vp, pk.row_start, pk.row_count, Q, rows=r, workspace=ws, out=out)

    step()                                          # warm-up (kernel attributes), then restore
    st.draft_len.copy_(snap[0])
    pk.totals.zero_()
    graph = torch.cuda.CUDAGraph()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        with torch.cuda.graph(graph):
            step()
    torch.cuda.current_stream().wait_stream(s)
    graph.replay()
    torch.cuda.synchronize()
    got = [t.clone() for t in (out, pk.ids, pk.row_start, pk.row_count, pk.totals, st.draft_len)]
    st.draft_len.copy_(snap[0])
    pk.totals.zero_()
    step()
    torch.cuda.synchronize()
    want = (out, pk.ids, pk.row_start, pk.row_count, pk.totals, st.draft_len)
    for a, b in zip(got, want):
        assert torch.equal(a.view(torch.uint8) if a.dtype == dtype else a, b.view(torch.uint8) if b.dtype == dtype else b), \
            "a graph replay differs from a host launch"


@pytest.fixture(autouse=True)
def _restore():
    yield
    from pyramidkv.monkeypatch import restore
    restore()


@pytest.mark.parametrize("method, fp8, gqa", [("pyramidkv", False, False), ("pyramidkv", True, True), ("adakv", False, False)])
def test_loop_end_to_end(libpkv, method, fp8, gqa, monkeypatch):
    import test_continuous_spec as TCS
    import test_spec as TS
    from pyramidkv_b200 import generate as G
    model = TGS._model_8b_geometry(method, fp8, gqa)
    prompts = [p.reshape(1, -1).to(_dev()) for p in TS._prompts(model, [2100, 1500, 900, 1200, 700], repeat=True)]
    caps = [40, 25, 33, 12, 30]
    TCS._check(model, prompts, caps, 3, 5, monkeypatch=monkeypatch, use_graph=False)
    on, st_on = G.greedy_generate_continuous(model, prompts, caps, 3, prompt_lookup_num_tokens=5, use_graph=True,
                                             return_stats=True)
    off = G.greedy_generate_continuous(model, prompts, caps, 3, prompt_lookup_num_tokens=5, use_graph=False)
    for a, b in zip(on, off):
        assert torch.equal(a, b), "graph on and graph off differ"
    # the admitted prompts are no longer than the first ones: only a buffer regrowth captures again
    assert st_on["graph_captures"] == 1 + st_on["regrowths"], st_on
    print({k: st_on[k] for k in ("decode_steps", "live_slot_steps", "granted_drafts", "accepted_drafts", "graph_captures")})
