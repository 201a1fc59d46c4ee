"""Prompt-lookup speculative decoding on the H100 (-m gpu): `pkv_decode_attn_multi` against fp64 attention over exactly the
rows each query sees (the error bound of tests/test_gpu_landscapes.py: one ulp of the output plus eps * max|v|, eps derived
from the fp32 sums the kernel forms), its stored rows, its out-of-range rule and its graph replay; `pkv_prompt_lookup` and
`pkv_spec_step` bit for bit against their CPU twins (oracle/spec.py); and the loop end to end at the Llama-3-8B attention
geometry, graph on against graph off and against the CPU checks of tests/test_spec.py."""
import pytest
import torch

import oracle_spec_backend as OSB
from oracle_fp8_backend import dequantize, quantize_rows

pytestmark = pytest.mark.gpu

U = 2.0 ** -24


def _dev():
    return torch.device("cuda", 0)


def _ref(q, K, V, n0, scale):
    """fp64 attention of q [Q, D] over K / V [n0 + Q, D] (float64) with query j seeing rows [0, n0 + j + 1)."""
    Qn = q.shape[0]
    s = (q.double() @ K.T) * scale
    mask = torch.arange(n0 + Qn)[None, :] > (n0 + torch.arange(Qn))[:, None]
    p = torch.softmax(s.masked_fill(mask, float("-inf")), dim=-1)
    A = float(((q.double().abs() @ K.abs().T) * scale).max())
    return p @ V, float(s.abs().max()), A


def _splits(Hq, T):
    """decode_splits_for (pkv_internal.h): the split rule of the batched decode, which the verify launch follows."""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    return max(1, min(-(-T // 256), -(-(sms * 4) // Hq), 64))


def _bound(ref, dtype, D, T, s_max, A, vmax, ns):
    chunk = -(-T // ns)
    eps = U * (2 * (D + 2) * A + 4 * s_max + 2 * (chunk + ns + 16))
    mant = 8 if dtype == torch.bfloat16 else 11
    ulp = torch.exp2(torch.floor(torch.log2(ref.abs().clamp(min=1e-30))) - (mant - 1))
    return ulp + eps * vmax


# (dtype, D, Hq, Hkv, fp8, gqa, Q, B, largest n0)
CASES = [(torch.bfloat16, 128, 32, 8, False, False, 5, 2, 3000), (torch.float16, 128, 32, 8, False, False, 16, 1, 26000),
         (torch.bfloat16, 64, 8, 8, False, False, 1, 3, 700), (torch.bfloat16, 128, 32, 8, True, False, 11, 2, 9000),
         (torch.float16, 64, 16, 8, False, True, 2, 2, 4000), (torch.bfloat16, 128, 16, 4, False, True, 16, 1, 26000),
         (torch.bfloat16, 128, 32, 4, True, True, 5, 2, 12000), (torch.float16, 128, 16, 2, False, True, 11, 1, 2000),
         (torch.bfloat16, 128, 16, 2, True, True, 16, 2, 5000), (torch.float16, 64, 8, 8, True, False, 2, 4, 300)]


def _setup(dtype, D, Hq, Hkv, fp8, gqa, Q, B, n_max, seed=0):
    g = torch.Generator().manual_seed(seed)
    H = Hkv if gqa else Hq
    cap = n_max + Q + 8
    rows = torch.randint(1, n_max + 1, (B, H), generator=g, dtype=torch.int32)
    rows[0, 0] = n_max
    k16 = torch.randn(B, H, cap, D, generator=g).to(dtype)
    v16 = torch.randn(B, H, cap, D, generator=g).to(dtype)
    q = torch.randn(B, Q, Hq, D, generator=g).to(dtype)
    kn = torch.randn(B, Q, Hkv, D, generator=g).to(dtype)
    vn = torch.randn(B, Q, Hkv, D, generator=g).to(dtype)
    if fp8:
        kq, ks = quantize_rows(k16)
        vq, vs = quantize_rows(v16)
        bufs = (kq.to(_dev()), vq.to(_dev()), (ks.to(_dev()), vs.to(_dev())))
    else:
        bufs = (k16.to(_dev()), v16.to(_dev()), None)
    return q, kn, vn, rows, bufs, cap


def _rows_of(buf, scales, b, c, n):
    if scales is None:
        return buf[b, c, :n].double().cpu()
    return dequantize(buf[b, c, :n], scales[b, c, :n]).double()


@pytest.mark.parametrize("dtype, D, Hq, Hkv, fp8, gqa, Q, B, n_max", CASES)
def test_verify_attention(libpkv, dtype, D, Hq, Hkv, fp8, gqa, Q, B, n_max):
    from pyramidkv_b200 import ops
    q, kn, vn, rows, (kb, vb, sc), cap = _setup(dtype, D, Hq, Hkv, fp8, gqa, Q, B, n_max)
    H = kb.shape[1]
    before_k, before_v = kb.clone(), vb.clone()
    before_s = None if sc is None else (sc[0].clone(), sc[1].clone())
    rows_d = rows.reshape(-1).to(_dev())
    # HF's layout: q [B, Q, Hq, D] as a view of the projection output
    qd, knd, vnd = q.to(_dev()), kn.to(_dev()), vn.to(_dev())
    out = ops.decode_attn_multi(qd, kb, vb, knd, vnd, rows=rows_d, scales=sc, gqa=gqa)
    torch.cuda.synchronize()
    G = Hq // Hkv
    scale = D ** -0.5
    for b in range(B):
        for c in range(H):
            n0 = int(rows[b, c])
            g = c if gqa else c // G
            # the new rows as stored: byte copies, or the E4M3 rule; nothing else written
            if sc is None:
                assert torch.equal(kb[b, c, n0:n0 + Q].cpu(), kn[b, :, g]) and torch.equal(vb[b, c, n0:n0 + Q].cpu(), vn[b, :, g])
            else:
                for buf, s_, new in ((kb, sc[0], kn), (vb, sc[1], vn)):
                    qb, s = quantize_rows(new[b, :, g])
                    assert torch.equal(buf.view(torch.uint8)[b, c, n0:n0 + Q].cpu(), qb.view(torch.uint8))
                    assert torch.equal(s_[b, c, n0:n0 + Q].cpu(), s)
            olds = ((kb, before_k), (vb, before_v)) + (() if sc is None else ((sc[0], before_s[0]), (sc[1], before_s[1])))
            for buf, old in olds:
                assert torch.equal(buf[b, c, :n0].view(torch.uint8), old[b, c, :n0].view(torch.uint8))
                assert torch.equal(buf[b, c, n0 + Q:].view(torch.uint8), old[b, c, n0 + Q:].view(torch.uint8))
            K = _rows_of(kb, None if sc is None else sc[0], b, c, n0 + Q)
            V = _rows_of(vb, None if sc is None else sc[1], b, c, n0 + Q)
            heads = range(c * G, c * G + G) if gqa else [c]
            for h in heads:
                ref, s_max, A = _ref(q[b, :, h], K, V, n0, scale)
                bound = _bound(ref, dtype, D, n0 + Q, s_max, A, float(V.abs().max()), _splits(Hq, n0 + Q))
                err = (out[b, :, h].double().cpu() - ref).abs()
                assert bool((err <= bound).all()), f"(b={b}, h={h}, n0={n0}): error {float(err.max()):.3g}"


def test_verify_out_of_range_and_graph(libpkv):
    from pyramidkv_b200 import ops
    dtype, D, Hq, Hkv, Q, B = torch.bfloat16, 128, 32, 8, 5, 2
    q, kn, vn, rows, (kb, vb, _), cap = _setup(dtype, D, Hq, Hkv, False, False, Q, B, 2000)
    qd, knd, vnd = q.to(_dev()), kn.to(_dev()), vn.to(_dev())
    ws = torch.empty(ops.decode_workspace_bytes(B * Hq * Q, D), dtype=torch.uint8, device=_dev())
    out = torch.empty(B, Q, Hq, D, dtype=dtype, device=_dev())
    rows_d = rows.reshape(-1).to(_dev())
    ops.decode_attn_multi(qd, kb, vb, knd, vnd, rows=rows_d, workspace=ws, out=out)     # warm-up, in range
    rows[1, 3] = cap - Q + 1            # one row past the capacity
    rows[0, 5] = -1
    rows_d.copy_(rows.reshape(-1).to(_dev()))
    kb0 = kb.clone()
    torch.cuda.synchronize()
    # the capacity check of the wrapper reads the rows; the kernel's own rule is what a captured launch relies on
    graph = torch.cuda.CUDAGraph()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        with torch.cuda.graph(graph):
            ops.decode_attn_multi(qd, kb, vb, knd, vnd, rows=rows_d, workspace=ws, out=out)
    torch.cuda.current_stream().wait_stream(s)
    graph.replay()
    torch.cuda.synchronize()
    assert torch.isnan(out[1, :, 3]).all() and torch.isnan(out[0, :, 5]).all()
    assert torch.equal(kb[1, 3], kb0[1, 3]) and torch.equal(kb[0, 5], kb0[0, 5])
    assert not torch.isnan(out[0, :, 0]).any()
    host = torch.empty_like(out)
    rows[1, 3], rows[0, 5] = 7, 9
    rows_d.copy_(rows.reshape(-1).to(_dev()))
    ops.decode_attn_multi(qd, kb, vb, knd, vnd, rows=rows_d, workspace=ws, out=host)
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(out.view(torch.int16), host.view(torch.int16)), "a graph replay differs from a host launch"


# ---- lookup and step kernels against their twins ----
def _state(B, K, N, n_eos, lengths, V, device, seed):
    from pyramidkv_b200.generate import SpecState
    g = torch.Generator().manual_seed(seed)
    prompts = [torch.randint(0, V, (n,), generator=g) for n in lengths]
    first = torch.randint(0, V, (B,), generator=g)
    eos = list(range(V, V + n_eos - 1)) + ([V - 1] if n_eos else [])
    return SpecState([p.to(device) for p in prompts], first.to(device), 40, K, N, eos or None, 0, device)


def _same(a, b, what):
    for name in ("hist", "hist_len", "budget", "done", "out", "out_len", "ids", "pos", "draft_len", "emitted"):
        x, y = getattr(a, name).cpu(), getattr(b, name).cpu()
        if name == "hist":
            for r in range(x.shape[0]):
                n = int(a.hist_len[r])
                assert torch.equal(x[r, :n], y[r, :n]), f"{what}: hist row {r}"
            continue
        assert torch.equal(x, y), f"{what}: {name}"


@pytest.mark.parametrize("B, K, N, n_eos, L", [(1, 4, 2, 0, 131072), (8, 15, 8, 4, 3000), (64, 1, 1, 1, 500),
                                               (8, 7, 3, 2, 20000), (64, 10, 5, 0, 64)])
def test_lookup_and_step_match_twins(libpkv, B, K, N, n_eos, L):
    from pyramidkv_b200 import ops
    lengths = [max(2, L - 37 * b) for b in range(B)]
    V = 7 if L < 10000 else 50
    gpu = _state(B, K, N, n_eos, lengths, V, _dev(), 1)
    cpu = _state(B, K, N, n_eos, lengths, V, torch.device("cpu"), 1)
    ops.prompt_lookup(gpu)
    OSB.lookup_twin(cpu)
    _same(gpu, cpu, "lookup")
    g = torch.Generator().manual_seed(2)
    rows_c = [torch.randint(0, 1000, (B * 8,), generator=g, dtype=torch.int32) for _ in range(33)]
    rows_g = [r.to(_dev()) for r in rows_c]
    for step in range(4):
        t = cpu.ids.roll(-1, dims=1).clone()                         # drafts accepted ...
        flip = torch.rand(B, K + 1, generator=g) < 0.3                # ... up to a random mismatch
        t[flip] = torch.randint(0, V, (int(flip.sum()),), generator=g)
        cpu.tokens.copy_(t)
        gpu.tokens.copy_(t.to(_dev()))
        ops.spec_step(gpu, rows_g)
        OSB.step_twin(cpu, rows_c)
        _same(gpu, cpu, f"step {step}")
        for i, (rg, rc) in enumerate(zip(rows_g, rows_c)):
            assert torch.equal(rg.cpu(), rc), f"step {step}: layer {i} row counts"


# ---- end to end ----
def _model_8b_geometry(method="pyramidkv", fp8=False, gqa=False):
    from pyramidkv_b200 import runner
    import transformers
    runner.patch(method)
    cfg = transformers.LlamaConfig(hidden_size=4096, intermediate_size=1024, num_hidden_layers=2, num_attention_heads=32,
                                   num_key_value_heads=8, head_dim=128, vocab_size=4096, rope_theta=500000.0,
                                   max_position_embeddings=65536)
    cfg._attn_implementation = "sdpa"
    torch.manual_seed(42)
    with torch.device(_dev()):
        model = transformers.LlamaForCausalLM(cfg).to(torch.bfloat16).eval()
    runner.set_knobs(model, method, 256)
    model.config.pkv_fused_rope = True
    if fp8:
        model.config.pkv_kv_cache_dtype = "fp8_e4m3"
    if gqa:
        model.config.pkv_gqa_shared = True
    return model


@pytest.fixture(autouse=True)
def _restore():
    yield
    from pyramidkv.monkeypatch import restore
    restore()


@pytest.mark.parametrize("method, fp8, gqa", [("pyramidkv", False, False), ("pyramidkv", True, True), ("adakv", False, False)])
def test_loop_end_to_end(libpkv, method, fp8, gqa):
    import test_spec as TS
    from pyramidkv_b200 import generate as G
    model = _model_8b_geometry(method, fp8, gqa)
    prompts = [p.to(_dev()) for p in TS._prompts(model, [1500, 900, 2100], repeat=True)]
    gen, dec = TS._check_loop(model, prompts, 40, 5)
    graphed = G.greedy_generate_batch(model, prompts, 40, prompt_lookup_num_tokens=5, use_graph=True)
    eager = G.greedy_generate_batch(model, prompts, 40, prompt_lookup_num_tokens=5, use_graph=False)
    for a, b, p, g in zip(graphed, eager, prompts, gen):
        assert torch.equal(a, b), "graph on and graph off differ"
        assert a[p.numel() + 1:].tolist() == g
