"""-m gpu: GQA-shared caches (PKV_FLAG_GQA_SHARED, knob pkv_gqa_shared).

Eviction: the per-KV-head scores the library leaves at `pooled_kv_off` are the torch twin of the group reduction applied to the
library's own per-query-head `pooled`, bit for bit; the indices are the tie rule's top-k of them; the cache rows are byte copies
of K / V and the slack behind them is untouched; StreamingLLM and L2Norm give the flagless cache with the duplicate heads
removed. Decode: `pkv_decode_attn_batch_gqa(_fp8)` gives every query head the bits of `pkv_decode_attn_batch(_fp8)` over the
repeat-interleaved cache, appends the row once, writes nothing past each (sequence, KV head)'s rows, replays in a graph with
the host launch's bits, gives NaN for an out-of-range row count and takes the same launches for any batch size."""
import ctypes as C

import pytest
import torch

from gpu_util import dev, hf_layout
from oracle_fp8_backend import quantize_rows
from oracle_gqa_backend import group_reduce

pytestmark = pytest.mark.gpu

SENTINEL = 7.0
SENTINEL_BYTE = 0x55


def _bits(t):
    return t.view(torch.int16) if t.element_size() == 2 else t.view(torch.uint8)


# ---------------- eviction ----------------
# (method, Hq, Hkv, D, S, budget, W, dtype, pooling, kernel, layer)
EVICT = [
    ("pyramidkv", 32, 8, 128, 1024, 128, 32, torch.bfloat16, "maxpool", 7, 5),
    ("snapkv", 32, 8, 128, 12288, 2048, 32, torch.bfloat16, "avgpool", 5, 0),
    ("pyramidkv", 32, 8, 128, 32768, 2048, 32, torch.bfloat16, "maxpool", 7, 20),
    ("snapkv", 64, 8, 128, 4500, 2048, 32, torch.bfloat16, "maxpool", 7, 0),       # Llama-3-70B heads: G = 8
    ("pyramidkv", 16, 4, 64, 2048, 256, 16, torch.float16, "avgpool", 5, 3),        # D = 64, fp16
    ("h2o", 32, 8, 128, 1024, 128, 32, torch.float16, "avgpool", 5, 0),
    ("h2o", 64, 8, 128, 2048, 512, 32, torch.bfloat16, "avgpool", 5, 0),
    ("streamingllm", 32, 8, 128, 12288, 2048, 32, torch.bfloat16, "avgpool", 5, 0),
    ("streamingllm", 16, 4, 64, 1000, 128, 8, torch.float16, "avgpool", 5, 0),
    ("l2norm", 32, 8, 128, 4096, 512, 0, torch.bfloat16, "avgpool", 5, 0),
    ("l2norm", 64, 8, 64, 1024, 128, 0, torch.float16, "avgpool", 5, 0),
]


def _inputs(Hq, Hkv, S, D, dtype, seed):
    g = torch.Generator().manual_seed(seed)
    q = torch.randn(Hq, S, D, generator=g).to(dtype)
    k = torch.randn(Hkv, S, D, generator=g).to(dtype)
    v = torch.randn(Hkv, S, D, generator=g).to(dtype)
    return q, k, v


def _evict(method, qd, kd, vd, W, top_k, H, D, dtype, kernel, pooling, gqa_shared):
    from pyramidkv_b200 import ops
    kc = torch.full((H, top_k + W + 3, D), SENTINEL, dtype=dtype, device=dev())
    vc = torch.full_like(kc, SENTINEL)
    idx = torch.full((H, top_k), -1, dtype=torch.int64, device=dev())
    plan = ops.plan_evict(method, qd, kd, vd, W, top_k, kc, vc, kernel, pooling, idx_out=idx, gqa_shared=gqa_shared)
    ops.run_stage(plan, "all")
    return plan, kc, vc, idx


@pytest.mark.parametrize("method,Hq,Hkv,D,S,budget,W,dtype,pooling,kernel,layer", EVICT)
def test_eviction(oracle, libpkv, method, Hq, Hkv, D, S, budget, W, dtype, pooling, kernel, layer):
    from oracle import pkv_oracle as O
    from pyramidkv_b200 import ops
    G = Hq // Hkv
    q, k, v = _inputs(Hq, Hkv, S, D, dtype, S + Hq)
    qd, kd, vd = hf_layout(q), hf_layout(k), hf_layout(v)
    mode, top_k = ops.layer_budget(method, budget, W, 32, layer, S)
    assert mode == 1
    plan, kc, vc, idx = _evict(method, qd, kd, vd, W, top_k, Hkv, D, dtype, kernel, pooling, True)
    torch.cuda.synchronize()
    kc, vc, idx = kc.cpu(), vc.cpu(), idx.cpu()
    rows = top_k + W
    assert bool((kc[:, rows:] == SENTINEL).all()) and bool((vc[:, rows:] == SENTINEL).all())
    if method in ("streamingllm", "l2norm"):
        # the flagless cache with its G identical copies removed
        _, kq, vq, iq = _evict(method, qd, kd, vd, W, top_k, Hq, D, dtype, kernel, pooling, False)
        torch.cuda.synchronize()
        assert torch.equal(idx, iq.cpu()[::G])
        assert torch.equal(_bits(kc[:, :rows]), _bits(kq.cpu()[::G, :rows])) and torch.equal(_bits(vc[:, :rows]), _bits(vq.cpu()[::G, :rows]))
        return
    pooled = ops.ws_pooled(plan).cpu().contiguous()
    s_kv = ops.ws_pooled_kv(plan).cpu().contiguous()
    assert torch.equal(_bits(s_kv), _bits(group_reduce(pooled, G)))
    assert torch.equal(idx, O.topk(s_kv, top_k, O.TIE_LOWEST_INDEX))
    assert torch.equal(_bits(kc[:, :rows]), _bits(O.gather(k, idx, W, Hkv))) and torch.equal(_bits(vc[:, :rows]), _bits(O.gather(v, idx, W, Hkv)))


def test_eviction_refusals(libpkv):
    from pyramidkv_b200 import _lib, ops
    Hq, Hkv, S, D, W = 32, 8, 2048, 128, 32
    q, k, v = (t.to(dev()) for t in _inputs(Hq, Hkv, S, D, torch.bfloat16, 1))
    kc = torch.empty(Hkv, 128 + W, D, dtype=torch.bfloat16, device=dev())
    with pytest.raises(ValueError, match="Hkv"):
        ops.plan_evict("snapkv", q, k, v, W, 128, kc.new_empty(Hq, 128 + W, D), kc.new_empty(Hq, 128 + W, D), gqa_shared=True)
    for kw in (dict(fused=True), dict(single_launch=True)):
        with pytest.raises(NotImplementedError, match="GQA_SHARED"):
            ops.plan_evict("snapkv", q, k, v, W, 128, kc, kc.clone(), gqa_shared=True, **kw)
    # the layer batch is not built for the flag
    plans = [ops.plan_evict("snapkv", q, k, v, W, 128, kc, kc.clone(), gqa_shared=True, workspace=ws)
             for ws in ops.batch_workspaces(ops.plan_evict("snapkv", q, k, v, W, 128, kc, kc.clone(), gqa_shared=True), 2)]
    assert not ops.batch_supported(plans)
    with pytest.raises(NotImplementedError, match="GQA_SHARED"):
        ops.evict_prefill_batch(plans)
    # unknown flag bits are an argument error
    d = _lib.EvictDesc.from_buffer_copy(plans[0].desc)
    d.flags |= 1 << 12
    assert _lib.lib().pkv_evict_prefill(C.byref(d), torch.cuda.current_stream().cuda_stream) == _lib.PKV_ERR_INVALID_ARG
    assert b"flags" in _lib.lib().pkv_last_error()


# ---------------- decode ----------------
BASE = [0, 16, 255, 256, 2055]
STEPS = 3


def _decode_case(B, Hkv, G, D, dtype, fp8, seed):
    """Ragged rows per (sequence, KV head), a cache with sentinels behind them, and STEPS steps of inputs (CPU)."""
    g = torch.Generator().manual_seed(seed)
    Hq = Hkv * G
    rows = torch.tensor([[max(0, BASE[(b + j) % len(BASE)] - 3 * j) for j in range(Hkv)] for b in range(B)], dtype=torch.int32)
    cap = int(rows.max()) + STEPS + 2
    if fp8:
        kc = torch.full((B, Hkv, cap, D), SENTINEL_BYTE, dtype=torch.uint8)
        vc = torch.full_like(kc, SENTINEL_BYTE)
        ks = torch.full((B, Hkv, cap), -1.0)
        vs = torch.full_like(ks, -1.0)
    else:
        kc = torch.full((B, Hkv, cap, D), SENTINEL, dtype=dtype)
        vc = torch.full_like(kc, SENTINEL)
        ks = vs = None
    for b in range(B):
        for j in range(Hkv):
            n = int(rows[b, j])
            x, y = (torch.randn(n, D, generator=g) * 0.8).to(dtype), torch.randn(n, D, generator=g).to(dtype)
            if fp8:
                (kq, ksc), (vq, vsc) = quantize_rows(x), quantize_rows(y)
                kc[b, j, :n], ks[b, j, :n] = kq.view(torch.uint8), ksc
                vc[b, j, :n], vs[b, j, :n] = vq.view(torch.uint8), vsc
            else:
                kc[b, j, :n], vc[b, j, :n] = x, y
    q = (torch.randn(STEPS, B, Hq, D, generator=g) * 0.8).to(dtype)
    kn = torch.randn(STEPS, B, Hkv, D, generator=g).to(dtype)
    vn = torch.randn(STEPS, B, Hkv, D, generator=g).to(dtype)
    return rows, kc, vc, ks, vs, q, kn, vn


def _run(fp8, grouped, q, bufs, length, kn, vn, **kw):
    from pyramidkv_b200 import ops
    k, v, ks, vs = bufs
    if fp8:
        k8, v8 = k.view(torch.float8_e4m3fn), v.view(torch.float8_e4m3fn)
        fn = ops.decode_attn_batch_gqa_fp8 if grouped else ops.decode_attn_batch_fp8
        return fn(q, k8, v8, ks, vs, length, kn, vn, **kw)
    fn = ops.decode_attn_batch_gqa if grouped else ops.decode_attn_batch
    return fn(q, k, v, length, kn, vn, **kw)


def _expand(G, bufs):
    return [t.repeat_interleave(G, dim=1).contiguous() if t is not None else None for t in bufs]


def _check_bits_against_expanded(B, Hkv, G, D, dtype, fp8, seed):
    from pyramidkv_b200 import ops
    rows, kc, vc, ks, vs, q, kn, vn = _decode_case(B, Hkv, G, D, dtype, fp8, seed)
    Hq, cap = Hkv * G, kc.shape[2]
    grp = [t.to(dev()) if t is not None else None for t in (kc, vc, ks, vs)]
    ref = _expand(G, grp)
    rows_kv = rows.reshape(-1).to(dev())
    rows_q = rows.repeat_interleave(G, dim=1).reshape(-1).to(dev())
    step = torch.zeros(1, dtype=torch.int32, device=dev())
    ws_g = torch.empty(ops.decode_workspace_bytes(B * Hq, D), dtype=torch.uint8, device=dev())
    ws_r = torch.empty_like(ws_g)
    for t in range(STEPS):
        step.fill_(t)
        args = (q[t].to(dev()), 1, kn[t].to(dev()), vn[t].to(dev()))
        a = _run(fp8, True, args[0], grp, *args[1:], rows=rows_kv, step=step, max_length=cap, workspace=ws_g)
        b = _run(fp8, False, args[0], ref, *args[1:], rows=rows_q, step=step, max_length=cap, workspace=ws_r)
        assert torch.equal(_bits(a), _bits(b)), t
        assert not bool(a.isnan().any())
    torch.cuda.synchronize()
    # the group cache equals every copy of the expanded one: old rows, the appended rows, and the untouched slack
    for x, y in zip(grp, ref):
        if x is None:
            continue
        xe = x.cpu().repeat_interleave(G, dim=1)
        assert torch.equal(_bits(xe), _bits(y.cpu()))
    kg = grp[0].cpu()
    for b in range(B):
        for j in range(Hkv):
            n = int(rows[b, j])
            if fp8:
                assert bool((kg[b, j, n + STEPS:] == SENTINEL_BYTE).all())
                for t in range(STEPS):
                    wq, wsc = quantize_rows(kn[t, b, j])
                    assert torch.equal(kg[b, j, n + t], wq.view(torch.uint8)) and grp[2][b, j, n + t].item() == wsc.item()
            else:
                assert bool((kg[b, j, n + STEPS:] == SENTINEL).all())
                for t in range(STEPS):
                    assert torch.equal(_bits(kg[b, j, n + t]), _bits(kn[t, b, j]))


@pytest.mark.parametrize("fp8,dtype", [(False, torch.bfloat16), (False, torch.float16), (True, torch.bfloat16)])
@pytest.mark.parametrize("G", [2, 4, 8])
@pytest.mark.parametrize("D", [64, 128])
def test_decode_bits_equal_the_expanded_cache(libpkv, fp8, dtype, G, D):
    _check_bits_against_expanded(3, 2, G, D, dtype, fp8, seed=G * D)


@pytest.mark.parametrize("fp8", [False, True])
@pytest.mark.parametrize("B", [1, 64])
def test_decode_batch_sizes(libpkv, fp8, B):
    """Llama-3-8B heads (32 query heads, 8 KV heads)."""
    _check_bits_against_expanded(B, 8, 4, 128, torch.bfloat16, fp8, seed=B)


@pytest.mark.parametrize("fp8", [False, True])
def test_graph_replay_equals_host_launches(libpkv, fp8):
    from pyramidkv_b200 import ops
    B, Hkv, G, D = 3, 8, 4, 128
    rows, kc, vc, ks, vs, q, kn, vn = _decode_case(B, Hkv, G, D, torch.bfloat16, fp8, seed=9)
    cap = kc.shape[2]
    rows_d = rows.reshape(-1).to(dev())
    qd, knd, vnd = q[0].to(dev()), kn[0].to(dev()), vn[0].to(dev())
    ws = torch.empty(ops.decode_workspace_bytes(B * Hkv * G, D), dtype=torch.uint8, device=dev())
    todev = lambda: [t.to(dev()) if t is not None else None for t in (kc, vc, ks, vs)]
    host_bufs, step = todev(), torch.zeros(1, dtype=torch.int32, device=dev())
    host = []
    for t in range(STEPS):
        step.fill_(t)
        host.append(_run(fp8, True, qd, host_bufs, 1, knd, vnd, rows=rows_d, step=step, max_length=cap, workspace=ws).clone())
    gbufs, gstep = todev(), torch.zeros(1, dtype=torch.int32, device=dev())
    out = torch.empty(B, Hkv * G, D, dtype=torch.bfloat16, device=dev())
    _run(fp8, True, qd, todev(), 1, knd, vnd, rows=rows_d, step=gstep, max_length=cap, workspace=ws, out=out)   # warm-up
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        _run(fp8, True, qd, gbufs, 1, knd, vnd, rows=rows_d, step=gstep, max_length=cap, workspace=ws, out=out)
        gstep.add_(1)
    replayed = []
    for _ in range(STEPS):
        graph.replay()
        replayed.append(out.clone())
    torch.cuda.synchronize()
    for a, b in zip(host, replayed):
        assert torch.equal(_bits(a), _bits(b))
    for a, b in zip(host_bufs, gbufs):
        if a is not None:
            assert torch.equal(_bits(a), _bits(b))


@pytest.mark.parametrize("fp8", [False, True])
def test_out_of_range_row_count_gives_nan(libpkv, fp8):
    """A (sequence, KV head) whose count falls below 1 reads and writes nothing; its G query heads are NaN, the others not."""
    B, Hkv, G, D = 2, 4, 4, 64
    rows, kc, vc, ks, vs, q, kn, vn = _decode_case(B, Hkv, G, D, torch.bfloat16, fp8, seed=4)
    rows[1, 2] = -5
    bufs = [t.to(dev()) if t is not None else None for t in (kc, vc, ks, vs)]
    before = [t.clone() for t in bufs if t is not None]
    out = _run(fp8, True, q[0].to(dev()), bufs, 1, kn[0].to(dev()), vn[0].to(dev()), rows=rows.reshape(-1).to(dev()))
    torch.cuda.synchronize()
    o = out.cpu().float().reshape(B, Hkv, G, D)
    assert bool(o[1, 2].isnan().all())
    o[1, 2] = 0
    assert not bool(o.isnan().any())
    for a, b in zip([t for t in bufs if t is not None], before):
        assert torch.equal(_bits(a[1, 2].cpu()), _bits(b[1, 2].cpu()))


@pytest.mark.parametrize("fp8", [False, True])
def test_one_launch_whatever_the_batch_size(libpkv, fp8):
    from pyramidkv_b200 import _lib
    D, Hkv, G = 128, 8, 4
    counts = []
    for B in (1, 8):
        rows, kc, vc, ks, vs, q, kn, vn = _decode_case(B, Hkv, G, D, torch.bfloat16, fp8, seed=B)
        bufs = [t.to(dev()) if t is not None else None for t in (kc, vc, ks, vs)]
        rows_d, step = torch.full((B * Hkv,), 299, dtype=torch.int32, device=dev()), torch.zeros(1, dtype=torch.int32, device=dev())
        call = lambda: _run(fp8, True, q[0].to(dev()), bufs, 1, kn[0].to(dev()), vn[0].to(dev()), rows=rows_d, step=step,
                            max_length=bufs[0].shape[2])
        call()
        n0 = _lib.launch_count()
        call()
        counts.append(_lib.launch_count() - n0)
    torch.cuda.synchronize()
    assert counts[0] == counts[1] == 2             # 300 rows: two splits, then the combine kernel


def test_decode_argument_errors(libpkv):
    from pyramidkv_b200 import _lib, ops
    B, Hkv, G, D, cap = 2, 4, 4, 128, 16
    kc = torch.zeros(B, Hkv, cap, D, dtype=torch.bfloat16, device=dev())
    q = torch.zeros(B, Hkv * G, D, dtype=torch.bfloat16, device=dev())
    kn = torch.zeros(B, Hkv, D, dtype=torch.bfloat16, device=dev())
    ok = torch.full((B * Hkv,), 3, dtype=torch.int32, device=dev())
    ops.decode_attn_batch_gqa(q, kc, kc.clone(), 1, kn, kn, rows=ok)
    with pytest.raises(ValueError, match="B\\*Hkv"):
        ops.decode_attn_batch_gqa(q, kc, kc.clone(), 1, kn, kn, rows=torch.full((B * Hkv * G,), 3, dtype=torch.int32, device=dev()))
    with pytest.raises(ValueError, match="k_new"):
        ops.decode_attn_batch_gqa(q, kc, kc.clone(), 1, q, q, rows=ok)
    with pytest.raises(ValueError, match="capacity"):
        ops.decode_attn_batch_gqa(q, kc, kc.clone(), cap + 1, kn, kn)
    with pytest.raises(ValueError, match="multiple"):
        ops.decode_attn_batch_gqa(q[:, :Hkv * G - 1], kc, kc.clone(), 1, kn, kn)
    with pytest.raises(NotImplementedError, match="group size"):   # G = 3 is not built
        ops.decode_attn_batch_gqa(torch.zeros(B, Hkv * 3, D, dtype=torch.bfloat16, device=dev()), kc, kc.clone(), 1, kn, kn)
    kq = torch.zeros(B, Hkv, cap, D, dtype=torch.float8_e4m3fn, device=dev())
    ks = torch.zeros(B, Hkv, cap, device=dev())
    ops.decode_attn_batch_gqa_fp8(q, kq, kq.clone(), ks, ks.clone(), 1, kn, kn, rows=ok)
    with pytest.raises(ValueError, match="scales"):
        ops.decode_attn_batch_gqa_fp8(q, kq, kq.clone(), ks[:, :, :-1].contiguous(), ks.clone(), 1, kn, kn, rows=ok)
    # the C entry points: strides too small, misaligned pointers, null scales
    out = torch.empty_like(q)
    d = _lib.DecodeDesc()
    d.struct_bytes = C.sizeof(_lib.DecodeDesc)
    d.dtype, d.num_q_heads, d.num_kv_heads, d.head_dim, d.device = 0, Hkv * G, Hkv, D, dev().index or 0
    d.length, d.q, d.out = 4, q.data_ptr(), out.data_ptr()
    d.k_cache, d.v_cache, d.cache_stride_h = kc.data_ptr(), kc.data_ptr(), cap * D
    ws = torch.empty(ops.decode_workspace_bytes(B * Hkv * G, D), dtype=torch.uint8, device=dev())
    d.workspace, d.workspace_bytes = ws.data_ptr(), ws.numel()
    L, st = _lib.lib(), torch.cuda.current_stream().cuda_stream
    assert L.pkv_decode_attn_batch_gqa(C.byref(d), B, Hkv * cap * D, None, None, cap, st) == _lib.PKV_OK
    assert L.pkv_decode_attn_batch_gqa(C.byref(d), B, Hkv * cap * D - 8, None, None, cap, st) == _lib.PKV_ERR_INVALID_ARG
    assert L.pkv_decode_attn_batch_gqa(C.byref(d), B, Hkv * cap * D, None, None, cap + 1, st) == _lib.PKV_ERR_INVALID_ARG
    assert L.pkv_decode_attn_batch_gqa(C.byref(d), B, Hkv * cap * D, ok.data_ptr() + 2, None, cap, st) == _lib.PKV_ERR_INVALID_ARG
    assert L.pkv_decode_attn_batch_gqa(C.byref(d), 0, Hkv * cap * D, None, None, cap, st) == _lib.PKV_ERR_INVALID_ARG
    d.k_cache, d.v_cache, d.cache_stride_h = kq.data_ptr(), kq.data_ptr(), cap * D
    fn = L.pkv_decode_attn_batch_gqa_fp8
    assert fn(C.byref(d), B, Hkv * cap * D, None, None, cap, ks.data_ptr(), ks.data_ptr(), cap, Hkv * cap, st) == _lib.PKV_OK
    assert fn(C.byref(d), B, Hkv * cap * D, None, None, cap, None, ks.data_ptr(), cap, Hkv * cap, st) == _lib.PKV_ERR_INVALID_ARG
    assert fn(C.byref(d), B, Hkv * cap * D, None, None, cap, ks.data_ptr(), ks.data_ptr(), cap, Hkv * cap - 1, st) == _lib.PKV_ERR_INVALID_ARG
    d.dtype = 7
    assert fn(C.byref(d), B, Hkv * cap * D, None, None, cap, ks.data_ptr(), ks.data_ptr(), cap, Hkv * cap, st) == _lib.PKV_ERR_UNSUPPORTED_DTYPE
    torch.cuda.synchronize()
