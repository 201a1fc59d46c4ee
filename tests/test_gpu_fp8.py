"""-m gpu: the FP8 cache kernels. `pkv_cache_quantize_fp8` (ops.cache_quantize_fp8) writes exactly the bytes and scales of
the torch rule and nothing past each (sequence, head)'s rows, in one launch for a whole prompt. `pkv_decode_attn_batch_fp8`
(ops.decode_attn_batch_fp8) is within 1e-3 + 1 output ulp of the exact attention over the dequantised rows, stores the rule
applied to the new token, writes nothing past the rows, gives every sequence the bits of its num_seqs = 1 launch, replays
in a CUDA graph with the host launch's bits and takes the same launches for any batch size."""
import pytest
import torch

from gpu_util import dev
from oracle_fp8_backend import dequantize, quantize_rows

pytestmark = pytest.mark.gpu

ATOL = 1e-3
BASE = [0, 16, 255, 256, 2055]             # rows before the append: {1, 17, 256, 257, 2056} attended at step 0
STEPS = 10
SENTINEL_BYTE = 0x55
SENTINEL_SCALE = -1.0


def _ulp(t):
    mant = 8 if t.dtype == torch.bfloat16 else 11
    return torch.exp2(torch.floor(torch.log2(t.float().abs().clamp_min(1e-8))) - (mant - 1))


def _u8(t):
    return t.view(torch.uint8)


def _fp8_empty(shape, device):
    q = torch.full(shape, SENTINEL_BYTE, dtype=torch.uint8, device=device).view(torch.float8_e4m3fn)
    s = torch.full(shape[:3], SENTINEL_SCALE, dtype=torch.float32, device=device)
    return q, s


def _rows16(n, D, dtype, g, scale=1.0):
    x = torch.randn(n, D, generator=g) * scale
    if n > 4:                                       # a zero row, a tiny row, a row with one large element
        x[1] = 0
        x[2] *= 1e-4
        x[3, 7] = 60.0
    return x.to(dtype)


# ---------------- pkv_cache_quantize_fp8 ----------------
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("D", [64, 128])
@pytest.mark.parametrize("n_layers,ragged", [(1, False), (32, False), (3, True), (32, True)])
def test_quantize_bit_equal_to_the_rule(libpkv, dtype, D, n_layers, ragged):
    from pyramidkv_b200 import _lib, ops
    g = torch.Generator().manual_seed(D + n_layers)
    B, Hq = 2, 4
    items, want = [], []
    for l in range(n_layers):
        rows = 40 + 13 * l
        cap16, cap8 = rows + 7, rows + 3
        k = torch.zeros(B, Hq, cap16, D, dtype=dtype)
        v = torch.zeros_like(k)
        for b in range(B):
            for h in range(Hq):
                k[b, h, :rows] = _rows16(rows, D, dtype, g, 2.0)
                v[b, h, :rows] = _rows16(rows, D, dtype, g)
        counts = torch.tensor([[rows - (5 * h + 3 * b + l) % 17 for h in range(Hq)] for b in range(B)], dtype=torch.int32) if ragged \
            else torch.full((B, Hq), rows, dtype=torch.int32)
        kq, ks = _fp8_empty((B, Hq, cap8, D), dev())
        vq, vs = _fp8_empty((B, Hq, cap8, D), dev())
        items.append((k.to(dev()), v.to(dev()), kq, vq, ks, vs, rows, counts.reshape(-1).to(dev()) if ragged else None))
        want.append((k, v, counts))
    ops.cache_quantize_fp8(items[:1])                                   # load the module before counting
    n0 = _lib.launch_count()
    ops.cache_quantize_fp8(items)
    assert _lib.launch_count() - n0 == 1
    torch.cuda.synchronize()
    for (k, v, counts), it in zip(want, items):
        for src, q, s in ((k, it[2], it[4]), (v, it[3], it[5])):
            qc, sc = _u8(q.cpu()), s.cpu()
            for b in range(B):
                for h in range(Hq):
                    n = int(counts[b, h])
                    wq, ws = quantize_rows(src[b, h, :n])
                    assert torch.equal(qc[b, h, :n], _u8(wq)), (b, h)
                    assert torch.equal(sc[b, h, :n], ws), (b, h)
                    assert bool((qc[b, h, n:] == SENTINEL_BYTE).all()) and bool((sc[b, h, n:] == SENTINEL_SCALE).all())


def test_quantize_whole_prompt_is_one_launch(libpkv):
    """Llama-3-8B geometry at budget 128: the 32 layers of one prompt convert in one launch."""
    from pyramidkv_b200 import _lib, ops
    items = []
    for l in range(32):
        k = torch.randn(1, 32, 128 + 256, 128, device=dev()).bfloat16()
        kq, ks = _fp8_empty((1, 32, 128 + 256, 128), dev())
        vq, vs = _fp8_empty((1, 32, 128 + 256, 128), dev())
        items.append((k, k, kq, vq, ks, vs, 128, None))
    ops.cache_quantize_fp8(items)
    n0 = _lib.launch_count()
    ops.cache_quantize_fp8(items)
    assert _lib.launch_count() - n0 == 1
    torch.cuda.synchronize()


# ---------------- pkv_decode_attn_batch_fp8 ----------------
def _case(dtype, D, Hq, Hkv, ragged, seed=0):
    g = torch.Generator().manual_seed(seed + D + Hq)
    B, cap = len(BASE), max(BASE) + STEPS + 2
    rows = torch.tensor([[max(0, r - (7 * h) % 40) if ragged else r for h in range(Hq)] for r in BASE], dtype=torch.int32)
    kq = torch.full((B, Hq, cap, D), SENTINEL_BYTE, dtype=torch.uint8)
    vq = torch.full((B, Hq, cap, D), SENTINEL_BYTE, dtype=torch.uint8)
    ks = torch.full((B, Hq, cap), SENTINEL_SCALE)
    vs = torch.full((B, Hq, cap), SENTINEL_SCALE)
    for b in range(B):
        for h in range(Hq):
            n = int(rows[b, h])
            q8, s8 = quantize_rows((torch.randn(n, D, generator=g) * 0.8).to(dtype))
            kq[b, h, :n], ks[b, h, :n] = _u8(q8), s8
            q8, s8 = quantize_rows(torch.randn(n, D, generator=g).to(dtype))
            vq[b, h, :n], vs[b, h, :n] = _u8(q8), s8
    q = (torch.randn(STEPS, B, Hq, D, generator=g) * 0.8).to(dtype)
    kn = torch.randn(STEPS, B, Hkv, D, generator=g).to(dtype)
    vn = torch.randn(STEPS, B, Hkv, D, generator=g).to(dtype)
    return rows, kq.view(torch.float8_e4m3fn), vq.view(torch.float8_e4m3fn), ks, vs, q, kn, vn


def _to(*ts):
    return [t.to(dev()) for t in ts]


GEOMS = [(torch.bfloat16, 128, 32, 8), (torch.float16, 128, 8, 8), (torch.bfloat16, 64, 16, 2), (torch.float16, 64, 8, 2)]


@pytest.mark.parametrize("ragged", [False, True])
@pytest.mark.parametrize("dtype,D,Hq,Hkv", GEOMS)
def test_decode_batch_accuracy_append_and_solo_bits(oracle, libpkv, dtype, D, Hq, Hkv, ragged):
    from pyramidkv_b200 import ops
    rows, kq, vq, ks, vs, q, kn, vn = _case(dtype, D, Hq, Hkv, ragged)
    B, cap = kq.shape[0], kq.shape[2]
    kb, vb, kbs, vbs = _to(kq, vq, ks, vs)                  # the batch
    solo = [_to(kq[b:b + 1], vq[b:b + 1], ks[b:b + 1], vs[b:b + 1]) for b in range(B)]
    rows_d = rows.to(dev()).reshape(-1)
    step = torch.zeros(1, dtype=torch.int32, device=dev())
    ws = torch.empty(ops.decode_workspace_bytes(B * Hq, D), dtype=torch.uint8, device=dev())
    G = Hq // Hkv
    for t in range(3):
        step.fill_(t)
        out = ops.decode_attn_batch_fp8(q[t].to(dev()), kb, vb, kbs, vbs, 1, kn[t].to(dev()), vn[t].to(dev()), rows=rows_d, step=step,
                                        max_length=cap, workspace=ws)
        for b in range(B):
            one = ops.decode_attn_batch_fp8(q[t, b:b + 1].to(dev()), *solo[b], 1, kn[t, b:b + 1].to(dev()), vn[t, b:b + 1].to(dev()),
                                            rows=rows_d[b * Hq:(b + 1) * Hq].contiguous(), step=step, max_length=cap)
            assert torch.equal(out[b].view(torch.int16), one[0].view(torch.int16)), (t, b)
            assert torch.equal(_u8(solo[b][0]), _u8(kb[b:b + 1])) and torch.equal(solo[b][2], kbs[b:b + 1])
            assert torch.equal(_u8(solo[b][1]), _u8(vb[b:b + 1])) and torch.equal(solo[b][3], vbs[b:b + 1])
        # accuracy: exact (fp64) attention over the dequantised rows the cache now holds
        kc, vc, kcs, vcs, o = kb.cpu(), vb.cpu(), kbs.cpu(), vbs.cpu(), out.cpu()
        for b in range(B):
            for h in range(Hq):
                T = int(rows[b, h]) + t + 1
                K = dequantize(kc[b, h, :T], kcs[b, h, :T]).double()
                V = dequantize(vc[b, h, :T], vcs[b, h, :T]).double()
                p = torch.softmax((K @ q[t, b, h].double()) * D ** -0.5, dim=0)
                exact = p @ V
                assert torch.all((o[b, h].float().double() - exact).abs() <= ATOL + _ulp(o[b, h]).double()), (b, h)
    # the appended rows are the rule applied to k_new / v_new of the sequence's kv head; nothing else was written
    kc, vc, kcs, vcs = _u8(kb.cpu()), _u8(vb.cpu()), kbs.cpu(), vbs.cpu()
    for b in range(B):
        for h in range(Hq):
            n = int(rows[b, h])
            for t in range(3):
                wq, wsc = quantize_rows(kn[t, b, h // G])
                assert torch.equal(kc[b, h, n + t], _u8(wq)) and kcs[b, h, n + t] == wsc
                wq, wsc = quantize_rows(vn[t, b, h // G])
                assert torch.equal(vc[b, h, n + t], _u8(wq)) and vcs[b, h, n + t] == wsc
            assert torch.equal(kc[b, h, :n], _u8(kq[b, h, :n])) and torch.equal(kcs[b, h, :n], ks[b, h, :n])
            assert bool((kc[b, h, n + 3:] == SENTINEL_BYTE).all()) and bool((vc[b, h, n + 3:] == SENTINEL_BYTE).all())
            assert bool((kcs[b, h, n + 3:] == SENTINEL_SCALE).all()) and bool((vcs[b, h, n + 3:] == SENTINEL_SCALE).all())


def test_host_launch_single_sequence(oracle, libpkv):
    """num_seqs = 1, step_dev = NULL, rows = NULL: `length` rows, the same bits as the device-length form."""
    from pyramidkv_b200 import ops
    rows, kq, vq, ks, vs, q, kn, vn = _case(torch.bfloat16, 128, 32, 8, ragged=False, seed=3)
    b = 3                                                       # 257 rows after the append: two splits
    cap = kq.shape[2]
    a = _to(kq[b:b + 1], vq[b:b + 1], ks[b:b + 1], vs[b:b + 1])
    c = _to(kq[b:b + 1], vq[b:b + 1], ks[b:b + 1], vs[b:b + 1])
    n = int(rows[b, 0])
    host = ops.decode_attn_batch_fp8(q[0, b:b + 1].to(dev()), *a, n + 1, kn[0, b:b + 1].to(dev()), vn[0, b:b + 1].to(dev()))
    zero = torch.zeros(1, dtype=torch.int32, device=dev())
    devlen = ops.decode_attn_batch_fp8(q[0, b:b + 1].to(dev()), *c, n + 1, kn[0, b:b + 1].to(dev()), vn[0, b:b + 1].to(dev()),
                                       step=zero, max_length=cap)
    assert torch.equal(host.view(torch.int16), devlen.view(torch.int16))
    assert torch.equal(_u8(a[0]), _u8(c[0])) and torch.equal(a[2], c[2])


def test_graph_replay_equals_host_launches(libpkv):
    from pyramidkv_b200 import ops
    rows, kq, vq, ks, vs, q, kn, vn = _case(torch.bfloat16, 128, 32, 8, ragged=True, seed=5)
    B, Hq, cap, D = kq.shape
    rows_d = rows.to(dev()).reshape(-1)
    qd, knd, vnd = q[0].to(dev()), kn[0].to(dev()), vn[0].to(dev())
    ws = torch.empty(ops.decode_workspace_bytes(B * Hq, D), dtype=torch.uint8, device=dev())
    h = _to(kq, vq, ks, vs)
    step = torch.zeros(1, dtype=torch.int32, device=dev())
    host = []
    for t in range(STEPS):
        step.fill_(t)
        host.append(ops.decode_attn_batch_fp8(qd, *h, 1, knd, vnd, rows=rows_d, step=step, max_length=cap, workspace=ws).clone())
    gbuf = _to(kq, vq, ks, vs)
    gstep = torch.zeros(1, dtype=torch.int32, device=dev())
    out = torch.empty(B, Hq, D, dtype=torch.bfloat16, device=dev())
    warm = [t.clone() for t in gbuf]
    ops.decode_attn_batch_fp8(qd, *warm, 1, knd, vnd, rows=rows_d, step=gstep, max_length=cap, workspace=ws, out=out)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        ops.decode_attn_batch_fp8(qd, *gbuf, 1, knd, vnd, rows=rows_d, step=gstep, max_length=cap, workspace=ws, out=out)
        gstep.add_(1)
    replayed = []
    for _ in range(STEPS):
        graph.replay()
        replayed.append(out.clone())
    torch.cuda.synchronize()
    for a, b in zip(host, replayed):
        assert torch.equal(a.view(torch.int16), b.view(torch.int16))
    for a, b in zip(h, gbuf):
        assert torch.equal(a.view(torch.uint8), b.view(torch.uint8))


def test_one_launch_whatever_the_batch_size(libpkv):
    from pyramidkv_b200 import _lib, ops
    D, Hq, Hkv, cap = 128, 32, 8, 400
    counts = []
    for B in (1, 8):
        kq = torch.randint(0, 0x70, (B, Hq, cap, D), dtype=torch.uint8, device=dev()).view(torch.float8_e4m3fn)
        ks = torch.rand(B, Hq, cap, device=dev())
        q = torch.randn(B, Hq, D, device=dev()).bfloat16()
        kn = torch.randn(B, Hkv, D, device=dev()).bfloat16()
        rows = torch.full((B * Hq,), 299, dtype=torch.int32, device=dev())
        step = torch.zeros(1, dtype=torch.int32, device=dev())
        ops.decode_attn_batch_fp8(q, kq, kq.clone(), ks, ks.clone(), 1, kn, kn, rows=rows, step=step)
        n0 = _lib.launch_count()
        ops.decode_attn_batch_fp8(q, kq, kq.clone(), ks, ks.clone(), 1, kn, kn, rows=rows, step=step)
        counts.append(_lib.launch_count() - n0)
    torch.cuda.synchronize()
    assert counts[0] == counts[1] >= 1


def test_argument_errors(libpkv):
    import ctypes as C
    from pyramidkv_b200 import _lib, ops
    B, Hq, D, cap = 2, 4, 128, 16
    kq = torch.zeros(B, Hq, cap, D, dtype=torch.float8_e4m3fn, device=dev())
    ks = torch.zeros(B, Hq, cap, device=dev())
    q = torch.zeros(B, Hq, D, dtype=torch.bfloat16, device=dev())
    ok = torch.full((B * Hq,), 3, dtype=torch.int32, device=dev())
    ops.decode_attn_batch_fp8(q, kq, kq.clone(), ks, ks.clone(), 1, rows=ok)
    with pytest.raises(ValueError, match="float8_e4m3fn"):
        ops.decode_attn_batch_fp8(q, kq.view(torch.uint8), kq.clone().view(torch.uint8), ks, ks.clone(), 1, rows=ok)
    with pytest.raises(ValueError, match="scales"):
        ops.decode_attn_batch_fp8(q, kq, kq.clone(), ks.double(), ks.clone(), 1, rows=ok)
    with pytest.raises(ValueError, match="capacity"):
        ops.decode_attn_batch_fp8(q, kq, kq.clone(), ks, ks.clone(), cap + 1)
    with pytest.raises(ValueError, match="aligned"):
        big = torch.zeros(B * Hq * cap * D + 8, dtype=torch.uint8, device=dev())
        mis = big[8:].view(torch.float8_e4m3fn).view(B, Hq, cap, D)
        ops.decode_attn_batch_fp8(q, mis, kq.clone(), ks, ks.clone(), 1, rows=ok)
    # the C entry point itself: null scales, misalignment, max_length above the capacity, a wrong dtype
    out = torch.empty_like(q)
    d = _lib.DecodeDesc()
    d.struct_bytes = C.sizeof(_lib.DecodeDesc)
    d.dtype, d.num_q_heads, d.num_kv_heads, d.head_dim, d.device = 0, Hq, Hq, D, dev().index or 0
    d.length, d.q, d.out = 4, q.data_ptr(), out.data_ptr()
    d.k_cache, d.v_cache, d.cache_stride_h = kq.data_ptr(), kq.data_ptr(), cap * D
    ws = torch.empty(ops.decode_workspace_bytes(B * Hq, D), dtype=torch.uint8, device=dev())
    d.workspace, d.workspace_bytes = ws.data_ptr(), ws.numel()
    L = _lib.lib()
    st = torch.cuda.current_stream().cuda_stream
    fn = L.pkv_decode_attn_batch_fp8
    assert fn(C.byref(d), B, Hq * cap * D, None, None, cap, ks.data_ptr(), ks.data_ptr(), cap, Hq * cap, st) == _lib.PKV_OK
    assert fn(C.byref(d), B, Hq * cap * D, None, None, cap, None, ks.data_ptr(), cap, Hq * cap, st) == _lib.PKV_ERR_INVALID_ARG
    assert fn(C.byref(d), B, Hq * cap * D, None, None, cap, ks.data_ptr() + 2, ks.data_ptr(), cap, Hq * cap, st) == _lib.PKV_ERR_INVALID_ARG
    assert fn(C.byref(d), B, Hq * cap * D, None, None, cap + 1, ks.data_ptr(), ks.data_ptr(), cap, Hq * cap, st) == _lib.PKV_ERR_INVALID_ARG
    assert fn(C.byref(d), B, Hq * cap * D, None, None, cap, ks.data_ptr(), ks.data_ptr(), cap - 1, Hq * cap, st) == _lib.PKV_ERR_INVALID_ARG
    assert fn(C.byref(d), B, Hq * cap * D - 8, None, None, cap, ks.data_ptr(), ks.data_ptr(), cap, Hq * cap, st) == _lib.PKV_ERR_INVALID_ARG
    d.k_cache = kq.data_ptr() + 8
    assert fn(C.byref(d), B, Hq * cap * D, None, None, cap, ks.data_ptr(), ks.data_ptr(), cap, Hq * cap, st) == _lib.PKV_ERR_INVALID_ARG
    d.k_cache, d.dtype = kq.data_ptr(), 7
    assert fn(C.byref(d), B, Hq * cap * D, None, None, cap, ks.data_ptr(), ks.data_ptr(), cap, Hq * cap, st) == _lib.PKV_ERR_UNSUPPORTED_DTYPE
    torch.cuda.synchronize()
    # quantize: a 16-bit source of the wrong dtype, rows above the capacity, misaligned destination
    k16 = torch.zeros(1, Hq, cap, D, dtype=torch.bfloat16, device=dev())
    k8, s8 = _fp8_empty((1, Hq, cap, D), dev())
    with pytest.raises(NotImplementedError):
        ops.cache_quantize_fp8([(k16.float(), k16.float(), k8, k8.clone(), s8, s8.clone(), 4, None)])
    with pytest.raises(ValueError, match="capacity"):
        ops.cache_quantize_fp8([(k16, k16, k8, k8.clone(), s8, s8.clone(), cap + 1, None)])
    with pytest.raises(ValueError, match="float8_e4m3fn"):
        ops.cache_quantize_fp8([(k16, k16, k16, k16, s8, s8.clone(), 4, None)])
