"""`pkv_token_logprobs` on the H100 against the fp64 oracle of its rules (oracle/logprobs.py): log-probabilities within
1e-5 (the bound of DESIGN.md §4.8) and exact top ids over a sweep of vocabulary sizes, batch sizes, dtypes, top N and
strided rows; constant rows and rows with many ties at the N-th value; NaN / inf rows and out-of-range tokens; graph replay
equal to host launches with one launch per call; the argument errors."""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import logprobs as LP

pytestmark = pytest.mark.gpu


def _dev(libpkv):
    from gpu_util import dev
    return dev()


def _logits(B, V, dtype, seed, dev, pad=0):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, V + pad, generator=g) * 2.5
    x[:, :: max(1, V // 97)] += 4.0                     # a head of likely tokens, and ties from the 16-bit rounding
    return x.to(dtype).to(dev)[:, :V]                   # rows pad elements apart when pad > 0


def _run(logits, tokens, N, cols=1, col=0, cursor=None):
    from pyramidkv_b200 import ops
    B = logits.shape[0]
    dev = logits.device
    lp = torch.full((B, cols), -7.0, dtype=torch.float32, device=dev)
    ids = torch.full((B, cols, N), -7, dtype=torch.long, device=dev)
    top = torch.full((B, cols, N), -7.0, dtype=torch.float32, device=dev)
    ops.token_logprobs(logits, tokens, lp, ids, top, col, 0, cursor)
    return lp, ids, top


def _check(logits, tokens, lp, ids, top, N, c=0, tol=1e-5):
    host = logits.float().cpu().numpy()
    toks = tokens[:, 0].cpu().tolist()
    lp, ids, top = lp[:, c].cpu().numpy(), ids[:, c].cpu().numpy(), top[:, c].cpu().numpy()
    for b in range(host.shape[0]):
        w_lp, w_ids, w_top = LP.logprobs_row(host[b], toks[b], N)
        bound = tol + abs(w_lp) * 2.0 ** -24 if np.isfinite(w_lp) else 0
        assert (np.isnan(lp[b]) and np.isnan(w_lp)) or abs(lp[b] - w_lp) <= bound, (b, lp[b], w_lp)
        assert ids[b].tolist() == w_ids.tolist(), (b, ids[b], w_ids)
        fin = np.isfinite(w_top)
        assert (np.isnan(top[b][~fin])).all()
        assert (np.abs(top[b][fin] - w_top[fin]) <= tol + np.abs(w_top[fin]) * 2.0 ** -24).all(), b


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("V", [257, 1000, 32000, 128256])
def test_kernel_matches_oracle(libpkv, V, dtype):
    dev = _dev(libpkv)
    for B in (1, 7, 64):
        for N in (0, 1, 5, 20):
            for pad in (0, 3):                                                # contiguous and strided rows
                logits = _logits(B, V, dtype, V + B + N + pad, dev, pad)
                g = torch.Generator().manual_seed(B + N)
                tokens = torch.randint(0, V, (B, 1), generator=g).to(dev)
                tokens[0, 0] = int(logits[0].float().argmax())
                lp, ids, top = _run(logits, tokens, N)
                _check(logits, tokens, lp, ids, top, N)
                if N:
                    assert torch.equal(ids[:, 0, 0], logits.argmax(dim=-1))


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_ties_constant_and_non_finite_rows(libpkv, dtype):
    dev = _dev(libpkv)
    V = 32000
    logits = _logits(10, V, dtype, 3, dev)
    logits[0] = 1.5                                                           # all ties
    logits[1] = -2.0
    logits[2] = 0.0
    logits[2, 5000::7] = 3.0                                                  # many ties at the top, scattered
    logits[3] = -1.0
    logits[3, :4] = 2.0
    logits[3, 9000::13] = 1.0                                                 # many ties at the N-th value
    logits[4, 77] = float("nan")
    logits[5, 300] = float("inf")
    logits[6] = float("-inf")
    logits[7, 31999] = float("-inf")
    logits[8, 0] = -0.0
    logits[8, 1] = 0.0
    tokens = torch.tensor([[3], [0], [5007], [9000], [1], [2], [3], [4], [V], [-1]], device=dev)
    for N in (0, 1, 5, 20):
        lp, ids, top = _run(logits, tokens, N)
        _check(logits, tokens, lp, ids, top, N)
    lp = lp.cpu()
    assert abs(float(lp[0, 0]) + np.log(V)) < 1e-5
    assert all(np.isnan(float(lp[b, 0])) for b in (4, 5, 6, 7, 8, 9))
    assert (ids[4:8].cpu() == -1).all() and ids[0, 0].cpu().tolist() == list(range(20))
    assert ids[2, 0, :5].cpu().tolist() == [5000, 5007, 5014, 5021, 5028]
    assert ids[3, 0, :6].cpu().tolist() == [0, 1, 2, 3, 9000, 9013]
    # fewer tokens than top_n: the entries past the vocabulary are -1 / NaN
    small = _logits(2, 3, dtype, 1, dev)
    lp, ids, top = _run(small, torch.zeros(2, 1, dtype=torch.long, device=dev), 5)
    _check(small, torch.zeros(2, 1, dtype=torch.long, device=dev), lp, ids, top, 5)
    assert (ids[:, 0, 3:].cpu() == -1).all() and torch.isnan(top[:, 0, 3:]).all()


def test_graph_replay_equals_host_launches_one_launch_per_call(libpkv):
    from pyramidkv_b200 import _lib, ops
    dev = _dev(libpkv)
    B, V, N, steps = 8, 128256, 5, 4
    rows = [_logits(B, V, torch.bfloat16, 21 + s, dev) for s in range(steps)]
    tokens = torch.randint(0, V, (B, 1), generator=torch.Generator().manual_seed(1)).to(dev)
    lp_h = torch.zeros(B, steps, device=dev)
    ids_h = torch.zeros(B, steps, N, dtype=torch.long, device=dev)
    top_h = torch.zeros(B, steps, N, device=dev)
    for s in range(steps):
        n0 = _lib.launch_count()
        ops.token_logprobs(rows[s], tokens, lp_h, ids_h, top_h, s)
        assert _lib.launch_count() - n0 == 1
    logits = rows[0].clone()
    cursor = torch.zeros(1, dtype=torch.long, device=dev)
    lp = torch.zeros_like(lp_h)
    ids = torch.zeros_like(ids_h)
    top = torch.zeros_like(top_h)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        ops.token_logprobs(logits, tokens, lp, ids, top, 0, 0, cursor)      # warm-up
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        ops.token_logprobs(logits, tokens, lp, ids, top, 0, 0, cursor)
        cursor.add_(1)
    cursor.zero_()
    for s in range(steps):
        logits.copy_(rows[s])
        graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(lp.view(torch.int32), lp_h.view(torch.int32))
    assert torch.equal(ids, ids_h) and torch.equal(top.view(torch.int32), top_h.view(torch.int32))
    assert int(cursor) == steps


def _desc(lg, tk, lp, ids, top, **over):
    from pyramidkv_b200 import _lib
    d = _lib.LogprobsDesc()
    d.struct_bytes = C.sizeof(_lib.LogprobsDesc)
    d.dtype, d.device, d.batch, d.vocab, d.top_n = 0, 0, lg.shape[0], lg.shape[1], ids.shape[2]
    d.logits, d.logits_stride = lg.data_ptr(), lg.stride(0)
    d.tokens, d.tokens_stride, d.tokens_column = tk.data_ptr(), tk.stride(0), 0
    d.column, d.logprob, d.logprob_stride = 1, lp.data_ptr(), lp.shape[1]
    d.top_ids, d.top_logprobs, d.top_stride = ids.data_ptr(), top.data_ptr(), ids.shape[1] * ids.shape[2]
    for k, v in over.items():
        setattr(d, k, v)
    return d


def test_argument_errors(libpkv):
    from pyramidkv_b200 import _lib, ops
    dev = _dev(libpkv)
    logits = _logits(4, 1000, torch.bfloat16, 2, dev)
    tokens = torch.zeros(4, 1, dtype=torch.long, device=dev)
    lp = torch.zeros(4, 2, device=dev)
    ids = torch.zeros(4, 2, 3, dtype=torch.long, device=dev)
    top = torch.zeros(4, 2, 3, device=dev)
    L = _lib.lib()
    stream = torch.cuda.current_stream().cuda_stream
    assert L.pkv_token_logprobs(C.byref(_desc(logits, tokens, lp, ids, top)), stream) == _lib.PKV_OK
    assert L.pkv_token_logprobs(C.byref(_desc(logits, tokens, lp, ids, top, top_n=0, top_ids=None, top_logprobs=None)),
                                stream) == _lib.PKV_OK
    bad = [dict(batch=0), dict(batch=2 ** 20 + 1), dict(vocab=0), dict(vocab=2 ** 24 + 1), dict(logits_stride=999),
           dict(top_n=21), dict(top_n=-1), dict(tokens_column=1), dict(tokens_column=-1), dict(column=2), dict(column=-1),
           dict(top_stride=5), dict(flags=1), dict(logits=logits.data_ptr() + 1), dict(logits=None), dict(tokens=None),
           dict(tokens=tokens.data_ptr() + 4), dict(logprob=None), dict(logprob=lp.data_ptr() + 2), dict(top_ids=None),
           dict(top_ids=ids.data_ptr() + 4), dict(top_logprobs=top.data_ptr() + 1), dict(cursor=tokens.data_ptr() + 4),
           dict(struct_bytes=8)]
    for over in bad:
        assert L.pkv_token_logprobs(C.byref(_desc(logits, tokens, lp, ids, top, **over)), stream) == _lib.PKV_ERR_INVALID_ARG, over
        assert _lib.last_error()
    assert L.pkv_token_logprobs(C.byref(_desc(logits, tokens, lp, ids, top, dtype=5)), stream) == _lib.PKV_ERR_UNSUPPORTED_DTYPE
    assert L.pkv_token_logprobs(None, stream) == _lib.PKV_ERR_INVALID_ARG
    with pytest.raises(ValueError):
        ops.token_logprobs(logits, tokens.int(), lp, ids, top)
    with pytest.raises(ValueError):
        ops.token_logprobs(logits[:3], tokens, lp, ids, top)
    with pytest.raises(ValueError):
        ops.token_logprobs(logits, tokens, lp, ids.float(), top)
    with pytest.raises(NotImplementedError):
        ops.token_logprobs(logits.float(), tokens, lp, ids, top)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        ops.token_logprobs(logits.cpu(), tokens, lp, ids, top)
    torch.cuda.synchronize()
