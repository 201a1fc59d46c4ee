"""`pkv_sample_tokens` on the H100 against the CPU oracle of its rules (oracle/sampling.py): tokens and kept sets over a sweep
of vocabulary sizes, batch sizes, dtypes and parameters, a fixed-seed chi-square test of the draw's distribution, the
greedy and NaN rules, graph replay, one launch per step, and the argument errors."""
import ctypes as C
import itertools

import numpy as np
import pytest
import torch

from oracle import sampling as S

pytestmark = pytest.mark.gpu

TEMPS, TOPKS, TOPPS = (0.0, 0.3, 1.0, 1.7), (0, 1, 50, None), (1e-6, 0.5, 0.9, 1.0)   # top_k None: V
COMBOS = list(itertools.product(TEMPS, TOPKS, TOPPS))                                 # 64


class _State:
    def __init__(self, temps, topks, topps, seeds, index, dev):
        self.temperature = torch.tensor(temps, dtype=torch.float32, device=dev)
        self.top_k = torch.tensor(topks, dtype=torch.int32, device=dev)
        self.top_p = torch.tensor(topps, dtype=torch.float32, device=dev)
        self.seed = torch.tensor([s - 2 ** 64 if s >= 2 ** 63 else s for s in seeds], dtype=torch.int64, device=dev)
        self.index = torch.tensor(index, dtype=torch.int64, device=dev)


def _dev(libpkv):
    from gpu_util import dev
    return dev()


def _logits(B, V, dtype, seed, dev):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, V, generator=g) * 2.5
    x[:, :: max(1, V // 97)] += 4.0                     # a head of likely tokens, and ties from the 16-bit rounding
    return x.to(dtype).to(dev)


def _ulp_tol(scale):
    return 16 * max(scale, 1.0) * 2.0 ** -23


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("V", [257, 1000, 32000, 128256])
def test_kernel_matches_oracle(libpkv, V, dtype):
    from pyramidkv_b200 import ops
    dev = _dev(libpkv)
    rows = checked = near = close = 0
    for B, off in ((1, 5), (7, 17), (64, 0)):
        combos = [COMBOS[(b + off) % 64] for b in range(B)]
        temps = [c[0] for c in combos]
        topks = [V if c[1] is None else c[1] for c in combos]
        topps = [c[2] for c in combos]
        seeds = [(0x9E3779B97F4A7C15 * (b + 1 + V)) % 2 ** 64 for b in range(B)]
        index = [b * 3 + 2 ** 33 * (b % 2) for b in range(B)]
        logits = _logits(B, V, dtype, V + B, dev)
        st = _State(temps, topks, topps, seeds, index, dev)
        out = torch.full((B, 3), -7, dtype=torch.long, device=dev)
        ops.sample_tokens(logits, st, out, 1)
        torch.cuda.synchronize()
        got = out[:, 1].cpu().tolist()
        assert out[:, 0].cpu().tolist() == [-7] * B and out[:, 2].cpu().tolist() == [-7] * B
        assert st.index.cpu().tolist() == [i + 1 for i in index]
        host = logits.float().cpu().numpy()
        for b in range(B):
            rows += 1
            d = S.sample_row(host[b], temps[b], topks[b], topps[b], seeds[b], index[b])
            if d.kept is None:
                assert got[b] == d.token, (B, b, combos[b])
                checked += 1
                continue
            if d.near_top_p:                                          # the kept set is only known up to the tolerance
                near += 1
                continue
            assert d.kept[got[b]], (B, b, combos[b], got[b])         # never outside the kept set
            if d.gap <= _ulp_tol(d.scale):
                close += 1
                continue
            assert got[b] == d.token, (B, b, combos[b], got[b], d.token)
            checked += 1
    print(f"V={V} {dtype}: rows={rows} exact={checked} top_p_within_tolerance={near} perturbed_scores_within_ulps={close}")
    assert near + close <= max(2, rows // 20)


def test_chi_square_of_the_draw(libpkv):
    """2^18 draws of one row through 4096 seeds x 64 token indices: every draw inside the kept set, and the frequencies
    match softmax(x) over the kept set (Pearson chi-square, p-value above 1e-3; fixed seeds, so deterministic)."""
    from scipy.stats import chisquare
    from pyramidkv_b200 import ops
    dev = _dev(libpkv)
    V, B, steps = 1000, 4096, 64
    g = torch.Generator().manual_seed(5)
    row = torch.cat([torch.linspace(3.0, 0.0, 60), torch.randn(V - 60, generator=g) - 3.0]).to(torch.bfloat16)
    T, k, p = 0.8, 50, 0.9
    probs = S.kept_probabilities(row.float().numpy(), T, k, p)
    kept = probs > 0
    logits = row.to(dev).reshape(1, V).expand(B, V).contiguous()
    st = _State([T] * B, [k] * B, [p] * B, [1000 + b for b in range(B)], [0] * B, dev)
    out = torch.empty(B, steps, dtype=torch.long, device=dev)
    for s in range(steps):
        ops.sample_tokens(logits, st, out, s)
    toks = out.cpu().numpy().reshape(-1)
    assert ((toks >= 0) & (toks < V)).all() and kept[toks].all()
    counts = np.bincount(toks, minlength=V)[kept]
    exp = probs[kept] * toks.size
    assert exp.min() >= 5
    res = chisquare(counts, exp)
    print(f"chi-square: kept={int(kept.sum())} draws={toks.size} stat={res.statistic:.1f} p={res.pvalue:.3f}")
    assert res.pvalue > 1e-3


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_greedy_constant_and_nan_rows(libpkv, dtype):
    from pyramidkv_b200 import ops
    dev = _dev(libpkv)
    V = 32000
    logits = _logits(8, V, dtype, 3, dev)
    logits[0] = 1.5                                            # all ties
    logits[1] = -2.0
    logits[4, 77] = float("nan")
    logits[5, 300] = float("inf")
    logits[6] = float("-inf")
    st = _State([0.0, 0.9, 0.0, 1.2, 0.7, 1.0, 1.0, 0.5], [0, 1, 0, 1, 0, 0, 0, 0], [1.0, 0.3, 0.5, 0.9, 0.9, 1.0, 1.0, 1.0],
                list(range(8)), [0] * 8, dev)
    out = torch.empty(8, 1, dtype=torch.long, device=dev)
    ops.sample_tokens(logits, st, out, 0)
    got = out[:, 0].cpu().tolist()
    am = logits.argmax(dim=-1).cpu().tolist()
    assert got[:5] == am[:5] == [0, 0, am[2], am[3], 77]
    assert got[5] == 300 and got[6] == 0
    d = S.sample_row(logits[7].float().cpu().numpy(), 0.5, 0, 1.0, 7, 0)
    assert got[7] == d.token
    # constant row, sampling on: a uniform draw, the oracle's token
    st = _State([1.0], [0], [1.0], [42], [3], dev)
    ops.sample_tokens(logits[:1], st, out[:1], 0)
    assert int(out[0, 0]) == S.sample_row(logits[0].float().cpu().numpy(), 1.0, 0, 1.0, 42, 3).token


def test_invalid_row_parameters_give_minus_one(libpkv):
    from pyramidkv_b200 import ops
    dev = _dev(libpkv)
    logits = _logits(5, 1000, torch.bfloat16, 9, dev)
    st = _State([-1.0, float("nan"), 1.0, 1.0, 1.0], [0, 0, -1, 0, 0], [1.0, 1.0, 1.0, 0.0, 1.5], [1] * 5, [0] * 5, dev)
    out = torch.empty(5, 1, dtype=torch.long, device=dev)
    ops.sample_tokens(logits, st, out, 0)
    assert out[:, 0].cpu().tolist() == [-1] * 5


def test_graph_replay_equals_host_launches_one_launch_per_step(libpkv):
    from pyramidkv_b200 import _lib, ops
    dev = _dev(libpkv)
    B, V, steps = 8, 32000, 5
    logits = _logits(B, V, torch.bfloat16, 21, dev)
    params = ([0.7] * B, [0, 40] * (B // 2), [0.9] * B, [77 + b for b in range(B)], [1] * B)
    host = _State(*params, dev)
    want = torch.empty(B, steps, dtype=torch.long, device=dev)
    for s in range(steps):
        n0 = _lib.launch_count()
        ops.sample_tokens(logits, host, want, s)
        assert _lib.launch_count() - n0 == 1
    st = _State(*params, dev)
    out = torch.empty(B, 1, dtype=torch.long, device=dev)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        ops.sample_tokens(logits, st, out, 0)                 # warm-up, then restore the token index
    torch.cuda.current_stream().wait_stream(side)
    st.index.fill_(1)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        ops.sample_tokens(logits, st, out, 0)
    got = []
    for _ in range(steps):
        graph.replay()
        got.append(out.clone())
    assert torch.equal(torch.cat(got, dim=1), want)
    assert st.index.cpu().tolist() == [1 + steps] * B
    big = _State([1.0] * 64, [0] * 64, [1.0] * 64, list(range(64)), [0] * 64, dev)
    n0 = _lib.launch_count()
    ops.sample_tokens(_logits(64, V, torch.bfloat16, 1, dev), big, torch.empty(64, 1, dtype=torch.long, device=dev), 0)
    assert _lib.launch_count() - n0 == 1


def _desc(logits_t, st, out, col, **over):
    from pyramidkv_b200 import _lib
    d = _lib.SampleDesc()
    d.struct_bytes = C.sizeof(_lib.SampleDesc)
    d.dtype, d.device, d.batch, d.vocab = 0, 0, logits_t.shape[0], logits_t.shape[1]
    d.logits, d.logits_stride = logits_t.data_ptr(), logits_t.stride(0)
    d.temperature, d.top_k, d.top_p = st.temperature.data_ptr(), st.top_k.data_ptr(), st.top_p.data_ptr()
    d.seed, d.token_index = st.seed.data_ptr(), st.index.data_ptr()
    d.tokens, d.tokens_stride, d.column, d.flags = out.data_ptr(), out.stride(0), col, 1
    for k, v in over.items():
        setattr(d, k, v)
    return d


def test_argument_errors(libpkv):
    from pyramidkv_b200 import _lib, ops
    dev = _dev(libpkv)
    logits = _logits(4, 1000, torch.bfloat16, 2, dev)
    st = _State([1.0] * 4, [0] * 4, [1.0] * 4, [0] * 4, [0] * 4, dev)
    out = torch.empty(4, 2, dtype=torch.long, device=dev)
    L = _lib.lib()
    stream = torch.cuda.current_stream().cuda_stream
    assert L.pkv_sample_tokens(C.byref(_desc(logits, st, out, 1)), stream) == _lib.PKV_OK
    bad = [dict(batch=0), dict(batch=2 ** 20 + 1), dict(vocab=0), dict(vocab=2 ** 24 + 1), dict(logits_stride=999),
           dict(column=2), dict(column=-1), dict(flags=2), dict(logits=logits.data_ptr() + 1), dict(logits=None),
           dict(temperature=None), dict(top_k=st.top_k.data_ptr() + 2), dict(top_p=st.top_p.data_ptr() + 1),
           dict(seed=st.seed.data_ptr() + 4), dict(token_index=None), dict(tokens=out.data_ptr() + 4),
           dict(struct_bytes=8)]
    for over in bad:
        assert L.pkv_sample_tokens(C.byref(_desc(logits, st, out, 1, **over)), stream) == _lib.PKV_ERR_INVALID_ARG, over
        assert _lib.last_error()
    assert L.pkv_sample_tokens(C.byref(_desc(logits, st, out, 1, dtype=5)), stream) == _lib.PKV_ERR_UNSUPPORTED_DTYPE
    assert L.pkv_sample_tokens(None, stream) == _lib.PKV_ERR_INVALID_ARG
    with pytest.raises(ValueError):
        ops.sample_tokens(logits, st, out.int(), 0)
    with pytest.raises(ValueError):
        ops.sample_tokens(logits[:3], st, out[:3], 0)
    with pytest.raises(NotImplementedError):
        ops.sample_tokens(logits.float(), st, out, 0)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        ops.sample_tokens(logits.cpu(), st, out, 0)
    torch.cuda.synchronize()
