"""`pkv_sample_tokens_penalized` on the H100 against the CPU restatement of its rules (tests/oracle_penalty_backend.py):
tokens, kept sets and count updates over a sweep of vocabulary sizes, batch sizes, dtypes and a grid of penalties, min-p,
temperature, top-k and top-p with prompt masks of up to 32K ids and counts up to 4096; rows at the defaults bit-equal to
`pkv_sample_tokens` in the same launch; the NaN / inf rules; a fixed-seed chi-square test of the penalized draw; graph replay
with its count updates and one launch per step; and the argument errors."""
import ctypes as C
import itertools

import numpy as np
import pytest
import torch

import oracle_penalty_backend as OP

pytestmark = pytest.mark.gpu

RHOS, PRES, FREQS, MINPS = (1.0, 0.8, 1.3), (0.0, 0.5, -0.5, 1.5), (0.0, 0.5, -0.5, 1.5), (0.0, 0.05, 0.5, 1.0)
TEMPS, TOPKS, TOPPS = (0.0, 0.7, 1.3), (0, 50), (0.9, 1.0)
COMBOS = list(itertools.product(RHOS, PRES, FREQS, MINPS, TEMPS, TOPKS, TOPPS))      # 2304


class _State:
    def __init__(self, rows, dev, V, stride=None, masks=None, counts=None):
        """rows: (T, top_k, top_p, seed, index, rho, presence, frequency, min_p) per row."""
        B = len(rows)
        col = list(zip(*rows))
        self.temperature = torch.tensor(col[0], dtype=torch.float32, device=dev)
        self.top_k = torch.tensor(col[1], dtype=torch.int32, device=dev)
        self.top_p = torch.tensor(col[2], dtype=torch.float32, device=dev)
        self.seed = torch.tensor([s - 2 ** 64 if s >= 2 ** 63 else s for s in col[3]], dtype=torch.int64, device=dev)
        self.index = torch.tensor(col[4], dtype=torch.int64, device=dev)
        for name, c in zip(("repetition_penalty", "presence_penalty", "frequency_penalty", "min_p"), col[5:]):
            setattr(self, name, torch.tensor(c, dtype=torch.float32, device=dev))
        S = stride or V
        self.prompt_mask = torch.zeros(B, S, dtype=torch.uint8, device=dev) if masks is None else masks.to(dev).contiguous()
        self.counts = torch.zeros(B, S, dtype=torch.int32, device=dev) if counts is None else counts.to(dev).contiguous()


def _dev(libpkv):
    from gpu_util import dev
    return dev()


def _logits(B, V, dtype, seed, dev):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, V, generator=g) * 2.5
    x[:, :: max(1, V // 97)] += 4.0                     # a head of likely tokens, and ties from the 16-bit rounding
    return x.to(dtype).to(dev)


def _history(B, V, S, seed):
    """A prompt mask of up to 32K ids and counts up to 4096 per row, biased toward the likely head of _logits."""
    g = np.random.default_rng(seed)
    mask = np.zeros((B, S), np.uint8)
    counts = np.zeros((B, S), np.int32)
    for b in range(B):
        n = int(g.integers(1, min(V, 32768) + 1))
        mask[b, g.choice(V, size=n, replace=False)] = 1
        m = int(g.integers(1, min(V, 600) + 1))
        ids = g.choice(V, size=m, replace=False)
        ids[: m // 3] = (ids[: m // 3] // max(1, V // 97)) * max(1, V // 97)
        counts[b, ids] = g.integers(1, 4097, size=m)
    return torch.from_numpy(mask), torch.from_numpy(counts)


def _ulp_tol(scale):
    return 16 * max(scale, 1.0) * 2.0 ** -23


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("V", [257, 32000, 128256])
def test_kernel_matches_oracle(libpkv, V, dtype):
    from pyramidkv_b200 import ops
    dev = _dev(libpkv)
    rows = checked = near = close = 0
    for B, off in ((1, 5), (7, 17), (64, 0)):
        S = V + (3 if B == 7 else 0)                       # a row stride above V: unaligned rows of mask and counts
        combos = [COMBOS[(b * 37 + off + V) % len(COMBOS)] for b in range(B)]
        params = [(c[4], c[5], c[6], (0x9E3779B97F4A7C15 * (b + 1 + V)) % 2 ** 64, b * 3 + 2 ** 33 * (b % 2), c[0], c[1], c[2],
                   c[3]) for b, c in enumerate(combos)]
        logits = _logits(B, V, dtype, V + B, dev)
        mask, counts = _history(B, V, S, V + B)
        st = _State(params, dev, V, S, mask, counts)
        out = torch.full((B, 3), -7, dtype=torch.long, device=dev)
        ops.sample_tokens_penalized(logits, st, out, 1)
        torch.cuda.synchronize()
        got = out[:, 1].cpu().tolist()
        assert out[:, 0].cpu().tolist() == [-7] * B and out[:, 2].cpu().tolist() == [-7] * B
        assert st.index.cpu().tolist() == [p[4] + 1 for p in params]
        after = st.counts.cpu()
        host = logits.float().cpu().numpy()
        for b in range(B):
            rows += 1
            T, k, p, seed, t, rho, pr, fq, mp = params[b]
            want_counts = counts[b].clone()
            if got[b] >= 0:
                want_counts[got[b]] += 1
            assert torch.equal(after[b], want_counts), (B, b)
            d = OP.sample_row_penalized(host[b], T, k, p, seed, t, rho, pr, fq, mp, mask[b, :V].numpy(), counts[b, :V].numpy())
            if d.kept is None:
                assert got[b] == d.token, (B, b, params[b])
                checked += 1
                continue
            if d.near_top_p:
                near += 1
                continue
            assert d.kept[got[b]], (B, b, params[b], got[b])
            if d.gap <= _ulp_tol(d.scale):
                close += 1
                continue
            assert got[b] == d.token, (B, b, params[b], got[b], d.token)
            checked += 1
    print(f"V={V} {dtype}: rows={rows} exact={checked} top_p_or_min_p_within_tolerance={near} perturbed_scores_within_ulps={close}")
    assert near + close <= max(2, rows // 20)


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_default_rows_equal_sample_tokens_in_a_mixed_batch(libpkv, dtype):
    """Rows at the defaults get pkv_sample_tokens' token bit for bit, whatever their mask and counts and whatever the other
    rows of the launch do; their counts still count the drawn token."""
    from pyramidkv_b200 import ops
    dev = _dev(libpkv)
    V, B = 128256, 64
    logits = _logits(B, V, dtype, 77, dev)
    mask, counts = _history(B, V, V, 78)
    base = [((0.0, 0.3, 1.0, 1.7)[b % 4], (0, 1, 50, V)[(b // 4) % 4], (1e-6, 0.5, 0.9, 1.0)[(b // 16) % 4], 1000 + b, b)
            for b in range(B)]
    pen = [bp + ((1.0, 0.0, 0.0, 0.0) if b % 2 == 0 else (1.3, 0.5, 0.5, 0.05)) for b, bp in enumerate(base)]
    st = _State(pen, dev, V, V, mask, counts)
    ref = _State([bp + (1.0, 0.0, 0.0, 0.0) for bp in base], dev, V)
    got = torch.empty(B, 1, dtype=torch.long, device=dev)
    want = torch.empty(B, 1, dtype=torch.long, device=dev)
    for step in range(3):
        ops.sample_tokens_penalized(logits, st, got, 0)
        ops.sample_tokens(logits, ref, want, 0)
        assert got[0::2].cpu().tolist() == want[0::2].cpu().tolist(), step
    assert got[1::2].cpu().tolist() != want[1::2].cpu().tolist()
    assert int((st.counts.cpu() - counts).sum()) == 3 * B


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_nan_inf_and_invalid_rows(libpkv, dtype):
    from pyramidkv_b200 import ops
    dev = _dev(libpkv)
    V = 32000
    logits = _logits(10, V, dtype, 3, dev)
    logits[0, 77] = float("nan")
    logits[1, 300] = float("inf")
    logits[2] = float("-inf")
    logits[3, 500] = float("inf")
    logits[3, 501] = float("-inf")
    mask, counts = _history(10, V, V, 4)
    counts[1, 300] = 9                                   # inf - 9 * f stays inf
    counts[3, 500] = 1
    base = (1.0, 0, 1.0, 5, 0)
    rows = [base + (1.3, 0.5, 0.5, 0.1)] * 4 + [base + bad for bad in
                                              ((0.0, 0, 0, 0), (float("inf"), 0, 0, 0), (1.0, float("nan"), 0, 0),
                                               (1.0, 0, float("inf"), 0), (1.0, 0, 0, 1.01), (1.0, 0, 0, float("nan")))]
    st = _State(rows, dev, V, V, mask, counts)
    out = torch.empty(10, 1, dtype=torch.long, device=dev)
    ops.sample_tokens_penalized(logits, st, out, 0)
    got = out[:, 0].cpu().tolist()
    host = logits.float().cpu().numpy()
    for b in range(10):
        d = OP.sample_row_penalized(host[b], *rows[b], mask[b].numpy(), counts[b].numpy())
        assert got[b] == d.token, b
    assert got[:3] == [77, 300, 0] and got[4:] == [-1] * 6
    assert torch.equal(st.counts[4:].cpu(), counts[4:])                # token -1 counts nothing


def test_chi_square_of_the_penalized_draw(libpkv):
    """2^18 draws of one penalized row through 4096 seeds x 64 token indices (advance off: the counts stay fixed): every
    draw inside the kept set, frequencies matching softmax over it (Pearson chi-square, p above 1e-3; fixed seeds)."""
    from scipy.stats import chisquare
    from pyramidkv_b200 import ops
    dev = _dev(libpkv)
    V, B, steps = 1000, 4096, 64
    g = torch.Generator().manual_seed(5)
    row = torch.cat([torch.linspace(3.0, 0.0, 60), torch.randn(V - 60, generator=g) - 3.0]).to(torch.bfloat16)
    mask = torch.zeros(V, dtype=torch.uint8)
    mask[0:60:3] = 1
    counts = torch.zeros(V, dtype=torch.int32)
    counts[1:60:4] = torch.arange(1, 16, dtype=torch.int32)
    T, k, p, rho, pr, fq, mp = 0.8, 50, 0.95, 1.3, 0.2, 0.05, 0.02
    x = OP.penalize(row.float().numpy(), rho, pr, fq, mask.numpy(), counts.numpy())
    d = OP.sample_row_penalized(row.float().numpy(), T, k, p, 0, 0, rho, pr, fq, mp, mask.numpy(), counts.numpy())
    kept = d.kept
    y = (x / np.float32(T)).astype(np.float32).astype(np.float64)
    probs = np.where(kept, np.exp(y - y[kept].max()), 0.0)
    probs /= probs.sum()
    logits = row.to(dev).reshape(1, V).expand(B, V).contiguous()
    st = _State([(T, k, p, 1000 + b, 0, rho, pr, fq, mp) for b in range(B)], dev, V, V,
                mask.reshape(1, V).expand(B, V), counts.reshape(1, V).expand(B, V))
    out = torch.empty(B, steps, dtype=torch.long, device=dev)
    for s in range(steps):
        ops.sample_tokens_penalized(logits, st, out, s)
        st.counts.copy_(counts.reshape(1, V).expand(B, V))
    toks = out.cpu().numpy().reshape(-1)
    assert ((toks >= 0) & (toks < V)).all() and kept[toks].all()
    obs = np.bincount(toks, minlength=V)[kept]
    exp = probs[kept] * toks.size
    assert exp.min() >= 5
    res = chisquare(obs, exp)
    print(f"chi-square (penalized): kept={int(kept.sum())} draws={toks.size} stat={res.statistic:.1f} p={res.pvalue:.3f}")
    assert res.pvalue > 1e-3


def test_graph_replay_equals_host_launches_with_counts_one_launch_per_step(libpkv):
    from pyramidkv_b200 import _lib, ops
    dev = _dev(libpkv)
    B, V, steps = 8, 32000, 6
    logits = _logits(B, V, torch.bfloat16, 21, dev)
    mask, counts = _history(B, V, V, 22)
    params = [(0.7, (0, 40)[b % 2], 0.9, 77 + b, 1, (1.0, 1.3)[b % 2], 0.4, 0.3, (0.0, 0.05)[b % 2]) for b in range(B)]
    host = _State(params, dev, V, V, mask, counts)
    want = torch.empty(B, steps, dtype=torch.long, device=dev)
    for s in range(steps):
        n0 = _lib.launch_count()
        ops.sample_tokens_penalized(logits, host, want, s)
        assert _lib.launch_count() - n0 == 1
    st = _State(params, dev, V, V, mask, counts)
    out = torch.empty(B, 1, dtype=torch.long, device=dev)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        ops.sample_tokens_penalized(logits, st, out, 0)            # warm-up, then restore the token index and counts
    torch.cuda.current_stream().wait_stream(side)
    st.index.fill_(1)
    st.counts.copy_(counts)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        ops.sample_tokens_penalized(logits, st, out, 0)
    got = []
    for _ in range(steps):
        graph.replay()
        got.append(out.clone())
    assert torch.equal(torch.cat(got, dim=1), want)
    assert st.index.cpu().tolist() == [1 + steps] * B
    assert torch.equal(st.counts, host.counts)
    # the same logits every step: the counts change the draws (the repeated token is penalized)
    assert any(len(set(r)) > 1 for r in want.cpu().tolist())


def _desc(logits_t, st, out, col):
    from pyramidkv_b200 import _lib
    d = _lib.SampleDesc()
    d.struct_bytes = C.sizeof(_lib.SampleDesc)
    d.dtype, d.device, d.batch, d.vocab = 0, 0, logits_t.shape[0], logits_t.shape[1]
    d.logits, d.logits_stride = logits_t.data_ptr(), logits_t.stride(0)
    d.temperature, d.top_k, d.top_p = st.temperature.data_ptr(), st.top_k.data_ptr(), st.top_p.data_ptr()
    d.seed, d.token_index = st.seed.data_ptr(), st.index.data_ptr()
    d.tokens, d.tokens_stride, d.column, d.flags = out.data_ptr(), out.stride(0), col, 1
    return d


def _pen(st, **over):
    from pyramidkv_b200 import _lib
    p = _lib.SamplePenalty()
    p.struct_bytes = C.sizeof(_lib.SamplePenalty)
    p.repetition_penalty, p.presence_penalty = st.repetition_penalty.data_ptr(), st.presence_penalty.data_ptr()
    p.frequency_penalty, p.min_p = st.frequency_penalty.data_ptr(), st.min_p.data_ptr()
    p.prompt_mask, p.counts, p.stride = st.prompt_mask.data_ptr(), st.counts.data_ptr(), st.prompt_mask.shape[1]
    for k, v in over.items():
        setattr(p, k, v)
    return p


def test_argument_errors(libpkv):
    from pyramidkv_b200 import _lib, ops
    dev = _dev(libpkv)
    V = 1000
    logits = _logits(4, V, torch.bfloat16, 2, dev)
    st = _State([(1.0, 0, 1.0, 0, 0, 1.2, 0.0, 0.0, 0.0)] * 4, dev, V)
    out = torch.empty(4, 2, dtype=torch.long, device=dev)
    L = _lib.lib()
    stream = torch.cuda.current_stream().cuda_stream
    assert L.pkv_sample_tokens_penalized(C.byref(_desc(logits, st, out, 1)), C.byref(_pen(st)), stream) == _lib.PKV_OK
    bad = [dict(struct_bytes=8), dict(repetition_penalty=None), dict(presence_penalty=st.presence_penalty.data_ptr() + 2),
           dict(frequency_penalty=None), dict(min_p=st.min_p.data_ptr() + 1), dict(prompt_mask=None), dict(counts=None),
           dict(counts=st.counts.data_ptr() + 2), dict(stride=V - 1)]
    for over in bad:
        assert L.pkv_sample_tokens_penalized(C.byref(_desc(logits, st, out, 1)), C.byref(_pen(st, **over)), stream) == \
            _lib.PKV_ERR_INVALID_ARG, over
        assert _lib.last_error()
    d = _desc(logits, st, out, 1)
    d.column = 2                                                    # the errors of pkv_sample_tokens stay
    assert L.pkv_sample_tokens_penalized(C.byref(d), C.byref(_pen(st)), stream) == _lib.PKV_ERR_INVALID_ARG
    d = _desc(logits, st, out, 1)
    d.dtype = 5
    assert L.pkv_sample_tokens_penalized(C.byref(d), C.byref(_pen(st)), stream) == _lib.PKV_ERR_UNSUPPORTED_DTYPE
    assert L.pkv_sample_tokens_penalized(C.byref(_desc(logits, st, out, 1)), None, stream) == _lib.PKV_ERR_INVALID_ARG
    assert L.pkv_sample_tokens_penalized(None, C.byref(_pen(st)), stream) == _lib.PKV_ERR_INVALID_ARG
    for name, val in (("prompt_mask", st.prompt_mask.bool()), ("counts", st.counts.long()),
                      ("prompt_mask", st.prompt_mask[:, : V - 1].contiguous()), ("min_p", st.min_p.double())):
        keep = getattr(st, name)
        setattr(st, name, val)
        with pytest.raises(ValueError):
            ops.sample_tokens_penalized(logits, st, out, 0)
        setattr(st, name, keep)
    with pytest.raises(NotImplementedError):
        ops.sample_tokens_penalized(logits.float(), st, out, 0)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        ops.sample_tokens_penalized(logits.cpu(), st, out, 0)
    torch.cuda.synchronize()
