"""CPU: the oracle against the restated torch chain (oracle/torch_chain.py) on the attention landscapes of
tests/attention_landscapes.py (sinks, heavy hitters, near one-hot rows, bf16-subnormal probabilities, outlier channels,
repeated keys, fp16 masks that round to -inf).

The GPU tests lean on the oracle in exactly these regimes, so it is pinned to the reference there first:
- every landscape's regime check passes (the regime is really present);
- exact-dot landscapes: the oracle's pooled scores equal torch_chain.scores bit for bit, and its indices equal
  select(tie_rule="lowest_index"), set and order, on every head;
- the others: logits within 2 ulp (rounding order of the dot product), and pooled scores within 2 ulp of their own magnitude
  when the oracle's softmax, window sum and pool run on torch's own logits."""
import pytest
import torch

from attention_landscapes import NAMES, assert_stage2, build


def _dtype_for(name):
    return torch.float16 if name == "fp16mask" else torch.bfloat16


CASES = [(name, Hq, Hkv, S, D, W, kernel, pooling)
         for name in NAMES
         for (Hq, Hkv, S, D, W, kernel, pooling) in [(4, 1, 600, 128, 8, 7, "maxpool"), (8, 2, 777, 64, 16, 5, "avgpool"),
                                                     (4, 2, 1100, 128, 32, 7, "maxpool")]]


def _torch_scores(L, kernel, pooling):
    from oracle import torch_chain as tc
    G = L.q.shape[0] // L.k.shape[0]
    return tc.scores("snapkv", tc.repeat_kv(L.k[None], G), L.q[None], L.W, kernel, pooling)[0]


@pytest.mark.parametrize("name,Hq,Hkv,S,D,W,kernel,pooling", CASES)
def test_landscape_oracle_equals_torch_chain(oracle, name, Hq, Hkv, S, D, W, kernel, pooling):
    from oracle import torch_chain as tc
    dt = _dtype_for(name)
    if name == "outlier" and D == 64:
        dt = torch.float16                      # the fp16 variant (|q.k| < 65504)
    L = build(name, Hq, Hkv, S, D, W, dt, seed=S + W)
    L.check(oracle)
    n = S - W
    top_k = min(n, max(8, n // 8))
    if name == "subnormal":
        top_k = min(n, L.info["normal"] + 8)    # reach into the subnormal band
    r = oracle.evict("snapkv", L.q, L.k, L.v, W, top_k, kernel, pooling)
    ts = _torch_scores(L, kernel, pooling)
    if L.exact:
        assert torch.equal(r.pooled.view(torch.int16), ts.view(torch.int16)), "pooled scores differ from torch_chain"
        assert torch.equal(r.idx, tc.select(ts, top_k, tie_rule="lowest_index")), "indices differ from select(lowest_index)"
    else:
        G = Hq // Hkv
        tl = torch.matmul(L.q[None][..., -W:, :], tc.repeat_kv(L.k[None], G).transpose(2, 3)) / (D ** 0.5)
        tl[:, :, :, -W:] += tc._window_mask(W, tl.dtype, tl.device)
        tl = tl[0]
        fin = torch.isfinite(r.logits.float()) & (r.logits.float() > -1e30)
        assert torch.equal(fin, torch.isfinite(tl.float()) & (tl.float() > -1e30))
        from attention_landscapes import ulp_own
        assert float(ulp_own(r.logits[fin], tl[fin], dt).max()) <= 2
        re = oracle.pool(oracle.window_sum(oracle.softmax_rows(tl.contiguous())), kernel, pooling)
        assert_stage2(re, ts, "pooled on torch's logits")
        assert torch.equal(oracle.topk(ts.contiguous(), top_k), tc.select(ts, top_k, tie_rule="lowest_index"))


def test_subnormal_band_is_what_a_flushing_exp_loses(oracle):
    """The issue's reproduction: with probabilities below 2^-126 flushed (as ex2.approx.ftz does), most non-zero pooled
    scores vanish and the selection changes; the oracle keeps them, as torch does."""
    L = build("subnormal", 4, 1, 600, 128, 8, torch.bfloat16, seed=3, band=9)
    r = oracle.evict("snapkv", L.q, L.k, L.v, 8, 64, 7, "maxpool")
    pr = r.probs.float()
    flushed = torch.where(pr.abs() < 2.0 ** -126, torch.zeros_like(pr), pr).to(torch.bfloat16)
    pooled_ftz = oracle.pool(oracle.window_sum(flushed.contiguous()), 7, "maxpool")
    nz, nz_ftz = int((r.pooled.float() != 0).sum()), int((pooled_ftz.float() != 0).sum())
    assert nz > 2 * nz_ftz
    assert not torch.equal(oracle.topk(pooled_ftz, 64), r.idx)
