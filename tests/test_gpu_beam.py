"""The beam search kernels (include/pkv.h: pkv_beam_candidates, pkv_beam_step, pkv_cache_reorder) against their
restatement (oracle/beam.py) and torch: candidate ids exactly (ties by index), the step exactly when fed the kernel's own
candidates, every reorder byte-equal to a torch gather with prompt rows, rows past n and other prompts untouched, and a
graph replay equal to a host launch."""
import numpy as np
import pytest
import torch

from oracle import beam as OB
from oracle_beam_backend import reorder_twin, state_view
from pyramidkv_b200 import generate as G
from pyramidkv_b200 import kv_cluster

pytestmark = pytest.mark.gpu
BK = kv_cluster.CudaBackend()


def test_cuda_division_by_host_scalar(libpkv):
    """torch's CUDA division of an fp32 tensor by a Python float d multiplies by f32(1 / d), the reciprocal taken in
    double (what the kernel and oracle/beam.py's "cuda" form do); its CPU division divides by f32(d)."""
    from gpu_util import dev
    g = torch.Generator().manual_seed(0)
    x = -torch.rand(1 << 16, generator=g) * 40
    for t in range(1, 300):          # 299 lengths x 5 penalties: 1495 (t, lp) pairs of 65536 values each
        for lp in (1.0, 2.0, -1.0, 0.5, 1.3):
            d = t ** lp
            got = (x.to(dev()) / d).cpu()
            assert torch.equal(got.view(torch.int32), (x * torch.tensor(1.0 / d, dtype=torch.float32)).view(torch.int32))
            assert torch.equal((x / d).view(torch.int32), (x / torch.tensor(d, dtype=torch.float32)).view(torch.int32))


@pytest.mark.parametrize("V", [1000, 32000, 128256])
@pytest.mark.parametrize("k", [2, 4, 8, 16])
@pytest.mark.parametrize("n_eos", [0, 1, 2, 3, 4])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_candidates(libpkv, V, k, n_eos, dtype):
    from gpu_util import dev
    K = max(2, 1 + n_eos) * k
    g = torch.Generator().manual_seed(V + k)
    x = (torch.randn(k, V, generator=g) * 3).to(dtype)
    x[0, :K + 5] = x[0, 7]                      # ties inside a row
    x[1] = x[0]                                 # and across rows
    if k > 2:
        x[2, 5] = float("nan")
        x[3 % k, 9] = float("inf")
    st = G.BeamState(1, k, 4, list(range(n_eos)), 1.0, False, dev())
    logits = x.to(dev())
    BK.beam_candidates(logits, st)
    torch.cuda.synchronize()
    xf = x.float()
    for r in range(k):
        row = xf[r]
        if not torch.isfinite(row).all():
            assert (st.cand_id[r].cpu() == -1).all() and torch.isinf(st.cand_lp[r].cpu()).all()
            continue
        ids = torch.sort(row, descending=True, stable=True).indices[:K]
        assert torch.equal(st.cand_id[r].cpu().long(), ids)
        ref = torch.log_softmax(row.double(), -1)[ids]
        assert (st.cand_lp[r].cpu().double() - ref).abs().max() < 1e-5 + 1e-6 * ref.abs().max()
        assert float(st.m[r]) == float(row.max())
        # log Z within the bound of pkv_token_logprobs (DESIGN.md §4.8): 1.3e-6 absolute and one ulp of log Z
        log_z = torch.logsumexp(row.double() - row.double().max(), -1)
        assert abs(float(st.log_z[r]) - float(log_z)) <= 1.3e-6 + 2.0 ** -23 * float(log_z)


def _crafted(P, k, T, n_eos, es, lp, seed, dev):
    """A state some steps in: random running scores, a partly filled pool, some frozen prompts."""
    st = G.BeamState(P, k, T, list(range(3, 3 + n_eos)), lp, es, dev)
    g = torch.Generator().manual_seed(seed)
    B = P * k
    run = (-torch.rand(B, generator=g) * 20).round() / 2           # ties across beams
    st.running.copy_(torch.sort(run.view(P, k), descending=True).values.reshape(-1).to(dev))
    pool = torch.where(torch.rand(B, generator=g) < 0.5, -torch.rand(B, generator=g) * 5, torch.full((B,), -1e9))
    pool = torch.sort(pool.view(P, k), descending=True).values.reshape(-1)
    st.pool_score.copy_(pool.to(dev))
    st.pool_done.copy_((pool > -1e8).to(torch.uint8).to(dev))
    st.pool_step.copy_(torch.where(pool > -1e8, 0, -1).to(torch.int32).to(dev))
    st.done.copy_((torch.rand(P, generator=g) < 0.2).to(torch.uint8).to(dev))
    st.cp.copy_(torch.randint(0, 3, (P, k, k), generator=g, dtype=torch.int32).to(dev))
    return st


@pytest.mark.parametrize("k", [2, 4, 16])
@pytest.mark.parametrize("n_eos", [0, 1, 4])
@pytest.mark.parametrize("es", [False, True, "never"])
@pytest.mark.parametrize("lp", [1.0, 0.0, -1.0, 2.0])
def test_step_matches_oracle(libpkv, k, n_eos, es, lp):
    from gpu_util import dev
    P, T, V = 5, 6, 50          # a small vocabulary: EOS ids and ties among candidates are frequent
    st = _crafted(P, k, T, n_eos, es, lp, k * 100 + n_eos, dev())
    g = torch.Generator().manual_seed(k)
    step = torch.zeros(1, dtype=torch.int32, device=dev())
    for t in (2, T - 1):        # a middle iteration and the last one
        logits = (torch.randn(P * k, V, generator=g) * 2).round().to(torch.bfloat16).to(dev())   # many ties
        step.fill_(t)
        BK.beam_candidates(logits, st)
        ref = {f: getattr(st, f).cpu().clone() for f in ("cand_lp", "cand_id")}
        host = G.BeamState(P, k, T, st.eos, lp, es, "cpu")
        for f in ("running", "pool_score", "pool_step", "pool_parent", "pool_token", "pool_done", "heuristic", "done",
                  "bp_token", "bp_parent", "cp", "next_token", "parent", "diverge"):
            getattr(host, f).copy_(getattr(st, f).cpu())
        BK.beam_step(st, k, step, 0)
        OB.step(state_view(host), ref["cand_lp"].numpy(), ref["cand_id"].numpy(), k, t, "cuda")
        for f in ("running", "pool_score", "pool_step", "pool_parent", "pool_token", "pool_done", "heuristic", "done",
                  "bp_token", "bp_parent", "cp", "next_token", "parent", "diverge"):
            a, b = getattr(st, f).cpu(), getattr(host, f)
            if a.dtype == torch.float32:
                a, b = a.view(torch.int32), b.view(torch.int32)
            assert torch.equal(a, b), (f, t)


def _cache(form, P, k, H, cap, D, dev, g):
    fp8, window, heavy = form
    B = P * k
    if fp8:
        kb = (torch.randn(B, H, cap, D, generator=g)).to(torch.float8_e4m3fn).to(dev)
        vb = (torch.randn(B, H, cap, D, generator=g)).to(torch.float8_e4m3fn).to(dev)
        ks, vs = torch.rand(B, H, cap, generator=g).to(dev), torch.rand(B, H, cap, generator=g).to(dev)
    else:
        kb = torch.randn(B, H, cap, D, generator=g).bfloat16().to(dev)
        vb = torch.randn(B, H, cap, D, generator=g).bfloat16().to(dev)
        ks = vs = None
    prompt = torch.randint(3, 9, (P, 1, H), generator=g).expand(P, k, H).reshape(-1).to(torch.int32).to(dev)
    hstate = None
    if heavy:
        hstate = (torch.rand(B, H, window, generator=g).to(dev), torch.randint(0, 50, (B, H, window), generator=g,
                  dtype=torch.int32).to(dev), torch.randint(0, window, (B * H,), generator=g, dtype=torch.int32).to(dev))
    return (kb, vb, ks, vs, prompt.contiguous(), window, hstate)


@pytest.mark.parametrize("form", [(False, None, False), (True, None, False), (False, 5, False), (True, 5, False),
                                  (False, 6, True), (True, 6, True)])
@pytest.mark.parametrize("pattern", ["identity", "swap", "cycle", "one", "random"])
@pytest.mark.parametrize("graph", [False, True])
def test_reorder(libpkv, form, pattern, graph):
    from gpu_util import dev
    P, k, H, D, n = 3, 4, 4, 128, 13
    g = torch.Generator().manual_seed(hash((form, pattern)) % 1000)
    layers = [_cache(form, P, k, H, 8 + n + 3, D, dev(), g) for _ in range(3)]
    par = {"identity": [list(range(k))], "swap": [[1, 0, 3, 2]], "cycle": [[1, 2, 3, 0]], "one": [[2] * k],
           "random": [torch.randint(0, k, (k,), generator=g).tolist()]}[pattern] * P
    parent = torch.tensor([x for row in par for x in row], dtype=torch.int32, device=dev())
    diverge = torch.randint(0, n + 1, (P * k,), generator=g, dtype=torch.int32).to(dev())
    diverge = torch.where(parent == torch.arange(P * k, device=dev(), dtype=torch.int32) % k, n, diverge)
    step = torch.tensor([n - 1], dtype=torch.int32, device=dev())
    cl = lambda t: None if t is None else t.cpu().clone()   # noqa: E731
    ref = [(cl(a), cl(b), cl(c), cl(d), cl(e), w, None if h is None else tuple(cl(x) for x in h))
           for a, b, c, d, e, w, h in layers]
    reorder_twin(ref, P, k, parent.cpu(), diverge.cpu(), step.cpu(), 1)
    if graph:
        gr = torch.cuda.CUDAGraph()
        with torch.cuda.graph(gr):
            BK.cache_reorder(layers, P, k, parent, diverge, step, 1)
        gr.replay()
    else:
        BK.cache_reorder(layers, P, k, parent, diverge, step, 1)
    torch.cuda.synchronize()
    for got, want in zip(layers, ref):
        for a, b in zip(got[:4], want[:4]):
            if a is not None:
                assert torch.equal(a.cpu().view(torch.uint8), b.view(torch.uint8))
        if got[6] is not None:
            for a, b in zip(got[6], want[6]):
                assert torch.equal(a.cpu(), b)
