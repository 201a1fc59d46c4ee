"""Token log-probabilities (the `logprobs=` argument of the three loops, `generate.score_continuations`,
`pkv_token_logprobs`). The CPU oracle of the rules (oracle/logprobs.py) against a direct fp64 log_softmax; then the loops
through the test-only backend on the CPU (`-m gpu`: through libpkv on a tiny random-init model, graph on and off) over every
cache form: the tokens do not change, the top entry is the greedy token, scoring the greedy continuations reproduces the
generated log-probabilities bit for bit, continuous batching adds no dependence on the slot, and with nothing evicted the
scores are those of a dense forward."""
import math

import numpy as np
import pytest
import torch

from oracle import logprobs as LP
from oracle_logprobs_backend import OracleLogprobsBackend
from pyramidkv_b200 import generate as G
from pyramidkv_b200 import runner

DEVICES = ["cpu", pytest.param("cuda", marks=pytest.mark.gpu)]
# (method, kv cache dtype FP8, GQA-shared, decode window R)
FORMS = [("pyramidkv", False, False, None), ("pyramidkv", True, False, None), ("pyramidkv", False, True, None),
         ("pyramidkv", True, True, None), ("adakv", False, False, None), ("headkv", False, False, None),
         ("pyramidkv", False, False, 3)]
LENGTHS = (150, 37, 300, 20, 90)
CAPS = [5, 9, 3, 7, 4]


@pytest.fixture(autouse=True)
def _restore():
    yield
    from pyramidkv.monkeypatch import restore
    restore()


def _model(request, device, method="pyramidkv", fp8=False, gqa=False, window=None, capacity=48):
    runner.patch(method)
    if device == "cpu":
        dev = torch.device("cpu")
        model = runner.build_model("tiny-llama", dev, torch.bfloat16, "eager")
        runner.set_knobs(model, method, capacity, backend_factory=OracleLogprobsBackend)
    else:
        request.getfixturevalue("libpkv")
        from gpu_util import dev as gpu
        dev = gpu()
        model = runner.build_model("tiny-llama", dev, torch.bfloat16, "sdpa")
        runner.set_knobs(model, method, capacity)
    if fp8:
        model.config.pkv_kv_cache_dtype = "fp8_e4m3"
    if gqa:
        model.config.pkv_gqa_shared = True
    model.config.pkv_decode_window = window
    return model, dev


def _graph_modes(device):
    return [False] if device == "cpu" else [False, True]


def _prompts(model, dev, lengths, seed=11):
    return [runner.synthetic_prompt(model.config.vocab_size, n, seed + i, dev) for i, n in enumerate(lengths)]


def _lists(seqs):
    return [t.tolist() for t in seqs]


def _same(a: G.TokenLogprobs, b: G.TokenLogprobs) -> bool:
    """Equal bit for bit (NaN included)."""
    return (torch.equal(a.token_ids, b.token_ids) and torch.equal(a.top_ids, b.top_ids)
            and torch.equal(a.logprobs.view(torch.int32), b.logprobs.view(torch.int32))
            and torch.equal(a.top_logprobs.view(torch.int32), b.top_logprobs.view(torch.int32)))


def _check_greedy_entries(seqs, prompts, lps, N):
    for s, p, e in zip(seqs, prompts, lps):
        gen = s[p.reshape(-1).shape[0]:].cpu()
        n = gen.shape[0]
        assert e.token_ids.tolist() == gen.tolist()
        assert e.logprobs.shape == (n,) and e.logprobs.dtype == torch.float32
        assert e.top_ids.shape == (n, N) and e.top_logprobs.shape == (n, N)
        assert torch.isfinite(e.logprobs).all() and (e.logprobs <= 0).all()
        if N:
            assert torch.equal(e.top_ids[:, 0], gen)                       # the greedy token is the top entry
            assert torch.equal(e.top_logprobs[:, 0], e.logprobs)
            assert (e.top_logprobs[:, :-1] >= e.top_logprobs[:, 1:]).all()


# ---- the oracle ----
def test_oracle_against_log_softmax():
    g = np.random.default_rng(3)
    for V, N in ((1, 0), (1, 3), (7, 5), (1000, 20), (32000, 1)):
        x = torch.from_numpy(g.standard_normal(V) * 3).to(torch.bfloat16).float().numpy()
        ref = torch.log_softmax(torch.from_numpy(x).double(), dim=0).numpy()
        for t in (0, V - 1, V // 2):
            lp, ids, top = LP.logprobs_row(x, t, N)
            assert abs(lp - ref[t]) < 1e-12
        n = min(N, V)
        order = sorted(range(V), key=lambda i: (-x[i], i))[:n]
        assert ids[:n].tolist() == order and np.allclose(top[:n], ref[order], rtol=0, atol=1e-12)
        assert (ids[n:] == -1).all() and np.isnan(top[n:]).all()
        assert math.isnan(LP.logprobs_row(x, V, N)[0]) and math.isnan(LP.logprobs_row(x, -1, N)[0])


def test_oracle_ties_and_non_finite_rows():
    x = np.array([1.0, 3.0, 2.0, 3.0, 2.0, 2.0, 0.5], dtype=np.float32)
    _, ids, top = LP.logprobs_row(x, 0, 4)
    assert ids.tolist() == [1, 3, 2, 4]                                    # logit descending, index ascending
    assert top[0] == top[1] and top[2] == top[3]
    assert LP.logprobs_row(np.full(5, 1.5, dtype=np.float32), 2, 3)[1].tolist() == [0, 1, 2]
    assert abs(LP.logprobs_row(np.full(5, 1.5, dtype=np.float32), 2, 0)[0] + math.log(5)) < 1e-12
    for bad in (np.nan, np.inf, -np.inf):
        y = x.copy()
        y[4] = bad
        lp, ids, top = LP.logprobs_row(y, 1, 3)
        assert math.isnan(lp) and ids.tolist() == [-1, -1, -1] and np.isnan(top).all()


# ---- the loops ----
@pytest.mark.parametrize("device", DEVICES)
@pytest.mark.parametrize("method,fp8,gqa,window", FORMS)
def test_loops_report_logprobs_and_score_reproduces_them(oracle, request, device, method, fp8, gqa, window):
    """logprobs=N leaves the tokens of logprobs=None, reports the greedy token as the top entry at every step, and
    score_continuations on the greedy continuations returns the same log-probabilities, bit for bit."""
    model, dev = _model(request, device, method, fp8, gqa, window)
    prompts = _prompts(model, dev, LENGTHS)
    for use_graph in _graph_modes(device):
        one = G.greedy_generate(model, prompts[0].reshape(1, -1), 6, use_graph=use_graph)
        got, lps = G.greedy_generate(model, prompts[0].reshape(1, -1), 6, use_graph=use_graph, logprobs=5)
        assert got.tolist() == one.tolist() and len(lps) == 1
        _check_greedy_entries([got[0]], prompts[:1], lps, 5)
        ref = G.greedy_generate_batch(model, prompts[:3], 6, use_graph=use_graph)
        seqs, lps = G.greedy_generate_batch(model, prompts[:3], 6, use_graph=use_graph, logprobs=2)
        assert _lists(seqs) == _lists(ref)
        _check_greedy_entries(seqs, prompts[:3], lps, 2)
        scored = G.score_continuations(model, prompts[:3], [e.token_ids for e in lps], top_n=2, use_graph=use_graph)
        assert all(_same(a, b) for a, b in zip(scored, lps)), use_graph
        seqs0, lps0 = G.greedy_generate_batch(model, prompts[:3], 6, use_graph=use_graph, logprobs=0)
        assert _lists(seqs0) == _lists(ref) and all(e.top_ids.shape == (6, 0) for e in lps0)
        assert all(torch.equal(a.logprobs, b.logprobs) for a, b in zip(lps0, lps))
        cont = G.greedy_generate_continuous(model, prompts, CAPS, 2, use_graph=use_graph, check_every=3)
        got, lpc = G.greedy_generate_continuous(model, prompts, CAPS, 2, use_graph=use_graph, check_every=3, logprobs=3)
        assert _lists(got) == _lists(cont)
        _check_greedy_entries(got, prompts, lpc, 3)


@pytest.mark.parametrize("device", DEVICES)
@pytest.mark.parametrize("method,fp8,gqa,window", [FORMS[1], FORMS[2], FORMS[4], FORMS[6]])
def test_continuous_logprobs_equal_lockstep(oracle, request, device, method, fp8, gqa, window):
    """Each request's log-probabilities in continuous batching equal those of a lock-step batch of three (the setting in
    which tests/test_continuous.py shows the greedy tokens equal), greedy and sampled."""
    model, dev = _model(request, device, method, fp8, gqa, window)
    prompts = _prompts(model, dev, LENGTHS)
    n = len(prompts)
    sps = [G.SamplingParams(temperature=(0.6, 1.0, 1.3)[i % 3], top_k=(0, 50, 7)[i % 3], seed=100 + i) for i in range(n)]
    for use_graph in _graph_modes(device):
        for samp in (None, sps):
            want = []
            for r in range(n):
                trio = [r, (r + 1) % n, (r + 2) % n]
                _, lps = G.greedy_generate_batch(model, [prompts[i] for i in trio], CAPS[r], use_graph=use_graph, logprobs=4,
                                                 sampling=None if samp is None else [samp[i] for i in trio])
                want.append(lps[0])
            got, st, lpc = G.greedy_generate_continuous(model, prompts, CAPS, 3, use_graph=use_graph, check_every=2,
                                                        return_stats=True, sampling=samp, logprobs=4)
            assert st["admissions"] == 2
            for r in range(n):
                assert _same(lpc[r], want[r]), (use_graph, samp is None, r)
                assert lpc[r].token_ids.tolist() == got[r][LENGTHS[r]:].tolist()


@pytest.mark.parametrize("device", DEVICES)
def test_sampled_tokens_scored_under_the_raw_distribution(oracle, request, device):
    """With sampling the entries score the drawn tokens under log_softmax(logits): the tokens are those of logprobs=None,
    and forcing them through score_continuations gives the same numbers (temperature and filters play no part)."""
    model, dev = _model(request, device)
    prompts = _prompts(model, dev, (150, 90))
    sp = [G.SamplingParams(temperature=1.3, top_k=20, top_p=0.9, seed=7), G.SamplingParams(temperature=0.5, seed=8)]
    for use_graph in _graph_modes(device):
        ref = G.greedy_generate_batch(model, prompts, 8, use_graph=use_graph, sampling=sp)
        seqs, lps = G.greedy_generate_batch(model, prompts, 8, use_graph=use_graph, sampling=sp, logprobs=3)
        assert _lists(seqs) == _lists(ref)
        for s, p, e in zip(seqs, prompts, lps):
            assert e.token_ids.tolist() == s[p.shape[1]:].tolist()
        scored = G.score_continuations(model, prompts, [e.token_ids for e in lps], top_n=3, use_graph=use_graph)
        assert all(_same(a, b) for a, b in zip(scored, lps))


@pytest.mark.parametrize("device", DEVICES)
@pytest.mark.parametrize("method,fp8,gqa,window", [FORMS[0], FORMS[2], FORMS[4], ("pyramidkv", False, False, 8)])
def test_score_without_eviction_matches_a_dense_forward(oracle, request, device, method, fp8, gqa, window):
    """Budget above every prompt length (and a decode window above the steps taken): nothing is evicted, and the scores of continuations of different lengths (trimmed
    on the host) are the log_softmax of one dense forward over prompt + continuation, within the bf16 rounding of the two
    computations (tolerance 0.05, against log-probabilities of about -7 for the tiny model's 32000 tokens)."""
    model, dev = _model(request, device, method, fp8, gqa, window, capacity=512)
    prompts = _prompts(model, dev, (40, 25, 60))
    g = torch.Generator().manual_seed(4)
    conts = [torch.randint(1, model.config.vocab_size, (n,), generator=g) for n in (6, 1, 4)]
    for use_graph in _graph_modes(device):
        scored = G.score_continuations(model, prompts, conts, top_n=1, use_graph=use_graph)
        assert [e.token_ids.tolist() for e in scored] == [c.tolist() for c in conts]
        from pyramidkv.monkeypatch import restore
        restore()
        for p, c, e in zip(prompts, conts, scored):
            full = torch.cat([p.reshape(-1), c.to(p.device)]).reshape(1, -1)
            with torch.no_grad():
                logits = model(input_ids=full).logits[0].float()
            S = p.shape[1]
            ref = torch.log_softmax(logits[S - 1:S - 1 + c.numel()], dim=-1)
            want = ref.gather(1, c.to(ref.device).reshape(-1, 1))[:, 0].cpu()
            err = float((e.logprobs - want).abs().max())
            assert err < 0.05, (use_graph, err)
        runner.patch(method)


def test_logprobs_argument_errors(oracle, request):
    model, dev = _model(request, "cpu")
    prompts = _prompts(model, dev, (150, 37))
    for bad in (-1, 21, 1.5, True, "3"):
        with pytest.raises((ValueError, TypeError)):
            G.greedy_generate(model, prompts[0].reshape(1, -1), 3, logprobs=bad)
        with pytest.raises((ValueError, TypeError)):
            G.greedy_generate_batch(model, prompts, 3, logprobs=bad)
        with pytest.raises((ValueError, TypeError)):
            G.greedy_generate_continuous(model, prompts, 3, 2, logprobs=bad)
        with pytest.raises((ValueError, TypeError)):
            G.score_continuations(model, prompts, [[1], [2]], top_n=bad)
    with pytest.raises(ValueError, match="one per prompt"):
        G.score_continuations(model, prompts, [[1, 2]])
    with pytest.raises(ValueError, match="at least one token"):
        G.score_continuations(model, prompts, [[1, 2], []])
    # the return value gains one element, the cache and the stats stay where they were
    seq, cache, lps = G.greedy_generate(model, prompts[0].reshape(1, -1), 3, return_cache=True, logprobs=0)
    assert seq.shape == (1, 153) and len(lps) == 1 and lps[0].logprobs.shape == (3,)
    seqs, st, lps = G.greedy_generate_continuous(model, prompts, 3, 1, return_stats=True, logprobs=1)
    assert st["admissions"] == 1 and [e.top_ids.shape for e in lps] == [(3, 1), (3, 1)]


def test_score_continuations_refuses_fullkv(oracle):
    runner.patch("fullkv")
    model = runner.build_model("tiny-llama", torch.device("cpu"), torch.bfloat16, "eager")
    p = runner.synthetic_prompt(model.config.vocab_size, 30, 1, torch.device("cpu"))
    with pytest.raises(RuntimeError, match="fullkv"):
        G.score_continuations(model, [p], [[5, 6]])
