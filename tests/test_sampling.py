"""Sampled decoding (generate.SamplingParams, the `sampling=` argument of the three loops, `pkv_sample_tokens`). The CPU
oracle of the rules (oracle/sampling.py) on known-answer vectors and hand-built rows; then the loops through the test-only
backend on the CPU (`-m gpu`: through libpkv on a tiny random-init model, graph on and off): temperature 0 and top_k 1 give
the greedy tokens bit for bit on every cache form, seeds decide the tokens, and continuous batching adds no dependence on
the slot."""
import numpy as np
import pytest
import torch

from oracle import sampling as S
from oracle_sampling_backend import OracleSamplingBackend
from pyramidkv_b200 import generate as G
from pyramidkv_b200 import runner

DEVICES = ["cpu", pytest.param("cuda", marks=pytest.mark.gpu)]
# (method, kv cache dtype FP8, GQA-shared)
FORMS = [("pyramidkv", False, False), ("pyramidkv", True, False), ("pyramidkv", False, True), ("pyramidkv", True, True),
         ("adakv", False, False), ("headkv", False, False)]
LENGTHS = (150, 37, 300, 20, 90)
CAPS = [5, 9, 3, 7, 4]


@pytest.fixture(autouse=True)
def _restore():
    yield
    from pyramidkv.monkeypatch import restore
    restore()


def _model(request, device, method="pyramidkv", fp8=False, gqa=False, capacity=48):
    runner.patch(method)
    if device == "cpu":
        dev = torch.device("cpu")
        model = runner.build_model("tiny-llama", dev, torch.bfloat16, "eager")
        runner.set_knobs(model, method, capacity, backend_factory=OracleSamplingBackend)
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
    return model, dev


def _graph_modes(device):
    return [False] if device == "cpu" else [False, True]


def _prompts(model, dev, lengths, seed=11):
    return [runner.synthetic_prompt(model.config.vocab_size, n, seed + i, dev) for i, n in enumerate(lengths)]


def _lists(seqs):
    return [t.tolist() for t in seqs]


# ---- the oracle ----
def test_philox_known_answers():
    """Random123's kat_vectors for philox4x32_10."""
    cases = [([0, 0, 0, 0], [0, 0], "6627e8d5 e169c58d bc57ac4c 9b00dbd8"),
             ([0xffffffff] * 4, [0xffffffff] * 2, "408f276d 41c83b0e a20bc7c6 6d5451fd"),
             ([0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344], [0xa4093822, 0x299f31d0], "d16cfe09 94fdcceb 5001e420 24126ea1")]
    for ctr, key, want in cases:
        assert " ".join("%08x" % int(w) for w in S.philox4x32_10(ctr, key)) == want
    u = S.uniforms(1001, 2 ** 64 - 1, 2 ** 40 + 3)
    assert u.shape == (1001,) and (u > 0).all() and (u < 1).all()


def test_oracle_top_k_keeps_ties():
    l = np.array([1.0, 3.0, 2.0, 3.0, 2.0, 2.0, 0.5], dtype=np.float32)
    d = S.sample_row(l, 1.0, 3, 1.0, 7, 0)
    assert d.kept.tolist() == [False, True, True, True, True, True, False]       # the 3rd largest is 2: all three 2s stay
    d = S.sample_row(l, 1.0, 2, 1.0, 7, 0)
    assert d.kept.tolist() == [False, True, False, True, False, False, False]


def test_oracle_top_p_boundary_and_at_least_one():
    # four equal largest logits of mass p4 each: a top_p just under 2 * p4 keeps exactly two of them, the lower indices
    l = np.array([0.0, 5.0, 0.0, 5.0, 5.0, 5.0], dtype=np.float32)
    p4 = np.exp(5.0) / (4 * np.exp(5.0) + 2)
    d = S.sample_row(l, 1.0, 0, 2 * p4 - 0.01, 3, 0)
    assert d.kept.tolist() == [False, True, False, True, False, False]
    d = S.sample_row(l, 1.0, 0, 2 * p4 + 0.01, 3, 0)
    assert d.kept.tolist() == [False, True, False, True, True, False]
    # a tiny top_p keeps one token: the largest, lowest index among ties
    d = S.sample_row(l, 1.0, 0, 1e-6, 3, 0)
    assert d.kept.tolist() == [False, True, False, False, False, False] and d.token == 1
    # top-k applies first: top_p over the renormalised kept set
    l2 = np.array([2.0, 1.0, 0.0, -1.0], dtype=np.float32)
    d = S.sample_row(l2, 1.0, 2, 0.7, 3, 0)                 # softmax over {2, 1}: 0.731, 0.269
    assert d.kept.tolist() == [True, False, False, False]


def test_oracle_greedy_and_nan_rules():
    l = np.array([1.0, 4.0, 4.0, -2.0], dtype=np.float32)
    assert S.sample_row(l, 0.0, 0, 1.0, 1, 5).token == 1
    assert S.sample_row(l, 0.7, 1, 0.9, 1, 5).token == 1
    n = l.copy()
    n[2] = np.nan
    assert S.sample_row(n, 1.0, 0, 1.0, 1, 5).token == 2                        # NaN: torch.argmax's token
    assert S.sample_row(l, 1e-45, 0, 1.0, 1, 5).token == 1                      # x overflows: the argmax
    assert S.sample_row(l, -1.0, 0, 1.0, 1, 5).token == -1


def test_sampling_params_validation():
    G.SamplingParams(0.0, 0, 1.0, 2 ** 64 - 1)
    for bad in (dict(temperature=-0.1), dict(temperature=float("nan")), dict(top_k=-1), dict(top_k=1.5), dict(top_p=0.0),
                dict(top_p=1.01), dict(seed=-1), dict(seed=2 ** 64)):
        with pytest.raises(ValueError):
            G.SamplingParams(**bad)


# ---- the loops ----
@pytest.mark.parametrize("device", DEVICES)
@pytest.mark.parametrize("method,fp8,gqa", FORMS)
def test_greedy_settings_give_greedy_tokens(oracle, request, device, method, fp8, gqa):
    """temperature 0 and top_k 1 give the tokens of sampling=None in all three loops."""
    model, dev = _model(request, device, method, fp8, gqa)
    prompts = _prompts(model, dev, LENGTHS)
    greedy = [G.SamplingParams(temperature=0.0, seed=5), G.SamplingParams(temperature=0.8, top_k=1, top_p=0.5, seed=6)]
    for use_graph in _graph_modes(device):
        ref_one = G.greedy_generate(model, prompts[0].reshape(1, -1), 6, use_graph=use_graph)
        ref_batch = G.greedy_generate_batch(model, prompts[:3], 6, use_graph=use_graph)
        ref_cont = G.greedy_generate_continuous(model, prompts, CAPS, 2, use_graph=use_graph, check_every=3)
        for sp in greedy:
            assert G.greedy_generate(model, prompts[0].reshape(1, -1), 6, use_graph=use_graph, sampling=sp).tolist() == ref_one.tolist()
            assert _lists(G.greedy_generate_batch(model, prompts[:3], 6, use_graph=use_graph, sampling=sp)) == _lists(ref_batch)
        mixed = [greedy[i % 2] for i in range(len(prompts))]
        got = G.greedy_generate_continuous(model, prompts, CAPS, 2, use_graph=use_graph, check_every=3, sampling=mixed)
        assert _lists(got) == _lists(ref_cont), use_graph


@pytest.mark.parametrize("device", DEVICES)
def test_seed_decides_the_tokens(oracle, request, device):
    model, dev = _model(request, device)
    prompts = _prompts(model, dev, (150, 90))
    sp = G.SamplingParams(temperature=1.0, top_k=0, top_p=0.95, seed=1234)
    for use_graph in _graph_modes(device):
        a = G.greedy_generate(model, prompts[0].reshape(1, -1), 12, use_graph=use_graph, sampling=sp)
        b = G.greedy_generate(model, prompts[0].reshape(1, -1), 12, use_graph=use_graph, sampling=sp)
        c = G.greedy_generate(model, prompts[0].reshape(1, -1), 12, use_graph=use_graph,
                              sampling=G.SamplingParams(1.0, 0, 0.95, seed=1235))
        greedy = G.greedy_generate(model, prompts[0].reshape(1, -1), 12, use_graph=use_graph)
        assert a.tolist() == b.tolist()
        assert a[0, 150:].tolist() != c[0, 150:].tolist() and a[0, 150:].tolist() != greedy[0, 150:].tolist()
        # a batch: the prompt's tokens do not depend on its batch position
        ab = G.greedy_generate_batch(model, [prompts[1], prompts[0]], 12, use_graph=use_graph,
                                     sampling=[G.SamplingParams(0.7, 40, 0.9, seed=9), sp])
        assert ab[1].tolist() == a[0].tolist()


@pytest.mark.parametrize("device", DEVICES)
@pytest.mark.parametrize("method,fp8,gqa", [FORMS[0], FORMS[1], FORMS[2], FORMS[4]])
def test_continuous_sampled_equals_lockstep(oracle, request, device, method, fp8, gqa):
    """Each request's sampled tokens in continuous batching equal its tokens in a lock-step batch of three (the setting in
    which tests/test_continuous.py shows the greedy tokens equal): sampling adds no dependence on the slot."""
    model, dev = _model(request, device, method, fp8, gqa)
    prompts = _prompts(model, dev, LENGTHS)
    n = len(prompts)
    sps = [G.SamplingParams(temperature=(0.6, 1.0, 1.3)[i % 3], top_k=(0, 50, 7)[i % 3], top_p=(0.9, 1.0, 0.8)[i % 3],
                            seed=100 + i) for i in range(n)]
    for use_graph in _graph_modes(device):
        want = [G.greedy_generate_batch(model, [prompts[r], prompts[(r + 1) % n], prompts[(r + 2) % n]], CAPS[r], use_graph=use_graph,
                                        sampling=[sps[r], sps[(r + 1) % n], sps[(r + 2) % n]])[0].tolist() for r in range(n)]
        for every in (1, 4):
            got, st = G.greedy_generate_continuous(model, prompts, CAPS, 3, use_graph=use_graph, check_every=every,
                                                   return_stats=True, sampling=sps)
            assert _lists(got) == want, (use_graph, every)
            assert st["admissions"] == 2


def test_sampling_argument_errors(oracle, request):
    model, dev = _model(request, "cpu")
    prompts = _prompts(model, dev, (150, 37))
    with pytest.raises(ValueError, match="one per prompt"):
        G.greedy_generate_batch(model, prompts, 3, sampling=[G.SamplingParams()])
    with pytest.raises(ValueError, match="one per prompt"):
        G.greedy_generate_continuous(model, prompts, 3, 2, sampling=[G.SamplingParams()] * 3)
    with pytest.raises(ValueError, match="SamplingParams"):
        G.greedy_generate(model, prompts[0].reshape(1, -1), 3, sampling=[G.SamplingParams()])
