"""Repetition, presence and frequency penalties and min-p (SamplingParams' new fields, `pkv_sample_tokens_penalized`,
DESIGN.md §4.10). The CPU restatement of the rules (tests/oracle_penalty_backend.py) on hand-built rows; then the loops
through the test-only backend (`-m gpu`: through libpkv on the tiny models, graph on and off): greedy with a repetition
penalty gives HF `generate(do_sample=False, repetition_penalty=r)`'s tokens on every cache form and with a decode window
of 3 rows, default fields give today's tokens, continuous batching equals lock-step batches, and an admission rebuilds only
its own slot's prompt mask and counts."""
import numpy as np
import pytest
import torch

import oracle_penalty_backend as OP
from oracle import sampling as S
from oracle_penalty_backend import OraclePenaltyBackend
from pyramidkv_b200 import generate as G
from pyramidkv_b200 import runner

DEVICES = ["cpu", pytest.param("cuda", marks=pytest.mark.gpu)]
# (arch, method, kv cache dtype FP8, GQA-shared, decode window)
FORMS = [("tiny-llama", "pyramidkv", False, False, None), ("tiny-mistral", "snapkv", False, False, None),
         ("tiny-llama", "pyramidkv", True, False, None), ("tiny-llama", "pyramidkv", False, True, None),
         ("tiny-llama", "adakv", False, False, None), ("tiny-llama", "headkv", False, False, None),
         ("tiny-llama", "pyramidkv", False, False, 3)]
LENGTHS = (150, 37, 300, 20, 90)
CAPS = [9, 4, 12, 7, 5]


@pytest.fixture(autouse=True)
def _restore():
    yield
    from pyramidkv.monkeypatch import restore
    restore()


def _model(request, device, arch="tiny-llama", method="pyramidkv", fp8=False, gqa=False, window=None, capacity=48):
    runner.patch(method)
    if device == "cpu":
        dev = torch.device("cpu")
        model = runner.build_model(arch, dev, torch.bfloat16, "eager")
        runner.set_knobs(model, method, capacity, backend_factory=OraclePenaltyBackend)
    else:
        request.getfixturevalue("libpkv")
        from gpu_util import dev as gpu
        dev = gpu()
        model = runner.build_model(arch, dev, torch.bfloat16, "sdpa")
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


def _hf(model, ids, new, rho):
    ids = ids.reshape(1, -1)
    with torch.no_grad():
        return model.generate(ids, attention_mask=torch.ones_like(ids), max_new_tokens=new, min_new_tokens=new, num_beams=1,
                              do_sample=False, repetition_penalty=rho, pad_token_id=0)


# ---- the rules ----
def test_repetition_sign_rule_and_prompt_only_tokens():
    l = np.array([2.0, -2.0, 0.0, -0.0, 3.0, -1.0], dtype=np.float32)
    mask = np.array([1, 1, 1, 1, 0, 0], dtype=np.uint8)
    counts = np.array([0, 0, 0, 0, 0, 2], dtype=np.int32)
    x = OP.penalize(l, 2.0, 0.0, 0.0, mask, counts)
    assert x.tolist() == [1.0, -4.0, 0.0, 0.0, 3.0, -2.0]        # divide the positive, multiply the negative; ±0 stay 0
    assert np.signbit(x[3]) and not np.signbit(x[2])
    x = OP.penalize(l, 0.5, 0.0, 0.0, mask, counts)              # rho < 1 promotes
    assert x.tolist() == [4.0, -1.0, 0.0, 0.0, 3.0, -0.5]
    # presence and frequency count generated tokens only: a prompt-only token is untouched by them
    x = OP.penalize(l, 1.0, 0.25, 0.5, mask, counts)
    assert x.tolist() == [2.0, -2.0, 0.0, 0.0, 3.0, np.float32(-1.0 - 0.5 * 2 - 0.25)]


def test_counts_above_one_and_fp32_rounding():
    l = np.array([1.0, 1.0, 1.0], dtype=np.float32)
    counts = np.array([0, 1, 7], dtype=np.int32)
    x = OP.penalize(l, 1.3, 0.1, 0.3, np.zeros(3, np.uint8), counts)
    r = np.float32(1.0) / np.float32(1.3)
    want2 = np.float32(np.float32(r - np.float32(np.float32(0.3) * np.float32(7))) - np.float32(0.1))
    assert x[0] == 1.0 and x[2] == want2 and x[1] > x[2]


def test_penalty_demotes_the_argmax_and_ties_go_to_the_lower_index():
    l = np.array([1.0, 4.0, 2.0, 3.0], dtype=np.float32)
    counts = np.array([0, 1, 0, 0], dtype=np.int32)
    assert OP.sample_row_penalized(l, 0.0, 0, 1.0, 1, 0).token == 1
    assert OP.sample_row_penalized(l, 0.0, 0, 1.0, 1, 0, repetition=2.0, counts=counts).token == 3     # 4 / 2 = 2 < 3
    assert OP.sample_row_penalized(l, 0.0, 0, 1.0, 1, 0, presence=1.5, counts=counts).token == 3       # 4 - 1.5 < 3
    # penalty-made ties: 4 - 2 * 1 = 2 = x_2, and 2 > 1.5: the lower index wins
    l2 = np.array([1.0, 4.0, 2.0, 1.5], dtype=np.float32)
    assert OP.sample_row_penalized(l2, 0.0, 0, 1.0, 1, 0, frequency=2.0, counts=counts).token == 1
    l3 = np.array([2.0, 4.0, 2.0], dtype=np.float32)
    assert OP.sample_row_penalized(l3, 0.0, 0, 1.0, 1, 0, repetition=2.0, counts=np.array([0, 1, 0], np.int32)).token == 0
    # invalid parameters: token -1
    assert OP.sample_row_penalized(l, 1.0, 0, 1.0, 1, 0, repetition=0.0).token == -1
    assert OP.sample_row_penalized(l, 1.0, 0, 1.0, 1, 0, presence=float("inf")).token == -1
    assert OP.sample_row_penalized(l, 1.0, 0, 1.0, 1, 0, min_p=1.5).token == -1


def test_min_p_at_zero_one_boundary_and_after_top_k_top_p():
    l = np.log(np.array([0.5, 0.25, 0.125, 0.125], dtype=np.float64)).astype(np.float32)
    d0 = OP.sample_row_penalized(l, 1.0, 0, 1.0, 5, 0, min_p=0.0)
    assert d0.kept.all()
    d1 = OP.sample_row_penalized(l, 1.0, 0, 1.0, 5, 0, min_p=1.0)
    assert d1.kept.tolist() == [True, False, False, False] and d1.token == 0
    # at the boundary: exp(x_1 - x_0) = 0.5 exactly in fp32 for these logits -> kept at min_p 0.5, dropped just above
    assert float(np.exp(np.float64(l[1]) - np.float64(l[0]))) == pytest.approx(0.5, rel=1e-6)
    dlo = OP.sample_row_penalized(l, 1.0, 0, 1.0, 5, 0, min_p=0.4)
    dhi = OP.sample_row_penalized(l, 1.0, 0, 1.0, 5, 0, min_p=0.6)
    assert dlo.kept.tolist() == [True, True, False, False] and dhi.kept.tolist() == [True, False, False, False]
    assert OP.sample_row_penalized(l, 1.0, 0, 1.0, 5, 0, min_p=0.5).near_top_p          # counted as a boundary case
    # after top-k / top-p: min-p only removes from their set
    d = OP.sample_row_penalized(l, 1.0, 1 + 1, 1.0, 5, 0, min_p=0.1)
    assert d.kept.tolist() == [True, True, False, False]
    d = OP.sample_row_penalized(l, 1.0, 0, 0.6, 5, 0, min_p=0.1)
    assert d.kept.tolist() == [True, True, False, False]


def test_defaults_are_the_unpenalized_rules():
    g = np.random.default_rng(3)
    for s in range(20):
        l = (g.standard_normal(300) * 2).astype(np.float32)
        a = OP.sample_row_penalized(l, 0.8, (0, 20)[s % 2], (1.0, 0.9)[s % 2], s, s, mask=np.ones(300, np.uint8),
                                    counts=np.full(300, 0, np.int32))
        b = S.sample_row(l, 0.8, (0, 20)[s % 2], (1.0, 0.9)[s % 2], s, s)
        assert a.token == b.token and (a.kept == b.kept).all()


def test_sampling_params_validation():
    G.SamplingParams(0.0, 0, 1.0, 0, 1.2, -0.5, 1.5, 0.05)                  # positional construction, new fields last
    p = G.SamplingParams(0.7, 0, 0.9, 3)
    assert (p.repetition_penalty, p.presence_penalty, p.frequency_penalty, p.min_p) == (1.0, 0.0, 0.0, 0.0)
    assert not p.penalized and G.SamplingParams(min_p=0.1).penalized and G.SamplingParams(repetition_penalty=0.9).penalized
    for bad in (dict(repetition_penalty=0.0), dict(repetition_penalty=-1.0), dict(repetition_penalty=float("inf")),
                dict(repetition_penalty=float("nan")), dict(presence_penalty=float("nan")),
                dict(frequency_penalty=float("-inf")), dict(min_p=-0.01), dict(min_p=1.01), dict(min_p=float("nan"))):
        with pytest.raises(ValueError):
            G.SamplingParams(**bad)


# ---- the loops ----
@pytest.mark.parametrize("device", DEVICES)
@pytest.mark.parametrize("arch,method,fp8,gqa,window", FORMS)
def test_greedy_repetition_penalty_matches_hf(request, device, arch, method, fp8, gqa, window):
    """temperature 0 with repetition_penalty rho: HF's greedy generate with the same penalty, in all three loops (each
    prompt against its own HF run). With a decode window of 3 the count table still penalizes tokens the ring dropped."""
    model, dev = _model(request, device, arch, method, fp8, gqa, window)
    prompts = _prompts(model, dev, LENGTHS[:3])
    rho = 1.8
    sp = G.SamplingParams(temperature=0.0, repetition_penalty=rho)
    want = [_hf(model, p, CAPS[i], rho)[0].tolist() for i, p in enumerate(prompts)]
    plain = _hf(model, prompts[0], CAPS[0], 1.0)[0].tolist()
    assert want[0] != plain                                    # the penalty changes the tokens here
    for use_graph in _graph_modes(device):
        assert G.greedy_generate(model, prompts[0].reshape(1, -1), CAPS[0], use_graph=use_graph, sampling=sp)[0].tolist() == want[0]
        got = G.greedy_generate_batch(model, prompts, max(CAPS[:3]), use_graph=use_graph, sampling=sp)
        assert [g.tolist()[: len(w)] for g, w in zip(got, want)] == want
        got = G.greedy_generate_continuous(model, prompts, CAPS[:3], 2, use_graph=use_graph, check_every=4, sampling=sp)
        assert _lists(got) == want, use_graph


@pytest.mark.parametrize("device", DEVICES)
def test_default_fields_give_todays_tokens(request, device):
    """Rows at the defaults, next to penalized rows in the same launch, get the tokens of a batch without penalties."""
    model, dev = _model(request, device)
    prompts = _prompts(model, dev, LENGTHS[:3])
    plain = [G.SamplingParams(0.9, 0, 0.95, seed=40 + i) for i in range(3)]
    for use_graph in _graph_modes(device):
        want = G.greedy_generate_batch(model, prompts, 8, use_graph=use_graph, sampling=plain)
        mixed = [plain[0], G.SamplingParams(0.9, 0, 0.95, seed=41, repetition_penalty=1.5, frequency_penalty=0.7, min_p=1.0), plain[2]]
        got = G.greedy_generate_batch(model, prompts, 8, use_graph=use_graph, sampling=mixed)
        assert got[0].tolist() == want[0].tolist() and got[2].tolist() == want[2].tolist()
        assert got[1].tolist() != want[1].tolist()


@pytest.mark.parametrize("device", DEVICES)
@pytest.mark.parametrize("method,fp8,window", [("pyramidkv", False, None), ("pyramidkv", True, None), ("pyramidkv", False, 3)])
def test_continuous_penalized_equals_lockstep(request, device, method, fp8, window):
    model, dev = _model(request, device, method=method, fp8=fp8, window=window)
    prompts = _prompts(model, dev, LENGTHS)
    n = len(prompts)
    sps = [G.SamplingParams(temperature=(0.0, 0.8, 1.2)[i % 3], top_k=(0, 50, 0)[i % 3], top_p=(1.0, 0.9, 1.0)[i % 3],
                            seed=200 + i, repetition_penalty=(1.3, 1.0, 0.9)[i % 3], presence_penalty=(0.0, 0.5, -0.5)[i % 3],
                            frequency_penalty=(0.2, 0.0, 1.5)[i % 3], min_p=(0.0, 0.05, 0.5)[i % 3]) for i in range(n)]
    sps[3] = G.SamplingParams(0.7, 0, 1.0, seed=203)          # one request at the defaults
    for use_graph in _graph_modes(device):
        want = [G.greedy_generate_batch(model, [prompts[r], prompts[(r + 1) % n], prompts[(r + 2) % n]], CAPS[r], use_graph=use_graph,
                                        sampling=[sps[r], sps[(r + 1) % n], sps[(r + 2) % n]])[0].tolist() for r in range(n)]
        for every in (1, 4):
            got, st = G.greedy_generate_continuous(model, prompts, CAPS, 3, use_graph=use_graph, check_every=every,
                                                   return_stats=True, sampling=sps)
            assert _lists(got) == want, (use_graph, every)
            assert st["admissions"] == 2


def test_admission_rebuilds_only_its_slot(request):
    model, dev = _model(request, "cpu")
    prompts = _prompts(model, dev, LENGTHS[:3])
    V = model.lm_head.weight.shape[0]
    sp = G.SamplingParams(0.8, 0, 1.0, seed=1, repetition_penalty=1.4, frequency_penalty=0.3)
    firsts, caches = zip(*[G._prefill(model, p, sp) for p in prompts[:2]])
    from pyramidkv_b200.cache import join_caches
    cache = join_caches(list(caches), reserve=16)
    dec = G.ContinuousDecoder(model, cache, torch.cat(firsts), [6, 6], 4, use_graph=False, sampling=[sp, sp],
                              prompts=prompts[:2])
    st = dec.sampling
    for b in range(2):
        assert st.prompt_mask[b].nonzero().reshape(-1).tolist() == sorted(set(prompts[b].reshape(-1).tolist()))
        assert st.counts[b].sum() == 1 and int(st.counts[b, int(firsts[b])]) == 1
    toks = dec.run_chunk(4)
    for b in range(2):
        assert st.counts[b].sum() == 5
        want = np.bincount([int(firsts[b])] + toks[b].tolist(), minlength=V)
        assert st.counts[b].tolist() == want.tolist()
    keep_mask, keep_counts = st.prompt_mask[0].clone(), st.counts[0].clone()
    first2, single = G._prefill(model, prompts[2], sp)
    dec.grow_for(single, 6)
    dec.admit(1, single, first2, 5, sp, prompts[2])
    assert torch.equal(st.prompt_mask[0], keep_mask) and torch.equal(st.counts[0], keep_counts)
    assert st.prompt_mask[1].nonzero().reshape(-1).tolist() == sorted(set(prompts[2].reshape(-1).tolist()))
    assert st.counts[1].sum() == 1 and int(st.counts[1, int(first2)]) == 1
    assert float(st.repetition_penalty[1]) == pytest.approx(1.4) and int(st.index[1]) == 1
    with pytest.raises(ValueError, match="prompt"):
        dec.admit(1, single, first2, 5, sp)
    plain = G.ContinuousDecoder(model, cache, torch.cat(firsts), [6, 6], 4, use_graph=False,
                                sampling=[G.SamplingParams(), G.SamplingParams()])
    assert not plain.sampling.penalized and not hasattr(plain.sampling, "counts")
    with pytest.raises(ValueError, match="penalties"):
        plain.admit(1, single, first2, 5, sp, prompts[2])
    dec.finish()
