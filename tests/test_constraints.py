"""Generation constraints (SamplingParams' sequence_bias, no_repeat_ngram_size, bad_words_ids, min_new_tokens and
stop_sequences; `pkv_token_rules` + `pkv_sample_tokens_constrained`, DESIGN.md §4.11). The numpy restatement
(oracle/constraints.py) pinned bit for bit against transformers' own processors; then the three loops through the test-only
backend (`-m gpu`: through libpkv, graph on and off) against HF `generate(do_sample=False, ...)` with the matching kwargs
and, for stop sequences, a StoppingCriteria over the ids."""
import numpy as np
import pytest
import torch
from transformers import StoppingCriteria, StoppingCriteriaList
from transformers.generation import logits_process as LP

from oracle import constraints as OC
from oracle_constraint_backend import OracleConstraintBackend
from pyramidkv_b200 import generate as G
from pyramidkv_b200 import runner

DEVICES = ["cpu", pytest.param("cuda", marks=pytest.mark.gpu)]


@pytest.fixture(autouse=True)
def _restore():
    yield
    from pyramidkv.monkeypatch import restore
    restore()


# ---- the restatement against transformers' processors, bit for bit ----
def _scores(g, V):
    x = (g.standard_normal(V) * 3).astype(np.float32)
    x[g.integers(0, V, 4)] = -0.0
    x[g.integers(0, V, 2)] = np.inf
    x[g.integers(0, V, 2)] = -np.inf
    x[g.integers(0, V, 1)] = np.nan
    return x


def _same(a, b):
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    assert a.view(np.int32).tolist() == b.view(np.int32).tolist() or (
        np.array_equal(np.isnan(a), np.isnan(b)) and a[~np.isnan(a)].view(np.int32).tolist() == b[~np.isnan(b)].view(np.int32).tolist())


def _hf_call(proc, hist, x):
    return proc(torch.tensor([hist]), torch.from_numpy(x.copy()).reshape(1, -1))[0].numpy()


@pytest.mark.parametrize("seed", range(6))
def test_restatement_matches_hf_processors(seed):
    g = np.random.default_rng(seed)
    V = 40
    for trial in range(12):
        n_hist = int(g.integers(1, 12))
        hist = g.integers(0, 6, n_hist).tolist()             # a small alphabet: n-grams and prefixes recur
        x = _scores(g, V)
        # sequence bias: single and longer sequences, longer than the history too, several ending in one token
        pairs, seen = [], set()
        for _ in range(int(g.integers(1, 8))):
            L = int(g.integers(1, 5)) if trial % 3 else int(g.integers(n_hist, n_hist + 3))
            s = tuple(int(t) for t in g.integers(0, 6, L))
            if s not in seen:
                seen.add(s)
                pairs.append((s, float(np.float32(g.standard_normal() * 4))))
        want = _hf_call(LP.SequenceBiasLogitsProcessor({s: w for s, w in pairs}), hist, x)
        _same(OC.add_bias(x, OC.sequence_bias(hist, pairs, V)), want)
        # no-repeat n-grams, n = 1 .. 5 (n > len + 1 included)
        for n in range(1, 6):
            want = _hf_call(LP.NoRepeatNGramLogitsProcessor(n), hist, x)
            _same(OC.apply_bans(x, OC.ngram_bans(hist, n, V)), want)
        # bad words, a single-token EOS among them
        eos = [int(g.integers(0, 6))]
        bad = [list(s) for s, _ in pairs] + [eos]
        want = _hf_call(LP.NoBadWordsLogitsProcessor(bad, eos), hist, x)
        _same(OC.apply_bans(x, np.zeros(V, bool), OC.bad_word_bans(hist, [tuple(b) for b in bad], eos, V)), want)
        # min_new_tokens, below and at the bound
        plen = int(g.integers(0, n_hist + 1))
        for m in (0, n_hist - plen, n_hist - plen + 1):
            want = _hf_call(LP.MinNewTokensLengthLogitsProcessor(plen, m, eos + [7]), hist, x)
            _same(OC.apply_bans(x, OC.min_new_bans(hist, plen, m, eos + [7], V)), want)


def test_restatement_quirks():
    V = 8
    # a bias sequence longer than the history is skipped; the untouched tokens get + 0.0 (-0.0 -> +0.0)
    x = np.array([-0.0, 1, 2, 3, 4, 5, 6, 7], np.float32)
    y = OC.add_bias(x, OC.sequence_bias([1, 2], [((0, 1, 2), 5.0), ((2,), 1.5)], V))
    assert y[2] == 3.5 and y[2 + 0] == 3.5 and not np.signbit(y[0])
    # biases ending in one token sum in order
    b = OC.sequence_bias([2, 3, 4], [((4, 5), 1e8), ((5,), 1.0), ((3, 4, 5), -1e8)], V)
    assert b[5] == np.float32(np.float32(np.float32(0 + 1.0) + 1e8) - 1e8)
    # n-grams: nothing while len + 1 < n; n = 1 bans the whole history
    assert not OC.ngram_bans([1, 2], 4, V).any() and OC.ngram_bans([1, 2, 1], 1, V).nonzero()[0].tolist() == [1, 2]
    # a bad word equal to an EOS id is dropped; a +inf logit under a bad word becomes NaN
    assert not OC.bad_word_bans([1], [(3,)], [3], V).any()
    z = OC.apply_bans(np.array([np.inf] * V, np.float32), np.zeros(V, bool), OC.bad_word_bans([1], [(3,)], [], V))
    assert np.isnan(z[3]) and z[2] == np.inf
    # min_new_tokens without an EOS id does nothing
    assert not OC.min_new_bans([1, 2], 2, 5, [], V).any()
    assert OC.stopped([1, 2, 3], [(2, 3)]) and not OC.stopped([3], [(2, 3)])


def test_sampling_params_validation_and_freezing():
    G.SamplingParams(0.0, 0, 1.0, 0, 1.0, 0.0, 0.0, 0.0, [([1, 2], -1.0)], 3, [[4]], 2, [[5, 6]])     # positional
    p = G.SamplingParams(sequence_bias=[[[1, 2], 2.0]], bad_words_ids=[[3, 4]], stop_sequences=[[9]])
    assert p.sequence_bias == (((1, 2), 2.0),) and p.bad_words_ids == ((3, 4),) and p.stop_sequences == ((9,),)
    assert p.constrained and not G.SamplingParams().constrained and hash(p) == hash(
        G.SamplingParams(sequence_bias=(((1, 2), 2.0),), bad_words_ids=((3, 4),), stop_sequences=((9,),)))
    d = G.SamplingParams()
    assert (d.sequence_bias, d.no_repeat_ngram_size, d.bad_words_ids, d.min_new_tokens, d.stop_sequences) == ((), 0, (), 0, ())
    for bad in (dict(sequence_bias=[([1], float("inf"))]), dict(sequence_bias=[([], 1.0)]), dict(sequence_bias=[([1], 1.0, 2)]),
                dict(sequence_bias=[([1], 1.0), ([1], 2.0)]), dict(sequence_bias=[([-1], 1.0)]), dict(no_repeat_ngram_size=-1),
                dict(no_repeat_ngram_size=1.5), dict(bad_words_ids=[[]]), dict(bad_words_ids=[3]), dict(min_new_tokens=-2),
                dict(stop_sequences=[[1, -2]]), dict(stop_sequences=["ab"])):
        with pytest.raises(ValueError):
            G.SamplingParams(**bad)


def test_forced_tokens_refuse_constraints(request):
    model, dev = _model(request, "cpu")
    prompt = _prompts(model, dev, (40,))[0].reshape(1, -1)
    first, cache = G._prefill(model, prompt)
    with pytest.raises(ValueError, match="exclude"):
        G.StaticDecoder(model, cache, first, 2, use_graph=False, sampling=[G.SamplingParams(0.0, stop_sequences=[[1]])],
                        prompts=[prompt], forced=torch.zeros(1, 2, dtype=torch.long))


# ---- the loops ----
def _model(request, device, arch="tiny-llama", method="pyramidkv", fp8=False, gqa=False, window=None, capacity=48):
    runner.patch(method)
    if device == "cpu":
        dev = torch.device("cpu")
        model = runner.build_model(arch, dev, torch.bfloat16, "eager")
        runner.set_knobs(model, method, capacity, backend_factory=OracleConstraintBackend)
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


def _prompts(model, dev, lengths, seed=11):
    return [runner.synthetic_prompt(model.config.vocab_size, n, seed + i, dev) for i, n in enumerate(lengths)]


class _StopOn(StoppingCriteria):
    def __init__(self, seqs):
        self.seqs = seqs

    def __call__(self, input_ids, scores, **kwargs):
        return torch.tensor([OC.stopped(r.tolist(), self.seqs) for r in input_ids], device=input_ids.device)


def _hf(model, ids, new, p: G.SamplingParams, eos):
    ids = ids.reshape(1, -1)
    kw = {}
    if p.sequence_bias:
        kw["sequence_bias"] = {s: w for s, w in p.sequence_bias}
    if p.no_repeat_ngram_size:
        kw["no_repeat_ngram_size"] = p.no_repeat_ngram_size
    if p.bad_words_ids:
        kw["bad_words_ids"] = [list(s) for s in p.bad_words_ids]
    if p.min_new_tokens:
        kw["min_new_tokens"] = p.min_new_tokens
    if p.repetition_penalty != 1.0:
        kw["repetition_penalty"] = p.repetition_penalty
    if p.stop_sequences:
        kw["stopping_criteria"] = StoppingCriteriaList([_StopOn(p.stop_sequences)])
    with torch.no_grad():
        out = model.generate(ids, attention_mask=torch.ones_like(ids), max_new_tokens=new, num_beams=1, do_sample=False,
                             eos_token_id=eos, pad_token_id=0, **kw)
    return out[0].tolist()


def _rule_sets(prompt, plain):
    """Requests whose rules change the tokens of the unconstrained greedy run `plain` (its generated part) on this prompt:
    each rule alone, the first token included, and all together."""
    g, last = plain, int(prompt.reshape(-1)[-1])

    def unique(pairs):                          # the greedy run may repeat tokens: one bias per sequence
        return [(s, w) for i, (s, w) in enumerate(pairs) if all(s != q for q, _ in pairs[:i])]
    return {
        "bias": dict(sequence_bias=unique([((g[0],), -30.0), ((g[1], g[2]), -30.0), ((g[2], g[3]), 2.5), ((g[3],), 0.5)])),
        "ngram": dict(no_repeat_ngram_size=2),
        "bad": dict(bad_words_ids=[(g[0],), (g[2], g[3])]),
        "min_new": dict(min_new_tokens=6),
        "stop": dict(stop_sequences=[(g[3], g[4]), (last, g[0], g[1], g[2], g[3])]),
        "stop_prompt": dict(stop_sequences=[(last, g[0], g[1])]),
        "all": dict(sequence_bias=[((g[1],), -30.0)], no_repeat_ngram_size=3, bad_words_ids=[(g[2],)], min_new_tokens=4,
                    stop_sequences=[(g[5],)]),
    }


CAP = 10


def _case(model, prompts, rule, penalty):
    """(requests, eos, HF's tokens per prompt) for one rule set."""
    plain = [_hf(model, p, CAP, G.SamplingParams(0.0), None)[p.numel():] for p in prompts]
    eos = plain[0][1] if rule in ("min_new", "all") else None    # an EOS the unconstrained run emits at its second token
    sps = [G.SamplingParams(0.0, repetition_penalty=penalty, **_rule_sets(p, plain[i])[rule]) for i, p in enumerate(prompts)]
    want = [_hf(model, p, CAP, sp, eos) for p, sp in zip(prompts, sps)]
    return plain, sps, eos, want


RULES = ["bias", "ngram", "bad", "min_new", "stop", "stop_prompt", "all"]


@pytest.mark.parametrize("device", DEVICES)
@pytest.mark.parametrize("rule", RULES)
@pytest.mark.parametrize("penalty", [1.0, 1.3])
def test_loops_match_hf(request, device, rule, penalty):
    model, dev = _model(request, device)
    prompts = _prompts(model, dev, (90, 37, 150))
    plain, sps, eos, want = _case(model, prompts, rule, penalty)
    if rule in ("bias", "bad", "stop", "stop_prompt", "min_new") and penalty == 1.0:
        assert want[0] != prompts[0].tolist() + plain[0], "the rule must change the tokens here"
    if rule in ("bias", "bad"):
        assert want[0][prompts[0].numel()] != plain[0][0]          # it fires on the prefill's token
    for use_graph in ([False] if device == "cpu" else [False, True]):
        got = G.greedy_generate(model, prompts[0].reshape(1, -1), CAP, use_graph=use_graph, eos_token_id=eos,
                                sampling=sps[0], check_every=3)
        assert got[0].tolist() == want[0], use_graph
        got = G.greedy_generate_batch(model, prompts, CAP, eos_token_id=eos, use_graph=use_graph, sampling=sps, check_every=3)
        assert [t.tolist() for t in got] == want, use_graph
        got = G.greedy_generate_continuous(model, prompts, CAP, 2, eos_token_id=eos, use_graph=use_graph, check_every=3,
                                           sampling=sps)
        assert [t.tolist() for t in got] == want, use_graph


@pytest.mark.parametrize("device", DEVICES)
def test_constrained_next_to_unconstrained(request, device):
    """A constrained and an unconstrained request in one batch each get their solo tokens."""
    model, dev = _model(request, device)
    prompts = _prompts(model, dev, (90, 37))
    plain = _hf(model, prompts[0], CAP, G.SamplingParams(0.0), None)[prompts[0].numel():]
    sps = [G.SamplingParams(0.0, **_rule_sets(prompts[0], plain)["all"]), G.SamplingParams(0.0)]
    solo = [G.greedy_generate_batch(model, [p], CAP, sampling=[sp], use_graph=False)[0].tolist() for p, sp in zip(prompts, sps)]
    got = G.greedy_generate_batch(model, prompts, CAP, sampling=sps, use_graph=device != "cpu")
    assert [t.tolist() for t in got] == solo
    assert solo[1] == _hf(model, prompts[1], CAP, G.SamplingParams(0.0), None)


@pytest.mark.parametrize("device", DEVICES)
def test_stop_leaves_the_cache_at_the_stop_token(request, device):
    model, dev = _model(request, device)
    prompts = _prompts(model, dev, (90, 37))
    plain = [_hf(model, p, CAP, G.SamplingParams(0.0), None)[p.numel():] for p in prompts]
    sps = [G.SamplingParams(0.0, stop_sequences=[tuple(plain[0][:4])]), G.SamplingParams(0.0)]
    seqs, cache = G.greedy_generate_batch(model, prompts, CAP, sampling=sps, use_graph=device != "cpu", return_cache=True)
    assert seqs[0].tolist() == prompts[0].reshape(-1).tolist() + plain[0][:4]
    ref_seqs, ref_cache = G.greedy_generate_batch(model, prompts, CAP, sampling=[G.SamplingParams(0.0)] * 2,
                                                  use_graph=False, return_cache=True)
    l0, r0 = cache.layers[0], ref_cache.layers[0]
    # the stop token is the last one kept, and, like an EOS, never fed back: the cache holds the tokens before it
    assert l0.seq_seen[0] == prompts[0].numel() + 3 and l0.seq_seen[1] == r0.seq_seen[1]


@pytest.mark.parametrize("device", DEVICES)
def test_stop_sequence_longer_than_the_prompt(request, device):
    """Prompts shorter than their stop sequences: the host keeps the last tokens of prompt + generated, however short the
    prompt, in all three loops."""
    model, dev = _model(request, device)
    prompts = _prompts(model, dev, (3, 37, 2))
    new = 14
    plain = [_hf(model, p, new, G.SamplingParams(0.0), None)[p.numel():] for p in prompts]
    sps = [G.SamplingParams(0.0, stop_sequences=[tuple(plain[0][4:9])]),
           G.SamplingParams(0.0, stop_sequences=[tuple(plain[1][2:8])]),
           G.SamplingParams(0.0, stop_sequences=[tuple(prompts[2].reshape(-1).tolist()) + tuple(plain[2][:4])])]
    want = [_hf(model, p, new, sp, None) for p, sp in zip(prompts, sps)]
    assert all(len(w) < p.numel() + new for w, p in zip(want, prompts))       # every stop sequence ends its sequence
    for use_graph in ([False] if device == "cpu" else [False, True]):
        got = G.greedy_generate(model, prompts[0].reshape(1, -1), new, use_graph=use_graph, sampling=sps[0], check_every=3)
        assert got[0].tolist() == want[0], use_graph
        got = G.greedy_generate_batch(model, prompts, new, use_graph=use_graph, sampling=sps, check_every=3)
        assert [t.tolist() for t in got] == want, use_graph
        for slots in (1, 2):
            got = G.greedy_generate_continuous(model, prompts, new, slots, use_graph=use_graph, check_every=3, sampling=sps)
            assert [t.tolist() for t in got] == want, (use_graph, slots)


def test_sampling_params_take_numpy_and_tensor_ids():
    p = G.SamplingParams(sequence_bias=[(np.array([1, 2]), np.float32(1.5)), (torch.tensor([3]), torch.tensor(-2.0))],
                         bad_words_ids=[np.array([4, 5], dtype=np.int64)], stop_sequences=[torch.tensor([6, 7])],
                         no_repeat_ngram_size=np.int64(3), min_new_tokens=np.int32(2))
    assert p.sequence_bias == (((1, 2), 1.5), ((3,), -2.0)) and p.bad_words_ids == ((4, 5),) and p.stop_sequences == ((6, 7),)
    assert all(type(t) is int for s in p.bad_words_ids + p.stop_sequences for t in s)
    assert (p.no_repeat_ngram_size, p.min_new_tokens) == (3, 2) and hash(p) is not None
    for bad in (dict(sequence_bias=[([1], "1.0")]), dict(sequence_bias=[([1], True)]), dict(bad_words_ids=[[1.5]]),
                dict(bad_words_ids=[torch.tensor(3)]), dict(stop_sequences=[np.array([-1])]),
                dict(sequence_bias=[([1], np.float32("nan"))])):
        with pytest.raises(ValueError):
            G.SamplingParams(**bad)


def test_set_row_checks_ids_before_the_row_changes():
    sp = G.SamplingParams(0.5, seed=1, bad_words_ids=[(3,)], stop_sequences=[(4, 5)])
    st = G.SamplingState([sp, sp], torch.device("cpu"), vocab=16, prompts=[torch.tensor([1, 2]), torch.tensor([7])])
    keep = {k: v.clone() for k, v in vars(st).items() if torch.is_tensor(v)}
    for bad, prompt in ((G.SamplingParams(0.9, seed=9, bad_words_ids=[(16,)]), torch.tensor([1])),
                        (G.SamplingParams(0.9, seed=9, stop_sequences=[(2, 99)]), torch.tensor([1])),
                        (G.SamplingParams(0.9, seed=9, bad_words_ids=[(2,)]), torch.tensor([1, 16]))):
        with pytest.raises(ValueError, match="outside"):
            st.set_row(1, bad, 1, prompt)
        assert all(torch.equal(getattr(st, k), v) for k, v in keep.items())
