"""Prompt-lookup speculative decoding (`greedy_generate(prompt_lookup_num_tokens=K)`, DESIGN.md §4.13) on the CPU, through
the test-only backend (tests/oracle_spec_backend.py): rule 1 against HF's PromptLookupCandidateGenerator, rule 3 against
HF's acceptance count, the loop end to end over every non-window cache form, forced drafts, and the refusals. The ctypes
mirrors of the new structs are checked against the header here as well."""
import ctypes as C
import os
import random
import re

import pytest
import torch
from transformers.generation.candidate_generator import PromptLookupCandidateGenerator

import oracle_spec_backend as OSB
from oracle import spec as OS
from oracle_spec_backend import OracleSpecBackend
from pyramidkv_b200 import _lib
from pyramidkv_b200 import generate as G
from pyramidkv_b200 import runner


@pytest.fixture(autouse=True)
def _restore():
    yield
    from pyramidkv.monkeypatch import restore
    restore()


# ---- rule 1 and rule 3 ----
def _hf_draft(h, K, N, eos, m):
    gen = PromptLookupCandidateGenerator(eos_token_id=torch.tensor(eos or [-1]), num_output_tokens=K,
                                         max_matching_ngram_size=N, max_length=len(h) + m)
    ids = torch.tensor([h])
    cand, _ = gen.get_candidates(ids)
    return cand[0, len(h):].tolist()


def _histories():
    rng = random.Random(0)
    out = [([1, 2, 3, 4, 5], 4, 2, [], 5),                      # no match
           ([7, 8, 9, 7], 4, 2, [], 5),                         # a match only at the start, reaching the end
           ([1, 2, 3, 9, 2, 3, 5, 1, 2, 3], 3, 3, [], 9),       # several n-gram sizes: the 3-gram wins
           ([5, 6, 0, 4, 1, 9, 5, 6], 5, 2, [4], 9),            # EOS inside the draft
           ([3, 1, 2, 3, 1, 2, 3], 15, 2, [], 20),              # K at the length cap
           ([3, 1, 2, 3, 1, 2, 3], 4, 2, [], 1),                # a budget of 1: no draft
           ([4, 4, 4, 4], 3, 8, [4], 5)]                        # the draft starts with EOS: empty
    for _ in range(300):
        L = rng.randint(2, 40)
        V = rng.choice([3, 5, 20])
        h = [rng.randrange(V) for _ in range(L)]
        eos = rng.sample(range(V), rng.randint(0, min(4, V)))
        out.append((h, rng.randint(1, 15), rng.randint(1, 8), eos, rng.randint(1, 20)))
    return out


@pytest.mark.parametrize("h, K, N, eos, m", _histories())
def test_draft_matches_hf(h, K, N, eos, m):
    assert OS.draft(h, K, N, eos, m) == _hf_draft(h, K, N, eos, m)


def test_accept_matches_hf_n_matches():
    rng = random.Random(1)
    for _ in range(500):
        d = rng.randint(0, 15)
        draft = [rng.randrange(4) for _ in range(d)]
        t = [rng.randrange(4) for _ in range(d + 1)]
        m = rng.randint(1, 20)
        cand = torch.tensor([draft])
        sel = torch.tensor([t])
        n = int(((~(cand == sel[:, :-1])).cumsum(dim=-1) < 1).sum())    # _assisted_decoding, greedy branch
        assert OS.accept(draft, t, m) == t[: min(n, m - 1) + 1]


def test_accept_stops_after_eos():
    assert OS.accept([5, 6, 7], [5, 6, 7, 8], 10, eos=[6]) == [5, 6]


# ---- the loop end to end ----
FORMS = [("pyramidkv", False, False), ("pyramidkv", True, False), ("pyramidkv", False, True), ("pyramidkv", True, True),
         ("adakv", False, False), ("headkv", False, False)]


def _model(arch="tiny-llama", method="pyramidkv", fp8=False, gqa=False, dtype=torch.bfloat16, capacity=48):
    runner.patch(method)
    model = runner.build_model(arch, torch.device("cpu"), dtype, "eager")
    runner.set_knobs(model, method, capacity, backend_factory=OracleSpecBackend)
    if fp8:
        model.config.pkv_kv_cache_dtype = "fp8_e4m3"
    if gqa:
        model.config.pkv_gqa_shared = True
    return model


def _prompts(model, lengths, seed=0, repeat=False):
    out = []
    for i, n in enumerate(lengths):
        p = runner.synthetic_prompt(model.config.vocab_size, n if not repeat else 24, seed + i, torch.device("cpu"))[0]
        out.append(p.repeat((n + 23) // 24)[:n] if repeat else p)
    return out


class _Recording(G.SpeculativeDecoder):
    """Keeps, per step, the verify logits and the state the step started from."""

    def _verify_logits(self):
        logits = super()._verify_logits()
        st = self.spec
        self.records.append((logits.float().clone(), st.ids.clone(), st.out_len.clone(), st.done.clone()))
        return logits


def _spec_run(model, prompts, T, K, N=2, eos=None, forced=None, cls=_Recording):
    firsts, caches = [], []
    for p in prompts:
        f, c = G._prefill(model, p.reshape(1, -1))
        firsts.append(f)
        caches.append(c)
    prompt_rows = [[l.rows_host[0] for l in c.layers] for c in caches]
    cache = G.join_caches(caches, reserve=T + K)
    first = torch.cat(firsts)
    cls.records = []
    dec = cls(model, cache, first, [p.reshape(-1) for p in prompts], T, K, N, use_graph=False, eos_token_id=eos,
              forced_drafts=forced)
    dec.records = []
    dec.run_to_end(4)
    gen = dec.generated()
    dec.finish([len(g) for g in gen])
    return first[:, 0].tolist(), gen, cache, prompt_rows, dec


def _check_loop(model, prompts, T, K, eos=None):
    """Every emitted token is the argmax of its verify row; every layer counts prompt rows + emitted tokens; against plain
    greedy the tokens agree up to a divergence that is a near tie of the verify row. Returns the near ties seen."""
    first, gen, cache, prompt_rows, dec = _spec_run(model, prompts, T, K, eos=eos)
    for logits, ids, out_len, done in dec.records:
        for b in range(len(prompts)):
            if bool(done[b]):
                continue
            o0 = int(out_len[b])
            am = logits[b].argmax(dim=-1)
            for k in range(K + 1):
                if o0 + k < len(gen[b]) and (k == 0 or int(ids[b, k]) == int(am[k - 1])):
                    assert gen[b][o0 + k] == int(am[k]), "an emitted token is not the argmax of its verify row"
                else:
                    break
    for i, l in enumerate(cache.layers):
        for b in range(len(prompts)):
            assert l.rows_host[b] == [r + len(gen[b]) for r in prompt_rows[b][i]]
    ties = 0
    for b, p in enumerate(prompts):
        ref = G.greedy_generate(model, p.reshape(1, -1), T, eos_token_id=eos)[0, p.numel():].tolist()
        got = [first[b]] + gen[b]
        if got == ref:
            continue
        j = next(i for i, (x, y) in enumerate(zip(got, ref)) if x != y)
        # the verify row that produced got[j] (j >= 1: a decode-loop token)
        row = None
        for logits, ids, out_len, done in dec.records:
            o0 = int(out_len[b])
            if not bool(done[b]) and o0 <= j - 1 <= o0 + K:
                row = logits[b, j - 1 - o0]
        assert row is not None
        gap = float(row[got[j]] - row[ref[j]])
        assert 0 <= gap <= 0.05 * max(1.0, float(row.abs().max())), f"sequence {b} diverges at {j} by {gap}: not a near tie"
        ties += 1
    if ties:
        print(f"near ties: {ties}")
    return gen, dec


@pytest.mark.parametrize("method, fp8, gqa", FORMS)
@pytest.mark.parametrize("B", [1, 4])
def test_loop_every_form(method, fp8, gqa, B):
    model = _model(method=method, fp8=fp8, gqa=gqa)
    _check_loop(model, _prompts(model, [90, 61, 120, 75][:B], repeat=True), 24, 4)


@pytest.mark.parametrize("arch, dtype", [("tiny-mistral", torch.bfloat16), ("tiny-llama", torch.float16)])
def test_loop_arch_dtype(arch, dtype):
    model = _model(arch=arch, dtype=dtype)
    _check_loop(model, _prompts(model, [70, 101], repeat=True), 20, 3)


def test_loop_eos_and_budget():
    model = _model()
    prompts = _prompts(model, [80, 64, 99], seed=3, repeat=True)
    plain = [G.greedy_generate(model, p.reshape(1, -1), 20)[0, p.numel():].tolist() for p in prompts]
    eos = [plain[0][7], plain[1][3]]
    gen, _ = _check_loop(model, prompts, 20, 5, eos=eos)
    for b in range(3):
        assert len(gen[b]) <= 19


def test_public_entry_points_match_the_loop():
    model = _model()
    prompts = _prompts(model, [64, 90], repeat=True)
    first, gen, _, _, _ = _spec_run(model, prompts, 16, 6, 3)
    seqs = G.greedy_generate_batch(model, prompts, 16, prompt_lookup_num_tokens=6, max_matching_ngram_size=3)
    for b, p in enumerate(prompts):
        assert seqs[b].tolist() == p.tolist() + [first[b]] + gen[b]
    one = G.greedy_generate(model, prompts[0].reshape(1, -1), 16, prompt_lookup_num_tokens=6, max_matching_ngram_size=3)
    assert one[0].tolist() == seqs[0].tolist()


def test_forced_drafts():
    model = _model()
    prompts = _prompts(model, [70, 96], seed=5)
    T, K = 25, 4
    plain = [[int(x) for x in G.greedy_generate(model, p.reshape(1, -1), T)[0, p.numel():]] for p in prompts]
    table = torch.tensor(plain)
    _, gen, _, _, dec = _spec_run(model, prompts, T, K, forced=table)
    near = sum(g != t[1:] for g, t in zip(gen, plain))
    steps = sum(not bool(r[3].all()) for r in dec.records)        # replays past the last sequence's end emit nothing
    if not near:
        assert steps == -(-(T - 1) // (K + 1)), "drafts equal to the greedy continuation are not all accepted"
    print(f"all-accepted drafts: {steps} steps, near ties {near}")
    wrong = (table + 1) % model.config.vocab_size
    _, gen, _, _, dec = _spec_run(model, prompts, T, K, forced=wrong)
    assert sum(not bool(r[3].all()) for r in dec.records) == T - 1 and all(len(g) == T - 1 for g in gen), \
        "wrong drafts must emit one token per step"


def test_repeating_prompt_accepts_more_than_one_token_per_step():
    model = _model()
    prompts = _prompts(model, [120], seed=9, repeat=True)
    _, gen, _, _, dec = _spec_run(model, prompts, 40, 6)
    rate = len(gen[0]) / sum(not bool(r[3].all()) for r in dec.records)
    print(f"tokens per step: {rate:.2f}")
    assert rate > 1.0


def test_refusals():
    model = _model()
    p = _prompts(model, [40])[0].reshape(1, -1)
    for kw in (dict(prompt_lookup_num_tokens=0), dict(prompt_lookup_num_tokens=16), dict(prompt_lookup_num_tokens=True),
               dict(prompt_lookup_num_tokens=4, max_matching_ngram_size=9), dict(max_matching_ngram_size=2),
               dict(prompt_lookup_num_tokens=4, sampling=G.SamplingParams()), dict(prompt_lookup_num_tokens=4, logprobs=2)):
        with pytest.raises(ValueError):
            G.greedy_generate(model, p, 8, **kw)
    with pytest.raises(ValueError):
        G.greedy_generate_batch(model, [p], 8, prompt_lookup_num_tokens=4, sampling=G.SamplingParams())
    for knob, val in (("pkv_decode_window", 8), ("pkv_decode_heavy", 2)):
        model.config.pkv_decode_window = 8
        setattr(model.config, knob, val)
        with pytest.raises(NotImplementedError, match=knob):
            G.greedy_generate(model, p, 8, prompt_lookup_num_tokens=4)
        with pytest.raises(NotImplementedError, match=knob):
            G.greedy_generate_batch(model, [p], 8, prompt_lookup_num_tokens=4)
        model.config.pkv_decode_window = model.config.pkv_decode_heavy = None


def test_default_is_unchanged():
    model = _model()
    p = _prompts(model, [60])[0].reshape(1, -1)
    assert torch.equal(G.greedy_generate(model, p, 10), G.greedy_generate(model, p, 10, prompt_lookup_num_tokens=None))


# ---- the ABI of the new structs ----
def _header_struct(name):
    text = open(os.path.join(os.path.dirname(__file__), "..", "include", "pkv.h")).read()
    body = re.search(r"typedef struct %s \{(.*?)\} %s;" % (name, name), text, re.S).group(1)
    body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    fields = []
    for decl in body.split(";"):
        decl = decl.strip()
        if not decl:
            continue
        parts = decl.replace("*", " * ").split()
        ptr = "*" in parts
        toks = [t for t in parts if t not in ("const",)]
        typ = toks[0]
        rest = " ".join(toks[1:]).replace("*", "").split(",")
        for r in rest:
            fields.append((r.strip(), "ptr" if ptr else typ))
    return fields


SIZES = {"uint32_t": 4, "int32_t": 4, "int64_t": 8, "uint64_t": 8, "ptr": 8, "float": 4}


@pytest.mark.parametrize("name, cls", [("pkv_decode_multi", _lib.DecodeMulti), ("pkv_spec_desc", _lib.SpecDesc)])
def test_struct_mirrors_match_header(name, cls):
    fields = _header_struct(name)
    assert [f for f, _ in fields] == [f for f, _ in cls._fields_]
    off = 0
    for (f, typ), (g, ct) in zip(fields, cls._fields_):
        size = SIZES[typ]
        off = (off + size - 1) // size * size
        assert getattr(cls, g).offset == off, f"{name}.{f}: offset {getattr(cls, g).offset} != {off}"
        assert C.sizeof(ct) == size
        off += size
    assert C.sizeof(cls) == (off + 7) // 8 * 8


def test_twin_out_of_range_writes_nothing():
    k = torch.zeros(1, 2, 8, 64, dtype=torch.bfloat16)
    v = torch.zeros_like(k)
    q = torch.randn(1, 3, 2, 64).bfloat16()
    kn = torch.randn(1, 3, 2, 64).bfloat16()
    out = OSB.multi_twin(q, k, v, kn, kn, rows=torch.tensor([6, 5], dtype=torch.int32))
    assert torch.isnan(out[0, :, 0]).all() and not torch.isnan(out[0, :, 1]).any()
    assert not k[0, 0].any() and torch.equal(k[0, 1, 5:8], kn[0, :, 1])


def test_runner_flag():
    rec = runner.run_suite("tiny-llama", "pyramidkv", 48, [("t", 80, 9)], device=torch.device("cpu"), dtype=torch.bfloat16,
                           attn_implementation="eager", backend_factory=OracleSpecBackend, decode_loop="static-eager",
                           prompt_lookup_num_tokens=3)[0]
    assert rec["prompt_lookup_num_tokens"] == 3 and len(rec["pred_ids"]) == 9
    with pytest.raises(NotImplementedError):
        runner.run_suite("tiny-llama", "pyramidkv", 48, [("t", 80, 9)], device=torch.device("cpu"), decode_loop="hf",
                         backend_factory=OracleSpecBackend, prompt_lookup_num_tokens=3)
