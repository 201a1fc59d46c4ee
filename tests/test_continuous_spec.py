"""Prompt-lookup speculation in the continuous loop (`greedy_generate_continuous(prompt_lookup_num_tokens=K)`,
`ContinuousSpecDecoder`, DESIGN.md §4.14) on the CPU, through the test-only backend (tests/oracle_continuous_spec_backend.py):
rule 2' (pack) on hand cases and against the scan the kernel computes, the loop end to end over every non-window cache form
against the plain continuous loop (divergences only at counted near ties), the draft budget D, forced drafts, the row
counts, the refusals, the runner flag and the ctypes mirrors of the new structs."""
import random

import pytest
import torch

import test_spec as TS
from oracle_continuous_spec_backend import OracleContinuousSpecBackend, pack
from pyramidkv_b200 import _lib
from pyramidkv_b200 import generate as G
from pyramidkv_b200 import runner


@pytest.fixture(autouse=True)
def _restore():
    yield
    from pyramidkv.monkeypatch import restore
    restore()


# ---- rule 2' ----
def test_pack_hand_cases():
    # four live slots wanting 3, 2, 4, 1 drafts, D = 5, rotation from slot 0: 3, 2, then nothing left
    assert pack([0, 0, 0, 0], [3, 2, 4, 1], [9, 9, 9, 9], 5, 0) == ([3, 2, 0, 0], [4, 3, 1, 1], [0, 4, 7, 8])
    # the same from slot 2 (step 6, B = 4): slot 2 takes 4, slot 3 takes 1, slots 0 and 1 none
    assert pack([0, 0, 0, 0], [3, 2, 4, 1], [9, 9, 9, 9], 5, 6) == ([0, 0, 4, 1], [1, 1, 5, 2], [0, 1, 2, 7])
    # a done slot gets no row and takes no budget; the m - 1 cap: budget 2 leaves one draft token, budget 1 none
    assert pack([0, 1, 0, 0], [3, 3, 3, 3], [2, 9, 1, 9], 4, 0) == ([1, 0, 0, 3], [2, 0, 1, 4], [0, 2, 2, 3])
    # every slot done: no rows at all
    assert pack([1, 1], [2, 2], [5, 5], 4, 1) == ([0, 0], [0, 0], [0, 0])


def _pack_by_scan(done, draft_len, budget, D, step):
    """The formulation of pkv_spec_pack: one scan in rotation order; d' = min(want, max(0, D - P)), P the drafts wanted
    before; the rows before position k are L + min(P, D); slot order shifts the starts by the rows of slots 0 .. r0 - 1."""
    B = len(done)
    r0 = step % B
    P = L = 0
    granted, count, R = [0] * B, [0] * B, [0] * B
    for k in range(B):
        b = (r0 + k) % B
        live = 0 if done[b] else 1
        want = max(0, min(draft_len[b], budget[b] - 1)) if live else 0
        granted[b] = min(want, max(0, D - P))
        count[b] = live + granted[b]
        R[b] = L + min(P, D)
        P += want
        L += live
    rows = L + min(P, D)
    shift = rows - R[0] if r0 else 0
    start = [R[b] + shift if b >= r0 else R[b] - R[0] for b in range(B)]
    return granted, count, start


def test_pack_random_against_the_scan():
    rng = random.Random(3)
    for _ in range(2000):
        B = rng.randint(1, 40)
        K = rng.randint(1, 15)
        done = [rng.random() < 0.3 for _ in range(B)]
        dl = [rng.randint(0, K) for _ in range(B)]
        bud = [rng.randint(0, 30) for _ in range(B)]
        D = rng.randint(1, B * K)
        step = rng.randint(0, 10 ** 6)
        got = pack(done, dl, bud, D, step)
        assert got == _pack_by_scan(done, dl, bud, D, step)
        granted, count, start = got
        assert sum(granted) <= D and sum(count) <= B + D
        assert all(start[b] + count[b] == start[b + 1] for b in range(B - 1))
        # a slot before the rotation start gets a draft only when every slot from it on got all it wanted
        r0 = step % B
        order = [(r0 + k) % B for k in range(B)]
        short = [b for b in order if not done[b] and granted[b] < max(0, min(dl[b], bud[b] - 1))]
        if short:
            assert all(granted[b] == 0 for b in order[order.index(short[0]) + 1:])


# ---- the loop end to end ----
FORMS = TS.FORMS


def _model(arch="tiny-llama", method="pyramidkv", fp8=False, gqa=False, dtype=torch.bfloat16):
    runner.patch(method)
    model = runner.build_model(arch, torch.device("cpu"), dtype, "eager")
    runner.set_knobs(model, method, 48, backend_factory=OracleContinuousSpecBackend)
    if fp8:
        model.config.pkv_kv_cache_dtype = "fp8_e4m3"
    if gqa:
        model.config.pkv_gqa_shared = True
    return model


class _Recording(G.ContinuousSpecDecoder):
    """Checks, at every step, that each slot emitted the argmaxes of its own verify rows (the first always, draft j while
    it equals the argmax before it), and keeps per request (keyed by its prompt's storage) the logits row of each emitted
    token, the slot's cache rows at admission and its emitted count; `steps`: per step, (row counts, tokens emitted)."""
    made = []

    def __init__(self, model, cache, first_token, prompts, *args, **kwargs):
        super().__init__(model, cache, first_token, prompts, *args, **kwargs)
        _Recording.made.append(self)
        self.slot_key = [p.data_ptr() for p in prompts]
        self.slot_rows0 = [[list(l.rows_host[b]) for l in self.layers] for b in range(len(prompts))]
        self.slot_emitted = [0] * len(prompts)
        self.by_req = {k: [] for k in self.slot_key}
        self.steps = []

    def admit(self, slot, src_cache, first_token, left, sampling=None, prompt=None, forced=None):
        super().admit(slot, src_cache, first_token, left, sampling, prompt, forced)
        self.slot_key[slot] = prompt.data_ptr()
        self.slot_rows0[slot] = [list(l.rows_host[0]) for l in src_cache.layers]
        self.slot_emitted[slot] = 0
        self.by_req[prompt.data_ptr()] = []

    def _verify_logits(self):
        logits = super()._verify_logits()
        pk = self.state.pack
        self._rec = (logits[0].float().clone(), pk.row_start.tolist(), pk.row_count.tolist(), pk.ids[0].tolist())
        return logits

    def _step(self):
        st = self.spec
        o0 = st.out_len.tolist()
        super()._step()
        logits, start, count, ids = self._rec
        o1 = st.out_len.tolist()
        emitted = []
        for b in range(len(o0)):
            toks = st.out[b, o0[b]:o1[b]].tolist()
            assert len(toks) <= count[b], "a slot emitted more tokens than it had rows"
            for k, t in enumerate(toks):
                row = logits[start[b] + k]
                assert t == int(row.argmax()), "an emitted token is not the argmax of its verify row"
                if k:
                    assert ids[start[b] + k] == toks[k - 1], "a token after a rejected draft was emitted"
                self.by_req[self.slot_key[b]].append(row)
            self.slot_emitted[b] += len(toks)
            emitted.append(len(toks))
        self.steps.append((count, emitted))


def _run(model, prompts, caps, slots, K, D=None, eos=None, forced=None, monkeypatch=None, use_graph=None):
    monkeypatch.setattr(G, "ContinuousSpecDecoder", _Recording)
    _Recording.made = []
    seqs, stats = G.greedy_generate_continuous(model, prompts, caps, slots, eos_token_id=eos, check_every=3,
                                               return_stats=True, prompt_lookup_num_tokens=K, max_draft_tokens=D,
                                               _forced_drafts=forced, use_graph=use_graph)
    monkeypatch.undo()
    return seqs, stats, _Recording.made[0]


def _check(model, prompts, caps, slots, K, D=None, eos=None, forced=None, monkeypatch=None, ref=None, use_graph=None):
    """The loop against the plain continuous loop: equal tokens per request up to a divergence that is a near tie of the
    verify row that produced it (test_spec._check_loop's rule), and every layer's row counts of each slot's last request
    equal its prompt rows plus the tokens it emitted. Returns (sequences, stats, decoder, near ties)."""
    if ref is None:
        ref = G.greedy_generate_continuous(model, prompts, caps, slots, eos_token_id=eos, check_every=3)
    seqs, stats, dec = _run(model, prompts, caps, slots, K, D, eos, forced, monkeypatch, use_graph)
    ties = 0
    for p, a, r in zip(prompts, seqs, ref):
        got, want = a[p.numel():].tolist(), r[p.numel():].tolist()
        if got == want:
            continue
        j = next((i for i, (x, y) in enumerate(zip(got, want)) if x != y), None)
        assert j is not None and j >= 1, "the spec loop ends a request at another length without a divergence"
        row = dec.by_req[p.data_ptr()][j - 1]
        gap = float(row[got[j]] - row[want[j]])
        assert 0 <= gap <= 0.05 * max(1.0, float(row.abs().max())), f"diverges at {j} by {gap}: not a near tie"
        ties += 1
    for b in range(len(dec.slot_key)):
        for i, l in enumerate(dec.cache.layers):
            H = len(dec.slot_rows0[b][i])
            got = l.rows[b * H:(b + 1) * H].tolist()
            assert got == [r + dec.slot_emitted[b] for r in dec.slot_rows0[b][i]], f"slot {b} layer {i} row counts"
    assert stats["accepted_drafts"] <= stats["granted_drafts"]
    if ties:
        print(f"near ties: {ties}")
    return seqs, stats, dec, ties


LENGTHS = [90, 61, 120, 75, 50, 100, 70]
CAPS = [9, 14, 5, 12, 3, 10, 7]


def _prompts(model, n, seed=0):
    return [p.reshape(1, -1) for p in TS._prompts(model, LENGTHS[:n], seed=seed, repeat=True)]


@pytest.mark.parametrize("method, fp8, gqa", FORMS)
@pytest.mark.parametrize("slots", [1, 3])
def test_loop_every_form(method, fp8, gqa, slots, monkeypatch):
    model = _model(method=method, fp8=fp8, gqa=gqa)
    prompts = _prompts(model, 5 + slots % 3)
    _check(model, prompts, CAPS[:len(prompts)], slots, 4, monkeypatch=monkeypatch)


@pytest.mark.parametrize("arch, dtype, slots", [("tiny-mistral", torch.bfloat16, 2), ("tiny-llama", torch.float16, 2)])
def test_loop_arch_dtype_eos(arch, dtype, slots, monkeypatch):
    model = _model(arch=arch, dtype=dtype)
    prompts = _prompts(model, 7, seed=4)
    caps = CAPS[:7]
    plain = G.greedy_generate_continuous(model, prompts, caps, slots)
    eos = [plain[0][prompts[0].numel() + 3].item(), plain[3][prompts[3].numel() + 5].item()]
    _, stats, _, _ = _check(model, prompts, caps, slots, 3, eos=eos, monkeypatch=monkeypatch)
    assert stats["admissions"] > 0 and stats["decode_steps"] > 0


@pytest.mark.parametrize("D", ["1", "K", "BK"])
def test_draft_budget(D, monkeypatch):
    model = _model()
    prompts = _prompts(model, 6, seed=2)
    caps, K, B = CAPS[:6], 4, 3
    d = {"1": 1, "K": K, "BK": B * K}[D]
    ref = G.greedy_generate_continuous(model, prompts, caps, B, check_every=3)
    _, stats, dec, _ = _check(model, prompts, caps, B, K, D=d, monkeypatch=monkeypatch, ref=ref)
    assert all(sum(c) <= B + d for c, _ in dec.steps)
    assert stats["granted_drafts"] <= d * stats["decode_steps"]


def test_forced_drafts(monkeypatch):
    model = _model()
    prompts = _prompts(model, 5, seed=5)
    caps, K, B = [13, 9, 11, 6, 10], 3, 2
    ref = G.greedy_generate_continuous(model, prompts, caps, B, check_every=3)
    table = [r[p.numel():] for r, p in zip(ref, prompts)]
    seqs, stats, dec, ties = _check(model, prompts, caps, B, K, D=B * K, forced=table, monkeypatch=monkeypatch, ref=ref)
    full = sum(all(e == c for c, e in zip(counts, emitted)) for counts, emitted in dec.steps)
    print(f"all-accepted steps: {full} of {len(dec.steps)}, near ties {ties}")
    if not ties:
        assert full == len(dec.steps), "drafts equal to the greedy continuation are not all accepted"
        assert stats["accepted_drafts"] == stats["granted_drafts"]
    wrong = [(t + 1) % model.config.vocab_size for t in table]
    _, stats, dec, _ = _check(model, prompts, caps, B, K, D=B * K, forced=wrong, monkeypatch=monkeypatch, ref=ref)
    assert all(e == (1 if c else 0) for counts, emitted in dec.steps for c, e in zip(counts, emitted)), \
        "wrong drafts must emit one token per step"
    assert stats["accepted_drafts"] == 0


def test_repeating_prompts_accept_drafts(monkeypatch):
    model = _model()
    prompts = [p.reshape(1, -1) for p in TS._prompts(model, [120, 96, 144], seed=9, repeat=True)]
    _, stats, _, _ = _check(model, prompts, [30, 30, 30], 2, 6, monkeypatch=monkeypatch)
    print(f"granted {stats['granted_drafts']}, accepted {stats['accepted_drafts']}")
    assert stats["accepted_drafts"] > 0


def test_refusals():
    model = _model()
    p = _prompts(model, 1)
    f = G.greedy_generate_continuous
    for kw in (dict(prompt_lookup_num_tokens=0), dict(prompt_lookup_num_tokens=16), dict(prompt_lookup_num_tokens=True),
               dict(prompt_lookup_num_tokens=4, max_matching_ngram_size=9), dict(max_matching_ngram_size=2),
               dict(max_draft_tokens=3), dict(prompt_lookup_num_tokens=4, max_draft_tokens=0),
               dict(prompt_lookup_num_tokens=4, max_draft_tokens=9), dict(prompt_lookup_num_tokens=4, max_draft_tokens=True),
               dict(prompt_lookup_num_tokens=4, sampling=G.SamplingParams()), dict(prompt_lookup_num_tokens=4, logprobs=2)):
        with pytest.raises(ValueError):
            f(model, p, 8, 2, **kw)
    for knob, val in (("pkv_decode_window", 8), ("pkv_decode_heavy", 2)):
        model.config.pkv_decode_window = 8
        setattr(model.config, knob, val)
        with pytest.raises(NotImplementedError, match=knob):
            f(model, p, 8, 2, prompt_lookup_num_tokens=4)
        model.config.pkv_decode_window = model.config.pkv_decode_heavy = None


def test_default_is_unchanged():
    model = _model()
    prompts = _prompts(model, 5)
    a, sa = G.greedy_generate_continuous(model, prompts, CAPS[:5], 2, return_stats=True)
    b, sb = G.greedy_generate_continuous(model, prompts, CAPS[:5], 2, return_stats=True, prompt_lookup_num_tokens=None,
                                         max_matching_ngram_size=None, max_draft_tokens=None)
    assert all(torch.equal(x, y) for x, y in zip(a, b))
    timing = ("prefill_s", "decode_s", "prefill_ms")
    assert {k: v for k, v in sa.items() if k not in timing} == {k: v for k, v in sb.items() if k not in timing}
    assert "granted_drafts" not in sa


def test_runner_flag():
    kw = dict(device=torch.device("cpu"), dtype=torch.bfloat16, attn_implementation="eager",
              backend_factory=OracleContinuousSpecBackend)
    tasks = [("a", 80, 9), ("b", 60, 5), ("c", 70, 7)]
    recs = runner.run_suite("tiny-llama", "pyramidkv", 48, tasks, decode_loop="continuous", eval_batch_size=2,
                            prompt_lookup_num_tokens=3, **kw)
    for rec, (_, _, n) in zip(recs, tasks):
        assert rec["prompt_lookup_num_tokens"] == 3 and len(rec["pred_ids"]) == n
        assert {"granted_drafts", "accepted_drafts"} <= set(rec["continuous"])
    for loop, bs in (("hf", 1), ("static-eager", 2)):
        with pytest.raises(NotImplementedError):
            runner.run_suite("tiny-llama", "pyramidkv", 48, tasks, decode_loop=loop, eval_batch_size=bs,
                             prompt_lookup_num_tokens=3, **kw)
    with pytest.raises(NotImplementedError):
        runner.run_suite("tiny-llama", "fullkv", 48, tasks, decode_loop="continuous", eval_batch_size=2,
                         prompt_lookup_num_tokens=3, **kw)


@pytest.mark.parametrize("name, cls", [("pkv_decode_packed", _lib.DecodePacked), ("pkv_spec_pack_desc", _lib.SpecPackDesc)])
def test_struct_mirrors_match_header(name, cls):
    TS.test_struct_mirrors_match_header(name, cls)
