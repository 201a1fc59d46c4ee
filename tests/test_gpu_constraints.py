"""`pkv_token_rules` and `pkv_sample_tokens_constrained` on the H100 against the CPU restatement of the rules
(oracle/constraints.py through tests/oracle_constraint_backend.py): bias sums bit-equal, ban sets and stop flags equal over
vocabulary sizes, batch sizes, histories up to 131 072 tokens with n-grams that recur thousands of times and n-grams across
the prompt / generated boundary, and 1 to 1 000 rule sequences per row; the constrained draw against the oracle over the
§4.6 / §4.10 grid with the near-tie cases counted and bounded; unconstrained rows bit-equal to
`pkv_sample_tokens_penalized` in the same launch; graph replay; and the loops over every cache form."""
import itertools

import numpy as np
import pytest
import torch

import oracle_constraint_backend as OCB
import oracle_penalty_backend as OP
from pyramidkv_b200 import generate as G

pytestmark = pytest.mark.gpu


def _dev(libpkv):
    from gpu_util import dev
    return dev()


def _requests(g, B, V, n_seq_max, hist_len, eos):
    """B requests with every rule, their prompts (length hist_len - a few generated tokens) and generated tokens. The
    history uses a small alphabet, so n-grams recur thousands of times in long histories."""
    reqs, prompts, gens = [], [], []
    for b in range(B):
        alpha = g.integers(0, V, 24)
        alpha[0] = V - 1                                       # the last token: the last, partial word of the ban bitmaps
        n = int(hist_len[b])
        hist = alpha[g.integers(0, 24, n)]
        n_gen = int(g.integers(0, min(8, n - 1) + 1))
        ns = int(g.integers(1, n_seq_max + 1))
        seqs = []
        for j in range(ns):
            L = int(g.integers(1, 6)) if j % 7 else int(g.integers(2, 5))
            # often the history's own tail (so it applies), sometimes spanning the prompt / generated boundary
            if j % 3 == 0 and L <= n:
                s = tuple(int(t) for t in hist[n - L + 1:]) + (int(alpha[g.integers(0, 24)]),) if L > 1 else (int(alpha[0]),)
            else:
                s = tuple(int(t) for t in alpha[g.integers(0, 24, L)])
            seqs.append(s)
        bias, seen = [], set()
        for s in seqs[: len(seqs) // 2 + 1]:
            if s not in seen:
                seen.add(s)
                bias.append((s, float(np.float32(g.standard_normal() * 3))))
        stops = [tuple(int(t) for t in hist[n - k:]) for k in (1, 3) if k <= n] if b % 2 else [seqs[-1]]
        kw = dict(sequence_bias=bias, no_repeat_ngram_size=int(1 + b % 5), bad_words_ids=seqs[len(seqs) // 2:] + [(eos[0],)],
                  min_new_tokens=int(g.integers(0, 10)), stop_sequences=stops)
        if b % 5 == 4:
            kw = {}                                            # an unconstrained row
        reqs.append(G.SamplingParams(0.0, **kw))
        prompts.append(torch.from_numpy(hist[: n - n_gen].astype(np.int64)))
        gens.append(hist[n - n_gen:].tolist())
    return reqs, prompts, gens


def _state(reqs, prompts, gens, V, dev, eos):
    st = G.SamplingState(reqs, dev, index=0, vocab=V, prompts=prompts, eos=eos, constraints=True, history=16)
    for b, gen in enumerate(gens):                             # the generated part of the history, appended in place
        for t in gen:
            n = int(st.history_len[b])
            st.history[b, n] = t
            st.history_len[b] = n + 1
    return st


# (V, B, history, extra bias / ban columns); an odd V takes the scalar bias clear (rows not 16-byte aligned) or, with rows
# padded to a multiple of 4, the vector clear and its scalar tail, and the bans of the last, partial word
CASES = [(V, B, L, 0) for V, B, L in itertools.product((1000, 32000, 128256), (1, 7, 64), (40, 4096, 131072))
         if not (B == 64 and L == 131072)] + [(1001, 64, 40, 0), (1001, 7, 4096, 3)]


@pytest.mark.parametrize("V,B,L,pad", CASES)
def test_token_rules_match_oracle(libpkv, V, B, L, pad):
    from pyramidkv_b200 import ops
    dev = _dev(libpkv)
    g = np.random.default_rng(V + B + L)
    eos = [int(g.integers(0, V)), int(g.integers(0, V))]
    lens = g.integers(max(2, L // 2), L + 1, B)
    reqs, prompts, gens = _requests(g, B, V, 1000 if B < 64 else 200, lens, eos)
    st = _state(reqs, prompts, gens, V, dev, eos)
    if pad:
        st.bias = torch.zeros(B, V + pad, dtype=torch.float32, device=dev)
        st.ban = torch.zeros(B, st.ban.shape[1] + pad, dtype=torch.int32, device=dev)
    append = torch.from_numpy(g.integers(0, V, (B, 1)))
    for b in range(1, B, 2):                                   # odd rows: the token completes their (last token,) stop sequence
        append[b, 0] = int(st.history[b, int(st.history_len[b]) - 1])
    append = append.to(dev)
    st.bias.fill_(7.0)
    st.ban.fill_(-1)                                           # stale state from an earlier step must be cleared
    cpu = _cpu_copy(st)
    ops.token_rules(st, V, append, 0)
    torch.cuda.synchronize()
    OCB.token_rules_twin(cpu, V, append.cpu(), 0)
    W = (V + 31) // 32
    for b in range(B):
        flags = int(cpu.rule_flags[b])
        if flags & 1:
            assert torch.equal(st.bias[b].cpu().view(torch.int32), cpu.bias[b].view(torch.int32)), b
        if flags & 6:
            assert torch.equal(st.ban[b, : 2 * W].cpu(), cpu.ban[b, : 2 * W]), b
        assert bool(st.stop[b]) == bool(cpu.stop[b]), b
    assert torch.equal(st.history.cpu(), cpu.history) and torch.equal(st.history_len.cpu(), cpu.history_len)
    assert any(bool(cpu.stop[b]) for b in range(B)) or B == 1


def _cpu_copy(st):
    class C:
        pass
    c = C()
    for k, v in vars(st).items():
        setattr(c, k, v.cpu().clone() if torch.is_tensor(v) else v)
    return c


TEMPS, TOPKS, TOPPS, RHOS, MINPS = (0.0, 0.7, 1.3), (0, 50), (0.9, 1.0), (1.0, 1.3), (0.0, 0.05)


@pytest.mark.parametrize("V", [1000, 1001, 32000, 128256])      # 1001: unaligned bias rows, a partial last group of 4
def test_constrained_sampler_matches_oracle(libpkv, V):
    from pyramidkv_b200 import ops
    dev = _dev(libpkv)
    g = np.random.default_rng(V)
    eos = [3]
    rows = checked = near = 0
    for B in (7, 64):
        lens = g.integers(20, 3000, B)
        reqs, prompts, gens = _requests(g, B, V, 100, lens, eos)
        combos = list(itertools.product(TEMPS, TOPKS, TOPPS, RHOS, MINPS))
        reqs = [G.SamplingParams(c[0], c[1], c[2], seed=1000 + b, repetition_penalty=c[3], min_p=c[4],
                                 **{k: getattr(r, k) for k in ("sequence_bias", "no_repeat_ngram_size", "bad_words_ids",
                                                               "min_new_tokens", "stop_sequences")})
                for b, (r, c) in enumerate(zip(reqs, (combos[(b * 5 + V) % len(combos)] for b in range(B))))]
        st = _state(reqs, prompts, gens, V, dev, eos)
        ops.token_rules(st, V)
        x = torch.randn(B, V, generator=torch.Generator().manual_seed(B)) * 2.5
        x[:, :: max(1, V // 97)] += 4.0
        hist_tok = [int(st.history[b, int(st.history_len[b]) - 1]) for b in range(B)]
        for b in range(B):
            x[b, hist_tok[b]] += 6.0                           # likely tokens the bans and biases act on
        logits = x.to(torch.bfloat16).to(dev)
        out = torch.full((B, 1), -7, dtype=torch.long, device=dev)
        pen = torch.full((B, 1), -7, dtype=torch.long, device=dev)
        ops.sample_tokens_penalized(logits, st, pen, 0, advance=False)
        ops.sample_tokens_constrained(logits, st, out, 0, advance=False)
        torch.cuda.synchronize()
        cpu = _cpu_copy(st)
        want = torch.zeros(B, 1, dtype=torch.long)
        OCB.sample_constrained_twin(logits.cpu(), cpu, want, 0, advance=False)
        for b in range(B):
            rows += 1
            if int(cpu.rule_flags[b]) & 7 == 0:
                assert int(out[b]) == int(pen[b]), b            # an unconstrained row: the penalized token, bit for bit
            if int(out[b]) == int(want[b]):
                checked += 1
                continue
            # a differing token must be a near tie of the oracle (top-p / min-p boundary within its tolerance)
            xr = OCB.constrained_x(logits[b].float().cpu().numpy(), int(cpu.rule_flags[b]) & 7, cpu.bias[b].numpy(),
                                   cpu.ban[b].numpy(), float(cpu.repetition_penalty[b]), 0.0, 0.0,
                                   cpu.prompt_mask[b].numpy(), cpu.counts[b].numpy())
            d = OP.sample_row_penalized(xr, float(cpu.temperature[b]), int(cpu.top_k[b]), float(cpu.top_p[b]),
                                        int(cpu.seed[b]) % 2 ** 64, int(cpu.index[b]), 1.0, 0.0, 0.0, float(cpu.min_p[b]))
            assert d.near_top_p, (b, int(out[b]), int(want[b]))
            near += 1
    assert near <= max(1, rows // 50), (near, rows)


def test_all_banned_row_and_argmax_rules(libpkv):
    from pyramidkv_b200 import ops
    dev = _dev(libpkv)
    V = 64
    prompt = torch.arange(V)                                   # n = 1 bans every token of the history: all of them
    reqs = [G.SamplingParams(0.0, no_repeat_ngram_size=1), G.SamplingParams(0.9, seed=3, no_repeat_ngram_size=1),
            G.SamplingParams(0.0, bad_words_ids=[(5,)])]
    st = G.SamplingState(reqs, dev, vocab=V, prompts=[prompt, prompt, prompt[:3]], eos=None)
    ops.token_rules(st, V)
    logits = torch.randn(3, V).to(torch.bfloat16)
    logits[2, 5] = float("inf")                                 # +inf under a bad word: NaN, the largest for the argmax
    logits = logits.to(dev)
    out = torch.zeros(3, 1, dtype=torch.long, device=dev)
    ops.sample_tokens_constrained(logits, st, out, 0, advance=False)
    assert out[:, 0].tolist() == [0, 0, 5]


def test_graph_replay_equals_eager(libpkv):
    from pyramidkv_b200 import ops
    dev = _dev(libpkv)
    V, B, steps = 32000, 8, 12
    g = np.random.default_rng(5)
    reqs, prompts, gens = _requests(g, B, V, 50, g.integers(50, 400, B), [1])
    logits = [torch.randn(B, V, generator=torch.Generator().manual_seed(s)).to(torch.bfloat16).to(dev) for s in range(steps)]
    buf = torch.empty_like(logits[0])

    def run(graph):
        st = _state(reqs, prompts, gens, V, dev, [1])
        ops.token_rules(st, V)
        out = torch.zeros(B, steps, dtype=torch.long, device=dev)
        col = torch.zeros(B, 1, dtype=torch.long, device=dev)
        stops = []

        def step():
            ops.sample_tokens_constrained(buf, st, col, 0)
            ops.token_rules(st, V, col, 0)
        if graph:
            snap = [t.clone() for t in (st.index, st.counts, *st.rule_state())]
            s = torch.cuda.Stream()
            s.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(s):
                step()
            torch.cuda.current_stream().wait_stream(s)
            for t, v in zip((st.index, st.counts, *st.rule_state()), snap):
                t.copy_(v)
            gr = torch.cuda.CUDAGraph()
            with torch.cuda.graph(gr):
                step()
        for i in range(steps):
            buf.copy_(logits[i])
            gr.replay() if graph else step()
            out[:, i] = col[:, 0]
            stops.append(st.stop[:, 0].clone())
        return out.cpu(), torch.stack(stops).cpu(), st.history.cpu()
    a, b = run(False), run(True)
    assert all(torch.equal(x, y) for x, y in zip(a, b))


# (arch, method, FP8, GQA-shared, decode window, heavy hitters)
FORMS = [("tiny-llama", "pyramidkv", False, False, None, False), ("tiny-llama", "pyramidkv", True, False, None, False),
         ("tiny-llama", "pyramidkv", False, True, None, False), ("tiny-llama", "pyramidkv", False, False, 3, False),
         ("tiny-llama", "pyramidkv", False, False, 4, True), ("tiny-llama", "adakv", False, False, None, False)]


@pytest.mark.parametrize("arch,method,fp8,gqa,window,heavy", FORMS)
def test_loops_every_cache_form(request, arch, method, fp8, gqa, window, heavy):
    """Every rule together in the three loops, graph and eager, against HF's generate on the same cache form; and the
    continuous loop equals the batch loop."""
    import test_constraints as TC
    model, dev = TC._model(request, "cuda", arch, method, fp8, gqa, window)
    if heavy:
        model.config.pkv_decode_heavy = 2
    prompts = TC._prompts(model, dev, (90, 37, 150))
    for rule in ("all", "stop"):
        plain, sps, eos, want = TC._case(model, prompts, rule, 1.0)
        if heavy:                                  # HF's generate has no heavy-hitter window: the eager batch loop is the reference
            want = [t.tolist() for t in G.greedy_generate_batch(model, prompts, TC.CAP, eos_token_id=eos, use_graph=False,
                                                                sampling=sps)]
        for use_graph in (False, True):
            got = G.greedy_generate(model, prompts[0].reshape(1, -1), TC.CAP, use_graph=use_graph, eos_token_id=eos,
                                    sampling=sps[0], check_every=3)
            assert got[0].tolist() == want[0], (rule, use_graph)
            batch = G.greedy_generate_batch(model, prompts, TC.CAP, eos_token_id=eos, use_graph=use_graph, sampling=sps)
            assert [t.tolist() for t in batch] == want, (rule, use_graph)
            cont = G.greedy_generate_continuous(model, prompts, TC.CAP, 2, eos_token_id=eos, use_graph=use_graph,
                                                check_every=3, sampling=sps)
            assert [t.tolist() for t in cont] == [t.tolist() for t in batch], (rule, use_graph)
