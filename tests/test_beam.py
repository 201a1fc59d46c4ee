"""Beam search in the static loop (`generate.beam_search_generate`, DESIGN.md §4.12) on the CPU, through the test-only
backend (tests/oracle_beam_backend.py; `-m gpu`: through libpkv on a tiny random-init model, graph on and off).

HF's reference is `generate(num_beams=k, do_sample=False)` on the same patched model. transformers 5.5 reorders a cache
layer with `reorder_cache`, which on a compacted layer re-slices its `keys` view but leaves the buffers the decode kernel
reads in beam order of the prefill; the reference therefore runs with a test-local `reorder_cache` that gathers the
buffers (`batch_select_indices`), which is what beam search over this cache means."""
import numpy as np
import pytest
import torch

import oracle_beam_backend
from oracle_beam_backend import OracleBeamBackend
from pyramidkv_b200 import generate as G
from pyramidkv_b200 import runner
from pyramidkv_b200.cache import PkvCacheLayer

DEVICES = ["cpu", pytest.param("cuda", marks=pytest.mark.gpu)]
# (method, FP8, GQA-shared, decode window R, heavy hitters H)
FORMS = [("pyramidkv", False, False, None, None), ("pyramidkv", True, False, None, None), ("pyramidkv", False, True, None, None),
         ("pyramidkv", True, True, None, None), ("adakv", False, False, None, None), ("headkv", False, False, None, None),
         ("pyramidkv", False, False, 3, None), ("pyramidkv", False, False, 4, 2)]


@pytest.fixture(autouse=True)
def _restore():
    yield
    from pyramidkv.monkeypatch import restore
    restore()


@pytest.fixture
def hf_reorder(monkeypatch):
    monkeypatch.setattr(PkvCacheLayer, "reorder_cache", lambda self, idx: self.batch_select_indices(idx), raising=False)


def _model(request, device, arch="tiny-llama", method="pyramidkv", fp8=False, gqa=False, window=None, heavy=None,
           capacity=48):
    runner.patch(method)
    if device == "cpu":
        dev = torch.device("cpu")
        model = runner.build_model(arch, dev, torch.bfloat16, "eager")
        runner.set_knobs(model, method, capacity, backend_factory=OracleBeamBackend)
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
    model.config.pkv_decode_heavy = heavy
    return model, dev


def _prompt(model, dev, n, seed):
    return runner.synthetic_prompt(model.config.vocab_size, n, seed, dev)


def _eos_ids(model, prompt, n):
    """n tokens the first step ranks 2nd, 3rd, ...: EOS candidates that really occur."""
    if n == 0:
        return None
    with torch.no_grad():
        logits, _ = G._prefill_logits(model, prompt.reshape(1, -1))
    ids = torch.sort(logits[0].float(), descending=True, stable=True).indices[1:1 + n].tolist()
    return ids[0] if n == 1 else ids


def _hf(model, prompt, T, k, n, lp, es, eos):
    out = model.generate(prompt.reshape(1, -1), num_beams=k, do_sample=False, max_new_tokens=T, num_return_sequences=n,
                         length_penalty=lp, early_stopping=es, eos_token_id=eos, pad_token_id=0,
                         output_scores=True, output_logits=True, return_dict_in_generate=True)
    return (out.sequences.cpu(), out.sequences_scores.cpu(), [x.float().cpu() for x in out.scores],
            [x.float().cpu() for x in out.logits])


def _fill(model, eos):
    """HF's fill of the sequences shorter than the longest returned (pad_token_id 0 is falsy there): the first EOS id, or
    -1 without one."""
    e = eos if eos is not None else model.generation_config.eos_token_id
    if e is None:
        return -1
    return int(e[0] if isinstance(e, (list, tuple)) else e)


def _check_hf(res, hf, plen, fill, tol=0.0):
    """Every hypothesis equals HF's at its rank: its tokens, then only HF's fill; its score bit for bit (tol = 0), or
    within tol."""
    seqs, scores = hf[0], hf[1]
    assert len(res) == seqs.shape[0]
    for (s, sc), row, ref in zip(res, seqs, scores):
        s = s.cpu()
        assert sc.dtype == torch.float32
        assert torch.equal(s, row[: s.shape[0]]), (s[plen:].tolist(), row[plen:].tolist())
        assert (row[s.shape[0]:] == fill).all(), (s[plen:].tolist(), row[plen:].tolist())
        if tol == 0.0:
            assert sc.view(torch.int32) == ref.view(torch.int32), (sc, ref)
        else:
            assert abs(float(sc) - float(ref)) <= tol, (float(sc), float(ref), tol)


# GPU: the kernel's log-probabilities and torch's CUDA log_softmax each lie within 1e-5 + 2^-24 |lp| of the exact ones
# (DESIGN.md §4.8), and each fp32 addition of a running score rounds once, so after t + 1 tokens two runs' scores of the
# same beam differ by at most E_t = (t + 1) * (2e-5 + 2^-22 |score|) (times the length-penalty scale in the pool). Where
# one of HF's cuts (candidates K / K+1, running beams k / k+1, pool k / k+1) separates two values by no more than 2 E_t,
# the runs may keep different beams from there on: such runs are counted, and compared up to that iteration.
NEAR_CUTS = []
DECODE_INPUT_RUNS = []


def _err(t, x, scale=1.0):
    return (t + 1) * (2e-5 + 2.0 ** -22 * abs(float(x))) * max(1.0, abs(float(scale)))


def _near(t, a, b, scale=1.0, same_row=False):
    a, b = float(a), float(b)
    if a <= -5e8 and b <= -5e8:           # both carry HF's -1e9 sentinel: what is left of a score is absorbed alike
        return False
    if same_row and a == b:               # equal logits of one row: equal in both runs, cut by index in both
        return False
    return abs(a - b) <= 2 * _err(t, max(abs(a), abs(b)), scale)


def _first_near_cut(hf_scores, k, T, eos, lp, es, hf_logits):
    """Replays HF's iterations from its own log-probabilities (`output_scores`) with oracle/beam.py, ties by index, and
    returns (the first iteration with a cut whose margin is within the error bound, or None; the replayed state)."""
    from oracle import beam as OB
    from oracle_beam_backend import state_view
    st = G.BeamState(1, k, T, [] if eos is None else ([eos] if isinstance(eos, int) else eos), lp, es, "cpu")
    S, K = state_view(st), st.K
    for t, rows in enumerate(hf_scores):
        srt, idx = torch.sort(rows, dim=-1, descending=True, stable=True)
        lp_k, ids = srt[:, : K + 1].numpy(), idx[:, : K + 1].to(torch.int32).numpy()
        ent = sorted(((np.float32(S.running[r] + lp_k[r, j]), r, int(ids[r, j])) for r in range(k) for j in range(K + 1)),
                     key=lambda e: (-float(e[0]), e[1], e[2]))
        x = hf_logits[t]

        def same(e1, e2):                  # one row's equal logits: equal in both runs, cut by index in both
            return e1[1] == e2[1] and float(x[e1[1], e1[2]]) == float(x[e2[1], e2[2]])
        if _near(t, ent[K - 1][0], ent[K][0], same_row=same(ent[K - 1], ent[K])):
            return t, st
        cand = ent[:K]
        hit = [t + 1 >= T or c[2] in S.eos for c in cand]
        run = sorted(((float(np.float32(c[0] + (OB.NEG if h else OB.NEG0))), c) for c, h in zip(cand, hit)),
                     key=lambda e: -e[0])
        if _near(t, run[k - 1][0], run[k][0], same_row=same(run[k - 1][1], run[k][1])):
            return t, st
        pool_before = [float(x) for x in S.pool_score]
        xs = [float(OB.scale(c[0], st.divisors[t][0], "cuda")) for c in cand]
        merged = sorted(pool_before + [x if (h and c < k) else -1e9 for c, (x, h) in enumerate(zip(xs, hit))], reverse=True)
        if S.heuristic[0] and _near(t, merged[k - 1], merged[k], 1.0 / st.divisors[t][0]):
            return t, st
        heur = bool(S.heuristic[0])
        OB.step(S, lp_k[:, :K], ids[:, :K], k, t, "cuda")
        # the early-stop heuristic compares the best running score with the worst finished one
        best = float(OB.scale(S.running[0], st.divisors[t][1], "cuda"))
        if heur and t + 1 < T and S.pool_done[:k].any() and _near(t, best, float(S.pool_score[:k].min()), 1.0 / st.divisors[t][1]):
            return t, st
        if S.done[0]:
            return None, st
    return None, st


# (k, length_penalty, early_stopping, return all, n_eos, max_new_tokens)
SWEEP = [(2, 1.0, False, False, 0, 10), (3, 0.0, True, True, 1, 12), (4, -1.0, "never", False, 2, 12),
         (4, 2.0, "never", True, 1, 14), (8, 1.0, True, True, 2, 9), (16, 2.0, False, False, 1, 6),
         (4, 1.0, False, True, 1, 1), (3, 1.0, "never", True, 0, 1), (2, 0.0, "never", True, 2, 16),
         (8, -1.0, False, True, 0, 7), (16, 0.0, True, True, 2, 5)]


@pytest.mark.parametrize("device", DEVICES)
@pytest.mark.parametrize("arch", ["tiny-llama", "tiny-mistral"])
@pytest.mark.parametrize("case", SWEEP, ids=lambda c: "k{}-lp{}-es{}-all{}-eos{}-T{}".format(*c))
def test_beam_matches_hf(request, hf_reorder, device, arch, case):
    k, lp, es, everything, n_eos, T = case
    model, dev = _model(request, device, arch)
    prompt = _prompt(model, dev, 90, 3 + k)
    eos = _eos_ids(model, prompt, n_eos)
    n = k if everything else 1
    res = G.beam_search_generate(model, prompt, T, k, length_penalty=lp, early_stopping=es, num_return_sequences=n,
                                 eos_token_id=eos)
    hf = _hf(model, prompt, T, k, n, lp, es, eos)
    fill = _fill(model, eos)
    if device == "cpu":                   # the test backend computes HF's own candidates: bit for bit
        _check_hf(res, hf, 90, fill)
        return
    # the GPU: HF's decisions are replayed from its own log-probabilities with the index tie rule (torch.topk leaves the
    # order of exact ties unspecified); up to the first cut with a margin within the error bound the kernels must take
    # the replay's beams; a run with such a cut is counted and compared at the longest length that has none
    scale = float(T) ** -lp if lp < 0 else 1.0
    T2, hf2 = T, hf
    while T2 > 0:
        cut, st = _first_near_cut(hf2[2], k, T2, eos, lp, es, hf2[3])
        if cut is None:
            break
        NEAR_CUTS.append((arch, k, lp, es, n_eos, T2, cut))
        print(f"near cut at iteration {cut} of {T2}: {len(NEAR_CUTS)} run(s) so far")
        T2 = cut
        hf2 = _hf(model, prompt, T2, k, n, lp, es, eos) if T2 else None
    if T2 == 0:
        return                               # a cut at iteration 0: nothing precedes it
    res2 = res if T2 == T else G.beam_search_generate(model, prompt, T2, k, length_penalty=lp, early_stopping=es,
                                                      num_return_sequences=n, eos_token_id=eos)
    replay = [(torch.cat([prompt.reshape(-1).cpu(), torch.tensor(g, dtype=torch.long)]), sc)
              for g, sc in st.hypotheses(n)[0]]
    tol = _err(T2, max(abs(float(x)) for _, x in replay), scale)
    first = [s.cpu().tolist()[90:] for s, _ in res2] == [r.tolist()[90:] for r, _ in replay]
    if not first:
        # HF's loop decodes the patched cache with the host-length batch launch, the static loop with the device-length
        # one: their logits after iteration 0 may differ by more than the log-softmax bound above (the prefill logits are
        # bit-identical). Such runs are counted; the one-token search, whose inputs are the same, must still agree.
        DECODE_INPUT_RUNS.append((arch, k, lp, es, n_eos, T2))
        print(f"decode-input divergence from HF's replay: {len(DECODE_INPUT_RUNS)} run(s) so far")
        hf1 = _hf(model, prompt, 1, k, n, lp, es, eos)
        cut1, st1 = _first_near_cut(hf1[2], k, 1, eos, lp, es, hf1[3])
        if cut1 is None:
            res1 = G.beam_search_generate(model, prompt, 1, k, length_penalty=lp, early_stopping=es,
                                          num_return_sequences=n, eos_token_id=eos)
            assert [s.cpu().tolist()[90:] for s, _ in res1] == [g for g, _ in st1.hypotheses(n)[0]]
            assert [int(x.view(torch.int32)) for _, x in res1] == [int(x.view(torch.int32)) for _, x in st1.hypotheses(n)[0]]
        return
    for (s, sc), (r, rs) in zip(res2, replay):
        assert abs(float(sc) - float(rs)) <= tol, (float(sc), float(rs), tol)
    if [s.tolist() for s, _ in replay] != [row[: len(s)].tolist() for (s, _), row in zip(replay, hf2[0])]:
        print("HF's tie order differs from the index rule in this run")


@pytest.mark.parametrize("device", DEVICES)
def test_prompts_are_independent(request, device):
    model, dev = _model(request, device)
    prompts = [_prompt(model, dev, n, 20 + i) for i, n in enumerate((150, 37, 300, 20))]
    eos = _eos_ids(model, prompts[1], 1)
    for graph in ([False] if device == "cpu" else [False, True]):
        together = G.beam_search_generate(model, prompts, 12, 4, num_return_sequences=4, eos_token_id=eos,
                                          early_stopping=True, use_graph=graph)
        for p, got in zip(prompts, together):
            alone = G.beam_search_generate(model, p, 12, 4, num_return_sequences=4, eos_token_id=eos,
                                           early_stopping=True, use_graph=graph)
            assert [s.tolist() for s, _ in got] == [s.tolist() for s, _ in alone]
            assert [float(x) for _, x in got] == [float(x) for _, x in alone]


@pytest.mark.parametrize("device", DEVICES)
@pytest.mark.parametrize("form", FORMS, ids=lambda f: "-".join(str(x) for x in f))
def test_every_form_matches_gather_loop(request, monkeypatch, device, form):
    """Every cache form against the same search with the reorder replaced by a whole-slot gather (`gather_reorder`:
    torch indexing, every generated row or the whole ring with the heavy-hitter state): hypotheses and scores bit-equal,
    with the graph on and off on the GPU. An EOS id freezes one prompt early."""
    method, fp8, gqa, window, heavy = form
    model, dev = _model(request, device, method=method, fp8=fp8, gqa=gqa, window=window, heavy=heavy)
    prompts = [_prompt(model, dev, n, 40 + i) for i, n in enumerate((120, 60, 90))]
    eos = _eos_ids(model, prompts[1], 1)
    kw = dict(num_return_sequences=4, eos_token_id=eos, early_stopping=True)
    runs = [G.beam_search_generate(model, prompts, 12, 4, use_graph=g, **kw)
            for g in ([False] if device == "cpu" else [False, True])]
    with monkeypatch.context() as m:
        m.setattr(G, "reorder_caches", oracle_beam_backend.gather_reorder)
        ref = G.beam_search_generate(model, prompts, 12, 4, use_graph=False, **kw)
    for got in runs:
        assert [[s.tolist() for s, _ in h] for h in got] == [[s.tolist() for s, _ in h] for h in ref]
        assert [[int(x.view(torch.int32)) for _, x in h] for h in got] == [[int(x.view(torch.int32)) for _, x in h] for h in ref]
    # the beams did move: some hypotheses of a prompt share a prefix and then differ
    assert any(len({tuple(s.tolist()) for s, _ in h}) > 1 for h in ref)


def test_argument_checks():
    class Fake:
        class lm_head:
            weight = torch.zeros(10, 1)
    p = torch.zeros(5, dtype=torch.long)
    bad = [dict(num_beams=1), dict(num_beams=17), dict(num_beams=4, early_stopping="sometimes"),
           dict(num_beams=4, num_return_sequences=5), dict(num_beams=4, num_return_sequences=0),
           dict(num_beams=4, eos_token_id=[1, 2, 3, 4, 5]), dict(num_beams=4, eos_token_id=10),
           dict(num_beams=4, length_penalty=float("nan")), dict(num_beams=4, max_new_tokens=0)]
    for kw in bad:
        kw = dict(kw)
        T = kw.pop("max_new_tokens", 4)
        with pytest.raises(ValueError):
            G.beam_search_generate(Fake, p, T, **kw)


def test_fullkv_raises(request):
    model, dev = _model(request, "cpu", method="fullkv")
    with pytest.raises(RuntimeError):
        G.beam_search_generate(model, _prompt(model, dev, 30, 1), 4, 2)
