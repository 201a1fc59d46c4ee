"""The decode window (knob `pkv_decode_window` = R): each sequence's cache holds its compacted prompt plus its last R generated
rows, the j-th appended row at physical row P + j mod R. Through the test-only backend on the CPU (`-m gpu`: through libpkv
on a tiny random-init model, graph on and off), over every cache form and the static, batched and continuous loops plus HF
`generate()`: R at least the steps taken gives the tokens and caches of the knob off; a small R keeps the ring rows a
restatement of the semantics names, equal across the loops, without regrowth in continuous batching."""
import ctypes as C

import pytest
import torch

from oracle_window_backend import OracleWindowBackend
from pyramidkv_b200 import cache as PC
from pyramidkv_b200 import generate as G
from pyramidkv_b200 import runner

DEVICES = ["cpu", pytest.param("cuda", marks=pytest.mark.gpu)]
# (method, kv cache dtype FP8, GQA-shared)
FORMS = [("pyramidkv", False, False), ("pyramidkv", True, False), ("pyramidkv", False, True), ("pyramidkv", True, True),
         ("adakv", False, False), ("headkv", False, False)]
LENGTHS = (150, 37, 300, 20, 90)
CAPS = [9, 4, 12, 7, 5]


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
        runner.set_knobs(model, method, capacity, backend_factory=OracleWindowBackend)
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


def _hf(model, ids, new):
    with torch.no_grad():
        return model.generate(ids, attention_mask=torch.ones_like(ids), max_new_tokens=new, min_new_tokens=new, num_beams=1,
                              do_sample=False, pad_token_id=0)


def _bytes(t):
    return t.view(torch.uint8) if t.dtype == torch.float8_e4m3fn else t


def _valid_rows(layer, b, h):
    """(K, V[, k_scale, v_scale]) of the rows sequence b, head h holds."""
    r = layer.rows_host[b][h]
    return [_bytes(getattr(layer, n)[b, h, :r]).cpu() for n in layer._BUFFERS]


# ---- the knob ----
def test_knob_values():
    class Cfg:
        pass
    c = Cfg()
    assert PC.decode_window(c) is None
    for ok in (1, 7, 4096):
        c.pkv_decode_window = ok
        assert PC.decode_window(c) == ok
    for bad in (0, -3, 1.5, "8", True):
        c.pkv_decode_window = bad
        with pytest.raises(ValueError):
            PC.decode_window(c)


def test_window_struct_layout_matches_header(libpkv, tmp_path):
    """sizeof / offsetof of pkv_decode_window against its ctypes mirror."""
    import os
    import subprocess
    from pyramidkv_b200 import _lib
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    src = tmp_path / "w.c"
    src.write_text('#include <stddef.h>\n#include <stdio.h>\n#include "pkv.h"\nint main(void){printf("%zu %zu %zu %zu\\n", '
                   'sizeof(pkv_decode_window), offsetof(pkv_decode_window, prompt_rows), offsetof(pkv_decode_window, k_scale), '
                   'offsetof(pkv_decode_window, window));return 0;}\n')
    exe = tmp_path / "w"
    subprocess.run(["gcc", "-I", os.path.join(root, "include"), "-I", "/usr/local/cuda/include", str(src), "-o", str(exe)],
                   check=True)
    W = _lib.DecodeWindow
    got = [int(x) for x in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]
    assert got == [C.sizeof(W), W.prompt_rows.offset, W.k_scale.offset, W.window.offset]


def test_bad_values_raise_in_prefill_and_refusals(request):
    model, dev = _model(request, "cpu", window=0)
    with pytest.raises(ValueError):
        G.greedy_generate(model, _prompts(model, dev, (60,))[0], 3)
    with pytest.raises(NotImplementedError):
        runner.run_suite("tiny-llama", "fullkv", -1, [("t", 16, 2)], device=torch.device("cpu"), decode_window=8)


# ---- R >= the steps taken: the knob changes nothing ----
@pytest.mark.parametrize("device", DEVICES)
@pytest.mark.parametrize("method,fp8,gqa", FORMS)
def test_large_window_equals_knob_off(request, device, method, fp8, gqa):
    off, dev = _model(request, device, method, fp8, gqa)
    prompts = _prompts(off, dev, LENGTHS)
    N = max(CAPS)
    for use_graph in _graph_modes(device):
        want_one, want_cache = G.greedy_generate(off, prompts[0], N, use_graph=use_graph, return_cache=True)
        want_batch, want_joined = G.greedy_generate_batch(off, prompts[:3], N, use_graph=use_graph, return_cache=True)
        want_cont = G.greedy_generate_continuous(off, prompts, CAPS, 3, use_graph=use_graph)
        want_hf = _hf(off, prompts[1], 6)
        for R in (N, 64):
            off.config.pkv_decode_window = R
            got_one, got_cache = G.greedy_generate(off, prompts[0], N, use_graph=use_graph, return_cache=True)
            got_batch, got_joined = G.greedy_generate_batch(off, prompts[:3], N, use_graph=use_graph, return_cache=True)
            got_cont, st = G.greedy_generate_continuous(off, prompts, CAPS, 3, use_graph=use_graph, return_stats=True)
            got_hf = _hf(off, prompts[1], 6)
            off.config.pkv_decode_window = None
            assert got_one.tolist() == want_one.tolist() and _lists(got_batch) == _lists(want_batch), (R, use_graph)
            assert _lists(got_cont) == _lists(want_cont) and got_hf.tolist() == want_hf.tolist(), (R, use_graph)
            assert st["regrowths"] == 0
            for got_c, want_c, B in ((got_cache, want_cache, 1), (got_joined, want_joined, 3)):
                for lg, lw in zip(got_c.layers, want_c.layers):
                    assert lg.window == R and lg.seq_seen == lw.seq_seen
                    assert lg.rows_host == [lw.rows_host[b] for b in range(B)]
                    for b in range(B):
                        for h in range(len(lg.rows_host[b])):
                            for x, y in zip(_valid_rows(lg, b, h), _valid_rows(lw, b, h)):
                                assert torch.equal(x, y), (R, b, h)


# ---- a small R: the ring the semantics name ----
def _teacher_layer0(model, ids, steps):
    """Layer 0's cache rows for `ids` (prompt + generated) with the knob off, the generated tokens fed one at a time: its K/V
    rows depend on the tokens and positions only, so they are what any decode of these tokens appends."""
    S = ids.shape[1] - steps - 1
    R = model.config.pkv_decode_window
    model.config.pkv_decode_window = None
    try:
        _, cache = G._prefill(model, ids[:, :S])
        with torch.no_grad():
            for t in range(S, S + steps):
                model(input_ids=ids[:, t:t + 1], past_key_values=cache, use_cache=True)
    finally:
        model.config.pkv_decode_window = R
    return cache.layers[0]


@pytest.mark.parametrize("device", DEVICES)
@pytest.mark.parametrize("method,fp8,gqa", FORMS)
def test_small_window_ring_and_loops(request, device, method, fp8, gqa):
    R, N = 3, 11
    model, dev = _model(request, device, method, fp8, gqa, window=R)
    prompts = _prompts(model, dev, LENGTHS)
    for use_graph in _graph_modes(device):
        seq, win = G.greedy_generate(model, prompts[0], N, use_graph=use_graph, return_cache=True)
        assert _hf(model, prompts[0], N).tolist() == seq.tolist()
        steps = N - 1
        ref = _teacher_layer0(model, seq, steps)
        l0 = win.layers[0]
        P = l0.prompt_rows_host[0]
        assert l0.generated == [steps] and l0.rows_host[0] == [p + R for p in P] and l0.seq_seen == [seq.shape[1] - 1]
        for h, p in enumerate(P):
            want = [t for t in _ref_rows(ref, h)]
            got = _valid_rows(l0, 0, h)
            for x, y in zip(got, want):
                assert torch.equal(x[:p], y[:p])                                   # the prompt rows stay
                for i in range(R):                                                 # ring slot i: the latest j = i mod R
                    j = max(j for j in range(steps) if j % R == i)
                    assert torch.equal(x[p + i], y[p + j]), (h, i, j)
        # lock-step batches and continuous batching of the same N agree, with no regrowth and one capture
        n = len(prompts)
        want = [G.greedy_generate_batch(model, [prompts[r], prompts[(r + 1) % n], prompts[(r + 2) % n]], CAPS[r],
                                        use_graph=use_graph)[0].tolist() for r in range(n)]
        got, st = G.greedy_generate_continuous(model, prompts, CAPS, 3, use_graph=use_graph, check_every=4, return_stats=True)
        assert _lists(got) == want
        assert st["regrowths"] == 0 and st["graph_captures"] == int(use_graph)


def _ref_rows(layer, h):
    """Rows of head h of a knob-off layer in token order, in the format of `_valid_rows`."""
    if isinstance(layer, PC.PkvBatchCacheLayer):
        return _valid_rows(layer, 0, h)
    r = layer.head_rows_host[h] + layer.appended if isinstance(layer, PC.PkvRaggedCacheLayer) else layer.length
    return [_bytes(getattr(layer, n)[0, h, :r]).cpu() for n in layer._BUFFERS]


@pytest.mark.parametrize("device", DEVICES)
@pytest.mark.parametrize("method,fp8,gqa", [FORMS[0], FORMS[1], FORMS[3]])
def test_returned_batch_cache_with_eos(request, device, method, fp8, gqa):
    """greedy_generate_batch(..., return_cache=True): sequence b holds P + min(kept_b, R) rows, and a sequence that stopped
    at its EOS holds the ring of a run that took exactly its kept steps: the steps after its EOS wrote nothing."""
    R, N = 4, 12
    model, dev = _model(request, device, method, fp8, gqa, window=R)
    prompts = _prompts(model, dev, LENGTHS[:3])
    for use_graph in _graph_modes(device):
        free = G.greedy_generate_batch(model, prompts, N, use_graph=use_graph)
        firsts = {f[LENGTHS[b]].item() for b, f in enumerate(free)}
        dec1 = free[1][LENGTHS[1] + 1:].tolist()
        # sequence 1's EOS: of the tokens that start no sequence, the one it first emits last (before its final step)
        eos = max(((i, t) for i, t in enumerate(dec1[:-1]) if t not in firsts and t not in dec1[:i]), default=(0, None))[1]
        assert eos is not None
        hit_at = dec1.index(eos)
        got, cache = G.greedy_generate_batch(model, prompts, N, eos_token_id=eos, use_graph=use_graph, return_cache=True)
        kept = []
        for b, (g, f) in enumerate(zip(got, free)):
            gen = g[LENGTHS[b] + 1:].tolist()        # the decode steps' tokens
            assert gen == f[LENGTHS[b] + 1:LENGTHS[b] + 1 + len(gen)].tolist()
            hit = next((i for i, t in enumerate(gen) if t == eos), None)
            kept.append(N - 1 if hit is None else hit + 1)
            for l in cache.layers:
                assert l.generated[b] == kept[b] and l.rows_host[b] == [p + min(kept[b], R) for p in l.prompt_rows_host[b]]
        assert kept[1] == hit_at + 1
        _, short = G.greedy_generate_batch(model, prompts, kept[1] + 1, use_graph=use_graph, return_cache=True)
        for l, ls in zip(cache.layers, short.layers):
            for h in range(len(l.rows_host[1])):
                for x, y in zip(_valid_rows(l, 1, h), _valid_rows(ls, 1, h)):
                    assert torch.equal(x, y), h


def test_multi_token_update_raises(request):
    model, dev = _model(request, "cpu", window=4)
    _, cache = G.greedy_generate(model, _prompts(model, dev, (60,))[0], 3, return_cache=True)
    with pytest.raises(NotImplementedError):
        cache.layers[0].update(torch.zeros(1, 2, 2, 64), torch.zeros(1, 2, 2, 64))


def test_runner_records_carry_the_window(request):
    recs = runner.run_suite("tiny-llama", "pyramidkv", 48, [("t", 90, 6)], device=torch.device("cpu"),
                            backend_factory=OracleWindowBackend, decode_loop="static-eager", decode_window=3)
    assert recs[0]["decode_window"] == 3 and len(recs[0]["pred_ids"]) == 6
