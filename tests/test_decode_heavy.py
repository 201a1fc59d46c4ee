"""Heavy hitters in the decode window (knob `pkv_decode_heavy` = H with `pkv_decode_window` = R): once the window is full, the
new row replaces the generated row with the least accumulated attention among all but the R - H - 1 most recent. Through
the test-only backend on the CPU (`-m gpu`: through libpkv on a tiny random-init model, graph on and off), over every cache
form and the static, batched and continuous loops plus HF `generate()`: R at least the steps taken gives the tokens and
caches of the knob off, and (CPU) H = 0 gives the ring's. A planted heavy hitter stays under the rule and leaves the ring."""
import ctypes as C

import pytest
import torch

from oracle_heavy_backend import OracleHeavyBackend, decode_heavy_twin
from oracle_window_backend import decode_window_twin
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


class _RingBackend(OracleHeavyBackend):
    heavy_override = 0


def _model(request, device, method="pyramidkv", fp8=False, gqa=False, window=None, heavy=None, factory=OracleHeavyBackend):
    runner.patch(method)
    if device == "cpu":
        dev = torch.device("cpu")
        model = runner.build_model("tiny-llama", dev, torch.bfloat16, "eager")
        runner.set_knobs(model, method, 48, backend_factory=factory)
    else:
        request.getfixturevalue("libpkv")
        from gpu_util import dev as gpu
        dev = gpu()
        model = runner.build_model("tiny-llama", dev, torch.bfloat16, "sdpa")
        runner.set_knobs(model, method, 48)
    if fp8:
        model.config.pkv_kv_cache_dtype = "fp8_e4m3"
    if gqa:
        model.config.pkv_gqa_shared = True
    model.config.pkv_decode_window = window
    model.config.pkv_decode_heavy = heavy
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
    r = layer.rows_host[b][h]
    return [_bytes(getattr(layer, n)[b, h, :r]).cpu() for n in layer._BUFFERS]


def _run_loops(model, prompts, N, use_graph):
    one, c1 = G.greedy_generate(model, prompts[0], N, use_graph=use_graph, return_cache=True)
    batch, cb = G.greedy_generate_batch(model, prompts[:3], N, use_graph=use_graph, return_cache=True)
    cont, st = G.greedy_generate_continuous(model, prompts, CAPS, 3, use_graph=use_graph, check_every=4, return_stats=True)
    # a static run stopped by an EOS: the first token sequence 1 emits after its first decode step
    eos = int(batch[1][LENGTHS[1] + 2])
    stopped, cs = G.greedy_generate_batch(model, prompts[:3], N, eos_token_id=eos, use_graph=use_graph, return_cache=True)
    hf = _hf(model, prompts[1], 6)
    return dict(one=one.tolist(), batch=_lists(batch), cont=_lists(cont), stopped=_lists(stopped), hf=hf.tolist()), \
        [(c1, 1), (cb, 3), (cs, 3)], st


def _same_caches(got, want, check_layer=None):
    for (gc, B), (wc, _) in zip(got, want):
        for lg, lw in zip(gc.layers, wc.layers):
            if check_layer is not None:
                check_layer(lg)
            assert lg.seq_seen == lw.seq_seen and lg.rows_host == [lw.rows_host[b] for b in range(B)]
            for b in range(B):
                for h in range(len(lg.rows_host[b])):
                    for x, y in zip(_valid_rows(lg, b, h), _valid_rows(lw, b, h)):
                        assert torch.equal(x, y), (b, h)


# ---- the knob ----
def test_knob_values():
    class Cfg:
        pass
    c = Cfg()
    assert PC.decode_heavy(c) is None
    c.pkv_decode_heavy = 2
    with pytest.raises(ValueError):          # no window
        PC.decode_heavy(c)
    c.pkv_decode_window = 8
    for ok in (1, 4, 7):
        c.pkv_decode_heavy = ok
        assert PC.decode_heavy(c) == ok
    for bad in (0, 8, 9, -1, 1.5, "2", True):
        c.pkv_decode_heavy = bad
        with pytest.raises(ValueError):
            PC.decode_heavy(c)
    c.pkv_decode_window, c.pkv_decode_heavy = 1, 1  # R = 1 leaves no H
    with pytest.raises(ValueError):
        PC.decode_heavy(c)


def test_heavy_struct_layout_matches_header(libpkv, tmp_path):
    """sizeof / offsetof of pkv_decode_heavy against its ctypes mirror."""
    import os
    import subprocess
    from pyramidkv_b200 import _lib
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    src = tmp_path / "h.c"
    src.write_text('#include <stddef.h>\n#include <stdio.h>\n#include "pkv.h"\nint main(void){printf("%zu %zu %zu %zu %zu %zu\\n", '
                   'sizeof(pkv_decode_heavy), offsetof(pkv_decode_heavy, heavy), offsetof(pkv_decode_heavy, scores), '
                   'offsetof(pkv_decode_heavy, victim), offsetof(pkv_decode_heavy, scratch), '
                   'offsetof(pkv_decode_heavy, scratch_bytes));return 0;}\n')
    exe = tmp_path / "h"
    subprocess.run(["gcc", "-I", os.path.join(root, "include"), "-I", "/usr/local/cuda/include", str(src), "-o", str(exe)],
                   check=True)
    Hv = _lib.DecodeHeavy
    got = [int(x) for x in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]
    assert got == [C.sizeof(Hv), Hv.heavy.offset, Hv.scores.offset, Hv.victim.offset, Hv.scratch.offset, Hv.scratch_bytes.offset]


def test_bad_values_raise_in_prefill_and_refusals(request):
    for window, heavy in ((None, 2), (4, 4), (4, 0)):
        model, dev = _model(request, "cpu", window=window, heavy=heavy)
        with pytest.raises(ValueError):
            G.greedy_generate(model, _prompts(model, dev, (60,))[0], 3)
    with pytest.raises(NotImplementedError):
        runner.run_suite("tiny-llama", "fullkv", -1, [("t", 16, 2)], device=torch.device("cpu"), decode_window=8, decode_heavy=2)
    with pytest.raises(ValueError):
        runner.run_suite("tiny-llama", "pyramidkv", 48, [("t", 16, 2)], device=torch.device("cpu"),
                         backend_factory=OracleHeavyBackend, decode_heavy=2)
    model, dev = _model(request, "cpu", window=4, heavy=2)
    _, cache = G.greedy_generate(model, _prompts(model, dev, (60,))[0], 3, return_cache=True)
    with pytest.raises(NotImplementedError):
        cache.layers[0].update(torch.zeros(1, 2, 2, 64), torch.zeros(1, 2, 2, 64))


def test_heavy_and_ring_caches_do_not_join(request):
    model, dev = _model(request, "cpu", window=4, heavy=2)
    p = _prompts(model, dev, (60,))[0]
    _, heavy = G.greedy_generate(model, p, 2, return_cache=True)
    model.config.pkv_decode_heavy = None
    _, ring = G.greedy_generate(model, p, 2, return_cache=True)
    with pytest.raises(ValueError):
        PC.join_caches([heavy, ring])


# ---- R >= the steps taken: the knob changes nothing ----
@pytest.mark.parametrize("device", DEVICES)
@pytest.mark.parametrize("method,fp8,gqa", FORMS)
def test_large_window_equals_knob_off(request, device, method, fp8, gqa):
    off, dev = _model(request, device, method, fp8, gqa)
    prompts = _prompts(off, dev, LENGTHS)
    N = max(CAPS)
    for use_graph in _graph_modes(device):
        want, want_caches, _ = _run_loops(off, prompts, N, use_graph)
        for R in (N, 64):
            off.config.pkv_decode_window, off.config.pkv_decode_heavy = R, R // 2
            got, got_caches, st = _run_loops(off, prompts, N, use_graph)
            off.config.pkv_decode_window = off.config.pkv_decode_heavy = None
            assert got == want and st["regrowths"] == 0, (R, use_graph)

            def check(layer, R=R):
                assert layer.window == R and layer.heavy == R // 2
            _same_caches(got_caches, want_caches, check)


# ---- H = 0 (the twin only: the knob refuses it) is the ring ----
@pytest.mark.parametrize("method,fp8,gqa", FORMS)
def test_heavy_zero_is_the_ring(request, method, fp8, gqa):
    R, N = 3, 11
    ring, dev = _model(request, "cpu", method, fp8, gqa, window=R)
    prompts = _prompts(ring, dev, LENGTHS)
    want, want_caches, _ = _run_loops(ring, prompts, N, False)
    zero, _ = _model(request, "cpu", method, fp8, gqa, window=R, heavy=1, factory=_RingBackend)
    got, got_caches, st = _run_loops(zero, prompts, N, False)
    assert got == want and st["regrowths"] == 0
    _same_caches(got_caches, want_caches)


# ---- a small window that wraps inside the loops ----
# the first three prompts keep every row (shorter than the budget); the fourth, admitted into a slot while the others have
# wrapped, has more rows than the batch holds, so the batch regrows and the decode graph is captured again mid-generation
WRAP_LENGTHS = (20, 37, 30, 150, 90)
WRAP_CAPS = [9, 14, 12, 8, 5]


@pytest.mark.parametrize("device", DEVICES)
@pytest.mark.parametrize("method,fp8,gqa", FORMS)
def test_small_heavy_window_loops(request, device, method, fp8, gqa):
    """R = 3, H = 1: the static loop (graph on and off) gives HF generate()'s tokens and the same held rows, and continuous
    batching with admissions, a regrowth and a recapture gives the tokens of lock-step batches of the same prompts."""
    R, H, N = 3, 1, 11
    model, dev = _model(request, device, method, fp8, gqa, window=R, heavy=H)
    prompts = _prompts(model, dev, WRAP_LENGTHS)
    n = len(prompts)
    want = [G.greedy_generate_batch(model, [prompts[r], prompts[(r + 1) % n], prompts[(r + 2) % n]], WRAP_CAPS[r],
                                    use_graph=False)[0].tolist() for r in range(n)]
    ref_cache = None
    for use_graph in _graph_modes(device):
        seq, cache = G.greedy_generate(model, prompts[0], N, use_graph=use_graph, return_cache=True)
        assert _hf(model, prompts[0], N).tolist() == seq.tolist(), use_graph
        l0 = cache.layers[0]
        assert l0.generated == [N - 1] and l0.rows_host[0] == [p + R for p in l0.prompt_rows_host[0]]
        held = sorted(int(g) for g in l0.heavy_gen[0, 0])
        assert held[-(R - H):] == list(range(N - 1 - (R - H), N - 1)), held    # the R - H most recent rows stay
        if ref_cache is None:
            ref_cache = cache
        else:                                                                   # graph on: the rows and state of graph off
            _same_caches([(cache, 1)], [(ref_cache, 1)])
            for lg, lw in zip(cache.layers, ref_cache.layers):
                assert torch.equal(lg.heavy_gen, lw.heavy_gen) and torch.equal(lg.heavy_scores, lw.heavy_scores)
        got, st = G.greedy_generate_continuous(model, prompts, WRAP_CAPS, 3, use_graph=use_graph, check_every=4,
                                               return_stats=True)
        assert _lists(got) == want, use_graph
        assert st["admissions"] == 2 and st["regrowths"] >= 1, st
        if use_graph:
            assert st["graph_captures"] == 1 + st["regrowths"], st


def test_admission_resets_the_slot_state(request):
    """Admitting a prompt into a slot of a heavy batch zeroes that slot's scores, sets its generation indices and victim to
    -1, and leaves the other slots' state as it was."""
    model, dev = _model(request, "cpu", window=3, heavy=1)
    prompts = _prompts(model, dev, (60, 37, 30))
    _, batch = G.greedy_generate_batch(model, prompts[:2], 8, return_cache=True)
    before = [(l.heavy_scores.clone(), l.heavy_gen.clone(), l.victim.clone()) for l in batch.layers]
    assert all(bool((g >= 0).all()) and bool((s > 0).any()) for s, g, _ in before)
    _, single = G._prefill(model, prompts[2])
    PC.admit_cache(batch, 1, single, torch.zeros(1, dtype=torch.int32), G._backend(model))
    for l, (s, g, v) in zip(batch.layers, before):
        H = l.heavy_gen.shape[1]
        assert bool((l.heavy_scores[1] == 0).all()) and bool((l.heavy_gen[1] == -1).all()) and bool((l.victim[H:] == -1).all())
        assert torch.equal(l.heavy_scores[0], s[0]) and torch.equal(l.heavy_gen[0], g[0]) and torch.equal(l.victim[:H], v[:H])
        assert l.generated == [7, 0]
    model.config.pkv_decode_heavy = None
    _, ring = G._prefill(model, prompts[2])
    with pytest.raises(ValueError, match="heavy hitters"):
        PC.admit_cache(batch, 1, ring, torch.zeros(1, dtype=torch.int32), G._backend(model))


# ---- a planted heavy hitter ----
def _planted(R, steps, D=64, P=8, seed=0):
    """q / k_new / v_new of `steps` steps over P random prompt rows: generated row 5's key is a large multiple of a direction u
    every later query leans on; every other key is small noise."""
    g = torch.Generator().manual_seed(seed)
    u = torch.randn(D, generator=g)
    u = u / u.norm()
    cap = P + steps + 1
    k = torch.zeros(1, 1, cap, D, dtype=torch.bfloat16)
    v = torch.zeros_like(k)
    k[0, 0, :P] = (torch.randn(P, D, generator=g) * 0.3).bfloat16()
    v[0, 0, :P] = torch.randn(P, D, generator=g).bfloat16()
    q = (torch.randn(steps, 1, 1, D, generator=g) * 0.3 + 2.5 * u).bfloat16()
    kn = (torch.randn(steps, 1, 1, D, generator=g) * 0.3).bfloat16()
    kn[5, 0, 0] = (20.0 * u).bfloat16()   # about 80 % of every later query's attention over the unwindowed cache
    vn = torch.randn(steps, 1, 1, D, generator=g).bfloat16()
    return q, k, v, kn, vn, P, cap


def test_planted_heavy_hitter_stays_and_leaves_the_ring():
    R, H = 16, 8
    steps = R + 100
    q, k0, v0, kn, vn, P, cap = _planted(R, steps)
    prompt_rows = torch.tensor([P], dtype=torch.int32)
    kh, vh, kr, vr, kf, vf = k0.clone(), v0.clone(), k0.clone(), v0.clone(), k0.clone(), v0.clone()
    scores = torch.zeros(1, 1, R, dtype=torch.float64)
    gen = torch.full((1, 1, R), -1, dtype=torch.int32)
    victim = torch.full((1,), -1, dtype=torch.int32)
    for t in range(steps):
        rows = torch.tensor([P + t], dtype=torch.int32)
        out_h = decode_heavy_twin(q[t], kh, vh, None, 1, kn[t], vn[t], prompt_rows, R, H, scores, gen, victim, rows)
        out_r = decode_window_twin(q[t], kr, vr, None, 1, kn[t], vn[t], prompt_rows, R, rows)
        kf[0, 0, P + t], vf[0, 0, P + t] = kn[t, 0, 0], vn[t, 0, 0]       # the unwindowed cache
    held = sorted(int(x) for x in gen.reshape(-1))
    assert 5 in held and len(set(held)) == R
    assert held[-(R - H):] == list(range(steps - (R - H), steps))         # the R - H most recent rows stay
    ring_held = [int(j) for j in range(steps - R, steps)]
    assert 5 not in ring_held and not any(torch.equal(kr[0, 0, P + i], kn[5, 0, 0]) for i in range(R))
    assert any(torch.equal(kh[0, 0, P + i], kn[5, 0, 0]) for i in range(R))
    # the last step's output against the unwindowed cache's (fp64 attention over every row)
    T = P + steps
    K, V = kf[0, 0, :T].double(), vf[0, 0, :T].double()
    full = torch.softmax(K @ q[-1, 0, 0].double() * 64 ** -0.5, dim=0) @ V
    err_h = float((out_h[0, 0].double() - full).norm())
    err_r = float((out_r[0, 0].double() - full).norm())
    assert err_h < err_r, (err_h, err_r)


def test_runner_records_carry_heavy(request):
    recs = runner.run_suite("tiny-llama", "pyramidkv", 48, [("t", 90, 6)], device=torch.device("cpu"),
                            backend_factory=OracleHeavyBackend, decode_loop="static-eager", decode_window=3, decode_heavy=1)
    assert recs[0]["decode_window"] == 3 and recs[0]["decode_heavy"] == 1 and len(recs[0]["pred_ids"]) == 6
