"""Continuous batching (generate.greedy_generate_continuous, generate.ContinuousDecoder, PkvBatchCacheLayer.admit / park /
grow): slots of a batched cache take new prompts in place while the step keeps replaying. CPU: host logic through the
test-only backend (with the torch twin of pkv_cache_install); `-m gpu`: the same checks through libpkv, graph on and off."""
import pytest
import torch

from oracle_continuous_backend import OracleContinuousBackend
from pyramidkv_b200 import generate as G
from pyramidkv_b200 import runner
from pyramidkv_b200.cache import PkvBatchCacheLayer, PkvFp8CacheLayer, admit_cache, join_caches, park_cache

DEVICES = ["cpu", pytest.param("cuda", marks=pytest.mark.gpu)]
# (method, kv cache dtype FP8, GQA-shared)
FORMS = [("pyramidkv", False, False), ("snapkv", False, False), ("streamingllm", False, False), ("adakv", False, False),
         ("headkv", False, False), ("pyramidkv", True, False), ("adakv", True, False), ("pyramidkv", False, True),
         ("pyramidkv", True, True)]
LENGTHS = (150, 37, 300, 20, 90, 61, 200)      # 37, 20: shorter than the budget (kept whole)
CAPS = [5, 9, 3, 12, 7, 4, 6]


@pytest.fixture(autouse=True)
def _restore():
    yield
    from pyramidkv.monkeypatch import restore
    restore()


def _model(request, device, arch="tiny-llama", method="pyramidkv", capacity=48, fp8=False, gqa=False):
    runner.patch(method)
    if device == "cpu":
        dev = torch.device("cpu")
        model = runner.build_model(arch, dev, torch.bfloat16, "eager")
        runner.set_knobs(model, method, capacity, backend_factory=OracleContinuousBackend)
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
    return model, dev


def _graph_modes(device):
    return [False] if device == "cpu" else [False, True]


def _prompts(model, dev, lengths, seed=11):
    return [runner.synthetic_prompt(model.config.vocab_size, n, seed + i, dev) for i, n in enumerate(lengths)]


def _lockstep(model, prompts, caps, eos, use_graph):
    """Request r's tokens from greedy_generate_batch in a batch of three sequences (r and the two prompts after it)."""
    n = len(prompts)
    return [G.greedy_generate_batch(model, [prompts[r], prompts[(r + 1) % n], prompts[(r + 2) % n]], caps[r], eos_token_id=eos,
                                    use_graph=use_graph)[0].tolist() for r in range(n)]


@pytest.mark.parametrize("device", DEVICES)
@pytest.mark.parametrize("arch,method,capacity", [("tiny-llama", "pyramidkv", 48), ("tiny-mistral", "snapkv", 40)])
def test_enough_slots_equals_greedy_generate_batch(oracle, request, device, arch, method, capacity):
    model, dev = _model(request, device, arch, method, capacity)
    prompts = _prompts(model, dev, (150, 37, 300))
    for use_graph in _graph_modes(device):
        ref = G.greedy_generate_batch(model, prompts, 9, use_graph=use_graph)
        for slots in (3, 5):
            got, st = G.greedy_generate_continuous(model, prompts, 9, slots, use_graph=use_graph, check_every=4, return_stats=True)
            assert [t.tolist() for t in got] == [t.tolist() for t in ref], (use_graph, slots)
            assert st["admissions"] == 0 and st["decode_steps"] == 8 and st["live_slot_steps"] == 3 * 8
            assert st["graph_captures"] == int(use_graph)


@pytest.mark.parametrize("device", DEVICES)
@pytest.mark.parametrize("method,fp8,gqa", FORMS)
def test_seven_prompts_three_slots_equal_lockstep(oracle, request, device, method, fp8, gqa):
    """Mixed lengths and max_new_tokens, forced EOS ids: every request gets the tokens it gets in a lock-step batch of three
    (the GEMMs have the same row count and each row's attention does not depend on the other sequences)."""
    model, dev = _model(request, device, method=method, fp8=fp8, gqa=gqa)
    prompts = _prompts(model, dev, LENGTHS)
    free = G.greedy_generate_continuous(model, prompts, CAPS, 3, use_graph=False)
    eos = sorted({free[1][LENGTHS[1] + 3].item(), free[4][LENGTHS[4] + 2].item()})
    for use_graph in _graph_modes(device):
        want = _lockstep(model, prompts, CAPS, eos, use_graph)
        for every in (1, 4, 16):
            got, st = G.greedy_generate_continuous(model, prompts, CAPS, 3, eos_token_id=eos, use_graph=use_graph,
                                                   check_every=every, return_stats=True)
            assert [t.tolist() for t in got] == want, (use_graph, every)
            assert any(len(g) < n + c for g, n, c in zip(want, LENGTHS, CAPS))          # some request stopped at an EOS
            admitted = sum(len(g) > n + 1 for g, n in zip(want[3:], LENGTHS[3:]))      # a first token that is an EOS needs no slot
            assert st["admissions"] == admitted and st["live_slot_steps"] == sum(len(g) - n - 1 for g, n in zip(want, LENGTHS))
            assert st["decode_steps"] < sum(CAPS)
            assert st["graph_captures"] == (1 + st["regrowths"] if use_graph else 0)


def _single_rows(layer):
    return [r + layer.appended for r in layer.head_rows_host] if hasattr(layer, "head_rows_host") else (
        list(layer.rows_host[0]) if isinstance(layer, PkvBatchCacheLayer) else [layer.length] * layer.k_buf.shape[1])


def _raw(t):
    """The bits (buffers past the rows hold uninitialised values, NaNs among them)."""
    return t.view({torch.float8_e4m3fn: torch.uint8, torch.float32: torch.int32}.get(t.dtype, torch.int16))


@pytest.mark.parametrize("device", DEVICES)
@pytest.mark.parametrize("method,fp8,gqa", [f for f in FORMS if f[0] in ("pyramidkv", "adakv")])
def test_admitted_slot_equals_join_and_others_untouched(oracle, request, device, method, fp8, gqa):
    model, dev = _model(request, device, method=method, fp8=fp8, gqa=gqa)
    prompts = _prompts(model, dev, (150, 37, 300, 90))
    caches = [G._prefill(model, p)[1] for p in prompts]
    backend = model.model.layers[0].self_attn.kv_cluster.backend
    batch = join_caches(caches[:3], reserve=40)
    ref = join_caches([caches[3]])
    before = [[_raw(getattr(l, n)).clone() for n in l._BUFFERS] for l in batch.layers]
    step = torch.tensor([5], dtype=torch.int32, device=dev)
    admit_cache(batch, 1, caches[3], step, backend)
    for i, (l, r) in enumerate(zip(batch.layers, ref.layers)):
        assert type(l) is type(r) and l.rows_host[1] == r.rows_host[0] == _single_rows(caches[3].layers[i])
        assert l.seq_seen == [150, 90, 300]
        H = l.k_buf.shape[1]
        assert l.rows.cpu().tolist()[H:2 * H] == [n - 5 for n in r.rows_host[0]]
        for name, old in zip(l._BUFFERS, before[i]):
            new, want = _raw(getattr(l, name)), _raw(getattr(r, name))
            assert torch.equal(new[0], old[0]) and torch.equal(new[2], old[2])          # the other slots: every byte
            for h in range(H):
                n = r.rows_host[0][h]
                assert torch.equal(new[1, h, :n], want[0, h, :n])
                assert torch.equal(new[1, h, n:], old[1, h, n:])                         # past the rows: untouched
    park_cache(batch, 2, step, backend)
    for l in batch.layers:
        H = l.k_buf.shape[1]
        assert l.rows.cpu().tolist()[2 * H:] == [-5] * H and l.rows_host[2] == [0] * H and l.seq_seen[2] == 0


@pytest.mark.parametrize("device", DEVICES)
def test_parked_slots_stay_within_capacity(oracle, request, device):
    model, dev = _model(request, device)
    prompts = _prompts(model, dev, (150, 37, 20))
    firsts, caches = zip(*[G._prefill(model, p) for p in prompts])
    for use_graph in _graph_modes(device):
        batch = join_caches(list(caches), reserve=20)
        cap = [l.capacity for l in batch.layers]
        dec = G.ContinuousDecoder(model, batch, torch.cat(firsts), [0, 40, 0], chunk=4, use_graph=use_graph)
        dec.park(0)
        dec.park(2)
        H = batch.layers[0].k_buf.shape[1]
        for _ in range(4):
            toks = dec.run_chunk(4)
            assert toks[0].tolist() == toks[2].tolist() == [0] * 4 and 0 not in toks[1].tolist()[:1]
            step = int(dec.state.step)
            for l, c in zip(batch.layers, cap):
                rows = l.rows.cpu().reshape(3, H) + 1 + step
                assert (rows[0] == 1).all() and (rows[2] == 1).all() and (rows <= c).all()
        dec.finish()


@pytest.mark.parametrize("device", DEVICES)
@pytest.mark.parametrize("fp8", [False, True])
def test_regrowth_keeps_tokens(oracle, request, device, fp8):
    """Short first prompts (small buffers), then a long prompt with a long max_new_tokens: the batch grows, the graph is
    captured again (one capture per buffer set) and every request's tokens stay those of the lock-step batch."""
    model, dev = _model(request, device, fp8=fp8)
    lengths, caps = (20, 25, 30, 300, 40), [3, 3, 3, 14, 4]
    prompts = _prompts(model, dev, lengths)
    for use_graph in _graph_modes(device):
        want = _lockstep(model, prompts, caps, None, use_graph)
        got, st = G.greedy_generate_continuous(model, prompts, caps, 3, use_graph=use_graph, check_every=2, return_stats=True)
        assert [t.tolist() for t in got] == want
        assert st["regrowths"] >= 1 and st["admissions"] == 2
        assert st["graph_captures"] == (1 + st["regrowths"] if use_graph else 0)


def test_argument_errors(oracle, request):
    model, dev = _model(request, "cpu")
    prompts = _prompts(model, dev, (150, 37))
    caches = [G._prefill(model, p)[1] for p in prompts]
    backend = model.model.layers[0].self_attn.kv_cluster.backend
    batch = join_caches(caches)
    step = torch.zeros(1, dtype=torch.int32)
    with pytest.raises(ValueError, match="slot"):
        admit_cache(batch, 2, caches[0], step, backend)
    with pytest.raises(ValueError, match="slot"):
        park_cache(batch, -1, step, backend)
    small = join_caches([caches[1], caches[1]])
    with pytest.raises(ValueError, match="capacity"):
        admit_cache(small, 0, caches[0], step, backend)                       # 150 tokens keep more rows than 37
    model.config.pkv_kv_cache_dtype = "fp8_e4m3"
    fp8 = G._prefill(model, prompts[0])[1]
    assert isinstance(fp8.layers[0], PkvFp8CacheLayer)
    with pytest.raises(ValueError, match="do not mix"):
        admit_cache(batch, 0, fp8, step, backend)
    with pytest.raises(ValueError, match="do not mix"):
        admit_cache(join_caches([fp8]), 0, caches[0], step, backend)
    model.config.pkv_kv_cache_dtype = None
    model.config.pkv_gqa_shared = True
    gqa = G._prefill(model, prompts[0])[1]
    with pytest.raises(ValueError, match="do not mix"):
        admit_cache(batch, 0, gqa, step, backend)
    model.config.pkv_gqa_shared = False
    with pytest.raises(ValueError, match="layers"):
        admit_cache(batch, 0, type(caches[0])(), step, backend)
    with pytest.raises(ValueError, match="max_new_tokens"):
        G.greedy_generate_continuous(model, prompts, [3], 2)
    with pytest.raises(ValueError, match="num_slots"):
        G.greedy_generate_continuous(model, prompts, 3, 0)
    with pytest.raises(ValueError, match="no prompts"):
        G.greedy_generate_continuous(model, [], 3, 2)


def test_runner_continuous_records(oracle):
    """run_longbench.py --decode_loop continuous: one record per prompt with its own tokens (those of the batch-1 static
    loop), prefill time and cache rows, and the continuous block; mixed max_new_tokens go through one call."""
    import run_longbench
    base = ["--method", "PyramidKV", "--model_path", "tiny-llama", "--max_capacity_prompts", "48", "--attn_implementation", "eager",
            "--dataset", "lcc", "--prompt_tokens", "150", "--max_new_tokens", "5", "--max_num_examples", "3", "--dtype", "bfloat16"]
    one = run_longbench.main(base + ["--decode_loop", "static-eager"], backend_factory=OracleContinuousBackend, device=torch.device("cpu"))
    cont = run_longbench.main(base + ["--decode_loop", "continuous", "--eval_batch_size", "2"], backend_factory=OracleContinuousBackend,
                              device=torch.device("cpu"))
    assert [r["pred_ids"] for r in cont] == [r["pred_ids"] for r in one]
    assert [r["cache_rows_first_last"] for r in cont] == [r["cache_rows_first_last"] for r in one]
    for r in cont:
        c = r["continuous"]
        assert r["decode_loop"] == "continuous" and r["prefill_ms"] > 0 and "decode_tok_per_s" not in r
        assert c["slots"] == 2 and c["decode_steps"] == 8 and c["occupancy"] == pytest.approx(12 / 16) and c["aggregate_tok_per_s"] > 0
    recs = runner.run_suite("tiny-llama", "pyramidkv", 48, [("a", 150, 5), ("b", 37, 3), ("c", 90, 7)], device=torch.device("cpu"),
                            dtype=torch.bfloat16, attn_implementation="eager", backend_factory=OracleContinuousBackend,
                            decode_loop="continuous", eval_batch_size=2)
    assert [len(r["pred_ids"]) for r in recs] == [5, 3, 7]
    with pytest.raises(NotImplementedError, match="static"):
        runner.run_suite("tiny-llama", "fullkv", 48, [("a", 150, 5)], device=torch.device("cpu"), dtype=torch.bfloat16,
                         attn_implementation="eager", decode_loop="continuous", eval_batch_size=2)
    with pytest.raises(NotImplementedError, match="ratio"):
        runner.run_suite("tiny-llama", "pyramidkv", -1, [("a", 150, 5), ("b", 90, 5)], device=torch.device("cpu"),
                         dtype=torch.bfloat16, attn_implementation="eager", backend_factory=OracleContinuousBackend,
                         decode_loop="continuous", eval_batch_size=2, capacity_ratio=0.5)
