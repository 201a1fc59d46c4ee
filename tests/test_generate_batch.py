"""Batched greedy decoding over the joined compacted caches of several prompts (generate.greedy_generate_batch,
cache.join_caches, the batched StaticDecoder). CPU: host logic through the test backend; `-m gpu`: the same checks on a
random-init small Llama / Mistral in bf16 through libpkv (graph and eager)."""
import pytest
import torch

from oracle_batch_backend import OracleBatchBackend
from pyramidkv_b200 import generate as G
from pyramidkv_b200 import runner
from pyramidkv_b200.cache import PkvBatchCacheLayer, PkvCacheLayer, PkvRaggedCacheLayer, join_caches

DEVICES = ["cpu", pytest.param("cuda", marks=pytest.mark.gpu)]


@pytest.fixture(autouse=True)
def _restore():
    yield
    from pyramidkv.monkeypatch import restore
    restore()


def _model(request, device, arch="tiny-llama", method="pyramidkv", capacity=48):
    runner.patch(method)
    if device == "cpu":
        dev = torch.device("cpu")
        model = runner.build_model(arch, dev, torch.bfloat16, "eager")
        runner.set_knobs(model, method, capacity, backend_factory=OracleBatchBackend)
    else:
        request.getfixturevalue("libpkv")
        from gpu_util import dev as gpu
        dev = gpu()
        model = runner.build_model(arch, dev, torch.bfloat16, "sdpa")
        runner.set_knobs(model, method, capacity)
    return model, dev


def _graph_modes(device):
    return [False] if device == "cpu" else [False, True]


def _prompts(model, dev, lengths, seed=11):
    return [runner.synthetic_prompt(model.config.vocab_size, n, seed + i, dev) for i, n in enumerate(lengths)]


@pytest.mark.parametrize("device", DEVICES)
@pytest.mark.parametrize("arch,method,capacity", [("tiny-llama", "pyramidkv", 48), ("tiny-mistral", "snapkv", 40)])
def test_equal_length_batch_matches_hf_generate(oracle, request, device, arch, method, capacity):
    """B = 3 equal-length prompts prefilled as ONE forward: the batched static loop (one decode launch per layer and step)
    gives HF generate's tokens on the same batch, and the same caches; fused RoPE (one launch for the batch) changes no bit."""
    from transformers import DynamicCache
    model, dev = _model(request, device, arch, method, capacity)
    ids = torch.cat(_prompts(model, dev, (150, 150, 150)))
    new = 9
    with torch.no_grad():
        ref = model.generate(ids, attention_mask=torch.ones_like(ids), max_new_tokens=new, min_new_tokens=new, num_beams=1,
                             do_sample=False, pad_token_id=0, return_dict_in_generate=True)
    for fused_rope in (False, True):
        model.config.pkv_fused_rope = fused_rope
        for use_graph in _graph_modes(device):
            for layer in model.model.layers:
                layer.self_attn.kv_seq_len = 0
            cache = DynamicCache(config=model.config)
            with torch.no_grad():
                first = model(input_ids=ids, past_key_values=cache, use_cache=True, logits_to_keep=1).logits[:, -1].argmax(-1, keepdim=True)
            dec = G.StaticDecoder(model, cache, first, new - 1, use_graph=use_graph)
            toks = dec.run(new - 1)
            assert torch.cat([ids, first, toks], dim=1).tolist() == ref.sequences.tolist(), (fused_rope, use_graph)
            dec.finish()
            for mine, theirs in zip(cache.layers, ref.past_key_values.layers):
                assert isinstance(mine, PkvCacheLayer) and mine.k_buf.shape[0] == 3
                assert mine.length == theirs.length and mine.get_seq_length() == theirs.get_seq_length() == 150 + new - 1
                assert torch.equal(mine.keys, theirs.keys) and torch.equal(mine.values, theirs.values)
    model.config.pkv_fused_rope = False


@pytest.mark.parametrize("device", DEVICES)
@pytest.mark.parametrize("method", ["pyramidkv", "adakv"])
def test_join_equals_single_caches(oracle, request, device, method):
    """Prompts of 150, 37 (shorter than the budget: kept whole) and 300 tokens, prefilled alone and joined: every layer's
    joined buffers and row counts (host and device) equal the single-prompt caches."""
    model, dev = _model(request, device, method=method)
    prompts = _prompts(model, dev, (150, 37, 300))
    singles = [G._prefill(model, p)[1] for p in prompts]
    joined = join_caches(singles, reserve=5)
    Hq = model.config.num_attention_heads
    ragged_seen = False
    for i, layer in enumerate(joined.layers):
        assert isinstance(layer, PkvBatchCacheLayer) and layer.k_buf.shape[:2] == (3, Hq)
        assert layer.seq_seen == [150, 37, 300] and layer.seen_tokens == 300
        want = []
        for b, c in enumerate(singles):
            s = c.layers[i]
            ragged_seen |= isinstance(s, PkvRaggedCacheLayer)
            hr = [r + s.appended for r in s.head_rows_host] if isinstance(s, PkvRaggedCacheLayer) else [s.length] * Hq
            want.append(hr)
            assert layer.rows_host[b] == hr
            for h in range(Hq):
                assert torch.equal(layer.k_buf[b, h, :hr[h]], s.k_buf[0, h, :hr[h]])
                assert torch.equal(layer.v_buf[b, h, :hr[h]], s.v_buf[0, h, :hr[h]])
        assert layer.rows.dtype == torch.int32 and layer.rows.cpu().tolist() == [r for row in want for r in row]
        assert layer.length == max(max(r) for r in want) and layer.capacity == layer.length + 5
        assert want[1] == [37] * Hq                                          # the short prompt keeps every row
    assert ragged_seen == (method == "adakv")


def test_join_rejects_stock_caches_and_batch_layer_limits(oracle):
    from transformers import DynamicCache
    model = runner.build_model("tiny-llama", torch.device("cpu"), torch.bfloat16, "eager")
    ids = runner.synthetic_prompt(model.config.vocab_size, 20, 1, torch.device("cpu"))
    stock = DynamicCache(config=model.config)
    with torch.no_grad():
        model(input_ids=ids, past_key_values=stock, use_cache=True)
    with pytest.raises(RuntimeError):
        join_caches([stock])
    k = torch.zeros(2, 4, 8, 64, dtype=torch.bfloat16)
    layer = PkvBatchCacheLayer(k, k.clone(), [[3, 4, 5, 6], [2, 2, 2, 2]], [10, 7])
    assert layer.length == 6 and layer.rows.tolist() == [3, 4, 5, 6, 2, 2, 2, 2]
    layer.settle([2, 0])
    assert layer.rows_host == [[5, 6, 7, 8], [2, 2, 2, 2]] and layer.seq_seen == [12, 7] and layer.length == 8
    for call in (lambda: layer.update(k[:, :1], k[:, :1]), lambda: layer.crop(3), lambda: layer.batch_repeat_interleave(2),
                 lambda: layer.batch_select_indices(torch.tensor([0]))):
        with pytest.raises(NotImplementedError):
            call()


@pytest.mark.parametrize("device", DEVICES)
def test_batch_order_does_not_matter(oracle, request, device):
    """Each prompt gets the same tokens whichever batch row it sits in (any mixing of sequences would show here)."""
    model, dev = _model(request, device)
    prompts = _prompts(model, dev, (150, 37, 300))
    for use_graph in _graph_modes(device):
        a = G.greedy_generate_batch(model, prompts, 7, use_graph=use_graph)
        b = G.greedy_generate_batch(model, [prompts[2], prompts[0], prompts[1]], 7, use_graph=use_graph)
        assert [t.tolist() for t in a] == [t.tolist() for t in (b[1], b[2], b[0])]
        assert all(t.shape[0] == p.shape[1] + 7 and torch.equal(t[: p.shape[1]], p[0]) for t, p in zip(a, prompts))


@pytest.mark.parametrize("device", DEVICES)
def test_batch_against_solo_teacher_forced(oracle, request, device):
    """Every sequence of the batch, fed alone through the single-sequence decode path with the tokens the batch produced,
    gives the batch's step logits within a tolerance (GEMMs of different M may round differently)."""
    model, dev = _model(request, device)
    prompts = _prompts(model, dev, (150, 37, 300))
    new = 8
    firsts, caches = zip(*[G._prefill(model, p) for p in prompts])
    joined = join_caches(list(caches), reserve=new)
    got = []
    hook = model.lm_head.register_forward_hook(lambda m, i, o: got.append(o.float().clone()))
    try:
        dec = G.StaticDecoder(model, joined, torch.cat(firsts), new - 1, use_graph=False)
        toks = dec.run(new - 1).clone()
    finally:
        hook.remove()
    batch_logits = torch.stack(got, dim=1)                                # [B, steps, vocab]
    worst = 0.0
    for b, p in enumerate(prompts):
        first, cache = G._prefill(model, p)
        feed = [int(firsts[b])] + toks[b, :-1].tolist()
        for t, tok in enumerate(feed):
            with torch.no_grad():
                lg = model(input_ids=torch.tensor([[tok]], device=dev), past_key_values=cache, use_cache=True).logits[0, -1].float()
            err = (lg - batch_logits[b, t]).abs().max().item()
            worst = max(worst, err)
            assert err <= 0.05 * max(lg.abs().max().item(), 1.0), (b, t, err)
    print(f"[{device}] batch vs solo teacher-forced: largest |logit difference| {worst:.5f}")


@pytest.mark.parametrize("device", DEVICES)
def test_eos_per_sequence(oracle, request, device):
    """A different EOS per sequence stops each one at its solo-stop index; tokens after it are pad_token_id, and finish()
    leaves per-sequence row counts that end at the EOS - for every check_every."""
    model, dev = _model(request, device)
    lengths = (150, 37, 300)
    prompts = _prompts(model, dev, lengths)
    free = [G.greedy_generate(model, p, 12)[0, n:].tolist() for p, n in zip(prompts, lengths)]
    eos = sorted({free[0][3], free[1][6]})
    solo = [G.greedy_generate(model, p, 12, eos_token_id=eos, return_cache=True) for p in prompts]
    for every in (1, 3, 16):
        seqs, cache = G.greedy_generate_batch(model, prompts, 12, eos_token_id=eos, check_every=every, return_cache=True)
        for b, (s, sc) in enumerate(solo):
            assert seqs[b].tolist() == s[0].tolist(), (every, b)
            for jl, sl in zip(cache.layers, sc.layers):
                assert max(jl.rows_host[b]) == sl.length and jl.seq_seen[b] == sl.get_seq_length()
    # on the device: finished sequences emit the pad token from then on
    firsts, caches = zip(*[G._prefill(model, p) for p in prompts])
    dec = G.StaticDecoder(model, join_caches(list(caches), reserve=11), torch.cat(firsts), 11, use_graph=device != "cpu",
                          eos_token_id=eos, pad_token_id=0)
    toks = dec.run(11).cpu()
    for b, (s, _) in enumerate(solo):
        stop = s.shape[1] - lengths[b] - 1                                 # decode steps up to and including the EOS
        assert toks[b, :stop].tolist() == s[0, lengths[b] + 1:].tolist()
        if stop < 11:
            assert toks[b, stop:].tolist() == [0] * (11 - stop)
    assert dec.done.cpu().tolist() == [[int(s.shape[1]) - n - 1 < 11 or s[0, -1].item() in eos] for (s, _), n in zip(solo, lengths)]
    dec.finish()


@pytest.mark.parametrize("device", DEVICES)
def test_batch_of_one_equals_greedy_generate(oracle, request, device):
    model, dev = _model(request, device)
    ids = _prompts(model, dev, (150,))[0]
    for use_graph in _graph_modes(device):
        assert G.greedy_generate_batch(model, [ids], 8, use_graph=use_graph)[0].tolist() == \
            G.greedy_generate(model, ids, 8, use_graph=use_graph)[0].tolist()
