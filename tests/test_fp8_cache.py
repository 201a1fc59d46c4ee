"""The opt-in FP8 (E4M3) compacted cache (model.config.pkv_kv_cache_dtype = "fp8_e4m3"): the quantisation rule, the
conversion after the prefill, PkvFp8CacheLayer, join_caches, the static and HF decode loops, and the runners' knob.
CPU: host logic through the FP8 test backend (torch twin of the two kernels); `-m gpu`: the same model-level checks on a
random-init small Llama / Mistral in bf16 through libpkv (graph and eager)."""
import pytest
import torch

from oracle_batch_backend import OracleBatchBackend
from oracle_fp8_backend import OracleFp8Backend, dequantize, quantize_rows
from pyramidkv_b200 import generate as G
from pyramidkv_b200 import runner
from pyramidkv_b200.cache import (PkvBatchCacheLayer, PkvCacheLayer, PkvFp8CacheLayer, PkvRaggedCacheLayer, join_caches,
                                  quantize_caches_fp8)

DEVICES = ["cpu", pytest.param("cuda", marks=pytest.mark.gpu)]


@pytest.fixture(autouse=True)
def _restore():
    yield
    from pyramidkv.monkeypatch import restore
    restore()


def _bytes(q):
    return q.view(torch.uint8)


# ---------------- the quantisation rule ----------------
def _within_bound(x, q, scale):
    """|x^ - x| <= 2^-4 |x| where the byte is a normal E4M3 value, <= 2^-10 * scale where it is subnormal (half the spacing
    of each range; the fp32 roundings of inv and scale add ~2^-23 relative, far inside the slack of the tie cases)."""
    xd, qd = x.double(), q.float().double()
    xh = qd * scale.double()[..., None]
    err = (xh - xd).abs()
    normal = qd.abs() >= 2.0 ** -6
    ok_n = err <= 2.0 ** -4 * xd.abs() * (1 + 2.0 ** -10)
    ok_s = err <= 2.0 ** -10 * scale.double()[..., None] * (1 + 2.0 ** -10)
    return bool(torch.where(normal, ok_n, ok_s).all())


def test_zero_row():
    q, s = quantize_rows(torch.zeros(3, 64, dtype=torch.bfloat16))
    assert bool((_bytes(q) == 0).all()) and bool((s == 0).all())
    x = torch.zeros(2, 64, dtype=torch.float16)
    x[0] = -0.0
    q, s = quantize_rows(x)
    assert bool((_bytes(q) == 0).all()) and s.tolist() == [0.0, 0.0]


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_random_rows_within_bound(dtype):
    g = torch.Generator().manual_seed(0)
    x = (torch.randn(512, 128, generator=g) * torch.logspace(-3, 2, 512)[:, None]).to(dtype)
    q, s = quantize_rows(x)
    assert _within_bound(x, q, s)
    # the largest element of every row lands on +-448
    top = x.float().abs().argmax(dim=-1)
    assert bool((q.float().gather(1, top[:, None]).abs() == 448).all())
    assert torch.allclose(s, x.float().abs().amax(dim=-1) / 448, rtol=2 ** -23, atol=0)


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_tiny_amax_goes_subnormal(dtype):
    """One element sets the scale; the others scale into E4M3's subnormal range (below 2^-6) or to zero."""
    x = torch.full((1, 64), 2e-5, dtype=dtype)     # * 448 / 2 = 0.00448: subnormal
    x[0, 5] = 2.0
    x[0, 9] = -8e-6                                  # -0.0018: rounds to -2^-9
    q, s = quantize_rows(x)
    qf = q.float()
    assert qf[0, 5] == 448 and bool((qf[0, [0, 1, 9]].abs() < 2 ** -6).all()) and bool((qf[0, [0, 1]] > 0).all())
    assert _within_bound(x, q, s)
    # a row whose own amax is tiny still uses the full range
    y = torch.full((1, 64), 3e-5, dtype=dtype)
    qy, sy = quantize_rows(y)
    assert bool((qy.float() == 448).all()) and sy.item() > 0 and _within_bound(y, qy, sy)


def test_top_of_range_satfinite_agrees_with_torch():
    """x * inv can exceed 448 by one fp32 ulp. torch's float8_e4m3fn conversion rounds to nearest even up to 464 (the
    midpoint between 448 and the NaN encoding) and gives 448 there; cvt.rn.satfinite gives 448 for any value above 448. The
    two agree on every value the rule produces. Find amax values where the overshoot happens and check the byte."""
    g = torch.Generator().manual_seed(1)
    a = torch.rand(20000, generator=g).bfloat16().float() * 100 + 1e-3
    inv = torch.full_like(a, 448.0) / a
    over = a[(a * inv) > 448]
    assert over.numel() > 0, "no overshooting amax found"
    y = over * (torch.full_like(over, 448.0) / over)
    assert bool((y > 448).all()) and bool((y < 448 * (1 + 2 ** -22)).all())
    assert bool((_bytes(y.to(torch.float8_e4m3fn)) == 0x7E).all())
    for b in over[:16].tolist():
        row = torch.tensor([[b, -b, b / 2]], dtype=torch.float32).bfloat16()
        q, _ = quantize_rows(row)
        assert _bytes(q)[0].tolist()[:2] == [0x7E, 0xFE]
    edge = torch.tensor([448.0, torch.nextafter(torch.tensor(448.0), torch.tensor(1e9)).item(), 460.0, 464.0])
    assert _bytes(edge.to(torch.float8_e4m3fn)).tolist() == [0x7E] * 4


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_round_half_even(dtype):
    """amax = 448 makes inv exactly 1: the elements are the scaled values themselves, chosen on rounding ties."""
    vals = [448.0, 1.0625, 1.1875, -1.0625, 2.0 ** -10, 3 * 2.0 ** -10, 5 * 2.0 ** -10, 2.0 ** -9]
    want = [0x7E, 0x38, 0x3A, 0xB8, 0x00, 0x02, 0x02, 0x01]     # 1.0, 1.25, -1.0; 0, 2^-8, 2^-8 (even), 2^-9
    x = torch.tensor([vals + [0.0] * (64 - len(vals))], dtype=dtype)
    q, s = quantize_rows(x)
    assert s.item() == 1.0 and _bytes(q)[0, :len(vals)].tolist() == want


# ---------------- plugin, static loop, HF loop ----------------
def _model(request, device, arch="tiny-llama", method="pyramidkv", capacity=48, fp8=True, backend=OracleFp8Backend):
    runner.patch(method)
    if device == "cpu":
        dev = torch.device("cpu")
        model = runner.build_model(arch, dev, torch.bfloat16, "eager")
        runner.set_knobs(model, method, capacity, backend_factory=backend)
    else:
        request.getfixturevalue("libpkv")
        from gpu_util import dev as gpu
        dev = gpu()
        model = runner.build_model(arch, dev, torch.bfloat16, "sdpa")
        runner.set_knobs(model, method, capacity)
    model.config.pkv_kv_cache_dtype = "fp8_e4m3" if fp8 else None
    return model, dev


def _prompts(model, dev, lengths, seed=11):
    return [runner.synthetic_prompt(model.config.vocab_size, n, seed + i, dev) for i, n in enumerate(lengths)]


def _graph_modes(device):
    return [False] if device == "cpu" else [False, True]


def test_knob_off_keeps_the_16bit_caches(oracle):
    """Knob unset: the FP8 backend's model builds exactly the caches of the batched backend (same classes, same bytes)."""
    a, dev = _model(None, "cpu", fp8=False)
    b, _ = _model(None, "cpu", fp8=False, backend=OracleBatchBackend)
    del a.config.pkv_kv_cache_dtype
    ids = _prompts(a, dev, (150,))[0]
    for method in ("pyramidkv", "adakv"):
        for m in (a, b):
            runner.patch(method)
            runner.set_knobs(m, method, 48, backend_factory=OracleFp8Backend if m is a else OracleBatchBackend)
        ca, cb = G._prefill(a, ids)[1], G._prefill(b, ids)[1]
        for la, lb in zip(ca.layers, cb.layers):
            assert type(la) is type(lb) and type(la) in (PkvCacheLayer, PkvRaggedCacheLayer)
            assert la.k_buf.dtype == torch.bfloat16 and la.length == lb.length
            assert torch.equal(la.keys, lb.keys) and torch.equal(la.values, lb.values)


@pytest.mark.parametrize("device", DEVICES)
@pytest.mark.parametrize("method", ["pyramidkv", "snapkv", "h2o", "streamingllm", "adakv", "headkv"])
def test_knob_on_converts_every_layer(oracle, request, device, method):
    """Knob on: every layer is a PkvFp8CacheLayer with the 16-bit cache's row counts, and its dequantised rows are within the
    E4M3 bound of the 16-bit rows."""
    cap = 48 if method != "streamingllm" else 40
    model, dev = _model(request, device, method=method, capacity=cap)
    ids = _prompts(model, dev, (150,))[0]
    c8 = G._prefill(model, ids)[1]
    model.config.pkv_kv_cache_dtype = None
    c16 = G._prefill(model, ids)[1]
    Hq = model.config.num_attention_heads
    for l8, l16 in zip(c8.layers, c16.layers):
        assert isinstance(l8, PkvFp8CacheLayer) and l8.k_buf.dtype == torch.float8_e4m3fn
        rows = [r + l16.appended for r in l16.head_rows_host] if isinstance(l16, PkvRaggedCacheLayer) else [l16.length] * Hq
        assert l8.rows_host == [rows] and l8.rows.cpu().tolist() == rows and l8.seq_seen == [150]
        assert l8.capacity == l16.capacity and l8.get_seq_length() == 150
        for h in range(Hq):
            k16, v16 = (l16.head_view(h) if isinstance(l16, PkvRaggedCacheLayer) else (l16.k_buf[0, h, :rows[h]], l16.v_buf[0, h, :rows[h]]))
            for t16, q8, s8 in ((k16, l8.k_buf[0, h, :rows[h]], l8.k_scale[0, h, :rows[h]]),
                                (v16, l8.v_buf[0, h, :rows[h]], l8.v_scale[0, h, :rows[h]])):
                assert _within_bound(t16.cpu(), q8.cpu(), s8.cpu())
                wq, ws = quantize_rows(t16)
                assert torch.equal(_bytes(q8.cpu()), _bytes(wq)) and torch.equal(s8.cpu(), ws)
            kd, _ = l8.head_view(0, h)
            assert torch.equal(kd.cpu(), dequantize(l8.k_buf[0, h, :rows[h]], l8.k_scale[0, h, :rows[h]]))


@pytest.mark.parametrize("device", DEVICES)
@pytest.mark.parametrize("arch,method", [("tiny-llama", "pyramidkv"), ("tiny-mistral", "snapkv"), ("tiny-llama", "adakv")])
def test_static_loop_graph_eager_and_hf_generate(oracle, request, device, arch, method):
    """HF model.generate over the FP8 cache gives the static loop's tokens; graph replay gives the eager loop's tokens; the
    cache ends with one more row per head and step."""
    model, dev = _model(request, device, arch, method, 40)
    ids = _prompts(model, dev, (150,))[0]
    new = 8
    with torch.no_grad():
        ref = model.generate(ids, attention_mask=torch.ones_like(ids), max_new_tokens=new, min_new_tokens=new, num_beams=1,
                             do_sample=False, pad_token_id=0, return_dict_in_generate=True)
    assert all(isinstance(l, PkvFp8CacheLayer) for l in ref.past_key_values.layers)
    for use_graph in _graph_modes(device):
        seq, cache = G.greedy_generate(model, ids, new, use_graph=use_graph, return_cache=True)
        assert seq.tolist() == ref.sequences.tolist(), use_graph
        for mine, theirs in zip(cache.layers, ref.past_key_values.layers):
            assert isinstance(mine, PkvFp8CacheLayer) and mine.rows_host == theirs.rows_host
            assert mine.get_seq_length() == theirs.get_seq_length() == 150 + new - 1
            for h in range(mine.k_buf.shape[1]):
                a, b = mine.head_view(0, h), theirs.head_view(0, h)
                assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])


@pytest.mark.parametrize("device", DEVICES)
@pytest.mark.parametrize("arch", ["tiny-llama", "tiny-mistral"])
def test_batch_of_one_and_batch_order(oracle, request, device, arch):
    model, dev = _model(request, device, arch)
    prompts = _prompts(model, dev, (150, 37, 300))
    for use_graph in _graph_modes(device):
        assert G.greedy_generate_batch(model, [prompts[0]], 7, use_graph=use_graph)[0].tolist() == \
            G.greedy_generate(model, prompts[0], 7, use_graph=use_graph)[0].tolist()
        a = G.greedy_generate_batch(model, prompts, 7, use_graph=use_graph)
        b = G.greedy_generate_batch(model, [prompts[2], prompts[0], prompts[1]], 7, use_graph=use_graph)
        assert [t.tolist() for t in a] == [t.tolist() for t in (b[1], b[2], b[0])]
        assert all(t.shape[0] == p.shape[1] + 7 and torch.equal(t[: p.shape[1]], p[0]) for t, p in zip(a, prompts))


@pytest.mark.parametrize("device", DEVICES)
def test_eos_per_sequence(oracle, request, device):
    """Each sequence of an FP8 batch stops at its solo EOS; finish() books its own row count."""
    model, dev = _model(request, device)
    lengths = (150, 37, 300)
    prompts = _prompts(model, dev, lengths)
    free = [G.greedy_generate(model, p, 12)[0, n:].tolist() for p, n in zip(prompts, lengths)]
    eos = sorted({free[0][3], free[1][6]})
    solo = [G.greedy_generate(model, p, 12, eos_token_id=eos, return_cache=True) for p in prompts]
    seqs, cache = G.greedy_generate_batch(model, prompts, 12, eos_token_id=eos, check_every=3, return_cache=True)
    for b, (s, sc) in enumerate(solo):
        assert seqs[b].tolist() == s[0].tolist(), b
        for jl, sl in zip(cache.layers, sc.layers):
            assert isinstance(jl, PkvFp8CacheLayer) and jl.rows_host[b] == sl.rows_host[0] and jl.seq_seen[b] == sl.get_seq_length()


@pytest.mark.parametrize("device", DEVICES)
@pytest.mark.parametrize("method", ["pyramidkv", "adakv"])
def test_join_fp8_caches(oracle, request, device, method):
    """FP8 single-prompt caches join into one PkvFp8CacheLayer per layer, bytes and scales copied as they are."""
    model, dev = _model(request, device, method=method)
    prompts = _prompts(model, dev, (150, 37, 300))
    singles = [G._prefill(model, p)[1] for p in prompts]
    joined = join_caches(singles, reserve=5)
    Hq = model.config.num_attention_heads
    for i, layer in enumerate(joined.layers):
        assert isinstance(layer, PkvFp8CacheLayer) and layer.k_buf.shape[:2] == (3, Hq)
        assert layer.seq_seen == [150, 37, 300]
        want = [c.layers[i].rows_host[0] for c in singles]
        assert layer.rows_host == want and layer.rows.cpu().tolist() == [r for row in want for r in row]
        assert layer.capacity == max(max(r) for r in want) + 5
        for b, c in enumerate(singles):
            s = c.layers[i]
            for h in range(Hq):
                n = want[b][h]
                assert torch.equal(_bytes(layer.k_buf[b, h, :n]), _bytes(s.k_buf[0, h, :n]))
                assert torch.equal(_bytes(layer.v_buf[b, h, :n]), _bytes(s.v_buf[0, h, :n]))
                assert torch.equal(layer.k_scale[b, h, :n], s.k_scale[0, h, :n]) and torch.equal(layer.v_scale[b, h, :n], s.v_scale[0, h, :n])
    model.config.pkv_kv_cache_dtype = None
    plain = G._prefill(model, prompts[0])[1]
    with pytest.raises(ValueError, match="FP8"):
        join_caches([singles[0], plain])


def test_refused_operations(oracle):
    k = torch.zeros(2, 4, 8, 64, dtype=torch.float8_e4m3fn)
    s = torch.zeros(2, 4, 8)
    layer = PkvFp8CacheLayer(k, k.clone(), s, s.clone(), [[3, 4, 5, 6], [2, 2, 2, 2]], [10, 7])
    assert layer.length == 6 and layer.rows.tolist() == [3, 4, 5, 6, 2, 2, 2, 2]
    layer.reserve(5)
    assert layer.capacity >= 11 and layer.k_scale.shape[2] == layer.capacity and layer.v_buf.dtype == torch.float8_e4m3fn
    layer.settle([2, 0])
    assert layer.rows_host == [[5, 6, 7, 8], [2, 2, 2, 2]] and layer.seq_seen == [12, 7]
    x = torch.zeros(2, 4, 2, 64, dtype=torch.bfloat16)
    for call in (lambda: layer.update(x, x), lambda: layer.crop(3), lambda: layer.batch_repeat_interleave(2),
                 lambda: layer.batch_select_indices(torch.tensor([0]))):
        with pytest.raises(NotImplementedError):
            call()
    with pytest.raises(NotImplementedError):
        from pyramidkv_b200.pipeline import PipelineRunner
        from types import SimpleNamespace
        PipelineRunner(SimpleNamespace(config=SimpleNamespace(pkv_kv_cache_dtype="fp8_e4m3")))


def test_multi_token_forward_refused(oracle):
    model, dev = _model(None, "cpu")
    ids = _prompts(model, dev, (150,))[0]
    _, cache = G._prefill(model, ids)
    with torch.no_grad(), pytest.raises(NotImplementedError, match="FP8"):
        model(input_ids=ids[:, :3], past_key_values=cache, use_cache=True)


def test_bad_knob_value(oracle):
    model, dev = _model(None, "cpu")
    model.config.pkv_kv_cache_dtype = "int4"
    with pytest.raises(ValueError, match="pkv_kv_cache_dtype"):
        G._prefill(model, _prompts(model, dev, (150,))[0])


@pytest.mark.parametrize("device", DEVICES)
@pytest.mark.parametrize("arch", ["tiny-llama", "tiny-mistral"])
def test_teacher_forced_logits_against_16bit(oracle, request, device, arch):
    """The same tokens fed through the FP8 cache and through the 16-bit cache. E4M3 keeps 3 mantissa bits, so every cached
    element may move by up to 2^-4 of itself: attention scores move by up to ~6 % of |q||k| and the attention output by up
    to ~6 % of the largest |V|. Through o_proj, the residual stream and lm_head that bounds the logit change by a small
    fraction of the logits' own range; 0.15 * max(|logit|) is that bound with margin (the measured value is printed)."""
    model, dev = _model(request, device, arch)
    ids = _prompts(model, dev, (300,))[0]
    seq = G.greedy_generate(model, ids, 10)[0, 300:].tolist()
    worst = 0.0
    top1 = 0
    caches = {}
    for knob in ("fp8_e4m3", None):
        model.config.pkv_kv_cache_dtype = knob
        _, caches[knob] = G._prefill(model, ids)
    for tok in seq[:-1]:
        lg = {}
        for knob, cache in caches.items():
            with torch.no_grad():
                lg[knob] = model(input_ids=torch.tensor([[tok]], device=dev), past_key_values=cache, use_cache=True).logits[0, -1].float()
        err = (lg["fp8_e4m3"] - lg[None]).abs().max().item()
        worst = max(worst, err)
        top1 += int(lg["fp8_e4m3"].argmax() == lg[None].argmax())
        assert err <= 0.15 * max(lg[None].abs().max().item(), 1.0), err
    assert isinstance(caches["fp8_e4m3"].layers[0], PkvFp8CacheLayer) and type(caches[None].layers[0]) is PkvCacheLayer
    print(f"[{device} {arch}] FP8 vs 16-bit teacher-forced: largest |logit difference| {worst:.5f}, top-1 agreement {top1}/{len(seq) - 1}")


def test_quantize_caches_skips_non_compacted_layers(oracle):
    from transformers import DynamicCache
    c = DynamicCache()
    c.layers = []
    assert quantize_caches_fp8(c, OracleFp8Backend()) == 0


def test_runner_records_the_cache_dtype(oracle):
    import run_longbench
    base = ["--method", "PyramidKV", "--model_path", "tiny-llama", "--max_capacity_prompts", "48", "--attn_implementation", "eager",
            "--dataset", "lcc", "--prompt_tokens", "150", "--max_new_tokens", "5", "--max_num_examples", "2", "--dtype", "bfloat16",
            "--decode_loop", "static-eager"]
    plain = run_longbench.main(base, backend_factory=OracleFp8Backend, device=torch.device("cpu"))
    assert all("kv_cache_dtype" not in r for r in plain)
    ref = run_longbench.main(base, backend_factory=OracleBatchBackend, device=torch.device("cpu"))
    drop = ("prefill_ms", "decode_tok_per_s")
    assert [{k: v for k, v in r.items() if k not in drop} for r in plain] == [{k: v for k, v in r.items() if k not in drop} for r in ref]
    for extra in ([], ["--eval_batch_size", "2"]):
        fp8 = run_longbench.main(base + ["--kv_cache_dtype", "fp8_e4m3"] + extra, backend_factory=OracleFp8Backend, device=torch.device("cpu"))
        assert all(r["kv_cache_dtype"] == "fp8_e4m3" and len(r["pred_ids"]) == 5 for r in fp8)
        assert [r["cache_rows_first_last"] for r in fp8] == [r["cache_rows_first_last"] for r in plain]
    import run_needle_in_haystack
    needle = run_needle_in_haystack.main(["--method", "pyramidkv", "--model_name", "tiny-llama", "--s_len", "150", "--e_len", "151",
                                          "--max_capacity_prompt", "48", "--max_new_tokens", "3",
                                          "--decode_loop", "static-eager", "--kv_cache_dtype", "fp8_e4m3", "--dtype", "bfloat16"],
                                         backend_factory=OracleFp8Backend, device=torch.device("cpu"))
    assert needle[0]["kv_cache_dtype"] == "fp8_e4m3"
    with pytest.raises(NotImplementedError, match="FullKV"):
        run_longbench.main(["--method", "FullKV", "--model_path", "tiny-llama", "--dataset", "lcc", "--prompt_tokens", "20",
                            "--max_new_tokens", "2", "--kv_cache_dtype", "fp8_e4m3"], device=torch.device("cpu"))
