"""The GQA-shared cache (knob `model.config.pkv_gqa_shared`): the torch twin of the group reduction, the per-KV-head caches the
patched prefill installs, the static / batched / HF decode loops over them (alone and with the FP8 knob), joins, and the
refusals. On the CPU through the test-only oracle backend; the `cuda` parameters run the same checks on the GPU kernels."""
import pytest
import torch

from oracle_gqa_backend import OracleGqaBackend, group_reduce
from pyramidkv_b200 import generate as G
from pyramidkv_b200 import runner
from pyramidkv_b200.cache import PkvBatchCacheLayer, PkvCacheLayer, PkvFp8CacheLayer, join_caches

DEVICES = ["cpu", pytest.param("cuda", marks=pytest.mark.gpu)]


@pytest.fixture(autouse=True)
def _restore():
    yield
    from pyramidkv.monkeypatch import restore
    restore()


# ---------------- the group reduction ----------------
def _loop_reduce(pooled, G_):
    """The rule written out element by element in numpy fp32 (no torch reduction)."""
    import numpy as np
    x = pooled.float().numpy()
    out = np.empty((x.shape[0] // G_, x.shape[1]), dtype=np.float32)
    for j in range(out.shape[0]):
        for t in range(out.shape[1]):
            s = np.float32(0)
            for g in range(G_):
                s = np.float32(s + x[j * G_ + g, t])
            out[j, t] = np.float32(s / np.float32(G_))
    return torch.from_numpy(out).to(pooled.dtype)


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("G_", [2, 4])
def test_twin_equals_the_fp32_loop(dtype, G_):
    g = torch.Generator().manual_seed(G_)
    x = (torch.rand(4 * G_, 300, generator=g) * 3e-3).to(dtype)
    x[:, :40] = x[:1, :40]                         # ties: equal scores in every head of the group
    x[0, 50:60] = 0
    x[1, 60:70] = torch.finfo(dtype).tiny            # the smallest normal, summed with zeros and tiny values
    got = group_reduce(x, G_)
    assert got.shape == (4, 300) and got.dtype == dtype
    assert torch.equal(got.view(torch.int16), _loop_reduce(x, G_).view(torch.int16))
    assert torch.equal(got[:, :40], x[::G_, :40])   # the mean of equal values is that value


# ---------------- the plugin ----------------
def _model(request, device, arch="tiny-llama", method="pyramidkv", capacity=48, gqa=True, fp8=False):
    runner.patch(method)
    if device == "cpu":
        dev = torch.device("cpu")
        model = runner.build_model(arch, dev, torch.bfloat16, "eager")
        runner.set_knobs(model, method, capacity, backend_factory=OracleGqaBackend)
    else:
        request.getfixturevalue("libpkv")
        from gpu_util import dev as gpu
        dev = gpu()
        model = runner.build_model(arch, dev, torch.bfloat16, "sdpa")
        runner.set_knobs(model, method, capacity)
    model.config.pkv_gqa_shared = gqa
    model.config.pkv_kv_cache_dtype = "fp8_e4m3" if fp8 else None
    return model, dev


def _prompts(model, dev, lengths, seed=11):
    return [runner.synthetic_prompt(model.config.vocab_size, n, seed + i, dev) for i, n in enumerate(lengths)]


def _graph_modes(device):
    return [False] if device == "cpu" else [False, True]


@pytest.mark.parametrize("device", DEVICES)
@pytest.mark.parametrize("method", ["pyramidkv", "snapkv", "h2o", "streamingllm", "l2norm"])
@pytest.mark.parametrize("fp8", [False, True])
def test_cache_shapes_and_bytes(oracle, request, device, method, fp8):
    """Every layer holds [1, Hkv, capacity, D]: G times fewer bytes than the per-query-head cache at the same rows."""
    model, dev = _model(request, device, method=method, capacity=48 if method != "streamingllm" else 40, fp8=fp8)
    ids = _prompts(model, dev, (150,))[0]
    c = G._prefill(model, ids)[1]
    model.config.pkv_gqa_shared = False
    c0 = G._prefill(model, ids)[1]
    Hq, Hkv = model.config.num_attention_heads, model.config.num_key_value_heads
    for l, l0 in zip(c.layers, c0.layers):
        assert isinstance(l, PkvBatchCacheLayer) and l.group == Hq // Hkv and l.num_q_heads == Hq
        assert isinstance(l, PkvFp8CacheLayer) == fp8 and l.k_buf.shape[:2] == (1, Hkv) and l0.k_buf.shape[:2] == (1, Hq)
        rows = l0.rows_host[0][0] if isinstance(l0, PkvBatchCacheLayer) else l0.length
        assert l.rows_host == [[rows] * Hkv] and l.rows.cpu().tolist() == [rows] * Hkv and l.seq_seen == [150]
        assert l.capacity == l0.capacity and l.get_seq_length() == 150
        assert l.k_buf.numel() * Hq // Hkv == l0.k_buf.numel()


@pytest.mark.parametrize("device", DEVICES)
@pytest.mark.parametrize("method", ["streamingllm", "l2norm"])
def test_query_independent_methods_unchanged(oracle, request, device, method):
    """StreamingLLM and L2Norm select the same rows for every head of a group: with the knob the cache is the knob-off cache
    with the duplicates removed, and decoding gives the same tokens and the same logits."""
    cap = 40 if method == "streamingllm" else 48
    model, dev = _model(request, device, method=method, capacity=cap)
    ids = _prompts(model, dev, (150,))[0]
    Gr = model.config.num_attention_heads // model.config.num_key_value_heads
    seq = {}
    caches = {}
    for knob in (True, False):
        model.config.pkv_gqa_shared = knob
        seq[knob] = G.greedy_generate(model, ids, 8)[0].tolist()
        caches[knob] = G._prefill(model, ids)[1]
    assert seq[True] == seq[False]
    for l, l0 in zip(caches[True].layers, caches[False].layers):
        n = l.length
        assert torch.equal(l.k_buf[:, :, :n], l0.k_buf[:, ::Gr, :n]) and torch.equal(l.v_buf[:, :, :n], l0.v_buf[:, ::Gr, :n])
    for tok in seq[True][150:157]:
        lg = {}
        for knob, cache in caches.items():
            with torch.no_grad():
                lg[knob] = model(input_ids=torch.tensor([[tok]], device=dev), past_key_values=cache, use_cache=True).logits[0, -1]
        assert torch.equal(lg[True], lg[False])


@pytest.mark.parametrize("device", DEVICES)
@pytest.mark.parametrize("arch,method,fp8", [("tiny-llama", "pyramidkv", False), ("tiny-mistral", "snapkv", False),
                                              ("tiny-llama", "h2o", False), ("tiny-llama", "snapkv", True)])
def test_static_loop_graph_eager_and_hf_generate(oracle, request, device, arch, method, fp8):
    model, dev = _model(request, device, arch, method, 40, fp8=fp8)
    ids = _prompts(model, dev, (150,))[0]
    new = 8
    with torch.no_grad():
        ref = model.generate(ids, attention_mask=torch.ones_like(ids), max_new_tokens=new, min_new_tokens=new, num_beams=1,
                             do_sample=False, pad_token_id=0, return_dict_in_generate=True)
    assert all(isinstance(l, PkvBatchCacheLayer) and l.group > 1 for l in ref.past_key_values.layers)
    for use_graph in _graph_modes(device):
        seq, cache = G.greedy_generate(model, ids, new, use_graph=use_graph, return_cache=True)
        assert seq.tolist() == ref.sequences.tolist(), use_graph
        for mine, theirs in zip(cache.layers, ref.past_key_values.layers):
            assert mine.rows_host == theirs.rows_host and mine.get_seq_length() == theirs.get_seq_length() == 150 + new - 1
            n = mine.length
            assert torch.equal(mine.k_buf[:, :, :n].view(torch.uint8), theirs.k_buf[:, :, :n].view(torch.uint8))


@pytest.mark.parametrize("device", DEVICES)
@pytest.mark.parametrize("fp8", [False, True])
def test_batch_equals_solo(oracle, request, device, fp8):
    model, dev = _model(request, device, fp8=fp8)
    prompts = _prompts(model, dev, (150, 37, 300))
    for use_graph in _graph_modes(device):
        solo = [G.greedy_generate(model, p, 7, use_graph=use_graph)[0].tolist() for p in prompts]
        batch = G.greedy_generate_batch(model, prompts, 7, use_graph=use_graph)
        assert [t.tolist() for t in batch] == solo


@pytest.mark.parametrize("device", DEVICES)
@pytest.mark.parametrize("fp8", [False, True])
def test_join_group_caches(oracle, request, device, fp8):
    model, dev = _model(request, device, fp8=fp8)
    prompts = _prompts(model, dev, (150, 37, 300))
    singles = [G._prefill(model, p)[1] for p in prompts]
    joined = join_caches(singles, reserve=5)
    Hkv = model.config.num_key_value_heads
    for i, layer in enumerate(joined.layers):
        want = [c.layers[i].rows_host[0] for c in singles]
        assert type(layer) is type(singles[0].layers[i]) and layer.group == singles[0].layers[i].group
        assert layer.k_buf.shape[:2] == (3, Hkv) and layer.rows_host == want and layer.seq_seen == [150, 37, 300]
        assert layer.capacity == max(max(r) for r in want) + 5
        for b, c in enumerate(singles):
            n = want[b][0]
            assert torch.equal(layer.k_buf[b, :, :n].view(torch.uint8), c.layers[i].k_buf[0, :, :n].view(torch.uint8))
    model.config.pkv_gqa_shared = False
    plain = G._prefill(model, prompts[0])[1]
    with pytest.raises(ValueError, match="GQA-shared"):
        join_caches([singles[0], plain])


def test_refusals(oracle):
    for method in ("adakv", "headkv"):
        model, dev = _model(None, "cpu", method=method)
        if method == "headkv":
            model.config.head_capacity = [[40] * model.config.num_attention_heads] * model.config.num_hidden_layers
        with pytest.raises(NotImplementedError, match="per QUERY head"):
            G._prefill(model, _prompts(model, dev, (150,))[0])
    model, dev = _model(None, "cpu")
    ids = _prompts(model, dev, (150,))[0]
    _, cache = G._prefill(model, ids)
    layer = cache.layers[0]
    x = torch.zeros(1, 2, 2, 64, dtype=torch.bfloat16)
    for call in (lambda: layer.update(x, x), lambda: layer.crop(3), lambda: layer.batch_repeat_interleave(2),
                 lambda: layer.batch_select_indices(torch.tensor([0]))):
        with pytest.raises(NotImplementedError):
            call()
    with torch.no_grad(), pytest.raises(NotImplementedError):
        model(input_ids=ids[:, :3], past_key_values=cache, use_cache=True)
    with pytest.raises(NotImplementedError, match="pkv_gqa_shared"):
        from types import SimpleNamespace
        from pyramidkv_b200.pipeline import PipelineRunner
        PipelineRunner(SimpleNamespace(config=SimpleNamespace(pkv_gqa_shared=True)))
    model.config.pkv_gqa_shared = "yes"
    with pytest.raises(ValueError, match="pkv_gqa_shared"):
        G._prefill(model, ids)


def test_runner_flag(oracle):
    import run_longbench
    import run_needle_in_haystack
    base = ["--method", "StreamingLLM", "--model_path", "tiny-llama", "--max_capacity_prompts", "40", "--attn_implementation",
            "eager", "--dataset", "lcc", "--prompt_tokens", "150", "--max_new_tokens", "5", "--max_num_examples", "2", "--dtype",
            "bfloat16", "--decode_loop", "static-eager"]
    cpu = torch.device("cpu")
    plain = run_longbench.main(base, backend_factory=OracleGqaBackend, device=cpu)
    assert all("gqa_shared" not in r for r in plain)
    for extra in ([], ["--eval_batch_size", "2"], ["--kv_cache_dtype", "fp8_e4m3"]):
        got = run_longbench.main(base + ["--gqa_shared"] + extra, backend_factory=OracleGqaBackend, device=cpu)
        assert all(r["gqa_shared"] is True for r in got)
        if not extra:      # StreamingLLM: the same tokens with the knob on and off
            assert [r["pred_ids"] for r in got] == [r["pred_ids"] for r in plain]
    needle = run_needle_in_haystack.main(["--method", "pyramidkv", "--model_name", "tiny-llama", "--s_len", "150", "--e_len", "151",
                                          "--max_capacity_prompt", "48", "--max_new_tokens", "3", "--decode_loop", "static-eager",
                                          "--gqa_shared", "--dtype", "bfloat16"], backend_factory=OracleGqaBackend, device=cpu)
    assert needle[0]["gqa_shared"] is True
    for method in ("FullKV", "AdaKV", "HeadKV"):
        with pytest.raises(NotImplementedError, match="gqa_shared"):
            run_longbench.main(["--method", method, "--model_path", "tiny-llama", "--dataset", "lcc", "--prompt_tokens", "20",
                                "--max_new_tokens", "2", "--max_capacity_prompts", "40", "--gqa_shared"], device=cpu)


def test_pooled_kv_offset_query(libpkv):
    """pkv_evict_pooled_kv_offset (host arithmetic only): the per-KV-head segment exists only with PKV_FLAG_GQA_SHARED and a
    scoring method, lies inside the workspace behind the per-query-head scores (L2Norm: is them), and pkv_ws_layout keeps
    its size; unknown flag bits and the fused forms are refused."""
    import ctypes as C
    from pyramidkv_b200 import _lib
    L = _lib.lib()
    d = _lib.EvictDesc()
    d.struct_bytes = C.sizeof(_lib.EvictDesc)
    d.method, d.dtype, d.pooling, d.kernel_size = _lib.METHODS["snapkv"], 0, 0, 5
    d.num_q_heads, d.num_kv_heads, d.head_dim, d.window, d.seq_len, d.top_k = 32, 8, 128, 32, 4096, 512
    off, lay = C.c_uint64(0), _lib.WsLayout()
    assert L.pkv_evict_pooled_kv_offset(C.byref(d), C.byref(off)) == _lib.PKV_ERR_INVALID_ARG
    plain = L.pkv_evict_workspace_bytes(C.byref(d))
    d.flags = _lib.FLAG_GQA_SHARED
    assert L.pkv_evict_pooled_kv_offset(C.byref(d), C.byref(off)) == _lib.PKV_OK
    assert L.pkv_evict_workspace_layout(C.byref(d), C.byref(lay)) == _lib.PKV_OK
    pitch = lay.pooled_pitch
    assert off.value >= lay.pooled_off + 32 * pitch * 2 and off.value % 256 == 0
    assert off.value + 8 * pitch * 2 <= lay.total_bytes and lay.total_bytes > plain
    d.flags = _lib.FLAG_GQA_SHARED | 64
    assert L.pkv_evict_pooled_kv_offset(C.byref(d), C.byref(off)) == _lib.PKV_ERR_UNSUPPORTED
    d.flags = 1 << 12
    assert L.pkv_evict_workspace_bytes(C.byref(d)) == 0
    d.flags = _lib.FLAG_GQA_SHARED
    d.method, d.window = _lib.METHODS["l2norm"], 0
    assert L.pkv_evict_pooled_kv_offset(C.byref(d), C.byref(off)) == _lib.PKV_OK
    assert L.pkv_evict_workspace_layout(C.byref(d), C.byref(lay)) == _lib.PKV_OK and off.value == lay.pooled_off
    d.method, d.window = _lib.METHODS["streamingllm"], 32
    assert L.pkv_evict_pooled_kv_offset(C.byref(d), C.byref(off)) == _lib.PKV_ERR_INVALID_ARG
