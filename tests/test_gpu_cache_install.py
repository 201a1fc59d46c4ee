"""`pkv_cache_install` (ops.cache_install) on the GPU against its torch twin (tests/oracle_continuous_backend.py): bytes, scales,
row counts relative to the device step counter, untouched sentinels and slots, one launch per 32 layers, graph replay,
argument errors; and the continuous decoder's decode launches per step."""
import pytest
import torch

from oracle_continuous_backend import install_twin

pytestmark = pytest.mark.gpu

FP8 = torch.float8_e4m3fn
# cache form -> (heads, FP8, per-head device counts)
FORMS = {"uniform": (8, False, False), "ragged": (8, False, True), "fp8": (8, True, False), "fp8_ragged": (8, True, True),
         "gqa": (2, False, False), "gqa_fp8": (2, True, False)}


def _bits(t):
    return t.view({FP8: torch.uint8, torch.float32: torch.int32}.get(t.dtype, torch.int16))


def _layer(dev, H, D, fp8, ragged, B=4, cap=96, src_cap=80, rows=70, seed=0, dtype=torch.bfloat16):
    """One layer: a prompt's source buffers and a batched destination filled with sentinel bytes."""
    g = torch.Generator(device="cpu").manual_seed(seed)
    def rnd(*shape):
        x = torch.randn(*shape, generator=g).to(dev)
        return x.to(FP8) if fp8 else x.to(dtype)
    sk, sv = rnd(1, H, src_cap, D), rnd(1, H, src_cap, D)
    if fp8:
        dk = torch.full((B, H, cap, D), 0x3C, dtype=torch.uint8, device=dev).view(FP8)
    else:
        dk = torch.full((B, H, cap, D), 7.0, dtype=dtype, device=dev)
    dv = dk.clone()
    ss = ds = None
    if fp8:
        ss = (torch.rand(1, H, src_cap, generator=g).to(dev), torch.rand(1, H, src_cap, generator=g).to(dev))
        ds = (torch.full((B, H, cap), -3.0, device=dev), torch.full((B, H, cap), -4.0, device=dev))
    rows_dev = torch.randint(1, rows + 1, (H,), generator=g, dtype=torch.int32).to(dev) if ragged else None
    dr = torch.full((B * H,), 1234, dtype=torch.int32, device=dev)
    return [sk, sv, ss, rows, rows_dev, dk, dv, ds, dr]


def _clone(item):
    c = lambda t: None if t is None else (tuple(x.clone() for x in t) if isinstance(t, tuple) else (t.clone() if torch.is_tensor(t) else t))
    return [c(t) for t in item]


def _same(a, b):
    for x, y in zip(a, b):
        if x is None or isinstance(x, int):
            continue
        for u, v in (zip(x, y) if isinstance(x, tuple) else [(x, y)]):
            assert torch.equal(_bits(u), _bits(v))


@pytest.mark.parametrize("form", list(FORMS))
@pytest.mark.parametrize("D", [64, 128])
def test_install_equals_twin(libpkv, form, D):
    from pyramidkv_b200 import ops
    dev = torch.device("cuda")
    H, fp8, ragged = FORMS[form]
    layers = [_layer(dev, H, D, fp8, ragged, seed=i, rows=70 - 9 * i) for i in range(3)]
    want = [_clone(l) for l in layers]
    step = torch.tensor([13], dtype=torch.int32, device=dev)
    ops.cache_install(layers, 2, step)
    install_twin(want, 2, step.cpu())
    for got, ref in zip(layers, want):
        _same(got, ref)                              # bytes, scales, sentinels past the rows, the other slots, row counts
        n = [min(got[3], int(r)) for r in got[4].tolist()] if ragged else [got[3]] * H
        assert got[8].tolist()[2 * H:3 * H] == [x - 13 for x in n] and got[8].tolist()[:2 * H] == [1234] * (2 * H)
    # parking: zero rows, only the row counts change
    before = [_clone(l) for l in layers]
    ops.cache_install([[None, None, None, 0, None, *l[5:]] for l in layers], 1, step)
    for got, old in zip(layers, before):
        assert got[8].tolist()[H:2 * H] == [-13] * H
        old[8][H:2 * H] = -13
        _same(got, old)


def test_fp16_and_one_launch_per_32_layers(libpkv):
    from pyramidkv_b200 import _lib, ops
    dev = torch.device("cuda")
    step = torch.tensor([2], dtype=torch.int32, device=dev)
    for n_layers, launches in ((1, 1), (32, 1), (33, 2)):
        layers = [_layer(dev, 8, 128, False, i % 2 == 1, seed=i, dtype=torch.float16) for i in range(n_layers)]
        want = [_clone(l) for l in layers]
        torch.cuda.synchronize()
        c0 = _lib.launch_count()
        ops.cache_install(layers, 0, step)
        assert _lib.launch_count() - c0 == launches
        install_twin(want, 0, step.cpu())
        for got, ref in zip(layers, want):
            _same(got, ref)


def test_install_replays_in_a_graph(libpkv):
    from pyramidkv_b200 import ops
    dev = torch.device("cuda")
    layers = [_layer(dev, 8, 128, True, True, seed=i) for i in range(4)]
    step = torch.zeros(1, dtype=torch.int32, device=dev)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        ops.cache_install(layers, 3, step)          # warm-up outside the capture
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        ops.cache_install(layers, 3, step)
    for it in range(3):
        for l in layers:                            # new source contents and step, same pointers
            l[0].view(torch.uint8).random_(0, 120)
            l[2][0].uniform_()
            l[4].random_(1, 71)
        step.fill_(7 * it + 1)
        want = [_clone(l) for l in layers]
        graph.replay()
        install_twin(want, 3, step.cpu())
        for got, ref in zip(layers, want):
            _same(got, ref)


def _misaligned(t):
    """A contiguous copy of t that starts 2 bytes past a 16-byte boundary."""
    m = torch.empty(t.numel() + 8, dtype=t.dtype, device=t.device)[1:1 + t.numel()].view(t.shape)
    m.copy_(t)
    return m


def test_argument_errors(libpkv):
    from pyramidkv_b200 import ops
    dev = torch.device("cuda")
    step = torch.zeros(1, dtype=torch.int32, device=dev)
    base = _layer(dev, 8, 64, False, False)
    cases = {
        "slot": (lambda: [base], 4),
        "slot-neg": (lambda: [base], -1),
        "rows above the destination": (lambda: [base[:3] + [97] + base[4:]], 0),
        "rows above the source": (lambda: [base[:3] + [81] + base[4:]], 0),
        "dtype": (lambda: [[base[0].half(), base[1].half()] + base[2:]], 0),
        "heads": (lambda: [[base[0][:, :4].contiguous(), base[1][:, :4].contiguous()] + base[2:]], 0),
        "misaligned": (lambda: [[_misaligned(base[0]), base[1]] + base[2:]], 0),
        "dst rows": (lambda: [base[:8] + [base[8][:-1]]], 0),
        "fp8 without scales": (lambda: [_layer(dev, 8, 64, True, False)[:7] + [None, base[8]]], 0),
        "scales on a 16-bit cache": (lambda: [base[:7] + [(torch.zeros(4, 8, 96, device=dev),) * 2, base[8]]], 0),
    }
    for name, (make, slot) in cases.items():
        items = make()
        snapshot = [_clone(l) for l in items]
        with pytest.raises(ValueError):
            ops.cache_install(items, slot, step)
        for got, old in zip(items, snapshot):
            _same(got, old)                          # a refused call writes nothing
    with pytest.raises(ValueError):
        ops.cache_install([base], 0, torch.zeros(1, dtype=torch.int64, device=dev))


@pytest.mark.parametrize("fp8,gqa", [(False, False), (True, True)])
def test_decode_launches_per_step_unchanged(libpkv, fp8, gqa):
    """One decode launch per layer and step for any number of slots, as in the lock-step loop; admission is one launch."""
    from pyramidkv_b200 import _lib, generate as G, runner
    from pyramidkv_b200.cache import join_caches
    from gpu_util import dev as gpu
    runner.patch("pyramidkv")
    try:
        dev = gpu()
        model = runner.build_model("tiny-llama", dev, torch.bfloat16, "sdpa")
        runner.set_knobs(model, "pyramidkv", 48)
        model.config.pkv_kv_cache_dtype = "fp8_e4m3" if fp8 else None
        model.config.pkv_gqa_shared = gqa
        L = model.config.num_hidden_layers
        for n in (2, 5):
            prompts = [runner.synthetic_prompt(model.config.vocab_size, 100 + 7 * i, i, dev) for i in range(n + 1)]
            firsts, caches = zip(*[G._prefill(model, p) for p in prompts])
            dec = G.ContinuousDecoder(model, join_caches(list(caches[:n]), reserve=8), torch.cat(firsts[:n]), [6] * n, chunk=2,
                                      use_graph=False)
            torch.cuda.synchronize()
            c0 = _lib.launch_count()
            dec.run_chunk(2)
            assert _lib.launch_count() - c0 == 2 * L
            c0 = _lib.launch_count()
            dec.admit(0, caches[n], firsts[n], 4)
            assert _lib.launch_count() - c0 == 1
            dec.finish()
    finally:
        from pyramidkv.monkeypatch import restore
        restore()
