"""-m gpu: the layer batch's select + gather launch (one CTA per head where a head's keys fit its shared memory) holds, for
every layer and every head of every test_gpu_batch shape, exactly the top-k of the pooled rows the batch itself wrote (value
descending, lowest index among equal scores) and byte copies of those K / V rows followed by the window. The per-layer test
compares only the heads whose pooled rows came out identical; this one checks all of them against the oracle's selection."""
import pytest
import torch

from gpu_util import dev
from test_gpu_batch import CASES, _layers, _run

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("Hq,Hkv,S,D,W,budget,kernel,pooling,dtype,L", CASES)
def test_batch_select_is_the_topk_of_its_pooled_rows(oracle, libpkv, Hq, Hkv, S, D, W, budget, kernel, pooling, dtype, L):
    layers = _layers(Hq, Hkv, S, D, dtype, L, seed=300)
    got, ks, _ = _run("pyramidkv", layers, W, budget, kernel, pooling, batch=True)
    G = Hq // Hkv
    for l in range(L):
        pooled, idx, kc, vc = (t.cpu() for t in got[l])
        assert torch.equal(oracle.topk(pooled.contiguous(), ks[l], oracle.TIE_LOWEST_INDEX), idx), f"layer {l}: indices"
        k_src, v_src = layers[l][1].cpu(), layers[l][2].cpu()
        win = torch.arange(S - W, S)
        for h in range(Hq):
            rows = torch.cat([idx[h], win])
            assert torch.equal(kc[h, :ks[l] + W], k_src[h // G][rows]), f"layer {l} head {h}: K rows"
            assert torch.equal(vc[h, :ks[l] + W], v_src[h // G][rows]), f"layer {l} head {h}: V rows"
