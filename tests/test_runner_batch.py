"""CPU: run_longbench.py --eval_batch_size N decodes the prompts N at a time with the static loop (test backend)."""
import pytest
import torch

from oracle_batch_backend import OracleBatchBackend


def test_eval_batch_size_gives_the_batch_size_one_tokens(oracle):
    import run_longbench
    base = ["--method", "PyramidKV", "--model_path", "tiny-llama", "--max_capacity_prompts", "48", "--attn_implementation", "eager",
            "--dataset", "lcc", "--prompt_tokens", "150", "--max_new_tokens", "5", "--max_num_examples", "3", "--dtype", "bfloat16",
            "--decode_loop", "static-eager"]
    one = run_longbench.main(base, backend_factory=OracleBatchBackend, device=torch.device("cpu"))
    two = run_longbench.main(base + ["--eval_batch_size", "2"], backend_factory=OracleBatchBackend, device=torch.device("cpu"))
    assert [r["pred_ids"] for r in two] == [r["pred_ids"] for r in one]
    assert [r["cache_rows_first_last"] for r in two] == [r["cache_rows_first_last"] for r in one]
    assert [r["batch_size"] for r in two] == [2, 2, 1] and all(r["eval_batch_size"] == 2 for r in two)
    assert all(r["prefill_ms"] > 0 and r["batch_decode_tok_per_s_aggregate"] > 0 for r in two)
    with pytest.raises(NotImplementedError, match="static"):
        run_longbench.main(base[:-2] + ["--eval_batch_size", "2"], backend_factory=OracleBatchBackend, device=torch.device("cpu"))
