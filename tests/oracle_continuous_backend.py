"""TEST-ONLY backend for continuous batching: the GQA / FP8 / batched oracle backend plus `cache_install`, the torch twin of
`pkv_cache_install` (include/pkv.h). Never importable from product code."""
import torch

from oracle_gqa_backend import OracleGqaBackend


def _bytes(t: torch.Tensor) -> torch.Tensor:
    return t.view(torch.uint8) if t.dtype == torch.float8_e4m3fn else t


def install_twin(layers, slot, step):
    """Per layer: head h of slot `slot` receives the source's first n_h = rows (or min(rows, rows_dev[h])) rows of K, V and
    (FP8) their scales; the slot's row counts become n_h - *step. The argument errors of the C entry raise ValueError."""
    s = int(step.reshape(-1)[0])
    for sk, sv, ss, rows, rows_dev, dk, dv, ds, dr in layers:
        B, H, cap, D = dk.shape
        if not 0 <= int(slot) < B:
            raise ValueError(f"slot {slot} outside [0, {B})")
        rows = int(rows)
        if rows < 0 or rows > cap or (rows > 0 and rows > sk.shape[2]):
            raise ValueError(f"rows={rows} outside [0, capacity]")
        if rows > 0 and (sk.dtype != dk.dtype or sk.shape[1] != H or sk.shape[3] != D):
            raise ValueError("source heads, head_dim or dtype differ from the batched cache")
        if (ds is not None) != (dk.dtype == torch.float8_e4m3fn):
            raise ValueError("scales go with FP8 caches only")
        for h in range(H):
            n = min(rows, int(rows_dev[h])) if rows_dev is not None and rows > 0 else rows
            if n > 0:
                _bytes(dk)[slot, h, :n] = _bytes(sk)[0, h, :n]
                _bytes(dv)[slot, h, :n] = _bytes(sv)[0, h, :n]
                if ds is not None:
                    ds[0][slot, h, :n] = ss[0][0, h, :n]
                    ds[1][slot, h, :n] = ss[1][0, h, :n]
            dr[int(slot) * H + h] = n - s


class OracleContinuousBackend(OracleGqaBackend):
    name = "oracle-cpu continuous (tests only)"

    def cache_install(self, layers, slot, step):
        install_twin(layers, slot, step)
