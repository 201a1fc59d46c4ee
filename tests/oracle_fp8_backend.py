"""TEST-ONLY backend for the FP8 compacted cache: the batched oracle backend plus `cache_quantize_fp8` (the torch form of the
quantisation rule of include/pkv.h) and `decode_attn_batch_fp8` (fp64 attention over the dequantised rows, after quantising
and storing the new row). Never importable from product code."""
import torch

from oracle_batch_backend import OracleBatchBackend

E4M3_MAX = 448.0


def quantize_rows(x: torch.Tensor):
    """x [..., D] bf16 / fp16 -> (E4M3 bytes as float8_e4m3fn [..., D], fp32 scales [...]), on the CPU:
    amax = max|x_e|; amax == 0: scale 0, bytes 0; else inv = rn_f32(448 / amax), q_e = e4m3(rn_f32(x_e * inv)),
    scale = rn_f32(amax / 448). Every division is tensor by tensor (an IEEE fp32 division)."""
    xf = x.detach().cpu().float()
    amax = xf.abs().amax(dim=-1)
    nz = amax != 0
    safe = torch.where(nz, amax, torch.ones_like(amax))
    inv = torch.full_like(safe, E4M3_MAX) / safe
    q = (xf * inv[..., None]).to(torch.float8_e4m3fn).view(torch.uint8) * nz[..., None].to(torch.uint8)
    scale = torch.where(nz, amax / torch.full_like(amax, E4M3_MAX), torch.zeros_like(amax))
    return q.view(torch.float8_e4m3fn), scale


def dequantize(q: torch.Tensor, scale: torch.Tensor) -> torch.Tensor:
    return q.cpu().float() * scale.cpu()[..., None]


class OracleFp8Backend(OracleBatchBackend):
    name = "oracle-cpu fp8 (tests only)"

    def cache_quantize_fp8(self, layers):
        for k, v, kq, vq, ks, vs, rows, rows_dev in layers:
            B, H = k.shape[:2]
            for b in range(B):
                for h in range(H):
                    n = min(int(rows_dev[b * H + h]), int(rows)) if rows_dev is not None else int(rows)
                    for src, dst, sc in ((k, kq, ks), (v, vq, vs)):
                        q, s = quantize_rows(src[b, h, :n])
                        dst.view(torch.uint8)[b, h, :n] = q.view(torch.uint8).to(dst.device)
                        sc[b, h, :n] = s.to(sc.device)

    def decode_attn_batch_fp8(self, q, k_q, v_q, k_scale, v_scale, length, k_new, v_new, rows=None, step=None, max_length=0,
                              workspace=None, out=None, softmax_scale=0.0):
        B, Hq, cap, D = k_q.shape
        extra = int(length) + (int(step.item()) if step is not None else 0)
        G = Hq // k_new.shape[1]
        kq_new, ks_new = quantize_rows(k_new)
        vq_new, vs_new = quantize_rows(v_new)
        scale = softmax_scale or D ** -0.5
        res = torch.empty(B, Hq, D, dtype=q.dtype)
        for b in range(B):
            for h in range(Hq):
                T = (int(rows.reshape(-1)[b * Hq + h]) if rows is not None else 0) + extra
                assert 1 <= T <= (max_length or cap) <= cap
                k_q.view(torch.uint8)[b, h, T - 1] = kq_new.view(torch.uint8)[b, h // G].to(k_q.device)
                v_q.view(torch.uint8)[b, h, T - 1] = vq_new.view(torch.uint8)[b, h // G].to(v_q.device)
                k_scale[b, h, T - 1] = ks_new[b, h // G]
                v_scale[b, h, T - 1] = vs_new[b, h // G]
                K = dequantize(k_q[b, h, :T], k_scale[b, h, :T]).double()
                V = dequantize(v_q[b, h, :T], v_scale[b, h, :T]).double()
                p = torch.softmax((K @ q[b, h].cpu().double()) * scale, dim=0)
                res[b, h] = (p @ V).to(q.dtype)
        res = res.to(q.device)
        if out is not None:
            out.copy_(res)
            return out
        return res
