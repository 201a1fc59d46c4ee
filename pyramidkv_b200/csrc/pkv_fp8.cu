// pkv_fp8.cu — the opt-in FP8 (E4M3) compacted cache: the conversion of the 16-bit cache the eviction wrote to E4M3 rows with
// one fp32 scale per row (format in pkv_rows.cuh). The decode step over those rows is decode_kernel (pkv_decode.cu).
#include <algorithm>

#include "pkv_common.cuh"
#include "pkv_internal.h"
#include "pkv_rows.cuh"

namespace pkv {
namespace {

constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;

// ---------------- conversion of the compacted 16-bit cache ----------------
// grid (x: row groups, y: layer). A group of D/16 lanes converts one row of K or V: two 128-bit loads per lane, the row max
// across the group, packed conversion, one 128-bit store per lane and one scale. Rows past a (sequence, head)'s count are
// neither read nor written.
template <typename T, int D>
__global__ void __launch_bounds__(kThreads) quantize_fp8_kernel(const __grid_constant__ QuantArgs a) {
    constexpr int LPR = D / 16, GPW = 32 / LPR;
    const QuantLayer& L = a.layer[blockIdx.y];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, sub = lane / LPR, piece = lane % LPR;
    const int64_t per_kv = int64_t(a.num_seqs) * a.H * L.rows;   // rows of K (then as many of V)
    const int64_t total = 2 * per_kv;
    const int64_t stride = int64_t(gridDim.x) * kWarps * GPW;
    // warp-uniform trip count (the row max shuffles need every lane)
    for (int64_t base = (int64_t(blockIdx.x) * kWarps + warp) * GPW; base < total; base += stride) {
        const int64_t i = base + sub;
        bool ok = i < total;
        int kv = 0;
        int64_t sh = 0, r = 0;
        float x[16];
#pragma unroll
        for (int e = 0; e < 16; ++e) x[e] = 0.f;
        if (ok) {
            kv = i >= per_kv ? 1 : 0;
            const int64_t j = i - kv * per_kv;
            sh = j / L.rows;                 // sequence * H + head
            r = j - sh * L.rows;
            if (L.rows_dev) ok = r < int64_t(__ldg(L.rows_dev + sh));
            if (ok) load16<T>(L.src[kv] + (sh * L.src_cap + r) * D + piece * 16, x);
        }
        const float amax = row_amax<LPR>(x);
        if (ok) {
            float s;
            const uint4 q = quantize16(x, amax, s);
            *reinterpret_cast<uint4*>(L.dst[kv] + (sh * L.dst_cap + r) * D + piece * 16) = q;
            if (piece == 0) L.scale[kv][sh * L.dst_cap + r] = s;
        }
    }
}

template <typename T, int D>
cudaError_t launch_quantize_t(const QuantArgs& a, int num_sms, cudaStream_t st) {
    constexpr int rows_per_cta = kWarps * (32 / (D / 16));
    int64_t most = 0;
    for (int l = 0; l < a.n_layers; ++l) most = std::max(most, 2 * int64_t(a.num_seqs) * a.H * a.layer[l].rows);
    int64_t gx = (most + rows_per_cta - 1) / rows_per_cta;
    const int64_t cap = std::max<int64_t>(1, int64_t(num_sms) * 16);   // grid-stride beyond ~16 CTAs per SM
    gx = std::max<int64_t>(1, std::min(gx, cap));
    quantize_fp8_kernel<T, D><<<dim3(unsigned(gx), unsigned(a.n_layers)), kThreads, 0, st>>>(a);
    count_launch();
    return cudaGetLastError();
}

}  // namespace

cudaError_t launch_quantize_fp8(const QuantArgs& a, int num_sms, cudaStream_t st) {
    if (a.dtype == PKV_BF16) return a.D == 128 ? launch_quantize_t<__nv_bfloat16, 128>(a, num_sms, st) : launch_quantize_t<__nv_bfloat16, 64>(a, num_sms, st);
    return a.D == 128 ? launch_quantize_t<__half, 128>(a, num_sms, st) : launch_quantize_t<__half, 64>(a, num_sms, st);
}

}  // namespace pkv
