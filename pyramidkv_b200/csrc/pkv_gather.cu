// pkv_gather.cu — stage 4: K/V gather + last-window concat, written straight into the cache.
//
// Replaces  k_past = K[:, :, :-W].gather(2, idx.expand(D)); torch.cat([k_past, K[:, :, -W:]], 2)
// (and the same for V): pyramidkv_utils.py:271-282, :335-346, :563-574, :607-619 — four launches and an
// int64 index per ELEMENT in the reference; here one launch, one int32 index per ROW, 128-bit row copies.
// The source is the un-repeated [Hkv, S, D] tensor; query head h copies from kv head h / G.
#include "pkv_common.cuh"
#include "pkv_internal.h"

namespace pkv {
namespace {

struct GatherParams {
    const uint16_t* src[2];
    int64_t s_sh[2], s_ss[2];
    uint16_t* dst[2];
    int64_t cache_sh;
    const int32_t* idx32;  // [Hq][k]; nullptr => identity 0..k-1 (StreamingLLM)
    int64_t k, S;
    int W, G;
};

constexpr int kGatherRowsPerCta = 128;   // 16 rows per warp: 8 independent 128-bit loads in flight per lane (D = 128)

template <int D>
__global__ void __launch_bounds__(256) gather_kernel(const GatherParams p) {
    constexpr int LPR = D / 8;         // lanes per row (16-byte pieces)
    constexpr int RPW = 32 / LPR;      // rows per warp instruction
    constexpr int ITER = 16 / RPW;     // each warp moves 16 rows
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int h = blockIdx.y, which = blockIdx.z;
    const int64_t rows = p.k + p.W;
    const int64_t r_base = int64_t(blockIdx.x) * kGatherRowsPerCta + warp * 16 + lane / LPR;
    const int piece = lane % LPR;
    // (selects instead of indexing the parameter arrays with a run-time index, which would spill them to local memory)
    const uint16_t* src = (which ? p.src[1] : p.src[0]) + int64_t(h / p.G) * (which ? p.s_sh[1] : p.s_sh[0]);
    uint16_t* dst = (which ? p.dst[1] : p.dst[0]) + int64_t(h) * p.cache_sh;
    const int64_t ss = which ? p.s_ss[1] : p.s_ss[0];

    uint4 v[ITER];
    int64_t tok[ITER];
#pragma unroll
    for (int it = 0; it < ITER; ++it) {
        const int64_t r = r_base + it * RPW;
        tok[it] = -1;
        if (r < rows) tok[it] = (r < p.k) ? (p.idx32 ? int64_t(p.idx32[int64_t(h) * p.k + r]) : r) : (p.S - p.W + (r - p.k));
    }
#pragma unroll
    for (int it = 0; it < ITER; ++it)
        if (tok[it] >= 0) v[it] = ldg_nc_v4(src + tok[it] * ss + piece * 8);
#pragma unroll
    for (int it = 0; it < ITER; ++it) {
        const int64_t r = r_base + it * RPW;
        if (tok[it] >= 0) *reinterpret_cast<uint4*>(dst + r * D + piece * 8) = v[it];
    }
}

// StreamingLLM keeps tokens 0..k-1 (pyramidkv_utils.py:607): materialise them only if the caller asks.
__global__ void iota_idx_kernel(int64_t* idx64, int64_t k, int64_t total) {
    const int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i < total) idx64[i] = i % k;
}

// PKV_FLAG_GQA_SHARED: out[j][t] = rn_dtype((sum_g f32(in[j*G+g][t]), g ascending) / f32(G)) over whole pooled rows (the pitch
// is a multiple of 8 elements); 8 elements per thread, grid (row blocks, kv head). The division is correctly rounded, so the
// result does not depend on how the compiler would treat a multiply by 1/G.
template <typename T>
__global__ void __launch_bounds__(256) group_reduce_kernel(const uint16_t* __restrict__ in, uint16_t* __restrict__ out, int64_t pitch, int G) {
    const int64_t i = (int64_t(blockIdx.x) * blockDim.x + threadIdx.x) * 8;
    if (i >= pitch) return;
    const int j = blockIdx.y;
    float s[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) s[e] = 0.f;
    for (int g = 0; g < G; ++g) {
        const uint4 v = ldg_nc_v4(in + (int64_t(j) * G + g) * pitch + i);
        const uint32_t u[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
        for (int e = 0; e < 4; ++e) {
            s[2 * e] = __fadd_rn(s[2 * e], DT<T>::to_f32(uint16_t(u[e] & 0xffffu)));
            s[2 * e + 1] = __fadd_rn(s[2 * e + 1], DT<T>::to_f32(uint16_t(u[e] >> 16)));
        }
    }
    const float fg = float(G);
    uint32_t w[4];
#pragma unroll
    for (int e = 0; e < 4; ++e)
        w[e] = uint32_t(DT<T>::from_f32(__fdiv_rn(s[2 * e], fg))) | (uint32_t(DT<T>::from_f32(__fdiv_rn(s[2 * e + 1], fg))) << 16);
    *reinterpret_cast<uint4*>(out + int64_t(j) * pitch + i) = make_uint4(w[0], w[1], w[2], w[3]);
}

}  // namespace

cudaError_t launch_group_reduce(const EvictArgs& a, cudaStream_t st) {
    const uint16_t* in = reinterpret_cast<const uint16_t*>(a.ws_base + a.ws.pooled_off);
    uint16_t* out = reinterpret_cast<uint16_t*>(a.ws_base + a.pooled_kv_off);
    const int64_t vecs = a.ws.pooled_pitch / 8;
    const dim3 grid(unsigned((vecs + 255) / 256), unsigned(a.Hkv));
    if (a.dtype == PKV_BF16) group_reduce_kernel<__nv_bfloat16><<<grid, 256, 0, st>>>(in, out, a.ws.pooled_pitch, a.G);
    else group_reduce_kernel<__half><<<grid, 256, 0, st>>>(in, out, a.ws.pooled_pitch, a.G);
    count_launch();
    return cudaGetLastError();
}

cudaError_t launch_gather(const EvictArgs& a, cudaStream_t st) {
    GatherParams p;
    p.src[0] = a.kk; p.src[1] = a.vv;
    p.s_sh[0] = a.k_sh; p.s_sh[1] = a.v_sh;
    p.s_ss[0] = a.k_ss; p.s_ss[1] = a.v_ss;
    p.dst[0] = a.k_cache; p.dst[1] = a.v_cache;
    p.cache_sh = a.cache_sh;
    p.idx32 = (a.method == PKV_STREAMINGLLM || a.k == 0) ? nullptr : reinterpret_cast<const int32_t*>(a.ws_base + a.ws.idx32_off);
    p.k = a.k; p.S = a.S; p.W = a.W; p.G = a.G;
    const int64_t rows = a.k + a.W;
    const dim3 grid(unsigned((rows + kGatherRowsPerCta - 1) / kGatherRowsPerCta), unsigned(a.Hq), 2);
    if (a.D == 128) gather_kernel<128><<<grid, 256, 0, st>>>(p);
    else gather_kernel<64><<<grid, 256, 0, st>>>(p);
    count_launch();
    if (a.method == PKV_STREAMINGLLM && a.idx_out && a.k > 0) {
        const int64_t total = int64_t(a.Hq) * a.k;
        iota_idx_kernel<<<unsigned((total + 255) / 256), 256, 0, st>>>(a.idx_out, a.k, total);
        count_launch();
    }
    return cudaGetLastError();
}

}  // namespace pkv
