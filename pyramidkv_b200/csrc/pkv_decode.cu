// pkv_decode.cu — decode step over the compacted per-query-head cache: in-place append + attention.
//
// Replaces, per layer and token: DynamicCache.update's torch.cat of the whole layer cache
// (cache_utils_think.py:383-384, called at llama_model.py:170 / :288 / :403), the two transposes and the
// attention launch (eager llama_model.py:174-183, sdpa :291-313, flash :411-445 -> flash_attn_func :77).
// q_len == 1 and every cached row is visible, so there is no mask. One launch for T <= 256 rows per
// head; longer caches are split along T (flash-decoding) and merged by a second small kernel.
// Several sequences decoded in lock-step share one launch: the grid is (split, q head, sequence), and every
// (sequence, head) divides its own rows among the splits a one-sequence launch would use.
// HBM-bound: reads 2*Hq*T*D*2 bytes per sequence; each row is fetched with 128-bit loads, D/8 lanes per row.
#include "pkv_common.cuh"
#include "pkv_internal.h"

namespace pkv {
namespace {

constexpr int kDecodeThreads = 256;
constexpr int kDecodeWarps = kDecodeThreads / 32;
constexpr int kDecodeUnroll = 4;

__host__ __device__ inline int64_t splits_for(int64_t Hq, int64_t T, int64_t num_sms) { return decode_splits_for(Hq, T, num_sms); }

struct DecodeParams {
    const uint16_t *q, *k_new, *v_new;   // q [num_seqs][Hq][D], k_new / v_new [num_seqs][Hkv][D]
    uint16_t *k_cache, *v_cache, *out;   // caches at + s*cache_sb + h*cache_sh; out [num_seqs][Hq][D]
    int64_t cache_sh, cache_sb, T, chunk, max_rows;
    int G, nsplit, num_sms;
    int Hq;     // query heads per sequence (the grouped kernel's split rule; the per-head kernel reads gridDim.y)
    float scale;
    float* ws;  // [num_seqs*Hq][nsplit][2 + D] partial (m, l, acc) when nsplit > 1
    const int32_t* step_dev;  // DEVLEN kernels: rows = T + *step_dev (graph-replayable decode; the grid is sized for the maximum)
    const int32_t* rows;      // DEVLEN kernels: + rows[s*Hq + h] (rows of each sequence and head: joined prompts, AdaKV / HeadKV)
};

template <typename T>
__device__ __forceinline__ void unpack8(const uint4& v, float (&f)[8]) {
    const uint32_t u[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
    for (int e = 0; e < 4; ++e) {
        f[2 * e] = DT<T>::to_f32(uint16_t(u[e] & 0xffffu));
        f[2 * e + 1] = DT<T>::to_f32(uint16_t(u[e] >> 16));
    }
}

// DEVLEN = false: the row count is the launch parameter p.T. DEVLEN = true: p.T is the row count at step 0 and the
// current step is read from device memory, so that ONE captured launch (CUDA graph) serves every decode step; the grid
// is sized for the cache capacity, and the rows are divided in-kernel among the splits a host launch for the current row
// count would use (the others stay empty), so both forms add the same terms in the same order: the same output bits.
// The split count comes from the per-sequence head count gridDim.y, so a sequence gets the same bits in a batch as alone.
// A row count outside [1, max_rows] (the capacity the launch was checked against) is treated as 0: nothing is read or
// written but the output, which becomes NaN.
template <typename T, int D, bool DEVLEN>
__global__ void __launch_bounds__(kDecodeThreads) decode_kernel(const DecodeParams p) {
    constexpr int LPR = D / 8;     // lanes per cached row
    constexpr int RPW = 32 / LPR;  // rows per warp step
    __shared__ float s_m[kDecodeWarps], s_l[kDecodeWarps];
    __shared__ float s_acc[kDecodeWarps][D];

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int split = blockIdx.x, h = blockIdx.y, g = h / p.G;
    const int64_t sh = int64_t(blockIdx.z) * gridDim.y + h;            // (sequence, head) index
    const int64_t sg = int64_t(blockIdx.z) * (gridDim.y / p.G) + g;    // (sequence, kv head) index
    const int sub = lane / LPR, piece = lane % LPR;
    uint16_t* kc = p.k_cache + int64_t(blockIdx.z) * p.cache_sb + int64_t(h) * p.cache_sh;
    uint16_t* vc = p.v_cache + int64_t(blockIdx.z) * p.cache_sb + int64_t(h) * p.cache_sh;
    const uint16_t* k_new = p.k_new + sg * D;
    const uint16_t* v_new = p.v_new + sg * D;
    int64_t rows = p.T, chunk = p.chunk;
    if constexpr (DEVLEN) {
        if (p.step_dev) rows += int64_t(__ldg(p.step_dev));
        if (p.rows) rows += int64_t(__ldg(p.rows + sh));
        if (rows < 1 || rows > p.max_rows) rows = 0;
        const int64_t ns = min(int64_t(p.nsplit), splits_for(gridDim.y, rows, p.num_sms));
        chunk = (rows + ns - 1) / ns;
    }
    const int64_t r_begin = int64_t(split) * chunk;
    const int64_t r_end = min(rows, r_begin + chunk);   // may be <= r_begin (empty split): the partial is (-inf, 0, 0)
    const bool has_new = p.k_new != nullptr;
    const int64_t new_row = rows - 1;

    // fused append: the CTA that owns the last row stores the new token's K/V (this head's copy)
    if (has_new && new_row >= r_begin && new_row < r_end && warp == 0 && lane < LPR) {
        *reinterpret_cast<uint4*>(kc + new_row * D + lane * 8) = *reinterpret_cast<const uint4*>(k_new + lane * 8);
        *reinterpret_cast<uint4*>(vc + new_row * D + lane * 8) = *reinterpret_cast<const uint4*>(v_new + lane * 8);
    }

    float qf[8];
    unpack8<T>(*reinterpret_cast<const uint4*>(p.q + sh * D + piece * 8), qf);

    float m = -INFINITY, l = 0.f, acc[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) acc[e] = 0.f;

    // warp-uniform trip count (the shuffles below need every lane); rows are checked per lane group
    for (int64_t rb = r_begin + warp * RPW; rb < r_end; rb += int64_t(kDecodeWarps) * RPW * kDecodeUnroll) {
        uint4 kv[kDecodeUnroll], vv[kDecodeUnroll];
        bool ok[kDecodeUnroll];
#pragma unroll
        for (int u = 0; u < kDecodeUnroll; ++u) {
            const int64_t r = rb + sub + int64_t(u) * kDecodeWarps * RPW;
            kv[u] = make_uint4(0, 0, 0, 0);
            vv[u] = make_uint4(0, 0, 0, 0);
            ok[u] = r < r_end;
            if (ok[u]) {
                const bool is_new = has_new && r == new_row;   // read the appended row from its source
                const uint16_t* kr = is_new ? k_new : kc + r * D;
                const uint16_t* vr = is_new ? v_new : vc + r * D;
                kv[u] = *reinterpret_cast<const uint4*>(kr + piece * 8);
                vv[u] = *reinterpret_cast<const uint4*>(vr + piece * 8);
            }
        }
#pragma unroll
        for (int u = 0; u < kDecodeUnroll; ++u) {
            float kf[8], vf[8];
            unpack8<T>(kv[u], kf);
            unpack8<T>(vv[u], vf);
            float dot = 0.f;
#pragma unroll
            for (int e = 0; e < 8; ++e) dot = fmaf(qf[e], kf[e], dot);
#pragma unroll
            for (int o = 1; o < LPR; o <<= 1) dot += __shfl_xor_sync(0xffffffffu, dot, o);
            if (ok[u]) {   // uniform within the LPR-lane row group
                const float s = dot * p.scale;
                const float mn = fmaxf(m, s);
                const float corr = expf(m - mn), pe = expf(s - mn);
                l = l * corr + pe;
#pragma unroll
                for (int e = 0; e < 8; ++e) acc[e] = acc[e] * corr + pe * vf[e];
                m = mn;
            }
        }
    }

    // merge the RPW row groups of the warp (same dims, different rows)
#pragma unroll
    for (int o = LPR; o < 32; o <<= 1) {
        const float m2 = __shfl_xor_sync(0xffffffffu, m, o);
        const float l2 = __shfl_xor_sync(0xffffffffu, l, o);
        const float mn = fmaxf(m, m2);
        const float c1 = (mn == -INFINITY) ? 0.f : expf(m - mn), c2 = (mn == -INFINITY) ? 0.f : expf(m2 - mn);
        l = l * c1 + l2 * c2;
#pragma unroll
        for (int e = 0; e < 8; ++e) {
            const float a2 = __shfl_xor_sync(0xffffffffu, acc[e], o);
            acc[e] = acc[e] * c1 + a2 * c2;
        }
        m = mn;
    }
    if (sub == 0) {
        if (piece == 0) { s_m[warp] = m; s_l[warp] = l; }
#pragma unroll
        for (int e = 0; e < 8; ++e) s_acc[warp][piece * 8 + e] = acc[e];
    }
    __syncthreads();
    if (tid < D) {
        float mn = -INFINITY;
#pragma unroll
        for (int w = 0; w < kDecodeWarps; ++w) mn = fmaxf(mn, s_m[w]);
        float lt = 0.f, at = 0.f;
#pragma unroll
        for (int w = 0; w < kDecodeWarps; ++w) {
            const float c = (s_m[w] == -INFINITY) ? 0.f : expf(s_m[w] - mn);
            lt += s_l[w] * c;
            at += s_acc[w][tid] * c;
        }
        if (p.nsplit == 1) {
            p.out[sh * D + tid] = DT<T>::from_f32(at / lt);
        } else {
            float* w = p.ws + (sh * p.nsplit + split) * (2 + D);
            if (tid == 0) { w[0] = mn; w[1] = lt; }
            w[2 + tid] = at;
        }
    }
}

// decode_kernel<T, D, true> over a GQA-shared cache ([num_seqs][Hkv][capacity][D], rows[s*Hkv + j]): the CTA of (split, KV
// head j, sequence) loads every row of its split once and runs, for each of the GH query heads h0..h0+GH-1 of the group, the
// arithmetic decode_kernel runs for that head on the repeat-interleaved cache - the same rows per warp and lane group, the same
// dot-product and online-softmax order, the same merges - so each head's output is bit-identical to it. The split count is
// the per-query-head kernel's for Hq heads, and the partials are written per query head for decode_combine_kernel.
// GH < G: the group is covered by G / GH CTAs (blockIdx.y = j * (G / GH) + part); part 0 appends the new row.
template <typename T, int D, int GH>
__global__ void __launch_bounds__(kDecodeThreads) decode_gqa_kernel(const DecodeParams p) {
    constexpr int LPR = D / 8;
    constexpr int RPW = 32 / LPR;
    __shared__ float s_m[GH][kDecodeWarps], s_l[GH][kDecodeWarps];
    __shared__ float s_acc[GH][kDecodeWarps][D];

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int parts = p.G / GH, split = blockIdx.x, j = blockIdx.y / parts, part = blockIdx.y % parts;
    const int Hkv = p.Hq / p.G;
    const int64_t sg = int64_t(blockIdx.z) * Hkv + j;                          // (sequence, kv head) index
    const int64_t sh0 = int64_t(blockIdx.z) * p.Hq + int64_t(j) * p.G + part * GH;   // (sequence, first query head) index
    const int sub = lane / LPR, piece = lane % LPR;
    uint16_t* kc = p.k_cache + int64_t(blockIdx.z) * p.cache_sb + int64_t(j) * p.cache_sh;
    uint16_t* vc = p.v_cache + int64_t(blockIdx.z) * p.cache_sb + int64_t(j) * p.cache_sh;
    const uint16_t* k_new = p.k_new + sg * D;
    const uint16_t* v_new = p.v_new + sg * D;
    int64_t rows = p.T;
    if (p.step_dev) rows += int64_t(__ldg(p.step_dev));
    if (p.rows) rows += int64_t(__ldg(p.rows + sg));
    if (rows < 1 || rows > p.max_rows) rows = 0;
    const int64_t ns = min(int64_t(p.nsplit), splits_for(p.Hq, rows, p.num_sms));
    const int64_t chunk = (rows + ns - 1) / ns;
    const int64_t r_begin = int64_t(split) * chunk;
    const int64_t r_end = min(rows, r_begin + chunk);
    const bool has_new = p.k_new != nullptr;
    const int64_t new_row = rows - 1;

    // fused append, once per KV head
    if (has_new && part == 0 && new_row >= r_begin && new_row < r_end && warp == 0 && lane < LPR) {
        *reinterpret_cast<uint4*>(kc + new_row * D + lane * 8) = *reinterpret_cast<const uint4*>(k_new + lane * 8);
        *reinterpret_cast<uint4*>(vc + new_row * D + lane * 8) = *reinterpret_cast<const uint4*>(v_new + lane * 8);
    }

    float qf[GH][8], m[GH], l[GH], acc[GH][8];
#pragma unroll
    for (int i = 0; i < GH; ++i) {
        unpack8<T>(*reinterpret_cast<const uint4*>(p.q + (sh0 + i) * D + piece * 8), qf[i]);
        m[i] = -INFINITY;
        l[i] = 0.f;
#pragma unroll
        for (int e = 0; e < 8; ++e) acc[i][e] = 0.f;
    }

    for (int64_t rb = r_begin + warp * RPW; rb < r_end; rb += int64_t(kDecodeWarps) * RPW * kDecodeUnroll) {
        uint4 kv[kDecodeUnroll], vv[kDecodeUnroll];
        bool ok[kDecodeUnroll];
#pragma unroll
        for (int u = 0; u < kDecodeUnroll; ++u) {
            const int64_t r = rb + sub + int64_t(u) * kDecodeWarps * RPW;
            kv[u] = make_uint4(0, 0, 0, 0);
            vv[u] = make_uint4(0, 0, 0, 0);
            ok[u] = r < r_end;
            if (ok[u]) {
                const bool is_new = has_new && r == new_row;
                const uint16_t* kr = is_new ? k_new : kc + r * D;
                const uint16_t* vr = is_new ? v_new : vc + r * D;
                kv[u] = *reinterpret_cast<const uint4*>(kr + piece * 8);
                vv[u] = *reinterpret_cast<const uint4*>(vr + piece * 8);
            }
        }
#pragma unroll
        for (int u = 0; u < kDecodeUnroll; ++u) {
            float kf[8], vf[8];
            unpack8<T>(kv[u], kf);
            unpack8<T>(vv[u], vf);
#pragma unroll
            for (int i = 0; i < GH; ++i) {
                float dot = 0.f;
#pragma unroll
                for (int e = 0; e < 8; ++e) dot = fmaf(qf[i][e], kf[e], dot);
#pragma unroll
                for (int o = 1; o < LPR; o <<= 1) dot += __shfl_xor_sync(0xffffffffu, dot, o);
                if (ok[u]) {
                    // Explicit roundings: the forms the compiler picks for decode_kernel (with the G heads unrolled it may
                    // contract a*b + c*d around the other product, or fuse dot * scale into s - mn), so the bits match it.
                    const float s = __fmul_rn(dot, p.scale);
                    const float mn = fmaxf(m[i], s);
                    const float corr = expf(m[i] - mn), pe = expf(s - mn);
                    l[i] = __fmaf_rn(l[i], corr, pe);
#pragma unroll
                    for (int e = 0; e < 8; ++e) acc[i][e] = __fmaf_rn(acc[i][e], corr, __fmul_rn(pe, vf[e]));
                    m[i] = mn;
                }
            }
        }
    }

#pragma unroll
    for (int i = 0; i < GH; ++i) {
#pragma unroll
        for (int o = LPR; o < 32; o <<= 1) {
            const float m2 = __shfl_xor_sync(0xffffffffu, m[i], o);
            const float l2 = __shfl_xor_sync(0xffffffffu, l[i], o);
            const float mn = fmaxf(m[i], m2);
            const float c1 = (mn == -INFINITY) ? 0.f : expf(m[i] - mn), c2 = (mn == -INFINITY) ? 0.f : expf(m2 - mn);
            l[i] = __fmaf_rn(l[i], c1, __fmul_rn(l2, c2));
#pragma unroll
            for (int e = 0; e < 8; ++e) {
                const float a2 = __shfl_xor_sync(0xffffffffu, acc[i][e], o);
                acc[i][e] = __fmaf_rn(acc[i][e], c1, __fmul_rn(a2, c2));
            }
            m[i] = mn;
        }
        if (sub == 0) {
            if (piece == 0) { s_m[i][warp] = m[i]; s_l[i][warp] = l[i]; }
#pragma unroll
            for (int e = 0; e < 8; ++e) s_acc[i][warp][piece * 8 + e] = acc[i][e];
        }
    }
    __syncthreads();
    for (int x = tid; x < GH * D; x += kDecodeThreads) {
        const int i = x / D, d = x % D;
        float mn = -INFINITY;
#pragma unroll
        for (int w = 0; w < kDecodeWarps; ++w) mn = fmaxf(mn, s_m[i][w]);
        float lt = 0.f, at = 0.f;
#pragma unroll
        for (int w = 0; w < kDecodeWarps; ++w) {
            const float c = (s_m[i][w] == -INFINITY) ? 0.f : expf(s_m[i][w] - mn);
            lt += s_l[i][w] * c;
            at += s_acc[i][w][d] * c;
        }
        if (p.nsplit == 1) {
            p.out[(sh0 + i) * D + d] = DT<T>::from_f32(at / lt);
        } else {
            float* w = p.ws + ((sh0 + i) * p.nsplit + split) * (2 + D);
            if (d == 0) { w[0] = mn; w[1] = lt; }
            w[2 + d] = at;
        }
    }
}

template <typename T, int D>
__global__ void decode_combine_kernel(const DecodeParams p) {   // one CTA per (sequence, head)
    const int64_t h = blockIdx.x;
    const int d = threadIdx.x;
    const float* w = p.ws + int64_t(h) * p.nsplit * (2 + D);
    float mn = -INFINITY;
    for (int s = 0; s < p.nsplit; ++s) mn = fmaxf(mn, w[s * (2 + D)]);
    float lt = 0.f, at = 0.f;
    for (int s = 0; s < p.nsplit; ++s) {
        const float ms = w[s * (2 + D)];
        const float c = (ms == -INFINITY) ? 0.f : expf(ms - mn);
        lt += w[s * (2 + D) + 1] * c;
        at += w[s * (2 + D) + 2 + d] * c;
    }
    p.out[h * D + d] = DT<T>::from_f32(at / lt);
}

template <int D>
__global__ void append_kernel(const DecodeParams p) {  // (host-length only; the graph path appends inside decode_kernel)
    constexpr int LPR = D / 8;
    const int h = blockIdx.x, g = h / p.G, lane = threadIdx.x;
    if (lane >= 2 * LPR) return;
    const bool is_v = lane >= LPR;
    const int piece = lane % LPR;
    const uint16_t* src = (is_v ? p.v_new : p.k_new) + int64_t(g) * D + piece * 8;
    uint16_t* dst = (is_v ? p.v_cache : p.k_cache) + int64_t(h) * p.cache_sh + (p.T - 1) * D + piece * 8;
    *reinterpret_cast<uint4*>(dst) = *reinterpret_cast<const uint4*>(src);
}

DecodeParams make_params(const DecodeArgs& a) {
    DecodeParams p;
    p.q = a.q; p.k_new = a.k_new; p.v_new = a.v_new;
    p.k_cache = a.k_cache; p.v_cache = a.v_cache; p.out = a.out;
    p.cache_sh = a.cache_sh; p.cache_sb = a.cache_sb; p.T = a.T; p.max_rows = a.max_rows;
    p.G = a.G; p.nsplit = a.nsplit; p.num_sms = a.num_sms;
    p.Hq = a.Hq;
    p.chunk = (a.T + a.nsplit - 1) / a.nsplit;
    p.scale = a.scale;
    p.ws = a.ws;
    p.step_dev = a.step_dev;
    p.rows = a.rows;
    return p;
}

template <typename T, int D>
cudaError_t launch_decode_t(const DecodeArgs& a, cudaStream_t st) {
    const DecodeParams p = make_params(a);
    const dim3 grid(unsigned(a.nsplit), unsigned(a.Hq), unsigned(a.num_seqs));
    if (a.devlen) decode_kernel<T, D, true><<<grid, kDecodeThreads, 0, st>>>(p);
    else decode_kernel<T, D, false><<<grid, kDecodeThreads, 0, st>>>(p);
    count_launch();
    if (a.nsplit > 1) {
        decode_combine_kernel<T, D><<<unsigned(int64_t(a.num_seqs) * a.Hq), D, 0, st>>>(p);
        count_launch();
    }
    return cudaGetLastError();
}

template <typename T, int D>
cudaError_t launch_decode_gqa_t(const DecodeArgs& a, cudaStream_t st) {
    const DecodeParams p = make_params(a);
    const dim3 grid(unsigned(a.nsplit), unsigned(a.Hkv), unsigned(a.num_seqs));
    if (a.G == 2) decode_gqa_kernel<T, D, 2><<<grid, kDecodeThreads, 0, st>>>(p);
    else if (a.G == 4) decode_gqa_kernel<T, D, 4><<<grid, kDecodeThreads, 0, st>>>(p);
    else decode_gqa_kernel<T, D, 8><<<grid, kDecodeThreads, 0, st>>>(p);
    count_launch();
    const cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess || a.nsplit == 1) return e;
    return launch_decode_combine(a, st);
}

}  // namespace

cudaError_t launch_decode_gqa(const DecodeArgs& a, cudaStream_t st) {
    if (a.dtype == PKV_BF16) return a.D == 128 ? launch_decode_gqa_t<__nv_bfloat16, 128>(a, st) : launch_decode_gqa_t<__nv_bfloat16, 64>(a, st);
    return a.D == 128 ? launch_decode_gqa_t<__half, 128>(a, st) : launch_decode_gqa_t<__half, 64>(a, st);
}

int decode_num_splits(int Hq, int64_t T, int num_sms) { return int(splits_for(Hq, T, num_sms)); }

cudaError_t launch_decode(const DecodeArgs& a, cudaStream_t st) {
    if (a.dtype == PKV_BF16) return a.D == 128 ? launch_decode_t<__nv_bfloat16, 128>(a, st) : launch_decode_t<__nv_bfloat16, 64>(a, st);
    return a.D == 128 ? launch_decode_t<__half, 128>(a, st) : launch_decode_t<__half, 64>(a, st);
}

cudaError_t launch_decode_combine(const DecodeArgs& a, cudaStream_t st) {
    const DecodeParams p = make_params(a);
    const unsigned grid = unsigned(int64_t(a.num_seqs) * a.Hq);
    if (a.dtype == PKV_BF16) {
        if (a.D == 128) decode_combine_kernel<__nv_bfloat16, 128><<<grid, 128, 0, st>>>(p);
        else decode_combine_kernel<__nv_bfloat16, 64><<<grid, 64, 0, st>>>(p);
    } else {
        if (a.D == 128) decode_combine_kernel<__half, 128><<<grid, 128, 0, st>>>(p);
        else decode_combine_kernel<__half, 64><<<grid, 64, 0, st>>>(p);
    }
    count_launch();
    return cudaGetLastError();
}

cudaError_t launch_append(const DecodeArgs& a, cudaStream_t st) {
    const DecodeParams p = make_params(a);
    if (a.D == 128) append_kernel<128><<<unsigned(a.Hq), 32, 0, st>>>(p);
    else append_kernel<64><<<unsigned(a.Hq), 32, 0, st>>>(p);
    count_launch();
    return cudaGetLastError();
}

}  // namespace pkv
