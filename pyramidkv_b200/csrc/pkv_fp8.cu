// pkv_fp8.cu — the opt-in FP8 (E4M3) compacted cache: the conversion of the 16-bit cache the eviction wrote, and the decode
// step over FP8 rows (in-place append of the quantised new token + attention).
//
// Format (per layer): E4M3 bytes [num_seqs, Hq, capacity, D] for K and for V, and one fp32 scale per (sequence, head, row)
// for each. A row x of D 16-bit values is stored as
//     amax = max_e |x_e| (fp32);  amax == 0: scale = 0, every byte 0;
//     else inv = rn_f32(448 / amax), q_e = e4m3_satfinite_rne(rn_f32(x_e * inv)), scale = rn_f32(amax / 448)
// and stands for x^_e = float(q_e) * scale. Each row carries its own scale, so appending a row never touches another one.
// The decode reads D bytes per row instead of 2*D: its 128-bit loads carry 16 elements (D/16 lanes per row), which
// `cvt.rn.f16x2.e4m3x2` widens exactly; the K scale multiplies the finished dot product and the V scale is folded into the
// softmax weight, so neither costs a multiply per element.
#include <algorithm>

#include <cuda_fp8.h>

#include "pkv_common.cuh"
#include "pkv_internal.h"

namespace pkv {
namespace {

constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;
constexpr int kUnroll = 4;
constexpr float kE4M3Max = 448.f;

template <typename T>
__device__ __forceinline__ void unpack8(const uint4& v, float* f) {
    const uint32_t u[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
    for (int e = 0; e < 4; ++e) {
        f[2 * e] = DT<T>::to_f32(uint16_t(u[e] & 0xffffu));
        f[2 * e + 1] = DT<T>::to_f32(uint16_t(u[e] >> 16));
    }
}

// 16 consecutive 16-bit elements (two 128-bit loads) -> fp32
template <typename T>
__device__ __forceinline__ void load16(const uint16_t* src, float (&x)[16]) {
    unpack8<T>(*reinterpret_cast<const uint4*>(src), x);
    unpack8<T>(*reinterpret_cast<const uint4*>(src + 8), x + 8);
}

// 16 E4M3 bytes (element e in byte e) -> fp32, exactly (cvt.rn.f16x2.e4m3x2, then f16 -> f32)
__device__ __forceinline__ void fp8x16_to_f32(const uint4& v, float (&f)[16]) {
    const uint32_t u[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
    for (int e = 0; e < 4; ++e) {
#pragma unroll
        for (int hlf = 0; hlf < 2; ++hlf) {
            const __half2 h2(__nv_cvt_fp8x2_to_halfraw2(__nv_fp8x2_storage_t(u[e] >> (16 * hlf)), __NV_E4M3));
            const float2 f2 = __half22float2(h2);
            f[4 * e + 2 * hlf] = f2.x;
            f[4 * e + 2 * hlf + 1] = f2.y;
        }
    }
}

// four fp32 -> four E4M3 bytes, first value in the low byte (cvt.rn.satfinite.e4m3x2.f32)
__device__ __forceinline__ uint32_t pack_fp8x4(float a, float b, float c, float d) {
    const uint32_t lo = __nv_cvt_float2_to_fp8x2(make_float2(a, b), __NV_SATFINITE, __NV_E4M3);
    const uint32_t hi = __nv_cvt_float2_to_fp8x2(make_float2(c, d), __NV_SATFINITE, __NV_E4M3);
    return lo | (hi << 16);
}

// largest |x| of a row spread over LPR consecutive lanes (every lane of the warp takes part)
template <int LPR>
__device__ __forceinline__ float row_amax(const float (&x)[16]) {
    float a = 0.f;
#pragma unroll
    for (int e = 0; e < 16; ++e) a = fmaxf(a, fabsf(x[e]));
#pragma unroll
    for (int o = 1; o < LPR; o <<= 1) a = fmaxf(a, __shfl_xor_sync(0xffffffffu, a, o));
    return a;
}

// this lane's 16 elements of a row whose amax is known -> E4M3 bytes; `scale` receives the row scale
__device__ __forceinline__ uint4 quantize16(const float (&x)[16], float amax, float& scale) {
    if (amax == 0.f) {
        scale = 0.f;
        return make_uint4(0, 0, 0, 0);
    }
    const float inv = __fdiv_rn(kE4M3Max, amax);
    uint32_t w[4];
#pragma unroll
    for (int e = 0; e < 4; ++e)
        w[e] = pack_fp8x4(__fmul_rn(x[4 * e], inv), __fmul_rn(x[4 * e + 1], inv), __fmul_rn(x[4 * e + 2], inv),
                          __fmul_rn(x[4 * e + 3], inv));
    scale = __fdiv_rn(amax, kE4M3Max);
    return make_uint4(w[0], w[1], w[2], w[3]);
}

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

// ---------------- decode step over the FP8 cache ----------------
struct Fp8DecodeParams {
    const uint16_t *q, *k_new, *v_new;   // q [num_seqs][Hq][D], k_new / v_new [num_seqs][Hkv][D]
    uint16_t* out;                       // [num_seqs][Hq][D]
    uint8_t *k_cache, *v_cache;          // at + s*cache_sb + h*cache_sh (bytes)
    float *k_scale, *v_scale;            // at + s*scale_sb + h*scale_sh
    int64_t cache_sh, cache_sb, scale_sh, scale_sb, T, max_rows;
    int G, nsplit, num_sms;
    int Hq;   // query heads per sequence (the grouped kernel's split rule)
    float scale;
    float* ws;
    const int32_t* step_dev;
    const int32_t* rows;
};

// decode_kernel<T, D, DEVLEN = true> (pkv_decode.cu) over E4M3 rows: the same row count rule, the same split rule and the
// same fp32 online softmax, so a sequence gets the same bits in a batch as alone and a graph replay equals a host launch.
// The CTA that owns row rows-1 quantises the new token (this head's kv head copy), stores its bytes and scale, and attends
// that quantised row (kept in shared memory), so the output is attention over exactly what the cache now holds.
template <typename T, int D>
__global__ void __launch_bounds__(kThreads) decode_fp8_kernel(const Fp8DecodeParams p) {
    constexpr int LPR = D / 16;    // lanes per cached row (16 elements each)
    constexpr int RPW = 32 / LPR;  // rows per warp step
    __shared__ float s_m[kWarps], s_l[kWarps];
    __shared__ float s_acc[kWarps][D];
    __shared__ uint4 s_new[2][LPR];
    __shared__ float s_new_scale[2];

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int split = blockIdx.x, h = blockIdx.y, g = h / p.G;
    const int64_t sh = int64_t(blockIdx.z) * gridDim.y + h;            // (sequence, head) index
    const int64_t sg = int64_t(blockIdx.z) * (gridDim.y / p.G) + g;    // (sequence, kv head) index
    const int sub = lane / LPR, piece = lane % LPR;
    uint8_t* kc = p.k_cache + int64_t(blockIdx.z) * p.cache_sb + int64_t(h) * p.cache_sh;
    uint8_t* vc = p.v_cache + int64_t(blockIdx.z) * p.cache_sb + int64_t(h) * p.cache_sh;
    float* ksc = p.k_scale + int64_t(blockIdx.z) * p.scale_sb + int64_t(h) * p.scale_sh;
    float* vsc = p.v_scale + int64_t(blockIdx.z) * p.scale_sb + int64_t(h) * p.scale_sh;
    int64_t rows = p.T;
    if (p.step_dev) rows += int64_t(__ldg(p.step_dev));
    if (p.rows) rows += int64_t(__ldg(p.rows + sh));
    if (rows < 1 || rows > p.max_rows) rows = 0;
    const int64_t ns = min(int64_t(p.nsplit), decode_splits_for(gridDim.y, rows, p.num_sms));
    const int64_t chunk = (rows + ns - 1) / ns;
    const int64_t r_begin = int64_t(split) * chunk;
    const int64_t r_end = min(rows, r_begin + chunk);   // may be <= r_begin (empty split): the partial is (-inf, 0, 0)
    const int64_t new_row = rows - 1;
    const bool own_new = p.k_new != nullptr && new_row >= r_begin && new_row < r_end;   // uniform over the CTA

    // fused append: warp 0 quantises the new K row (lane groups 0, 2, ...) and V row (1, 3, ...); groups 0 and 1 store them
    if (own_new && warp == 0) {
        const int which = sub & 1;
        float x[16];
        load16<T>((which ? p.v_new : p.k_new) + sg * D + piece * 16, x);
        const float amax = row_amax<LPR>(x);
        float s;
        const uint4 qv = quantize16(x, amax, s);
        if (sub < 2) {
            *reinterpret_cast<uint4*>((which ? vc : kc) + new_row * D + piece * 16) = qv;
            s_new[which][piece] = qv;
            if (piece == 0) {
                (which ? vsc : ksc)[new_row] = s;
                s_new_scale[which] = s;
            }
        }
    }
    __syncthreads();

    float qf[16];
    load16<T>(p.q + sh * D + piece * 16, qf);

    float m = -INFINITY, l = 0.f, acc[16];
#pragma unroll
    for (int e = 0; e < 16; ++e) acc[e] = 0.f;

    // warp-uniform trip count (the shuffles below need every lane); rows are checked per lane group
    for (int64_t rb = r_begin + warp * RPW; rb < r_end; rb += int64_t(kWarps) * RPW * kUnroll) {
        uint4 kv[kUnroll], vv[kUnroll];
        float ks[kUnroll], vs[kUnroll];
        bool ok[kUnroll];
#pragma unroll
        for (int u = 0; u < kUnroll; ++u) {
            const int64_t r = rb + sub + int64_t(u) * kWarps * RPW;
            kv[u] = make_uint4(0, 0, 0, 0);
            vv[u] = make_uint4(0, 0, 0, 0);
            ks[u] = vs[u] = 0.f;
            ok[u] = r < r_end;
            if (ok[u]) {
                if (own_new && r == new_row) {   // the appended row: from shared memory, as stored
                    kv[u] = s_new[0][piece];
                    vv[u] = s_new[1][piece];
                    ks[u] = s_new_scale[0];
                    vs[u] = s_new_scale[1];
                } else {
                    kv[u] = *reinterpret_cast<const uint4*>(kc + r * D + piece * 16);
                    vv[u] = *reinterpret_cast<const uint4*>(vc + r * D + piece * 16);
                    ks[u] = ksc[r];
                    vs[u] = vsc[r];
                }
            }
        }
#pragma unroll
        for (int u = 0; u < kUnroll; ++u) {
            float kf[16];
            fp8x16_to_f32(kv[u], kf);
            float dot = 0.f;
#pragma unroll
            for (int e = 0; e < 16; ++e) dot = fmaf(qf[e], kf[e], dot);
#pragma unroll
            for (int o = 1; o < LPR; o <<= 1) dot += __shfl_xor_sync(0xffffffffu, dot, o);
            if (ok[u]) {   // uniform within the LPR-lane row group
                const float s = dot * ks[u] * p.scale;
                const float mn = fmaxf(m, s);
                const float corr = expf(m - mn), pe = expf(s - mn);
                l = l * corr + pe;
                const float pv = pe * vs[u];
                float vf[16];
                fp8x16_to_f32(vv[u], vf);
#pragma unroll
                for (int e = 0; e < 16; ++e) acc[e] = acc[e] * corr + pv * vf[e];
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
        for (int e = 0; e < 16; ++e) {
            const float a2 = __shfl_xor_sync(0xffffffffu, acc[e], o);
            acc[e] = acc[e] * c1 + a2 * c2;
        }
        m = mn;
    }
    if (sub == 0) {
        if (piece == 0) { s_m[warp] = m; s_l[warp] = l; }
#pragma unroll
        for (int e = 0; e < 16; ++e) s_acc[warp][piece * 16 + e] = acc[e];
    }
    __syncthreads();
    if (tid < D) {
        float mn = -INFINITY;
#pragma unroll
        for (int w = 0; w < kWarps; ++w) mn = fmaxf(mn, s_m[w]);
        float lt = 0.f, at = 0.f;
#pragma unroll
        for (int w = 0; w < kWarps; ++w) {
            const float c = (s_m[w] == -INFINITY) ? 0.f : expf(s_m[w] - mn);
            lt += s_l[w] * c;
            at += s_acc[w][tid] * c;
        }
        if (p.nsplit == 1) {
            p.out[sh * D + tid] = DT<T>::from_f32(at / lt);
        } else {
            float* w = p.ws + (sh * p.nsplit + split) * (2 + D);   // the layout decode_combine_kernel merges
            if (tid == 0) { w[0] = mn; w[1] = lt; }
            w[2 + tid] = at;
        }
    }
}

// decode_fp8_kernel over a GQA-shared FP8 cache ([num_seqs][Hkv][capacity][D] bytes, [num_seqs][Hkv][capacity] scales, rows
// [s*Hkv + j]): the CTA of (split, KV head j, sequence) loads every row of its split once and runs, for each of the GH query
// heads of the group it covers, the arithmetic decode_fp8_kernel runs for that head on the repeat-interleaved cache, so each
// head's output is bit-identical to it. GH < G (G = 8: GH = 4, the registers of eight heads do not fit): G / GH CTAs per group,
// blockIdx.y = j * (G / GH) + part. Every part quantises the new row into shared memory; part 0 stores it.
template <typename T, int D, int GH>
__global__ void __launch_bounds__(kThreads) decode_gqa_fp8_kernel(const Fp8DecodeParams p) {
    constexpr int LPR = D / 16;
    constexpr int RPW = 32 / LPR;
    __shared__ float s_m[GH][kWarps], s_l[GH][kWarps];
    __shared__ float s_acc[GH][kWarps][D];
    __shared__ uint4 s_new[2][LPR];
    __shared__ float s_new_scale[2];

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int parts = p.G / GH, split = blockIdx.x, j = blockIdx.y / parts, part = blockIdx.y % parts;
    const int Hkv = p.Hq / p.G;
    const int64_t sg = int64_t(blockIdx.z) * Hkv + j;
    const int64_t sh0 = int64_t(blockIdx.z) * p.Hq + int64_t(j) * p.G + part * GH;
    const int sub = lane / LPR, piece = lane % LPR;
    uint8_t* kc = p.k_cache + int64_t(blockIdx.z) * p.cache_sb + int64_t(j) * p.cache_sh;
    uint8_t* vc = p.v_cache + int64_t(blockIdx.z) * p.cache_sb + int64_t(j) * p.cache_sh;
    float* ksc = p.k_scale + int64_t(blockIdx.z) * p.scale_sb + int64_t(j) * p.scale_sh;
    float* vsc = p.v_scale + int64_t(blockIdx.z) * p.scale_sb + int64_t(j) * p.scale_sh;
    int64_t rows = p.T;
    if (p.step_dev) rows += int64_t(__ldg(p.step_dev));
    if (p.rows) rows += int64_t(__ldg(p.rows + sg));
    if (rows < 1 || rows > p.max_rows) rows = 0;
    const int64_t ns = min(int64_t(p.nsplit), decode_splits_for(p.Hq, rows, p.num_sms));
    const int64_t chunk = (rows + ns - 1) / ns;
    const int64_t r_begin = int64_t(split) * chunk;
    const int64_t r_end = min(rows, r_begin + chunk);
    const int64_t new_row = rows - 1;
    const bool own_new = p.k_new != nullptr && new_row >= r_begin && new_row < r_end;

    if (own_new && warp == 0) {
        const int which = sub & 1;
        float x[16];
        load16<T>((which ? p.v_new : p.k_new) + sg * D + piece * 16, x);
        const float amax = row_amax<LPR>(x);
        float s;
        const uint4 qv = quantize16(x, amax, s);
        if (sub < 2) {
            if (part == 0) *reinterpret_cast<uint4*>((which ? vc : kc) + new_row * D + piece * 16) = qv;
            s_new[which][piece] = qv;
            if (piece == 0) {
                if (part == 0) (which ? vsc : ksc)[new_row] = s;
                s_new_scale[which] = s;
            }
        }
    }
    __syncthreads();

    float qf[GH][16], m[GH], l[GH], acc[GH][16];
#pragma unroll
    for (int i = 0; i < GH; ++i) {
        load16<T>(p.q + (sh0 + i) * D + piece * 16, qf[i]);
        m[i] = -INFINITY;
        l[i] = 0.f;
#pragma unroll
        for (int e = 0; e < 16; ++e) acc[i][e] = 0.f;
    }

    for (int64_t rb = r_begin + warp * RPW; rb < r_end; rb += int64_t(kWarps) * RPW * kUnroll) {
        uint4 kv[kUnroll], vv[kUnroll];
        float ks[kUnroll], vs[kUnroll];
        bool ok[kUnroll];
#pragma unroll
        for (int u = 0; u < kUnroll; ++u) {
            const int64_t r = rb + sub + int64_t(u) * kWarps * RPW;
            kv[u] = make_uint4(0, 0, 0, 0);
            vv[u] = make_uint4(0, 0, 0, 0);
            ks[u] = vs[u] = 0.f;
            ok[u] = r < r_end;
            if (ok[u]) {
                if (own_new && r == new_row) {
                    kv[u] = s_new[0][piece];
                    vv[u] = s_new[1][piece];
                    ks[u] = s_new_scale[0];
                    vs[u] = s_new_scale[1];
                } else {
                    kv[u] = *reinterpret_cast<const uint4*>(kc + r * D + piece * 16);
                    vv[u] = *reinterpret_cast<const uint4*>(vc + r * D + piece * 16);
                    ks[u] = ksc[r];
                    vs[u] = vsc[r];
                }
            }
        }
#pragma unroll
        for (int u = 0; u < kUnroll; ++u) {
            float kf[16];
            fp8x16_to_f32(kv[u], kf);
            float vf[16];
            fp8x16_to_f32(vv[u], vf);
#pragma unroll
            for (int i = 0; i < GH; ++i) {
                float dot = 0.f;
#pragma unroll
                for (int e = 0; e < 16; ++e) dot = fmaf(qf[i][e], kf[e], dot);
#pragma unroll
                for (int o = 1; o < LPR; o <<= 1) dot += __shfl_xor_sync(0xffffffffu, dot, o);
                if (ok[u]) {
                    const float s = dot * ks[u] * p.scale;
                    const float mn = fmaxf(m[i], s);
                    const float corr = expf(m[i] - mn), pe = expf(s - mn);
                    l[i] = l[i] * corr + pe;
                    const float pv = pe * vs[u];
#pragma unroll
                    for (int e = 0; e < 16; ++e) acc[i][e] = acc[i][e] * corr + pv * vf[e];
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
            // explicit roundings: the contraction the compiler picks in decode_fp8_kernel (with the heads unrolled it may
            // contract l * c1 + l2 * c2 around the other product), so the bits match it
            l[i] = __fmaf_rn(l[i], c1, __fmul_rn(l2, c2));
#pragma unroll
            for (int e = 0; e < 16; ++e) {
                const float a2 = __shfl_xor_sync(0xffffffffu, acc[i][e], o);
                acc[i][e] = __fmaf_rn(acc[i][e], c1, __fmul_rn(a2, c2));
            }
            m[i] = mn;
        }
        if (sub == 0) {
            if (piece == 0) { s_m[i][warp] = m[i]; s_l[i][warp] = l[i]; }
#pragma unroll
            for (int e = 0; e < 16; ++e) s_acc[i][warp][piece * 16 + e] = acc[i][e];
        }
    }
    __syncthreads();
    for (int x = tid; x < GH * D; x += kThreads) {
        const int i = x / D, d = x % D;
        float mn = -INFINITY;
#pragma unroll
        for (int w = 0; w < kWarps; ++w) mn = fmaxf(mn, s_m[i][w]);
        float lt = 0.f, at = 0.f;
#pragma unroll
        for (int w = 0; w < kWarps; ++w) {
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
cudaError_t launch_decode_fp8_t(const DecodeArgs& a, cudaStream_t st) {
    Fp8DecodeParams p;
    p.q = a.q; p.k_new = a.k_new; p.v_new = a.v_new; p.out = a.out;
    p.k_cache = reinterpret_cast<uint8_t*>(a.k_cache); p.v_cache = reinterpret_cast<uint8_t*>(a.v_cache);
    p.k_scale = a.k_scale; p.v_scale = a.v_scale;
    p.cache_sh = a.cache_sh; p.cache_sb = a.cache_sb; p.scale_sh = a.scale_sh; p.scale_sb = a.scale_sb;
    p.T = a.T; p.max_rows = a.max_rows;
    p.G = a.G; p.nsplit = a.nsplit; p.num_sms = a.num_sms;
    p.Hq = a.Hq;
    p.scale = a.scale;
    p.ws = a.ws;
    p.step_dev = a.step_dev;
    p.rows = a.rows;
    if (a.gqa) {
        const unsigned parts = a.G > 4 ? unsigned(a.G / 4) : 1u;
        const dim3 grid(unsigned(a.nsplit), unsigned(a.Hkv) * parts, unsigned(a.num_seqs));
        if (a.G == 2) decode_gqa_fp8_kernel<T, D, 2><<<grid, kThreads, 0, st>>>(p);
        else decode_gqa_fp8_kernel<T, D, 4><<<grid, kThreads, 0, st>>>(p);
    } else {
        const dim3 grid(unsigned(a.nsplit), unsigned(a.Hq), unsigned(a.num_seqs));
        decode_fp8_kernel<T, D><<<grid, kThreads, 0, st>>>(p);
    }
    count_launch();
    if (a.nsplit > 1) {
        const cudaError_t e = cudaGetLastError();
        if (e != cudaSuccess) return e;
        return launch_decode_combine(a, st);
    }
    return cudaGetLastError();
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

cudaError_t launch_decode_fp8(const DecodeArgs& a, cudaStream_t st) {
    if (a.dtype == PKV_BF16) return a.D == 128 ? launch_decode_fp8_t<__nv_bfloat16, 128>(a, st) : launch_decode_fp8_t<__nv_bfloat16, 64>(a, st);
    return a.D == 128 ? launch_decode_fp8_t<__half, 128>(a, st) : launch_decode_fp8_t<__half, 64>(a, st);
}

cudaError_t launch_decode_gqa_fp8(const DecodeArgs& a, cudaStream_t st) {
    DecodeArgs g = a;
    g.gqa = true;
    return launch_decode_fp8(g, st);
}

cudaError_t launch_quantize_fp8(const QuantArgs& a, int num_sms, cudaStream_t st) {
    if (a.dtype == PKV_BF16) return a.D == 128 ? launch_quantize_t<__nv_bfloat16, 128>(a, num_sms, st) : launch_quantize_t<__nv_bfloat16, 64>(a, num_sms, st);
    return a.D == 128 ? launch_quantize_t<__half, 128>(a, num_sms, st) : launch_quantize_t<__half, 64>(a, num_sms, st);
}

}  // namespace pkv
