// pkv_rowsel.cuh — block-wide selection over one row of 16-bit logits, one CTA of kThreads per row. Shared by the sampling
// kernel (pkv_sample.cu), the log-probability kernel (pkv_logprobs.cu) and the beam candidates (pkv_beam.cu):
//   - the 16-bit order key (okey / key_bits) and per-lane replicated byte histograms walked from the top, which find the
//     n-th largest logit in two passes over the row;
//   - expf masses in 64-bit fixed point (2^-40 units), so that every sum is an integer sum, independent of the schedule;
//   - block reductions (best (value, index), sum) and the index of the n-th element of a predicate in index order;
//   - row_top: m, log Z and the row's top N in three passes.
#pragma once

#include <cmath>

#include "pkv_common.cuh"

namespace pkv {
namespace rowsel {

constexpr int kThreads = 1024;
constexpr int kWarps = kThreads / 32;
constexpr float kFixScale = 1099511627776.0f;   // 2^40: e_i in (0, 1] -> at most 2^40 units, V <= 2^24 rows sum below 2^64

// bf16 / fp16 bits -> a 16-bit key whose unsigned order is the numeric order (-0 is folded onto +0; NaN never gets here)
__device__ __forceinline__ uint32_t okey(uint32_t b) {
    if ((b & 0x7fffu) == 0) b = 0;
    return (b & 0x8000u) ? (~b & 0xffffu) : (b | 0x8000u);
}
__device__ __forceinline__ uint16_t key_bits(uint32_t k) { return uint16_t((k & 0x8000u) ? (k & 0x7fffu) : (~k & 0xffffu)); }
// the same for fp32 values (the penalized sampler, whose values are not 16-bit logits); for a bf16 logit l,
// okey32(f32(l)) == okey(bits(l)) << 16
__device__ __forceinline__ uint32_t okey32(float v) {
    uint32_t b = __float_as_uint(v);
    if ((b & 0x7fffffffu) == 0) b = 0;
    return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}
__device__ __forceinline__ float key_value32(uint32_t k) { return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k); }

__device__ __forceinline__ unsigned long long fixed_mass(float x, float m) {
    return __float2ull_rn(expf(x - m) * kFixScale);
}

// (value, index) is better: larger value, NaN above everything, then the lower index
__device__ __forceinline__ bool better_nan(float v, int i, float bv, int bi) {
    const bool n = v != v, bn = bv != bv;
    if (n != bn) return n;
    if (!n && v != bv) return v > bv;
    return i < bi;
}
__device__ __forceinline__ bool better(float v, int i, float bv, int bi) { return v > bv || (v == bv && i < bi); }

struct Shared {
    uint32_t cnt[256];
    unsigned long long mass[256];
    float rf[kWarps];
    int ri[kWarps];
    unsigned long long ru[kWarps];
    int wc[kWarps];
    int bin;
    unsigned long long above;
    unsigned long long in_bin;
    int cut;
};

// elements 4g .. 4g+3 of the row (0 past its end): one 8-byte load where the row allows it
__device__ __forceinline__ void load4(const uint16_t* lg, int g, int V, bool vec, uint32_t (&b)[4]) {
    const int i = 4 * g;
    if (vec && i + 3 < V) {
        const uint2 u = __ldg(reinterpret_cast<const uint2*>(lg) + g);
        b[0] = u.x & 0xffffu; b[1] = u.x >> 16; b[2] = u.y & 0xffffu; b[3] = u.y >> 16;
    } else {
#pragma unroll
        for (int j = 0; j < 4; ++j) b[j] = i + j < V ? __ldg(lg + i + j) : 0u;
    }
}

template <bool NaN>
__device__ __forceinline__ void block_best(Shared& S, float& v, int& i) {
#pragma unroll
    for (int o = 16; o; o >>= 1) {
        const float ov = __shfl_xor_sync(0xffffffffu, v, o);
        const int oi = __shfl_xor_sync(0xffffffffu, i, o);
        if (NaN ? better_nan(ov, oi, v, i) : better(ov, oi, v, i)) { v = ov; i = oi; }
    }
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (lane == 0) { S.rf[warp] = v; S.ri[warp] = i; }
    __syncthreads();
    v = S.rf[0]; i = S.ri[0];
    for (int w = 1; w < kWarps; ++w)
        if (NaN ? better_nan(S.rf[w], S.ri[w], v, i) : better(S.rf[w], S.ri[w], v, i)) { v = S.rf[w]; i = S.ri[w]; }
    __syncthreads();
}

__device__ __forceinline__ unsigned long long block_sum(Shared& S, unsigned long long s) {
#pragma unroll
    for (int o = 16; o; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if ((threadIdx.x & 31) == 0) S.ru[threadIdx.x >> 5] = s;
    __syncthreads();
    s = 0;
    for (int w = 0; w < kWarps; ++w) s += S.ru[w];
    __syncthreads();
    return s;
}

// Histograms are replicated per lane (bin * 32 + lane): lanes of a warp never add to the same word, whatever the logits
// (a row's 16-bit keys crowd into a few high-byte bins). reduce_hist folds the replicas into one table before a walk.
// The replicas of each bin summed into red[bin] (warp w: bins 8w .. 8w+7) and cleared. Caller synchronises before and after.
template <typename T>
__device__ __forceinline__ void reduce_hist(T* rep, T* red) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int j = 0; j < 256 / kWarps; ++j) {
        const int bin = warp * (256 / kWarps) + j;
        T v = rep[bin * 32 + lane];
        rep[bin * 32 + lane] = 0;
#pragma unroll
        for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
        if (lane == 0) red[bin] = v;
    }
}

// Warp 0 walks hist[255..0] from the top: the bin b with above(b) < target <= above(b) + hist[b] -> S.bin, S.above,
// S.in_bin = hist[b]. Bins are cleared for the next pass. Caller synchronises before and after; target <= the total.
template <typename T>
__device__ void walk_top(Shared& S, T* hist, unsigned long long target) {
    if (threadIdx.x >= 32) return;
    const int lane = threadIdx.x;
    T v[8];
    unsigned long long own = 0;
#pragma unroll
    for (int j = 0; j < 8; ++j) { v[j] = hist[255 - 8 * lane - j]; own += v[j]; }
    unsigned long long incl = own;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const unsigned long long t = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += t;
    }
    const unsigned hit = __ballot_sync(0xffffffffu, incl >= target);
    const int first = hit ? __ffs(hit) - 1 : 31;
    if (lane == first) {
        unsigned long long above = incl - own;
        int b = 255 - 8 * lane - 7;
        unsigned long long in_bin = v[7];
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            if (above + v[j] >= target) { b = 255 - 8 * lane - j; in_bin = v[j]; break; }
            above += v[j];
        }
        S.bin = b;
        S.above = above;
        S.in_bin = in_bin;
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) hist[8 * lane + j] = 0;
}

// The index of the n-th (n >= 1) element i < V with pred(i), in index order; V - 1 when fewer than n do. One ballot per
// kThreads elements, stopping at the chunk that holds it. Every thread of the block calls it and gets the same index.
template <typename Pred>
__device__ int nth_index(Shared& S, int V, long long n, Pred pred) {
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    long long left = n;
    if (tid == 0) S.cut = V - 1;
    for (int base = 0; base < V; base += kThreads) {
        const int i = base + tid;
        const bool f = i < V && pred(i);
        const unsigned bal = __ballot_sync(0xffffffffu, f);
        if (lane == 0) S.wc[warp] = __popc(bal);
        __syncthreads();
        int before = 0, total = 0;
        for (int w = 0; w < kWarps; ++w) { const int c = S.wc[w]; before += w < warp ? c : 0; total += c; }
        if (f && before + __popc(bal & ((1u << lane) - 1u)) + 1 == left) S.cut = i;
        __syncthreads();
        if (left <= total) break;
        left -= total;
    }
    return S.cut;
}

template <int MaxN>
struct Top {
    uint32_t key[MaxN];
    int idx[MaxN];
    int n;
};

// The three passes over one row of V 16-bit logits lg (every thread of the block calls it): the maximum mx, log_z =
// logf(Z) with Z = sum expf(x_i - mx) in 64-bit fixed point, and (n_top > 0, n_top <= min(MaxN, V)) the row's n_top
// largest keys with their indices in top (in no order; ties at the n_top-th key go to the lowest indices). hist is
// 256 * 32 words of shared memory. False (and log_z NaN, top empty) when the row holds a NaN or +-inf.
//   1. the maximum, whether any logit is NaN or +-inf, and (n_top > 0) a count histogram of the high byte of the key;
//   2. Z and (n_top > 0) the low-byte histogram inside the high-byte bin of the n_top-th largest key -> that key k_N,
//      how many keys lie above it and how many equal it;
//   3. (n_top > 0) every key above k_N and the lowest-index ties at k_N (when more tie than are needed, the index of the
//      last one kept comes from one ballot scan in index order, which stops at the chunk that holds it).
template <typename E, int MaxN>
__device__ bool row_top(Shared& S, Top<MaxN>& top, uint32_t* hist, const uint16_t* lg, int V, int n_top, float& mx_out,
                        float& log_z_out) {
    const int tid = threadIdx.x, lane = tid & 31;
    const bool vec = (reinterpret_cast<uintptr_t>(lg) & 7u) == 0;
    if (n_top > 0)
        for (int b = tid; b < 256 * 32; b += kThreads) hist[b] = 0;
    if (tid == 0) top.n = 0;
    __syncthreads();

    // pass 1: the maximum, the non-finite flag, the high-byte histogram
    float mx = -INFINITY;
    int bad = 0;
    for (int g = tid; 4 * g < V; g += kThreads) {
        uint32_t bb[4];
        load4(lg, g, V, vec, bb);
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            if (4 * g + j < V) {
                const float x = DT<E>::to_f32(uint16_t(bb[j]));
                bad |= !isfinite(x);
                mx = fmaxf(mx, x);
                if (n_top > 0) atomicAdd(&hist[(okey(bb[j]) >> 8) * 32 + lane], 1u);
            }
        }
    }
    int mi = 0;
    block_best<false>(S, mx, mi);
    const bool finite = !__syncthreads_or(bad);
    float log_z = NAN;
    int hb = 0;
    if (finite) {
        if (n_top > 0) {
            reduce_hist(hist, S.cnt);
            __syncthreads();
            walk_top(S, S.cnt, (unsigned long long)n_top);
            __syncthreads();
            hb = S.bin;
        }
        // pass 2: Z; the low-byte histogram inside bin hb
        unsigned long long z = 0;
        for (int g = tid; 4 * g < V; g += kThreads) {
            uint32_t bb[4];
            load4(lg, g, V, vec, bb);
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                if (4 * g + j < V) {
                    z += fixed_mass(DT<E>::to_f32(uint16_t(bb[j])), mx);
                    if (n_top > 0) {
                        const uint32_t k = okey(bb[j]);
                        if (int(k >> 8) == hb) atomicAdd(&hist[(k & 255u) * 32 + lane], 1u);
                    }
                }
            }
        }
        z = block_sum(S, z);   // >= 2^40: the maximum contributes expf(0) = 1
        log_z = logf(__ull2float_rn(z) * (1.0f / kFixScale));   // the scaling is exact: log Z in [0, log V]
    }
    if (finite && n_top > 0) {
        const int rest = n_top - int(S.above);
        __syncthreads();
        reduce_hist(hist, S.cnt);
        __syncthreads();
        walk_top(S, S.cnt, (unsigned long long)rest);
        __syncthreads();
        const uint32_t kn = (uint32_t(hb) << 8) | uint32_t(S.bin);
        const int need = rest - int(S.above);             // ties at k_N to keep, >= 1
        const int ties = int(S.in_bin);
        // pass 3: keys above k_N, and the ties at k_N up to the need-th one in index order
        const int cut = need < ties ? nth_index(S, V, need, [&](int i) { return okey(__ldg(lg + i)) == kn; }) : V - 1;
        for (int g = tid; 4 * g < V; g += kThreads) {
            uint32_t bb[4];
            load4(lg, g, V, vec, bb);
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const int i = 4 * g + j;
                if (i < V) {
                    const uint32_t k = okey(bb[j]);
                    if (k > kn || (k == kn && i <= cut)) {
                        const int s = atomicAdd(&top.n, 1);
                        if (s < MaxN) { top.key[s] = k; top.idx[s] = i; }
                    }
                }
            }
        }
        __syncthreads();
    }
    mx_out = mx;
    log_z_out = log_z;
    return finite;
}

}  // namespace rowsel
}  // namespace pkv
