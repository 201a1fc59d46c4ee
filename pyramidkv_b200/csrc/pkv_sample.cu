// pkv_sample.cu — one sampled token per row of logits (include/pkv.h: pkv_sample_tokens): temperature, top-k, top-p and a
// Gumbel-max draw keyed by Philox4x32-10, one CTA per row, in one launch for the whole batch.
//
// The CTA streams its row (bf16 / fp16, 256 KB for Llama-3's 128256 tokens; it stays in L2 between passes) several times:
//   1. argmax (torch's first-index rule, NaN largest) and, with top-k, a count histogram of the high byte of the 16-bit key;
//   2. top-k: the low-byte histogram inside the chosen high-byte bin -> the k-th largest logit l_k, kappa = f32(l_k) / T;
//   3. Z = sum of e_i = expf(x_i - m) over the kept set in 64-bit fixed point (2^-40 units: exact, order-free sums), and with
//      top-p a mass histogram of the high byte;
//   4. top-p: the low-byte mass histogram -> the largest logit lambda whose upper mass reaches ceil(top_p * Z), tau = lambda / T;
//   5. the mass above tau and the number of ties at tau; 6. (only when the ties must be cut) the index of the last kept tie;
//   7. Philox + Gumbel noise + argmax over the kept set.
// Division by T > 0 is monotone, so the order of x = f32(l) / T is the order of the logits (with ties where the division
// rounds distinct logits together): the k-th largest x is f32(l_k) / T, and both selections can walk histograms of the
// 16-bit logit keys. Every sum is an integer sum and every tie is broken by index, so the token does not depend on the
// thread schedule: a graph replay and a host launch give the same token.
#include <cmath>

#include "pkv_common.cuh"
#include "pkv_internal.h"

namespace pkv {
namespace {

constexpr int kThreads = 1024;
constexpr int kWarps = kThreads / 32;
constexpr float kFixScale = 1099511627776.0f;   // 2^40: e_i in (0, 1] -> at most 2^40 units, V <= 2^24 rows sum below 2^64

// bf16 / fp16 bits -> a 16-bit key whose unsigned order is the numeric order (-0 is folded onto +0; NaN never gets here)
__device__ __forceinline__ uint32_t okey(uint32_t b) {
    if ((b & 0x7fffu) == 0) b = 0;
    return (b & 0x8000u) ? (~b & 0xffffu) : (b | 0x8000u);
}
__device__ __forceinline__ uint16_t key_bits(uint32_t k) { return uint16_t((k & 0x8000u) ? (k & 0x7fffu) : (~k & 0xffffu)); }

// Philox4x32-10 (Salmon et al., SC'11; the Random123 reference constants)
__device__ __forceinline__ uint4 philox(uint4 c, uint32_t k0, uint32_t k1) {
#pragma unroll
    for (int r = 0; r < 10; ++r) {
        if (r) { k0 += 0x9E3779B9u; k1 += 0xBB67AE85u; }
        const uint32_t lo0 = 0xD2511F53u * c.x, hi0 = __umulhi(0xD2511F53u, c.x);
        const uint32_t lo1 = 0xCD9E8D57u * c.z, hi1 = __umulhi(0xCD9E8D57u, c.z);
        c = make_uint4(hi1 ^ c.y ^ k0, lo1, hi0 ^ c.w ^ k1, lo0);
    }
    return c;
}

// u = (2 * (r >> 9) + 1) * 2^-24 in (0, 1), exact in fp32; g = -log(-log u)
__device__ __forceinline__ float gumbel(uint32_t r) {
    const float u = float(((r >> 9) << 1) | 1u) * 5.9604644775390625e-08f;
    return -logf(-logf(u));
}

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

// Histograms are replicated per lane (bin * 32 + lane): lanes of a warp never add to the same word, whatever the logits
// (a row's 16-bit keys crowd into a few high-byte bins). reduce_hist folds the replicas into one table before a walk.
struct Hist {
    uint32_t cnt[256 * 32];
    unsigned long long mass[256 * 32];
};
constexpr size_t kHistBytes = sizeof(Hist);

struct Shared {
    uint32_t cnt[256];
    unsigned long long mass[256];
    float rf[kWarps];
    int ri[kWarps];
    unsigned long long ru[kWarps];
    int wc[kWarps];
    int bin;
    unsigned long long above;
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

// Warp 0 walks hist[255..0] from the top: the bin b with above(b) < target <= above(b) + hist[b] -> S.bin, S.above.
// Bins are cleared for the next pass. Caller synchronises before and after.
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
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            if (above + v[j] >= target) { b = 255 - 8 * lane - j; break; }
            above += v[j];
        }
        S.bin = b;
        S.above = above;
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) hist[8 * lane + j] = 0;
}

template <typename E>   // element type of the logits
__global__ void __launch_bounds__(kThreads, 1) sample_kernel(const __grid_constant__ SampleArgs a) {
    __shared__ Shared S;
    extern __shared__ __align__(16) unsigned char smem_raw[];
    Hist& H = *reinterpret_cast<Hist*>(smem_raw);
    const int row = blockIdx.x, tid = threadIdx.x, lane = tid & 31;
    const uint16_t* lg = a.logits + int64_t(row) * a.ld;
    const int V = a.V;
    const bool vec = (reinterpret_cast<uintptr_t>(lg) & 7u) == 0;
    const float T = a.temperature[row];
    const int K = a.top_k[row];
    const float P = a.top_p[row];
    const uint64_t seed = a.seed[row];
    const int64_t t = a.token_index[row];
    const bool valid = T >= 0.f && K >= 0 && P > 0.f && P <= 1.f;   // false for NaN
    const bool use_k = K > 1 && K < V;
    for (int b = tid; b < 256 * 32; b += kThreads) { H.cnt[b] = 0; H.mass[b] = 0; }
    __syncthreads();

    // pass 1: argmax of the logits; top-k level 1
    float bv = -INFINITY;
    int bi = 0x7fffffff;
    for (int g = tid; 4 * g < V; g += kThreads) {
        uint32_t bb[4];
        load4(lg, g, V, vec, bb);
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int i = 4 * g + j;
            if (i < V) {
                const uint32_t b = bb[j];
                const float v = DT<E>::to_f32(uint16_t(b));
                if (better_nan(v, i, bv, bi)) { bv = v; bi = i; }
                if (use_k) atomicAdd(&H.cnt[(okey(b) >> 8) * 32 + lane], 1u);
            }
        }
    }
    block_best<true>(S, bv, bi);
    int64_t tok = bi;
    const float m = __fdiv_rn(bv, T);
    if (!valid) tok = -1;
    else if (!(T == 0.f || K == 1 || bv != bv || !isfinite(m))) {
        // pass 2: the k-th largest logit -> kappa
        float kappa = -INFINITY;
        if (use_k) {
            reduce_hist(H.cnt, S.cnt);
            __syncthreads();
            walk_top(S, S.cnt, (unsigned long long)K);
            __syncthreads();
            const int hb = S.bin, rest = K - int(S.above);
            for (int g = tid; 4 * g < V; g += kThreads) {
                uint32_t bb[4];
                load4(lg, g, V, vec, bb);
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    const int i = 4 * g + j;
                    if (i < V) {
                        const uint32_t k = okey(bb[j]);
                        if (int(k >> 8) == hb) atomicAdd(&H.cnt[(k & 255u) * 32 + lane], 1u);
                    }
                }
            }
            __syncthreads();
            reduce_hist(H.cnt, S.cnt);
            __syncthreads();
            walk_top(S, S.cnt, (unsigned long long)rest);
            __syncthreads();
            kappa = __fdiv_rn(DT<E>::to_f32(key_bits((uint32_t(hb) << 8) | uint32_t(S.bin))), T);
        }
        // pass 3: Z over the kept set; top-p level 1
        const bool use_p = P < 1.f;
        unsigned long long z = 0;
        for (int g = tid; 4 * g < V; g += kThreads) {
            uint32_t bb[4];
            load4(lg, g, V, vec, bb);
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const int i = 4 * g + j;
                if (i < V) {
                    const uint32_t b = bb[j];
                    const float x = __fdiv_rn(DT<E>::to_f32(uint16_t(b)), T);
                    if (x >= kappa) {
                        const unsigned long long e = fixed_mass(x, m);
                        z += e;
                        if (use_p && e) atomicAdd(&H.mass[(okey(b) >> 8) * 32 + lane], e);
                    }
                }
            }
        }
        z = block_sum(S, z);
        float tau = kappa;
        int cut = 0x7fffffff;
        if (use_p) {
            // pass 4: the largest logit lambda with mass{l >= lambda} >= ceil(top_p * Z) -> tau
            unsigned long long target = (unsigned long long)ceil(double(P) * double(z));
            if (target < 1) target = 1;
            reduce_hist(H.mass, S.mass);
            __syncthreads();
            walk_top(S, S.mass, target);
            __syncthreads();
            const int hb = S.bin;
            const unsigned long long rest = target - S.above;
            for (int g = tid; 4 * g < V; g += kThreads) {
                uint32_t bb[4];
                load4(lg, g, V, vec, bb);
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    const int i = 4 * g + j;
                    if (i < V) {
                        const uint32_t b = bb[j];
                        const uint32_t k = okey(b);
                        if (int(k >> 8) == hb) {
                            const float x = __fdiv_rn(DT<E>::to_f32(uint16_t(b)), T);
                            if (x >= kappa) {
                                const unsigned long long e = fixed_mass(x, m);
                                if (e) atomicAdd(&H.mass[(k & 255u) * 32 + lane], e);
                            }
                        }
                    }
                }
            }
            __syncthreads();
            reduce_hist(H.mass, S.mass);
            __syncthreads();
            walk_top(S, S.mass, rest);
            __syncthreads();
            tau = __fdiv_rn(DT<E>::to_f32(key_bits((uint32_t(hb) << 8) | uint32_t(S.bin))), T);
            // pass 5: the mass above tau and the ties at tau (every x >= tau is kept by top-k: tau >= kappa)
            unsigned long long above = 0, ties = 0;
            for (int g = tid; 4 * g < V; g += kThreads) {
                uint32_t bb[4];
                load4(lg, g, V, vec, bb);
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    const int i = 4 * g + j;
                    if (i < V) {
                        const float x = __fdiv_rn(DT<E>::to_f32(bb[j]), T);
                        if (x > tau) above += fixed_mass(x, m);
                        else if (x == tau) ties += 1;
                    }
                }
            }
            above = block_sum(S, above);
            ties = block_sum(S, ties);
            // the ties at tau share one e: keep the first `need` of them in index order (need >= 1: above < target)
            const unsigned long long e_tau = fixed_mass(tau, m);
            const unsigned long long need = (e_tau && above < target) ? (target - above + e_tau - 1) / e_tau : 1;
            if (need < ties) {
                // pass 6: the index of the need-th tie
                long long left = (long long)need;
                const int warp = tid >> 5;
                if (tid == 0) S.cut = V - 1;
                for (int base = 0; base < V; base += kThreads) {
                    const int i = base + tid;
                    const bool f = i < V && __fdiv_rn(DT<E>::to_f32(__ldg(lg + i)), T) == tau;
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
                cut = S.cut;
            }
        }
        // pass 7: Gumbel-max over the kept set {x > tau} + {x == tau, index <= cut}
        float bs = -INFINITY;
        int bj = 0x7fffffff;
        const uint32_t k0 = uint32_t(seed), k1 = uint32_t(seed >> 32);
        const uint32_t t0 = uint32_t(uint64_t(t)), t1 = uint32_t(uint64_t(t) >> 32);
        for (int g = tid; 4 * g < V; g += kThreads) {
            uint32_t bb[4];
            load4(lg, g, V, vec, bb);
            float x[4];
            bool keep[4], any = false;
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const int i = 4 * g + j;
                x[j] = i < V ? __fdiv_rn(DT<E>::to_f32(bb[j]), T) : -INFINITY;
                keep[j] = i < V && (x[j] > tau || (x[j] == tau && i <= cut));
                any |= keep[j];
            }
            if (!any) continue;
            const uint4 r = philox(make_uint4(uint32_t(g), 0u, t0, t1), k0, k1);
            const uint32_t w[4] = {r.x, r.y, r.z, r.w};
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                if (!keep[j]) continue;
                const float s = x[j] + gumbel(w[j]);
                if (better(s, 4 * g + j, bs, bj)) { bs = s; bj = 4 * g + j; }
            }
        }
        block_best<false>(S, bs, bj);
        tok = bj;
    }
    if (tid == 0) {
        a.tokens[int64_t(row) * a.tokens_ld + a.col] = tok;
        if (a.advance) a.token_index[row] = t + 1;
    }
}

template <typename E>
cudaError_t launch_sample_t(const SampleArgs& a, cudaStream_t st) {
    // per device (the current one): set on every launch, a host-side attribute write
    const cudaError_t attr = cudaFuncSetAttribute(sample_kernel<E>, cudaFuncAttributeMaxDynamicSharedMemorySize, int(kHistBytes));
    if (attr != cudaSuccess) return attr;
    sample_kernel<E><<<a.B, kThreads, kHistBytes, st>>>(a);
    count_launch();
    return cudaGetLastError();
}

}  // namespace

cudaError_t launch_sample(const SampleArgs& a, cudaStream_t st) {
    return a.dtype == PKV_BF16 ? launch_sample_t<__nv_bfloat16>(a, st) : launch_sample_t<__half>(a, st);
}

}  // namespace pkv
