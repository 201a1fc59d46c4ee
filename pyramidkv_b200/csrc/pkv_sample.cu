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
#include "pkv_internal.h"
#include "pkv_rowsel.cuh"

namespace pkv {
namespace {

using namespace rowsel;

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

// the per-lane replicated count and mass histograms (rowsel::reduce_hist)
struct Hist {
    uint32_t cnt[256 * 32];
    unsigned long long mass[256 * 32];
};
constexpr size_t kHistBytes = sizeof(Hist);

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
                cut = nth_index(S, V, (long long)need,
                                [&](int i) { return __fdiv_rn(DT<E>::to_f32(__ldg(lg + i)), T) == tau; });
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

// ---- the penalized form (pkv_sample_tokens_penalized) ----
// The penalized value x_v (before the temperature) of one row: f32(logit), then the repetition penalty over the prompt and
// the generated tokens, then frequency * count and presence over the generated ones. Each operation is rounded once
// (no contraction), as the rules in include/pkv.h state them.
struct PenRow {
    const uint16_t* lg;
    const uint8_t* mask;
    const int32_t* cnt;
    int V;
    bool vec;           // 8-byte logit loads
    bool vec_pc;        // 4-byte mask and 16-byte count loads
    bool use_mask;      // repetition_penalty != 1
    bool pen;           // some penalty is on: counts (and the mask) are read
    float rho, pres, freq;
    // the rule terms of the constrained form (pkv_sample_tokens_constrained); rules = 0 in the penalized form
    int rules;          // PKV_RULE_BIAS | PKV_RULE_BAN | PKV_RULE_BAD of the row
    bool vec_bias;      // 16-byte bias loads
    const float* bias;
    const uint32_t* ban;
    int W;
};

__device__ __forceinline__ float penalize(const PenRow& r, float x, uint32_t in_prompt, int c) {
    if (r.use_mask && (in_prompt || c > 0)) x = x < 0.f ? __fmul_rn(x, r.rho) : __fdiv_rn(x, r.rho);
    if (c > 0) x = __fsub_rn(__fsub_rn(x, __fmul_rn(r.freq, float(c))), r.pres);
    return x;
}

// the bans of element i after the penalties: set to -inf (n-grams, min_new_tokens), else add -inf or 0 (bad words)
__device__ __forceinline__ float ban_term(const PenRow& r, float x, int i) {
    if ((r.rules & PKV_RULE_BAN) && ((__ldg(r.ban + (i >> 5)) >> (i & 31)) & 1u)) return -INFINITY;
    if (r.rules & PKV_RULE_BAD) x = __fadd_rn(x, ((__ldg(r.ban + r.W + (i >> 5)) >> (i & 31)) & 1u) ? -INFINITY : 0.f);
    return x;
}

// steps 2-3 (the penalties) on elements 4g .. 4g+3
__device__ __forceinline__ void penalize4(const PenRow& r, int g, float (&x)[4]) {
    if (!r.pen) return;
    const int i = 4 * g;
    int c[4];
    uint32_t mk[4] = {0u, 0u, 0u, 0u};
    if (r.vec_pc && i + 3 < r.V) {
        const int4 cv = __ldg(reinterpret_cast<const int4*>(r.cnt) + g);
        c[0] = cv.x; c[1] = cv.y; c[2] = cv.z; c[3] = cv.w;
        if (r.use_mask) {
            const uint32_t m = __ldg(reinterpret_cast<const uint32_t*>(r.mask) + g);
#pragma unroll
            for (int j = 0; j < 4; ++j) mk[j] = (m >> (8 * j)) & 255u;
        }
    } else {
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            c[j] = i + j < r.V ? __ldg(r.cnt + i + j) : 0;
            if (r.use_mask) mk[j] = i + j < r.V ? __ldg(r.mask + i + j) : 0u;
        }
    }
#pragma unroll
    for (int j = 0; j < 4; ++j) x[j] = penalize(r, x[j], mk[j], c[j]);
}

// x of elements 4g .. 4g+3 (those past V are not meaningful: callers test i < V); kRules adds the rule terms
template <typename E, bool kRules>
__device__ __forceinline__ void load_x4(const PenRow& r, int g, float (&x)[4]) {
    uint32_t bb[4];
    load4(r.lg, g, r.V, r.vec, bb);
#pragma unroll
    for (int j = 0; j < 4; ++j) x[j] = DT<E>::to_f32(uint16_t(bb[j]));
    const int i = 4 * g;
    if (kRules && (r.rules & PKV_RULE_BIAS)) {
        if (r.vec_bias && i + 3 < r.V) {
            const float4 bv = __ldg(reinterpret_cast<const float4*>(r.bias) + g);
            x[0] = __fadd_rn(x[0], bv.x); x[1] = __fadd_rn(x[1], bv.y); x[2] = __fadd_rn(x[2], bv.z); x[3] = __fadd_rn(x[3], bv.w);
        } else {
#pragma unroll
            for (int j = 0; j < 4; ++j)
                if (i + j < r.V) x[j] = __fadd_rn(x[j], __ldg(r.bias + i + j));
        }
    }
    penalize4(r, g, x);
    if (kRules && (r.rules & (PKV_RULE_BAN | PKV_RULE_BAD))) {
#pragma unroll
        for (int j = 0; j < 4; ++j)
            if (i + j < r.V) x[j] = ban_term(r, x[j], i + j);
    }
}

template <typename E, bool kRules>
__device__ __forceinline__ float load_x1(const PenRow& r, int i) {
    float x = DT<E>::to_f32(__ldg(r.lg + i));
    if (kRules && (r.rules & PKV_RULE_BIAS)) x = __fadd_rn(x, __ldg(r.bias + i));
    if (r.pen) x = penalize(r, x, r.use_mask ? uint32_t(__ldg(r.mask + i)) : 0u, __ldg(r.cnt + i));
    if (kRules && (r.rules & (PKV_RULE_BAN | PKV_RULE_BAD))) x = ban_term(r, x, i);
    return x;
}

// The walks of sample_kernel, over 32-bit keys of x (okey32) in four 8-bit digits: the penalties do not keep the order of
// the logits. Level 0 histograms the top digit; level lv > 0 the digit below `prefix` (the lv digits chosen so far).
// kRules (pkv_sample_tokens_constrained) adds the rule terms of RuleTermArgs to x; rows with none read nothing of them.
template <typename E, bool kRules>
__global__ void __launch_bounds__(kThreads, 1) sample_penalized_kernel(const __grid_constant__ SampleArgs a,
                                                                       const __grid_constant__ PenaltyArgs p,
                                                                       const __grid_constant__ RuleTermArgs q) {
    __shared__ Shared S;
    extern __shared__ __align__(16) unsigned char smem_raw[];
    Hist& H = *reinterpret_cast<Hist*>(smem_raw);
    const int row = blockIdx.x, tid = threadIdx.x, lane = tid & 31;
    const int V = a.V;
    PenRow r;
    r.lg = a.logits + int64_t(row) * a.ld;
    r.mask = p.mask + int64_t(row) * p.ld;
    r.cnt = p.counts + int64_t(row) * p.ld;
    r.V = V;
    r.vec = (reinterpret_cast<uintptr_t>(r.lg) & 7u) == 0;
    r.vec_pc = (reinterpret_cast<uintptr_t>(r.cnt) & 15u) == 0 && (reinterpret_cast<uintptr_t>(r.mask) & 3u) == 0;
    r.rho = p.repetition[row];
    r.pres = p.presence[row];
    r.freq = p.frequency[row];
    const float minp = p.min_p[row];
    r.use_mask = r.rho != 1.f;
    r.pen = r.use_mask || r.pres != 0.f || r.freq != 0.f;
    r.rules = kRules ? (q.flags[row] & (PKV_RULE_BIAS | PKV_RULE_BAN | PKV_RULE_BAD)) : 0;
    r.bias = kRules ? q.bias + int64_t(row) * q.bias_ld : nullptr;
    r.ban = kRules ? q.ban + int64_t(row) * q.ban_ld : nullptr;
    r.W = q.W;
    r.vec_bias = (reinterpret_cast<uintptr_t>(r.bias) & 15u) == 0;
    const float T = a.temperature[row];
    const int K = a.top_k[row];
    const float P = a.top_p[row];
    const uint64_t seed = a.seed[row];
    const int64_t t = a.token_index[row];
    const bool valid = T >= 0.f && K >= 0 && P > 0.f && P <= 1.f && r.rho > 0.f && isfinite(r.rho) && isfinite(r.pres) &&
                       isfinite(r.freq) && minp >= 0.f && minp <= 1.f;   // false for NaN
    const bool use_k = K > 1 && K < V;
    for (int b = tid; b < 256 * 32; b += kThreads) { H.cnt[b] = 0; H.mass[b] = 0; }
    __syncthreads();

    // pass 1: argmax of x; top-k level 0
    float bv = -INFINITY;
    int bi = 0x7fffffff;
    for (int g = tid; 4 * g < V; g += kThreads) {
        float x[4];
        load_x4<E, kRules>(r, g, x);
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int i = 4 * g + j;
            if (i < V) {
                if (better_nan(x[j], i, bv, bi)) { bv = x[j]; bi = i; }
                if (use_k) atomicAdd(&H.cnt[(okey32(x[j]) >> 24) * 32 + lane], 1u);
            }
        }
    }
    block_best<true>(S, bv, bi);
    int64_t tok = bi;
    const float m = __fdiv_rn(bv, T);
    if (!valid) tok = -1;
    else if (!(T == 0.f || K == 1 || bv != bv || !isfinite(m))) {
        // top-k levels 1-3: the k-th largest x -> kappa
        float kappa = -INFINITY;
        if (use_k) {
            uint32_t prefix = 0;
            unsigned long long rest = (unsigned long long)K;
            for (int lv = 0; lv < 4; ++lv) {
                if (lv > 0) {
                    const int hs = 32 - 8 * lv, ds = 24 - 8 * lv;
                    for (int g = tid; 4 * g < V; g += kThreads) {
                        float x[4];
                        load_x4<E, kRules>(r, g, x);
#pragma unroll
                        for (int j = 0; j < 4; ++j) {
                            const uint32_t k = okey32(x[j]);
                            if (4 * g + j < V && (k >> hs) == prefix) atomicAdd(&H.cnt[((k >> ds) & 255u) * 32 + lane], 1u);
                        }
                    }
                    __syncthreads();
                }
                reduce_hist(H.cnt, S.cnt);
                __syncthreads();
                walk_top(S, S.cnt, rest);
                __syncthreads();
                rest -= S.above;
                prefix = (prefix << 8) | uint32_t(S.bin);
            }
            kappa = __fdiv_rn(key_value32(prefix), T);
        }
        // Z over the kept set; top-p level 0
        const bool use_p = P < 1.f;
        unsigned long long z = 0;
        for (int g = tid; 4 * g < V; g += kThreads) {
            float x[4];
            load_x4<E, kRules>(r, g, x);
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                if (4 * g + j < V) {
                    const float y = __fdiv_rn(x[j], T);
                    if (y >= kappa) {
                        const unsigned long long e = fixed_mass(y, m);
                        z += e;
                        if (use_p && e) atomicAdd(&H.mass[(okey32(x[j]) >> 24) * 32 + lane], e);
                    }
                }
            }
        }
        z = block_sum(S, z);
        float tau = kappa;
        int cut = 0x7fffffff;
        if (use_p) {
            // top-p levels 0-3: the largest x lambda with mass{x >= lambda} >= ceil(top_p * Z) -> tau
            unsigned long long target = (unsigned long long)ceil(double(P) * double(z));
            if (target < 1) target = 1;
            uint32_t prefix = 0;
            unsigned long long rest = target;
            for (int lv = 0; lv < 4; ++lv) {
                if (lv > 0) {
                    const int hs = 32 - 8 * lv, ds = 24 - 8 * lv;
                    for (int g = tid; 4 * g < V; g += kThreads) {
                        float x[4];
                        load_x4<E, kRules>(r, g, x);
#pragma unroll
                        for (int j = 0; j < 4; ++j) {
                            const uint32_t k = okey32(x[j]);
                            if (4 * g + j < V && (k >> hs) == prefix) {
                                const float y = __fdiv_rn(x[j], T);
                                if (y >= kappa) {
                                    const unsigned long long e = fixed_mass(y, m);
                                    if (e) atomicAdd(&H.mass[((k >> ds) & 255u) * 32 + lane], e);
                                }
                            }
                        }
                    }
                    __syncthreads();
                }
                reduce_hist(H.mass, S.mass);
                __syncthreads();
                walk_top(S, S.mass, rest);
                __syncthreads();
                rest -= S.above;
                prefix = (prefix << 8) | uint32_t(S.bin);
            }
            tau = __fdiv_rn(key_value32(prefix), T);
            // the mass above tau and the ties at tau (every y >= tau is kept by top-k: tau >= kappa)
            unsigned long long above = 0, ties = 0;
            for (int g = tid; 4 * g < V; g += kThreads) {
                float x[4];
                load_x4<E, kRules>(r, g, x);
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    if (4 * g + j < V) {
                        const float y = __fdiv_rn(x[j], T);
                        if (y > tau) above += fixed_mass(y, m);
                        else if (y == tau) ties += 1;
                    }
                }
            }
            above = block_sum(S, above);
            ties = block_sum(S, ties);
            const unsigned long long e_tau = fixed_mass(tau, m);
            const unsigned long long need = (e_tau && above < target) ? (target - above + e_tau - 1) / e_tau : 1;
            if (need < ties)
                cut = nth_index(S, V, (long long)need, [&](int i) { return __fdiv_rn(load_x1<E, kRules>(r, i), T) == tau; });
        }
        // Gumbel-max over the kept set {y > tau} + {y == tau, index <= cut}, less the tokens min-p drops
        float bs = -INFINITY;
        int bj = 0x7fffffff;
        const uint32_t k0 = uint32_t(seed), k1 = uint32_t(seed >> 32);
        const uint32_t t0 = uint32_t(uint64_t(t)), t1 = uint32_t(uint64_t(t) >> 32);
        for (int g = tid; 4 * g < V; g += kThreads) {
            float x[4];
            load_x4<E, kRules>(r, g, x);
            bool keep[4], any = false;
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const int i = 4 * g + j;
                x[j] = i < V ? __fdiv_rn(x[j], T) : -INFINITY;
                keep[j] = i < V && (x[j] > tau || (x[j] == tau && i <= cut)) && (minp == 0.f || expf(x[j] - m) >= minp);
                any |= keep[j];
            }
            if (!any) continue;
            const uint4 rr = philox(make_uint4(uint32_t(g), 0u, t0, t1), k0, k1);
            const uint32_t w[4] = {rr.x, rr.y, rr.z, rr.w};
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
        if (a.advance) {
            a.token_index[row] = t + 1;
            if (tok >= 0) p.counts[int64_t(row) * p.ld + tok] += 1;
        }
    }
}

template <typename E, bool kRules>
cudaError_t launch_sample_penalized_t(const SampleArgs& a, const PenaltyArgs& p, const RuleTermArgs& q, cudaStream_t st) {
    const cudaError_t attr = cudaFuncSetAttribute(sample_penalized_kernel<E, kRules>,
                                                  cudaFuncAttributeMaxDynamicSharedMemorySize, int(kHistBytes));
    if (attr != cudaSuccess) return attr;
    sample_penalized_kernel<E, kRules><<<a.B, kThreads, kHistBytes, st>>>(a, p, q);
    count_launch();
    return cudaGetLastError();
}

}  // namespace

cudaError_t launch_sample(const SampleArgs& a, cudaStream_t st) {
    return a.dtype == PKV_BF16 ? launch_sample_t<__nv_bfloat16>(a, st) : launch_sample_t<__half>(a, st);
}

cudaError_t launch_sample_penalized(const SampleArgs& a, const PenaltyArgs& p, cudaStream_t st) {
    const RuleTermArgs none{};
    return a.dtype == PKV_BF16 ? launch_sample_penalized_t<__nv_bfloat16, false>(a, p, none, st)
                               : launch_sample_penalized_t<__half, false>(a, p, none, st);
}

cudaError_t launch_sample_constrained(const SampleArgs& a, const PenaltyArgs& p, const RuleTermArgs& q, cudaStream_t st) {
    return a.dtype == PKV_BF16 ? launch_sample_penalized_t<__nv_bfloat16, true>(a, p, q, st)
                               : launch_sample_penalized_t<__half, true>(a, p, q, st);
}

}  // namespace pkv
