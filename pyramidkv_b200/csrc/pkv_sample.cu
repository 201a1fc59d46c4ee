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

}  // namespace

cudaError_t launch_sample(const SampleArgs& a, cudaStream_t st) {
    return a.dtype == PKV_BF16 ? launch_sample_t<__nv_bfloat16>(a, st) : launch_sample_t<__half>(a, st);
}

}  // namespace pkv
