// pkv_logprobs.cu — log-probabilities of one row of logits (include/pkv.h: pkv_token_logprobs): the log-softmax read at a
// given token and at the row's top N, one CTA per row, in one launch for the whole batch.
//
// The CTA streams its row (bf16 / fp16, 256 KB for Llama-3's 128256 tokens; it stays in L2 between passes):
//   1. the maximum m, whether any logit is NaN or +-inf, and (N > 0) a count histogram of the high byte of the 16-bit key;
//   2. Z = sum of expf(x_i - m) in 64-bit fixed point (2^-40 units: exact, order-free sums) and (N > 0) the low-byte
//      histogram inside the high-byte bin of the N-th largest key -> that key k_N, how many keys lie above it and how many
//      equal it;
//   3. (N > 0) the N entries: every key above k_N and the lowest-index ties at k_N (when more tie than are needed, the index
//      of the last one kept comes from one ballot scan in index order, which stops at the chunk that holds it).
// The (at most 20) entries are then sorted by (logit descending, index ascending) by one thread. Every sum is an integer
// sum and every tie is cut by index, so a graph replay and a host launch write the same bits.
#include "pkv_internal.h"
#include "pkv_rowsel.cuh"

namespace pkv {
namespace {

using namespace rowsel;

struct Top {
    uint32_t key[kMaxTopLogprobs];
    int idx[kMaxTopLogprobs];
    int n;
};

template <typename E>   // element type of the logits
__global__ void __launch_bounds__(kThreads, 1) logprobs_kernel(const __grid_constant__ LogprobsArgs a) {
    __shared__ Shared S;
    __shared__ Top top;
    __shared__ uint32_t hist[256 * 32];
    const int row = blockIdx.x, tid = threadIdx.x, lane = tid & 31;
    const uint16_t* lg = a.logits + int64_t(row) * a.ld;
    const int V = a.V, N = a.N;
    const int n_top = N < V ? N : V;                   // entries past the vocabulary: id -1, NaN
    const bool vec = (reinterpret_cast<uintptr_t>(lg) & 7u) == 0;
    const int64_t col = a.col + (a.cursor ? *a.cursor : 0);
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
                        if (s < kMaxTopLogprobs) { top.key[s] = k; top.idx[s] = i; }
                    }
                }
            }
        }
        __syncthreads();
    }
    if (tid == 0) {
        const int64_t t = a.tokens[int64_t(row) * a.tokens_ld + a.tokens_col];
        float lp = NAN;
        if (finite && t >= 0 && t < V) lp = (DT<E>::to_f32(__ldg(lg + t)) - mx) - log_z;
        a.lp[int64_t(row) * a.lp_ld + col] = lp;
        if (N > 0) {
            // insertion sort of the n_top entries: key descending, index ascending
            const int n = finite ? n_top : 0;
            for (int p = 1; p < n; ++p) {
                const uint32_t k = top.key[p];
                const int i = top.idx[p];
                int q = p;
                for (; q > 0 && (top.key[q - 1] < k || (top.key[q - 1] == k && top.idx[q - 1] > i)); --q) {
                    top.key[q] = top.key[q - 1];
                    top.idx[q] = top.idx[q - 1];
                }
                top.key[q] = k;
                top.idx[q] = i;
            }
            int64_t* ids = a.top_ids + int64_t(row) * a.top_ld + col * N;
            float* tlp = a.top_lp + int64_t(row) * a.top_ld + col * N;
            for (int p = 0; p < N; ++p) {
                ids[p] = p < n ? int64_t(top.idx[p]) : int64_t(-1);
                tlp[p] = p < n ? (DT<E>::to_f32(key_bits(top.key[p])) - mx) - log_z : NAN;
            }
        }
    }
}

template <typename E>
cudaError_t launch_logprobs_t(const LogprobsArgs& a, cudaStream_t st) {
    logprobs_kernel<E><<<a.B, kThreads, 0, st>>>(a);
    count_launch();
    return cudaGetLastError();
}

}  // namespace

cudaError_t launch_logprobs(const LogprobsArgs& a, cudaStream_t st) {
    return a.dtype == PKV_BF16 ? launch_logprobs_t<__nv_bfloat16>(a, st) : launch_logprobs_t<__half>(a, st);
}

}  // namespace pkv
