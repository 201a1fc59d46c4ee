// pkv_logprobs.cu — log-probabilities of one row of logits (include/pkv.h: pkv_token_logprobs): the log-softmax read at a
// given token and at the row's top N, one CTA per row, in one launch for the whole batch.
//
// The CTA streams its row (bf16 / fp16, 256 KB for Llama-3's 128256 tokens; it stays in L2 between passes) through the
// three passes of rowsel::row_top (pkv_rowsel.cuh): the maximum m, Z = sum of expf(x_i - m) in 64-bit fixed point (2^-40
// units: exact, order-free sums) and the N largest logits found by a radix walk over the 16-bit keys.
// The (at most 20) entries are then sorted by (logit descending, index ascending) by one thread. Every sum is an integer
// sum and every tie is cut by index, so a graph replay and a host launch write the same bits.
#include "pkv_internal.h"
#include "pkv_rowsel.cuh"

namespace pkv {
namespace {

using namespace rowsel;

template <typename E>   // element type of the logits
__global__ void __launch_bounds__(kThreads, 1) logprobs_kernel(const __grid_constant__ LogprobsArgs a) {
    __shared__ Shared S;
    __shared__ Top<kMaxTopLogprobs> top;
    __shared__ uint32_t hist[256 * 32];
    const int row = blockIdx.x, tid = threadIdx.x;
    const uint16_t* lg = a.logits + int64_t(row) * a.ld;
    const int V = a.V, N = a.N;
    const int n_top = N < V ? N : V;                   // entries past the vocabulary: id -1, NaN
    const int64_t col = a.col + (a.cursor ? *a.cursor : 0);
    float mx, log_z;
    const bool finite = row_top<E>(S, top, hist, lg, V, n_top, mx, log_z);
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
