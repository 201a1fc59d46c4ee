// pkv_rules.cu — the per-row rule terms of one decode step (include/pkv.h: pkv_token_rules, DESIGN.md §4.11): sequence-bias
// sums, the two ban bitmaps (set to -inf: no-repeat n-grams and min_new_tokens; add -inf: bad words) and the stop flag,
// from each row's token history. One CTA per row:
//   0. append the step's token to the history (thread 0);
//   1. clear the row's dense bias row and ban words (only the kinds its flags name);
//   2. the rule sequences, one thread per sequence: a bias thread that heads a run of sequences with one last token sums
//      the run in order (so the sum is HF's, whatever the thread schedule); bad words and stop sequences test the tail;
//   3. the n-gram scan: one thread per start position of the history, O(history * N) compares per row;
//   4. the EOS bans of min_new_tokens.
// Bits are set with atomicOr and every bias entry has one writer, so the outputs do not depend on the schedule.
#include "pkv_internal.h"

namespace pkv {
namespace {

constexpr int kRuleThreads = 512;

// the last len tokens of h[0, n) equal s[0, len) (the caller checks len <= n)
__device__ __forceinline__ bool tail_is(const int32_t* h, int n, const int32_t* s, int len) {
    for (int k = 0; k < len; ++k)
        if (h[n - len + k] != s[k]) return false;
    return true;
}

__device__ __forceinline__ void set_bit(uint32_t* words, int v, int V) {
    if (v >= 0 && v < V) atomicOr(words + (v >> 5), 1u << (v & 31));
}

__global__ void __launch_bounds__(kRuleThreads) token_rules_kernel(const __grid_constant__ TokenRulesArgs a) {
    const int b = blockIdx.x, tid = threadIdx.x;
    int32_t* h = a.hist + int64_t(b) * a.hist_ld;
    __shared__ int s_len, s_stop;
    if (tid == 0) {
        int n = a.hist_len[b];
        if (a.append && n < a.hist_ld) {
            h[n] = int32_t(a.append[int64_t(b) * a.append_ld + a.append_col]);
            a.hist_len[b] = ++n;
        }
        s_len = n;
        s_stop = 0;
    }
    __syncthreads();
    const int n = s_len, V = a.V, W = a.W;
    const int flags = a.flags[b];
    float* bias = a.bias + int64_t(b) * a.bias_ld;
    uint32_t* ban = a.ban + int64_t(b) * a.ban_ld;
    if (flags & PKV_RULE_BIAS) {
        if ((a.bias_ld & 3) == 0 && (reinterpret_cast<uintptr_t>(a.bias) & 15u) == 0) {
            for (int g = tid; 4 * g + 3 < V; g += kRuleThreads) reinterpret_cast<float4*>(bias)[g] = make_float4(0.f, 0.f, 0.f, 0.f);
            for (int v = (V & ~3) + tid; v < V; v += kRuleThreads) bias[v] = 0.f;
        } else {
            for (int v = tid; v < V; v += kRuleThreads) bias[v] = 0.f;
        }
    }
    if (flags & (PKV_RULE_BAN | PKV_RULE_BAD))
        for (int w = tid; w < 2 * W; w += kRuleThreads) ban[w] = 0u;
    __syncthreads();
    if (!(flags & (PKV_RULE_BIAS | PKV_RULE_BAN | PKV_RULE_BAD | PKV_RULE_STOP))) {
        if (tid == 0) a.stop[b] = 0;
        return;
    }

    // 2. the rule sequences
    const int ns = a.n_seq[b];
    const int32_t* off = a.seq_off + int64_t(b) * a.seq_ld;
    const int32_t* kind = a.seq_kind + int64_t(b) * a.seq_ld;
    const float* wt = a.seq_bias + int64_t(b) * a.seq_ld;
    const int32_t* tok = a.seq_tok + int64_t(b) * a.tok_ld;
    for (int j = tid; j < ns; j += kRuleThreads) {
        const int o = off[j], L = off[j + 1] - o, k = kind[j];
        if (L < 1) continue;
        const int last = tok[o + L - 1];
        if (k == PKV_SEQ_BIAS) {
            if (j > 0 && kind[j - 1] == PKV_SEQ_BIAS && off[j] > off[j - 1] && tok[o - 1] == last) continue;   // not a run head
            float s = 0.f;
            for (int i = j; i < ns && kind[i] == PKV_SEQ_BIAS; ++i) {
                const int oi = off[i], Li = off[i + 1] - oi;
                if (Li < 1 || tok[oi + Li - 1] != last) break;
                const bool m = Li == 1 || (Li <= n && tail_is(h, n, tok + oi, Li - 1));
                s = __fadd_rn(s, m ? wt[i] : 0.f);
            }
            if (last >= 0 && last < V && (flags & PKV_RULE_BIAS)) bias[last] = s;
        } else if (k == PKV_SEQ_BAD) {
            if ((flags & PKV_RULE_BAD) && (L == 1 || (L <= n && tail_is(h, n, tok + o, L - 1)))) set_bit(ban + W, last, V);
        } else if (k == PKV_SEQ_STOP) {
            if ((flags & PKV_RULE_STOP) && L <= n && tail_is(h, n, tok + o, L)) s_stop = 1;
        }
    }

    if (flags & PKV_RULE_BAN) {
        // 3. no-repeat n-grams: the N-grams h[i, i + N) whose first N - 1 tokens are the last N - 1 of h
        const int N = a.ngram[b];
        if (N > 0 && n >= N) {
            const int32_t* pre = h + n - N + 1;
            for (int i = tid; i <= n - N; i += kRuleThreads) {
                int k = 0;
                while (k < N - 1 && h[i + k] == pre[k]) ++k;
                if (k == N - 1) set_bit(ban, h[i + N - 1], V);
            }
        }
        // 4. min_new_tokens: EOS is set to -inf while fewer tokens than that have been generated
        if (n - a.prompt_len[b] < a.min_new[b])
            for (int e = tid; e < a.n_eos; e += kRuleThreads) set_bit(ban, a.eos[e], V);
    }
    __syncthreads();
    if (tid == 0) a.stop[b] = uint8_t(s_stop);
}

}  // namespace

cudaError_t launch_token_rules(const TokenRulesArgs& a, cudaStream_t st) {
    token_rules_kernel<<<a.B, kRuleThreads, 0, st>>>(a);
    count_launch();
    return cudaGetLastError();
}

}  // namespace pkv
