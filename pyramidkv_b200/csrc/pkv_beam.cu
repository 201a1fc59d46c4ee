// pkv_beam.cu — beam search on the device (include/pkv.h: pkv_beam_candidates, pkv_beam_step, pkv_cache_reorder;
// DESIGN.md §4.12): HF's `_beam_search` with do_sample=False, step by step, with fixed launch arguments so that the
// decode step graph replays it.
//
//   - beam_candidates_kernel: one CTA per beam row streams the row through rowsel::row_top (the passes of
//     pkv_token_logprobs: m, log Z in 64-bit fixed point, the radix walk over the 16-bit keys and the ordered tie scan)
//     and writes the row's top K tokens (logit descending, index ascending) with lp = (f32(l) - m) - log Z.
//   - beam_step_kernel: one CTA per prompt merges its k * K entries into the global top K (score descending, flat index
//     r * V + v ascending), then runs steps d-g of `_beam_search`: running beams, the finished pool, the early-stop
//     heuristic, and the bookkeeping the host and pkv_cache_reorder read (backpointers, parents, divergence rows).
//   - cache_reorder_kernel: one CTA per (layer, prompt, head) copies the generated rows each beam slot takes from its
//     parent, chunk by chunk; every source row of a chunk is in shared memory before any destination row of it is
//     written, so any parent map (a swap, a cycle, many-to-one) is safe in place.
#include "pkv_internal.h"
#include "pkv_rowsel.cuh"

namespace pkv {
namespace {

using namespace rowsel;

template <typename E>
__global__ void __launch_bounds__(kThreads, 1) beam_candidates_kernel(const __grid_constant__ BeamCandArgs a) {
    __shared__ Shared S;
    __shared__ Top<kMaxBeamCandidates> top;
    __shared__ uint32_t hist[256 * 32];
    const int row = blockIdx.x, tid = threadIdx.x;
    const uint16_t* lg = a.logits + int64_t(row) * a.ld;
    const int K = a.K, n_top = K < a.V ? K : a.V;
    float mx, log_z;
    const bool finite = row_top<E>(S, top, hist, lg, a.V, n_top, mx, log_z);
    // entry p's place in (key descending, index ascending) order: the entries are distinct indices, so ranks are distinct
    const int n = finite ? n_top : 0;
    float* lp = a.cand_lp + int64_t(row) * K;
    int32_t* ids = a.cand_id + int64_t(row) * K;
    if (tid < n) {
        const uint32_t k = top.key[tid];
        const int i = top.idx[tid];
        int r = 0;
        for (int q = 0; q < n; ++q) r += top.key[q] > k || (top.key[q] == k && top.idx[q] < i);
        lp[r] = (DT<E>::to_f32(key_bits(k)) - mx) - log_z;
        ids[r] = i;
    } else if (tid < K) {
        lp[tid] = -INFINITY;   // past the vocabulary, or a row with a NaN or +-inf logit: never a candidate before a real one
        ids[tid] = -1;
    }
    if (tid == 0) {
        a.m[row] = mx;
        a.log_z[row] = log_z;
    }
}

constexpr int kStepThreads = 1024;
constexpr float kNeg = -1.0e9f;   // HF's sentinel

// (s, i) before (t, j): score descending (NaN ranked as -inf), then index ascending
__device__ __forceinline__ bool ahead(float s, int i, float t, int j) {
    s = s != s ? -INFINITY : s;
    t = t != t ? -INFINITY : t;
    return s > t || (s == t && i < j);
}

__global__ void __launch_bounds__(kStepThreads, 1) beam_step_kernel(const __grid_constant__ BeamStepArgs a) {
    __shared__ float e_score[kMaxBeams * kMaxBeamCandidates];
    __shared__ int e_id[kMaxBeams * kMaxBeamCandidates];
    __shared__ float c_score[kMaxBeamCandidates];
    __shared__ int c_beam[kMaxBeamCandidates], c_tok[kMaxBeamCandidates];
    __shared__ bool c_hit[kMaxBeamCandidates];
    __shared__ float m_score[kMaxBeams + kMaxBeamCandidates];
    __shared__ int new_par[kMaxBeams], new_tok[kMaxBeams], div[kMaxBeams];
    __shared__ float new_run[kMaxBeams];
    __shared__ float pool_s[kMaxBeams];
    __shared__ int pool_st[kMaxBeams], pool_pa[kMaxBeams], pool_tk[kMaxBeams];
    __shared__ bool pool_f[kMaxBeams];
    __shared__ int cp_new[kMaxBeams * kMaxBeams];
    const int p = blockIdx.x, tid = threadIdx.x;
    const int k = a.k, K = a.K, T = a.max_steps;
    const int t = *a.step + a.step_offset;        // the iteration: t tokens generated before it, t rows in each beam's cache
    const int bk = p * k;
    if (a.done[p] || t >= T) {
        // a finished prompt keeps decoding in lock-step, frozen: every beam stays in its slot and copies nothing
        if (tid < k) {
            a.next_token[bk + tid] = 0;
            a.parent[bk + tid] = tid;
            a.diverge[bk + tid] = t;
        }
        return;
    }
    // c. the k * K scored entries, running[r] + lp
    const int nE = k * K;
    for (int e = tid; e < nE; e += kStepThreads) {
        const int r = e / K;
        const int src = (a.rows_per_prompt == 1 ? p : bk + r) * K + e % K;
        e_score[e] = a.running[bk + r] + a.cand_lp[src];
        e_id[e] = a.cand_id[src];
    }
    __syncthreads();
    // the global top K: flat index r * V + v ascending is (r, v) ascending; within a row the entries are distinct ids
    for (int e = tid; e < nE; e += kStepThreads) {
        const float s = e_score[e];
        const int r = e / K;
        const int v = e_id[e];
        const float s1 = s != s ? -INFINITY : s;
        int rank = 0;
        for (int f = 0; f < nE && rank < K; ++f) {
            const int rf = f / K, vf = e_id[f];
            const float sf = e_score[f];
            const float s2 = sf != sf ? -INFINITY : sf;
            // (vf, v) as unsigned: an id of -1 (no entry: a non-finite row) sorts after every token of its row, and such
            // entries by their position, so that every rank is taken exactly once
            rank += s2 > s1 || (s2 == s1 && (rf < r || (rf == r && (unsigned(vf) < unsigned(v) ||
                                                                    (vf == v && f < e)))));
        }
        if (rank < K) {
            c_score[rank] = s;
            c_beam[rank] = r;
            c_tok[rank] = v < 0 ? 0 : v;   // a prompt whose rows are all non-finite still feeds a valid token
        }
    }
    __syncthreads();
    // d. which candidates hit a stopping criterion: an EOS id, or the maximum length
    const bool last = t + 1 >= T;
    if (tid < K) {
        bool hit = last;
        for (int j = 0; j < a.n_eos; ++j) hit |= c_tok[tid] == a.eos[j];
        c_hit[tid] = hit;
    }
    __syncthreads();
    // e. the running beams: the top k of score + hit * -1e9 (ties: candidate order)
    if (tid < K) {
        const float s = c_score[tid] + (c_hit[tid] ? kNeg : -0.0f);
        int rank = 0;
        for (int c = 0; c < K; ++c) rank += ahead(c_score[c] + (c_hit[c] ? kNeg : -0.0f), c, s, tid);
        if (rank < k) {
            new_run[rank] = s;
            new_par[rank] = c_beam[tid];
            new_tok[rank] = c_tok[tid];
        }
    }
    // f. the pool: the old k entries, then the K candidates with the length penalty and the sentinels, top k
    const float* scale = a.scale + 2 * int64_t(t);
    const bool full = a.early_stopping == 1;
    bool all_fin = true;
    for (int j = 0; j < k; ++j) all_fin &= a.pool_done[bk + j] != 0;
    const bool heur = a.heur[p] != 0;
    if (tid < k) m_score[tid] = a.pool_score[bk + tid];
    if (tid < K) {
        float s = c_score[tid] * scale[0];
        s += (all_fin && full) ? kNeg : -0.0f;
        s += heur ? -0.0f : kNeg;
        s += (c_hit[tid] && tid < k) ? -0.0f : kNeg;
        m_score[k + tid] = s;
    }
    __syncthreads();
    if (tid < k + K) {
        const float s = m_score[tid];
        int rank = 0;
        for (int c = 0; c < k + K; ++c) rank += ahead(m_score[c], c, s, tid);
        if (rank < k) {
            pool_s[rank] = s;
            if (tid < k) {
                pool_st[rank] = a.pool_step[bk + tid];
                pool_pa[rank] = a.pool_parent[bk + tid];
                pool_tk[rank] = a.pool_token[bk + tid];
                pool_f[rank] = a.pool_done[bk + tid] != 0;
            } else {
                const int c = tid - k;
                pool_st[rank] = t;
                pool_pa[rank] = c_beam[c];
                pool_tk[rank] = c_tok[c];
                pool_f[rank] = c_hit[c] && c < k;
            }
        }
    }
    __syncthreads();
    // the divergence rows and the new common-prefix matrix: cp'[a][b] = (pa == pb) ? t : cp[pa][pb]
    const int32_t* cp = a.cp + int64_t(p) * k * k;
    for (int ij = tid; ij < k * k; ij += kStepThreads) {
        const int i = ij / k, j = ij % k;
        const int pi = new_par[i], pj = new_par[j];
        cp_new[ij] = pi == pj ? t : cp[pi * k + pj];
    }
    if (tid < k) div[tid] = new_par[tid] == tid ? t : cp[tid * k + new_par[tid]];
    __syncthreads();
    int32_t* cpw = a.cp + int64_t(p) * k * k;
    for (int ij = tid; ij < k * k; ij += kStepThreads) cpw[ij] = cp_new[ij];
    if (tid < k) {
        const int b = bk + tid;
        a.running[b] = new_run[tid];
        a.pool_score[b] = pool_s[tid];
        a.pool_step[b] = pool_st[tid];
        a.pool_parent[b] = pool_pa[tid];
        a.pool_token[b] = pool_tk[tid];
        a.pool_done[b] = pool_f[tid];
        a.bp_token[int64_t(b) * T + t] = new_tok[tid];
        a.bp_parent[int64_t(b) * T + t] = new_par[tid];
        a.next_token[b] = new_tok[tid];
        a.parent[b] = new_par[tid];
        a.diverge[b] = div[tid];
    }
    // g. the early-stop heuristic after the step, and whether the prompt is done
    if (tid == 0) {
        const float best = new_run[0] * scale[1];
        float worst = pool_s[0];
        bool fin = true;
        for (int j = 1; j < k; ++j) worst = fminf(worst, pool_s[j]);
        bool any = false;
        for (int j = 0; j < k; ++j) {
            any |= best > (pool_f[j] ? worst : kNeg);
            fin &= pool_f[j];
        }
        const bool h = heur && any;
        a.heur[p] = h;
        a.done[p] = !h || (fin && full) || last;
    }
}

constexpr int kReorderThreads = 256;
constexpr int kChunk = 4;   // generated rows per chunk
constexpr int kNone = 1 << 30;

__global__ void __launch_bounds__(kReorderThreads) cache_reorder_kernel(const __grid_constant__ ReorderArgs a) {
    extern __shared__ uint4 smem[];
    const ReorderLayer& L = a.layer[blockIdx.y];
    const int p = blockIdx.x / a.H, h = blockIdx.x % a.H, k = a.k, H = a.H, R = a.window;
    const int n = *a.step + a.step_offset;
    const int S = R > 0 ? min(n, R) : n;             // generated slots held
    const int vecs = a.row_bytes / 16;               // 16-byte words per K / V row
    uint4* kv = smem;                                // [k][kChunk][2][vecs]
    uint32_t* aux = reinterpret_cast<uint32_t*>(smem + k * kChunk * 2 * vecs);   // [k][kChunk][4] scales, heavy state
    uint32_t* vic = aux + k * kChunk * 4;            // [k]
    __shared__ int par[kMaxBeams], lo[kMaxBeams];
    __shared__ int first;
    if (threadIdx.x < k) {
        const int b = p * k + threadIdx.x;
        const int pa = a.parent[b], d = a.diverge[b];
        par[threadIdx.x] = pa;
        // the first slot to copy: the divergence row (no window), the ring slots of positions >= d (window), every slot
        // (heavy hitters: not position-indexed); kNone: nothing
        lo[threadIdx.x] = pa == int(threadIdx.x) ? kNone : (R == 0 ? d : (a.heavy ? 0 : max(d, n - R)));
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        int m = kNone;
        for (int j = 0; j < k; ++j) m = min(m, lo[j]);
        first = m;
    }
    __syncthreads();
    if (first == kNone) return;                      // every beam kept its own rows
    const int64_t cap = L.cap;
    // slot s of a ring holds the latest position j = s mod R below n; with no window slot s is position s
    auto needed = [&](int j, int s) {
        if (s >= S) return false;
        if (R == 0 || a.heavy) return s >= lo[j];
        return s + int64_t(R) * ((n - 1 - s) / R) >= lo[j];
    };
    const int start = R > 0 && !a.heavy ? 0 : first;   // ring slots are not in position order
    for (int c0 = start - start % kChunk; c0 < S; c0 += kChunk) {
        // load every needed source row of the chunk
        for (int w = threadIdx.x; w < k * kChunk * 2 * vecs; w += kReorderThreads) {
            const int j = w / (kChunk * 2 * vecs), rest = w % (kChunk * 2 * vecs);
            const int sl = rest / (2 * vecs), kvi = (rest / vecs) & 1, x = rest % vecs;
            const int s = c0 + sl;
            if (!needed(j, s)) continue;
            const int64_t src = int64_t(p * k + par[j]) * H + h;
            const int64_t row = L.base[src] + s;
            kv[w] = reinterpret_cast<const uint4*>(L.plane[kvi])[(src * cap + row) * vecs + x];
        }
        for (int w = threadIdx.x; w < k * kChunk; w += kReorderThreads) {
            const int j = w / kChunk, s = c0 + w % kChunk;
            if (!needed(j, s)) continue;
            const int64_t src = int64_t(p * k + par[j]) * H + h;
            const int64_t row = L.base[src] + s;
            if (L.plane[2]) {
                aux[4 * w] = reinterpret_cast<const uint32_t*>(L.plane[2])[src * cap + row];
                aux[4 * w + 1] = reinterpret_cast<const uint32_t*>(L.plane[3])[src * cap + row];
            }
            if (a.heavy) {
                aux[4 * w + 2] = __float_as_uint(L.heavy_scores[src * R + s]);
                aux[4 * w + 3] = uint32_t(L.heavy_gen[src * R + s]);
            }
        }
        if (a.heavy && c0 == 0 && threadIdx.x < k && par[threadIdx.x] != int(threadIdx.x))
            vic[threadIdx.x] = uint32_t(L.victim[int64_t(p * k + par[threadIdx.x]) * H + h]);
        __syncthreads();
        for (int w = threadIdx.x; w < k * kChunk * 2 * vecs; w += kReorderThreads) {
            const int j = w / (kChunk * 2 * vecs), rest = w % (kChunk * 2 * vecs);
            const int sl = rest / (2 * vecs), kvi = (rest / vecs) & 1, x = rest % vecs;
            const int s = c0 + sl;
            if (!needed(j, s)) continue;
            const int64_t dst = int64_t(p * k + j) * H + h;
            const int64_t row = L.base[dst] + s;
            reinterpret_cast<uint4*>(L.plane[kvi])[(dst * cap + row) * vecs + x] = kv[w];
        }
        for (int w = threadIdx.x; w < k * kChunk; w += kReorderThreads) {
            const int j = w / kChunk, s = c0 + w % kChunk;
            if (!needed(j, s)) continue;
            const int64_t dst = int64_t(p * k + j) * H + h;
            const int64_t row = L.base[dst] + s;
            if (L.plane[2]) {
                reinterpret_cast<uint32_t*>(L.plane[2])[dst * cap + row] = aux[4 * w];
                reinterpret_cast<uint32_t*>(L.plane[3])[dst * cap + row] = aux[4 * w + 1];
            }
            if (a.heavy) {
                L.heavy_scores[dst * R + s] = __uint_as_float(aux[4 * w + 2]);
                L.heavy_gen[dst * R + s] = int32_t(aux[4 * w + 3]);
            }
        }
        if (a.heavy && c0 == 0 && threadIdx.x < k && par[threadIdx.x] != int(threadIdx.x))
            L.victim[int64_t(p * k + threadIdx.x) * H + h] = int32_t(vic[threadIdx.x]);
        __syncthreads();
    }
}

}  // namespace

cudaError_t launch_beam_candidates(const BeamCandArgs& a, cudaStream_t st) {
    if (a.dtype == PKV_BF16) beam_candidates_kernel<__nv_bfloat16><<<a.rows, kThreads, 0, st>>>(a);
    else beam_candidates_kernel<__half><<<a.rows, kThreads, 0, st>>>(a);
    count_launch();
    return cudaGetLastError();
}

cudaError_t launch_beam_step(const BeamStepArgs& a, cudaStream_t st) {
    beam_step_kernel<<<a.P, kStepThreads, 0, st>>>(a);
    count_launch();
    return cudaGetLastError();
}

size_t reorder_smem_bytes(int k, int row_bytes) {
    return size_t(k) * kChunk * 2 * row_bytes + size_t(k) * kChunk * 16 + size_t(k) * 4;
}

cudaError_t launch_cache_reorder(const ReorderArgs& a, cudaStream_t st) {
    const size_t smem = reorder_smem_bytes(a.k, a.row_bytes);
    dim3 grid(a.P * a.H, a.n_layers);
    cache_reorder_kernel<<<grid, kReorderThreads, smem, st>>>(a);
    count_launch();
    return cudaGetLastError();
}

}  // namespace pkv
