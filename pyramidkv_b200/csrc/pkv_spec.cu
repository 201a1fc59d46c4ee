// pkv_spec.cu — prompt-lookup speculative decoding: the verify attention over K + 1 new rows per sequence, the device
// n-gram lookup that drafts them and the acceptance step (include/pkv.h: pkv_decode_attn_multi, pkv_prompt_lookup,
// pkv_spec_step; DESIGN.md §4.13).
//
// Verify attention: one CTA per (split, cache head, sequence) stages tiles of 32 cached rows in shared memory, widened to fp32,
// and every one of its M = GH * Q query rows (GH query heads of the cache head, Q new tokens each) reads them from there:
// each cached row leaves HBM once per CTA, not once per query. The Q new rows of a (sequence, cache head) are built in shared
// memory first (16-bit: as given; E4M3: quantised with the rule of pkv_rows.cuh), split 0 stores them at n0 .. n0 + Q - 1,
// and every split attends them from shared memory, so no CTA reads a row another CTA is writing. Query j of a head attends
// rows [0, n0 + j + 1). Per (query row, tile): lane r computes the dot with row r (K tile padded to D + 1 floats per row, so
// the 32 lanes hit 32 banks), one warp max / sum gives the online softmax step, and the lanes then own D / 32 output dims
// each. Accumulators live in shared memory, so the register count does not grow with Q or the group.
// The packed launch (pkv_decode_attn_packed) runs the same body with a per-sequence row count c <= Q read on the device:
// the CTA works on GH * c query rows, and a count of 0 returns before anything of the sequence is read or written.
#include "pkv_common.cuh"
#include "pkv_internal.h"
#include "pkv_rows.cuh"

namespace pkv {
namespace {

constexpr int kMultiThreads = 256;
constexpr int kMultiWarps = kMultiThreads / 32;
constexpr int kTile = 32;   // cached rows per shared-memory tile: one per lane

struct MultiSmem {   // float offsets into the dynamic shared memory of one CTA
    int q, acc, ml, k, v, kvs, nk, nv, ns, p, total;
};

__host__ __device__ inline MultiSmem multi_smem(int M, int Q, int D) {
    MultiSmem s;
    s.q = 0;
    s.acc = s.q + M * D;
    s.ml = s.acc + M * D;          // (m, l) per query row
    s.k = s.ml + 2 * M;
    s.v = s.k + kTile * (D + 1);
    s.kvs = s.v + kTile * D;       // K / V scale per tile row
    s.nk = s.kvs + 2 * kTile;
    s.nv = s.nk + Q * D;           // the Q new rows, as the cache holds them (widened)
    s.ns = s.nv + Q * D;           // their K / V scales
    s.p = s.ns + 2 * Q;            // per warp: the 32 softmax weights of the current tile
    s.total = s.p + kMultiWarps * kTile;
    return s;
}

// The token rows of sequence s: [*base, *base + *cnt). Dense: s*Q and Q. Packed: row_start / row_count; false when the range
// leaves [0, M) or the count exceeds Q (the sequence is then skipped).
__device__ __forceinline__ bool seq_rows(const MultiArgs& p, int s, int64_t* base, int* cnt) {
    if (!p.row_count) {
        *base = int64_t(s) * p.Q;
        *cnt = p.Q;
        return true;
    }
    *base = __ldg(p.row_start + s);
    *cnt = __ldg(p.row_count + s);
    return *cnt >= 0 && *cnt <= p.Q && *base >= 0 && *base + *cnt <= p.M;
}

// Packed: zero the output rows of heads [h0, h0 + GH) between sequence s's last row and the next sequence's first (the
// last sequence: up to M; sequence 0 also those before its first).
__device__ void zero_gaps(const MultiArgs& p, int s, int h0, int GH, int D) {
    const int64_t start = __ldg(p.row_start + s);
    const int64_t end = max(int64_t(0), start + max(0, __ldg(p.row_count + s)));
    const int64_t next = s + 1 < p.num_seqs ? int64_t(__ldg(p.row_start + s + 1)) : p.M;
    const uint16_t zero = 0;
    for (int part = 0; part < 2; ++part) {
        const int64_t lo = part ? end : 0, hi = min(p.M, part ? next : (s == 0 ? start : 0));
        for (int64_t x = threadIdx.x; x < (hi - lo) * GH * D; x += kMultiThreads) {
            const int64_t r = lo + x / (int64_t(GH) * D);
            const int hi_ = int(x / D % GH), d = int(x % D);
            p.out[r * p.out_st + int64_t(h0 + hi_) * p.out_sh + d] = zero;
        }
    }
}

template <typename T, int D, bool kE4M3>
__global__ void __launch_bounds__(kMultiThreads) decode_multi_kernel(const MultiArgs p) {
    using Elem = typename std::conditional<kE4M3, uint8_t, uint16_t>::type;
    constexpr int DPL = D / 32;   // output dims per lane
    extern __shared__ float smem[];
    const int Q = p.Q, GH = p.heads_per_cache;
    const MultiSmem L = multi_smem(GH * Q, Q, D);
    float* s_q = smem + L.q;
    float* s_acc = smem + L.acc;
    float* s_ml = smem + L.ml;
    float* s_k = smem + L.k;
    float* s_v = smem + L.v;
    float* s_kvs = smem + L.kvs;
    float* s_nk = smem + L.nk;
    float* s_nv = smem + L.nv;
    float* s_ns = smem + L.ns;
    float* s_p = smem + L.p;

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int split = blockIdx.x, c = blockIdx.y, s = blockIdx.z;
    const int heads = p.Hq / GH;                                       // cache heads per sequence
    const int64_t sc = int64_t(s) * heads + c;                         // (sequence, cache head)
    const int kvh = GH > 1 ? c : c / p.G;                              // the kv head whose new rows this cache head takes
    const int h0 = GH > 1 ? c * GH : c;                                // first query head
    if (p.row_count && split == 0) zero_gaps(p, s, h0, GH, D);
    int64_t base;                                                      // token row of the sequence's query 0
    int cnt;                                                           // its new rows (queries per head)
    if (!seq_rows(p, s, &base, &cnt) || cnt == 0) return;
    const int M = GH * cnt;
    Elem* kc = static_cast<Elem*>(p.k_cache) + int64_t(s) * p.cache_sb + int64_t(c) * p.cache_sh;
    Elem* vc = static_cast<Elem*>(p.v_cache) + int64_t(s) * p.cache_sb + int64_t(c) * p.cache_sh;
    const int64_t scale_off = int64_t(s) * p.scale_sb + int64_t(c) * p.scale_sh;

    int64_t n0 = p.T;   // rows held before this step's Q rows
    if (p.step_dev) n0 += int64_t(__ldg(p.step_dev));
    if (p.rows) n0 += int64_t(__ldg(p.rows + sc));
    const bool valid = n0 >= 0 && n0 + cnt <= p.max_rows;
    const int64_t rows = valid ? n0 + cnt : 0;                         // the largest attended count
    const int64_t ns = min(int64_t(p.nsplit), decode_splits_for(p.Hq, rows, p.num_sms));
    const int64_t chunk = (rows + ns - 1) / ns;
    const int64_t r_begin = int64_t(split) * chunk;
    const int64_t r_end = min(rows, r_begin + chunk);

    // queries (fp32) and fresh accumulators
    for (int x = tid; x < M * D; x += kMultiThreads) {
        const int i = x / D, d = x % D, hi = i / cnt, j = i % cnt;
        const uint16_t* src = p.q + (base + j) * p.q_st + int64_t(h0 + hi) * p.q_sh;
        s_q[x] = DT<T>::to_f32(src[d]);
        s_acc[x] = 0.f;
    }
    for (int i = tid; i < M; i += kMultiThreads) {
        s_ml[2 * i] = -INFINITY;
        s_ml[2 * i + 1] = 0.f;
    }
    // the Q new rows: warp w builds rows w, w + 8, ... of K and V (lane l holds dims l*DPL .. l*DPL + DPL - 1)
    for (int x = warp; x < 2 * cnt; x += kMultiWarps) {
        const int j = x >> 1, which = x & 1;
        const uint16_t* src = (which ? p.v_new : p.k_new) + (base + j) * p.kv_st + int64_t(kvh) * p.kv_sh + lane * DPL;
        float v[DPL];
#pragma unroll
        for (int e = 0; e < DPL; ++e) v[e] = DT<T>::to_f32(src[e]);
        float* dst = (which ? s_nv : s_nk) + j * D + lane * DPL;
        const int64_t row = n0 + j;
        const bool store = valid && split == 0;
        if constexpr (kE4M3) {
            float amax = 0.f;
#pragma unroll
            for (int e = 0; e < DPL; ++e) amax = fmaxf(amax, fabsf(v[e]));
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, o));
            float scale = 0.f;
            uint8_t bytes[DPL];
            if (amax != 0.f) {
                const float inv = __fdiv_rn(kE4M3Max, amax);
                scale = __fdiv_rn(amax, kE4M3Max);
#pragma unroll
                for (int e = 0; e < DPL; e += 2) {
                    const uint16_t two = __nv_cvt_float2_to_fp8x2(make_float2(__fmul_rn(v[e], inv), __fmul_rn(v[e + 1], inv)),
                                                                  __NV_SATFINITE, __NV_E4M3);
                    bytes[e] = uint8_t(two & 0xffu);
                    bytes[e + 1] = uint8_t(two >> 8);
                }
            } else {
#pragma unroll
                for (int e = 0; e < DPL; ++e) bytes[e] = 0;
            }
#pragma unroll
            for (int e = 0; e < DPL; e += 2) {
                const __half2 h2(__nv_cvt_fp8x2_to_halfraw2(__nv_fp8x2_storage_t(bytes[e] | (uint16_t(bytes[e + 1]) << 8)), __NV_E4M3));
                const float2 f2 = __half22float2(h2);
                dst[e] = f2.x;
                dst[e + 1] = f2.y;
            }
            if (lane == 0) s_ns[2 * j + which] = scale;
            if (store) {
                Elem* crow = (which ? vc : kc) + row * D + lane * DPL;
#pragma unroll
                for (int e = 0; e < DPL; ++e) crow[e] = bytes[e];
                if (lane == 0) (which ? p.v_scale : p.k_scale)[scale_off + row] = scale;
            }
        } else {
#pragma unroll
            for (int e = 0; e < DPL; ++e) dst[e] = v[e];
            if (lane == 0) s_ns[2 * j + which] = 1.f;
            if (store) {
                Elem* crow = (which ? vc : kc) + row * D + lane * DPL;
#pragma unroll
                for (int e = 0; e < DPL; ++e) crow[e] = src[e];
            }
        }
    }
    __syncthreads();

    for (int64_t t0 = r_begin; t0 < r_end; t0 += kTile) {
        // stage the tile: cached rows from global memory, new rows from shared memory
        constexpr int E = kE4M3 ? 16 : 8, LPR = D / E;   // one 128-bit load per thread and row piece
        for (int x = tid; x < kTile * LPR; x += kMultiThreads) {
            const int r = x / LPR, d0 = (x % LPR) * E;
            const int64_t row = t0 + r;
            float kf[16], vf[16];
#pragma unroll
            for (int e = 0; e < E; ++e) kf[e] = vf[e] = 0.f;
            if (row < r_end) {
                if (row >= n0) {
#pragma unroll
                    for (int e = 0; e < E; ++e) {
                        kf[e] = s_nk[int(row - n0) * D + d0 + e];
                        vf[e] = s_nv[int(row - n0) * D + d0 + e];
                    }
                } else {
                    const uint4 kv = *reinterpret_cast<const uint4*>(kc + row * D + d0);
                    const uint4 vv = *reinterpret_cast<const uint4*>(vc + row * D + d0);
                    if constexpr (kE4M3) {
                        fp8x16_to_f32(kv, kf);
                        fp8x16_to_f32(vv, vf);
                    } else {
                        unpack8<T>(kv, kf);
                        unpack8<T>(vv, vf);
                    }
                }
            }
#pragma unroll
            for (int e = 0; e < E; ++e) {
                s_k[r * (D + 1) + d0 + e] = kf[e];
                s_v[r * D + d0 + e] = vf[e];
            }
        }
        for (int r = tid; r < kTile; r += kMultiThreads) {
            const int64_t row = t0 + r;
            float ks = 1.f, vs = 1.f;
            if constexpr (kE4M3) {
                ks = vs = 0.f;
                if (row < r_end) {
                    if (row >= n0) {
                        ks = s_ns[2 * int(row - n0)];
                        vs = s_ns[2 * int(row - n0) + 1];
                    } else {
                        ks = p.k_scale[scale_off + row];
                        vs = p.v_scale[scale_off + row];
                    }
                }
            }
            s_kvs[2 * r] = ks;
            s_kvs[2 * r + 1] = vs;
        }
        __syncthreads();
        const int64_t row = t0 + lane;
        const float* krow = s_k + lane * (D + 1);
        for (int i = warp; i < M; i += kMultiWarps) {
            const int j = i % cnt;
            const float* qrow = s_q + i * D;
            float dot = 0.f;
#pragma unroll 16
            for (int d = 0; d < D; ++d) dot = fmaf(qrow[d], krow[d], dot);
            const bool vis = row < r_end && row < n0 + j + 1;
            float sc_ = -INFINITY;
            if (vis) sc_ = kE4M3 ? __fmul_rn(__fmul_rn(dot, s_kvs[2 * lane]), p.scale) : __fmul_rn(dot, p.scale);
            float tmax = sc_;
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) tmax = fmaxf(tmax, __shfl_xor_sync(0xffffffffu, tmax, o));
            const float m_old = s_ml[2 * i], l_old = s_ml[2 * i + 1];
            const float mn = fmaxf(m_old, tmax);
            if (mn == -INFINITY) continue;   // nothing visible yet (uniform over the warp)
            const float corr = expf(m_old - mn);
            const float pe = vis ? expf(sc_ - mn) : 0.f;
            float psum = pe;
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) psum += __shfl_xor_sync(0xffffffffu, psum, o);
            s_p[warp * kTile + lane] = kE4M3 ? __fmul_rn(pe, s_kvs[2 * lane + 1]) : pe;
            __syncwarp();
            float* acc = s_acc + i * D;
#pragma unroll
            for (int e = 0; e < DPL; ++e) {
                const int d = lane + 32 * e;
                float a = acc[d] * corr;
#pragma unroll 8
                for (int r = 0; r < kTile; ++r) a = fmaf(s_p[warp * kTile + r], s_v[r * D + d], a);
                acc[d] = a;
            }
            __syncwarp();
            if (lane == 0) {
                s_ml[2 * i] = mn;
                s_ml[2 * i + 1] = __fmaf_rn(l_old, corr, psum);
            }
            __syncwarp();
        }
        __syncthreads();
    }

    for (int x = tid; x < M * D; x += kMultiThreads) {
        const int i = x / D, d = x % D, hi = i / cnt, j = i % cnt;
        const float m = s_ml[2 * i], l = s_ml[2 * i + 1], a = s_acc[x];
        const int64_t h = h0 + hi;
        if (p.nsplit == 1) {
            p.out[(base + j) * p.out_st + h * p.out_sh + d] = DT<T>::from_f32(a / l);
        } else {
            float* w = p.ws + (((int64_t(s) * p.Hq + h) * Q + j) * p.nsplit + split) * (2 + D);
            if (d == 0) { w[0] = m; w[1] = l; }
            w[2 + d] = a;
        }
    }
}

template <typename T, int D>
__global__ void decode_multi_combine_kernel(const MultiArgs p) {   // one CTA per (sequence, query head, query)
    const int64_t x = blockIdx.x;
    const int d = threadIdx.x;
    const int64_t j = x % p.Q, h = (x / p.Q) % p.Hq, s = x / (int64_t(p.Q) * p.Hq);
    int64_t base;
    int cnt;
    if (!seq_rows(p, int(s), &base, &cnt) || j >= cnt) return;   // a row no query of s owns (zeroed by split 0)
    const float* w = p.ws + x * p.nsplit * (2 + D);
    float mn = -INFINITY;
    for (int k = 0; k < p.nsplit; ++k) mn = fmaxf(mn, w[k * (2 + D)]);
    float lt = 0.f, at = 0.f;
    for (int k = 0; k < p.nsplit; ++k) {
        const float ms = w[k * (2 + D)];
        const float c = (ms == -INFINITY) ? 0.f : expf(ms - mn);
        lt += w[k * (2 + D) + 1] * c;
        at += w[k * (2 + D) + 2 + d] * c;
    }
    p.out[(base + j) * p.out_st + h * p.out_sh + d] = DT<T>::from_f32(at / lt);
}

template <typename T, int D, bool kE4M3>
cudaError_t launch_multi_t(const MultiArgs& a, cudaStream_t st) {
    const int M = a.heads_per_cache * a.Q;
    const size_t bytes = size_t(multi_smem(M, a.Q, D).total) * sizeof(float);
    auto kern = decode_multi_kernel<T, D, kE4M3>;
    static size_t granted = 0;   // the attribute is set outside the launches a graph captures (the warm-up step runs first)
    if (bytes > granted) {
        const cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, int(bytes));
        if (e != cudaSuccess) return e;
        granted = bytes;
    }
    const dim3 grid(unsigned(a.nsplit), unsigned(a.Hq / a.heads_per_cache), unsigned(a.num_seqs));
    kern<<<grid, kMultiThreads, bytes, st>>>(a);
    count_launch();
    if (a.nsplit > 1) {
        decode_multi_combine_kernel<T, D><<<unsigned(int64_t(a.num_seqs) * a.Hq * a.Q), D, 0, st>>>(a);
        count_launch();
    }
    return cudaGetLastError();
}

template <typename T, int D>
cudaError_t launch_multi_d(const MultiArgs& a, cudaStream_t st) {
    return a.k_scale ? launch_multi_t<T, D, true>(a, st) : launch_multi_t<T, D, false>(a, st);
}

// ---- prompt lookup and the acceptance step: integer logic, one CTA per sequence ----
constexpr int kSpecThreads = 512;

__device__ __forceinline__ bool is_eos(const SpecArgs& p, int64_t t) {
    for (int k = 0; k < p.n_eos; ++k)
        if (p.eos[k] == t) return true;
    return false;
}

// Rule 1 for sequence b over its history h[0, L): the largest n <= min(N, L - 1) with a start i, i + n < L, h[i, i + n) ==
// h[L - n, L); the lowest such i; the draft h[i + n, min(i + n + K, L)) cut before its first EOS. One pass: for every end
// e = i + n - 1 <= L - 2, c(e) = the length of the common suffix of h[0, e] and h[0, L) (capped at min(N, L - 1)); the lowest
// start for n is then the lowest e with c(e) >= n, minus n - 1. Writes the next verify inputs [last, draft.., pad..], their
// positions L - 1 + j and the draft length.
__device__ void lookup_one(const SpecArgs& p, int b) {
    __shared__ int64_t s_suf[kMaxNgram];
    __shared__ int s_best[kMaxNgram];
    const int64_t* h = p.hist + int64_t(b) * p.hist_cap;
    const int64_t Lh = p.hist_len[b];
    const int Q = p.Q, K = Q - 1;
    const bool draft = !p.done[b] && p.budget[b] > 1 && Lh >= 2;
    const int nmax = draft ? int(min(int64_t(p.N), Lh - 1)) : 0;
    if (threadIdx.x < kMaxNgram) {
        s_best[threadIdx.x] = INT32_MAX;
        if (int(threadIdx.x) < nmax) s_suf[threadIdx.x] = h[Lh - 1 - threadIdx.x];
    }
    __syncthreads();
    if (nmax > 0) {
        int best[kMaxNgram];
#pragma unroll
        for (int k = 0; k < kMaxNgram; ++k) best[k] = INT32_MAX;
        for (int64_t e = threadIdx.x; e <= Lh - 2; e += kSpecThreads) {
            if (h[e] != s_suf[0]) continue;
            int cnt = 1;
            while (cnt < nmax && cnt <= e && h[e - cnt] == s_suf[cnt]) ++cnt;
#pragma unroll
            for (int k = 0; k < kMaxNgram; ++k)
                if (k < cnt && best[k] == INT32_MAX) best[k] = int(e);   // e ascends per thread: the first hit is the lowest
        }
#pragma unroll
        for (int k = 0; k < kMaxNgram; ++k)
            if (k < nmax && best[k] != INT32_MAX) atomicMin(&s_best[k], best[k]);
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        int d = 0;
        int64_t start = 0;
        for (int n = nmax; n >= 1; --n) {
            if (s_best[n - 1] != INT32_MAX) {
                start = int64_t(s_best[n - 1]) + 1;
                d = int(min(int64_t(K), Lh - start));
                break;
            }
        }
        int64_t* ids = p.ids + int64_t(b) * Q;
        int64_t* pos = p.pos + int64_t(b) * Q;
        int kept = 0;
        for (; kept < d; ++kept) {
            const int64_t t = h[start + kept];
            if (is_eos(p, t)) break;
            ids[1 + kept] = t;
        }
        for (int j = 1 + kept; j < Q; ++j) ids[j] = p.pad;
        ids[0] = h[Lh - 1];
        for (int j = 0; j < Q; ++j) pos[j] = Lh - 1 + j;
        p.draft_len[b] = kept;
    }
}

__global__ void __launch_bounds__(kSpecThreads) prompt_lookup_kernel(const SpecArgs p) { lookup_one(p, blockIdx.x); }

// Rule 3, then the row counts of the first (up to 32) layers, then rule 1 for the next step.
__global__ void __launch_bounds__(kSpecThreads) spec_step_kernel(const SpecArgs p) {
    __shared__ int s_n;
    const int b = blockIdx.x, Q = p.Q;
    if (threadIdx.x == 0) {
        int n = 0;
        if (!p.done[b]) {
            const int64_t* t = p.tokens + int64_t(b) * Q;
            const int64_t* ids = p.ids + int64_t(b) * Q;
            const int d = p.draft_len[b];
            int a = 0;
            while (a < d && ids[1 + a] == t[a]) ++a;
            const int m = p.budget[b];
            a = min(a, m - 1);
            int64_t L = p.hist_len[b], o = p.out_len[b];
            bool stop = false;
            for (int k = 0; k <= a && !stop; ++k) {
                const int64_t tok = t[k];
                if (L < p.hist_cap) p.hist[int64_t(b) * p.hist_cap + L] = tok;
                if (o < p.out_cap) p.out[int64_t(b) * p.out_cap + o] = tok;
                ++L;
                ++o;
                ++n;
                stop = is_eos(p, tok);
            }
            p.hist_len[b] = int32_t(L);
            p.out_len[b] = int32_t(o);
            p.budget[b] = m - n;
            if (stop || m - n <= 0) p.done[b] = 1;
        }
        p.emitted[b] = n;
        s_n = n;
    }
    __syncthreads();
    const int n = s_n;
    if (n) {
        for (int x = threadIdx.x; x < p.n_layers * p.H; x += kSpecThreads) p.rows[x / p.H][int64_t(b) * p.H + x % p.H] += n;
    }
    lookup_one(p, b);
}

__global__ void spec_rows_kernel(const SpecArgs p) {   // the row counts of layers past the first 32: one CTA per sequence
    const int b = blockIdx.x, n = p.emitted[b];
    if (!n) return;
    for (int x = threadIdx.x; x < p.n_layers * p.H; x += blockDim.x) p.rows[x / p.H][int64_t(b) * p.H + x % p.H] += n;
}

// ---- rule 2' (pack): one CTA; one scan over the slots in rotation order, then each slot's rows ----
constexpr int kPackThreads = 1024;

// Exclusive block scan of v (all threads take part); *total gets the sum over the block.
__device__ long long block_exclusive_scan(long long v, long long* total) {
    __shared__ long long s_warp[kPackThreads / 32];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    long long x = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const long long y = __shfl_up_sync(0xffffffffu, x, o);
        if (lane >= o) x += y;
    }
    if (lane == 31) s_warp[warp] = x;
    __syncthreads();
    if (warp == 0) {
        long long w = s_warp[lane];
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const long long y = __shfl_up_sync(0xffffffffu, w, o);
            if (lane >= o) w += y;
        }
        s_warp[lane] = w;   // inclusive over warps
    }
    __syncthreads();
    const long long before = (warp ? s_warp[warp - 1] : 0) + x - v;
    *total = s_warp[kPackThreads / 32 - 1];
    __syncthreads();        // s_warp is reused by the next call
    return before;
}

// Slot b at rotation position k = (b - r0) mod B. The scan runs over k and carries (draft tokens wanted, live slots) in one
// 64-bit value: the budget granted before position k is min(P_k, D), so d' = min(want, max(0, D - P_k)), and the rows of
// the positions before k are R_k = L_k + min(P_k, D). Slot order then shifts every start by the rows of slots 0 .. r0 - 1.
__global__ void __launch_bounds__(kPackThreads) spec_pack_kernel(const SpecArgs p, const PackArgs k) {
    __shared__ long long s_r0;   // R of slot 0
    const int B = p.num_seqs, Q = p.Q;
    const int r0 = int(((int64_t(__ldg(k.step)) % B) + B) % B);
    long long carry = 0;         // (wanted << 0) + (live << 32), summed over the positions already scanned
    for (int k0 = 0; k0 < B; k0 += kPackThreads) {
        const int pos = k0 + int(threadIdx.x);
        const int b = pos < B ? (r0 + pos) % B : 0;
        long long want = 0, live = 0;
        if (pos < B && !p.done[b]) {
            live = 1;
            want = max(0, min(p.draft_len[b], p.budget[b] - 1));
        }
        long long total;
        const long long before = carry + block_exclusive_scan(want + (live << 32), &total);
        if (pos < B) {
            const long long P = before & 0xffffffffll, L = before >> 32;
            const int granted = int(min(want, max(0ll, k.D - P)));
            p.draft_len[b] = granted;
            k.row_count[b] = int(live) + granted;
            const long long R = L + min(P, (long long)k.D);
            k.row_start[b] = int(R);   // rotation order for now
            if (b == 0) s_r0 = R;
        }
        carry += total;
    }
    __syncthreads();
    const long long Ptot = carry & 0xffffffffll, Ltot = carry >> 32;
    const long long rows = Ltot + min(Ptot, (long long)k.D);
    const long long shift = r0 ? rows - s_r0 : 0;   // the rows of slots 0 .. r0 - 1
    if (threadIdx.x == 0 && k.totals) {
        k.totals[0] += min(Ptot, (long long)k.D);
        k.totals[1] += Ltot;
    }
    for (int b = threadIdx.x; b < B; b += kPackThreads) {
        const long long R = k.row_start[b];
        const int start = int(b >= r0 ? R + shift : R - s_r0);
        k.row_start[b] = start;
        for (int j = 0; j < k.row_count[b]; ++j) {
            k.ids[start + j] = p.ids[int64_t(b) * Q + j];
            k.pos[start + j] = p.pos[int64_t(b) * Q + j];
        }
    }
    for (long long r = rows + threadIdx.x; r < k.M; r += kPackThreads) {
        k.ids[r] = p.pad;
        k.pos[r] = 0;
    }
}

}  // namespace

cudaError_t launch_spec_pack(const SpecArgs& a, const PackArgs& k, cudaStream_t st) {
    spec_pack_kernel<<<1, kPackThreads, 0, st>>>(a, k);
    count_launch();
    return cudaGetLastError();
}

size_t decode_multi_smem_bytes(int heads_per_cache, int Q, int D) {
    return size_t(multi_smem(heads_per_cache * Q, Q, D).total) * sizeof(float);
}

cudaError_t launch_decode_multi(const MultiArgs& a, cudaStream_t st) {
    if (a.dtype == PKV_BF16) return a.D == 128 ? launch_multi_d<__nv_bfloat16, 128>(a, st) : launch_multi_d<__nv_bfloat16, 64>(a, st);
    return a.D == 128 ? launch_multi_d<__half, 128>(a, st) : launch_multi_d<__half, 64>(a, st);
}

cudaError_t launch_prompt_lookup(const SpecArgs& a, cudaStream_t st) {
    prompt_lookup_kernel<<<unsigned(a.num_seqs), kSpecThreads, 0, st>>>(a);
    count_launch();
    return cudaGetLastError();
}

cudaError_t launch_spec_step(const SpecArgs& a, bool first, cudaStream_t st) {
    if (first) spec_step_kernel<<<unsigned(a.num_seqs), kSpecThreads, 0, st>>>(a);
    else spec_rows_kernel<<<unsigned(a.num_seqs), 256, 0, st>>>(a);
    count_launch();
    return cudaGetLastError();
}

}  // namespace pkv
