// pkv_decode.cu — decode step over the compacted cache: in-place append + attention, one kernel for every cache form.
//
// Replaces, per layer and token: DynamicCache.update's torch.cat of the whole layer cache
// (cache_utils_think.py:383-384, called at llama_model.py:170 / :288 / :403), the two transposes and the
// attention launch (eager llama_model.py:174-183, sdpa :291-313, flash :411-445 -> flash_attn_func :77).
// q_len == 1 and every cached row is visible, so there is no mask. One launch for T <= 256 rows per
// head; longer caches are split along T (flash-decoding) and merged by a second small kernel.
// Several sequences decoded in lock-step share one launch: the grid is (split, cache head part, sequence), and every
// (sequence, head) divides its own rows among the splits a one-sequence launch would use.
// HBM-bound: reads 2*T*D*elem bytes per cache head and sequence; each row is fetched with 128-bit loads, D/8 lanes per row
// for 16-bit rows, D/16 for E4M3 rows (the per-row K scale multiplies the finished dot product and the V scale is folded
// into the softmax weight, so neither costs a multiply per element).
#include "pkv_common.cuh"
#include "pkv_internal.h"
#include "pkv_rows.cuh"

namespace pkv {
namespace {

constexpr int kDecodeThreads = 256;
constexpr int kDecodeWarps = kDecodeThreads / 32;
constexpr int kDecodeUnroll = 4;

struct DecodeParams {
    const uint16_t *q, *k_new, *v_new;   // q [num_seqs][Hq][D], k_new / v_new [num_seqs][Hkv][D]
    void *k_cache, *v_cache;             // cache head c of sequence s at + s*cache_sb + c*cache_sh elements
    uint16_t* out;                       // [num_seqs][Hq][D]
    float *k_scale, *v_scale;            // E4M3 rows: at + s*scale_sb + c*scale_sh
    int64_t cache_sh, cache_sb, scale_sh, scale_sb, T, max_rows;
    int G, nsplit, num_sms;
    int Hq;     // query heads per sequence: the split rule
    float scale;
    float* ws;  // [num_seqs*Hq][nsplit][2 + D] partial (m, l, acc) when nsplit > 1
    const int32_t* step_dev;  // rows = T + *step_dev (graph-replayable decode; the grid is sized for the maximum)
    const int32_t* rows;      // + rows[s*(cache heads) + c] (rows of each sequence and cache head: joined prompts, AdaKV / HeadKV)
    int64_t window;           // decode window R (0: off): rows past prompt_rows[s*(cache heads) + c] form a ring of R rows
    const int32_t* prompt_rows;
    // heavy-hitter window (pkv_decode_attn_heavy): the slot of the next row past a full window, the per-step scratch and the
    // accumulated state (decode_heavy_kernel)
    int32_t* victim;     // [num_seqs*(cache heads)] absolute row index
    float* hv_logit;     // [num_seqs*Hq][window] s of each attended generated row (index row - P)
    float* hv_ml;        // [num_seqs*Hq][2] (m, l) the output of the step is normalised by
    float* hv_scores;    // [num_seqs*(cache heads)][window] accumulated attention A of the row in each slot
    int32_t* hv_gen;     // [num_seqs*(cache heads)][window] generation index of the row in each slot
    int64_t heavy;       // H: rows past the R - H most recent that may stay
    int heads_per_cache;
};

// Decode window modes (template parameter of decode_kernel): none, the ring (oldest row replaced) and heavy hitters (the
// row decode_heavy_kernel chose replaced).
enum WindowMode { kNoWindow = 0, kRing = 1, kHeavy = 2 };

// Row formats. A lane holds kElems elements of a row (one 128-bit load). score() and weight() give the softmax input of a
// row and the factor of its V elements, with the roundings the fp32 online softmax below is defined by.
template <typename T>
struct Rows16 {   // bf16 / fp16 rows, as the eviction wrote them
    using Elem = uint16_t;
    static constexpr int kElems = 8;
    static constexpr bool kE4M3 = false;
    static __device__ __forceinline__ void widen(const uint4& v, float (&f)[kElems]) { unpack8<T>(v, f); }
    static __device__ __forceinline__ float score(float dot, float /*k_scale*/, float scale) { return __fmul_rn(dot, scale); }
    static __device__ __forceinline__ float weight(float pe, float /*v_scale*/) { return pe; }
};
struct RowsE4M3 {   // E4M3 rows with one fp32 scale per row for K and for V (pkv_rows.cuh)
    using Elem = uint8_t;
    static constexpr int kElems = 16;
    static constexpr bool kE4M3 = true;
    static __device__ __forceinline__ void widen(const uint4& v, float (&f)[kElems]) { fp8x16_to_f32(v, f); }
    static __device__ __forceinline__ float score(float dot, float k_scale, float scale) { return __fmul_rn(__fmul_rn(dot, k_scale), scale); }
    static __device__ __forceinline__ float weight(float pe, float v_scale) { return __fmul_rn(pe, v_scale); }
};

// One CTA per (split, cache head part, sequence) attends GH query heads over the rows of its split, loading each row once.
// GH = 1: a cache per query head (h = blockIdx.y; the new row comes from kv head h / G). GH > 1: a GQA-shared cache per KV
// head c, read by its G query heads, GH of them per CTA: blockIdx.y = c * (G / GH) + part, and part 0 appends the new row.
//
// The row count is T (+ *step_dev) (+ rows[...]), read on the device, so that ONE captured launch (CUDA graph) serves every
// decode step; the grid is sized for the capacity, and the rows are divided in-kernel among the splits a launch for the
// current row count would use (the others stay empty), so every launch adds the same terms in the same order: the same
// output bits. The split count is that of Hq query heads, so a sequence gets the same bits in a batch as alone, and every
// head of a shared cache the bits it gets from the repeat-interleaved cache. A row count outside [1, max_rows] (the capacity
// the launch was checked against) is treated as 0: nothing is read or written but the output, which becomes NaN.
// With a decode window (window > 0, pkv_decode_attn_window) the count n past P = prompt_rows[...] wraps: once n > P + window
// the new row goes to P + (n-1-P) mod window and P + window rows are attended, with the split rule of that count.
// Heavy mode (pkv_decode_attn_heavy) goes to victim[s*(cache heads) + c] instead (a victim outside [P, P + window) is treated
// as an out-of-range count), stores the softmax input s of every attended generated row r >= P and query head (the lane of
// piece 0, which holds the reduced dot) at hv_logit[head][r - P], and with nsplit == 1 the (m, l) the output is divided by
// at hv_ml[head] (decode_combine_kernel stores them otherwise). The output arithmetic is the ring's.
//
// Registers: the GH = 1 forms must stay within the ceilings of their occupancy, 80 per thread for 16-bit rows (3 CTAs per
// SM; 64-79 now) and 128 for E4M3 rows (2 CTAs per SM; at 128 now, no headroom). ptxas -v prints the counts. The window mode
// is a template parameter so that the launches without one keep the code (and the speed) they had before it existed.
template <typename T, int D, typename Rows, int GH, int kMode>
__global__ void __launch_bounds__(kDecodeThreads) decode_kernel(const DecodeParams p) {
    using Elem = typename Rows::Elem;
    constexpr int E = Rows::kElems;
    constexpr int LPR = D / E;        // lanes per cached row
    constexpr int RPW = 32 / LPR;     // rows per warp step
    constexpr bool kShared = GH > 1;
    __shared__ float s_m[GH][kDecodeWarps], s_l[GH][kDecodeWarps];
    __shared__ float s_acc[GH][kDecodeWarps][D];
    __shared__ uint4 s_new[2][LPR];   // E4M3: the appended K and V rows and their scales, as stored
    __shared__ float s_new_scale[2];

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int sub = lane / LPR, piece = lane % LPR;
    const int Hkv = p.Hq / p.G, parts = kShared ? p.G / GH : 1;
    const int split = blockIdx.x, c = blockIdx.y / parts, part = blockIdx.y % parts;
    const int64_t sc = int64_t(blockIdx.z) * (kShared ? Hkv : p.Hq) + c;                               // (sequence, cache head)
    const int64_t sk = int64_t(blockIdx.z) * Hkv + (kShared ? c : c / p.G);                           // (sequence, kv head)
    const int64_t sh0 = int64_t(blockIdx.z) * p.Hq + (kShared ? int64_t(c) * p.G : c) + part * GH;   // (sequence, first query head)
    const int64_t cache_off = int64_t(blockIdx.z) * p.cache_sb + int64_t(c) * p.cache_sh;
    const int64_t scale_off = int64_t(blockIdx.z) * p.scale_sb + int64_t(c) * p.scale_sh;
    Elem* kc = static_cast<Elem*>(p.k_cache) + cache_off;
    Elem* vc = static_cast<Elem*>(p.v_cache) + cache_off;
    const uint16_t* k_new = p.k_new + sk * D;
    const uint16_t* v_new = p.v_new + sk * D;
    int64_t rows = p.T;   // logical row count n: the new row is the n-th
    if (p.step_dev) rows += int64_t(__ldg(p.step_dev));
    if (p.rows) rows += int64_t(__ldg(p.rows + sc));
    int64_t ring_row = rows - 1;
    [[maybe_unused]] int64_t P = 0;
    if constexpr (kMode != kNoWindow) {
        // decode window: the prompt's P rows stay, appended row j (= n-1-P) lives at P + j mod R (heavy: at the victim), and
        // P + R rows are attended once the window is full (before that the rows are those of the unwindowed launch)
        if (rows >= 1) {
            P = int64_t(__ldg(p.prompt_rows + sc));
            if (P < 0) {
                rows = 0;
            } else if (rows > P + p.window) {
                if constexpr (kMode == kHeavy) {
                    ring_row = int64_t(p.victim[sc]);
                    rows = (ring_row >= P && ring_row < P + p.window) ? P + p.window : 0;
                } else {
                    ring_row = P + (rows - 1 - P) % p.window;
                    rows = P + p.window;
                }
            }
        }
    }
    if (rows < 1 || rows > p.max_rows) rows = 0;
    const int64_t new_row = kMode != kNoWindow ? ring_row : rows - 1;
    const int64_t ns = min(int64_t(p.nsplit), decode_splits_for(p.Hq, rows, p.num_sms));
    const int64_t chunk = (rows + ns - 1) / ns;
    const int64_t r_begin = int64_t(split) * chunk;
    const int64_t r_end = min(rows, r_begin + chunk);   // may be <= r_begin (empty split): the partial is (-inf, 0, 0)
    const bool own_new = p.k_new != nullptr && new_row >= r_begin && new_row < r_end;   // uniform over the CTA

    // fused append: the CTA that owns the last row stores the new token's K/V
    if constexpr (Rows::kE4M3) {
        // warp 0 quantises the new K row (lane groups 0, 2, ...) and V row (1, 3, ...); groups 0 and 1 store them, and every
        // part keeps them in shared memory to attend the row exactly as the cache holds it
        if (own_new && warp == 0) {
            const int which = sub & 1;
            float x[16];
            load16<T>((which ? v_new : k_new) + piece * 16, x);
            const float amax = row_amax<LPR>(x);
            float s;
            const uint4 qv = quantize16(x, amax, s);
            if (sub < 2) {
                if (part == 0) *reinterpret_cast<uint4*>((which ? vc : kc) + new_row * D + piece * 16) = qv;
                s_new[which][piece] = qv;
                if (piece == 0) {
                    if (part == 0) (which ? p.v_scale : p.k_scale)[scale_off + new_row] = s;
                    s_new_scale[which] = s;
                }
            }
        }
        __syncthreads();
    } else {
        if (own_new && part == 0 && warp == 0 && lane < LPR) {
            *reinterpret_cast<uint4*>(kc + new_row * D + lane * 8) = *reinterpret_cast<const uint4*>(k_new + lane * 8);
            *reinterpret_cast<uint4*>(vc + new_row * D + lane * 8) = *reinterpret_cast<const uint4*>(v_new + lane * 8);
        }
    }

    float qf[GH][E], m[GH], l[GH], acc[GH][E];
#pragma unroll
    for (int i = 0; i < GH; ++i) {
#pragma unroll
        for (int b = 0; b < E; b += 8) unpack8<T>(*reinterpret_cast<const uint4*>(p.q + (sh0 + i) * D + piece * E + b), qf[i] + b);
        m[i] = -INFINITY;
        l[i] = 0.f;
#pragma unroll
        for (int e = 0; e < E; ++e) acc[i][e] = 0.f;
    }

    // warp-uniform trip count (the shuffles below need every lane); rows are checked per lane group
    for (int64_t rb = r_begin + warp * RPW; rb < r_end; rb += int64_t(kDecodeWarps) * RPW * kDecodeUnroll) {
        uint4 kv[kDecodeUnroll], vv[kDecodeUnroll];
        float ks[kDecodeUnroll], vs[kDecodeUnroll];   // E4M3 row scales
        bool ok[kDecodeUnroll];
#pragma unroll
        for (int u = 0; u < kDecodeUnroll; ++u) {
            const int64_t r = rb + sub + int64_t(u) * kDecodeWarps * RPW;
            kv[u] = make_uint4(0, 0, 0, 0);
            vv[u] = make_uint4(0, 0, 0, 0);
            ks[u] = vs[u] = 0.f;
            ok[u] = r < r_end;
            if (ok[u]) {
                const bool is_new = own_new && r == new_row;   // the appended row: from its source
                if constexpr (Rows::kE4M3) {
                    if (is_new) {
                        kv[u] = s_new[0][piece];
                        vv[u] = s_new[1][piece];
                        ks[u] = s_new_scale[0];
                        vs[u] = s_new_scale[1];
                    } else {
                        kv[u] = *reinterpret_cast<const uint4*>(kc + r * D + piece * E);
                        vv[u] = *reinterpret_cast<const uint4*>(vc + r * D + piece * E);
                        ks[u] = p.k_scale[scale_off + r];
                        vs[u] = p.v_scale[scale_off + r];
                    }
                } else {
                    const uint16_t* kr = is_new ? k_new : kc + r * D;
                    const uint16_t* vr = is_new ? v_new : vc + r * D;
                    kv[u] = *reinterpret_cast<const uint4*>(kr + piece * E);
                    vv[u] = *reinterpret_cast<const uint4*>(vr + piece * E);
                }
            }
        }
#pragma unroll
        for (int u = 0; u < kDecodeUnroll; ++u) {
            float kf[E], vf[E];
            Rows::widen(kv[u], kf);
            Rows::widen(vv[u], vf);
#pragma unroll
            for (int i = 0; i < GH; ++i) {
                float dot = 0.f;
#pragma unroll
                for (int e = 0; e < E; ++e) dot = fmaf(qf[i][e], kf[e], dot);
#pragma unroll
                for (int o = 1; o < LPR; o <<= 1) dot += __shfl_xor_sync(0xffffffffu, dot, o);
                if (ok[u]) {   // uniform within the LPR-lane row group
                    // Explicit roundings, so that the compiler cannot contract differently for different GH (a*b + c*d around
                    // either product, or dot * scale into s - mn): every head gets the bits of its per-query-head cache.
                    const float s = Rows::score(dot, ks[u], p.scale);
                    if constexpr (kMode == kHeavy) {   // (32-bit: a row index fits, and the E4M3 GH = 4 form has no registers to spare)
                        const int rel = int(rb - P) + sub + u * kDecodeWarps * RPW;   // generated row rel = r - P
                        if (piece == 0 && rel >= 0) p.hv_logit[(sh0 + i) * p.window + rel] = s;
                    }
                    const float mn = fmaxf(m[i], s);
                    const float corr = expf(m[i] - mn), pe = expf(s - mn);
                    l[i] = __fmaf_rn(l[i], corr, pe);
                    const float pv = Rows::weight(pe, vs[u]);
#pragma unroll
                    for (int e = 0; e < E; ++e) acc[i][e] = __fmaf_rn(acc[i][e], corr, __fmul_rn(pv, vf[e]));
                    m[i] = mn;
                }
            }
        }
    }

    // merge the RPW row groups of each warp (same dims, different rows), then the warps
#pragma unroll
    for (int i = 0; i < GH; ++i) {
#pragma unroll
        for (int o = LPR; o < 32; o <<= 1) {
            const float m2 = __shfl_xor_sync(0xffffffffu, m[i], o);
            const float l2 = __shfl_xor_sync(0xffffffffu, l[i], o);
            const float mn = fmaxf(m[i], m2);
            const float c1 = (mn == -INFINITY) ? 0.f : expf(m[i] - mn), c2 = (mn == -INFINITY) ? 0.f : expf(m2 - mn);
            l[i] = __fmaf_rn(l[i], c1, __fmul_rn(l2, c2));
#pragma unroll
            for (int e = 0; e < E; ++e) {
                const float a2 = __shfl_xor_sync(0xffffffffu, acc[i][e], o);
                acc[i][e] = __fmaf_rn(acc[i][e], c1, __fmul_rn(a2, c2));
            }
            m[i] = mn;
        }
        if (sub == 0) {
            if (piece == 0) { s_m[i][warp] = m[i]; s_l[i][warp] = l[i]; }
#pragma unroll
            for (int e = 0; e < E; ++e) s_acc[i][warp][piece * E + e] = acc[i][e];
        }
    }
    __syncthreads();
    for (int x = tid; x < GH * D; x += kDecodeThreads) {
        const int i = x / D, d = x % D;
        float mn = -INFINITY;
#pragma unroll
        for (int w = 0; w < kDecodeWarps; ++w) mn = fmaxf(mn, s_m[i][w]);
        float lt = 0.f, at = 0.f;
#pragma unroll
        for (int w = 0; w < kDecodeWarps; ++w) {
            const float c = (s_m[i][w] == -INFINITY) ? 0.f : expf(s_m[i][w] - mn);
            lt += s_l[i][w] * c;
            at += s_acc[i][w][d] * c;
        }
        if (p.nsplit == 1) {
            p.out[(sh0 + i) * D + d] = DT<T>::from_f32(at / lt);
            if constexpr (kMode == kHeavy) {
                if (d == 0) { p.hv_ml[2 * (sh0 + i)] = mn; p.hv_ml[2 * (sh0 + i) + 1] = lt; }
            }
        } else {
            float* w = p.ws + ((sh0 + i) * p.nsplit + split) * (2 + D);
            if (d == 0) { w[0] = mn; w[1] = lt; }
            w[2 + d] = at;
        }
    }
}

template <typename T, int D, bool kHeavy>
__global__ void decode_combine_kernel(const DecodeParams p) {   // one CTA per (sequence, head)
    const int64_t h = blockIdx.x;
    const int d = threadIdx.x;
    const float* w = p.ws + int64_t(h) * p.nsplit * (2 + D);
    float mn = -INFINITY;
    for (int s = 0; s < p.nsplit; ++s) mn = fmaxf(mn, w[s * (2 + D)]);
    float lt = 0.f, at = 0.f;
    for (int s = 0; s < p.nsplit; ++s) {
        const float ms = w[s * (2 + D)];
        const float c = (ms == -INFINITY) ? 0.f : expf(ms - mn);
        lt += w[s * (2 + D) + 1] * c;
        at += w[s * (2 + D) + 2 + d] * c;
    }
    p.out[h * D + d] = DT<T>::from_f32(at / lt);
    if constexpr (kHeavy) {
        if (d == 0) { p.hv_ml[2 * h] = mn; p.hv_ml[2 * h + 1] = lt; }
    }
}

// 512 threads: one pass over the slots of a window up to 512 rows. The kernel is latency-bound (a few dependent loads per
// slot), so each thread issues all of its slot's loads before the arithmetic.
constexpr int kHeavyThreads = 512;
constexpr int kHeavyMaxGroup = 8;   // query heads per cache head: 1, or a GQA group of 2, 4 or 8

// (A, generation index) of a victim candidate; the smaller A wins, ties go to the smaller generation index. A total order on
// the distinct generation indices, so the reduction order does not change the winner.
struct HeavyPick {
    float a;
    int32_t g, slot;
};
__device__ __forceinline__ bool heavy_before(const HeavyPick& x, const HeavyPick& y) { return x.a < y.a || (x.a == y.a && x.g < y.g); }

// The heavy-hitter bookkeeping of one decode step, after the decode (and combine) launch: one CTA per (sequence, cache head).
// With n, P and the appended slot as decode_kernel derived them (the same out-of-range rule: nothing is written), the row
// appended as generation j = n-1-P starts from A = 0 with gen = j; every held generated row (slots [0, min(j+1, R)) past P)
// adds sum_h expf(s - m_h) / l_h over the query heads reading this cache head, in ascending head order, in fp32; and when the
// next step's count n + 1 exceeds P + R, victim = P + the slot of the smallest A among the rows of generation index
// <= j + 1 - (R - H). Each thread owns whole slots, so every value is one fixed sequence of fp32 operations: no atomics.
__global__ void __launch_bounds__(kHeavyThreads) decode_heavy_kernel(const DecodeParams p) {
    __shared__ HeavyPick s_best[kHeavyThreads / 32];
    const int64_t sc = blockIdx.x;
    const int heads = p.Hq / p.heads_per_cache;   // cache heads per sequence
    const int64_t sh0 = (sc / heads) * p.Hq + (sc % heads) * p.heads_per_cache;
    int64_t n = p.T;
    if (p.step_dev) n += int64_t(__ldg(p.step_dev));
    if (p.rows) n += int64_t(__ldg(p.rows + sc));
    const int64_t P = int64_t(__ldg(p.prompt_rows + sc)), R = p.window;
    if (n < 1 || P < 0 || n <= P || min(n, P + R) > p.max_rows) return;   // out of range, or an append inside the prompt
    const int64_t slot = n > P + R ? int64_t(p.victim[sc]) : n - 1;
    if (slot < P || slot >= P + R) return;
    const int64_t j = n - 1 - P, held = min(j + 1, R), k_new = slot - P;
    const bool pick = j + 1 >= R;
    const int64_t last = j + 1 - (R - p.heavy);   // the candidates' largest generation index
    float* A = p.hv_scores + sc * R;
    int32_t* gen = p.hv_gen + sc * R;
    HeavyPick best{INFINITY, INT32_MAX, -1};
    float m[kHeavyMaxGroup], l[kHeavyMaxGroup];
#pragma unroll
    for (int h = 0; h < kHeavyMaxGroup; ++h) {
        if (h < p.heads_per_cache) { m[h] = p.hv_ml[2 * (sh0 + h)]; l[h] = p.hv_ml[2 * (sh0 + h) + 1]; }
    }
    for (int64_t k = threadIdx.x; k < held; k += kHeavyThreads) {
        float s[kHeavyMaxGroup];
#pragma unroll
        for (int h = 0; h < kHeavyMaxGroup; ++h) {
            if (h < p.heads_per_cache) s[h] = p.hv_logit[(sh0 + h) * R + k];
        }
        float a = 0.f;
        int32_t g = int32_t(j);
        if (k == k_new) gen[k] = g;
        else { a = A[k]; g = gen[k]; }
        float sum = 0.f;   // ascending head order
#pragma unroll
        for (int h = 0; h < kHeavyMaxGroup; ++h) {
            if (h < p.heads_per_cache) sum = __fadd_rn(sum, __fdiv_rn(expf(__fsub_rn(s[h], m[h])), l[h]));
        }
        a = __fadd_rn(a, sum);
        A[k] = a;
        const HeavyPick c{a, g, int32_t(k)};
        if (pick && g <= last && heavy_before(c, best)) best = c;
    }
    if (!pick) return;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        HeavyPick c;
        c.a = __shfl_xor_sync(0xffffffffu, best.a, o);
        c.g = __shfl_xor_sync(0xffffffffu, best.g, o);
        c.slot = __shfl_xor_sync(0xffffffffu, best.slot, o);
        if (heavy_before(c, best)) best = c;
    }
    if ((threadIdx.x & 31) == 0) s_best[threadIdx.x >> 5] = best;
    __syncthreads();
    if (threadIdx.x == 0) {
        for (int w = 1; w < kHeavyThreads / 32; ++w)
            if (heavy_before(s_best[w], best)) best = s_best[w];
        p.victim[sc] = best.slot < 0 ? -1 : int32_t(P + best.slot);   // -1 (no candidate: A is NaN): the next step is out of range
    }
}

template <int D>
__global__ void append_kernel(const DecodeParams p) {  // (pkv_cache_append; decode_kernel appends the new row itself)
    constexpr int LPR = D / 8;
    const int h = blockIdx.x, g = h / p.G, lane = threadIdx.x;
    if (lane >= 2 * LPR) return;
    const bool is_v = lane >= LPR;
    const int piece = lane % LPR;
    const uint16_t* src = (is_v ? p.v_new : p.k_new) + int64_t(g) * D + piece * 8;
    uint16_t* dst = static_cast<uint16_t*>(is_v ? p.v_cache : p.k_cache) + int64_t(h) * p.cache_sh + (p.T - 1) * D + piece * 8;
    *reinterpret_cast<uint4*>(dst) = *reinterpret_cast<const uint4*>(src);
}

DecodeParams make_params(const DecodeArgs& a) {
    DecodeParams p;
    p.q = a.q; p.k_new = a.k_new; p.v_new = a.v_new;
    p.k_cache = a.k_cache; p.v_cache = a.v_cache; p.out = a.out;
    p.k_scale = a.k_scale; p.v_scale = a.v_scale;
    p.cache_sh = a.cache_sh; p.cache_sb = a.cache_sb; p.scale_sh = a.scale_sh; p.scale_sb = a.scale_sb;
    p.T = a.T; p.max_rows = a.max_rows;
    p.G = a.G; p.nsplit = a.nsplit; p.num_sms = a.num_sms;
    p.Hq = a.Hq;
    p.scale = a.scale;
    p.ws = a.ws;
    p.step_dev = a.step_dev;
    p.rows = a.rows;
    p.window = a.window;
    p.prompt_rows = a.prompt_rows;
    p.victim = a.victim;
    p.hv_logit = a.hv_scratch;
    p.hv_ml = a.hv_scratch ? a.hv_scratch + int64_t(a.num_seqs) * a.Hq * a.window : nullptr;
    p.hv_scores = a.hv_scores;
    p.hv_gen = a.hv_gen;
    p.heavy = a.heavy;
    p.heads_per_cache = a.heads_per_cache;
    return p;
}

template <typename T, int D, typename Rows, int kMode>
cudaError_t launch_decode_t(const DecodeArgs& a, cudaStream_t st) {
    const DecodeParams p = make_params(a);
    // query heads per CTA: 1 on a cache per query head; on a shared cache the whole group, for E4M3 at most 4 (the registers
    // of eight heads do not fit)
    const int GH = a.heads_per_cache == 1 ? 1 : Rows::kE4M3 ? min(a.G, 4) : a.G;
    const dim3 grid(unsigned(a.nsplit), unsigned(a.Hq / GH), unsigned(a.num_seqs));
    if (GH == 1) decode_kernel<T, D, Rows, 1, kMode><<<grid, kDecodeThreads, 0, st>>>(p);
    else if (GH == 2) decode_kernel<T, D, Rows, 2, kMode><<<grid, kDecodeThreads, 0, st>>>(p);
    else if (GH == 4) decode_kernel<T, D, Rows, 4, kMode><<<grid, kDecodeThreads, 0, st>>>(p);
    else if (!Rows::kE4M3 && GH == 8) {
        if constexpr (!Rows::kE4M3) decode_kernel<T, D, Rows, 8, kMode><<<grid, kDecodeThreads, 0, st>>>(p);
    } else {
        return cudaErrorInvalidValue;   // no instantiation for this group size
    }
    count_launch();
    if (a.nsplit > 1) {
        decode_combine_kernel<T, D, kMode == kHeavy><<<unsigned(int64_t(a.num_seqs) * a.Hq), D, 0, st>>>(p);
        count_launch();
    }
    if constexpr (kMode == kHeavy) {
        decode_heavy_kernel<<<unsigned(int64_t(a.num_seqs) * (a.Hq / a.heads_per_cache)), kHeavyThreads, 0, st>>>(p);
        count_launch();
    }
    return cudaGetLastError();
}

template <typename T, int D, int kMode>
cudaError_t launch_decode_rows(const DecodeArgs& a, cudaStream_t st) {
    return a.k_scale ? launch_decode_t<T, D, RowsE4M3, kMode>(a, st) : launch_decode_t<T, D, Rows16<T>, kMode>(a, st);
}

template <int kMode>
cudaError_t launch_decode_w(const DecodeArgs& a, cudaStream_t st) {
    if (a.dtype == PKV_BF16) return a.D == 128 ? launch_decode_rows<__nv_bfloat16, 128, kMode>(a, st) : launch_decode_rows<__nv_bfloat16, 64, kMode>(a, st);
    return a.D == 128 ? launch_decode_rows<__half, 128, kMode>(a, st) : launch_decode_rows<__half, 64, kMode>(a, st);
}

}  // namespace

int decode_num_splits(int Hq, int64_t T, int num_sms) { return int(decode_splits_for(Hq, T, num_sms)); }

cudaError_t launch_decode(const DecodeArgs& a, cudaStream_t st) {
    if (a.victim) return launch_decode_w<kHeavy>(a, st);
    return a.window > 0 ? launch_decode_w<kRing>(a, st) : launch_decode_w<kNoWindow>(a, st);
}

cudaError_t launch_append(const DecodeArgs& a, cudaStream_t st) {
    const DecodeParams p = make_params(a);
    if (a.D == 128) append_kernel<128><<<unsigned(a.Hq), 32, 0, st>>>(p);
    else append_kernel<64><<<unsigned(a.Hq), 32, 0, st>>>(p);
    count_launch();
    return cudaGetLastError();
}

}  // namespace pkv
