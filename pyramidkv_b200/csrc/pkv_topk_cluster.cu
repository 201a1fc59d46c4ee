// pkv_topk_cluster.cu — stages 2+3+4 per (layer, query head) on one thread-block CLUSTER.
//
//   select_cluster_kernel<T, POOL, GATHER>
//     POOL   = false : keys come from the pooled scores in the workspace (stage 3 alone: `pkv_stage_topk`)
//     POOL   = true  : the cluster first computes its head's pooled scores itself — softmax(fp32) -> round ->
//                      window-row sum -> round -> 1-D pool (pyramidkv_utils.py:262-269) — straight into the key buffer
//     GATHER = true  : after the selection every CTA of the cluster copies its share of the K/V rows into the cache
//                      (pyramidkv_utils.py:271-282)
//   so `pkv_evict_prefill` is two launches per layer (window scores; select) instead of four.
//
// Top-k (pyramidkv_utils.py:270): the keys of a head are split over the C = 2/4/8 CTAs of the cluster (one SM each,
// C*Hq <= #SMs). The k-th largest key is found by a radix select with THREE DSMEM exchanges in total: the cluster-wide
// min/max (bits shared by all keys are skipped), then one or two 256-bin histogram passes over the remaining bits;
// every CTA st.async's its histogram into every peer's shared memory (completion counted on the receiver's mbarrier —
// no cluster barrier, no fence), sums the C histograms and finds the bin by a suffix scan. The per-CTA histograms also
// give every CTA the output offsets of its winners. For k <= 1024 the winners are broadcast to every CTA, each CTA
// RANKS its k/C share against all k (k^2/C comparisons, no sort network, no barrier) and immediately copies the K/V
// rows of exactly those winners; larger k falls back to a bitonic sort in the leader CTA. Same tie rule as topk_kernel
// (pkv_topk.cu): all keys above the k-th value, then the lowest indices among equals; order (value desc, index asc).
// Deterministic.
#include <algorithm>

#include "pkv_common.cuh"
#include "pkv_internal.h"

namespace pkv {
namespace {

constexpr int kThreads = 512;
constexpr int kWarps = kThreads / 32;
constexpr uint32_t kH = 0x80008000u;
constexpr int kMaxCluster = 8;
constexpr int kMaxPad = 32;     // kernel_size <= 65
constexpr int kMaxW = 64;
constexpr int kBins = 256;        // histogram bins per radix pass
constexpr int kRankMaxK = 1024;   // k up to this: distributed rank sort (k^2/C comparisons); above: bitonic sort in the leader

struct SelectParams {
    // ---- top-k ----
    const uint16_t* scores;  // [Hq][pitch] pooled scores (read when !POOL, written when POOL)
    uint16_t* scores_out;
    int64_t pitch;
    int n, n8, k, P;         // n8 = ceil(n/8) key words; P = power of two >= max(k, 2)
    int rank_path;           // 1: k <= rank_limit() -> broadcast + rank sort; 0: bitonic sort in the leader
    int sort_cap;            // u64 entries at the start of dynamic smem: P (leader sort buffer) or blk (my outgoing block)
    int words_per_cta;       // ceil(n8 / C)
    int hist_off;            // byte offset of the histogram exchange area in dynamic shared memory (16-byte aligned)
    int stage_off, kcap, blk; // rank path: staging area [C][blk] u64 (blk = k + 1 rounded up to even: count + winners), kcap = k rounded up to even
    int radix_off;           // leader-sort path: byte offset of the second [k] u64 buffer of the LSD radix sort (0 = bitonic network instead)
    int32_t* idx32;          // [Hq][k]
    int64_t* idx64;          // optional [Hq][k]
    // ---- pool (POOL) ----
    const uint16_t* logits;  // [Hkv][s_pad][NW]
    const float2* partial;   // [Hkv][n_slots][NW]
    int64_t s_pad, n_slots;
    int W, G, NW, kernel, pooling;
    int score_grid, tiles_per_g, total_tiles;
    int g_base;              // layer batch: kv heads of the layers in front of this one (the score kernel numbers kv heads across layers)
    // ---- gather (GATHER) ----
    const uint16_t* src[2];
    int64_t s_sh[2], s_ss[2];
    uint16_t* dst[2];
    int64_t cache_sh, S;
    int D;
    unsigned long long* stamps;   // diagnostics (PKV_STAMPS=1), else nullptr
};

// ---- cluster / DSMEM primitives ----
__device__ __forceinline__ uint32_t cluster_ctarank() { uint32_t r; asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r)); return r; }
__device__ __forceinline__ uint32_t cluster_nctarank() { uint32_t r; asm volatile("mov.u32 %0, %%cluster_nctarank;" : "=r"(r)); return r; }
__device__ __forceinline__ void cluster_sync() {
    asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}
__device__ __forceinline__ uint32_t map_remote(const void* local_smem, uint32_t rank) {
    uint32_t la = static_cast<uint32_t>(__cvta_generic_to_shared(local_smem)), ra;
    asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(ra) : "r"(la), "r"(rank));
    return ra;
}
__device__ __forceinline__ void st_remote_u64(uint32_t raddr, uint64_t v) {
    asm volatile("st.shared::cluster.u64 [%0], %1;" ::"r"(raddr), "l"(v) : "memory");
}
// asynchronous 8-byte store into another CTA's shared memory that completes 8 bytes on that CTA's mbarrier: the DSMEM
// mailbox primitive (no cluster-wide barrier, no memory fence on the critical path)
__device__ __forceinline__ void st_async_u64(uint32_t raddr, uint64_t v, uint32_t rbar) {
    asm volatile("st.async.weak.shared::cluster.mbarrier::complete_tx::bytes.b64 [%0], %1, [%2];" ::"r"(raddr), "l"(v), "r"(rbar) : "memory");
}
// bulk copy of `bytes` (multiple of 16, 16-byte aligned both sides) from MY shared memory into a peer CTA's shared memory:
// ONE transaction that completes `bytes` on the receiver's mbarrier (hundreds of 8-byte st.async's serialise on it).
// Generic-proxy writes to the source must be fenced (fence_proxy_async) and barrier'd before the issuing thread gets here,
// and the source CTA must stay alive until the receiver has the data (cluster_arrive_relaxed / cluster_wait below).
__device__ __forceinline__ void bulk_copy_to_peer(uint32_t remote_dst, const void* local_src, uint32_t bytes, uint32_t remote_bar) {
    asm volatile("cp.async.bulk.shared::cluster.shared::cta.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(remote_dst), "r"(static_cast<uint32_t>(__cvta_generic_to_shared(local_src))), "r"(bytes), "r"(remote_bar) : "memory");
}
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void cluster_arrive_relaxed() { asm volatile("barrier.cluster.arrive.relaxed.aligned;" ::: "memory"); }
__device__ __forceinline__ void cluster_wait() { asm volatile("barrier.cluster.wait.aligned;" ::: "memory"); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(static_cast<uint32_t>(__cvta_generic_to_shared(bar))), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(static_cast<uint32_t>(__cvta_generic_to_shared(bar))), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    asm volatile(
        "{\n"
        ".reg .pred P1;\n"
        "LAB_WAIT:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 P1, [%0], %1;\n"
        "@P1 bra DONE;\n"
        "bra LAB_WAIT;\n"
        "DONE:\n"
        "}\n" ::"r"(static_cast<uint32_t>(__cvta_generic_to_shared(bar))), "r"(parity) : "memory");
}

// ---- SWAR compare of 8 packed 16-bit keys against one candidate (see pkv_topk.cu) ----
__device__ __forceinline__ uint32_t ge_mask2(uint32_t a, uint32_t cl2, bool ctop) {
    const uint32_t t = (a | kH) - cl2;
    return ctop ? (t & a & kH) : ((t | a) & kH);
}
__device__ __forceinline__ uint32_t ge_bits8(uint4 v, uint32_t cand) {   // cand in [0, 0xffff]
    const uint32_t cl2 = (cand & 0x7fffu) * 0x10001u;
    const bool ctop = (cand & 0x8000u) != 0;
    return ge_mask2(v.x, cl2, ctop) | (ge_mask2(v.y, cl2, ctop) >> 1) | (ge_mask2(v.z, cl2, ctop) >> 2) | (ge_mask2(v.w, cl2, ctop) >> 3);
}
// order-preserving key of two packed 16-bit floats: bits ^ (sign ? 0xffff : 0x8000)
__device__ __forceinline__ uint32_t sort_key2(uint32_t u) {
    const uint32_t sign = (u >> 15) & 0x00010001u;
    return u ^ ((sign * 0x7fffu) | 0x80008000u);
}

// layer batch (pkv_evict_prefill_batch): blockIdx.z = layer, every layer with its own budget k (hence its own shared-memory
// layout), score rows, index outputs and K / V source and cache pointers. LB = 1 is the per-layer launch.
template <int LB> struct SelectLayers { SelectParams p[LB]; };

// OCC: CTAs per SM the register allocation aims at.
// SOLO (layer batch): one CTA per head, launched without a cluster. Heads outnumber the SMs many times over, so the kernel
// wants throughput: every exchange becomes CTA-local (__syncthreads, the CTA's own histograms and winner list), the
// leader-sort path reuses the dead key buffer for its radix buffers (two CTAs per SM at k ~ 4K, 32K tokens), and the gather
// takes the indices from shared memory.
template <typename T, bool POOL, bool GATHER, int LB, int OCC = 1, bool SOLO = false>
__global__ void __launch_bounds__(kThreads, OCC) select_cluster_kernel(const __grid_constant__ SelectLayers<LB> layers) {
    static_assert(!(SOLO && POOL), "the one-CTA form reads pooled scores");
    const SelectParams& p = layers.p[LB == 1 ? 0 : blockIdx.z];
    extern __shared__ __align__(16) uint8_t smem_raw[];
    uint64_t* sortbuf = reinterpret_cast<uint64_t*>(smem_raw);                  // [P] (used in the leader CTA only)
    uint4* keys_s = reinterpret_cast<uint4*>(smem_raw + size_t(p.sort_cap) * 8); // [words_per_cta]
    float* sbuf = reinterpret_cast<float*>(keys_s + p.words_per_cta);           // [words_per_cta*8 + 2*pad] window sums (POOL)
    uint32_t* hist_all = reinterpret_cast<uint32_t*>(smem_raw + p.hist_off);   // [2 passes][C][kBins] every CTA's histograms (!SOLO)
    int2* mine_s = SOLO ? reinterpret_cast<int2*>(smem_raw + p.hist_off)       // [ceil(k/C) + 1] (output row, token) of my winners
                        : reinterpret_cast<int2*>(hist_all + 2 * kMaxCluster * kBins);
    uint64_t* stage_in = reinterpret_cast<uint64_t*>(smem_raw + p.stage_off);  // [C][blk] every CTA's {count, winners...} (rank path)
    uint64_t* flat_s = stage_in + size_t(kMaxCluster) * p.blk;                 // [k] all winners, concatenated in rank order
    __shared__ int gt_cnt_s[kMaxCluster];
    __shared__ __align__(16) uint32_t hist_loc[2][kBins];
    __shared__ __align__(8) uint64_t hbar[2], wbar;                             // histogram / winner broadcast mbarriers
    __shared__ int pick_s[2];
    __shared__ int wsum_s[kBins / 32];
    __shared__ uint32_t scan_s[kWarps];
    __shared__ __align__(8) uint64_t slots[2][kMaxCluster];                     // all-gather mailboxes (double-buffered)
    __shared__ __align__(8) uint64_t xbar[2];                                   // one mbarrier per mailbox buffer
    __shared__ StatR stat[POOL ? kMaxW : 1];
    __shared__ __align__(16) StatP stat_p[POOL ? kMaxW / 2 : 1];                // the same as packed row pairs (fp32 pair operands as loaded)

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const uint32_t rank = SOLO ? 0u : cluster_ctarank(), C = SOLO ? 1u : cluster_nctarank();
    const int h = blockIdx.y;
    const int w_begin = min(int(rank) * p.words_per_cta, p.n8), w_end = min(w_begin + p.words_per_cta, p.n8);
    const int nw = w_end - w_begin;                                             // my key words (possibly 0)
    int xchg = 0;                                                                // mailbox parity
    unsigned long long* const stamps = (tid == 0 && rank == 0 && blockIdx.y == 0 && blockIdx.z == 0) ? p.stamps : nullptr;
    int stamp_i = 0;
    stamp(stamps, stamp_i++);   // 0: entry
    if (tid == 0 && rank == C - 1 && blockIdx.y == 0 && blockIdx.z == 0) stamp(p.stamps, 43);

    // All-gather of one 64-bit value per CTA through DSMEM mailboxes: thread 0 arms its own mbarrier for C*8 bytes and
    // st.async's its value into slot[rank] of every CTA (each store completes 8 bytes on the RECEIVER's mbarrier); everyone
    // then waits on the local mbarrier only. Two buffers alternate: a CTA can start exchange e+2 only after every CTA has
    // contributed to e+1, i.e. after it finished reading e.
    auto allgather = [&](uint64_t v) -> const uint64_t* {
        const int buf = xchg & 1;
        const uint32_t phase = (xchg >> 1) & 1;
        ++xchg;
        uint64_t* box = slots[buf];
        if (tid == 0) {
            mbar_expect_tx(&xbar[buf], C * 8u);
            for (uint32_t r = 0; r < C; ++r) st_async_u64(map_remote(box + rank, r), v, map_remote(&xbar[buf], r));
        }
        mbar_wait(&xbar[buf], phase);
        return box;
    };

    const bool rank_path = p.rank_path != 0;
    if (!SOLO && tid == 0) {
        mbar_init(&xbar[0], 1);
        mbar_init(&xbar[1], 1);
        mbar_init(&hbar[0], 1);
        mbar_init(&hbar[1], 1);
        mbar_init(&wbar, 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        // each of these is used exactly once per launch: arm them now, the bytes may arrive any time after the barrier below
        mbar_expect_tx(&hbar[0], C * kBins * 4u);
        mbar_expect_tx(&hbar[1], C * kBins * 4u);
        if (rank_path) mbar_expect_tx(&wbar, C * uint32_t(p.blk) * 8u);   // every CTA sends one fixed-size block to every CTA
    }
    for (int i = tid; i < 2 * kBins; i += kThreads) (&hist_loc[0][0])[i] = 0u;
    if (rank == 0 && !rank_path)
        for (int i = tid; i < p.P; i += kThreads) sortbuf[i] = ~0ull;
    if constexpr (SOLO) __syncthreads();
    else cluster_sync();   // mbarriers initialised everywhere, sort buffer cleared: remote traffic may start
    stamp(stamps, stamp_i++);   // 1: first cluster barrier
    // everything above overlaps the previous kernel's tail (PDL)
    pdl_wait();      // the previous kernel has finished writing the logits / partials / scores
    pdl_trigger();
    stamp(stamps, stamp_i++);   // 2: predecessor complete

    // ================= keys of my words: from the workspace, or computed here (stage 2) =================
    uint32_t mn2 = 0xffffffffu, mx2 = 0u;
    auto take_word = [&](int i, uint32_t (&o)[4]) {   // o = 4 words of raw 16-bit scores -> keys; min/max; store
        const int i8 = w_begin + i;
#pragma unroll
        for (int e = 0; e < 4; ++e) o[e] = sort_key2(o[e]);
        if (i8 != p.n8 - 1) {
            mx2 = __vimax3_u16x2(mx2, o[0], o[1]); mx2 = __vimax3_u16x2(mx2, o[2], o[3]);
            mn2 = __vimin3_u16x2(mn2, o[0], o[1]); mn2 = __vimin3_u16x2(mn2, o[2], o[3]);
        } else {                        // last word of the row: keys beyond n become 0 (never above a real key, highest indices)
            const int valid = p.n - i8 * 8;
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                if (2 * e >= valid) o[e] = 0u;
                else if (2 * e + 1 >= valid) o[e] &= 0xffffu;
            }
            for (int e = 0; e < valid; ++e) {
                const uint32_t key = (o[e >> 1] >> ((e & 1) * 16)) & 0xffffu;
                mx2 = __vimax3_u16x2(mx2, key * 0x10001u, key * 0x10001u);
                mn2 = __vimin3_u16x2(mn2, key * 0x10001u, key * 0x10001u);
            }
        }
        keys_s[i] = make_uint4(o[0], o[1], o[2], o[3]);
    };

    if constexpr (!POOL) {
        const uint16_t* row = p.scores + int64_t(h) * p.pitch;
        for (int i0 = tid; i0 < nw; i0 += 4 * kThreads) {   // four loads in flight per thread, then their keys
            uint4 raw[4];
#pragma unroll
            for (int u = 0; u < 4; ++u)
                if (i0 + u * kThreads < nw) raw[u] = *reinterpret_cast<const uint4*>(row + size_t(w_begin + i0 + u * kThreads) * 8);
#pragma unroll
            for (int u = 0; u < 4; ++u)
                if (i0 + u * kThreads < nw) {
                    uint32_t o[4] = {raw[u].x, raw[u].y, raw[u].z, raw[u].w};
                    take_word(i0 + u * kThreads, o);
                }
        }
    } else {
        const int g = h / p.G, col0 = (h % p.G) * p.W;
        const int pad = p.kernel / 2;
        // ---- softmax statistics of this head's W rows: merge the stage-1 partials (slot order => deterministic) ----
        const int n_valid = p.score_grid > 0 ? tc5_slot_count(p.g_base + g, p.tiles_per_g, p.total_tiles, p.score_grid) : int(p.n_slots);
        for (int w = warp; w < p.W; w += kWarps) {
            const StatR merged = warp_merge_partials(p.partial + int64_t(g) * p.n_slots * p.NW + col0 + w, p.NW, n_valid, lane);
            if (lane == 0) {
                stat[w] = merged;
                float* f = reinterpret_cast<float*>(&stat_p[w >> 1]);
                f[w & 1] = -merged.m; f[2 + (w & 1)] = -merged.l; f[4 + (w & 1)] = merged.r;
            }
        }
        __syncthreads();
        // ---- window-row sums s[j] for my tokens plus the pooling halo ----
        const bool is_max = p.pooling == PKV_MAXPOOL;
        const float fill = is_max ? -INFINITY : 0.f;
        const uint16_t* __restrict__ base = p.logits + int64_t(g) * p.s_pad * p.NW + col0;
        const int j_begin = w_begin * 8;
        const int total = nw * 8 + 2 * pad;
        if (p.W == 8) {
            StatP st_p[4];                                                      // the 8 rows' statistics, packed pairs (fp32 pair path)
#pragma unroll
            for (int e = 0; e < 4; ++e) st_p[e] = stat_p[e];
            for (int i0 = 0; i0 < total; i0 += kThreads * 4) {
                uint4 v[4];
                bool ok[4];
#pragma unroll
                for (int u = 0; u < 4; ++u) {                                   // loads first (memory-level parallelism)
                    const int i = i0 + u * kThreads + tid, j = j_begin - pad + i;
                    ok[u] = i < total && j >= 0 && j < p.n;
                    if (ok[u]) v[u] = *reinterpret_cast<const uint4*>(base + int64_t(j) * p.NW);
                }
#pragma unroll
                for (int u = 0; u < 4; ++u) {
                    const int i = i0 + u * kThreads + tid;
                    if (i < total) {
                        float s = fill;
                        if (ok[u]) { float acc = 0.f; window_sum8_packed<T, false>(v[u], st_p, acc); s = round_dt<T>(acc); }   // tokens < n: never masked
                        sbuf[i] = s;
                    }
                }
            }
        } else {
            for (int i = tid; i < total; i += kThreads) {
                const int j = j_begin - pad + i;
                float s = fill;
                if (j >= 0 && j < p.n) {
                    float acc = 0.f;
                    for (int w8 = 0; w8 < p.W; w8 += 8) window_sum8<T>(*reinterpret_cast<const uint4*>(base + int64_t(j) * p.NW + w8), stat + w8, acc);
                    s = round_dt<T>(acc);
                }
                sbuf[i] = s;
            }
        }
        __syncthreads();
        // ---- 1-D pool -> pooled scores (written for inspection / parity checks) -> keys ----
        uint16_t* out_row = p.scores_out + int64_t(h) * p.pitch;
        const float kern_f = float(p.kernel);                     // count_include_pad=True: always / kernel_size
        for (int i = tid; i < nw; i += kThreads) {
            uint32_t o[4];
#pragma unroll
            for (int e2 = 0; e2 < 4; ++e2) {
                float r2[2];
#pragma unroll
                for (int q = 0; q < 2; ++q) {
                    const int t = i * 8 + e2 * 2 + q;           // local token; its window is sbuf[t .. t + 2*pad]
                    float r;
                    if (is_max) {
                        r = -INFINITY;
                        for (int d = 0; d <= 2 * pad; ++d) r = fmaxf(r, sbuf[t + d]);
                    } else {
                        float sum = 0.f;
                        for (int d = 0; d <= 2 * pad; ++d) sum += sbuf[t + d];
                        r = __fdiv_rn(sum, kern_f);
                    }
                    r2[q] = r;
                }
                o[e2] = DT<T>::pack2(r2[0], r2[1]);
            }
            *reinterpret_cast<uint4*>(out_row + size_t(w_begin + i) * 8) = make_uint4(o[0], o[1], o[2], o[3]);
            take_word(i, o);
        }
    }

    stamp(stamps, stamp_i++);   // 3: keys loaded
    // ================= cluster-wide min / max of the real keys =================
    uint32_t kmin = min(mn2 & 0xffffu, mn2 >> 16), kmax = max(mx2 & 0xffffu, mx2 >> 16);
    kmin = __reduce_min_sync(0xffffffffu, kmin);
    kmax = __reduce_max_sync(0xffffffffu, kmax);
    if (lane == 0) { scan_s[warp] = kmin | (kmax << 16); }
    __syncthreads();
    {
        const uint32_t v = lane < kWarps ? scan_s[lane] : 0x0000ffffu;
        kmin = __reduce_min_sync(0xffffffffu, v & 0xffffu);
        kmax = __reduce_max_sync(0xffffffffu, v >> 16);
        if constexpr (!SOLO) {
            const uint64_t* box = allgather(uint64_t(kmin) | (uint64_t(kmax) << 32));
            for (uint32_t r = 0; r < C; ++r) { kmin = min(kmin, uint32_t(box[r] & 0xffffu)); kmax = max(kmax, uint32_t(box[r] >> 32)); }
        }
    }

    stamp(stamps, stamp_i++);   // 4: min/max exchanged

    // ---- k-th largest key = largest v with count(key >= v) >= k. Bits above `nbits` are common to all real keys; the
    //      remaining bits are resolved by one (nbits <= 8) or two 256-bin histogram passes. ----
    const int nbits = 32 - __clz(kmin ^ kmax);                   // 0 when all keys are equal
    const uint32_t common = (nbits >= 16) ? 0u : (kmax >> nbits) << nbits;
    const bool two_pass = nbits > 8;
    const int shift1 = two_pass ? nbits - 8 : 0;
    const uint32_t mask1 = two_pass ? 0xffu : ((1u << nbits) - 1u);
    const uint32_t mask2 = (1u << shift1) - 1u;

    // histogram of my real keys: pass 0 on bits [shift1, shift1+8), pass 1 on the low shift1 bits of the keys in bin `sel`.
    // Branch-free (one predicated shared-memory reduction per key): every instruction here is paid by 16 warps.
    auto build_hist = [&](int pass, uint32_t sel) {
        uint32_t* hl = hist_loc[pass];
        for (int i = tid; i < nw; i += kThreads) {
            const uint4 v = keys_s[i];
            const uint32_t u[4] = {v.x, v.y, v.z, v.w};
            const int valid = p.n - (w_begin + i) * 8;             // < 8 only in the last word of the row
#pragma unroll
            for (int e = 0; e < 8; ++e) {
                const uint32_t key = (e & 1) ? (u[e >> 1] >> 16) : (u[e >> 1] & 0xffffu);
                const uint32_t hi = (key >> shift1) & mask1;
                const uint32_t bin = pass == 0 ? hi : (key & mask2);
                const bool take = e < valid && (pass == 0 || hi == sel);
                if (take) atomicAdd(&hl[bin], 1u);
            }
        }
        if constexpr (!SOLO) fence_proxy_async();      // the atomics above are read by the async proxy below
        __syncthreads();
        stamp(stamps, 32 + 2 * pass);
        if constexpr (SOLO) return;   // pick_bin reads this CTA's histogram in place
        // broadcast my histogram: one 1 KB bulk copy to each of the C CTAs (completes on the receiver's mbarrier)
        if (tid < int(C))
            bulk_copy_to_peer(map_remote(hist_all + (size_t(pass) * kMaxCluster + rank) * kBins, uint32_t(tid)), hl, kBins * 4u,
                              map_remote(&hbar[pass], uint32_t(tid)));
        mbar_wait(&hbar[pass], 0);
        stamp(stamps, 33 + 2 * pass);
        if (pass == 1 && tid == 0 && rank == C - 1 && blockIdx.y == 0 && blockIdx.z == 0) stamp(p.stamps, 46);
    };
    // bin B = largest bin whose suffix count reaches `need`; returns B and the number of keys in the bins above it
    auto pick_bin = [&](int pass, int need, int& B, int& above) {
        const uint32_t* ha = SOLO ? hist_loc[pass] : hist_all + size_t(pass) * kMaxCluster * kBins;
        int tot = 0;
        if (tid < kBins)
            for (uint32_t r = 0; r < C; ++r) tot += int(ha[r * kBins + tid]);
        int suf = tot;                                            // inclusive suffix sum inside the warp (32 bins)
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const int t = __shfl_down_sync(0xffffffffu, suf, o);
            if (lane + o < 32) suf += t;
        }
        if (tid < kBins && lane == 0) wsum_s[warp] = suf;
        __syncthreads();
        if (tid < kBins) {
            for (int w2 = warp + 1; w2 < kBins / 32; ++w2) suf += wsum_s[w2];
            if (suf >= need && suf - tot < need) { pick_s[0] = tid; pick_s[1] = suf - tot; }
        }
        __syncthreads();
        B = pick_s[0];
        above = pick_s[1];
    };

    int B1 = 0, above1 = 0, B2 = 0, above2 = 0;
    build_hist(0, 0u);
    pick_bin(0, p.k, B1, above1);
    stamp(stamps, stamp_i++);   // 5: first histogram pass
    if (two_pass) {
        build_hist(1, uint32_t(B1));
        pick_bin(1, p.k - above1, B2, above2);
    }
    stamp(stamps, stamp_i++);   // 6: second histogram pass
    const uint32_t thr = common | (uint32_t(B1) << shift1) | uint32_t(B2);
    const int count_gt = above1 + above2;
    const int need = p.k - count_gt;                              // ties to take, lowest index first (>= 1)

    // ---- ties held by the CTAs before me (ties are taken lowest index first, cluster-wide): one histogram entry per CTA ----
    int tie_base = 0;
    {
        const uint32_t* hl = hist_all + (two_pass ? size_t(kMaxCluster) * kBins + B2 : size_t(B1));
        for (uint32_t r = 0; r < rank; ++r) tie_base += int(hl[r * kBins]);
    }
    int gt_base = 0;                             // keys above thr held by the CTAs before me: only the leader-sort path needs it
    if (!SOLO && !rank_path) {
        if (warp < int(C)) {
            const uint32_t* h1 = hist_all + size_t(warp) * kBins;
            const uint32_t* h2 = hist_all + (size_t(kMaxCluster) + warp) * kBins;
            int part = 0;
            for (int bb = lane; bb < kBins; bb += 32) {
                if (bb > B1) part += int(h1[bb]);
                if (two_pass && bb > B2) part += int(h2[bb]);
            }
            part = __reduce_add_sync(0xffffffffu, part);
            if (lane == 0) gt_cnt_s[warp] = part;
        }
        __syncthreads();
        for (uint32_t r = 0; r < rank; ++r) gt_base += gt_cnt_s[r];
    }
    stamp(stamps, stamp_i++);   // 7: bases
    if (tid == 0 && rank == C - 1 && blockIdx.y == 0 && blockIdx.z == 0) stamp(p.stamps, 47);

    // ---- emit my winners. Thread t owns the contiguous words [t*wpt, (t+1)*wpt) so ONE block scan gives index-order slots:
    //      into my own staging block (k <= 1024: {count, keys above thr..., my ties...}; broadcast below) or straight into
    //      the LEADER's sort buffer (DSMEM stores) ----
    const int wpt = (p.words_per_cta + kThreads - 1) / kThreads;
    const int wt_begin = min(tid * wpt, nw), wt_end = min(wt_begin + wpt, nw);
    uint32_t my_g = 0, my_t = 0;
    for (int i = wt_begin; i < wt_end; ++i) {
        const uint4 v = keys_s[i];
        const uint32_t ge = ge_bits8(v, thr);
        const uint32_t gt = (thr < 0xffffu && ge) ? ge_bits8(v, thr + 1) : 0u;
        my_g += __popc(gt);
        my_t += __popc(ge & ~gt);
    }
    uint32_t inc_g = my_g, inc_t = my_t;         // two independent inclusive scans (tie counts can exceed 16 bits)
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const uint32_t a = __shfl_up_sync(0xffffffffu, inc_g, o), b2 = __shfl_up_sync(0xffffffffu, inc_t, o);
        if (lane >= o) { inc_g += a; inc_t += b2; }
    }
    __shared__ uint32_t wtot_g[kWarps], wtot_t[kWarps];
    if (lane == 31) { wtot_g[warp] = inc_g; wtot_t[warp] = inc_t; }
    __syncthreads();
    uint32_t cta_g = 0, cta_t = 0;               // my CTA's totals
    {
        const uint32_t wg = lane < kWarps ? wtot_g[lane] : 0u, wt = lane < kWarps ? wtot_t[lane] : 0u;
        uint32_t ig = wg, it = wt;
#pragma unroll
        for (int o = 1; o < kWarps; o <<= 1) {
            const uint32_t a = __shfl_up_sync(0xffffffffu, ig, o), b2 = __shfl_up_sync(0xffffffffu, it, o);
            if (lane >= o) { ig += a; it += b2; }
        }
        cta_g = __shfl_sync(0xffffffffu, ig, kWarps - 1);
        cta_t = __shfl_sync(0xffffffffu, it, kWarps - 1);
        inc_g += __shfl_sync(0xffffffffu, ig - wg, warp);
        inc_t += __shfl_sync(0xffffffffu, it - wt, warp);
    }
    const int taken_t = max(0, min(int(cta_t), need - tie_base));       // my ties that make it
    const uint32_t sort_remote = SOLO ? 0u : map_remote(sortbuf, 0);
    if (my_g + my_t) {
        int gt_pos = int(inc_g - my_g);                             // among MY keys above thr, index order
        int tie_pos = int(inc_t - my_t);                            // among MY ties, index order
        for (int i = wt_begin; i < wt_end; ++i) {
            const uint4 v = keys_s[i];
            const uint32_t u[4] = {v.x, v.y, v.z, v.w};
            const uint32_t ge = ge_bits8(v, thr);
            if (!ge) continue;
            const uint32_t gt = (thr < 0xffffu) ? ge_bits8(v, thr + 1) : 0u;
            const int i8 = w_begin + i;
#pragma unroll
            for (int e = 0; e < 8; ++e) {
                const int bit = ((e & 1) ? 31 : 15) - (e >> 1);
                if ((ge >> bit) & 1u) {
                    const uint32_t key = (u[e >> 1] >> ((e & 1) * 16)) & 0xffffu;
                    const uint64_t comp = (uint64_t(0xffffu - key) << 32) | uint64_t(uint32_t(i8 * 8 + e));
                    if ((gt >> bit) & 1u) {
                        if (rank_path) sortbuf[1 + gt_pos] = comp;
                        else if (SOLO) sortbuf[gt_pos] = comp;
                        else st_remote_u64(sort_remote + uint32_t(gt_base + gt_pos) * 8u, comp);
                        ++gt_pos;
                    } else {
                        if (tie_base + tie_pos < need) {
                            if (rank_path) sortbuf[1 + int(cta_g) + tie_pos] = comp;
                            else if (SOLO) sortbuf[count_gt + tie_pos] = comp;
                            else st_remote_u64(sort_remote + uint32_t(count_gt + tie_base + tie_pos) * 8u, comp);
                        }
                        ++tie_pos;
                    }
                }
            }
        }
    }
    if (rank_path) {
        // ================= k <= 1024: distributed rank sort + gather of exactly my winners =================
        if (tid == 0) sortbuf[0] = uint64_t(int(cta_g) + taken_t);      // block header: how many winners follow
        if constexpr (!SOLO) fence_proxy_async();
        __syncthreads();
        stamp(stamps, 36);
        if (tid == 0 && rank == C - 1 && blockIdx.y == 0 && blockIdx.z == 0) stamp(p.stamps, 44);
#ifdef PKV_STAMPS_BUILD
        if (tid == 0 && blockIdx.y == 0 && blockIdx.z == 0 && p.stamps) { stamp(p.stamps, 48 + int(rank)); p.stamps[56 + rank] = (uint64_t(cta_g) << 32) | cta_t; }
#endif
        // SOLO: the CTA holds all k winners already; they are the flat list
        const uint64_t* flat = SOLO ? sortbuf + 1 : flat_s;
        if constexpr (!SOLO) {
            if (tid < int(C))          // my block -> row `rank` of every CTA's staging area, one transaction each
                bulk_copy_to_peer(map_remote(stage_in + size_t(rank) * p.blk, uint32_t(tid)), sortbuf, uint32_t(p.blk) * 8u,
                                  map_remote(&wbar, uint32_t(tid)));
            mbar_wait(&wbar, 0);       // every CTA's block has landed in MY staging area
            cluster_arrive_relaxed();  // (peers may still be reading my block / histograms: I must not exit before they all got here)
            if (tid == 0 && rank == C - 1 && blockIdx.y == 0 && blockIdx.z == 0) stamp(p.stamps, 45);
            stamp(stamps, stamp_i);   // 8: winners broadcast
            // flat list of all k winners in CTA order (any order would do: composites are unique, the rank is a count)
            for (int t = tid; t < p.k; t += kThreads) {
                uint64_t cand = ~0ull;
                int rem = t;
                for (uint32_t r = 0; r < C; ++r) {
                    const int c = int(stage_in[size_t(r) * p.blk]);
                    if (rem >= 0 && rem < c) cand = stage_in[size_t(r) * p.blk + 1 + rem];
                    rem -= c;
                }
                flat_s[t] = cand;
            }
        }
        ++stamp_i;
        const int s_begin = int((int64_t(rank) * p.k) / int(C)), s_end = int((int64_t(rank + 1) * p.k) / int(C));
        const int n_mine = s_end - s_begin;
        if constexpr (!SOLO) __syncthreads();
        stamp(stamps, 37);
        // 8 lanes per winner, 64 winners per step: each lane counts the candidates below its winner in its slice of the
        // flat list (independent loads; composites are unique, so the rank is that count)
        {
            const int gi = tid >> 3, sub8 = tid & 7;
            for (int e0 = 0; e0 < n_mine; e0 += kThreads / 8) {
                const int e = e0 + gi;
                const bool active = e < n_mine;
                const uint64_t me = active ? flat[s_begin + e] : 0ull;
                int below = 0;
                if (active) {
#pragma unroll 4
                    for (int j = sub8; j < p.k; j += 8) below += (flat[j] < me) ? 1 : 0;
                }
                below += __shfl_xor_sync(0xffffffffu, below, 1);
                below += __shfl_xor_sync(0xffffffffu, below, 2);
                below += __shfl_xor_sync(0xffffffffu, below, 4);
                if (active && sub8 == 0) {
                    const int32_t idx = int32_t(uint32_t(me & 0xffffffffull));
                    p.idx32[int64_t(h) * p.k + below] = idx;
                    if (p.idx64) p.idx64[int64_t(h) * p.k + below] = int64_t(idx);
                    mine_s[e] = make_int2(below, idx);
                }
            }
        }
        stamp(stamps, stamp_i++);   // 9: ranked, indices written
        if constexpr (GATHER) {
            __syncthreads();
            // ---- stage 4 for my winners (+ my share of the window rows): half-warp (D=128) / quarter-warp (D=64) per
            //      16-byte piece of a row; K and V rows of two units in flight per lane ----
            const int lpr = p.D / 8, rpw = 32 / lpr;
            const int subrow = lane / lpr, piece = lane % lpr;
            const int n_win = (p.W > int(rank)) ? (p.W - 1 - int(rank)) / int(C) + 1 : 0;
            const int total = n_mine + n_win;
            const int kvh = h / p.G;
            const uint16_t* srcK = p.src[0] + int64_t(kvh) * p.s_sh[0];
            const uint16_t* srcV = p.src[1] + int64_t(kvh) * p.s_sh[1];
            uint16_t* dstK = p.dst[0] + int64_t(h) * p.cache_sh;
            uint16_t* dstV = p.dst[1] + int64_t(h) * p.cache_sh;
            const int stride = kWarps * rpw;
            for (int u0 = warp * rpw + subrow; u0 < total; u0 += 2 * stride) {
                int64_t tok[2], row[2];
                uint4 vk[2], vv[2];
#pragma unroll
                for (int x = 0; x < 2; ++x) {
                    const int u = u0 + x * stride;
                    tok[x] = -1; row[x] = 0;
                    if (u < n_mine) { const int2 m = mine_s[u]; row[x] = m.x; tok[x] = m.y; }
                    else if (u < total) { const int w = int(rank) + (u - n_mine) * int(C); row[x] = p.k + w; tok[x] = p.S - p.W + w; }
                }
#pragma unroll
                for (int x = 0; x < 2; ++x)
                    if (tok[x] >= 0) {
                        vk[x] = ldg_nc_v4(srcK + tok[x] * p.s_ss[0] + piece * 8);
                        vv[x] = ldg_nc_v4(srcV + tok[x] * p.s_ss[1] + piece * 8);
                    }
#pragma unroll
                for (int x = 0; x < 2; ++x)
                    if (tok[x] >= 0) {
                        *reinterpret_cast<uint4*>(dstK + row[x] * p.D + piece * 8) = vk[x];
                        *reinterpret_cast<uint4*>(dstV + row[x] * p.D + piece * 8) = vv[x];
                    }
            }
        }
        stamp(stamps, stamp_i++);   // 10: done
        if constexpr (!SOLO) cluster_wait();   // everyone has received everything this CTA sent: its shared memory may go away
        return;
    }

    // ================= k > 1024: bitonic sort in the leader, then the whole cluster gathers =================
    if constexpr (SOLO) __syncthreads();
    else cluster_sync();          // every winner is in the leader's sort buffer
    if (!GATHER && rank != 0) return;

    uint64_t* sorted = sortbuf;
    if (rank == 0) {
        if (p.radix_off) {
            // ---- leader: stable LSD radix sort on the 16-bit inverted score (4 passes x 4 bits). The winners arrived in index
            //      order (above-threshold block, then the ties, CTA by CTA), so stability alone yields (score desc, index asc).
            //      Thread t owns the contiguous elements [t*E, (t+1)*E): per-thread digit counts are packed bytes, one
            //      block-wide scan over [16 digits][512 threads] gives every thread its 16 write cursors. ~20 barriers in
            //      all, against 78 for the bitonic network at k = 3978. ----
            uint64_t* const buf0 = sortbuf;
            uint64_t* const buf1 = reinterpret_cast<uint64_t*>(smem_raw + p.radix_off);
            // [16][kThreads]: the histograms are dead by now (SOLO: behind buf1, in the dead key buffer)
            uint16_t* cnt = SOLO ? reinterpret_cast<uint16_t*>(smem_raw + p.radix_off + ((size_t(p.k) * 8 + 15) & ~size_t(15)))
                                 : reinterpret_cast<uint16_t*>(hist_all);
            __shared__ uint32_t wsum[kWarps];
            const int E = (p.k + kThreads - 1) / kThreads;                          // <= 16 (k <= 8192)
            const int e0 = min(tid * E, p.k), e1 = min(e0 + E, p.k);
            int cur = 0;
#pragma unroll 1
            for (int pass = 0; pass < 4; ++pass) {
                const uint64_t* src = cur ? buf1 : buf0;
                uint64_t* dst = cur ? buf0 : buf1;
                const int sh = 32 + 4 * pass;
                unsigned long long c_lo = 0ull, c_hi = 0ull;                        // counts of digits 0-7 / 8-15, one byte each
                for (int e = e0; e < e1; ++e) {
                    const uint32_t d = uint32_t(src[e] >> sh) & 15u;
                    if (d < 8) c_lo += 1ull << (8 * d); else c_hi += 1ull << (8 * (d - 8));
                }
#pragma unroll
                for (int d = 0; d < 16; ++d) cnt[d * kThreads + tid] = uint16_t(((d < 8 ? c_lo >> (8 * d) : c_hi >> (8 * (d - 8)))) & 0xffu);
                __syncthreads();
                // exclusive scan of the flattened [digit][thread] table: thread t takes entries [16t, 16t + 16) (one digit per warp)
                uint32_t loc[16], tot = 0;
#pragma unroll
                for (int x = 0; x < 16; ++x) { loc[x] = tot; tot += cnt[16 * tid + x]; }
                uint32_t inc = tot;
#pragma unroll
                for (int o = 1; o < 32; o <<= 1) { const uint32_t v = __shfl_up_sync(0xffffffffu, inc, o); if (lane >= o) inc += v; }
                if (lane == 31) wsum[warp] = inc;
                __syncthreads();
                uint32_t base = inc - tot;
                for (int w2 = 0; w2 < warp; ++w2) base += wsum[w2];
#pragma unroll
                for (int x = 0; x < 16; ++x) cnt[16 * tid + x] = uint16_t(base + loc[x]);   // k <= 8192 fits 16 bits
                __syncthreads();
                uint32_t cursor[16];
#pragma unroll
                for (int d = 0; d < 16; ++d) cursor[d] = cnt[d * kThreads + tid];
                for (int e = e0; e < e1; ++e) {
                    const uint64_t v = src[e];
                    const uint32_t d = uint32_t(v >> sh) & 15u;
                    uint32_t pos = 0;
#pragma unroll
                    for (int x = 0; x < 16; ++x) if (uint32_t(x) == d) { pos = cursor[x]; cursor[x] = pos + 1; }
                    dst[pos] = v;
                }
                __syncthreads();
                cur ^= 1;
            }
            sorted = cur ? buf1 : buf0;                                             // 4 passes: back in sortbuf
        } else {
        // ---- leader: bitonic sort (ascending composite = score descending, index ascending); see pkv_topk.cu ----
        const int pairs = p.P >> 1;
        const int sort_threads = min(kThreads, (pairs + 31) & ~31);
        if (tid < sort_threads) {
            for (int size = 2; size <= p.P; size <<= 1) {
                for (int stride = size >> 1; stride > 0; stride >>= 1) {
                    for (int t = tid; t < pairs; t += kThreads) {
                        const int i = 2 * t - (t & (stride - 1));
                        const int j = i + stride;
                        const bool up = (i & size) == 0;
                        const uint64_t x = sortbuf[i], y = sortbuf[j];
                        if ((x > y) == up) { sortbuf[i] = y; sortbuf[j] = x; }
                    }
                    const int next_stride = (stride > 1) ? (stride >> 1) : size;
                    if (stride >= 32 || next_stride >= 32) asm volatile("bar.sync 1, %0;" ::"r"(sort_threads) : "memory");
                    else __syncwarp();
                }
            }
        }
        }
        __syncthreads();
        for (int r = tid; r < p.k; r += kThreads) {
            const uint32_t idx = uint32_t(sorted[r] & 0xffffffffull);
            p.idx32[int64_t(h) * p.k + r] = int32_t(idx);
            if (p.idx64) p.idx64[int64_t(h) * p.k + r] = int64_t(idx);
        }
        if (GATHER && !SOLO) __threadfence();   // idx32 must be visible to the other CTAs of the cluster
    }
    stamp(stamps, stamp_i++);   // 19: sorted + indices written
    if constexpr (GATHER && SOLO) {
        // ---- stage 4 from the sorted list in shared memory: K and V rows of four slots in flight per lane ----
        const int lpr = p.D / 8, rpw = 32 / lpr;
        const int rows = p.k + p.W;
        const int sub = lane / lpr, piece = lane % lpr;
        const int kvh = h / p.G;
        const uint16_t* srcK = p.src[0] + int64_t(kvh) * p.s_sh[0];
        const uint16_t* srcV = p.src[1] + int64_t(kvh) * p.s_sh[1];
        uint16_t* dstK = p.dst[0] + int64_t(h) * p.cache_sh;
        uint16_t* dstV = p.dst[1] + int64_t(h) * p.cache_sh;
        const int stride = kWarps * rpw;
        for (int r0 = warp * rpw + sub; r0 < rows; r0 += stride * 4) {
            uint4 vk[4], vv[4];
            int64_t tok[4];
#pragma unroll
            for (int u = 0; u < 4; ++u) {
                const int r = r0 + u * stride;
                tok[u] = -1;
                if (r < rows) tok[u] = (r < p.k) ? int64_t(uint32_t(sorted[r] & 0xffffffffull)) : (p.S - p.W + (r - p.k));
            }
#pragma unroll
            for (int u = 0; u < 4; ++u)
                if (tok[u] >= 0) {
                    vk[u] = ldg_nc_v4(srcK + tok[u] * p.s_ss[0] + piece * 8);
                    vv[u] = ldg_nc_v4(srcV + tok[u] * p.s_ss[1] + piece * 8);
                }
#pragma unroll
            for (int u = 0; u < 4; ++u)
                if (tok[u] >= 0) {
                    const int64_t o = int64_t(r0 + u * stride) * p.D + piece * 8;
                    *reinterpret_cast<uint4*>(dstK + o) = vk[u];
                    *reinterpret_cast<uint4*>(dstV + o) = vv[u];
                }
        }
    } else if constexpr (GATHER) {
        cluster_sync();
        stamp(stamps, stamp_i++);   // 20
        // ---- stage 4: rows r = rank, rank + C, ... of this head; half-warp (D=128) / quarter-warp (D=64) per 16-byte piece ----
        const int lpr = p.D / 8;                       // lanes per row
        const int rpw = 32 / lpr;                      // rows per warp step
        const int rows = p.k + p.W;
        const int sub = lane / lpr, piece = lane % lpr;
        const int32_t* idx = p.idx32 + int64_t(h) * p.k;
        const int kvh = h / p.G;
#pragma unroll
        for (int which = 0; which < 2; ++which) {
            const uint16_t* src = (which ? p.src[1] : p.src[0]) + int64_t(kvh) * (which ? p.s_sh[1] : p.s_sh[0]);
            uint16_t* dst = (which ? p.dst[1] : p.dst[0]) + int64_t(h) * p.cache_sh;
            const int64_t ss = which ? p.s_ss[1] : p.s_ss[0];
            // row slots are dealt round-robin over (CTA, warp, sub-group); 4 independent loads in flight per lane
            const int stride = int(C) * kWarps * rpw;
            for (int r0 = (int(rank) * kWarps + warp) * rpw + sub; r0 < rows; r0 += stride * 4) {
                uint4 v[4];
                int64_t tok[4];
#pragma unroll
                for (int u = 0; u < 4; ++u) {
                    const int r = r0 + u * stride;
                    tok[u] = -1;
                    if (r < rows) tok[u] = (r < p.k) ? int64_t(__ldcg(idx + r)) : (p.S - p.W + (r - p.k));
                }
#pragma unroll
                for (int u = 0; u < 4; ++u)
                    if (tok[u] >= 0) v[u] = ldg_nc_v4(src + tok[u] * ss + piece * 8);
#pragma unroll
                for (int u = 0; u < 4; ++u)
                    if (tok[u] >= 0) *reinterpret_cast<uint4*>(dst + int64_t(r0 + u * stride) * p.D + piece * 8) = v[u];
            }
        }
    }
    stamp(stamps, stamp_i++);   // 21 (20 without gather): done
}

constexpr size_t kSmemBudget = 200 * 1024;
constexpr size_t kExclusiveSmem = 116 * 1024;   // > 227 KB / 2

int next_pow2(int64_t v) { int p = 2; while (p < v) p <<= 1; return p; }

int pick_cluster(const EvictArgs& a) {
    int c = kMaxCluster;
    while (c > 1 && a.Hq * c > a.num_sms) c >>= 1;
    return c;
}

// Largest k that takes the distributed rank sort (k^2 / C comparisons); above it the leader sorts (LSD radix sort). Per-layer launch:
// 1024 (the cluster has the SM to itself and the distributed form has the shorter critical path). Layer batch: 512 - with four
// clusters' CTAs sharing an SM the k^2 work is what counts. Experiment knob PKV_RANK_MAX (<= kRankMaxK) overrides both.
int rank_limit(bool batch = false) {
    static const int v = [] { const char* e = getenv("PKV_RANK_MAX"); const int x = e ? atoi(e) : 0; return x < kRankMaxK ? x : kRankMaxK; }();
    return v > 0 ? v : batch ? 512 : kRankMaxK;
}

int blk_entries(const EvictArgs& a) { return int((a.k + 2) & ~int64_t(1)); }   // count + k winners, even (16-byte multiple)

constexpr int kRadixMaxK = 8192;   // leader-sort path: LSD radix sort (16-bit cursors, second buffer in shared memory) up to this k

size_t select_smem(const EvictArgs& a, int c, bool pool, size_t* hist_off = nullptr, size_t* stage_off = nullptr, size_t* radix_off = nullptr,
                   bool batch = false) {
    const int64_t n8 = (a.n + 7) / 8, words = (n8 + c - 1) / c;
    const bool rank_path = a.k <= rank_limit(batch);
    if (batch && c == 1) {
        // one CTA per head (SOLO): sort buffer / winner list, keys, then the (row, token) list of the rank path. The radix
        // sort's second buffer and digit table reuse the key buffer, dead once the winners are listed.
        size_t b = size_t(rank_path ? blk_entries(a) : next_pow2(a.k > 0 ? a.k : 1)) * 8;
        size_t keys = size_t(words) * 16;
        if (!rank_path && a.k <= kRadixMaxK) {
            if (radix_off) *radix_off = b;
            keys = std::max(keys, ((size_t(a.k) * 8 + 15) & ~size_t(15)) + size_t(16) * kThreads * sizeof(uint16_t));
        }
        b = (b + keys + 15) & ~size_t(15);
        if (hist_off) *hist_off = b;
        if (rank_path) b += (size_t(a.k) + 2) * sizeof(int2);
        return b;
    }
    // sort buffer of the leader (bitonic path) / my outgoing block (rank path)
    size_t b = size_t(rank_path ? blk_entries(a) : next_pow2(a.k > 0 ? a.k : 1)) * 8 + size_t(words) * 16;
    if (pool) b += (size_t(words) * 8 + 2 * kMaxPad) * sizeof(float);
    b = (b + 15) & ~size_t(15);
    if (hist_off) *hist_off = b;
    b += size_t(2) * kMaxCluster * kBins * 4;                 // every CTA's two histograms
    b += (size_t(a.k) / c + 2) * sizeof(int2);                // (output row, token) of the winners this CTA ranks
    b = (b + 15) & ~size_t(15);
    if (stage_off) *stage_off = b;
    if (rank_path) {
        b += size_t(kMaxCluster) * blk_entries(a) * 8;        // every CTA's block
        b += size_t((a.k + 1) & ~int64_t(1)) * 8;             // flat list
        b += (size_t(a.k) / c + 2) * sizeof(int);             // rank accumulators
    } else if (a.k <= kRadixMaxK) {
        b = (b + 15) & ~size_t(15);
        if (radix_off) *radix_off = b;
        b += size_t((a.k + 1) & ~int64_t(1)) * 8;             // second buffer of the leader's radix sort
    }
    return b;
}

// CTAs per head of the layer batch: one (the SOLO form) where the head's keys and buffers fit one CTA's shared memory, else
// the fewest whose share fits
int batch_cluster(const EvictArgs& a) {
    int c = 1;
    while (c < kMaxCluster && select_smem(a, c, false, nullptr, nullptr, nullptr, true) > kSmemBudget) c <<= 1;
    return c;
}

// one layer's parameters; returns the dynamic shared memory it needs
template <bool POOL, bool GATHER>
size_t fill_select_params(const EvictArgs& a, int c, SelectParams* out, int layer = 0, int n_layers = 1, int batch_grid = 0, bool batch = false) {
    SelectParams p = {};
    p.scores = reinterpret_cast<const uint16_t*>(a.ws_base + a.ws.pooled_off);
    p.scores_out = reinterpret_cast<uint16_t*>(a.ws_base + a.ws.pooled_off);
    p.pitch = a.ws.pooled_pitch;
    p.n = int(a.n);
    p.n8 = int((a.n + 7) / 8);
    p.k = int(a.k);
    p.P = next_pow2(a.k);
    p.words_per_cta = (p.n8 + c - 1) / c;
    p.idx32 = reinterpret_cast<int32_t*>(a.ws_base + a.ws.idx32_off);
    p.idx64 = a.idx_out;
    if (POOL) {
        p.logits = reinterpret_cast<const uint16_t*>(a.ws_base + a.ws.logits_off);
        p.partial = reinterpret_cast<const float2*>(a.ws_base + a.ws.partial_off);
        p.s_pad = a.ws.s_pad; p.n_slots = a.ws.n_slots;
        p.W = a.W; p.G = a.G; p.NW = int(a.ws.nw); p.kernel = a.kernel_size; p.pooling = a.pooling;
        p.score_grid = a.score_impl == 1 ? (n_layers > 1 ? batch_grid : a.score_grid) : 0;
        p.tiles_per_g = int(a.ws.s_pad / kTileTokens);
        p.total_tiles = p.tiles_per_g * a.Hkv * n_layers;
        p.g_base = layer * a.Hkv;
    }
    p.W = a.W; p.G = a.G;
    if (GATHER) {
        p.src[0] = a.kk; p.src[1] = a.vv;
        p.s_sh[0] = a.k_sh; p.s_sh[1] = a.v_sh;
        p.s_ss[0] = a.k_ss; p.s_ss[1] = a.v_ss;
        p.dst[0] = a.k_cache; p.dst[1] = a.v_cache;
        p.cache_sh = a.cache_sh; p.S = a.S; p.D = a.D;
    }
    p.stamps = debug_stamps();
    size_t hist_off = 0, stage_off = 0, radix_off = 0;
    const size_t smem = select_smem(a, c, POOL, &hist_off, &stage_off, &radix_off, batch);
    p.radix_off = int(radix_off);
    p.hist_off = int(hist_off);
    p.stage_off = int(stage_off);
    p.kcap = int((a.k + 1) & ~int64_t(1));
    p.blk = blk_entries(a);
    p.rank_path = a.k <= rank_limit(batch) ? 1 : 0;
    p.sort_cap = p.rank_path ? p.blk : p.P;
    *out = p;
    return smem;
}

template <typename T, bool POOL, bool GATHER, int LB, int OCC = 1, bool SOLO = false>
cudaError_t launch_select_t(const EvictArgs* as, int n, int c, cudaStream_t st, int batch_grid = 0) {
    const EvictArgs& a = as[0];
    SelectLayers<LB> layers;
    size_t smem = 0;
    for (int l = 0; l < LB; ++l) {
        const size_t b = fill_select_params<POOL, GATHER>(as[l < n ? l : 0], c, &layers.p[l], l < n ? l : 0, n, batch_grid, LB > 1);
        if (b > smem) smem = b;
    }
    // Per-layer launch, one CTA per SM: the kernel is a chain of short latency-bound phases, two CTAs sharing an SM's
    // schedulers stretch all of them (and skew the cluster, which waits for its slowest member at every exchange). Asking for
    // more than half of the SM's shared memory keeps the block scheduler from doubling up. A layer batch has many more
    // clusters than SMs and wants throughput, not latency: there the CTAs share SMs as far as their shared memory allows.
    static const bool exclusive = [] { const char* e = getenv("PKV_SELECT_EXCLUSIVE"); return e ? atoi(e) != 0 : true; }();
    const size_t smem_req = (exclusive && LB == 1) ? (smem > kExclusiveSmem ? smem : kExclusiveSmem) : smem;
    auto kern = select_cluster_kernel<T, POOL, GATHER, LB, OCC, SOLO>;
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, int(kSmemBudget));
    if (e != cudaSuccess) return e;
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(unsigned(c), unsigned(a.Hq), unsigned(n));
    cfg.blockDim = dim3(kThreads, 1, 1);
    cfg.dynamicSmemBytes = smem_req;
    cfg.stream = st;
    cudaLaunchAttribute attr[2];
    int na = 0;
    if (!SOLO) {
        attr[na].id = cudaLaunchAttributeClusterDimension;
        attr[na].val.clusterDim.x = unsigned(c);
        attr[na].val.clusterDim.y = 1;
        attr[na].val.clusterDim.z = 1;
        ++na;
    }
    if (pdl_mask() & 4) {
        attr[na].id = cudaLaunchAttributeProgrammaticStreamSerialization;
        attr[na].val.programmaticStreamSerializationAllowed = 1;
        ++na;
    }
    cfg.attrs = attr;
    cfg.numAttrs = unsigned(na);
    e = cudaLaunchKernelEx(&cfg, kern, layers);
    count_launch();
    return e != cudaSuccess ? e : cudaGetLastError();
}

template <bool POOL, bool GATHER>
cudaError_t launch_select(const EvictArgs& a, cudaStream_t st) {
    const int c = pick_cluster(a);
    return a.dtype == PKV_BF16 ? launch_select_t<__nv_bfloat16, POOL, GATHER, 1>(&a, 1, c, st) : launch_select_t<__half, POOL, GATHER, 1>(&a, 1, c, st);
}

template <int OCC, bool SOLO>
cudaError_t launch_select_batch(const EvictArgs* as, int n, int c, cudaStream_t st) {
    return as[0].dtype == PKV_BF16 ? launch_select_t<__nv_bfloat16, false, true, kMaxLayerBatch, OCC, SOLO>(as, n, c, st)
                                   : launch_select_t<__half, false, true, kMaxLayerBatch, OCC, SOLO>(as, n, c, st);
}

}  // namespace

// The cluster variant needs every CTA's share of the keys (plus window sums when pooling) and the leader's sort
// buffer in shared memory, and at least 2 CTAs per head that are all resident at once.
bool topk_cluster_supported(const EvictArgs& a) {
    const int c = pick_cluster(a);
    if (c < 2 || a.k < 1 || a.k > (1 << 14) || a.n >= (int64_t(1) << 20)) return false;   // limits the tests cover (counts are 32-bit)
    return select_smem(a, c, false) <= kSmemBudget;
}
// layer batch: any CTA count per head up to kMaxCluster whose buffers fit
bool select_batch_supported(const EvictArgs& a) {
    if (a.k < 1 || a.k > (1 << 14) || a.n >= (int64_t(1) << 20)) return false;
    if (a.D != 64 && a.D != 128) return false;
    return select_smem(a, batch_cluster(a), false, nullptr, nullptr, nullptr, true) <= kSmemBudget;
}
bool select_fused_supported(const EvictArgs& a, bool pool) {
    const int c = pick_cluster(a);
    if (c < 2 || a.k < 1 || a.k > (1 << 14) || a.n >= (int64_t(1) << 20)) return false;
    if (a.D != 64 && a.D != 128) return false;
    if (pool && (a.W > kMaxW || a.kernel_size / 2 > kMaxPad)) return false;
    return select_smem(a, c, pool) <= kSmemBudget;
}

cudaError_t launch_topk_cluster(const EvictArgs& a, cudaStream_t st) {
    if (a.k == 0) return cudaSuccess;
    return launch_select<false, false>(a, st);
}
// stages 2+3+4 (window methods) or 3+4 (H2O, whose scores are already in the workspace) in one launch
cudaError_t launch_select_fused(const EvictArgs& a, bool pool, cudaStream_t st) {
    return pool ? launch_select<true, true>(a, st) : launch_select<false, true>(a, st);
}
// stages 3+4 of n layers of identical geometry (budgets may differ) in one launch: blockIdx.z = layer
cudaError_t launch_select_layers(const EvictArgs* as, int n, cudaStream_t st) {
    if (n < 1 || n > kMaxLayerBatch) return cudaErrorInvalidValue;
    // one CTA count per launch: the largest any layer needs
    int c = 1, kmax = 0;
    for (int l = 0; l < n; ++l) { c = std::max(c, batch_cluster(as[l])); kmax = std::max(kmax, int(as[l].k)); }
    // Register builds: 40 registers (three 512-thread CTAs per SM) for the rank sort; where the leader sorts, 64 registers for the
    // one-CTA form (two CTAs per SM, which its shared memory allows up to k = 8192 at 32K tokens) and 56 for the cluster form
    if (c == 1) return kmax > rank_limit(true) ? launch_select_batch<2, true>(as, n, c, st) : launch_select_batch<3, true>(as, n, c, st);
    return kmax > kRankMaxK ? launch_select_batch<1, false>(as, n, c, st) : launch_select_batch<3, false>(as, n, c, st);
}

}  // namespace pkv
