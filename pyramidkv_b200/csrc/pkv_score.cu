// pkv_score.cu — stage 1 (mma.sync variant) and stage 2 of the window-scoring eviction.
//
// Stage 1  score_mma_kernel     : logits[g][tok][col] = mask(round(round(K.q)/sqrt(D)))   (model dtype)
//                                 + per-tile softmax partials (max, sumexp) per column.
//                                 Reference ops: pyramidkv_utils.py:253-260 (matmul, /sqrt, mask add).
// Stage 2  softmax_pool_kernel  : p = round(exp(x-M)/L); s = round(sum_w p); pooled = pool1d(s).
//                                 Reference ops: pyramidkv_utils.py:262-269.
//
// K is read ONCE per kv head (GQA-aware): one CTA scores a 128-token tile of one kv head against the
// window rows of all G query heads of the group (columns col = head_in_group*W + w).
#include <cstdlib>

#include "pkv_common.cuh"
#include "pkv_internal.h"

namespace pkv {

namespace {

__device__ __forceinline__ void ldmatrix_x4(uint32_t (&r)[4], uint32_t addr) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];"
                 : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(addr));
}
template <typename T>
__device__ __forceinline__ void mma_16816(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1);
template <>
__device__ __forceinline__ void mma_16816<__nv_bfloat16>(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                 : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
template <>
__device__ __forceinline__ void mma_16816<__half>(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                 : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

struct ScoreParams {
    const uint16_t* q;
    const uint16_t* k;
    int64_t q_sh, q_ss, k_sh, k_ss;
    int64_t S, s_pad, n_slots;
    int W, G, NW;
    float sqrt_d, inv_sqrt_d;
    uint16_t* logits;
    float2* partial;
};

// The reference's rounding chain for one logit (fp32 accumulator in, model-dtype value out), mask excluded.
template <typename T, int D>
__device__ __forceinline__ float finish_logit(float acc, float sqrt_d, float inv_sqrt_d) {
    const float x = round_dt<T>(acc);                                // matmul output in the model dtype
    return round_dt<T>(div_sqrt_d<T, D>(x, sqrt_d, inv_sqrt_d));     // / math.sqrt(head_dim)
}
// attn_weights[..., -W:, -W:] += mask (fp32 {0, finfo.min}); jw = token index inside the window, w = window row
template <typename T>
__device__ __forceinline__ float add_window_mask(float x, int jw, int w) {
    return (jw > w) ? round_dt<T>(x + DT<T>::finfo_min()) : x;
}

template <typename T, int D>
__global__ void __launch_bounds__(256) score_mma_kernel(const ScoreParams p) {
    constexpr int CH = D / 8;  // 16-byte chunks per row
    extern __shared__ __align__(16) uint8_t smem_raw[];
    uint16_t* Ks = reinterpret_cast<uint16_t*>(smem_raw);              // [128][D], chunk-swizzled
    uint16_t* Qs = Ks + kTileTokens * D;                               // [NW][D],  chunk-swizzled
    MS* stat_s = reinterpret_cast<MS*>(Qs + size_t(p.NW) * D);         // [8 warps][NW]

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int tile = blockIdx.x, g = blockIdx.y;
    const int64_t tok0 = int64_t(tile) * kTileTokens;

    // ---- stage the K tile and the group's window rows of Q (cp.async, 16 B per request) ----
    const uint16_t* kg = p.k + int64_t(g) * p.k_sh;
    for (int i = tid; i < kTileTokens * CH; i += 256) {
        const int r = i / CH, c = i % CH;
        const int64_t tok = tok0 + r;
        const bool valid = tok < p.S;
        cp_async16(Ks + (r * CH + (c ^ (r & 7))) * 8, kg + (valid ? tok : 0) * p.k_ss + c * 8, valid);
    }
    for (int i = tid; i < p.NW * CH; i += 256) {
        const int r = i / CH, c = i % CH;
        const int hq = g * p.G + r / p.W, w = r % p.W;
        cp_async16(Qs + (r * CH + (c ^ (r & 7))) * 8, p.q + int64_t(hq) * p.q_sh + (p.S - p.W + w) * p.q_ss + c * 8, true);
    }
    cp_async_commit();
    cp_async_wait<0>();
    __syncthreads();

    // ---- A fragments (this warp's 16 tokens x D) stay in registers for all column tiles ----
    uint32_t a[D / 16][4];
    {
        const int row = warp * 16 + (lane & 15);
#pragma unroll
        for (int ks = 0; ks < D / 16; ++ks) {
            const int chunk = ks * 2 + (lane >> 4);
            ldmatrix_x4(a[ks], static_cast<uint32_t>(__cvta_generic_to_shared(Ks + (row * CH + (chunk ^ (row & 7))) * 8)));
        }
    }

    const int64_t tokA = tok0 + warp * 16 + (lane >> 2), tokB = tokA + 8;
    const bool validA = tokA < p.S, validB = tokB < p.S;
    uint16_t* outA = p.logits + (int64_t(g) * p.s_pad + tokA) * p.NW;
    uint16_t* outB = p.logits + (int64_t(g) * p.s_pad + tokB) * p.NW;

    // only the tile(s) that overlap the last W tokens need the mask (block-uniform branch)
    const bool window_tile = tok0 + kTileTokens > p.S - p.W;
    const int jwA = int(tokA - (p.S - p.W)), jwB = jwA + 8;
    int wbase = 0;   // (nt * 8) % W without a division: W is a multiple of 8
    for (int nt = 0; nt < p.NW / 8; ++nt) {
        float c[4] = {0.f, 0.f, 0.f, 0.f};
        const int qrow = nt * 8 + (lane & 7);
#pragma unroll
        for (int ks = 0; ks < D / 16; ks += 2) {
            uint32_t b[4];
            const int chunk = ks * 2 + (lane >> 3);
            ldmatrix_x4(b, static_cast<uint32_t>(__cvta_generic_to_shared(Qs + (qrow * CH + (chunk ^ (qrow & 7))) * 8)));
            mma_16816<T>(c, a[ks], b[0], b[1]);
            mma_16816<T>(c, a[ks + 1], b[2], b[3]);
        }
        const int col0 = nt * 8 + (lane & 3) * 2;
        float xA0 = finish_logit<T, D>(c[0], p.sqrt_d, p.inv_sqrt_d);
        float xA1 = finish_logit<T, D>(c[1], p.sqrt_d, p.inv_sqrt_d);
        float xB0 = finish_logit<T, D>(c[2], p.sqrt_d, p.inv_sqrt_d);
        float xB1 = finish_logit<T, D>(c[3], p.sqrt_d, p.inv_sqrt_d);
        if (window_tile) {
            const int w0 = wbase + (lane & 3) * 2;
            xA0 = add_window_mask<T>(xA0, jwA, w0); xA1 = add_window_mask<T>(xA1, jwA, w0 + 1);
            xB0 = add_window_mask<T>(xB0, jwB, w0); xB1 = add_window_mask<T>(xB1, jwB, w0 + 1);
        }
        wbase += 8;
        if (wbase == p.W) wbase = 0;
        *reinterpret_cast<uint32_t*>(outA + col0) = uint32_t(DT<T>::from_f32(xA0)) | (uint32_t(DT<T>::from_f32(xA1)) << 16);
        *reinterpret_cast<uint32_t*>(outB + col0) = uint32_t(DT<T>::from_f32(xB0)) | (uint32_t(DT<T>::from_f32(xB1)) << 16);

        // per-column (max, sumexp) over this warp's 16 tokens. The partial sums use the fast exp (ex2.approx): they only
        // feed the softmax denominator, whose last bits already depend on the summation order.
        const float vA0 = validA ? xA0 : -INFINITY, vA1 = validA ? xA1 : -INFINITY;
        const float vB0 = validB ? xB0 : -INFINITY, vB1 = validB ? xB1 : -INFINITY;
        float m0 = fmaxf(vA0, vB0), m1 = fmaxf(vA1, vB1);
#pragma unroll
        for (int o = 4; o < 32; o <<= 1) {
            m0 = fmaxf(m0, __shfl_xor_sync(0xffffffffu, m0, o));
            m1 = fmaxf(m1, __shfl_xor_sync(0xffffffffu, m1, o));
        }
        float l0 = (m0 == -INFINITY) ? 0.f : __expf(vA0 - m0) + __expf(vB0 - m0);
        float l1 = (m1 == -INFINITY) ? 0.f : __expf(vA1 - m1) + __expf(vB1 - m1);
#pragma unroll
        for (int o = 4; o < 32; o <<= 1) {
            l0 += __shfl_xor_sync(0xffffffffu, l0, o);
            l1 += __shfl_xor_sync(0xffffffffu, l1, o);
        }
        if (lane < 4) {
            stat_s[warp * p.NW + col0] = MS{m0, l0};
            stat_s[warp * p.NW + col0 + 1] = MS{m1, l1};
        }
    }
    __syncthreads();
    for (int col = tid; col < p.NW; col += 256) {
        MS acc = stat_s[col];
#pragma unroll
        for (int wv = 1; wv < 8; ++wv) acc = ms_merge(acc, stat_s[wv * p.NW + col]);
        p.partial[(int64_t(g) * p.n_slots + tile) * p.NW + col] = make_float2(acc.m, acc.l);
    }
}

// ------------------------------------------------------------------------------------------------
struct PoolParams {
    const uint16_t* logits;
    const float2* partial;
    int64_t S, n, s_pad, n_slots, pooled_pitch;
    int W, G, NW, kernel, pooling;
    int score_grid, tiles_per_g, total_tiles;   // score_grid > 0: partials come from the wgmma kernel (one per CTA and kv head)
    int early_trigger;
    uint16_t* pooled;
    float inv_w;   // MEAN instantiation only: 1 / W (exact: W is a power of two)
    int Hkv;       // layer batch: kv heads per layer (the score kernel numbers kv heads across the layers)
    const int* done;   // layer-major batch: the partials are laid out per layer. With under_scan the launch runs WHILE the score
    int done_target;   // kernel does and polls done[layer] until it reaches done_target (all score CTAs finished the layer)
    int under_scan;
    int use_merged;    // layer batch: the rows' merged statistics were written by merge_partials_kernel (ly.merged[layer][g * NW + column])
};
// layer batch (pkv_evict_prefill_batch): blockIdx.z = layer; the workspace pointers of each layer travel as a kernel parameter
template <int LB> struct PoolLayers { const uint16_t* logits[LB]; const float2* partial[LB]; uint16_t* pooled[LB]; float4* merged[LB]; };
template <> struct PoolLayers<1> {};

// Layer batch: merges the softmax partials of every (layer, head, window row) ONCE - softmax_pool_kernel runs 32 CTAs per head at
// 32K, each of which would otherwise repeat the merge (two dependent strided reads of the partials at the head of every CTA).
// Same function and slot order as the in-kernel merge: identical statistics. Grid (Hq, layers), one warp per window row.
template <int LB>
__global__ void __launch_bounds__(256) merge_partials_kernel(const PoolParams p, const __grid_constant__ PoolLayers<LB> ly) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int h = blockIdx.x, z = blockIdx.y, g = h / p.G, col0 = (h % p.G) * p.W;
    const int gg = p.done ? g : g + z * p.Hkv;
    pdl_wait();
    pdl_trigger();
    const int n_valid = p.score_grid > 0 ? tc5_slot_count(gg, p.tiles_per_g, p.total_tiles, p.score_grid) : int(p.n_slots);
    for (int w = warp; w < p.W; w += 8) {
        const StatR m = warp_merge_partials(ly.partial[z] + int64_t(g) * p.n_slots * p.NW + col0 + w, p.NW, n_valid, lane);
        if (lane == 0) ly.merged[z][g * p.NW + col0 + w] = make_float4(m.m, m.l, m.r, 0.f);
    }
}

constexpr int kPoolTok = 1024;    // tokens per CTA
constexpr int kPoolMaxPad = 32;   // kernel_size <= 65
constexpr int kPoolMaxW = 64;

// WT: window size known at compile time (8) or 0 = any multiple of 8; KS: pooling kernel size known at compile time
// (5, 7) or 0 = any odd size. The specialised path (WT = 8, KS > 0) is the one the reference's defaults hit.
// MEAN: the window rows are averaged instead of summed (`.mean(dim=-2)`, AdaKV / HeadKV calcul_attn_sore,
// pyramidkv_utils.py:661 / :795): fp32 sum times the exact power of two 1/W, one rounding.
template <typename T, int WT, int KS, bool MEAN = false, int LB = 1>
__global__ void __launch_bounds__(256) softmax_pool_kernel(const PoolParams p, const __grid_constant__ PoolLayers<LB> ly) {
    __shared__ StatR stat[kPoolMaxW];
    __shared__ __align__(16) StatP stat_p[kPoolMaxW / 2];    // the same statistics as packed row pairs {-m, -m'}, {-l, -l'}, {r, r'}: fp32 pair operands as loaded
    __shared__ __align__(16) float sbuf[kPoolTok + 2 * kPoolMaxPad];

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int h = blockIdx.y, g = h / p.G, col0 = (h % p.G) * p.W;
    const int pad = KS > 0 ? KS / 2 : p.kernel / 2;
    const int64_t j0 = int64_t(blockIdx.x) * kPoolTok;
    const bool is_max = p.pooling == PKV_MAXPOOL;
    const float fill = is_max ? -INFINITY : 0.f;
    const uint16_t* lg = p.logits;
    const float2* part = p.partial;
    uint16_t* pooled = p.pooled;
    int gg = g;                                   // kv head index as the score kernel counts it
    if constexpr (LB > 1) {
        lg = ly.logits[blockIdx.z]; part = ly.partial[blockIdx.z]; pooled = ly.pooled[blockIdx.z];
        if (!p.done) gg += int(blockIdx.z) * p.Hkv;      // (the layer-major score walk numbers the kv heads per layer)
    }
    const uint16_t* __restrict__ base = lg + int64_t(g) * p.s_pad * p.NW + col0;
    const int total = kPoolTok + 2 * pad;

    if (LB > 1 && p.under_scan) {
        // Layer-major batch: this launch starts as soon as every CTA of the score launch is resident (programmatic dependent
        // launch; that kernel triggers at its start) and follows it one layer behind: the logits are read back from L2 while
        // the score kernel streams the next layer's K. No griddepcontrol.wait here - it would wait for the whole scan.
        pdl_trigger();
        if (tid == 0) {
            int v;
            do {
                asm volatile("ld.acquire.gpu.global.s32 %0, [%1];" : "=r"(v) : "l"(p.done + blockIdx.z) : "memory");
                if (v < p.done_target) __nanosleep(256);
            } while (v < p.done_target);
        }
        __syncthreads();
    } else {
        pdl_wait();      // stage 1 has finished writing the logits and the softmax partials
        if (p.early_trigger) pdl_trigger();
    }

    constexpr int kIt = (kPoolTok + 2 * kPoolMaxPad + 255) / 256;       // 5 tokens per thread at most
    uint4 v[kIt];
    bool ok[kIt];
    if constexpr (WT == 8) {                                             // all logit loads first: they fly during the merge
        const int64_t jt = j0 - pad + tid;
        const uint16_t* ptr = base + jt * p.NW;
#pragma unroll
        for (int it = 0; it < kIt; ++it) {
            const int64_t j = jt + it * 256;
            ok[it] = (tid + it * 256) < total && j >= 0 && j < p.n;
            if (ok[it]) v[it] = *reinterpret_cast<const uint4*>(ptr + int64_t(it) * 256 * p.NW);
        }
    }

    // merge the softmax partials of this head's W rows (slot order => deterministic), or pick up the merged statistics
    bool have_stats = false;
    if constexpr (LB > 1) {
        if (p.use_merged) {
            if (tid < p.W) {
                const float4 v = ly.merged[blockIdx.z][g * p.NW + col0 + tid];
                stat[tid] = StatR{v.x, v.y, v.z};
                float* f = reinterpret_cast<float*>(&stat_p[tid >> 1]);
                f[tid & 1] = -v.x; f[2 + (tid & 1)] = -v.y; f[4 + (tid & 1)] = v.z;
            }
            have_stats = true;
        }
    }
    if (!have_stats) {
        const int n_valid = p.score_grid > 0 ? tc5_slot_count(gg, p.tiles_per_g, p.total_tiles, p.score_grid) : int(p.n_slots);
        for (int w = warp; w < p.W; w += 8) {
            const StatR merged = warp_merge_partials(part + int64_t(g) * p.n_slots * p.NW + col0 + w, p.NW, n_valid, lane);
            if (lane == 0) {
                stat[w] = merged;
                float* f = reinterpret_cast<float*>(&stat_p[w >> 1]);
                f[w & 1] = -merged.m; f[2 + (w & 1)] = -merged.l; f[4 + (w & 1)] = merged.r;
            }
        }
    }
    __syncthreads();

    if constexpr (WT == 8) {
        StatP st_p[4];                                                   // the 8 rows' statistics live in registers
#pragma unroll
        for (int e = 0; e < 4; ++e) st_p[e] = stat_p[e];
#pragma unroll
        for (int it = 0; it < kIt; ++it) {
            const int i = tid + it * 256;
            if (it < kIt - 1 || i < total) {
                float s = fill;
                // (tokens j < n only: never inside the masked W x W block, so the -150 guard of the exp is not needed: pkv_common.cuh)
                if (ok[it]) { float acc = 0.f; window_sum8_packed<T, false>(v[it], st_p, acc); s = round_dt<T>(acc); }   // sum(dim=-2) in the model dtype
                sbuf[i] = s;
            }
        }
    } else {
        for (int i = tid; i < total; i += 256) {
            const int64_t j = j0 - pad + i;
            float s = fill;
            if (j >= 0 && j < p.n) {
                float acc = 0.f;
                for (int w8 = 0; w8 < p.W; w8 += 8) window_sum8<T>(*reinterpret_cast<const uint4*>(base + j * p.NW + w8), stat + w8, acc);
                if constexpr (MEAN) acc = __fmul_rn(acc, p.inv_w);
                s = round_dt<T>(acc);
            }
            sbuf[i] = s;
        }
    }
    __syncthreads();

    uint16_t* __restrict__ out = pooled + int64_t(h) * p.pooled_pitch;
    if constexpr (KS > 0) {
        // four consecutive tokens per thread: 4 + 2*pad window sums from shared memory as vectors, one 8-byte store
        constexpr int kNv = 4 + 2 * (KS / 2);
        const int t0 = 4 * tid;
        const int64_t j = j0 + t0;
        if (j < p.n) {
            float sv[(kNv + 3) / 4 * 4];
#pragma unroll
            for (int q = 0; q < (kNv + 3) / 4; ++q) {
                const float4 f = *reinterpret_cast<const float4*>(&sbuf[t0 + 4 * q]);
                sv[4 * q] = f.x; sv[4 * q + 1] = f.y; sv[4 * q + 2] = f.z; sv[4 * q + 3] = f.w;
            }
            float r[4];
            if (is_max) {
#pragma unroll
                for (int q = 0; q < 4; ++q) {
                    r[q] = sv[q];
#pragma unroll
                    for (int d = 1; d < KS; ++d) r[q] = fmaxf(r[q], sv[q + d]);
                }
            } else {
                const float ks = float(KS);
#pragma unroll
                for (int q = 0; q < 4; ++q) {
                    float sum = 0.f;
#pragma unroll
                    for (int d = 0; d < KS; ++d) sum += sv[q + d];       // zero padding, ascending order
                    r[q] = __fdiv_rn(sum, ks);                            // count_include_pad=True
                }
            }
            if (j + 3 < p.n) {
                *reinterpret_cast<uint2*>(out + j) = make_uint2(DT<T>::pack2(r[0], r[1]), DT<T>::pack2(r[2], r[3]));
            } else {
#pragma unroll
                for (int q = 0; q < 4; ++q)
                    if (j + q < p.n) out[j + q] = DT<T>::from_f32(r[q]);
            }
        }
    } else {
        for (int t = tid; t < kPoolTok; t += 256) {
            const int64_t j = j0 + t;
            if (j >= p.n) break;
            float r;
            if (is_max) {
                r = -INFINITY;
                for (int d = 0; d <= 2 * pad; ++d) r = fmaxf(r, sbuf[t + d]);
            } else {
                float sum = 0.f;
                for (int d = 0; d <= 2 * pad; ++d) sum += sbuf[t + d];   // zero padding, ascending order
                r = __fdiv_rn(sum, float(p.kernel));                      // count_include_pad=True
            }
            out[j] = DT<T>::from_f32(r);
        }
    }
}

template <typename T, int D>
cudaError_t launch_score_t(const EvictArgs& a, cudaStream_t st) {
    ScoreParams p;
    p.q = a.q; p.k = a.kk;
    p.q_sh = a.q_sh; p.q_ss = a.q_ss; p.k_sh = a.k_sh; p.k_ss = a.k_ss;
    p.S = a.S; p.s_pad = a.ws.s_pad; p.n_slots = a.ws.n_slots;
    p.W = a.W; p.G = a.G; p.NW = int(a.ws.nw);
    p.sqrt_d = sqrtf(float(a.D));
    p.inv_sqrt_d = 1.0f / p.sqrt_d;
    p.logits = reinterpret_cast<uint16_t*>(a.ws_base + a.ws.logits_off);
    p.partial = reinterpret_cast<float2*>(a.ws_base + a.ws.partial_off);
    const size_t smem = size_t(kTileTokens) * D * 2 + size_t(p.NW) * D * 2 + size_t(8) * p.NW * sizeof(MS);
    auto kern = score_mma_kernel<T, D>;
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, int(smem));
    if (e != cudaSuccess) return e;
    const dim3 grid(unsigned(a.ws.s_pad / kTileTokens), unsigned(a.Hkv));
    kern<<<grid, 256, smem, st>>>(p);
    count_launch();
    return cudaGetLastError();
}

}  // namespace

cudaError_t launch_score_mma(const EvictArgs& a, cudaStream_t st) {
    if (a.dtype == PKV_BF16) return a.D == 128 ? launch_score_t<__nv_bfloat16, 128>(a, st) : launch_score_t<__nv_bfloat16, 64>(a, st);
    return a.D == 128 ? launch_score_t<__half, 128>(a, st) : launch_score_t<__half, 64>(a, st);
}

// n == 1: the per-layer launch; n > 1: one launch over n layers of identical geometry (blockIdx.z = layer), whose
// softmax partials were written by ONE score launch over the same n layers (batch_grid = its persistent grid)
cudaError_t launch_softmax_pool_layers(const EvictArgs* as, int n, int batch_grid, cudaStream_t st, const int* done, bool under_scan) {
    if (n < 1 || n > kMaxLayerBatch) return cudaErrorInvalidValue;
    const EvictArgs& a = as[0];
    PoolParams p;
    p.logits = reinterpret_cast<const uint16_t*>(a.ws_base + a.ws.logits_off);
    p.partial = reinterpret_cast<const float2*>(a.ws_base + a.ws.partial_off);
    p.S = a.S; p.n = a.n; p.s_pad = a.ws.s_pad; p.n_slots = a.ws.n_slots; p.pooled_pitch = a.ws.pooled_pitch;
    p.W = a.W; p.G = a.G; p.NW = int(a.ws.nw); p.kernel = a.kernel_size; p.pooling = a.pooling;
    const bool layer_major = n > 1 && done != nullptr;     // partials laid out per layer, exactly like the per-layer launches'
    p.score_grid = a.score_impl == 1 ? ((n > 1 && !layer_major) ? batch_grid : a.score_grid) : 0;
    p.tiles_per_g = int(a.ws.s_pad / kTileTokens);
    p.total_tiles = p.tiles_per_g * a.Hkv * (layer_major ? 1 : n);
    p.Hkv = a.Hkv;
    p.done = layer_major ? done : nullptr;
    p.done_target = a.score_grid;
    p.under_scan = (layer_major && under_scan) ? 1 : 0;
    p.use_merged = 0;
    p.pooled = reinterpret_cast<uint16_t*>(a.ws_base + a.ws.pooled_off);
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(unsigned((a.n + kPoolTok - 1) / kPoolTok), unsigned(a.Hq), unsigned(n));
    cfg.blockDim = dim3(256);
    cfg.dynamicSmemBytes = 0;
    cfg.stream = st;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;   // start while stage 1 drains; the kernel waits itself
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = ((pdl_mask() & 2) || p.under_scan) ? 1 : 0;    // (under_scan: the launch must start WITH the score kernel)
    p.early_trigger = (pdl_mask() & 8) ? 1 : 0;
    const int ks = (a.W == 8 && (a.kernel_size == 7 || a.kernel_size == 5)) ? a.kernel_size : 0;
    cudaError_t e;
    p.inv_w = 1.0f / float(a.W);
    if (n > 1) {
        if (a.window_mean) return cudaErrorInvalidValue;     // AdaKV / HeadKV are evicted layer by layer
        PoolLayers<kMaxLayerBatch> ly;
        const uint64_t merged_off = fused_ws_layout(a.Hq, a.G, a.k).hist_off;     // 2 * Hq * 1 KB of the fused kernel's area >= Hkv * NW * 16 B
        for (int l = 0; l < kMaxLayerBatch; ++l) {
            const EvictArgs& b = as[l < n ? l : 0];
            ly.logits[l] = reinterpret_cast<const uint16_t*>(b.ws_base + b.ws.logits_off);
            ly.partial[l] = reinterpret_cast<const float2*>(b.ws_base + b.ws.partial_off);
            ly.pooled[l] = reinterpret_cast<uint16_t*>(b.ws_base + b.ws.pooled_off);
            ly.merged[l] = reinterpret_cast<float4*>(b.ws_base + b.ws.fused_off + merged_off);
        }
        // PKV_BATCH_MERGE=0: every pool CTA merges the partials itself (A/B runs)
        static const bool merge_env = []() { const char* e = getenv("PKV_BATCH_MERGE"); return !e || atoi(e) != 0; }();
        p.use_merged = (merge_env && !p.under_scan) ? 1 : 0;
        if (p.use_merged) {
            cudaLaunchConfig_t mc = cfg;
            mc.gridDim = dim3(unsigned(a.Hq), unsigned(n), 1);
            e = cudaLaunchKernelEx(&mc, merge_partials_kernel<kMaxLayerBatch>, p, ly);
            count_launch();
            if (e != cudaSuccess) return e;
        }
        // The builds without a register cap (about 60 registers, four CTAs per SM): the stage is bound by the dependency latency of
        // the window sums, and capping at 48 or 40 registers for five or six CTAs per SM costs more of each thread's ILP than the
        // extra CTAs hide (H100: 0.28 instead of 0.32 ms per 32 x 32K batch, DESIGN.md section 4.1).
#define PKV_POOL_LAUNCH_B(T)                                                                                        \
    (a.W != 8 ? cudaLaunchKernelEx(&cfg, softmax_pool_kernel<T, 0, 0, false, kMaxLayerBatch>, p, ly)                \
     : ks == 7 ? cudaLaunchKernelEx(&cfg, softmax_pool_kernel<T, 8, 7, false, kMaxLayerBatch>, p, ly)               \
     : ks == 5 ? cudaLaunchKernelEx(&cfg, softmax_pool_kernel<T, 8, 5, false, kMaxLayerBatch>, p, ly)               \
               : cudaLaunchKernelEx(&cfg, softmax_pool_kernel<T, 8, 0, false, kMaxLayerBatch>, p, ly))
        if (a.dtype == PKV_BF16) e = PKV_POOL_LAUNCH_B(__nv_bfloat16);
        else e = PKV_POOL_LAUNCH_B(__half);
#undef PKV_POOL_LAUNCH_B
        count_launch();
        return e != cudaSuccess ? e : cudaGetLastError();
    }
    const PoolLayers<1> one;
    if (a.window_mean) {   // AdaKV / HeadKV scores: generic-window instantiation with the mean (any power-of-two W, any odd kernel)
        if (a.dtype == PKV_BF16) e = cudaLaunchKernelEx(&cfg, softmax_pool_kernel<__nv_bfloat16, 0, 0, true>, p, one);
        else e = cudaLaunchKernelEx(&cfg, softmax_pool_kernel<__half, 0, 0, true>, p, one);
        count_launch();
        return e != cudaSuccess ? e : cudaGetLastError();
    }
#define PKV_POOL_LAUNCH(T)                                                                      \
    (a.W != 8 ? cudaLaunchKernelEx(&cfg, softmax_pool_kernel<T, 0, 0>, p, one)                  \
     : ks == 7 ? cudaLaunchKernelEx(&cfg, softmax_pool_kernel<T, 8, 7>, p, one)                 \
     : ks == 5 ? cudaLaunchKernelEx(&cfg, softmax_pool_kernel<T, 8, 5>, p, one)                 \
               : cudaLaunchKernelEx(&cfg, softmax_pool_kernel<T, 8, 0>, p, one))
    if (a.dtype == PKV_BF16) e = PKV_POOL_LAUNCH(__nv_bfloat16);
    else e = PKV_POOL_LAUNCH(__half);
#undef PKV_POOL_LAUNCH
    count_launch();
    return e != cudaSuccess ? e : cudaGetLastError();
}
cudaError_t launch_softmax_pool(const EvictArgs& a, cudaStream_t st) { return launch_softmax_pool_layers(&a, 1, 0, st, nullptr, false); }

}  // namespace pkv
