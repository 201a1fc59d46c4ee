// pkv_oracle.cpp — CPU restatement of the PyramidKV eviction hot path.
//
// *** TEST INFRASTRUCTURE, NOT PRODUCT CODE. ***
// Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference
// legs may load this library. The product path (pyramidkv_b200/) never imports it and
// has no CPU fallback.
//
// Parity pin: the reference ships no tests/golden vectors for this path (SURVEY.md §4),
// so this restatement is pinned against outputs of the reference's own Python code
// (`pyramidkv/pyramidkv_utils.py`, imported unmodified) captured by
// tests/golden/make_golden.py and committed under tests/golden/*.npz.
//
// Every function cites the reference lines it follows (paths relative to the reference's root).
// Arithmetic model ("rounding chain", SURVEY.md §2.1): all tensors live in the model
// dtype (bf16 / fp16); every torch op computes in fp32 and rounds its result to the
// model dtype (round-to-nearest-even). The dot product is accumulated in double and
// rounded once to fp32 (the "ideal" fp32 GEMM result; real GEMMs differ from it only
// in the last fp32 bits, which survive the following bf16/fp16 rounding with
// probability ~2^-16 per element).
//
// Build: see oracle/Makefile (g++ -O3 -fopenmp -shared).

#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <limits>
#include <utility>
#include <vector>

#if defined(_OPENMP)
#include <omp.h>
#endif

namespace {

enum { DT_BF16 = 0, DT_FP16 = 1 };
enum { M_PYRAMIDKV = 0, M_SNAPKV = 1, M_H2O = 2, M_STREAMINGLLM = 3, M_L2NORM = 4 };
enum { POOL_AVG = 0, POOL_MAX = 1 };
enum { TIE_LOWEST_INDEX = 0, TIE_TORCH_CPU = 1 };

inline float bits_to_f32(uint32_t u) { float f; std::memcpy(&f, &u, 4); return f; }
inline uint32_t f32_to_bits(float f) { uint32_t u; std::memcpy(&u, &f, 4); return u; }

inline float bf16_to_f32(uint16_t h) { return bits_to_f32(uint32_t(h) << 16); }
inline uint16_t f32_to_bf16(float f) {
    uint32_t u = f32_to_bits(f);
    if ((u & 0x7fffffffu) > 0x7f800000u) return uint16_t((u >> 16) | 0x0040u);  // quiet NaN
    u += 0x7fffu + ((u >> 16) & 1u);                                               // RNE
    return uint16_t(u >> 16);
}

inline float fp16_to_f32(uint16_t h) {
    const uint32_t sign = uint32_t(h & 0x8000u) << 16;
    uint32_t exp = (h >> 10) & 0x1fu;
    uint32_t man = h & 0x3ffu;
    if (exp == 0) {
        if (man == 0) return bits_to_f32(sign);
        // subnormal: normalise
        int e = -1;
        do { man <<= 1; ++e; } while ((man & 0x400u) == 0);
        man &= 0x3ffu;
        return bits_to_f32(sign | uint32_t(127 - 15 - e) << 23 | man << 13);
    }
    if (exp == 31) return bits_to_f32(sign | 0x7f800000u | man << 13);
    return bits_to_f32(sign | (exp + 112u) << 23 | man << 13);
}
inline uint16_t f32_to_fp16(float f) {
    const uint32_t u = f32_to_bits(f);
    const uint16_t sign = uint16_t((u >> 16) & 0x8000u);
    const uint32_t a = u & 0x7fffffffu;
    if (a > 0x7f800000u) return sign | 0x7e00u;       // NaN
    if (a >= 0x477ff000u) return sign | 0x7c00u;      // >= 65520 rounds to inf (RNE)
    if (a < 0x33000001u) return sign;                 // <= 2^-25 rounds to zero (tie -> even = 0)
    int32_t exp = int32_t(a >> 23) - 127;
    uint32_t man = (a & 0x7fffffu) | 0x800000u;       // 24-bit significand
    int shift;
    uint32_t base;
    if (exp < -14) { shift = 13 + (-14 - exp); base = 0; }       // subnormal result
    else { shift = 13; base = uint32_t(exp + 15) << 10; man &= 0x7fffffu; }
    const uint32_t q = man >> shift;
    const uint32_t rem = man & ((1u << shift) - 1u);
    const uint32_t half = 1u << (shift - 1);
    uint32_t r = base + q;
    if (rem > half || (rem == half && (q & 1u))) ++r;  // carries propagate into the exponent correctly
    return sign | uint16_t(r);
}

inline float to_f32(uint16_t h, int dt) { return dt == DT_BF16 ? bf16_to_f32(h) : fp16_to_f32(h); }
inline uint16_t from_f32(float f, int dt) { return dt == DT_BF16 ? f32_to_bf16(f) : f32_to_fp16(f); }
inline float round_dt(float f, int dt) { return to_f32(from_f32(f, dt), dt); }
inline float finfo_min(int dt) { return dt == DT_BF16 ? bf16_to_f32(0xff7f) : -65504.0f; }

// One score element of `attn_weights` before softmax, as the reference builds it:
//   matmul (fp32 acc, rounded) -> / sqrt(head_dim) (fp32 divide, rounded)
// pyramidkv_utils.py:253 (PyramidKV), :317 (SnapKV), :544 (H2O).
inline float score_elem(const uint16_t* q, const uint16_t* k, int D, int dt, float sqrt_d) {
    double acc = 0.0;
    for (int d = 0; d < D; ++d) acc += double(to_f32(q[d], dt)) * double(to_f32(k[d], dt));
    const float r1 = round_dt(float(acc), dt);
    return round_dt(r1 / sqrt_d, dt);
}

// In-place `attn_weights[..., -W:, -W:] += mask` with an fp32 mask of {0, finfo(dtype).min}
// pyramidkv_utils.py:254-260. (bf16: stays finfo.min; fp16: may round to -inf.)
inline float add_mask(float x, int dt) { return round_dt(x + finfo_min(dt), dt); }

}  // namespace

extern "C" {

int pkvo_version() { return 1; }

int pkvo_num_threads() {
#if defined(_OPENMP)
    return omp_get_max_threads();
#else
    return 1;
#endif
}

// Per-layer budget. Returns 0 on success.
//   *mode = 0 -> q_len < max_capacity_prompt: K/V returned unchanged (no eviction)
//   *mode = 1 -> evict, keep *k_out rows of the first S-W plus the last W rows
// PyramidKV: pyramidkv_utils.py:205-215 (budget), :218-220 (branches; note the middle
// branch uses k = B-W like SnapKV). SnapKV :314-334, H2O :541-562, StreamingLLM :603-608.
int pkvo_layer_budget(int method, int64_t max_capacity_prompt, int64_t window, int num_layers,
                      int layer_idx, int64_t q_len, int beta, int64_t* k_out, int* mode) {
    const int64_t B = max_capacity_prompt, W = window, S = q_len;
    if (B - W <= 0) return 1;  // assert self.max_capacity_prompt - self.window_size > 0  (:184)
    if (S < B) { *mode = 0; *k_out = S; return 0; }
    *mode = 1;
    if (method != M_PYRAMIDKV) { *k_out = B - W; return 0; }
    if (num_layers < 2 || beta <= 0) return 1;
    int64_t min_num = (B - W) / beta;
    int64_t max_num = (B - W) * 2 - min_num;
    if (max_num >= S - W) {
        max_num = S - W;
        min_num = (B - W) * 2 - max_num;
    }
    // Python floor division (operands may be negative in the clamped branch)
    const int64_t num = max_num - min_num, den = num_layers - 1;
    int64_t steps = num / den;
    if ((num % den != 0) && ((num < 0) != (den < 0))) --steps;
    if (S < (B - W) * 2) { *k_out = B - W; return 0; }
    *k_out = max_num - int64_t(layer_idx) * steps;
    return 0;
}

// Observation-window logits after the mask add, model dtype, layout [Hq][W][S].
// q: [Hq] x [S] x [D] with element strides (q_sh, q_ss); only rows S-W..S-1 are read.
// k: [Hkv] x [S] x [D] with strides (k_sh, k_ss); query head h reads kv head h / (Hq/Hkv)
// (== repeat_kv, pyramidkv_utils.py:108-117 / llama_model.py:158).
// pyramidkv_utils.py:253-260.
void pkvo_window_logits(const uint16_t* q, const uint16_t* k, int dt, int Hq, int Hkv, int64_t S, int D,
                        int W, int64_t q_sh, int64_t q_ss, int64_t k_sh, int64_t k_ss, uint16_t* logits) {
    const int G = Hq / Hkv;
    const float sqrt_d = float(std::sqrt(double(D)));  // math.sqrt(head_dim) as an fp32 scalar
#pragma omp parallel for collapse(2) schedule(static)
    for (int h = 0; h < Hq; ++h) {
        for (int w = 0; w < W; ++w) {
            const uint16_t* qrow = q + int64_t(h) * q_sh + (S - W + w) * q_ss;
            const uint16_t* kh = k + int64_t(h / G) * k_sh;
            uint16_t* out = logits + (int64_t(h) * W + w) * S;
            for (int64_t j = 0; j < S; ++j) {
                float x = score_elem(qrow, kh + j * k_ss, D, dt, sqrt_d);
                const int64_t jw = j - (S - W);
                if (jw >= 0) x = (jw > w) ? add_mask(x, dt) : round_dt(x + 0.0f, dt);
                out[j] = from_f32(x, dt);
            }
        }
    }
}

// softmax(dim=-1, dtype=float32).to(dtype) over rows of length S. pyramidkv_utils.py:262.
void pkvo_softmax_rows(const uint16_t* logits, int dt, int64_t rows, int64_t S, uint16_t* probs) {
#pragma omp parallel for schedule(static)
    for (int64_t r = 0; r < rows; ++r) {
        const uint16_t* x = logits + r * S;
        uint16_t* p = probs + r * S;
        float mx = -std::numeric_limits<float>::infinity();
        for (int64_t j = 0; j < S; ++j) mx = std::max(mx, to_f32(x[j], dt));
        double sum = 0.0;
        for (int64_t j = 0; j < S; ++j) sum += double(std::exp(to_f32(x[j], dt) - mx));
        const float fsum = float(sum);
        for (int64_t j = 0; j < S; ++j) p[j] = from_f32(std::exp(to_f32(x[j], dt) - mx) / fsum, dt);
    }
}

// attn_weights[:, :, -W:, :-W].sum(dim=-2): fp32 accumulate over the W rows, one rounding.
// probs [Hq][W][S] -> wsum [Hq][S-W]. pyramidkv_utils.py:263.
void pkvo_window_sum(const uint16_t* probs, int dt, int Hq, int W, int64_t S, uint16_t* wsum) {
    const int64_t n = S - W;
#pragma omp parallel for schedule(static)
    for (int h = 0; h < Hq; ++h)
        for (int64_t j = 0; j < n; ++j) {
            float acc = 0.0f;
            for (int w = 0; w < W; ++w) acc += to_f32(probs[(int64_t(h) * W + w) * S + j], dt);
            wsum[int64_t(h) * n + j] = from_f32(acc, dt);
        }
}

// attn_weights[:, :, -W:, :-W].mean(dim=-2) of AdaKV / HeadKV (`calcul_attn_sore`, pyramidkv_utils.py:661 / :795): fp32
// accumulate over the W rows, fp32 divide by W, one rounding. (torch's CPU kernel rounds the sum first and divides in the
// model dtype — identical for the power-of-two window sizes the CUDA path accepts, where the division is exact.)
void pkvo_window_mean(const uint16_t* probs, int dt, int Hq, int W, int64_t S, uint16_t* wmean) {
    const int64_t n = S - W;
#pragma omp parallel for schedule(static)
    for (int h = 0; h < Hq; ++h)
        for (int64_t j = 0; j < n; ++j) {
            float acc = 0.0f;
            for (int w = 0; w < W; ++w) acc += to_f32(probs[(int64_t(h) * W + w) * S + j], dt);
            wmean[int64_t(h) * n + j] = from_f32(acc / float(W), dt);
        }
}

// Per-head budgets of AdaKVCluster.update_kv (pyramidkv_utils.py:702-717). score [H][n] (pooled mean scores).
//   per head: sort descending; normalize: ratio = round(round(sum top-base) / round(sum all)), scaled = round(v * ratio)
//   flat top-(H*base) over the [H][n] scaled values -> how many fall into each head (c'_h)
//   caps[h] = round_half_even(float32(c'_h) * one_minus_floor + floor_capacity)
// Ties at the global threshold are implementation-defined in the reference (torch.topk on the flattened tensor); the
// rule here is the CUDA path's: lower flat index first, i.e. lower heads take the tied slots first. cnt_gt / cnt_eq
// (optional) report, per head, the scaled values above / equal to the threshold *thr_out.
int pkvo_adakv_capacities(const uint16_t* score, int dt, int H, int64_t n, int64_t base, float one_minus_floor,
                          int64_t floor_capacity, int normalize, int32_t* caps, int64_t* cnt_gt, int64_t* cnt_eq,
                          uint16_t* thr_out, uint16_t* scaled_out /* optional [H][n]: the (normalised) scores the flat top-k sees */,
                          float* ratio_out /* optional [H]: ratio_h (1 without normalize) */) {
    if (H <= 0 || base < 1 || base > n) return 1;
    std::vector<uint16_t> scaled(size_t(H) * size_t(n));
    for (int h = 0; h < H; ++h) {
        const uint16_t* row = score + int64_t(h) * n;
        float ratio = 1.0f;
        if (normalize) {
            std::vector<float> v(static_cast<size_t>(n));
            for (int64_t j = 0; j < n; ++j) v[size_t(j)] = to_f32(row[j], dt);
            std::vector<float> srt(v);
            std::sort(srt.begin(), srt.end(), [](float a, float b) { return a > b; });
            double top = 0.0, all = 0.0;
            for (int64_t j = 0; j < n; ++j) { all += double(srt[size_t(j)]); if (j < base) top += double(srt[size_t(j)]); }
            const float s_top = round_dt(float(top), dt), s_all = round_dt(float(all), dt);      // .sum(dim=-1) in the model dtype
            ratio = round_dt(s_top / s_all, dt);        // 0 / 0 = NaN for a head whose scores are all zero
        }
        if (ratio_out) ratio_out[h] = ratio;
        for (int64_t j = 0; j < n; ++j)
            scaled[size_t(h) * size_t(n) + size_t(j)] = normalize ? from_f32(to_f32(row[j], dt) * ratio, dt) : row[j];
    }
    if (scaled_out) std::memcpy(scaled_out, scaled.data(), scaled.size() * 2);
    const int64_t K = int64_t(H) * base;
    std::vector<float> flat(scaled.size());
    for (size_t i = 0; i < scaled.size(); ++i) flat[i] = to_f32(scaled[i], dt);
    std::vector<float> tmp(flat);
    // NaN (the scaled scores of a NaN-ratio head) ranks above every value and equals every NaN, as in torch.sort / topk
    const auto above = [](float a, float b) { return (std::isnan(a) && !std::isnan(b)) || a > b; };
    const auto same = [](float a, float b) { return (std::isnan(a) && std::isnan(b)) || a == b; };
    std::nth_element(tmp.begin(), tmp.begin() + (K - 1), tmp.end(), above);
    const float thr = tmp[size_t(K - 1)];
    if (thr_out) *thr_out = from_f32(thr, dt);
    int64_t need = K;
    std::vector<int64_t> gt(static_cast<size_t>(H), 0), eq(static_cast<size_t>(H), 0);
    for (int h = 0; h < H; ++h)
        for (int64_t j = 0; j < n; ++j) {
            const float x = flat[size_t(h) * size_t(n) + size_t(j)];
            if (above(x, thr)) ++gt[size_t(h)]; else if (same(x, thr)) ++eq[size_t(h)];
        }
    for (int h = 0; h < H; ++h) need -= gt[size_t(h)];
    for (int h = 0; h < H; ++h) {
        const int64_t take = std::min(need, eq[size_t(h)]);
        need -= take;
        const float f = float(gt[size_t(h)] + take) * one_minus_floor + float(floor_capacity);
        caps[h] = int32_t(std::nearbyint(f));                           // torch.round: half to even
        if (cnt_gt) cnt_gt[h] = gt[size_t(h)];
        if (cnt_eq) cnt_eq[h] = eq[size_t(h)];
    }
    return 0;
}

// F.max_pool1d / F.avg_pool1d(kernel, padding=kernel//2, stride=1) along the token axis.
// max: -inf padding (exact). avg: zero padding, count_include_pad=True (always / kernel),
// fp32 sum in ascending order, fp32 divide, one rounding. Odd kernel sizes only (an even
// kernel makes the reference's pooled row one element longer than the gather source).
// pyramidkv_utils.py:264-269.
int pkvo_pool(const uint16_t* wsum, int dt, int Hq, int64_t n, int kernel, int pooling, uint16_t* pooled) {
    if (kernel < 1 || (kernel & 1) == 0) return 1;
    if (pooling != POOL_AVG && pooling != POOL_MAX) return 2;  // ValueError('Pooling method not supported') :237
    const int pad = kernel / 2;
#pragma omp parallel for schedule(static)
    for (int h = 0; h < Hq; ++h) {
        const uint16_t* in = wsum + int64_t(h) * n;
        uint16_t* out = pooled + int64_t(h) * n;
        for (int64_t j = 0; j < n; ++j) {
            if (pooling == POOL_MAX) {
                float m = -std::numeric_limits<float>::infinity();
                for (int64_t t = j - pad; t <= j + pad; ++t)
                    if (t >= 0 && t < n) m = std::max(m, to_f32(in[t], dt));
                out[j] = from_f32(m, dt);
            } else {
                float s = 0.0f;
                for (int64_t t = j - pad; t <= j + pad; ++t)
                    if (t >= 0 && t < n) s += to_f32(in[t], dt);
                out[j] = from_f32(s / float(kernel), dt);
            }
        }
    }
    return 0;
}

// attn_cache.topk(k, dim=-1).indices (largest, sorted). pyramidkv_utils.py:270 (:334, :562).
// scores [Hq][n] model dtype -> idx [Hq][k] int64.
//   TIE_LOWEST_INDEX: the contract the CUDA path implements — every element strictly above the
//     k-th value, then the lowest indices among elements equal to it; emitted in
//     (value descending, index ascending) order.
//   TIE_TORCH_CPU: restates what the un-vendored dependency torch (2.11.0, CPU `topk`,
//     ATen/native/TopKImpl.h) does: (value, index) pairs, comparator on value only (NaN first),
//     std::partial_sort when k*64 <= n, else std::nth_element(k-1) + std::sort of the first k-1.
//     Tie order is then whatever libstdc++ produces; reproduced by calling the same algorithms.
int pkvo_topk(const uint16_t* scores, int dt, int Hq, int64_t n, int64_t k, int tie_mode, int64_t* idx) {
    if (k < 0 || k > n) return 1;
    if (k == 0) return 0;
    using elem_t = std::pair<float, int64_t>;
    int rc = 0;
#pragma omp parallel for schedule(dynamic)
    for (int h = 0; h < Hq; ++h) {
        std::vector<elem_t> queue(n);
        for (int64_t j = 0; j < n; ++j) queue[j] = elem_t(to_f32(scores[int64_t(h) * n + j], dt), j);
        if (tie_mode == TIE_LOWEST_INDEX) {
            auto cmp = [](const elem_t& x, const elem_t& y) {
                if (x.first != y.first) return x.first > y.first;
                return x.second < y.second;
            };
            std::partial_sort(queue.begin(), queue.begin() + k, queue.end(), cmp);
        } else {
            auto cmp = [](const elem_t& x, const elem_t& y) {
                return (std::isnan(x.first) && !std::isnan(y.first)) || (x.first > y.first);
            };
            if (k * 64 <= n) {
                std::partial_sort(queue.begin(), queue.begin() + k, queue.end(), cmp);
            } else {
                std::nth_element(queue.begin(), queue.begin() + k - 1, queue.end(), cmp);
                std::sort(queue.begin(), queue.begin() + k - 1, cmp);
            }
        }
        for (int64_t j = 0; j < k; ++j) idx[int64_t(h) * k + j] = queue[j].second;
    }
    return rc;
}

// K' = cat(K[:, :, :-W].gather(2, idx), K[:, :, -W:]) (same for V) written into a cache of
// row capacity `cap` per query head: out[h][r][:], r < k + W. src: [Hkv][S][D] strided.
// idx == nullptr -> identity indices 0..k-1 (StreamingLLM, pyramidkv_utils.py:607-608).
// pyramidkv_utils.py:271-282.
void pkvo_gather(const uint16_t* src, int Hq, int Hkv, int64_t S, int D, int W, int64_t s_sh, int64_t s_ss,
                 const int64_t* idx, int64_t k, uint16_t* out, int64_t cap) {
    const int G = Hq / Hkv;
#pragma omp parallel for schedule(static)
    for (int h = 0; h < Hq; ++h) {
        const uint16_t* sh = src + int64_t(h / G) * s_sh;
        uint16_t* oh = out + int64_t(h) * cap * D;
        for (int64_t r = 0; r < k; ++r) {
            const int64_t j = idx ? idx[int64_t(h) * k + r] : r;
            std::memcpy(oh + r * D, sh + j * s_ss, size_t(D) * 2);
        }
        for (int w = 0; w < W; ++w) std::memcpy(oh + (k + w) * D, sh + (S - W + w) * s_ss, size_t(D) * 2);
    }
}

// H2O scores: full softmax(QK^T/sqrt(D)) with the causal mask applied ONLY to the last WxW
// block, column sum over ALL S rows (fp32 accumulate, one rounding), no pooling.
// out: colsum [Hq][S-W]. Row statistics in double-accumulated fp32 like pkvo_softmax_rows.
// pyramidkv_utils.py:544-561.
void pkvo_h2o_scores(const uint16_t* q, const uint16_t* k, int dt, int Hq, int Hkv, int64_t S, int D, int W,
                     int64_t q_sh, int64_t q_ss, int64_t k_sh, int64_t k_ss, uint16_t* colsum) {
    const int G = Hq / Hkv;
    const float sqrt_d = float(std::sqrt(double(D)));
    const int64_t n = S - W;
#pragma omp parallel for schedule(dynamic)
    for (int h = 0; h < Hq; ++h) {
        const uint16_t* kh = k + int64_t(h / G) * k_sh;
        std::vector<float> acc(size_t(n), 0.0f);
        std::vector<float> row(static_cast<size_t>(S));
        for (int64_t i = 0; i < S; ++i) {
            const uint16_t* qrow = q + int64_t(h) * q_sh + i * q_ss;
            float mx = -std::numeric_limits<float>::infinity();
            for (int64_t j = 0; j < S; ++j) {
                float x = score_elem(qrow, kh + j * k_ss, D, dt, sqrt_d);
                const int64_t iw = i - n, jw = j - n;
                if (iw >= 0 && jw >= 0) x = (jw > iw) ? add_mask(x, dt) : round_dt(x + 0.0f, dt);
                row[size_t(j)] = x;
                mx = std::max(mx, x);
            }
            double sum = 0.0;
            for (int64_t j = 0; j < S; ++j) sum += double(std::exp(row[size_t(j)] - mx));
            const float fsum = float(sum);
            for (int64_t j = 0; j < n; ++j) acc[size_t(j)] += round_dt(std::exp(row[size_t(j)] - mx) / fsum, dt);
        }
        for (int64_t j = 0; j < n; ++j) colsum[int64_t(h) * n + j] = from_f32(acc[size_t(j)], dt);
    }
}

// Whole prefill eviction of one layer (the body of *KVCluster.update_kv for merge=None).
// Optional stage outputs (may be nullptr): logits [Hq][W][S], probs [Hq][W][S],
// wsum [Hq][S-W], pooled [Hq][S-W] (for H2O: wsum == pooled == column sums, logits/probs unused),
// idx [Hq][k]. k_cache / v_cache: [Hq][cap][D].
// Returns 0 ok, 1 bad argument, 2 unsupported pooling.
// L2Norm scores (SURVEY.md §8 f4): `token_norms = torch.norm(key_states, p=2, dim=-1)` — pyramidkv_utils.py:420.
// One torch op: fp32-class accumulation of the squares (restated as a double accumulation rounded once to fp32),
// fp32 sqrt, one rounding to the model dtype. Bit-identical to torch 2.11 CPU on 32768/32768 bf16 and 32765/32768
// fp16 probe values (tests/golden/l2norm_*.npz pin it). norms [Hkv][S].
void pkvo_key_norms(const uint16_t* k, int dt, int Hkv, int64_t S, int D, int64_t k_sh, int64_t k_ss, uint16_t* norms) {
#pragma omp parallel for schedule(static)
    for (int64_t i = 0; i < int64_t(Hkv) * S; ++i) {
        const int64_t h = i / S, t = i % S;
        const uint16_t* row = k + h * k_sh + t * k_ss;
        double acc = 0.0;
        for (int d = 0; d < D; ++d) { const double x = double(to_f32(row[d], dt)); acc += x * x; }
        norms[i] = from_f32(std::sqrt(float(acc)), dt);
    }
}

// pyramidkv_utils.py:197-283 (PyramidKV), :306-347 (SnapKV), :533-575 (H2O), :595-620 (StreamingLLM),
// :406-431 (L2Norm: W == 0, keeps the k = max_capacity_prompt tokens of smallest key norm in (norm asc, index asc)
// order — `argsort` is not stable in the reference, so the order among equal norms is implementation-defined there;
// o_pooled receives the NEGATED norms of each query head's kv head, i.e. the keys a descending top-k selects on).
int pkvo_evict(int method, int dt, int pooling, int kernel, int tie_mode, int Hq, int Hkv, int64_t S, int D, int W,
               int64_t k, const uint16_t* q, int64_t q_sh, int64_t q_ss, const uint16_t* kk, int64_t k_sh,
               int64_t k_ss, const uint16_t* vv, int64_t v_sh, int64_t v_ss, uint16_t* k_cache, uint16_t* v_cache,
               int64_t cap, uint16_t* o_logits, uint16_t* o_probs, uint16_t* o_wsum, uint16_t* o_pooled,
               int64_t* o_idx) {
    if (Hq <= 0 || Hkv <= 0 || Hq % Hkv || W < (method == M_L2NORM ? 0 : 1) || W > S || k < 0 || k > S - W || cap < k + W) return 1;
    if (method == M_L2NORM && W != 0) return 1;
    const int64_t n = S - W;
    std::vector<int64_t> idx_buf;
    int64_t* idx = o_idx;
    if (method == M_STREAMINGLLM) {
        if (o_idx)
            for (int h = 0; h < Hq; ++h)
                for (int64_t r = 0; r < k; ++r) o_idx[int64_t(h) * k + r] = r;
        idx = nullptr;
    } else {
        if (!idx) { idx_buf.resize(size_t(Hq) * size_t(std::max<int64_t>(k, 1))); idx = idx_buf.data(); }
        std::vector<uint16_t> pooled_buf;
        uint16_t* pooled = o_pooled;
        if (!pooled) { pooled_buf.resize(size_t(Hq) * size_t(n)); pooled = pooled_buf.data(); }
        if (method == M_L2NORM) {
            std::vector<uint16_t> norms(size_t(Hkv) * size_t(S));
            pkvo_key_norms(kk, dt, Hkv, S, D, k_sh, k_ss, norms.data());
            const int G = Hq / Hkv;
            for (int h = 0; h < Hq; ++h)
                for (int64_t t = 0; t < S; ++t) pooled[int64_t(h) * n + t] = norms[size_t(h / G) * size_t(S) + size_t(t)] ^ 0x8000u;
            if (o_wsum) std::memcpy(o_wsum, pooled, size_t(Hq) * size_t(n) * 2);
            tie_mode = TIE_LOWEST_INDEX;
        } else if (method == M_H2O) {
            pkvo_h2o_scores(q, kk, dt, Hq, Hkv, S, D, W, q_sh, q_ss, k_sh, k_ss, pooled);
            if (o_wsum) std::memcpy(o_wsum, pooled, size_t(Hq) * size_t(n) * 2);
        } else {
            std::vector<uint16_t> lb, pb, wb;
            uint16_t* logits = o_logits; if (!logits) { lb.resize(size_t(Hq) * W * S); logits = lb.data(); }
            uint16_t* probs = o_probs;   if (!probs)  { pb.resize(size_t(Hq) * W * S); probs = pb.data(); }
            uint16_t* wsum = o_wsum;     if (!wsum)   { wb.resize(size_t(Hq) * size_t(n)); wsum = wb.data(); }
            pkvo_window_logits(q, kk, dt, Hq, Hkv, S, D, W, q_sh, q_ss, k_sh, k_ss, logits);
            pkvo_softmax_rows(logits, dt, int64_t(Hq) * W, S, probs);
            pkvo_window_sum(probs, dt, Hq, W, S, wsum);
            const int rc = pkvo_pool(wsum, dt, Hq, n, kernel, pooling, pooled);
            if (rc) return rc == 2 ? 2 : 1;
        }
        if (pkvo_topk(pooled, dt, Hq, n, k, tie_mode, idx)) return 1;
    }
    pkvo_gather(kk, Hq, Hkv, S, D, W, k_sh, k_ss, idx, k, k_cache, cap);
    pkvo_gather(vv, Hq, Hkv, S, D, W, v_sh, v_ss, idx, k, v_cache, cap);
    return 0;
}

// Decode attention over the compacted cache, eager semantics (q_len = 1, every cached row
// visible): logits = round(round(q.k) / sqrt(D)); p = round(softmax_fp32(logits));
// out = round(sum_fp32 p*v). q [Hq][D]; k_cache/v_cache [Hq][cap][D]; T rows valid; out [Hq][D].
// llama_model.py:174-183 (eager); the flash/sdpa variants (:291-313, :411-445) keep p in fp32 —
// both are within the 1e-3 tolerance north_star states.
void pkvo_decode_attn(const uint16_t* q, const uint16_t* k_cache, const uint16_t* v_cache, int dt, int Hq, int D,
                      int64_t T, int64_t cap, uint16_t* out) {
    const float sqrt_d = float(std::sqrt(double(D)));
#pragma omp parallel for schedule(static)
    for (int h = 0; h < Hq; ++h) {
        const uint16_t* qh = q + int64_t(h) * D;
        const uint16_t* kh = k_cache + int64_t(h) * cap * D;
        const uint16_t* vh = v_cache + int64_t(h) * cap * D;
        std::vector<float> x(static_cast<size_t>(T));
        float mx = -std::numeric_limits<float>::infinity();
        for (int64_t t = 0; t < T; ++t) { x[size_t(t)] = score_elem(qh, kh + t * D, D, dt, sqrt_d); mx = std::max(mx, x[size_t(t)]); }
        double sum = 0.0;
        for (int64_t t = 0; t < T; ++t) sum += double(std::exp(x[size_t(t)] - mx));
        const float fsum = float(sum);
        std::vector<double> acc(size_t(D), 0.0);
        for (int64_t t = 0; t < T; ++t) {
            const float p = round_dt(std::exp(x[size_t(t)] - mx) / fsum, dt);
            for (int d = 0; d < D; ++d) acc[size_t(d)] += double(p) * double(to_f32(vh[t * D + d], dt));
        }
        for (int d = 0; d < D; ++d) out[int64_t(h) * D + d] = from_f32(float(acc[size_t(d)]), dt);
    }
}

// Exact (double) attention output as fp32, for tolerance checks that do not depend on any
// intermediate rounding convention. out32 [Hq][D].
void pkvo_decode_attn_exact(const uint16_t* q, const uint16_t* k_cache, const uint16_t* v_cache, int dt, int Hq,
                            int D, int64_t T, int64_t cap, float* out32) {
    const double inv = 1.0 / std::sqrt(double(D));
#pragma omp parallel for schedule(static)
    for (int h = 0; h < Hq; ++h) {
        const uint16_t* qh = q + int64_t(h) * D;
        const uint16_t* kh = k_cache + int64_t(h) * cap * D;
        const uint16_t* vh = v_cache + int64_t(h) * cap * D;
        std::vector<double> x(static_cast<size_t>(T));
        double mx = -1e300;
        for (int64_t t = 0; t < T; ++t) {
            double a = 0.0;
            for (int d = 0; d < D; ++d) a += double(to_f32(qh[d], dt)) * double(to_f32(kh[t * D + d], dt));
            x[size_t(t)] = a * inv; mx = std::max(mx, x[size_t(t)]);
        }
        double sum = 0.0;
        for (int64_t t = 0; t < T; ++t) { x[size_t(t)] = std::exp(x[size_t(t)] - mx); sum += x[size_t(t)]; }
        for (int d = 0; d < D; ++d) {
            double a = 0.0;
            for (int64_t t = 0; t < T; ++t) a += x[size_t(t)] * double(to_f32(vh[t * D + d], dt));
            out32[int64_t(h) * D + d] = float(a / sum);
        }
    }
}

// Rotary embedding in place (SURVEY.md §8 f2): HF `apply_rotary_pos_emb` as the patched forwards call it
// (llama_model.py:157 / :276 / :378): x*cos + rotate_half(x)*sin, rotate_half(x) = cat(-x[D/2:], x[:D/2]); every torch op
// (two products, one sum) computes in fp32 and rounds once to the model dtype. x: [H][S][D] strided; cos/sin [S][D].
void pkvo_rope_inplace(uint16_t* x, int dt, int H, int64_t S, int D, int64_t x_sh, int64_t x_ss, const uint16_t* cos,
                       const uint16_t* sin, int64_t cs_ss) {
    const int half = D / 2;
#pragma omp parallel for schedule(static)
    for (int64_t i = 0; i < int64_t(H) * S; ++i) {
        const int64_t h = i / S, t = i % S;
        uint16_t* row = x + h * x_sh + t * x_ss;
        const uint16_t* c = cos + t * cs_ss;
        const uint16_t* sn = sin + t * cs_ss;
        uint16_t out[512];
        for (int d = 0; d < D; ++d) {
            const float xv = to_f32(row[d], dt);
            const float rot = d < half ? -to_f32(row[d + half], dt) : to_f32(row[d - half], dt);
            const float t1 = round_dt(xv * to_f32(c[d], dt), dt);
            const float t2 = round_dt(rot * to_f32(sn[d], dt), dt);
            out[d] = from_f32(t1 + t2, dt);
        }
        std::memcpy(row, out, size_t(D) * 2);
    }
}

// dtype helpers exported for tests
float pkvo_to_f32(uint16_t h, int dt) { return to_f32(h, dt); }
uint16_t pkvo_from_f32(float f, int dt) { return from_f32(f, dt); }

}  // extern "C"
