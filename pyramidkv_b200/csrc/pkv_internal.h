// pkv_internal.h — host-side launcher prototypes shared by the .cu translation units.
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/pkv.h"

namespace pkv {

// Resolved, validated view of a pkv_evict_desc plus the workspace segments.
struct EvictArgs {
    int method, dtype, pooling, kernel_size;
    int Hq, Hkv, G, D, W;
    int64_t S, n /* S-W */, k;
    const uint16_t *q, *kk, *vv;
    int64_t q_sh, q_ss, k_sh, k_ss, v_sh, v_ss;
    uint16_t *k_cache, *v_cache;
    int64_t cache_sh;
    int64_t* idx_out;
    pkv_ws_layout ws;
    uint8_t* ws_base;
    uint32_t flags;
    int device;
    int num_sms;
    bool window_mean = false;   // PKV_FLAG_WINDOW_MEAN: stage 2 averages the window rows (AdaKV / HeadKV scores)
    bool gqa_shared = false;    // PKV_FLAG_GQA_SHARED with G > 1: one cache per KV head (stages 3-4 run on kv_view(*this))
    uint64_t pooled_kv_off = 0; // PKV_FLAG_GQA_SHARED: workspace offset of the per-KV-head top-k input (pkv_evict_pooled_kv_offset)
    int score_impl;   // 0 = mma.sync (one softmax partial per tile), 1 = TMA + wgmma (one partial per CTA and kv head)
    int score_grid;   // persistent grid of the wgmma kernel
};

void count_launch(int n = 1);
// Timing diagnostics (env PKV_STAMPS=1): a device buffer of 128 u64 that chosen threads of the score kernel
// ([64, 128)) and the select kernel ([0, 64)) write %clock64 / %globaltimer stamps into. nullptr when disabled.
unsigned long long* debug_stamps();

// stage 1 (window methods): logits + per-slot (max,sumexp) partials
cudaError_t launch_score_mma(const EvictArgs& a, cudaStream_t st);
bool score_tc5_supported(const EvictArgs& a);
int tc5_grid(const EvictArgs& a);
cudaError_t launch_score_tc5(const EvictArgs& a, cudaStream_t st);
constexpr int kMaxLayerBatch = 32;   // layers one launch of the batch kernels covers (their per-layer tables travel as kernel parameters)
cudaError_t launch_score_tc5_layers(const EvictArgs* as, int n, cudaStream_t st, int max_stages = 0, int* done = nullptr);
bool tc5_layer_major_ok(const EvictArgs& a);
// stage 2 (window methods): softmax -> round -> window sum -> pool
cudaError_t launch_softmax_pool(const EvictArgs& a, cudaStream_t st);
cudaError_t launch_softmax_pool_layers(const EvictArgs* as, int n, int batch_grid, cudaStream_t st, const int* done = nullptr, bool under_scan = false);
// H2O stages 1/2
cudaError_t launch_h2o_rowstats(const EvictArgs& a, cudaStream_t st);
cudaError_t launch_h2o_colsum(const EvictArgs& a, cudaStream_t st);
// L2Norm stage 1: negated key norms -> `pooled` (pkv_l2norm.cu)
cudaError_t launch_l2norm_scores(const EvictArgs& a, cudaStream_t st);
// H2O on TMA + wgmma (pkv_h2o_tc5.cu; PKV_H2O=tc5). stats4 = float4 {M, L, rn(1/L), 0} per query row, placed behind
// the float2 statistics inside the workspace (same formula in compute_layout and in the kernels' launcher)
inline uint64_t h2o_stats4_offset(const pkv_ws_layout& L, int Hq) {
    const uint64_t end = L.h2o_stats_off + uint64_t(Hq) * uint64_t(L.s_pad) * 8u;
    return (end + 255u) / 256u * 256u;
}
bool h2o_tc5_supported(const EvictArgs& a);
cudaError_t launch_h2o_tc5_rowstats(const EvictArgs& a, cudaStream_t st);
cudaError_t launch_h2o_tc5_colsum(const EvictArgs& a, cudaStream_t st);
// stage 3
bool topk_supported(const EvictArgs& a, const char** why);
cudaError_t launch_topk(const EvictArgs& a, cudaStream_t st);          // picks the cluster variant when it applies
cudaError_t launch_topk_single(const EvictArgs& a, cudaStream_t st);   // one CTA per head
bool topk_cluster_supported(const EvictArgs& a);
cudaError_t launch_topk_cluster(const EvictArgs& a, cudaStream_t st);  // one thread-block cluster per head
// stages 2+3+4 (pool = true, window methods) or 3+4 (pool = false) in ONE cluster launch per layer
bool select_fused_supported(const EvictArgs& a, bool pool);
cudaError_t launch_select_fused(const EvictArgs& a, bool pool, cudaStream_t st);
cudaError_t launch_select_layers(const EvictArgs* as, int n, cudaStream_t st);
bool select_batch_supported(const EvictArgs& a);
// stage 4
cudaError_t launch_gather(const EvictArgs& a, cudaStream_t st);
// PKV_FLAG_GQA_SHARED: pooled [Hq][pitch] -> pooled_kv [Hkv][pitch], the fp32 mean over each group rounded once (pkv_gather.cu)
cudaError_t launch_group_reduce(const EvictArgs& a, cudaStream_t st);

// ---- the whole eviction of a window method in ONE persistent launch (pkv_evict_fused.cu) ----
constexpr int kFusedStages = 5;        // cross-CTA exchanges: statistics, pooling halo, histogram pass 0 / 1, winners
constexpr int kFusedMaxGrid = 160;     // flag slots per stage (>= the SM count of an H100 SXM, 132)
constexpr int kFusedMaxPad = 32;       // kernel_size <= 65
constexpr int kFusedFixedSmem = 24576; // Q window tile + statistics + mbarriers, in front of the logit store (multiple of 1024)
// Segment `fused_off` of the workspace. Nothing in it needs initialising: flags carry a per-launch token, the tables are
// cleared by the launch that uses them.
struct FusedWs { uint64_t epoch_off, status_off, flags_off, hist_off, cursor_off, lhist_off, halo_off, win_off, total; };
inline FusedWs fused_ws_layout(int Hq, int G, int64_t k) {
    FusedWs w;
    uint64_t off = 0;
    auto seg = [&](uint64_t bytes) { const uint64_t o = off; off = (off + bytes + 255) / 256 * 256; return o; };
    w.epoch_off = seg(64);
    w.status_off = w.epoch_off + 8;
    w.flags_off = seg(uint64_t(kFusedStages) * kFusedMaxGrid * 8);
    w.hist_off = seg(uint64_t(2) * Hq * 256 * 4);
    w.cursor_off = seg(uint64_t(Hq) * 4);
    w.lhist_off = seg(uint64_t(kFusedMaxGrid) * G * 256 * 2);
    w.halo_off = seg(uint64_t(kFusedMaxGrid) * G * 2 * kFusedMaxPad * 4);
    w.win_off = seg(uint64_t(Hq) * uint64_t((k + 1) & ~int64_t(1)) * 8);
    w.total = off;
    return w;
}
bool evict_fused_supported(const EvictArgs& a);
int fused_tiles_per_cta(const EvictArgs& a);   // largest number of 128-token tiles one CTA of the fused kernel would hold
// pool_only = true: stages 1-2 (K scan, softmax, window sums, pool -> `pooled` in the workspace) in one launch; the select
// kernel follows as its own launch. false: stages 1-4, everything in one launch.
cudaError_t launch_evict_fused(const EvictArgs& a, bool pool_only, cudaStream_t st);

// One decode step over a compacted cache of any form. The row count of each (sequence, cache head) is read on the device:
// T (+ *step_dev) (+ rows[s*(cache heads) + c]); counts outside [1, max_rows] (with a window: attended counts above
// max_rows) are not attended (NaN output, nothing written).
struct DecodeArgs {
    int dtype, Hq, Hkv, G, D;
    int64_t T;  // valid rows after append (at step 0)
    const uint16_t *q, *k_new, *v_new;
    void *k_cache, *v_cache;
    uint16_t* out;
    int64_t cache_sh;
    int64_t cache_sb = 0;   // elements between the caches of consecutive sequences
    int num_seqs = 1;
    int heads_per_cache = 1;   // 1: a cache per query head; G: a GQA-shared cache per KV head ([num_seqs][Hkv][capacity][D])
    int64_t max_rows = 0;
    float* ws;
    float scale;
    int nsplit;
    int num_sms;
    const int32_t* step_dev = nullptr;  // device step counter added to T inside the kernel
    const int32_t* rows = nullptr;      // [num_seqs * cache heads] row counts added to T inside the kernel
    // E4M3 cache when k_scale is set: k_cache / v_cache hold E4M3 bytes, one fp32 scale per (sequence, cache head, row)
    float *k_scale = nullptr, *v_scale = nullptr;
    int64_t scale_sh = 0, scale_sb = 0;   // floats between the scales of consecutive heads / sequences
    // decode window (pkv_decode_attn_window) when window > 0: the n-th row of (sequence s, cache head c) with n > P + window,
    // P = prompt_rows[s*(cache heads) + c], is stored at P + (n-1-P) mod window and P + window rows are attended
    int64_t window = 0;
    const int32_t* prompt_rows = nullptr;
    // heavy-hitter window (pkv_decode_attn_heavy) when victim is set: past P + window the new row goes to victim[s*(cache
    // heads) + c], and decode_heavy_kernel updates the state and picks the next victim. hv_scratch: [num_seqs*Hq][window]
    // logits then [num_seqs*Hq][2] (m, l)
    int32_t* victim = nullptr;
    float *hv_scratch = nullptr, *hv_scores = nullptr;
    int32_t* hv_gen = nullptr;
    int64_t heavy = 0;
};
// split count for T rows (decode_num_splits); shared by the launch and the decode kernel
__host__ __device__ inline int64_t decode_splits_for(int64_t Hq, int64_t T, int64_t num_sms) {
    int64_t ns = (T + 255) / 256;                       // ~256 rows (32 per warp) per CTA
    const int64_t cap = (num_sms * 4 + Hq - 1) / Hq;    // at most ~4 CTAs per SM in flight
    if (ns > cap) ns = cap;
    if (ns < 1) ns = 1;
    if (ns > 64) ns = 64;
    return ns;
}
int decode_num_splits(int Hq, int64_t T, int num_sms);
// decode_kernel for the cache form (16-bit or E4M3 rows, per query head or GQA-shared), plus the merge of the split partials
cudaError_t launch_decode(const DecodeArgs& a, cudaStream_t st);
cudaError_t launch_append(const DecodeArgs& a, cudaStream_t st);

// ---- speculative decoding (pkv_spec.cu) ----
// The verify attention: Q new rows per (sequence, cache head) stored at n0 .. n0 + Q - 1, n0 = T (+ *step_dev) (+ rows[..]);
// query j attends rows [0, n0 + j + 1). n0 < 0 or n0 + Q > max_rows: NaN output, nothing written. Packed (row_count set):
// sequence s has row_count[s] new rows at token rows row_start[s] + j of M; split 0 zeroes the output rows no sequence owns.
struct MultiArgs {
    int dtype, Hq, Hkv, G, D, Q, num_seqs, heads_per_cache, nsplit, num_sms;
    const uint16_t *q, *k_new, *v_new;   // token s*Q + j, head h at + (s*Q + j)**_st + h*_sh elements
    uint16_t* out;
    int64_t q_st, q_sh, kv_st, kv_sh, out_st, out_sh;
    void *k_cache, *v_cache;
    int64_t cache_sh, cache_sb;
    float *k_scale, *v_scale;            // E4M3 rows when set
    int64_t scale_sh, scale_sb;
    int64_t T, max_rows;
    const int32_t* step_dev;
    const int32_t* rows;
    float scale;
    float* ws;                           // [num_seqs*Hq*Q][nsplit][2 + D] when nsplit > 1
    const int32_t* row_start;            // packed rows (pkv_decode_attn_packed); NULL: the dense layout start s*Q, count Q
    const int32_t* row_count;
    int64_t M;                           // packed token rows
};
size_t decode_multi_smem_bytes(int heads_per_cache, int Q, int D);
cudaError_t launch_decode_multi(const MultiArgs& a, cudaStream_t st);
constexpr int kMaxNgram = 8;
struct SpecArgs {
    int num_seqs, Q, N, n_eos, n_layers, H;   // n_layers <= kMaxLayerBatch
    int64_t hist_cap, out_cap, pad;
    int64_t* hist; int32_t* hist_len; int32_t* budget; uint8_t* done;
    int64_t* out; int32_t* out_len;
    int64_t* ids; int64_t* pos; int32_t* draft_len; int32_t* emitted;
    const int64_t* tokens; const int64_t* eos;
    int32_t* rows[kMaxLayerBatch];
};
cudaError_t launch_prompt_lookup(const SpecArgs& a, cudaStream_t st);
// first: the step kernel (rule 3, the rows of a.rows, rule 1); otherwise only the rows of a.rows, by emitted[b]
cudaError_t launch_spec_step(const SpecArgs& a, bool first, cudaStream_t st);
struct PackArgs {   // rule 2' (pkv_spec_pack)
    int D, M;
    const int32_t* step;
    int64_t *ids, *pos;
    int32_t *row_start, *row_count;
    int64_t* totals;
};
cudaError_t launch_spec_pack(const SpecArgs& a, const PackArgs& k, cudaStream_t st);

// ---- conversion of the compacted cache to FP8 (E4M3) rows (pkv_fp8.cu) ----
struct QuantLayer {
    const uint16_t* src[2];   // K, V: 16-bit [num_seqs][H][src_cap][D]
    uint8_t* dst[2];          // K, V: E4M3 [num_seqs][H][dst_cap][D]
    float* scale[2];          // K, V: fp32 [num_seqs][H][dst_cap]
    int64_t src_cap, dst_cap;
    int64_t rows;             // rows per (sequence, head); with rows_dev the bound of the device counts
    const int32_t* rows_dev;  // optional device int32 [num_seqs*H]
};
struct QuantArgs {
    int dtype, num_seqs, H, D, n_layers;   // n_layers <= kMaxLayerBatch
    QuantLayer layer[kMaxLayerBatch];
};
cudaError_t launch_quantize_fp8(const QuantArgs& a, int num_sms, cudaStream_t st);

// ---- admission into one slot of a batched cache (pkv_install.cu) ----
struct InstallLayer {
    const uint8_t* src[2];      // K, V: [H][src_cap][row_bytes] (one prompt); unused when rows == 0
    uint8_t* dst[2];            // K, V: [num_seqs][H][dst_cap][row_bytes]
    const float* src_scale[2];  // FP8 only: [H][src_cap]
    float* dst_scale[2];        // FP8 only: [num_seqs][H][dst_cap]
    int64_t src_cap, dst_cap;
    int64_t rows;               // rows per head; with rows_dev the bound of the device counts
    const int32_t* rows_dev;    // optional device int32 [H]
    int32_t* dst_rows;          // device int32 [num_seqs*H]: row counts of the decode kernels
};
struct InstallArgs {
    int H, slot, n_layers;      // n_layers <= kMaxLayerBatch
    const int32_t* step_dev;
    InstallLayer layer[kMaxLayerBatch];
};
cudaError_t launch_install(const InstallArgs& a, int row_bytes, int num_sms, cudaStream_t st);

// one sampled token per row of logits (pkv_sample.cu): one CTA per row
struct SampleArgs {
    int dtype, B, V;
    const uint16_t* logits;
    int64_t ld;                 // elements between rows
    const float* temperature;   // per-row device parameters [B]
    const int32_t* top_k;
    const float* top_p;
    const uint64_t* seed;
    int64_t* token_index;
    int64_t* tokens;            // token of row b at tokens[b * tokens_ld + col]
    int64_t tokens_ld, col;
    bool advance;               // token_index[b] += 1 after the draw
};
cudaError_t launch_sample(const SampleArgs& a, cudaStream_t st);
// the penalties and min-p of pkv_sample_tokens_penalized, per row b
struct PenaltyArgs {
    const float* repetition;    // [B] device parameters
    const float* presence;
    const float* frequency;
    const float* min_p;
    const uint8_t* mask;        // prompt_mask[b * ld + v]
    int32_t* counts;            // counts[b * ld + v], incremented at the drawn token with SampleArgs::advance
    int64_t ld;
};
cudaError_t launch_sample_penalized(const SampleArgs& a, const PenaltyArgs& p, cudaStream_t st);
// the rule terms of pkv_sample_tokens_constrained, per row b (flags: PKV_RULE_*)
struct RuleTermArgs {
    const int32_t* flags;       // [B]
    const float* bias;          // bias[b * bias_ld + v]
    int64_t bias_ld;
    const uint32_t* ban;        // words [0, W) of row b: set to -inf; [W, 2W): add -inf
    int64_t ban_ld;
    int W;
};
cudaError_t launch_sample_constrained(const SampleArgs& a, const PenaltyArgs& p, const RuleTermArgs& q, cudaStream_t st);

// the per-row rule terms of one step from the token history (pkv_rules.cu): one CTA per row
struct TokenRulesArgs {
    int B, V, W, n_eos;
    int32_t* hist; int64_t hist_ld;
    int32_t* hist_len;
    const int32_t* prompt_len;
    const int32_t* flags;
    const int32_t* ngram;
    const int32_t* min_new;
    const int32_t* n_seq;
    const int32_t* seq_off; const int32_t* seq_kind; const float* seq_bias; int64_t seq_ld;
    const int32_t* seq_tok; int64_t tok_ld;
    const int32_t* eos;
    const int64_t* append; int64_t append_ld, append_col;   // optional
    float* bias; int64_t bias_ld;
    uint32_t* ban; int64_t ban_ld;
    uint8_t* stop;
};
cudaError_t launch_token_rules(const TokenRulesArgs& a, cudaStream_t st);

// log-probabilities of one row of logits at a token and at its top N (pkv_logprobs.cu): one CTA per row
constexpr int kMaxTopLogprobs = 20;
struct LogprobsArgs {
    int dtype, B, V, N;         // N: top entries per row, <= kMaxTopLogprobs
    const uint16_t* logits;
    int64_t ld;                 // elements between rows
    const int64_t* tokens;      // token of row b at tokens[b * tokens_ld + tokens_col]
    int64_t tokens_ld, tokens_col;
    const int64_t* cursor;      // optional device column added to col
    int64_t col;
    float* lp;                  // lp[b * lp_ld + c], c = col (+ *cursor)
    int64_t lp_ld;
    int64_t* top_ids;           // top_ids / top_lp[b * top_ld + c * N + n]
    float* top_lp;
    int64_t top_ld;
};
cudaError_t launch_logprobs(const LogprobsArgs& a, cudaStream_t st);

// beam search (pkv_beam.cu, DESIGN.md §4.12)
constexpr int kMaxBeams = 16;
constexpr int kMaxBeamCandidates = 80;   // K = max(2, 1 + n_eos) * k with k <= 16 and n_eos <= 4
struct BeamCandArgs {
    int dtype, rows, V, K;
    const uint16_t* logits;
    int64_t ld;
    float* m;                   // [rows]
    float* log_z;               // [rows]
    float* cand_lp;             // [rows][K]
    int32_t* cand_id;           // [rows][K]
};
cudaError_t launch_beam_candidates(const BeamCandArgs& a, cudaStream_t st);
struct BeamStepArgs {
    int P, k, K, rows_per_prompt, n_eos, early_stopping, max_steps, step_offset;
    const float* cand_lp; const int32_t* cand_id;
    const int32_t* eos;
    const float* scale;         // [max_steps][2]
    const int32_t* step;
    float* running;
    float* pool_score; int32_t* pool_step; int32_t* pool_parent; int32_t* pool_token; uint8_t* pool_done;
    uint8_t* heur; uint8_t* done;
    int32_t* bp_token; int32_t* bp_parent;
    int32_t* cp;
    int64_t* next_token;
    int32_t* parent; int32_t* diverge;
};
cudaError_t launch_beam_step(const BeamStepArgs& a, cudaStream_t st);
struct ReorderLayer {
    void* plane[4];             // K, V rows [B][H][cap][row_bytes]; K, V fp32 scales [B][H][cap] (FP8) or null
    int64_t cap;
    const int32_t* base;        // [B*H]: the row of generated slot 0
    float* heavy_scores;        // heavy hitters: [B*H][window]
    int32_t* heavy_gen;         // [B*H][window]
    int32_t* victim;            // [B*H]
};
struct ReorderArgs {
    int P, k, H, row_bytes, window, heavy, n_layers, step_offset;
    const int32_t* parent; const int32_t* diverge;   // [P*k]
    const int32_t* step;
    ReorderLayer layer[kMaxLayerBatch];
};
size_t reorder_smem_bytes(int k, int row_bytes);
cudaError_t launch_cache_reorder(const ReorderArgs& a, cudaStream_t st);

// RoPE in place on Q and K (pkv_rope.cu)
struct RopeArgs {
    int dtype, Hq, Hkv, D;
    int64_t S;
    uint16_t *q, *k;
    int64_t q_sh, q_ss, k_sh, k_ss;
    const uint16_t *cos, *sin;
    int64_t cs_ss;
    int num_sms;
};
cudaError_t launch_rope(const RopeArgs& a, cudaStream_t st);

// AdaKV budgets + ragged-cache window placement (pkv_adakv.cu)
size_t adakv_scratch_bytes(int Hq);
cudaError_t launch_adakv_counts(const EvictArgs& a, int64_t base, int normalize, void* scratch, int32_t* counts, cudaStream_t st);
cudaError_t launch_ragged_window(const EvictArgs& a, const int32_t* caps_dev, cudaStream_t st);
// flat ragged cache append (pkv_flatten.cu)
cudaError_t launch_flatten_append(void* dst, const void* src, const void* state, const int32_t* head_lens, const int32_t* cu_lens,
                                  int num_heads, int row_bytes, int num_sms, cudaStream_t st);

}  // namespace pkv
