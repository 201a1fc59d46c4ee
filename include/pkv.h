/* pkv.h — C ABI of libpkv.so: H100 (sm_90a) KV-cache eviction hot path.
 *
 * Drop-in boundary for the prefill-time eviction of Zefan-Cai/PyramidKV and for decode attention over
 * the compacted cache. Each entry point names the reference code it replaces (paths relative to the
 * reference repository root). Plain pointers and sizes only — no torch types.
 *
 * Conventions
 *  - All tensors hold 16-bit elements of `dtype` (PKV_BF16 / PKV_FP16); strides are in ELEMENTS.
 *    The innermost (head_dim) axis is contiguous; base pointers and row strides are 16-byte aligned.
 *  - Batch size is 1 (as in the reference: README.md:47, batch inference unsupported), except for
 *    pkv_decode_attn_batch, which decodes the compacted caches of several prompts in one launch.
 *  - Q is [num_q_heads, seq_len, head_dim]; K/V are [num_kv_heads, seq_len, head_dim] and are NOT
 *    repeated: query head h reads kv head h / (num_q_heads / num_kv_heads). Passing
 *    num_kv_heads == num_q_heads reproduces the reference's post-`repeat_kv` call exactly
 *    (pyramidkv/llama_model.py:158-159).
 *  - The compacted cache is per QUERY head: [num_q_heads, capacity, head_dim] (the reference caches
 *    K/V after repeat_kv, llama_model.py:167-168). Rows 0..top_k-1 are the selected tokens in
 *    (score descending, index ascending) order, rows top_k..top_k+window-1 are the last `window` tokens.
 *  - Every launch function takes the CUDA stream as an opaque `void*` (cudaStream_t) and is fully
 *    asynchronous: no device synchronisation, no default-stream launches, no device allocation.
 *    Scratch memory is caller-provided (`workspace`), sized by the *_workspace_bytes queries.
 *  - Functions return a pkv_status; pkv_last_error() gives a thread-local message for the last failure.
 *  - There is no CPU fallback: on a device that is not compute capability 10.x every launch returns
 *    PKV_ERR_UNSUPPORTED_ARCH.
 */
#ifndef PKV_H_
#define PKV_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define PKV_ABI_VERSION 3

typedef enum pkv_status {
    PKV_OK = 0,
    PKV_ERR_INVALID_ARG = 1,       /* reference: Python assert / shape errors */
    PKV_ERR_UNSUPPORTED_DTYPE = 2,
    PKV_ERR_UNSUPPORTED_ARCH = 3,
    PKV_ERR_CUDA = 4,
    PKV_ERR_WORKSPACE = 5,         /* workspace missing or too small */
    PKV_ERR_UNSUPPORTED = 6,       /* valid in the reference, not built here (e.g. merge != None) */
    PKV_ERR_POOLING = 7            /* reference: ValueError('Pooling method not supported'), pyramidkv_utils.py:237 */
} pkv_status;

typedef enum pkv_dtype { PKV_BF16 = 0, PKV_FP16 = 1 } pkv_dtype;

/* monkeypatch.py:19-87 method strings: "pyramidkv", "snapkv", "h2o", "streamingllm", "l2norm".
 * PKV_L2NORM (L2NormCluster, pyramidkv_utils.py:394-431): window must be 0 and top_k = max_capacity_prompt; the
 * cache receives the top_k tokens of smallest key L2 norm in (norm ascending, index ascending) order, no window rows;
 * q is not read (may be NULL). */
typedef enum pkv_method { PKV_PYRAMIDKV = 0, PKV_SNAPKV = 1, PKV_H2O = 2, PKV_STREAMINGLLM = 3, PKV_L2NORM = 4 } pkv_method;

/* self.config.pooling: "avgpool" / "maxpool" (pyramidkv_utils.py:264-269) */
typedef enum pkv_pooling { PKV_AVGPOOL = 0, PKV_MAXPOOL = 1 } pkv_pooling;

/* Which window-scoring kernel to use (pkv_evict_desc.flags bits 0-1). */
#define PKV_SCORE_AUTO 0u    /* TMA + wgmma kernel when the shape allows, else the mma.sync kernel */
#define PKV_SCORE_MMA 1u     /* force the mma.sync kernel */
#define PKV_SCORE_TCGEN05 2u /* force the TMA + wgmma kernel (error if the shape is unsupported; the name is kept for ABI compatibility) */
/* pkv_evict_desc.flags bit 2: stage 2 AVERAGES the window rows instead of summing them — `calcul_attn_sore` of AdaKV /
 * HeadKV (pyramidkv_utils.py:661 / :795: `.mean(dim=-2)`). Power-of-two window sizes only (the mean is the fp32 sum
 * times an exact power of two, the value every torch back end agrees on). */
#define PKV_FLAG_WINDOW_MEAN 4u
/* pkv_evict_desc.flags bit 3: the caller promises that q, k and v were NOT written by the kernel that immediately
 * precedes this call in the stream (they are older). pkv_evict_prefill then starts streaming K while that kernel is
 * still draining (programmatic dependent launch); without the flag the first load waits for its completion. */
#define PKV_FLAG_INPUTS_READY 8u
/* pkv_evict_desc.flags bit 4: pkv_evict_prefill runs the staged kernels (stages 1-4 as separate launches) even where the
 * single-launch kernel applies. Results are identical; for A/B measurements and tests. */
#define PKV_FLAG_STAGED 16u
/* pkv_evict_desc.flags bit 5: pkv_evict_prefill runs the WHOLE eviction (stages 1-4) as one persistent launch where the
 * shape allows. Identical results; it adds five cross-CTA exchanges through global memory. Kept for experiments and tests. */
#define PKV_FLAG_SINGLE_LAUNCH 32u
/* pkv_evict_desc.flags bit 6: run stages 1-2 as ONE persistent launch (pkv_evict_fused.cu: the logits stay in shared
 * memory, the CTAs of a kv head exchange softmax partials and pooling halos through flag words) followed by the select
 * kernel, for every shape that kernel supports. Identical results. Not the default: its flag waits need every CTA to be
 * co-resident, which only the slower cooperative launch guarantees. */
#define PKV_FLAG_FUSED 64u
/* pkv_evict_desc.flags bit 7: GQA-shared selection — ONE compacted cache per KV head instead of one per query head.
 * k_cache / v_cache / cache_stride_h then describe [num_kv_heads, >= top_k+window, head_dim] and idx_out is
 * [num_kv_heads, top_k]. With G = num_q_heads / num_kv_heads:
 *  - PyramidKV, SnapKV, H2O: stage 2 writes `pooled` [num_q_heads][S-W] exactly as without the flag; a group reduction then
 *    writes pooled_kv[j][t] = rn_dtype((sum over g = 0..G-1, ascending, in fp32, of f32(pooled[j*G+g][t])) / f32(G)) (one
 *    correctly rounded fp32 division, one rounding to the model dtype) into a workspace segment of its own
 *    (pkv_evict_pooled_kv_offset), and
 *    stages 3-4 run over num_kv_heads "heads" with G = 1 on it: KV head j keeps K[j] / V[j] at its top_k indices under the
 *    stage-3 tie rule, in score order, followed by the last `window` rows. The reduction follows the pooling, so with
 *    maxpool the mean of pooled scores is not the pool of the mean.
 *  - StreamingLLM, L2Norm: the selection does not depend on the query head; each KV head is selected directly (the cache
 *    of the flagless call with the G identical copies removed). L2Norm's key norms are computed per KV head in `pooled`.
 * With G = 1 the flag changes nothing. PKV_FLAG_FUSED / PKV_FLAG_SINGLE_LAUNCH and the layer batch (pkv_evict_prefill_batch,
 * pkv_evict_batch_supported, pkv_stage_batch) return PKV_ERR_UNSUPPORTED with it, as do pkv_stage_scan_pool,
 * pkv_adakv_counts and pkv_ragged_place_window. The stage entry points follow the same split: pkv_stage_pool includes
 * the group reduction, pkv_stage_topk / pkv_stage_gather run per KV head. */
#define PKV_FLAG_GQA_SHARED 128u
/* Flags outside this set are rejected with PKV_ERR_INVALID_ARG. */
#define PKV_EVICT_KNOWN_FLAGS 255u

/* One layer's prefill eviction: the body of *KVCluster.update_kv with merge=None. */
typedef struct pkv_evict_desc {
    uint32_t struct_bytes; /* = sizeof(pkv_evict_desc); ABI check */
    int32_t method;        /* pkv_method */
    int32_t dtype;         /* pkv_dtype */
    int32_t pooling;       /* pkv_pooling (ignored by H2O / StreamingLLM) */
    int32_t kernel_size;   /* pooling kernel, odd */
    int32_t num_q_heads;
    int32_t num_kv_heads;
    int32_t head_dim;      /* 64 or 128 */
    int32_t window;        /* self.window_size; multiple of 8 for the scoring methods; 0 for PKV_L2NORM */
    int32_t device;        /* CUDA device ordinal the pointers live on */
    int64_t seq_len;       /* q_len == kv_len of the prompt */
    int64_t top_k;         /* rows kept from the first seq_len-window tokens (pkv_layer_budget) */
    const void* q; int64_t q_stride_h; int64_t q_stride_s;
    const void* k; int64_t k_stride_h; int64_t k_stride_s;
    const void* v; int64_t v_stride_h; int64_t v_stride_s;
    void* k_cache;         /* [num_q_heads, >= top_k+window rows, head_dim] */
    void* v_cache;
    int64_t cache_stride_h; /* elements between consecutive heads of the cache (= capacity*head_dim) */
    int64_t* idx_out;      /* optional [num_q_heads, top_k] int64 selected token indices, may be NULL */
    void* workspace;
    uint64_t workspace_bytes;
    uint32_t flags;        /* PKV_SCORE_* | PKV_FLAG_WINDOW_MEAN | PKV_FLAG_INPUTS_READY | PKV_FLAG_STAGED | PKV_FLAG_SINGLE_LAUNCH |
                            * PKV_FLAG_FUSED | PKV_FLAG_GQA_SHARED */
    uint32_t reserved;
} pkv_evict_desc;

/* Byte offsets of the scratch segments inside `workspace` (for stage-injection tests and debugging). */
typedef struct pkv_ws_layout {
    uint64_t total_bytes;
    uint64_t logits_off;    /* dtype [num_kv_heads][s_pad][nw], nw = group*window; masked logits */
    uint64_t partial_off;   /* float2 (max, sumexp) [num_kv_heads][n_slots][nw] */
    uint64_t pooled_off;    /* dtype [num_q_heads][pooled_pitch]: pooled scores = top-k input (L2Norm: negated key norms) */
    uint64_t idx32_off;     /* int32 [num_q_heads][top_k] */
    uint64_t h2o_stats_off; /* float2 (row max, row sumexp) [num_q_heads][s_pad] (H2O only) */
    uint64_t h2o_acc_off;   /* float [num_q_heads][pooled_pitch] column-sum accumulators (H2O only) */
    int64_t s_pad;          /* seq_len rounded up to the 128-token tile */
    int64_t n_slots;        /* partial-statistics slots per kv head */
    int64_t nw;             /* columns per token in `logits` */
    int64_t pooled_pitch;   /* elements per pooled row */
    uint64_t fused_off;     /* window methods: exchange area of the single-launch kernel (epoch u64, status u32 at +8, flags,
                             * histogram tables, winner lists). status != 0 after a launch = a cross-CTA wait timed out. */
} pkv_ws_layout;

int pkv_version(void);
const char* pkv_last_error(void);
/* Number of CUDA kernels this library has launched in the calling process (for bench accounting). */
uint64_t pkv_launch_count(void);
/* Host-buffer plugin path only (no device work): picks rows of a HOST-resident [Hkv, S, row] tensor into a dense
 * host [Hq, n_rows, row] buffer, query head h reading kv head h / (Hq/Hkv) — the host half of
 * `past_key_value` compaction (pyramidkv_utils.py:271-282) when V lives in host memory: the GPU selects the indices
 * from K and Q, V itself never crosses the bus. `rows` is [Hq][n_rows] int64 (selected indices, then the window).
 * Returns PKV_OK or PKV_ERR_INVALID_ARG (null pointer, bad head counts, a row index outside [0, seq_len)). */
int pkv_host_pick_rows(const void* src, int64_t src_stride_h_bytes, int64_t src_stride_s_bytes, int64_t seq_len,
                       int32_t num_kv_heads, int32_t num_q_heads, int64_t row_bytes, const int64_t* rows, int64_t n_rows,
                       void* dst);

/* Diagnostics only (not part of the reference-facing boundary): with PKV_STAMPS=1 in the environment, one CTA of the
 * score kernel and one cluster leader of the select kernel write %globaltimer stamps (ns) at their phase boundaries into
 * a device buffer; this copies up to 128 of them out (caller synchronises the stream first). Returns the count
 * copied, 0 when disabled. Slots: [0,64) select kernel, [64,128) score kernel (tools/stamps.py names them). */
int pkv_debug_read_stamps(uint64_t* out, int count);

/* Per-layer budget: pyramidkv_utils.py:205-215 (PyramidKV pyramid), branches :218-220, and
 * k = max_capacity_prompt - window_size for SnapKV (:334) / H2O (:562) / StreamingLLM (:607);
 * PKV_L2NORM (window = 0): k = max_capacity_prompt (:429-430).
 * *mode_out: 0 = q_len < max_capacity_prompt, K/V kept whole (no eviction); 1 = evict with *top_k_out.
 * PKV_ERR_INVALID_ARG mirrors `assert self.max_capacity_prompt - self.window_size > 0` (:184). */
int pkv_layer_budget(int method, int64_t max_capacity_prompt, int64_t window, int num_layers, int layer_idx,
                     int64_t q_len, int beta, int64_t* top_k_out, int* mode_out);

/* Workspace size / layout for pkv_evict_prefill and its stage entry points. */
int pkv_evict_workspace_layout(const pkv_evict_desc* d, pkv_ws_layout* out);
uint64_t pkv_evict_workspace_bytes(const pkv_evict_desc* d);
/* PKV_FLAG_GQA_SHARED with a scoring method (not StreamingLLM): *off_out = byte offset in the workspace of the per-KV-head top-k
 * input, dtype [num_kv_heads][pooled_pitch] (the group reduction of `pooled`; = pooled_off for L2Norm and when G = 1). For
 * stage-level tests and debugging; kept out of pkv_ws_layout so that the struct callers allocate keeps its size.
 * PKV_ERR_INVALID_ARG without the flag, for StreamingLLM (no scores) or a null pointer. */
int pkv_evict_pooled_kv_offset(const pkv_evict_desc* d, uint64_t* off_out);

/* Whole eviction of one layer = stages 1-4 below on `stream` (three launches: window scores; softmax + pool; select +
 * gather). PKV_FLAG_FUSED / PKV_FLAG_SINGLE_LAUNCH select the fused forms (identical results) where the shape allows
 * (group*window in {32, 64}, window 8 or 16, <= 15-16 score tiles per CTA: e.g. Llama-3-8B up to ~37K tokens).
 * Replaces PyramidKVCluster.update_kv pyramidkv_utils.py:197-283, SnapKVCluster.update_kv :306-347,
 * H2OKVCluster.update_kv :533-575, StreamingLLMKVCluster.update_kv :595-620 and the repeat_kv copies
 * in front of them (llama_model.py:158-159). */
int pkv_evict_prefill(const pkv_evict_desc* d, void* stream);
/* The eviction of SEVERAL layers of one prompt in one pass: four launches per 32 layers (window scores of all layers on one
 * persistent grid; merge of the softmax partials; softmax + pool; select + gather) instead of three per layer. Results are those of pkv_evict_prefill on
 * each descriptor. The reference evicts inside every layer's attention forward (llama_model.py:165-168), but a layer's
 * eviction reads only that layer's q / k / v and writes only that layer's cache, and nothing reads the compacted cache before
 * the first decode step - so the patched forward may park the descriptors and evict all layers once the last layer's K / V
 * exist (pyramidkv_b200/attention.py, knob pkv_defer_eviction). `descs` = n_layers descriptors, each with its own tensors,
 * caches, workspace and top_k (PyramidKV budgets differ per layer); method in {PKV_PYRAMIDKV, PKV_SNAPKV}, identical geometry,
 * dtype, knobs and flags, seq_len >= 897, every top_k inside the cluster select kernel: otherwise PKV_ERR_UNSUPPORTED and
 * nothing is launched (pkv_evict_batch_supported asks without launching; the caller then evicts layer by layer). */
int pkv_evict_prefill_batch(const pkv_evict_desc* descs, int n_layers, void* stream);
int pkv_evict_batch_supported(const pkv_evict_desc* descs, int n_layers);
/* One stage of the layer batch, for measurements and stage-level tests: 0 = all (= pkv_evict_prefill_batch), 1 = window scores
 * (pkv_stage_scores of every layer), 2 = softmax + pool, 3 = select + gather. */
int pkv_stage_batch(const pkv_evict_desc* descs, int n_layers, int stage, void* stream);
/* How pkv_evict_prefill(d) runs: 0 = staged launches (or d is invalid); 1 = stages 1-2 in one persistent launch
 * (pkv_evict_fused.cu) followed by the select kernel; 2 = stages 1-4 in one launch (PKV_FLAG_SINGLE_LAUNCH). */
int pkv_evict_single_launch(const pkv_evict_desc* d);
/* Stages 1+2 in one launch for every shape the fused kernel supports (PKV_ERR_UNSUPPORTED otherwise): leaves `pooled` in the
 * workspace like pkv_stage_scores + pkv_stage_pool (the logits segment is not written). */
int pkv_stage_scan_pool(const pkv_evict_desc* d, void* stream);

/* Stage 1 — observation-window logits: matmul, /sqrt(head_dim), mask add with the reference's rounding
 * chain; writes `logits` and per-tile softmax partials into the workspace. pyramidkv_utils.py:253-260.
 * (H2O: row statistics of the full S x S product, :544-551.) */
int pkv_stage_scores(const pkv_evict_desc* d, void* stream);
/* Stage 2 — softmax(fp32)->dtype, window-row sum, 1-D pool -> `pooled`. pyramidkv_utils.py:262-269.
 * (H2O: column sums over all rows, :553-561.) */
int pkv_stage_pool(const pkv_evict_desc* d, void* stream);
/* Stage 3 — per-head top-k of `pooled` -> idx32 (and idx_out). pyramidkv_utils.py:270. Tie rule: every
 * element above the k-th value, then the lowest indices among those equal to it; order (value desc, index asc). */
int pkv_stage_topk(const pkv_evict_desc* d, void* stream);
/* Stage 4 — K/V gather + last-window concat written into the cache. pyramidkv_utils.py:271-282. */
int pkv_stage_gather(const pkv_evict_desc* d, void* stream);

/* Decode step over the compacted cache (q_len == 1, every cached row visible).
 * Replaces DynamicCache.update's torch.cat (cache_utils_think.py:383-384 / llama_model.py:170) and the
 * attention call llama_model.py:174-183 (eager) / :291-313 (sdpa) / :411-445 (flash). */
typedef struct pkv_decode_desc {
    uint32_t struct_bytes;
    int32_t dtype;
    int32_t num_q_heads;
    int32_t num_kv_heads;
    int32_t head_dim;       /* 64 or 128 */
    int32_t device;
    int64_t length;         /* valid rows per head AFTER the optional append */
    const void* q;          /* [num_q_heads, head_dim] contiguous */
    const void* k_new;      /* optional [num_kv_heads, head_dim]: appended as row length-1 of every head */
    const void* v_new;
    void* k_cache;          /* [num_q_heads, capacity, head_dim] */
    void* v_cache;
    int64_t cache_stride_h;
    void* out;              /* [num_q_heads, head_dim] contiguous */
    void* workspace;        /* pkv_decode_workspace_bytes */
    uint64_t workspace_bytes;
    float softmax_scale;    /* 0 => 1/sqrt(head_dim) */
    uint32_t reserved;
} pkv_decode_desc;

uint64_t pkv_decode_workspace_bytes(const pkv_decode_desc* d);
int pkv_decode_attn(const pkv_decode_desc* d, void* stream);
/* The same decode step in a form a CUDA graph can replay (SURVEY.md §8 f3: the generate loop after the path —
 * llama_model.py:401-404, cache_utils_think.py:383-384, positions llama_model.py:2617-2631). `d->length` is the row
 * count AFTER the append at step 0; the kernel adds the int32 `*step_dev` (device memory, advanced by the caller once
 * per generated token, shared by all layers) so the captured launch parameters never change. The launch is sized for
 * `max_length` rows (>= length + largest step; must fit the cache: cache_stride_h >= max_length*head_dim) and needs
 * the same workspace as pkv_decode_attn. Results are those of pkv_decode_attn with length + *step_dev up to the
 * summation order across splits. */
int pkv_decode_attn_graph(const pkv_decode_desc* d, const int32_t* step_dev, int64_t max_length, void* stream);
/* The decode step of num_seqs sequences in ONE launch (grid: split x q head x sequence). Replaces, for a batch, the
 * per-layer torch.cat of the whole batched cache (cache_utils_think.py:383-384, llama_model.py:170) and the attention call
 * llama_model.py:174-183 / :291-313 / :411-445 — batch inference, which the reference lists as unsupported (README.md:47).
 * Sequence s, query head h: cache at k_cache + s*cache_stride_b + h*cache_stride_h, query q[s][h], output out[s][h]
 * (q, out: [num_seqs, num_q_heads, head_dim] contiguous); it appends k_new[s][h / group] / v_new[s][h / group]
 * (k_new, v_new: [num_seqs, num_kv_heads, head_dim] contiguous, optional) as its last row and attends
 *     rows = d->length (+ *step_dev when step_dev != NULL) (+ rows[s*num_q_heads + h] when rows != NULL)
 * rows; `rows` is DEVICE int32 [num_seqs*num_q_heads] (prompts whose compacted caches differ in length, AdaKV / HeadKV
 * heads). Graph-replayable like pkv_decode_attn_graph: the launch is sized for `max_length` rows (cache_stride_h >=
 * max_length*head_dim), row counts are read on the device, and each (sequence, head) divides its rows among the splits a
 * one-sequence launch uses, so every sequence's output and appended row are bit-identical to pkv_decode_attn_graph /
 * pkv_decode_attn_ragged on that sequence alone. A (sequence, head) whose row count falls outside [1, max_length] reads
 * and writes no row; its output is NaN. Workspace: pkv_decode_workspace_bytes with num_q_heads = num_seqs*num_q_heads.
 * PKV_ERR_INVALID_ARG: num_seqs outside [1, 65535], cache_stride_b < num_q_heads*cache_stride_h, max_length < length or
 * above the capacity, misaligned rows / step_dev. */
int pkv_decode_attn_batch(const pkv_decode_desc* d, int32_t num_seqs, int64_t cache_stride_b, const int32_t* rows,
                          const int32_t* step_dev, int64_t max_length, void* stream);
/* The opt-in FP8 compacted cache. K and V are stored as E4M3 bytes ([num_seqs, num_q_heads, capacity, head_dim], one byte
 * per element) with one fp32 scale per (sequence, head, row) for each: [num_seqs, num_q_heads, capacity]. A 16-bit row x
 * is stored as amax = max|x_e| (fp32); amax == 0: scale 0 and every byte 0; otherwise inv = rn_f32(448 / amax),
 * q_e = E4M3(rn_f32(x_e * inv)) rounded to nearest even and saturated to +-448 (cvt.rn.satfinite.e4m3x2.f32), scale =
 * rn_f32(amax / 448). Row e stands for float(q_e) * scale. (The reference's --quant_method caches are HQQ-based and are
 * not built here.)
 *
 * pkv_decode_attn_batch_fp8 = pkv_decode_attn_batch over such a cache, with the same row count rule, split rule,
 * out-of-range behaviour (NaN output, nothing read or written), workspace (pkv_decode_workspace_bytes with num_q_heads =
 * num_seqs*num_q_heads) and graph replayability: every sequence's output and appended row are bit-identical to a
 * num_seqs = 1 launch on that sequence alone. It is the only FP8 decode entry point: a single sequence (host-launched or
 * in a graph) is num_seqs = 1, with step_dev = NULL and rows = NULL for a host launch of `length` rows. d->dtype is the
 * dtype of q, k_new, v_new and out; d->k_cache / d->v_cache point at the E4M3 bytes and cache_stride_h counts bytes
 * (a multiple of 16, >= max_length*head_dim; cache_stride_b likewise). Sequence s, head h reads its scales at
 * k_scale / v_scale + s*scale_stride_b + h*scale_stride_h (floats; scale_stride_h >= max_length). The CTA that owns the
 * last row quantises k_new[s][h / group] / v_new[s][h / group] with the rule above, stores its bytes and scale, and attends
 * that quantised row: the output is the attention (fp32 online softmax, as pkv_decode_attn) over exactly the rows the
 * cache holds. PKV_ERR_INVALID_ARG additionally for null or misaligned scale pointers and too small scale strides. */
int pkv_decode_attn_batch_fp8(const pkv_decode_desc* d, int32_t num_seqs, int64_t cache_stride_b, const int32_t* rows,
                              const int32_t* step_dev, int64_t max_length, float* k_scale, float* v_scale, int64_t scale_stride_h,
                              int64_t scale_stride_b, void* stream);
/* The decode step over GQA-shared caches (PKV_FLAG_GQA_SHARED): one cache per KV head, [num_seqs, num_kv_heads, capacity,
 * head_dim], read ONCE for the G = num_q_heads / num_kv_heads query heads of its group (G in {2, 4, 8}). q / out are
 * [num_seqs, num_q_heads, head_dim] and k_new / v_new [num_seqs, num_kv_heads, head_dim]; cache_stride_h counts the elements
 * (FP8: bytes) between KV heads and cache_stride_b those between sequences (>= num_kv_heads*cache_stride_h). Sequence s, KV
 * head j attends rows = d->length (+ *step_dev) (+ rows[s*num_kv_heads + j]), `rows` DEVICE int32 [num_seqs*num_kv_heads].
 * Grid (split, KV head, sequence): one CTA reads each row once and computes all G query heads (G = 8 on the FP8 cache: two
 * CTAs of four heads each). The split count is the one pkv_decode_attn_batch uses for num_q_heads heads and that row count,
 * and the partials stay per query head, so the workspace is pkv_decode_workspace_bytes with num_q_heads =
 * num_seqs*num_q_heads. Query head h's output and the appended row are bit-identical to pkv_decode_attn_batch /
 * pkv_decode_attn_batch_fp8 over the same cache repeat-interleaved G times along the heads. The CTA that owns the last row
 * stores (FP8: quantises and stores) k_new / v_new of its KV head once and attends it as stored. Graph replayability,
 * NaN output for a row count outside [1, max_length] and argument errors follow pkv_decode_attn_batch /
 * pkv_decode_attn_batch_fp8; G outside {2, 4, 8} is PKV_ERR_UNSUPPORTED. FP8 scales: [num_seqs, num_kv_heads, capacity]. */
int pkv_decode_attn_batch_gqa(const pkv_decode_desc* d, int32_t num_seqs, int64_t cache_stride_b, const int32_t* rows,
                              const int32_t* step_dev, int64_t max_length, void* stream);
int pkv_decode_attn_batch_gqa_fp8(const pkv_decode_desc* d, int32_t num_seqs, int64_t cache_stride_b, const int32_t* rows,
                                  const int32_t* step_dev, int64_t max_length, float* k_scale, float* v_scale,
                                  int64_t scale_stride_h, int64_t scale_stride_b, void* stream);
/* The decode step with a decode window: each (sequence, cache head) keeps its P prompt rows plus a ring of its last
 * `window` = R appended rows, so generation of any length needs P + R rows. Any cache form: a cache per query head or a
 * GQA-shared one (`gqa_shared`), 16-bit rows or E4M3 rows (`k_scale` / `v_scale` non-NULL, with the layout, quantisation
 * and strides of pkv_decode_attn_batch_fp8). The logical row count n = d->length (+ *step_dev) (+ rows[s*H + c]) is that
 * of pkv_decode_attn_batch / _gqa / _fp8 (H = num_q_heads, or num_kv_heads when gqa_shared), and P = prompt_rows[s*H + c]
 * (DEVICE int32). While n <= P + R the step is exactly the unwindowed one: it stores the new row at n - 1 and attends
 * rows [0, n). Once n > P + R, the j-th appended row (j = n - 1 - P) is stored at P + j mod R, replacing the oldest, and
 * rows [0, P + R) are attended, in physical order, the new row as stored; positions are those the caller rotated K with.
 * Every output, appended row and scale is then bit-identical to pkv_decode_attn_batch / _gqa / _fp8 / _gqa_fp8 run
 * without k_new on the same buffer with the new row already at its ring slot and P + min(n - P, R) rows. A count n < 1,
 * P < 0 or an attended count above max_length reads and writes no row; its output is NaN. The caller keeps max_length
 * >= P + R for every (sequence, cache head) whose ring fills (it cannot be checked on the host for device P), as it keeps
 * the counts of `rows` within max_length. Graph-replayable like pkv_decode_attn_batch: n and P are read on the device.
 * Workspace: pkv_decode_workspace_bytes with num_q_heads = num_seqs*num_q_heads. PKV_ERR_INVALID_ARG, in addition to the
 * errors of the entry point of the same cache form: w NULL or w->struct_bytes != sizeof(pkv_decode_window), window < 1,
 * prompt_rows NULL or not 4-byte aligned. */
typedef struct pkv_decode_window {
    uint32_t struct_bytes;
    int32_t num_seqs;
    int64_t cache_stride_b;     /* elements (E4M3: bytes) between the caches of consecutive sequences */
    int32_t gqa_shared;         /* 0: a cache per query head; 1: one per KV head (group in {2, 4, 8}) */
    int32_t reserved;
    const int32_t* rows;        /* optional DEVICE int32 [num_seqs*H], as pkv_decode_attn_batch */
    const int32_t* prompt_rows; /* DEVICE int32 [num_seqs*H]: P of each (sequence, cache head) */
    const int32_t* step_dev;    /* optional DEVICE int32 step counter */
    int64_t max_length;         /* the rows the launch is sized for: cache_stride_h >= max_length*head_dim */
    float* k_scale;             /* E4M3 rows: fp32 row scales [num_seqs, H, capacity]; NULL for 16-bit rows */
    float* v_scale;
    int64_t scale_stride_h, scale_stride_b;
    int64_t window;             /* R >= 1 */
} pkv_decode_window;
int pkv_decode_attn_window(const pkv_decode_desc* d, const pkv_decode_window* w, void* stream);
/* The decode window with heavy hitters (H2O's decode-time rule): the victim is the generated row with the least
 * accumulated attention, while the R - H most recent rows always stay. `w` is the window of pkv_decode_attn_window (same
 * forms, layouts, row counts, checks and out-of-range rule); `h` adds H = h->heavy in [0, R - 1] and the state of one layer,
 * DEVICE memory the caller owns, with H = num_q_heads (or num_kv_heads when gqa_shared) cache heads per sequence:
 *   scores fp32  [num_seqs*H][R]  A, the accumulated attention of the generated row held in each slot (slot k = row P + k);
 *   gen    int32 [num_seqs*H][R]  the generation index of that row;
 *   victim int32 [num_seqs*H]     the row the next appended row replaces once the window is full.
 * Semantics, per (sequence, cache head) with P prompt rows. The j-th generated row (j = 0 is the prefill's token, appended at
 * logical count n = P + j + 1) has a score A_j that starts from 0 at the step that appends it. At every step, query head h
 * gives each row r it attends the probability p = expf(s_r - m_h) / l_h (an IEEE fp32 division), where s_r is the softmax
 * input of the row as the kernel computes it (for E4M3 rows with the row's K scale) and m_h, l_h are the fp32 maximum and
 * sum the output of head h is normalised by at this step. Every held generated row, the new one included, then adds
 * (sum over the query heads reading this cache head, in ascending head order, of p), in fp32: one head for a cache per query
 * head, the G heads of the group for a GQA-shared one. Prompt rows are never scored or evicted.
 *   While n <= P + R the step is the ring's (and the unwindowed one's): the row goes to n - 1.
 *   Once n > P + R the new row j takes the slot of the victim: among the held generated rows of generation index
 *   <= j - (R - H) (every held row but the R - H - 1 most recent), the one with the smallest A after step n - 1, ties to the
 *   smallest generation index. So H + 1 rows compete at each step, and the R - H most recent rows always stay.
 *   When no row qualifies (a count that repeats appends generation j again, as a finished slot of continuous batching
 *   does, until every held row is that recent), victim = -1 and the following full-window steps are out of range.
 *   H = 0 is the ring: the only candidate is the oldest row, at P + j mod R, so the cache is bit-identical to
 *   pkv_decode_attn_window's.
 * A step's output and appended row are bit-identical to pkv_decode_attn_batch / _gqa / _fp8 / _gqa_fp8 run without k_new
 * over the same buffer with the new row already at its slot. A count n < 1, P < 0, an attended count above max_length, or a
 * victim outside [P, P + R) reads and writes nothing (no cache row, no score, no victim) and gives a NaN output; a count
 * n <= P appends inside the prompt as the unwindowed step does and scores nothing. Every write stays inside rows
 * [0, P + R). The arithmetic is fixed-order fp32 without atomics: state and outputs do not depend on the thread schedule,
 * and a graph replay writes the bits of a host launch. A new (sequence, cache head) needs no reset: the rows it appends
 * overwrite the slots it reads. Launches: the decode (and its combine) and one small bookkeeping kernel.
 * `scratch` holds the per-step logits and (m, l): pkv_decode_heavy_workspace_bytes(num_seqs, num_q_heads, R) bytes, one
 * buffer for every layer (the launches are stream-ordered). PKV_ERR_INVALID_ARG, in addition to pkv_decode_attn_window's
 * errors: h NULL or h->struct_bytes != sizeof(pkv_decode_heavy), heavy outside [0, R - 1], k_new or v_new NULL, a NULL or
 * not 4-byte aligned scores / gen / victim / scratch. PKV_ERR_WORKSPACE: scratch_bytes too small. */
typedef struct pkv_decode_heavy {
    uint32_t struct_bytes;
    int32_t reserved;
    int64_t heavy;              /* H in [0, window - 1] */
    float* scores;              /* DEVICE fp32 [num_seqs*H][window] */
    int32_t* gen;               /* DEVICE int32 [num_seqs*H][window] */
    int32_t* victim;            /* DEVICE int32 [num_seqs*H] */
    void* scratch;              /* DEVICE, pkv_decode_heavy_workspace_bytes */
    uint64_t scratch_bytes;
} pkv_decode_heavy;
int pkv_decode_attn_heavy(const pkv_decode_desc* d, const pkv_decode_window* w, const pkv_decode_heavy* h, void* stream);
/* Bytes of the per-step scratch of pkv_decode_attn_heavy: num_seqs*num_q_heads*(window + 2) floats; 0 for a count below 1. */
uint64_t pkv_decode_heavy_workspace_bytes(int32_t num_seqs, int32_t num_q_heads, int64_t window);
/* Conversion of the compacted 16-bit caches of num_layers layers (one prompt, or one equal-length batch of num_seqs
 * sequences) to the FP8 format above, in one launch per 32 layers; the per-layer tables travel as kernel parameters.
 * Layer l: src[2l] / src[2l+1] = K / V, 16-bit contiguous [num_seqs, num_heads, src_capacity[l], head_dim]; dst[2l] /
 * dst[2l+1] = E4M3 [num_seqs, num_heads, dst_capacity[l], head_dim]; scales[2l] / scales[2l+1] = fp32 [num_seqs,
 * num_heads, dst_capacity[l]]. Every (sequence, head) converts rows[l] rows, or, when rows_dev != NULL and rows_dev[l] !=
 * NULL, the DEVICE int32 count rows_dev[l][s*num_heads + h] (AdaKV / HeadKV heads), which must not exceed rows[l]. Rows
 * past the count are neither read nor written. Pointers to 16-bit / E4M3 data are 16-byte aligned. */
int pkv_cache_quantize_fp8(int32_t dtype, int32_t num_seqs, int32_t num_heads, int32_t head_dim, int32_t device, int32_t num_layers,
                           const void* const* src, void* const* dst, float* const* scales, const int64_t* src_capacity,
                           const int64_t* dst_capacity, const int64_t* rows, const int32_t* const* rows_dev, void* stream);
/* Admission of one prompt into slot `slot` of a batched compacted cache (continuous batching), in one launch per 32 layers;
 * the per-layer tables travel as kernel parameters. Layer l: src[2l] / src[2l+1] = the prompt's K / V, [num_heads,
 * src_capacity[l], head_dim] elements of elem_bytes bytes (2: bf16 / fp16; 1: E4M3); dst[2l] / dst[2l+1] = the batched
 * buffers [num_seqs, num_heads, dst_capacity[l], head_dim]. With elem_bytes 1, src_scales / dst_scales hold the fp32 row
 * scales, [num_heads, src_capacity[l]] and [num_seqs, num_heads, dst_capacity[l]]; with elem_bytes 2 dst_scales is NULL.
 * Head h copies n_h = rows[l] rows, or, when rows_dev != NULL and rows_dev[l] != NULL, n_h = min(rows[l],
 * rows_dev[l][h]) (DEVICE int32, AdaKV / HeadKV heads). The same launch writes the decode row counts
 *     dst_rows[l][slot*num_heads + h] = n_h - *step_dev
 * so that the next decode step (which attends length 1 + *step_dev + rows rows) appends row n_h and attends n_h + 1 rows:
 * the host never reads the step counter. rows[l] = 0 parks the slot (src may be NULL): each later step attends and
 * overwrites row 0. Rows past n_h and every other slot are neither read nor written; the launch replays in a CUDA graph.
 * PKV_ERR_INVALID_ARG: slot outside [0, num_seqs), rows above a capacity, null or misaligned pointers (16 bytes for K / V,
 * 4 for scales and row counts), scale tables that do not match elem_bytes. */
int pkv_cache_install(int32_t elem_bytes, int32_t num_seqs, int32_t num_heads, int32_t head_dim, int32_t device, int32_t num_layers,
                      int32_t slot, const void* const* src, void* const* dst, const float* const* src_scales, float* const* dst_scales,
                      const int64_t* src_capacity, const int64_t* dst_capacity, const int64_t* rows, const int32_t* const* rows_dev,
                      int32_t* const* dst_rows, const int32_t* step_dev, void* stream);
/* Append only (no attention): writes k_new/v_new as row length-1. */
int pkv_cache_append(const pkv_decode_desc* d, void* stream);

/* The step in front of the path (SURVEY.md §8 f2): rotary embedding of Q [num_q_heads, seq_len, head_dim] and
 * K [num_kv_heads, seq_len, head_dim] IN PLACE, one launch. Replaces `apply_rotary_pos_emb(query_states, key_states,
 * cos, sin)` at llama_model.py:157 / :276 / :378 (mistral_model.py likewise): q*cos + rotate_half(q)*sin with the torch
 * rounding chain (every product and the sum rounded once to the model dtype) — results are bit-identical to the
 * torch op chain. cos / sin are [seq_len, head_dim] in the model dtype (what `rotary_emb` returns for one batch row),
 * `cs_stride_s` elements between tokens. Strides in elements, multiples of 8; pointers 16-byte aligned. */
typedef struct pkv_rope_desc {
    uint32_t struct_bytes;
    int32_t dtype;
    int32_t num_q_heads;
    int32_t num_kv_heads;
    int32_t head_dim;       /* 64 or 128 */
    int32_t device;
    int64_t seq_len;
    void* q; int64_t q_stride_h; int64_t q_stride_s;
    void* k; int64_t k_stride_h; int64_t k_stride_s;
    const void* cos;
    const void* sin;
    int64_t cs_stride_s;
} pkv_rope_desc;
int pkv_rope_inplace(const pkv_rope_desc* d, void* stream);

/* ---- ragged per-head budgets: AdaKV (pyramidkv_utils.py:622-757) and HeadKV (:760-878) ----
 * The cache keeps the padded [num_q_heads, capacity, head_dim] layout; head h holds head_rows[h] = cap_h + window rows
 * (then the decoded tokens) instead of the reference's flat tensor that is re-allocated and copied on every token
 * (update_flatten_view). Prefill of one layer, all on `stream`:
 *   1. pkv_stage_scores + pkv_stage_pool with method = PKV_SNAPKV and PKV_FLAG_WINDOW_MEAN (`calcul_attn_sore` :647-672).
 *   2. (AdaKV) pkv_adakv_counts: per head, how many of the globally largest num_q_heads*base_capacity (normalised)
 *      scores it owns — `counts` (DEVICE int32 [2*num_q_heads + 2]) = values above the threshold per head, values equal
 *      to it per head, the threshold's bit pattern, the total above. The host gives the tied slots to the lower heads
 *      first and applies the reference's float32 floor mix + round-half-even (:715). HeadKV takes its budgets from the
 *      runner's head-score file instead.
 *   3. pkv_stage_topk + pkv_stage_gather with top_k = max_h cap_h, then pkv_ragged_place_window: the last `window` rows go
 *      to rows [cap_h, cap_h + window) of head h (`caps` DEVICE int32 [num_q_heads], every cap_h <= top_k).
 * Decode: pkv_decode_attn_ragged = pkv_decode_attn with rows_h = d->length + head_rows[h] (+ *step_dev when given, as in
 * pkv_decode_attn_graph); d->length counts the rows appended so far including this step's. */
uint64_t pkv_adakv_scratch_bytes(int32_t num_q_heads);
int pkv_adakv_counts(const pkv_evict_desc* d, int64_t base_capacity, int32_t normalize, void* scratch, uint64_t scratch_bytes,
                     int32_t* counts, void* stream);
int pkv_ragged_place_window(const pkv_evict_desc* d, const int32_t* caps, void* stream);
int pkv_decode_attn_ragged(const pkv_decode_desc* d, const int32_t* head_rows, const int32_t* step_dev, int64_t max_length,
                           void* stream);

/* sm_90a counterpart of the reference's only native kernel: `update_flatten_view(cache, state, headlens, cu_headlens)`
 * (csrc/csrc/cuda_api.cu:11-85, Python binding tiny_api_cuda.update_flatten_view, called from
 * DynamicCacheSplitHeadFlatten.update pyramidkv_utils.py:63-66 for the AdaKV / HeadKV ragged caches). `src` is the flat
 * [total_rows, row] cache (heads back to back), `state` [num_heads, row] the new row of every head, `head_lens[h]` the
 * rows head h holds and `cu_lens[h]` the rows before it (int32, DEVICE memory, as the reference passes them; only
 * entries 0..num_heads-1 are read). Writes dst [total_rows + num_heads, row] = cat_h(src rows of h, state[h]).
 * `row_bytes` = head_dim * element size, a multiple of 16; all pointers 16-byte aligned. The reference allocates the
 * result inside the call and launches on the legacy default stream (cuda_api.cu:78); here the caller provides `dst`
 * and the stream. */
int pkv_update_flatten_view(void* dst, const void* src, const void* state, const int32_t* head_lens, const int32_t* cu_lens,
                            int32_t num_heads, int32_t row_bytes, int32_t device, void* stream);

/* ---- sampled decoding: one token per row of logits, in one launch for the batch (DESIGN.md §4.6) ----
 * Row b (logits[b*logits_stride .. + vocab), dtype bf16 / fp16) is drawn with its own device parameters temperature[b] = T
 * (fp32), top_k[b], top_p[b] (fp32), seed[b] and token index t = token_index[b]:
 *  1. T == 0 or top_k == 1: the argmax of the logits, first index among ties (torch.argmax); no random numbers.
 *  2. x_i = f32(logit_i) / T (IEEE fp32 division).
 *  3. top_k in [2, vocab): kappa = the top_k-th largest x; every token with x_i >= kappa is kept (ties at kappa included).
 *  4. top_p < 1: the kept tokens in (x descending, index ascending) order; the shortest prefix whose mass (softmax of x over
 *     the kept set) reaches top_p, at least one token. The masses are expf(x_i - max x) summed exactly in 64-bit fixed
 *     point (2^-40 units), so the prefix equals the exact one unless a prefix mass at the boundary lies within a relative
 *     1e-5 of top_p.
 *  5. token = argmax over the kept set of x_i + g_i (lowest index among ties), g_i = -log(-log(u_i)), u_i = (2*(r >> 9) + 1)
 *     * 2^-24 with r = word (i & 3) of Philox4x32-10(counter = {i >> 2, 0, lo32(t), hi32(t)}, key = {lo32(seed),
 *     hi32(seed)}): a draw from softmax(x) over the kept set that depends only on the logits, the parameters, seed and t.
 *  6. A row whose largest logit is NaN (torch.argmax's order: NaN above everything) or whose largest x is not finite
 *     (+-inf, or an overflow of the division) gets the argmax of rule 1.
 * Parameters are read on the device, so they are not checked at the call: a row with T < 0, top_k < 0 or top_p outside
 * (0, 1] (or NaN) gets token -1. The token goes to tokens[b*tokens_stride + column]; with PKV_SAMPLE_ADVANCE, token_index[b]
 * is incremented after the draw. No allocation, no synchronisation, fixed launch arguments: the launch replays in a CUDA
 * graph with all per-request state in device memory. PKV_ERR_INVALID_ARG: batch outside [1, 2^20], vocab outside
 * [1, 2^24], logits_stride < vocab, column outside [0, tokens_stride), null or misaligned pointers (2 bytes for the
 * logits, 4 for temperature / top_k / top_p, 8 for seed / token_index / tokens), unknown flags. */
#define PKV_SAMPLE_ADVANCE 1u
typedef struct pkv_sample_desc {
    uint32_t struct_bytes;  /* = sizeof(pkv_sample_desc) */
    int32_t dtype;          /* pkv_dtype of the logits */
    int32_t device;
    int32_t batch;          /* rows */
    int64_t vocab;          /* logits per row */
    const void* logits; int64_t logits_stride;   /* elements between rows */
    const float* temperature;   /* [batch] device arrays */
    const int32_t* top_k;       /* 0: off */
    const float* top_p;         /* 1: off */
    const uint64_t* seed;
    int64_t* token_index;
    int64_t* tokens; int64_t tokens_stride; int64_t column;   /* int64 [batch, tokens_stride] */
    uint32_t flags;         /* PKV_SAMPLE_ADVANCE */
    uint32_t reserved;
} pkv_sample_desc;
int pkv_sample_tokens(const pkv_sample_desc* d, void* stream);
/* ---- the same draw with repetition, presence and frequency penalties and min-p (DESIGN.md §4.10) ----
 * Row b also has rho = repetition_penalty[b], presence = presence_penalty[b], frequency = frequency_penalty[b] and
 * min_p[b] (fp32), its prompt set P (prompt_mask[b*stride + v] != 0) and its generated-token counts
 * c[v] = counts[b*stride + v] (>= 0). Every operation below is one IEEE fp32 operation (no contraction):
 *  1. x_v = f32(logit_v).
 *  2. rho != 1 and (v in P or c[v] > 0): x_v = x_v < 0 ? x_v * rho : x_v / rho (HF's RepetitionPenaltyLogitsProcessor
 *     over the prompt and generated ids).
 *  3. c[v] > 0: x_v = (x_v - frequency * f32(c[v])) - presence (vLLM's order; generated tokens only).
 *  4. Rules 1-6 of pkv_sample_tokens on x in place of f32(logit): T == 0 or top_k == 1 gives the argmax of x (first index,
 *     NaN largest), as does a row whose largest x / T is not finite; top-k and top-p as there; then min-p keeps, of the
 *     top-p set, the tokens with expf(x_i / T - max_j x_j / T) >= min_p (fp32; the largest always stays).
 *  5. With PKV_SAMPLE_ADVANCE, counts[b*stride + token] += 1 as well as token_index[b] (not for a token -1).
 * A row with rho = 1, presence = frequency = 0 and min_p = 0 gets exactly pkv_sample_tokens' token (and its mask and counts
 * are not read); every row reads the parameters of both structs on the device: rho not in (0, inf), a non-finite presence
 * or frequency, or min_p outside [0, 1] (or NaN) also give token -1. Same launch properties as pkv_sample_tokens (one CTA
 * per row, no scratch, no allocation, no synchronisation, graph-replayable). PKV_ERR_INVALID_ARG: those of
 * pkv_sample_tokens, a null penalty struct or struct_bytes mismatch, null or misaligned parameter arrays (4 bytes) or counts
 * (4 bytes), a null prompt_mask, stride < vocab. */
typedef struct pkv_sample_penalty {
    uint32_t struct_bytes;  /* = sizeof(pkv_sample_penalty) */
    uint32_t reserved;
    const float* repetition_penalty;   /* [batch] device arrays; 1: off */
    const float* presence_penalty;     /* 0: off */
    const float* frequency_penalty;    /* 0: off */
    const float* min_p;                /* 0: off */
    const uint8_t* prompt_mask;        /* uint8 [batch, stride]: nonzero for the row's prompt tokens */
    int32_t* counts;                   /* int32 [batch, stride]: generated-token counts, updated by the launch */
    int64_t stride;                    /* elements between rows of prompt_mask and counts, >= vocab */
} pkv_sample_penalty;
int pkv_sample_tokens_penalized(const pkv_sample_desc* d, const pkv_sample_penalty* p, void* stream);

/* ---- generation constraints: the per-row rule terms of one step, from the row's token history (DESIGN.md §4.11) ----
 * Row b has a history h = history[b*history_stride ..] of n = history_len[b] token ids (its prompt, then every token
 * generated so far), prompt_len[b], flags[b] (PKV_RULE_*), no-repeat n-gram size N = ngram[b] (0: off), min_new =
 * min_new_tokens[b], and n_seq[b] rule sequences: sequence j has the tokens seq_tokens[b*tokens_stride + seq_off[b*
 * seq_stride + j] .. seq_off[.. + j + 1]) (length L >= 1), the kind seq_kind[b*seq_stride + j] and, for a bias, the fp32
 * value seq_bias[b*seq_stride + j]. One CTA per row:
 *  0. With `append`, h[n] = append[b*append_stride + append_column] and history_len[b] = n + 1 first (not when n already
 *     equals history_stride: a full history takes no more tokens).
 *  1. PKV_RULE_BIAS: bias[b*bias_stride + v] = 0 for every v < vocab, then, for each run of consecutive bias sequences
 *     with one last token v (the caller orders them: the single-token one first, then in its own order), bias[v] =
 *     (((0 + w_1) + m_2 w_2) + ...), where m_j w_j is w_j when the sequence applies and 0 otherwise; a single-token sequence
 *     always applies, a longer one when L <= n and its first L - 1 tokens equal the last L - 1 of h (HF's
 *     SequenceBiasLogitsProcessor, its dict order and its skip of sequences longer than the context).
 *  2. PKV_RULE_BAN | PKV_RULE_BAD: the 2 * W words (W = ceil(vocab / 32)) of ban[b*ban_stride ..] are cleared; bit v of
 *     words [0, W) ("set to -inf") is set for every token N > 0 bans (the last token of every N-gram of h whose first N - 1
 *     tokens are the last N - 1 of h: HF's NoRepeatNGramLogitsProcessor, nothing while n + 1 < N) and, while n -
 *     prompt_len[b] < min_new, for each of the n_eos ids eos[] (HF's MinNewTokensLengthLogitsProcessor); bit v of words
 *     [W, 2W) ("add -inf") for the last token of every bad-word sequence that applies as in 1 (HF's
 *     NoBadWordsLogitsProcessor; the caller drops the single-token bad words equal to an EOS id).
 *  3. stop[b] = 1 when a stop sequence equals the last L tokens of h (L <= n), else 0.
 * Token ids outside [0, vocab) in h, in the sequences or in eos[] ban nothing. A row with flags 0 only appends and writes
 * stop[b] = 0. No allocation, no synchronisation, fixed launch arguments: graph-replayable. PKV_ERR_INVALID_ARG: batch
 * outside [1, 2^20], vocab outside [1, 2^24], a null or misaligned (4 bytes; 8 for append) pointer, a null eos with n_eos
 * > 0, strides smaller than what they index (history_stride < 1, bias_stride < vocab, ban_stride < 2W, seq_stride < 2,
 * tokens_stride < 1, append_column outside [0, append_stride)). The device tables must hold n_seq[b] + 1 offsets per row
 * (n_seq[b] < seq_stride) and the sequences' tokens; they are not checked. */
#define PKV_RULE_BIAS 1     /* flags[b]: sequence bias */
#define PKV_RULE_BAN 2      /* no-repeat n-grams or min_new_tokens: "set to -inf" */
#define PKV_RULE_BAD 4      /* bad words: "add -inf" */
#define PKV_RULE_STOP 8     /* stop sequences */
#define PKV_SEQ_BIAS 0      /* seq_kind values */
#define PKV_SEQ_BAD 1
#define PKV_SEQ_STOP 2
typedef struct pkv_token_rules_desc {
    uint32_t struct_bytes;  /* = sizeof(pkv_token_rules_desc) */
    int32_t device;
    int32_t batch;
    int32_t vocab;
    int32_t* history; int64_t history_stride;   /* int32 [batch, history_stride] */
    int32_t* history_len;                       /* [batch] device arrays */
    const int32_t* prompt_len;
    const int32_t* flags;
    const int32_t* ngram;
    const int32_t* min_new_tokens;
    const int32_t* n_seq;
    const int32_t* seq_off; const int32_t* seq_kind; const float* seq_bias; int64_t seq_stride;   /* [batch, seq_stride] */
    const int32_t* seq_tokens; int64_t tokens_stride;                                                /* [batch, tokens_stride] */
    const int32_t* eos; int32_t n_eos;          /* the EOS ids of min_new_tokens */
    int32_t reserved;
    const int64_t* append; int64_t append_stride; int64_t append_column;   /* optional (null): the token to append */
    float* bias; int64_t bias_stride;           /* fp32 [batch, bias_stride] */
    uint32_t* ban; int64_t ban_stride;          /* uint32 [batch, ban_stride] */
    uint8_t* stop;                              /* [batch] */
} pkv_token_rules_desc;
int pkv_token_rules(const pkv_token_rules_desc* d, void* stream);

/* ---- the penalized draw with the rule terms of pkv_token_rules (DESIGN.md §4.11) ----
 * Row b with f = flags[b]: x_v = f32(logit_v); f & PKV_RULE_BIAS: x_v = x_v + bias[b*bias_stride + v]; then steps 2-3 of
 * pkv_sample_tokens_penalized; then f & PKV_RULE_BAN and bit v of the "set" words of ban[b*ban_stride ..]: x_v = -inf;
 * otherwise, f & PKV_RULE_BAD: x_v = x_v + (-inf if bit v of the "add" words is set, else 0) (so a +inf logit becomes
 * NaN, as in HF); then steps 4-5 of pkv_sample_tokens_penalized on x. Each operation is one IEEE fp32 operation. A row with
 * f & 7 == 0 reads none of bias and ban and gets exactly pkv_sample_tokens_penalized's token. Same launch properties as
 * pkv_sample_tokens. PKV_ERR_INVALID_ARG: those of pkv_sample_tokens_penalized, a null rules struct or struct_bytes
 * mismatch, null or misaligned (4 bytes) flags / bias / ban, bias_stride < vocab, ban_stride < 2 * ceil(vocab / 32). */
typedef struct pkv_sample_rules {
    uint32_t struct_bytes;  /* = sizeof(pkv_sample_rules) */
    uint32_t reserved;
    const int32_t* flags;                      /* [batch] */
    const float* bias; int64_t bias_stride;    /* as written by pkv_token_rules */
    const uint32_t* ban; int64_t ban_stride;
} pkv_sample_rules;
int pkv_sample_tokens_constrained(const pkv_sample_desc* d, const pkv_sample_penalty* p, const pkv_sample_rules* r,
                                  void* stream);

/* ---- token log-probabilities: the log-softmax of each row of logits at a token and at its top N (DESIGN.md §4.8) ----
 * Row b (logits[b*logits_stride .. + vocab), bf16 / fp16) is read as the model's raw distribution: x_i = f32(logit_i),
 * temperature 1, no filters (whatever a sampler does with the row). With m = max_i x_i and Z = sum_i expf(x_i - m), summed
 * exactly in 64-bit fixed point (2^-40 units, as pkv_sample_tokens sums its masses, so the result does not depend on the
 * thread schedule):  lp_i = (x_i - m) - logf(Z).  Written, at column c = column (+ *cursor when cursor is not NULL):
 *  - logprob[b*logprob_stride + c] (fp32) = lp_t of the token t = tokens[b*tokens_stride + tokens_column];
 *  - for n < top_n: top_ids[b*top_stride + c*top_n + n] (int64) and top_logprobs[same] (fp32), the row's top_n tokens in
 *    (logit descending, index ascending) order with their lp, so entry 0 is torch.argmax's token of a finite row.
 * A row with a NaN or +-inf logit gets NaN log-probabilities and top ids -1; so do top entries n >= vocab. A token outside
 * [0, vocab) gets NaN (device data: not an error). The error of lp against the exact log-softmax of the row is bounded in
 * DESIGN.md §4.8 (below 1e-5 absolute plus half an fp32 ulp of lp). No allocation, no synchronisation, fixed launch
 * arguments: the launch replays in a CUDA graph. PKV_ERR_INVALID_ARG: batch outside [1, 2^20], vocab outside [1, 2^24],
 * logits_stride < vocab, top_n outside [0, 20], tokens_column outside [0, tokens_stride), column < 0, logprob_stride <=
 * column, top_stride < (column + 1) * top_n, null or misaligned pointers (2 bytes for the logits, 4 for logprob /
 * top_logprobs, 8 for tokens / top_ids / cursor; top_ids and top_logprobs may be NULL when top_n = 0), unknown flags.
 * With a cursor the strides cannot bound the column it adds: the caller keeps column + *cursor inside its buffers. */
typedef struct pkv_logprobs_desc {
    uint32_t struct_bytes;  /* = sizeof(pkv_logprobs_desc) */
    int32_t dtype;          /* pkv_dtype of the logits */
    int32_t device;
    int32_t batch;          /* rows */
    int64_t vocab;          /* logits per row */
    const void* logits; int64_t logits_stride;   /* elements between rows */
    const int64_t* tokens; int64_t tokens_stride; int64_t tokens_column;   /* int64 [batch, tokens_stride] */
    int32_t top_n;          /* 0 .. 20 */
    uint32_t flags;         /* none defined: 0 */
    const int64_t* cursor;  /* optional device int64 added to column */
    int64_t column;
    float* logprob; int64_t logprob_stride;           /* fp32 [batch, logprob_stride] */
    int64_t* top_ids; float* top_logprobs; int64_t top_stride;   /* [batch, top_stride], top_n entries per column */
} pkv_logprobs_desc;
int pkv_token_logprobs(const pkv_logprobs_desc* d, void* stream);

/* ---- beam search: HF's `_beam_search` (do_sample=False) on the device (DESIGN.md §4.12) ----
 * The rules, restated in oracle/beam.py. P prompts of k = num_beams beams each (2 <= k <= 16), beam b = p*k + r. At
 * iteration t (t tokens generated before it, so each beam's cache holds t generated rows; t = 0 reads the prefill's
 * logits), with n_eos <= 4 EOS ids and K = max(2, 1 + n_eos) * k <= 80:
 *  1. pkv_beam_candidates, per beam row: m = max f32(l_v), log Z = logf(sum expf(f32(l_v) - m)) with Z summed exactly in
 *     64-bit fixed point (pkv_token_logprobs' rule), and the row's top K tokens (logit descending, index ascending) with
 *     lp_v = (f32(l_v) - m) - log Z. A row with a NaN or +-inf logit has no candidates (lp -inf, id -1).
 *  2. pkv_beam_step, per prompt (one CTA), every value fp32:
 *     c. score(r, v) = running[r] + lp_v; the top K of the k rows' entries by (score descending, flat index r*V + v
 *        ascending) are the candidates c = 0 .. K-1 (the global top K lies inside the union of each row's top K); entries
 *        of a non-finite row (id -1) come after every token of their row, in row order, and stand for token 0;
 *     d. hit_c: token v_c is an EOS id, or t + 1 = max_steps (the maximum length);
 *     e. running: the top k of score_c + (hit_c ? -1e9 : -0), (value descending, c ascending); beam slot a takes the
 *        a-th: its token, its parent slot r_c and that running score;
 *     f. pool: x_c = score_c * scale[t][0], then + -1e9 when every pool entry is finished and early_stopping is True, + -1e9
 *        when the early-stop heuristic already failed, + -1e9 unless hit_c and c < k; the new pool is the top k of the old
 *        k entries followed by the K x_c (value descending, index ascending); a new entry is finished when hit_c and c < k;
 *     g. heuristic' = heuristic && any_j (running[0] * scale[t][1] > (finished_j ? min pool score : -1e9));
 *        done = !heuristic' || (every pool entry finished && early_stopping is True) || t + 1 = max_steps.
 *     scale[t] = (f32(1 / (t + 1)^length_penalty), f32(1 / L^length_penalty)), the reciprocals taken in double, with L =
 *     max_steps when early_stopping is "never" and length_penalty > 0, else t + 1: torch's CUDA division of an fp32
 *     tensor by a Python float d multiplies by f32(1 / d). A done prompt is frozen: its state is not written; its beams take token 0 and keep their rows.
 *  3. pkv_cache_reorder moves each beam's cache to its parent's: slot a copies the generated rows [diverge[a], t) of slot
 *     parent[a] (nothing when parent[a] = a), where diverge[a] comes from the common-prefix matrix cp (k x k per prompt,
 *     generated rows two slots share): diverge[a] = parent[a] == a ? t : cp[a][parent[a]], cp'[a][b] = (pa == pb) ? t :
 *     cp[pa][pb]. */
#define PKV_MAX_BEAMS 16
#define PKV_MAX_BEAM_CANDIDATES 80
/* Candidates of `rows` rows of logits (bf16 / fp16, logits_stride elements apart), top_k = K <= 80: m [rows], log_z [rows],
 * cand_lp [rows, K] (fp32) and cand_id [rows, K] (int32), all DEVICE and contiguous. One CTA per row, fixed launch
 * arguments: it replays in a CUDA graph. PKV_ERR_INVALID_ARG: rows outside [1, 2^20], vocab outside [1, 2^24], stride <
 * vocab, top_k outside [1, 80], null or misaligned pointers (2 bytes for the logits, 4 for the outputs). */
int pkv_beam_candidates(int32_t dtype, int32_t device, int32_t rows, int64_t vocab, const void* logits, int64_t logits_stride,
                        int32_t top_k, float* m, float* log_z, float* cand_lp, int32_t* cand_id, void* stream);
/* One beam step of every prompt (rule 2 above). Every pointer is DEVICE memory; the iteration t = *step + step_offset is
 * read on the device, so the launch replays in a CUDA graph. cand_lp / cand_id: [P*k, K] from pkv_beam_candidates, or
 * with cand_rows_per_prompt = 1 one row per prompt, read for each of its k beams (iteration 0: the prefill's row).
 * running [P*k] fp32 (initially 0, -1e9, ..., -1e9 per prompt); the pool [P*k]: score (initially -1e9), its (step,
 * parent, token) handle (int32) and finished flag (uint8, initially 0); heuristic [P] (uint8, initially 1) and done [P]
 * (initially 0); backpointers bp_token / bp_parent [P*k, max_steps] (int32: iteration t writes column t); cp [P, k, k]
 * (int32, initially 0); outputs next_token [P*k] (int64), parent and diverge [P*k] (int32). */
typedef struct pkv_beam_step_desc {
    uint32_t struct_bytes;        /* = sizeof(pkv_beam_step_desc) */
    int32_t device;
    int32_t num_prompts, num_beams, top_k, cand_rows_per_prompt;
    int32_t n_eos;                /* 0 .. 4 */
    int32_t early_stopping;       /* 0: False, 1: True, 2: "never" */
    int32_t max_steps;            /* max_new_tokens */
    int32_t step_offset;
    const int32_t* step;
    const float* cand_lp; const int32_t* cand_id;
    const int32_t* eos;           /* [n_eos] */
    const float* scale;           /* [max_steps, 2] */
    float* running;
    float* pool_score; int32_t* pool_step; int32_t* pool_parent; int32_t* pool_token; uint8_t* pool_done;
    uint8_t* heuristic; uint8_t* done;
    int32_t* bp_token; int32_t* bp_parent;
    int32_t* cp;
    int64_t* next_token; int32_t* parent; int32_t* diverge;
} pkv_beam_step_desc;
int pkv_beam_step(const pkv_beam_step_desc* d, void* stream);
/* The beam reorder of num_layers layers of a batched compacted cache of P*k sequences (rule 3 above), one launch per 32
 * layers, the per-layer tables as kernel parameters; n = *step + step_offset generated rows. Layer l: planes[4l .. 4l+3]
 * = K, V rows [P*k, num_heads, capacity[l], row_bytes] and, for E4M3 rows, their fp32 scales [P*k, num_heads,
 * capacity[l]] (NULL for 16-bit rows); base[l] (DEVICE int32 [P*k*num_heads]): the row of generated slot 0 of each
 * (sequence, head). Without a window generated row j is slot j. With window R > 0 slot j mod R holds the latest position j,
 * and slot a copies the slots of positions [max(diverge, n - R), n); with heavy != 0 the slots are not position-indexed:
 * a beam whose parent changed copies every slot [0, min(n, R)) and heavy_scores[l] / heavy_gen[l] ([P*k*num_heads, R])
 * and victim[l] ([P*k*num_heads]). Prompt rows are never read or written. PKV_ERR_INVALID_ARG: num_beams outside [2,
 * 16], row_bytes not a positive multiple of 16 up to 256, null or misaligned pointers. */
int pkv_cache_reorder(int32_t num_prompts, int32_t num_beams, int32_t num_heads, int32_t row_bytes, int32_t device,
                      int32_t num_layers, int32_t window, int32_t heavy, void* const* planes, const int64_t* capacity,
                      const int32_t* const* base, float* const* heavy_scores, int32_t* const* heavy_gen,
                      int32_t* const* victim, const int32_t* parent, const int32_t* diverge, const int32_t* step,
                      int32_t step_offset, void* stream);

/* ---- prompt-lookup speculative decoding, greedy (DESIGN.md §4.13; the rules restated in oracle/spec.py) ----
 * HF's generate(prompt_lookup_num_tokens=K, max_matching_ngram_size=N) without logits processors, for num_seqs sequences
 * at once, K in [1, 15], N in [1, 8], Q = K + 1. Per sequence, with history h = prompt + tokens emitted so far (length L)
 * and remaining budget m (tokens it may still emit):
 *  1. Draft (PromptLookupCandidateGenerator.get_candidates): for n = min(N, L - 1) down to 1, the lowest start i with
 *     h[i, i + n) == h[L - n, L) and i + n < L; the draft is h[i + n, min(i + n + K, L)), cut before its first EOS id. No
 *     n matches: no draft. No draft when m <= 1 or the sequence is done. Draft length d <= K.
 *  2. Verify: one forward over the Q tokens [last emitted, draft.., padding] at positions L - 1 .. L - 1 + K gives the
 *     argmaxes t_0 .. t_K (torch.argmax: the first index among ties).
 *  3. Accept (_assisted_decoding, greedy): a = the number of leading j < d with draft[j] == t_j, then a = min(a, m - 1);
 *     the sequence emits t_0 .. t_a, stopping after the first EOS id among them. It is done after an EOS or when m reaches
 *     0; a done sequence emits nothing (pad_token_id) and advances nothing.
 *  4. Cache: the verify step writes the Q new rows of every layer and cache head at n0 .. n0 + K (n0: the rows held);
 *     acceptance advances that row count by the tokens emitted. Rejected rows stay in the buffers uncounted and are
 *     overwritten by the next step. A cache reserves its rows + max_new_tokens + K: a sequence whose budget ran out
 *     still takes part in the verify steps of the others, writing (uncounted) Q rows behind its last. */
#define PKV_MAX_SPEC_QUERIES 16
#define PKV_MAX_NGRAM 8
/* The verify attention: the batched decode of pkv_decode_attn_batch with Q = num_queries new rows per sequence. `d` gives
 * dtype, head counts, head_dim, device, length, the caches (cache_stride_h), q, k_new, v_new, out, the workspace and the
 * softmax scale. Sequence s, token j, query head h reads q at q + (s*Q + j)*q_stride_t + h*q_stride_h (so HF's [b, q, H, D]
 * projections are read in place), kv head g's new rows at k_new / v_new + (s*Q + j)*kv_stride_t + g*kv_stride_h, and
 * writes out + (s*Q + j)*out_stride_t + h*out_stride_h. Per (sequence s, cache head c), n0 = d->length (+ *step_dev)
 * (+ rows[s*H + c]) rows are held (H = num_q_heads, or num_kv_heads when gqa_shared): the launch stores the Q new rows at
 * n0 .. n0 + Q - 1 (16-bit rows: byte copies; E4M3 rows: the quantisation rule of pkv_decode_attn_batch_fp8, scale
 * included) and query j of every head of the cache attends rows [0, n0 + j + 1) in fp32 (online softmax; E4M3: the row's
 * K scale multiplies the fp32 dot, its V scale the softmax weight), the new rows as stored. One CTA per (split, cache head,
 * sequence) reads each cached row once for all its GH*Q query rows; the split count is pkv_decode_attn_batch's for the
 * largest attended count n0 + Q. n0 < 0 or n0 + Q > max_length: nothing is read or written, the outputs are NaN. Graph-
 * replayable: every count is read on the device. Workspace: pkv_decode_workspace_bytes with num_q_heads =
 * num_seqs*num_q_heads*num_queries. PKV_ERR_INVALID_ARG: m NULL or its struct_bytes wrong, num_queries outside [1, 16],
 * num_seqs outside [1, 65535], d->length < 0, max_length above the capacity, strides that misalign rows, null or
 * misaligned pointers; gqa_shared with a group outside {2, 4, 8} is PKV_ERR_UNSUPPORTED. */
typedef struct pkv_decode_multi {
    uint32_t struct_bytes;
    int32_t num_seqs;
    int32_t num_queries;        /* Q in [1, 16] */
    int32_t gqa_shared;         /* 0: a cache per query head; 1: one per KV head */
    int64_t cache_stride_b;     /* elements (E4M3: bytes) between the caches of consecutive sequences */
    const int32_t* rows;        /* optional DEVICE int32 [num_seqs*H]: rows held */
    const int32_t* step_dev;    /* optional DEVICE int32 added to every count */
    int64_t max_length;         /* rows the launch is sized for: cache_stride_h >= max_length*head_dim */
    float* k_scale;             /* E4M3 rows: fp32 row scales [num_seqs, H, capacity]; NULL for 16-bit rows */
    float* v_scale;
    int64_t scale_stride_h, scale_stride_b;
    int64_t q_stride_t, q_stride_h;      /* elements; multiples of 8 */
    int64_t kv_stride_t, kv_stride_h;    /* k_new and v_new alike */
    int64_t out_stride_t, out_stride_h;
} pkv_decode_multi;
int pkv_decode_attn_multi(const pkv_decode_desc* d, const pkv_decode_multi* m, void* stream);
/* The device state of rules 1 and 3, all DEVICE memory, contiguous: hist int64 [num_seqs, hist_cap] (the history; its
 * length hist_len int32 [num_seqs]), budget int32 [num_seqs] (m), done uint8 [num_seqs], out int64 [num_seqs, out_cap]
 * (the tokens emitted by the steps; out_len int32 [num_seqs] each sequence's cursor), ids and pos int64 [num_seqs, Q] (the
 * next verify step's input ids and positions), draft_len int32 [num_seqs], emitted int32 [num_seqs] (the tokens the last
 * step emitted), tokens int64 [num_seqs, Q] (the verify argmaxes t), eos int64 [n_eos] (n_eos in [0, 4]). rows: a HOST
 * table of num_layers DEVICE int32 [num_seqs*num_heads] row counts (pkv_spec_step only; may be NULL with num_layers 0). */
typedef struct pkv_spec_desc {
    uint32_t struct_bytes;
    int32_t device;
    int32_t num_seqs;
    int32_t num_queries;        /* Q = K + 1 in [2, 16] */
    int32_t max_ngram;          /* N in [1, 8] */
    int32_t n_eos;
    int64_t pad_token_id;       /* the padding of ids past the draft */
    int64_t hist_cap, out_cap;
    int64_t* hist; int32_t* hist_len; int32_t* budget; uint8_t* done;
    int64_t* out; int32_t* out_len;
    int64_t* ids; int64_t* pos; int32_t* draft_len; int32_t* emitted;
    const int64_t* tokens; const int64_t* eos;
    int32_t num_layers, num_heads;
    int32_t* const* rows;
} pkv_spec_desc;
/* Rule 1 for every sequence (one CTA each, a single pass over its history): ids = [h[L - 1], draft.., pad_token_id..],
 * pos[j] = L - 1 + j, draft_len = d. Runs once before the first verify step. */
int pkv_prompt_lookup(const pkv_spec_desc* d, void* stream);
/* Rule 3 for every sequence from `tokens` and the current ids / draft_len: appends the emitted tokens to hist and out at
 * the sequence's cursors, advances hist_len, out_len, budget, done and every layer's row counts (by emitted), then rule 1
 * for the next ids / pos / draft_len. One launch per 32 layers; integer logic, no host reads: graph-replayable.
 * PKV_ERR_INVALID_ARG (both): a wrong struct_bytes, num_seqs outside [1, 65535], Q outside [2, 16], N outside [1, 8],
 * n_eos outside [0, 4], caps below 1, null or misaligned pointers. */
int pkv_spec_step(const pkv_spec_desc* d, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* PKV_H_ */
