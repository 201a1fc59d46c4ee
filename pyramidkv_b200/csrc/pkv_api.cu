// pkv_api.cu — the extern "C" boundary declared in include/pkv.h: validation, workspace layout, dispatch.
#include <algorithm>
#include <atomic>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "pkv_common.cuh"
#include "pkv_internal.h"

namespace pkv {

static thread_local char g_err[512] = "";
static std::atomic<uint64_t> g_launches{0};

unsigned long long* debug_stamps() {
    static unsigned long long* buf = [] {
        const char* e = getenv("PKV_STAMPS");
        void* p = nullptr;
        if (e && atoi(e) && cudaMalloc(&p, 128 * sizeof(unsigned long long)) == cudaSuccess) cudaMemset(p, 0, 128 * sizeof(unsigned long long));
        return static_cast<unsigned long long*>(p);
    }();
    return buf;
}
void count_launch(int n) { g_launches.fetch_add(uint64_t(n), std::memory_order_relaxed); }

static int fail(int code, const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
    return code;
}
static int fail_cuda(cudaError_t e, const char* what) {
    return fail(PKV_ERR_CUDA, "%s: %s", what, cudaGetErrorString(e));
}

// Per-device facts, queried once. sm_90a cubins only load on compute capability 9.0.
struct DevInfo { int ok = -1; int sms = 0; int major = 0, minor = 0; };
static DevInfo g_dev[64];

static int device_info(int dev, const DevInfo** out) {
    if (dev < 0 || dev >= 64) return fail(PKV_ERR_INVALID_ARG, "device ordinal %d out of range", dev);
    DevInfo& d = g_dev[dev];
    if (d.ok < 0) {
        cudaError_t e = cudaDeviceGetAttribute(&d.major, cudaDevAttrComputeCapabilityMajor, dev);
        if (e == cudaSuccess) e = cudaDeviceGetAttribute(&d.minor, cudaDevAttrComputeCapabilityMinor, dev);
        if (e == cudaSuccess) e = cudaDeviceGetAttribute(&d.sms, cudaDevAttrMultiProcessorCount, dev);
        if (e != cudaSuccess) return fail_cuda(e, "cudaDeviceGetAttribute (is a CUDA device present?)");
        d.ok = (d.major == 9 && d.minor == 0) ? 1 : 0;
    }
    if (!d.ok) return fail(PKV_ERR_UNSUPPORTED_ARCH, "device %d is sm_%d%d; libpkv is built for sm_90a only (no fallback)", dev, d.major, d.minor);
    *out = &d;
    return PKV_OK;
}

struct DeviceGuard {
    int prev = -1;
    bool switched = false;
    explicit DeviceGuard(int dev) {
        if (cudaGetDevice(&prev) == cudaSuccess && prev != dev) switched = (cudaSetDevice(dev) == cudaSuccess);
    }
    ~DeviceGuard() { if (switched) cudaSetDevice(prev); }
};

static inline uint64_t align_up(uint64_t v, uint64_t a) { return (v + a - 1) / a * a; }
static inline bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }

static bool is_window_method(int m) { return m == PKV_PYRAMIDKV || m == PKV_SNAPKV; }

// PKV_FLAG_GQA_SHARED: the selection stages seen as Hkv "heads" with G = 1 — top-k over the group-reduced scores, the gather
// writing KV head j's cache from K[j] / V[j]. (The caller's cache is [Hkv, capacity, D].)
static EvictArgs kv_view(const EvictArgs& a) {
    EvictArgs b = a;
    b.Hq = a.Hkv;
    b.G = 1;
    b.ws.nw = a.W;
    b.ws.pooled_off = a.pooled_kv_off;
    b.gqa_shared = false;
    return b;
}

// Shape-only validation + layout (no device access): shared by the workspace queries and the launches. *pooled_kv_off: the
// PKV_FLAG_GQA_SHARED segment (0 without the flag or for StreamingLLM).
static int compute_layout(const pkv_evict_desc* d, pkv_ws_layout* L, uint64_t* pooled_kv_off = nullptr) {
    if (!d) return fail(PKV_ERR_INVALID_ARG, "null descriptor");
    if (d->struct_bytes != sizeof(pkv_evict_desc))
        return fail(PKV_ERR_INVALID_ARG, "pkv_evict_desc.struct_bytes=%u, library expects %zu (ABI mismatch)", d->struct_bytes, sizeof(pkv_evict_desc));
    if (d->dtype != PKV_BF16 && d->dtype != PKV_FP16) return fail(PKV_ERR_UNSUPPORTED_DTYPE, "dtype %d: only bf16 (0) and fp16 (1) are supported", d->dtype);
    if (d->method < PKV_PYRAMIDKV || d->method > PKV_L2NORM) return fail(PKV_ERR_INVALID_ARG, "unknown method %d", d->method);
    if (d->flags & ~PKV_EVICT_KNOWN_FLAGS) return fail(PKV_ERR_INVALID_ARG, "unknown pkv_evict_desc.flags bits 0x%x", d->flags & ~PKV_EVICT_KNOWN_FLAGS);
    if ((d->flags & PKV_FLAG_GQA_SHARED) && (d->flags & (PKV_FLAG_FUSED | PKV_FLAG_SINGLE_LAUNCH)))
        return fail(PKV_ERR_UNSUPPORTED, "PKV_FLAG_GQA_SHARED runs the staged kernels: PKV_FLAG_FUSED / PKV_FLAG_SINGLE_LAUNCH are not built with it");
    if (d->num_q_heads <= 0 || d->num_kv_heads <= 0 || d->num_q_heads % d->num_kv_heads)
        return fail(PKV_ERR_INVALID_ARG, "num_q_heads=%d must be a positive multiple of num_kv_heads=%d", d->num_q_heads, d->num_kv_heads);
    if (d->head_dim != 64 && d->head_dim != 128) return fail(PKV_ERR_UNSUPPORTED, "head_dim=%d: only 64 and 128 are built", d->head_dim);
    if (d->method == PKV_L2NORM) {
        if (d->window != 0 || d->seq_len < 1) return fail(PKV_ERR_INVALID_ARG, "l2norm keeps no window: window must be 0 (got %d) and seq_len >= 1", d->window);
    } else if (d->seq_len < 1 || d->window < 1 || d->window > d->seq_len)
        return fail(PKV_ERR_INVALID_ARG, "need 1 <= window (%d) <= seq_len (%lld)", d->window, (long long)d->seq_len);
    if (d->top_k < 0 || d->top_k > d->seq_len - d->window)
        return fail(PKV_ERR_INVALID_ARG, "top_k=%lld out of range [0, seq_len-window=%lld] (selected index k out of range)", (long long)d->top_k, (long long)(d->seq_len - d->window));
    const int G = d->num_q_heads / d->num_kv_heads;
    if (is_window_method(d->method)) {
        if (d->pooling != PKV_AVGPOOL && d->pooling != PKV_MAXPOOL) return fail(PKV_ERR_POOLING, "Pooling method not supported");
        if (d->kernel_size < 1 || (d->kernel_size & 1) == 0 || d->kernel_size > 65)
            return fail(PKV_ERR_UNSUPPORTED, "kernel_size=%d: odd sizes 1..65 are supported", d->kernel_size);
        if (d->window % 8 != 0 || d->window > 64) return fail(PKV_ERR_UNSUPPORTED, "window_size=%d: multiples of 8 up to 64 are supported by the scoring kernels", d->window);
    }
    memset(L, 0, sizeof(*L));
    L->s_pad = int64_t(align_up(uint64_t(d->seq_len), kTileTokens));
    L->n_slots = L->s_pad / kTileTokens;
    L->nw = int64_t(G) * d->window;
    const int64_t n = d->seq_len - d->window;
    L->pooled_pitch = int64_t(align_up(uint64_t(n > 0 ? n : 1), 8));
    uint64_t off = 0;
    auto seg = [&](uint64_t bytes) { const uint64_t o = off; off = align_up(off + bytes, 256); return o; };
    if (is_window_method(d->method)) {
        L->logits_off = seg(uint64_t(d->num_kv_heads) * uint64_t(L->s_pad) * uint64_t(L->nw) * 2);
        L->partial_off = seg(uint64_t(d->num_kv_heads) * uint64_t(L->n_slots) * uint64_t(L->nw) * sizeof(float2));
    }
    if (d->method != PKV_STREAMINGLLM) {
        L->pooled_off = seg(uint64_t(d->num_q_heads) * uint64_t(L->pooled_pitch) * 2);
        L->idx32_off = seg(uint64_t(d->num_q_heads) * uint64_t(d->top_k > 0 ? d->top_k : 1) * 4);
    }
    if (is_window_method(d->method)) L->fused_off = seg(fused_ws_layout(d->num_q_heads, G, d->top_k).total);
    if (d->method == PKV_H2O) {
        L->h2o_stats_off = seg(uint64_t(d->num_q_heads) * uint64_t(L->s_pad) * sizeof(float2));
        L->h2o_acc_off = L->h2o_stats_off;  // column sums are accumulated in registers; no extra segment
        seg(uint64_t(d->num_q_heads) * uint64_t(L->s_pad) * sizeof(float4));   // stats4 of the wgmma kernels: h2o_stats4_offset()
    }
    uint64_t kv_off = 0;
    if ((d->flags & PKV_FLAG_GQA_SHARED) && d->method != PKV_STREAMINGLLM)
        kv_off = (G > 1 && d->method != PKV_L2NORM) ? seg(uint64_t(d->num_kv_heads) * uint64_t(L->pooled_pitch) * 2) : L->pooled_off;
    if (pooled_kv_off) *pooled_kv_off = kv_off;
    L->total_bytes = off > 0 ? off : 256;
    return PKV_OK;
}

static int resolve(const pkv_evict_desc* d, EvictArgs* a) {
    pkv_ws_layout L;
    uint64_t kv_off = 0;
    int rc = compute_layout(d, &L, &kv_off);
    if (rc) return rc;
    const DevInfo* di = nullptr;
    rc = device_info(d->device, &di);
    if (rc) return rc;
    if ((!d->q && d->method != PKV_L2NORM) || !d->k || !d->v || !d->k_cache || !d->v_cache) return fail(PKV_ERR_INVALID_ARG, "null tensor pointer");
    if (!aligned16(d->q) || !aligned16(d->k) || !aligned16(d->v) || !aligned16(d->k_cache) || !aligned16(d->v_cache))
        return fail(PKV_ERR_INVALID_ARG, "tensor base pointers must be 16-byte aligned");
    const int64_t st[] = {d->q_stride_h, d->q_stride_s, d->k_stride_h, d->k_stride_s, d->v_stride_h, d->v_stride_s, d->cache_stride_h};
    for (int64_t s : st)
        if (s % 8 != 0 || s < 0) return fail(PKV_ERR_INVALID_ARG, "strides must be non-negative multiples of 8 elements (16 bytes), got %lld", (long long)s);
    if (d->q_stride_s < d->head_dim || d->k_stride_s < d->head_dim || d->v_stride_s < d->head_dim)
        return fail(PKV_ERR_INVALID_ARG, "token strides must be >= head_dim (last dim contiguous)");
    if (d->cache_stride_h < (d->top_k + d->window) * int64_t(d->head_dim))
        return fail(PKV_ERR_INVALID_ARG, "cache_stride_h=%lld holds fewer than top_k+window=%lld rows", (long long)d->cache_stride_h, (long long)(d->top_k + d->window));
    if (!d->workspace || d->workspace_bytes < L.total_bytes)
        return fail(PKV_ERR_WORKSPACE, "workspace of %llu bytes required, got %llu", (unsigned long long)L.total_bytes, (unsigned long long)(d->workspace ? d->workspace_bytes : 0));
    if ((reinterpret_cast<uintptr_t>(d->workspace) & 255u) != 0) return fail(PKV_ERR_WORKSPACE, "workspace must be 256-byte aligned");
    a->method = d->method; a->dtype = d->dtype; a->pooling = d->pooling; a->kernel_size = d->kernel_size;
    a->Hq = d->num_q_heads; a->Hkv = d->num_kv_heads; a->G = a->Hq / a->Hkv; a->D = d->head_dim; a->W = d->window;
    a->S = d->seq_len; a->n = d->seq_len - d->window; a->k = d->top_k;
    a->q = static_cast<const uint16_t*>(d->q); a->kk = static_cast<const uint16_t*>(d->k); a->vv = static_cast<const uint16_t*>(d->v);
    a->q_sh = d->q_stride_h; a->q_ss = d->q_stride_s; a->k_sh = d->k_stride_h; a->k_ss = d->k_stride_s; a->v_sh = d->v_stride_h; a->v_ss = d->v_stride_s;
    a->k_cache = static_cast<uint16_t*>(d->k_cache); a->v_cache = static_cast<uint16_t*>(d->v_cache);
    a->cache_sh = d->cache_stride_h;
    a->idx_out = d->idx_out;
    a->ws = L; a->ws_base = static_cast<uint8_t*>(d->workspace);
    a->flags = d->flags; a->device = d->device; a->num_sms = di->sms;
    a->window_mean = (d->flags & PKV_FLAG_WINDOW_MEAN) != 0;
    a->gqa_shared = (d->flags & PKV_FLAG_GQA_SHARED) != 0 && a->G > 1;
    a->pooled_kv_off = kv_off;
    if (a->window_mean && (!is_window_method(a->method) || (a->W & (a->W - 1)) != 0))
        return fail(PKV_ERR_UNSUPPORTED, "PKV_FLAG_WINDOW_MEAN needs a window method and a power-of-two window_size (got %d)", a->W);
    // which stage-1 kernel runs is a pure function of the descriptor (stage 2 must read the partials it wrote)
    a->score_impl = 0; a->score_grid = 0;
    if (is_window_method(a->method)) {
        const uint32_t sel = a->flags & 3u;
        const bool tc5_ok = score_tc5_supported(*a);
        if (sel == PKV_SCORE_TCGEN05 && !tc5_ok) return fail(PKV_ERR_UNSUPPORTED, "wgmma score kernel does not support this shape (needs group*window in {32, 64})");
        if ((sel == PKV_SCORE_AUTO && tc5_ok) || sel == PKV_SCORE_TCGEN05) { a->score_impl = 1; a->score_grid = tc5_grid(*a); }
    }
    if (a->method != PKV_STREAMINGLLM) {
        const char* why = nullptr;
        if (!topk_supported(a->gqa_shared ? kv_view(*a) : *a, &why)) return fail(PKV_ERR_UNSUPPORTED, "%s", why);
    }
    return PKV_OK;
}

// H2O scoring runs on the TMA + wgmma kernels (pkv_h2o_tc5.cu; the mma.sync kernels of pkv_h2o.cu remain for shapes the
// tensor maps or the ring cannot take; PKV_H2O=mma forces them for A/B runs).
// Both passes follow the same choice (pass 1 reads what pass 0 wrote).
static bool h2o_use_tc5() {
    static const bool v = []() { const char* e = getenv("PKV_H2O"); return !(e && e[0] == 'm'); }();
    return v;
}

static int run_scores(const EvictArgs& a, cudaStream_t st) {
    if (a.gqa_shared && a.method == PKV_L2NORM) return run_scores(kv_view(a), st);   // the key norms of each KV head, once
    cudaError_t e = cudaSuccess;
    if (a.method == PKV_H2O) e = (h2o_use_tc5() && h2o_tc5_supported(a)) ? launch_h2o_tc5_rowstats(a, st) : launch_h2o_rowstats(a, st);
    else if (a.method == PKV_L2NORM) e = launch_l2norm_scores(a, st);
    else if (is_window_method(a.method)) e = a.score_impl == 1 ? launch_score_tc5(a, st) : launch_score_mma(a, st);
    return e == cudaSuccess ? PKV_OK : fail_cuda(e, "score launch");
}
static int run_pool(const EvictArgs& a, cudaStream_t st) {
    cudaError_t e = cudaSuccess;
    if (a.method == PKV_H2O) e = (h2o_use_tc5() && h2o_tc5_supported(a)) ? launch_h2o_tc5_colsum(a, st) : launch_h2o_colsum(a, st);
    else if (is_window_method(a.method)) e = launch_softmax_pool(a, st);
    if (e == cudaSuccess && a.gqa_shared && (a.method == PKV_H2O || is_window_method(a.method))) e = launch_group_reduce(a, st);
    return e == cudaSuccess ? PKV_OK : fail_cuda(e, "pool launch");
}
static int run_topk(const EvictArgs& a, cudaStream_t st) {
    if (a.method == PKV_STREAMINGLLM) return PKV_OK;
    const cudaError_t e = launch_topk(a.gqa_shared ? kv_view(a) : a, st);
    return e == cudaSuccess ? PKV_OK : fail_cuda(e, "topk launch");
}
static int run_gather(const EvictArgs& a, cudaStream_t st) {
    const cudaError_t e = launch_gather(a.gqa_shared ? kv_view(a) : a, st);
    return e == cudaSuccess ? PKV_OK : fail_cuda(e, "gather launch");
}

}  // namespace pkv

using namespace pkv;

extern "C" {

int pkv_version(void) { return PKV_ABI_VERSION; }
const char* pkv_last_error(void) { return g_err; }
uint64_t pkv_launch_count(void) { return g_launches.load(std::memory_order_relaxed); }
int pkv_host_pick_rows(const void* src, int64_t src_stride_h_bytes, int64_t src_stride_s_bytes, int64_t seq_len,
                       int32_t num_kv_heads, int32_t num_q_heads, int64_t row_bytes, const int64_t* rows, int64_t n_rows,
                       void* dst) {
    if (!src || !rows || !dst || num_kv_heads <= 0 || num_q_heads <= 0 || num_q_heads % num_kv_heads || row_bytes <= 0 || n_rows < 0)
        return fail(PKV_ERR_INVALID_ARG, "pkv_host_pick_rows: bad argument");
    const int g = num_q_heads / num_kv_heads;
    const char* s = static_cast<const char*>(src);
    char* d = static_cast<char*>(dst);
    for (int h = 0; h < num_q_heads; ++h) {
        const char* sh = s + int64_t(h / g) * src_stride_h_bytes;
        for (int64_t r = 0; r < n_rows; ++r) {
            const int64_t tok = rows[int64_t(h) * n_rows + r];
            if (tok < 0 || tok >= seq_len) return fail(PKV_ERR_INVALID_ARG, "pkv_host_pick_rows: row index %lld outside [0, %lld)", (long long)tok, (long long)seq_len);
            memcpy(d + (int64_t(h) * n_rows + r) * row_bytes, sh + tok * src_stride_s_bytes, size_t(row_bytes));
        }
    }
    return PKV_OK;
}
int pkv_debug_read_stamps(uint64_t* out, int count) {
    unsigned long long* b = pkv::debug_stamps();
    if (!b || !out) return 0;
    if (count > 128) count = 128;
    if (cudaMemcpy(out, b, size_t(count) * sizeof(uint64_t), cudaMemcpyDeviceToHost) != cudaSuccess) return 0;
    return count;
}

int pkv_layer_budget(int method, int64_t max_capacity_prompt, int64_t window, int num_layers, int layer_idx,
                     int64_t q_len, int beta, int64_t* top_k_out, int* mode_out) {
    if (!top_k_out || !mode_out) return fail(PKV_ERR_INVALID_ARG, "null output pointer");
    const int64_t B = max_capacity_prompt, W = window, S = q_len;
    if (B - W <= 0) return fail(PKV_ERR_INVALID_ARG, "assert max_capacity_prompt - window_size > 0 failed (%lld - %lld)", (long long)B, (long long)W);
    if (method < PKV_PYRAMIDKV || method > PKV_L2NORM) return fail(PKV_ERR_INVALID_ARG, "unknown method %d", method);
    if (method == PKV_L2NORM && W != 0) return fail(PKV_ERR_INVALID_ARG, "l2norm keeps no window: window must be 0");
    if (S < B) { *mode_out = 0; *top_k_out = S; return PKV_OK; }   // q_len < max_capacity_prompt: keep everything
    *mode_out = 1;
    if (method != PKV_PYRAMIDKV) { *top_k_out = B - W; return PKV_OK; }
    if (num_layers < 2 || beta <= 0 || layer_idx < 0 || layer_idx >= num_layers)
        return fail(PKV_ERR_INVALID_ARG, "pyramidkv needs num_layers >= 2, beta > 0, 0 <= layer_idx < num_layers");
    int64_t min_num = (B - W) / beta;                 // non-negative operands: C division == Python //
    int64_t max_num = (B - W) * 2 - min_num;
    if (max_num >= S - W) { max_num = S - W; min_num = (B - W) * 2 - max_num; }
    const int64_t num = max_num - min_num, den = num_layers - 1;
    int64_t steps = num / den;
    if (num % den != 0 && num < 0) --steps;           // floor like Python
    *top_k_out = (S < (B - W) * 2) ? (B - W) : (max_num - int64_t(layer_idx) * steps);
    return PKV_OK;
}

int pkv_evict_workspace_layout(const pkv_evict_desc* d, pkv_ws_layout* out) {
    if (!out) return fail(PKV_ERR_INVALID_ARG, "null output pointer");
    return compute_layout(d, out);
}

uint64_t pkv_evict_workspace_bytes(const pkv_evict_desc* d) {
    pkv_ws_layout L;
    return compute_layout(d, &L) == PKV_OK ? L.total_bytes : 0;
}

int pkv_evict_pooled_kv_offset(const pkv_evict_desc* d, uint64_t* off_out) {
    if (!off_out) return fail(PKV_ERR_INVALID_ARG, "null output pointer");
    pkv_ws_layout L;
    uint64_t off = 0;
    const int rc = compute_layout(d, &L, &off);
    if (rc) return rc;
    if (!(d->flags & PKV_FLAG_GQA_SHARED) || d->method == PKV_STREAMINGLLM)
        return fail(PKV_ERR_INVALID_ARG, "pkv_evict_pooled_kv_offset: per-KV-head scores exist only with PKV_FLAG_GQA_SHARED and a scoring method");
    *off_out = off;
    return PKV_OK;
}

#define PKV_STAGE_PROLOGUE()                      \
    EvictArgs a;                                  \
    int rc = resolve(d, &a);                      \
    if (rc) return rc;                            \
    DeviceGuard guard(a.device);                  \
    cudaStream_t st = static_cast<cudaStream_t>(stream)

// 0 staged launches, 1 fused stages 1-2 + select kernel, 2 everything in one launch.
// Default: STAGED. The fused forms rely on every CTA being resident for their cross-CTA flag waits, which only the
// cooperative launch guarantees; they stay available (PKV_FLAG_FUSED / PKV_FLAG_SINGLE_LAUNCH, or PKV_ONEPASS=1 / 2 for A/B runs).
static int fused_mode(const EvictArgs& a) {
    static const int env = []() { const char* e = getenv("PKV_ONEPASS"); return e ? atoi(e) : 0; }();
    if ((a.flags & PKV_FLAG_STAGED) || a.gqa_shared || a.score_impl != 1 || !evict_fused_supported(a)) return 0;
    if (a.flags & PKV_FLAG_SINGLE_LAUNCH) return 2;
    if (a.flags & PKV_FLAG_FUSED) return 1;
    return env < 0 ? 0 : env > 2 ? 2 : env;
}

int pkv_evict_single_launch(const pkv_evict_desc* d) {
    EvictArgs a;
    if (resolve(d, &a)) return 0;
    return fused_mode(a);
}

int pkv_stage_scan_pool(const pkv_evict_desc* d, void* stream) {
    PKV_STAGE_PROLOGUE();
    if ((a.flags & PKV_FLAG_STAGED) || a.gqa_shared || a.score_impl != 1 || !evict_fused_supported(a))
        return fail(PKV_ERR_UNSUPPORTED, "pkv_stage_scan_pool: this shape runs as staged launches (pkv_stage_scores + pkv_stage_pool)");
    const cudaError_t e = launch_evict_fused(a, true, st);
    return e == cudaSuccess ? PKV_OK : fail_cuda(e, "fused scan+pool launch");
}

int pkv_stage_scores(const pkv_evict_desc* d, void* stream) { PKV_STAGE_PROLOGUE(); return run_scores(a, st); }
int pkv_stage_pool(const pkv_evict_desc* d, void* stream) { PKV_STAGE_PROLOGUE(); return run_pool(a, st); }
int pkv_stage_topk(const pkv_evict_desc* d, void* stream) { PKV_STAGE_PROLOGUE(); return run_topk(a, st); }
int pkv_stage_gather(const pkv_evict_desc* d, void* stream) { PKV_STAGE_PROLOGUE(); return run_gather(a, st); }

int pkv_evict_prefill(const pkv_evict_desc* d, void* stream) {
    PKV_STAGE_PROLOGUE();
    // PKV_FUSED: 0 = four launches per layer; 1 = stage 2, then stages 3+4 on one cluster launch;
    // 2 = stages 2+3+4 on one cluster launch (slower at 32K: 16 warps/SM starve the exp/div-heavy pool phase; faster <= 8K)
    // unset = 1, with 2 chosen by prompt length below
    static const int fused_env = []() { const char* e = getenv("PKV_FUSED"); return e ? atoi(e) : -1; }();
    static const int fused = fused_env < 0 ? 1 : fused_env;
    constexpr int64_t kPoolInSelectMaxS = 12288;
    // window methods whose logits fit on chip: stages 1-2 in one persistent launch, then the select kernel (or all in one)
    if (const int fm = fused_mode(a)) {
        cudaError_t e = launch_evict_fused(a, fm == 1, st);
        if (e != cudaSuccess) return fail_cuda(e, "fused eviction launch");
        if (fm == 2) return PKV_OK;
        if (select_fused_supported(a, false)) {
            e = launch_select_fused(a, false, st);
            return e == cudaSuccess ? PKV_OK : fail_cuda(e, "select launch");
        }
        if ((rc = run_topk(a, st))) return rc;
        return run_gather(a, st);
    }
    if ((rc = run_scores(a, st))) return rc;
    if (a.gqa_shared) {
        // scores and pool per query head, the group reduction, then select + gather per KV head (never pooling inside the select
        // cluster: the reduction sits between the pool and the select)
        if ((rc = run_pool(a, st))) return rc;
        const EvictArgs b = kv_view(a);
        if (a.method != PKV_STREAMINGLLM && fused > 0 && select_fused_supported(b, false)) {
            const cudaError_t e = launch_select_fused(b, false, st);
            return e == cudaSuccess ? PKV_OK : fail_cuda(e, "select launch");
        }
        if ((rc = run_topk(a, st))) return rc;
        return run_gather(a, st);
    }
    if (a.method != PKV_STREAMINGLLM && fused > 0) {
        // Pooling inside the select cluster saves one launch; it wins while the three kernels are launch-bound (short prompts)
        // and loses once the exp-heavy pool phase is big enough to want the whole-chip pool grid. PKV_FUSED=1 / 2 pin either form.
        bool pool = (fused >= 2 || (fused_env < 0 && a.ws.s_pad <= kPoolInSelectMaxS)) && is_window_method(a.method) && !a.window_mean;
        if (pool && !select_fused_supported(a, true)) pool = false;
        if (select_fused_supported(a, pool)) {
            if (!pool && (rc = run_pool(a, st))) return rc;
            const cudaError_t e = launch_select_fused(a, pool, st);
            return e == cudaSuccess ? PKV_OK : fail_cuda(e, "select launch");
        }
    }
    if ((rc = run_pool(a, st))) return rc;
    if ((rc = run_topk(a, st))) return rc;
    return run_gather(a, st);
}

// ---- layer batch: the eviction of all layers of one prompt in one pass (three launches per <= 32 layers) ----
// Why layers cannot differ: the persistent score grid walks ONE (layer, kv head, tile) list and the pool / select grids
// index the layer with blockIdx.z, so geometry, dtype and pooling knobs are shared; budgets (top_k), tensors, caches and
// workspaces are per layer.
static const char* batch_mismatch(const EvictArgs& a, const EvictArgs& b) {
    if (a.method != b.method || a.dtype != b.dtype || a.pooling != b.pooling || a.kernel_size != b.kernel_size) return "method / dtype / pooling knobs differ";
    if (a.Hq != b.Hq || a.Hkv != b.Hkv || a.D != b.D || a.W != b.W || a.S != b.S) return "head counts, head_dim, window or seq_len differ";
    if (a.device != b.device || a.flags != b.flags || a.score_impl != b.score_impl) return "device, flags or score kernel differ";
    if (a.ws.s_pad != b.ws.s_pad || a.ws.nw != b.ws.nw || a.ws.n_slots != b.ws.n_slots || a.ws.pooled_pitch != b.ws.pooled_pitch) return "workspace layouts differ";
    return nullptr;
}
static int resolve_batch(const pkv_evict_desc* descs, int n, std::vector<EvictArgs>* out) {
    if (!descs || n < 1) return fail(PKV_ERR_INVALID_ARG, "pkv_evict_prefill_batch: need >= 1 descriptor");
    out->resize(size_t(n));
    for (int l = 0; l < n; ++l) {
        if (descs[l].struct_bytes != sizeof(pkv_evict_desc)) return fail(PKV_ERR_INVALID_ARG, "descriptor %d: struct_bytes mismatch", l);
        const int rc = resolve(&descs[l], &(*out)[size_t(l)]);
        if (rc) return rc;
    }
    const EvictArgs& a = (*out)[0];
    if (a.flags & PKV_FLAG_GQA_SHARED) return fail(PKV_ERR_UNSUPPORTED, "layer batch: not built for PKV_FLAG_GQA_SHARED (evict layer by layer)");
    if (!is_window_method(a.method) || a.window_mean || a.score_impl != 1)
        return fail(PKV_ERR_UNSUPPORTED, "layer batch: window methods (pyramidkv / snapkv) on the wgmma score kernel only");
    if (a.ws.s_pad / kTileTokens < 8) return fail(PKV_ERR_UNSUPPORTED, "layer batch: prompts of at least 897 tokens (8 K tiles per kv head)");
    for (int l = 0; l < n; ++l) {
        const EvictArgs& b = (*out)[size_t(l)];
        if (const char* why = batch_mismatch(a, b)) return fail(PKV_ERR_UNSUPPORTED, "layer batch: layer %d: %s", l, why);
        if (!select_batch_supported(b)) return fail(PKV_ERR_UNSUPPORTED, "layer batch: layer %d: top_k=%lld is outside the cluster select kernel", l, (long long)b.k);
    }
    return PKV_OK;
}

extern "C" int pkv_evict_batch_supported(const pkv_evict_desc* descs, int n_layers) {
    std::vector<EvictArgs> as;
    return resolve_batch(descs, n_layers, &as) == PKV_OK ? 1 : 0;
}

// Auxiliary stream of the overlapped layer batch: chunk c's pool + select launches run on it while the caller's stream scans
// chunk c + 1 (the scan is HBM-bound with one 64-register CTA per SM; the pool is issue-bound and the select latency-bound:
// they fit next to it). Forked from and joined to the caller's stream with events (the pattern is stream-capturable); one per
// thread and device, created on first use.
constexpr int kMaxChunks = 64;
struct BatchAux {
    cudaStream_t s = nullptr;
    cudaEvent_t fork = nullptr, join = nullptr, ev[kMaxChunks] = {};
};
static BatchAux* batch_aux(int device) {
    static thread_local BatchAux aux[64];
    if (device < 0 || device >= 64) return nullptr;
    BatchAux& a = aux[device];
    if (!a.s) {
        if (cudaStreamCreateWithFlags(&a.s, cudaStreamNonBlocking) != cudaSuccess) { a.s = nullptr; return nullptr; }
        bool ok = cudaEventCreateWithFlags(&a.fork, cudaEventDisableTiming) == cudaSuccess && cudaEventCreateWithFlags(&a.join, cudaEventDisableTiming) == cudaSuccess;
        for (int i = 0; ok && i < kMaxChunks; ++i) ok = cudaEventCreateWithFlags(&a.ev[i], cudaEventDisableTiming) == cudaSuccess;
        if (!ok) return nullptr;
    }
    return &a;
}

// stage: 0 = all four launches, 1 = window scores, 2 = partial merge + softmax + pool, 3 = select + gather (2 and 3 read what the
// earlier stages of the SAME batch left in the workspaces)
extern "C" int pkv_stage_batch(const pkv_evict_desc* descs, int n_layers, int stage, void* stream) {
    if (stage < 0 || stage > 3) return fail(PKV_ERR_INVALID_ARG, "pkv_stage_batch: stage %d outside [0, 3]", stage);
    std::vector<EvictArgs> as;
    const int rc = resolve_batch(descs, n_layers, &as);
    if (rc) return rc;
    DeviceGuard guard(as[0].device);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    // experiment knob PKV_BATCH_CHUNK = layers per launch (<= 32). Default 32: smaller chunks do not keep the logits in L2 (the K
    // stream evicts them either way) and add launches
    static const int chunk_env = []() { const char* e = getenv("PKV_BATCH_CHUNK"); const int v = e ? atoi(e) : kMaxLayerBatch; return v < 2 ? 2 : v > kMaxLayerBatch ? kMaxLayerBatch : v; }();
    // PKV_BATCH_OVERLAP = c (2..32): chunks of c layers; chunk i's pool + select run on the auxiliary stream under the scan of
    // chunk i + 1 (score kernel limited to 4 ring stages so that their shared memory fits next to it)
    static const int overlap_env = []() { const char* e = getenv("PKV_BATCH_OVERLAP"); const int v = e ? atoi(e) : 0; return v < 0 ? 0 : v > kMaxLayerBatch ? kMaxLayerBatch : v; }();
    if (stage == 0 && overlap_env >= 2 && n_layers > overlap_env && (n_layers + overlap_env - 1) / overlap_env <= kMaxChunks) {
        BatchAux* aux = batch_aux(as[0].device);
        if (!aux) return fail(PKV_ERR_CUDA, "layer batch: could not create the auxiliary stream");
        cudaError_t e = cudaEventRecord(aux->fork, st);
        if (e == cudaSuccess) e = cudaStreamWaitEvent(aux->s, aux->fork, 0);
        if (e != cudaSuccess) return fail_cuda(e, "layer-batch fork");
        int c = 0;
        for (int l0 = 0; l0 < n_layers; l0 += overlap_env, ++c) {
            const int n = n_layers - l0 < overlap_env ? n_layers - l0 : overlap_env;
            const EvictArgs* chunk = as.data() + l0;
            if (n == 1) {   // left-over single layer: per-layer launches on the caller's stream
                const int r1 = pkv_evict_prefill(&descs[l0], stream);
                if (r1) return r1;
                continue;
            }
            const int total_tiles = int(chunk[0].ws.s_pad / kTileTokens) * chunk[0].Hkv * n;
            const int grid = total_tiles < chunk[0].num_sms ? total_tiles : chunk[0].num_sms;
            e = launch_score_tc5_layers(chunk, n, st, 4);
            if (e != cudaSuccess) return fail_cuda(e, "layer-batch score launch");
            e = cudaEventRecord(aux->ev[c], st);
            if (e == cudaSuccess) e = cudaStreamWaitEvent(aux->s, aux->ev[c], 0);
            if (e != cudaSuccess) return fail_cuda(e, "layer-batch chunk event");
            e = launch_softmax_pool_layers(chunk, n, grid, aux->s);
            if (e != cudaSuccess) return fail_cuda(e, "layer-batch pool launch");
            e = launch_select_layers(chunk, n, aux->s);
            if (e != cudaSuccess) return fail_cuda(e, "layer-batch select launch");
        }
        e = cudaEventRecord(aux->join, aux->s);
        if (e == cudaSuccess) e = cudaStreamWaitEvent(st, aux->join, 0);
        return e == cudaSuccess ? PKV_OK : fail_cuda(e, "layer-batch join");
    }
    for (int l0 = 0; l0 < n_layers; l0 += chunk_env) {
        const int n = n_layers - l0 < chunk_env ? n_layers - l0 : chunk_env;
        const EvictArgs* chunk = as.data() + l0;
        if (n == 1) {      // a single layer left over: the per-layer launches
            if (stage != 0) return fail(PKV_ERR_UNSUPPORTED, "pkv_stage_batch: a left-over single layer has no batch stages");
            const int r1 = pkv_evict_prefill(&descs[l0], stream);
            if (r1) return r1;
            continue;
        }
        const int total_tiles = int(chunk[0].ws.s_pad / kTileTokens) * chunk[0].Hkv * n;
        const int grid = total_tiles < chunk[0].num_sms ? total_tiles : chunk[0].num_sms;
        cudaError_t e = cudaSuccess;
        // Layer-major form (>= 8 tiles per CTA and layer): every CTA scans its range of layer 0, then of layer 1, ... - the softmax
        // partials keep the per-layer layout (pooled scores bit-identical to the per-layer calls') and the pool launch can follow the
        // scan layer by layer. done[layer] counts the CTAs that finished a layer; the counters live in the first layer's
        // workspace (flag area of the fused kernel, unused here) and are zeroed in stream order.
        // PKV_BATCH_FOLLOW: 0 = one contiguous tile range per CTA over all layers; 1 (default) = layer-major walk; 2 = layer-major
        // with the pool launch started WITH the scan (programmatic dependent launch) and following it one layer behind through the
        // counters (with one or two pool CTAs per SM next to the scan the pool is latency-bound and the scan loses more than the
        // pool gains)
        static const int follow_env = []() { const char* e = getenv("PKV_BATCH_FOLLOW"); return e ? atoi(e) : 1; }();
        static const int stages_env = []() { const char* e = getenv("PKV_BATCH_STAGES"); return e ? atoi(e) : 4; }();
        int* done = nullptr;
        if (follow_env > 0 && tc5_layer_major_ok(chunk[0]))
            done = reinterpret_cast<int*>(chunk[0].ws_base + chunk[0].ws.fused_off + fused_ws_layout(chunk[0].Hq, chunk[0].G, chunk[0].k).flags_off);
        if (stage == 0 || stage == 1) {
            if (done) e = cudaMemsetAsync(done, 0, sizeof(int) * size_t(n), st);
            if (e == cudaSuccess) e = launch_score_tc5_layers(chunk, n, st, stages_env, done);     // 4 ring stages (PKV_BATCH_STAGES)
        }
        if (e != cudaSuccess) return fail_cuda(e, "layer-batch score launch");
        if (stage == 0 || stage == 2) e = launch_softmax_pool_layers(chunk, n, grid, st, done, follow_env >= 2);
        if (e != cudaSuccess) return fail_cuda(e, "layer-batch pool launch");
        if (stage == 0 || stage == 3) e = launch_select_layers(chunk, n, st);
        if (e != cudaSuccess) return fail_cuda(e, "layer-batch select launch");
    }
    return PKV_OK;
}
extern "C" int pkv_evict_prefill_batch(const pkv_evict_desc* descs, int n_layers, void* stream) { return pkv_stage_batch(descs, n_layers, 0, stream); }

// max_length > 0: graph-replayable launch — `length` is the row count at step 0 and the launch (split count, workspace,
// capacity check) is sized for max_length rows. num_seqs sequences: q / out / k_new / v_new hold num_seqs blocks back to back.
static int resolve_decode(const pkv_decode_desc* d, DecodeArgs* a, bool need_q, int64_t max_length = 0, int num_seqs = 1) {
    if (!d) return fail(PKV_ERR_INVALID_ARG, "null descriptor");
    if (d->struct_bytes != sizeof(pkv_decode_desc))
        return fail(PKV_ERR_INVALID_ARG, "pkv_decode_desc.struct_bytes=%u, library expects %zu (ABI mismatch)", d->struct_bytes, sizeof(pkv_decode_desc));
    if (d->dtype != PKV_BF16 && d->dtype != PKV_FP16) return fail(PKV_ERR_UNSUPPORTED_DTYPE, "dtype %d: only bf16 (0) and fp16 (1) are supported", d->dtype);
    if (d->num_q_heads <= 0 || d->num_kv_heads <= 0 || d->num_q_heads % d->num_kv_heads) return fail(PKV_ERR_INVALID_ARG, "bad head counts");
    if (d->head_dim != 64 && d->head_dim != 128) return fail(PKV_ERR_UNSUPPORTED, "head_dim=%d: only 64 and 128 are built", d->head_dim);
    if (d->length < 1) return fail(PKV_ERR_INVALID_ARG, "length must be >= 1");
    if (max_length != 0 && max_length < d->length) return fail(PKV_ERR_INVALID_ARG, "max_length=%lld is smaller than length=%lld", (long long)max_length, (long long)d->length);
    const int64_t rows_bound = max_length > 0 ? max_length : d->length;
    if (d->cache_stride_h < rows_bound * d->head_dim || d->cache_stride_h % 8) return fail(PKV_ERR_INVALID_ARG, "cache_stride_h too small for `length` rows (cache capacity exceeded)");
    if (!d->k_cache || !d->v_cache || (need_q && (!d->q || !d->out))) return fail(PKV_ERR_INVALID_ARG, "null tensor pointer");
    if ((d->k_new == nullptr) != (d->v_new == nullptr)) return fail(PKV_ERR_INVALID_ARG, "k_new and v_new must be given together");
    if (!aligned16(d->k_cache) || !aligned16(d->v_cache) || !aligned16(d->q) || !aligned16(d->out) || !aligned16(d->k_new) || !aligned16(d->v_new))
        return fail(PKV_ERR_INVALID_ARG, "tensor base pointers must be 16-byte aligned");
    const DevInfo* di = nullptr;
    int rc = device_info(d->device, &di);
    if (rc) return rc;
    a->dtype = d->dtype; a->Hq = d->num_q_heads; a->Hkv = d->num_kv_heads; a->G = a->Hq / a->Hkv; a->D = d->head_dim;
    a->T = d->length;
    a->q = static_cast<const uint16_t*>(d->q); a->k_new = static_cast<const uint16_t*>(d->k_new); a->v_new = static_cast<const uint16_t*>(d->v_new);
    a->k_cache = d->k_cache; a->v_cache = d->v_cache; a->out = static_cast<uint16_t*>(d->out);
    a->cache_sh = d->cache_stride_h;
    a->scale = d->softmax_scale != 0.f ? d->softmax_scale : 1.0f / sqrtf(float(d->head_dim));
    a->num_sms = di->sms;
    a->nsplit = decode_num_splits(a->Hq, rows_bound, a->num_sms);
    a->ws = static_cast<float*>(d->workspace);
    a->num_seqs = num_seqs;
    a->max_rows = rows_bound;
    if (need_q && a->nsplit > 1) {
        const uint64_t need = uint64_t(num_seqs) * a->Hq * a->nsplit * (2 + a->D) * sizeof(float);
        if (!d->workspace || d->workspace_bytes < need) return fail(PKV_ERR_WORKSPACE, "decode workspace of %llu bytes required", (unsigned long long)need);
    }
    return PKV_OK;
}

uint64_t pkv_decode_workspace_bytes(const pkv_decode_desc* d) {
    if (!d || d->num_q_heads <= 0 || d->head_dim <= 0) return 0;
    // upper bound over any length: at most 64 splits
    return uint64_t(d->num_q_heads) * 64 * (2 + uint64_t(d->head_dim)) * sizeof(float);
}

// The argument checks every device-length decode entry point shares.
static int check_devlen_args(const char* fn, int32_t num_seqs, const int32_t* rows, const int32_t* step_dev, int64_t max_length) {
    if ((reinterpret_cast<uintptr_t>(rows) & 3u) || (reinterpret_cast<uintptr_t>(step_dev) & 3u)) return fail(PKV_ERR_INVALID_ARG, "%s: misaligned int32 pointer", fn);
    if (max_length < 1) return fail(PKV_ERR_INVALID_ARG, "%s: max_length must be >= 1", fn);
    if (num_seqs < 1 || num_seqs > 65535) return fail(PKV_ERR_INVALID_ARG, "%s: num_seqs=%d outside [1, 65535]", fn, num_seqs);
    return PKV_OK;
}

// E4M3 caches: one fp32 scale per row for K and for V, `stride_h` / `stride_b` floats between heads / sequences
struct DecodeScales {
    float *k, *v;
    int64_t stride_h, stride_b;
};

// The decode of every cache form behind the seven entry points: num_seqs sequences with a cache per query head, or with a
// GQA-shared cache per KV head (`shared`), of 16-bit rows or of E4M3 rows (`scales`). host_length: pkv_decode_attn, the
// `length` rows of one sequence (num_seqs, rows, step_dev and max_length are not used); otherwise every device-length
// argument is checked.
static int decode(const char* fn, const pkv_decode_desc* d, bool shared, const DecodeScales* scales, bool host_length, int32_t num_seqs,
                  int64_t cache_stride_b, const int32_t* rows, const int32_t* step_dev, int64_t max_length, void* stream,
                  int64_t window = 0, const int32_t* prompt_rows = nullptr, const pkv_decode_heavy* heavy = nullptr) {
    int rc = host_length ? PKV_OK : check_devlen_args(fn, num_seqs, rows, step_dev, max_length);
    if (rc) return rc;
    if (scales && (!scales->k || !scales->v)) return fail(PKV_ERR_INVALID_ARG, "%s: null scale pointer", fn);
    if (scales && ((reinterpret_cast<uintptr_t>(scales->k) & 3u) || (reinterpret_cast<uintptr_t>(scales->v) & 3u)))
        return fail(PKV_ERR_INVALID_ARG, "%s: misaligned scale pointer", fn);
    DecodeArgs a;
    rc = resolve_decode(d, &a, true, host_length ? 0 : max_length, num_seqs);
    if (rc) return rc;
    if (shared && a.G != 2 && a.G != 4 && a.G != 8)
        return fail(PKV_ERR_UNSUPPORTED, "%s: group size num_q_heads/num_kv_heads = %d: the grouped kernels are built for 2, 4 and 8", fn, a.G);
    const int64_t align = scales ? 16 : 8;   // cache strides in elements that keep every row 16-byte aligned
    if (a.cache_sh % align) return fail(PKV_ERR_INVALID_ARG, "%s: cache_stride_h=%lld is not a multiple of 16 bytes", fn, (long long)a.cache_sh);
    const int heads = shared ? a.Hkv : a.Hq;   // cache heads per sequence
    a.cache_sb = heads * a.cache_sh;
    if (num_seqs > 1) {
        if (cache_stride_b < a.cache_sb || cache_stride_b % align)
            return fail(PKV_ERR_INVALID_ARG, "%s: cache_stride_b=%lld is below num_%s_heads*cache_stride_h=%lld or not a multiple of 16 bytes", fn,
                        (long long)cache_stride_b, shared ? "kv" : "q", (long long)a.cache_sb);
        a.cache_sb = cache_stride_b;
    }
    if (scales) {
        if (scales->stride_h < max_length || (num_seqs > 1 && scales->stride_b < heads * scales->stride_h))
            return fail(PKV_ERR_INVALID_ARG, "%s: scale strides (%lld, %lld) hold fewer than max_length=%lld rows per cache head", fn,
                        (long long)scales->stride_h, (long long)scales->stride_b, (long long)max_length);
        a.k_scale = scales->k;
        a.v_scale = scales->v;
        a.scale_sh = scales->stride_h;
        a.scale_sb = num_seqs > 1 ? scales->stride_b : heads * scales->stride_h;
    }
    a.heads_per_cache = shared ? a.G : 1;
    a.rows = rows;
    a.step_dev = step_dev;
    a.window = window;
    a.prompt_rows = prompt_rows;
    if (heavy) {
        const uint64_t need = pkv_decode_heavy_workspace_bytes(num_seqs, a.Hq, window);
        if (heavy->scratch_bytes < need) return fail(PKV_ERR_WORKSPACE, "%s: heavy scratch of %llu bytes required", fn, (unsigned long long)need);
        a.victim = heavy->victim;
        a.hv_scratch = static_cast<float*>(heavy->scratch);
        a.hv_scores = heavy->scores;
        a.hv_gen = heavy->gen;
        a.heavy = heavy->heavy;
    }
    DeviceGuard guard(d->device);
    const cudaError_t e = launch_decode(a, static_cast<cudaStream_t>(stream));
    return e == cudaSuccess ? PKV_OK : fail_cuda(e, fn);
}

int pkv_decode_attn(const pkv_decode_desc* d, void* stream) { return decode("pkv_decode_attn", d, false, nullptr, true, 1, 0, nullptr, nullptr, 0, stream); }

int pkv_decode_attn_batch(const pkv_decode_desc* d, int32_t num_seqs, int64_t cache_stride_b, const int32_t* rows,
                          const int32_t* step_dev, int64_t max_length, void* stream) {
    return decode("pkv_decode_attn_batch", d, false, nullptr, false, num_seqs, cache_stride_b, rows, step_dev, max_length, stream);
}

int pkv_decode_attn_batch_fp8(const pkv_decode_desc* d, int32_t num_seqs, int64_t cache_stride_b, const int32_t* rows,
                              const int32_t* step_dev, int64_t max_length, float* k_scale, float* v_scale, int64_t scale_stride_h,
                              int64_t scale_stride_b, void* stream) {
    const DecodeScales scales{k_scale, v_scale, scale_stride_h, scale_stride_b};
    return decode("pkv_decode_attn_batch_fp8", d, false, &scales, false, num_seqs, cache_stride_b, rows, step_dev, max_length, stream);
}

int pkv_decode_attn_batch_gqa(const pkv_decode_desc* d, int32_t num_seqs, int64_t cache_stride_b, const int32_t* rows,
                              const int32_t* step_dev, int64_t max_length, void* stream) {
    return decode("pkv_decode_attn_batch_gqa", d, true, nullptr, false, num_seqs, cache_stride_b, rows, step_dev, max_length, stream);
}

int pkv_decode_attn_batch_gqa_fp8(const pkv_decode_desc* d, int32_t num_seqs, int64_t cache_stride_b, const int32_t* rows,
                                  const int32_t* step_dev, int64_t max_length, float* k_scale, float* v_scale,
                                  int64_t scale_stride_h, int64_t scale_stride_b, void* stream) {
    const DecodeScales scales{k_scale, v_scale, scale_stride_h, scale_stride_b};
    return decode("pkv_decode_attn_batch_gqa_fp8", d, true, &scales, false, num_seqs, cache_stride_b, rows, step_dev, max_length, stream);
}

// The checks of the window arguments, then the decode (with the heavy-hitter state when `h` is set).
static int decode_window(const char* fn, const pkv_decode_desc* d, const pkv_decode_window* w, const pkv_decode_heavy* h, void* stream) {
    if (!w || w->struct_bytes != sizeof(pkv_decode_window))
        return fail(PKV_ERR_INVALID_ARG, "%s: null pkv_decode_window or struct_bytes != %zu (ABI mismatch)", fn, sizeof(pkv_decode_window));
    if (w->window < 1) return fail(PKV_ERR_INVALID_ARG, "%s: window=%lld must be >= 1", fn, (long long)w->window);
    if (!w->prompt_rows || (reinterpret_cast<uintptr_t>(w->prompt_rows) & 3u)) return fail(PKV_ERR_INVALID_ARG, "%s: null or misaligned prompt_rows", fn);
    if ((w->k_scale == nullptr) != (w->v_scale == nullptr)) return fail(PKV_ERR_INVALID_ARG, "%s: null scale pointer", fn);
    const DecodeScales scales{w->k_scale, w->v_scale, w->scale_stride_h, w->scale_stride_b};
    return decode(fn, d, w->gqa_shared != 0, w->k_scale ? &scales : nullptr, false, w->num_seqs, w->cache_stride_b, w->rows,
                  w->step_dev, w->max_length, stream, w->window, w->prompt_rows, h);
}

int pkv_decode_attn_window(const pkv_decode_desc* d, const pkv_decode_window* w, void* stream) {
    return decode_window("pkv_decode_attn_window", d, w, nullptr, stream);
}

uint64_t pkv_decode_heavy_workspace_bytes(int32_t num_seqs, int32_t num_q_heads, int64_t window) {
    if (num_seqs < 1 || num_q_heads < 1 || window < 1) return 0;
    return uint64_t(num_seqs) * uint64_t(num_q_heads) * uint64_t(window + 2) * sizeof(float);
}

int pkv_decode_attn_heavy(const pkv_decode_desc* d, const pkv_decode_window* w, const pkv_decode_heavy* h, void* stream) {
    const char* fn = "pkv_decode_attn_heavy";
    if (!h || h->struct_bytes != sizeof(pkv_decode_heavy))
        return fail(PKV_ERR_INVALID_ARG, "%s: null pkv_decode_heavy or struct_bytes != %zu (ABI mismatch)", fn, sizeof(pkv_decode_heavy));
    if (w && w->struct_bytes == sizeof(pkv_decode_window) && (h->heavy < 0 || h->heavy >= w->window))
        return fail(PKV_ERR_INVALID_ARG, "%s: heavy=%lld outside [0, window - 1 = %lld]", fn, (long long)h->heavy, (long long)w->window - 1);
    if (d && (!d->k_new || !d->v_new)) return fail(PKV_ERR_INVALID_ARG, "%s: the heavy-hitter step appends a row: k_new / v_new required", fn);
    const auto bad = [](const void* ptr) { return !ptr || (reinterpret_cast<uintptr_t>(ptr) & 3u); };
    if (bad(h->scores) || bad(h->gen) || bad(h->victim) || bad(h->scratch))
        return fail(PKV_ERR_INVALID_ARG, "%s: null or misaligned scores / gen / victim / scratch", fn);
    return decode_window(fn, d, w, h, stream);
}

int pkv_cache_quantize_fp8(int32_t dtype, int32_t num_seqs, int32_t num_heads, int32_t head_dim, int32_t device, int32_t num_layers,
                           const void* const* src, void* const* dst, float* const* scales, const int64_t* src_capacity,
                           const int64_t* dst_capacity, const int64_t* rows, const int32_t* const* rows_dev, void* stream) {
    const char* fn = "pkv_cache_quantize_fp8";
    if (dtype != PKV_BF16 && dtype != PKV_FP16) return fail(PKV_ERR_UNSUPPORTED_DTYPE, "%s: dtype %d: only bf16 (0) and fp16 (1) are supported", fn, dtype);
    if (head_dim != 64 && head_dim != 128) return fail(PKV_ERR_UNSUPPORTED, "%s: head_dim=%d: only 64 and 128 are built", fn, head_dim);
    if (num_seqs < 1 || num_heads < 1 || num_layers < 1) return fail(PKV_ERR_INVALID_ARG, "%s: need num_seqs, num_heads, num_layers >= 1", fn);
    if (!src || !dst || !scales || !src_capacity || !dst_capacity || !rows) return fail(PKV_ERR_INVALID_ARG, "%s: null table", fn);
    for (int l = 0; l < num_layers; ++l) {
        for (int kv = 0; kv < 2; ++kv) {
            const void* s = src[2 * l + kv];
            const void* t = dst[2 * l + kv];
            const float* c = scales[2 * l + kv];
            if (!s || !t || !c) return fail(PKV_ERR_INVALID_ARG, "%s: layer %d: null tensor pointer", fn, l);
            if (!aligned16(s) || !aligned16(t) || (reinterpret_cast<uintptr_t>(c) & 3u)) return fail(PKV_ERR_INVALID_ARG, "%s: layer %d: misaligned tensor pointer", fn, l);
        }
        if (rows[l] < 0 || rows[l] > src_capacity[l] || rows[l] > dst_capacity[l])
            return fail(PKV_ERR_INVALID_ARG, "%s: layer %d: rows=%lld outside [0, capacity] (source %lld, destination %lld)", fn, l,
                        (long long)rows[l], (long long)src_capacity[l], (long long)dst_capacity[l]);
        if (rows_dev && (reinterpret_cast<uintptr_t>(rows_dev[l]) & 3u)) return fail(PKV_ERR_INVALID_ARG, "%s: layer %d: misaligned row counts", fn, l);
    }
    const DevInfo* di = nullptr;
    int rc = device_info(device, &di);
    if (rc) return rc;
    DeviceGuard guard(device);
    for (int l0 = 0; l0 < num_layers; l0 += kMaxLayerBatch) {
        QuantArgs a;
        a.dtype = dtype; a.num_seqs = num_seqs; a.H = num_heads; a.D = head_dim;
        a.n_layers = std::min(kMaxLayerBatch, num_layers - l0);
        for (int i = 0; i < a.n_layers; ++i) {
            const int l = l0 + i;
            QuantLayer& q = a.layer[i];
            for (int kv = 0; kv < 2; ++kv) {
                q.src[kv] = static_cast<const uint16_t*>(src[2 * l + kv]);
                q.dst[kv] = static_cast<uint8_t*>(dst[2 * l + kv]);
                q.scale[kv] = scales[2 * l + kv];
            }
            q.src_cap = src_capacity[l];
            q.dst_cap = dst_capacity[l];
            q.rows = rows[l];
            q.rows_dev = rows_dev ? rows_dev[l] : nullptr;
        }
        const cudaError_t e = launch_quantize_fp8(a, di->sms, static_cast<cudaStream_t>(stream));
        if (e != cudaSuccess) return fail_cuda(e, "fp8 quantize launch");
    }
    return PKV_OK;
}

int pkv_cache_install(int32_t elem_bytes, int32_t num_seqs, int32_t num_heads, int32_t head_dim, int32_t device, int32_t num_layers,
                      int32_t slot, const void* const* src, void* const* dst, const float* const* src_scales, float* const* dst_scales,
                      const int64_t* src_capacity, const int64_t* dst_capacity, const int64_t* rows, const int32_t* const* rows_dev,
                      int32_t* const* dst_rows, const int32_t* step_dev, void* stream) {
    const char* fn = "pkv_cache_install";
    if (elem_bytes != 1 && elem_bytes != 2) return fail(PKV_ERR_INVALID_ARG, "%s: elem_bytes=%d: 2 (bf16 / fp16) or 1 (E4M3)", fn, elem_bytes);
    if (head_dim != 64 && head_dim != 128) return fail(PKV_ERR_UNSUPPORTED, "%s: head_dim=%d: only 64 and 128 are built", fn, head_dim);
    if (num_seqs < 1 || num_heads < 1 || num_heads > 4096 || num_layers < 1)
        return fail(PKV_ERR_INVALID_ARG, "%s: need num_seqs >= 1, 1 <= num_heads <= 4096, num_layers >= 1", fn);
    if (slot < 0 || slot >= num_seqs) return fail(PKV_ERR_INVALID_ARG, "%s: slot %d outside [0, %d)", fn, slot, num_seqs);
    if (!step_dev || (reinterpret_cast<uintptr_t>(step_dev) & 3u)) return fail(PKV_ERR_INVALID_ARG, "%s: null or misaligned step counter", fn);
    if (!dst || !dst_rows || !src_capacity || !dst_capacity || !rows) return fail(PKV_ERR_INVALID_ARG, "%s: null table", fn);
    const bool fp8 = elem_bytes == 1;
    if (fp8 != (dst_scales != nullptr)) return fail(PKV_ERR_INVALID_ARG, "%s: scale tables go with elem_bytes 1 (E4M3) only, and it needs them", fn);
    for (int l = 0; l < num_layers; ++l) {
        if (rows[l] < 0 || rows[l] > dst_capacity[l] || (rows[l] > 0 && rows[l] > src_capacity[l]))
            return fail(PKV_ERR_INVALID_ARG, "%s: layer %d: rows=%lld outside [0, capacity] (source %lld, destination %lld)", fn, l,
                        (long long)rows[l], (long long)src_capacity[l], (long long)dst_capacity[l]);
        if (!dst_rows[l] || (reinterpret_cast<uintptr_t>(dst_rows[l]) & 3u)) return fail(PKV_ERR_INVALID_ARG, "%s: layer %d: null or misaligned row counts", fn, l);
        if (rows_dev && (reinterpret_cast<uintptr_t>(rows_dev[l]) & 3u)) return fail(PKV_ERR_INVALID_ARG, "%s: layer %d: misaligned source row counts", fn, l);
        for (int kv = 0; kv < 2; ++kv) {
            const void* t = dst[2 * l + kv];
            if (!t || !aligned16(t)) return fail(PKV_ERR_INVALID_ARG, "%s: layer %d: null or misaligned destination", fn, l);
            if (fp8 && (!dst_scales[2 * l + kv] || (reinterpret_cast<uintptr_t>(dst_scales[2 * l + kv]) & 3u)))
                return fail(PKV_ERR_INVALID_ARG, "%s: layer %d: null or misaligned destination scales", fn, l);
            if (rows[l] == 0) continue;
            const void* s = src ? src[2 * l + kv] : nullptr;
            if (!s || !aligned16(s)) return fail(PKV_ERR_INVALID_ARG, "%s: layer %d: null or misaligned source", fn, l);
            if (fp8 && (!src_scales || !src_scales[2 * l + kv] || (reinterpret_cast<uintptr_t>(src_scales[2 * l + kv]) & 3u)))
                return fail(PKV_ERR_INVALID_ARG, "%s: layer %d: null or misaligned source scales", fn, l);
        }
    }
    const DevInfo* di = nullptr;
    int rc = device_info(device, &di);
    if (rc) return rc;
    DeviceGuard guard(device);
    for (int l0 = 0; l0 < num_layers; l0 += kMaxLayerBatch) {
        InstallArgs a;
        a.H = num_heads; a.slot = slot; a.step_dev = step_dev;
        a.n_layers = std::min(kMaxLayerBatch, num_layers - l0);
        for (int i = 0; i < a.n_layers; ++i) {
            const int l = l0 + i;
            InstallLayer& q = a.layer[i];
            for (int kv = 0; kv < 2; ++kv) {
                q.src[kv] = rows[l] > 0 ? static_cast<const uint8_t*>(src[2 * l + kv]) : nullptr;
                q.dst[kv] = static_cast<uint8_t*>(dst[2 * l + kv]);
                q.src_scale[kv] = fp8 && rows[l] > 0 ? src_scales[2 * l + kv] : nullptr;
                q.dst_scale[kv] = fp8 ? dst_scales[2 * l + kv] : nullptr;
            }
            q.src_cap = src_capacity[l];
            q.dst_cap = dst_capacity[l];
            q.rows = rows[l];
            q.rows_dev = rows_dev && rows[l] > 0 ? rows_dev[l] : nullptr;
            q.dst_rows = dst_rows[l];
        }
        const cudaError_t e = launch_install(a, head_dim * elem_bytes, di->sms, static_cast<cudaStream_t>(stream));
        if (e != cudaSuccess) return fail_cuda(e, "cache install launch");
    }
    return PKV_OK;
}

int pkv_decode_attn_graph(const pkv_decode_desc* d, const int32_t* step_dev, int64_t max_length, void* stream) {
    if (!step_dev) return fail(PKV_ERR_INVALID_ARG, "pkv_decode_attn_graph: null step counter");
    return decode("pkv_decode_attn_graph", d, false, nullptr, false, 1, 0, nullptr, step_dev, max_length, stream);
}

int pkv_rope_inplace(const pkv_rope_desc* d, void* stream) {
    if (!d) return fail(PKV_ERR_INVALID_ARG, "null descriptor");
    if (d->struct_bytes != sizeof(pkv_rope_desc))
        return fail(PKV_ERR_INVALID_ARG, "pkv_rope_desc.struct_bytes=%u, library expects %zu (ABI mismatch)", d->struct_bytes, sizeof(pkv_rope_desc));
    if (d->dtype != PKV_BF16 && d->dtype != PKV_FP16) return fail(PKV_ERR_UNSUPPORTED_DTYPE, "dtype %d: only bf16 (0) and fp16 (1) are supported", d->dtype);
    if (d->num_q_heads <= 0 || d->num_kv_heads <= 0) return fail(PKV_ERR_INVALID_ARG, "bad head counts");
    if (d->head_dim != 64 && d->head_dim != 128) return fail(PKV_ERR_UNSUPPORTED, "head_dim=%d: only 64 and 128 are built", d->head_dim);
    if (d->seq_len < 1) return fail(PKV_ERR_INVALID_ARG, "seq_len must be >= 1");
    if (!d->q || !d->k || !d->cos || !d->sin) return fail(PKV_ERR_INVALID_ARG, "null tensor pointer");
    if (!aligned16(d->q) || !aligned16(d->k) || !aligned16(d->cos) || !aligned16(d->sin)) return fail(PKV_ERR_INVALID_ARG, "tensor base pointers must be 16-byte aligned");
    const int64_t st[] = {d->q_stride_h, d->q_stride_s, d->k_stride_h, d->k_stride_s, d->cs_stride_s};
    for (int64_t s : st)
        if (s % 8 != 0 || s < 0) return fail(PKV_ERR_INVALID_ARG, "strides must be non-negative multiples of 8 elements (16 bytes), got %lld", (long long)s);
    if (d->q_stride_s < d->head_dim || d->k_stride_s < d->head_dim || d->cs_stride_s < d->head_dim)
        return fail(PKV_ERR_INVALID_ARG, "token strides must be >= head_dim (last dim contiguous)");
    const DevInfo* di = nullptr;
    int rc = device_info(d->device, &di);
    if (rc) return rc;
    RopeArgs a;
    a.dtype = d->dtype; a.Hq = d->num_q_heads; a.Hkv = d->num_kv_heads; a.D = d->head_dim; a.S = d->seq_len;
    a.q = static_cast<uint16_t*>(d->q); a.k = static_cast<uint16_t*>(d->k);
    a.q_sh = d->q_stride_h; a.q_ss = d->q_stride_s; a.k_sh = d->k_stride_h; a.k_ss = d->k_stride_s;
    a.cos = static_cast<const uint16_t*>(d->cos); a.sin = static_cast<const uint16_t*>(d->sin); a.cs_ss = d->cs_stride_s;
    a.num_sms = di->sms;
    DeviceGuard guard(d->device);
    const cudaError_t e = launch_rope(a, static_cast<cudaStream_t>(stream));
    return e == cudaSuccess ? PKV_OK : fail_cuda(e, "rope launch");
}

uint64_t pkv_adakv_scratch_bytes(int32_t num_q_heads) { return num_q_heads > 0 ? uint64_t(adakv_scratch_bytes(num_q_heads)) : 0; }

int pkv_adakv_counts(const pkv_evict_desc* d, int64_t base_capacity, int32_t normalize, void* scratch, uint64_t scratch_bytes,
                     int32_t* counts, void* stream) {
    PKV_STAGE_PROLOGUE();
    if (!is_window_method(a.method)) return fail(PKV_ERR_INVALID_ARG, "pkv_adakv_counts: the scores come from a window method (use PKV_SNAPKV)");
    if (a.flags & PKV_FLAG_GQA_SHARED) return fail(PKV_ERR_UNSUPPORTED, "pkv_adakv_counts: per-query-head budgets are not built for PKV_FLAG_GQA_SHARED");
    if (!a.window_mean) return fail(PKV_ERR_INVALID_ARG, "pkv_adakv_counts: the scores must come from stage 2 with PKV_FLAG_WINDOW_MEAN (calcul_attn_sore averages the window rows)");
    if (base_capacity < 1 || base_capacity > a.n) return fail(PKV_ERR_INVALID_ARG, "base_capacity=%lld out of range [1, seq_len-window=%lld]", (long long)base_capacity, (long long)a.n);
    if (!scratch || !counts || scratch_bytes < adakv_scratch_bytes(a.Hq)) return fail(PKV_ERR_WORKSPACE, "pkv_adakv_counts: scratch of %zu bytes and a counts buffer are required", adakv_scratch_bytes(a.Hq));
    if ((reinterpret_cast<uintptr_t>(scratch) & 15u) || (reinterpret_cast<uintptr_t>(counts) & 3u)) return fail(PKV_ERR_INVALID_ARG, "pkv_adakv_counts: misaligned scratch / counts");
    const cudaError_t e = launch_adakv_counts(a, base_capacity, normalize != 0, scratch, counts, st);
    return e == cudaSuccess ? PKV_OK : fail_cuda(e, "adakv counts launch");
}

int pkv_ragged_place_window(const pkv_evict_desc* d, const int32_t* caps, void* stream) {
    PKV_STAGE_PROLOGUE();
    if (!caps) return fail(PKV_ERR_INVALID_ARG, "pkv_ragged_place_window: null caps");
    if (a.flags & PKV_FLAG_GQA_SHARED) return fail(PKV_ERR_UNSUPPORTED, "pkv_ragged_place_window: per-query-head budgets are not built for PKV_FLAG_GQA_SHARED");
    const cudaError_t e = launch_ragged_window(a, caps, st);
    return e == cudaSuccess ? PKV_OK : fail_cuda(e, "ragged window launch");
}

int pkv_decode_attn_ragged(const pkv_decode_desc* d, const int32_t* head_rows, const int32_t* step_dev, int64_t max_length, void* stream) {
    if (!head_rows) return fail(PKV_ERR_INVALID_ARG, "pkv_decode_attn_ragged: null head_rows");
    return decode("pkv_decode_attn_ragged", d, false, nullptr, false, 1, 0, head_rows, step_dev, max_length, stream);
}

int pkv_update_flatten_view(void* dst, const void* src, const void* state, const int32_t* head_lens, const int32_t* cu_lens,
                            int32_t num_heads, int32_t row_bytes, int32_t device, void* stream) {
    if (!dst || !src || !state || !head_lens || !cu_lens) return fail(PKV_ERR_INVALID_ARG, "pkv_update_flatten_view: null pointer");
    if (num_heads <= 0 || num_heads > 65535) return fail(PKV_ERR_INVALID_ARG, "pkv_update_flatten_view: num_heads=%d out of range", num_heads);
    if (row_bytes <= 0 || row_bytes % 16 != 0 || row_bytes > 16 * 256) return fail(PKV_ERR_INVALID_ARG, "pkv_update_flatten_view: row_bytes=%d must be a multiple of 16 (at most 4096)", row_bytes);
    if (!aligned16(dst) || !aligned16(src) || !aligned16(state)) return fail(PKV_ERR_INVALID_ARG, "tensor base pointers must be 16-byte aligned");
    const DevInfo* di = nullptr;
    int rc = device_info(device, &di);
    if (rc) return rc;
    DeviceGuard guard(device);
    const cudaError_t e = launch_flatten_append(dst, src, state, head_lens, cu_lens, num_heads, row_bytes, di->sms, static_cast<cudaStream_t>(stream));
    return e == cudaSuccess ? PKV_OK : fail_cuda(e, "flatten append launch");
}

// The checks of pkv_sample_tokens, then its launch, or the penalized one when `pen` is set, or the constrained one when `rules`
// is also set (both already checked).
static int sample(const char* fn, const pkv_sample_desc* d, const pkv_sample_penalty* pen, void* stream,
                  const pkv_sample_rules* rules = nullptr) {
    if (!d) return fail(PKV_ERR_INVALID_ARG, "%s: null descriptor", fn);
    if (d->struct_bytes != sizeof(pkv_sample_desc))
        return fail(PKV_ERR_INVALID_ARG, "pkv_sample_desc.struct_bytes=%u, library expects %zu (ABI mismatch)", d->struct_bytes, sizeof(pkv_sample_desc));
    if (d->dtype != PKV_BF16 && d->dtype != PKV_FP16) return fail(PKV_ERR_UNSUPPORTED_DTYPE, "%s: dtype %d: only bf16 (0) and fp16 (1) logits", fn, d->dtype);
    if (d->batch < 1 || d->batch > (1 << 20)) return fail(PKV_ERR_INVALID_ARG, "%s: batch=%d outside [1, 2^20]", fn, d->batch);
    if (d->vocab < 1 || d->vocab > (int64_t(1) << 24)) return fail(PKV_ERR_INVALID_ARG, "%s: vocab=%lld outside [1, 2^24]", fn, (long long)d->vocab);
    if (d->logits_stride < d->vocab) return fail(PKV_ERR_INVALID_ARG, "%s: logits_stride=%lld < vocab=%lld", fn, (long long)d->logits_stride, (long long)d->vocab);
    if (d->column < 0 || d->column >= d->tokens_stride)
        return fail(PKV_ERR_INVALID_ARG, "%s: column=%lld outside [0, tokens_stride=%lld)", fn, (long long)d->column, (long long)d->tokens_stride);
    if (d->flags & ~PKV_SAMPLE_ADVANCE) return fail(PKV_ERR_INVALID_ARG, "%s: unknown flags 0x%x", fn, d->flags);
    auto bad = [](const void* p, uintptr_t align) { return !p || (reinterpret_cast<uintptr_t>(p) & (align - 1)); };
    if (bad(d->logits, 2)) return fail(PKV_ERR_INVALID_ARG, "%s: null or misaligned logits (2 bytes)", fn);
    if (bad(d->temperature, 4) || bad(d->top_k, 4) || bad(d->top_p, 4))
        return fail(PKV_ERR_INVALID_ARG, "%s: null or misaligned temperature / top_k / top_p (4 bytes)", fn);
    if (bad(d->seed, 8) || bad(d->token_index, 8) || bad(d->tokens, 8))
        return fail(PKV_ERR_INVALID_ARG, "%s: null or misaligned seed / token_index / tokens (8 bytes)", fn);
    const DevInfo* di = nullptr;
    int rc = device_info(d->device, &di);
    if (rc) return rc;
    SampleArgs a;
    a.dtype = d->dtype; a.B = d->batch; a.V = int(d->vocab);
    a.logits = static_cast<const uint16_t*>(d->logits); a.ld = d->logits_stride;
    a.temperature = d->temperature; a.top_k = d->top_k; a.top_p = d->top_p; a.seed = d->seed; a.token_index = d->token_index;
    a.tokens = d->tokens; a.tokens_ld = d->tokens_stride; a.col = d->column;
    a.advance = (d->flags & PKV_SAMPLE_ADVANCE) != 0;
    DeviceGuard guard(d->device);
    if (!pen) {
        const cudaError_t e = launch_sample(a, static_cast<cudaStream_t>(stream));
        return e == cudaSuccess ? PKV_OK : fail_cuda(e, "sample launch");
    }
    if (pen->stride < d->vocab) return fail(PKV_ERR_INVALID_ARG, "%s: stride=%lld < vocab=%lld", fn, (long long)pen->stride, (long long)d->vocab);
    PenaltyArgs p;
    p.repetition = pen->repetition_penalty; p.presence = pen->presence_penalty; p.frequency = pen->frequency_penalty;
    p.min_p = pen->min_p; p.mask = pen->prompt_mask; p.counts = pen->counts; p.ld = pen->stride;
    if (!rules) {
        const cudaError_t e = launch_sample_penalized(a, p, static_cast<cudaStream_t>(stream));
        return e == cudaSuccess ? PKV_OK : fail_cuda(e, "penalized sample launch");
    }
    const int64_t W = (d->vocab + 31) / 32;
    if (rules->bias_stride < d->vocab || rules->ban_stride < 2 * W)
        return fail(PKV_ERR_INVALID_ARG, "%s: bias_stride=%lld < vocab=%lld or ban_stride=%lld < %lld", fn, (long long)rules->bias_stride,
                    (long long)d->vocab, (long long)rules->ban_stride, (long long)(2 * W));
    RuleTermArgs q;
    q.flags = rules->flags; q.bias = rules->bias; q.bias_ld = rules->bias_stride; q.ban = rules->ban; q.ban_ld = rules->ban_stride;
    q.W = int(W);
    const cudaError_t e = launch_sample_constrained(a, p, q, static_cast<cudaStream_t>(stream));
    return e == cudaSuccess ? PKV_OK : fail_cuda(e, "constrained sample launch");
}

int pkv_sample_tokens(const pkv_sample_desc* d, void* stream) { return sample("pkv_sample_tokens", d, nullptr, stream); }

static int check_penalty(const char* fn, const pkv_sample_penalty* pen) {
    if (!pen || pen->struct_bytes != sizeof(pkv_sample_penalty))
        return fail(PKV_ERR_INVALID_ARG, "%s: null pkv_sample_penalty or struct_bytes != %zu (ABI mismatch)", fn, sizeof(pkv_sample_penalty));
    const auto bad = [](const void* ptr, uintptr_t align) { return !ptr || (reinterpret_cast<uintptr_t>(ptr) & (align - 1)); };
    if (bad(pen->repetition_penalty, 4) || bad(pen->presence_penalty, 4) || bad(pen->frequency_penalty, 4) || bad(pen->min_p, 4))
        return fail(PKV_ERR_INVALID_ARG, "%s: null or misaligned repetition / presence / frequency penalty or min_p (4 bytes)", fn);
    if (bad(pen->prompt_mask, 1) || bad(pen->counts, 4)) return fail(PKV_ERR_INVALID_ARG, "%s: null prompt_mask, or null or misaligned counts (4 bytes)", fn);
    return PKV_OK;
}

int pkv_sample_tokens_penalized(const pkv_sample_desc* d, const pkv_sample_penalty* pen, void* stream) {
    const char* fn = "pkv_sample_tokens_penalized";
    const int rc = check_penalty(fn, pen);
    return rc ? rc : sample(fn, d, pen, stream);
}

int pkv_sample_tokens_constrained(const pkv_sample_desc* d, const pkv_sample_penalty* pen, const pkv_sample_rules* r,
                                  void* stream) {
    const char* fn = "pkv_sample_tokens_constrained";
    int rc = check_penalty(fn, pen);
    if (rc) return rc;
    if (!r || r->struct_bytes != sizeof(pkv_sample_rules))
        return fail(PKV_ERR_INVALID_ARG, "%s: null pkv_sample_rules or struct_bytes != %zu (ABI mismatch)", fn, sizeof(pkv_sample_rules));
    const auto bad = [](const void* ptr, uintptr_t align) { return !ptr || (reinterpret_cast<uintptr_t>(ptr) & (align - 1)); };
    if (bad(r->flags, 4) || bad(r->bias, 4) || bad(r->ban, 4))
        return fail(PKV_ERR_INVALID_ARG, "%s: null or misaligned flags / bias / ban (4 bytes)", fn);
    return sample(fn, d, pen, stream, r);
}

int pkv_token_rules(const pkv_token_rules_desc* d, void* stream) {
    const char* fn = "pkv_token_rules";
    if (!d) return fail(PKV_ERR_INVALID_ARG, "%s: null descriptor", fn);
    if (d->struct_bytes != sizeof(pkv_token_rules_desc))
        return fail(PKV_ERR_INVALID_ARG, "pkv_token_rules_desc.struct_bytes=%u, library expects %zu (ABI mismatch)", d->struct_bytes, sizeof(pkv_token_rules_desc));
    if (d->batch < 1 || d->batch > (1 << 20)) return fail(PKV_ERR_INVALID_ARG, "%s: batch=%d outside [1, 2^20]", fn, d->batch);
    if (d->vocab < 1 || d->vocab > (1 << 24)) return fail(PKV_ERR_INVALID_ARG, "%s: vocab=%d outside [1, 2^24]", fn, d->vocab);
    const int64_t W = (int64_t(d->vocab) + 31) / 32;
    if (d->history_stride < 1 || d->history_stride > INT32_MAX || d->bias_stride < d->vocab || d->ban_stride < 2 * W ||
        d->seq_stride < 2 || d->tokens_stride < 1 || d->n_eos < 0)
        return fail(PKV_ERR_INVALID_ARG, "%s: history_stride=%lld, bias_stride=%lld (vocab %d), ban_stride=%lld (>= %lld), seq_stride=%lld, "
                    "tokens_stride=%lld or n_eos=%d out of range", fn, (long long)d->history_stride, (long long)d->bias_stride, d->vocab,
                    (long long)d->ban_stride, (long long)(2 * W), (long long)d->seq_stride, (long long)d->tokens_stride, d->n_eos);
    const auto bad = [](const void* ptr, uintptr_t align) { return !ptr || (reinterpret_cast<uintptr_t>(ptr) & (align - 1)); };
    if (bad(d->history, 4) || bad(d->history_len, 4) || bad(d->prompt_len, 4) || bad(d->flags, 4) || bad(d->ngram, 4) ||
        bad(d->min_new_tokens, 4) || bad(d->n_seq, 4) || bad(d->seq_off, 4) || bad(d->seq_kind, 4) || bad(d->seq_bias, 4) ||
        bad(d->seq_tokens, 4) || bad(d->bias, 4) || bad(d->ban, 4) || bad(d->stop, 1) || (d->n_eos > 0 && bad(d->eos, 4)))
        return fail(PKV_ERR_INVALID_ARG, "%s: null or misaligned device array (4 bytes)", fn);
    if (d->append && ((reinterpret_cast<uintptr_t>(d->append) & 7u) || d->append_column < 0 || d->append_column >= d->append_stride))
        return fail(PKV_ERR_INVALID_ARG, "%s: misaligned append (8 bytes) or append_column=%lld outside [0, append_stride=%lld)", fn,
                    (long long)d->append_column, (long long)d->append_stride);
    const DevInfo* di = nullptr;
    const int rc = device_info(d->device, &di);
    if (rc) return rc;
    TokenRulesArgs a;
    a.B = d->batch; a.V = d->vocab; a.W = int(W); a.n_eos = d->n_eos;
    a.hist = d->history; a.hist_ld = d->history_stride; a.hist_len = d->history_len; a.prompt_len = d->prompt_len;
    a.flags = d->flags; a.ngram = d->ngram; a.min_new = d->min_new_tokens; a.n_seq = d->n_seq;
    a.seq_off = d->seq_off; a.seq_kind = d->seq_kind; a.seq_bias = d->seq_bias; a.seq_ld = d->seq_stride;
    a.seq_tok = d->seq_tokens; a.tok_ld = d->tokens_stride; a.eos = d->eos;
    a.append = d->append; a.append_ld = d->append_stride; a.append_col = d->append_column;
    a.bias = d->bias; a.bias_ld = d->bias_stride; a.ban = d->ban; a.ban_ld = d->ban_stride; a.stop = d->stop;
    DeviceGuard guard(d->device);
    const cudaError_t e = launch_token_rules(a, static_cast<cudaStream_t>(stream));
    return e == cudaSuccess ? PKV_OK : fail_cuda(e, "token rules launch");
}

int pkv_token_logprobs(const pkv_logprobs_desc* d, void* stream) {
    const char* fn = "pkv_token_logprobs";
    if (!d) return fail(PKV_ERR_INVALID_ARG, "%s: null descriptor", fn);
    if (d->struct_bytes != sizeof(pkv_logprobs_desc))
        return fail(PKV_ERR_INVALID_ARG, "pkv_logprobs_desc.struct_bytes=%u, library expects %zu (ABI mismatch)", d->struct_bytes, sizeof(pkv_logprobs_desc));
    if (d->dtype != PKV_BF16 && d->dtype != PKV_FP16) return fail(PKV_ERR_UNSUPPORTED_DTYPE, "%s: dtype %d: only bf16 (0) and fp16 (1) logits", fn, d->dtype);
    if (d->batch < 1 || d->batch > (1 << 20)) return fail(PKV_ERR_INVALID_ARG, "%s: batch=%d outside [1, 2^20]", fn, d->batch);
    if (d->vocab < 1 || d->vocab > (int64_t(1) << 24)) return fail(PKV_ERR_INVALID_ARG, "%s: vocab=%lld outside [1, 2^24]", fn, (long long)d->vocab);
    if (d->logits_stride < d->vocab) return fail(PKV_ERR_INVALID_ARG, "%s: logits_stride=%lld < vocab=%lld", fn, (long long)d->logits_stride, (long long)d->vocab);
    if (d->top_n < 0 || d->top_n > kMaxTopLogprobs) return fail(PKV_ERR_INVALID_ARG, "%s: top_n=%d outside [0, %d]", fn, d->top_n, kMaxTopLogprobs);
    if (d->tokens_column < 0 || d->tokens_column >= d->tokens_stride)
        return fail(PKV_ERR_INVALID_ARG, "%s: tokens_column=%lld outside [0, tokens_stride=%lld)", fn, (long long)d->tokens_column, (long long)d->tokens_stride);
    if (d->column < 0 || d->logprob_stride <= d->column)
        return fail(PKV_ERR_INVALID_ARG, "%s: column=%lld outside [0, logprob_stride=%lld)", fn, (long long)d->column, (long long)d->logprob_stride);
    if (d->top_n > 0 && d->top_stride < (d->column + 1) * d->top_n)
        return fail(PKV_ERR_INVALID_ARG, "%s: top_stride=%lld < (column + 1) * top_n = %lld", fn, (long long)d->top_stride, (long long)((d->column + 1) * d->top_n));
    if (d->flags) return fail(PKV_ERR_INVALID_ARG, "%s: unknown flags 0x%x", fn, d->flags);
    auto bad = [](const void* p, uintptr_t align) { return !p || (reinterpret_cast<uintptr_t>(p) & (align - 1)); };
    if (bad(d->logits, 2)) return fail(PKV_ERR_INVALID_ARG, "%s: null or misaligned logits (2 bytes)", fn);
    if (bad(d->tokens, 8)) return fail(PKV_ERR_INVALID_ARG, "%s: null or misaligned tokens (8 bytes)", fn);
    if (bad(d->logprob, 4)) return fail(PKV_ERR_INVALID_ARG, "%s: null or misaligned logprob (4 bytes)", fn);
    if (d->cursor && (reinterpret_cast<uintptr_t>(d->cursor) & 7u)) return fail(PKV_ERR_INVALID_ARG, "%s: misaligned cursor (8 bytes)", fn);
    if (d->top_n > 0 && (bad(d->top_ids, 8) || bad(d->top_logprobs, 4)))
        return fail(PKV_ERR_INVALID_ARG, "%s: null or misaligned top_ids (8 bytes) / top_logprobs (4 bytes)", fn);
    const DevInfo* di = nullptr;
    int rc = device_info(d->device, &di);
    if (rc) return rc;
    LogprobsArgs a;
    a.dtype = d->dtype; a.B = d->batch; a.V = int(d->vocab); a.N = d->top_n;
    a.logits = static_cast<const uint16_t*>(d->logits); a.ld = d->logits_stride;
    a.tokens = d->tokens; a.tokens_ld = d->tokens_stride; a.tokens_col = d->tokens_column;
    a.cursor = d->cursor; a.col = d->column;
    a.lp = d->logprob; a.lp_ld = d->logprob_stride;
    a.top_ids = d->top_ids; a.top_lp = d->top_logprobs; a.top_ld = d->top_stride;
    DeviceGuard guard(d->device);
    const cudaError_t e = launch_logprobs(a, static_cast<cudaStream_t>(stream));
    return e == cudaSuccess ? PKV_OK : fail_cuda(e, "logprobs launch");
}

int pkv_cache_append(const pkv_decode_desc* d, void* stream) {
    DecodeArgs a;
    int rc = resolve_decode(d, &a, false);
    if (rc) return rc;
    if (!a.k_new) return fail(PKV_ERR_INVALID_ARG, "k_new/v_new required");
    DeviceGuard guard(d->device);
    const cudaError_t e = launch_append(a, static_cast<cudaStream_t>(stream));
    return e == cudaSuccess ? PKV_OK : fail_cuda(e, "append launch");
}

int pkv_beam_candidates(int32_t dtype, int32_t device, int32_t rows, int64_t vocab, const void* logits, int64_t logits_stride,
                        int32_t top_k, float* m, float* log_z, float* cand_lp, int32_t* cand_id, void* stream) {
    const char* fn = "pkv_beam_candidates";
    if (dtype != PKV_BF16 && dtype != PKV_FP16) return fail(PKV_ERR_UNSUPPORTED_DTYPE, "%s: dtype %d: only bf16 (0) and fp16 (1) logits", fn, dtype);
    if (rows < 1 || rows > (1 << 20)) return fail(PKV_ERR_INVALID_ARG, "%s: rows=%d outside [1, 2^20]", fn, rows);
    if (vocab < 1 || vocab > (int64_t(1) << 24)) return fail(PKV_ERR_INVALID_ARG, "%s: vocab=%lld outside [1, 2^24]", fn, (long long)vocab);
    if (logits_stride < vocab) return fail(PKV_ERR_INVALID_ARG, "%s: logits_stride=%lld < vocab", fn, (long long)logits_stride);
    if (top_k < 1 || top_k > kMaxBeamCandidates) return fail(PKV_ERR_INVALID_ARG, "%s: top_k=%d outside [1, %d]", fn, top_k, kMaxBeamCandidates);
    auto bad = [](const void* p, uintptr_t align) { return !p || (reinterpret_cast<uintptr_t>(p) & (align - 1)); };
    if (bad(logits, 2) || bad(m, 4) || bad(log_z, 4) || bad(cand_lp, 4) || bad(cand_id, 4))
        return fail(PKV_ERR_INVALID_ARG, "%s: null or misaligned pointer", fn);
    const DevInfo* di = nullptr;
    int rc = device_info(device, &di);
    if (rc) return rc;
    BeamCandArgs a;
    a.dtype = dtype; a.rows = rows; a.V = int(vocab); a.K = top_k;
    a.logits = static_cast<const uint16_t*>(logits); a.ld = logits_stride;
    a.m = m; a.log_z = log_z; a.cand_lp = cand_lp; a.cand_id = cand_id;
    DeviceGuard guard(device);
    const cudaError_t e = launch_beam_candidates(a, static_cast<cudaStream_t>(stream));
    return e == cudaSuccess ? PKV_OK : fail_cuda(e, "beam candidates launch");
}

int pkv_beam_step(const pkv_beam_step_desc* d, void* stream) {
    const char* fn = "pkv_beam_step";
    if (!d) return fail(PKV_ERR_INVALID_ARG, "%s: null descriptor", fn);
    if (d->struct_bytes != sizeof(pkv_beam_step_desc))
        return fail(PKV_ERR_INVALID_ARG, "pkv_beam_step_desc.struct_bytes=%u, library expects %zu (ABI mismatch)", d->struct_bytes, sizeof(pkv_beam_step_desc));
    const int k = d->num_beams;
    if (d->num_prompts < 1 || d->num_prompts > (1 << 16)) return fail(PKV_ERR_INVALID_ARG, "%s: num_prompts=%d outside [1, 65536]", fn, d->num_prompts);
    if (k < 2 || k > kMaxBeams) return fail(PKV_ERR_INVALID_ARG, "%s: num_beams=%d outside [2, %d]", fn, k, kMaxBeams);
    if (d->n_eos < 0 || d->n_eos > 4) return fail(PKV_ERR_INVALID_ARG, "%s: n_eos=%d outside [0, 4]", fn, d->n_eos);
    const int n_eos = d->n_eos;
    if (d->top_k != (n_eos + 1 > 2 ? n_eos + 1 : 2) * k) return fail(PKV_ERR_INVALID_ARG, "%s: top_k=%d is not max(2, 1 + n_eos) * num_beams", fn, d->top_k);
    if (d->cand_rows_per_prompt != 1 && d->cand_rows_per_prompt != k) return fail(PKV_ERR_INVALID_ARG, "%s: cand_rows_per_prompt must be 1 or num_beams", fn);
    if (d->early_stopping < 0 || d->early_stopping > 2) return fail(PKV_ERR_INVALID_ARG, "%s: early_stopping=%d outside [0, 2]", fn, d->early_stopping);
    if (d->max_steps < 1) return fail(PKV_ERR_INVALID_ARG, "%s: max_steps=%d < 1", fn, d->max_steps);
    auto bad = [](const void* p, uintptr_t align) { return !p || (reinterpret_cast<uintptr_t>(p) & (align - 1)); };
    if (bad(d->step, 4) || bad(d->cand_lp, 4) || bad(d->cand_id, 4) || (n_eos && bad(d->eos, 4)) || bad(d->scale, 4) ||
        bad(d->running, 4) || bad(d->pool_score, 4) || bad(d->pool_step, 4) || bad(d->pool_parent, 4) || bad(d->pool_token, 4) ||
        bad(d->pool_done, 1) || bad(d->heuristic, 1) || bad(d->done, 1) || bad(d->bp_token, 4) || bad(d->bp_parent, 4) ||
        bad(d->cp, 4) || bad(d->next_token, 8) || bad(d->parent, 4) || bad(d->diverge, 4))
        return fail(PKV_ERR_INVALID_ARG, "%s: null or misaligned pointer", fn);
    const DevInfo* di = nullptr;
    int rc = device_info(d->device, &di);
    if (rc) return rc;
    BeamStepArgs a;
    a.P = d->num_prompts; a.k = k; a.K = d->top_k; a.rows_per_prompt = d->cand_rows_per_prompt; a.n_eos = n_eos;
    a.early_stopping = d->early_stopping; a.max_steps = d->max_steps; a.step_offset = d->step_offset; a.step = d->step;
    a.cand_lp = d->cand_lp; a.cand_id = d->cand_id; a.eos = d->eos; a.scale = d->scale; a.running = d->running;
    a.pool_score = d->pool_score; a.pool_step = d->pool_step; a.pool_parent = d->pool_parent; a.pool_token = d->pool_token;
    a.pool_done = d->pool_done; a.heur = d->heuristic; a.done = d->done; a.bp_token = d->bp_token; a.bp_parent = d->bp_parent;
    a.cp = d->cp; a.next_token = d->next_token; a.parent = d->parent; a.diverge = d->diverge;
    DeviceGuard guard(d->device);
    const cudaError_t e = launch_beam_step(a, static_cast<cudaStream_t>(stream));
    return e == cudaSuccess ? PKV_OK : fail_cuda(e, "beam step launch");
}

int pkv_cache_reorder(int32_t num_prompts, int32_t num_beams, int32_t num_heads, int32_t row_bytes, int32_t device,
                      int32_t num_layers, int32_t window, int32_t heavy, void* const* planes, const int64_t* capacity,
                      const int32_t* const* base, float* const* heavy_scores, int32_t* const* heavy_gen,
                      int32_t* const* victim, const int32_t* parent, const int32_t* diverge, const int32_t* step,
                      int32_t step_offset, void* stream) {
    const char* fn = "pkv_cache_reorder";
    if (num_beams < 2 || num_beams > kMaxBeams) return fail(PKV_ERR_INVALID_ARG, "%s: num_beams=%d outside [2, %d]", fn, num_beams, kMaxBeams);
    if (num_prompts < 1 || num_heads < 1 || num_heads > 4096 || num_layers < 1 || int64_t(num_prompts) * num_heads > (1 << 24))
        return fail(PKV_ERR_INVALID_ARG, "%s: need num_prompts >= 1, 1 <= num_heads <= 4096, num_layers >= 1", fn);
    if (row_bytes < 16 || row_bytes > 256 || row_bytes % 16) return fail(PKV_ERR_INVALID_ARG, "%s: row_bytes=%d: a multiple of 16 in [16, 256]", fn, row_bytes);
    if (window < 0 || (heavy && window == 0)) return fail(PKV_ERR_INVALID_ARG, "%s: window=%d, heavy=%d", fn, window, heavy);
    auto bad = [](const void* p, uintptr_t align) { return !p || (reinterpret_cast<uintptr_t>(p) & (align - 1)); };
    if (!planes || !capacity || !base || bad(parent, 4) || bad(diverge, 4) || bad(step, 4))
        return fail(PKV_ERR_INVALID_ARG, "%s: null or misaligned table", fn);
    const bool scaled = planes[2] != nullptr;
    for (int l = 0; l < num_layers; ++l) {
        if (bad(planes[4 * l], 16) || bad(planes[4 * l + 1], 16) || bad(base[l], 4) || capacity[l] < 1)
            return fail(PKV_ERR_INVALID_ARG, "%s: layer %d: null or misaligned rows or row table", fn, l);
        if (scaled != (planes[4 * l + 2] != nullptr) || (scaled && (bad(planes[4 * l + 2], 4) || bad(planes[4 * l + 3], 4))))
            return fail(PKV_ERR_INVALID_ARG, "%s: layer %d: scales must be given for every layer or none", fn, l);
        if (heavy && (!heavy_scores || !heavy_gen || !victim || bad(heavy_scores[l], 4) || bad(heavy_gen[l], 4) || bad(victim[l], 4)))
            return fail(PKV_ERR_INVALID_ARG, "%s: layer %d: null or misaligned heavy-hitter state", fn, l);
    }
    const DevInfo* di = nullptr;
    int rc = device_info(device, &di);
    if (rc) return rc;
    DeviceGuard guard(device);
    for (int l0 = 0; l0 < num_layers; l0 += kMaxLayerBatch) {
        ReorderArgs a;
        a.P = num_prompts; a.k = num_beams; a.H = num_heads; a.row_bytes = row_bytes; a.window = window; a.heavy = heavy != 0;
        a.n_layers = std::min(kMaxLayerBatch, num_layers - l0); a.step_offset = step_offset;
        a.parent = parent; a.diverge = diverge; a.step = step;
        for (int i = 0; i < a.n_layers; ++i) {
            const int l = l0 + i;
            ReorderLayer& q = a.layer[i];
            for (int j = 0; j < 4; ++j) q.plane[j] = planes[4 * l + j];
            q.cap = capacity[l];
            q.base = base[l];
            q.heavy_scores = heavy ? heavy_scores[l] : nullptr;
            q.heavy_gen = heavy ? heavy_gen[l] : nullptr;
            q.victim = heavy ? victim[l] : nullptr;
        }
        const cudaError_t e = launch_cache_reorder(a, static_cast<cudaStream_t>(stream));
        if (e != cudaSuccess) return fail_cuda(e, "cache reorder launch");
    }
    return PKV_OK;
}

// pkv_decode_attn_multi (pk NULL) and pkv_decode_attn_packed: one launch of the verify kernel.
static int decode_multi_run(const char* fn, const pkv_decode_desc* d, const pkv_decode_multi* m, const pkv_decode_packed* pk,
                            void* stream) {
    if (!d || !m) return fail(PKV_ERR_INVALID_ARG, "%s: null descriptor", fn);
    if (d->struct_bytes != sizeof(pkv_decode_desc) || m->struct_bytes != sizeof(pkv_decode_multi))
        return fail(PKV_ERR_INVALID_ARG, "%s: struct_bytes mismatch (ABI)", fn);
    if (d->dtype != PKV_BF16 && d->dtype != PKV_FP16) return fail(PKV_ERR_UNSUPPORTED_DTYPE, "%s: dtype %d", fn, d->dtype);
    if (d->num_q_heads <= 0 || d->num_kv_heads <= 0 || d->num_q_heads % d->num_kv_heads) return fail(PKV_ERR_INVALID_ARG, "%s: bad head counts", fn);
    if (d->head_dim != 64 && d->head_dim != 128) return fail(PKV_ERR_UNSUPPORTED, "%s: head_dim=%d: only 64 and 128 are built", fn, d->head_dim);
    const int Q = m->num_queries, G = d->num_q_heads / d->num_kv_heads;
    if (Q < 1 || Q > PKV_MAX_SPEC_QUERIES) return fail(PKV_ERR_INVALID_ARG, "%s: num_queries=%d outside [1, %d]", fn, Q, PKV_MAX_SPEC_QUERIES);
    if (m->num_seqs < 1 || m->num_seqs > 65535) return fail(PKV_ERR_INVALID_ARG, "%s: num_seqs=%d outside [1, 65535]", fn, m->num_seqs);
    if (m->gqa_shared && G != 2 && G != 4 && G != 8)
        return fail(PKV_ERR_UNSUPPORTED, "%s: group size %d: the grouped form is built for 2, 4 and 8", fn, G);
    const bool e4m3 = m->k_scale != nullptr;
    if (e4m3 != (m->v_scale != nullptr)) return fail(PKV_ERR_INVALID_ARG, "%s: k_scale and v_scale go together", fn);
    const int heads = m->gqa_shared ? d->num_kv_heads : d->num_q_heads;
    const int64_t align = e4m3 ? 16 : 8;
    if (d->length < 0 || m->max_length < Q || d->cache_stride_h < m->max_length * d->head_dim || d->cache_stride_h % align ||
        (m->num_seqs > 1 && (m->cache_stride_b < heads * d->cache_stride_h || m->cache_stride_b % align)))
        return fail(PKV_ERR_INVALID_ARG, "%s: length, max_length or cache strides out of range (cache capacity exceeded)", fn);
    if (e4m3 && (m->scale_stride_h < m->max_length || (m->num_seqs > 1 && m->scale_stride_b < heads * m->scale_stride_h)))
        return fail(PKV_ERR_INVALID_ARG, "%s: scale strides hold fewer than max_length rows", fn);
    if (m->q_stride_t % 8 || m->q_stride_h % 8 || m->kv_stride_t % 8 || m->kv_stride_h % 8 || m->out_stride_t < 0 || m->out_stride_h < 0)
        return fail(PKV_ERR_INVALID_ARG, "%s: token / head strides must be multiples of 8 elements", fn);
    if (!d->q || !d->out || !d->k_new || !d->v_new || !d->k_cache || !d->v_cache || !aligned16(d->q) || !aligned16(d->k_new) ||
        !aligned16(d->v_new) || !aligned16(d->k_cache) || !aligned16(d->v_cache) || (reinterpret_cast<uintptr_t>(d->out) & 1u) ||
        (reinterpret_cast<uintptr_t>(m->rows) & 3u) || (reinterpret_cast<uintptr_t>(m->step_dev) & 3u) ||
        (e4m3 && ((reinterpret_cast<uintptr_t>(m->k_scale) & 3u) || (reinterpret_cast<uintptr_t>(m->v_scale) & 3u))))
        return fail(PKV_ERR_INVALID_ARG, "%s: null or misaligned pointer", fn);
    const DevInfo* di = nullptr;
    int rc = device_info(d->device, &di);
    if (rc) return rc;
    MultiArgs a;
    a.dtype = d->dtype; a.Hq = d->num_q_heads; a.Hkv = d->num_kv_heads; a.G = G; a.D = d->head_dim; a.Q = Q;
    a.num_seqs = m->num_seqs; a.heads_per_cache = m->gqa_shared ? G : 1; a.num_sms = di->sms;
    a.nsplit = decode_num_splits(a.Hq, m->max_length, a.num_sms);
    a.q = static_cast<const uint16_t*>(d->q); a.k_new = static_cast<const uint16_t*>(d->k_new);
    a.v_new = static_cast<const uint16_t*>(d->v_new); a.out = static_cast<uint16_t*>(d->out);
    a.q_st = m->q_stride_t; a.q_sh = m->q_stride_h; a.kv_st = m->kv_stride_t; a.kv_sh = m->kv_stride_h;
    a.out_st = m->out_stride_t; a.out_sh = m->out_stride_h;
    a.k_cache = d->k_cache; a.v_cache = d->v_cache; a.cache_sh = d->cache_stride_h;
    a.cache_sb = m->num_seqs > 1 ? m->cache_stride_b : heads * d->cache_stride_h;
    a.k_scale = m->k_scale; a.v_scale = m->v_scale; a.scale_sh = m->scale_stride_h;
    a.scale_sb = m->num_seqs > 1 ? m->scale_stride_b : heads * m->scale_stride_h;
    a.T = d->length; a.max_rows = m->max_length; a.step_dev = m->step_dev; a.rows = m->rows;
    a.scale = d->softmax_scale != 0.f ? d->softmax_scale : 1.0f / sqrtf(float(d->head_dim));
    a.ws = static_cast<float*>(d->workspace);
    a.row_start = pk ? pk->row_start : nullptr;
    a.row_count = pk ? pk->row_count : nullptr;
    a.M = pk ? pk->total_rows : int64_t(m->num_seqs) * Q;
    if (a.nsplit > 1) {
        const uint64_t need = uint64_t(a.num_seqs) * a.Hq * Q * a.nsplit * (2 + a.D) * sizeof(float);
        if (!d->workspace || d->workspace_bytes < need || (reinterpret_cast<uintptr_t>(d->workspace) & 15u))
            return fail(PKV_ERR_WORKSPACE, "%s: workspace of %llu bytes required", fn, (unsigned long long)need);
    }
    DeviceGuard guard(d->device);
    const cudaError_t e = launch_decode_multi(a, static_cast<cudaStream_t>(stream));
    return e == cudaSuccess ? PKV_OK : fail_cuda(e, fn);
}

int pkv_decode_attn_multi(const pkv_decode_desc* d, const pkv_decode_multi* m, void* stream) {
    return decode_multi_run("pkv_decode_attn_multi", d, m, nullptr, stream);
}

int pkv_decode_attn_packed(const pkv_decode_desc* d, const pkv_decode_multi* m, const pkv_decode_packed* p, void* stream) {
    const char* fn = "pkv_decode_attn_packed";
    if (!p) return fail(PKV_ERR_INVALID_ARG, "%s: null descriptor", fn);
    if (p->struct_bytes != sizeof(pkv_decode_packed)) return fail(PKV_ERR_INVALID_ARG, "%s: struct_bytes mismatch (ABI)", fn);
    if (p->total_rows < 1) return fail(PKV_ERR_INVALID_ARG, "%s: total_rows=%d below 1", fn, p->total_rows);
    if (!p->row_start || !p->row_count || (reinterpret_cast<uintptr_t>(p->row_start) & 3u) ||
        (reinterpret_cast<uintptr_t>(p->row_count) & 3u))
        return fail(PKV_ERR_INVALID_ARG, "%s: null or misaligned row_start / row_count", fn);
    return decode_multi_run(fn, d, m, p, stream);
}

static int spec_args(const char* fn, const pkv_spec_desc* d, bool step, SpecArgs* a) {
    if (!d) return fail(PKV_ERR_INVALID_ARG, "%s: null descriptor", fn);
    if (d->struct_bytes != sizeof(pkv_spec_desc))
        return fail(PKV_ERR_INVALID_ARG, "pkv_spec_desc.struct_bytes=%u, library expects %zu (ABI mismatch)", d->struct_bytes, sizeof(pkv_spec_desc));
    if (d->num_seqs < 1 || d->num_seqs > 65535) return fail(PKV_ERR_INVALID_ARG, "%s: num_seqs=%d outside [1, 65535]", fn, d->num_seqs);
    if (d->num_queries < 2 || d->num_queries > PKV_MAX_SPEC_QUERIES) return fail(PKV_ERR_INVALID_ARG, "%s: num_queries=%d outside [2, 16]", fn, d->num_queries);
    if (d->max_ngram < 1 || d->max_ngram > PKV_MAX_NGRAM) return fail(PKV_ERR_INVALID_ARG, "%s: max_ngram=%d outside [1, 8]", fn, d->max_ngram);
    if (d->n_eos < 0 || d->n_eos > 4) return fail(PKV_ERR_INVALID_ARG, "%s: n_eos=%d outside [0, 4]", fn, d->n_eos);
    if (d->hist_cap < 1 || d->hist_cap > INT32_MAX || d->out_cap < 1) return fail(PKV_ERR_INVALID_ARG, "%s: hist_cap / out_cap out of range", fn);
    auto bad = [](const void* p, uintptr_t align) { return !p || (reinterpret_cast<uintptr_t>(p) & (align - 1)); };
    if (bad(d->hist, 8) || bad(d->hist_len, 4) || bad(d->budget, 4) || bad(d->done, 1) || bad(d->out, 8) || bad(d->out_len, 4) ||
        bad(d->ids, 8) || bad(d->pos, 8) || bad(d->draft_len, 4) || bad(d->emitted, 4) || (d->n_eos && bad(d->eos, 8)) ||
        (step && bad(d->tokens, 8)))
        return fail(PKV_ERR_INVALID_ARG, "%s: null or misaligned pointer", fn);
    if (step && (d->num_layers < 0 || (d->num_layers > 0 && (!d->rows || d->num_heads < 1))))
        return fail(PKV_ERR_INVALID_ARG, "%s: num_layers / num_heads / rows table", fn);
    for (int l = 0; step && l < d->num_layers; ++l)
        if (bad(d->rows[l], 4)) return fail(PKV_ERR_INVALID_ARG, "%s: layer %d: null or misaligned row counts", fn, l);
    const DevInfo* di = nullptr;
    int rc = device_info(d->device, &di);
    if (rc) return rc;
    a->num_seqs = d->num_seqs; a->Q = d->num_queries; a->N = d->max_ngram; a->n_eos = d->n_eos; a->n_layers = 0; a->H = d->num_heads;
    a->hist_cap = d->hist_cap; a->out_cap = d->out_cap; a->pad = d->pad_token_id;
    a->hist = d->hist; a->hist_len = d->hist_len; a->budget = d->budget; a->done = d->done; a->out = d->out; a->out_len = d->out_len;
    a->ids = d->ids; a->pos = d->pos; a->draft_len = d->draft_len; a->emitted = d->emitted; a->tokens = d->tokens; a->eos = d->eos;
    return PKV_OK;
}

int pkv_prompt_lookup(const pkv_spec_desc* d, void* stream) {
    SpecArgs a;
    int rc = spec_args("pkv_prompt_lookup", d, false, &a);
    if (rc) return rc;
    DeviceGuard guard(d->device);
    const cudaError_t e = launch_prompt_lookup(a, static_cast<cudaStream_t>(stream));
    return e == cudaSuccess ? PKV_OK : fail_cuda(e, "prompt lookup launch");
}

int pkv_spec_pack(const pkv_spec_desc* d, const pkv_spec_pack_desc* k, void* stream) {
    const char* fn = "pkv_spec_pack";
    SpecArgs a;
    int rc = spec_args(fn, d, false, &a);
    if (rc) return rc;
    if (!k) return fail(PKV_ERR_INVALID_ARG, "%s: null descriptor", fn);
    if (k->struct_bytes != sizeof(pkv_spec_pack_desc))
        return fail(PKV_ERR_INVALID_ARG, "pkv_spec_pack_desc.struct_bytes=%u, library expects %zu (ABI mismatch)", k->struct_bytes, sizeof(pkv_spec_pack_desc));
    const int64_t most = int64_t(d->num_seqs) * (d->num_queries - 1);
    if (k->max_draft_tokens < 1 || k->max_draft_tokens > most)
        return fail(PKV_ERR_INVALID_ARG, "%s: max_draft_tokens=%d outside [1, %lld]", fn, k->max_draft_tokens, (long long)most);
    if (int64_t(k->total_rows) < int64_t(d->num_seqs) + k->max_draft_tokens)
        return fail(PKV_ERR_INVALID_ARG, "%s: total_rows=%d below num_seqs + max_draft_tokens", fn, k->total_rows);
    auto bad = [](const void* p, uintptr_t align) { return !p || (reinterpret_cast<uintptr_t>(p) & (align - 1)); };
    if (bad(k->step, 4) || bad(k->ids, 8) || bad(k->pos, 8) || bad(k->row_start, 4) || bad(k->row_count, 4) ||
        (k->totals && bad(k->totals, 8)))
        return fail(PKV_ERR_INVALID_ARG, "%s: null or misaligned pointer", fn);
    PackArgs p;
    p.D = k->max_draft_tokens; p.M = k->total_rows; p.step = k->step; p.ids = k->ids; p.pos = k->pos;
    p.row_start = k->row_start; p.row_count = k->row_count; p.totals = k->totals;
    DeviceGuard guard(d->device);
    const cudaError_t e = launch_spec_pack(a, p, static_cast<cudaStream_t>(stream));
    return e == cudaSuccess ? PKV_OK : fail_cuda(e, "spec pack launch");
}

int pkv_spec_step(const pkv_spec_desc* d, void* stream) {
    SpecArgs a;
    int rc = spec_args("pkv_spec_step", d, true, &a);
    if (rc) return rc;
    DeviceGuard guard(d->device);
    int l0 = 0;
    do {   // the step with the first 32 layers, then the row counts of the next 32 per launch
        a.n_layers = std::min(kMaxLayerBatch, d->num_layers - l0);
        for (int i = 0; i < a.n_layers; ++i) a.rows[i] = d->rows[l0 + i];
        const cudaError_t e = launch_spec_step(a, l0 == 0, static_cast<cudaStream_t>(stream));
        if (e != cudaSuccess) return fail_cuda(e, "spec step launch");
        l0 += kMaxLayerBatch;
    } while (l0 < d->num_layers);
    return PKV_OK;
}

}  // extern "C"
