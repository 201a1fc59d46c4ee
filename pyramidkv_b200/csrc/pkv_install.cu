// pkv_install.cu — admission of one prompt into one slot of a batched compacted cache (continuous batching): every layer's
// K / V rows (FP8: and their scales) are copied from the prompt's single-sequence buffers into slot `slot` of the batched
// buffers, and the slot's row counts are set relative to the device step counter, all in one launch per 32 layers. Parking
// a slot is the same launch with zero rows.
#include <algorithm>

#include "pkv_common.cuh"
#include "pkv_internal.h"

namespace pkv {
namespace {

constexpr int kThreads = 256;

// grid (x: chunks of one head's rows, y: layer, z: K / V x head). A (layer, K or V, head)'s n rows are contiguous in the
// source and in the destination slot, so the copy is a flat run of 16-byte vectors; rows past n are neither read nor written.
template <int VPR>   // 16-byte vectors per row
__global__ void __launch_bounds__(kThreads) install_kernel(const __grid_constant__ InstallArgs a) {
    const InstallLayer& L = a.layer[blockIdx.y];
    const int kv = int(blockIdx.z) / a.H, h = int(blockIdx.z) - kv * a.H;
    int64_t n = L.rows;
    if (L.rows_dev) n = min(n, int64_t(__ldg(L.rows_dev + h)));
    const int64_t sh = int64_t(a.slot) * a.H + h;
    // the decode kernels attend 1 + *step_dev + rows[sh] rows: the next step appends row n and attends n + 1
    if (blockIdx.x == 0 && kv == 0 && threadIdx.x == 0) L.dst_rows[sh] = int32_t(n - int64_t(*a.step_dev));
    if (n <= 0) return;
    const uint4* src = reinterpret_cast<const uint4*>(L.src[kv]) + int64_t(h) * L.src_cap * VPR;
    uint4* dst = reinterpret_cast<uint4*>(L.dst[kv]) + sh * L.dst_cap * VPR;
    const int64_t first = int64_t(blockIdx.x) * kThreads + threadIdx.x, stride = int64_t(gridDim.x) * kThreads;
    for (int64_t i = first; i < n * VPR; i += stride) dst[i] = ldg_nc_v4(src + i);
    if (L.src_scale[kv]) {
        const float* ss = L.src_scale[kv] + int64_t(h) * L.src_cap;
        float* ds = L.dst_scale[kv] + sh * L.dst_cap;
        for (int64_t r = first; r < n; r += stride) ds[r] = __ldg(ss + r);
    }
}

template <int VPR>
cudaError_t launch_install_t(const InstallArgs& a, int num_sms, cudaStream_t st) {
    int64_t most = 0;
    for (int l = 0; l < a.n_layers; ++l) most = std::max(most, a.layer[l].rows * VPR);
    const int64_t heads = int64_t(a.n_layers) * 2 * a.H;
    int64_t gx = (most + kThreads - 1) / kThreads;
    gx = std::max<int64_t>(1, std::min(gx, std::max<int64_t>(1, int64_t(num_sms) * 16 / heads)));   // grid-stride beyond ~16 CTAs per SM
    install_kernel<VPR><<<dim3(unsigned(gx), unsigned(a.n_layers), unsigned(2 * a.H)), kThreads, 0, st>>>(a);
    count_launch();
    return cudaGetLastError();
}

}  // namespace

cudaError_t launch_install(const InstallArgs& a, int row_bytes, int num_sms, cudaStream_t st) {
    switch (row_bytes) {
        case 64: return launch_install_t<4>(a, num_sms, st);
        case 128: return launch_install_t<8>(a, num_sms, st);
        default: return launch_install_t<16>(a, num_sms, st);
    }
}

}  // namespace pkv
