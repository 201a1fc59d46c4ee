// pkv_rows.cuh — per-lane pieces of a cached row: widening 16-bit and E4M3 elements to fp32, and the E4M3 row quantisation.
// Shared by the decode kernel (pkv_decode.cu) and the conversion of the 16-bit cache to E4M3 (pkv_fp8.cu).
//
// E4M3 row format: a row x of D 16-bit values is stored as
//     amax = max_e |x_e| (fp32);  amax == 0: scale = 0, every byte 0;
//     else inv = rn_f32(448 / amax), q_e = e4m3_satfinite_rne(rn_f32(x_e * inv)), scale = rn_f32(amax / 448)
// and stands for x^_e = float(q_e) * scale. Each row carries its own scale, so appending a row never touches another one.
#pragma once

#include <cuda_fp8.h>

#include "pkv_common.cuh"

namespace pkv {

constexpr float kE4M3Max = 448.f;

// eight 16-bit elements (one 128-bit load) -> fp32
template <typename T>
__device__ __forceinline__ void unpack8(const uint4& v, float* f) {
    const uint32_t u[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
    for (int e = 0; e < 4; ++e) {
        f[2 * e] = DT<T>::to_f32(uint16_t(u[e] & 0xffffu));
        f[2 * e + 1] = DT<T>::to_f32(uint16_t(u[e] >> 16));
    }
}

// 16 consecutive 16-bit elements (two 128-bit loads) -> fp32
template <typename T>
__device__ __forceinline__ void load16(const uint16_t* src, float (&x)[16]) {
    unpack8<T>(*reinterpret_cast<const uint4*>(src), x);
    unpack8<T>(*reinterpret_cast<const uint4*>(src + 8), x + 8);
}

// 16 E4M3 bytes (element e in byte e) -> fp32, exactly (cvt.rn.f16x2.e4m3x2, then f16 -> f32)
__device__ __forceinline__ void fp8x16_to_f32(const uint4& v, float (&f)[16]) {
    const uint32_t u[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
    for (int e = 0; e < 4; ++e) {
#pragma unroll
        for (int hlf = 0; hlf < 2; ++hlf) {
            const __half2 h2(__nv_cvt_fp8x2_to_halfraw2(__nv_fp8x2_storage_t(u[e] >> (16 * hlf)), __NV_E4M3));
            const float2 f2 = __half22float2(h2);
            f[4 * e + 2 * hlf] = f2.x;
            f[4 * e + 2 * hlf + 1] = f2.y;
        }
    }
}

// four fp32 -> four E4M3 bytes, first value in the low byte (cvt.rn.satfinite.e4m3x2.f32)
__device__ __forceinline__ uint32_t pack_fp8x4(float a, float b, float c, float d) {
    const uint32_t lo = __nv_cvt_float2_to_fp8x2(make_float2(a, b), __NV_SATFINITE, __NV_E4M3);
    const uint32_t hi = __nv_cvt_float2_to_fp8x2(make_float2(c, d), __NV_SATFINITE, __NV_E4M3);
    return lo | (hi << 16);
}

// largest |x| of a row spread over LPR consecutive lanes (every lane of the warp takes part)
template <int LPR>
__device__ __forceinline__ float row_amax(const float (&x)[16]) {
    float a = 0.f;
#pragma unroll
    for (int e = 0; e < 16; ++e) a = fmaxf(a, fabsf(x[e]));
#pragma unroll
    for (int o = 1; o < LPR; o <<= 1) a = fmaxf(a, __shfl_xor_sync(0xffffffffu, a, o));
    return a;
}

// this lane's 16 elements of a row whose amax is known -> E4M3 bytes; `scale` receives the row scale
__device__ __forceinline__ uint4 quantize16(const float (&x)[16], float amax, float& scale) {
    if (amax == 0.f) {
        scale = 0.f;
        return make_uint4(0, 0, 0, 0);
    }
    const float inv = __fdiv_rn(kE4M3Max, amax);
    uint32_t w[4];
#pragma unroll
    for (int e = 0; e < 4; ++e)
        w[e] = pack_fp8x4(__fmul_rn(x[4 * e], inv), __fmul_rn(x[4 * e + 1], inv), __fmul_rn(x[4 * e + 2], inv),
                          __fmul_rn(x[4 * e + 3], inv));
    scale = __fdiv_rn(amax, kE4M3Max);
    return make_uint4(w[0], w[1], w[2], w[3]);
}

}  // namespace pkv
