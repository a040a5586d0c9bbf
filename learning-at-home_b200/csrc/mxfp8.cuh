// mxfp8.cuh — the MXFP8 operand rules shared by every kernel that emits an operand of the block-scaled FP8 GEMM
// (csrc/grouped_gemm_fp8.cu): the UE8M0 scale of a 32-element block, the E4M3 conversion, and the byte of a scale in the
// activation layout (tile_rows = 128, one group; the layout itself is described in grouped_gemm_fp8.cu).
#pragma once
#include "sm90.cuh"
#include <cuda_fp8.h>

namespace lah {

// smallest power of two s with amax / s <= 448 (the E4M3 maximum), as a biased exponent clamped to [1, 253]: no element
// saturates, and 2^(127 - e) (the reciprocal applied before the conversion) stays a normal fp32 number
__device__ __forceinline__ uint32_t e8m0_from_amax(float amax) {
    const float s = amax * (1.f / 448.f);
    uint32_t bits = __float_as_uint(s);
    uint32_t e = (bits >> 23) & 0xFFu;
    if (bits & 0x7FFFFFu) e += 1;
    return min(max(e, 1u), 253u);
}

// 2^(127 - e): the exact reciprocal of the block scale 2^(e - 127)
__device__ __forceinline__ float e8m0_inv(uint32_t e) { return __uint_as_float((254u - e) << 23); }

// eight values times inv, rounded to E4M3 (nearest even, saturating), packed little-endian into two words
__device__ __forceinline__ uint2 e4m3x8(const float (&y)[8], float inv) {
    uint2 o;
    o.x = static_cast<uint32_t>(__nv_cvt_float2_to_fp8x2(make_float2(y[0] * inv, y[1] * inv), __NV_SATFINITE, __NV_E4M3)) |
          (static_cast<uint32_t>(__nv_cvt_float2_to_fp8x2(make_float2(y[2] * inv, y[3] * inv), __NV_SATFINITE, __NV_E4M3)) << 16);
    o.y = static_cast<uint32_t>(__nv_cvt_float2_to_fp8x2(make_float2(y[4] * inv, y[5] * inv), __NV_SATFINITE, __NV_E4M3)) |
          (static_cast<uint32_t>(__nv_cvt_float2_to_fp8x2(make_float2(y[6] * inv, y[7] * inv), __NV_SATFINITE, __NV_E4M3)) << 16);
    return o;
}

// byte offset of the scale of (row, 32-column block kb32) of a [rows, K] activation operand
__device__ __forceinline__ long long act_sf_byte(long long row, int K, int kb32) {
    const int ra = static_cast<int>(row & 127);
    const long long chunk = (row >> 7) * (K / 128) + (kb32 >> 2);
    return chunk * 512 + ((ra & 31) * 4 + (ra >> 5)) * 4 + (kb32 & 3);
}

// Quantise the 8 values a lane holds of a 32-column block that 4 adjacent lanes (a quad: lanes 4i .. 4i + 3, in column
// order) share: the quad's amax in two shuffles over `mask` (which must include the whole quad), then the lane's 8 payload
// bytes and the block's scale byte (written by the quad's first lane)
__device__ __forceinline__ void quant_quad8(const float (&y)[8], unsigned mask, int lane, uint8_t* __restrict__ payload,
                                            uint8_t* __restrict__ sf_byte) {
    float amax = 0.f;
#pragma unroll
    for (int t = 0; t < 8; ++t) amax = fmaxf(amax, fabsf(y[t]));
    amax = fmaxf(amax, __shfl_xor_sync(mask, amax, 1));
    amax = fmaxf(amax, __shfl_xor_sync(mask, amax, 2));
    const uint32_t e = e8m0_from_amax(amax);
    const uint2 o8 = e4m3x8(y, e8m0_inv(e));
    asm volatile("st.global.v2.u32 [%0], {%1, %2};" ::"l"(payload), "r"(o8.x), "r"(o8.y) : "memory");
    if ((lane & 3) == 0) *sf_byte = static_cast<uint8_t>(e);
}

}  // namespace lah
