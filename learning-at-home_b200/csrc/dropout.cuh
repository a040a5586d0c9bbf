// dropout.cuh — the one definition of the transformer expert's dropout masks (counter-based Philox4x32-10).
//
// A keep decision is a pure function of (seed, site, position): no state, no dependence on tiling, launch shape or thread
// layout.  One Philox call returns 128 bits = eight 16-bit lanes and decides a GRANULE of 8 elements; an element is kept iff
// its lane u16 >= thr, with thr = min(65535, round(p * 65536)) (ops/kernels.py::dropout_threshold), so the realised drop
// probability is thr / 65536 (within 2^-17 of p; p = 0.1 -> 6554 / 65536 = 0.1000061).  Kept values are scaled by 1 / (1 - p).
//
//   site 0 (attention probabilities), position (batch, head, query q, key k), q, k < MAX_SEQ:
//     a 16-element block {a, a+1, a+8, a+9} x {b, b+1, b+8, b+9} (a, b even, a % 16 < 8, b % 16 < 8) is split by query parity
//     into two granules of {q, q+8} x {b, b+1, b+8, b+9}.  Forward threads hold rows {g, g+8} x key pairs {2c, 2c+1} of every
//     8-key group, so one call covers 8 of their elements; backward threads hold the transpose and use half of two calls.
//       counter = ((gq & 127) * 128 + (gk & 127) | (q & 1) << 14, head, batch, (gq >> 7) << 8 | (gk >> 7) << 20)
//                 gq = (q >> 4) * 4 + ((q >> 1) & 3), same for gk
//       lane    = ((q >> 3) & 1) * 4 + ((k & 1) | ((k >> 3) & 1) << 1)
//     For q, k < 512 the last word is 0 (the layout of the 512-token kernels, so their masks are unchanged); its low byte is
//     always 0 (= SITE_ATTN), which keeps site 0 apart from sites 1-3.  The 12-bit fields hold gq >> 7 and gk >> 7 up to
//     4095, i.e. q, k < 2^21; MAX_SEQ stays far below, so a whole S x S plane is indexed in 32 bits.
//   sites 1-3 (dropout1, dropout, dropout2), position (token row r, column n): granule {r, r+8} x {b, b+1, b+8, b+9}, which is
//     exactly what a thread of a wgmma accumulator holds for two adjacent 8-column groups.
//       counter = (gn, gr, 0, site), gr = (r >> 4) * 8 + (r & 7), gn = (n >> 4) * 4 + ((n >> 1) & 3)
//       lane    = ((r >> 3) & 1) * 4 + ((n & 1) | ((n >> 3) & 1) << 1)
//   key = (seed & 0xffffffff, seed >> 32)
//
// ops/kernels.py::dropout_keep_ref is an independent CPU implementation of the same definition.
#pragma once

#include <stdint.h>

namespace lah {
namespace drop {

constexpr int SITE_ATTN = 0;
constexpr int MAX_SEQ = 65536;   // longest attention sequence (csrc/attention.cu, attention_bwd.cu)

__host__ __device__ __forceinline__ uint4 philox4x32_10(uint4 c, uint32_t k0, uint32_t k1) {
    constexpr uint32_t M0 = 0xD2511F53u, M1 = 0xCD9E8D57u, W0 = 0x9E3779B9u, W1 = 0xBB67AE85u;
#pragma unroll
    for (int r = 0; r < 10; ++r) {
#ifdef __CUDA_ARCH__
        const uint32_t hi0 = __umulhi(M0, c.x), hi1 = __umulhi(M1, c.z);
#else
        const uint32_t hi0 = static_cast<uint32_t>((static_cast<uint64_t>(M0) * c.x) >> 32);
        const uint32_t hi1 = static_cast<uint32_t>((static_cast<uint64_t>(M1) * c.z) >> 32);
#endif
        const uint32_t lo0 = M0 * c.x, lo1 = M1 * c.z;
        c = make_uint4(hi1 ^ c.y ^ k0, lo1, hi0 ^ c.w ^ k1, lo0);
        k0 += W0;
        k1 += W1;
    }
    return c;
}

// the 8 decisions of one attention granule: gq / gk are the granule coordinates of (q, k), parity = q & 1
__device__ __forceinline__ uint4 attn_bits(unsigned long long seed, int batch, int head, uint32_t gq, uint32_t gk,
                                           uint32_t parity) {
    return philox4x32_10(make_uint4(((gq & 127u) * 128u + (gk & 127u)) | (parity << 14), static_cast<uint32_t>(head),
                                    static_cast<uint32_t>(batch), SITE_ATTN | (gq >> 7) << 8 | (gk >> 7) << 20),
                         static_cast<uint32_t>(seed), static_cast<uint32_t>(seed >> 32));
}

// the 8 decisions of one (row, column) granule of sites 1-3
__device__ __forceinline__ uint4 rc_bits(unsigned long long seed, int site, uint32_t gr, uint32_t gn) {
    return philox4x32_10(make_uint4(gn, gr, 0u, static_cast<uint32_t>(site)), static_cast<uint32_t>(seed),
                         static_cast<uint32_t>(seed >> 32));
}

__device__ __forceinline__ uint32_t granule_row(uint32_t r) { return (r >> 4) * 8u + (r & 7u); }
__device__ __forceinline__ uint32_t granule_col(uint32_t n) { return (n >> 4) * 4u + ((n >> 1) & 3u); }
__device__ __forceinline__ uint32_t granule_attn(uint32_t q) { return (q >> 4) * 4u + ((q >> 1) & 3u); }

// keep decision of lane e (0..7) of a granule
__device__ __forceinline__ bool keep(uint4 bits, int e, uint32_t thr) {
    const uint32_t w = (e >> 1) == 0 ? bits.x : (e >> 1) == 1 ? bits.y : (e >> 1) == 2 ? bits.z : bits.w;
    return ((e & 1) ? (w >> 16) : (w & 0xffffu)) >= thr;
}

// single-element forms (mask materialisation, elementwise kernels)
__device__ __forceinline__ bool keep_attn(unsigned long long seed, int batch, int head, uint32_t q, uint32_t k, uint32_t thr) {
    const uint4 b = attn_bits(seed, batch, head, granule_attn(q), granule_attn(k), q & 1u);
    return keep(b, static_cast<int>(((q >> 3) & 1u) * 4u + ((k & 1u) | ((k >> 3) & 1u) << 1)), thr);
}
__device__ __forceinline__ bool keep_rc(unsigned long long seed, int site, uint32_t r, uint32_t n, uint32_t thr) {
    const uint4 b = rc_bits(seed, site, granule_row(r), granule_col(n));
    return keep(b, static_cast<int>(((r >> 3) & 1u) * 4u + ((n & 1u) | ((n >> 3) & 1u) << 1)), thr);
}

}  // namespace drop
}  // namespace lah
