// dropout.cu — elementwise dropout kernels of the transformer expert and the mask materialiser (masks: dropout.cuh).
//
//   op 0  out = M o x / (1 - p)                            backward of dropout1 / dropout2 (the branch side of the residual)
//   op 1  out = M o gelu(x) / (1 - p)                      forward of linear1's activation + dropout
//   op 2  out = gelu'(f) o M o x / (1 - p)   (x = dg)      backward of the same
//   op 3  out = M o relu(x) / (1 - p)                      the same pair for a ReLU activation
//   op 4  out = [f > 0] o M o x / (1 - p)    (x = dg)
//
// One thread owns one mask granule ({r, r+8} x {b, b+1, b+8, b+9}): one Philox call, eight elements, 4-byte accesses that a
// quad of threads turns into 32 contiguous bytes per row.  GELU is the erf form, as nn.GELU().
//
// The gated activation of GatedFeedforwardBlock lives here too (no dropout): over the stacked pre-activation
// h = [g | u] ([rows, 2 inner], the output of the one GEMM over [W1; W3])
//   forward   a  = silu(g) o u
//   backward  dh = [da o u o s (1 + g (1 - s)) | da o silu(g)],  s = sigmoid(g)
// in fp32 with one bf16 rounding per output, 16-byte accesses (one thread per 8 columns of a row).
// swiglu_quant_kernel is the forward of the FP8 expert: it ALSO writes a as the MXFP8 operand of the W2 GEMM (E4M3 payload
// and scales in the activation layout, from the fp32 product before its bf16 rounding), and the bf16 a only when asked.
#include "mxfp8.cuh"
#include "sm90.cuh"
#include "dropout.cuh"

namespace lah {
namespace drop {

constexpr int OP_APPLY = 0, OP_GELU_FWD = 1, OP_GELU_BWD = 2, OP_RELU_FWD = 3, OP_RELU_BWD = 4;

__device__ __forceinline__ float gelu_f(float v) { return 0.5f * v * (1.f + erff(v * 0.70710678118654752f)); }
__device__ __forceinline__ float gelu_grad(float v) {
    return 0.5f * (1.f + erff(v * 0.70710678118654752f)) + v * 0.39894228040143268f * __expf(-0.5f * v * v);
}

template <int OP>
__global__ void __launch_bounds__(256) dropout_ew_kernel(const bf16* __restrict__ x, const bf16* __restrict__ f,
                                                         bf16* __restrict__ out, long long granules, int cols,
                                                         unsigned long long seed, int site, uint32_t thr, float scale) {
    const long long t = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (t >= granules) return;
    const int col_granules = cols >> 2;
    const uint32_t gr = static_cast<uint32_t>(t / col_granules), gn = static_cast<uint32_t>(t % col_granules);
    const uint4 bits = rc_bits(seed, site, gr, gn);
    const long long r0 = static_cast<long long>(gr >> 3) * 16 + (gr & 7);
    const int n0 = static_cast<int>(gn >> 2) * 16 + 2 * static_cast<int>(gn & 3);
#pragma unroll
    for (int h = 0; h < 2; ++h) {
#pragma unroll
        for (int jl = 0; jl < 2; ++jl) {
            const long long off = (r0 + 8 * h) * cols + n0 + 8 * jl;
            const float2 xv = unpack_bf16x2(__ldg(reinterpret_cast<const uint32_t*>(x + off)));
            float v[2] = {xv.x, xv.y};
            float fv[2] = {0.f, 0.f};
            if (OP == OP_GELU_BWD || OP == OP_RELU_BWD) {
                const float2 t2 = unpack_bf16x2(__ldg(reinterpret_cast<const uint32_t*>(f + off)));
                fv[0] = t2.x;
                fv[1] = t2.y;
            }
#pragma unroll
            for (int i = 0; i < 2; ++i) {
                const float s = keep(bits, h * 4 + jl * 2 + i, thr) ? scale : 0.f;
                if (OP == OP_APPLY) v[i] = v[i] * s;
                if (OP == OP_GELU_FWD) v[i] = gelu_f(v[i]) * s;
                if (OP == OP_GELU_BWD) v[i] = gelu_grad(fv[i]) * (v[i] * s);
                if (OP == OP_RELU_FWD) v[i] = v[i] > 0.f ? v[i] * s : 0.f;
                if (OP == OP_RELU_BWD) v[i] = fv[i] > 0.f ? v[i] * s : 0.f;
            }
            *reinterpret_cast<uint32_t*>(out + off) = pack_bf16x2(v[0], v[1]);
        }
    }
}

// mask[b, h, r, c] (uint8 0 / 1): site 0 -> keep_attn(b, h, query r, key c); sites 1-3 -> keep_rc(r, c) (b = h = 0)
__global__ void __launch_bounds__(256) dropout_mask_kernel(uint8_t* __restrict__ out, int site, int heads, int rows,
                                                           int cols, long long total, unsigned long long seed, uint32_t thr) {
    const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i >= total) return;
    const uint32_t c = static_cast<uint32_t>(i % cols);
    const long long br = i / cols;
    const uint32_t r = static_cast<uint32_t>(br % rows);
    const long long bh = br / rows;
    const bool k = site == SITE_ATTN ? keep_attn(seed, static_cast<int>(bh / heads), static_cast<int>(bh % heads), r, c, thr)
                                     : keep_rc(seed, site, r, c, thr);
    out[i] = k ? 1 : 0;
}

}  // namespace drop

// sigmoid that saturates to exactly 0 / 1 for large |g| (exp overflows to inf, 1 / inf = 0), so that no product below
// meets inf * 0
__device__ __forceinline__ float sigmoid_f(float g) { return 1.f / (1.f + __expf(-g)); }

__device__ __forceinline__ void unpack8(const int4& q, float (&f)[8]) {
    const uint32_t w[4] = {(uint32_t)q.x, (uint32_t)q.y, (uint32_t)q.z, (uint32_t)q.w};
#pragma unroll
    for (int t = 0; t < 4; ++t) {
        const float2 v = unpack_bf16x2(w[t]);
        f[2 * t] = v.x;
        f[2 * t + 1] = v.y;
    }
}

__device__ __forceinline__ int4 pack8(const float (&f)[8]) {
    return make_int4(pack_bf16x2(f[0], f[1]), pack_bf16x2(f[2], f[3]), pack_bf16x2(f[4], f[5]), pack_bf16x2(f[6], f[7]));
}

// thread t: row t / (inner / 8), columns 8 (t % (inner / 8)) .. + 7 of g, u, a / da and dg, du
template <bool BWD>
__global__ void __launch_bounds__(256) swiglu_kernel(const bf16* __restrict__ h, const bf16* __restrict__ da,
                                                     bf16* __restrict__ out, long long vecs, int inner) {
    const long long t = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (t >= vecs) return;
    const int per_row = inner >> 3;
    const long long row = t / per_row;
    const int col = static_cast<int>(t - row * per_row) * 8;
    const bf16* hr = h + row * 2 * inner;
    float g[8], u[8];
    unpack8(__ldg(reinterpret_cast<const int4*>(hr + col)), g);
    unpack8(__ldg(reinterpret_cast<const int4*>(hr + inner + col)), u);
    if (!BWD) {
        float a[8];
#pragma unroll
        for (int i = 0; i < 8; ++i) a[i] = g[i] * sigmoid_f(g[i]) * u[i];
        *reinterpret_cast<int4*>(out + row * inner + col) = pack8(a);
    } else {
        float d[8], dg[8], du[8];
        unpack8(__ldg(reinterpret_cast<const int4*>(da + row * inner + col)), d);
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            const float s = sigmoid_f(g[i]);
            dg[i] = d[i] * u[i] * (s * (1.f + g[i] * (1.f - s)));
            du[i] = d[i] * (g[i] * s);
        }
        bf16* o = out + row * 2 * inner;
        *reinterpret_cast<int4*>(o + col) = pack8(dg);
        *reinterpret_cast<int4*>(o + inner + col) = pack8(du);
    }
}

// the forward above plus the MXFP8 copy of a (aq, sf; a may be nullptr).  The 4 threads of a 32-column block are adjacent
// lanes of one row (inner / 8 is a multiple of 4), so a quad is wholly live or wholly skipped and shuffles within itself.
// Rows of tiles whose group is -1 (tile_group128: one entry per 128 rows) and rows >= *total_rows are skipped.
__global__ void __launch_bounds__(256) swiglu_quant_kernel(const bf16* __restrict__ h, bf16* __restrict__ a,
                                                           uint8_t* __restrict__ aq, uint8_t* __restrict__ sf,
                                                           long long vecs, int inner,
                                                           const int* __restrict__ tile_group128,
                                                           const int* __restrict__ total_rows) {
    const long long t = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (t >= vecs) return;
    const int per_row = inner >> 3;
    const long long row = t / per_row;
    if (total_rows && row >= __ldg(total_rows)) return;
    if (tile_group128 && __ldg(tile_group128 + (row >> 7)) < 0) return;
    const int v = static_cast<int>(t - row * per_row), col = v * 8;
    const bf16* hr = h + row * 2 * inner;
    float g[8], u[8], y[8];
    unpack8(__ldg(reinterpret_cast<const int4*>(hr + col)), g);
    unpack8(__ldg(reinterpret_cast<const int4*>(hr + inner + col)), u);
#pragma unroll
    for (int i = 0; i < 8; ++i) y[i] = g[i] * sigmoid_f(g[i]) * u[i];
    if (a) *reinterpret_cast<int4*>(a + row * inner + col) = pack8(y);
    const int lane = threadIdx.x & 31;
    quant_quad8(y, 0xFu << (lane & ~3), lane, aq + row * inner + col, sf + act_sf_byte(row, inner, v >> 2));
}

}  // namespace lah

using namespace lah;
using namespace lah::drop;

extern "C" {

// out[batch, heads, rows, cols] uint8 keep mask of `site` (sites 1-3: batch = heads = 1)
int lah_dropout_mask(void* out, int site, int batch, int heads, int rows, int cols, unsigned long long seed, int thr,
                     cudaStream_t st) {
    if (site < 0 || site > 3 || batch < 0 || heads < 1 || rows < 0 || cols < 1 || thr < 0 || thr > 65535) return -2;
    if (site != SITE_ATTN && (batch != 1 || heads != 1)) return -2;
    const long long total = static_cast<long long>(batch) * heads * rows * cols;
    if (total == 0) return 0;
    dropout_mask_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>((uint8_t*)out, site, heads, rows, cols, total, seed,
                                                                       static_cast<uint32_t>(thr));
    return -(int)cudaGetLastError();
}

// elementwise dropout op (see the top of this file) over contiguous [rows, cols] bf16 tensors; rows, cols multiples of 16
int lah_dropout_ew(int op, const void* x, const void* f, void* out, long long rows, int cols, unsigned long long seed,
                   int site, int thr, float scale, cudaStream_t st) {
    if ((rows % 16) || (cols % 16) || cols <= 0 || site < 1 || site > 3 || thr < 0 || thr > 65535) return -2;
    const long long granules = rows * cols / 8;
    if (granules == 0) return 0;
    const unsigned grid = (unsigned)((granules + 255) / 256);
    const uint32_t t = static_cast<uint32_t>(thr);
    if (op == OP_APPLY)
        dropout_ew_kernel<OP_APPLY><<<grid, 256, 0, st>>>((const bf16*)x, nullptr, (bf16*)out, granules, cols, seed, site, t, scale);
    else if (op == OP_GELU_FWD)
        dropout_ew_kernel<OP_GELU_FWD><<<grid, 256, 0, st>>>((const bf16*)x, nullptr, (bf16*)out, granules, cols, seed, site, t, scale);
    else if (op == OP_GELU_BWD)
        dropout_ew_kernel<OP_GELU_BWD><<<grid, 256, 0, st>>>((const bf16*)x, (const bf16*)f, (bf16*)out, granules, cols, seed, site, t,
                                                            scale);
    else if (op == OP_RELU_FWD)
        dropout_ew_kernel<OP_RELU_FWD><<<grid, 256, 0, st>>>((const bf16*)x, nullptr, (bf16*)out, granules, cols, seed, site, t, scale);
    else if (op == OP_RELU_BWD)
        dropout_ew_kernel<OP_RELU_BWD><<<grid, 256, 0, st>>>((const bf16*)x, (const bf16*)f, (bf16*)out, granules, cols, seed, site, t,
                                                            scale);
    else
        return -3;
    return -(int)cudaGetLastError();
}

// SwiGLU forward: a [rows, inner] = silu(g) o u of h = [g | u] [rows, 2 inner]; contiguous bf16, inner a multiple of 128
int lah_swiglu_fwd(const void* h, void* a, long long rows, int inner, cudaStream_t st) {
    if (rows < 0 || inner <= 0 || inner % 128) return -2;
    const long long vecs = rows * (inner / 8);
    if (vecs == 0) return 0;
    swiglu_kernel<false><<<(unsigned)((vecs + 255) / 256), 256, 0, st>>>((const bf16*)h, nullptr, (bf16*)a, vecs, inner);
    return -(int)cudaGetLastError();
}

// the same + a as an MXFP8 GEMM operand (aq: e4m3 [rows, inner]; sf: activation scale layout, tile_rows = 128); a may be
// NULL.  tile_group128 (optional): the group of every 128 rows, -1 = skipped; total_rows (optional, device): rows past it
// are skipped.  inner a multiple of 128; h and a 16-byte aligned, aq 8-byte aligned (the vector widths of the kernel)
int lah_swiglu_fwd_q(const void* h, void* a, void* aq, void* sf, long long rows, int inner, const int* tile_group128,
                     const int* total_rows, cudaStream_t st) {
    if (rows < 0 || inner <= 0 || inner % 128 || !aq || !sf) return -2;
    if ((reinterpret_cast<uintptr_t>(h) % 16) || (reinterpret_cast<uintptr_t>(a) % 16) ||
        (reinterpret_cast<uintptr_t>(aq) % 8))
        return -2;
    const long long vecs = rows * (inner / 8);
    if (vecs == 0) return 0;
    swiglu_quant_kernel<<<(unsigned)((vecs + 255) / 256), 256, 0, st>>>((const bf16*)h, (bf16*)a, (uint8_t*)aq,
                                                                       (uint8_t*)sf, vecs, inner, tile_group128,
                                                                       total_rows);
    return -(int)cudaGetLastError();
}

// SwiGLU backward: dh [rows, 2 inner] = [dg | du] from da [rows, inner] and the forward's h
int lah_swiglu_bwd(const void* da, const void* h, void* dh, long long rows, int inner, cudaStream_t st) {
    if (rows < 0 || inner <= 0 || inner % 128) return -2;
    const long long vecs = rows * (inner / 8);
    if (vecs == 0) return 0;
    swiglu_kernel<true><<<(unsigned)((vecs + 255) / 256), 256, 0, st>>>((const bf16*)h, (const bf16*)da, (bf16*)dh, vecs,
                                                                       inner);
    return -(int)cudaGetLastError();
}

}  // extern "C"
