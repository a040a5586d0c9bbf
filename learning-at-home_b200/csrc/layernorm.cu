// layernorm.cu — fused (bias already added by the GEMM epilogue) LayerNorm + ReLU forward / backward over
// expert-grouped rows, plus grouped column sums (bias gradients).
//
// Reference semantics: nn.LayerNorm(4h) -> nn.ReLU between the expert's Linear layers
// (/root/reference/experiments/throughput/layers.py:9-15); per-expert affine parameters gamma/beta are stacked [G, C].
//
// Rows are grouped by expert in 128-row tiles; tile_group[t] gives the expert (or -1: tile unused, skipped).
#include "sm90.cuh"
#include <cuda_fp8.h>
#include <stdlib.h>

namespace lah {

constexpr float LN_EPS = 1e-5f;

// ------------------------------------------------------------------------------------------------
// forward: one warp per R consecutive rows (same 128-row tile => same expert), lane owns C/32 columns as chunks of 8
// (coalesced 16B accesses)
//   a = relu((h - mean) * rstd * gamma + beta);  saves mean / rstd per row
// Why R rows per warp: gamma / beta are 2 x 4 B per column against 2 B of payload, i.e. with one row per warp 2/3 of
// the bytes through the L1/LSU pipe were affine parameters (ncu: 3.4 TB/s DRAM, L1 the limiter); holding a parameter
// chunk in registers and applying it to R rows divides that traffic by R.
// ------------------------------------------------------------------------------------------------
// With QUANT the kernel ALSO emits the MXFP8 operand of the next expert GEMM (csrc/grouped_gemm_fp8.cu): E4M3 payload +
// one UE8M0 scale per 32 columns (4 adjacent lanes share a block: two shuffles), quantised from the fp32 value before it
// is rounded to bf16.  The bf16 copy is optional (a == nullptr in forward-only runs).
template <int C>
struct LnFwdCfg {
    static constexpr int R = (C >= 4096) ? 1 : ((C >= 2048) ? 2 : 4);   // rows per warp (64 packed registers)
};

static int ln_rows_per_warp(int dflt) {   // LAH_LN_ROWS=1 selects the one-row-per-warp variant (A/B measurements)
    static int forced = -1;
    if (forced < 0) {
        const char* e = getenv("LAH_LN_ROWS");
        forced = e ? atoi(e) : 0;
    }
    return forced == 1 ? 1 : dflt;
}

template <int C, bool QUANT, int R>
__global__ void __launch_bounds__(256, 2) ln_relu_fwd_kernel(
    const bf16* __restrict__ h, bf16* __restrict__ a, float* __restrict__ mean_out, float* __restrict__ rstd_out,
    const float* __restrict__ gamma, const float* __restrict__ beta, const int* __restrict__ tile_group, int rows,
    int relu, uint8_t* __restrict__ aq, uint8_t* __restrict__ sf, int tile_shift) {
    constexpr int NV = C / 256;  // int4 (8 x bf16) chunks per lane
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int row0 = (blockIdx.x * 8 + warp) * R;
    if (row0 >= rows) return;
    const int g = tile_group ? __ldg(tile_group + (row0 >> tile_shift)) : 0;
    if (g < 0) return;
    // rows stay PACKED (bf16x2) in registers: 4 regs per 8 values; values are unpacked on the fly in each pass
    int4 q[R][NV];
#pragma unroll
    for (int r = 0; r < R; ++r) {
        const int4* hp = reinterpret_cast<const int4*>(h + static_cast<long long>(min(row0 + r, rows - 1)) * C);
#pragma unroll
        for (int j = 0; j < NV; ++j) q[r][j] = ld_nc_v4(hp + j * 32 + lane);
    }
    float mean[R], rstd[R];
#pragma unroll
    for (int r = 0; r < R; ++r) {
        // one pass: sum and sum of squares in fp32 (inputs are bf16: 8 mantissa bits, C <= 4096 -> ample head-room)
        float s = 0.f, ss = 0.f;
#pragma unroll
        for (int j = 0; j < NV; ++j) {
            const uint32_t w[4] = {(uint32_t)q[r][j].x, (uint32_t)q[r][j].y, (uint32_t)q[r][j].z, (uint32_t)q[r][j].w};
#pragma unroll
            for (int t = 0; t < 4; ++t) {
                const float2 f = unpack_bf16x2(w[t]);
                s += f.x + f.y;
                ss += f.x * f.x + f.y * f.y;
            }
        }
        s = warp_sum(s);
        ss = warp_sum(ss);
        mean[r] = s * (1.f / C);
        rstd[r] = rsqrtf(fmaxf(ss * (1.f / C) - mean[r] * mean[r], 0.f) + LN_EPS);
        if (lane == 0 && mean_out && row0 + r < rows) {
            mean_out[row0 + r] = mean[r];
            rstd_out[row0 + r] = rstd[r];
        }
    }
    const float* gp = gamma + static_cast<long long>(g) * C;
    const float* bp = beta + static_cast<long long>(g) * C;
#pragma unroll
    for (int j = 0; j < NV; ++j) {
        const int col = (j * 32 + lane) * 8;
        // volatile asm loads: ordered with the volatile asm stores below, so the compiler cannot hoist the parameter
        // loads of all later chunks to the top (16 registers per chunk -> spills)
        const int4 g0 = ld_nc_v4(reinterpret_cast<const int4*>(gp + col));
        const int4 g1 = ld_nc_v4(reinterpret_cast<const int4*>(gp + col + 4));
        const int4 b0 = ld_nc_v4(reinterpret_cast<const int4*>(bp + col));
        const int4 b1 = ld_nc_v4(reinterpret_cast<const int4*>(bp + col + 4));
        const float gg[8] = {__int_as_float(g0.x), __int_as_float(g0.y), __int_as_float(g0.z), __int_as_float(g0.w),
                             __int_as_float(g1.x), __int_as_float(g1.y), __int_as_float(g1.z), __int_as_float(g1.w)};
        const float bb[8] = {__int_as_float(b0.x), __int_as_float(b0.y), __int_as_float(b0.z), __int_as_float(b0.w),
                             __int_as_float(b1.x), __int_as_float(b1.y), __int_as_float(b1.z), __int_as_float(b1.w)};
#pragma unroll
        for (int r = 0; r < R; ++r) {
            const int row = row0 + r;
            if (row >= rows) continue;   // warp-uniform
            const uint32_t w[4] = {(uint32_t)q[r][j].x, (uint32_t)q[r][j].y, (uint32_t)q[r][j].z, (uint32_t)q[r][j].w};
            float y[8];
#pragma unroll
            for (int t = 0; t < 4; ++t) {
                const float2 f = unpack_bf16x2(w[t]);
                y[2 * t] = (f.x - mean[r]) * rstd[r] * gg[2 * t] + bb[2 * t];
                y[2 * t + 1] = (f.y - mean[r]) * rstd[r] * gg[2 * t + 1] + bb[2 * t + 1];
            }
            if (relu) {
#pragma unroll
                for (int t = 0; t < 8; ++t) y[t] = fmaxf(y[t], 0.f);
            }
            if (!QUANT || a) {
                int4 o;
                o.x = pack_bf16x2(y[0], y[1]);
                o.y = pack_bf16x2(y[2], y[3]);
                o.z = pack_bf16x2(y[4], y[5]);
                o.w = pack_bf16x2(y[6], y[7]);
                // asm store with a memory clobber: keeps the compiler from hoisting the parameter loads of all later
                // chunks above it (which costs 16 registers per chunk and spills)
                st_v4(reinterpret_cast<int4*>(a + static_cast<long long>(row) * C) + j * 32 + lane, o);
            }
            if (QUANT) {
                float amax = 0.f;
#pragma unroll
                for (int t = 0; t < 8; ++t) amax = fmaxf(amax, fabsf(y[t]));
                amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, 1));
                amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, 2));
                // smallest power-of-two scale with amax / scale <= 448 (same rule as quant_mxfp8_kernel)
                const uint32_t bits = __float_as_uint(amax * (1.f / 448.f));
                uint32_t e = ((bits >> 23) & 0xFFu) + ((bits & 0x7FFFFFu) ? 1u : 0u);
                e = min(max(e, 1u), 253u);
                const float inv = __uint_as_float((254u - e) << 23);
                uint2 o8;
                o8.x = static_cast<uint32_t>(__nv_cvt_float2_to_fp8x2(make_float2(y[0] * inv, y[1] * inv), __NV_SATFINITE, __NV_E4M3)) |
                       (static_cast<uint32_t>(__nv_cvt_float2_to_fp8x2(make_float2(y[2] * inv, y[3] * inv), __NV_SATFINITE, __NV_E4M3)) << 16);
                o8.y = static_cast<uint32_t>(__nv_cvt_float2_to_fp8x2(make_float2(y[4] * inv, y[5] * inv), __NV_SATFINITE, __NV_E4M3)) |
                       (static_cast<uint32_t>(__nv_cvt_float2_to_fp8x2(make_float2(y[6] * inv, y[7] * inv), __NV_SATFINITE, __NV_E4M3)) << 16);
                asm volatile("st.global.v2.u32 [%0], {%1, %2};" ::"l"(reinterpret_cast<uint2*>(aq + static_cast<long long>(row) * C) + j * 32 + lane),
                             "r"(o8.x), "r"(o8.y)
                             : "memory");
                if ((lane & 3) == 0) {
                    const int kb32 = j * 8 + (lane >> 2);   // 32-column block of this lane quad
                    const int ra = row & 127;
                    const long long chunk = static_cast<long long>(row >> 7) * (C / 128) + (kb32 >> 2);
                    sf[chunk * 512 + ((ra & 31) * 4 + (ra >> 5)) * 4 + (kb32 & 3)] = static_cast<uint8_t>(e);
                }
            }
        }
    }
}

// ------------------------------------------------------------------------------------------------
// backward: one CTA (C/8 threads) per 128-row tile; thread owns 8 consecutive columns, keeps fp32 column
// accumulators (dgamma, dbeta, dbias) in registers for the whole tile, block-reduces the two row statistics.  The
// tile's column sums go to part[tile][0..2][C]; group_tile_sum_kernel adds them to the group's gradients in tile order, so
// the result does not depend on the order in which the CTAs finish.
//   y    = xhat*gamma + beta            (recomputed; relu mask = y > 0)
//   g    = da * mask                    dbeta += g        dgamma += g * xhat
//   dxh  = g * gamma
//   dh   = rstd * (dxh - mean_c(dxh) - xhat * mean_c(dxh * xhat))     dbias += dh
// ------------------------------------------------------------------------------------------------
template <int C>
__global__ void __launch_bounds__(C / 8, (C <= 2048) ? 2 : 1) ln_relu_bwd_kernel(const bf16* __restrict__ da, const bf16* __restrict__ h,
                                                            const float* __restrict__ mean_in,
                                                            const float* __restrict__ rstd_in,
                                                            const float* __restrict__ gamma,
                                                            const float* __restrict__ beta, bf16* __restrict__ dh,
                                                            float* __restrict__ part,
                                                            const int* __restrict__ tile_group, int rows, int relu, int tile_rows) {
    constexpr int THREADS = C / 8;
    constexpr int WARPS = THREADS / 32;
    constexpr int RB = (C >= 4096) ? 2 : 4;  // rows per batch (register blocking)
    __shared__ float red[WARPS][2 * RB];
    __shared__ float tot[2 * RB];
    const int tile = blockIdx.x;
    const int g = tile_group ? __ldg(tile_group + tile) : 0;
    if (g < 0) return;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int col = tid * 8;
    float gam[8], bet[8];
    {
        const float* gp = gamma + static_cast<long long>(g) * C + col;
        const float* bp = beta + static_cast<long long>(g) * C + col;
        const float4 g0 = __ldg(reinterpret_cast<const float4*>(gp)), g1 = __ldg(reinterpret_cast<const float4*>(gp + 4));
        const float4 b0 = __ldg(reinterpret_cast<const float4*>(bp)), b1 = __ldg(reinterpret_cast<const float4*>(bp + 4));
        gam[0] = g0.x; gam[1] = g0.y; gam[2] = g0.z; gam[3] = g0.w; gam[4] = g1.x; gam[5] = g1.y; gam[6] = g1.z; gam[7] = g1.w;
        bet[0] = b0.x; bet[1] = b0.y; bet[2] = b0.z; bet[3] = b0.w; bet[4] = b1.x; bet[5] = b1.y; bet[6] = b1.z; bet[7] = b1.w;
    }
    float acc_dg[8], acc_db[8], acc_dbias[8];
#pragma unroll
    for (int t = 0; t < 8; ++t) acc_dg[t] = acc_db[t] = acc_dbias[t] = 0.f;

    const int row0 = tile * tile_rows;
    const int row_end = min(rows, row0 + tile_rows);
    // software pipeline: the loads of batch i+1 are in flight while batch i is reduced / written
    int4 nqa[RB], nqh[RB];
    float nmu[RB], nrs[RB];
    auto issue_loads = [&](int rb) {
#pragma unroll
        for (int r = 0; r < RB; ++r) {
            const int row = rb + r;
            const int rr = row < row_end ? row : row0;
            const long long off = static_cast<long long>(rr) * C + col;
            nqa[r] = ld_nc_v4(reinterpret_cast<const int4*>(da + off));
            nqh[r] = ld_nc_v4(reinterpret_cast<const int4*>(h + off));
            nmu[r] = __ldg(mean_in + rr);
            nrs[r] = __ldg(rstd_in + rr);
        }
    };
    issue_loads(row0);
    for (int rb = row0; rb < row_end; rb += RB) {
        float rs[RB];
        float part[2 * RB];
        int4 qa_c[RB], qh_c[RB];
        float mu_c[RB];
#pragma unroll
        for (int r = 0; r < RB; ++r) {
            qa_c[r] = nqa[r];
            qh_c[r] = nqh[r];
            mu_c[r] = nmu[r];
            rs[r] = nrs[r];
        }
        if (rb + RB < row_end) issue_loads(rb + RB);
        // masked gradient g and xhat of one (row, 8 columns) slice, from the PACKED inputs: phase 2 recomputes them
        // instead of keeping 16 floats per row alive across the block reduction (214 -> <= 128 registers: 2 CTAs / SM)
        auto slice = [&](int r, bool ok, float (&gvv)[8], float (&xhh)[8]) {
            const uint32_t wa[4] = {(uint32_t)qa_c[r].x, (uint32_t)qa_c[r].y, (uint32_t)qa_c[r].z, (uint32_t)qa_c[r].w};
            const uint32_t wh[4] = {(uint32_t)qh_c[r].x, (uint32_t)qh_c[r].y, (uint32_t)qh_c[r].z, (uint32_t)qh_c[r].w};
#pragma unroll
            for (int t = 0; t < 4; ++t) {
                const float2 fa = unpack_bf16x2(wa[t]);
                const float2 fh = unpack_bf16x2(wh[t]);
                const float x0 = (fh.x - mu_c[r]) * rs[r], x1 = (fh.y - mu_c[r]) * rs[r];
                const float y0 = x0 * gam[2 * t] + bet[2 * t], y1 = x1 * gam[2 * t + 1] + bet[2 * t + 1];
                gvv[2 * t] = (ok && (!relu || y0 > 0.f)) ? fa.x : 0.f;
                gvv[2 * t + 1] = (ok && (!relu || y1 > 0.f)) ? fa.y : 0.f;
                xhh[2 * t] = x0;
                xhh[2 * t + 1] = x1;
            }
        };
#pragma unroll
        for (int r = 0; r < RB; ++r) {
            float gvv[8], xhh[8];
            slice(r, rb + r < row_end, gvv, xhh);
            float s1 = 0.f, s2 = 0.f;
#pragma unroll
            for (int t = 0; t < 8; ++t) {
                const float d = gvv[t] * gam[t];
                s1 += d;
                s2 += d * xhh[t];
            }
            part[2 * r] = s1;
            part[2 * r + 1] = s2;
        }
#pragma unroll
        for (int i = 0; i < 2 * RB; ++i) part[i] = warp_sum(part[i]);
        if (lane == 0) {
#pragma unroll
            for (int i = 0; i < 2 * RB; ++i) red[warp][i] = part[i];
        }
        __syncthreads();
        if (tid < 2 * RB) {
            float s = 0.f;
#pragma unroll
            for (int w = 0; w < WARPS; ++w) s += red[w][tid];
            tot[tid] = s * (1.f / C);
        }
        __syncthreads();
#pragma unroll
        for (int r = 0; r < RB; ++r) {
            const int row = rb + r;
            if (row >= row_end) continue;
            float gvv[8], xhh[8];
            slice(r, true, gvv, xhh);
            const float m1 = tot[2 * r], m2 = tot[2 * r + 1];
            float o[8];
#pragma unroll
            for (int t = 0; t < 8; ++t) {
                o[t] = rs[r] * (gvv[t] * gam[t] - m1 - xhh[t] * m2);
                acc_db[t] += gvv[t];
                acc_dg[t] += gvv[t] * xhh[t];
                acc_dbias[t] += o[t];
            }
            int4 q;
            q.x = pack_bf16x2(o[0], o[1]);
            q.y = pack_bf16x2(o[2], o[3]);
            q.z = pack_bf16x2(o[4], o[5]);
            q.w = pack_bf16x2(o[6], o[7]);
            *reinterpret_cast<int4*>(dh + static_cast<long long>(row) * C + col) = q;
        }
        // `tot` is rewritten only after the next batch's first __syncthreads, which every thread reaches
        // after it finished reading tot above -> no extra barrier needed.
    }
    float* pg = part + static_cast<long long>(tile) * 3 * C + col;
#pragma unroll
    for (int t = 0; t < 8; ++t) {
        pg[t] = acc_dg[t];
        pg[C + t] = acc_db[t];
        pg[2 * C + t] = acc_dbias[t];
    }
}

// ------------------------------------------------------------------------------------------------
// grouped column sum: out[g, c] += sum over the rows of every 128-row tile of group g of x[row, c]
// CTA = (tile, 256-column slab); thread owns one column pair, 4 row phases; the tile's sums go to part[tile][C] and are
// added to out by group_tile_sum_kernel
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(512) grouped_colsum_kernel(const bf16* __restrict__ x, long long ldx,
                                                             float* __restrict__ part, int C,
                                                             const int* __restrict__ tile_group, int rows, int tile_rows) {
    __shared__ float2 sm[4][128];
    const int tile = blockIdx.x;
    const int g = tile_group ? __ldg(tile_group + tile) : 0;
    if (g < 0) return;
    const int cp = threadIdx.x & 127;         // column pair inside the slab
    const int phase = threadIdx.x >> 7;       // 0..3
    const int col = blockIdx.y * 256 + cp * 2;
    if (col >= C) return;                      // C is a multiple of 256 in practice; whole warps exit together
    const int row0 = tile * tile_rows, row_end = min(rows, row0 + tile_rows);
    float2 acc = make_float2(0.f, 0.f);
    for (int r = row0 + phase; r < row_end; r += 4) {
        const uint32_t u = __ldg(reinterpret_cast<const uint32_t*>(x + static_cast<long long>(r) * ldx + col));
        const float2 f = unpack_bf16x2(u);
        acc.x += f.x;
        acc.y += f.y;
    }
    sm[phase][cp] = acc;
    __syncthreads();
    if (phase == 0) {
        float2 s = sm[0][cp];
#pragma unroll
        for (int p = 1; p < 4; ++p) {
            s.x += sm[p][cp].x;
            s.y += sm[p][cp].y;
        }
        *reinterpret_cast<float2*>(part + static_cast<long long>(tile) * C + col) = s;
    }
}

// out_v[g, c] += sum over the tiles t of group g (in increasing t) of part[t][v][c], v < V: a fixed summation order, so
// the per-group gradients are the same in every run.  Thread = (v, c); tiles with group -1 are skipped.
__global__ void __launch_bounds__(256) group_tile_sum_kernel(const float* __restrict__ part, int num_tiles, int V, int C,
                                                             const int* __restrict__ tile_group, float* out0, float* out1,
                                                             float* out2) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= V * C) return;
    const int v = i / C, c = i - v * C;
    float* out = v == 0 ? out0 : (v == 1 ? out1 : out2);
    int cur = -1;
    float acc = 0.f;
    for (int t = 0; t < num_tiles; ++t) {
        const int g = tile_group ? __ldg(tile_group + t) : 0;
        if (g < 0) continue;
        if (g != cur) {
            if (cur >= 0) out[static_cast<long long>(cur) * C + c] += acc;
            cur = g;
            acc = 0.f;
        }
        acc += __ldg(part + (static_cast<long long>(t) * V + v) * C + c);
    }
    if (cur >= 0) out[static_cast<long long>(cur) * C + c] += acc;
}

}  // namespace lah

using namespace lah;

extern "C" {

static int shift_of(int tile_rows) {
    int s = 0;
    while ((1 << s) < tile_rows) ++s;
    return ((1 << s) == tile_rows && tile_rows >= 8) ? s : -1;
}

// tile_rows: rows per tile_group entry (power of two >= 8; 128 for the padded big-batch layout, 16 for the small-M layout)
int lah_ln_relu_fwd_t(const void* h, void* a, float* mean, float* rstd, const float* gamma, const float* beta,
                      const int* tile_group, int rows, int C, int relu, int tile_rows, cudaStream_t st) {
    if (rows <= 0) return 0;
    const int tile_shift = shift_of(tile_rows);
    if (tile_shift < 0) return -2;
#define LAH_LN_FWD(CC)                                                                                          \
    if (C == CC) {                                                                                              \
        constexpr int RR = LnFwdCfg<CC>::R;                                                                     \
        if (ln_rows_per_warp(RR) == 1)                                                                          \
            ln_relu_fwd_kernel<CC, false, 1><<<(rows + 7) / 8, 256, 0, st>>>(                                  \
                (const bf16*)h, (bf16*)a, mean, rstd, gamma, beta, tile_group, rows, relu, nullptr, nullptr, tile_shift);   \
        else                                                                                                    \
            ln_relu_fwd_kernel<CC, false, RR><<<(rows + 8 * RR - 1) / (8 * RR), 256, 0, st>>>(                 \
                (const bf16*)h, (bf16*)a, mean, rstd, gamma, beta, tile_group, rows, relu, nullptr, nullptr, tile_shift);   \
        return -(int)cudaGetLastError();                                                                        \
    }
    LAH_LN_FWD(256) LAH_LN_FWD(512) LAH_LN_FWD(1024) LAH_LN_FWD(2048) LAH_LN_FWD(4096)
#undef LAH_LN_FWD
    return -2;
}

int lah_ln_relu_fwd(const void* h, void* a, float* mean, float* rstd, const float* gamma, const float* beta,
                    const int* tile_group, int rows, int C, int relu, cudaStream_t st) {
    return lah_ln_relu_fwd_t(h, a, mean, rstd, gamma, beta, tile_group, rows, C, relu, 128, st);
}

// same + MXFP8 copy of the output (aq: e4m3 [rows, C]; sf: activation scale layout, tile_rows = 128); a may be NULL
int lah_ln_relu_fwd_q(const void* h, void* a, float* mean, float* rstd, const float* gamma, const float* beta,
                      const int* tile_group, int rows, int C, int relu, void* aq, void* sf, cudaStream_t st) {
    if (rows <= 0) return 0;
#define LAH_LN_FWD(CC)                                                                                          \
    if (C == CC) {                                                                                              \
        constexpr int RR = LnFwdCfg<CC>::R;                                                                     \
        if (ln_rows_per_warp(RR) == 1)                                                                          \
            ln_relu_fwd_kernel<CC, true, 1><<<(rows + 7) / 8, 256, 0, st>>>(                                  \
                (const bf16*)h, (bf16*)a, mean, rstd, gamma, beta, tile_group, rows, relu, (uint8_t*)aq, (uint8_t*)sf, 7);   \
        else                                                                                                    \
            ln_relu_fwd_kernel<CC, true, RR><<<(rows + 8 * RR - 1) / (8 * RR), 256, 0, st>>>(                 \
                (const bf16*)h, (bf16*)a, mean, rstd, gamma, beta, tile_group, rows, relu, (uint8_t*)aq, (uint8_t*)sf, 7);   \
        return -(int)cudaGetLastError();                                                                        \
    }
    LAH_LN_FWD(256) LAH_LN_FWD(512) LAH_LN_FWD(1024) LAH_LN_FWD(2048) LAH_LN_FWD(4096)
#undef LAH_LN_FWD
    return -2;
}

// part: scratch of [ceil(rows / tile_rows), 3, C] fp32 (per-tile column sums, reduced in tile order)
int lah_ln_relu_bwd_t(const void* da, const void* h, const float* mean, const float* rstd, const float* gamma,
                      const float* beta, void* dh, float* dgamma, float* dbeta, float* dbias, float* part,
                      const int* tile_group, int rows, int C, int relu, int tile_rows, cudaStream_t st) {
    if (rows <= 0) return 0;
    if (shift_of(tile_rows) < 0) return -2;
    const int grid = (rows + tile_rows - 1) / tile_rows;
#define LAH_LN_BWD(CC)                                                                                          \
    if (C == CC) {                                                                                              \
        ln_relu_bwd_kernel<CC><<<grid, CC / 8, 0, st>>>((const bf16*)da, (const bf16*)h, mean, rstd, gamma,    \
                                                        beta, (bf16*)dh, part, tile_group, rows, relu,         \
                                                        tile_rows);                                             \
        group_tile_sum_kernel<<<(3 * CC + 255) / 256, 256, 0, st>>>(part, grid, 3, CC, tile_group, dgamma,     \
                                                                     dbeta, dbias);                            \
        return -(int)cudaGetLastError();                                                                        \
    }
    LAH_LN_BWD(256) LAH_LN_BWD(512) LAH_LN_BWD(1024) LAH_LN_BWD(2048) LAH_LN_BWD(4096)
#undef LAH_LN_BWD
    return -2;
}

int lah_ln_relu_bwd(const void* da, const void* h, const float* mean, const float* rstd, const float* gamma,
                    const float* beta, void* dh, float* dgamma, float* dbeta, float* dbias, float* part,
                    const int* tile_group, int rows, int C, int relu, cudaStream_t st) {
    return lah_ln_relu_bwd_t(da, h, mean, rstd, gamma, beta, dh, dgamma, dbeta, dbias, part, tile_group, rows, C, relu, 128,
                             st);
}

// part: scratch of [ceil(rows / tile_rows), C] fp32 (per-tile column sums, reduced in tile order)
int lah_grouped_colsum_t(const void* x, long long ldx, float* out, float* part, int C, const int* tile_group, int rows,
                         int tile_rows, cudaStream_t st) {
    if (rows <= 0) return 0;
    if (C % 256 || shift_of(tile_rows) < 0) return -2;
    const int tiles = (rows + tile_rows - 1) / tile_rows;
    dim3 grid(tiles, (C + 255) / 256);
    grouped_colsum_kernel<<<grid, 512, 0, st>>>((const bf16*)x, ldx, part, C, tile_group, rows, tile_rows);
    group_tile_sum_kernel<<<(C + 255) / 256, 256, 0, st>>>(part, tiles, 1, C, tile_group, out, nullptr, nullptr);
    return -(int)cudaGetLastError();
}

int lah_grouped_colsum(const void* x, long long ldx, float* out, float* part, int C, const int* tile_group, int rows,
                       cudaStream_t st) {
    return lah_grouped_colsum_t(x, ldx, out, part, C, tile_group, rows, 128, st);
}

}  // extern "C"
