// grouped_gemm_fp8.cu — block-scaled FP8 (MXFP8: E4M3 data, one UE8M0 scale per 1x32 block along K) grouped GEMM on
// Hopper FP8 tensor cores (wgmma ... e4m3.e4m3), plus the quantisation kernels that produce its operands.
//
//   C[r, :] = (A_q[r, :] * 2^sfa) @ (W_q[g(r)] * 2^sfb)^T (+ bias) (+ act) (+ residual)       bf16 / fp32 out
//
// Same structure as grouped_gemm.cu (one TMA producer warp, two consumer warpgroups of 64 rows, 128 x 128 tiles, epilogue
// from registers).  Differences:
//   * 8-bit operands: BLOCK_K = 128 elements (one 128 B swizzle row), MMA K = 32 -> twice the math per smem byte;
//   * the tensor core has no block scaling here, so every 32-element K block is one wgmma into a scratch accumulator that
//     is added to the running accumulator times 2^sfa[row] * 2^sfb[col] (exact: powers of two); the scale words come
//     straight from the quantiser's layout (sf_word) through the read-only cache.
//
// Used for the expert FFN forward GEMMs (BASELINE.json config "fp8 expert GEMM"); dgrad / wgrad stay in bf16.
#include "mxfp8.cuh"
#include "sm90.cuh"
#include <cuda_fp8.h>

namespace lah {
namespace f8 {

constexpr int TILE_M = 128;
constexpr int TILE_N = 128;
constexpr int BLOCK_K = 128;  // elements == bytes
constexpr int MMA_K = 32;
constexpr int STAGES = 6;
constexpr int NUM_THREADS = 288;     // two consumer warpgroups + one TMA producer warp
constexpr int A_TILE_ROWS = 128;     // scale-factor tiling of activations / weights (see the storage layout below)
constexpr int W_TILE_ROWS = 192;

constexpr int A_BYTES = TILE_M * BLOCK_K;       // 16 KB
constexpr int B_BYTES = TILE_N * BLOCK_K;       // 16 KB
constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
constexpr int BAR_OFFSET = STAGES * STAGE_BYTES;
constexpr int SMEM_TOTAL = BAR_OFFSET + 2 * STAGES * 8 + 1024;
static_assert(SMEM_TOTAL <= 227 * 1024, "shared memory budget");

struct Params {
    int N, K, M, num_groups, num_m_tiles, n_tiles, num_kb;
    const int* tile_group;
    void* C;
    long long ldc;
    const float* bias;
    const bf16* residual;
    long long ldr;
    const int* wait_flags;
    int wait_count, wait_epoch;
    const int* epoch_base;   // device-side epoch base added to wait_epoch (nullptr: 0), see moe.cu Peers::step_ctr
    int* status;
    int act;
    const uint32_t* sfa;   // activation scales (tile_rows = 128)
    const uint32_t* sfb;   // weight scales (tile_rows = 192)
};

// D (64 x 128 per warpgroup) = A * B for one 32-element K block, E4M3 inputs (both K-major), fp32 accumulate, D overwritten
__device__ __forceinline__ void wgmma_e4m3_n128(float (&d)[64], uint64_t da, uint64_t db) {
    asm volatile(
        "wgmma.mma_async.sync.aligned.m64n128k32.f32.e4m3.e4m3 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, 0, 1, 1;\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "l"(da), "l"(db));
}

// the four UE8M0 scale bytes (k-steps of 32 elements) of row r of a 128-element K block, see the storage layout below
__device__ __forceinline__ uint32_t sf_word(const uint32_t* __restrict__ sf, int g, int r, int tiles_per_group, int tile_rows,
                                            int num_kb, int kb) {
    const int tile = r / tile_rows, rt = r - tile * tile_rows;
    const int atoms = (tile_rows + 127) >> 7, atom = rt >> 7, ra = rt & 127;
    const long long chunk = ((static_cast<long long>(g) * tiles_per_group + tile) * num_kb + kb) * atoms + atom;
    return __ldg(sf + chunk * 128 + (ra & 31) * 4 + (ra >> 5));
}
__device__ __forceinline__ float e8m0_scale(uint32_t word, int ks) { return __uint_as_float(((word >> (8 * ks)) & 0xFFu) << 23); }

template <bool OUT_F32>
__global__ void __launch_bounds__(NUM_THREADS, 1)
gemm_fp8_kernel(const Params p, const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + BAR_OFFSET);
    uint64_t* empty_bar = full_bar + STAGES;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

    if (warp == 8 && lane == 0) {
        tma_prefetch_desc(&tmA);
        tma_prefetch_desc(&tmB);
        for (int i = 0; i < STAGES; ++i) {
            mbar_init(&full_bar[i], 1);
            mbar_init(&empty_bar[i], 8);   // one arrive per consumer warp
        }
        fence_mbar_init();
    }
    __syncthreads();
    const int total_tiles = p.num_m_tiles * p.n_tiles;

    if (warp == 8) {
        if (lane != 0) return;
        // =============================================================== TMA producer
        if (p.wait_flags) {   // rows pushed by peer GPUs over NVLink must have landed before the first TMA load
            const unsigned long long t_wait = globaltimer_ns();
            for (int sidx = 0; sidx < p.wait_count; ++sidx)
                spin_flag_ft(p.wait_flags + sidx, p.wait_epoch + (p.epoch_base ? p.epoch_base[0] : 0), p.status, sidx,
                             p.epoch_base ? p.epoch_base[1] : 0);
            if (blockIdx.x == 0) atomicAdd(reinterpret_cast<unsigned long long*>(p.status + 2), globaltimer_ns() - t_wait);
            fence_proxy_async_global();
        }
        int stage = 0;
        uint32_t phase = 0;
        for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
            const int m_tile = tile / p.n_tiles, n_tile = tile - m_tile * p.n_tiles;
            const int g = p.tile_group ? __ldg(p.tile_group + m_tile) : 0;
            if (g < 0) continue;
            for (int kb = 0; kb < p.num_kb; ++kb) {
                mbar_wait(&empty_bar[stage], phase ^ 1);
                uint8_t* sa = smem + stage * STAGE_BYTES;
                mbar_arrive_expect_tx(&full_bar[stage], STAGE_BYTES);
                tma_load_2d(sa, &tmA, &full_bar[stage], kb * BLOCK_K, m_tile * TILE_M);
                tma_load_3d(sa + A_BYTES, &tmB, &full_bar[stage], kb * BLOCK_K, n_tile * TILE_N, g);
                if (++stage == STAGES) {
                    stage = 0;
                    phase ^= 1;
                }
            }
        }
        return;
    }

    // =================================================================== consumers (two warpgroups of 64 rows)
    const int wg = warp >> 2;
    const int row_in_tile = wg * 64 + (warp & 3) * 16 + (lane >> 2);   // and + 8
    const int col_in_tile = 2 * (lane & 3);                             // + 8 j (+ 1)
    const int w_tiles_per_group = (p.N + W_TILE_ROWS - 1) / W_TILE_ROWS;
    int stage = 0;
    uint32_t phase = 0;
    float acc[TILE_N / 2], part[TILE_N / 2];
    for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
        const int m_tile = tile / p.n_tiles, n_tile = tile - m_tile * p.n_tiles;
        const int g = p.tile_group ? __ldg(p.tile_group + m_tile) : 0;
        if (g < 0) continue;
        const int m_row = m_tile * TILE_M, n_col = n_tile * TILE_N;
#pragma unroll
        for (int i = 0; i < TILE_N / 2; ++i) acc[i] = 0.f;
        for (int kb = 0; kb < p.num_kb; ++kb) {
            // block scales of this thread's 2 rows and 32 columns (one 32-bit word = the 4 k-steps of the K block)
            uint32_t wa[2], wb[TILE_N / 8][2];
#pragma unroll
            for (int h = 0; h < 2; ++h) wa[h] = sf_word(p.sfa, 0, m_row + row_in_tile + 8 * h, 0, A_TILE_ROWS, p.num_kb, kb);
#pragma unroll
            for (int j = 0; j < TILE_N / 8; ++j)
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    const int n = min(n_col + 8 * j + col_in_tile + e, p.N - 1);
                    wb[j][e] = sf_word(p.sfb, g, n, w_tiles_per_group, W_TILE_ROWS, p.num_kb, kb);
                }
            mbar_wait(&full_bar[stage], phase);
            const uint32_t sa = smem_u32(smem + stage * STAGE_BYTES) + wg * (64 * 128);
            const uint32_t sb = smem_u32(smem + stage * STAGE_BYTES + A_BYTES);
#pragma unroll
            for (int ks = 0; ks < BLOCK_K / MMA_K; ++ks) {
                wgmma_fence();
                wgmma_e4m3_n128(part, make_smem_desc_sw128(sa + ks * 32, 0, 1024), make_smem_desc_sw128(sb + ks * 32, 0, 1024));
                wgmma_commit();
                wgmma_wait<0>();
                wgmma_fence_regs(part);
                // the 1x32 block scales are powers of two: scaling the block's partial product is exact
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const float sa_h = e8m0_scale(wa[h], ks);
#pragma unroll
                    for (int j = 0; j < TILE_N / 8; ++j)
#pragma unroll
                        for (int e = 0; e < 2; ++e)
                            acc[4 * j + 2 * h + e] = fmaf(part[4 * j + 2 * h + e] * sa_h, e8m0_scale(wb[j][e], ks),
                                                          acc[4 * j + 2 * h + e]);
                }
            }
            __syncwarp();
            if (lane == 0) mbar_arrive(&empty_bar[stage]);
            if (++stage == STAGES) {
                stage = 0;
                phase ^= 1;
            }
        }
        // ------------------------------------------------------------ epilogue from registers
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int row = m_row + row_in_tile + 8 * h;
            if (row >= p.M) continue;
#pragma unroll
            for (int j = 0; j < TILE_N / 8; ++j) {
                const int col = n_col + 8 * j + col_in_tile;
                if (col >= p.N) continue;
                float v0 = acc[4 * j + 2 * h], v1 = acc[4 * j + 2 * h + 1];
                if (p.bias) {
                    const float2 b = __ldg(reinterpret_cast<const float2*>(p.bias + static_cast<long long>(g) * p.N + col));
                    v0 += b.x;
                    v1 += b.y;
                }
                if (p.act == 1) {
                    v0 = fmaxf(v0, 0.f);
                    v1 = fmaxf(v1, 0.f);
                } else if (p.act == 2) {
                    v0 = 0.5f * v0 * (1.f + erff(v0 * 0.70710678118654752f));
                    v1 = 0.5f * v1 * (1.f + erff(v1 * 0.70710678118654752f));
                }
                if (p.residual) {
                    const float2 r = unpack_bf16x2(
                        __ldg(reinterpret_cast<const unsigned int*>(p.residual + static_cast<long long>(row) * p.ldr + col)));
                    v0 += r.x;
                    v1 += r.y;
                }
                if (OUT_F32)
                    *reinterpret_cast<float2*>(reinterpret_cast<float*>(p.C) + static_cast<long long>(row) * p.ldc + col) =
                        make_float2(v0, v1);
                else
                    *reinterpret_cast<uint32_t*>(reinterpret_cast<bf16*>(p.C) + static_cast<long long>(row) * p.ldc + col) =
                        pack_bf16x2(v0, v1);
            }
        }
    }
}

// ------------------------------------------------------------------------------------------------ quantisation
// Scale-factor storage.  Rows are split into tiles of `tile_rows` rows (128 for activations, 192 for weights), every
// tile into atoms of 128 rows, K into blocks of 128 elements.  One (atom, K block) chunk is 128 32-bit words = 512 B:
//   word (r % 32) * 4 + (r / 32)  holds the four UE8M0 bytes (k-steps of 32 elements) of row r of the atom.
// Chunk index = ((tile * num_kb + kb) * atoms_per_tile + atom).
__host__ __device__ inline long long sf_chunks(long long rows, int tile_rows, int num_kb) {
    const long long tiles = (rows + tile_rows - 1) / tile_rows;
    return tiles * num_kb * ((tile_rows + 127) / 128);
}

// one thread per (row, 32-element block): 64 B (bf16) or 128 B (fp32) in, 32 B + one scale byte out
template <typename T>
__global__ void __launch_bounds__(256) quant_mxfp8_kernel(const T* __restrict__ in, long long ld_in,
                                                          uint8_t* __restrict__ out, long long ld_out,
                                                          uint8_t* __restrict__ sf, int rows_per_group, int groups, int K,
                                                          int tile_rows, const int* __restrict__ tile_group128,
                                                          const int* __restrict__ total_rows_dev) {
    const int blocks_per_row = K >> 5;
    const long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
    const long long grow = idx / blocks_per_row;  // row over all groups
    const int kb32 = static_cast<int>(idx - grow * blocks_per_row);
    if (grow >= static_cast<long long>(rows_per_group) * groups) return;
    if (total_rows_dev && grow >= *total_rows_dev) return;
    if (tile_group128 && __ldg(tile_group128 + (grow >> 7)) < 0) return;
    const int g = static_cast<int>(grow / rows_per_group);
    const int r = static_cast<int>(grow - static_cast<long long>(g) * rows_per_group);
    const T* src = in + grow * ld_in + kb32 * 32;
    float v[32];
    if (sizeof(T) == 2) {
        const int4* p4 = reinterpret_cast<const int4*>(src);
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int4 q = __ldg(p4 + j);
            const uint32_t w[4] = {(uint32_t)q.x, (uint32_t)q.y, (uint32_t)q.z, (uint32_t)q.w};
#pragma unroll
            for (int t = 0; t < 4; ++t) {
                const float2 f = unpack_bf16x2(w[t]);
                v[8 * j + 2 * t] = f.x;
                v[8 * j + 2 * t + 1] = f.y;
            }
        }
    } else {
        const float4* p4 = reinterpret_cast<const float4*>(src);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const float4 f = __ldg(p4 + j);
            v[4 * j] = f.x; v[4 * j + 1] = f.y; v[4 * j + 2] = f.z; v[4 * j + 3] = f.w;
        }
    }
    float amax = 0.f;
#pragma unroll
    for (int j = 0; j < 32; ++j) amax = fmaxf(amax, fabsf(v[j]));
    const uint32_t e = e8m0_from_amax(amax);   // csrc/mxfp8.cuh
    const float inv = __uint_as_float((254u - e) << 23);
    uint32_t packed[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        const uint32_t lo = __nv_cvt_float2_to_fp8x2(make_float2(v[4 * j] * inv, v[4 * j + 1] * inv), __NV_SATFINITE, __NV_E4M3);
        const uint32_t hi = __nv_cvt_float2_to_fp8x2(make_float2(v[4 * j + 2] * inv, v[4 * j + 3] * inv), __NV_SATFINITE, __NV_E4M3);
        packed[j] = lo | (hi << 16);
    }
    int4* dst = reinterpret_cast<int4*>(out + grow * ld_out + kb32 * 32);
    dst[0] = make_int4(packed[0], packed[1], packed[2], packed[3]);
    dst[1] = make_int4(packed[4], packed[5], packed[6], packed[7]);
    // scale byte
    const int num_kb = K >> 7;
    const int tiles_per_group = (rows_per_group + tile_rows - 1) / tile_rows;
    const int atoms = (tile_rows + 127) >> 7;
    const int tile = r / tile_rows;
    const int rt = r - tile * tile_rows;
    const int atom = rt >> 7, ra = rt & 127;
    const long long chunk = ((static_cast<long long>(g) * tiles_per_group + tile) * num_kb + (kb32 >> 2)) * atoms + atom;
    sf[chunk * 512 + ((ra & 31) * 4 + (ra >> 5)) * 4 + (kb32 & 3)] = static_cast<uint8_t>(e);
}

// ------------------------------------------------------------------------------------------------ host
template <bool OUT_F32>
static int launch_fp8(const Params& p, const CUtensorMap& tmA, const CUtensorMap& tmB, int max_ctas, cudaStream_t st) {
    if (const int e = set_max_dynamic_smem<gemm_fp8_kernel<OUT_F32>>(SMEM_TOTAL)) return e;
    const long long total = 1ll * p.num_m_tiles * p.n_tiles;
    if (total <= 0) return 0;
    gemm_fp8_kernel<OUT_F32><<<persistent_grid(total, max_ctas), NUM_THREADS, SMEM_TOTAL, st>>>(p, tmA, tmB);
    cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? 0 : -static_cast<int>(e);
}

}  // namespace f8
}  // namespace lah

using namespace lah;
using namespace lah::f8;

extern "C" const int* lah_get_epoch_base();

extern "C" {

// bytes of the scale-factor buffer for `rows` rows per group (tile_rows = 128: activations, 192: weights)
long long lah_mxfp8_sf_bytes(long long rows_per_group, int groups, int K, int tile_rows) {
    return sf_chunks(rows_per_group, tile_rows, K / 128) * groups * 512;
}

// in [groups * rows_per_group, K] (bf16: in_f32 = 0, fp32: 1) -> out e4m3 (same shape, ld_out bytes per row) + scales
int lah_quant_mxfp8(const void* in, long long ld_in, int in_f32, void* out, long long ld_out, void* sf, int rows_per_group,
                    int groups, int K, int tile_rows, const int* tile_group128, const int* total_rows_dev,
                    cudaStream_t stream) {
    if ((K % 128) || (ld_out % 16) || (tile_rows != 128 && tile_rows != 192)) return -2;
    // every thread reads its 32 input elements and writes its 32 payload bytes as 16-byte vectors: the input row stride
    // (in bytes) and both bases must be multiples of 16
    if (((ld_in * (in_f32 ? 4 : 2)) % 16) || (reinterpret_cast<uintptr_t>(in) % 16) || (reinterpret_cast<uintptr_t>(out) % 16))
        return -2;
    const long long threads = static_cast<long long>(rows_per_group) * groups * (K / 32);
    if (threads == 0) return 0;
    const int blocks = static_cast<int>((threads + 255) / 256);
    if (in_f32)
        quant_mxfp8_kernel<float><<<blocks, 256, 0, stream>>>(reinterpret_cast<const float*>(in), ld_in,
                                                             reinterpret_cast<uint8_t*>(out), ld_out,
                                                             reinterpret_cast<uint8_t*>(sf), rows_per_group, groups, K,
                                                             tile_rows, tile_group128, total_rows_dev);
    else
        quant_mxfp8_kernel<bf16><<<blocks, 256, 0, stream>>>(reinterpret_cast<const bf16*>(in), ld_in,
                                                            reinterpret_cast<uint8_t*>(out), ld_out,
                                                            reinterpret_cast<uint8_t*>(sf), rows_per_group, groups, K,
                                                            tile_rows, tile_group128, total_rows_dev);
    cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? 0 : -static_cast<int>(e);
}

// A: e4m3 [a_rows, K] (lda bytes), sfa: activation scales (tile_rows = 128); B: e4m3 [G, N, K], sfb: weight scales
// (tile_rows = 192).  tile_group has one entry per 128 rows.
int lah_gemm_mgroup_fp8(const void* A, long long lda, int a_rows, const void* sfa, const void* B, const void* sfb, int G,
                        int N, int K, void* C, long long ldc, int out_f32, int m_valid, int num_m_tiles128,
                        const int* tile_group, const float* bias, const void* residual, long long ldr, int max_ctas,
                        const int* wait_flags, int wait_count, int wait_epoch, int* status, int act, cudaStream_t stream) {
    if ((K % 128) || (N % 64) || (lda % 16)) return -2;
    // the epilogue reads the residual and writes a bf16 C as 4-byte pairs, writes an fp32 C as 8-byte pairs and reads the
    // bias as float2: even row strides and bases aligned to those widths
    if ((ldc % 2) || (reinterpret_cast<uintptr_t>(C) % (out_f32 ? 8 : 4))) return -2;
    if (residual && ((ldr % 2) || (reinterpret_cast<uintptr_t>(residual) % 4))) return -2;
    if (bias && (reinterpret_cast<uintptr_t>(bias) % 8)) return -2;
    const int num_kb = K / 128;
    const int n_tiles = (N + TILE_N - 1) / TILE_N;
    CUtensorMap tmA, tmB;
    {
        uint64_t dims[2] = {(uint64_t)K, (uint64_t)a_rows};
        uint64_t str[1] = {(uint64_t)lda};
        uint32_t box[2] = {BLOCK_K, TILE_M};
        int r = make_tmap(&tmA, CU_TENSOR_MAP_DATA_TYPE_UINT8, 2, A, dims, str, box);
        if (r) return r;
    }
    {
        uint64_t dims[3] = {(uint64_t)K, (uint64_t)N, (uint64_t)G};
        uint64_t str[2] = {(uint64_t)K, (uint64_t)N * K};
        uint32_t box[3] = {BLOCK_K, TILE_N, 1};
        int r = make_tmap(&tmB, CU_TENSOR_MAP_DATA_TYPE_UINT8, 3, B, dims, str, box);
        if (r) return r;
    }
    Params p;
    p.N = N; p.K = K; p.M = m_valid; p.num_groups = G; p.num_m_tiles = num_m_tiles128; p.n_tiles = n_tiles;
    p.num_kb = num_kb; p.tile_group = tile_group; p.C = C; p.ldc = ldc; p.bias = bias;
    p.residual = reinterpret_cast<const bf16*>(residual); p.ldr = ldr;
    p.wait_flags = wait_flags; p.wait_count = wait_count; p.wait_epoch = wait_epoch; p.epoch_base = lah_get_epoch_base(); p.status = status; p.act = act;
    p.sfa = reinterpret_cast<const uint32_t*>(sfa); p.sfb = reinterpret_cast<const uint32_t*>(sfb);
    return out_f32 ? launch_fp8<true>(p, tmA, tmB, max_ctas, stream)
                   : launch_fp8<false>(p, tmA, tmB, max_ctas, stream);
}

}  // extern "C"
