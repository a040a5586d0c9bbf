// grouped_gemm.cu — persistent, warp-specialised wgmma GEMM for sm_90a.
//
// One kernel template covers every GEMM-shaped op of the DMoE expert path
// (reference hot loops: experiments/throughput/layers.py:8-19 forward, lib/runtime/expert_backend.py:73-93 backward):
//
//   MODE_MGROUP  C[rows, N] = act(A[rows, K] * B[g(rows)]^T (+bias[g])) (+residual)
//                rows are grouped by expert, every group padded to a multiple of 128 rows; the group of a
//                128-row tile comes from a device-side table written by the dispatch kernel (no host sync).
//                B is either K-major  ([G, N, K], forward:  x @ W^T)
//                      or MN-major    ([G, K, N], dgrad:    dy @ W  with W stored [K=out, N=in]).
//   MODE_KGROUP  C[g][M, N] (+)= A_g^T * B_g   (wgrad: dW = dY^T X, reduction over the tokens of expert g)
//                A = dY [tokens, M], B = X [tokens, N], both "MN-major" operands; fp32 output per group.
//
// Structure (one CTA per SM, 288 threads):
//   warps 0-7  two consumer warpgroups: warpgroup w owns rows [64w, 64w + 64) of the 128 x BLOCK_N tile, issues
//              wgmma.m64nBLOCK_Nk16 from the shared-memory ring (accumulator in registers) and runs the epilogue
//              (bias / activation / residual / accumulate -> bf16 | fp32 -> global) straight from its registers
//   warp 8     TMA producer (one lane): cp.async.bulk.tensor -> 128B-swizzled smem ring, mbarrier complete_tx; it runs
//              ahead into the next tile while the consumers drain the previous one
#include "sm90.cuh"

namespace lah {

constexpr int BLOCK_M = 128;
constexpr int BLOCK_K = 64;   // 64 bf16 = 128 bytes = one swizzle-128B row
constexpr int MMA_K = 16;
constexpr int NUM_THREADS = 288;
constexpr int MODE_MGROUP = 0;
constexpr int MODE_KGROUP = 1;

struct GemmParams {
    int N;               // columns of C
    int K;               // MGROUP: reduction length
    int M;               // KGROUP: rows of C per group (multiple of 128). MGROUP: number of valid rows of C.
    int num_groups;      // KGROUP: number of groups
    int num_m_tiles;     // MGROUP: number of 128-row tiles to visit (upper bound; unused tiles have group -1)
    const int* tile_group;  // MGROUP: [num_m_tiles] group of each m tile, -1 = skip; nullptr => group 0
    const int* group_off;   // KGROUP: [G+1] padded token offsets (multiples of 128)
    void* C;
    long long ldc;
    long long c_group_stride;  // KGROUP: elements between consecutive groups of C
    const float* bias;         // MGROUP: [G, N] or nullptr
    const bf16* residual;      // MGROUP: [rows, ldr] or nullptr
    long long ldr;
    // receive-side fusion: the TMA producer waits until every source rank's dispatch flag reached `wait_epoch`
    const int* wait_flags;     // [wait_count] local flag words written by the peers (st.release.sys), or nullptr
    int wait_count, wait_epoch;
    const int* epoch_base;   // device-side epoch base added to wait_epoch (nullptr: 0), see moe.cu Peers::step_ctr
    int* status;
    int act;                 // MGROUP epilogue activation after the bias: 0 none, 1 ReLU, 2 GELU (erf)
    int accumulate;          // KGROUP: C += result (gradient accumulation across steps, update_every_*)
};

template <int BLOCK_N, int STAGES>
struct SmemLayout {
    static constexpr int A_BYTES = BLOCK_M * BLOCK_K * 2;
    static constexpr int B_BYTES = BLOCK_N * BLOCK_K * 2;
    static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
    static constexpr int BAR_OFFSET = STAGES * STAGE_BYTES;
    static constexpr int TOTAL = BAR_OFFSET + 2 * STAGES * 8 + 1024;  // + alignment slack
    static_assert(TOTAL <= 227 * 1024, "shared memory budget");
};

template <int BLOCK_N, bool A_MN, bool B_MN>
__device__ __forceinline__ void mma_kblock(float (&acc)[BLOCK_N / 2], uint32_t sa, uint32_t sb, int wg, bool first) {
    // A: this warpgroup's 64 rows. K-major: rows 64wg.. (8 KB in). MN-major: the wg-th 64-wide atom (BLOCK_K*128 B).
    const uint32_t a0 = sa + wg * (A_MN ? BLOCK_K * 128 : 64 * 128);
    constexpr uint32_t A_KSTEP = A_MN ? MMA_K * 128 : MMA_K * 2, B_KSTEP = B_MN ? MMA_K * 128 : MMA_K * 2;
    constexpr uint32_t LBO = BLOCK_K * 128;
#pragma unroll
    for (int k = 0; k < BLOCK_K / MMA_K; ++k) {
        const uint64_t da = make_smem_desc_sw128(a0 + k * A_KSTEP, LBO, 1024);
        const uint64_t db = make_smem_desc_sw128(sb + k * B_KSTEP, LBO, 1024);
        const uint32_t accum = (first && k == 0) ? 0u : 1u;
        if constexpr (BLOCK_N == 256) wgmma_bf16_n256<A_MN, B_MN>(acc, da, db, accum);
        if constexpr (BLOCK_N == 128) wgmma_bf16_n128<A_MN, B_MN>(acc, da, db, accum);
        if constexpr (BLOCK_N == 64) wgmma_bf16_n64<A_MN, B_MN>(acc, da, db, accum);
    }
}

template <int BLOCK_N, int STAGES, int MODE, bool A_MN, bool B_MN, bool OUT_F32>
__global__ void __launch_bounds__(NUM_THREADS, 1)
gemm_kernel(const GemmParams p, const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB) {
    using L = SmemLayout<BLOCK_N, STAGES>;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + L::BAR_OFFSET);
    uint64_t* empty_bar = full_bar + STAGES;

    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;

    if (warp == 8 && lane == 0) {
        tma_prefetch_desc(&tmA);
        tma_prefetch_desc(&tmB);
        for (int i = 0; i < STAGES; ++i) {
            mbar_init(&full_bar[i], 1);
            mbar_init(&empty_bar[i], 8);  // one arrive per consumer warp
        }
        fence_mbar_init();
    }
    __syncthreads();

    // ------------------------------------------------------------------ tile enumeration
    const int n_tiles = (p.N + BLOCK_N - 1) / BLOCK_N;
    int total_tiles, tiles_per_group = 0;
    if (MODE == MODE_MGROUP) {
        total_tiles = p.num_m_tiles * n_tiles;
    } else {
        tiles_per_group = (p.M / BLOCK_M) * n_tiles;
        total_tiles = p.num_groups * tiles_per_group;
    }

    // decode one tile; returns false when the tile must be skipped (identical decision in all roles)
    auto decode = [&](int tile, int& m_row, int& n_col, int& group, int& k_begin, int& num_kb) -> bool {
        if (MODE == MODE_MGROUP) {
            const int m_tile = tile / n_tiles;
            const int n_tile = tile - m_tile * n_tiles;
            group = p.tile_group ? __ldg(p.tile_group + m_tile) : 0;
            m_row = m_tile * BLOCK_M;
            n_col = n_tile * BLOCK_N;
            k_begin = 0;
            num_kb = (p.K + BLOCK_K - 1) / BLOCK_K;
            return group >= 0;
        } else {
            group = tile / tiles_per_group;
            const int r = tile - group * tiles_per_group;
            const int m_tile = r / n_tiles;
            const int n_tile = r - m_tile * n_tiles;
            m_row = m_tile * BLOCK_M;
            n_col = n_tile * BLOCK_N;
            k_begin = __ldg(p.group_off + group);
            num_kb = (__ldg(p.group_off + group + 1) - k_begin) / BLOCK_K;
            return num_kb > 0;
        }
    };

    if (warp == 8) {
        if (lane != 0) return;
        // =============================================================== TMA producer
        if (p.wait_flags) {  // rows pushed by peer GPUs over NVLink must have landed before the first TMA load
            const unsigned long long t_wait = globaltimer_ns();
            for (int sidx = 0; sidx < p.wait_count; ++sidx)
                spin_flag_ft(p.wait_flags + sidx, p.wait_epoch + (p.epoch_base ? p.epoch_base[0] : 0), p.status, sidx,
                             p.epoch_base ? p.epoch_base[1] : 0);
            // exposed communication wait (ns) of this rank: status[2..3] is a 64-bit counter (EngineContext.wait_ns)
            if (blockIdx.x == 0) atomicAdd(reinterpret_cast<unsigned long long*>(p.status + 2), globaltimer_ns() - t_wait);
            fence_proxy_async_global();
        }
        int stage = 0;
        uint32_t phase = 0;
        for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
            int m_row, n_col, g, k_begin, num_kb;
            if (!decode(tile, m_row, n_col, g, k_begin, num_kb)) continue;
            for (int kb = 0; kb < num_kb; ++kb) {
                mbar_wait(&empty_bar[stage], phase ^ 1);
                uint8_t* sa = smem + stage * L::STAGE_BYTES;
                uint8_t* sb = sa + L::A_BYTES;
                const int k = k_begin + kb * BLOCK_K;
                mbar_arrive_expect_tx(&full_bar[stage], L::STAGE_BYTES);
                // ---- A
                if (!A_MN) {
                    tma_load_2d(sa, &tmA, &full_bar[stage], k, m_row);
                } else {
#pragma unroll
                    for (int i = 0; i < BLOCK_M / 64; ++i)
                        tma_load_2d(sa + i * (BLOCK_K * 128), &tmA, &full_bar[stage], m_row + i * 64, k);
                }
                // ---- B
                if (MODE == MODE_MGROUP) {
                    if (!B_MN) {
                        tma_load_3d(sb, &tmB, &full_bar[stage], k, n_col, g);
                    } else {
#pragma unroll
                        for (int i = 0; i < BLOCK_N / 64; ++i)
                            tma_load_3d(sb + i * (BLOCK_K * 128), &tmB, &full_bar[stage], n_col + i * 64, k, g);
                    }
                } else {
                    if (!B_MN) {
                        tma_load_2d(sb, &tmB, &full_bar[stage], k, n_col);
                    } else {
#pragma unroll
                        for (int i = 0; i < BLOCK_N / 64; ++i)
                            tma_load_2d(sb + i * (BLOCK_K * 128), &tmB, &full_bar[stage], n_col + i * 64, k);
                    }
                }
                if (++stage == STAGES) {
                    stage = 0;
                    phase ^= 1;
                }
            }
        }
        return;
    }

    // =================================================================== consumers (two warpgroups)
    const int wg = warp >> 2;
    const int row_in_tile = wg * 64 + (warp & 3) * 16 + (lane >> 2);   // and + 8
    const int col_in_tile = 2 * (lane & 3);                             // + 8 j (+ 1)
    int stage = 0;
    uint32_t phase = 0;
    float acc[BLOCK_N / 2];
    for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
        int m_row, n_col, g, k_begin, num_kb;
        if (!decode(tile, m_row, n_col, g, k_begin, num_kb)) continue;
        int prev_stage = -1;
        for (int kb = 0; kb < num_kb; ++kb) {
            mbar_wait(&full_bar[stage], phase);
            const uint32_t sa = smem_u32(smem + stage * L::STAGE_BYTES);
            wgmma_fence();
            mma_kblock<BLOCK_N, A_MN, B_MN>(acc, sa, sa + L::A_BYTES, wg, kb == 0);
            wgmma_commit();
            wgmma_wait<1>();   // the k-block before this one is done: release its stage
            if (prev_stage >= 0) {
                __syncwarp();
                if (lane == 0) mbar_arrive(&empty_bar[prev_stage]);
            }
            prev_stage = stage;
            if (++stage == STAGES) {
                stage = 0;
                phase ^= 1;
            }
        }
        wgmma_wait<0>();
        wgmma_fence_regs(acc);
        __syncwarp();
        if (lane == 0) mbar_arrive(&empty_bar[prev_stage]);

        // ------------------------------------------------------------ epilogue from registers
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int row = m_row + row_in_tile + 8 * h;
            const bool row_ok = (MODE == MODE_KGROUP) ? true : (row < p.M);
            if (!row_ok) continue;
            const long long gbase = (MODE == MODE_KGROUP ? static_cast<long long>(g) * p.c_group_stride : 0ll) +
                                    static_cast<long long>(row) * p.ldc;
#pragma unroll
            for (int j = 0; j < BLOCK_N / 8; ++j) {
                const int col = n_col + 8 * j + col_in_tile;
                if (col >= p.N) continue;
                float v0 = acc[4 * j + 2 * h], v1 = acc[4 * j + 2 * h + 1];
                if (MODE == MODE_MGROUP) {
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
                }
                if (OUT_F32) {
                    float2* cp = reinterpret_cast<float2*>(reinterpret_cast<float*>(p.C) + gbase + col);
                    if (MODE == MODE_KGROUP && p.accumulate) {
                        const float2 o = *cp;
                        v0 += o.x;
                        v1 += o.y;
                    }
                    *cp = make_float2(v0, v1);
                } else {
                    *reinterpret_cast<uint32_t*>(reinterpret_cast<bf16*>(p.C) + gbase + col) = pack_bf16x2(v0, v1);
                }
            }
        }
    }
}

// ------------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------------
typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static PFN_encodeTiled get_encode_fn() {
    static PFN_encodeTiled fn = nullptr;
    if (!fn) {
        void* ptr = nullptr;
        cudaDriverEntryPointQueryResult qres;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &ptr, cudaEnableDefault, &qres) != cudaSuccess || !ptr)
            return nullptr;
        fn = reinterpret_cast<PFN_encodeTiled>(ptr);
    }
    return fn;
}

// bf16 tensor map, up to 3 dims (dim0 = contiguous), 128B swizzle, zero OOB fill.
static int make_tmap_bf16(CUtensorMap* tm, const void* ptr, int rank, const uint64_t* dims, const uint64_t* strides_bytes,
                          const uint32_t* box) {
    PFN_encodeTiled fn = get_encode_fn();
    if (!fn) return -100;
    cuuint64_t gdims[3];
    cuuint64_t gstr[2];
    cuuint32_t gbox[3];
    cuuint32_t estr[3] = {1, 1, 1};
    for (int i = 0; i < rank; ++i) {
        gdims[i] = dims[i];
        gbox[i] = box[i];
    }
    for (int i = 0; i < rank - 1; ++i) gstr[i] = strides_bytes[i];
    CUresult r = fn(tm, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, rank, const_cast<void*>(ptr), gdims, gstr, gbox, estr,
                    CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                    CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    return r == CUDA_SUCCESS ? 0 : -static_cast<int>(r) - 1000;
}

static int g_num_sms = 0;
static int num_sms() {
    if (!g_num_sms) {
        int dev = 0;
        cudaGetDevice(&dev);
        cudaDeviceGetAttribute(&g_num_sms, cudaDevAttrMultiProcessorCount, dev);
    }
    return g_num_sms;
}

template <int BLOCK_N, int STAGES, int MODE, bool A_MN, bool B_MN, bool OUT_F32>
static int launch(const GemmParams& p, const CUtensorMap& tmA, const CUtensorMap& tmB, int max_ctas, cudaStream_t st) {
    using L = SmemLayout<BLOCK_N, STAGES>;
    auto kern = gemm_kernel<BLOCK_N, STAGES, MODE, A_MN, B_MN, OUT_F32>;
    static bool configured = false;
    if (!configured) {
        cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, L::TOTAL);
        if (e != cudaSuccess) return -static_cast<int>(e);
        configured = true;
    }
    const int n_tiles = (p.N + BLOCK_N - 1) / BLOCK_N;
    long long total = (MODE == MODE_MGROUP) ? 1ll * p.num_m_tiles * n_tiles : 1ll * p.num_groups * (p.M / BLOCK_M) * n_tiles;
    if (total <= 0) return 0;
    int grid = num_sms();
    if (max_ctas > 0 && max_ctas < grid) grid = max_ctas;
    if (total < grid) grid = static_cast<int>(total);
    kern<<<grid, NUM_THREADS, L::TOTAL, st>>>(p, tmA, tmB);
    cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? 0 : -static_cast<int>(e);
}

static int gemm_mgroup(const void* A, long long lda, int a_rows, const void* B, int G, int N, int K, int b_mn, void* C,
                       long long ldc, int out_f32, int m_valid, int num_m_tiles, const int* tile_group, const float* bias,
                       const void* residual, long long ldr, int block_n, int max_ctas, const int* wait_flags,
                       int wait_count, int wait_epoch, int* status, int act, const int* epoch_base, cudaStream_t stream) {
    if ((K % 8) || (N % 32) || (lda % 8)) return -2;
    if (block_n != 256 && block_n != 128 && block_n != 64) return -3;
    CUtensorMap tmA, tmB;
    {
        uint64_t dims[2] = {(uint64_t)K, (uint64_t)a_rows};
        uint64_t str[1] = {(uint64_t)lda * 2};
        uint32_t box[2] = {BLOCK_K, BLOCK_M};
        int r = make_tmap_bf16(&tmA, A, 2, dims, str, box);
        if (r) return r;
    }
    if (!b_mn) {
        uint64_t dims[3] = {(uint64_t)K, (uint64_t)N, (uint64_t)G};
        uint64_t str[2] = {(uint64_t)K * 2, (uint64_t)N * K * 2};
        uint32_t box[3] = {BLOCK_K, (uint32_t)block_n, 1};
        int r = make_tmap_bf16(&tmB, B, 3, dims, str, box);
        if (r) return r;
    } else {
        uint64_t dims[3] = {(uint64_t)N, (uint64_t)K, (uint64_t)G};
        uint64_t str[2] = {(uint64_t)N * 2, (uint64_t)N * K * 2};
        uint32_t box[3] = {64, BLOCK_K, 1};
        int r = make_tmap_bf16(&tmB, B, 3, dims, str, box);
        if (r) return r;
    }
    GemmParams p;
    p.N = N; p.K = K; p.M = m_valid; p.num_groups = G; p.num_m_tiles = num_m_tiles; p.tile_group = tile_group;
    p.group_off = nullptr; p.C = C; p.ldc = ldc; p.c_group_stride = 0; p.bias = bias;
    p.residual = reinterpret_cast<const bf16*>(residual); p.ldr = ldr;
    p.wait_flags = wait_flags; p.wait_count = wait_count; p.wait_epoch = wait_epoch; p.epoch_base = epoch_base; p.status = status;
    p.act = act; p.accumulate = 0;
#define LAH_LAUNCH_M(BN, ST)                                                                                   \
    if (!b_mn && !out_f32) return launch<BN, ST, MODE_MGROUP, false, false, false>(p, tmA, tmB, max_ctas, stream); \
    if (b_mn && !out_f32) return launch<BN, ST, MODE_MGROUP, false, true, false>(p, tmA, tmB, max_ctas, stream);   \
    if (!b_mn && out_f32) return launch<BN, ST, MODE_MGROUP, false, false, true>(p, tmA, tmB, max_ctas, stream);   \
    return launch<BN, ST, MODE_MGROUP, false, true, true>(p, tmA, tmB, max_ctas, stream);
    if (block_n == 256) { LAH_LAUNCH_M(256, 4) }
    if (block_n == 128) { LAH_LAUNCH_M(128, 6) }
    LAH_LAUNCH_M(64, 8)
#undef LAH_LAUNCH_M
}

static int gemm_kgroup(const void* A, long long lda, const void* B, long long ldb, int total_rows, int G, int M, int N,
                       const int* group_off, float* C, long long ldc, long long c_group_stride, int block_n, int max_ctas,
                       int accumulate, cudaStream_t stream) {
    if ((M % 128) || (N % 32) || (lda % 8) || (ldb % 8)) return -2;
    CUtensorMap tmA, tmB;
    {
        uint64_t dims[2] = {(uint64_t)M, (uint64_t)total_rows};
        uint64_t str[1] = {(uint64_t)lda * 2};
        uint32_t box[2] = {64, BLOCK_K};
        int r = make_tmap_bf16(&tmA, A, 2, dims, str, box);
        if (r) return r;
    }
    {
        uint64_t dims[2] = {(uint64_t)N, (uint64_t)total_rows};
        uint64_t str[1] = {(uint64_t)ldb * 2};
        uint32_t box[2] = {64, BLOCK_K};
        int r = make_tmap_bf16(&tmB, B, 2, dims, str, box);
        if (r) return r;
    }
    GemmParams p;
    p.N = N; p.K = 0; p.M = M; p.num_groups = G; p.num_m_tiles = 0; p.tile_group = nullptr; p.group_off = group_off;
    p.C = C; p.ldc = ldc; p.c_group_stride = c_group_stride; p.bias = nullptr; p.residual = nullptr; p.ldr = 0;
    p.wait_flags = nullptr; p.wait_count = 0; p.wait_epoch = 0; p.epoch_base = nullptr; p.status = nullptr;
    p.act = 0; p.accumulate = accumulate;
    if (block_n == 256) return launch<256, 4, MODE_KGROUP, true, true, true>(p, tmA, tmB, max_ctas, stream);
    if (block_n == 128) return launch<128, 6, MODE_KGROUP, true, true, true>(p, tmA, tmB, max_ctas, stream);
    if (block_n == 64) return launch<64, 8, MODE_KGROUP, true, true, true>(p, tmA, tmB, max_ctas, stream);
    return -3;
}

}  // namespace lah

using namespace lah;

// ------------------------------------------------------------------------------------------------
// C ABI (called from python via ctypes; see ops/native.py)
// ------------------------------------------------------------------------------------------------
extern "C" const int* lah_get_epoch_base();

extern "C" {

// C[rows, N] = A[rows, K] @ B[g]^T (+bias) (+residual)
//   b_mn == 0: B is [G, N, K] (K contiguous);  b_mn == 1: B is [G, K, N] (N contiguous)
//   a_rows: rows of the A buffer (TMA bound); m_valid: rows of C that may be written
//   tile_group: device int[num_m_tiles] or null; out_f32: 0 => bf16 C, 1 => fp32 C
int lah_gemm_mgroup(const void* A, long long lda, int a_rows, const void* B, int G, int N, int K, int b_mn, void* C,
                    long long ldc, int out_f32, int m_valid, int num_m_tiles, const int* tile_group,
                    const float* bias, const void* residual, long long ldr, int block_n, int max_ctas,
                    const int* wait_flags, int wait_count, int wait_epoch, int* status, cudaStream_t stream) {
    return gemm_mgroup(A, lda, a_rows, B, G, N, K, b_mn, C, ldc, out_f32, m_valid, num_m_tiles, tile_group, bias, residual,
                       ldr, block_n, max_ctas, wait_flags, wait_count, wait_epoch, status, 0, lah_get_epoch_base(), stream);
}

// C[g][M, N] (fp32) = A[off[g]:off[g+1], :M]^T @ B[off[g]:off[g+1], :N]   (A, B row-major token matrices)
int lah_gemm_kgroup(const void* A, long long lda, const void* B, long long ldb, int total_rows, int G, int M, int N,
                    const int* group_off, float* C, long long ldc, long long c_group_stride, int block_n,
                    int max_ctas, cudaStream_t stream) {
    return gemm_kgroup(A, lda, B, ldb, total_rows, G, M, N, group_off, C, ldc, c_group_stride, block_n, max_ctas, 0, stream);
}

// Wide-tile entry points of the big-batch expert path (expert groups padded to 256 rows, N a multiple of 256):
// 128 x 256 tiles with the fused epilogue activation (act: 0 none, 1 ReLU, 2 GELU) and, for the weight gradient,
// accumulation into C across steps.  tile_group has one entry per 128 rows.
int lah_gemm_mgroup2(const void* A, long long lda, int a_rows, const void* B, int G, int N, int K, int b_mn, void* C,
                     long long ldc, int out_f32, int m_valid, int num_m_tiles128, const int* tile_group,
                     const float* bias, const void* residual, long long ldr, int max_ctas, const int* wait_flags,
                     int wait_count, int wait_epoch, int* status, int act, cudaStream_t stream) {
    return gemm_mgroup(A, lda, a_rows, B, G, N, K, b_mn, C, ldc, out_f32, m_valid, num_m_tiles128, tile_group, bias,
                       residual, ldr, 256, max_ctas, wait_flags, wait_count, wait_epoch, status, act, lah_get_epoch_base(),
                       stream);
}

int lah_gemm_kgroup2(const void* A, long long lda, const void* B, long long ldb, int total_rows, int G, int M, int N,
                     const int* group_off, float* C, long long ldc, long long c_group_stride, int max_ctas,
                     int accumulate, cudaStream_t stream) {
    if (N % 256) return -2;
    return gemm_kgroup(A, lda, B, ldb, total_rows, G, M, N, group_off, C, ldc, c_group_stride, 256, max_ctas, accumulate,
                       stream);
}

}  // extern "C"
