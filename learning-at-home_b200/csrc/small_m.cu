// small_m.cu — the "many small requests" regime of the reference (64 trainers x batch 4 -> O(1..64) rows per expert and
// step; reference: experiments/convergence notebooks, lib/runtime/task_pool.py:105-125) on sm_90a.
//
// With a handful of rows per expert every expert GEMM is a WEIGHT-STREAMING problem (12.6 MB of bf16 weights per
// active expert and forward at hid 512) and the optimizer is a STATE-STREAMING problem (fp32 p, m, v, vmax).  Two
// kernels, both persistent / warp-specialised / TMA-fed, with wgmma accumulators in registers (two consumer warpgroups of
// 64 MMA rows each, one TMA producer warp):
//
//   swapab_kernel      D^T[out_features, tokens] = W[out_features, K] * X^T[K, tokens]   ("swap-AB": the weights sit on
//                      the 128-wide MMA-M side, the expert's 16..128 tokens on the MMA-N side, so a group of 16 rows
//                      costs N=16 instructions instead of a 128-row padded tile).  A tile = (expert, 128-token
//                      chunk, 128-row slice of the weight matrix) streamed through a 6-stage TMA ring; experts with
//                      more than 128 rows are spread over several CTAs (hot experts).  A_MN selects dgrad
//                      (W^T read straight from the same [out, in] tensor as an MN-major operand).
//   wgrad_adam_kernel  dW tile = dY^T X with wgmma (both operands MN-major, two 32-token stages, reduction over the
//                      expert's tokens = the gradient reduction over all trainers that routed to it) with the per-expert AMSGrad step FUSED
//                      INTO THE EPILOGUE: every thread reads p / m / v / vmax at the positions of its accumulator
//                      registers (four 8-column groups at a time, so 32 loads are in flight per thread), updates them
//                      and writes them back together with the bf16 mirror.  The weight gradient never exists in HBM: 34 B / parameter
//                      instead of 46 (wgrad write 4 + Adam 38 + re-read 4).
//                      Reference semantics: one torch.optim.Adam(amsgrad=True) step per expert right after its backward
//                      (/root/reference/lib/runtime/expert_backend.py:90-97).
#include "sm90.cuh"

namespace lah {
namespace smallm {

constexpr int BM = 128;      // MMA M: weight rows (swapab) / dY features (wgrad)
constexpr int BK = 64;       // k elements per stage row (128 B of bf16 = one swizzle row)
constexpr int MMA_K = 16;
constexpr int BN_MAX = 128;  // max tokens per MMA (swapab) / X features per tile (wgrad)
constexpr int NUM_THREADS = 288;   // two consumer warpgroups + one producer warp

typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static PFN_encodeTiled encode_fn() {
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

static int make_tmap(CUtensorMap* tm, CUtensorMapDataType dt, int esize, const void* ptr, int rank, const uint64_t* dims,
                     const uint64_t* strides_bytes, const uint32_t* box) {
    PFN_encodeTiled fn = encode_fn();
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
    (void)esize;
    CUresult r = fn(tm, dt, rank, const_cast<void*>(ptr), gdims, gstr, gbox, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                    CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    return r == CUDA_SUCCESS ? 0 : -static_cast<int>(r) - 1000;
}

static int num_sms() {
    static int sms = 0;
    if (!sms) {
        int dev = 0;
        cudaGetDevice(&dev);
        cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    }
    return sms;
}

// =====================================================================================================================
// swap-AB grouped linear
// =====================================================================================================================
namespace sab {

constexpr int STAGES = 6;
constexpr int A_BYTES = BM * BK * 2;          // 16 KB
constexpr int B_BYTES = BN_MAX * BK * 2;      // 16 KB (only box_rows * 128 B are filled)
constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
constexpr int BAR_OFFSET = STAGES * STAGE_BYTES;
constexpr int QD = 4;                         // depth of the tile queue (dynamic scheduler)
constexpr int MAX_G = 1023;                   // groups per launch (prefix table of 128-token chunks lives in smem)
constexpr int CUM_OFFSET = BAR_OFFSET + (2 * STAGES + 2 * QD) * 8 + QD * 4 + 16;
constexpr int SMEM_TOTAL = CUM_OFFSET + (MAX_G + 1) * 4 + 1024;
static_assert(SMEM_TOTAL <= 232448, "shared memory budget");

struct Params {
    int G, M_out, K;          // groups, output features (rows of the weight operand), reduction length
    const int* group_off;     // [G] first row of the group inside the token-major buffers
    const int* group_rows;    // [G] valid rows (0: skip the group)
    bf16* out;                // [rows, M_out]  token-major
    long long ldo;
    const float* bias;        // [G, M_out] or nullptr
    const bf16* residual;     // [rows, ldr] or nullptr
    long long ldr;
    const int* wait_flags;    // receive-side fusion: rows pushed by the peers must have landed (see grouped_gemm.cu)
    int wait_count, wait_epoch;
    const int* epoch_base;    // optional device-side epoch base added to wait_epoch (CUDA-graph replay)
    int* status;
    int* tile_counter;        // work-stealing tile counter (zeroed before the launch)
};

__device__ __forceinline__ int box_rows_of(int nn) { return nn <= 16 ? 16 : (nn <= 32 ? 32 : (nn <= 64 ? 64 : 128)); }

// Tiles are handed out DYNAMICALLY: SMs do not get equal shares of HBM bandwidth (a static split leaves the fast SMs idle
// while they wait for the slowest one), so the TMA-producer thread of every CTA draws the next tile from a global
// counter and publishes it to the consumer warps of its CTA through a small smem queue.
// A tile is (group, 128-token chunk, 128-feature slice): a HOT expert (routing collapses while training; with 8 experts per
// rank one of them can hold > 1000 of the rank's rows) is split over as many CTAs as it has chunks instead of one CTA
// walking all of its chunks back to back - the slowest rank of a step is the one that owns the hottest expert, and every
// other rank waits for it in the combine.  Every CTA builds the prefix table of chunks per group in shared memory.
__device__ __forceinline__ int find_group(const int* cum, int G, int gc) {   // largest g with cum[g] <= gc
    int lo = 0, hi = G - 1;
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (cum[mid] <= gc) lo = mid; else hi = mid - 1;
    }
    return lo;
}

// mainloop + epilogue of one tile for a token box of NB rows (MMA N = NB); warpgroup wg owns weight rows [64wg, 64wg + 64)
template <int NB, bool A_MN>
__device__ __forceinline__ void sab_tile(const Params& p, uint8_t* smem, uint64_t* full_bar, uint64_t* empty_bar, int& stage,
                                         uint32_t& phase, int num_kb, int wg, int warp, int lane, int g, int ms, int row0,
                                         int nn) {
    float acc[NB / 2];
    constexpr uint32_t A_KSTEP = A_MN ? MMA_K * 128 : MMA_K * 2;
    int prev_stage = -1;
    for (int kb = 0; kb < num_kb; ++kb) {
        mbar_wait(&full_bar[stage], phase);
        const uint32_t sa = smem_u32(smem + stage * STAGE_BYTES) + wg * (A_MN ? BK * 128 : 64 * 128);
        const uint32_t sb = smem_u32(smem + stage * STAGE_BYTES + A_BYTES);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < BK / MMA_K; ++k) {
            const uint64_t da = make_smem_desc_sw128(sa + k * A_KSTEP, BK * 128, 1024);
            const uint64_t db = make_smem_desc_sw128(sb + k * (MMA_K * 2), 0, 1024);
            const uint32_t accum = (kb > 0 || k > 0) ? 1u : 0u;
            if constexpr (NB == 16) wgmma_bf16_n16<A_MN, 0>(acc, da, db, accum);
            if constexpr (NB == 32) wgmma_bf16_n32<A_MN, 0>(acc, da, db, accum);
            if constexpr (NB == 64) wgmma_bf16_n64<A_MN, 0>(acc, da, db, accum);
            if constexpr (NB == 128) wgmma_bf16_n128<A_MN, 0>(acc, da, db, accum);
        }
        wgmma_commit();
        wgmma_wait<1>();
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
    if (lane == 0 && prev_stage >= 0) mbar_arrive(&empty_bar[prev_stage]);

    // epilogue: accumulator row = output feature, column = token.  The padding rows of the group's last 16-row block are
    // WRITTEN too (their inputs are zero rows, so they get bias / zero): every later kernel may then read whole 16-row
    // blocks without meeting stale memory, and the k-step masked wgrad sees exact zeros there
    const int n16 = (nn + 15) & ~15;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        const int feat = ms * BM + wg * 64 + (warp & 3) * 16 + (lane >> 2) + 8 * h;
        const float bias = p.bias ? __ldg(p.bias + static_cast<long long>(g) * p.M_out + feat) : 0.f;
#pragma unroll
        for (int j = 0; j < NB / 8; ++j) {
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                const int n = 8 * j + 2 * (lane & 3) + e;
                if (n < n16) {
                    const long long row = row0 + n;
                    float v = acc[4 * j + 2 * h + e] + bias;
                    if (p.residual) v += __bfloat162float(p.residual[row * p.ldr + feat]);
                    p.out[row * p.ldo + feat] = __float2bfloat16(v);
                }
            }
        }
    }
}

template <bool A_MN>
__global__ void __launch_bounds__(NUM_THREADS, 1)
swapab_kernel(const Params p, const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB16,
              const __grid_constant__ CUtensorMap tmB32, const __grid_constant__ CUtensorMap tmB64,
              const __grid_constant__ CUtensorMap tmB128) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + BAR_OFFSET);
    uint64_t* empty_bar = full_bar + STAGES;
    uint64_t* q_full = empty_bar + STAGES;
    uint64_t* q_empty = q_full + QD;
    volatile int* q_tile = reinterpret_cast<volatile int*>(q_empty + QD);
    int* cum = reinterpret_cast<int*>(smem + CUM_OFFSET);   // cum[g] = 128-token chunks of the groups before g

    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;

    if (warp == 0) {   // prefix table of chunks (warp scan, 32 groups per round)
        int carry = 0;
        for (int base = 0; base < p.G; base += 32) {
            const int g = base + lane;
            int x = g < p.G ? (__ldg(p.group_rows + g) + BN_MAX - 1) / BN_MAX : 0;
#pragma unroll
            for (int d = 1; d < 32; d <<= 1) {
                const int y = __shfl_up_sync(0xffffffffu, x, d);
                if (lane >= d) x += y;
            }
            if (g < p.G) cum[g + 1] = carry + x;
            carry += __shfl_sync(0xffffffffu, x, 31);
        }
        if (lane == 0) cum[0] = 0;
    }
    if (warp == 8 && lane == 0) {
        tma_prefetch_desc(&tmA);
        tma_prefetch_desc(&tmB16);
        tma_prefetch_desc(&tmB32);
        tma_prefetch_desc(&tmB64);
        tma_prefetch_desc(&tmB128);
        for (int i = 0; i < STAGES; ++i) {
            mbar_init(&full_bar[i], 1);
            mbar_init(&empty_bar[i], 8);   // one arrive per consumer warp
        }
        for (int i = 0; i < QD; ++i) {
            mbar_init(&q_full[i], 1);
            mbar_init(&q_empty[i], 8);
        }
        fence_mbar_init();
    }
    __syncthreads();

    const int m_slices = p.M_out / BM;
    const int total = cum[p.G] * m_slices;
    const int num_kb = p.K / BK;

    if (warp == 8) {
        if (lane != 0) return;
        // =============================================================== scheduler + TMA producer
        if (p.wait_flags) {
            const int epoch = p.wait_epoch + (p.epoch_base ? *p.epoch_base : 0);
            const unsigned long long t_wait = globaltimer_ns();
            for (int sidx = 0; sidx < p.wait_count; ++sidx)
                spin_flag_ft(p.wait_flags + sidx, epoch, p.status, sidx, p.epoch_base ? p.epoch_base[1] : 0);
            if (blockIdx.x == 0) atomicAdd(reinterpret_cast<unsigned long long*>(p.status + 2), globaltimer_ns() - t_wait);
            fence_proxy_async_global();
        }
        int stage = 0, qi = 0;
        uint32_t phase = 0, qphase = 0;
        while (true) {
            const int tile = atomicAdd(p.tile_counter, 1);
            mbar_wait(&q_empty[qi], qphase ^ 1);
            q_tile[qi] = tile;
            mbar_arrive(&q_full[qi]);
            if (++qi == QD) {
                qi = 0;
                qphase ^= 1;
            }
            if (tile >= total) break;
            const int gc = tile / m_slices, ms = tile - gc * m_slices;
            const int g = find_group(cum, p.G, gc);
            const int n0 = (gc - cum[g]) * BN_MAX;
            const int rows = __ldg(p.group_rows + g);
            const int off = __ldg(p.group_off + g);
            const int box = box_rows_of(min(rows - n0, BN_MAX));
            const CUtensorMap* tmB = box == 16 ? &tmB16 : (box == 32 ? &tmB32 : (box == 64 ? &tmB64 : &tmB128));
            for (int kb = 0; kb < num_kb; ++kb) {
                mbar_wait(&empty_bar[stage], phase ^ 1);
                uint8_t* sa = smem + stage * STAGE_BYTES;
                uint8_t* sb = sa + A_BYTES;
                const int k = kb * BK;
                mbar_arrive_expect_tx(&full_bar[stage], A_BYTES + box * 128);
                if (!A_MN) {
                    tma_load_3d(sa, &tmA, &full_bar[stage], k, ms * BM, g);
                } else {
#pragma unroll
                    for (int i = 0; i < BM / 64; ++i)
                        tma_load_3d(sa + i * (BK * 128), &tmA, &full_bar[stage], ms * BM + i * 64, k, g);
                }
                tma_load_2d(sb, tmB, &full_bar[stage], k, off + n0);
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
    int stage = 0, qi = 0;
    uint32_t phase = 0, qphase = 0;
    while (true) {
        mbar_wait(&q_full[qi], qphase);
        const int tile = q_tile[qi];
        __syncwarp();
        if (lane == 0) mbar_arrive(&q_empty[qi]);
        if (++qi == QD) {
            qi = 0;
            qphase ^= 1;
        }
        if (tile >= total) break;
        const int gc = tile / m_slices, ms = tile - gc * m_slices;
        const int g = find_group(cum, p.G, gc);
        const int n0 = (gc - cum[g]) * BN_MAX;
        const int nn = min(__ldg(p.group_rows + g) - n0, BN_MAX);
        const int row0 = __ldg(p.group_off + g) + n0;
        switch (box_rows_of(nn)) {
            case 16: sab_tile<16, A_MN>(p, smem, full_bar, empty_bar, stage, phase, num_kb, wg, warp, lane, g, ms, row0, nn); break;
            case 32: sab_tile<32, A_MN>(p, smem, full_bar, empty_bar, stage, phase, num_kb, wg, warp, lane, g, ms, row0, nn); break;
            case 64: sab_tile<64, A_MN>(p, smem, full_bar, empty_bar, stage, phase, num_kb, wg, warp, lane, g, ms, row0, nn); break;
            default: sab_tile<128, A_MN>(p, smem, full_bar, empty_bar, stage, phase, num_kb, wg, warp, lane, g, ms, row0, nn); break;
        }
    }
}

}  // namespace sab

// =====================================================================================================================
// fused wgrad + AMSGrad
// =====================================================================================================================
namespace wa {

constexpr int WBK = 32;                                  // tokens per operand stage
constexpr int OP_STAGES = 4;                             // a hot expert has tens of k-blocks: loads run ahead of the MMAs
constexpr int OP_STAGE_BYTES = 2 * (WBK * BM * 2);       // A [32 t][128 n] + B [32 t][128 k] (two 64-wide MN atoms each)
constexpr int OP_BYTES = OP_STAGES * OP_STAGE_BYTES;
constexpr int BAR_OFFSET = OP_BYTES;
constexpr int QD = 4;                                    // depth of the tile queue (dynamic scheduler)
constexpr int SMEM_TOTAL = BAR_OFFSET + (2 * OP_STAGES + 2 * QD) * 8 + QD * 4 + 16 + 1024;
constexpr int JB = 4;                                    // 8-column groups whose state is loaded together
static_assert(SMEM_TOTAL <= 232448, "shared memory budget");

struct Params {
    int G, N, K;              // groups (slots of the segment), rows (= features of dY) and columns (= features of X) of W
    const int* group_off;     // [G] first token row of the group in dy / x
    const int* group_rows;    // [G] valid rows (0: the expert is not stepped)
    const int* skip;          // optional [G, 2]: skip[2g] >= 0 -> handled by the unfused path (shadowed experts)
    const int* step;          // [G] per-expert step count AFTER this update
    float* p;                 // [G, N, K] fp32 master weights and AMSGrad state
    float* m;
    float* v;
    float* vmax;
    bf16* p_bf16;             // [G, N, K] bf16 mirror consumed by the GEMMs
    float lr, beta1, beta2, eps;
    int amsgrad;
    int* tile_counter;        // work-stealing tile counter (zeroed before the launch)
    const int* poison;        // optional status word: a step that timed out on a peer must not update anything
};

struct Tile {
    int g, mt, nt;
};

__global__ void __launch_bounds__(NUM_THREADS, 1)
wgrad_adam_kernel(const Params p, const __grid_constant__ CUtensorMap tmDY, const __grid_constant__ CUtensorMap tmX) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint64_t* op_full = reinterpret_cast<uint64_t*>(smem + BAR_OFFSET);
    uint64_t* op_empty = op_full + OP_STAGES;
    uint64_t* q_full = op_empty + OP_STAGES;
    uint64_t* q_empty = q_full + QD;
    volatile int* q_tile = reinterpret_cast<volatile int*>(q_empty + QD);

    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;
    if (p.poison && (*p.poison & 1)) return;   // degraded step (a peer timed out): no optimizer step from partial data

    if (warp == 8 && lane == 0) {
        tma_prefetch_desc(&tmDY);
        tma_prefetch_desc(&tmX);
        for (int i = 0; i < OP_STAGES; ++i) {
            mbar_init(&op_full[i], 1);
            mbar_init(&op_empty[i], 8);
        }
        for (int i = 0; i < QD; ++i) {
            mbar_init(&q_full[i], 1);
            mbar_init(&q_empty[i], 8);
        }
        fence_mbar_init();
    }
    __syncthreads();

    const int n_tiles = p.K / BN_MAX;
    const int tiles_per_group = (p.N / BM) * n_tiles;
    const int total = p.G * tiles_per_group;
    auto decode = [&](int tile) {
        Tile t;
        t.g = tile / tiles_per_group;
        const int r = tile - t.g * tiles_per_group;
        t.mt = r / n_tiles;
        t.nt = r - t.mt * n_tiles;
        return t;
    };

    if (warp == 8) {
        if (lane != 0) return;
        // =============================================================== scheduler + operand producer (dY^T / X^T k-blocks)
        // tiles are drawn from a global counter (work stealing: SMs see different HBM bandwidth, a static split leaves the
        // fast ones idle) and published to the consumer warps through a queue
        uint32_t phase = 0, qphase = 0;
        int qi = 0, stage = 0;
        while (true) {
            int tile;
            while (true) {
                tile = atomicAdd(p.tile_counter, 1);
                if (tile >= total) break;
                const int g = tile / tiles_per_group;
                if (__ldg(p.group_rows + g) > 0 && !(p.skip && __ldg(p.skip + 2 * g) >= 0)) break;
                atomicMax(p.tile_counter, (g + 1) * tiles_per_group);   // skip the rest of an inactive group
            }
            mbar_wait(&q_empty[qi], qphase ^ 1);
            q_tile[qi] = tile;
            mbar_arrive(&q_full[qi]);
            if (++qi == QD) {
                qi = 0;
                qphase ^= 1;
            }
            if (tile >= total) break;
            const Tile t = decode(tile);
            const int off = __ldg(p.group_off + t.g), rows = __ldg(p.group_rows + t.g);
            for (int t0 = 0; t0 < rows; t0 += WBK) {
                mbar_wait(&op_empty[stage], phase ^ 1);
                mbar_arrive_expect_tx(&op_full[stage], OP_STAGE_BYTES);
                uint8_t* sa = smem + stage * OP_STAGE_BYTES;
                uint8_t* sb = sa + WBK * BM * 2;
#pragma unroll
                for (int i = 0; i < BM / 64; ++i)
                    tma_load_2d(sa + i * (WBK * 128), &tmDY, &op_full[stage], t.mt * BM + i * 64, off + t0);
#pragma unroll
                for (int i = 0; i < BN_MAX / 64; ++i)
                    tma_load_2d(sb + i * (WBK * 128), &tmX, &op_full[stage], t.nt * BN_MAX + i * 64, off + t0);
                if (++stage == OP_STAGES) {
                    stage = 0;
                    phase ^= 1;
                }
            }
        }
        return;
    }

    // =================================================================== consumers: wgrad tile (MMA) + AMSGrad epilogue
    const int wg = warp >> 2;
    int qi = 0, stage = 0;
    uint32_t phase = 0, qphase = 0;
    float acc[BN_MAX / 2];
    while (true) {
        mbar_wait(&q_full[qi], qphase);
        const int tile = q_tile[qi];
        __syncwarp();
        if (lane == 0) mbar_arrive(&q_empty[qi]);
        if (++qi == QD) {
            qi = 0;
            qphase ^= 1;
        }
        if (tile >= total) break;
        const Tile t = decode(tile);
        const int rows = __ldg(p.group_rows + t.g);
        // ---- dW tile: only ceil(rows/16) k-steps of the last block (the group's padding rows up to 16 are zero)
        int prev_stage = -1;
        for (int t0 = 0; t0 < rows; t0 += WBK) {
            mbar_wait(&op_full[stage], phase);
            const uint32_t sa = smem_u32(smem + stage * OP_STAGE_BYTES) + wg * (WBK * 128);
            const uint32_t sb = smem_u32(smem + stage * OP_STAGE_BYTES + WBK * BM * 2);
            const int ksteps = min(WBK / MMA_K, (rows - t0 + MMA_K - 1) / MMA_K);
            wgmma_fence();
            for (int k = 0; k < ksteps; ++k) {
                const uint64_t da = make_smem_desc_sw128(sa + k * (MMA_K * 128), WBK * 128, 1024);
                const uint64_t db = make_smem_desc_sw128(sb + k * (MMA_K * 128), WBK * 128, 1024);
                wgmma_bf16_n128<1, 1>(acc, da, db, (t0 > 0 || k > 0) ? 1u : 0u);
            }
            wgmma_commit();
            wgmma_wait<1>();
            if (prev_stage >= 0) {
                __syncwarp();
                if (lane == 0) mbar_arrive(&op_empty[prev_stage]);
            }
            prev_stage = stage;
            if (++stage == OP_STAGES) {
                stage = 0;
                phase ^= 1;
            }
        }
        wgmma_wait<0>();
        wgmma_fence_regs(acc);
        __syncwarp();
        if (lane == 0 && prev_stage >= 0) mbar_arrive(&op_empty[prev_stage]);

        // ---- AMSGrad on the accumulator positions: rows r (+8), columns 8j + 2(lane%4) (+1)
        const float st = static_cast<float>(__ldg(p.step + t.g));
        const float step_size = p.lr / (1.f - powf(p.beta1, st));
        const float inv_sqrt_bc2 = rsqrtf(1.f - powf(p.beta2, st));
        const long long row_base = static_cast<long long>(t.g) * p.N + t.mt * BM + wg * 64 + (warp & 3) * 16 + (lane >> 2);
        const int col_base = t.nt * BN_MAX + 2 * (lane & 3);
#pragma unroll
        for (int j0 = 0; j0 < BN_MAX / 8; j0 += JB) {
            float2 pw[JB][2], m[JB][2], v[JB][2], vm[JB][2];
#pragma unroll
            for (int jj = 0; jj < JB; ++jj)
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const long long o = (row_base + 8 * h) * p.K + col_base + 8 * (j0 + jj);
                    pw[jj][h] = *reinterpret_cast<const float2*>(p.p + o);
                    m[jj][h] = *reinterpret_cast<const float2*>(p.m + o);
                    v[jj][h] = *reinterpret_cast<const float2*>(p.v + o);
                    vm[jj][h] = p.amsgrad ? *reinterpret_cast<const float2*>(p.vmax + o) : make_float2(0.f, 0.f);
                }
#pragma unroll
            for (int jj = 0; jj < JB; ++jj)
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    float* pp = &pw[jj][h].x; float* mp = &m[jj][h].x; float* vp = &v[jj][h].x; float* vmp = &vm[jj][h].x;
#pragma unroll
                    for (int e = 0; e < 2; ++e) {
                        const float grad = acc[4 * (j0 + jj) + 2 * h + e];
                        mp[e] = mp[e] + (1.f - p.beta1) * (grad - mp[e]);
                        vp[e] = vp[e] * p.beta2 + (1.f - p.beta2) * grad * grad;
                        float denom;
                        if (p.amsgrad) {
                            vmp[e] = fmaxf(vmp[e], vp[e]);
                            denom = sqrtf(vmp[e]) * inv_sqrt_bc2 + p.eps;
                        } else {
                            denom = sqrtf(vp[e]) * inv_sqrt_bc2 + p.eps;
                        }
                        pp[e] -= step_size * (mp[e] / denom);
                    }
                    const long long o = (row_base + 8 * h) * p.K + col_base + 8 * (j0 + jj);
                    *reinterpret_cast<float2*>(p.p + o) = pw[jj][h];
                    *reinterpret_cast<float2*>(p.m + o) = m[jj][h];
                    *reinterpret_cast<float2*>(p.v + o) = v[jj][h];
                    if (p.amsgrad) *reinterpret_cast<float2*>(p.vmax + o) = vm[jj][h];
                    *reinterpret_cast<uint32_t*>(p.p_bf16 + o) = pack_bf16x2(pw[jj][h].x, pw[jj][h].y);
                }
        }
    }
}

}  // namespace wa
}  // namespace smallm
}  // namespace lah

using namespace lah;
using namespace lah::smallm;

extern "C" const int* lah_get_epoch_base();

// work-stealing tile counter shared by the launches of this file (stream-ordered: memset -> kernel); allocated on first use
static int* tile_counter() {
    static int* ctr = nullptr;
    if (!ctr) {
        if (cudaMalloc(&ctr, 256) != cudaSuccess) return nullptr;
        cudaMemset(ctr, 0, 256);
    }
    return ctr;
}
static const int* g_poison = nullptr;

extern "C" {

// status word whose bit 0 (a peer-flag wait timed out in this step) turns the optimizer kernels into no-ops; NULL disables
int lah_set_poison_word(const int* status) {
    g_poison = status;
    return 0;
}
const int* lah_get_poison_word() { return g_poison; }

// out[row, :] = act_rows[row, :] @ W[g]^T (+bias[g]) (+residual[row, :]) for the rows of every group, swap-AB tiles.
//   a_mn == 0: W is [G, M_out, K] (forward);  a_mn == 1: W is [G, K, M_out] and the product is x @ W (dgrad)
int lah_swapab_linear(const void* x, long long ldx, int x_rows, const void* W, int G, int M_out, int K, int a_mn,
                      void* out, long long ldo, const int* group_off, const int* group_rows, const float* bias,
                      const void* residual, long long ldr, const int* wait_flags, int wait_count, int wait_epoch,
                      const int* epoch_base, int* status, int max_ctas, cudaStream_t st) {
    if ((K % BK) || (M_out % BM) || (ldx % 8) || G > sab::MAX_G) return -2;
    CUtensorMap tmA, tmB[4];
    if (!a_mn) {
        uint64_t dims[3] = {(uint64_t)K, (uint64_t)M_out, (uint64_t)G};
        uint64_t str[2] = {(uint64_t)K * 2, (uint64_t)M_out * K * 2};
        uint32_t box[3] = {BK, BM, 1};
        int r = make_tmap(&tmA, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, W, 3, dims, str, box);
        if (r) return r;
    } else {
        uint64_t dims[3] = {(uint64_t)M_out, (uint64_t)K, (uint64_t)G};
        uint64_t str[2] = {(uint64_t)M_out * 2, (uint64_t)M_out * K * 2};
        uint32_t box[3] = {64, BK, 1};
        int r = make_tmap(&tmA, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, W, 3, dims, str, box);
        if (r) return r;
    }
    const uint32_t boxes[4] = {16, 32, 64, 128};
    for (int i = 0; i < 4; ++i) {
        uint64_t dims[2] = {(uint64_t)K, (uint64_t)x_rows};
        uint64_t str[1] = {(uint64_t)ldx * 2};
        uint32_t box[2] = {BK, boxes[i]};
        int r = make_tmap(&tmB[i], CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, x, 2, dims, str, box);
        if (r) return r;
    }
    sab::Params p;
    p.G = G; p.M_out = M_out; p.K = K; p.group_off = group_off; p.group_rows = group_rows; p.out = (bf16*)out; p.ldo = ldo;
    p.bias = bias; p.residual = (const bf16*)residual; p.ldr = ldr; p.wait_flags = wait_flags; p.wait_count = wait_count;
    p.wait_epoch = wait_epoch; p.epoch_base = epoch_base ? epoch_base : lah_get_epoch_base(); p.status = status;
    p.tile_counter = tile_counter();
    if (!p.tile_counter) return -3;
    // upper bound of the tile count (the real one depends on the device-side row counts): every group has at least one
    // 128-token chunk per 128-feature slice, and all groups together at most x_rows / 128 + G chunks
    const long long total = 1ll * (M_out / BM) * (G + x_rows / BN_MAX);
    if (total <= 0 || G <= 0) return 0;
    if (cudaMemsetAsync(p.tile_counter, 0, sizeof(int), st) != cudaSuccess) return -4;
    int ctas = num_sms();
    if (max_ctas > 0 && max_ctas < ctas) ctas = max_ctas;
    if (total < ctas) ctas = static_cast<int>(total);
    static bool configured[2] = {false, false};
    if (!a_mn) {
        if (!configured[0]) {
            cudaError_t e = cudaFuncSetAttribute(sab::swapab_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, sab::SMEM_TOTAL);
            if (e != cudaSuccess) return -(int)e;
            configured[0] = true;
        }
        sab::swapab_kernel<false><<<ctas, NUM_THREADS, sab::SMEM_TOTAL, st>>>(p, tmA, tmB[0], tmB[1], tmB[2], tmB[3]);
    } else {
        if (!configured[1]) {
            cudaError_t e = cudaFuncSetAttribute(sab::swapab_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, sab::SMEM_TOTAL);
            if (e != cudaSuccess) return -(int)e;
            configured[1] = true;
        }
        sab::swapab_kernel<true><<<ctas, NUM_THREADS, sab::SMEM_TOTAL, st>>>(p, tmA, tmB[0], tmB[1], tmB[2], tmB[3]);
    }
    return -(int)cudaGetLastError();
}

// W[g] -= AMSGrad(dW[g] = dy_g^T x_g) for every group with rows > 0; p / m / v / vmax are [G, N, K] fp32, p_bf16 the mirror
int lah_wgrad_adam(const void* dy, long long lddy, const void* x, long long ldx, int total_rows, int G, int N, int K,
                   const int* group_off, const int* group_rows, const int* skip, const int* step, float* p, float* m,
                   float* v, float* vmax, void* p_bf16, float lr, float beta1, float beta2, float eps, int amsgrad,
                   int max_ctas, cudaStream_t st) {
    if ((N % BM) || (K % BN_MAX) || (lddy % 8) || (ldx % 8)) return -2;
    CUtensorMap tmDY, tmX;
    {
        uint64_t dims[2] = {(uint64_t)N, (uint64_t)total_rows};
        uint64_t str[1] = {(uint64_t)lddy * 2};
        uint32_t box[2] = {64, wa::WBK};
        int r = make_tmap(&tmDY, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, dy, 2, dims, str, box);
        if (r) return r;
    }
    {
        uint64_t dims[2] = {(uint64_t)K, (uint64_t)total_rows};
        uint64_t str[1] = {(uint64_t)ldx * 2};
        uint32_t box[2] = {64, wa::WBK};
        int r = make_tmap(&tmX, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, x, 2, dims, str, box);
        if (r) return r;
    }
    wa::Params a;
    a.G = G; a.N = N; a.K = K; a.group_off = group_off; a.group_rows = group_rows; a.skip = skip; a.step = step;
    a.p = p; a.m = m; a.v = v; a.vmax = vmax; a.p_bf16 = (bf16*)p_bf16; a.lr = lr; a.beta1 = beta1; a.beta2 = beta2; a.eps = eps; a.amsgrad = amsgrad;
    a.tile_counter = tile_counter() ? tile_counter() + 16 : nullptr;   // own word (64 B apart from the GEMM's)
    a.poison = g_poison;
    if (!a.tile_counter) return -3;
    const long long total = 1ll * G * (N / BM) * (K / BN_MAX);
    if (total <= 0) return 0;
    if (cudaMemsetAsync(a.tile_counter, 0, sizeof(int), st) != cudaSuccess) return -4;
    int ctas = num_sms();
    if (max_ctas > 0 && max_ctas < ctas) ctas = max_ctas;
    if (total < ctas) ctas = (int)total;
    static bool configured = false;
    if (!configured) {
        cudaError_t e = cudaFuncSetAttribute(wa::wgrad_adam_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, wa::SMEM_TOTAL);
        if (e != cudaSuccess) return -(int)e;
        configured = true;
    }
    wa::wgrad_adam_kernel<<<ctas, NUM_THREADS, wa::SMEM_TOTAL, st>>>(a, tmDY, tmX);
    return -(int)cudaGetLastError();
}

}  // extern "C"
