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
//                      INTO THE EPILOGUE: p / m / v / vmax stream through a TMA ring of 4-rows-per-band chunks of the tile
//                      (loaded while the MMAs run), every thread updates them in shared memory at the positions of its
//                      accumulator registers and writes the bf16 mirror, and the chunk goes back to HBM by TMA store.
//                      The weight gradient never exists in HBM: 34 B / parameter
//                      instead of 46 (wgrad write 4 + Adam 38 + re-read 4).  The SPLIT instantiation keeps the master
//                      weight as its bf16 mirror plus a 16-bit low half (split_decode, sm90.cuh): both planes stream
//                      through the ring like the rest of the state, and nothing is stored from registers: 32 B / parameter.
//                      Reference semantics: one torch.optim.Adam(amsgrad=True) step per expert right after its backward
//                      (/root/reference/lib/runtime/expert_backend.py:90-97).
#include "sm90.cuh"
#include <climits>

namespace lah {
namespace smallm {

constexpr int BM = 128;      // MMA M: weight rows (swapab) / dY features (wgrad)
constexpr int BK = 64;       // k elements per stage row (128 B of bf16 = one swizzle row)
constexpr int MMA_K = 16;
constexpr int BN_MAX = 128;  // max tokens per MMA (swapab) / X features per tile (wgrad)
constexpr int NUM_THREADS = 288;   // two consumer warpgroups + one producer warp

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
constexpr int OP_STAGES = 2;                             // a hot expert has tens of k-blocks: loads run ahead of the MMAs
constexpr int OP_STAGE_BYTES = 2 * (WBK * BM * 2);       // A [32 t][128 n] + B [32 t][128 k] (two 64-wide MN atoms each)
constexpr int OP_BYTES = OP_STAGES * OP_STAGE_BYTES;
// optimizer state streams through its own ring.  Chunk c of a tile holds rows 4c .. 4c + 3 of each of the tile's eight
// 16-row bands (one band per consumer warp) over all 128 columns, so every row is read and written as one 512-B run.  Per
// array it is four [8 bands][4 rows][32 fp32] boxes of a 3-D view (K, 16, G*N / 16) with 128-B swizzle, side by side.
constexpr int BAND_ROWS = 4;                             // rows of every 16-row band in one chunk
constexpr int CHUNKS = 16 / BAND_ROWS;                   // chunks per tile
constexpr int SUB_COLS = 32;                             // columns of one box (128 B: the swizzle row)
constexpr int SUB_BYTES = BM / CHUNKS * SUB_COLS * 4;    // 4 KB: one box
constexpr int ARR_BYTES = (BN_MAX / SUB_COLS) * SUB_BYTES;   // 16 KB: one state array of a chunk
constexpr int ST_STAGES = 3;
constexpr int ST_STAGE_BYTES = 4 * ARR_BYTES;
constexpr int ST_OFFSET = OP_BYTES;
constexpr int BAR_OFFSET = ST_OFFSET + ST_STAGES * ST_STAGE_BYTES;
constexpr int QD = 4;                                    // depth of the tile queue (dynamic scheduler)
constexpr int SMEM_TOTAL = BAR_OFFSET + (2 * OP_STAGES + 2 * ST_STAGES + 2 * QD) * 8 + QD * 4 + 16 + 1024;
static_assert(ST_STAGES <= CHUNKS, "the producer issues a tile's first ST_STAGES chunks before its remaining k-blocks");
static_assert(OP_STAGE_BYTES % 1024 == 0 && SUB_BYTES % 1024 == 0, "128-B swizzle atoms need 1 KB alignment");
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
    float wd;                 // WD_L2: grad += wd * p;  WD_DECOUPLED: p *= wd before the moments, wd = 1 - lr * weight_decay
                              // rounded to fp32 by the caller (in the padding after amsgrad: the layout stays as it was)
    int* tile_counter;        // work-stealing tile counter (zeroed before the launch)
    const int* poison;        // optional status word: a step that timed out on a peer must not update anything
};
// the tensor maps follow Params in parameter space at 64-B alignment.  Params fills its 128 B exactly, so the device-resident
// learning rate is not a field here (one more pointer would move the maps by 64 B) but the kernel's last parameter
static_assert(sizeof(Params) == 128 && sizeof(Params) % alignof(CUtensorMap) == 0, "Params layout");

// weight-decay form of one launch (a template parameter: the WD_NONE instantiation is the kernel without decay)
constexpr int WD_NONE = 0, WD_L2 = 1, WD_DECOUPLED = 2;

struct Tile {
    int g, mt, nt;
};

// state tensor maps: p, m, v, vmax viewed as [G * N / 16][16][K] fp32 (vmax only read when amsgrad).  SPLIT: the hi and lo
// planes of the master weight as [G * N / 16][16][K] 16-bit, then m, v, vmax
template <bool SPLIT>
struct StateMaps {
    CUtensorMap a[SPLIT ? 5 : 4];
};
// SPLIT: a chunk's 16 KB of p hold the two planes, 8 KB each as two [8 bands][4 rows][64 x 16 bit] boxes (128-B swizzle);
// m, v and vmax keep their places
constexpr int PLANE_COLS = 64;
constexpr int PLANE_BYTES = ARR_BYTES / 2;
static_assert(PLANE_BYTES == (BN_MAX / PLANE_COLS) * SUB_BYTES, "a plane box has the rows and bytes of an fp32 box");

// TMA load (bar != nullptr) or store of chunk c of the tile whose rows start at srow and columns at col0, 16-KB arrays
// [0, n_arr) (array 0: p, or the two planes)
template <bool SPLIT>
__device__ __forceinline__ void state_chunk_tma(const StateMaps<SPLIT>& tm, int n_arr, uint8_t* ss, uint64_t* bar, int col0,
                                                int srow, int c) {
    if constexpr (SPLIT) {
        for (int a = 0; a < 2; ++a)
#pragma unroll
            for (int q = 0; q < BN_MAX / PLANE_COLS; ++q) {
                uint8_t* s = ss + a * PLANE_BYTES + q * SUB_BYTES;
                if (bar) tma_load_3d(s, &tm.a[a], bar, col0 + q * PLANE_COLS, BAND_ROWS * c, srow / 16);
                else tma_store_3d(&tm.a[a], s, col0 + q * PLANE_COLS, BAND_ROWS * c, srow / 16);
            }
    }
    for (int a = SPLIT ? 1 : 0; a < n_arr; ++a)
#pragma unroll
        for (int q = 0; q < BN_MAX / SUB_COLS; ++q) {
            uint8_t* s = ss + a * ARR_BYTES + q * SUB_BYTES;
            const CUtensorMap* m = &tm.a[SPLIT ? a + 1 : a];
            if (bar) tma_load_3d(s, m, bar, col0 + q * SUB_COLS, BAND_ROWS * c, srow / 16);
            else tma_store_3d(m, s, col0 + q * SUB_COLS, BAND_ROWS * c, srow / 16);
        }
}

// DEV_LR: the learning rate and, with WD_DECOUPLED, the factor 1 - lr * weight_decay come from lr_dev = {lr, decay} in device
// memory instead of p.lr / p.wd, so a captured CUDA graph follows a schedule.  Read once per consumer thread; the update
// expressions are the same, so a launch whose block holds x is bit-identical to a by-value launch with x.
// SPLIT: the master weight is decoded from its planes in shared memory, updated by the same expressions and encoded back
// (p.p and p.p_bf16 are unused), so p, m, v, vmax and the mirror get the bits of the fp32 instantiation
template <int WD, bool DEV_LR, bool SPLIT>
__global__ void __launch_bounds__(NUM_THREADS, 1)
wgrad_adam_kernel(const Params p, const __grid_constant__ CUtensorMap tmDY, const __grid_constant__ CUtensorMap tmX,
                  const __grid_constant__ StateMaps<SPLIT> tmS, const float* __restrict__ lr_dev) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint8_t* st_smem = smem + ST_OFFSET;
    uint64_t* op_full = reinterpret_cast<uint64_t*>(smem + BAR_OFFSET);
    uint64_t* op_empty = op_full + OP_STAGES;
    uint64_t* st_full = op_empty + OP_STAGES;
    uint64_t* st_empty = st_full + ST_STAGES;
    uint64_t* q_full = st_empty + ST_STAGES;
    uint64_t* q_empty = q_full + QD;
    volatile int* q_tile = reinterpret_cast<volatile int*>(q_empty + QD);

    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;
    if (p.poison && (*p.poison & 1)) return;   // degraded step (a peer timed out): no optimizer step from partial data
    const int n_arr = p.amsgrad ? 4 : 3;

    if (warp == 8 && lane == 0) {
        tma_prefetch_desc(&tmDY);
        tma_prefetch_desc(&tmX);
        for (int a = 0; a < n_arr + (SPLIT ? 1 : 0); ++a) tma_prefetch_desc(&tmS.a[a]);
        for (int i = 0; i < OP_STAGES; ++i) {
            mbar_init(&op_full[i], 1);
            mbar_init(&op_empty[i], 8);
        }
        for (int i = 0; i < ST_STAGES; ++i) {
            mbar_init(&st_full[i], 1);
            mbar_init(&st_empty[i], 1);   // released by the thread that stored the chunk back
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
        // =============================================================== scheduler + operand / state producer
        // tiles are drawn from a global counter (work stealing: SMs see different HBM bandwidth, a static split leaves the
        // fast ones idle) and published to the consumer warps through a queue.  Per tile: the dY^T / X^T k-blocks and the
        // state chunks.  The state does not depend on the gradient, so the first ST_STAGES chunks go out right after the
        // first k-block (their slots are freed by the previous tile's epilogue) and stream in during the MMA; the rest
        // follow the last k-block.  The consumers take the same order, so no wait of the producer can deadlock.
        uint32_t phase = 0, qphase = 0, sphase = 0;
        int qi = 0, stage = 0, sstage = 0;
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
            const int srow = t.g * p.N + t.mt * BM;
            auto load_chunk = [&](int c) {
                mbar_wait(&st_empty[sstage], sphase ^ 1);
                mbar_arrive_expect_tx(&st_full[sstage], n_arr * ARR_BYTES);
                state_chunk_tma(tmS, n_arr, st_smem + sstage * ST_STAGE_BYTES, &st_full[sstage], t.nt * BN_MAX, srow, c);
                if (++sstage == ST_STAGES) {
                    sstage = 0;
                    sphase ^= 1;
                }
            };
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
                if (t0 == 0)
                    for (int c = 0; c < ST_STAGES; ++c) load_chunk(c);
            }
            for (int c = ST_STAGES; c < CHUNKS; ++c) load_chunk(c);
        }
        return;
    }

    // =================================================================== consumers: wgrad tile (MMA) + AMSGrad epilogue
    float lr = p.lr, wd = p.wd;
    if constexpr (DEV_LR) {
        lr = lr_dev[0];
        if constexpr (WD == WD_DECOUPLED) wd = lr_dev[1];
    }
    const int wg = warp >> 2;
    int qi = 0, stage = 0, sstage = 0;
    uint32_t phase = 0, qphase = 0, sphase = 0;
    float acc[BN_MAX / 2];
    float xg[BN_MAX / 8];   // gradient of the partner lane's row, columns 64 .. 127
    // this thread's accumulator rows of the tile: lrow and lrow + 8, rows lane / 4 and lane / 4 + 8 of its warp's 16-row band
    const int lrow = wg * 64 + (warp & 3) * 16 + (lane >> 2);
    // Chunk c holds band rows 4c .. 4c + 3: row lrow + 8 (c / 2) of the lanes whose half (lane / 16) is c % 2, and the same
    // row number of their partner lane ^ 16 in the other half.  Every lane works on every chunk: the row's owner on its
    // columns 0 .. 63 (j < 8), the partner on columns 64 .. 127 with the owner's gradient fetched by a shuffle.  In a chunk's
    // boxes both see the row as row R = 4 warp + (lane / 4) % 4 (128 B, 16-B unit u at u ^ (R % 8)).
    const int brow = (lane >> 2) & 3;
    const int R = warp * BAND_ROWS + brow;
    const int jflip = 2 * (brow & 1);
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

        // ---- AMSGrad on the accumulator positions: rows r (+8), columns 8j + 2(lane%4) (+1), state from the chunk ring
        const float st = static_cast<float>(__ldg(p.step + t.g));
        const float step_size = lr / (1.f - powf(p.beta1, st));
        const float inv_sqrt_bc2 = rsqrtf(1.f - powf(p.beta2, st));
        const int srow = t.g * p.N + t.mt * BM;
        const int col_base = t.nt * BN_MAX + 2 * (lane & 3);
#pragma unroll
        for (int c = 0; c < CHUNKS; ++c) {
            mbar_wait(&st_full[sstage], sphase);
            uint8_t* ss = st_smem + sstage * ST_STAGE_BYTES;
            if ((c & 1) == 0) {   // the partner's gradient of columns 64 .. 127 in the current row pair (r, r ^ 4)
#pragma unroll
                for (int i = 0; i < BN_MAX / 8; ++i) xg[i] = __shfl_xor_sync(0xffffffffu, acc[4 * (BN_MAX / 16 + i / 2) + i % 2], 16);
            }
            const bool own = (lane >> 4) == (c & 1);
            const long long o_row = (static_cast<long long>(srow) + (own ? lrow : lrow ^ 4) + 8 * (c >> 1)) * p.K + col_base;
            const int jbase = own ? 0 : BN_MAX / 16;
#pragma unroll
            for (int k = 0; k < BN_MAX / 16; ++k) {
                // column group j = k of even rows, k ^ 2 of odd rows: rows R and R ^ 1 put the same j in the same two 16-B
                // units, so this way the 16 lanes of each half cover eight distinct units, and the owners' columns
                // (boxes 0, 1) and the partners' (boxes 2, 3) one wavefront each: no bank conflict
                const int j = jbase + (k ^ jflip);
                const int so = (j >> 2) * SUB_BYTES + R * 128 + (((2 * (j & 3) + ((lane & 3) >> 1)) ^ (R & 7)) << 4) +
                               8 * (lane & 1);
                float2* sp = reinterpret_cast<float2*>(ss + so);
                float2* sm = reinterpret_cast<float2*>(ss + ARR_BYTES + so);
                float2* sv = reinterpret_cast<float2*>(ss + 2 * ARR_BYTES + so);
                float2* svm = reinterpret_cast<float2*>(ss + 3 * ARR_BYTES + so);
                // SPLIT: columns 8j + 2 (lane % 4) + {0, 1} of a plane are one 32-bit word of 16-B unit j % 8 of box j / 8
                const int po = (j >> 3) * SUB_BYTES + R * 128 + (((j & 7) ^ (R & 7)) << 4) + 4 * (lane & 3);
                uint32_t* shi = reinterpret_cast<uint32_t*>(ss + po);
                uint32_t* slo = reinterpret_cast<uint32_t*>(ss + PLANE_BYTES + po);
                float2 pw, m = *sm, v = *sv;
                if constexpr (SPLIT) {
                    const uint32_t hw = *shi, lw = *slo;
                    pw.x = split_decode(hw & 0xffffu, lw & 0xffffu, __float_as_uint(v.x) >> 31);
                    pw.y = split_decode(hw >> 16, lw >> 16, __float_as_uint(v.y) >> 31);
                    v.x = without_tie_bit(v.x);
                    v.y = without_tie_bit(v.y);
                } else {
                    pw = *sp;
                }
                float2 vm = p.amsgrad ? *svm : make_float2(0.f, 0.f);
                float* pp = &pw.x; float* mp = &m.x; float* vp = &v.x; float* vmp = &vm.x;
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    float grad = own ? (jflip ? acc[4 * (k ^ 2) + e] : acc[4 * k + e])
                                     : (jflip ? xg[2 * (k ^ 2) + e] : xg[2 * k + e]);
                    if constexpr (WD == WD_L2) grad += wd * pp[e];
                    if constexpr (WD == WD_DECOUPLED) pp[e] = __fmul_rn(pp[e], wd);   // rounded alone, as p.mul_()
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
                if constexpr (SPLIT) {
                    *shi = pack_bf16x2(pw.x, pw.y);
                    *slo = (__float_as_uint(pw.x) & 0xffffu) | (__float_as_uint(pw.y) << 16);
                    v.x = with_tie_bit(v.x, split_tie_up(pw.x));
                    v.y = with_tie_bit(v.y, split_tie_up(pw.y));
                } else {
                    *sp = pw;
                }
                *sm = m;
                *sv = v;
                if (p.amsgrad) *svm = vm;
                if constexpr (!SPLIT) *reinterpret_cast<uint32_t*>(p.p_bf16 + o_row + 8 * j) = pack_bf16x2(pw.x, pw.y);
            }
            // the updated chunk goes back to HBM by TMA; its slot returns to the producer once the store has read it
            fence_proxy_async_smem();
            named_bar_sync(1, 256);
            if (threadIdx.x == 0) {
                state_chunk_tma(tmS, n_arr, ss, nullptr, t.nt * BN_MAX, srow, c);
                tma_store_commit();
                tma_store_wait_read<0>();
                mbar_arrive(&st_empty[sstage]);
            }
            if (++sstage == ST_STAGES) {
                sstage = 0;
                sphase ^= 1;
            }
            // after the first two chunks the gradient of row lrow + 8 moves to the slots of row lrow: a run-time index into
            // the accumulator would put it in local memory
            if (c == 1) {
#pragma unroll
                for (int j = 0; j < BN_MAX / 8; ++j) {
                    acc[4 * j] = acc[4 * j + 2];
                    acc[4 * j + 1] = acc[4 * j + 3];
                }
            }
        }
    }
    if (threadIdx.x == 0) tma_store_wait<0>();
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
                      int* status, int max_ctas, cudaStream_t st) {
    if ((K % BK) || (M_out % BM) || (ldx % 8) || G > sab::MAX_G) return -2;
    CUtensorMap tmA, tmB[4];
    if (!a_mn) {
        uint64_t dims[3] = {(uint64_t)K, (uint64_t)M_out, (uint64_t)G};
        uint64_t str[2] = {(uint64_t)K * 2, (uint64_t)M_out * K * 2};
        uint32_t box[3] = {BK, BM, 1};
        int r = make_tmap(&tmA, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, W, dims, str, box);
        if (r) return r;
    } else {
        uint64_t dims[3] = {(uint64_t)M_out, (uint64_t)K, (uint64_t)G};
        uint64_t str[2] = {(uint64_t)M_out * 2, (uint64_t)M_out * K * 2};
        uint32_t box[3] = {64, BK, 1};
        int r = make_tmap(&tmA, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, W, dims, str, box);
        if (r) return r;
    }
    const uint32_t boxes[4] = {16, 32, 64, 128};
    for (int i = 0; i < 4; ++i) {
        uint64_t dims[2] = {(uint64_t)K, (uint64_t)x_rows};
        uint64_t str[1] = {(uint64_t)ldx * 2};
        uint32_t box[2] = {BK, boxes[i]};
        int r = make_tmap(&tmB[i], CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, x, dims, str, box);
        if (r) return r;
    }
    sab::Params p;
    p.G = G; p.M_out = M_out; p.K = K; p.group_off = group_off; p.group_rows = group_rows; p.out = (bf16*)out; p.ldo = ldo;
    p.bias = bias; p.residual = (const bf16*)residual; p.ldr = ldr; p.wait_flags = wait_flags; p.wait_count = wait_count;
    p.wait_epoch = wait_epoch; p.epoch_base = lah_get_epoch_base(); p.status = status;
    p.tile_counter = tile_counter();
    if (!p.tile_counter) return -3;
    // upper bound of the tile count (the real one depends on the device-side row counts): every group has at least one
    // 128-token chunk per 128-feature slice, and all groups together at most x_rows / 128 + G chunks
    const long long total = 1ll * (M_out / BM) * (G + x_rows / BN_MAX);
    if (total <= 0 || G <= 0) return 0;
    if (cudaMemsetAsync(p.tile_counter, 0, sizeof(int), st) != cudaSuccess) return -4;
    const int ctas = persistent_grid(total, max_ctas);
    if (!a_mn) {
        if (int e = set_max_dynamic_smem<sab::swapab_kernel<false>>(sab::SMEM_TOTAL)) return e;
        sab::swapab_kernel<false><<<ctas, NUM_THREADS, sab::SMEM_TOTAL, st>>>(p, tmA, tmB[0], tmB[1], tmB[2], tmB[3]);
    } else {
        if (int e = set_max_dynamic_smem<sab::swapab_kernel<true>>(sab::SMEM_TOTAL)) return e;
        sab::swapab_kernel<true><<<ctas, NUM_THREADS, sab::SMEM_TOTAL, st>>>(p, tmA, tmB[0], tmB[1], tmB[2], tmB[3]);
    }
    return -(int)cudaGetLastError();
}

}  // extern "C"

template <int WD, bool DEV_LR, bool SPLIT>
static int launch_wgrad_adam(const wa::Params& a, const CUtensorMap& tmDY, const CUtensorMap& tmX,
                             const wa::StateMaps<SPLIT>& tmS, const float* lr_dev, int ctas, cudaStream_t st) {
    if (int e = set_max_dynamic_smem<wa::wgrad_adam_kernel<WD, DEV_LR, SPLIT>>(wa::SMEM_TOTAL)) return e;
    wa::wgrad_adam_kernel<WD, DEV_LR, SPLIT><<<ctas, NUM_THREADS, wa::SMEM_TOTAL, st>>>(a, tmDY, tmX, tmS, lr_dev);
    return -(int)cudaGetLastError();
}

// the two entry points below; SPLIT: p is the hi plane (p_bf16 is unused), lo the low-half plane
template <bool SPLIT>
static int wgrad_adam(const void* dy, long long lddy, const void* x, long long ldx, int total_rows, int G, int N, int K,
                      const int* group_off, const int* group_rows, const int* skip, const int* step, void* p, void* lo,
                      float* m, float* v, float* vmax, void* p_bf16, float lr, const float* lr_dev, float beta1, float beta2,
                      float eps, int amsgrad, float weight_decay, float decay, int decoupled, int max_ctas, cudaStream_t st) {
    if ((N % BM) || (K % BN_MAX) || (lddy % 8) || (ldx % 8) || 1ll * G * N > INT_MAX) return -2;
    if (decoupled && weight_decay != 0.f) return -2;
    if (amsgrad && !vmax) return -2;   // AMSGrad streams vmax through its own tensor map
    CUtensorMap tmDY, tmX;
    wa::StateMaps<SPLIT> tmS;
    {
        void* arrs[5] = {p, m, v, amsgrad ? vmax : (float*)m, nullptr};   // without amsgrad the vmax map is never used
        if (SPLIT) {
            arrs[1] = lo; arrs[2] = m; arrs[3] = v; arrs[4] = amsgrad ? vmax : m;
        }
        uint64_t dims[3] = {(uint64_t)K, 16, (uint64_t)G * N / 16};
        uint64_t str[2] = {(uint64_t)K * 4, (uint64_t)K * 64};
        uint32_t box[3] = {wa::SUB_COLS, wa::BAND_ROWS, BM / 16};
        for (int a = 0; a < (SPLIT ? 5 : 4); ++a) {
            int r;
            if (SPLIT && a < 2) {
                uint64_t pstr[2] = {(uint64_t)K * 2, (uint64_t)K * 32};
                uint32_t pbox[3] = {wa::PLANE_COLS, wa::BAND_ROWS, BM / 16};
                r = make_tmap(&tmS.a[a], CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, arrs[a], dims, pstr, pbox);
            } else {
                r = make_tmap(&tmS.a[a], CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, arrs[a], dims, str, box);
            }
            if (r) return r;
        }
    }
    {
        uint64_t dims[2] = {(uint64_t)N, (uint64_t)total_rows};
        uint64_t str[1] = {(uint64_t)lddy * 2};
        uint32_t box[2] = {64, wa::WBK};
        int r = make_tmap(&tmDY, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, dy, dims, str, box);
        if (r) return r;
    }
    {
        uint64_t dims[2] = {(uint64_t)K, (uint64_t)total_rows};
        uint64_t str[1] = {(uint64_t)ldx * 2};
        uint32_t box[2] = {64, wa::WBK};
        int r = make_tmap(&tmX, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, x, dims, str, box);
        if (r) return r;
    }
    wa::Params a;
    a.G = G; a.N = N; a.K = K; a.group_off = group_off; a.group_rows = group_rows; a.skip = skip; a.step = step;
    a.p = SPLIT ? nullptr : (float*)p; a.m = m; a.v = v; a.vmax = vmax; a.p_bf16 = (bf16*)p_bf16; a.lr = lr; a.beta1 = beta1; a.beta2 = beta2; a.eps = eps; a.amsgrad = amsgrad;
    a.wd = decoupled ? decay : weight_decay;
    a.tile_counter = tile_counter() ? tile_counter() + 16 : nullptr;   // own word (64 B apart from the GEMM's)
    a.poison = g_poison;
    if (!a.tile_counter) return -3;
    const long long total = 1ll * G * (N / BM) * (K / BN_MAX);
    if (total <= 0) return 0;
    if (cudaMemsetAsync(a.tile_counter, 0, sizeof(int), st) != cudaSuccess) return -4;
    const int ctas = persistent_grid(total, max_ctas);
    if (lr_dev) {
        if (decoupled) return launch_wgrad_adam<wa::WD_DECOUPLED, true, SPLIT>(a, tmDY, tmX, tmS, lr_dev, ctas, st);
        if (weight_decay != 0.f) return launch_wgrad_adam<wa::WD_L2, true, SPLIT>(a, tmDY, tmX, tmS, lr_dev, ctas, st);
        return launch_wgrad_adam<wa::WD_NONE, true, SPLIT>(a, tmDY, tmX, tmS, lr_dev, ctas, st);
    }
    if (decoupled) return launch_wgrad_adam<wa::WD_DECOUPLED, false, SPLIT>(a, tmDY, tmX, tmS, nullptr, ctas, st);
    if (weight_decay != 0.f) return launch_wgrad_adam<wa::WD_L2, false, SPLIT>(a, tmDY, tmX, tmS, nullptr, ctas, st);
    return launch_wgrad_adam<wa::WD_NONE, false, SPLIT>(a, tmDY, tmX, tmS, nullptr, ctas, st);
}

extern "C" {

// W[g] -= AMSGrad(dW[g] = dy_g^T x_g) for every group with rows > 0; p / m / v / vmax are [G, N, K] fp32, p_bf16 the mirror.
// weight_decay: the L2 coefficient (WD_L2); decay: the decoupled weight-decay factor 1 - lr * wd, read only when `decoupled`
// is set, which selects WD_DECOUPLED.  At most one of the two forms per launch.  lr_dev == NULL: lr and decay by value;
// otherwise lr_dev = {lr, 1 - lr * wd} in device memory (the factor computed on the host in double and rounded to fp32
// once) and the DEV_LR instantiation, which ignores lr and decay, so a captured CUDA graph follows a schedule
int lah_wgrad_adam(const void* dy, long long lddy, const void* x, long long ldx, int total_rows, int G, int N, int K,
                   const int* group_off, const int* group_rows, const int* skip, const int* step, float* p, float* m,
                   float* v, float* vmax, void* p_bf16, float lr, const float* lr_dev, float beta1, float beta2, float eps,
                   int amsgrad, float weight_decay, float decay, int decoupled, int max_ctas, cudaStream_t st) {
    return wgrad_adam<false>(dy, lddy, x, ldx, total_rows, G, N, K, group_off, group_rows, skip, step, p, nullptr, m, v,
                             vmax, p_bf16, lr, lr_dev, beta1, beta2, eps, amsgrad, weight_decay, decay, decoupled, max_ctas,
                             st);
}

// the same step on a split master weight: hi ([G, N, K] bf16, the GEMM operand) and lo ([G, N, K] 16 bit) instead of p and
// its mirror, the tie bits in the sign of v (split_decode, sm90.cuh).  p, m, v, vmax and hi come out as lah_wgrad_adam's
int lah_wgrad_adam_split(const void* dy, long long lddy, const void* x, long long ldx, int total_rows, int G, int N, int K,
                         const int* group_off, const int* group_rows, const int* skip, const int* step, void* hi, void* lo,
                         float* m, float* v, float* vmax, float lr, const float* lr_dev, float beta1, float beta2, float eps,
                         int amsgrad, float weight_decay, float decay, int decoupled, int max_ctas, cudaStream_t st) {
    if (!hi || !lo) return -2;
    return wgrad_adam<true>(dy, lddy, x, ldx, total_rows, G, N, K, group_off, group_rows, skip, step, hi, lo, m, v, vmax,
                            nullptr, lr, lr_dev, beta1, beta2, eps, amsgrad, weight_decay, decay, decoupled, max_ctas, st);
}

}  // extern "C"
