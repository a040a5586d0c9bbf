// opt_stream_probe.cu — the optimizer-state stream of wgrad_adam_kernel (csrc/small_m.cu) without its MMA and its math:
// a persistent, warp-specialised kernel that walks 128 x 128 tiles of four fp32 [G*N, K] arrays (p, m, v, vmax), brings
// each tile in as four 64 KB chunks through a 3-stage TMA ring, optionally reads p back from shared memory at the
// accumulator positions of the fused kernel and writes the bf16 mirror, and stores every chunk back by TMA.  The chunk
// geometry is a run-time argument, so one process can compare the ways of cutting a tile into chunks.  GEO_SPLIT streams the
// master weight as two 16-bit planes (its bf16 GEMM operand and its low half) instead of fp32 p + a bf16 mirror.
//
// Built and driven by tools/opt_stream_probe.py.
#include "sm90.cuh"

using namespace lah;

namespace {

constexpr int BM = 128, BN = 128;
constexpr int CHUNKS = 4;
constexpr int ARR_BYTES = 16384;                   // one array of a chunk: 4096 fp32
constexpr int STAGES = 3;
constexpr int STAGE_BYTES = 4 * ARR_BYTES;
constexpr int BAR_OFFSET = STAGES * STAGE_BYTES;
constexpr int QD = 4;
constexpr int SMEM_TOTAL = BAR_OFFSET + (2 * STAGES + 2 * QD) * 8 + QD * 4 + 16 + 1024;
constexpr int NUM_THREADS = 288;

// chunk c of a tile is
//   GEO_COLS        columns [32c, 32c + 32) of all 128 rows: one [128 rows][32 fp32] box per array, 128-B row runs
//   GEO_ROWS        rows [32c, 32c + 32), all 128 columns: four adjacent [32][32] boxes per array, 512-B row runs
//   GEO_BANDS       rows 4c .. 4c + 3 of each of the tile's eight 16-row bands, all 128 columns: a 3-D map (K, 16, G*N/16)
//                   and four [8 bands][4 rows][32 fp32] boxes per array, 512-B row runs
//   GEO_BANDS_FLAT  the same rows as one unswizzled [8][4][128 fp32] box per array
//   GEO_SPLIT       the rows of GEO_BANDS for five arrays: the hi and lo 16-bit planes of the master weight, two
//                   [8 bands][4 rows][64 x 16 bit] boxes each (256-B row runs, 8 KB per plane), then m, v, vmax as in
//                   GEO_BANDS; 64 KB per chunk as before, everything moved by TMA
enum { GEO_COLS = 0, GEO_ROWS = 1, GEO_BANDS = 2, GEO_BANDS_FLAT = 3, GEO_SPLIT = 4 };

struct Maps {
    CUtensorMap a[5];
};

__device__ __forceinline__ void chunk_tma(int geo, bool store, const Maps& tm, uint8_t* ss, uint64_t* bar, int col0, int srow,
                                          int c) {
    if (geo == GEO_SPLIT) {
        for (int a = 0; a < 5; ++a) {
            const int plane = a < 2;
            uint8_t* s = ss + (plane ? a * 8192 : (a - 1) * ARR_BYTES);
            for (int q = 0; q < (plane ? 2 : 4); ++q) {
                const int x = col0 + (plane ? 64 : 32) * q;
                if (store) tma_store_3d(&tm.a[a], s + q * 4096, x, 4 * c, srow / 16);
                else tma_load_3d(s + q * 4096, &tm.a[a], bar, x, 4 * c, srow / 16);
            }
        }
        return;
    }
    for (int a = 0; a < 4; ++a) {
        uint8_t* s = ss + a * ARR_BYTES;
        const CUtensorMap* m = &tm.a[a];
        if (geo == GEO_COLS) {
            if (store) tma_store_2d(m, s, col0 + 32 * c, srow);
            else tma_load_2d(s, m, bar, col0 + 32 * c, srow);
        } else if (geo == GEO_ROWS) {
            for (int q = 0; q < 4; ++q) {
                if (store) tma_store_2d(m, s + q * 4096, col0 + 32 * q, srow + 32 * c);
                else tma_load_2d(s + q * 4096, m, bar, col0 + 32 * q, srow + 32 * c);
            }
        } else if (geo == GEO_BANDS) {
            for (int q = 0; q < 4; ++q) {
                if (store) tma_store_3d(m, s + q * 4096, col0 + 32 * q, 4 * c, srow / 16);
                else tma_load_3d(s + q * 4096, m, bar, col0 + 32 * q, 4 * c, srow / 16);
            }
        } else {
            if (store) tma_store_3d(m, s, col0, 4 * c, srow / 16);
            else tma_load_3d(s, m, bar, col0, 4 * c, srow / 16);
        }
    }
}

// the consumer side of one chunk: p read back from shared memory at this thread's accumulator positions (rows lrow, lrow + 8
// of warp w's 16-row band; columns 8j + 2(lane % 4) + {0, 1}) and written to the bf16 mirror
__device__ __forceinline__ void chunk_mirror(int geo, const uint8_t* sp, bf16* mirror, long long K, int srow, int col0, int c,
                                             int warp, int lane) {
    const int lrow = warp * 16 + (lane >> 2);
    const int cq = 2 * (lane & 3);
    if (geo == GEO_COLS) {
        for (int h = 0; h < 2; ++h)
            for (int jj = 0; jj < 4; ++jj) {
                const int r = lrow + 8 * h;
                const int so = r * 128 + (((2 * jj + ((lane & 3) >> 1)) ^ (r & 7)) << 4) + 8 * (lane & 1);
                const float2 v = *reinterpret_cast<const float2*>(sp + so);
                *reinterpret_cast<uint32_t*>(mirror + (srow + r) * K + col0 + 32 * c + 8 * jj + cq) = pack_bf16x2(v.x, v.y);
            }
    } else if (geo == GEO_ROWS) {
        if ((warp >> 1) != c) return;
        for (int h = 0; h < 2; ++h)
            for (int j = 0; j < 16; ++j) {
                const int r = lrow + 8 * h, R = r - 32 * c;
                const int so = (j >> 2) * 4096 + R * 128 + (((2 * (j & 3) + ((lane & 3) >> 1)) ^ (R & 7)) << 4) + 8 * (lane & 1);
                const float2 v = *reinterpret_cast<const float2*>(sp + so);
                *reinterpret_cast<uint32_t*>(mirror + (srow + r) * K + col0 + 8 * j + cq) = pack_bf16x2(v.x, v.y);
            }
    } else {
        if (((lane >> 4) & 1) != (c & 1)) return;
        const int i = (lane >> 2) & 3, R = warp * 4 + i;
        const int r = lrow + 8 * (c >> 1);
        for (int j0 = 0; j0 < 16; ++j0) {
            const int j = j0 ^ (2 * (i & 1));
            int so;
            if (geo == GEO_BANDS)
                so = (j >> 2) * 4096 + R * 128 + (((2 * (j & 3) + ((lane & 3) >> 1)) ^ (R & 7)) << 4) + 8 * (lane & 1);
            else
                so = R * 512 + (8 * j + cq) * 4;
            const float2 v = *reinterpret_cast<const float2*>(sp + so);
            *reinterpret_cast<uint32_t*>(mirror + (srow + r) * K + col0 + 8 * j + cq) = pack_bf16x2(v.x, v.y);
        }
    }
}

__global__ void __launch_bounds__(NUM_THREADS, 1)
probe_kernel(int geo, int mirror_on, int GN, int K, bf16* mirror, int* tile_counter, const __grid_constant__ Maps tm) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint64_t* st_full = reinterpret_cast<uint64_t*>(smem + BAR_OFFSET);
    uint64_t* st_empty = st_full + STAGES;
    uint64_t* q_full = st_empty + STAGES;
    uint64_t* q_empty = q_full + QD;
    volatile int* q_tile = reinterpret_cast<volatile int*>(q_empty + QD);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (warp == 8 && lane == 0) {
        for (int a = 0; a < (geo == GEO_SPLIT ? 5 : 4); ++a) tma_prefetch_desc(&tm.a[a]);
        for (int i = 0; i < STAGES; ++i) {
            mbar_init(&st_full[i], 1);
            mbar_init(&st_empty[i], 1);
        }
        for (int i = 0; i < QD; ++i) {
            mbar_init(&q_full[i], 1);
            mbar_init(&q_empty[i], 8);
        }
        fence_mbar_init();
    }
    __syncthreads();
    const int n_tiles = K / BN;
    const int total = (GN / BM) * n_tiles;

    if (warp == 8) {
        if (lane != 0) return;
        int qi = 0, sstage = 0;
        uint32_t qphase = 0, sphase = 0;
        while (true) {
            const int tile = atomicAdd(tile_counter, 1);
            mbar_wait(&q_empty[qi], qphase ^ 1);
            q_tile[qi] = tile;
            mbar_arrive(&q_full[qi]);
            if (++qi == QD) {
                qi = 0;
                qphase ^= 1;
            }
            if (tile >= total) break;
            const int srow = (tile / n_tiles) * BM, col0 = (tile % n_tiles) * BN;
            for (int c = 0; c < CHUNKS; ++c) {
                mbar_wait(&st_empty[sstage], sphase ^ 1);
                mbar_arrive_expect_tx(&st_full[sstage], STAGE_BYTES);
                chunk_tma(geo, false, tm, smem + sstage * STAGE_BYTES, &st_full[sstage], col0, srow, c);
                if (++sstage == STAGES) {
                    sstage = 0;
                    sphase ^= 1;
                }
            }
        }
        return;
    }

    int qi = 0, sstage = 0;
    uint32_t qphase = 0, sphase = 0;
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
        const int srow = (tile / n_tiles) * BM, col0 = (tile % n_tiles) * BN;
        for (int c = 0; c < CHUNKS; ++c) {
            mbar_wait(&st_full[sstage], sphase);
            uint8_t* ss = smem + sstage * STAGE_BYTES;
            if (mirror_on) chunk_mirror(geo, ss, mirror, K, srow, col0, c, warp, lane);
            fence_proxy_async_smem();
            named_bar_sync(1, 256);
            if (threadIdx.x == 0) {
                chunk_tma(geo, true, tm, ss, nullptr, col0, srow, c);
                tma_store_commit();
                tma_store_wait_read<0>();
                mbar_arrive(&st_empty[sstage]);
            }
            if (++sstage == STAGES) {
                sstage = 0;
                sphase ^= 1;
            }
        }
    }
    if (threadIdx.x == 0) tma_store_wait<0>();
}

int* counter() {
    static int* ctr = nullptr;
    if (!ctr && cudaMalloc(&ctr, 256) != cudaSuccess) ctr = nullptr;
    return ctr;
}

}  // namespace

// GEO_SPLIT: mirror is the hi plane, lo the low-half plane, p unused; mirror_on must be 0 (the planes go back by TMA)
extern "C" int probe_stream(int geo, int mirror_on, int GN, int K, float* p, float* m, float* v, float* vmax, void* mirror,
                            void* lo, int ctas, cudaStream_t st) {
    if (geo < 0 || geo > GEO_SPLIT || GN % BM || K % BN || (geo == GEO_SPLIT && mirror_on)) return -2;
    Maps tm;
    void* arrs[5] = {p, m, v, vmax, nullptr};
    if (geo == GEO_SPLIT) {
        arrs[0] = mirror; arrs[1] = lo; arrs[2] = m; arrs[3] = v; arrs[4] = vmax;
    }
    for (int a = 0; a < (geo == GEO_SPLIT ? 5 : 4); ++a) {
        int r;
        if (geo == GEO_SPLIT && a < 2) {
            const uint64_t dims[3] = {(uint64_t)K, 16, (uint64_t)GN / 16};
            const uint64_t str[2] = {(uint64_t)K * 2, (uint64_t)K * 32};
            const uint32_t box[3] = {64, 4, 8};
            r = make_tmap(&tm.a[a], CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, arrs[a], dims, str, box);
        } else if (geo == GEO_COLS || geo == GEO_ROWS) {
            const uint64_t dims[2] = {(uint64_t)K, (uint64_t)GN};
            const uint64_t str[1] = {(uint64_t)K * 4};
            const uint32_t box[2] = {32, geo == GEO_COLS ? 128u : 32u};
            r = make_tmap(&tm.a[a], CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, arrs[a], dims, str, box);
        } else {
            const uint64_t dims[3] = {(uint64_t)K, 16, (uint64_t)GN / 16};
            const uint64_t str[2] = {(uint64_t)K * 4, (uint64_t)K * 64};
            const uint32_t box[3] = {geo == GEO_BANDS_FLAT ? 128u : 32u, 4, 8};
            r = make_tmap(&tm.a[a], CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, arrs[a], dims, str, box,
                          geo == GEO_BANDS_FLAT ? CU_TENSOR_MAP_SWIZZLE_NONE : CU_TENSOR_MAP_SWIZZLE_128B);
        }
        if (r) return r;
    }
    int* ctr = counter();
    if (!ctr) return -3;
    if (cudaMemsetAsync(ctr, 0, sizeof(int), st) != cudaSuccess) return -4;
    if (int e = set_max_dynamic_smem<probe_kernel>(SMEM_TOTAL)) return e;
    probe_kernel<<<persistent_grid((long long)(GN / BM) * (K / BN), ctas), NUM_THREADS, SMEM_TOTAL, st>>>(
        geo, mirror_on, GN, K, (bf16*)mirror, ctr, tm);
    return -(int)cudaGetLastError();
}
