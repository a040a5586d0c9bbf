// attention_bwd.cu — wgmma self-attention BACKWARD for the transformer expert (d_model 1024, 16 heads x 64, seq 512).
// The reference's transformer expert cannot be trained at all (in-place transpose of a leaf, SURVEY.md §0.3); this kernel is
// what makes the sm_90a transformer expert trainable without falling back to eager PyTorch.
//
// One CTA = one (batch, head, 128-key block j); consumer warpgroup w owns keys [64w, 64w + 64) of the block.  K_j / V_j stay
// in shared memory; the four 128-query blocks i stream through a 2-stage TMA pipeline (Q_i and dO_i).  Per query block, all
// on tensor cores with accumulators in registers (transposed problem: keys are the MMA rows):
//
//     S^T = K_j Q_i^T               (64 x 128 per warpgroup)     dP^T = V_j dO_i^T            (64 x 128)
//     P^T = exp2(S^T * scale*log2e - LSE_i)   [recomputed from the forward's row log-sum-exp: no second softmax pass]
//     dS^T = P^T o (dP^T - Delta_i) * scale   [Delta = rowsum(dO o O)]
//     dV_j += P^T dO_i   (64 x 64)   dK_j += dS^T Q_i  (64 x 64)   dQ_i^(j) = dS K_j  (128 x 64, one partial per key block j)
//
// P^T and dS^T are fed to dV / dK straight from registers (the accumulator layout IS the wgmma A fragment layout); dS^T is
// also stored once to shared memory (bf16, 128B-swizzled [key rows][64 queries] atoms), where it is the MN-major A operand
// of dQ.  Q_i, dO_i, K_j are consumed both K-major (S, dP) and MN-major (dV, dK, dQ) straight from their TMA tiles.
// Nothing of size S x S touches HBM.  Thread 0 also drives TMA.
#include "sm90.cuh"

namespace lah {
namespace attnb {

constexpr int S_LEN = 512;
constexpr int HEAD_DIM = 64;
constexpr int BLK = 128;                       // query block == key block
constexpr int NUM_QB = S_LEN / BLK;            // 4
constexpr int NUM_THREADS = 256;
constexpr int TILE = BLK * HEAD_DIM * 2;       // 16 KB: 128 x 64 bf16
constexpr int ATOM = BLK * 128;                // 16 KB: one [128 key rows][64 queries] atom of dS^T
constexpr int OFF_K = 0;
constexpr int OFF_V = OFF_K + TILE;
constexpr int OFF_Q = OFF_V + TILE;            // 2 stages
constexpr int OFF_DO = OFF_Q + 2 * TILE;       // 2 stages
constexpr int OFF_DS = OFF_DO + 2 * TILE;      // dS^T: two atoms (queries 0-63, 64-127)
constexpr int OFF_LSE = OFF_DS + 2 * ATOM;     // lse2 / delta of the current query block: 2 x 128 fp32
constexpr int OFF_BAR = OFF_LSE + 2 * BLK * 4;
constexpr int NUM_BARS = 1 + 2;
constexpr int SMEM_TOTAL = OFF_BAR + NUM_BARS * 8 + 16 + 1024;

__global__ void __launch_bounds__(NUM_THREADS, 1)
attention_bwd_kernel(const __grid_constant__ CUtensorMap tm_qkv, const __grid_constant__ CUtensorMap tm_do,
                     const float* __restrict__ lse2, const float* __restrict__ delta, bf16* __restrict__ dqkv,
                     bf16* __restrict__ dq_part, long long total_tokens, int d_model, int num_heads, float scale,
                     float scale_log2e) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint64_t* bars = reinterpret_cast<uint64_t*>(smem + OFF_BAR);
    uint64_t* kv_full = bars;
    uint64_t* q_full = bars + 1;     // [2]
    float* s_lse = reinterpret_cast<float*>(smem + OFF_LSE);
    float* s_delta = s_lse + BLK;

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, wg = warp >> 2;
    const int j = blockIdx.x & 3;
    const int head = (blockIdx.x >> 2) % num_heads;
    const int batch = (blockIdx.x >> 2) / num_heads;
    const int seq0 = batch * S_LEN;

    auto load_q = [&](int i) {   // thread 0 only; stage i & 1 must be free
        const int st = i & 1;
        mbar_arrive_expect_tx(&q_full[st], 2 * TILE);
        tma_load_2d(smem + OFF_Q + st * TILE, &tm_qkv, &q_full[st], head * HEAD_DIM, seq0 + i * BLK);
        tma_load_2d(smem + OFF_DO + st * TILE, &tm_do, &q_full[st], head * HEAD_DIM, seq0 + i * BLK);
    };
    if (tid == 0) {
        tma_prefetch_desc(&tm_qkv);
        tma_prefetch_desc(&tm_do);
        mbar_init(kv_full, 1);
        mbar_init(&q_full[0], 1);
        mbar_init(&q_full[1], 1);
        fence_mbar_init();
        mbar_arrive_expect_tx(kv_full, 2 * TILE);
        tma_load_2d(smem + OFF_K, &tm_qkv, kv_full, d_model + head * HEAD_DIM, seq0 + j * BLK);
        tma_load_2d(smem + OFF_V, &tm_qkv, kv_full, 2 * d_model + head * HEAD_DIM, seq0 + j * BLK);
        load_q(0);
        load_q(1);
    }
    __syncthreads();

    const uint32_t sk = smem_u32(smem + OFF_K), sv = smem_u32(smem + OFF_V), sds = smem_u32(smem + OFF_DS);
    const int key_row = wg * 64 + (warp & 3) * 16 + (lane >> 2);   // row of the block (+ 8 for h = 1)
    const int qcol = 2 * (lane & 3);                               // query column (+ 8 jj, + 1)
    float dv[HEAD_DIM / 2], dk[HEAD_DIM / 2];
#pragma unroll
    for (int e = 0; e < HEAD_DIM / 2; ++e) dv[e] = dk[e] = 0.f;
    mbar_wait(kv_full, 0);
#pragma unroll 1
    for (int i = 0; i < NUM_QB; ++i) {
        const int st = i & 1;
        const long long tok0 = seq0 + i * BLK;
        if (tid < BLK) s_lse[tid] = __ldg(lse2 + (tok0 + tid) * num_heads + head);
        else s_delta[tid - BLK] = __ldg(delta + (tok0 + tid - BLK) * num_heads + head);
        mbar_wait(&q_full[st], (i >> 1) & 1);
        const uint32_t sq = smem_u32(smem + OFF_Q + st * TILE), sdo = smem_u32(smem + OFF_DO + st * TILE);
        float sacc[BLK / 2], dpacc[BLK / 2];
        wgmma_fence();
#pragma unroll
        for (int ks = 0; ks < HEAD_DIM / 16; ++ks)
            wgmma_bf16_n128<0, 0>(sacc, make_smem_desc_sw128(sk + wg * 8192 + ks * 32, 0, 1024),
                                  make_smem_desc_sw128(sq + ks * 32, 0, 1024), ks > 0 ? 1u : 0u);
#pragma unroll
        for (int ks = 0; ks < HEAD_DIM / 16; ++ks)
            wgmma_bf16_n128<0, 0>(dpacc, make_smem_desc_sw128(sv + wg * 8192 + ks * 32, 0, 1024),
                                  make_smem_desc_sw128(sdo + ks * 32, 0, 1024), ks > 0 ? 1u : 0u);
        wgmma_commit();
        named_bar_sync(1, NUM_THREADS);   // lse / delta of this block are in shared memory
        wgmma_wait<0>();
        wgmma_fence_regs(sacc);
        wgmma_fence_regs(dpacc);
        uint32_t pa[BLK / 16][4], da[BLK / 16][4];
#pragma unroll
        for (int jj = 0; jj < BLK / 8; ++jj) {
            const int q = 8 * jj + qcol;
            const float l0 = s_lse[q], l1 = s_lse[q + 1], d0 = s_delta[q], d1 = s_delta[q + 1];
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const float p0 = exp2f(sacc[4 * jj + 2 * h] * scale_log2e - l0);
                const float p1 = exp2f(sacc[4 * jj + 2 * h + 1] * scale_log2e - l1);
                const uint32_t pp = pack_bf16x2(p0, p1);
                const uint32_t dd = pack_bf16x2(p0 * (dpacc[4 * jj + 2 * h] - d0) * scale,
                                                p1 * (dpacc[4 * jj + 2 * h + 1] - d1) * scale);
                pa[jj >> 1][(jj & 1) * 2 + h] = pp;
                da[jj >> 1][(jj & 1) * 2 + h] = dd;
                // dS^T[key][q]: atom q / 64, 16 B chunk (q % 64) / 8 swizzled with key & 7
                const int key = key_row + 8 * h;
                *reinterpret_cast<uint32_t*>(smem + OFF_DS + (jj >> 3) * ATOM + key * 128 + (((jj & 7) ^ (key & 7)) << 4) +
                                             4 * (lane & 3)) = dd;
            }
        }
        // dV += P^T dO, dK += dS^T Q: reduction over the 128 queries of the block, B operands MN-major (16 rows per step)
        wgmma_fence();
#pragma unroll
        for (int kc = 0; kc < BLK / 16; ++kc)
            wgmma_bf16_rs_n64<1>(dv, pa[kc], make_smem_desc_sw128(sdo + kc * 2048, 0, 1024), 1u);
#pragma unroll
        for (int kc = 0; kc < BLK / 16; ++kc)
            wgmma_bf16_rs_n64<1>(dk, da[kc], make_smem_desc_sw128(sq + kc * 2048, 0, 1024), 1u);
        wgmma_commit();
        fence_proxy_async_smem();          // generic-proxy smem writes (dS^T) -> visible to the tensor core
        named_bar_sync(1, NUM_THREADS);    // dS^T of both warpgroups is in shared memory
        // dQ (this warpgroup's 64 queries) = dS K_j: A = dS^T atom wg (MN-major), B = K_j (MN-major), 8 steps of 16 keys
        float dq[HEAD_DIM / 2];
        wgmma_fence();
#pragma unroll
        for (int kc = 0; kc < BLK / 16; ++kc)
            wgmma_bf16_n64<1, 1>(dq, make_smem_desc_sw128(sds + wg * ATOM + kc * 2048, ATOM, 1024),
                                 make_smem_desc_sw128(sk + kc * 2048, 0, 1024), kc > 0 ? 1u : 0u);
        wgmma_commit();
        wgmma_wait<0>();
        wgmma_fence_regs(dq);
        wgmma_fence_regs(dv);
        wgmma_fence_regs(dk);
        // partial dQ of THIS key block into slice j of dq_part ([4, T, D] bf16; attn_dq_reduce_kernel sums the four slices in
        // fp32) — no atomics, half the bytes of fp32 partials
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const long long token = tok0 + wg * 64 + (warp & 3) * 16 + (lane >> 2) + 8 * h;
            bf16* dqp = dq_part + (static_cast<long long>(j) * total_tokens + token) * d_model + head * HEAD_DIM + qcol;
#pragma unroll
            for (int jj = 0; jj < HEAD_DIM / 8; ++jj)
                *reinterpret_cast<uint32_t*>(dqp + 8 * jj) = pack_bf16x2(dq[4 * jj + 2 * h], dq[4 * jj + 2 * h + 1]);
        }
        named_bar_sync(1, NUM_THREADS);    // dS^T, Q_i, dO_i, lse / delta of this block are no longer read
        if (tid == 0 && i + 2 < NUM_QB) load_q(i + 2);
    }
    // dK_j / dV_j
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        const long long key = seq0 + j * BLK + key_row + 8 * h;
        bf16* dkp = dqkv + key * (3ll * d_model) + d_model + head * HEAD_DIM + qcol;
        bf16* dvp = dqkv + key * (3ll * d_model) + 2 * d_model + head * HEAD_DIM + qcol;
#pragma unroll
        for (int jj = 0; jj < HEAD_DIM / 8; ++jj) {
            *reinterpret_cast<uint32_t*>(dkp + 8 * jj) = pack_bf16x2(dk[4 * jj + 2 * h], dk[4 * jj + 2 * h + 1]);
            *reinterpret_cast<uint32_t*>(dvp + 8 * jj) = pack_bf16x2(dv[4 * jj + 2 * h], dv[4 * jj + 2 * h + 1]);
        }
    }
}

typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

// prologue: delta[t, h] = sum_d dO[t, h, d] * O[t, h, d]  (one warp per (token, head): 64 bf16 = one 128 B row segment each)
__global__ void __launch_bounds__(256) attn_delta_kernel(const bf16* __restrict__ dout, const bf16* __restrict__ out,
                                                         float* __restrict__ delta, long long pairs) {
    const long long w = (static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (w >= pairs) return;
    const __nv_bfloat162 a = reinterpret_cast<const __nv_bfloat162*>(dout + w * HEAD_DIM)[lane];
    const __nv_bfloat162 b = reinterpret_cast<const __nv_bfloat162*>(out + w * HEAD_DIM)[lane];
    float acc = __bfloat162float(a.x) * __bfloat162float(b.x) + __bfloat162float(a.y) * __bfloat162float(b.y);
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, d);
    if (lane == 0) delta[w] = acc;
}

// epilogue: dQ = sum of the per-key-block partials, written as bf16 into the Q third of dqkv
__global__ void __launch_bounds__(256) attn_dq_reduce_kernel(const bf16* __restrict__ dq_part, bf16* __restrict__ dqkv,
                                                             long long tokens, int d_model, int parts) {
    const long long i8 = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;   // 8-element (16 B) index inside [T, D]
    const long long n8 = tokens * d_model / 8;
    if (i8 >= n8) return;
    float acc[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) acc[e] = 0.f;
    for (int p = 0; p < parts; ++p) {
        const int4 t = reinterpret_cast<const int4*>(dq_part)[i8 + p * n8];
        const uint32_t w[4] = {(uint32_t)t.x, (uint32_t)t.y, (uint32_t)t.z, (uint32_t)t.w};
#pragma unroll
        for (int e = 0; e < 4; ++e) {
            const float2 f = unpack_bf16x2(w[e]);
            acc[2 * e] += f.x;
            acc[2 * e + 1] += f.y;
        }
    }
    const long long el = i8 * 8, tok = el / d_model, col = el - tok * d_model;
    *reinterpret_cast<int4*>(dqkv + tok * 3 * d_model + col) =
        make_int4(pack_bf16x2(acc[0], acc[1]), pack_bf16x2(acc[2], acc[3]), pack_bf16x2(acc[4], acc[5]), pack_bf16x2(acc[6], acc[7]));
}

}  // namespace attnb
}  // namespace lah

using namespace lah;
using namespace lah::attnb;

extern "C" {

// qkv [T, 3D] bf16 (forward input), out [T, D] bf16 (forward output), dout [T, D] bf16, lse2 [T, H] fp32 (forward output)
// -> dqkv [T, 3D] bf16.  Scratch: delta [T, H] fp32 (rowsum(dout o out), computed here), dq_part [4, T, D] bf16 (the four
// per-key-block partials of dQ, reduced into the Q third of dqkv here).  Three launches, no PyTorch ops around them.
int lah_attention_bwd(const void* qkv, const void* out, const void* dout, const float* lse2, float* delta, void* dqkv,
                      void* dq_part, int batch, int num_heads, int d_model, cudaStream_t st) {
    if (d_model != num_heads * HEAD_DIM) return -2;
    static PFN_encodeTiled fn = nullptr;
    if (!fn) {
        void* ptr = nullptr;
        cudaDriverEntryPointQueryResult qres;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &ptr, cudaEnableDefault, &qres) != cudaSuccess || !ptr)
            return -100;
        fn = reinterpret_cast<PFN_encodeTiled>(ptr);
    }
    CUtensorMap tm_qkv, tm_do;
    cuuint32_t box[2] = {HEAD_DIM, BLK};
    cuuint32_t estr[2] = {1, 1};
    {
        cuuint64_t dims[2] = {(cuuint64_t)3 * d_model, (cuuint64_t)batch * S_LEN};
        cuuint64_t strides[1] = {(cuuint64_t)3 * d_model * 2};
        CUresult r = fn(&tm_qkv, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(qkv), dims, strides, box, estr,
                        CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                        CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
        if (r != CUDA_SUCCESS) return -1000 - (int)r;
    }
    {
        cuuint64_t dims[2] = {(cuuint64_t)d_model, (cuuint64_t)batch * S_LEN};
        cuuint64_t strides[1] = {(cuuint64_t)d_model * 2};
        CUresult r = fn(&tm_do, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(dout), dims, strides, box, estr,
                        CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                        CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
        if (r != CUDA_SUCCESS) return -1000 - (int)r;
    }
    static bool configured = false;
    if (!configured) {
        cudaError_t e = cudaFuncSetAttribute(attention_bwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_TOTAL);
        if (e != cudaSuccess) return -(int)e;
        configured = true;
    }
    if (batch <= 0) return 0;
    const float scale = 1.f / sqrtf((float)HEAD_DIM);
    const long long tokens = (long long)batch * S_LEN, pairs = tokens * num_heads;
    attn_delta_kernel<<<(unsigned)((pairs * 32 + 255) / 256), 256, 0, st>>>((const bf16*)dout, (const bf16*)out, delta, pairs);
    attention_bwd_kernel<<<batch * num_heads * (S_LEN / BLK), NUM_THREADS, SMEM_TOTAL, st>>>(
        tm_qkv, tm_do, lse2, delta, (bf16*)dqkv, (bf16*)dq_part, tokens, d_model, num_heads, scale,
        scale * 1.4426950408889634f);
    attn_dq_reduce_kernel<<<(unsigned)((tokens * d_model / 8 + 255) / 256), 256, 0, st>>>((const bf16*)dq_part, (bf16*)dqkv, tokens, d_model,
                                                                                         S_LEN / BLK);
    return -(int)cudaGetLastError();
}

}  // extern "C"
