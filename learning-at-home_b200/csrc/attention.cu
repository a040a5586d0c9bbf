// attention.cu — wgmma self-attention for the transformer expert (d_model 1024, 16 heads x 64, seq 512;
// reference: nn.MultiheadAttention inside experiments/throughput/layers.py:22-51).
//
// FORWARD (this file): flash attention.  One CTA owns one 128-query tile of one (batch, head); two consumer warpgroups own
// 64 query rows each.  K / V stream through a 2-stage TMA pipeline in 128-key blocks; per block S = Q K^T is computed by
// wgmma into registers, the online softmax runs on those registers (a row is spread over the 4 lanes of a quad), and the
// bf16 probabilities are fed straight from registers as the A operand of O += P V (their accumulator layout IS the A
// fragment layout).  S and P never touch shared memory or HBM.  The kernel also emits the row log-sum-exp (base 2) that the
// BACKWARD kernel (attention_bwd.cu) needs to recompute P without a second softmax pass.
//
// Input : qkv [T = batch*512, 3*D] bf16 (output of the fused in_proj GEMM: [q | k | v] per token, heads contiguous)
// Output: out [T, D] bf16 (heads concatenated, ready for out_proj); lse2 [T, heads] fp32 (optional)
#include "sm90.cuh"
#include <stdlib.h>

namespace lah {
namespace attn {

constexpr int S_LEN = 512;      // keys per sequence
constexpr int HEAD_DIM = 64;
constexpr int Q_TILE = 128;

namespace v2 {

constexpr int KB = 128;                       // keys per block
constexpr int NUM_KB = S_LEN / KB;            // 4
constexpr int NUM_THREADS2 = 256;             // two consumer warpgroups; thread 0 also drives TMA
constexpr int TILE_BYTES = 128 * HEAD_DIM * 2;            // 16 KB: a 128 x 64 bf16 tile (Q tile, K block, V block)
constexpr int OFF_Q2 = 0;
constexpr int OFF_K2 = OFF_Q2 + TILE_BYTES;               // 2 stages
constexpr int OFF_V2 = OFF_K2 + 2 * TILE_BYTES;           // 2 stages
constexpr int OFF_BAR2 = OFF_V2 + 2 * TILE_BYTES;
constexpr int NUM_BARS = 1 + 2;
constexpr int SMEM_TOTAL2 = OFF_BAR2 + NUM_BARS * 8 + 16 + 1024;

__global__ void __launch_bounds__(NUM_THREADS2, 1)
attention_fwd_v2_kernel(const __grid_constant__ CUtensorMap tm_qkv, bf16* __restrict__ out, float* __restrict__ lse2,
                        int d_model, int num_heads, float scale_log2e) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint64_t* bars = reinterpret_cast<uint64_t*>(smem + OFF_BAR2);
    uint64_t* bar_q = bars;
    uint64_t* kv_full = bars + 1;   // [2]

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, wg = warp >> 2;
    const int qt = blockIdx.x & 3;
    const int head = (blockIdx.x >> 2) % num_heads;
    const int batch = (blockIdx.x >> 2) / num_heads;
    const int seq_row0 = batch * S_LEN;

    auto load_kv = [&](int j) {   // thread 0 only; stage j & 1 must be free
        const int st = j & 1;
        mbar_arrive_expect_tx(&kv_full[st], 2 * TILE_BYTES);
        tma_load_2d(smem + OFF_K2 + st * TILE_BYTES, &tm_qkv, &kv_full[st], d_model + head * HEAD_DIM, seq_row0 + j * KB);
        tma_load_2d(smem + OFF_V2 + st * TILE_BYTES, &tm_qkv, &kv_full[st], 2 * d_model + head * HEAD_DIM, seq_row0 + j * KB);
    };
    if (tid == 0) {
        tma_prefetch_desc(&tm_qkv);
        mbar_init(bar_q, 1);
        mbar_init(&kv_full[0], 1);
        mbar_init(&kv_full[1], 1);
        fence_mbar_init();
        mbar_arrive_expect_tx(bar_q, TILE_BYTES);
        tma_load_2d(smem + OFF_Q2, &tm_qkv, bar_q, head * HEAD_DIM, seq_row0 + qt * Q_TILE);
        load_kv(0);
        load_kv(1);
    }
    __syncthreads();

    const uint32_t sq = smem_u32(smem + OFF_Q2) + wg * (64 * 128);   // this warpgroup's 64 query rows
    float o[HEAD_DIM / 2];
#pragma unroll
    for (int i = 0; i < HEAD_DIM / 2; ++i) o[i] = 0.f;
    // m = running row maximum (raw score units), l = this thread's share of the row sum (reduced over the quad at the end)
    float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};
    mbar_wait(bar_q, 0);
#pragma unroll 1
    for (int j = 0; j < NUM_KB; ++j) {
        const int st = j & 1;
        mbar_wait(&kv_full[st], (j >> 1) & 1);
        const uint32_t sk = smem_u32(smem + OFF_K2 + st * TILE_BYTES), sv = smem_u32(smem + OFF_V2 + st * TILE_BYTES);
        float s[KB / 2];
        wgmma_fence();
#pragma unroll
        for (int ks = 0; ks < HEAD_DIM / 16; ++ks)
            wgmma_bf16_n128<0, 0>(s, make_smem_desc_sw128(sq + ks * 32, 0, 1024), make_smem_desc_sw128(sk + ks * 32, 0, 1024),
                                  ks > 0 ? 1u : 0u);
        wgmma_commit();
        wgmma_wait<0>();
        wgmma_fence_regs(s);
        uint32_t pa[KB / 16][4];
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            float mx = -INFINITY;
#pragma unroll
            for (int jj = 0; jj < KB / 8; ++jj) mx = fmaxf(mx, fmaxf(s[4 * jj + 2 * h], s[4 * jj + 2 * h + 1]));
            mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
            mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
            const float m_new = fmaxf(m[h], mx);
            const float alpha = exp2f((m[h] - m_new) * scale_log2e);   // j == 0: m = -inf -> 0 (O and l are 0 then)
            m[h] = m_new;
            const float ms = m_new * scale_log2e;
            float sum = 0.f;
#pragma unroll
            for (int jj = 0; jj < KB / 8; ++jj) {
                const uint32_t pk = pack_bf16x2(exp2f(s[4 * jj + 2 * h] * scale_log2e - ms),
                                                exp2f(s[4 * jj + 2 * h + 1] * scale_log2e - ms));
                const float2 back = unpack_bf16x2(pk);   // sum what the tensor core will actually see
                sum += back.x + back.y;
                // A fragment of key chunk jj/2: regs {row g, keys 0-7 | row g+8, keys 0-7 | row g, keys 8-15 | row g+8, ...}
                pa[jj >> 1][(jj & 1) * 2 + h] = pk;
            }
            l[h] = l[h] * alpha + sum;
#pragma unroll
            for (int jj = 0; jj < HEAD_DIM / 8; ++jj) {
                o[4 * jj + 2 * h] *= alpha;
                o[4 * jj + 2 * h + 1] *= alpha;
            }
        }
        wgmma_fence();
#pragma unroll
        for (int kc = 0; kc < KB / 16; ++kc)   // V block as an MN-major B operand: 16 keys = 16 rows of 128 B per step
            wgmma_bf16_rs_n64<1>(o, pa[kc], make_smem_desc_sw128(sv + kc * 2048, 0, 1024), 1u);
        wgmma_commit();
        wgmma_wait<0>();
        wgmma_fence_regs(o);
        if (j + 2 < NUM_KB) {
            named_bar_sync(1, NUM_THREADS2);   // both warpgroups are done with stage st
            if (tid == 0) load_kv(j + 2);
        }
    }
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        float lt = l[h];
        lt += __shfl_xor_sync(0xffffffffu, lt, 1);
        lt += __shfl_xor_sync(0xffffffffu, lt, 2);
        const float inv = 1.f / lt;
        const long long token = seq_row0 + qt * Q_TILE + wg * 64 + (warp & 3) * 16 + (lane >> 2) + 8 * h;
        if (lse2 && (lane & 3) == 0) lse2[token * num_heads + head] = m[h] * scale_log2e + log2f(lt);
        bf16* op = out + token * d_model + head * HEAD_DIM + 2 * (lane & 3);
#pragma unroll
        for (int jj = 0; jj < HEAD_DIM / 8; ++jj)
            *reinterpret_cast<uint32_t*>(op + 8 * jj) = pack_bf16x2(o[4 * jj + 2 * h] * inv, o[4 * jj + 2 * h + 1] * inv);
    }
}

}  // namespace v2

typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

}  // namespace attn
}  // namespace lah

using namespace lah;
using namespace lah::attn;

extern "C" {

// qkv: [tokens, 3*d_model] bf16, tokens = batch * 512; out: [tokens, d_model] bf16; lse2: [tokens, heads] fp32 or NULL
int lah_attention_fwd(const void* qkv, void* out, float* lse2, int batch, int num_heads, int d_model, cudaStream_t st) {
    if (d_model != num_heads * HEAD_DIM) return -2;
    static PFN_encodeTiled fn = nullptr;
    if (!fn) {
        void* ptr = nullptr;
        cudaDriverEntryPointQueryResult qres;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &ptr, cudaEnableDefault, &qres) != cudaSuccess || !ptr)
            return -100;
        fn = reinterpret_cast<PFN_encodeTiled>(ptr);
    }
    CUtensorMap tm;
    cuuint64_t dims[2] = {(cuuint64_t)3 * d_model, (cuuint64_t)batch * S_LEN};
    cuuint64_t strides[1] = {(cuuint64_t)3 * d_model * 2};
    cuuint32_t box[2] = {HEAD_DIM, 128};
    cuuint32_t estr[2] = {1, 1};
    CUresult r = fn(&tm, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(qkv), dims, strides, box, estr,
                    CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                    CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) return -1000 - (int)r;
    static bool configured = false;
    if (!configured) {
        cudaError_t e = cudaFuncSetAttribute(v2::attention_fwd_v2_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, v2::SMEM_TOTAL2);
        if (e != cudaSuccess) return -(int)e;
        configured = true;
    }
    if (batch <= 0) return 0;
    const float scale_log2e = 1.4426950408889634f / sqrtf((float)HEAD_DIM);
    v2::attention_fwd_v2_kernel<<<batch * num_heads * (S_LEN / Q_TILE), v2::NUM_THREADS2, v2::SMEM_TOTAL2, st>>>(
        tm, (bf16*)out, lse2, d_model, num_heads, scale_log2e);
    return -(int)cudaGetLastError();
}

}  // extern "C"
