// attention.cu — wgmma self-attention for the transformer expert (head_dim 64, any sequence length S in 1..MAX_SEQ;
// reference: nn.MultiheadAttention inside experiments/throughput/layers.py:22-51).
//
// FORWARD (this file): flash attention.  One CTA owns one 128-query tile of one (batch, head); two consumer warpgroups own
// 64 query rows each.  K / V stream through a 2-stage TMA pipeline in 128-key blocks; per block S = Q K^T is computed by
// wgmma into registers, the online softmax runs on those registers (a row is spread over the 4 lanes of a quad), and the
// bf16 probabilities are fed straight from registers as the A operand of O += P V (their accumulator layout IS the A
// fragment layout).  S and P never touch shared memory or HBM.  The kernel also emits the row log-sum-exp (base 2) that the
// BACKWARD kernel (attention_bwd.cu) needs to recompute P without a second softmax pass.
//
// Input : qkv [T = batch*S, 3*D] bf16 (output of the fused in_proj GEMM: [q | k | v] per token, heads contiguous)
// Output: out [T, D] bf16 (heads concatenated, ready for out_proj); lse2 [T, heads] fp32 (optional)
//
// Sequence length: ceil(S / 128) query tiles and key blocks per sequence.  The tensor map is 3-D {3*D, S, batch}, so TMA
// zero-fills the rows past the end of a sequence and no tile reads the next one.  In the last key block of a partial
// sequence (S % 128 != 0) the scores of keys >= S are set to -inf before the row maximum, so they enter neither l nor the
// LSE; rows of queries >= S are computed on zeros and not stored.  Full blocks take exactly the arithmetic of the
// 512-token kernel: the tail test is one uniform branch per key block.
#include "sm90.cuh"
#include "dropout.cuh"
#include <stdlib.h>

namespace lah {
namespace attn {

constexpr int HEAD_DIM = 64;
constexpr int Q_TILE = 128;

namespace v2 {

constexpr int KB = 128;                       // keys per block
constexpr int NUM_THREADS2 = 256;             // two consumer warpgroups; thread 0 also drives TMA
constexpr int TILE_BYTES = 128 * HEAD_DIM * 2;            // 16 KB: a 128 x 64 bf16 tile (Q tile, K block, V block)
constexpr int OFF_Q2 = 0;
constexpr int OFF_K2 = OFF_Q2 + TILE_BYTES;               // 2 stages
constexpr int OFF_V2 = OFF_K2 + 2 * TILE_BYTES;           // 2 stages
constexpr int OFF_BAR2 = OFF_V2 + 2 * TILE_BYTES;
constexpr int NUM_BARS = 1 + 2;
constexpr int SMEM_TOTAL2 = OFF_BAR2 + NUM_BARS * 8 + 16 + 1024;

// DROP: attention dropout (dropout.cuh, site 0).  The kept bf16 probabilities feed O += P V; the row sum l (and so the LSE)
// keeps summing ALL of them, and 1 / (1 - p) is folded into the final 1 / l.
template <bool DROP>
__global__ void __launch_bounds__(NUM_THREADS2, 1)
attention_fwd_v2_kernel(const __grid_constant__ CUtensorMap tm_qkv, bf16* __restrict__ out, float* __restrict__ lse2,
                        int d_model, int num_heads, int seq_len, float scale_log2e, unsigned long long seed, uint32_t thr,
                        float rescale) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint64_t* bars = reinterpret_cast<uint64_t*>(smem + OFF_BAR2);
    uint64_t* bar_q = bars;
    uint64_t* kv_full = bars + 1;   // [2]

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, wg = warp >> 2;
    const int num_kb = (seq_len + KB - 1) / KB;   // key blocks = query tiles per sequence
    const int qt = blockIdx.x % num_kb;
    const int head = (blockIdx.x / num_kb) % num_heads;
    const int batch = (blockIdx.x / num_kb) / num_heads;

    auto load_kv = [&](int j) {   // thread 0 only; stage j & 1 must be free
        const int st = j & 1;
        mbar_arrive_expect_tx(&kv_full[st], 2 * TILE_BYTES);
        tma_load_3d(smem + OFF_K2 + st * TILE_BYTES, &tm_qkv, &kv_full[st], d_model + head * HEAD_DIM, j * KB, batch);
        tma_load_3d(smem + OFF_V2 + st * TILE_BYTES, &tm_qkv, &kv_full[st], 2 * d_model + head * HEAD_DIM, j * KB, batch);
    };
    if (tid == 0) {
        tma_prefetch_desc(&tm_qkv);
        mbar_init(bar_q, 1);
        mbar_init(&kv_full[0], 1);
        mbar_init(&kv_full[1], 1);
        fence_mbar_init();
        mbar_arrive_expect_tx(bar_q, TILE_BYTES);
        tma_load_3d(smem + OFF_Q2, &tm_qkv, bar_q, head * HEAD_DIM, qt * Q_TILE, batch);
        load_kv(0);
        if (num_kb > 1) load_kv(1);
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
    for (int j = 0; j < num_kb; ++j) {
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
        // keep bits of this thread's 64 scores, bit i <-> s[i], generated while the S MMA runs: one Philox granule per
        // 16-key chunk kc covers rows {g, g+8} x keys {2c, 2c+1, 2c+8, 2c+9} = s[8kc .. 8kc+7]
        uint32_t km[2] = {0u, 0u};
        if constexpr (DROP) {
            const uint32_t q = qt * Q_TILE + wg * 64 + (warp & 3) * 16 + (lane >> 2);
#pragma unroll
            for (int kc = 0; kc < KB / 16; ++kc) {
                const uint4 bits = drop::attn_bits(seed, batch, head, drop::granule_attn(q), (8 * j + kc) * 4 + (lane & 3), q & 1u);
#pragma unroll
                for (int e = 0; e < 8; ++e) {   // lane e = h * 4 + jl * 2 + i  <->  s[4 (2kc + jl) + 2h + i]
                    const int idx = 8 * kc + 4 * ((e >> 1) & 1) + 2 * (e >> 2) + (e & 1);
                    km[idx >> 5] |= static_cast<uint32_t>(drop::keep(bits, e, thr)) << (idx & 31);
                }
            }
        }
        wgmma_wait<0>();
        wgmma_fence_regs(s);
        if (j * KB + KB > seq_len) {   // last block of a partial sequence: s[4 jj + 2 h + i] is key 8 jj + 2 (lane & 3) + i
#pragma unroll
            for (int jj = 0; jj < KB / 8; ++jj)
#pragma unroll
                for (int i = 0; i < 2; ++i)
                    if (j * KB + 8 * jj + 2 * (lane & 3) + i >= seq_len) s[4 * jj + i] = s[4 * jj + 2 + i] = -INFINITY;
        }
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
                uint32_t pk = pack_bf16x2(exp2f(s[4 * jj + 2 * h] * scale_log2e - ms),
                                          exp2f(s[4 * jj + 2 * h + 1] * scale_log2e - ms));
                const float2 back = unpack_bf16x2(pk);   // sum what the tensor core will actually see
                sum += back.x + back.y;
                if constexpr (DROP) {
                    const int idx = 4 * jj + 2 * h;
                    const uint32_t b2 = (km[idx >> 5] >> (idx & 31)) & 3u;
                    pk &= ((b2 & 1u) ? 0x0000ffffu : 0u) | ((b2 & 2u) ? 0xffff0000u : 0u);
                }
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
        if (j + 2 < num_kb) {
            named_bar_sync(1, NUM_THREADS2);   // both warpgroups are done with stage st
            if (tid == 0) load_kv(j + 2);
        }
    }
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        float lt = l[h];
        lt += __shfl_xor_sync(0xffffffffu, lt, 1);
        lt += __shfl_xor_sync(0xffffffffu, lt, 2);
        const float inv = DROP ? rescale / lt : 1.f / lt;
        const int q = qt * Q_TILE + wg * 64 + (warp & 3) * 16 + (lane >> 2) + 8 * h;
        if (q >= seq_len) continue;
        const long long token = static_cast<long long>(batch) * seq_len + q;
        if (lse2 && (lane & 3) == 0) lse2[token * num_heads + head] = m[h] * scale_log2e + log2f(lt);
        bf16* op = out + token * d_model + head * HEAD_DIM + 2 * (lane & 3);
#pragma unroll
        for (int jj = 0; jj < HEAD_DIM / 8; ++jj)
            *reinterpret_cast<uint32_t*>(op + 8 * jj) = pack_bf16x2(o[4 * jj + 2 * h] * inv, o[4 * jj + 2 * h + 1] * inv);
    }
}

}  // namespace v2

}  // namespace attn
}  // namespace lah

using namespace lah;
using namespace lah::attn;

extern "C" {

// qkv: [tokens, 3*d_model] bf16, tokens = batch * seq_len, 1 <= seq_len <= MAX_SEQ; out: [tokens, d_model] bf16;
// lse2: [tokens, heads] fp32 or NULL.  Returns -2 for a sequence length out of range or one that does not divide tokens.
// drop_thr < 0: no dropout; otherwise attention dropout with threshold drop_thr (dropout.cuh), seed, rescale = 1 / (1 - p)
int lah_attention_fwd(const void* qkv, void* out, float* lse2, long long tokens, int seq_len, int num_heads, int d_model,
                      unsigned long long seed, int drop_thr, float rescale, cudaStream_t st) {
    if (d_model != num_heads * HEAD_DIM || drop_thr > 65535) return -2;
    if (seq_len < 1 || seq_len > drop::MAX_SEQ || tokens < 0 || tokens % seq_len) return -2;
    const long long batch = tokens / seq_len;
    if (batch == 0) return 0;
    CUtensorMap tm;
    {   // 3-D {columns, position in sequence, sequence}: a tile never crosses into the next sequence
        uint64_t dims[3] = {(uint64_t)3 * d_model, (uint64_t)seq_len, (uint64_t)batch};
        uint64_t str[2] = {(uint64_t)3 * d_model * 2, (uint64_t)seq_len * 3 * d_model * 2};
        uint32_t box[3] = {HEAD_DIM, 128, 1};
        int r = make_tmap(&tm, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, qkv, dims, str, box);
        if (r) return r;
    }
    if (int e = set_max_dynamic_smem<v2::attention_fwd_v2_kernel<false>>(v2::SMEM_TOTAL2)) return e;
    if (int e = set_max_dynamic_smem<v2::attention_fwd_v2_kernel<true>>(v2::SMEM_TOTAL2)) return e;
    const float scale_log2e = 1.4426950408889634f / sqrtf((float)HEAD_DIM);
    const long long ctas = batch * num_heads * ((seq_len + Q_TILE - 1) / Q_TILE);
    if (ctas > 0x7fffffffll) return -2;
    auto kern = drop_thr < 0 ? v2::attention_fwd_v2_kernel<false> : v2::attention_fwd_v2_kernel<true>;
    kern<<<(unsigned)ctas, v2::NUM_THREADS2, v2::SMEM_TOTAL2, st>>>(
        tm, (bf16*)out, lse2, d_model, num_heads, seq_len, scale_log2e, seed, static_cast<uint32_t>(drop_thr < 0 ? 0 : drop_thr),
        rescale);
    return -(int)cudaGetLastError();
}

}  // extern "C"
