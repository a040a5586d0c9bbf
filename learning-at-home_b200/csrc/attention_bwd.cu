// attention_bwd.cu — wgmma self-attention BACKWARD for the transformer expert (head_dim 64, any sequence length S in
// 1..MAX_SEQ).
// The reference's transformer expert cannot be trained at all (in-place transpose of a leaf, SURVEY.md §0.3); this kernel is
// what makes the sm_90a transformer expert trainable without falling back to eager PyTorch.
//
// One CTA = one (batch, head, 128-key block j); consumer warpgroup w owns keys [64w, 64w + 64) of the block.  K_j / V_j stay
// in shared memory; the ceil(S / 128) query blocks i stream through a 2-stage TMA pipeline (Q_i and dO_i).  Per query block, all
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
//
// DROP (attention dropout, dropout.cuh site 0): the keep mask M is regenerated from the seed, never stored.  With
// Pd = M o P / (1 - p):  dV += Pd^T dO,  dS = P o (M o dP / (1 - p) - Delta) * scale, Delta = rowsum(dO o O) of the DROPPED
// output O (attn_delta_kernel, unchanged); LSE is that of the undropped softmax.  P^T is masked but not scaled in the dV
// MMA; 1 / (1 - p) is applied to dV once at the end.
//
// Sequence length: the tensor maps are 3-D {columns, S, batch}, so rows past the end of a sequence arrive as zeros.  Zeros
// alone do not make P vanish (exp2(0 - LSE) is not 0, and a garbage LSE can make it inf, and inf * 0 is NaN), so in a
// partial block P^T and dS^T are forced to exactly 0: queries >= S get LSE = +inf and Delta = 0 (LSE and Delta are only
// read for valid queries), keys >= S get S^T = -inf.  No dK / dV row is stored for keys >= S and no dQ-partial row for
// queries >= S.  Full blocks run exactly the arithmetic of the 512-token kernel.
#include "sm90.cuh"
#include "dropout.cuh"

namespace lah {
namespace attnb {

constexpr int HEAD_DIM = 64;
constexpr int BLK = 128;                       // query block == key block
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

template <bool DROP>
__global__ void __launch_bounds__(NUM_THREADS, 1)
attention_bwd_kernel(const __grid_constant__ CUtensorMap tm_qkv, const __grid_constant__ CUtensorMap tm_do,
                     const float* __restrict__ lse2, const float* __restrict__ delta, bf16* __restrict__ dqkv,
                     bf16* __restrict__ dq_part, long long total_tokens, int d_model, int num_heads, int seq_len, float scale,
                     float scale_log2e, unsigned long long seed, uint32_t thr, float rescale) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint64_t* bars = reinterpret_cast<uint64_t*>(smem + OFF_BAR);
    uint64_t* kv_full = bars;
    uint64_t* q_full = bars + 1;     // [2]
    float* s_lse = reinterpret_cast<float*>(smem + OFF_LSE);
    float* s_delta = s_lse + BLK;

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, wg = warp >> 2;
    const int num_qb = (seq_len + BLK - 1) / BLK;   // query blocks = key blocks per sequence
    const int j = blockIdx.x % num_qb;
    const int head = (blockIdx.x / num_qb) % num_heads;
    const int batch = (blockIdx.x / num_qb) / num_heads;
    const long long seq0 = static_cast<long long>(batch) * seq_len;

    auto load_q = [&](int i) {   // thread 0 only; stage i & 1 must be free
        const int st = i & 1;
        mbar_arrive_expect_tx(&q_full[st], 2 * TILE);
        tma_load_3d(smem + OFF_Q + st * TILE, &tm_qkv, &q_full[st], head * HEAD_DIM, i * BLK, batch);
        tma_load_3d(smem + OFF_DO + st * TILE, &tm_do, &q_full[st], head * HEAD_DIM, i * BLK, batch);
    };
    if (tid == 0) {
        tma_prefetch_desc(&tm_qkv);
        tma_prefetch_desc(&tm_do);
        mbar_init(kv_full, 1);
        mbar_init(&q_full[0], 1);
        mbar_init(&q_full[1], 1);
        fence_mbar_init();
        mbar_arrive_expect_tx(kv_full, 2 * TILE);
        tma_load_3d(smem + OFF_K, &tm_qkv, kv_full, d_model + head * HEAD_DIM, j * BLK, batch);
        tma_load_3d(smem + OFF_V, &tm_qkv, kv_full, 2 * d_model + head * HEAD_DIM, j * BLK, batch);
        load_q(0);
        if (num_qb > 1) load_q(1);
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
    for (int i = 0; i < num_qb; ++i) {
        const int st = i & 1;
        const long long tok0 = seq0 + i * BLK;
        const int qr = tid & (BLK - 1);   // query row of the block whose LSE (tid < 128) or Delta this thread loads
        const bool qvalid = i * BLK + qr < seq_len;
        if (tid < BLK) s_lse[qr] = qvalid ? __ldg(lse2 + (tok0 + qr) * num_heads + head) : INFINITY;
        else s_delta[qr] = qvalid ? __ldg(delta + (tok0 + qr) * num_heads + head) : 0.f;
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
        if (j * BLK + BLK > seq_len) {   // last key block of a partial sequence: sacc[4 jj + 2 h + par] is key key_row + 8 h
#pragma unroll
            for (int h = 0; h < 2; ++h)
                if (j * BLK + key_row + 8 * h >= seq_len)
#pragma unroll
                    for (int jj = 0; jj < BLK / 8; ++jj) sacc[4 * jj + 2 * h] = sacc[4 * jj + 2 * h + 1] = -INFINITY;
        }
        const uint32_t kk = j * BLK + key_row;   // this thread's keys: kk, kk + 8
        uint32_t km = 0u;
        uint32_t pa[BLK / 16][4], da[BLK / 16][4];
#pragma unroll
        for (int jj = 0; jj < BLK / 8; ++jj) {
            if constexpr (DROP) {
                // keep bits of the 16-query chunk jp = jj / 2, bit 4 jl + 2h + par <-> sacc[4 (2jp + jl) + 2h + par]
                // (keys kk + 8h x queries 16jp + qcol + 8jl + par): the granules of query parity 0 / 1 each hold 4 of them
                if ((jj & 1) == 0) {
                    km = 0u;
#pragma unroll
                    for (int par = 0; par < 2; ++par) {
                        const uint4 bits = drop::attn_bits(seed, batch, head, (8 * i + (jj >> 1)) * 4 + (lane & 3),
                                                           drop::granule_attn(kk), par);
#pragma unroll
                        for (int jl = 0; jl < 2; ++jl)
#pragma unroll
                            for (int h = 0; h < 2; ++h)   // lane = query bit 3 * 4 + (key bit 0 | key bit 3 << 1)
                                km |= static_cast<uint32_t>(drop::keep(bits, jl * 4 + static_cast<int>(kk & 1u) + 2 * h, thr))
                                      << (4 * jl + 2 * h + par);
                    }
                }
            }
            const int q = 8 * jj + qcol;
            const float l0 = s_lse[q], l1 = s_lse[q + 1], d0 = s_delta[q], d1 = s_delta[q + 1];
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const float p0 = exp2f(sacc[4 * jj + 2 * h] * scale_log2e - l0);
                const float p1 = exp2f(sacc[4 * jj + 2 * h + 1] * scale_log2e - l1);
                uint32_t pp, dd;
                if constexpr (DROP) {
                    const int idx = 4 * (jj & 1) + 2 * h;
                    const bool k0 = (km >> idx) & 1u, k1 = (km >> (idx + 1)) & 1u;
                    pp = pack_bf16x2(k0 ? p0 : 0.f, k1 ? p1 : 0.f);
                    dd = pack_bf16x2(p0 * ((k0 ? dpacc[4 * jj + 2 * h] * rescale : 0.f) - d0) * scale,
                                     p1 * ((k1 ? dpacc[4 * jj + 2 * h + 1] * rescale : 0.f) - d1) * scale);
                } else {
                    pp = pack_bf16x2(p0, p1);
                    dd = pack_bf16x2(p0 * (dpacc[4 * jj + 2 * h] - d0) * scale, p1 * (dpacc[4 * jj + 2 * h + 1] - d1) * scale);
                }
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
        // partial dQ of THIS key block into slice j of dq_part ([ceil(S / 128), T, D] bf16; attn_dq_reduce_kernel sums the
        // slices in fp32) — no atomics, half the bytes of fp32 partials
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int q = wg * 64 + (warp & 3) * 16 + (lane >> 2) + 8 * h;
            if (i * BLK + q >= seq_len) continue;
            const long long token = tok0 + q;
            bf16* dqp = dq_part + (static_cast<long long>(j) * total_tokens + token) * d_model + head * HEAD_DIM + qcol;
#pragma unroll
            for (int jj = 0; jj < HEAD_DIM / 8; ++jj)
                *reinterpret_cast<uint32_t*>(dqp + 8 * jj) = pack_bf16x2(dq[4 * jj + 2 * h], dq[4 * jj + 2 * h + 1]);
        }
        named_bar_sync(1, NUM_THREADS);    // dS^T, Q_i, dO_i, lse / delta of this block are no longer read
        if (tid == 0 && i + 2 < num_qb) load_q(i + 2);
    }
    // dK_j / dV_j
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        if (j * BLK + key_row + 8 * h >= seq_len) continue;
        const long long key = seq0 + j * BLK + key_row + 8 * h;
        bf16* dkp = dqkv + key * (3ll * d_model) + d_model + head * HEAD_DIM + qcol;
        bf16* dvp = dqkv + key * (3ll * d_model) + 2 * d_model + head * HEAD_DIM + qcol;
#pragma unroll
        for (int jj = 0; jj < HEAD_DIM / 8; ++jj) {
            *reinterpret_cast<uint32_t*>(dkp + 8 * jj) = pack_bf16x2(dk[4 * jj + 2 * h], dk[4 * jj + 2 * h + 1]);
            if constexpr (DROP)
                *reinterpret_cast<uint32_t*>(dvp + 8 * jj) = pack_bf16x2(dv[4 * jj + 2 * h] * rescale, dv[4 * jj + 2 * h + 1] * rescale);
            else
                *reinterpret_cast<uint32_t*>(dvp + 8 * jj) = pack_bf16x2(dv[4 * jj + 2 * h], dv[4 * jj + 2 * h + 1]);
        }
    }
}

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

// epilogue: dQ = sum of the per-key-block partials in key-block order (deterministic), written as bf16 into the Q third of dqkv
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
// -> dqkv [T, 3D] bf16, T = batch * seq_len, 1 <= seq_len <= MAX_SEQ (-2 otherwise, or when seq_len does not divide T).
// Scratch: delta [T, H] fp32 (rowsum(dout o out), computed here), dq_part [ceil(seq_len / 128), T, D] bf16 (one partial
// of dQ per key block, reduced into the Q third of dqkv here).  Three launches, no PyTorch ops around them.
// drop_thr < 0: the forward ran without dropout; otherwise the same (seed, drop_thr, rescale) as lah_attention_fwd.
int lah_attention_bwd(const void* qkv, const void* out, const void* dout, const float* lse2, float* delta, void* dqkv,
                      void* dq_part, long long tokens, int seq_len, int num_heads, int d_model, unsigned long long seed,
                      int drop_thr, float rescale, cudaStream_t st) {
    if (d_model != num_heads * HEAD_DIM || drop_thr > 65535) return -2;
    if (seq_len < 1 || seq_len > drop::MAX_SEQ || tokens < 0 || tokens % seq_len) return -2;
    const long long batch = tokens / seq_len;
    if (batch == 0) return 0;
    CUtensorMap tm_qkv, tm_do;
    const uint32_t box[3] = {HEAD_DIM, BLK, 1};
    {   // 3-D {columns, position in sequence, sequence}: a tile never crosses into the next sequence
        uint64_t dims[3] = {(uint64_t)3 * d_model, (uint64_t)seq_len, (uint64_t)batch};
        uint64_t str[2] = {(uint64_t)3 * d_model * 2, (uint64_t)seq_len * 3 * d_model * 2};
        int r = make_tmap(&tm_qkv, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, qkv, dims, str, box);
        if (r) return r;
    }
    {
        uint64_t dims[3] = {(uint64_t)d_model, (uint64_t)seq_len, (uint64_t)batch};
        uint64_t str[2] = {(uint64_t)d_model * 2, (uint64_t)seq_len * d_model * 2};
        int r = make_tmap(&tm_do, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, dout, dims, str, box);
        if (r) return r;
    }
    if (int e = set_max_dynamic_smem<attention_bwd_kernel<false>>(SMEM_TOTAL)) return e;
    if (int e = set_max_dynamic_smem<attention_bwd_kernel<true>>(SMEM_TOTAL)) return e;
    const float scale = 1.f / sqrtf((float)HEAD_DIM);
    const int blocks = (seq_len + BLK - 1) / BLK;
    const long long pairs = tokens * num_heads, ctas = batch * num_heads * blocks;
    if (ctas > 0x7fffffffll) return -2;
    attn_delta_kernel<<<(unsigned)((pairs * 32 + 255) / 256), 256, 0, st>>>((const bf16*)dout, (const bf16*)out, delta, pairs);
    auto kern = drop_thr < 0 ? attention_bwd_kernel<false> : attention_bwd_kernel<true>;
    kern<<<(unsigned)ctas, NUM_THREADS, SMEM_TOTAL, st>>>(
        tm_qkv, tm_do, lse2, delta, (bf16*)dqkv, (bf16*)dq_part, tokens, d_model, num_heads, seq_len, scale,
        scale * 1.4426950408889634f, seed, static_cast<uint32_t>(drop_thr < 0 ? 0 : drop_thr), rescale);
    attn_dq_reduce_kernel<<<(unsigned)((tokens * d_model / 8 + 255) / 256), 256, 0, st>>>((const bf16*)dq_part, (bf16*)dqkv, tokens, d_model,
                                                                                         blocks);
    return -(int)cudaGetLastError();
}

}  // extern "C"
