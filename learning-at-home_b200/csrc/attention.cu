// attention.cu — wgmma self-attention for the transformer expert (head_dim HD = 32, 64 or 128, any sequence length S in
// 1..MAX_SEQ; reference: nn.MultiheadAttention inside experiments/throughput/layers.py:22-51).
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
// Head dim: HD is a template parameter; the entry point dispatches on D / heads.  A tile row of a head is stored as swizzle
// atoms of 64 columns (128 B, 128B swizzle) or, at HD = 32, one atom of 32 columns (64 B, 64B swizzle: the head is never
// padded, since 64 columns would reach into the next head).  HD = 128 loads each 128-row tile as two 64-column atoms (two TMA
// boxes), runs the S MMA in 8 k16 steps across them and P V as m64n128 with V MN-major across the two atoms (LBO = one
// atom).  Shared memory: Q + 2 stages of K and V = 5 tiles of 128 x HD bf16 (40 / 80 / 160 KB).  Registers per thread: S 64,
// O HD / 2, P 32.
//
// Sequence length: ceil(S / 128) query tiles and key blocks per sequence.  The tensor map is 3-D {3*D, S, batch}, so TMA
// zero-fills the rows past the end of a sequence and no tile reads the next one.  In the last key block of a partial
// sequence (S % 128 != 0) the scores of keys >= S are set to -inf before the row maximum, so they enter neither l nor the
// LSE; rows of queries >= S are computed on zeros and not stored.  Full blocks take exactly the arithmetic of the
// 512-token kernel: the tail test is one uniform branch per key block.
//
// Key padding mask (MASK instantiations): key_mask is [batch, ceil(S / 32)] uint32, bit k % 32 of word k / 32 set iff key k
// is valid (attention_pack_key_mask_kernel; bits of keys >= S are clear, so the mask also covers the tail).  Producer and
// consumers walk the same list of key blocks that hold a valid key: a block without one is neither loaded nor computed.  In
// a partially valid block the scores of masked keys are set to -inf, as in the tail.  The mask is per key, so after the
// first block every row maximum is finite.  A sequence without a valid key processes no block: out = 0, lse2 = +inf.
//
// Causal attention (CAUSAL instantiations, never with MASK): query q attends to keys <= q.  Query tile i walks key blocks
// 0 .. i only (Q_TILE = KB, so block i is the diagonal one); producer and consumers both stop after it.  In the diagonal
// block the scores of keys > query are set to -inf before the row maximum (one uniform branch, as for the tail): that also
// covers keys >= S, which only the diagonal block of the last tile holds.  Every row keeps its own key, so l > 0.  CTAs are
// launched heaviest first within groups of CAUSAL_GROUP (batch, head) pairs: each group counts its query tiles down from
// the last one, so short tiles end each group and the grid, and the group's K / V stay in L2.
#include "sm90.cuh"
#include "dropout.cuh"
#include <stdlib.h>

namespace lah {
namespace attn {

constexpr int Q_TILE = 128;

namespace v2 {

constexpr int KB = 128;                       // keys per block
constexpr int NUM_THREADS2 = 256;             // two consumer warpgroups; thread 0 also drives TMA
constexpr int NUM_BARS = 1 + 2;
// causal launch order: heaviest query tiles first within groups of this many (batch, head) pairs, whose K / V (1 MB per pair
// at S = 2048, HD = 128) stay in L2 while the group's tiles run; one order over all pairs would stream every pair's K / V
// from HBM once per query tile
constexpr int CAUSAL_GROUP = 8;

// shared-memory layout of one head dim: a 128 x HD bf16 tile (Q tile, K block, V block) is HD / ATOM_COLS atoms of
// [128 rows][ATOM_COLS columns], each loaded by one TMA box
template <int HD>
struct Fwd {
    static_assert(HD == 32 || HD == 64 || HD == 128, "head_dim 32, 64 or 128");
    static constexpr int ATOM_COLS = HD < 64 ? HD : 64;
    static constexpr int ATOMS = HD / ATOM_COLS;
    static constexpr int ROW_BYTES = ATOM_COLS * 2;
    static constexpr int ATOM_BYTES = 128 * ROW_BYTES;
    static constexpr int TILE_BYTES = 128 * HD * 2;           // 8 / 16 / 32 KB
    static constexpr int OFF_Q2 = 0;
    static constexpr int OFF_K2 = OFF_Q2 + TILE_BYTES;        // 2 stages
    static constexpr int OFF_V2 = OFF_K2 + 2 * TILE_BYTES;    // 2 stages
    static constexpr int OFF_BAR2 = OFF_V2 + 2 * TILE_BYTES;
    static constexpr int SMEM_TOTAL2 = OFF_BAR2 + NUM_BARS * 8 + 16 + 1024;
};

// DROP: attention dropout (dropout.cuh, site 0).  The kept bf16 probabilities feed O += P V; the row sum l (and so the LSE)
// keeps summing ALL of them, and 1 / (1 - p) is folded into the final 1 / l.
// MASK without DROP at HD <= 64 is held to 128 registers, as the unmasked kernel is: two CTAs per SM (129 would allow one)
// CAUSAL without DROP at HD <= 64 is held to 128 registers for the same reason
template <int HD, bool DROP, bool MASK, bool CAUSAL>
__global__ void __launch_bounds__(NUM_THREADS2, (MASK || CAUSAL) && !DROP && HD <= 64 ? 2 : 1)
attention_fwd_v2_kernel(const __grid_constant__ CUtensorMap tm_qkv, bf16* __restrict__ out, float* __restrict__ lse2,
                        int d_model, int num_heads, int seq_len, float scale_log2e, unsigned long long seed, uint32_t thr,
                        float rescale, const uint32_t* __restrict__ key_mask) {
    using C = Fwd<HD>;
    constexpr int TILE_BYTES = C::TILE_BYTES, OFF_Q2 = C::OFF_Q2, OFF_K2 = C::OFF_K2, OFF_V2 = C::OFF_V2;
    constexpr int KSTEPS_PER_ATOM = C::ATOM_COLS / 16;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint64_t* bars = reinterpret_cast<uint64_t*>(smem + C::OFF_BAR2);
    uint64_t* bar_q = bars;
    uint64_t* kv_full = bars + 1;   // [2]

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, wg = warp >> 2;
    static_assert(!(MASK && CAUSAL), "causal attention takes no key padding mask");
    const int num_kb = (seq_len + KB - 1) / KB;   // key blocks = query tiles per sequence
    // CAUSAL: groups of CAUSAL_GROUP (batch, head) pairs, each group's last query tiles first; g0 = the group's first pair,
    // gs its size
    const int nbh = CAUSAL ? gridDim.x / num_kb : 0;
    const int g0 = CAUSAL ? blockIdx.x / (CAUSAL_GROUP * num_kb) * CAUSAL_GROUP : 0;
    const int gs = CAUSAL ? min(CAUSAL_GROUP, nbh - g0) : 1;
    const int r = CAUSAL ? blockIdx.x - g0 * num_kb : 0;
    const int qt = CAUSAL ? num_kb - 1 - r / gs : blockIdx.x % num_kb;
    const unsigned bh = CAUSAL ? g0 + r % gs : blockIdx.x / num_kb;
    const int head = bh % num_heads;
    const int batch = bh / num_heads;
    const int end_kb = CAUSAL ? qt + 1 : num_kb;   // key blocks 0 .. end_kb - 1 (CAUSAL: up to the diagonal block qt)

    // one 128-row tile of HD columns starting at column c0: one TMA box per atom
    auto load_tile = [&](uint8_t* dst, uint64_t* bar, int c0, int row) {
        tma_load_3d(dst, &tm_qkv, bar, c0, row, batch);
        if constexpr (C::ATOMS == 2) tma_load_3d(dst + C::ATOM_BYTES, &tm_qkv, bar, c0 + 64, row, batch);
    };
    // this sequence's mask words; valid-key bits of block j: words 4j .. 4j + 3 (0 past the last word)
    const int mask_words = (seq_len + 31) / 32;
    const uint32_t* kmask = MASK ? key_mask + static_cast<long long>(batch) * mask_words : nullptr;
    auto block_words = [&](int j, uint32_t (&w)[KB / 32]) {
#pragma unroll
        for (int i = 0; i < KB / 32; ++i) w[i] = j * (KB / 32) + i < mask_words ? __ldg(kmask + j * (KB / 32) + i) : 0u;
    };
    auto next_block = [&](int j) {   // first key block >= j holding a valid key, or num_kb
        if constexpr (MASK) {
            for (; j < num_kb; ++j) {
                uint32_t w[KB / 32];
                block_words(j, w);
                if (w[0] | w[1] | w[2] | w[3]) break;
            }
        }
        return j;
    };
    auto load_kv = [&](int st, int j) {   // thread 0 only; stage st must be free
        mbar_arrive_expect_tx(&kv_full[st], 2 * TILE_BYTES);
        load_tile(smem + OFF_K2 + st * TILE_BYTES, &kv_full[st], d_model + head * HD, j * KB);
        load_tile(smem + OFF_V2 + st * TILE_BYTES, &kv_full[st], 2 * d_model + head * HD, j * KB);
    };
    if (tid == 0) {
        tma_prefetch_desc(&tm_qkv);
        mbar_init(bar_q, 1);
        mbar_init(&kv_full[0], 1);
        mbar_init(&kv_full[1], 1);
        fence_mbar_init();
        mbar_arrive_expect_tx(bar_q, TILE_BYTES);
        load_tile(smem + OFF_Q2, bar_q, head * HD, qt * Q_TILE);
        if constexpr (!MASK) {
            load_kv(0, 0);
            if (end_kb > 1) load_kv(1, 1);
        }
    }
    // j: the key block being processed, n: how many blocks were processed before it (its stage and phase); without MASK
    // j = n.  j1 (MASK): the next block holding a valid key, already loaded into the other stage when < num_kb
    int j = 0, j1 = 0;
    if constexpr (MASK) {
        j = next_block(0);
        j1 = next_block(j + 1);
        if (tid == 0) {
            if (j < num_kb) load_kv(0, j);
            if (j1 < num_kb) load_kv(1, j1);
        }
    }
    __syncthreads();

    const uint32_t sq = smem_u32(smem + OFF_Q2) + wg * (64 * C::ROW_BYTES);   // this warpgroup's 64 query rows
    float o[HD / 2];
#pragma unroll
    for (int i = 0; i < HD / 2; ++i) o[i] = 0.f;
    // m = running row maximum (raw score units), l = this thread's share of the row sum (reduced over the quad at the end)
    float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};
    mbar_wait(bar_q, 0);
#pragma unroll 1
    for (int n = 0; j < end_kb; ++n) {
        const int st = (MASK ? n : j) & 1;
        // MASK: bit 2 jj + i of kbits = key 8 jj + 2 (lane & 3) + i of block j is valid, i.e. bits 2c, 2c + 1 of every byte of
        // the block's words, c = lane & 3; j2 = the block after j1, looked up before the MMAs so that its loads overlap them
        uint32_t kbits = ~0u;
        int j2 = 0;
        if constexpr (MASK) {
            uint32_t kw[KB / 32];
            block_words(j, kw);
            kbits = 0u;
#pragma unroll
            for (int w = 0; w < KB / 32; ++w) {
                uint32_t x = (kw[w] >> (2 * (lane & 3))) & 0x03030303u;
                x = (x | x >> 6) & 0x000F000Fu;
                kbits |= ((x | x >> 12) & 0xFFu) << (8 * w);
            }
            j2 = next_block(j1 + 1);
        }
        mbar_wait(&kv_full[st], ((MASK ? n : j) >> 1) & 1);
        const uint32_t sk = smem_u32(smem + OFF_K2 + st * TILE_BYTES), sv = smem_u32(smem + OFF_V2 + st * TILE_BYTES);
        float s[KB / 2];
        wgmma_fence();
#pragma unroll
        for (int ks = 0; ks < HD / 16; ++ks) {   // k16 step ks: atom ks / KSTEPS_PER_ATOM, 32 B into its swizzle row
            const uint32_t koff = (ks / KSTEPS_PER_ATOM) * C::ATOM_BYTES + (ks % KSTEPS_PER_ATOM) * 32;
            wgmma_bf16_n128<0, 0>(s, make_smem_desc_cols<C::ATOM_COLS>(sq + koff, 0),
                                  make_smem_desc_cols<C::ATOM_COLS>(sk + koff, 0), ks > 0 ? 1u : 0u);
        }
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
        if constexpr (MASK) {   // masked keys and keys >= S (clear bits): s[4 jj + 2 h + i] is key 8 jj + 2 (lane & 3) + i
            if (kbits != ~0u) {
#pragma unroll
                for (int jj = 0; jj < KB / 8; ++jj)
#pragma unroll
                    for (int i = 0; i < 2; ++i)
                        if (!((kbits >> (2 * jj + i)) & 1u)) s[4 * jj + i] = s[4 * jj + 2 + i] = -INFINITY;
            }
        } else if constexpr (CAUSAL) {
            if (j == qt) {   // diagonal block: s[4 jj + 2 h + i] is key 8 jj + 2 (lane & 3) + i of row r + 8 h, masked iff
                             // key > row, i.e. 8 (jj - h) + i > t = r - 2 (lane & 3)
                const int t = wg * 64 + (warp & 3) * 16 + (lane >> 2) - 2 * (lane & 3);
#pragma unroll
                for (int jj = 0; jj < KB / 8; ++jj)
#pragma unroll
                    for (int i = 0; i < 2; ++i) {
                        if (8 * jj + i > t) s[4 * jj + i] = -INFINITY;
                        if (8 * jj - 8 + i > t) s[4 * jj + 2 + i] = -INFINITY;
                    }
            }
        } else if (j * KB + KB > seq_len) {   // last block of a partial sequence: s[4 jj + 2 h + i] is key 8 jj + 2 (lane & 3) + i
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
            for (int jj = 0; jj < HD / 8; ++jj) {
                o[4 * jj + 2 * h] *= alpha;
                o[4 * jj + 2 * h + 1] *= alpha;
            }
        }
        wgmma_fence();
#pragma unroll
        for (int kc = 0; kc < KB / 16; ++kc)   // V block as an MN-major B operand: 16 keys = 16 rows per step, atoms ATOM_BYTES apart
            wgmma_bf16_rs<HD, 1>(o, pa[kc],
                                 make_smem_desc_cols<C::ATOM_COLS>(sv + kc * 16 * C::ROW_BYTES, C::ATOMS > 1 ? C::ATOM_BYTES : 0), 1u);
        wgmma_commit();
        wgmma_wait<0>();
        wgmma_fence_regs(o);
        if constexpr (!MASK) j2 = j + 2;
        if (j2 < end_kb) {
            named_bar_sync(1, NUM_THREADS2);   // both warpgroups are done with stage st
            if (tid == 0) load_kv((MASK ? n : j2) & 1, j2);
        }
        j = MASK ? j1 : j + 1;
        if constexpr (MASK) j1 = j2;
    }
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        float lt = l[h];
        lt += __shfl_xor_sync(0xffffffffu, lt, 1);
        lt += __shfl_xor_sync(0xffffffffu, lt, 2);
        // MASK: lt = 0 iff the sequence has no valid key (no block processed; otherwise the row maximum contributes 1)
        const float inv = MASK && lt == 0.f ? 0.f : DROP ? rescale / lt : 1.f / lt;
        const int q = qt * Q_TILE + wg * 64 + (warp & 3) * 16 + (lane >> 2) + 8 * h;
        if (q >= seq_len) continue;
        const long long token = static_cast<long long>(batch) * seq_len + q;
        if (lse2 && (lane & 3) == 0)
            lse2[token * num_heads + head] = MASK && lt == 0.f ? INFINITY : m[h] * scale_log2e + log2f(lt);
        bf16* op = out + token * d_model + head * HD + 2 * (lane & 3);
#pragma unroll
        for (int jj = 0; jj < HD / 8; ++jj)
            *reinterpret_cast<uint32_t*>(op + 8 * jj) = pack_bf16x2(o[4 * jj + 2 * h] * inv, o[4 * jj + 2 * h + 1] * inv);
    }
}

template <int HD, bool CAUSAL>
int launch_fwd(const void* qkv, void* out, float* lse2, long long batch, int seq_len, int num_heads, int d_model,
               unsigned long long seed, int drop_thr, float rescale, cudaStream_t st, const uint32_t* key_mask) {
    using C = Fwd<HD>;
    CUtensorMap tm;
    {   // 3-D {columns, position in sequence, sequence}: a tile never crosses into the next sequence
        uint64_t dims[3] = {(uint64_t)3 * d_model, (uint64_t)seq_len, (uint64_t)batch};
        uint64_t str[2] = {(uint64_t)3 * d_model * 2, (uint64_t)seq_len * 3 * d_model * 2};
        uint32_t box[3] = {C::ATOM_COLS, 128, 1};
        int r = make_tmap(&tm, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, qkv, dims, str, box,
                          C::ATOM_COLS == 32 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_128B);
        if (r) return r;
    }
    decltype(&attention_fwd_v2_kernel<HD, false, false, CAUSAL>) kern;
    if constexpr (CAUSAL) {
        if (int e = set_max_dynamic_smem<attention_fwd_v2_kernel<HD, false, false, true>>(C::SMEM_TOTAL2)) return e;
        if (int e = set_max_dynamic_smem<attention_fwd_v2_kernel<HD, true, false, true>>(C::SMEM_TOTAL2)) return e;
        kern = drop_thr < 0 ? attention_fwd_v2_kernel<HD, false, false, true> : attention_fwd_v2_kernel<HD, true, false, true>;
    } else {
        if (int e = set_max_dynamic_smem<attention_fwd_v2_kernel<HD, false, false, false>>(C::SMEM_TOTAL2)) return e;
        if (int e = set_max_dynamic_smem<attention_fwd_v2_kernel<HD, true, false, false>>(C::SMEM_TOTAL2)) return e;
        if (int e = set_max_dynamic_smem<attention_fwd_v2_kernel<HD, false, true, false>>(C::SMEM_TOTAL2)) return e;
        if (int e = set_max_dynamic_smem<attention_fwd_v2_kernel<HD, true, true, false>>(C::SMEM_TOTAL2)) return e;
        kern = key_mask ? (drop_thr < 0 ? attention_fwd_v2_kernel<HD, false, true, false> : attention_fwd_v2_kernel<HD, true, true, false>)
                        : (drop_thr < 0 ? attention_fwd_v2_kernel<HD, false, false, false> : attention_fwd_v2_kernel<HD, true, false, false>);
    }
    const float scale_log2e = 1.4426950408889634f / sqrtf((float)HD);
    const long long ctas = batch * num_heads * ((seq_len + Q_TILE - 1) / Q_TILE);
    if (ctas > 0x7fffffffll) return -2;
    kern<<<(unsigned)ctas, NUM_THREADS2, C::SMEM_TOTAL2, st>>>(
        tm, (bf16*)out, lse2, d_model, num_heads, seq_len, scale_log2e, seed, static_cast<uint32_t>(drop_thr < 0 ? 0 : drop_thr),
        rescale, key_mask);
    return -(int)cudaGetLastError();
}

// shape checks and head-dim dispatch of both entry points
template <bool CAUSAL>
int attention_fwd(const void* qkv, void* out, float* lse2, long long tokens, int seq_len, int num_heads, int d_model,
                  unsigned long long seed, int drop_thr, float rescale, cudaStream_t st, const uint32_t* key_mask) {
    if (num_heads < 1 || d_model % num_heads || drop_thr > 65535) return -2;
    const int hd = d_model / num_heads;
    if (hd != 32 && hd != 64 && hd != 128) return -2;
    if (seq_len < 1 || seq_len > drop::MAX_SEQ || tokens < 0 || tokens % seq_len) return -2;
    const long long batch = tokens / seq_len;
    if (batch == 0) return 0;
    if (hd == 32) return launch_fwd<32, CAUSAL>(qkv, out, lse2, batch, seq_len, num_heads, d_model, seed, drop_thr, rescale, st, key_mask);
    if (hd == 64) return launch_fwd<64, CAUSAL>(qkv, out, lse2, batch, seq_len, num_heads, d_model, seed, drop_thr, rescale, st, key_mask);
    return launch_fwd<128, CAUSAL>(qkv, out, lse2, batch, seq_len, num_heads, d_model, seed, drop_thr, rescale, st, key_mask);
}

}  // namespace v2

// words [batch, ceil(S / 32)]: bit k % 32 of word k / 32 = !pad[b, k] (key k valid), clear for k >= S; one thread per word
__global__ void __launch_bounds__(256) attention_pack_key_mask_kernel(const uint8_t* __restrict__ pad, uint32_t* __restrict__ words,
                                                                      long long batch, int seq_len) {
    const int per_seq = (seq_len + 31) / 32;
    const long long w = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (w >= batch * per_seq) return;
    const long long b = w / per_seq;
    const int k0 = static_cast<int>(w - b * per_seq) * 32;
    const uint8_t* row = pad + b * seq_len;
    uint32_t bits = 0u;
    for (int i = 0; i < 32 && k0 + i < seq_len; ++i) bits |= static_cast<uint32_t>(row[k0 + i] == 0) << i;
    words[w] = bits;
}

}  // namespace attn
}  // namespace lah

using namespace lah;
using namespace lah::attn;

extern "C" {

// qkv: [tokens, 3*d_model] bf16, tokens = batch * seq_len, 1 <= seq_len <= MAX_SEQ; out: [tokens, d_model] bf16;
// lse2: [tokens, heads] fp32 or NULL.  Returns -2 for a head dim d_model / num_heads other than 32, 64 or 128 (or heads that
// do not divide d_model), a sequence length out of range or one that does not divide tokens.
// drop_thr < 0: no dropout; otherwise attention dropout with threshold drop_thr (dropout.cuh), seed, rescale = 1 / (1 - p)
// key_mask: [batch, ceil(seq_len / 32)] uint32 key padding mask from lah_pack_key_mask, NULL for none.  A sequence without a
// valid key gets out = 0 and lse2 = +inf.
int lah_attention_fwd(const void* qkv, void* out, float* lse2, long long tokens, int seq_len, int num_heads, int d_model,
                      unsigned long long seed, int drop_thr, float rescale, cudaStream_t st, const uint32_t* key_mask) {
    return v2::attention_fwd<false>(qkv, out, lse2, tokens, seq_len, num_heads, d_model, seed, drop_thr, rescale, st, key_mask);
}

// causal self-attention (query q attends to keys <= q): the arguments and return codes of lah_attention_fwd without a key
// padding mask
int lah_attention_fwd_causal(const void* qkv, void* out, float* lse2, long long tokens, int seq_len, int num_heads, int d_model,
                             unsigned long long seed, int drop_thr, float rescale, cudaStream_t st) {
    return v2::attention_fwd<true>(qkv, out, lse2, tokens, seq_len, num_heads, d_model, seed, drop_thr, rescale, st, nullptr);
}

// pad: [batch, seq_len] bool (torch's src_key_padding_mask, true = ignored key) -> words [batch, ceil(seq_len / 32)] uint32
// of valid-key bits.  Returns -2 for a sequence length out of range.
int lah_pack_key_mask(const void* pad, void* words, long long batch, int seq_len, cudaStream_t st) {
    if (seq_len < 1 || seq_len > drop::MAX_SEQ || batch < 0) return -2;
    const long long n = batch * ((seq_len + 31) / 32);
    if (n == 0) return 0;
    attention_pack_key_mask_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>((const uint8_t*)pad, (uint32_t*)words, batch, seq_len);
    return -(int)cudaGetLastError();
}

}  // extern "C"
