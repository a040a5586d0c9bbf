// attention_bwd.cu — wgmma self-attention BACKWARD for the transformer expert (head_dim HD = 32, 64 or 128, any sequence
// length S in 1..MAX_SEQ).
// The reference's transformer expert cannot be trained at all (in-place transpose of a leaf, SURVEY.md §0.3); this kernel is
// what makes the sm_90a transformer expert trainable without falling back to eager PyTorch.
//
// One CTA = one (batch, head, 128-key block j); consumer warpgroup w owns keys [64w, 64w + 64) of the block.  K_j / V_j stay
// in shared memory; the ceil(S / QB) query blocks i of QB queries stream through a 2-stage TMA pipeline (Q_i and dO_i).  Per
// query block, all on tensor cores with accumulators in registers (transposed problem: keys are the MMA rows):
//
//     S^T = K_j Q_i^T               (64 x QB per warpgroup)      dP^T = V_j dO_i^T            (64 x QB)
//     P^T = exp2(S^T * scale*log2e - LSE_i)   [recomputed from the forward's row log-sum-exp: no second softmax pass]
//     dS^T = P^T o (dP^T - Delta_i) * scale   [Delta = rowsum(dO o O)]
//     dV_j += P^T dO_i   (64 x HD)   dK_j += dS^T Q_i  (64 x HD)   dQ_i^(j) = dS K_j  (QB x HD, one partial per key block j)
//
// P^T and dS^T are fed to dV / dK straight from registers (the accumulator layout IS the wgmma A fragment layout); dS^T is
// also stored once to shared memory (bf16, 128B-swizzled [key rows][64 queries] atoms), where it is the MN-major A operand
// of dQ.  Q_i, dO_i, K_j are consumed both K-major (S, dP) and MN-major (dV, dK, dQ) straight from their TMA tiles.
// Nothing of size S x S touches HBM.  Thread 0 also drives TMA.
//
// Head dim (template parameter HD; the entry point dispatches on D / heads).  Tiles are stored as atoms of 64 columns
// (128B swizzle) or, at HD = 32, of 32 columns (64B swizzle; the head is never padded into the next one).
//   HD = 32, 64: QB = 128.  Per thread S^T, dP^T 64 accumulators each, dV, dK HD / 2 each; warpgroup w computes dQ of
//     queries [64w, 64w + 64).  Shared memory K, V + 2 x (Q, dO) + dS^T (2 atoms): 81 / 129 KB.
//   HD = 128: QB = 64, so S^T and dP^T take 32 registers each beside the 64 + 64 of dV and dK (128 queries would need 256).
//     K_j / V_j are two 64-column atoms each; every operand spanning the head dim is two atoms (LBO = one atom).  dS^T is
//     one atom, and warpgroup w computes dQ of all 64 queries for head columns [64w, 64w + 64).  Shared memory 145 KB.
//   TMA boxes are {atom columns, QB rows}; at HD = 128 the 128 key rows of K_j / V_j take two boxes per atom.
//
// DROP (attention dropout, dropout.cuh site 0): the keep mask M is regenerated from the seed, never stored.  With
// Pd = M o P / (1 - p):  dV += Pd^T dO,  dS = P o (M o dP / (1 - p) - Delta) * scale, Delta = rowsum(dO o O) of the DROPPED
// output O (attn_delta_kernel, unchanged); LSE is that of the undropped softmax.  P^T is masked but not scaled in the dV
// MMA; 1 / (1 - p) is applied to dV once at the end.  The granules are addressed by absolute query / key position, so the
// mask is that of the forward at every QB.
//
// Sequence length: the tensor maps are 3-D {columns, S, batch}, so rows past the end of a sequence arrive as zeros.  Zeros
// alone do not make P vanish (exp2(0 - LSE) is not 0, and a garbage LSE can make it inf, and inf * 0 is NaN), so in a
// partial block P^T and dS^T are forced to exactly 0: queries >= S get LSE = +inf and Delta = 0 (LSE and Delta are only
// read for valid queries), keys >= S get S^T = -inf.  No dK / dV row is stored for keys >= S and no dQ-partial row for
// queries >= S.  Full blocks run exactly the arithmetic of the 512-token kernel.
//
// Key padding mask (MASK instantiations; format of attention.cu, bits of keys >= S clear): a CTA whose 128 keys hold no
// valid key does no MMA and loads nothing; it writes exact zeros to its dK / dV rows and a zero dQ partial (slice j), so
// attn_dq_reduce_kernel stays mask-blind.  In a partially valid block S^T of masked keys is set to -inf, as for keys >= S,
// so P^T and dS^T are exactly 0 and so are those dK / dV rows.  A sequence without a valid key has LSE = +inf.
//
// Causal attention (CAUSAL instantiations, never with MASK): key block j walks only the query blocks that hold a query
// >= 128 j, i.e. i >= 128 j / QB (at HD = 128 both 64-query halves of the diagonal, of which the first straddles it).  In
// a query block that starts inside the key block, S^T of keys > query is set to -inf, so P^T and dS^T are exactly 0 there;
// that also covers keys >= S for every valid query.  dQ partial j then holds only queries >= 128 j:
// attn_dq_reduce_kernel<true> sums, for query q, the partials j <= q / 128 in the same order, and the rows of partial j
// below 128 j are neither written nor read.  CTAs are launched heaviest first: blockIdx.x / (batch * heads) is j, and key
// block 0 walks every query block.
#include "sm90.cuh"
#include "dropout.cuh"

namespace lah {
namespace attnb {

constexpr int BLK = 128;                       // keys per CTA (key block); dq_part has one slice per key block
constexpr int NUM_THREADS = 256;
constexpr int ATOM = BLK * 128;                // 16 KB: one [128 key rows][64 queries] atom of dS^T
constexpr int NUM_BARS = 1 + 2;

template <int HD>
struct Bwd {
    static_assert(HD == 32 || HD == 64 || HD == 128, "head_dim 32, 64 or 128");
    static constexpr int QB = HD == 128 ? 64 : 128;              // queries per block
    static constexpr int ATOM_COLS = HD < 64 ? HD : 64;
    static constexpr int ATOMS = HD / ATOM_COLS;
    static constexpr int ROW_BYTES = ATOM_COLS * 2;
    static constexpr int KV_ATOM = BLK * ROW_BYTES;             // [128 key rows][ATOM_COLS]
    static constexpr int Q_ATOM = QB * ROW_BYTES;               // [QB query rows][ATOM_COLS]
    static constexpr int KV_TILE = BLK * HD * 2;                // 8 / 16 / 32 KB
    static constexpr int Q_TILE = QB * HD * 2;                  // 8 / 16 / 16 KB
    static constexpr int DQ_N = HD == 128 ? 64 : HD;            // dQ columns per warpgroup
    static constexpr int OFF_K = 0;
    static constexpr int OFF_V = OFF_K + KV_TILE;
    static constexpr int OFF_Q = OFF_V + KV_TILE;               // 2 stages
    static constexpr int OFF_DO = OFF_Q + 2 * Q_TILE;           // 2 stages
    static constexpr int OFF_DS = OFF_DO + 2 * Q_TILE;          // dS^T: QB / 64 atoms (queries 0-63, 64-127)
    static constexpr int OFF_LSE = OFF_DS + (QB / 64) * ATOM;   // lse2 / delta of the current query block: 2 x QB fp32
    static constexpr int OFF_BAR = OFF_LSE + 2 * QB * 4;
    static constexpr int SMEM_TOTAL = OFF_BAR + NUM_BARS * 8 + 16 + 1024;
};

template <int HD, bool DROP, bool MASK, bool CAUSAL>
__global__ void __launch_bounds__(NUM_THREADS, 1)
attention_bwd_kernel(const __grid_constant__ CUtensorMap tm_qkv, const __grid_constant__ CUtensorMap tm_do,
                     const float* __restrict__ lse2, const float* __restrict__ delta, bf16* __restrict__ dqkv,
                     bf16* __restrict__ dq_part, long long total_tokens, int d_model, int num_heads, int seq_len, float scale,
                     float scale_log2e, unsigned long long seed, uint32_t thr, float rescale,
                     const uint32_t* __restrict__ key_mask) {
    using C = Bwd<HD>;
    constexpr int QB = C::QB, ACOLS = C::ATOM_COLS, ROW_BYTES = C::ROW_BYTES;
    constexpr int OFF_K = C::OFF_K, OFF_V = C::OFF_V, OFF_Q = C::OFF_Q, OFF_DO = C::OFF_DO, OFF_DS = C::OFF_DS;
    constexpr int KSTEPS_PER_ATOM = ACOLS / 16;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint64_t* bars = reinterpret_cast<uint64_t*>(smem + C::OFF_BAR);
    uint64_t* kv_full = bars;
    uint64_t* q_full = bars + 1;     // [2]
    float* s_lse = reinterpret_cast<float*>(smem + C::OFF_LSE);
    float* s_delta = s_lse + QB;

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, wg = warp >> 2;
    const int num_kb = (seq_len + BLK - 1) / BLK;   // key blocks per sequence
    const int num_qb = (seq_len + QB - 1) / QB;     // query blocks per sequence
    static_assert(!(MASK && CAUSAL), "causal attention takes no key padding mask");
    const int nbh = CAUSAL ? gridDim.x / num_kb : 0;   // CAUSAL: (batch, head) pairs; key block 0 comes first
    const int j = CAUSAL ? static_cast<int>(blockIdx.x / nbh) : blockIdx.x % num_kb;
    const unsigned bh = CAUSAL ? blockIdx.x % nbh : blockIdx.x / num_kb;
    const int head = bh % num_heads;
    const int batch = bh / num_heads;
    const int i0 = CAUSAL ? j * (BLK / QB) : 0;     // first query block; CAUSAL: the first holding a query >= 128 j
    const long long seq0 = static_cast<long long>(batch) * seq_len;
    const int key_row = wg * 64 + (warp & 3) * 16 + (lane >> 2);   // row of the block (+ 8 for h = 1)
    uint32_t kvalid = 3u;   // MASK: bit h set iff key key_row + 8 h of this block is valid
    if constexpr (MASK) {
        const int mask_words = (seq_len + 31) / 32;
        uint32_t w[BLK / 32];
#pragma unroll
        for (int i = 0; i < BLK / 32; ++i)
            w[i] = j * (BLK / 32) + i < mask_words ? __ldg(key_mask + batch * mask_words + j * (BLK / 32) + i) : 0u;
        if (!(w[0] | w[1] | w[2] | w[3])) {   // no valid key: zero dK_j / dV_j rows and dQ partial j, nothing else
            constexpr int V8 = HD / 8;   // 16 B vectors per head row
            const int keys = min(BLK, seq_len - j * BLK);
            for (int e = tid; e < 2 * keys * V8; e += NUM_THREADS) {
                const int t = e / (keys * V8), r = (e / V8) % keys, c = e % V8;
                *reinterpret_cast<int4*>(dqkv + (seq0 + j * BLK + r) * (3ll * d_model) + (1 + t) * d_model + head * HD + 8 * c) =
                    make_int4(0, 0, 0, 0);
            }
            for (int e = tid; e < seq_len * V8; e += NUM_THREADS)
                *reinterpret_cast<int4*>(dq_part + (static_cast<long long>(j) * total_tokens + seq0 + e / V8) * d_model +
                                         head * HD + 8 * (e % V8)) = make_int4(0, 0, 0, 0);
            return;
        }
        const unsigned long long lo = w[0] | static_cast<unsigned long long>(w[1]) << 32,   // keys 0-63, 64-127
                                 hi = w[2] | static_cast<unsigned long long>(w[3]) << 32;
        const unsigned long long mine = (key_row < 64 ? lo : hi) >> (key_row & 63);   // key_row and key_row + 8: same half
        kvalid = static_cast<uint32_t>(mine & 1u) | static_cast<uint32_t>((mine >> 8) & 1u) << 1;
    }

    auto load_q = [&](int i) {   // thread 0 only; stage (i - i0) & 1 must be free
        const int st = (i - i0) & 1;
        mbar_arrive_expect_tx(&q_full[st], 2 * C::Q_TILE);
        tma_load_3d(smem + OFF_Q + st * C::Q_TILE, &tm_qkv, &q_full[st], head * HD, i * QB, batch);
        tma_load_3d(smem + OFF_DO + st * C::Q_TILE, &tm_do, &q_full[st], head * HD, i * QB, batch);
        if constexpr (C::ATOMS == 2) {
            tma_load_3d(smem + OFF_Q + st * C::Q_TILE + C::Q_ATOM, &tm_qkv, &q_full[st], head * HD + 64, i * QB, batch);
            tma_load_3d(smem + OFF_DO + st * C::Q_TILE + C::Q_ATOM, &tm_do, &q_full[st], head * HD + 64, i * QB, batch);
        }
    };
    if (tid == 0) {
        tma_prefetch_desc(&tm_qkv);
        tma_prefetch_desc(&tm_do);
        mbar_init(kv_full, 1);
        mbar_init(&q_full[0], 1);
        mbar_init(&q_full[1], 1);
        fence_mbar_init();
        if constexpr (QB == BLK) {
            mbar_arrive_expect_tx(kv_full, 2 * C::KV_TILE);
            tma_load_3d(smem + OFF_K, &tm_qkv, kv_full, d_model + head * HD, j * BLK, batch);
            tma_load_3d(smem + OFF_V, &tm_qkv, kv_full, 2 * d_model + head * HD, j * BLK, batch);
        } else {   // HD = 128: box (atom a, row half r) of K_j / V_j; a half wholly past S is not loaded but zeroed below
            const int halves = j * BLK + QB < seq_len ? 2 : 1;
            mbar_arrive_expect_tx(kv_full, halves * C::KV_TILE);
#pragma unroll
            for (int a = 0; a < C::ATOMS; ++a)
                for (int r = 0; r < halves; ++r) {
                    const int off = a * C::KV_ATOM + r * QB * ROW_BYTES;
                    tma_load_3d(smem + OFF_K + off, &tm_qkv, kv_full, d_model + head * HD + a * 64, j * BLK + r * QB, batch);
                    tma_load_3d(smem + OFF_V + off, &tm_qkv, kv_full, 2 * d_model + head * HD + a * 64, j * BLK + r * QB, batch);
                }
        }
        load_q(i0);
        if (i0 + 1 < num_qb) load_q(i0 + 1);
    }
    if constexpr (QB != BLK) {
        // key rows [QB, 128) all >= S: zeros, as TMA would have filled them (garbage there could be inf / NaN in dP^T)
        if (j * BLK + QB >= seq_len) {
            constexpr int HALF = QB * ROW_BYTES / 16;   // int4 per (tile, atom) half
            for (int e = tid; e < 2 * C::ATOMS * HALF; e += NUM_THREADS) {
                const int t = e / (C::ATOMS * HALF), a = (e / HALF) % C::ATOMS, x = e % HALF;
                reinterpret_cast<int4*>(smem + (t ? OFF_V : OFF_K) + a * C::KV_ATOM + QB * ROW_BYTES)[x] = make_int4(0, 0, 0, 0);
            }
            fence_proxy_async_smem();   // generic-proxy zeros -> visible to the tensor core
        }
    }
    __syncthreads();

    const uint32_t sk = smem_u32(smem + OFF_K), sv = smem_u32(smem + OFF_V), sds = smem_u32(smem + OFF_DS);
    const int qcol = 2 * (lane & 3);                               // query column (+ 8 jj, + 1)
    float dv[HD / 2], dk[HD / 2];
#pragma unroll
    for (int e = 0; e < HD / 2; ++e) dv[e] = dk[e] = 0.f;
    mbar_wait(kv_full, 0);
#pragma unroll 1
    for (int i = i0; i < num_qb; ++i) {
        const int st = (i - i0) & 1;
        const long long tok0 = seq0 + i * QB;
        const int qr = tid & (QB - 1);   // query row of the block whose LSE (tid < QB) or Delta this thread loads
        const bool qvalid = i * QB + qr < seq_len;
        if (tid < QB) s_lse[qr] = qvalid ? __ldg(lse2 + (tok0 + qr) * num_heads + head) : INFINITY;
        else if (QB == BLK || tid < 2 * QB) s_delta[qr] = qvalid ? __ldg(delta + (tok0 + qr) * num_heads + head) : 0.f;
        mbar_wait(&q_full[st], ((i - i0) >> 1) & 1);
        const uint32_t sq = smem_u32(smem + OFF_Q + st * C::Q_TILE), sdo = smem_u32(smem + OFF_DO + st * C::Q_TILE);
        float sacc[QB / 2], dpacc[QB / 2];
        wgmma_fence();
#pragma unroll
        for (int ks = 0; ks < HD / 16; ++ks) {   // k16 step ks: atom ks / KSTEPS_PER_ATOM, 32 B into its swizzle row
            const uint32_t a = ks / KSTEPS_PER_ATOM, kb = (ks % KSTEPS_PER_ATOM) * 32;
            wgmma_bf16_ss<QB, 0, 0>(sacc, make_smem_desc_cols<ACOLS>(sk + a * C::KV_ATOM + wg * (64 * ROW_BYTES) + kb, 0),
                                    make_smem_desc_cols<ACOLS>(sq + a * C::Q_ATOM + kb, 0), ks > 0 ? 1u : 0u);
        }
#pragma unroll
        for (int ks = 0; ks < HD / 16; ++ks) {
            const uint32_t a = ks / KSTEPS_PER_ATOM, kb = (ks % KSTEPS_PER_ATOM) * 32;
            wgmma_bf16_ss<QB, 0, 0>(dpacc, make_smem_desc_cols<ACOLS>(sv + a * C::KV_ATOM + wg * (64 * ROW_BYTES) + kb, 0),
                                    make_smem_desc_cols<ACOLS>(sdo + a * C::Q_ATOM + kb, 0), ks > 0 ? 1u : 0u);
        }
        wgmma_commit();
        named_bar_sync(1, NUM_THREADS);   // lse / delta of this block are in shared memory
        wgmma_wait<0>();
        wgmma_fence_regs(sacc);
        wgmma_fence_regs(dpacc);
        if constexpr (MASK) {   // masked keys and keys >= S: sacc[4 jj + 2 h + par] is key key_row + 8 h
#pragma unroll
            for (int h = 0; h < 2; ++h)
                if (!((kvalid >> h) & 1u))
#pragma unroll
                    for (int jj = 0; jj < QB / 8; ++jj) sacc[4 * jj + 2 * h] = sacc[4 * jj + 2 * h + 1] = -INFINITY;
        } else if constexpr (CAUSAL) {
            if (i * QB < j * BLK + BLK) {   // the block meets the diagonal: sacc[4 jj + 2 h + par] is key j BLK + key_row + 8 h,
                                           // query i QB + 8 jj + qcol + par; masked iff 8 jj + par < t + 8 h
                const int t = j * BLK + key_row - i * QB - qcol;
#pragma unroll
                for (int jj = 0; jj < QB / 8; ++jj)
#pragma unroll
                    for (int h = 0; h < 2; ++h)
#pragma unroll
                        for (int par = 0; par < 2; ++par)
                            if (8 * jj + par < t + 8 * h) sacc[4 * jj + 2 * h + par] = -INFINITY;
            }
        } else if (j * BLK + BLK > seq_len) {   // last key block of a partial sequence: sacc[4 jj + 2 h + par] is key key_row + 8 h
#pragma unroll
            for (int h = 0; h < 2; ++h)
                if (j * BLK + key_row + 8 * h >= seq_len)
#pragma unroll
                    for (int jj = 0; jj < QB / 8; ++jj) sacc[4 * jj + 2 * h] = sacc[4 * jj + 2 * h + 1] = -INFINITY;
        }
        const uint32_t kk = j * BLK + key_row;   // this thread's keys: kk, kk + 8
        uint32_t km = 0u;
        uint32_t pa[QB / 16][4], da[QB / 16][4];
#pragma unroll
        for (int jj = 0; jj < QB / 8; ++jj) {
            if constexpr (DROP) {
                // keep bits of the 16-query chunk jp = jj / 2, bit 4 jl + 2h + par <-> sacc[4 (2jp + jl) + 2h + par]
                // (keys kk + 8h x queries 16jp + qcol + 8jl + par): the granules of query parity 0 / 1 each hold 4 of them
                if ((jj & 1) == 0) {
                    km = 0u;
#pragma unroll
                    for (int par = 0; par < 2; ++par) {
                        const uint4 bits = drop::attn_bits(seed, batch, head, ((QB / 16) * i + (jj >> 1)) * 4 + (lane & 3),
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
        // dV += P^T dO, dK += dS^T Q: reduction over the QB queries of the block, B operands MN-major (16 rows per step,
        // head-dim atoms Q_ATOM apart)
        constexpr uint32_t LBO_Q = C::ATOMS > 1 ? C::Q_ATOM : 0;
        wgmma_fence();
#pragma unroll
        for (int kc = 0; kc < QB / 16; ++kc)
            wgmma_bf16_rs<HD, 1>(dv, pa[kc], make_smem_desc_cols<ACOLS>(sdo + kc * 16 * ROW_BYTES, LBO_Q), 1u);
#pragma unroll
        for (int kc = 0; kc < QB / 16; ++kc)
            wgmma_bf16_rs<HD, 1>(dk, da[kc], make_smem_desc_cols<ACOLS>(sq + kc * 16 * ROW_BYTES, LBO_Q), 1u);
        wgmma_commit();
        fence_proxy_async_smem();          // generic-proxy smem writes (dS^T) -> visible to the tensor core
        named_bar_sync(1, NUM_THREADS);    // dS^T of both warpgroups is in shared memory
        // dQ = dS K_j: A = dS^T (MN-major), B = K_j (MN-major), 8 steps of 16 keys.  QB = 128: this warpgroup's 64 queries
        // (dS^T atom wg), all HD columns; QB = 64: all 64 queries, head columns [64 wg, 64 wg + 64) (K_j atom wg)
        constexpr int DQ_N = C::DQ_N;
        const uint32_t sds_w = QB == BLK ? sds + wg * ATOM : sds;
        const uint32_t sk_w = HD == 128 ? sk + wg * C::KV_ATOM : sk;
        float dq[DQ_N / 2];
        wgmma_fence();
#pragma unroll
        for (int kc = 0; kc < BLK / 16; ++kc)
            wgmma_bf16_ss<DQ_N, 1, 1>(dq, make_smem_desc_sw128(sds_w + kc * 2048, ATOM, 1024),
                                      make_smem_desc_cols<ACOLS>(sk_w + kc * 16 * ROW_BYTES, 0), kc > 0 ? 1u : 0u);
        wgmma_commit();
        wgmma_wait<0>();
        wgmma_fence_regs(dq);
        wgmma_fence_regs(dv);
        wgmma_fence_regs(dk);
        // partial dQ of THIS key block into slice j of dq_part ([ceil(S / 128), T, D] bf16; attn_dq_reduce_kernel sums the
        // slices in fp32) — no atomics, half the bytes of fp32 partials
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int q = (QB == BLK ? wg * 64 : 0) + (warp & 3) * 16 + (lane >> 2) + 8 * h;
            if (i * QB + q >= seq_len) continue;
            const long long token = tok0 + q;
            bf16* dqp = dq_part + (static_cast<long long>(j) * total_tokens + token) * d_model + head * HD +
                        (HD == 128 ? wg * 64 : 0) + qcol;
#pragma unroll
            for (int jj = 0; jj < DQ_N / 8; ++jj)
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
        bf16* dkp = dqkv + key * (3ll * d_model) + d_model + head * HD + qcol;
        bf16* dvp = dqkv + key * (3ll * d_model) + 2 * d_model + head * HD + qcol;
#pragma unroll
        for (int jj = 0; jj < HD / 8; ++jj) {
            *reinterpret_cast<uint32_t*>(dkp + 8 * jj) = pack_bf16x2(dk[4 * jj + 2 * h], dk[4 * jj + 2 * h + 1]);
            if constexpr (DROP)
                *reinterpret_cast<uint32_t*>(dvp + 8 * jj) = pack_bf16x2(dv[4 * jj + 2 * h] * rescale, dv[4 * jj + 2 * h + 1] * rescale);
            else
                *reinterpret_cast<uint32_t*>(dvp + 8 * jj) = pack_bf16x2(dv[4 * jj + 2 * h], dv[4 * jj + 2 * h + 1]);
        }
    }
}

// prologue: delta[t, h] = sum_d dO[t, h, d] * O[t, h, d]  (one warp per (token, head); per lane one bf16 at HD = 32, else
// HD / 64 bf16 pairs, each pass of the warp reading one 128 B row segment)
template <int HD>
__global__ void __launch_bounds__(256) attn_delta_kernel(const bf16* __restrict__ dout, const bf16* __restrict__ out,
                                                         float* __restrict__ delta, long long pairs) {
    const long long w = (static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (w >= pairs) return;
    float acc;
    if constexpr (HD == 32) {
        acc = __bfloat162float(dout[w * HD + lane]) * __bfloat162float(out[w * HD + lane]);
    } else {
        const __nv_bfloat162 a = reinterpret_cast<const __nv_bfloat162*>(dout + w * HD)[lane];
        const __nv_bfloat162 b = reinterpret_cast<const __nv_bfloat162*>(out + w * HD)[lane];
        acc = __bfloat162float(a.x) * __bfloat162float(b.x) + __bfloat162float(a.y) * __bfloat162float(b.y);
#pragma unroll
        for (int c = 1; c < HD / 64; ++c) {
            const __nv_bfloat162 a2 = reinterpret_cast<const __nv_bfloat162*>(dout + w * HD)[32 * c + lane];
            const __nv_bfloat162 b2 = reinterpret_cast<const __nv_bfloat162*>(out + w * HD)[32 * c + lane];
            acc += __bfloat162float(a2.x) * __bfloat162float(b2.x) + __bfloat162float(a2.y) * __bfloat162float(b2.y);
        }
    }
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, d);
    if (lane == 0) delta[w] = acc;
}

// epilogue: dQ = sum of the per-key-block partials in key-block order (deterministic), written as bf16 into the Q third of dqkv.
// CAUSAL: query q of its sequence sums partials 0 .. q / BLK only (the key blocks that hold a key <= q)
template <bool CAUSAL>
__global__ void __launch_bounds__(256) attn_dq_reduce_kernel(const bf16* __restrict__ dq_part, bf16* __restrict__ dqkv,
                                                             long long tokens, int d_model, int parts, int seq_len) {
    const long long i8 = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;   // 8-element (16 B) index inside [T, D]
    const long long n8 = tokens * d_model / 8;
    if (i8 >= n8) return;
    if constexpr (CAUSAL) parts = static_cast<int>((i8 * 8 / d_model) % seq_len) / BLK + 1;
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

template <int HD, bool CAUSAL>
int launch_bwd(const void* qkv, const void* out, const void* dout, const float* lse2, float* delta, void* dqkv, void* dq_part,
               long long tokens, long long batch, int seq_len, int num_heads, int d_model, unsigned long long seed,
               int drop_thr, float rescale, cudaStream_t st, const uint32_t* key_mask) {
    using C = Bwd<HD>;
    CUtensorMap tm_qkv, tm_do;
    const uint32_t box[3] = {C::ATOM_COLS, C::QB, 1};
    const CUtensorMapSwizzle swz = C::ATOM_COLS == 32 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_128B;
    {   // 3-D {columns, position in sequence, sequence}: a tile never crosses into the next sequence
        uint64_t dims[3] = {(uint64_t)3 * d_model, (uint64_t)seq_len, (uint64_t)batch};
        uint64_t str[2] = {(uint64_t)3 * d_model * 2, (uint64_t)seq_len * 3 * d_model * 2};
        int r = make_tmap(&tm_qkv, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, qkv, dims, str, box, swz);
        if (r) return r;
    }
    {
        uint64_t dims[3] = {(uint64_t)d_model, (uint64_t)seq_len, (uint64_t)batch};
        uint64_t str[2] = {(uint64_t)d_model * 2, (uint64_t)seq_len * d_model * 2};
        int r = make_tmap(&tm_do, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, dout, dims, str, box, swz);
        if (r) return r;
    }
    decltype(&attention_bwd_kernel<HD, false, false, CAUSAL>) kern;
    if constexpr (CAUSAL) {
        if (int e = set_max_dynamic_smem<attention_bwd_kernel<HD, false, false, true>>(C::SMEM_TOTAL)) return e;
        if (int e = set_max_dynamic_smem<attention_bwd_kernel<HD, true, false, true>>(C::SMEM_TOTAL)) return e;
        kern = drop_thr < 0 ? attention_bwd_kernel<HD, false, false, true> : attention_bwd_kernel<HD, true, false, true>;
    } else {
        if (int e = set_max_dynamic_smem<attention_bwd_kernel<HD, false, false, false>>(C::SMEM_TOTAL)) return e;
        if (int e = set_max_dynamic_smem<attention_bwd_kernel<HD, true, false, false>>(C::SMEM_TOTAL)) return e;
        if (int e = set_max_dynamic_smem<attention_bwd_kernel<HD, false, true, false>>(C::SMEM_TOTAL)) return e;
        if (int e = set_max_dynamic_smem<attention_bwd_kernel<HD, true, true, false>>(C::SMEM_TOTAL)) return e;
        kern = key_mask ? (drop_thr < 0 ? attention_bwd_kernel<HD, false, true, false> : attention_bwd_kernel<HD, true, true, false>)
                        : (drop_thr < 0 ? attention_bwd_kernel<HD, false, false, false> : attention_bwd_kernel<HD, true, false, false>);
    }
    const float scale = 1.f / sqrtf((float)HD);
    const int blocks = (seq_len + BLK - 1) / BLK;
    const long long pairs = tokens * num_heads, ctas = batch * num_heads * blocks;
    if (ctas > 0x7fffffffll) return -2;
    attn_delta_kernel<HD><<<(unsigned)((pairs * 32 + 255) / 256), 256, 0, st>>>((const bf16*)dout, (const bf16*)out, delta, pairs);
    kern<<<(unsigned)ctas, NUM_THREADS, C::SMEM_TOTAL, st>>>(
        tm_qkv, tm_do, lse2, delta, (bf16*)dqkv, (bf16*)dq_part, tokens, d_model, num_heads, seq_len, scale,
        scale * 1.4426950408889634f, seed, static_cast<uint32_t>(drop_thr < 0 ? 0 : drop_thr), rescale, key_mask);
    attn_dq_reduce_kernel<CAUSAL><<<(unsigned)((tokens * d_model / 8 + 255) / 256), 256, 0, st>>>(
        (const bf16*)dq_part, (bf16*)dqkv, tokens, d_model, blocks, seq_len);
    return -(int)cudaGetLastError();
}

// shape checks and head-dim dispatch of both entry points
template <bool CAUSAL>
int attention_bwd(const void* qkv, const void* out, const void* dout, const float* lse2, float* delta, void* dqkv,
                  void* dq_part, long long tokens, int seq_len, int num_heads, int d_model, unsigned long long seed,
                  int drop_thr, float rescale, cudaStream_t st, const uint32_t* key_mask) {
    if (num_heads < 1 || d_model % num_heads || drop_thr > 65535) return -2;
    const int hd = d_model / num_heads;
    if (hd != 32 && hd != 64 && hd != 128) return -2;
    if (seq_len < 1 || seq_len > drop::MAX_SEQ || tokens < 0 || tokens % seq_len) return -2;
    const long long batch = tokens / seq_len;
    if (batch == 0) return 0;
    if (hd == 32)
        return launch_bwd<32, CAUSAL>(qkv, out, dout, lse2, delta, dqkv, dq_part, tokens, batch, seq_len, num_heads, d_model,
                                      seed, drop_thr, rescale, st, key_mask);
    if (hd == 64)
        return launch_bwd<64, CAUSAL>(qkv, out, dout, lse2, delta, dqkv, dq_part, tokens, batch, seq_len, num_heads, d_model,
                                      seed, drop_thr, rescale, st, key_mask);
    return launch_bwd<128, CAUSAL>(qkv, out, dout, lse2, delta, dqkv, dq_part, tokens, batch, seq_len, num_heads, d_model,
                                   seed, drop_thr, rescale, st, key_mask);
}

}  // namespace attnb
}  // namespace lah

using namespace lah;
using namespace lah::attnb;

extern "C" {

// qkv [T, 3D] bf16 (forward input), out [T, D] bf16 (forward output), dout [T, D] bf16, lse2 [T, H] fp32 (forward output)
// -> dqkv [T, 3D] bf16, T = batch * seq_len, 1 <= seq_len <= MAX_SEQ, head dim D / H in {32, 64, 128} (-2 otherwise, or
// when seq_len does not divide T or H does not divide D).
// Scratch: delta [T, H] fp32 (rowsum(dout o out), computed here), dq_part [ceil(seq_len / 128), T, D] bf16 (one partial
// of dQ per key block, reduced into the Q third of dqkv here).  Three launches, no PyTorch ops around them.
// drop_thr < 0: the forward ran without dropout; otherwise the same (seed, drop_thr, rescale) as lah_attention_fwd.
// key_mask: the key padding mask of lah_attention_fwd (NULL: no mask).
int lah_attention_bwd(const void* qkv, const void* out, const void* dout, const float* lse2, float* delta, void* dqkv,
                      void* dq_part, long long tokens, int seq_len, int num_heads, int d_model, unsigned long long seed,
                      int drop_thr, float rescale, cudaStream_t st, const uint32_t* key_mask) {
    return attention_bwd<false>(qkv, out, dout, lse2, delta, dqkv, dq_part, tokens, seq_len, num_heads, d_model, seed, drop_thr,
                                rescale, st, key_mask);
}

// backward of lah_attention_fwd_causal: the arguments and return codes of lah_attention_bwd without a key padding mask.
// Rows of dq_part's slice j below query 128 j are not written.
int lah_attention_bwd_causal(const void* qkv, const void* out, const void* dout, const float* lse2, float* delta, void* dqkv,
                             void* dq_part, long long tokens, int seq_len, int num_heads, int d_model, unsigned long long seed,
                             int drop_thr, float rescale, cudaStream_t st) {
    return attention_bwd<true>(qkv, out, dout, lse2, delta, dqkv, dq_part, tokens, seq_len, num_heads, d_model, seed, drop_thr,
                               rescale, st, nullptr);
}

}  // extern "C"
