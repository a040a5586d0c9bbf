// moe.cu — DMoE routing + expert all-to-all as peer-to-peer (NVLink/NVSwitch) kernels.
//
// What the reference does with Python threads, a Kademlia DHT and one blocking TCP RPC per (sample, expert)
// (/root/reference/lib/client/gating_function.py:25-153, lib/client/remote_expert.py:53-76,
//  lib/runtime/task_pool.py:141-172) is done here by five kernels operating on SYMMETRIC buffers (same offset on every
// GPU, every GPU's heap mapped into every peer):
//
//   gate_topk        product-key scores + liveness table + Bernoulli failure injection -> exact top-k, softmax over the
//                    survivors, per-expert slot allocation (the TaskPool "batch assembly" becomes a per-expert rank in token order)
//   layout_exchange  every rank stores its per-expert counts into every peer (P2P st), release/acquire flags, then each
//                    rank derives the SAME global layout: rows grouped by expert, groups padded to 128 rows
//   scatter_rows     fused permute + P2P store of token rows into the owner GPU's receive buffer (+ zero padding rows)
//   combine_rows     weighted un-permute: P2P loads of expert outputs from the owners, softmax-weighted sum
//   bwd_dispatch     d(weights) = <grad, expert_out> (P2P load), push w*grad to the owners (P2P store),
//                    softmax backward -> gradient w.r.t. the grid logits
//
// Memory ordering protocol (SURVEY.md §5.2): data is written with plain stores, then `__threadfence_system()` +
// `st.release.sys` of a monotonically increasing epoch into the consumer's flag word; consumers poll with
// `ld.acquire.sys`.  Flags never need resetting.  Every poll loop has a clock64() timeout that raises status[0].
#include "sm90.cuh"

namespace lah {

constexpr int MAX_WORLD = 8;
constexpr int MAX_GRID_DIMS = 4;
constexpr int MAX_K = 8;
constexpr long long SPIN_TIMEOUT_CYCLES = 20000000000ll;  // ~10 s

struct Peers {
    char* base[MAX_WORLD];  // base of every rank's symmetric heap, as mapped in THIS process
    int world;
    int me;
    unsigned long long* wait_ns;  // optional device counter: ns this rank spent blocked on peer flags ("exposed" comm)
    // device-resident step counters (CUDA-graph replay: nothing that changes from step to step is a kernel argument):
    //   step_ctr[0] = epoch base added to every (step-relative) epoch argument;  step_ctr[2..3] = 64-bit token base added to
    //   the gate's token_offset (failure-injection RNG stream).  Bumped by step_begin_kernel.  nullptr -> 0.
    int* step_ctr;
    int spin_timeout_ms;          // flag-wait timeout (0 -> ~10 s); a timed-out wait raises STATUS_TIMEOUT and goes on
    // NVSwitch multicast alias of the symmetric heap (same offsets; nullptr when the arena is a legacy IPC mapping): one
    // multimem.st reaches every rank's copy, multimem.ld_reduce returns the in-switch sum of all copies (NVLS)
    char* mc_base;
};

__device__ __forceinline__ void multimem_st_release_u32(void* mc_addr, int v) {
    asm volatile("multimem.st.release.sys.global.u32 [%0], %1;" ::"l"(mc_addr), "r"(v) : "memory");
}
__device__ __forceinline__ void multimem_st_u32(void* mc_addr, int v) {
    asm volatile("multimem.st.relaxed.sys.global.u32 [%0], %1;" ::"l"(mc_addr), "r"(v) : "memory");
}

// publish `epoch` into flag word [slot][me] of EVERY rank.  Call from the threads [0, world) of one warp after the data
// stores (each caller fences).  With a multicast mapping this is ONE store replicated by the switch.
__device__ __forceinline__ void signal_all_ranks(const Peers& peers, long long flags_off, int slot, int epoch, int tid) {
    if (peers.mc_base) {
        if (tid == 0) {
            __threadfence_system();
            multimem_st_release_u32(peers.mc_base + flags_off + (static_cast<long long>(slot) * MAX_WORLD + peers.me) * 4, epoch);
        }
    } else if (tid < peers.world) {
        __threadfence_system();
        st_release_sys(reinterpret_cast<int*>(peers.base[tid] + flags_off) + slot * MAX_WORLD + peers.me, epoch);
    }
}

__device__ __forceinline__ int epoch_of(const Peers& peers, int rel) {
    return rel + (peers.step_ctr ? *reinterpret_cast<volatile const int*>(peers.step_ctr) : 0);
}

struct GridSpec {
    int ndim;
    int size[MAX_GRID_DIMS];    // grid_size
    int offset[MAX_GRID_DIMS];  // offset of the dim's logits inside a logits row
    int total;                  // sum(size)
    int num_experts;            // prod(size)
};

enum Status { STATUS_TIMEOUT = 1, STATUS_OVERFLOW = 2 };

__device__ __forceinline__ float hash_uniform(unsigned long long x) {
    // splitmix64 -> uniform in [0, 1)
    x += 0x9E3779B97F4A7C15ull;
    x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ull;
    x = (x ^ (x >> 27)) * 0x94D049BB133111EBull;
    x = x ^ (x >> 31);
    return static_cast<float>(x >> 40) * (1.0f / 16777216.0f);
}

// rank: the peer whose flag this is.  Excluded ranks (status[1] bit) are never waited for; once a wait of this step timed
// out (status[0] bit 0) the remaining waits return at once — the step is abandoned, its optimizer updates are skipped
__device__ __forceinline__ bool spin_until_ge(const int* flag, int epoch, int* status, int timeout_ms = 0, int rank = -1) {
    if (status && rank >= 0) {
        const volatile int* vs = status;
        if ((vs[1] >> rank) & 1) return false;
        if (vs[0] & STATUS_TIMEOUT) return false;
    }
    const long long t0 = clock64();
    const long long limit = timeout_ms > 0 ? static_cast<long long>(timeout_ms) * 2000000ll : SPIN_TIMEOUT_CYCLES;
    while (ld_acquire_sys(flag) < epoch) {
        if (clock64() - t0 > limit) {
            atomicOr(status, STATUS_TIMEOUT);
            return false;
        }
    }
    return true;
}

// called by the threads [0, world) of one warp right after their spin: adds the LONGEST of their waits to the counter
__device__ __forceinline__ void account_wait(const Peers& peers, unsigned long long t0, int world) {
    const unsigned long long dt64 = globaltimer_ns() - t0;
    const unsigned mask = (world >= 32) ? 0xffffffffu : ((1u << world) - 1u);
    const unsigned dt = __reduce_max_sync(mask, dt64 > 0xffffffffull ? 0xffffffffu : static_cast<unsigned>(dt64));
    if (peers.wait_ns && (threadIdx.x & 31) == 0) atomicAdd(peers.wait_ns, static_cast<unsigned long long>(dt));
}

// ------------------------------------------------------------------------------------------------
// gate: one warp per token
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) gate_topk_kernel(const float* __restrict__ logits, int B, GridSpec gs, int k,
                                                        const unsigned char* __restrict__ alive, float failure_rate,
                                                        unsigned long long seed, long long token_offset,
                                                        int* __restrict__ idx_out, float* __restrict__ w_out,
                                                        int* __restrict__ pos_out, int* __restrict__ counts,
                                                        const int* __restrict__ step_ctr) {
    if (step_ctr) token_offset += *reinterpret_cast<const long long*>(step_ctr + 2);
    extern __shared__ float s_logits[];  // [8 warps][gs.total]
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int b = blockIdx.x * 8 + warp;
    if (b >= B) return;
    float* lg = s_logits + warp * gs.total;
    for (int i = lane; i < gs.total; i += 32) lg[i] = logits[static_cast<long long>(b) * gs.total + i];
    __syncwarp();

    // per-lane sorted top-k over the candidates this lane owns (c = lane, lane+32, ...)
    float best_v[MAX_K];
    int best_i[MAX_K];
#pragma unroll
    for (int j = 0; j < MAX_K; ++j) {
        best_v[j] = -INFINITY;
        best_i[j] = -1;
    }
    for (int c = lane; c < gs.num_experts; c += 32) {
        if (alive && !alive[c]) continue;
        if (failure_rate > 0.f) {
            const unsigned long long key = seed ^ (static_cast<unsigned long long>(token_offset + b) * 0x100000001B3ull +
                                                   static_cast<unsigned long long>(c));
            if (hash_uniform(key) < failure_rate) continue;
        }
        int rem = c;
        float s = 0.f;
#pragma unroll
        for (int d = MAX_GRID_DIMS - 1; d >= 0; --d) {
            if (d < gs.ndim) {
                const int i = rem % gs.size[d];
                rem /= gs.size[d];
                s += lg[gs.offset[d] + i];
            }
        }
        // insertion (ties keep the smaller expert id first because candidates arrive in increasing order)
        if (s > best_v[MAX_K - 1] || best_i[MAX_K - 1] < 0) {
            float v = s;
            int id = c;
            bool shifting = false;  // once inserted, everything below shifts down by one
#pragma unroll
            for (int j = 0; j < MAX_K; ++j) {
                const bool take = shifting || (best_i[j] < 0) || (v > best_v[j]);
                if (take) {
                    shifting = true;
                    const float tv = best_v[j];
                    const int ti = best_i[j];
                    best_v[j] = v;
                    best_i[j] = id;
                    v = tv;
                    id = ti;
                }
            }
        }
    }
    // merge: k rounds of warp arg-max over the heads of the per-lane lists
    float sel_v[MAX_K];
    int sel_i[MAX_K];
    int head = 0;
#pragma unroll
    for (int j = 0; j < MAX_K; ++j) {
        sel_v[j] = -INFINITY;
        sel_i[j] = -1;
        if (j < k) {
            float v = -INFINITY;
            int id = -1;
#pragma unroll
            for (int t = 0; t < MAX_K; ++t)
                if (t == head) {
                    v = best_v[t];
                    id = best_i[t];
                }
            float bv = v;
            int bi = id;
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) {
                const float ov = __shfl_xor_sync(0xffffffffu, bv, o);
                const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
                const bool better = (oi >= 0) && (bi < 0 || ov > bv || (ov == bv && oi < bi));
                if (better) {
                    bv = ov;
                    bi = oi;
                }
            }
            sel_v[j] = bv;
            sel_i[j] = bi;
            if (bi >= 0 && bi == id) ++head;  // the winning lane pops its head
        }
    }
    // softmax over the selected (alive) experts
    float mx = -INFINITY;
#pragma unroll
    for (int j = 0; j < MAX_K; ++j)
        if (sel_i[j] >= 0) mx = fmaxf(mx, sel_v[j]);
    float denom = 0.f;
#pragma unroll
    for (int j = 0; j < MAX_K; ++j)
        if (sel_i[j] >= 0) denom += __expf(sel_v[j] - mx);
    if (lane < k) {
        int id = -1;
        float v = 0.f;
#pragma unroll
        for (int j = 0; j < MAX_K; ++j)
            if (j == lane) {
                id = sel_i[j];
                v = sel_v[j];
            }
        const long long o = static_cast<long long>(b) * k + lane;
        idx_out[o] = id;
        w_out[o] = id >= 0 ? __expf(v - mx) / denom : 0.f;
        if (id < 0) pos_out[o] = 0;   // slots of the routed pairs: rank_slots_kernel
    }
}

// slot of every routed (token, choice) pair inside its expert = the number of EARLIER pairs (token-major order) routed to
// the same expert; counts[e] += pairs routed to e.  One CTA per expert: the row order inside every expert group, and with
// it every reduction over an expert's rows, is the same in every run (an atomic slot counter would order rows by arrival).
__global__ void __launch_bounds__(1024) rank_slots_kernel(const int* __restrict__ idx, int n, int* __restrict__ pos,
                                                          int* __restrict__ counts) {
    __shared__ int warp_off[32];
    __shared__ int s_total;
    const int e = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    int base = 0;
    for (int start = 0; start < n; start += 1024) {
        const int i = start + tid;
        const bool hit = i < n && __ldg(idx + i) == e;
        const unsigned m = __ballot_sync(0xffffffffu, hit);
        if (lane == 0) warp_off[warp] = __popc(m);
        __syncthreads();
        if (warp == 0) {
            const int v = warp_off[lane];
            int incl = v;
#pragma unroll
            for (int d = 1; d < 32; d <<= 1) {
                const int y = __shfl_up_sync(0xffffffffu, incl, d);
                if (lane >= d) incl += y;
            }
            warp_off[lane] = incl - v;
            if (lane == 31) s_total = incl;
        }
        __syncthreads();
        if (hit) pos[i] = base + warp_off[warp] + __popc(m & ((1u << lane) - 1u));
        base += s_total;
        __syncthreads();   // warp_off / s_total are rewritten by the next chunk
    }
    if (tid == 0 && base) counts[e] += base;
}

// ------------------------------------------------------------------------------------------------
// layout exchange: single CTA of 1024 threads
// ------------------------------------------------------------------------------------------------
struct LayoutArgs {
    long long cnt_all_off;   // symmetric int [MAX_WORLD][E]
    long long flags_off;     // symmetric int [slots][MAX_WORLD]
    int slot;
    int epoch;
    int E, E_loc;
    int max_rows;            // capacity of the receive buffers (rows)
    int max_tiles;           // max_rows / tile_rows
    int align;               // group padding in rows: 128 (1-CTA GEMM), 256 (wide-tile GEMM) or 16 (small-M swap-AB path)
    int tile_rows;           // rows per tile_group entry: min(align, 128)
    int* counts;             // [E] local counts (zeroed on exit)
    int* dst_row;            // [E]  row (in route_owner[e]'s buffer) where MY first row for expert e goes
    int* group_off;          // [E_loc + S_max + 1] padded offsets of my groups (owned experts, then shadow slots)
    int* group_rows;         // [E_loc + S_max] valid rows of my groups
    int* tile_group;         // [max_tiles]
    int* total_rows;         // [1] padded rows in my buffer
    int* status;
    // ---- hot-expert shadowing (dynamic data-parallel replicas; see the kernel comment)
    int S_max;               // shadow slots per rank (0 disables)
    float shadow_tol;        // stop once the most loaded rank is within tol x mean
    int min_shadow_rows;     // never shadow an expert with fewer total rows
    int* route_owner;        // [E]  rank whose buffer receives MY rows of expert e
    int* step_rows;          // [E_loc] GLOBAL rows of my owned experts (optimizer gating)
    int* shadow_info;        // [S_max][4]: expert (-1 = unused), owner, my rows in the slot (0 if I own it), rank mask
    int* owned_shadow;       // [E_loc][2]: shadow slot of my owned expert (-1 = none), mask of ranks that have rows
};

constexpr int LAYOUT_MAX_E = 4096;

// Load balancing.  Expert popularity is heavily skewed once training starts (a handful of experts receive most rows),
// so a static expert -> GPU placement leaves most GPUs idle behind the owner of a hot expert.  After the count exchange
// every rank knows the full [rank][expert] histogram and runs the SAME greedy selection: while the most loaded rank
// exceeds tol x mean, its largest expert becomes a SHADOWED expert.  Rows routed to a shadowed expert are not dispatched:
// every rank processes its own rows with a replica of the expert's weights (pulled from the owner over NVLink, see
// pull_shadow_kernel) in one of its S_max shadow groups, and the owner's optimizer sums the partial weight gradients of
// all ranks (adam.cu).  Shadowing an expert spreads its rows exactly like the tokens are spread (data parallel).
__global__ void __launch_bounds__(1024) layout_exchange_kernel(Peers peers, LayoutArgs a) {
    __shared__ int warp_tot[32];
    __shared__ int owner_base_s[MAX_WORLD + 1];
    __shared__ int s_tot[LAYOUT_MAX_E];
    __shared__ short s_slot[LAYOUT_MAX_E];
    __shared__ long long s_load[MAX_WORLD];
    __shared__ int s_shadow[MAX_WORLD * 2];   // S_max <= 16
    __shared__ int s_pick[2];
    __shared__ int s_red_v[32], s_red_i[32];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int me = peers.me, world = peers.world;
    a.epoch = epoch_of(peers, a.epoch);
    // 1. publish my counts to every peer (one multimem.st per word through the switch, or plain P2P stores), then
    //    release the epoch flag on every peer
    if (peers.mc_base) {
        int* dst = reinterpret_cast<int*>(peers.mc_base + a.cnt_all_off) + static_cast<long long>(me) * a.E;
        for (int e = tid; e < a.E; e += blockDim.x) multimem_st_u32(dst + e, a.counts[e]);
    } else {
        for (int r = 0; r < world; ++r) {
            int* dst = reinterpret_cast<int*>(peers.base[r] + a.cnt_all_off) + static_cast<long long>(me) * a.E;
            for (int e = tid; e < a.E; e += blockDim.x) dst[e] = a.counts[e];
        }
    }
    __threadfence_system();
    __syncthreads();
    signal_all_ranks(peers, a.flags_off, a.slot, a.epoch, tid);
    if (tid < world) {
        // 2. wait for everybody's counts
        const int* fw = reinterpret_cast<const int*>(peers.base[me] + a.flags_off) + a.slot * MAX_WORLD + tid;
        const unsigned long long t0 = globaltimer_ns();
        spin_until_ge(fw, a.epoch, a.status, peers.spin_timeout_ms, tid);
        account_wait(peers, t0, world);
    }
    __syncthreads();
    {   // excluded ranks (host-maintained mask in status[1]) contribute no rows: their (stale) count rows read as zero
        const int dead = reinterpret_cast<volatile int*>(a.status)[1];
        if (dead) {
            int* mine = reinterpret_cast<int*>(peers.base[me] + a.cnt_all_off);
            for (int r = 0; r < world; ++r)
                if ((dead >> r) & 1)
                    for (int e = tid; e < a.E; e += blockDim.x) mine[static_cast<long long>(r) * a.E + e] = 0;
        }
    }
    for (int t = tid; t < a.max_tiles; t += blockDim.x) a.tile_group[t] = -1;
    if (tid < MAX_WORLD) s_load[tid] = 0;
    if (tid < MAX_WORLD * 2) s_shadow[tid] = -1;
    __syncthreads();
    const int* cnt_all = reinterpret_cast<const int*>(peers.base[me] + a.cnt_all_off);
    // 3. totals per expert and the initial load of every rank (= rows of the experts it owns)
    for (int e = tid; e < a.E; e += blockDim.x) {
        int tot = 0;
        for (int s = 0; s < world; ++s) tot += cnt_all[static_cast<long long>(s) * a.E + e];
        s_tot[e] = tot;
        s_slot[e] = -1;
        if (tot) atomicAdd(reinterpret_cast<unsigned long long*>(&s_load[e / a.E_loc]), static_cast<unsigned long long>(tot));
    }
    __syncthreads();
    // 4. greedy shadow selection (identical on every rank: same inputs, deterministic tie-breaks)
    int num_shadow = 0;
    for (int it = 0; it < a.S_max && world > 1; ++it) {
        if (tid == 0) {
            long long total = 0, mx = -1;
            int rmax = 0;
            for (int r = 0; r < world; ++r) {
                total += s_load[r];
                if (s_load[r] > mx) {
                    mx = s_load[r];
                    rmax = r;
                }
            }
            const bool balanced = static_cast<float>(mx) * world <= a.shadow_tol * static_cast<float>(total);
            s_pick[0] = balanced ? -1 : rmax;
        }
        __syncthreads();
        const int rmax = s_pick[0];
        if (rmax < 0) break;
        // arg-max of tot[e] over the not yet shadowed experts of rank rmax (ties: smaller expert id)
        int bv = -1, bi = -1;
        for (int le = tid; le < a.E_loc; le += blockDim.x) {
            const int e = rmax * a.E_loc + le;
            if (s_slot[e] < 0 && s_tot[e] > bv) {
                bv = s_tot[e];
                bi = e;
            }
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            const int ov = __shfl_xor_sync(0xffffffffu, bv, o);
            const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
            if (ov > bv || (ov == bv && oi >= 0 && (bi < 0 || oi < bi))) {
                bv = ov;
                bi = oi;
            }
        }
        if (lane == 0) {
            s_red_v[warp] = bv;
            s_red_i[warp] = bi;
        }
        __syncthreads();
        if (tid == 0) {
            int v = -1, i = -1;
            for (int w = 0; w < 32; ++w)
                if (s_red_v[w] > v || (s_red_v[w] == v && s_red_i[w] >= 0 && (i < 0 || s_red_i[w] < i))) {
                    v = s_red_v[w];
                    i = s_red_i[w];
                }
            if (i < 0 || v < a.min_shadow_rows) {
                s_pick[1] = -1;
            } else {
                s_pick[1] = i;
                s_slot[i] = static_cast<short>(it);
                s_shadow[it] = i;
                s_load[rmax] -= v;
                for (int r = 0; r < world; ++r) s_load[r] += cnt_all[static_cast<long long>(r) * a.E + i];
            }
        }
        __syncthreads();
        if (s_pick[1] < 0) break;
        ++num_shadow;
    }
    // 5. layout of the OWNED groups of every rank, computed redundantly (and identically) everywhere:
    //    rows(e) = all rows of e, or only the owner's own rows when e is shadowed
    //    dst_row[e] <- exclusive prefix of padded group sizes over ALL experts (temporarily),
    //    counts[e]  <- rows of expert e that come from ranks < me (the local counts are consumed by now)
    int running = 0;
    for (int chunk = 0; chunk < a.E; chunk += blockDim.x) {
        const int e = chunk + tid;
        int rows = 0, before = 0;
        if (e < a.E) {
            if (s_slot[e] >= 0) {
                rows = cnt_all[static_cast<long long>(e / a.E_loc) * a.E + e];
            } else {
                rows = s_tot[e];
                for (int s = 0; s < me; ++s) before += cnt_all[static_cast<long long>(s) * a.E + e];
            }
        }
        const int padded = (rows + a.align - 1) / a.align * a.align;
        int v = padded;  // inclusive scan inside the warp
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const int n = __shfl_up_sync(0xffffffffu, v, o);
            if (lane >= o) v += n;
        }
        if (lane == 31) warp_tot[warp] = v;
        __syncthreads();
        if (warp == 0) {
            int w = warp_tot[lane];
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const int n = __shfl_up_sync(0xffffffffu, w, o);
                if (lane >= o) w += n;
            }
            warp_tot[lane] = w;
        }
        __syncthreads();
        const int excl = running + (warp > 0 ? warp_tot[warp - 1] : 0) + v - padded;
        running += warp_tot[31];
        if (e < a.E) {
            a.dst_row[e] = excl;
            a.counts[e] = before;
            if (e / a.E_loc == me) a.group_rows[e - me * a.E_loc] = rows;
        }
        __syncthreads();
    }
    if (tid < world) owner_base_s[tid] = a.dst_row[tid * a.E_loc];
    if (tid == 0) owner_base_s[world] = running;
    __syncthreads();
    // 6. my shadow groups follow my owned groups; every rank's total is checked against the buffer capacity
    const int G_own = a.E_loc;
    if (tid == 0) {
        int cur = owner_base_s[me + 1] - owner_base_s[me];
        for (int s = 0; s < a.S_max; ++s) {
            const int e = s_shadow[s];
            const int rows = (e >= 0 && e / a.E_loc != me) ? cnt_all[static_cast<long long>(me) * a.E + e] : 0;
            const int padded = (rows + a.align - 1) / a.align * a.align;
            a.group_off[G_own + s] = cur;
            a.group_rows[G_own + s] = rows;
            for (int t = cur / a.tile_rows; t < (cur + padded) / a.tile_rows && t < a.max_tiles; ++t) a.tile_group[t] = G_own + s;
            int mask = 0;
            if (e >= 0)
                for (int r = 0; r < world; ++r) mask |= (cnt_all[static_cast<long long>(r) * a.E + e] > 0) << r;
            a.shadow_info[4 * s + 0] = e;
            a.shadow_info[4 * s + 1] = e >= 0 ? e / a.E_loc : -1;
            a.shadow_info[4 * s + 2] = rows;
            a.shadow_info[4 * s + 3] = mask;
            cur += padded;
        }
        a.group_off[G_own + a.S_max] = cur;
        *a.total_rows = cur;
    }
    if (tid < world) {
        int total = owner_base_s[tid + 1] - owner_base_s[tid];
        for (int s = 0; s < a.S_max; ++s) {
            const int e = s_shadow[s];
            if (e >= 0 && e / a.E_loc != tid)
                total += (cnt_all[static_cast<long long>(tid) * a.E + e] + a.align - 1) / a.align * a.align;
        }
        if (total > a.max_rows) atomicOr(a.status, STATUS_OVERFLOW);
    }
    __syncthreads();
    // 7. make offsets owner-relative; routing tables; tables of my owned experts
    for (int e = tid; e < a.E; e += blockDim.x) {
        const int owner = e / a.E_loc;
        const int rel = a.dst_row[e] - owner_base_s[owner];
        const int before = a.counts[e];
        const int slot = s_slot[e];
        a.counts[e] = 0;  // leave the slot counters clean for the next gate call
        if (owner == me) {
            const int le = e - me * a.E_loc;
            a.group_off[le] = rel;
            const int padded = (a.group_rows[le] + a.align - 1) / a.align * a.align;
            for (int t = rel / a.tile_rows; t < (rel + padded) / a.tile_rows && t < a.max_tiles; ++t) a.tile_group[t] = le;
            if (a.step_rows) a.step_rows[le] = s_tot[e];
            if (a.owned_shadow) {
                int mask = 0;
                if (slot >= 0)
                    for (int r = 0; r < world; ++r) mask |= (cnt_all[static_cast<long long>(r) * a.E + e] > 0) << r;
                a.owned_shadow[2 * le] = slot;
                a.owned_shadow[2 * le + 1] = mask;
            }
        }
        int dst, route;
        if (slot < 0) {
            dst = rel + before;
            route = owner;
        } else if (owner == me) {
            dst = rel;
            route = me;
        } else {
            dst = a.group_off[G_own + slot];
            route = me;
        }
        a.dst_row[e] = dst;
        if (a.route_owner) a.route_owner[e] = route;
    }
}

// ------------------------------------------------------------------------------------------------
// scatter: warp per (token, slot) pair -> P2P store of the row; extra CTAs zero the padding rows of local experts;
// the last CTA to finish releases the epoch flag on every peer.
// ------------------------------------------------------------------------------------------------
struct ScatterArgs {
    const bf16* src;          // [B, H] rows to send (x in forward, grad in backward)
    const float* scale;       // [B*k] optional per-pair scale (backward: gate weights) or nullptr
    const int* idx;           // [B*k] expert ids
    const int* pos;           // [B*k] slot inside (me, expert)
    const int* dst_row;       // [E]
    int* pair_row;            // [B*k] out: row in the owner's buffer (or -1); nullptr in backward (rows known)
    long long dst_off;        // symmetric receive buffer [max_rows, H] bf16
    long long flags_off;
    int slot, epoch;
    int num_pairs, k, H, E_loc, max_rows;
    const int* group_off;     // local experts (for zero padding)
    const int* group_rows;
    int pair_blocks;          // CTAs that handle pairs; the rest zero padding
    int align;                // group padding in rows
    const int* route_owner;   // [E] destination rank of MY rows of expert e (nullptr: the owner e / E_loc)
    int num_groups;           // groups in my buffer (owned experts + shadow slots) whose padding rows are zeroed
    int* done_counter;
    int* status;
};

template <int VEC_PER_LANE>
__global__ void __launch_bounds__(256) scatter_rows_kernel(Peers peers, ScatterArgs a) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (static_cast<int>(blockIdx.x) < a.pair_blocks) {
        const int p = blockIdx.x * 8 + warp;
        if (p < a.num_pairs) {
            const int e = a.idx[p];
            int row = -1;
            if (e >= 0) {
                row = (a.pair_row && !a.dst_row) ? a.pair_row[p] : a.dst_row[e] + a.pos[p];
                if (row >= a.max_rows) {
                    if (lane == 0) atomicOr(a.status, STATUS_OVERFLOW);
                    row = -1;
                }
            }
            if (a.pair_row && a.dst_row && lane == 0) a.pair_row[p] = row;
            if (row >= 0) {
                const int owner = a.route_owner ? a.route_owner[e] : e / a.E_loc;
                const int b = p / a.k;
                const int4* sp = reinterpret_cast<const int4*>(a.src + static_cast<long long>(b) * a.H);
                int4* dp = reinterpret_cast<int4*>(peers.base[owner] + a.dst_off) +
                           static_cast<long long>(row) * (a.H / 8);
                int4 v[VEC_PER_LANE];
#pragma unroll
                for (int j = 0; j < VEC_PER_LANE; ++j) v[j] = ld_nc_v4(sp + j * 32 + lane);
                if (a.scale) {
                    const float s = a.scale[p];
#pragma unroll
                    for (int j = 0; j < VEC_PER_LANE; ++j) {
                        uint32_t* u = reinterpret_cast<uint32_t*>(&v[j]);
#pragma unroll
                        for (int t = 0; t < 4; ++t) {
                            const float2 f = unpack_bf16x2(u[t]);
                            u[t] = pack_bf16x2(f.x * s, f.y * s);
                        }
                    }
                }
#pragma unroll
                for (int j = 0; j < VEC_PER_LANE; ++j) st_v4(dp + j * 32 + lane, v[j]);
            }
        }
    } else {
        // zero the padding rows of my local experts (rows [off+rows, next off))
        const int nb = gridDim.x - a.pair_blocks;
        int4* base = reinterpret_cast<int4*>(peers.base[peers.me] + a.dst_off);
        const int4 z = make_int4(0, 0, 0, 0);
        for (int le = blockIdx.x - a.pair_blocks; le < a.num_groups; le += nb) {
            const int r0 = a.group_off[le] + a.group_rows[le];
            const int r1 = min(a.max_rows, a.group_off[le] + (a.group_rows[le] + a.align - 1) / a.align * a.align);
            for (int r = r0 + warp; r < r1; r += 8) {
                int4* dp = base + static_cast<long long>(r) * (a.H / 8);
#pragma unroll
                for (int j = 0; j < VEC_PER_LANE; ++j) dp[j * 32 + lane] = z;
            }
        }
    }
    // completion: last CTA publishes the epoch to every peer
    __syncthreads();
    if (threadIdx.x == 0) {
        __threadfence_system();
        const int prev = atomicAdd(a.done_counter, 1);
        if (prev == static_cast<int>(gridDim.x) - 1) {
            *a.done_counter = 0;
            __threadfence_system();
            const int epoch = epoch_of(peers, a.epoch);
            if (peers.mc_base) {
                multimem_st_release_u32(peers.mc_base + a.flags_off + (static_cast<long long>(a.slot) * MAX_WORLD + peers.me) * 4, epoch);
            } else {
                for (int r = 0; r < peers.world; ++r) {
                    int* f = reinterpret_cast<int*>(peers.base[r] + a.flags_off) + a.slot * MAX_WORLD + peers.me;
                    st_release_sys(f, epoch);
                }
            }
        }
    }
}

// ------------------------------------------------------------------------------------------------
// flag helpers: signal every peer / wait for every peer (single warp)
// ------------------------------------------------------------------------------------------------
__global__ void signal_wait_kernel(Peers peers, long long flags_off, int slot, int epoch, int do_signal, int do_wait,
                                   int* status) {
    const int lane = threadIdx.x;
    epoch = epoch_of(peers, epoch);
    if (do_signal) signal_all_ranks(peers, flags_off, slot, epoch, lane);
    if (do_wait && lane < peers.world) {
        const int* f = reinterpret_cast<const int*>(peers.base[peers.me] + flags_off) + slot * MAX_WORLD + lane;
        const unsigned long long t0 = globaltimer_ns();
        spin_until_ge(f, epoch, status, peers.spin_timeout_ms, lane);
        account_wait(peers, t0, peers.world);
    }
}

// NVLS all-reduce (in place, one shot) of a float buffer that lives at the same offset of every rank's symmetric heap:
// rank r owns the r-th slice: multimem.ld_reduce returns the sum of all ranks' copies (added INSIDE the switch), the
// scaled result goes back to every rank with one multimem.st.  Every rank therefore ends up with the bit-identical
// reduced gradient (replicated trainer parameters must not drift apart), and each element crosses NVLink once per
// direction instead of `world` P2P loads per rank.  Callers bracket it with flag barriers (all gradients written /
// all slices reduced).  Reference: the trainers of the emulator share these parameters under a lock (notebook cell 3).
__global__ void __launch_bounds__(256) nvls_allreduce_kernel(Peers peers, long long off, long long n, float scale) {
    const long long per = ((n / 4 + peers.world - 1) / peers.world) * 4;   // float4 granularity
    const long long lo = per * peers.me, hi = min(n, lo + per);
    float* mc = reinterpret_cast<float*>(peers.mc_base + off);
    for (long long i = lo + (static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x) * 4; i < hi;
         i += static_cast<long long>(gridDim.x) * blockDim.x * 4) {
        float4 r;
        asm volatile("multimem.ld_reduce.relaxed.sys.global.add.v4.f32 {%0, %1, %2, %3}, [%4];"
                     : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w)
                     : "l"(mc + i)
                     : "memory");
        r.x *= scale; r.y *= scale; r.z *= scale; r.w *= scale;
        asm volatile("multimem.st.relaxed.sys.global.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(mc + i), "f"(r.x), "f"(r.y),
                     "f"(r.z), "f"(r.w)
                     : "memory");
    }
}

// liveness broadcast: the owner of experts [first, first + count) stamps their heartbeat (ms, 64 bit) into the table of
// EVERY rank with one multimem.st per expert (declare_experts of the reference: one DHT store per uid and prefix,
// /root/reference/lib/network/__init__.py:69-86); without multicast: unicast P2P stores
__global__ void heartbeat_kernel(Peers peers, long long hb_off, int first, int count, long long now_ms) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= count) return;
    if (peers.mc_base) {
        asm volatile("multimem.st.relaxed.sys.global.u64 [%0], %1;" ::"l"(reinterpret_cast<long long*>(peers.mc_base + hb_off) + first + i),
                     "l"(now_ms)
                     : "memory");
    } else {
        for (int r = 0; r < peers.world; ++r) reinterpret_cast<long long*>(peers.base[r] + hb_off)[first + i] = now_ms;
    }
}

// alive[e] = (now - hb[e] <= max_age) for every expert: turns the heartbeat table into the mask the gate kernel reads
__global__ void alive_from_heartbeats_kernel(const long long* hb, unsigned char* alive, int E, long long now_ms, long long max_age_ms) {
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e < E) alive[e] = (hb[e] > 0 && now_ms - hb[e] <= max_age_ms) ? 1 : 0;
}

// one thread: advance the device-side step counters (see Peers::step_ctr)
__global__ void step_begin_kernel(int* step_ctr, int epoch_delta, long long token_delta) {
    step_ctr[0] += epoch_delta;
    *reinterpret_cast<long long*>(step_ctr + 2) += token_delta;
}

// ------------------------------------------------------------------------------------------------
// combine: warp per token; out[b] = sum_j w[b,j] * src_owner(j)[row(b,j)]     (w == nullptr -> plain sum)
// ------------------------------------------------------------------------------------------------
struct CombineArgs {
    long long src_off;        // symmetric [max_rows, H] bf16 on the owners
    const int* idx;           // [B*k]
    const int* pair_row;      // [B*k]
    const float* w;           // [B*k] or nullptr
    bf16* out;                // [B, H]
    int B, k, H, E_loc;
    // fused flag protocol: block 0 publishes 'my expert outputs are complete' to every peer, every block waits for all
    long long flags_off;
    int slot, epoch, do_signal, do_wait;
    int* status;
    const int* route_owner;   // [E] rank that holds MY rows of expert e (nullptr: e / E_loc)
};

template <int VEC_PER_LANE>
__global__ void __launch_bounds__(256) combine_rows_kernel(Peers peers, CombineArgs a) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (a.do_signal || a.do_wait) a.epoch = epoch_of(peers, a.epoch);
    if (a.do_signal && blockIdx.x == 0 && threadIdx.x < 32) {
        // everything launched before this kernel on the stream (the last expert GEMM) is complete: tell the peers
        signal_all_ranks(peers, a.flags_off, a.slot, a.epoch, threadIdx.x);
    }
    if (a.do_wait) {
        if (threadIdx.x < peers.world) {
            const int* f = reinterpret_cast<const int*>(peers.base[peers.me] + a.flags_off) + a.slot * MAX_WORLD + threadIdx.x;
            const unsigned long long t0 = globaltimer_ns();
            spin_until_ge(f, a.epoch, a.status, peers.spin_timeout_ms, threadIdx.x);
            if (blockIdx.x == 0) account_wait(peers, t0, peers.world);
        }
        __syncthreads();
    }
    const int b = blockIdx.x * 8 + warp;
    if (b >= a.B) return;
    float acc[VEC_PER_LANE * 8];
#pragma unroll
    for (int i = 0; i < VEC_PER_LANE * 8; ++i) acc[i] = 0.f;
    for (int j = 0; j < a.k; ++j) {
        const long long p = static_cast<long long>(b) * a.k + j;
        const int e = a.idx[p];
        const int row = a.pair_row[p];
        if (e < 0 || row < 0) continue;
        const float w = a.w ? a.w[p] : 1.f;
        const int4* sp = reinterpret_cast<const int4*>(peers.base[a.route_owner ? a.route_owner[e] : e / a.E_loc] + a.src_off) +
                         static_cast<long long>(row) * (a.H / 8);
#pragma unroll
        for (int v = 0; v < VEC_PER_LANE; ++v) {
            const int4 q = ld_v4(sp + v * 32 + lane);
            const uint32_t u[4] = {(uint32_t)q.x, (uint32_t)q.y, (uint32_t)q.z, (uint32_t)q.w};
#pragma unroll
            for (int t = 0; t < 4; ++t) {
                const float2 f = unpack_bf16x2(u[t]);
                acc[v * 8 + 2 * t] += w * f.x;
                acc[v * 8 + 2 * t + 1] += w * f.y;
            }
        }
    }
    int4* op = reinterpret_cast<int4*>(a.out + static_cast<long long>(b) * a.H);
#pragma unroll
    for (int v = 0; v < VEC_PER_LANE; ++v) {
        int4 q;
        q.x = pack_bf16x2(acc[v * 8 + 0], acc[v * 8 + 1]);
        q.y = pack_bf16x2(acc[v * 8 + 2], acc[v * 8 + 3]);
        q.z = pack_bf16x2(acc[v * 8 + 4], acc[v * 8 + 5]);
        q.w = pack_bf16x2(acc[v * 8 + 6], acc[v * 8 + 7]);
        op[v * 32 + lane] = q;
    }
}

// ------------------------------------------------------------------------------------------------
// backward of combine (gate side): dw[b,j] = <g[b], y_j>;  dlogit_j = w_j (dw_j - sum_i w_i dw_i)
// scattered into the gradient of the grid logits [B, gs.total]
// ------------------------------------------------------------------------------------------------
struct GateBwdArgs {
    long long yo_off;         // symmetric expert outputs [max_rows, H]
    const bf16* grad;         // [B, H] grad w.r.t. the layer output
    const int* idx;
    const int* pair_row;
    const float* w;
    float* dlogits;           // [B, gs.total]
    int B, k, H, E_loc;
    const int* route_owner;   // [E] or nullptr
};

template <int VEC_PER_LANE>
__global__ void __launch_bounds__(256) gate_bwd_kernel(Peers peers, GateBwdArgs a, GridSpec gs) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int b = blockIdx.x * 8 + warp;
    if (b >= a.B) return;
    float g[VEC_PER_LANE * 8];
    const int4* gp = reinterpret_cast<const int4*>(a.grad + static_cast<long long>(b) * a.H);
#pragma unroll
    for (int v = 0; v < VEC_PER_LANE; ++v) {
        const int4 q = ld_nc_v4(gp + v * 32 + lane);
        const uint32_t u[4] = {(uint32_t)q.x, (uint32_t)q.y, (uint32_t)q.z, (uint32_t)q.w};
#pragma unroll
        for (int t = 0; t < 4; ++t) {
            const float2 f = unpack_bf16x2(u[t]);
            g[v * 8 + 2 * t] = f.x;
            g[v * 8 + 2 * t + 1] = f.y;
        }
    }
    float dw[MAX_K], wj[MAX_K];
    int ej[MAX_K];
    float dot_sum = 0.f;
#pragma unroll
    for (int j = 0; j < MAX_K; ++j) {
        dw[j] = 0.f;
        wj[j] = 0.f;
        ej[j] = -1;
        if (j < a.k) {
            const long long p = static_cast<long long>(b) * a.k + j;
            const int e = a.idx[p];
            const int row = a.pair_row[p];
            if (e >= 0 && row >= 0) {
                const int4* sp = reinterpret_cast<const int4*>(peers.base[a.route_owner ? a.route_owner[e] : e / a.E_loc] + a.yo_off) +
                                 static_cast<long long>(row) * (a.H / 8);
                float d = 0.f;
#pragma unroll
                for (int v = 0; v < VEC_PER_LANE; ++v) {
                    const int4 q = ld_v4(sp + v * 32 + lane);
                    const uint32_t u[4] = {(uint32_t)q.x, (uint32_t)q.y, (uint32_t)q.z, (uint32_t)q.w};
#pragma unroll
                    for (int t = 0; t < 4; ++t) {
                        const float2 f = unpack_bf16x2(u[t]);
                        d += g[v * 8 + 2 * t] * f.x + g[v * 8 + 2 * t + 1] * f.y;
                    }
                }
                d = warp_sum(d);
                dw[j] = d;
                wj[j] = a.w[p];
                ej[j] = e;
                dot_sum += wj[j] * d;
            }
        }
    }
    float* dl = a.dlogits + static_cast<long long>(b) * gs.total;
    for (int i = lane; i < gs.total; i += 32) dl[i] = 0.f;
    __syncwarp();
    if (lane == 0) {
#pragma unroll
        for (int j = 0; j < MAX_K; ++j) {
            if (ej[j] < 0) continue;
            const float d = wj[j] * (dw[j] - dot_sum);
            int rem = ej[j];
            for (int dd = gs.ndim - 1; dd >= 0; --dd) {
                const int i = rem % gs.size[dd];
                rem /= gs.size[dd];
                dl[gs.offset[dd] + i] += d;
            }
        }
    }
}

// ------------------------------------------------------------------------------------------------
// shadow replicas: pull the parameters of the shadowed experts from their owners (P2P loads over NVLink)
// Flat parameter layout (ExpertShard): segment sg holds [slots, seg_n[sg]] values starting at seg_start[sg]; slots =
// E_loc owned experts followed by S_max shadow slots.  Big segments (weights) are pulled from the bf16 mirror that the
// GEMMs consume, small ones (biases, LayerNorm affine) from the fp32 master copy.
// ------------------------------------------------------------------------------------------------
struct SegLayout {
    int num_segs;
    long long seg_start[13];
    long long seg_n[12];
};

struct PullArgs {
    const int* shadow_info;   // [S_max][4] written by layout_exchange
    int E_loc;
    long long p_off, pbf16_off;  // symmetric offsets of the fp32 parameters / bf16 mirror
    SegLayout L;
    int small_mask;           // bit sg: segment sg is a small fp32 parameter
};

__global__ void __launch_bounds__(256) pull_shadow_kernel(Peers peers, PullArgs a) {
    const int s = blockIdx.y;
    const int e = a.shadow_info[4 * s + 0], owner = a.shadow_info[4 * s + 1], rows = a.shadow_info[4 * s + 2];
    if (e < 0 || owner == peers.me || rows <= 0) return;
    const int le = e - owner * a.E_loc;
    const long long tid = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
    const long long nthreads = static_cast<long long>(gridDim.x) * blockDim.x;
    for (int sg = 0; sg < a.L.num_segs; ++sg) {
        const long long n = a.L.seg_n[sg];
        const bool small = (a.small_mask >> sg) & 1;
        const long long esz = small ? 4 : 2;
        const long long off = small ? a.p_off : a.pbf16_off;
        const int4* src = reinterpret_cast<const int4*>(peers.base[owner] + off + (a.L.seg_start[sg] + le * n) * esz);
        int4* dst = reinterpret_cast<int4*>(peers.base[peers.me] + off + (a.L.seg_start[sg] + (a.E_loc + s) * n) * esz);
        const long long nvec = n * esz / 16;
#pragma unroll 4
        for (long long v = tid; v < nvec; v += nthreads) dst[v] = ld_v4(src + v);
    }
}

// zero the gradient slots [first_slot, first_slot + num_slots) of the segments selected by seg_mask
__global__ void __launch_bounds__(256) zero_slots_kernel(float* g, SegLayout L, int first_slot, int num_slots, int seg_mask) {
    const int sg = blockIdx.y;
    if (!((seg_mask >> sg) & 1)) return;
    float4* base = reinterpret_cast<float4*>(g + L.seg_start[sg] + first_slot * L.seg_n[sg]);
    const long long nvec = num_slots * L.seg_n[sg] / 4;
    for (long long v = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; v < nvec;
         v += static_cast<long long>(gridDim.x) * blockDim.x)
        base[v] = make_float4(0.f, 0.f, 0.f, 0.f);
}

static Peers g_peers = {};
static bool g_peers_set = false;

}  // namespace lah

using namespace lah;

extern "C" {

// ---- peer table (set once after the symmetric heap rendezvous; see symm.cu / parallel/symmetric.py)
int lah_set_peers(const unsigned long long* bases, int world, int me) {
    if (world < 1 || world > MAX_WORLD || me < 0 || me >= world) return -2;
    for (int i = 0; i < MAX_WORLD; ++i) g_peers.base[i] = i < world ? reinterpret_cast<char*>(bases[i]) : nullptr;
    g_peers.world = world;
    g_peers.me = me;
    g_peers.wait_ns = nullptr;
    g_peers.step_ctr = nullptr;
    g_peers.spin_timeout_ms = 0;
    g_peers.mc_base = nullptr;
    g_peers_set = true;
    return 0;
}

// multicast alias of the symmetric heap (0 = none): enables the multimem.* paths
int lah_set_multicast(unsigned long long mc_base) {
    g_peers.mc_base = reinterpret_cast<char*>(mc_base);
    return 0;
}
unsigned long long lah_get_multicast() { return reinterpret_cast<unsigned long long>(g_peers.mc_base); }

// device-side step counters: int32[4] (see Peers::step_ctr); NULL disables (epochs / token offsets are then absolute)
int lah_set_step_counters(int* step_ctr) {
    g_peers.step_ctr = step_ctr;
    return 0;
}
const int* lah_get_epoch_base() { return g_peers.step_ctr; }

// timeout of every peer-flag wait in ms of SM clock at ~2 GHz (0 = default ~10 s)
int lah_set_spin_timeout_ms(int ms) {
    g_peers.spin_timeout_ms = ms;
    return 0;
}

int lah_nvls_allreduce(long long off, long long n, float scale, cudaStream_t st) {
    if (!g_peers_set || !g_peers.mc_base) return -10;
    if (n % 4 || off % 16) return -2;
    long long blocks = (n / 4 / g_peers.world + 255) / 256;
    if (blocks < 1) blocks = 1;
    if (blocks > 132 * 4) blocks = 132 * 4;
    nvls_allreduce_kernel<<<(int)blocks, 256, 0, st>>>(g_peers, off, n, scale);
    return -(int)cudaGetLastError();
}

int lah_heartbeat(long long hb_off, int first, int count, long long now_ms, cudaStream_t st) {
    if (!g_peers_set) return -10;
    if (count <= 0) return 0;
    heartbeat_kernel<<<(count + 127) / 128, 128, 0, st>>>(g_peers, hb_off, first, count, now_ms);
    return -(int)cudaGetLastError();
}

int lah_alive_from_heartbeats(const long long* hb, unsigned char* alive, int E, long long now_ms, long long max_age_ms,
                              cudaStream_t st) {
    if (E <= 0) return 0;
    alive_from_heartbeats_kernel<<<(E + 255) / 256, 256, 0, st>>>(hb, alive, E, now_ms, max_age_ms);
    return -(int)cudaGetLastError();
}

int lah_step_begin(int epoch_delta, long long token_delta, cudaStream_t st) {
    if (!g_peers.step_ctr) return -10;
    step_begin_kernel<<<1, 1, 0, st>>>(g_peers.step_ctr, epoch_delta, token_delta);
    return -(int)cudaGetLastError();
}

// device counter (8 bytes) that accumulates the ns this rank spends blocked on peer flags; NULL disables
int lah_set_wait_counter(unsigned long long* counter) {
    g_peers.wait_ns = counter;
    return 0;
}

static int make_grid_spec(GridSpec* gs, const int* grid, int ndim) {
    if (ndim < 1 || ndim > MAX_GRID_DIMS) return -2;
    gs->ndim = ndim;
    gs->total = 0;
    gs->num_experts = 1;
    for (int d = 0; d < MAX_GRID_DIMS; ++d) {
        gs->size[d] = d < ndim ? grid[d] : 1;
        gs->offset[d] = gs->total;
        if (d < ndim) {
            gs->total += grid[d];
            gs->num_experts *= grid[d];
        }
    }
    return 0;
}

int lah_gate_topk(const float* logits, int B, const int* grid, int ndim, int k, const unsigned char* alive,
                  float failure_rate, unsigned long long seed, long long token_offset, int* idx, float* w, int* pos,
                  int* counts, cudaStream_t st) {
    GridSpec gs;
    if (make_grid_spec(&gs, grid, ndim)) return -2;
    if (k < 1 || k > MAX_K) return -3;
    if (B <= 0) return 0;
    gate_topk_kernel<<<(B + 7) / 8, 256, 8 * gs.total * sizeof(float), st>>>(logits, B, gs, k, alive, failure_rate, seed,
                                                                           token_offset, idx, w, pos, counts,
                                                                           g_peers.step_ctr);
    rank_slots_kernel<<<gs.num_experts, 1024, 0, st>>>(idx, B * k, pos, counts);
    return -(int)cudaGetLastError();
}

int lah_layout_exchange(long long cnt_all_off, long long flags_off, int slot, int epoch, int E, int E_loc, int max_rows,
                        int align, int tile_rows, int* counts, int* dst_row, int* group_off, int* group_rows, int* tile_group, int* total_rows,
                        int* status, int S_max, float shadow_tol, int min_shadow_rows, int* route_owner, int* step_rows,
                        int* shadow_info, int* owned_shadow, cudaStream_t st) {
    if (!g_peers_set) return -10;
    if (E > LAYOUT_MAX_E || S_max < 0 || S_max > 2 * MAX_WORLD) return -2;
    LayoutArgs a;
    a.cnt_all_off = cnt_all_off; a.flags_off = flags_off; a.slot = slot; a.epoch = epoch; a.E = E; a.E_loc = E_loc;
    if (tile_rows <= 0 || align % tile_rows) return -2;
    a.max_rows = max_rows; a.tile_rows = tile_rows; a.max_tiles = max_rows / tile_rows; a.align = align; a.counts = counts; a.dst_row = dst_row; a.group_off = group_off;
    a.group_rows = group_rows; a.tile_group = tile_group; a.total_rows = total_rows; a.status = status;
    a.S_max = S_max; a.shadow_tol = shadow_tol; a.min_shadow_rows = min_shadow_rows; a.route_owner = route_owner;
    a.step_rows = step_rows; a.shadow_info = shadow_info; a.owned_shadow = owned_shadow;
    layout_exchange_kernel<<<1, 1024, 0, st>>>(g_peers, a);
    return -(int)cudaGetLastError();
}

int lah_scatter_rows(const void* src, const float* scale, const int* idx, const int* pos, const int* dst_row,
                     int* pair_row, long long dst_off, long long flags_off, int slot, int epoch, int num_pairs, int k,
                     int H, int E_loc, int max_rows, int align, const int* group_off, const int* group_rows,
                     int* done_counter, int* status, const int* route_owner, int num_groups, cudaStream_t st) {
    if (!g_peers_set) return -10;
    ScatterArgs a;
    a.src = (const bf16*)src; a.scale = scale; a.idx = idx; a.pos = pos; a.dst_row = dst_row; a.pair_row = pair_row;
    a.dst_off = dst_off; a.flags_off = flags_off; a.slot = slot; a.epoch = epoch; a.num_pairs = num_pairs; a.k = k;
    a.H = H; a.E_loc = E_loc; a.max_rows = max_rows; a.group_off = group_off; a.group_rows = group_rows;
    a.pair_blocks = (num_pairs + 7) / 8; a.align = align; a.done_counter = done_counter; a.status = status;
    a.route_owner = route_owner; a.num_groups = num_groups > 0 ? num_groups : E_loc;
    const int pad_blocks = a.num_groups < 64 ? a.num_groups : 64;
    const int grid = a.pair_blocks + pad_blocks;
    if (H == 256) scatter_rows_kernel<1><<<grid, 256, 0, st>>>(g_peers, a);
    else if (H == 512) scatter_rows_kernel<2><<<grid, 256, 0, st>>>(g_peers, a);
    else if (H == 1024) scatter_rows_kernel<4><<<grid, 256, 0, st>>>(g_peers, a);
    else return -2;
    return -(int)cudaGetLastError();
}

int lah_signal_wait(long long flags_off, int slot, int epoch, int do_signal, int do_wait, int* status,
                    cudaStream_t st) {
    if (!g_peers_set) return -10;
    signal_wait_kernel<<<1, 32, 0, st>>>(g_peers, flags_off, slot, epoch, do_signal, do_wait, status);
    return -(int)cudaGetLastError();
}

int lah_combine_rows(long long src_off, const int* idx, const int* pair_row, const float* w, void* out, int B, int k,
                     int H, int E_loc, long long flags_off, int slot, int epoch, int do_signal, int do_wait, int* status,
                     const int* route_owner, cudaStream_t st) {
    if (!g_peers_set) return -10;
    if (B <= 0) return 0;
    CombineArgs a;
    a.src_off = src_off; a.idx = idx; a.pair_row = pair_row; a.w = w; a.out = (bf16*)out; a.B = B; a.k = k; a.H = H;
    a.E_loc = E_loc; a.flags_off = flags_off; a.slot = slot; a.epoch = epoch; a.do_signal = do_signal; a.do_wait = do_wait;
    a.status = status; a.route_owner = route_owner;
    const int grid = (B + 7) / 8;
    if (H == 256) combine_rows_kernel<1><<<grid, 256, 0, st>>>(g_peers, a);
    else if (H == 512) combine_rows_kernel<2><<<grid, 256, 0, st>>>(g_peers, a);
    else if (H == 1024) combine_rows_kernel<4><<<grid, 256, 0, st>>>(g_peers, a);
    else return -2;
    return -(int)cudaGetLastError();
}

int lah_gate_bwd(long long yo_off, const void* grad, const int* idx, const int* pair_row, const float* w,
                 float* dlogits, int B, int k, int H, int E_loc, const int* grid_sizes, int ndim, const int* route_owner,
                 cudaStream_t st) {
    if (!g_peers_set) return -10;
    if (B <= 0) return 0;
    GridSpec gs;
    if (make_grid_spec(&gs, grid_sizes, ndim)) return -2;
    if (k > MAX_K) return -3;
    GateBwdArgs a;
    a.yo_off = yo_off; a.grad = (const bf16*)grad; a.idx = idx; a.pair_row = pair_row; a.w = w; a.dlogits = dlogits;
    a.B = B; a.k = k; a.H = H; a.E_loc = E_loc; a.route_owner = route_owner;
    const int grid = (B + 7) / 8;
    if (H == 256) gate_bwd_kernel<1><<<grid, 256, 0, st>>>(g_peers, a, gs);
    else if (H == 512) gate_bwd_kernel<2><<<grid, 256, 0, st>>>(g_peers, a, gs);
    else if (H == 1024) gate_bwd_kernel<4><<<grid, 256, 0, st>>>(g_peers, a, gs);
    else return -2;
    return -(int)cudaGetLastError();
}

static int make_seg_layout(SegLayout* L, int num_segs, const long long* seg_n, int slots) {
    if (num_segs < 1 || num_segs > 12) return -2;
    L->num_segs = num_segs;
    long long off = 0;
    for (int s = 0; s < 12; ++s) {
        L->seg_start[s] = off;
        L->seg_n[s] = s < num_segs ? seg_n[s] : 8;
        if (s < num_segs) {
            if (seg_n[s] % 8) return -2;
            off += seg_n[s] * slots;
        }
    }
    L->seg_start[12] = off;
    return 0;
}

int lah_pull_shadow(const int* shadow_info, int S_max, int E_loc, long long p_off, long long pbf16_off, int num_segs,
                    const long long* seg_n, int small_mask, cudaStream_t st) {
    if (!g_peers_set) return -10;
    if (S_max <= 0) return 0;
    PullArgs a;
    a.shadow_info = shadow_info; a.E_loc = E_loc; a.p_off = p_off; a.pbf16_off = pbf16_off; a.small_mask = small_mask;
    if (make_seg_layout(&a.L, num_segs, seg_n, E_loc + S_max)) return -2;
    pull_shadow_kernel<<<dim3(64, S_max), 256, 0, st>>>(g_peers, a);
    return -(int)cudaGetLastError();
}

int lah_zero_slots(float* g, int num_segs, const long long* seg_n, int slots, int first_slot, int num_slots, int seg_mask,
                   cudaStream_t st) {
    if (num_slots <= 0) return 0;
    SegLayout L;
    if (make_seg_layout(&L, num_segs, seg_n, slots)) return -2;
    zero_slots_kernel<<<dim3(8, num_segs), 256, 0, st>>>(g, L, first_slot, num_slots, seg_mask);
    return -(int)cudaGetLastError();
}

}  // extern "C"
