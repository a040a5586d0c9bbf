// adam.cu — fused multi-group Adam / AMSGrad step + bf16 cast (+ gradient zeroing, + optional peer gradient reduce).
//
// Reference semantics: every expert owns a torch.optim.Adam(amsgrad=True) that is stepped right after each backward
// (/root/reference/lib/runtime/expert_backend.py:95-97; Adam(lr=1e-3, amsgrad=True) in the convergence notebooks), i.e.
// the step counter is PER EXPERT and experts that received no tokens are not stepped.  Parameters of the experts hosted
// on a rank are stacked [G, n]; `active[g]`/`step[g]` carry the per-expert state.
//
// One pass over HBM: reads p, g, m, v, vmax (fp32), writes p, m, v, vmax (fp32) + the bf16 copy consumed by the GEMMs,
// and (optionally) zeroes g for the atomically accumulated bias / LayerNorm gradients.
//
// Replicated (trainer-side) parameters: `peer_grad_off >= 0` makes the kernel read the gradient of every rank from the
// symmetric heap (P2P loads over NVLink) and average them before the update, so the data-parallel gradient reduce and
// the optimizer are one kernel; every rank computes the bit-identical sum in the same order.
#include "sm90.cuh"

namespace lah {

struct AdamArgs {
    float* p; float* g; float* m; float* v; float* vmax; bf16* p_bf16;
    // flat layout: segment s holds [G, seg_n[s]] contiguous values starting at seg_start[s]; total = end of last segment
    int num_segs; long long seg_start[13]; long long seg_n[12]; long long total;
    const int* step;      // [G] step count AFTER this update (already incremented); nullptr => use `step_scalar`
    const int* group_rows;  // [G] rows the expert received (0 => skip the group); nullptr => always active
    int step_scalar;
    float lr, beta1, beta2, eps, weight_decay;
    int amsgrad, zero_mask;   // zero_mask bit s => zero the gradient of segment s after use
    // peer reduce
    int world; long long peer_grad_off; char* peer_base[8]; float grad_scale;
    // experts: only the first G_active slots of every segment are owned (the rest are shadow replicas of other ranks'
    // experts).  shadow_of[2g] >= 0: expert g was SHADOWED this step -> its weight gradient is the sum of the partial
    // gradients that the ranks in mask shadow_of[2g+1] left in shadow slot shadow_of[2g] of their (symmetric) gradient
    // buffers (+ my own partial in the owned slot when my bit is set): the data-parallel reduce is fused into the update
    int G_active; const int* shadow_of; long long shadow_g_off; int me;
    // optional restriction to a subset of the segments (seg_mask != 0): the kernel then walks only the concatenation of the
    // selected segments (the fused wgrad+AMSGrad kernel of small_m.cu owns the weight matrices, this one the small vectors)
    int num_ranges; long long r_start[6]; long long r_cum[7];
    int dead_mask;       // ranks excluded from the peer gradient reduce (their buffers hold stale data)
    const int* poison;   // status word: bit 0 set (a peer-flag wait timed out in this step) -> no update from partial data
    // decoupled weight decay (AdamW, Adam(decoupled_weight_decay=True)): p *= decay before the moments, decay = 1 - lr * wd
    // computed in double by the caller and rounded to fp32 once, as torch's scalar multiply does.  Read only by the
    // DECOUPLED instantiation; the other one keeps the L2 form (grad += weight_decay * p)
    float decay;
    // DEV_LR instantiations: {lr, decay} in device memory, written by the host between steps (appended: the fields above
    // keep their offsets)
    const float* lr_dev;
};

// DEV_LR: the learning rate and the decoupled factor come from a.lr_dev = {lr, decay} in device memory instead of a.lr /
// a.decay, so a captured CUDA graph follows a schedule.  Read once per thread; the update expressions are the same, so a
// launch whose block holds x is bit-identical to a by-value launch with x
template <bool DECOUPLED, bool DEV_LR>
__global__ void __launch_bounds__(256) adam_kernel(AdamArgs a) {
    if (a.poison && (*a.poison & 1)) return;
    float dev_lr = 0.f, dev_decay = 1.f;   // the by-value instantiations read a.lr / a.decay where they are used
    if constexpr (DEV_LR) {
        dev_lr = a.lr_dev[0];
        if constexpr (DECOUPLED) dev_decay = a.lr_dev[1];
    }
    const long long stride = static_cast<long long>(gridDim.x) * blockDim.x * 4;
    const long long span = a.num_ranges ? a.r_cum[a.num_ranges] : a.total;
    for (long long j = (static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x) * 4; j < span; j += stride) {
        long long i = j;
        if (a.num_ranges) {
            int r = 0;
#pragma unroll
            for (int t = 1; t < 6; ++t)
                if (t < a.num_ranges && j >= a.r_cum[t]) r = t;
            i = a.r_start[r] + (j - a.r_cum[r]);
        }
        int sg = 0;
#pragma unroll
        for (int t = 1; t < 12; ++t)
            if (t < a.num_segs && i >= a.seg_start[t]) sg = t;
        const int g = static_cast<int>((i - a.seg_start[sg]) / a.seg_n[sg]);
        if (g >= a.G_active) continue;
        if (a.group_rows && a.group_rows[g] <= 0) continue;
        const int step = a.step ? a.step[g] : a.step_scalar;
        const float bc1 = 1.f - powf(a.beta1, static_cast<float>(step));
        const float bc2 = 1.f - powf(a.beta2, static_cast<float>(step));
        const float step_size = (DEV_LR ? dev_lr : a.lr) / bc1;
        const float inv_sqrt_bc2 = rsqrtf(bc2);
        float4 gr;
        if (a.peer_grad_off >= 0) {
            gr = make_float4(0.f, 0.f, 0.f, 0.f);
            for (int r = 0; r < a.world; ++r) {
                if ((a.dead_mask >> r) & 1) continue;
                const float4 t = *reinterpret_cast<const float4*>(
                    reinterpret_cast<const float*>(a.peer_base[r] + a.peer_grad_off) + i);
                gr.x += t.x; gr.y += t.y; gr.z += t.z; gr.w += t.w;
            }
            gr.x *= a.grad_scale; gr.y *= a.grad_scale; gr.z *= a.grad_scale; gr.w *= a.grad_scale;
        } else if (a.shadow_of && a.shadow_of[2 * g] >= 0) {
            const int slot = a.shadow_of[2 * g], mask = a.shadow_of[2 * g + 1];
            gr = ((mask >> a.me) & 1) ? *reinterpret_cast<const float4*>(a.g + i) : make_float4(0.f, 0.f, 0.f, 0.f);
            const long long pi = i + (a.G_active + slot - g) * a.seg_n[sg];
            for (int r = 0; r < a.world; ++r) {
                if (r == a.me || !((mask >> r) & 1)) continue;
                const float4 t = *reinterpret_cast<const float4*>(
                    reinterpret_cast<const float*>(a.peer_base[r] + a.shadow_g_off) + pi);
                gr.x += t.x; gr.y += t.y; gr.z += t.z; gr.w += t.w;
            }
        } else {
            gr = *reinterpret_cast<const float4*>(a.g + i);
        }
        float4 p = *reinterpret_cast<const float4*>(a.p + i);
        float4 m = *reinterpret_cast<const float4*>(a.m + i);
        float4 v = *reinterpret_cast<const float4*>(a.v + i);
        float4 vm = a.amsgrad ? *reinterpret_cast<const float4*>(a.vmax + i) : make_float4(0.f, 0.f, 0.f, 0.f);
        float* pp = &p.x; float* mp = &m.x; float* vp = &v.x; float* vmp = &vm.x; float* gp = &gr.x;
#pragma unroll
        for (int t = 0; t < 4; ++t) {
            float grad = gp[t];
            if constexpr (DECOUPLED) pp[t] = __fmul_rn(pp[t], DEV_LR ? dev_decay : a.decay);   // rounded on its own, as torch's p.mul_()
            else if (a.weight_decay != 0.f) grad += a.weight_decay * pp[t];
            mp[t] = mp[t] + (1.f - a.beta1) * (grad - mp[t]);
            vp[t] = vp[t] * a.beta2 + (1.f - a.beta2) * grad * grad;
            float denom;
            if (a.amsgrad) {
                vmp[t] = fmaxf(vmp[t], vp[t]);
                denom = sqrtf(vmp[t]) * inv_sqrt_bc2 + a.eps;
            } else {
                denom = sqrtf(vp[t]) * inv_sqrt_bc2 + a.eps;
            }
            pp[t] -= step_size * (mp[t] / denom);
        }
        *reinterpret_cast<float4*>(a.p + i) = p;
        *reinterpret_cast<float4*>(a.m + i) = m;
        *reinterpret_cast<float4*>(a.v + i) = v;
        if (a.amsgrad) *reinterpret_cast<float4*>(a.vmax + i) = vm;
        if (a.p_bf16) {
            uint2 q;
            q.x = pack_bf16x2(p.x, p.y);
            q.y = pack_bf16x2(p.z, p.w);
            *reinterpret_cast<uint2*>(a.p_bf16 + i) = q;
        }
        if (((a.zero_mask >> sg) & 1) && a.peer_grad_off < 0)
            *reinterpret_cast<float4*>(a.g + i) = make_float4(0.f, 0.f, 0.f, 0.f);
    }
}

// step[g] += (group_rows[g] > 0)
__global__ void bump_steps_kernel(int* step, const int* group_rows, int G) {
    const int g = blockIdx.x * blockDim.x + threadIdx.x;
    if (g < G && group_rows[g] > 0) step[g] += 1;
}

__global__ void cast_bf16_kernel(const float* __restrict__ src, bf16* __restrict__ dst, long long n) {
    const long long stride = static_cast<long long>(gridDim.x) * blockDim.x * 4;
    for (long long i = (static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x) * 4; i < n; i += stride) {
        const float4 p = *reinterpret_cast<const float4*>(src + i);
        uint2 q;
        q.x = pack_bf16x2(p.x, p.y);
        q.y = pack_bf16x2(p.z, p.w);
        *reinterpret_cast<uint2*>(dst + i) = q;
    }
}

// split master weight (split_decode, sm90.cuh): hi, lo and the tie bits in the sign of v from p
__global__ void split_encode_kernel(const float* __restrict__ p, bf16* __restrict__ hi, uint16_t* __restrict__ lo,
                                    float* __restrict__ v, long long n) {
    const long long stride = static_cast<long long>(gridDim.x) * blockDim.x * 4;
    for (long long i = (static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x) * 4; i < n; i += stride) {
        const float4 w = *reinterpret_cast<const float4*>(p + i);
        float4 s = *reinterpret_cast<const float4*>(v + i);
        uint2 h, l;
        h.x = pack_bf16x2(w.x, w.y);
        h.y = pack_bf16x2(w.z, w.w);
        l.x = (__float_as_uint(w.x) & 0xffffu) | (__float_as_uint(w.y) << 16);
        l.y = (__float_as_uint(w.z) & 0xffffu) | (__float_as_uint(w.w) << 16);
        s.x = with_tie_bit(without_tie_bit(s.x), split_tie_up(w.x));
        s.y = with_tie_bit(without_tie_bit(s.y), split_tie_up(w.y));
        s.z = with_tie_bit(without_tie_bit(s.z), split_tie_up(w.z));
        s.w = with_tie_bit(without_tie_bit(s.w), split_tie_up(w.w));
        *reinterpret_cast<uint2*>(hi + i) = h;
        *reinterpret_cast<uint2*>(lo + i) = l;
        *reinterpret_cast<float4*>(v + i) = s;
    }
}

// p from hi, lo and the tie bits
__global__ void split_decode_kernel(const bf16* __restrict__ hi, const uint16_t* __restrict__ lo,
                                    const float* __restrict__ v, float* __restrict__ p, long long n) {
    const long long stride = static_cast<long long>(gridDim.x) * blockDim.x * 4;
    for (long long i = (static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x) * 4; i < n; i += stride) {
        const uint2 h = *reinterpret_cast<const uint2*>(hi + i);
        const uint2 l = *reinterpret_cast<const uint2*>(lo + i);
        const float4 s = *reinterpret_cast<const float4*>(v + i);
        float4 w;
        w.x = split_decode(h.x & 0xffffu, l.x & 0xffffu, __float_as_uint(s.x) >> 31);
        w.y = split_decode(h.x >> 16, l.x >> 16, __float_as_uint(s.y) >> 31);
        w.z = split_decode(h.y & 0xffffu, l.y & 0xffffu, __float_as_uint(s.z) >> 31);
        w.w = split_decode(h.y >> 16, l.y >> 16, __float_as_uint(s.w) >> 31);
        *reinterpret_cast<float4*>(p + i) = w;
    }
}

}  // namespace lah

using namespace lah;

extern "C" const int* lah_get_poison_word();

extern "C" {

// weight_decay: the L2 coefficient; decay: the decoupled weight-decay factor 1 - lr * wd, read only when `decoupled` is set,
// which selects the DECOUPLED instantiation.  At most one of the two forms per launch.  lr_dev == NULL: lr and decay by
// value; otherwise lr_dev = {lr, 1 - lr * wd} in device memory (the factor computed on the host in double and rounded to
// fp32 once) and the DEV_LR instantiation, which ignores lr and decay, so a captured CUDA graph follows a schedule
int lah_adam_step(float* p, float* g, float* m, float* v, float* vmax, void* p_bf16, int num_segs, const long long* seg_n,
                  int G, const int* step, const int* group_rows, int step_scalar, float lr, const float* lr_dev, float beta1,
                  float beta2, float eps, float weight_decay, int amsgrad, int zero_mask, int world, long long peer_grad_off,
                  const unsigned long long* peer_bases, float grad_scale, int G_active, const int* shadow_of,
                  long long shadow_g_off, int me, int seg_mask, int dead_mask, float decay, int decoupled, cudaStream_t st) {
    if (num_segs < 1 || num_segs > 12) return -2;
    if (decoupled && weight_decay != 0.f) return -2;
    AdamArgs a;
    a.num_segs = num_segs;
    long long off = 0;
    for (int s = 0; s < 12; ++s) {
        a.seg_start[s] = off;
        a.seg_n[s] = s < num_segs ? seg_n[s] : 1;
        if (s < num_segs) {
            if (seg_n[s] % 4) return -2;
            off += seg_n[s] * G;
        }
    }
    a.seg_start[12] = off;
    a.p = p; a.g = g; a.m = m; a.v = v; a.vmax = vmax; a.p_bf16 = (bf16*)p_bf16;
    a.total = off; a.step = step; a.group_rows = group_rows; a.step_scalar = step_scalar; a.lr = lr;
    a.beta1 = beta1; a.beta2 = beta2; a.eps = eps; a.weight_decay = weight_decay; a.amsgrad = amsgrad;
    a.zero_mask = zero_mask; a.world = world; a.peer_grad_off = peer_grad_off; a.grad_scale = grad_scale;
    a.G_active = G_active > 0 ? G_active : G; a.shadow_of = shadow_of; a.shadow_g_off = shadow_g_off; a.me = me;
    for (int i = 0; i < 8; ++i) a.peer_base[i] = (peer_bases && i < world) ? (char*)peer_bases[i] : nullptr;
    a.poison = lah_get_poison_word();
    a.dead_mask = dead_mask;
    a.decay = decay;
    a.lr_dev = lr_dev;
    a.num_ranges = 0;
    a.r_cum[0] = 0;
    if (seg_mask) {   // adjacent selected segments merge into one range
        for (int s = 0; s < num_segs; ++s) {
            if (!((seg_mask >> s) & 1)) continue;
            const long long len = seg_n[s] * G;
            if (a.num_ranges && a.r_start[a.num_ranges - 1] + (a.r_cum[a.num_ranges] - a.r_cum[a.num_ranges - 1]) == a.seg_start[s]) {
                a.r_cum[a.num_ranges] += len;
            } else {
                if (a.num_ranges == 6) return -2;
                a.r_start[a.num_ranges] = a.seg_start[s];
                a.r_cum[a.num_ranges + 1] = a.r_cum[a.num_ranges] + len;
                ++a.num_ranges;
            }
        }
        if (!a.num_ranges) return 0;
    }
    const long long span = a.num_ranges ? a.r_cum[a.num_ranges] : a.total;
    if (span <= 0) return 0;
    long long blocks = (span / 4 + 255) / 256;
    if (blocks > 132 * 16) blocks = 132 * 16;
    if (lr_dev) {
        if (decoupled)
            adam_kernel<true, true><<<(int)blocks, 256, 0, st>>>(a);
        else
            adam_kernel<false, true><<<(int)blocks, 256, 0, st>>>(a);
    } else if (decoupled) {
        adam_kernel<true, false><<<(int)blocks, 256, 0, st>>>(a);
    } else {
        adam_kernel<false, false><<<(int)blocks, 256, 0, st>>>(a);
    }
    return -(int)cudaGetLastError();
}

int lah_bump_steps(int* step, const int* group_rows, int G, cudaStream_t st) {
    bump_steps_kernel<<<(G + 255) / 256, 256, 0, st>>>(step, group_rows, G);
    return -(int)cudaGetLastError();
}

int lah_cast_bf16(const float* src, void* dst, long long n, cudaStream_t st) {
    if (n % 4) return -2;
    if (n <= 0) return 0;
    long long blocks = (n / 4 + 255) / 256;
    if (blocks > 132 * 16) blocks = 132 * 16;
    cast_bf16_kernel<<<(int)blocks, 256, 0, st>>>(src, (bf16*)dst, n);
    return -(int)cudaGetLastError();
}

// split master weight of n values: encode == 1 writes hi, lo and v's tie bits from p; encode == 0 writes p from them
int lah_split_master(float* p, void* hi, void* lo, float* v, long long n, int encode, cudaStream_t st) {
    if (n % 4) return -2;
    if (n <= 0) return 0;
    long long blocks = (n / 4 + 255) / 256;
    if (blocks > 132 * 16) blocks = 132 * 16;
    if (encode)
        split_encode_kernel<<<(int)blocks, 256, 0, st>>>(p, (bf16*)hi, (uint16_t*)lo, v, n);
    else
        split_decode_kernel<<<(int)blocks, 256, 0, st>>>((const bf16*)hi, (const uint16_t*)lo, v, p, n);
    return -(int)cudaGetLastError();
}

}  // extern "C"
