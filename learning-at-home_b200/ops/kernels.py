"""
Python entry points for the non-GEMM sm_90a kernels (csrc/layernorm.cu, csrc/moe.cu, csrc/adam.cu) and their PyTorch
oracles.  All wrappers launch on the current CUDA stream, never synchronise, and are CUDA-graph capturable.
"""
import ctypes

import torch
import torch.nn.functional as F

from . import native
from .native import c_void_p, c_int, c_ll, c_float, ptr, stream_ptr

c_ull = ctypes.c_ulonglong
_configured = False

SLOT_COUNTS, SLOT_DISPATCH, SLOT_OUTPUT, SLOT_GRAD, SLOT_DINPUT, SLOT_TRAINER, SLOT_BARRIER, SLOT_SHADOW = range(8)
NUM_SLOTS = 8
MAX_WORLD = 8
STATUS_TIMEOUT, STATUS_OVERFLOW = 1, 2


def _lib():
    global _configured
    lib = native.cuda_lib()
    if _configured:
        return lib
    P, I, L, Fl = c_void_p, c_int, c_ll, c_float
    sigs = {
        "lah_ln_relu_fwd": [P, P, P, P, P, P, P, I, I, I, P],
        "lah_ln_relu_fwd_t": [P, P, P, P, P, P, P, I, I, I, I, P],
        "lah_ln_relu_bwd_t": [P, P, P, P, P, P, P, P, P, P, P, P, I, I, I, I, P],
        "lah_grouped_colsum_t": [P, L, P, P, I, P, I, I, P],
        "lah_set_step_counters": [P],
        "lah_set_multicast": [c_ull],
        "lah_set_poison_word": [P],
        "lah_nvls_allreduce": [L, L, Fl, P],
        "lah_heartbeat": [L, I, I, L, P],
        "lah_alive_from_heartbeats": [P, P, I, L, L, P],
        "lah_set_spin_timeout_ms": [I],
        "lah_step_begin": [I, L, P],
        "lah_swapab_linear": [P, L, I, P, I, I, I, I, P, L, P, P, P, P, L, P, I, I, P, P, I, P],
        "lah_wgrad_adam": [P, L, P, L, I, I, I, I, P, P, P, P, P, P, P, P, P, Fl, Fl, Fl, Fl, I, I, P],
        "lah_ln_relu_fwd_q": [P, P, P, P, P, P, P, I, I, I, P, P, P],
        "lah_ln_relu_bwd": [P, P, P, P, P, P, P, P, P, P, P, P, I, I, I, P],
        "lah_grouped_colsum": [P, L, P, P, I, P, I, P],
        "lah_set_peers": [P, I, I],
        "lah_set_wait_counter": [P],
        "lah_gate_topk": [P, I, P, I, I, P, Fl, c_ull, L, P, P, P, P, P],
        "lah_layout_exchange": [L, L, I, I, I, I, I, I, I, P, P, P, P, P, P, P, I, Fl, I, P, P, P, P, P],
        "lah_scatter_rows": [P, P, P, P, P, P, L, L, I, I, I, I, I, I, I, I, P, P, P, P, P, I, P],
        "lah_pull_shadow": [P, I, I, L, L, I, P, I, P],
        "lah_zero_slots": [P, I, P, I, I, I, I, P],
        "lah_signal_wait": [L, I, I, I, I, P, P],
        "lah_combine_rows": [L, P, P, P, P, I, I, I, I, L, I, I, I, I, P, P, P],
        "lah_gate_bwd": [L, P, P, P, P, P, I, I, I, I, P, I, P, P],
        "lah_adam_step": [P, P, P, P, P, P, I, P, I, P, P, I, Fl, Fl, Fl, Fl, Fl, I, I, I, L, P, Fl, I, P, L, I, I, I, P],
        "lah_bump_steps": [P, P, I, P],
        "lah_cast_bf16": [P, P, L, P],
        "lah_attention_fwd": [P, P, P, I, I, I, P],
        "lah_attention_bwd": [P, P, P, P, P, P, P, I, I, I, P],
        "lah_symm_alloc": [c_ull, ctypes.POINTER(c_void_p)],
        "lah_symm_free": [P],
        "lah_symm_get_handle": [P, ctypes.c_char_p],
        "lah_symm_open_handle": [ctypes.c_char_p, ctypes.POINTER(c_void_p)],
        "lah_symm_close_handle": [P],
        "lah_device_sync": [],
    }
    for name, argtypes in sigs.items():
        fn = getattr(lib, name)
        fn.restype = c_int
        fn.argtypes = argtypes
    _configured = True
    return lib


def _grid_array(grid_size):
    return (c_int * len(grid_size))(*[int(g) for g in grid_size])


# ---------------------------------------------------------------------------------------------------------
# LayerNorm + ReLU over expert-grouped rows
# ---------------------------------------------------------------------------------------------------------
def ln_relu_fwd(h, gamma, beta, tile_group, *, out, mean, rstd, relu=True, quant=None, tile_rows=128):
    """:param quant: optional ops.fp8.MXFP8Tensor that additionally receives the output as an MXFP8 GEMM operand
    (``out`` may then be None: forward-only runs do not need the bf16 copy)"""
    rows, C = h.shape
    assert h.is_contiguous() and gamma.dtype == torch.float32 and (out is None or out.is_contiguous())
    if quant is not None:
        assert quant.K == C and quant.groups == 1 and quant.rows_per_group >= rows and quant.tile_rows == 128
        native.check(_lib().lah_ln_relu_fwd_q(ptr(h), ptr(out), ptr(mean), ptr(rstd), ptr(gamma), ptr(beta),
                                              ptr(tile_group), rows, C, int(relu), ptr(quant.q), ptr(quant.sf),
                                              stream_ptr()), "lah_ln_relu_fwd_q")
    else:
        native.check(_lib().lah_ln_relu_fwd_t(ptr(h), ptr(out), ptr(mean), ptr(rstd), ptr(gamma), ptr(beta),
                                              ptr(tile_group), rows, C, int(relu), int(tile_rows), stream_ptr()),
                     "lah_ln_relu_fwd")
    native.count_launch()
    return out


def ln_relu_bwd(da, h, mean, rstd, gamma, beta, tile_group, *, dh, dgamma, dbeta, dbias, relu=True, tile_rows=128):
    """dgamma / dbeta / dbias (+)= the column sums of every group's rows, summed in a fixed order (run-to-run identical)"""
    rows, C = h.shape
    assert da.is_contiguous() and h.is_contiguous() and dh.is_contiguous()
    part = torch.empty((rows + tile_rows - 1) // tile_rows, 3, C, device=h.device, dtype=torch.float32)
    native.check(_lib().lah_ln_relu_bwd_t(ptr(da), ptr(h), ptr(mean), ptr(rstd), ptr(gamma), ptr(beta), ptr(dh),
                                          ptr(dgamma), ptr(dbeta), ptr(dbias), ptr(part), ptr(tile_group), rows, C,
                                          int(relu), int(tile_rows), stream_ptr()), "lah_ln_relu_bwd")
    native.count_launch(2)
    return dh


def grouped_colsum(x, tile_group, *, out, tile_rows=128):
    """out[g] += the column sums of group g's rows, summed in a fixed order (run-to-run identical)"""
    rows, C = x.shape
    part = torch.empty((rows + tile_rows - 1) // tile_rows, C, device=x.device, dtype=torch.float32)
    native.check(_lib().lah_grouped_colsum_t(ptr(x), x.stride(0), ptr(out), ptr(part), C, ptr(tile_group), rows,
                                             int(tile_rows), stream_ptr()), "lah_grouped_colsum")
    native.count_launch(2)
    return out


# ---------------------------------------------------------------------------------------------------------
# routing / P2P all-to-all
# ---------------------------------------------------------------------------------------------------------
def set_peers(bases, me):
    arr = (c_ull * len(bases))(*[int(b) for b in bases])
    native.check(_lib().lah_set_peers(ctypes.cast(arr, c_void_p), len(bases), me), "lah_set_peers")


def set_wait_counter(counter):
    """int64 device tensor [1] accumulating the ns this rank spends blocked on peer flags (None disables)"""
    native.check(_lib().lah_set_wait_counter(ptr(counter)), "lah_set_wait_counter")


def set_multicast(mc_base):
    """multicast (NVLS) alias of the symmetric heap, 0 = none; enables the multimem.* paths of csrc/moe.cu"""
    native.check(_lib().lah_set_multicast(int(mc_base)), "lah_set_multicast")


def nvls_allreduce(off, n, scale=1.0):
    """in-place one-shot NVLS all-reduce of the fp32 buffer at symmetric-heap offset ``off`` (multimem.ld_reduce + multimem.st);
    bracket with flag barriers"""
    native.check(_lib().lah_nvls_allreduce(int(off), int(n), float(scale), stream_ptr()), "lah_nvls_allreduce")
    native.count_launch()


def heartbeat(hb_off, first, count, now_ms):
    """stamp the heartbeat of experts [first, first+count) into EVERY rank's table (multimem.st / P2P stores)"""
    native.check(_lib().lah_heartbeat(int(hb_off), int(first), int(count), int(now_ms), stream_ptr()), "lah_heartbeat")
    native.count_launch()


def alive_from_heartbeats(hb, alive, now_ms, max_age_ms):
    native.check(_lib().lah_alive_from_heartbeats(ptr(hb), ptr(alive), alive.numel(), int(now_ms), int(max_age_ms),
                                                  stream_ptr()), "lah_alive_from_heartbeats")
    native.count_launch()


def set_poison_word(status):
    """int32 status tensor whose bit 0 (STATUS_TIMEOUT) disables every optimizer kernel of the step (None: never)"""
    native.check(_lib().lah_set_poison_word(ptr(status)), "lah_set_poison_word")


def set_step_counters(ctr):
    """int32 device tensor [4]: [0] epoch base added to every step-relative epoch, [2:4] int64 token base of the gate's
    failure-injection stream (None disables).  Nothing that changes from step to step is then a kernel ARGUMENT, so a
    whole training step can be captured in a CUDA graph and replayed."""
    native.check(_lib().lah_set_step_counters(ptr(ctr)), "lah_set_step_counters")


def step_begin(epoch_delta, token_delta=0):
    native.check(_lib().lah_step_begin(int(epoch_delta), int(token_delta), stream_ptr()), "lah_step_begin")
    native.count_launch()


def set_spin_timeout_ms(ms):
    """timeout of every peer-flag wait (0 = ~10 s); on expiry the waiter raises STATUS_TIMEOUT and CONTINUES"""
    native.check(_lib().lah_set_spin_timeout_ms(int(ms)), "lah_set_spin_timeout_ms")


def gate_topk(logits, grid_size, k, *, alive=None, failure_rate=0.0, seed=0, token_offset=0, idx, w, pos, counts):
    B = logits.shape[0]
    assert logits.dtype == torch.float32 and logits.is_contiguous() and logits.shape[1] == sum(grid_size)
    native.check(_lib().lah_gate_topk(ptr(logits), B, ctypes.cast(_grid_array(grid_size), c_void_p), len(grid_size), k,
                                      ptr(alive), float(failure_rate), int(seed) & (2 ** 64 - 1), int(token_offset),
                                      ptr(idx), ptr(w), ptr(pos), ptr(counts), stream_ptr()), "lah_gate_topk")
    native.count_launch(2)


def layout_exchange(cnt_all_off, flags_off, slot, epoch, E, E_loc, max_rows, *, align=128, tile_rows=None, counts, dst_row, group_off, group_rows,
                    tile_group, total_rows, status, shadow_slots=0, shadow_tol=1.1, min_shadow_rows=512, route_owner=None,
                    step_rows=None, shadow_info=None, owned_shadow=None):
    """count exchange + global layout; with ``shadow_slots`` > 0 also the hot-expert shadow selection (csrc/moe.cu)"""
    native.check(_lib().lah_layout_exchange(cnt_all_off, flags_off, slot, epoch, E, E_loc, max_rows, align,
                                            int(tile_rows or min(align, 128)), ptr(counts),
                                            ptr(dst_row), ptr(group_off), ptr(group_rows), ptr(tile_group),
                                            ptr(total_rows), ptr(status), int(shadow_slots), float(shadow_tol),
                                            int(min_shadow_rows), ptr(route_owner), ptr(step_rows), ptr(shadow_info),
                                            ptr(owned_shadow), stream_ptr()), "lah_layout_exchange")
    native.count_launch()


def pull_shadow(shadow_info, shadow_slots, E_loc, p_off, pbf16_off, seg_sizes, small_mask):
    """replicate the parameters of the shadowed experts from their owners into my shadow slots (P2P loads)"""
    segs = (c_ll * len(seg_sizes))(*[int(s) for s in seg_sizes])
    native.check(_lib().lah_pull_shadow(ptr(shadow_info), int(shadow_slots), E_loc, p_off, pbf16_off, len(seg_sizes),
                                        ctypes.cast(segs, c_void_p), int(small_mask), stream_ptr()), "lah_pull_shadow")
    native.count_launch()


def zero_slots(g, seg_sizes, slots, first_slot, num_slots, seg_mask):
    segs = (c_ll * len(seg_sizes))(*[int(s) for s in seg_sizes])
    native.check(_lib().lah_zero_slots(ptr(g), len(seg_sizes), ctypes.cast(segs, c_void_p), slots, first_slot, num_slots,
                                       int(seg_mask), stream_ptr()), "lah_zero_slots")
    native.count_launch()


def scatter_rows(src, scale, idx, pos, dst_row, pair_row, dst_off, flags_off, slot, epoch, k, E_loc, max_rows,
                 group_off, group_rows, done_counter, status, align=128, route_owner=None, num_groups=0):
    num_pairs = idx.numel()
    H = src.shape[1]
    assert src.is_contiguous() and src.dtype == torch.bfloat16
    native.check(_lib().lah_scatter_rows(ptr(src), ptr(scale), ptr(idx), ptr(pos), ptr(dst_row), ptr(pair_row), dst_off,
                                         flags_off, slot, epoch, num_pairs, k, H, E_loc, max_rows, align, ptr(group_off),
                                         ptr(group_rows), ptr(done_counter), ptr(status), ptr(route_owner),
                                         int(num_groups), stream_ptr()),
                 "lah_scatter_rows")
    native.count_launch()


def signal_wait(flags_off, slot, epoch, status, *, signal=True, wait=True):
    native.check(_lib().lah_signal_wait(flags_off, slot, epoch, int(signal), int(wait), ptr(status), stream_ptr()),
                 "lah_signal_wait")
    native.count_launch()


def combine_rows(src_off, idx, pair_row, w, out, k, E_loc, *, flags_off=0, slot=0, epoch=0, signal=False, wait=False,
                 status=None, route_owner=None):
    """weighted P2P gather; with signal/wait the kernel itself publishes 'my expert outputs are ready' to every peer
    and waits for all peers' flags before pulling their rows (no separate flag kernels)"""
    B, H = out.shape
    native.check(_lib().lah_combine_rows(src_off, ptr(idx), ptr(pair_row), ptr(w), ptr(out), B, k, H, E_loc, flags_off,
                                         slot, epoch, int(signal), int(wait), ptr(status), ptr(route_owner),
                                         stream_ptr()),
                 "lah_combine_rows")
    native.count_launch()
    return out


def gate_bwd(yo_off, grad, idx, pair_row, w, dlogits, k, E_loc, grid_size, route_owner=None):
    B, H = grad.shape
    assert grad.is_contiguous() and grad.dtype == torch.bfloat16 and dlogits.dtype == torch.float32
    native.check(_lib().lah_gate_bwd(yo_off, ptr(grad), ptr(idx), ptr(pair_row), ptr(w), ptr(dlogits), B, k, H, E_loc,
                                     ctypes.cast(_grid_array(grid_size), c_void_p), len(grid_size), ptr(route_owner),
                                     stream_ptr()),
                 "lah_gate_bwd")
    native.count_launch()
    return dlogits


# ---------------------------------------------------------------------------------------------------------
# attention (transformer expert)
# ---------------------------------------------------------------------------------------------------------
def attention_fwd(qkv, num_heads, *, out=None, lse=None):
    """
    Self-attention over 512-token sequences on wgmma (csrc/attention.cu).
    :param qkv: [batch*512, 3*d_model] bf16 = in_proj output, [q | k | v] per token; head_dim must be 64
    :param lse: optional fp32 [batch*512, num_heads]: receives the base-2 row log-sum-exp (needed by attention_bwd)
    :returns: [batch*512, d_model] bf16, heads concatenated (input of out_proj)
    """
    tokens, three_d = qkv.shape
    d_model = three_d // 3
    assert qkv.is_cuda and qkv.dtype == torch.bfloat16 and qkv.is_contiguous() and tokens % 512 == 0
    if out is None:
        out = torch.empty(tokens, d_model, dtype=torch.bfloat16, device=qkv.device)
    if lse is not None:
        assert lse.dtype == torch.float32 and lse.is_contiguous() and lse.numel() == tokens * num_heads
    native.check(_lib().lah_attention_fwd(ptr(qkv), ptr(out), ptr(lse), tokens // 512, num_heads, d_model, stream_ptr()),
                 "lah_attention_fwd")
    native.count_launch()
    return out


def attention_bwd(qkv, out, dout, lse, num_heads):
    """
    Backward of ``attention_fwd`` on wgmma (csrc/attention_bwd.cu): recomputes P from the saved log-sum-exp, forms dV / dK /
    dQ on tensor cores (nothing of size S x S touches HBM).  Returns dqkv [tokens, 3*d_model] bf16.
    """
    tokens, three_d = qkv.shape
    d_model = three_d // 3
    assert dout.dtype == torch.bfloat16 and dout.is_contiguous() and out.is_contiguous() and lse.dtype == torch.float32
    assert out.dtype == torch.bfloat16 and qkv.is_contiguous()
    delta = torch.empty(tokens, num_heads, dtype=torch.float32, device=qkv.device)      # rowsum(dout o out), filled by the prologue kernel
    dqkv = torch.empty_like(qkv)
    dq_part = torch.empty(4, tokens, d_model, dtype=torch.bfloat16, device=qkv.device)  # one partial per 128-key block
    native.check(_lib().lah_attention_bwd(ptr(qkv), ptr(out), ptr(dout), ptr(lse), ptr(delta), ptr(dqkv), ptr(dq_part),
                                          tokens // 512, num_heads, d_model, stream_ptr()), "lah_attention_bwd")
    native.count_launch(3)   # delta prologue, wgmma backward, dQ partial reduction
    return dqkv


def attention_ref(qkv, num_heads, seq_len=512):
    """fp32 oracle: softmax(q k^T / sqrt(d)) v per head"""
    tokens, three_d = qkv.shape
    d = three_d // 3
    q, k, v = qkv.float().view(tokens // seq_len, seq_len, 3, num_heads, d // num_heads).unbind(2)
    q, k, v = (t.transpose(1, 2) for t in (q, k, v))  # [B, H, S, hd]
    att = torch.softmax(q @ k.transpose(-1, -2) / (d // num_heads) ** 0.5, dim=-1) @ v
    return att.transpose(1, 2).reshape(tokens, d)


# ---------------------------------------------------------------------------------------------------------
# optimizer
# ---------------------------------------------------------------------------------------------------------
def adam_step(p, g, m, v, vmax, p_bf16, seg_sizes, G, *, step=None, group_rows=None, step_scalar=0, lr=1e-3,
              betas=(0.9, 0.999), eps=1e-8, weight_decay=0.0, amsgrad=True, zero_mask=0, world=1,
              peer_grad_off=-1, peer_bases=None, grad_scale=1.0, G_active=0, shadow_of=None, shadow_g_off=-1, me=0,
              seg_mask=0, dead_mask=0):
    arr = None
    if peer_bases is not None:
        arr = (c_ull * len(peer_bases))(*[int(b) for b in peer_bases])
    """
    One fused Adam/AMSGrad step over a flat fp32 buffer laid out as consecutive segments [G, seg_sizes[s]].
    :param step: int32 [G] per-group step counts (already incremented) or None -> step_scalar for everything
    :param group_rows: int32 [G]; groups with 0 rows are skipped (experts that received no tokens are not stepped)
    :param G_active: only the first G_active of the G slots per segment are updated (the rest are shadow replicas)
    :param shadow_of: int32 [G_active, 2] (slot, rank mask): gradient of a shadowed expert = sum of the partial
        gradients in shadow slot ``slot`` of the ranks in ``mask`` (buffers at symmetric offset ``shadow_g_off``)
    """
    if isinstance(seg_sizes, int):
        seg_sizes = [seg_sizes]
    segs = (c_ll * len(seg_sizes))(*[int(s) for s in seg_sizes])
    native.check(_lib().lah_adam_step(ptr(p), ptr(g), ptr(m), ptr(v), ptr(vmax), ptr(p_bf16), len(seg_sizes),
                                      ctypes.cast(segs, c_void_p), G, ptr(step),
                                      ptr(group_rows), int(step_scalar), lr, betas[0], betas[1], eps, weight_decay,
                                      int(amsgrad), int(zero_mask), world, peer_grad_off,
                                      ctypes.cast(arr, c_void_p) if arr is not None else c_void_p(0), grad_scale,
                                      int(G_active), ptr(shadow_of), int(shadow_g_off), int(me), int(seg_mask),
                                      int(dead_mask), stream_ptr()), "lah_adam_step")
    native.count_launch()


def swapab_linear(x, w, group_off, group_rows, *, out, bias=None, residual=None, w_is_kn=False, wait=None, max_ctas=0):
    """
    Small-M grouped linear on swap-AB wgmma tiles (csrc/small_m.cu): for the rows [group_off[g], +group_rows[g]) of every
    group, out = x @ W[g]^T (+bias[g]) (+residual)   (w_is_kn: out = x @ W[g], the dgrad of a Linear whose weight is W).
    Weights are streamed exactly once per 128 tokens; a group of r rows costs MMAs of N = ceil16(r).
    :param x: [rows, K] bf16;  w: [G, M_out, K] (or [G, K, M_out] with w_is_kn) bf16;  out: [rows, M_out] bf16
    """
    assert x.dtype == torch.bfloat16 and w.dtype == torch.bfloat16 and out.dtype == torch.bfloat16 and w.is_contiguous()
    rows, K = x.shape
    G = w.shape[0]
    M_out = w.shape[2] if w_is_kn else w.shape[1]
    assert (w.shape[1] if w_is_kn else w.shape[2]) == K and x.stride(1) == 1 and out.stride(1) == 1
    wait_flags, wait_count, wait_epoch, wait_status = (wait[0], wait[0].numel(), wait[1], wait[2]) if wait else (None, 0, 0, None)
    native.check(_lib().lah_swapab_linear(ptr(x), x.stride(0), rows, ptr(w), G, M_out, K, int(w_is_kn), ptr(out),
                                          out.stride(0), ptr(group_off), ptr(group_rows), ptr(bias), ptr(residual),
                                          residual.stride(0) if residual is not None else 0, ptr(wait_flags), wait_count,
                                          wait_epoch, c_void_p(0), ptr(wait_status), int(max_ctas), stream_ptr()),
                 "lah_swapab_linear")
    native.count_launch()
    return out


def swapab_linear_ref(x, w, group_off, group_rows, *, bias=None, residual=None, w_is_kn=False):
    off, rows = group_off.tolist(), group_rows.tolist()
    M_out = w.shape[2] if w_is_kn else w.shape[1]
    out = torch.zeros(x.shape[0], M_out, dtype=torch.float32, device=x.device)
    for g, (o, r) in enumerate(zip(off, rows)):
        if r <= 0:
            continue
        wg = w[g].float()
        y = x[o:o + r].float() @ (wg if w_is_kn else wg.t())
        if bias is not None:
            y = y + bias.view(w.shape[0], M_out)[g]
        if residual is not None:
            y = y + residual[o:o + r].float()
        out[o:o + r] = y
    return out


def wgrad_adam(dy, x, group_off, group_rows, *, p, m, v, vmax, p_bf16, step, skip=None, lr=1e-3, betas=(0.9, 0.999),
               eps=1e-8, amsgrad=True, max_ctas=0):
    """
    Fused weight gradient + per-expert AMSGrad (csrc/small_m.cu): for every group g with rows > 0,
    dW[g] = dy_g^T x_g is formed in registers and applied to p / m / v / vmax ([G, N, K] fp32) and the bf16 mirror in the same
    kernel; the gradient never reaches HBM.  ``step`` holds the per-expert step counts AFTER this update.
    """
    G, N, Kd = p.shape
    assert dy.shape[1] == N and x.shape[1] == Kd and dy.shape[0] == x.shape[0] and p.is_contiguous()
    assert dy.dtype == torch.bfloat16 and x.dtype == torch.bfloat16 and p.dtype == torch.float32
    native.check(_lib().lah_wgrad_adam(ptr(dy), dy.stride(0), ptr(x), x.stride(0), dy.shape[0], G, N, Kd, ptr(group_off),
                                       ptr(group_rows), ptr(skip), ptr(step), ptr(p), ptr(m), ptr(v), ptr(vmax),
                                       ptr(p_bf16), lr, betas[0], betas[1], eps, int(amsgrad), int(max_ctas),
                                       stream_ptr()), "lah_wgrad_adam")
    native.count_launch()


def bump_steps(step, group_rows):
    native.check(_lib().lah_bump_steps(ptr(step), ptr(group_rows), step.numel(), stream_ptr()), "lah_bump_steps")
    native.count_launch()


def cast_bf16(src, dst):
    assert src.dtype == torch.float32 and dst.dtype == torch.bfloat16 and src.numel() == dst.numel()
    native.check(_lib().lah_cast_bf16(ptr(src), ptr(dst), src.numel(), stream_ptr()), "lah_cast_bf16")
    native.count_launch()


# ---------------------------------------------------------------------------------------------------------
# PyTorch oracles
# ---------------------------------------------------------------------------------------------------------
def product_key_scores(logits, grid_size):
    """[B, sum(grid)] grid logits -> [B, prod(grid)] expert scores (expert id = row-major index over the grid)."""
    parts = torch.split(logits, list(grid_size), dim=-1)
    scores = parts[0]
    for part in parts[1:]:
        scores = (scores.unsqueeze(-1) + part.unsqueeze(-2)).flatten(-2)
    return scores


def gate_topk_ref(logits, grid_size, k, alive=None, fail_mask=None):
    """returns idx [B,k] (-1 for missing), weights [B,k] (softmax over alive selected)"""
    scores = product_key_scores(logits.float(), grid_size)
    dead = torch.zeros_like(scores, dtype=torch.bool)
    if alive is not None:
        dead |= ~alive.bool().view(1, -1)
    if fail_mask is not None:
        dead |= fail_mask
    scores = scores.masked_fill(dead, float("-inf"))
    top_v, top_i = torch.topk(scores, k, dim=-1)
    valid = torch.isfinite(top_v)
    w = torch.softmax(top_v.masked_fill(~valid, float("-inf")), dim=-1)
    w = torch.where(valid, w, torch.zeros_like(w)).nan_to_num(0.0)
    return torch.where(valid, top_i, torch.full_like(top_i, -1)), w


def ln_relu_ref(h, gamma, beta, relu=True):
    y = F.layer_norm(h.float(), (h.shape[-1],), gamma.float(), beta.float(), 1e-5)
    return F.relu(y) if relu else y


@torch.no_grad()
def adam_step_ref(p, g, m, v, vmax, seg_sizes, G, *, step, group_rows=None, lr=1e-3, betas=(0.9, 0.999), eps=1e-8,
                  amsgrad=True, zero_mask=0):
    """PyTorch implementation of csrc/adam.cu (flat segments [G, size]; per-group step; inactive groups skipped)."""
    if isinstance(seg_sizes, int):
        seg_sizes = [seg_sizes]
    off = 0
    active = torch.ones(G, dtype=torch.bool, device=p.device) if group_rows is None else (group_rows > 0)
    idx = active.nonzero().squeeze(1)          # only the active groups are touched (inactive experts are not stepped)
    stepf = step.to(torch.float32).clamp(min=1)[idx]
    bc1 = (1 - betas[0] ** stepf).view(-1, 1)
    bc2 = (1 - betas[1] ** stepf).view(-1, 1)
    for s, size in enumerate(seg_sizes):
        sl = slice(off, off + size * G)
        off += size * G
        if idx.numel() == 0:
            continue
        P, Gr, M, V = p[sl].view(G, size), g[sl].view(G, size), m[sl].view(G, size), v[sl].view(G, size)
        grad = Gr[idx]
        m_new = M[idx] + (1 - betas[0]) * (grad - M[idx])
        v_new = V[idx] * betas[1] + (1 - betas[1]) * grad * grad
        if amsgrad:
            VM = vmax[sl].view(G, size)
            vm_new = torch.maximum(VM[idx], v_new)
            denom = vm_new.sqrt() / bc2.sqrt() + eps
            VM[idx] = vm_new
        else:
            denom = v_new.sqrt() / bc2.sqrt() + eps
        P[idx] = P[idx] - (lr / bc1) * (m_new / denom)
        M[idx] = m_new
        V[idx] = v_new
        if (zero_mask >> s) & 1:
            Gr[idx] = 0.0
