"""
Python entry points for the non-GEMM sm_90a kernels (csrc/layernorm.cu, csrc/moe.cu, csrc/adam.cu) and their PyTorch
oracles.  All wrappers launch on the current CUDA stream, never synchronise, and are CUDA-graph capturable.
"""
import ctypes
import math

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
        "lah_ln_relu_fwd": [P, P, P, P, P, P, P, I, I, I, I, P],
        "lah_ln_relu_bwd": [P, P, P, P, P, P, P, P, P, P, P, P, I, I, I, I, P, P],
        "lah_grouped_colsum": [P, L, P, P, I, P, I, I, P],
        "lah_set_step_counters": [P],
        "lah_set_multicast": [c_ull],
        "lah_set_poison_word": [P],
        "lah_nvls_allreduce": [L, L, Fl, P],
        "lah_heartbeat": [L, I, I, L, P],
        "lah_alive_from_heartbeats": [P, P, I, L, L, P],
        "lah_set_spin_timeout_ms": [I],
        "lah_step_begin": [I, L, P],
        "lah_swapab_linear": [P, L, I, P, I, I, I, I, P, L, P, P, P, P, L, P, I, I, P, I, P],
        "lah_wgrad_adam": [P, L, P, L, I, I, I, I, P, P, P, P, P, P, P, P, P, Fl, P, Fl, Fl, Fl, I, Fl, Fl, I, I, P],
        "lah_wgrad_adam_split": [P, L, P, L, I, I, I, I, P, P, P, P, P, P, P, P, P, Fl, P, Fl, Fl, Fl, I, Fl, Fl, I, I, P],
        "lah_ln_relu_fwd_q": [P, P, P, P, P, P, P, I, I, I, P, P, P],
        "lah_set_peers": [P, I, I],
        "lah_set_wait_counter": [P],
        "lah_gate_topk": [P, I, P, I, I, P, Fl, c_ull, L, P, P, P, P, P, I, Fl, P, I, I, I, P, P],
        "lah_expert_bias_update": [P, I, I, P, Fl, P, P],
        "lah_layout_exchange": [L, L, I, I, I, I, I, I, I, P, P, P, P, P, P, P, I, Fl, I, P, P, P, P, ctypes.c_double, P,
                                P, P],
        "lah_scatter_rows": [P, P, P, P, P, P, L, L, I, I, I, I, I, I, I, I, P, P, P, P, P, I, P, P],
        "lah_pull_shadow": [P, I, I, L, L, I, P, I, P],
        "lah_zero_slots": [P, I, P, I, I, I, I, P],
        "lah_signal_wait": [L, I, I, I, I, P, P],
        "lah_combine_rows": [L, P, P, P, P, I, I, I, I, L, I, I, I, I, P, P, P, P, P, P],
        "lah_gate_bwd": [L, P, P, P, P, P, I, I, I, I, P, I, P, P, Fl, I, P, P, P, P, P],
        "lah_router_loss_fwd": [P, I, P, I, P, P, I, P, P, P, P, P, P, I, P],
        "lah_router_loss_bwd": [P, I, P, I, P, P, P, P, Fl, Fl, P, I, P],
        "lah_adam_step": [P, P, P, P, P, P, I, P, I, P, P, I, Fl, P, Fl, Fl, Fl, Fl, I, I, I, L, P, Fl, I, P, L, I, I, I, Fl,
                          I, P],
        "lah_bump_steps": [P, P, I, P],
        "lah_cast_bf16": [P, P, L, P],
        "lah_split_master": [P, P, P, P, L, I, P],
        "lah_attention_fwd": [P, P, P, L, I, I, I, c_ull, I, Fl, P, P],
        "lah_attention_bwd": [P, P, P, P, P, P, P, L, I, I, I, c_ull, I, Fl, P, P],
        "lah_attention_fwd_causal": [P, P, P, L, I, I, I, c_ull, I, Fl, P],
        "lah_attention_bwd_causal": [P, P, P, P, P, P, P, L, I, I, I, c_ull, I, Fl, P],
        "lah_pack_key_mask": [P, P, L, I, P],
        "lah_dropout_mask": [P, I, I, I, I, I, c_ull, I, P],
        "lah_dropout_ew": [I, P, P, P, L, I, c_ull, I, I, Fl, P],
        "lah_rms_norm_fwd": [P, P, P, P, I, I, Fl, P, I, P],
        "lah_rms_norm_fwd_q": [P, P, P, P, I, I, Fl, P, I, P, P, P],
        "lah_rms_norm_bwd": [P, P, P, P, P, P, P, I, I, I, P, P, P],
        "lah_swiglu_fwd": [P, P, L, I, P],
        "lah_swiglu_fwd_q": [P, P, P, P, L, I, P, P, P],
        "lah_swiglu_bwd": [P, P, P, L, I, P],
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
def _check_ln_width(C, what, max_width=None):
    """the LayerNorm kernels run the widths LN_WIDTHS, the grouped column sum any multiple of LN_WIDTH_STEP
    (csrc/layernorm.cu); the C entry points return -2 for any other"""
    if max_width is None and not ln_width_ok(C):
        raise ValueError(f"{what}: width {C} is not a multiple of {LN_WIDTH_STEP} in [{LN_WIDTH_STEP}, {LN_MAX_WIDTH}]")
    if max_width is not None and (C <= 0 or C % LN_WIDTH_STEP):
        raise ValueError(f"{what}: width {C} is not a positive multiple of {LN_WIDTH_STEP}")


def ln_relu_fwd(h, gamma, beta, tile_group, *, out, mean, rstd, relu=True, quant=None, tile_rows=128):
    """:param quant: optional ops.fp8.MXFP8Tensor that additionally receives the output as an MXFP8 GEMM operand
    (``out`` may then be None: forward-only runs do not need the bf16 copy); the MXFP8 path runs C in 256, 512, 1024,
    2048 and 4096 only"""
    rows, C = h.shape
    _check_ln_width(C, "ln_relu_fwd")
    assert h.is_contiguous() and gamma.dtype == torch.float32 and (out is None or out.is_contiguous())
    if quant is not None:
        assert quant.K == C and quant.groups == 1 and quant.rows_per_group >= rows and quant.tile_rows == 128
        native.check(_lib().lah_ln_relu_fwd_q(ptr(h), ptr(out), ptr(mean), ptr(rstd), ptr(gamma), ptr(beta),
                                              ptr(tile_group), rows, C, int(relu), ptr(quant.q), ptr(quant.sf),
                                              stream_ptr()), "lah_ln_relu_fwd_q")
    else:
        native.check(_lib().lah_ln_relu_fwd(ptr(h), ptr(out), ptr(mean), ptr(rstd), ptr(gamma), ptr(beta),
                                            ptr(tile_group), rows, C, int(relu), int(tile_rows), stream_ptr()),
                     "lah_ln_relu_fwd")
    native.count_launch()
    return out


def ln_relu_bwd(da, h, mean, rstd, gamma, beta, tile_group, *, dh, dgamma, dbeta, dbias, relu=True, tile_rows=128,
                dres=None):
    """dgamma / dbeta / dbias (+)= the column sums of every group's rows, summed in a fixed order (run-to-run identical)
    :param dres: optional bf16 [rows, C] gradient of a residual that bypasses the LayerNorm: dh = dres + LN backward, and
        dbias is the column sum of that total"""
    rows, C = h.shape
    _check_ln_width(C, "ln_relu_bwd")
    assert da.is_contiguous() and h.is_contiguous() and dh.is_contiguous()
    assert dres is None or (dres.shape == h.shape and dres.dtype == torch.bfloat16 and dres.is_contiguous())
    part = torch.empty((rows + tile_rows - 1) // tile_rows, 3, C, device=h.device, dtype=torch.float32)
    native.check(_lib().lah_ln_relu_bwd(ptr(da), ptr(h), ptr(mean), ptr(rstd), ptr(gamma), ptr(beta), ptr(dh),
                                        ptr(dgamma), ptr(dbeta), ptr(dbias), ptr(part), ptr(tile_group), rows, C,
                                        int(relu), int(tile_rows), ptr(dres), stream_ptr()), "lah_ln_relu_bwd")
    native.count_launch(2)
    return dh


def _bf16_rows(t, what, shape):
    if t.dtype != torch.bfloat16 or not t.is_contiguous() or tuple(t.shape) != tuple(shape):
        raise ValueError(f"{what}: expected a contiguous bf16 tensor of shape {tuple(shape)}, got {t.dtype} "
                         f"{tuple(t.shape)}{'' if t.is_contiguous() else ' (not contiguous)'}")


def _f32_vec(t, what, n):
    if t.dtype != torch.float32 or not t.is_contiguous() or t.numel() != n:
        raise ValueError(f"{what}: expected a contiguous float32 tensor of {n} elements, got {t.dtype} {tuple(t.shape)}")


def _check_rms_groups(what, gamma, tile_group, tile_rows, rows, C):
    """gamma of a grouped RMSNorm call: [G, C] with one row per group; tile_group: int32, one entry per tile_rows rows"""
    if tile_rows < 8 or tile_rows & (tile_rows - 1):
        raise ValueError(f"{what}: tile_rows must be a power of two >= 8, got {tile_rows}")
    if tile_group is None:
        return 1
    tiles = (rows + tile_rows - 1) // tile_rows
    if tile_group.dtype != torch.int32 or not tile_group.is_contiguous() or tile_group.numel() < tiles:
        raise ValueError(f"{what}: tile_group must be a contiguous int32 tensor of >= {tiles} entries, got "
                         f"{tile_group.dtype} {tuple(tile_group.shape)}")
    if gamma.numel() % C or gamma.numel() == 0:
        raise ValueError(f"{what}: grouped gamma must be [G, {C}], got {tuple(gamma.shape)}")
    return gamma.numel() // C


def _check_quant_out(what, quant, rows, K_):
    """``quant``: an activation-layout ops.fp8.MXFP8Tensor (one group, 128-row scale tiles) of width K_ and >= rows rows"""
    if quant.K != K_ or quant.groups != 1 or quant.rows_per_group < rows or quant.tile_rows != 128:
        raise ValueError(f"{what}: quant must be an activation MXFP8Tensor of width {K_} with >= {rows} rows, got "
                         f"K={quant.K}, groups={quant.groups}, rows={quant.rows_per_group}, tile_rows={quant.tile_rows}")
    if not quant.q.is_contiguous() or quant.q.data_ptr() % 8:
        raise ValueError(f"{what}: the payload of quant must be contiguous and 8-byte aligned")


def rms_norm_fwd(x, gamma, eps, *, out, rstd, tile_group=None, tile_rows=16, quant=None):
    """RMSNorm over the rows of x (csrc/layernorm.cu): out = bf16(x * rstd * gamma), rstd[r] = 1 / sqrt(mean(x_r^2) + eps)
    kept in fp32.  x, out: bf16 [rows, C] with C in LN_WIDTHS; gamma: fp32 [C]; rstd: fp32 [rows]; eps > 0.
    With ``tile_group`` (int32, the group of every ``tile_rows`` rows, -1 = unused) gamma is fp32 [G, C] and the rows of
    tile t are normalised with gamma[tile_group[t]]; the rows of -1 tiles are left as they were.
    :param quant: optional ops.fp8.MXFP8Tensor (activation layout) that additionally receives the output as an MXFP8 GEMM
        operand, quantised from the fp32 value before its bf16 rounding; ``out`` may then be None.  C a multiple of 256"""
    if x.dim() != 2:
        raise ValueError(f"rms_norm_fwd: x must be [rows, C], got {tuple(x.shape)}")
    rows, C = x.shape
    _check_ln_width(C, "rms_norm_fwd")
    _bf16_rows(x, "rms_norm_fwd x", (rows, C))
    if out is not None or quant is None:
        _bf16_rows(out, "rms_norm_fwd out", (rows, C))
    G = _check_rms_groups("rms_norm_fwd", gamma, tile_group, tile_rows, rows, C)
    _f32_vec(gamma, "rms_norm_fwd gamma", G * C)
    _f32_vec(rstd, "rms_norm_fwd rstd", rows)
    if not eps > 0:
        raise ValueError(f"rms_norm_fwd: eps must be > 0, got {eps}")
    if quant is None:
        native.check(_lib().lah_rms_norm_fwd(ptr(x), ptr(out), ptr(rstd), ptr(gamma), rows, C, float(eps),
                                             ptr(tile_group), int(tile_rows), stream_ptr()), "lah_rms_norm_fwd")
    else:
        if C % 256:
            raise ValueError(f"rms_norm_fwd: the MXFP8 output needs a width that is a multiple of 256, got {C}")
        _check_quant_out("rms_norm_fwd", quant, rows, C)
        native.check(_lib().lah_rms_norm_fwd_q(ptr(x), ptr(out), ptr(rstd), ptr(gamma), rows, C, float(eps),
                                               ptr(tile_group), int(tile_rows), ptr(quant.q), ptr(quant.sf),
                                               stream_ptr()), "lah_rms_norm_fwd_q")
    native.count_launch()
    return out


def rms_norm_bwd(dn, x, rstd, gamma, *, dx, dgamma, dres=None, tile_rows=16, tile_group=None):
    """backward of ``rms_norm_fwd``: dx = dres + rstd (gamma o dn - x mean(gamma o dn o x) rstd^2), rounded once;
    dgamma (+)= the column sums of dn o x rstd, per ``tile_rows`` rows (a power of two >= 8) and then in tile order
    (run-to-run identical).  dres: optional bf16 [rows, C] gradient of a residual that bypasses the norm.
    With ``tile_group`` gamma and dgamma are fp32 [G, C]: tile t uses gamma[g] and adds into dgamma[g], g = tile_group[t];
    -1 tiles are skipped (their rows of dx are not written)"""
    if x.dim() != 2:
        raise ValueError(f"rms_norm_bwd: x must be [rows, C], got {tuple(x.shape)}")
    rows, C = x.shape
    _check_ln_width(C, "rms_norm_bwd")
    for t, what in ((dn, "dn"), (x, "x"), (dx, "dx")) + (((dres, "dres"),) if dres is not None else ()):
        _bf16_rows(t, f"rms_norm_bwd {what}", (rows, C))
    G = _check_rms_groups("rms_norm_bwd", gamma, tile_group, tile_rows, rows, C)
    _f32_vec(gamma, "rms_norm_bwd gamma", G * C)
    _f32_vec(dgamma, "rms_norm_bwd dgamma", G * C)
    _f32_vec(rstd, "rms_norm_bwd rstd", rows)
    part = torch.empty((rows + tile_rows - 1) // tile_rows, C, device=x.device, dtype=torch.float32)
    native.check(_lib().lah_rms_norm_bwd(ptr(dn), ptr(x), ptr(rstd), ptr(gamma), ptr(dx), ptr(dgamma), ptr(part), rows, C,
                                         int(tile_rows), ptr(dres), ptr(tile_group), stream_ptr()), "lah_rms_norm_bwd")
    native.count_launch(2)
    return dx


def _tile_rows_of(tile_group, tile_rows, rows):
    """the group of every row (-1: an unused tile) from the per-tile table"""
    return tile_group.long().repeat_interleave(tile_rows)[:rows]


def rms_norm_grouped_fwd_ref(x, gamma, eps, tile_group, tile_rows):
    """oracle of the grouped ``rms_norm_fwd`` in fp32 (fp64 for a fp64 input): (n, rstd); rows of -1 tiles are 0 in n"""
    xf = x if x.dtype == torch.float64 else x.float()
    g = _tile_rows_of(tile_group.cpu(), tile_rows, x.shape[0]).to(x.device)
    live = (g >= 0)[:, None]
    gam = gamma.reshape(-1, x.shape[1]).to(xf.dtype)[g.clamp(min=0)]
    n, rstd = rms_norm_fwd_ref(xf, torch.ones(x.shape[1], dtype=xf.dtype, device=x.device), eps)
    return torch.where(live, n * gam, torch.zeros_like(n)), rstd


def rms_norm_grouped_bwd_ref(dn, x, gamma, eps, tile_group, tile_rows, dres=None):
    """oracle of the grouped ``rms_norm_bwd`` in fp32 (fp64 for a fp64 input): (dx, dgamma [G, C]); rows of -1 tiles are
    0 in dx and add nothing to dgamma"""
    xf = x if x.dtype == torch.float64 else x.float()
    C = x.shape[1]
    gam = gamma.reshape(-1, C).to(xf.dtype)
    g = _tile_rows_of(tile_group.cpu(), tile_rows, x.shape[0]).to(x.device)
    live = g >= 0
    d = dn.to(xf.dtype) * live[:, None]
    gr = gam[g.clamp(min=0)]
    rstd = torch.rsqrt(xf.pow(2).mean(-1, keepdim=True) + eps)
    dx = rstd * (gr * d - xf * (gr * d * xf).mean(-1, keepdim=True) * rstd * rstd)
    if dres is not None:
        dx = dx + dres.to(xf.dtype)
    dx = dx * live[:, None]
    dgamma = torch.zeros_like(gam).index_add_(0, g[live], (d * xf * rstd)[live])
    return dx, dgamma


def rms_norm_fwd_ref(x, gamma, eps):
    """oracle of ``rms_norm_fwd`` in fp32 (fp64 for a fp64 input): (n, rstd)"""
    xf = x if x.dtype == torch.float64 else x.float()
    rstd = torch.rsqrt(xf.pow(2).mean(-1) + eps)
    return xf * rstd[:, None] * gamma.to(xf.dtype), rstd


def rms_norm_bwd_ref(dn, x, gamma, eps, dres=None):
    """oracle of ``rms_norm_bwd`` in fp32 (fp64 for a fp64 input), closed form: (dx, dgamma)"""
    xf = x if x.dtype == torch.float64 else x.float()
    d, g = dn.to(xf.dtype), gamma.to(xf.dtype)
    rstd = torch.rsqrt(xf.pow(2).mean(-1, keepdim=True) + eps)
    dx = rstd * (g * d - xf * (g * d * xf).mean(-1, keepdim=True) * rstd * rstd)
    if dres is not None:
        dx = dx + dres.to(xf.dtype)
    return dx, (d * xf * rstd).sum(0)


def grouped_colsum(x, tile_group, *, out, tile_rows=128):
    """out[g] += the column sums of group g's rows, summed in a fixed order (run-to-run identical)"""
    rows, C = x.shape
    _check_ln_width(C, "grouped_colsum", max_width=0)
    part = torch.empty((rows + tile_rows - 1) // tile_rows, C, device=x.device, dtype=torch.float32)
    native.check(_lib().lah_grouped_colsum(ptr(x), x.stride(0), ptr(out), ptr(part), C, ptr(tile_group), rows,
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


def _check_expert_bias(what, bias, E, device):
    if bias.dtype != torch.float32 or bias.dim() != 1 or bias.numel() != E or not bias.is_contiguous() \
            or bias.device != device:
        raise ValueError(f"{what}: bias must be a contiguous float32 [{E}] tensor on {device}, got {bias.dtype} "
                         f"{tuple(bias.shape)} on {bias.device}")


ROUTER_SCORES = ("softmax", "sigmoid")   # the weight functions of the gate (DESIGN.md §6c), in csrc score_mode order


def _score_mode(what, score, scale, sig, n, device, norm=True):
    """csrc score_mode of ``score``; checks ``scale`` and the sigma array ``sig`` (float32, >= n entries) before any launch.
    The softmax gate takes a scale other than 1 only with ``norm=False`` (DESIGN.md §6e)"""
    if score not in ROUTER_SCORES:
        raise ValueError(f"{what}: score must be one of {ROUTER_SCORES}, got {score!r}")
    if not isinstance(norm, bool):
        raise ValueError(f"{what}: norm must be a bool, got {norm!r}")
    scale = float(scale)
    if score == "softmax":
        if sig is not None:
            raise ValueError(f"{what}: the softmax gate takes no sig array")
        if norm and scale != 1.0:
            raise ValueError(f"{what}: the normalised softmax gate takes no scale ({scale}); use norm=False")
    if not math.isfinite(scale) or scale <= 0.0:
        raise ValueError(f"{what}: scale must be a finite value > 0, got {scale}")
    if score == "softmax":
        return 0
        raise ValueError(f"{what}: scale must be a finite value > 0, got {scale}")
    if sig is None or sig.dtype != torch.float32 or not sig.is_contiguous() or sig.numel() < n or sig.device != device:
        got = "None" if sig is None else f"{sig.dtype} {tuple(sig.shape)} on {sig.device}"
        raise ValueError(f"{what}: the sigmoid gate needs sig, a contiguous float32 tensor of >= {n} entries on "
                         f"{device}, got {got}")
    return 1


MAX_EXPERT_GROUPS = 64   # csrc MAX_GROUPS: the group mask of group-limited routing is one 64-bit word


def check_expert_groups(what, E, n_group, topk_group, k=None):
    """group-limited routing (DESIGN.md §6d): n_group must be an int in [1, 64] dividing E (and E <= LAYOUT_MAX_E when
    n_group > 1), topk_group an int in [1, n_group]; with ``k``, k <= topk_group * E / n_group (else k pairs never fill)"""
    for name, v in (("n_group", n_group), ("topk_group", topk_group)):
        if not isinstance(v, int) or isinstance(v, bool):
            raise ValueError(f"{what}: {name} must be an int, got {v!r}")
    if not 1 <= n_group <= MAX_EXPERT_GROUPS or E % n_group:
        raise ValueError(f"{what}: n_group must be in [1, {MAX_EXPERT_GROUPS}] and divide the {E} experts, got {n_group}")
    if n_group > 1 and E > LAYOUT_MAX_E:
        raise ValueError(f"{what}: group-limited routing scores at most {LAYOUT_MAX_E} experts, got {E}")
    if not 1 <= topk_group <= n_group:
        raise ValueError(f"{what}: topk_group must be in [1, n_group = {n_group}], got {topk_group}")
    if k is not None and k > topk_group * (E // n_group):
        raise ValueError(f"{what}: k = {k} experts cannot come from topk_group = {topk_group} groups of "
                         f"{E // n_group} experts")


def _check_lse(what, lse, n, device, needed):
    """the float32 log-partition array of the unnormalised softmax gate: >= n entries when ``needed``, else None"""
    if not needed:
        if lse is not None:
            raise ValueError(f"{what}: lse belongs to the unnormalised softmax gate (score='softmax', norm=False)")
        return
    if lse is None or lse.dtype != torch.float32 or not lse.is_contiguous() or lse.numel() < n or lse.device != device:
        got = "None" if lse is None else f"{lse.dtype} {tuple(lse.shape)} on {lse.device}"
        raise ValueError(f"{what}: the unnormalised softmax gate needs lse, a contiguous float32 tensor of >= {n} "
                         f"entries on {device}, got {got}")


def gate_topk(logits, grid_size, k, *, alive=None, failure_rate=0.0, seed=0, token_offset=0, idx, w, pos, counts,
              bias=None, score="softmax", scale=1.0, sig=None, n_group=1, topk_group=1, norm=True, lse=None):
    """top-k routing of the grid logits (two launches).  ``bias``: float32 [prod(grid)] added to the selection key only
    (DESIGN.md §6b).  ``score="softmax"``: the weights are the softmax over the unbiased scores of the selected experts.
    ``score="sigmoid"`` (DeepSeek-V3, DESIGN.md §6c): the weights are scale * sigma_j / sum of sigma over the valid selected
    pairs, the bias is added to sigma(s), and sigma_j of every pair goes to ``sig`` (float32 [B * k], 0 for a missing pair).
    ``n_group`` / ``topk_group`` (DeepSeek-V2/V3 group-limited routing, DESIGN.md §6d): the experts form n_group groups of
    consecutive ids and each token picks its k experts from its topk_group best groups only.
    ``norm=False`` (norm_topk_prob=False, DESIGN.md §6e): the weights are not renormalised over the selection.  Softmax:
    scale * p_j with p the softmax over every live expert (failed and unchosen-group experts included), whose
    log-partition z_b goes to ``lse`` (float32 [B]); sigmoid: scale * sigma_j"""
    B = logits.shape[0]
    assert logits.dtype == torch.float32 and logits.is_contiguous() and logits.shape[1] == sum(grid_size)
    if bias is not None:
        _check_expert_bias("gate_topk", bias, math.prod(grid_size), logits.device)
    mode = _score_mode("gate_topk", score, scale, sig, B * k, logits.device, norm)
    _check_lse("gate_topk", lse, B, logits.device, score == "softmax" and not norm)
    check_expert_groups("gate_topk", math.prod(grid_size), n_group, topk_group)
    native.check(_lib().lah_gate_topk(ptr(logits), B, ctypes.cast(_grid_array(grid_size), c_void_p), len(grid_size), k,
                                      ptr(alive), float(failure_rate), int(seed) & (2 ** 64 - 1), int(token_offset),
                                      ptr(idx), ptr(w), ptr(pos), ptr(counts), ptr(bias), mode, float(scale), ptr(sig),
                                      n_group, topk_group, int(norm), ptr(lse), stream_ptr()), "lah_gate_topk")
    native.count_launch(2)


def expert_bias_update(counts, *, alive=None, bias, rate):
    """Auxiliary-loss-free balancing step (one launch): every live expert's ``bias`` moves by ``rate`` toward balance,
    + when N c_e < T, - when N c_e > T (c_e: routed pairs of the int32 [R, E] count table summed over R, T = sum_e c_e,
    N = live experts).  Dead experts and T = 0 change nothing (DESIGN.md §6b)."""
    if counts.dtype != torch.int32 or counts.dim() != 2 or not counts.is_contiguous() \
            or not 1 <= counts.shape[0] <= MAX_WORLD or not 1 <= counts.shape[1] <= LAYOUT_MAX_E:
        raise ValueError(f"expert_bias_update: counts must be a contiguous int32 [R <= {MAX_WORLD}, E <= {LAYOUT_MAX_E}] "
                         f"tensor, got {counts.dtype} {tuple(counts.shape)}")
    E = counts.shape[1]
    _check_expert_bias("expert_bias_update", bias, E, counts.device)
    if alive is not None and (alive.dtype != torch.uint8 or alive.numel() != E or not alive.is_contiguous()):
        raise ValueError(f"expert_bias_update: alive must be a contiguous uint8 tensor of {E} entries, got {alive.dtype} "
                         f"{tuple(alive.shape)}")
    rate = float(rate)
    if not math.isfinite(rate) or rate < 0.0:
        raise ValueError(f"expert_bias_update: rate must be a finite value >= 0, got {rate}")
    native.check(_lib().lah_expert_bias_update(ptr(counts), counts.shape[0], E, ptr(alive), rate, ptr(bias),
                                               stream_ptr()), "lah_expert_bias_update")
    native.count_launch()
    return bias


def layout_exchange(cnt_all_off, flags_off, slot, epoch, E, E_loc, max_rows, *, align=128, tile_rows=None, counts, dst_row, group_off, group_rows,
                    tile_group, total_rows, status, shadow_slots=0, shadow_tol=1.1, min_shadow_rows=512, route_owner=None,
                    step_rows=None, shadow_info=None, owned_shadow=None, capacity_factor=0.0, keep=None,
                    capacity_stats=None):
    """count exchange + global layout; with ``shadow_slots`` > 0 also the hot-expert shadow selection (csrc/moe.cu).
    ``capacity_factor`` > 0 (DESIGN.md §6f): every table follows the kept counts of ``expert_capacity_ref``; ``keep``
    (int32 [E]) receives this rank's kept pairs per expert, ``capacity_stats`` (int32 [2]) C and the box-wide dropped
    pairs.  0 (dropless) takes neither"""
    f = check_capacity_factor("layout_exchange", capacity_factor)
    if (f > 0.0) != (keep is not None and capacity_stats is not None):
        raise ValueError("layout_exchange: keep and capacity_stats go with capacity_factor > 0, and only with it")
    if f > 0.0:
        for name, t, n in (("keep", keep, E), ("capacity_stats", capacity_stats, 2)):
            if t.dtype != torch.int32 or not t.is_contiguous() or t.numel() < n or not t.is_cuda:
                raise ValueError(f"layout_exchange: {name} must be a contiguous CUDA int32 tensor of >= {n} entries")
    native.check(_lib().lah_layout_exchange(cnt_all_off, flags_off, slot, epoch, E, E_loc, max_rows, align,
                                            int(tile_rows or min(align, 128)), ptr(counts),
                                            ptr(dst_row), ptr(group_off), ptr(group_rows), ptr(tile_group),
                                            ptr(total_rows), ptr(status), int(shadow_slots), float(shadow_tol),
                                            int(min_shadow_rows), ptr(route_owner), ptr(step_rows), ptr(shadow_info),
                                            ptr(owned_shadow), f, ptr(keep), ptr(capacity_stats), stream_ptr()),
                 "lah_layout_exchange")
    native.count_launch()


CAPACITY_MAX = 2 ** 31 - 1   # C saturates here (csrc/moe.cu layout_exchange_kernel): no count table holds more pairs


def check_capacity_factor(what, f):
    """the expert capacity factor as a float: finite and >= 0 (0 = dropless)"""
    f = float(f)
    if not math.isfinite(f) or f < 0.0:
        raise ValueError(f"{what}: the expert capacity factor must be a finite value >= 0, got {f}")
    return f


def expert_capacity(factor, routed_pairs, num_experts):
    """C = max(1, ceil((factor * P) / E)) in float64, in this order (DESIGN.md §6f), saturated at CAPACITY_MAX"""
    c = math.ceil((float(factor) * float(routed_pairs)) / float(num_experts))
    return max(1, min(c, CAPACITY_MAX))


def expert_capacity_ref(cnt, factor):
    """the expert capacity of a count table ``cnt`` [world, E] (rank r's routed pairs per expert; rows of excluded ranks
    zero): dict(capacity=C, kept=[world, E] with kept(r, e) = clamp(C - sum_{s<r} cnt(s, e), 0, cnt(r, e)),
    dropped=P - sum(kept)).  Rank r keeps its pairs of expert e with pos < kept(r, e)"""
    cnt = torch.as_tensor(cnt).long().cpu()
    P = int(cnt.sum())
    C = expert_capacity(factor, P, cnt.shape[1])
    before = torch.cumsum(cnt, 0) - cnt
    kept = torch.minimum(torch.clamp(C - before, min=0), cnt)
    return dict(capacity=C, kept=kept, dropped=P - int(kept.sum()))


def capacity_keep_ref(idx, factor, num_experts):
    """world-1 form of ``expert_capacity_ref`` on one batch's expert ids ``idx`` [B, k] (-1: no pair): (kept mask [B, k],
    C, dropped).  A pair is kept when fewer than C earlier pairs (token-major order) chose its expert"""
    flat = idx.reshape(-1).long()
    valid = flat >= 0
    key = torch.where(valid, flat, torch.full_like(flat, num_experts))
    order = torch.sort(key, stable=True).indices
    srt = key[order]
    pos = torch.empty_like(flat)
    pos[order] = torch.arange(flat.numel(), device=flat.device) - torch.searchsorted(srt, srt)
    C = expert_capacity(factor, int(valid.sum()), num_experts)
    kept = valid & (pos < C)
    return kept.view(idx.shape), C, int(valid.sum() - kept.sum())


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
                 group_off, group_rows, done_counter, status, align=128, route_owner=None, num_groups=0, keep=None):
    """P2P dispatch of one row per routed pair.  ``keep`` (forward only: with ``dst_row`` and ``pair_row``): the kept
    pairs per expert of ``layout_exchange(capacity_factor > 0)``; a pair with pos >= keep[e] is dropped (pair_row -1)"""
    num_pairs = idx.numel()
    H = src.shape[1]
    assert src.is_contiguous() and src.dtype == torch.bfloat16
    if keep is not None and (dst_row is None or pair_row is None):
        raise ValueError("scatter_rows: keep drops pairs in the forward dispatch (dst_row and pair_row given) only")
    native.check(_lib().lah_scatter_rows(ptr(src), ptr(scale), ptr(idx), ptr(pos), ptr(dst_row), ptr(pair_row), dst_off,
                                         flags_off, slot, epoch, num_pairs, k, H, E_loc, max_rows, align, ptr(group_off),
                                         ptr(group_rows), ptr(done_counter), ptr(status), ptr(route_owner),
                                         int(num_groups), ptr(keep), stream_ptr()),
                 "lah_scatter_rows")
    native.count_launch()


def signal_wait(flags_off, slot, epoch, status, *, signal=True, wait=True):
    native.check(_lib().lah_signal_wait(flags_off, slot, epoch, int(signal), int(wait), ptr(status), stream_ptr()),
                 "lah_signal_wait")
    native.count_launch()


def combine_rows(src_off, idx, pair_row, w, out, k, E_loc, *, flags_off=0, slot=0, epoch=0, signal=False, wait=False,
                 status=None, route_owner=None, addend=None, pass_self=None, pass_w=None):
    """weighted P2P gather; with signal/wait the kernel itself publishes 'my expert outputs are ready' to every peer
    and waits for all peers' flags before pulling their rows (no separate flag kernels).
    :param addend: optional bf16 [B, H] (contiguous, 16-byte aligned) that starts every row's fp32 accumulator:
        out = bf16(addend + sum_j w_j src_j), rounded once.  None launches the plain kernel
    :param pass_self, pass_w: expert capacity (DESIGN.md §6f): a routed pair without a row (dropped) adds
        pass_w[p] * pass_self[b] instead, with pass_self bf16 [B, H] like the addend and pass_w float32 [B * k]"""
    B, H = out.shape
    if addend is not None:
        _bf16_rows(addend, "combine_rows addend", (B, H))
        if addend.data_ptr() % 16:
            raise ValueError("combine_rows: the addend must be 16-byte aligned")
    if (pass_self is None) != (pass_w is None):
        raise ValueError("combine_rows: pass_self and pass_w go together")
    if pass_self is not None:
        _bf16_rows(pass_self, "combine_rows pass_self", (B, H))
        _f32_vec(pass_w, "combine_rows pass_w", B * k)
        if pass_self.data_ptr() % 16:
            raise ValueError("combine_rows: pass_self must be 16-byte aligned")
    native.check(_lib().lah_combine_rows(src_off, ptr(idx), ptr(pair_row), ptr(w), ptr(out), B, k, H, E_loc, flags_off,
                                         slot, epoch, int(signal), int(wait), ptr(status), ptr(route_owner),
                                         ptr(addend), ptr(pass_self), ptr(pass_w), stream_ptr()),
                 "lah_combine_rows")
    native.count_launch()
    return out


def combine_rows_ref(src, idx, pair_row, w=None, addend=None, pass_self=None, pass_w=None):
    """exact oracle of ``combine_rows`` on one rank's rows: the float64 sum addend[b] + sum_j w[b, j] src[pair_row[b, j]]
    over the pairs with an expert and a row, rounded to bf16 once.  ``src``: [R, H]; idx, pair_row, w: [B, k].  With
    ``pass_self`` [B, H] and ``pass_w`` [B, k], every pair with an expert and no row adds pass_w[b, j] pass_self[b]"""
    present = ((idx >= 0) & (pair_row >= 0)).double()
    if w is not None:
        present = present * w.double()
    terms = src.double()[pair_row.clamp(min=0).long()] * present.unsqueeze(-1)
    total = terms.sum(1)
    if addend is not None:
        total = total + addend.double()
    if pass_self is not None:
        dropped = ((idx >= 0) & (pair_row < 0)).double() * pass_w.double()
        total = total + dropped.sum(1, keepdim=True) * pass_self.double()
    return total.to(torch.bfloat16)


def gate_bwd(yo_off, grad, idx, pair_row, w, dlogits, k, E_loc, grid_size, route_owner=None, *, score="softmax",
             scale=1.0, sig=None, norm=True, lse=None, alive=None, logits=None, pass_x=None):
    """gradient of the grid logits from the combine's (one launch).  ``score="sigmoid"``: the gate's ``sig`` array and
    ``scale`` of the same forward (DESIGN.md §6c).  ``norm=False`` (DESIGN.md §6e): the gate ran with norm=False; the
    softmax gate then also needs the forward's grid ``logits`` (float32 [B, sum(grid)]), its ``lse`` and the ``alive``
    table it routed with, and adds the dense term -p_e sum_j w_j dw_j of every live expert.  ``pass_x`` (expert
    capacity, DESIGN.md §6f): the layer input, bf16 [B, H]; a routed pair without a row then has dw_j = <g_b, x_b>"""
    B, H = grad.shape
    assert grad.is_contiguous() and grad.dtype == torch.bfloat16 and dlogits.dtype == torch.float32
    if pass_x is not None:
        _bf16_rows(pass_x, "gate_bwd pass_x", (B, H))
        if pass_x.data_ptr() % 16:
            raise ValueError("gate_bwd: pass_x must be 16-byte aligned")
    _score_mode("gate_bwd", score, scale, sig, B * k, grad.device, norm)
    dense = score == "softmax" and not norm
    _check_lse("gate_bwd", lse, B, grad.device, dense)
    E = math.prod(grid_size)
    if not dense:
        if logits is not None or alive is not None:
            raise ValueError("gate_bwd: logits and alive belong to the unnormalised softmax gate (norm=False)")
    else:
        if logits is None or logits.dtype != torch.float32 or not logits.is_contiguous() or logits.device != grad.device \
                or tuple(logits.shape) != (B, sum(grid_size)):
            got = "None" if logits is None else f"{logits.dtype} {tuple(logits.shape)} on {logits.device}"
            raise ValueError(f"gate_bwd: the unnormalised softmax gate needs logits, a contiguous float32 "
                             f"[{B}, {sum(grid_size)}] tensor on {grad.device}, got {got}")
        if alive is not None and (alive.dtype != torch.uint8 or alive.numel() != E or not alive.is_contiguous()
                                  or alive.device != grad.device):
            raise ValueError(f"gate_bwd: alive must be a contiguous uint8 tensor of {E} entries on {grad.device}")
        if E > LAYOUT_MAX_E or (len(grid_size) > 1 and sum(grid_size) + E + E // 32 + 1 > GATE_BWD_DENSE_MAX_FLOATS):
            raise ValueError(f"gate_bwd: the unnormalised softmax gate takes at most {LAYOUT_MAX_E} experts (and "
                             f"{GATE_BWD_DENSE_MAX_FLOATS - LAYOUT_MAX_E - LAYOUT_MAX_E // 32 - 1} grid logits on a "
                             f"grid of 2+ dims), got grid {tuple(grid_size)}")
    native.check(_lib().lah_gate_bwd(yo_off, ptr(grad), ptr(idx), ptr(pair_row), ptr(w), ptr(dlogits), B, k, H, E_loc,
                                     ctypes.cast(_grid_array(grid_size), c_void_p), len(grid_size), ptr(route_owner),
                                     ptr(sig), float(scale), int(norm), ptr(lse), ptr(logits), ptr(alive),
                                     ptr(pass_x), stream_ptr()),
                 "lah_gate_bwd")
    native.count_launch()
    return dlogits


# ---------------------------------------------------------------------------------------------------------
# router losses of the product-key gate (load balancing + z-loss; csrc/moe.cu router_*_kernel)
# ---------------------------------------------------------------------------------------------------------
MAX_GRID_DIMS = 4        # csrc/moe.cu MAX_GRID_DIMS
LAYOUT_MAX_E = 4096      # csrc/moe.cu LAYOUT_MAX_E: most experts (and grid logits) of a gate
# csrc GATE_BWD_DENSE_MAX_FLOATS: the shared memory per token of the dense pass of the unnormalised softmax gate_bwd
GATE_BWD_DENSE_MAX_FLOATS = LAYOUT_MAX_E // 2 + 2 + LAYOUT_MAX_E + LAYOUT_MAX_E // 32 + 1
ROUTER_WARPS = 4         # tokens per CTA of the router-loss kernels


def check_router_grid(grid_size):
    """the grids the router-loss kernels take: 1..MAX_GRID_DIMS positive sizes, at most LAYOUT_MAX_E experts and logits"""
    grid = tuple(int(g) for g in grid_size)
    if not 1 <= len(grid) <= MAX_GRID_DIMS or min(grid) < 1 or sum(grid) > LAYOUT_MAX_E or math.prod(grid) > LAYOUT_MAX_E:
        raise ValueError(f"router losses: grid_size must have 1..{MAX_GRID_DIMS} positive sizes with at most "
                         f"{LAYOUT_MAX_E} experts, got {grid_size}")
    return grid


def _router_args(what, logits, grid_size, alive):
    grid = check_router_grid(grid_size)
    if logits.dtype != torch.float32 or logits.dim() != 2 or logits.shape[1] != sum(grid) or not logits.is_contiguous():
        raise ValueError(f"{what}: logits must be a contiguous float32 [B, {sum(grid)}] tensor, got {logits.dtype} "
                         f"{tuple(logits.shape)}")
    E = math.prod(grid)
    if alive is not None and (alive.dtype != torch.uint8 or alive.numel() != E or not alive.is_contiguous()):
        raise ValueError(f"{what}: alive must be a contiguous uint8 tensor of {E} entries, got {alive.dtype} "
                         f"{tuple(alive.shape)}")
    return grid, logits.shape[0], E


def _router_score_mode(what, score):
    if score not in ROUTER_SCORES:
        raise ValueError(f"{what}: score must be one of {ROUTER_SCORES}, got {score!r}")
    return ROUTER_SCORES.index(score)


def router_loss_fwd(logits, grid_size, counts, *, alive=None, f, z, Fb, loss, partials=None, ticket=None,
                    score="softmax"):
    """Router losses of one training forward (two launches).  ``counts``: int32 [R, E] count table (one row per rank,
    R <= MAX_WORLD), summed over its rows.  Writes f (float32 [E + 1]: f_e = c_e / sum c, then N = live experts), z and
    Fb (float32, >= B entries: logsumexp z_b and F_b = sum_e f_e p_{b,e}) and loss (float32 [2]: unweighted L_aux, L_z).
    ``partials`` (float32, >= 2 * ceil(B / ROUTER_WARPS)) and ``ticket`` (int32 [1], zero between calls) are scratch,
    allocated when None.  ``score="sigmoid"`` (DESIGN.md §6c): p_{b,e} = sigma_{b,e} / S'_b over the live experts, z
    holds S'_b and L_z is 0."""
    grid, B, E = _router_args("router_loss_fwd", logits, grid_size, alive)
    mode = _router_score_mode("router_loss_fwd", score)
    if counts.dtype != torch.int32 or counts.dim() != 2 or counts.shape[1] != E or not counts.is_contiguous() \
            or not 1 <= counts.shape[0] <= MAX_WORLD:
        raise ValueError(f"router_loss_fwd: counts must be a contiguous int32 [R <= {MAX_WORLD}, {E}] tensor, got "
                         f"{counts.dtype} {tuple(counts.shape)}")
    nblk = (B + ROUTER_WARPS - 1) // ROUTER_WARPS
    if partials is None:
        partials = torch.empty(max(1, 2 * nblk), dtype=torch.float32, device=logits.device)
    if ticket is None:
        ticket = torch.zeros(1, dtype=torch.int32, device=logits.device)
    _f32_vec(f, "router_loss_fwd: f", E + 1)
    _f32_vec(loss, "router_loss_fwd: loss", 2)
    for t, name, n in ((z, "z", B), (Fb, "Fb", B), (partials, "partials", 2 * nblk)):
        if t.dtype != torch.float32 or not t.is_contiguous() or t.numel() < n:
            raise ValueError(f"router_loss_fwd: {name} must be a contiguous float32 tensor of >= {n} entries, got "
                             f"{t.dtype} {tuple(t.shape)}")
    if ticket.dtype != torch.int32 or ticket.numel() < 1:
        raise ValueError("router_loss_fwd: ticket must be an int32 tensor")
    native.check(_lib().lah_router_loss_fwd(ptr(logits), B, ctypes.cast(_grid_array(grid), c_void_p), len(grid),
                                            ptr(alive), ptr(counts), counts.shape[0], ptr(f), ptr(z), ptr(Fb), ptr(loss),
                                            ptr(partials), ptr(ticket), mode, stream_ptr()), "lah_router_loss_fwd")
    native.count_launch(2 if B > 0 else 1)
    return loss


def router_loss_bwd(logits, grid_size, *, alive=None, f, z, Fb, aux_coef, z_coef, dlogits, score="softmax"):
    """dlogits += the gradient of aux_coef * L_aux + z_coef * L_z w.r.t. the grid logits (f constant), from the f, z and
    Fb the forward wrote for the same logits and score (one launch).  The sigmoid router has no z-loss: z_coef must be 0"""
    grid, B, E = _router_args("router_loss_bwd", logits, grid_size, alive)
    mode = _router_score_mode("router_loss_bwd", score)
    if mode and z_coef != 0.0:
        raise ValueError(f"router_loss_bwd: the sigmoid router has no z-loss; z_coef must be 0, got {z_coef}")
    _f32_vec(f, "router_loss_bwd: f", E + 1)
    for t, name in ((z, "z"), (Fb, "Fb")):
        if t.dtype != torch.float32 or not t.is_contiguous() or t.numel() < B:
            raise ValueError(f"router_loss_bwd: {name} must be a contiguous float32 tensor of >= {B} entries")
    if dlogits.dtype != torch.float32 or tuple(dlogits.shape) != tuple(logits.shape) or not dlogits.is_contiguous():
        raise ValueError(f"router_loss_bwd: dlogits must be a contiguous float32 {tuple(logits.shape)} tensor, got "
                         f"{dlogits.dtype} {tuple(dlogits.shape)}")
    if not (math.isfinite(aux_coef) and math.isfinite(z_coef)):
        raise ValueError("router_loss_bwd: the coefficients must be finite")
    native.check(_lib().lah_router_loss_bwd(ptr(logits), B, ctypes.cast(_grid_array(grid), c_void_p), len(grid),
                                            ptr(alive), ptr(f), ptr(z), ptr(Fb), float(aux_coef), float(z_coef),
                                            ptr(dlogits), mode, stream_ptr()), "lah_router_loss_bwd")
    if B > 0:
        native.count_launch()
    return dlogits


# ---------------------------------------------------------------------------------------------------------
# attention (transformer expert)
# ---------------------------------------------------------------------------------------------------------
MAX_SEQ = 65536   # longest sequence of the attention kernels (csrc/dropout.cuh MAX_SEQ)
HEAD_DIMS = (32, 64, 128)   # head dims d_model / num_heads of the attention kernels (csrc/attention.cu, attention_bwd.cu)
# row widths of the LayerNorm kernels (csrc/layernorm.cu LN_MAX_C): every multiple of LN_WIDTH_STEP up to LN_MAX_WIDTH;
# the grouped column sum runs any multiple of LN_WIDTH_STEP (the in_proj bias gradient sums 3 d_model columns)
LN_WIDTH_STEP = 128
LN_MAX_WIDTH = 4096
LN_WIDTHS = tuple(range(LN_WIDTH_STEP, LN_MAX_WIDTH + 1, LN_WIDTH_STEP))


def ln_width_ok(C) -> bool:
    """True when ``C`` is a width the LayerNorm kernels run (LN_WIDTHS)"""
    return 0 < C <= LN_MAX_WIDTH and C % LN_WIDTH_STEP == 0


def pack_key_mask(pad):
    """
    Packs a key padding mask for ``attention_fwd`` / ``attention_bwd`` (csrc/attention.cu, one launch).
    :param pad: bool [batch, seq_len] CUDA tensor in torch's ``src_key_padding_mask`` convention: True = key ignored
    :returns: int32 [batch, ceil(seq_len / 32)]: bit k % 32 of word k / 32 is set iff key k is valid (not padding); bits of
        keys >= seq_len are clear
    """
    assert pad.is_cuda and pad.dtype == torch.bool and pad.dim() == 2 and pad.is_contiguous(), (pad.dtype, tuple(pad.shape))
    batch, seq_len = pad.shape
    assert 1 <= seq_len <= MAX_SEQ, seq_len
    words = torch.empty(batch, (seq_len + 31) // 32, dtype=torch.int32, device=pad.device)
    native.check(_lib().lah_pack_key_mask(ptr(pad), ptr(words), batch, seq_len, stream_ptr()), "lah_pack_key_mask")
    native.count_launch()
    return words


def pack_key_mask_ref(pad):
    """CPU oracle of ``pack_key_mask``"""
    batch, seq_len = pad.shape
    n = (seq_len + 31) // 32
    valid = torch.zeros(batch, n * 32, dtype=torch.int64)
    valid[:, :seq_len] = (~pad.cpu()).long()
    bits = (valid.view(batch, n, 32) << torch.arange(32)).sum(-1)
    return torch.where(bits >= 2 ** 31, bits - 2 ** 32, bits).to(torch.int32)


def _check_key_mask(key_mask, tokens, seq_len, device, causal):
    assert not (causal and key_mask is not None), "causal attention takes no key padding mask"
    if key_mask is not None:
        assert key_mask.dtype == torch.int32 and key_mask.is_contiguous() and key_mask.device == device
        assert key_mask.shape == (tokens // seq_len, (seq_len + 31) // 32), (tuple(key_mask.shape), tokens, seq_len)


def attention_fwd(qkv, num_heads, *, out=None, lse=None, dropout=None, seq_len=512, key_mask=None, causal=False):
    """
    Self-attention over sequences of ``seq_len`` tokens (1 <= seq_len <= MAX_SEQ) on wgmma (csrc/attention.cu).
    :param qkv: [batch*seq_len, 3*d_model] bf16 = in_proj output, [q | k | v] per token; num_heads must divide d_model and
        the head dim d_model / num_heads must be in HEAD_DIMS
    :param out: optional [batch*seq_len, d_model] bf16 destination (may be the leading rows of a larger buffer)
    :param lse: optional fp32 [batch*seq_len, num_heads]: receives the base-2 row log-sum-exp (needed by attention_bwd); with
        dropout it is still that of the undropped softmax.  A row with no valid key gets lse = +inf, which attention_bwd
        reads as "P is exactly 0"
    :param dropout: (p, seed): O = (M o P) V / (1 - p) with the site-0 mask of ``dropout_mask``; p = 0 or None launches the
        kernel without dropout
    :param key_mask: optional key padding mask from ``pack_key_mask``: masked keys are ignored by every query of their
        sequence (queries at padded positions are still computed); key blocks of 128 without a valid key are skipped.  A
        sequence without a valid key gets out = 0.  None launches the unmasked kernel
    :param causal: query q attends to keys <= q only (key blocks above the diagonal are neither loaded nor computed); takes
        no ``key_mask``
    :returns: [batch*seq_len, d_model] bf16, heads concatenated (input of out_proj)
    """
    tokens, three_d = qkv.shape
    d_model = three_d // 3
    assert 1 <= seq_len <= MAX_SEQ and tokens % seq_len == 0, (tokens, seq_len)
    assert qkv.is_cuda and qkv.dtype == torch.bfloat16 and qkv.is_contiguous()
    assert num_heads > 0 and d_model % num_heads == 0 and d_model // num_heads in HEAD_DIMS, (d_model, num_heads)
    if out is None:
        out = torch.empty(tokens, d_model, dtype=torch.bfloat16, device=qkv.device)
    assert out.dtype == torch.bfloat16 and out.is_contiguous() and out.shape == (tokens, d_model)
    if lse is not None:
        assert lse.dtype == torch.float32 and lse.is_contiguous() and lse.numel() == tokens * num_heads
    _check_key_mask(key_mask, tokens, seq_len, qkv.device, causal)
    seed, thr, rescale = _dropout_args(dropout)
    args = (ptr(qkv), ptr(out), ptr(lse), tokens, int(seq_len), num_heads, d_model, seed, thr, rescale, stream_ptr())
    if causal:
        native.check(_lib().lah_attention_fwd_causal(*args), "lah_attention_fwd_causal")
    else:
        native.check(_lib().lah_attention_fwd(*args, ptr(key_mask)), "lah_attention_fwd")
    native.count_launch()
    return out


def attention_bwd(qkv, out, dout, lse, num_heads, *, dropout=None, seq_len=512, dqkv=None, key_mask=None, causal=False):
    """
    Backward of ``attention_fwd`` on wgmma (csrc/attention_bwd.cu): recomputes P from the saved log-sum-exp, forms dV / dK /
    dQ on tensor cores (nothing of size S x S touches HBM).  Returns dqkv [tokens, 3*d_model] bf16.  Same head dims as
    ``attention_fwd``.
    Scratch: the per-key-block dQ partials, 2 * ceil(seq_len / 128) * tokens * d_model bytes (4x the bytes of dQ at 512
    tokens, 32x at 4096), and the fp32 [tokens, num_heads] row sums Delta.
    :param dropout: the (p, seed) of the forward that produced ``out``; the mask is regenerated, not read
    :param dqkv: optional contiguous [tokens, 3*d_model] bf16 destination
    :param key_mask: the ``pack_key_mask`` words of the forward.  dK / dV rows of masked keys are exactly 0; a 128-key block
        without a valid key does no MMA and writes a zero dQ partial
    :param causal: the ``causal`` of the forward: key block j walks only the query blocks that hold a query >= 128 j
    """
    tokens, three_d = qkv.shape
    d_model = three_d // 3
    assert 1 <= seq_len <= MAX_SEQ and tokens % seq_len == 0, (tokens, seq_len)
    assert dout.dtype == torch.bfloat16 and dout.is_contiguous() and out.is_contiguous() and lse.dtype == torch.float32
    assert out.dtype == torch.bfloat16 and qkv.is_contiguous()
    assert num_heads > 0 and d_model % num_heads == 0 and d_model // num_heads in HEAD_DIMS, (d_model, num_heads)
    delta = torch.empty(tokens, num_heads, dtype=torch.float32, device=qkv.device)      # rowsum(dout o out), filled by the prologue kernel
    if dqkv is None:
        dqkv = torch.empty_like(qkv)
    assert dqkv.dtype == torch.bfloat16 and dqkv.is_contiguous() and dqkv.shape == qkv.shape
    blocks = (seq_len + 127) // 128
    dq_part = torch.empty(blocks, tokens, d_model, dtype=torch.bfloat16, device=qkv.device)  # one partial per 128-key block
    _check_key_mask(key_mask, tokens, seq_len, qkv.device, causal)
    args = (ptr(qkv), ptr(out), ptr(dout), ptr(lse), ptr(delta), ptr(dqkv), ptr(dq_part), tokens, int(seq_len), num_heads,
            d_model, *_dropout_args(dropout), stream_ptr())
    if causal:
        native.check(_lib().lah_attention_bwd_causal(*args), "lah_attention_bwd_causal")
    else:
        native.check(_lib().lah_attention_bwd(*args, ptr(key_mask)), "lah_attention_bwd")
    native.count_launch(3)   # delta prologue, wgmma backward, dQ partial reduction
    return dqkv


def attention_ref(qkv, num_heads, seq_len=512, key_mask=None, causal=False):
    """fp32 oracle (fp64 for a fp64 input): softmax(q k^T / sqrt(d)) v per head.
    :param key_mask: optional bool [batch, seq_len], True = key ignored (torch's src_key_padding_mask): its scores are -inf;
        rows without a valid key give 0 (``softmax(...).nan_to_num(0)``, which is what torch's layer computes in training mode)
    :param causal: scores of keys > query are -inf"""
    tokens, three_d = qkv.shape
    d = three_d // 3
    x = qkv if qkv.dtype == torch.float64 else qkv.float()
    q, k, v = x.view(tokens // seq_len, seq_len, 3, num_heads, d // num_heads).unbind(2)
    q, k, v = (t.transpose(1, 2) for t in (q, k, v))  # [B, H, S, hd]
    s = q @ k.transpose(-1, -2) / (d // num_heads) ** 0.5
    if causal:
        s = s.masked_fill(torch.ones(seq_len, seq_len, dtype=torch.bool, device=s.device).triu(1), float("-inf"))
    if key_mask is None:
        att = torch.softmax(s, dim=-1) @ v
    else:
        s = s.masked_fill(key_mask.to(s.device).view(tokens // seq_len, 1, 1, seq_len), float("-inf"))
        att = torch.softmax(s, dim=-1).nan_to_num(0.0) @ v
    return att.transpose(1, 2).reshape(tokens, d)


# ---------------------------------------------------------------------------------------------------------
# dropout of the transformer expert (csrc/dropout.cuh: counter-based Philox4x32-10 masks, csrc/dropout.cu)
#   site 0 = attention probabilities, position (batch, head, query, key)
#   sites 1, 2, 3 = dropout1 (after out_proj), dropout (after linear1's GELU), dropout2 (after linear2), position (row, col)
# ---------------------------------------------------------------------------------------------------------
SITE_ATTN, SITE_OUT_PROJ, SITE_FF, SITE_LINEAR2 = range(4)


def dropout_threshold(p):
    """an element is kept iff its 16-bit Philox lane >= this; the realised drop probability is threshold / 65536"""
    assert 0.0 <= p < 1.0, p
    return min(65535, int(math.floor(p * 65536 + 0.5)))


def _dropout_args(dropout):
    """(seed, threshold, 1 / (1 - p)) for the C entry points; threshold -1 = no dropout"""
    if dropout is None or dropout[0] == 0:
        return 0, -1, 1.0
    p, seed = dropout[0], dropout[1]
    return int(seed) & (2 ** 64 - 1), dropout_threshold(p), 1.0 / (1.0 - p)


def dropout_mask(shape, p, seed, site, device=None):
    """
    Materialised keep mask (bool) from the same device functions the fused kernels use: ``shape`` is (batch, heads, queries,
    keys) for site 0 and (rows, cols) for sites 1-3.  For tests and oracles; the training path never stores a mask.
    """
    if site == SITE_ATTN:
        batch, heads, rows, cols = shape
    else:
        (rows, cols), batch, heads = shape, 1, 1
    out = torch.empty(*shape, dtype=torch.uint8, device=device or "cuda")
    native.check(_lib().lah_dropout_mask(ptr(out), int(site), batch, heads, rows, cols, int(seed) & (2 ** 64 - 1),
                                         dropout_threshold(p), stream_ptr()), "lah_dropout_mask")
    native.count_launch()
    return out.bool()


def _dropout_ew(op, x, f, p, seed, site, out):
    assert x.dtype == torch.bfloat16 and x.is_contiguous() and x.dim() == 2 and 1 <= site <= 3
    assert f is None or (f.shape == x.shape and f.dtype == torch.bfloat16 and f.is_contiguous())
    out = torch.empty_like(x) if out is None else out
    assert out.shape == x.shape and out.is_contiguous()
    rows, cols = x.shape
    native.check(_lib().lah_dropout_ew(op, ptr(x), ptr(f), ptr(out), rows, cols, int(seed) & (2 ** 64 - 1), int(site),
                                       dropout_threshold(p), 1.0 / (1.0 - p), stream_ptr()), "lah_dropout_ew")
    native.count_launch()
    return out


def dropout_apply(x, p, seed, site, *, out=None):
    """out = M o x / (1 - p) (bf16 [rows, cols], rows and cols multiples of 16): the gradient of a dropout site's branch"""
    return _dropout_ew(0, x, None, p, seed, site, out)


def gelu_dropout(f, p, seed, site, *, out=None):
    """out = M o gelu(f) / (1 - p) (erf GELU)"""
    return _dropout_ew(1, f, None, p, seed, site, out)


def gelu_dropout_bwd(dg, f, p, seed, site, *, out=None):
    """out = gelu'(f) o M o dg / (1 - p): backward of ``gelu_dropout``"""
    return _dropout_ew(2, dg, f, p, seed, site, out)


def relu_dropout(f, p, seed, site, *, out=None):
    """out = M o relu(f) / (1 - p)"""
    return _dropout_ew(3, f, None, p, seed, site, out)


def relu_dropout_bwd(dg, f, p, seed, site, *, out=None):
    """out = [f > 0] o M o dg / (1 - p): backward of ``relu_dropout``"""
    return _dropout_ew(4, dg, f, p, seed, site, out)


def relu_dropout_ref(f, mask, p):
    """fp32 oracle of ``relu_dropout`` with a materialised keep mask"""
    return mask.float() * F.relu(f.float()) / (1 - p)


def relu_dropout_bwd_ref(dg, f, mask, p):
    """fp32 oracle of ``relu_dropout_bwd``"""
    return (f.float() > 0).float() * mask.float() * dg.float() / (1 - p)


# ---------------------------------------------------------------------------------------------------------
# SwiGLU of the gated expert (csrc/dropout.cu): h = [g | u] is the output of the one GEMM over [W1; W3]
# ---------------------------------------------------------------------------------------------------------
def _check_swiglu(h, what):
    if h.dim() != 2 or h.shape[1] % 256:
        raise ValueError(f"{what}: h must be [rows, 2 * inner] with inner a multiple of 128, got {tuple(h.shape)}")
    rows, inner = h.shape[0], h.shape[1] // 2
    _bf16_rows(h, f"{what} h", (rows, 2 * inner))
    return rows, inner


def swiglu_fwd(h, *, out=None, quant=None, tile_group=None, total_rows=None):
    """a = silu(g) o u for h = [g | u] (bf16 [rows, 2 inner], inner a multiple of 128): bf16 [rows, inner], computed in
    fp32 and rounded once.
    :param quant: optional ops.fp8.MXFP8Tensor (activation layout) that additionally receives a as an MXFP8 GEMM operand,
        quantised from the fp32 product before its bf16 rounding; ``out`` is then written only when given.  With it,
        ``tile_group`` (int32, one entry per 128 rows, -1 = skipped) and ``total_rows`` (int32 [1] on the device: rows
        past it are skipped) limit the rows processed"""
    rows, inner = _check_swiglu(h, "swiglu_fwd")
    if quant is None:
        if tile_group is not None or total_rows is not None:
            raise ValueError("swiglu_fwd: tile_group and total_rows apply to the MXFP8 output (quant) only")
        out = torch.empty(rows, inner, dtype=torch.bfloat16, device=h.device) if out is None else out
        _bf16_rows(out, "swiglu_fwd out", (rows, inner))
        native.check(_lib().lah_swiglu_fwd(ptr(h), ptr(out), rows, inner, stream_ptr()), "lah_swiglu_fwd")
    else:
        if out is not None:
            _bf16_rows(out, "swiglu_fwd out", (rows, inner))
        _check_quant_out("swiglu_fwd", quant, rows, inner)
        if tile_group is not None and (tile_group.dtype != torch.int32 or not tile_group.is_contiguous()
                                       or tile_group.numel() < -(-rows // 128)):
            raise ValueError(f"swiglu_fwd: tile_group must be a contiguous int32 tensor of >= {-(-rows // 128)} entries")
        if total_rows is not None and (total_rows.dtype != torch.int32 or total_rows.numel() < 1):
            raise ValueError("swiglu_fwd: total_rows must be an int32 device tensor of one element")
        native.check(_lib().lah_swiglu_fwd_q(ptr(h), ptr(out), ptr(quant.q), ptr(quant.sf), rows, inner, ptr(tile_group),
                                             ptr(total_rows), stream_ptr()), "lah_swiglu_fwd_q")
    native.count_launch()
    return out


def swiglu_bwd(da, h, *, out=None):
    """dh = [da o u o s (1 + g (1 - s)) | da o silu(g)], s = sigmoid(g): bf16 [rows, 2 inner], the backward of
    ``swiglu_fwd``"""
    rows, inner = _check_swiglu(h, "swiglu_bwd")
    _bf16_rows(da, "swiglu_bwd da", (rows, inner))
    out = torch.empty_like(h) if out is None else out
    _bf16_rows(out, "swiglu_bwd out", (rows, 2 * inner))
    native.check(_lib().lah_swiglu_bwd(ptr(da), ptr(h), ptr(out), rows, inner, stream_ptr()), "lah_swiglu_bwd")
    native.count_launch()
    return out


def swiglu_ref(h):
    """oracle of ``swiglu_fwd`` in fp32 (fp64 for a fp64 input)"""
    hf = h if h.dtype == torch.float64 else h.float()
    g, u = hf.chunk(2, dim=-1)
    return F.silu(g) * u


def swiglu_bwd_ref(da, h):
    """oracle of ``swiglu_bwd`` in fp32 (fp64 for a fp64 input)"""
    hf = h if h.dtype == torch.float64 else h.float()
    g, u = hf.chunk(2, dim=-1)
    d = da.to(hf.dtype)
    s = torch.sigmoid(g)
    return torch.cat([d * u * s * (1 + g * (1 - s)), d * g * s], dim=-1)


_PHILOX_M0, _PHILOX_M1, _PHILOX_W0, _PHILOX_W1 = 0xD2511F53, 0xCD9E8D57, 0x9E3779B9, 0xBB67AE85
_U32 = 0xFFFFFFFF


def _mulhilo32(a, m):
    """(a * m) >> 32 and (a * m) & 0xffffffff for int64 tensors holding uint32 values, without 64-bit overflow"""
    t1, t2 = (a & 0xFFFF) * m, (a >> 16) * m
    return (t2 + (t1 >> 16)) >> 16, (((t2 & 0xFFFF) << 16) + t1) & _U32


def philox4x32_10_ref(ctr, key):
    """CPU Philox4x32-10 (Salmon et al., SC'11) on int64 tensors holding uint32 values; ctr: 4 words, key: 2 words"""
    c = [torch.as_tensor(w, dtype=torch.int64) for w in ctr]
    c = list(torch.broadcast_tensors(*c))
    k0, k1 = int(key[0]) & _U32, int(key[1]) & _U32
    for _ in range(10):
        hi0, lo0 = _mulhilo32(c[0], _PHILOX_M0)
        hi1, lo1 = _mulhilo32(c[2], _PHILOX_M1)
        c = [hi1 ^ c[1] ^ k0, lo1, hi0 ^ c[3] ^ k1, lo0]
        k0, k1 = (k0 + _PHILOX_W0) & _U32, (k1 + _PHILOX_W1) & _U32
    return c


def dropout_counter_ref(site, *index):
    """
    The Philox counter (four int64 tensors holding uint32 words) and the lane (0..7) of the keep decision at ``index``
    (csrc/dropout.cuh): ``index`` are broadcastable integer tensors, (batch, head, query, key) for site 0 and (row, col)
    for sites 1-3.
    """
    idx = torch.broadcast_tensors(*[torch.as_tensor(t, dtype=torch.int64) for t in index])
    zero = torch.zeros_like(idx[0])
    if site == SITE_ATTN:
        b, h, q, k = idx
        gq, gk = (q >> 4) * 4 + ((q >> 1) & 3), (k >> 4) * 4 + ((k >> 1) & 3)
        ctr = ((((gq & 127) * 128) + (gk & 127)) | ((q & 1) << 14), h, b, ((gq >> 7) << 8) | ((gk >> 7) << 20) | SITE_ATTN)
        lane = ((q >> 3) & 1) * 4 + ((k & 1) | (((k >> 3) & 1) << 1))
    else:
        r, n = idx
        gr, gn = (r >> 4) * 8 + (r & 7), (n >> 4) * 4 + ((n >> 1) & 3)
        ctr = (gn, gr, zero, zero + site)
        lane = ((r >> 3) & 1) * 4 + ((n & 1) | (((n >> 3) & 1) << 1))
    return ctr, lane


def dropout_keep_ref(p, seed, site, *index):
    """
    Independent CPU definition of the keep decision (the mask definition of csrc/dropout.cuh): ``index`` are broadcastable
    integer tensors, (batch, head, query, key) for site 0 and (row, col) for sites 1-3.  Returns a bool tensor.
    """
    ctr, lane = dropout_counter_ref(site, *index)
    seed = int(seed) & (2 ** 64 - 1)
    words = torch.stack(philox4x32_10_ref(ctr, (seed & _U32, seed >> 32)), dim=-1)
    w = words.gather(-1, (lane >> 1).unsqueeze(-1)).squeeze(-1)
    u16 = torch.where((lane & 1) == 1, w >> 16, w & 0xFFFF)
    return u16 >= dropout_threshold(p)


def dropout_mask_ref(shape, p, seed, site):
    """CPU counterpart of ``dropout_mask`` (same shape convention)"""
    grids = [torch.arange(n).view(*([1] * i), n, *([1] * (len(shape) - i - 1))) for i, n in enumerate(shape)]
    return dropout_keep_ref(p, seed, site, *grids)


# ---------------------------------------------------------------------------------------------------------
# optimizer
# ---------------------------------------------------------------------------------------------------------
def weight_decay_args(lr, weight_decay, decoupled):
    """(L2 coefficient, decoupled factor) the optimizer kernels take for torch's two weight-decay forms:
    Adam(weight_decay=wd) adds wd * p to the gradient; AdamW (decoupled) multiplies p by 1 - lr * wd, computed in double and
    rounded to fp32 once, as torch's ``p.mul_(1 - lr * wd)`` does.  A factor of 1 means no decoupled decay."""
    if decoupled:
        return 0.0, 1.0 - float(lr) * float(weight_decay)
    return float(weight_decay), 1.0


def lr_block_values(lr, weight_decay, decoupled):
    """the two floats of the device block that ``lr_dev`` points to: [lr, decoupled factor 1 - lr * wd] (the factor as
    ``weight_decay_args`` forms it, 1 without decoupled decay)"""
    return float(lr), weight_decay_args(lr, weight_decay, decoupled)[1]


def _check_lr_dev(lr_dev):
    assert (lr_dev.is_cuda and lr_dev.dtype == torch.float32 and lr_dev.numel() == 2 and lr_dev.is_contiguous()), \
        "lr_dev: a contiguous float32 CUDA tensor [lr, decay] (lr_block_values)"


def segment_views(flat, shapes, slots=1):
    """
    The layout ``adam_step`` / ``adam_step_ref`` work on, as views of ``flat``: consecutive segments, one per entry of
    ``shapes`` (name -> shape, in segment order), segment s holding ``slots`` tensors of its shape: {name: [slots, *shape]}.
    """
    views, off = {}, 0
    for name, shape in shapes.items():
        n = slots * math.prod(shape)
        views[name] = flat[off: off + n].view(slots, *shape)
        off += n
    assert off == flat.numel(), (off, flat.numel())
    return views


def adam_step(p, g, m, v, vmax, p_bf16, seg_sizes, G, *, step=None, group_rows=None, step_scalar=0, lr=1e-3,
              betas=(0.9, 0.999), eps=1e-8, weight_decay=0.0, decoupled=False, amsgrad=True, zero_mask=0, world=1,
              peer_grad_off=-1, peer_bases=None, grad_scale=1.0, G_active=0, shadow_of=None, shadow_g_off=-1, me=0,
              seg_mask=0, dead_mask=0, lr_dev=None):
    """
    One fused Adam/AMSGrad step over a flat fp32 buffer laid out as consecutive segments [G, seg_sizes[s]].
    :param lr_dev: optional float32 CUDA tensor [2] = ``lr_block_values(lr, weight_decay, decoupled)``: the kernel reads the
        learning rate and the decoupled factor from it when it runs (``lr`` is then not used), so a captured CUDA graph
        follows a schedule.  Bit-identical to the by-value launch with the same values
    :param step: int32 [G] per-group step counts (already incremented) or None -> step_scalar for everything
    :param group_rows: int32 [G]; groups with 0 rows are skipped (experts that received no tokens are not stepped)
    :param weight_decay: torch's ``weight_decay``: L2 (added to the gradient), or with ``decoupled`` AdamW's p *= 1 - lr wd
    :param G_active: only the first G_active of the G slots per segment are updated (the rest are shadow replicas)
    :param shadow_of: int32 [G_active, 2] (slot, rank mask): gradient of a shadowed expert = sum of the partial
        gradients in shadow slot ``slot`` of the ranks in ``mask`` (buffers at symmetric offset ``shadow_g_off``)
    """
    arr = None
    if peer_bases is not None:
        arr = (c_ull * len(peer_bases))(*[int(b) for b in peer_bases])
    if isinstance(seg_sizes, int):
        seg_sizes = [seg_sizes]
    segs = (c_ll * len(seg_sizes))(*[int(s) for s in seg_sizes])
    if lr_dev is not None:
        _check_lr_dev(lr_dev)
    l2, decay = weight_decay_args(lr, weight_decay, decoupled)
    native.check(_lib().lah_adam_step(ptr(p), ptr(g), ptr(m), ptr(v), ptr(vmax), ptr(p_bf16), len(seg_sizes),
                                      ctypes.cast(segs, c_void_p), G, ptr(step), ptr(group_rows), int(step_scalar), lr,
                                      ptr(lr_dev), betas[0], betas[1], eps, l2, int(amsgrad), int(zero_mask), world,
                                      peer_grad_off, ctypes.cast(arr, c_void_p) if arr is not None else c_void_p(0),
                                      grad_scale, int(G_active), ptr(shadow_of), int(shadow_g_off), int(me), int(seg_mask),
                                      int(dead_mask), decay, int(bool(decoupled and weight_decay)), stream_ptr()),
                 "lah_adam_step")
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
                                          wait_epoch, ptr(wait_status), int(max_ctas), stream_ptr()),
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
               eps=1e-8, amsgrad=True, weight_decay=0.0, decoupled=False, max_ctas=0, lr_dev=None, p_lo=None):
    """
    Fused weight gradient + per-expert AMSGrad (csrc/small_m.cu): for every group g with rows > 0,
    dW[g] = dy_g^T x_g is formed in registers and applied to p / m / v / vmax ([G, N, K] fp32) and the bf16 mirror in the same
    kernel; the gradient never reaches HBM.  ``step`` holds the per-expert step counts AFTER this update.
    ``weight_decay`` / ``decoupled`` / ``lr_dev``: as in ``adam_step``.
    ``p_lo``: a split master weight (``split_encode``): p=None, the weight is ``p_bf16`` plus its low half ``p_lo`` ([G, N, K]
    int16) with the tie bits in the sign of ``v``; the step computes the same bits as on fp32 p.
    """
    G, N, Kd = (p if p_lo is None else p_lo).shape
    assert dy.shape[1] == N and x.shape[1] == Kd and dy.shape[0] == x.shape[0]
    assert dy.dtype == torch.bfloat16 and x.dtype == torch.bfloat16
    if p_lo is None:
        assert p.is_contiguous() and p.dtype == torch.float32
    else:
        assert p is None and p_lo.dtype == torch.int16 and p_bf16.dtype == torch.bfloat16
        assert p_lo.is_contiguous() and p_bf16.is_contiguous() and p_bf16.shape[1:] == p_lo.shape[1:]
    if amsgrad and vmax is None:
        raise ValueError("wgrad_adam: amsgrad needs a vmax tensor (vmax=None only with amsgrad=False)")
    if lr_dev is not None:
        _check_lr_dev(lr_dev)
    l2, decay = weight_decay_args(lr, weight_decay, decoupled)
    common = (ptr(dy), dy.stride(0), ptr(x), x.stride(0), dy.shape[0], G, N, Kd, ptr(group_off), ptr(group_rows),
              ptr(skip), ptr(step))
    tail = (lr, ptr(lr_dev), betas[0], betas[1], eps, int(amsgrad), l2, decay, int(bool(decoupled and weight_decay)),
            int(max_ctas), stream_ptr())
    if p_lo is None:
        native.check(_lib().lah_wgrad_adam(*common, ptr(p), ptr(m), ptr(v), ptr(vmax), ptr(p_bf16), *tail),
                     "lah_wgrad_adam")
    else:
        native.check(_lib().lah_wgrad_adam_split(*common, ptr(p_bf16), ptr(p_lo), ptr(m), ptr(v), ptr(vmax), *tail),
                     "lah_wgrad_adam_split")
    native.count_launch()


def bump_steps(step, group_rows):
    native.check(_lib().lah_bump_steps(ptr(step), ptr(group_rows), step.numel(), stream_ptr()), "lah_bump_steps")
    native.count_launch()


def cast_bf16(src, dst):
    assert src.dtype == torch.float32 and dst.dtype == torch.bfloat16 and src.numel() == dst.numel()
    native.check(_lib().lah_cast_bf16(ptr(src), ptr(dst), src.numel(), stream_ptr()), "lah_cast_bf16")
    native.count_launch()


def _check_split(p, hi, lo, v):
    n = p.numel()
    assert p.dtype == torch.float32 and hi.dtype == torch.bfloat16 and lo.dtype == torch.int16 and v.dtype == torch.float32
    assert hi.numel() == n and lo.numel() == n and v.numel() == n
    assert all(t.is_contiguous() and t.is_cuda for t in (p, hi, lo, v))


def split_encode(p, hi, lo, v):
    """Split master weight: hi = bf16(p) (round to nearest even, the GEMM operand), lo = the low 16 bits of p, and the bit
    that tells a tie rounded up (low half 0x8000, p's upper half odd) in the sign of v (exp_avg_sq, >= 0).  csrc/sm90.cuh,
    split_decode, has the exact rule; ``split_decode`` inverts it for every finite p."""
    _check_split(p, hi, lo, v)
    native.check(_lib().lah_split_master(ptr(p), ptr(hi), ptr(lo), ptr(v), p.numel(), 1, stream_ptr()), "lah_split_master")
    native.count_launch()


def split_decode(hi, lo, v, out):
    """the fp32 master weight of a split one (``split_encode``), into ``out``"""
    _check_split(out, hi, lo, v)
    native.check(_lib().lah_split_master(ptr(out), ptr(hi), ptr(lo), ptr(v), out.numel(), 0, stream_ptr()),
                 "lah_split_master")
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


def sigmoid_weights_ref(sel, valid, scale=1.0):
    """weights of the sigmoid router (DESIGN.md §6c) from the selected scores ``sel`` [B, k] and their validity:
    scale * sigma_j / S_b with S_b the sum of sigma over the valid pairs; a token with S_b = 0 gets zeros.  Differentiable
    (no NaN reaches the gradient of an S_b = 0 token)."""
    sg = torch.where(valid, torch.sigmoid(sel), torch.zeros_like(sel))
    S = sg.sum(-1, keepdim=True)
    return torch.where(S > 0, scale * sg / torch.where(S > 0, S, torch.ones_like(S)), torch.zeros_like(sg))


def softmax_lse_ref(scores, alive=None):
    """[B] log-partition z_b of the softmax over the live experts (DESIGN.md §6a / §6e): logsumexp of ``scores`` [B, E]
    over the experts with ``alive`` (uint8 [E], None: all); 0 for a token without a finite live score.  Differentiable"""
    live = torch.ones(scores.shape[-1], dtype=torch.bool, device=scores.device) if alive is None \
        else alive.bool().reshape(-1).to(scores.device)
    masked = scores.masked_fill(~live.view(1, -1), float("-inf"))
    ok = torch.isfinite(masked).any(-1, keepdim=True)
    z = torch.logsumexp(torch.where(ok, masked, torch.zeros_like(masked)), -1, keepdim=True)
    return torch.where(ok, z, torch.zeros_like(z)).squeeze(-1)


def softmax_weights_ref(scores, idx, alive=None, scale=1.0):
    """weights of the unnormalised softmax router (norm_topk_prob=False, DESIGN.md §6e): scale * p_{b, idx} with p the
    softmax of ``scores`` [B, E] over the live experts (``softmax_lse_ref``), 0 for a missing pair (idx -1).  The
    selection does not enter the partition: failed experts and experts outside the chosen groups stay in it.
    Differentiable in ``scores``"""
    z = softmax_lse_ref(scores, alive)
    sel = torch.gather(scores, 1, idx.clamp(min=0))
    valid = idx >= 0
    return torch.where(valid, scale * torch.exp(sel.masked_fill(~valid, 0.0) - z.unsqueeze(-1)), torch.zeros_like(sel))


def expert_group_scores_ref(scores, bias, n_group, score="softmax"):
    """(score [B, G], has [B, G]) of group-limited routing (DESIGN.md §6d).  ``scores``: the float32 product-key scores
    with -inf for the experts that are not candidates (dead or failure-injected).  A candidate's group key is the key the
    selection ranks (s, s + b or sigma(s) + b), sigma(s) for the unbiased sigmoid router.  A group scores its largest key
    (softmax) or the sum of its two largest (sigmoid; one candidate scores its key); ``has``: the group has a candidate."""
    B, E = scores.shape
    gsz = E // n_group
    cand = torch.isfinite(scores)
    base = torch.sigmoid(scores) if score == "sigmoid" else scores
    key = base if bias is None else base + bias.to(device=scores.device, dtype=torch.float32).reshape(1, -1)
    key = key.masked_fill(~cand, float("-inf")).view(B, n_group, gsz)
    top = torch.sort(key, dim=-1, descending=True)[0]
    gscore = top[..., 0]
    if score == "sigmoid" and gsz > 1:
        gscore = torch.where(torch.isfinite(top[..., 1]), top[..., 0] + top[..., 1], top[..., 0])
    return gscore, cand.view(B, n_group, gsz).any(-1)


def expert_group_mask_ref(scores, bias, n_group, topk_group, score="softmax"):
    """[B, E] bool: the experts of each token's topk_group best groups (``expert_group_scores_ref``).  The groups are
    sorted by score stably, descending, so equal scores go to the smaller id; a group without candidates is never taken."""
    gscore, has = expert_group_scores_ref(scores, bias, n_group, score)
    order = torch.sort(gscore.masked_fill(~has, float("-inf")), dim=-1, descending=True, stable=True)[1]
    chosen = torch.zeros_like(has)
    chosen.scatter_(1, order[:, :topk_group], True)
    chosen &= has
    return chosen.repeat_interleave(scores.shape[1] // n_group, dim=1)


def gate_topk_ref(logits, grid_size, k, alive=None, fail_mask=None, bias=None, score="softmax", scale=1.0, n_group=1,
                  topk_group=1, norm=True):
    """returns idx [B,k] (-1 for missing), weights [B,k] (softmax over alive selected).  Equal scores select the smaller
    expert id first, like gate_topk_kernel (torch.topk leaves the order of ties unspecified, so it sorts stably instead).
    The scores are summed first grid dimension first and the kernel last dimension first: on 3-d and 4-d grids they can
    differ in the last bit unless the logits are exact in any order (e.g. small multiples of a power of two).
    ``bias`` ([E]): the selection ranks the float32 keys score + bias[e]; the weights stay the softmax over the unbiased
    scores of the selected experts.
    ``score="sigmoid"`` (DESIGN.md §6c): the weights are ``sigmoid_weights_ref`` of the selected scores, and a bias is
    added to sigmoid(score) in float32; without one the selection is the softmax router's.
    ``n_group`` / ``topk_group`` (DESIGN.md §6d): the candidates are narrowed to each token's topk_group best groups
    (``expert_group_mask_ref``) before the selection; 1 / 1 and topk_group = n_group leave them as they are.
    ``norm=False`` (DESIGN.md §6e): the same selection, weighted by ``softmax_weights_ref`` (softmax) or scale * sigma_j
    (sigmoid), without renormalisation."""
    if score not in ROUTER_SCORES:
        raise ValueError(f"gate_topk_ref: score must be one of {ROUTER_SCORES}, got {score!r}")
    scores = product_key_scores(logits.float(), grid_size)
    raw = scores
    check_expert_groups("gate_topk_ref", scores.shape[-1], n_group, topk_group)
    dead = torch.zeros_like(scores, dtype=torch.bool)
    if alive is not None:
        dead |= ~alive.bool().view(1, -1)
    if fail_mask is not None:
        dead |= fail_mask
    scores = scores.masked_fill(dead, float("-inf"))
    if topk_group < n_group:
        scores = scores.masked_fill(~expert_group_mask_ref(scores, bias, n_group, topk_group, score), float("-inf"))
    if scores.shape[-1] < k:
        scores = F.pad(scores, (0, k - scores.shape[-1]), value=float("-inf"))
    if bias is None:
        top_v, top_i = torch.sort(scores, dim=-1, descending=True, stable=True)
        top_v, top_i = top_v[..., :k], top_i[..., :k]
    else:
        b = bias.to(device=scores.device, dtype=torch.float32).reshape(1, -1)
        base = scores if score == "softmax" else torch.sigmoid(scores).masked_fill(~torch.isfinite(scores), float("-inf"))
        keys = base + F.pad(b, (0, scores.shape[-1] - b.shape[-1]))
        top_i = torch.sort(keys, dim=-1, descending=True, stable=True)[1][..., :k]
        top_v = torch.gather(scores, -1, top_i)
    valid = torch.isfinite(top_v)
    top_i = torch.where(valid, top_i, torch.full_like(top_i, -1))
    if not norm and score == "softmax":
        return top_i, softmax_weights_ref(raw, top_i, alive, scale)   # valid ids < E: padding never enters
    if not norm:
        return top_i, torch.where(valid, scale * torch.sigmoid(top_v.masked_fill(~valid, 0.0)), torch.zeros_like(top_v))
    if score == "sigmoid":
        w = sigmoid_weights_ref(top_v.masked_fill(~valid, 0.0), valid, scale)
        return torch.where(valid, top_i, torch.full_like(top_i, -1)), w
    w = torch.softmax(top_v.masked_fill(~valid, float("-inf")), dim=-1)
    w = torch.where(valid, w, torch.zeros_like(w)).nan_to_num(0.0)
    return torch.where(valid, top_i, torch.full_like(top_i, -1)), w


def router_loss_ref(logits, grid_size, counts, alive=None, score="softmax"):
    """Oracle of the router-loss kernels: (L_aux, L_z) as 0-d tensors in the dtype of ``logits`` (float64 works),
    differentiable in the logits with f detached.  ``counts``: [E] routed pairs per expert, or [R, E] (summed over R).
    L_aux = N * sum_e f_e * mean_b p_{b,e} over the N live experts, L_z = mean_b z_b^2; a token without a finite live
    score contributes 0 to both, and N = 0 gives zeros.  ``score="sigmoid"`` (DESIGN.md §6c): p_{b,e} = sigma_{b,e} / S'_b
    with S'_b the sum of sigma over the live experts (a token with S'_b = 0 contributes 0), and L_z = 0."""
    if score not in ROUTER_SCORES:
        raise ValueError(f"router_loss_ref: score must be one of {ROUTER_SCORES}, got {score!r}")
    scores = product_key_scores(logits, grid_size)
    B, E = scores.shape
    live = torch.ones(E, dtype=torch.bool, device=scores.device) if alive is None else alive.bool().reshape(-1).to(scores.device)
    c = counts.reshape(-1, E).sum(0).to(scores.dtype).to(scores.device)
    f = (c / c.sum() if float(c.sum()) > 0 else torch.zeros_like(c)).detach()
    N = int(live.sum())
    masked = scores.masked_fill(~live.view(1, -1), float("-inf"))
    ok = torch.isfinite(masked).any(-1, keepdim=True)   # tokens with at least one finite live score
    masked = torch.where(ok, masked, torch.zeros_like(masked))
    if N == 0 or B == 0:
        zero = scores.sum() * 0
        return zero, zero
    if score == "sigmoid":
        sg = torch.where(live.view(1, -1), torch.sigmoid(scores), torch.zeros_like(scores))
        S = sg.sum(-1, keepdim=True)
        p = sg / torch.where(S > 0, S, torch.ones_like(S))
        return N * (p * f).sum() / B, torch.zeros((), dtype=scores.dtype, device=scores.device)
    z = torch.logsumexp(masked, -1, keepdim=True)
    p = torch.where(live.view(1, -1) & ok, torch.exp(masked - z), torch.zeros_like(masked))
    z = torch.where(ok, z, torch.zeros_like(z)).squeeze(-1)
    return N * (p * f).sum() / B, (z * z).sum() / B


def expert_bias_update_ref(counts, bias, rate, alive=None):
    """Oracle of expert_bias_update: the updated float32 bias (a new tensor).  ``counts``: [E] or [R, E] routed pairs
    (summed over R).  The comparisons N c_e <> T are exact integers; a moving bias gets one float32 add of +-rate."""
    bias = bias.to(torch.float32)
    E = bias.numel()
    c = counts.reshape(-1, E).to(torch.int64).sum(0).cpu()
    live = torch.ones(E, dtype=torch.bool) if alive is None else alive.bool().reshape(-1).cpu()
    T, N = int(c.sum()), int(live.sum())
    step = torch.sign(T - N * c) * live   # +1: below the mean load, -1: above, 0: balanced or dead
    if T == 0:
        step.zero_()
    rate32 = torch.tensor(rate, dtype=torch.float32)
    out = torch.where(step != 0, bias.cpu() + step.to(torch.float32) * rate32, bias.cpu())
    return out.to(bias.device)


_SPLITMIX_GAMMA = 0x9E3779B97F4A7C15


def splitmix64_ref(x):
    """splitmix64 finaliser of csrc/moe.cu hash_uniform, x + gamma included (= the output of a splitmix64 generator whose
    state was x); numpy uint64 arrays wrap modulo 2**64 like the kernel's unsigned long long"""
    import numpy as np
    x = np.array(x, dtype=np.uint64, ndmin=1) + np.uint64(_SPLITMIX_GAMMA)
    x = (x ^ (x >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
    x = (x ^ (x >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
    return x ^ (x >> np.uint64(31))


def gate_fail_mask_ref(B, E, rate, seed, token_offset):
    """[B, E] bool: the (token, expert) pairs that gate_topk's failure injection drops.  Token b of a call draws
    u = (splitmix64(seed ^ ((token_offset + b) * 0x100000001B3 + e)) >> 40) / 2**24 for expert e and fails iff u < rate, with
    rate rounded to float32 as the kernel receives it.  u has 24 bits, so this is exact, not a statistical twin.
    ``token_offset`` is the kernel argument plus the device token base (step counters [2:4]) at the launch."""
    import numpy as np
    mask64 = 2 ** 64 - 1
    tok = (np.arange(B, dtype=np.uint64) + np.uint64(int(token_offset) & mask64)) * np.uint64(0x100000001B3)
    key = np.uint64(int(seed) & mask64) ^ (tok[:, None] + np.arange(E, dtype=np.uint64)[None, :])
    u = (splitmix64_ref(key) >> np.uint64(40)).astype(np.float64) / 2.0 ** 24
    return torch.from_numpy(u < float(np.float32(rate)))


def ln_relu_ref(h, gamma, beta, relu=True):
    y = F.layer_norm(h.float(), (h.shape[-1],), gamma.float(), beta.float(), 1e-5)
    return F.relu(y) if relu else y


def ln_relu_bwd_ref(da, h, gamma, beta, relu=True, dres=None):
    """fp32 closed-form oracle of ``ln_relu_bwd`` for one group: (dh, dgamma, dbeta, dbias), dbias = the column sum of dh"""
    hf = h.float()
    mu = hf.mean(-1, keepdim=True)
    rstd = torch.rsqrt(hf.var(-1, unbiased=False, keepdim=True) + 1e-5)
    xhat = (hf - mu) * rstd
    g = da.float()
    if relu:
        g = g * (xhat * gamma.float() + beta.float() > 0)
    dxh = g * gamma.float()
    dh = rstd * (dxh - dxh.mean(-1, keepdim=True) - xhat * (dxh * xhat).mean(-1, keepdim=True))
    if dres is not None:
        dh = dh + dres.float()
    return dh, (g * xhat).sum(0), g.sum(0), dh.sum(0)


@torch.no_grad()
def adam_step_ref(p, g, m, v, vmax, seg_sizes, G, *, step, group_rows=None, lr=1e-3, betas=(0.9, 0.999), eps=1e-8,
                  amsgrad=True, zero_mask=0, weight_decay=0.0, decoupled=False):
    """PyTorch implementation of csrc/adam.cu (flat segments [G, size]; per-group step; inactive groups skipped;
    weight decay as torch.optim.Adam / AdamW apply it)."""
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
        if weight_decay and decoupled:
            P[idx] = P[idx] * (1 - lr * weight_decay)
        elif weight_decay:
            grad = grad + weight_decay * P[idx]
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
