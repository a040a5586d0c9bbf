"""
Grouped GEMMs of the expert path (wgmma/TMA kernel in csrc/grouped_gemm.cu) + plain PyTorch oracles.

Layout contract shared with the dispatch kernel (ops/dispatch.py):
  * token rows are grouped by expert, every group is padded with ZERO rows to a multiple of 128,
  * ``tile_group[t]`` is the expert of the t-th 128-row tile (-1 = unused tile),
  * ``group_off[g]`` .. ``group_off[g+1]`` is the padded row range of expert g.

Replaces the cuBLAS calls behind ``nn.Linear`` in the reference's experts
(/root/reference/experiments/throughput/layers.py:8-19) and autograd's dgrad/wgrad
(/root/reference/lib/runtime/expert_backend.py:73-93).
"""
import ctypes

import torch

from . import native
from .kernels import _dropout_args
from .native import c_void_p, c_int, c_ll, ptr, stream_ptr

TILE_M = 128
_configured = False


def _lib():
    global _configured
    lib = native.cuda_lib()
    if not _configured:
        lib.lah_gemm_mgroup.restype = c_int
        lib.lah_gemm_mgroup.argtypes = [c_void_p, c_ll, c_int, c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_ll,
                                        c_int, c_int, c_int, c_void_p, c_void_p, c_void_p, c_ll, c_int, c_int, c_void_p, c_int, c_int,
                                        c_void_p, c_int, ctypes.c_ulonglong, c_int, ctypes.c_float, c_int, c_void_p]
        lib.lah_gemm_kgroup.restype = c_int
        lib.lah_gemm_kgroup.argtypes = [c_void_p, c_ll, c_void_p, c_ll, c_int, c_int, c_int, c_int, c_void_p,
                                        c_void_p, c_ll, c_ll, c_int, c_int, c_int, c_void_p]
        _configured = True
    return lib


def _pick_block_n(n: int) -> int:
    if n % 256 == 0 or n > 256:
        return 256
    if n > 64:
        return 128
    return 64


def _check_pairs(t, what, align):
    """the GEMM epilogue accesses ``t`` two elements at a time: its row stride must be even and its base ``align``-byte
    aligned (a misaligned vector access faults on the device)"""
    if (t.dim() > 1 and t.stride(0) % 2) or t.data_ptr() % align:
        raise ValueError(f"{what}: the row stride must be even and the base {align}-byte aligned "
                         f"(stride {t.stride(0)}, address {t.data_ptr():#x})")


def grouped_linear(a, w, *, tile_group=None, bias=None, residual=None, w_is_kn=False, out=None,
                   out_dtype=torch.bfloat16, m_valid=None, block_n=None, max_ctas=0, wait=None, act=0, dropout=None):
    """
    out[r, :] = act(a[r, :] @ W[g(r)]^T (+ bias[g(r)])) (+ residual[r, :])   on 128 x block_n tiles

    :param a: [rows, K] bf16, rows grouped by expert & padded to 128 (see module docstring)
    :param w: [G, N, K] bf16 (w_is_kn=False, y = x W^T)   or   [G, K, N] bf16 (w_is_kn=True, y = x W: dgrad)
    :param tile_group: int32 [ceil(rows/128)] expert of every 128-row tile (-1 skips the tile); None => expert 0
    :param bias: fp32 [G, N] or None;  residual: bf16 [rows, N] or None
    :param block_n: tile width 256, 128 or 64; None picks it from N (256 whenever N is a multiple of 256)
    :param act: activation fused after the bias: 0 none, 1 ReLU, 2 GELU(erf)
    :param wait: (flags int32 tensor [count], epoch, status tensor) — receive-side fusion: the kernel's TMA producer
        polls the peers' dispatch flags (ld.acquire.sys) before its first load instead of a separate wait kernel
    :param dropout: (p, seed, site): out = M o act(a W^T + bias) / (1 - p) (+ residual), M the (row, column) mask of
        ``kernels.dropout_mask`` site 1-3; needs 128 x 256 tiles, y = x W^T, bf16 output.  p = 0 or None: no dropout
    """
    wait_flags, wait_count, wait_epoch, wait_status = (wait[0], wait[0].numel(), wait[1], wait[2]) if wait else (None, 0, 0, None)
    assert a.is_cuda and a.dtype == torch.bfloat16 and w.dtype == torch.bfloat16 and a.dim() == 2 and w.dim() == 3
    assert a.stride(1) == 1 and w.is_contiguous()
    rows, K = a.shape
    G = w.shape[0]
    if w_is_kn:
        assert w.shape[1] == K
        N = w.shape[2]
    else:
        assert w.shape[2] == K
        N = w.shape[1]
    num_m_tiles = (rows + TILE_M - 1) // TILE_M
    if tile_group is not None:
        assert tile_group.dtype == torch.int32 and tile_group.numel() >= num_m_tiles
    if out is None:
        out = torch.empty(rows, N, device=a.device, dtype=out_dtype)
    assert out.stride(1) == 1 and out.shape[0] >= rows and out.shape[1] == N
    _check_pairs(out, "out", 2 * out.element_size())
    if bias is not None:
        assert bias.dtype == torch.float32 and bias.is_contiguous() and bias.numel() == G * N
        _check_pairs(bias, "bias", 8)
    if residual is not None:
        assert residual.dtype == torch.bfloat16 and residual.stride(1) == 1
        _check_pairs(residual, "residual", 4)
    bn = block_n or _pick_block_n(N)
    seed, thr, scale = _dropout_args(dropout)
    site = 0
    if thr >= 0:
        assert bn == 256 and not w_is_kn and out.dtype == torch.bfloat16 and wait is None, \
            "the dropout epilogue needs 128 x 256 tiles, y = x W^T and a bf16 output"
        site = int(dropout[2])
    code = _lib().lah_gemm_mgroup(
        ptr(a), a.stride(0), rows, ptr(w), G, N, K, int(w_is_kn), ptr(out), out.stride(0),
        int(out.dtype == torch.float32), rows if m_valid is None else m_valid, num_m_tiles, ptr(tile_group),
        ptr(bias), ptr(residual), residual.stride(0) if residual is not None else 0, bn, max_ctas, ptr(wait_flags),
        wait_count, wait_epoch, ptr(wait_status), int(act), seed, thr, scale, site, stream_ptr())
    native.check(code, "lah_gemm_mgroup")
    native.count_launch()
    return out


def grouped_wgrad(dy, x, group_off, num_groups, *, out=None, block_n=None, max_ctas=0, accumulate=False):
    """
    out[g] (+)= dy[off[g]:off[g+1]]^T @ x[off[g]:off[g+1]]   (fp32 [G, M, N]); groups with no rows are left untouched.
    The reduction over an expert's rows IS the gradient reduction over all trainers that routed tokens to it.
    :param accumulate: add to ``out`` instead of overwriting it (gradient accumulation across steps)
    """
    assert dy.is_cuda and dy.dtype == torch.bfloat16 and x.dtype == torch.bfloat16
    assert dy.stride(1) == 1 and x.stride(1) == 1 and dy.shape[0] == x.shape[0]
    assert group_off.dtype == torch.int32 and group_off.numel() >= num_groups + 1
    rows, M = dy.shape
    N = x.shape[1]
    if out is None:
        out = torch.zeros(num_groups, M, N, device=dy.device, dtype=torch.float32)
    assert out.dtype == torch.float32 and out.is_contiguous()
    _check_pairs(out, "out", 8)
    bn = block_n or _pick_block_n(N)
    code = _lib().lah_gemm_kgroup(ptr(dy), dy.stride(0), ptr(x), x.stride(0), rows, num_groups, M, N, ptr(group_off),
                                  ptr(out), N, M * N, bn, max_ctas, int(accumulate), stream_ptr())
    native.check(code, "lah_gemm_kgroup")
    native.count_launch()
    return out


# ---------------------------------------------------------------------------------------------------------
# PyTorch oracles (fp32 math) — used by the tests and by the CPU / baseline paths
# ---------------------------------------------------------------------------------------------------------
def grouped_linear_ref(a, w, *, tile_group=None, bias=None, residual=None, w_is_kn=False):
    rows = a.shape[0]
    N = w.shape[2] if w_is_kn else w.shape[1]
    out = torch.zeros(rows, N, dtype=torch.float32, device=a.device)
    num_m_tiles = (rows + TILE_M - 1) // TILE_M
    groups = tile_group.tolist() if tile_group is not None else [0] * num_m_tiles
    for t in range(num_m_tiles):
        g = groups[t]
        if g < 0:
            continue
        sl = slice(t * TILE_M, min(rows, (t + 1) * TILE_M))
        wg = w[g].float()
        y = a[sl].float() @ (wg if w_is_kn else wg.t())
        if bias is not None:
            y = y + bias.view(w.shape[0], N)[g]
        if residual is not None:
            y = y + residual[sl].float()
        out[sl] = y
    return out


def grouped_wgrad_ref(dy, x, group_off, num_groups):
    off = group_off.tolist()
    out = torch.zeros(num_groups, dy.shape[1], x.shape[1], dtype=torch.float32, device=dy.device)
    for g in range(num_groups):
        if off[g + 1] > off[g]:
            out[g] = dy[off[g]:off[g + 1]].float().t() @ x[off[g]:off[g + 1]].float()
    return out
