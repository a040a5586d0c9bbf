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
                                        c_void_p, c_void_p]
        lib.lah_gemm_kgroup.restype = c_int
        lib.lah_gemm_kgroup.argtypes = [c_void_p, c_ll, c_void_p, c_ll, c_int, c_int, c_int, c_int, c_void_p,
                                        c_void_p, c_ll, c_ll, c_int, c_int, c_void_p]
        lib.lah_gemm_mgroup2.restype = c_int
        lib.lah_gemm_mgroup2.argtypes = [c_void_p, c_ll, c_int, c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_ll,
                                         c_int, c_int, c_int, c_void_p, c_void_p, c_void_p, c_ll, c_int, c_void_p, c_int, c_int, c_void_p,
                                         c_int, c_void_p]
        lib.lah_gemm_kgroup2.restype = c_int
        lib.lah_gemm_kgroup2.argtypes = [c_void_p, c_ll, c_void_p, c_ll, c_int, c_int, c_int, c_int, c_void_p,
                                         c_void_p, c_ll, c_ll, c_int, c_int, c_void_p]
        _configured = True
    return lib


def _pick_block_n(n: int) -> int:
    if n % 256 == 0 or n > 256:
        return 256
    if n > 64:
        return 128
    return 64


def grouped_linear(a, w, *, tile_group=None, bias=None, residual=None, w_is_kn=False, out=None,
                   out_dtype=torch.bfloat16, m_valid=None, block_n=None, max_ctas=0, two_cta=False, wait=None, act=0):
    """
    out[r, :] = a[r, :] @ W[g(r)]^T (+ bias[g(r)]) (+ residual[r, :])

    :param a: [rows, K] bf16, rows grouped by expert & padded to 128 (see module docstring)
    :param w: [G, N, K] bf16 (w_is_kn=False, y = x W^T)   or   [G, K, N] bf16 (w_is_kn=True, y = x W: dgrad)
    :param tile_group: int32 [ceil(rows/128)] expert of every 128-row tile (-1 skips the tile); None => expert 0
    :param bias: fp32 [G, N] or None;  residual: bf16 [rows, N] or None
    :param act: activation fused after the bias (wide-tile kernel only): 0 none, 1 ReLU, 2 GELU(erf)
    :param wait: (flags int32 tensor [count], epoch, status tensor) — receive-side fusion: the kernel's TMA producer
        polls the peers' dispatch flags (ld.acquire.sys) before its first load instead of a separate wait kernel
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
    if bias is not None:
        assert bias.dtype == torch.float32 and bias.is_contiguous() and bias.numel() == G * N
    if residual is not None:
        assert residual.dtype == torch.bfloat16 and residual.stride(1) == 1
    if two_cta and N % 256 == 0:
        # wide-tile kernel (128x256 tiles): expert groups must be padded to 256 rows
        code = _lib().lah_gemm_mgroup2(
            ptr(a), a.stride(0), rows, ptr(w), G, N, K, int(w_is_kn), ptr(out), out.stride(0),
            int(out.dtype == torch.float32), rows if m_valid is None else m_valid, num_m_tiles, ptr(tile_group),
            ptr(bias), ptr(residual), residual.stride(0) if residual is not None else 0, max_ctas, ptr(wait_flags),
            wait_count, wait_epoch, ptr(wait_status), int(act), stream_ptr())
        native.check(code, "lah_gemm_mgroup2")
        native.count_launch()
        return out
    assert act == 0, "epilogue activations are implemented in the wide-tile kernel (two_cta=True, N % 256 == 0)"
    bn = block_n or _pick_block_n(N)
    code = _lib().lah_gemm_mgroup(
        ptr(a), a.stride(0), rows, ptr(w), G, N, K, int(w_is_kn), ptr(out), out.stride(0),
        int(out.dtype == torch.float32), rows if m_valid is None else m_valid, num_m_tiles, ptr(tile_group),
        ptr(bias), ptr(residual), residual.stride(0) if residual is not None else 0, bn, max_ctas, ptr(wait_flags),
        wait_count, wait_epoch, ptr(wait_status), stream_ptr())
    native.check(code, "lah_gemm_mgroup")
    native.count_launch()
    return out


def grouped_wgrad(dy, x, group_off, num_groups, *, out=None, block_n=None, max_ctas=0, two_cta=False, accumulate=False):
    """
    out[g] = dy[off[g]:off[g+1]]^T @ x[off[g]:off[g+1]]   (fp32 [G, M, N]); groups with no rows are left untouched.
    The reduction over an expert's rows IS the gradient reduction over all trainers that routed tokens to it.
    """
    assert dy.is_cuda and dy.dtype == torch.bfloat16 and x.dtype == torch.bfloat16
    assert dy.stride(1) == 1 and x.stride(1) == 1 and dy.shape[0] == x.shape[0]
    assert group_off.dtype == torch.int32 and group_off.numel() >= num_groups + 1
    rows, M = dy.shape
    N = x.shape[1]
    if out is None:
        out = torch.zeros(num_groups, M, N, device=dy.device, dtype=torch.float32)
    assert out.dtype == torch.float32 and out.is_contiguous()
    if two_cta and M % 256 == 0 and N % 256 == 0:
        code = _lib().lah_gemm_kgroup2(ptr(dy), dy.stride(0), ptr(x), x.stride(0), rows, num_groups, M, N,
                                       ptr(group_off), ptr(out), N, M * N, max_ctas, int(accumulate), stream_ptr())
        native.check(code, "lah_gemm_kgroup2")
        native.count_launch()
        return out
    assert not accumulate, "gradient accumulation is implemented in the wide-tile kernel (two_cta=True)"
    bn = block_n or _pick_block_n(N)
    code = _lib().lah_gemm_kgroup(ptr(dy), dy.stride(0), ptr(x), x.stride(0), rows, num_groups, M, N, ptr(group_off),
                                  ptr(out), N, M * N, bn, max_ctas, stream_ptr())
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
