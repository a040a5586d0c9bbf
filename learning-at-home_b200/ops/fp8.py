"""
Block-scaled FP8 (MXFP8) operands and the grouped GEMM that consumes them (csrc/grouped_gemm_fp8.cu):
E4M3 data + one UE8M0 (power-of-two) scale per 1x32 block along K, applied per 32-element K block to FP8 wgmma partials.

BASELINE.json config "DMoE 4096 experts ... fp8 expert GEMM": the expert FFN forward GEMMs
(/root/reference/experiments/throughput/layers.py:8-19 — nn.Linear in the reference, fp32 cuBLAS) run on FP8 tensor
cores; dgrad / wgrad stay bf16 (see DESIGN.md §5).

Scale-factor storage (shared with the kernel): rows are split into tiles of ``tile_rows`` rows (128 for activations,
192 for weights), tiles into atoms of 128 rows, K into blocks of 128; one (atom, K-block) chunk is
512 bytes (byte ``((r % 32) * 4 + r // 32) * 4 + kstep``).
"""
import ctypes

import torch

from . import gemm, native
from .native import c_void_p, c_int, c_ll, ptr, stream_ptr

ACT_TILE = 128      # tile_rows of activation scale factors
WEIGHT_TILE = 192   # tile_rows of weight scale factors (= TILE_N of the kernel)
_configured = False


def _lib():
    global _configured
    lib = native.cuda_lib()
    if not _configured:
        lib.lah_mxfp8_sf_bytes.restype = c_ll
        lib.lah_mxfp8_sf_bytes.argtypes = [c_ll, c_int, c_int, c_int]
        lib.lah_quant_mxfp8.restype = c_int
        lib.lah_quant_mxfp8.argtypes = [c_void_p, c_ll, c_int, c_void_p, c_ll, c_void_p, c_int, c_int, c_int, c_int,
                                        c_void_p, c_void_p, c_void_p]
        lib.lah_gemm_mgroup_fp8.restype = c_int
        lib.lah_gemm_mgroup_fp8.argtypes = [c_void_p, c_ll, c_int, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int,
                                            c_void_p, c_ll, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p, c_ll,
                                            c_int, c_void_p, c_int, c_int, c_void_p, c_int, c_void_p]
        _configured = True
    return lib


def sf_bytes(rows_per_group: int, groups: int, K: int, tile_rows: int) -> int:
    tiles = (rows_per_group + tile_rows - 1) // tile_rows
    return tiles * (K // 128) * ((tile_rows + 127) // 128) * groups * 512


class MXFP8Tensor:
    """e4m3 payload ``q`` (uint8 [groups*rows, K]) + packed UE8M0 scales ``sf`` (uint8, layout above)"""

    def __init__(self, rows_per_group, groups, K, tile_rows, device):
        self.rows_per_group, self.groups, self.K, self.tile_rows = rows_per_group, groups, K, tile_rows
        self.q = torch.empty(rows_per_group * groups, K, dtype=torch.uint8, device=device)
        # scales of rows that are never written (tile padding) must not be NaN (0xFF): zero-initialise once
        self.sf = torch.zeros(sf_bytes(rows_per_group, groups, K, tile_rows), dtype=torch.uint8, device=device)


def quantize(x, *, tile_rows=ACT_TILE, groups=1, out: MXFP8Tensor = None, tile_group=None, total_rows=None):
    """
    :param x: [groups * rows_per_group, K] bf16 or fp32 (row stride arbitrary, unit column stride), K % 128 == 0
    :param tile_group: optional int32 per-128-row-tile expert map; tiles with -1 are skipped
    """
    assert x.is_cuda and x.dim() == 2 and x.stride(1) == 1 and x.dtype in (torch.bfloat16, torch.float32)
    rows, K = x.shape
    assert rows % groups == 0 and K % 128 == 0
    if out is None:
        out = MXFP8Tensor(rows // groups, groups, K, tile_rows, x.device)
    assert out.K == K and out.groups == groups and out.rows_per_group == rows // groups and out.tile_rows == tile_rows
    # the kernel reads 32 input elements and writes 32 payload bytes per thread as 16-byte vectors
    if (x.stride(0) * x.element_size()) % 16 or x.data_ptr() % 16 or out.q.data_ptr() % 16:
        raise ValueError(f"quantize: the input row stride and both bases must be multiples of 16 bytes (input stride "
                         f"{x.stride(0)}, address {x.data_ptr():#x}; payload address {out.q.data_ptr():#x})")
    code = _lib().lah_quant_mxfp8(ptr(x), x.stride(0), int(x.dtype == torch.float32), ptr(out.q), out.q.stride(0),
                                  ptr(out.sf), rows // groups, groups, K, tile_rows, ptr(tile_group), ptr(total_rows),
                                  stream_ptr())
    native.check(code, "lah_quant_mxfp8")
    native.count_launch()
    return out


def grouped_linear_fp8(a: MXFP8Tensor, w: MXFP8Tensor, *, tile_group=None, bias=None, residual=None, out=None,
                       out_dtype=torch.bfloat16, m_valid=None, max_ctas=0, wait=None, act=0):
    """out[r, :] = dequant(a)[r, :] @ dequant(w)[g(r)]^T (+ bias[g(r)]) (+ act) (+ residual[r, :]);  groups padded to 256 rows"""
    assert a.tile_rows == ACT_TILE and w.tile_rows == WEIGHT_TILE and a.groups == 1 and a.K == w.K
    rows, K = a.q.shape
    G, N = w.groups, w.rows_per_group
    num_m_tiles = (rows + 127) // 128
    if out is None:
        out = torch.empty(rows, N, device=a.q.device, dtype=out_dtype)
    assert out.stride(1) == 1 and out.dtype in (torch.bfloat16, torch.float32)
    gemm._check_pairs(out, "out", 2 * out.element_size())
    if tile_group is not None:
        assert tile_group.dtype == torch.int32 and tile_group.numel() >= num_m_tiles
    if bias is not None:
        assert bias.dtype == torch.float32 and bias.is_contiguous() and bias.numel() == G * N
        gemm._check_pairs(bias, "bias", 8)
    if residual is not None:
        assert residual.dtype == torch.bfloat16 and residual.stride(1) == 1
        gemm._check_pairs(residual, "residual", 4)
    wait_flags, wait_count, wait_epoch, wait_status = None, 0, 0, None
    if wait is not None:
        wait_flags, wait_epoch, wait_status = wait
        wait_count = wait_flags.numel()
    code = _lib().lah_gemm_mgroup_fp8(
        ptr(a.q), a.q.stride(0), rows, ptr(a.sf), ptr(w.q), ptr(w.sf), G, N, K, ptr(out), out.stride(0),
        int(out.dtype == torch.float32), rows if m_valid is None else m_valid, num_m_tiles, ptr(tile_group), ptr(bias),
        ptr(residual), residual.stride(0) if residual is not None else 0, max_ctas, ptr(wait_flags), wait_count,
        wait_epoch, ptr(wait_status), int(act), stream_ptr())
    native.check(code, "lah_gemm_mgroup_fp8")
    native.count_launch()
    return out


# ---------------------------------------------------------------------------------------------------------
# PyTorch oracles
# ---------------------------------------------------------------------------------------------------------
def quantize_ref(x):
    """(q float8_e4m3fn [rows, K], exponent int32 [rows, K/32]) with the kernel's rule: the smallest power-of-two scale
    such that amax / scale <= 448"""
    rows, K = x.shape
    xb = x.float().view(rows, K // 32, 32)
    amax = xb.abs().amax(-1)
    s = amax / 448.0
    bits = s.view(torch.int32)
    e = ((bits >> 23) & 0xFF) + ((bits & 0x7FFFFF) != 0).to(torch.int32)
    e = e.clamp(1, 253)
    inv = ((254 - e) << 23).view(torch.float32)
    q = (xb * inv.unsqueeze(-1)).to(torch.float8_e4m3fn).view(rows, K)
    return q, e


def dequantize_ref(q, e):
    rows, K = q.shape
    scale = (e << 23).view(torch.float32)
    return (q.float().view(rows, K // 32, 32) * scale.unsqueeze(-1)).view(rows, K)


def unpack_sf(t: MXFP8Tensor):
    """packed scale bytes -> int32 exponents [groups * rows_per_group, K / 32] (inverse of the kernel's layout)"""
    R, G, K, T = t.rows_per_group, t.groups, t.K, t.tile_rows
    atoms, num_kb, tiles = (T + 127) // 128, K // 128, (R + T - 1) // T
    dev = t.sf.device
    r = torch.arange(R, device=dev)
    tile, rt = r // T, r % T
    atom, ra = rt // 128, rt % 128
    kb32 = torch.arange(K // 32, device=dev)
    g = torch.arange(G, device=dev)
    chunk = ((g[:, None, None] * tiles + tile[None, :, None]) * num_kb + (kb32 // 4)[None, None, :]) * atoms + atom[None, :, None]
    byte = chunk * 512 + (((ra % 32) * 4 + ra // 32) * 4)[None, :, None] + (kb32 % 4)[None, None, :]
    return t.sf[byte.reshape(-1)].to(torch.int32).view(G * R, K // 32)
