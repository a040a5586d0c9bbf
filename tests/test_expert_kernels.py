"""
The kernels of the expert hot path, one by one, element by element against float64 oracles: the grouped GEMM
(csrc/grouped_gemm.cu, M-grouped forward / dgrad and K-grouped wgrad), the swap-AB small-M linear (csrc/small_m.cu), the
LayerNorm forward / backward and grouped column sums (csrc/layernorm.cu) and the fused Adam step with its helpers
(csrc/adam.cu).

Every oracle is computed in float64 from the same bf16 / fp32 operands the kernel reads.  Each element is compared with its
own error bound, never one norm over a whole output.  For a GEMM the bound at (i, j) is

    |out - ref| <= eps_out |ref| + (1 + eps_out) E,    E = C_ACC K 2^-24 (|A| |B|)[i, j] + (bias, residual, activation terms)

with eps_out = 2^-8 for a bf16 output and 2^-23 for fp32, and (|A| |B|) the float64 product of the absolute values.  The
LayerNorm and Adam bounds are built the same way from the magnitudes of the terms each fp32 operation combines, with the
depth of every fp32 summation in place of K.  C_ACC is the one constant of all of them.  Results that are exact are compared
exactly: dropped elements with a residual, the bf16 mirrors, the padding rows of swap-AB, and every byte a kernel must not
touch (sentinel-filled canary rows and columns).  Two identical calls must give byte-equal results.

The CPU tests check the oracles themselves against torch.autograd and torch.optim.Adam, and the host-side refusals of the C
entry points, which return before anything reaches the device.
"""
import ctypes

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import lah_b200  # noqa: F401
from lah_b200.ops import kernels as K

BF16 = torch.bfloat16
U = 2.0 ** -24         # unit roundoff of fp32
EPS_BF16 = 2.0 ** -8
EPS_F32 = 2.0 ** -23
C_ACC = 4              # the constant of every error bound in this file
LN_EPS = 1e-5
SENTINEL = 0x7B        # canary byte: 0x7b7b (bf16) and 0x7b7b7b7b (fp32) are ~1.3e36, which no kernel here produces

WORST = {}             # kernel -> worst observed |error| / bound


def note(kernel, ratio):
    WORST[kernel] = max(WORST.get(kernel, 0.0), float(ratio))


@pytest.fixture(scope="module", autouse=True)
def report_worst_ratios():
    yield
    if WORST:
        print("\nworst |error| / bound per kernel: " + ", ".join(f"{k} {v:.3g}" for k, v in sorted(WORST.items())))


def within(got, ref, bound, what, kernel):
    """every element of got within its own bound of the float64 ref; returns the worst error / bound"""
    err = (got.double() - ref).abs()
    bad = ~(err <= bound)
    if bad.any():
        i = bad.nonzero()[0].tolist()
        raise AssertionError(f"{what}: {int(bad.sum())} of {bad.numel()} elements outside their bound; first at {i}: "
                             f"got {got[tuple(i)].item()!r}, ref {ref[tuple(i)].item()!r}, bound {bound[tuple(i)].item():.3g}")
    ratio = (err / (bound + 1e-300)).max().item() if err.numel() else 0.0
    note(kernel, ratio)
    return ratio


def sentinel_like(shape, dtype, device="cuda"):
    t = torch.empty(shape, dtype=dtype, device=device)
    t.view(torch.uint8).fill_(SENTINEL)
    return t


def untouched(t):
    """bool mask of the elements that still hold the canary pattern"""
    ref = sentinel_like((1,), t.dtype, t.device)
    return t.contiguous().view(torch.uint8).view(*t.shape, t.element_size()).eq(ref.view(torch.uint8)).all(-1)


def gelu64(x):
    return 0.5 * x * (1.0 + torch.special.erf(x / 2 ** 0.5))


def f32(x):
    """a Python float as the fp32 value a kernel receives through ctypes"""
    return float(np.float32(x))


# ---------------------------------------------------------------------------------------------------------------- oracles
def ln_fwd64(h, gamma, beta, relu):
    """float64 LayerNorm(+ReLU) of the bf16 rows h with per-row affine parameters; returns (y, mean, rstd, bound terms)"""
    x = h.double()
    C = x.shape[1]
    mu = x.mean(1, keepdim=True)
    var = ((x - mu) ** 2).mean(1, keepdim=True)
    rstd = (var + LN_EPS).rsqrt()
    xhat = (x - mu) * rstd
    y = xhat * gamma.double() + beta.double()
    if relu:
        y = y.clamp(min=0)
    # fp32 one-pass statistics: sum and sum of squares over C / 32 sequential terms per lane, then a 5-level warp tree
    D = C // 32 + 8
    e_abs, e_sq = x.abs().mean(1, keepdim=True), (x * x).mean(1, keepdim=True)
    d_mean = C_ACC * U * D * e_abs
    d_var = C_ACC * U * D * (e_sq + 2 * mu.abs() * e_abs) + 2 * U * mu * mu
    d_rstd = 0.5 * d_var / (var + LN_EPS) + 4 * U                           # relative (rsqrtf: 2 ulp)
    g = gamma.double().abs()
    xabs = (x.abs() + mu.abs()) * rstd
    e_y = g * (xhat.abs() * d_rstd + rstd * d_mean + 3 * U * xabs) + 2 * U * (xhat.abs() * g + beta.double().abs())
    return y, mu.squeeze(1), rstd.squeeze(1), dict(e_y=e_y, d_mean=d_mean.squeeze(1), d_rstd=d_rstd.squeeze(1))


def ln_bwd64(da, h, mean, rstd, gamma, beta, relu, dres=None):
    """float64 LayerNorm(+ReLU) backward per row from the statistics the kernel reads; returns (dh, g o xhat, g, y)
    with g = da masked by the ReLU; the per-group column sums of the last three and of dh are the parameter gradients"""
    x = (h.double() - mean.double()[:, None]) * rstd.double()[:, None]
    y = x * gamma.double() + beta.double()
    g = da.double() * (y > 0) if relu else da.double()
    dxh = g * gamma.double()
    dh = rstd.double()[:, None] * (dxh - dxh.mean(-1, keepdim=True) - x * (dxh * x).mean(-1, keepdim=True))
    if dres is not None:
        dh = dh + dres.double()
    return dh, g * x, g, y


def adam_layout(seg_sizes, G):
    """(segment, group) of every element of the flat [G, seg_sizes[s]] segments"""
    seg, grp = [], []
    for s, n in enumerate(seg_sizes):
        seg.append(torch.full((G * n,), s, dtype=torch.long))
        grp.append(torch.arange(G).repeat_interleave(n))
    return torch.cat(seg), torch.cat(grp)


def adam_ref64(p, g, m, v, vmax, seg_sizes, G, *, step, group_rows=None, lr=1e-3, betas=(0.9, 0.999), eps=1e-8,
               weight_decay=0.0, amsgrad=True, zero_mask=0, G_active=0, seg_mask=0, grad=None, zero_grad=True):
    """
    float64 oracle of ``adam_step`` (csrc/adam.cu) over flat segments [G, seg_sizes[s]].  An element of group gi and segment s
    is updated iff gi < G_active (0: all), group_rows[gi] > 0 and (seg_mask == 0 or bit s of seg_mask).  ``step`` is an int
    per group or one int for all.  ``grad`` replaces g as the gradient (peer reduce); ``zero_grad`` = False keeps g as it was
    (the peer-reduce branch never zeroes).  Returns (dict of new p, m, v, vmax, g as float64, bool update mask, bounds).
    """
    seg, grp = adam_layout(seg_sizes, G)
    dev = p.device
    seg, grp = seg.to(dev), grp.to(dev)
    upd = grp < (G_active or G)
    if group_rows is not None:
        upd &= group_rows.to(dev).long()[grp] > 0
    if seg_mask:
        upd &= ((seg_mask >> seg) & 1).bool()
    stepv = (step.to(dev).double()[grp] if torch.is_tensor(step) else torch.full_like(p, float(step), dtype=torch.float64))
    b1, b2 = betas
    P, Gr, M, V, VM = (t.double() for t in (p, g, m, v, vmax))
    gr = (Gr if grad is None else grad.double()) + weight_decay * P
    m1 = M + (1 - b1) * (gr - M)
    v1 = V * b2 + (1 - b2) * gr * gr
    vh = torch.maximum(VM, v1) if amsgrad else v1
    bc1, bc2 = 1 - b1 ** stepv, 1 - b2 ** stepv
    denom = vh.sqrt() / bc2.sqrt() + eps
    step_size = lr / bc1
    delta = step_size * (m1 / denom)
    p1 = P - delta
    new = dict(p=torch.where(upd, p1, P), m=torch.where(upd, m1, M), v=torch.where(upd, v1, V),
               vmax=torch.where(upd, vh, VM) if amsgrad else VM,
               g=torch.where(upd & ((zero_mask >> seg) & 1).bool(), torch.zeros_like(Gr), Gr) if zero_grad else Gr)
    # bounds: powf of the fast-math build is exp2(step * log2(beta)) with approximate exp2 / log2: abs error ~ step 2^-22
    d_bc = C_ACC * (stepv + 1) * 2.0 ** -22
    e_m = C_ACC * U * (M.abs() + gr.abs() + (weight_decay * P).abs() + 2 * (Gr if grad is None else grad.double()).abs())
    e_v = C_ACC * 4 * U * (V * b2 + (1 - b2) * gr * gr)
    rel = d_bc / bc1 + 0.5 * d_bc / bc2 + 16 * C_ACC * U
    e_p = delta.abs() * rel + step_size * e_m / denom + U * p1.abs()
    bounds = dict(p=e_p, m=e_m, v=e_v, vmax=e_v)
    return new, upd, bounds


# ---------------------------------------------------------------------------------------------------------------- CPU
@pytest.mark.parametrize("relu", [False, True])
def test_ln_fwd_oracle_matches_torch_layer_norm(relu):
    gen = torch.Generator().manual_seed(1)
    h = (torch.randn(37, 256, generator=gen) * 3 + 1).to(BF16)
    gamma, beta = torch.randn(256, generator=gen), torch.randn(256, generator=gen)
    y, mu, rstd, _ = ln_fwd64(h, gamma, beta, relu)
    ref = F.layer_norm(h.double(), (256,), gamma.double(), beta.double(), LN_EPS)
    torch.testing.assert_close(y, F.relu(ref) if relu else ref, rtol=1e-12, atol=1e-12)
    torch.testing.assert_close(mu, h.double().mean(1), rtol=1e-14, atol=1e-14)
    torch.testing.assert_close(rstd, 1 / (h.double().var(1, unbiased=False) + LN_EPS).sqrt(), rtol=1e-12, atol=0)


@pytest.mark.parametrize("relu", [False, True])
@pytest.mark.parametrize("with_dres", [False, True])
def test_ln_bwd_oracle_matches_autograd(relu, with_dres):
    """dh = d/dh [sum(da o act(LN(h))) + sum(dres o h)]; dgamma, dbeta = autograd's; dbias = the column sum of dh"""
    gen = torch.Generator().manual_seed(2)
    h = (torch.randn(29, 512, generator=gen) * 2 - 0.5).to(BF16)
    gamma, beta = torch.randn(512, generator=gen), torch.randn(512, generator=gen)
    da = torch.randn(29, 512, generator=gen).to(BF16)
    dres = torch.randn(29, 512, generator=gen).to(BF16) if with_dres else None
    hd = h.double().requires_grad_()
    gd, bd = gamma.double().requires_grad_(), beta.double().requires_grad_()
    y = F.layer_norm(hd, (512,), gd, bd, LN_EPS)
    loss = ((F.relu(y) if relu else y) * da.double()).sum()
    if with_dres:
        loss = loss + (hd * dres.double()).sum()
    loss.backward()
    mean = h.double().mean(1)
    rstd = 1 / (h.double().var(1, unbiased=False) + LN_EPS).sqrt()
    dh, gx, g, _ = ln_bwd64(da, h, mean, rstd, gamma, beta, relu, dres)
    torch.testing.assert_close(dh, hd.grad, rtol=1e-10, atol=1e-12)
    torch.testing.assert_close(gx.sum(0), gd.grad, rtol=1e-10, atol=1e-12)
    torch.testing.assert_close(g.sum(0), bd.grad, rtol=1e-10, atol=1e-12)
    torch.testing.assert_close(dh.sum(0), hd.grad.sum(0), rtol=1e-10, atol=1e-11)


@pytest.mark.parametrize("amsgrad", [True, False])
@pytest.mark.parametrize("weight_decay", [0.0, 0.05])
def test_adam_oracle_matches_torch_optim_step_for_step(amsgrad, weight_decay):
    gen = torch.Generator().manual_seed(3)
    G, n, lr, betas, eps = 1, 64, 3e-3, (0.8, 0.99), 1e-6
    w = torch.nn.Parameter(torch.randn(n, generator=gen, dtype=torch.float64))
    opt = torch.optim.Adam([w], lr=lr, betas=betas, eps=eps, weight_decay=weight_decay, amsgrad=amsgrad)
    p, m, v, vmax = w.detach().clone(), torch.zeros(n, dtype=torch.float64), torch.zeros(n, dtype=torch.float64), \
        torch.zeros(n, dtype=torch.float64)
    for step in range(1, 7):
        grad = torch.randn(n, generator=gen, dtype=torch.float64) * (0.1 if step % 2 else 2.0)
        w.grad = grad.clone()
        opt.step()
        new, upd, _ = adam_ref64(p, grad, m, v, vmax, [n], G, step=step, lr=lr, betas=betas, eps=eps,
                                 weight_decay=weight_decay, amsgrad=amsgrad)
        assert bool(upd.all())
        p, m, v, vmax = new["p"], new["m"], new["v"], new["vmax"]
        st = opt.state[w]
        torch.testing.assert_close(p, w.detach(), rtol=1e-13, atol=1e-15)
        torch.testing.assert_close(m, st["exp_avg"], rtol=1e-13, atol=1e-15)
        torch.testing.assert_close(v, st["exp_avg_sq"], rtol=1e-13, atol=1e-18)
        if amsgrad:
            torch.testing.assert_close(vmax, st["max_exp_avg_sq"], rtol=1e-13, atol=1e-18)


def test_adam_oracle_segment_range_and_shadow_slot_indexing_by_hand():
    """segments [3 groups x 4] then [3 x 8]: group 0 of segment 1 is the flat range [12, 20).  With G_active = 2 group 2 is a
    shadow slot, group 1 received no rows, and seg_mask = 0b10 leaves only segment 1: exactly [12, 20) is stepped.  At step 1
    with eps = 0, Adam moves every parameter by lr against the sign of its gradient."""
    G, segs = 3, [4, 8]
    n = G * sum(segs)
    p, g = torch.ones(n, dtype=torch.float64), torch.full((n,), 0.5, dtype=torch.float64)
    z = torch.zeros(n, dtype=torch.float64)
    rows = torch.tensor([1, 0, 5])
    kw = dict(step=torch.tensor([1, 4, 9]), group_rows=rows, lr=0.1, eps=0.0, G_active=2)
    new, upd, _ = adam_ref64(p, g, z, z, z, segs, G, seg_mask=0b10, zero_mask=0b11, **kw)
    assert upd.nonzero().squeeze(1).tolist() == list(range(12, 20))
    assert torch.allclose(new["p"][12:20], torch.full((8,), 0.9, dtype=torch.float64), rtol=0, atol=1e-15)
    assert bool((new["p"][upd.logical_not()] == 1).all())
    assert new["g"].eq(0).nonzero().squeeze(1).tolist() == list(range(12, 20))
    # without seg_mask: group 0 of segment 0 ([0, 4)) too; zero_mask bit 0 alone zeroes only that one
    new, upd, _ = adam_ref64(p, g, z, z, z, segs, G, zero_mask=0b01, **kw)
    assert upd.nonzero().squeeze(1).tolist() == list(range(0, 4)) + list(range(12, 20))
    assert new["g"].eq(0).nonzero().squeeze(1).tolist() == list(range(0, 4))
    # a per-element step: group 2's elements use step 9 once it is active
    new, upd, _ = adam_ref64(p, g, z, z, z, segs, G, **dict(kw, G_active=0, group_rows=None))
    assert bool(upd.all())


# The C entry points are called with fake device addresses that only their host checks look at.  Should a check ever stop
# refusing, the call would go on to a launch on those addresses, so these tests run only where there is no device: there
# a missing check shows as a wrong return code.  With a device, the wrappers' own refusals are tested instead
# (test_grouped_linear_refuses_misaligned_epilogue_operands).
host_abi_only = pytest.mark.skipif(torch.cuda.is_available(), reason="fake device addresses: run only without a device")


def _lib():
    from lah_b200 import build_native
    try:
        build_native._nvcc()
    except RuntimeError:
        pytest.skip("nvcc not found")
    from lah_b200.ops import gemm
    gemm._lib()
    return K._lib()


def _mgroup(lib, *, ldc=512, C=0x100000, out_f32=0, residual=0, ldr=0, bias=0, lda=64, K_=64, N=512):
    """lah_gemm_mgroup with fake (never dereferenced) device addresses: only the host checks before the launch run"""
    v = ctypes.c_void_p
    return lib.lah_gemm_mgroup(v(0x200000), lda, 128, v(0x300000), 1, N, K_, 0, v(C), ldc, out_f32, 128, 1, v(0),
                               v(bias), v(residual), ldr, 256, 0, v(0), 0, 0, v(0), 0, 0, -1, 1.0, 0, v(0))


@host_abi_only
def test_gemm_c_abi_refuses_misaligned_epilogue_operands():
    lib = _lib()
    assert _mgroup(lib, ldc=511) == -2                                    # odd ldc
    assert _mgroup(lib, C=0x100002) == -2                                 # bf16 C off its 4-byte pairs
    assert _mgroup(lib, C=0x100004, out_f32=1) == -2                      # fp32 C off its 8-byte pairs
    assert _mgroup(lib, residual=0x400000, ldr=511) == -2                 # odd ldr
    assert _mgroup(lib, residual=0x400002, ldr=512) == -2                 # residual off its 4-byte pairs
    assert _mgroup(lib, bias=0x500004) == -2                              # bias off float2
    assert _mgroup(lib, lda=60) == -2 and _mgroup(lib, K_=60) == -2 and _mgroup(lib, N=80) == -2
    v = ctypes.c_void_p
    kg = lambda C, ldc, stride: lib.lah_gemm_kgroup(v(0x200000), 128, v(0x300000), 64, 256, 1, 128, 64, v(0x600000),
                                                    v(C), ldc, stride, 64, 0, 0, v(0))
    assert kg(0x100004, 64, 128 * 64) == -2 and kg(0x100000, 63, 128 * 64) == -2 and kg(0x100000, 64, 8191) == -2


@host_abi_only
def test_swapab_linear_host_abi_refusals():
    lib = _lib()
    v = ctypes.c_void_p
    # 1024 groups: the prefix table of 128-token chunks holds at most MAX_G = 1023
    assert lib.lah_swapab_linear(v(0x200000), 64, 128, v(0x300000), 1024, 128, 64, 0, v(0x400000), 128, v(0x500000),
                                 v(0x600000), v(0), v(0), 0, v(0), 0, 0, v(0), 0, v(0)) == -2


@host_abi_only
def test_adam_step_host_abi_refusals():
    lib = _lib()
    v = ctypes.c_void_p
    # every case by value (lr_dev NULL) and with a device rate block (a fake address)
    for lr_dev in (0, 0x600000):
        def adam(segs=(4, 8), l2=0.0, decay=1.0, decoupled=0):
            arr = (ctypes.c_longlong * len(segs))(*segs)
            return lib.lah_adam_step(v(0x100000), v(0x200000), v(0x300000), v(0x400000), v(0x500000), v(0), len(segs),
                                     ctypes.cast(arr, v), 2, v(0), v(0), 1, 1e-3, v(lr_dev), 0.9, 0.999, 1e-8, l2, 1, 0, 1,
                                     -1, v(0), 1.0, 0, v(0), -1, 0, 0, 0, decay, decoupled, v(0))
        # the controls: these arguments pass the host checks, with either decay form
        assert adam() != -2 and adam(l2=0.1) != -2 and adam(decay=0.99, decoupled=1) != -2, lr_dev
        for segs in ((4,) * 13, (4, 6, 8), ()):           # 13 segments, a size not a multiple of 4, no segment at all
            assert adam(segs) == -2 and adam(segs, l2=0.1) == -2 and adam(segs, decay=0.99, decoupled=1) == -2, segs
        assert adam(l2=0.1, decay=0.99, decoupled=1) == -2, lr_dev     # L2 and decoupled decay at once


# ---------------------------------------------------------------------------------------------------------------- GPU
def cuda_randn(gen, *shape, scale=1.0, dtype=torch.float32):
    return (torch.randn(*shape, generator=gen) * scale).to(dtype).cuda()


def gemm_epilogue64(pre, mag, K, *, bias=None, act=0, keep=None, p=0.0, residual=None, out_f32=False, extra=None):
    """float64 epilogue of the grouped GEMM over the product pre = A B and mag = |A| |B|: (ref, bound).  ``extra`` is an
    error of the product that is not an fp32 summation (the FP8 tensor core's in-block accumulation)"""
    e = C_ACC * K * U * mag
    if extra is not None:
        e = e + extra
    if bias is not None:
        pre = pre + bias
        e = e + 2 * U * (pre.abs() + bias.abs())
    if act == 1:
        ref = pre.clamp(min=0)          # ReLU is 1-Lipschitz: an element at the kink stays within e
    elif act == 2:
        ref = gelu64(pre)               # |gelu'| <= 1.13
        e = 1.13 * e + 16 * U * pre.abs()
    else:
        ref = pre
    if keep is not None:
        scale = 1.0 / (1.0 - p)
        ref = torch.where(keep, ref * scale, torch.zeros_like(ref))
        e = torch.where(keep, e * scale + 2 * U * ref.abs(), torch.zeros_like(e))
    if residual is not None:
        r = residual.double()
        ref = ref + r
        e = e + U * (ref.abs() + r.abs())
    eps = EPS_F32 if out_f32 else EPS_BF16
    return ref, eps * ref.abs() + (1 + eps) * e


def tiles_of(rows_per_group, align=128, unused_tail=True):
    """tile_group of ragged groups padded to `align` rows: an unused tile before group 1 and (unused_tail) one at the end"""
    tiles = []
    for g, r in enumerate(rows_per_group):
        if g == 1:
            tiles.append(-1)
        tiles += [g] * (-(-r // align) * (align // 128))
    return tiles + [-1] * unused_tail


def run_mgroup(seed, rows_per_group, N, K_, *, block_n, w_is_kn=False, out_f32=False, bias=False, residual=False, act=0,
               align=128, m_valid_cut=0, max_ctas=0, strided=False, dropout=None):
    from lah_b200.ops import gemm
    gen = torch.Generator().manual_seed(seed)
    # with m_valid the last tiles belong to the last group, so the rows >= m_valid that must stay untouched are rows the
    # kernel would otherwise compute
    tiles = tiles_of(rows_per_group, align, unused_tail=not m_valid_cut)
    rows, G = len(tiles) * 128, len(rows_per_group)
    m_valid = rows - m_valid_cut
    assert not m_valid_cut or tiles[(m_valid - 1) // 128] >= 0 and tiles[-1] >= 0
    pad = 16 if strided else 0          # column slices of wider tensors: 16-byte aligned bases and strides
    a = cuda_randn(gen, rows, K_ + 3 * pad, dtype=BF16)[:, pad:pad + K_]
    w = cuda_randn(gen, G, *((K_, N) if w_is_kn else (N, K_)), scale=K_ ** -0.5, dtype=BF16)
    b = cuda_randn(gen, G, N) if bias else None
    res = cuda_randn(gen, rows, N + 3 * pad, dtype=BF16)[:, pad:pad + N] if residual else None
    out_full = sentinel_like((rows, N + 3 * pad), torch.float32 if out_f32 else BF16)
    out = out_full[:, pad:pad + N]
    tg = torch.tensor(tiles, dtype=torch.int32, device="cuda")
    call = lambda: gemm.grouped_linear(a, w, tile_group=tg, bias=b, residual=res, w_is_kn=w_is_kn, out=out,
                                       m_valid=m_valid if m_valid_cut else None, block_n=block_n, max_ctas=max_ctas,
                                       act=act, dropout=dropout)
    call()
    first = out_full.clone()
    out_full.view(torch.uint8).fill_(SENTINEL)
    call()
    torch.cuda.synchronize()
    assert torch.equal(first.view(torch.uint8), out_full.view(torch.uint8)), "two identical calls differ"
    # float64 oracle over the rows of every used tile
    grow = tg.long().repeat_interleave(128)
    valid = (grow >= 0) & (torch.arange(rows, device="cuda") < m_valid)
    pre = torch.zeros(rows, N, dtype=torch.float64, device="cuda")
    mag = torch.zeros_like(pre)
    for t, g in enumerate(tiles):
        if g >= 0:
            wg = w[g].double()
            B = wg if w_is_kn else wg.t()
            sl = slice(t * 128, (t + 1) * 128)
            pre[sl] = a[sl].double() @ B
            mag[sl] = a[sl].double().abs() @ B.abs()
    keep = K.dropout_mask((rows, N), dropout[0], dropout[1], dropout[2]) if dropout and dropout[0] > 0 else None
    ref, bound = gemm_epilogue64(pre, mag, K_, bias=b.double()[grow.clamp(min=0)] if bias else None, act=act, keep=keep,
                                 p=dropout[0] if dropout else 0.0, residual=res, out_f32=out_f32)
    ratio = within(out[valid], ref[valid], bound[valid], "grouped_linear", "grouped_linear")
    # canaries: rows of -1 tiles and rows >= m_valid, and the columns around the slice
    assert bool(untouched(out[~valid]).all()), "rows the kernel must skip were written"
    if pad:
        assert bool(untouched(out_full[:, :pad]).all()) and bool(untouched(out_full[:, pad + N:]).all())
    if keep is not None and residual:
        dropped = valid[:, None] & ~keep
        assert dropped.any() and torch.equal(out[dropped], res[dropped]), "a dropped element differs from its residual"
    return out_full, ratio


MGROUP_CASES = {
    "bn256_k200_n320_bias_res_strided": dict(rows_per_group=[300, 0, 77, 128], N=320, K_=200, block_n=256, bias=True,
                                             residual=True, strided=True),
    "bn256_kn_k72_res": dict(rows_per_group=[130, 5], N=512, K_=72, block_n=256, w_is_kn=True, residual=True),
    "bn256_align256_relu": dict(rows_per_group=[128, 300, 0, 1000], N=512, K_=200, block_n=256, bias=True, act=1, align=256),
    "bn256_kn_f32_ctas3": dict(rows_per_group=[200, 1, 260], N=320, K_=200, block_n=256, w_is_kn=True, out_f32=True,
                               residual=True, max_ctas=3),
    "bn128_k24_n96_f32_relu": dict(rows_per_group=[1, 200], N=96, K_=24, block_n=128, out_f32=True, bias=True, act=1),
    "bn128_kn_n320_gelu_f32": dict(rows_per_group=[129, 0, 40], N=320, K_=200, block_n=128, w_is_kn=True, out_f32=True,
                                   act=2, residual=True),
    "bn128_mvalid_ctas1": dict(rows_per_group=[300, 77], N=384, K_=200, block_n=128, bias=True, m_valid_cut=77,
                               max_ctas=1),
    "bn64_k72_n96_gelu_strided_ctas3": dict(rows_per_group=[50, 0, 140], N=96, K_=72, block_n=64, bias=True, residual=True,
                                            act=2, strided=True, max_ctas=3, m_valid_cut=200),
    "bn64_kn_k24_f32_strided": dict(rows_per_group=[256, 3], N=64, K_=24, block_n=64, w_is_kn=True, out_f32=True,
                                    residual=True, strided=True, act=1),
    "bn64_k200_ctas1": dict(rows_per_group=[20, 300], N=160, K_=200, block_n=64, bias=True, max_ctas=1),
}


@pytest.mark.gpu
@pytest.mark.parametrize("case", list(MGROUP_CASES))
def test_grouped_linear_elementwise(case, record_property):
    _, ratio = run_mgroup(list(MGROUP_CASES).index(case), **MGROUP_CASES[case])
    record_property("max_err_over_bound", ratio)


@pytest.mark.gpu
@pytest.mark.parametrize("site,p,act,residual", [(1, 0.1, 0, True), (1, 0.5, 0, False), (2, 0.1, 2, False),
                                                 (2, 0.5, 1, False), (3, 0.1, 0, True), (3, 0.5, 0, True)])
def test_grouped_linear_dropout_epilogue(site, p, act, residual, record_property):
    """N = 320: the second n tile and the mask granules straddle N; with a residual every dropped element IS the residual"""
    _, ratio = run_mgroup(17 * site, [300, 0, 77, 128], 320, 200, block_n=256, bias=True, residual=residual, act=act,
                          dropout=(p, 1234 + site, site))
    record_property("max_err_over_bound", ratio)


@pytest.mark.gpu
def test_grouped_linear_dropout_p0_is_no_dropout():
    """a contract of the wrapper, not of the kernel: p = 0 must launch the instantiation without dropout (the Python side
    maps it to threshold -1), so a model with dropout 0 computes exactly what one without dropout computes"""
    kw = dict(rows_per_group=[300, 77], N=320, K_=200, block_n=256, bias=True, residual=True, act=2)
    plain, _ = run_mgroup(5, **kw)
    p0, _ = run_mgroup(5, **kw, dropout=(0.0, 99, 2))
    assert torch.equal(plain.view(torch.uint8), p0.view(torch.uint8))


KGROUP_CASES = [  # block_n, N, M, rows per group, accumulate, max_ctas
    (64, 32, 128, [128, 0, 300, 77], False, 0),
    (128, 96, 256, [0, 512, 130], True, 1),
    (256, 96, 128, [1000, 0, 64], True, 0),
    (256, 32, 256, [5, 0], False, 1),
    (128, 32, 384, [300], False, 3),
    (64, 96, 128, [0, 640, 1], True, 1),
]


@pytest.mark.gpu
@pytest.mark.parametrize("block_n,N,M,rows_per_group,accumulate,max_ctas", KGROUP_CASES)
def test_grouped_wgrad_elementwise(block_n, N, M, rows_per_group, accumulate, max_ctas, record_property):
    from lah_b200.ops import gemm
    gen = torch.Generator().manual_seed(block_n + N + M)
    G = len(rows_per_group)
    off = [0]
    for r in rows_per_group:
        off.append(off[-1] + -(-r // 128) * 128)
    rows = off[-1] + 128                                   # trailing rows in no group
    dy, x = cuda_randn(gen, rows, M, dtype=BF16), cuda_randn(gen, rows, N, dtype=BF16)
    go = torch.tensor(off, dtype=torch.int32, device="cuda")
    out0 = cuda_randn(gen, G, M, N) if accumulate else sentinel_like((G, M, N), torch.float32)
    out = out0.clone()
    gemm.grouped_wgrad(dy, x, go, G, out=out, block_n=block_n, max_ctas=max_ctas, accumulate=accumulate)
    first = out.clone()
    out.copy_(out0)
    gemm.grouped_wgrad(dy, x, go, G, out=out, block_n=block_n, max_ctas=max_ctas, accumulate=accumulate)
    torch.cuda.synchronize()
    assert torch.equal(first.view(torch.uint8), out.view(torch.uint8)), "two identical calls differ"
    ratio = 0.0
    for g in range(G):
        if off[g + 1] == off[g]:
            assert torch.equal(out[g].view(torch.uint8), out0[g].view(torch.uint8)), f"empty group {g} was written"
            continue
        sl = slice(off[g], off[g + 1])
        ref = dy[sl].double().t() @ x[sl].double()
        e = C_ACC * (off[g + 1] - off[g]) * U * (dy[sl].double().abs().t() @ x[sl].double().abs())
        if accumulate:
            ref = ref + out0[g].double()
            e = e + U * (ref.abs() + out0[g].double().abs())
        ratio = max(ratio, within(out[g], ref, EPS_F32 * ref.abs() + (1 + EPS_F32) * e, f"group {g}", "grouped_wgrad"))
    record_property("max_err_over_bound", ratio)


@pytest.mark.gpu
def test_grouped_linear_refuses_misaligned_epilogue_operands():
    """the wrapper refuses on the host, before any launch"""
    from lah_b200.ops import gemm
    a = torch.zeros(128, 64, dtype=BF16, device="cuda")
    w = torch.zeros(1, 64, 64, dtype=BF16, device="cuda")
    wide = torch.zeros(128, 130, dtype=BF16, device="cuda")
    with pytest.raises(ValueError):
        gemm.grouped_linear(a, w, out=wide[:, 1:65])                            # bf16 out one element off
    with pytest.raises(ValueError):
        gemm.grouped_linear(a, w, out=torch.zeros(128 * 65, dtype=BF16, device="cuda").view(128, 65)[:, :64])  # odd ldc
    with pytest.raises(ValueError):
        gemm.grouped_linear(a, w, out=torch.zeros(128, 66, device="cuda")[:, 1:65], out_dtype=torch.float32)
    with pytest.raises(ValueError):
        gemm.grouped_linear(a, w, residual=wide[:, 1:65])                      # residual one element off
    with pytest.raises(ValueError):
        gemm.grouped_linear(a, w, residual=torch.zeros(128 * 65, dtype=BF16, device="cuda").view(128, 65)[:, :64])
    with pytest.raises(ValueError):
        gemm.grouped_linear(a, w, bias=torch.zeros(65, device="cuda")[1:])     # bias off float2
    with pytest.raises(ValueError):
        gemm.grouped_wgrad(a, a, torch.tensor([0, 128], dtype=torch.int32, device="cuda"), 1,
                           out=torch.zeros(64 * 64 + 1, device="cuda")[1:].view(1, 64, 64))


# ------------------------------------------------------------------ LayerNorm
LN_TILES = [0, 1, 0, -1, 2, 1]      # group 0's tiles are separated by group 1's, tile 3 unused, a partial last tile


def ln_inputs(seed, C, tile_rows, grouped, offset_ratio=None):
    """rows = 5 full tiles + 1, 3 or 5 rows; rows of very different scale (down to 1e-2, where the eps term matters) and
    offset, or a common offset of `offset_ratio` x the row's standard deviation"""
    gen = torch.Generator().manual_seed(seed)
    rows = 5 * tile_rows + (1, 3, 5)[(C // 256 + tile_rows) % 3]
    n_tiles = -(-rows // tile_rows)
    tiles = LN_TILES[:n_tiles] if grouped else [0] * n_tiles
    scale = 10 ** (torch.rand(rows, 1, generator=gen) * 2.5 - 2)
    if offset_ratio is None:
        offset = (torch.rand(rows, 1, generator=gen) * 4 - 2) * scale
    else:
        offset = offset_ratio * scale * torch.where(torch.rand(rows, 1, generator=gen) < 0.5, -1.0, 1.0)
    h = (torch.randn(rows, C, generator=gen) * scale + offset).to(BF16).cuda()
    G = 3
    gamma = (1 + 0.3 * torch.randn(G, C, generator=gen)).cuda()
    beta = (0.3 * torch.randn(G, C, generator=gen)).cuda()
    tg = torch.tensor(tiles, dtype=torch.int32, device="cuda") if grouped else None
    grow = torch.tensor(tiles, device="cuda").repeat_interleave(tile_rows)[:rows]
    return h, gamma, beta, tg, grow, gen


def check_ln_forward(h, gamma, beta, tg, grow, tile_rows, relu):
    rows, C = h.shape
    out, mean, rstd = sentinel_like((rows, C), BF16), sentinel_like((rows,), torch.float32), sentinel_like((rows,), torch.float32)
    K.ln_relu_fwd(h, gamma, beta, tg, out=out, mean=mean, rstd=rstd, relu=relu, tile_rows=tile_rows)
    torch.cuda.synchronize()
    valid = grow >= 0
    gi = grow.clamp(min=0)
    y, mu, rs, b = ln_fwd64(h[valid], gamma[gi[valid]], beta[gi[valid]], relu)
    r1 = within(out[valid], y, EPS_BF16 * y.abs() + (1 + EPS_BF16) * b["e_y"], "LayerNorm output", "ln_fwd")
    r2 = within(mean[valid], mu, b["d_mean"], "saved mean", "ln_fwd")
    r3 = within(rstd[valid], rs, b["d_rstd"] * rs, "saved rstd", "ln_fwd")
    assert bool(untouched(out[~valid]).all() and untouched(mean[~valid]).all() and untouched(rstd[~valid]).all())
    return out, mean, rstd, max(r1, r2, r3)


@pytest.mark.gpu
@pytest.mark.parametrize("relu", [False, True])
@pytest.mark.parametrize("grouped", [False, True], ids=["tile_group_none", "ragged"])
@pytest.mark.parametrize("tile_rows", [8, 16, 128])
@pytest.mark.parametrize("C", [256, 512, 1024, 2048, 4096])
def test_ln_forward_elementwise(C, tile_rows, grouped, relu, record_property):
    h, gamma, beta, tg, grow, _ = ln_inputs(C + tile_rows, C, tile_rows, grouped)
    record_property("max_err_over_bound", check_ln_forward(h, gamma, beta, tg, grow, tile_rows, relu)[3])


@pytest.mark.gpu
@pytest.mark.parametrize("C", [512, 4096])
def test_ln_forward_rows_with_a_large_common_offset(C, record_property):
    """|mean| = 64 x std: the one-pass fp32 variance E[x^2] - mean^2 loses about 12 bits; still within the normal bound"""
    h, gamma, beta, tg, grow, _ = ln_inputs(C, C, 128, True, offset_ratio=64.0)
    record_property("max_err_over_bound", check_ln_forward(h, gamma, beta, tg, grow, 128, True)[3])


@pytest.mark.gpu
@pytest.mark.parametrize("with_dres", [False, True], ids=["no_dres", "dres"])
@pytest.mark.parametrize("relu", [False, True])
@pytest.mark.parametrize("grouped", [False, True], ids=["tile_group_none", "ragged"])
@pytest.mark.parametrize("tile_rows", [8, 16, 128])
@pytest.mark.parametrize("C", [256, 512, 1024, 2048, 4096])
def test_ln_backward_elementwise(C, tile_rows, grouped, relu, with_dres, record_property):
    h, gamma, beta, tg, grow, gen = ln_inputs(7 * C + tile_rows, C, tile_rows, grouped)
    rows = h.shape[0]
    _, mean, rstd, _ = check_ln_forward(h, gamma, beta, tg, grow, tile_rows, relu)
    valid = grow >= 0
    gi = grow.clamp(min=0)
    gam, bet = gamma[gi], beta[gi]
    da = cuda_randn(gen, rows, C, dtype=BF16)
    # the ReLU mask at an element whose y is within rounding of 0 is either side: such elements get da = 0 (counted: rare)
    _, _, _, y = ln_bwd64(da, h, mean, rstd, gam, bet, relu)
    xabs = (h.double().abs() + mean.double().abs()[:, None]) * rstd.double()[:, None]
    kink = relu & valid[:, None] & (y.abs() <= C_ACC * U * (xabs * gam.double().abs() + bet.double().abs()))
    assert int(kink.sum()) <= max(2, kink.numel() // 10000), int(kink.sum())
    da = da.masked_fill(kink, 0)
    dres = cuda_randn(gen, rows, C, dtype=BF16) if with_dres else None
    d0 = [cuda_randn(gen, 3, C) for _ in range(3)]          # dgamma, dbeta, dbias start non-zero: the kernel adds
    outs = []
    for _ in range(2):
        dh = sentinel_like((rows, C), BF16)
        dg, db, dbias = (t.clone() for t in d0)
        K.ln_relu_bwd(da, h, mean, rstd, gamma, beta, tg, dh=dh, dgamma=dg, dbeta=db, dbias=dbias, relu=relu,
                      tile_rows=tile_rows, dres=dres)
        outs.append((dh, dg, db, dbias))
    torch.cuda.synchronize()
    for a, b in zip(*outs):
        assert torch.equal(a.view(torch.uint8), b.view(torch.uint8)), "two identical calls differ"
    dh, dg, db, dbias = outs[0]
    ref_dh, gx, g, _ = ln_bwd64(da, h, mean, rstd, gam, bet, relu, dres)
    # dh = rstd (g gamma - mean(g gamma) - xhat mean(g gamma xhat)) (+ dres): row means over <= 32 sequential fp32 sums
    D_row = 32
    r = rstd.double()[:, None]
    gg = (g * gam.double()).abs()
    m1, m2 = gg.mean(1, keepdim=True), (gg * xabs).mean(1, keepdim=True)
    e_dh = C_ACC * U * r * (gg + D_row * m1 + xabs * D_row * m2 + 3 * xabs * gg)
    if with_dres:
        e_dh = e_dh + U * ref_dh.abs()
    ratio = within(dh[valid], ref_dh[valid], EPS_BF16 * ref_dh[valid].abs() + (1 + EPS_BF16) * e_dh[valid], "dh", "ln_bwd")
    assert bool(untouched(dh[~valid]).all()), "rows of unused tiles were written"
    # parameter gradients: fp32 column sums over a tile, then over the group's tiles in tile order
    D_col = tile_rows + len(LN_TILES) + 4
    for grp in range(3):
        rows_g = valid & (grow == grp)
        for name, got, terms, mags in (("dgamma", dg, gx, (g.abs() * xabs)), ("dbeta", db, g, g.abs()),
                                       ("dbias", dbias, ref_dh, ref_dh.abs())):
            start = d0[("dgamma", "dbeta", "dbias").index(name)][grp].double()
            ref = start + terms[rows_g].sum(0)
            e = C_ACC * U * (D_col + 4) * mags[rows_g].sum(0) + U * (start.abs() + ref.abs())
            if name == "dbias":
                e = e + e_dh[rows_g].sum(0)
            ratio = max(ratio, within(got[grp], ref, e, f"{name} of group {grp}", "ln_bwd"))
    record_property("max_err_over_bound", ratio)


@pytest.mark.gpu
@pytest.mark.parametrize("tile_rows", [16, 128])
@pytest.mark.parametrize("C", [256, 768])
def test_grouped_colsum_elementwise(C, tile_rows, record_property):
    gen = torch.Generator().manual_seed(C + tile_rows)
    rows = 5 * tile_rows + 3
    tiles = LN_TILES[:-(-rows // tile_rows)]
    grow = torch.tensor(tiles, device="cuda").repeat_interleave(tile_rows)[:rows]
    x = cuda_randn(gen, rows, C + 128, dtype=BF16)[:, 64:64 + C]            # strided: ldx = C + 128 > C
    tg = torch.tensor(tiles, dtype=torch.int32, device="cuda")
    out0 = cuda_randn(gen, 3, C)
    outs = [K.grouped_colsum(x, tg, out=out0.clone(), tile_rows=tile_rows) for _ in range(2)]
    torch.cuda.synchronize()
    assert torch.equal(outs[0], outs[1]), "two identical calls differ"
    D = tile_rows // 4 + 4 + len(tiles) + 2
    ratio = 0.0
    for grp in range(3):
        xs = x[grow == grp].double()
        ref = out0[grp].double() + xs.sum(0)
        e = C_ACC * U * D * xs.abs().sum(0) + U * (out0[grp].double().abs() + ref.abs())
        ratio = max(ratio, within(outs[0][grp], ref, e, f"group {grp}", "grouped_colsum"))
    record_property("max_err_over_bound", ratio)


# ------------------------------------------------------------------ swap-AB
SAB_SIZES = [0, 1, 15, 16, 17, 127, 128, 129, 300]


def run_swapab(seed, sizes, K_, M_out, *, w_is_kn, bias, residual, max_ctas=0):
    """groups at 16-row aligned offsets, each followed by its zero padding rows up to a multiple of 16 and then 16 gap rows
    (random in x, canaries in out) that no group owns"""
    gen = torch.Generator().manual_seed(seed)
    G = len(sizes)
    offs, o = [], 0
    for r in sizes:
        offs.append(o)
        o += -(-r // 16) * 16 + 16
    rows = o
    x = cuda_randn(gen, rows, K_, dtype=BF16)
    own = torch.zeros(rows, dtype=torch.bool, device="cuda")       # rows of a group or of its padding
    real = torch.zeros_like(own)
    for off, r in zip(offs, sizes):
        x[off + r: off + -(-r // 16) * 16] = 0
        own[off: off + -(-r // 16) * 16] = True
        real[off: off + r] = True
    w = cuda_randn(gen, G, *((K_, M_out) if w_is_kn else (M_out, K_)), scale=K_ ** -0.5, dtype=BF16)
    b = cuda_randn(gen, G, M_out) if bias else None
    res = cuda_randn(gen, rows, M_out, dtype=BF16) if residual else None
    go = torch.tensor(offs, dtype=torch.int32, device="cuda")
    gr = torch.tensor(sizes, dtype=torch.int32, device="cuda")
    outs = []
    for _ in range(2):
        out = sentinel_like((rows, M_out), BF16)
        K.swapab_linear(x, w, go, gr, out=out, bias=b, residual=res, w_is_kn=w_is_kn, max_ctas=max_ctas)
        outs.append(out)
    torch.cuda.synchronize()
    out = outs[0]
    assert torch.equal(out.view(torch.uint8), outs[1].view(torch.uint8)), "two identical calls differ"
    assert bool(untouched(out[~own]).all()), "rows past a group's padding were written"
    grp = torch.full((rows,), -1, dtype=torch.long, device="cuda")
    for g, (off, r) in enumerate(zip(offs, sizes)):
        grp[off: off + -(-r // 16) * 16] = g
    pre = torch.zeros(rows, M_out, dtype=torch.float64, device="cuda")
    mag = torch.zeros_like(pre)
    for g, (off, r) in enumerate(zip(offs, sizes)):
        if r:
            sl = slice(off, off + -(-r // 16) * 16)
            B = w[g].double() if w_is_kn else w[g].double().t()
            pre[sl] = x[sl].double() @ B
            mag[sl] = x[sl].double().abs() @ B.abs()
    ref, bound = gemm_epilogue64(pre, mag, K_, bias=b.double()[grp.clamp(min=0)] if bias else None, residual=res)
    ratio = within(out[own], ref[own], bound[own], "swapab_linear", "swapab_linear")
    # padding rows: exactly the epilogue of a zero product, i.e. bf16(bias (+ residual)) computed in fp32, or zero
    pad = own & ~real
    if pad.any():
        expect = torch.zeros(int(pad.sum()), M_out, device="cuda")
        if bias:
            expect = expect + b[grp[pad]]
        if residual:
            expect = expect + res[pad].float()
        assert torch.equal(out[pad].float(), expect.to(BF16).float()), "padding rows differ from their contract"
    return ratio


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["fwd_bias_res", "fwd_bias", "dgrad", "dgrad_res"])
@pytest.mark.parametrize("K_,M_out", [(64, 128), (2048, 128), (64, 2048), (2048, 2048)])
def test_swapab_linear_elementwise(K_, M_out, mode, record_property):
    ratio = run_swapab(K_ + M_out, SAB_SIZES, K_, M_out, w_is_kn=mode.startswith("dgrad"), bias=mode.startswith("fwd"),
                       residual=mode.endswith("res"), max_ctas=1 if (K_, mode) == (64, "dgrad_res") else 0)
    record_property("max_err_over_bound", ratio)


@pytest.mark.gpu
@pytest.mark.parametrize("max_ctas", [0, 1])
def test_swapab_linear_1023_groups_one_launch(max_ctas, record_property):
    gen = torch.Generator().manual_seed(11)
    sizes = torch.randint(0, 40, (1023,), generator=gen).tolist()
    sizes[::97] = [0] * len(sizes[::97])
    sizes[-1] = 130
    ratio = run_swapab(12, sizes, 64, 128, w_is_kn=False, bias=True, residual=True, max_ctas=max_ctas)
    record_property("max_err_over_bound", ratio)


# ------------------------------------------------------------------ Adam, bump_steps, cast_bf16
@pytest.fixture
def poison():
    """a zeroed status word installed as the optimizer's poison word, and the previous one restored afterwards"""
    lib = K._lib()
    lib.lah_get_poison_word.restype = ctypes.c_void_p
    prev = lib.lah_get_poison_word()
    status = torch.zeros(4, dtype=torch.int32, device="cuda")
    K.set_poison_word(status)
    yield status
    torch.cuda.synchronize()
    lib.lah_set_poison_word(ctypes.c_void_p(prev))


def adam_state(seed, seg_sizes, G, amsgrad=True):
    gen = torch.Generator().manual_seed(seed)
    n = G * sum(seg_sizes)
    v = torch.rand(n, generator=gen) * 1e-3
    st = dict(p=torch.randn(n, generator=gen), g=torch.randn(n, generator=gen) * 0.1,
              m=torch.randn(n, generator=gen) * 0.01, v=v, vmax=v + torch.rand(n, generator=gen) * 1e-3)
    st = {k: t.cuda() for k, t in st.items()}
    st["p_bf16"] = sentinel_like((n,), BF16)
    return st


def run_adam(st, seg_sizes, G, oracle_kw=None, **kw):
    """one adam_step on copies of st; checks every array against adam_ref64 and the untouched elements byte for byte"""
    hyper = dict(lr=kw.pop("lr", 2e-3), betas=kw.pop("betas", (0.9, 0.999)), eps=kw.pop("eps", 1e-8),
                 weight_decay=kw.pop("weight_decay", 0.0))
    amsgrad = kw.get("amsgrad", True)
    t = {k: v.clone() for k, v in st.items()}
    K.adam_step(t["p"], t["g"], t["m"], t["v"], t["vmax"], t["p_bf16"], seg_sizes, G, **hyper, **kw)
    torch.cuda.synchronize()
    okw = dict(step=kw["step"] if kw.get("step") is not None else kw.get("step_scalar", 0), group_rows=kw.get("group_rows"),
               amsgrad=amsgrad, zero_mask=kw.get("zero_mask", 0), G_active=kw.get("G_active", 0),
               seg_mask=kw.get("seg_mask", 0), lr=f32(hyper["lr"]), betas=tuple(map(f32, hyper["betas"])),
               eps=f32(hyper["eps"]), weight_decay=f32(hyper["weight_decay"]))
    okw.update(oracle_kw or {})
    new, upd, bounds = adam_ref64(st["p"], st["g"], st["m"], st["v"], st["vmax"], seg_sizes, G, **okw)
    ratio = 0.0
    for name in ("p", "m", "v") + (("vmax",) if amsgrad else ()):
        ratio = max(ratio, within(t[name][upd], new[name][upd], bounds[name][upd], name, "adam_step"))
        assert torch.equal(t[name][~upd], st[name][~upd]), f"{name} changed outside the stepped elements"
    if not amsgrad:
        assert torch.equal(t["vmax"], st["vmax"]), "vmax written without amsgrad"
    assert torch.equal(t["g"], new["g"].float()), "the gradient is not zeroed exactly where zero_mask says"
    assert torch.equal(t["p_bf16"][upd], t["p"][upd].to(BF16)), "p_bf16 is not the bf16 rounding of p"
    assert bool(untouched(t["p_bf16"][~upd]).all())
    return t, upd, ratio


SEGS12 = [4, 8, 12, 36, 4, 100, 8, 64, 20, 4, 16, 260]
ADAM_CASES = {
    "all_segments_shadow_slots": dict(seg_mask=0, zero_mask=0b100000000101, G_active=3, amsgrad=True, step="group"),
    "five_merged_ranges": dict(seg_mask=0b110101101011, zero_mask=0b000001000011, G_active=4, amsgrad=True, step="group"),
    "six_ranges_scalar_step_wd": dict(seg_mask=0b010101010101, zero_mask=0b000000010001, G_active=5, amsgrad=False,
                                      step="scalar", weight_decay=0.01),
    "no_amsgrad_wd": dict(seg_mask=0, zero_mask=0xFFF, G_active=0, amsgrad=False, step="group", weight_decay=0.1),
}


@pytest.mark.gpu
@pytest.mark.parametrize("case", list(ADAM_CASES))
def test_adam_step_elementwise(case, poison, record_property):
    c = dict(ADAM_CASES[case])
    G = 5
    st = adam_state(len(case), SEGS12, G)
    rows = torch.tensor([3, 0, 1, 7, 2], dtype=torch.int32, device="cuda")
    step = torch.tensor([1, 4, 2, 9, 3], dtype=torch.int32, device="cuda")
    kind = c.pop("step")
    worst = 0.0
    for _ in range(2):                 # two consecutive steps, each against the oracle from the same inputs
        kw = dict(step=step, step_scalar=0) if kind == "group" else dict(step=None, step_scalar=int(step[0]) + 1)
        t, upd, ratio = run_adam(st, SEGS12, G, group_rows=rows, **kw, **c)
        assert upd.any() and not upd.all()
        worst = max(worst, ratio)
        st = dict(t)
        step = step + 1
    record_property("max_err_over_bound", worst)


@pytest.mark.gpu
def test_adam_step_peer_reduce_branch_at_world_1(poison, record_property):
    """the gradient read through the peer table (base + offset = g) times grad_scale; never zeroes g; a dead rank adds 0"""
    G, segs, off = 3, [8, 40], 4096
    st = adam_state(21, segs, G)
    kw = dict(step=torch.tensor([2, 1, 5], dtype=torch.int32, device="cuda"), world=1, peer_grad_off=off,
              peer_bases=[st["g"].data_ptr() - off], zero_mask=0b11)
    _, _, r1 = run_adam(st, segs, G, grad_scale=0.5, oracle_kw=dict(grad=st["g"] * 0.5, zero_grad=False), **kw)
    _, _, r2 = run_adam(st, segs, G, grad_scale=0.5, dead_mask=1,
                        oracle_kw=dict(grad=torch.zeros_like(st["g"]), zero_grad=False), **kw)
    record_property("max_err_over_bound", max(r1, r2))


@pytest.mark.gpu
def test_adam_step_poison_word_blocks_every_update(poison):
    G, segs = 2, [16, 4]
    st = adam_state(22, segs, G)
    t = {k: v.clone() for k, v in st.items()}
    poison[0] = K.STATUS_TIMEOUT
    K.adam_step(t["p"], t["g"], t["m"], t["v"], t["vmax"], t["p_bf16"], segs, G, step_scalar=3, zero_mask=0b11)
    torch.cuda.synchronize()
    poison[0] = 0
    for k in st:
        assert torch.equal(t[k].view(torch.uint8), st[k].view(torch.uint8)), f"{k} changed under the poison word"


@pytest.mark.gpu
def test_bump_steps_and_cast_bf16_are_exact():
    gen = torch.Generator().manual_seed(23)
    step = torch.randint(0, 100, (300,), generator=gen, dtype=torch.int32).cuda()
    rows = torch.randint(-2, 3, (300,), generator=gen, dtype=torch.int32).cuda()
    s = step.clone()
    K.bump_steps(s, rows)
    scale = 10.0 ** torch.randint(-30, 31, (4004,), generator=gen).double()      # magnitudes from 1e-30 to 1e30
    src = (torch.randn(4004, generator=gen, dtype=torch.float64) * scale).float().cuda()
    assert src.abs().min() < 1e-28 and src.abs().max() > 1e28 and bool((src != 0).all())
    dst = torch.empty(src.numel(), dtype=BF16, device="cuda")
    K.cast_bf16(src, dst)
    torch.cuda.synchronize()
    assert torch.equal(s, step + (rows > 0).int())
    assert torch.equal(dst.view(torch.int16), src.to(BF16).view(torch.int16))
