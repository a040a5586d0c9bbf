"""
The fused weight gradient + AMSGrad kernel of the small expert path (csrc/small_m.cu, ``wgrad_adam``) and the MXFP8
quantiser and grouped GEMM of the FP8 expert forward (csrc/grouped_gemm_fp8.cu, ops/fp8.py), element by element against
float64 oracles, with the machinery and the one constant C_ACC of test_expert_kernels.py.

wgrad_adam never writes its gradient to memory.  With beta1 = 0 and m = 0 the AMSGrad update is m <- m + (1 - 0)(g - m) = g
with no rounding, so the returned m IS the kernel's fp32 gradient dy_g^T x_g; it is held to the GEMM bound.  The optimizer
step is checked on operands whose gradient is exact in fp32 (small integers times powers of two), so that adam_ref64's
element bounds apply with the float64 gradient.  Everything a launch must not touch (empty and shadowed groups, vmax
without amsgrad, every array under the poison word) is compared byte for byte against canaries.

The quantiser is compared exactly: payload bytes and every scale byte.  The FP8 GEMM is compared with the float64 product of
its dequantised operands under a bound with two terms: the fp32 fmaf chain over the 32-element K blocks (and the epilogue),
and the tensor core's own accumulation inside a block, which cuts every product to a multiple of 2^-13 times the block's
largest one, an error below 2^-FP8_MMA_BITS sum |a_k b_k| (tools/fp8_mma_precision.py, DESIGN.md section 5).
"""
import ctypes
import types

import pytest
import torch
import torch.nn.functional as F

from test_expert_kernels import (BF16, C_ACC, EPS_F32, K, SENTINEL, U, _lib, adam_ref64, cuda_randn, f32,  # noqa: F401
                                 gemm_epilogue64, host_abi_only, poison, report_worst_ratios, sentinel_like, tiles_of,
                                 untouched, within)

OPT_CTAS = 132 * 17 // 28   # the optimizer stream's share of the SMs the engine gives the fused kernel
FP8_MMA_BITS = 8            # F: a 32-product e4m3 wgmma sum is within 2^-F sum |a_k b_k| (measured, DESIGN.md section 5)


def ceil16(r):
    return -(-r // 16) * 16


# ---------------------------------------------------------------------------------------------------------------- oracles
def wgrad64(dy, x, offs, rows_list):
    """per group: (float64 dy_g^T x_g, |dy_g|^T |x_g|), None for an empty group"""
    out = []
    for o, r in zip(offs, rows_list):
        if r == 0:
            out.append(None)
            continue
        d, xx = dy[o:o + r].double(), x[o:o + r].double()
        out.append((d.t() @ xx, d.abs().t() @ xx.abs()))
    return out


# ---------------------------------------------------------------------------------------------------------------- CPU
@pytest.mark.parametrize("amsgrad", [True, False])
def test_wgrad_adam_oracle_matches_linear_autograd_and_torch_adam(amsgrad):
    """float64 dy^T x followed by adam_ref64 is one torch.optim.Adam step per expert on an nn.Linear weight [out, in]:
    the gradient of sum(dy o x W^T) is dy^T x, and an expert with no rows in a step is not stepped (its step count stays)"""
    gen = torch.Generator().manual_seed(31)
    G, N, Kd, lr, betas, eps = 3, 8, 12, 3e-3, (0.8, 0.99), 1e-6
    ws = [torch.nn.Parameter(torch.randn(N, Kd, generator=gen, dtype=torch.float64)) for _ in range(G)]
    opts = [torch.optim.Adam([w], lr=lr, betas=betas, eps=eps, amsgrad=amsgrad) for w in ws]
    p = torch.stack([w.detach().clone() for w in ws]).view(-1)
    m, v, vmax = torch.zeros_like(p), torch.zeros_like(p), torch.zeros_like(p)
    step = torch.zeros(G, dtype=torch.long)
    for rows in ([3, 0, 5], [1, 4, 0], [0, 2, 7], [6, 1, 1], [2, 0, 3]):
        grad = torch.zeros(G, N, Kd, dtype=torch.float64)
        for g, r in enumerate(rows):
            if r == 0:
                continue
            x = torch.randn(r, Kd, generator=gen, dtype=torch.float64)
            dy = torch.randn(r, N, generator=gen, dtype=torch.float64)
            (F.linear(x, ws[g]) * dy).sum().backward()
            opts[g].step()
            opts[g].zero_grad(set_to_none=True)
            grad[g] = dy.t() @ x
        rows_t = torch.tensor(rows)
        step += (rows_t > 0).long()
        new, upd, _ = adam_ref64(p, grad.view(-1), m, v, vmax, [N * Kd], G, step=step, group_rows=rows_t, lr=lr,
                                 betas=betas, eps=eps, amsgrad=amsgrad, grad=grad.view(-1))
        assert upd.view(G, -1).all(1).tolist() == [r > 0 for r in rows]
        p, m, v, vmax = new["p"], new["m"], new["v"], new["vmax"]
        for g in range(G):
            torch.testing.assert_close(p.view(G, N, Kd)[g], ws[g].detach(), rtol=1e-13, atol=1e-15)
            st = opts[g].state[ws[g]]
            if not st:
                continue
            assert int(st["step"]) == int(step[g])
            torch.testing.assert_close(m.view(G, N, Kd)[g], st["exp_avg"], rtol=1e-13, atol=1e-15)
            torch.testing.assert_close(v.view(G, N, Kd)[g], st["exp_avg_sq"], rtol=1e-13, atol=1e-18)
            if amsgrad:
                torch.testing.assert_close(vmax.view(G, N, Kd)[g], st["max_exp_avg_sq"], rtol=1e-13, atol=1e-18)


@host_abi_only
def test_wgrad_adam_host_abi_refusals():
    lib = _lib()
    v = ctypes.c_void_p

    # every case by value (lr_dev NULL) and with a device rate block (a fake address)
    for lr_dev in (0, 0xa00000):
        def wa(N=256, K_=384, lddy=256, ldx=384, G=4, vmax=0x800000, l2=0.0, decay=1.0, decoupled=0):
            return lib.lah_wgrad_adam(v(0x200000), lddy, v(0x300000), ldx, 1024, G, N, K_, v(0x400000), v(0x400100), v(0),
                                      v(0x400200), v(0x500000), v(0x600000), v(0x700000), v(vmax), v(0x900000), 1e-3,
                                      v(lr_dev), 0.9, 0.999, 1e-8, 1, l2, decay, decoupled, 0, v(0))
        # the controls: these arguments pass the host checks, with either decay form
        assert wa() != -2 and wa(l2=0.1) != -2 and wa(decay=0.99, decoupled=1) != -2, lr_dev
        for kw in (dict(N=192), dict(K_=320),             # N, K not multiples of the 128 x 128 tile
                   dict(lddy=260), dict(ldx=388),         # row strides off the 16-byte TMA granule
                   dict(G=1 << 20, N=4096),               # G * N rows of the state maps overflow an int
                   dict(vmax=0)):                         # amsgrad without vmax
            assert wa(**kw) == -2 and wa(l2=0.1, **kw) == -2 and wa(decay=0.99, decoupled=1, **kw) == -2, (lr_dev, kw)
        assert wa(l2=0.1, decay=0.99, decoupled=1) == -2, lr_dev        # L2 and decoupled decay at once


@host_abi_only
def test_fp8_c_abi_refuses_misaligned_operands():
    lib = _lib()
    from lah_b200.ops import fp8
    fp8._lib()
    v = ctypes.c_void_p

    def gemm(ldc=64, C=0x100000, out_f32=0, residual=0, ldr=0, bias=0):
        return lib.lah_gemm_mgroup_fp8(v(0x200000), 128, 128, v(0x210000), v(0x300000), v(0x310000), 1, 64, 128, v(C),
                                       ldc, out_f32, 128, 1, v(0), v(bias), v(residual), ldr, 0, v(0), 0, 0, v(0), 0, v(0))
    assert gemm() != -2 and gemm(out_f32=1, residual=0x400000, ldr=64, bias=0x500000) != -2    # the controls
    assert gemm(ldc=63) == -2                                             # odd ldc
    assert gemm(C=0x100002) == -2                                         # bf16 C off its 4-byte pairs
    assert gemm(C=0x100004, out_f32=1) == -2                              # fp32 C off its 8-byte pairs
    assert gemm(residual=0x400000, ldr=63) == -2                          # odd ldr
    assert gemm(residual=0x400002, ldr=64) == -2                          # residual off its 4-byte pairs
    assert gemm(bias=0x500004) == -2                                      # bias off float2

    def quant(inp=0x200000, ld_in=128, in_f32=0, out=0x300000):
        return lib.lah_quant_mxfp8(v(inp), ld_in, in_f32, v(out), 128, v(0x400000), 128, 1, 128, 128, v(0), v(0), v(0))
    assert quant() != -2 and quant(ld_in=136) != -2 and quant(ld_in=132, in_f32=1) != -2            # the controls
    assert quant(ld_in=132) == -2 and quant(ld_in=130, in_f32=1) == -2    # row strides of 264 and 520 bytes
    assert quant(inp=0x200008) == -2 and quant(inp=0x200008, in_f32=1) == -2   # input base off 16 bytes
    assert quant(out=0x300008) == -2                                      # payload base off 16 bytes


# ---------------------------------------------------------------------------------------------------------------- GPU
# ------------------------------------------------------------------ wgrad_adam
def wa_inputs(gen, rows_list, N, K_, *, exact=False, strided=False):
    """dy [total, N], x [total, K_] bf16: groups at 16-row aligned offsets, each right after the previous one's padding,
    so the 32-row TMA box of a group with rows % 32 in [1, 16] covers the next group's first rows and the last group ends at
    the end of the buffer.  The padding rows [rows, ceil16(rows)) are zero in dy and non-zero in x, the layout the engine
    produces (scatter_rows zeroes the padding of the output gradient, the activations there are the LayerNorm of the bias):
    the kernel masks k-steps only at 16-row granularity and relies on dy being zero there.
    exact: dy = i 2^-6 (|i| <= 8, half of them 0) and x = j 2^-4 (1 <= |j| <= 16); every partial sum of a 1100-row
    reduction is a multiple of 2^-10 below 2^14, so the fp32 gradient is exact in any order."""
    offs, total = [], 0
    for r in rows_list:
        offs.append(total)
        total += ceil16(r)
    pad = 8 if strided else 0          # views into wider tensors: bases 16 B in, row strides > width
    if exact:
        i = torch.randint(-8, 9, (total, N), generator=gen) * (torch.rand(total, N, generator=gen) < 0.5)
        j = torch.randint(1, 17, (total, K_), generator=gen) * (torch.randint(0, 2, (total, K_), generator=gen) * 2 - 1)
        dyv, xv = i * 2.0 ** -6, j * 2.0 ** -4
    else:
        dyv, xv = torch.randn(total, N, generator=gen) * 0.5, torch.randn(total, K_, generator=gen)
    real = torch.zeros(total, dtype=torch.bool)
    for o, r in zip(offs, rows_list):
        real[o:o + r] = True
    dyv[~real] = 0
    dy_full = cuda_randn(gen, total, N + 2 * pad, dtype=BF16)
    x_full = cuda_randn(gen, total, K_ + 2 * pad, dtype=BF16)
    dy, x = dy_full[:, pad:pad + N], x_full[:, pad:pad + K_]
    dy.copy_(dyv.to(BF16))
    x.copy_(xv.to(BF16))
    assert bool((x != 0).all()) or not exact
    return dy, x, offs


def wa_state(seed, G, N, K_, stepped, *, m_zero=False, vmax_none=False):
    """p, m, v, vmax [G, N, K_] fp32 and the bf16 mirror: random state in stepped groups (vmax on both sides of v), canaries
    everywhere else and in the whole mirror"""
    cg = torch.Generator(device="cuda").manual_seed(seed)
    shape = (G, N, K_)
    v = torch.rand(shape, generator=cg, device="cuda") * 1e-3
    st = dict(p=torch.randn(shape, generator=cg, device="cuda"),
              m=torch.zeros(shape, device="cuda") if m_zero else torch.randn(shape, generator=cg, device="cuda") * 1e-2,
              v=v, vmax=None if vmax_none else v * (0.5 + torch.rand(shape, generator=cg, device="cuda")))
    for name, t in st.items():
        if t is not None:
            t[~torch.tensor(stepped, device="cuda")] = sentinel_like((1,), torch.float32)
    st["p_bf16"] = sentinel_like(shape, BF16)
    return st


def wa_launch(st, dy, x, go, gr, step, *, skip=None, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, amsgrad=True, max_ctas=0):
    t = {k: (v.clone() if v is not None else None) for k, v in st.items()}
    K.wgrad_adam(dy, x, go, gr, p=t["p"], m=t["m"], v=t["v"], vmax=t["vmax"], p_bf16=t["p_bf16"], step=step, skip=skip,
                 lr=lr, betas=betas, eps=eps, amsgrad=amsgrad, max_ctas=max_ctas)
    torch.cuda.synchronize()
    return t


def same_bytes(a, b):
    return torch.equal(a.contiguous().view(torch.uint8), b.contiguous().view(torch.uint8))


def assert_groups_untouched(before, after, groups, what):
    for g in groups:
        for name, t in after.items():
            if t is not None:
                assert same_bytes(t[g], before[name][g]), f"{what}: {name} of group {g} was written"


WA_ROWS = [0, 1, 15, 16, 17, 31, 32, 33, 63, 64, 65, 1100, 300]    # 1100 rows: 35 k-blocks; 300 % 32 = 12 ends the buffer
WA_GRAD_CASES = {
    "n128_k128_ctas1": dict(N=128, K_=128, max_ctas=1),
    "n256_k384_strided_ctas3": dict(N=256, K_=384, max_ctas=3, strided=True),
    "n2048_k512_opt_ctas": dict(N=2048, K_=512, max_ctas=OPT_CTAS),
    "n512_k2048_strided": dict(N=512, K_=2048, strided=True),
    "n2048_k2048": dict(N=2048, K_=2048),
    "g64_n128_k256_ctas3": dict(N=128, K_=256, max_ctas=3, G=64),
}


@pytest.mark.gpu
@pytest.mark.parametrize("case", list(WA_GRAD_CASES))
def test_wgrad_adam_gradient_elementwise(case, poison, record_property):
    """beta1 = 0, m = 0: the returned m is the kernel's fp32 gradient, held to the GEMM bound C_ACC rows 2^-24 |dy|^T |x|"""
    c = dict(WA_GRAD_CASES[case])
    N, K_, G = c["N"], c["K_"], c.get("G")
    gen = torch.Generator().manual_seed(list(WA_GRAD_CASES).index(case) + 40)
    rows_list = list(WA_ROWS)
    if G:
        choice = torch.randint(0, len(WA_ROWS) - 2, (G,), generator=gen).tolist()
        rows_list = [WA_ROWS[i] for i in choice]
        rows_list[G // 2], rows_list[-1] = 1100, 300
    G = len(rows_list)
    dy, x, offs = wa_inputs(gen, rows_list, N, K_, strided=c.get("strided", False))
    stepped = [r > 0 for r in rows_list]
    st = wa_state(G, G, N, K_, stepped, m_zero=True)
    go = torch.tensor(offs, dtype=torch.int32, device="cuda")
    gr = torch.tensor(rows_list, dtype=torch.int32, device="cuda")
    step = torch.randint(1, 50, (G,), generator=gen, dtype=torch.int32).cuda()
    t = wa_launch(st, dy, x, go, gr, step, betas=(0.0, 0.999), max_ctas=c.get("max_ctas", 0))
    assert_groups_untouched(st, t, [g for g in range(G) if not stepped[g]], "empty group")
    ratio = 0.0
    for g, ref in enumerate(wgrad64(dy, x, offs, rows_list)):
        if ref is None:
            continue
        pre, mag = ref
        bound = EPS_F32 * pre.abs() + (1 + EPS_F32) * C_ACC * rows_list[g] * U * mag
        ratio = max(ratio, within(t["m"][g], pre, bound, f"gradient of group {g} ({rows_list[g]} rows)", "wgrad_adam grad"))
        assert same_bytes(t["p_bf16"][g], t["p"][g].to(BF16)), f"p_bf16 of group {g} is not the bf16 rounding of p"
    record_property("max_err_over_bound", ratio)


# groups 2 (no rows) and 5 (shadowed: skip[2g] >= 0) are not stepped; the others carry the step counts 1 .. 100000
WA_ADAM_ROWS = [1, 17, 0, 33, 300, 5, 1100, 16, 64]
WA_ADAM_STEPS = [1, 2, 7, 10, 1000, 3, 100000, 1, 2]
WA_ADAM_SKIP = (5,)
WA_ADAM_CASES = {
    "amsgrad": dict(amsgrad=True),
    "amsgrad_betas_0.5_0.99": dict(amsgrad=True, betas=(0.5, 0.99)),
    "adam_vmax_canaries": dict(amsgrad=False),
    "adam_vmax_none_betas_0.5_0.99": dict(amsgrad=False, betas=(0.5, 0.99), vmax_none=True),
    "amsgrad_n2048_k512_opt_ctas": dict(amsgrad=True, N=2048, K_=512, max_ctas=OPT_CTAS),
}


def wa_adam_setup(seed, N, K_, vmax_none=False):
    gen = torch.Generator().manual_seed(seed)
    G = len(WA_ADAM_ROWS)
    dy, x, offs = wa_inputs(gen, WA_ADAM_ROWS, N, K_, exact=True)
    skip = torch.full((G, 2), -1, dtype=torch.int32, device="cuda")
    for g in WA_ADAM_SKIP:
        skip[g, 0] = 0
    rows_eff = torch.tensor([0 if g in WA_ADAM_SKIP else r for g, r in enumerate(WA_ADAM_ROWS)])
    stepped = (rows_eff > 0).tolist()
    st = wa_state(seed, G, N, K_, stepped, vmax_none=vmax_none)
    grad = torch.zeros(G, N, K_, dtype=torch.float64, device="cuda")
    for g, ref in enumerate(wgrad64(dy, x, offs, WA_ADAM_ROWS)):
        if ref is not None and stepped[g]:
            grad[g] = ref[0]
    go = torch.tensor(offs, dtype=torch.int32, device="cuda")
    gr = torch.tensor(WA_ADAM_ROWS, dtype=torch.int32, device="cuda")
    return dy, x, go, gr, skip, rows_eff, stepped, st, grad


@pytest.mark.gpu
@pytest.mark.parametrize("case", list(WA_ADAM_CASES))
def test_wgrad_adam_optimizer_step_elementwise(case, poison, record_property):
    """two consecutive launches, each against adam_ref64 from the state before it, on a gradient that is exact in fp32
    (checked bit for bit through the beta1 = 0 probe); many elements have g = 0 exactly"""
    c = dict(WA_ADAM_CASES[case])
    N, K_ = c.get("N", 256), c.get("K_", 384)
    amsgrad, betas, lr, eps = c["amsgrad"], c.get("betas", (0.9, 0.999)), 2e-3, 1e-8
    dy, x, go, gr, skip, rows_eff, stepped, st, grad = wa_adam_setup(list(WA_ADAM_CASES).index(case) + 60, N, K_,
                                                                     c.get("vmax_none", False))
    G = len(WA_ADAM_ROWS)
    unstepped = [g for g in range(G) if not stepped[g]]
    kw = dict(skip=skip, max_ctas=c.get("max_ctas", 0))
    # the gradient is exact: the beta1 = 0 probe returns it bit for bit
    assert bool((grad == 0).any()) and grad.abs().max().item() * 2 ** 10 < 2 ** 24
    probe = wa_launch(dict(st, m=torch.zeros_like(st["m"])), dy, x, go, gr, torch.ones(G, dtype=torch.int32, device="cuda"),
                      betas=(0.0, 0.999), amsgrad=amsgrad, **kw)
    sm = torch.tensor(stepped, device="cuda")
    assert torch.equal(probe["m"][sm], grad[sm].float()), "the kernel's fp32 gradient is not exact"
    step = torch.tensor(WA_ADAM_STEPS, dtype=torch.int32, device="cuda")
    worst = 0.0
    for launch in range(2):
        t = wa_launch(st, dy, x, go, gr, step, lr=lr, betas=betas, eps=eps, amsgrad=amsgrad, **kw)
        if launch == 0:
            again = wa_launch(st, dy, x, go, gr, step, lr=lr, betas=betas, eps=eps, amsgrad=amsgrad, **kw)
            for name, a in t.items():
                assert a is None or same_bytes(a, again[name]), f"two identical launches differ in {name}"
        vmax0 = st["vmax"] if st["vmax"] is not None else torch.zeros_like(st["p"])
        new, upd, bounds = adam_ref64(st["p"].view(-1), grad.view(-1), st["m"].view(-1), st["v"].view(-1),
                                      vmax0.view(-1), [N * K_], G, step=step, group_rows=rows_eff, lr=f32(lr),
                                      betas=tuple(map(f32, betas)), eps=f32(eps), amsgrad=amsgrad, grad=grad.view(-1))
        for name in ("p", "m", "v") + (("vmax",) if amsgrad else ()):
            got = t[name].view(-1)
            worst = max(worst, within(got[upd], new[name][upd], bounds[name][upd], f"{name} after launch {launch}",
                                      "wgrad_adam"))
        assert_groups_untouched(st, t, unstepped, "unstepped group")
        if not amsgrad and st["vmax"] is not None:
            assert same_bytes(t["vmax"], st["vmax"]), "vmax written without amsgrad"
        for g in range(G):
            if stepped[g]:
                assert same_bytes(t["p_bf16"][g], t["p"][g].to(BF16)), f"p_bf16 of group {g} is not the rounding of p"
        st = t
        step = step + torch.tensor(stepped, dtype=torch.int32, device="cuda")
    record_property("max_err_over_bound", worst)


@pytest.mark.gpu
def test_wgrad_adam_refuses_amsgrad_without_vmax():
    """the wrapper refuses on the host, before any launch"""
    dy, x, go, gr, skip, _, stepped, st, _ = wa_adam_setup(71, 256, 384, vmax_none=True)
    with pytest.raises(ValueError):
        wa_launch(st, dy, x, go, gr, torch.ones(len(stepped), dtype=torch.int32, device="cuda"), skip=skip, amsgrad=True)


@pytest.mark.gpu
def test_wgrad_adam_poison_word_blocks_every_update(poison):
    dy, x, go, gr, skip, _, stepped, st, _ = wa_adam_setup(70, 256, 384)
    step = torch.tensor(WA_ADAM_STEPS, dtype=torch.int32, device="cuda")
    control = wa_launch(st, dy, x, go, gr, step, skip=skip)
    for name in ("p", "m", "v", "vmax", "p_bf16"):
        assert not same_bytes(control[name], st[name]), f"the same launch without the poison word leaves {name} as it was"
    poison[0] = K.STATUS_TIMEOUT
    t = wa_launch(st, dy, x, go, gr, step, skip=skip)
    poison[0] = 0
    for name, a in st.items():
        assert same_bytes(t[name], a), f"{name} changed under the poison word"


# ------------------------------------------------------------------ MXFP8 quantiser
def e4m3_bytes(q):
    """payload bytes with -0 (0x80) read as +0: the sign of a zero is not part of its value"""
    return torch.where(q == 0x80, torch.zeros_like(q), q)


def sf_index(t):
    """byte offset in t.sf of the scale of every (row, 32-element block): unpack_sf applied to a table of offsets"""
    table = types.SimpleNamespace(rows_per_group=t.rows_per_group, groups=t.groups, K=t.K, tile_rows=t.tile_rows,
                                  sf=torch.arange(t.sf.numel(), device=t.sf.device))
    return fp8_mod().unpack_sf(table).long()


def fp8_mod():
    from lah_b200.ops import fp8
    return fp8


def edge_blocks(dtype, gen):
    """32-element blocks exact in dtype at the edges of the scale rule and of e4m3:
    all zeros (scale byte 1); amax exactly 448 2^k, one ulp above and one below (the rounding-up of the scale); elements
    that land in the e4m3 subnormals, on their rounding ties or below them; normal values with amax < 448 2^-126 (the
    e = 1 clamp); blocks at the largest finite value of dtype; fp32 significands bf16 would drop; mixed magnitudes."""
    itype = torch.int16 if dtype == BF16 else torch.int32
    sign = lambda n: torch.randint(0, 2, (n,), generator=gen).double() * 2 - 1
    body = lambda: (torch.rand(32, generator=gen).double() * 2 - 1)
    blocks = [torch.zeros(32, dtype=dtype)]
    for k in (-100, -20, -3, 0, 5, 40, 110):
        top = torch.tensor([448.0 * 2.0 ** k], dtype=dtype)
        for bump in (0, 1, -1):
            amax = (top.view(itype) + bump).view(dtype)
            b = (body() * 0.999 * amax.double()).to(dtype)
            b[int(torch.randint(0, 32, (1,), generator=gen))] = amax * float(sign(1))
            blocks.append(b)
    for k in (-4, 0, 7):
        vals = [448.0, 2 ** -6, 2 ** -7, 2 ** -8, 2 ** -9, 1.5 * 2 ** -9, 2 ** -10, 2 ** -11, 3 * 2 ** -10, 1.25 * 2 ** -9,
                0.75 * 2 ** -9, 2.5 * 2 ** -9, 7 * 2 ** -9, 15 * 2 ** -10]
        b = torch.zeros(32, dtype=torch.float64)
        b[:len(vals)] = torch.tensor(vals, dtype=torch.float64) * 2.0 ** k * sign(len(vals))
        blocks.append(b[torch.randperm(32, generator=gen)].to(dtype))
    tiny = (1 + torch.rand(32, generator=gen).double()) * 2.0 ** -121 * sign(32)
    blocks.append(tiny.to(dtype))
    b = torch.tensor([2.0 ** -126, 3 * 2.0 ** -126, 447 * 2.0 ** -126] + [0.0] * 29, dtype=torch.float64) * sign(32)
    blocks.append(b.to(dtype))
    big = torch.finfo(dtype).max
    for frac in (1.0, 0.75):
        b = (body() * big * frac).to(dtype)
        b[3] = -big * frac
        blocks.append(b)
    for _ in range(3):
        blocks.append((torch.randn(32, generator=gen, dtype=torch.float64) * 10.0 ** (torch.rand(32, generator=gen) * 6 - 3))
                      .to(dtype))
    out = torch.stack(blocks)
    assert bool(torch.isfinite(out.double()).all())
    assert bool(((out == 0) | (out.double().abs() >= 2.0 ** -126)).all()), "fp32 subnormal inputs are out of scope"
    return out


def quant_inputs(gen, rows, K_, dtype, edge_rows):
    """[rows, K_] in dtype, a view 16 elements into a wider tensor; the rows in edge_rows hold the edge blocks"""
    full = (torch.randn(rows, K_ + 48, generator=gen) * 10.0 ** (torch.rand(rows, 1, generator=gen) * 4 - 2)).to(dtype)
    x = full[:, 16:16 + K_]
    eb = edge_blocks(dtype, gen)
    per_row = K_ // 32
    n = -(-eb.shape[0] // per_row)
    eb = torch.cat([eb, x[:n].reshape(-1, 32)[:n * per_row - eb.shape[0]]]).view(n, K_)
    for r0 in edge_rows:
        x[r0:r0 + n] = eb
    return full.cuda()[:, 16:16 + K_]


def check_quant(x, tile_rows, groups, processed, *, tile_group=None, total_rows=None):
    fp8 = fp8_mod()
    rows, K_ = x.shape
    out = fp8.MXFP8Tensor(rows // groups, groups, K_, tile_rows, "cuda")
    out.q.fill_(SENTINEL)
    out.sf.fill_(SENTINEL)
    fp8.quantize(x, tile_rows=tile_rows, groups=groups, out=out, tile_group=tile_group,
                 total_rows=None if total_rows is None else torch.tensor([total_rows], dtype=torch.int32, device="cuda"))
    torch.cuda.synchronize()
    q_ref, e_ref = fp8.quantize_ref(x[processed])
    got = out.q[processed]
    bad = e4m3_bytes(got) != e4m3_bytes(q_ref.view(torch.uint8))
    if bad.any():
        i = bad.nonzero()[0].tolist()
        raise AssertionError(f"{int(bad.sum())} payload bytes differ; first at processed row {i[0]}, column {i[1]}: "
                             f"input {x[processed][i[0], i[1]].item()!r}, got {got[i[0], i[1]].item():#x}, "
                             f"ref {q_ref.view(torch.uint8)[i[0], i[1]].item():#x}")
    e_got = fp8.unpack_sf(out)[processed]
    assert torch.equal(e_got, e_ref), f"{int((e_got != e_ref).sum())} scale bytes differ"
    assert bool((out.q[~processed] == SENTINEL).all()), "payload rows the kernel must skip were written"
    written = torch.zeros(out.sf.numel(), dtype=torch.bool, device="cuda")
    written[sf_index(out)[processed].reshape(-1)] = True
    assert bool((out.sf[~written] == SENTINEL).all()), "scale bytes of skipped rows or of tile padding were written"
    return e_ref


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [BF16, torch.float32], ids=["bf16", "fp32"])
def test_quantize_activation_tiles_exact(dtype):
    """NaN and Inf inputs are out of scope, and so are fp32 subnormal inputs (the fast-math build flushes them to zero)"""
    gen = torch.Generator().manual_seed(80)
    rows, K_ = 5 * 128, 256
    tiles = [0, -1, 1, 0, 2]
    total_rows = 570                               # inside the last tile: rows 570 .. 639 stay untouched
    x = quant_inputs(gen, rows, K_, dtype, edge_rows=(0, 128, 300, 530))
    tg = torch.tensor(tiles, dtype=torch.int32, device="cuda")
    r = torch.arange(rows, device="cuda")
    processed = (tg.long()[r // 128] >= 0) & (r < total_rows)
    e = check_quant(x, fp8_mod().ACT_TILE, 1, processed, tile_group=tg, total_rows=total_rows)
    assert bool((e == 1).any()) and bool((e >= 245).any())      # the clamp and the top of the range were exercised


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [BF16, torch.float32], ids=["bf16", "fp32"])
def test_quantize_weight_tiles_exact(dtype):
    """3 groups of 200 rows in 192-row weight tiles: each group's second tile is mostly padding, whose scale bytes stay
    untouched"""
    gen = torch.Generator().manual_seed(81)
    groups, rpg, K_ = 3, 200, 384
    x = quant_inputs(gen, groups * rpg, K_, dtype, edge_rows=(0, 190, 400, 590))
    processed = torch.ones(groups * rpg, dtype=torch.bool, device="cuda")
    check_quant(x, fp8_mod().WEIGHT_TILE, groups, processed)


@pytest.mark.gpu
def test_fp8_wrappers_refuse_misaligned_operands():
    """the wrappers refuse on the host, before any launch"""
    fp8 = fp8_mod()
    with pytest.raises(ValueError):
        fp8.quantize(torch.zeros(128, 136, dtype=BF16, device="cuda")[:, 4:132])              # input base 8 B off
    with pytest.raises(ValueError):
        fp8.quantize(torch.zeros(128 * 132, dtype=BF16, device="cuda").view(128, 132)[:, :128])     # 264-byte rows
    with pytest.raises(ValueError):
        fp8.quantize(torch.zeros(128 * 130, device="cuda").view(128, 130)[:, :128])           # 520-byte fp32 rows
    t = fp8.MXFP8Tensor(128, 1, 128, fp8.ACT_TILE, "cuda")
    t.q = torch.zeros(128 * 128 + 16, dtype=torch.uint8, device="cuda")[8:8 + 128 * 128].view(128, 128)
    with pytest.raises(ValueError):
        fp8.quantize(torch.zeros(128, 128, dtype=BF16, device="cuda"), out=t)                # payload base 8 B off
    aq = fp8.MXFP8Tensor(128, 1, 128, fp8.ACT_TILE, "cuda")
    wq = fp8.MXFP8Tensor(64, 1, 128, fp8.WEIGHT_TILE, "cuda")
    wide = torch.zeros(128, 130, dtype=BF16, device="cuda")
    with pytest.raises(ValueError):
        fp8.grouped_linear_fp8(aq, wq, out=wide[:, 1:65])                                     # bf16 out one element off
    with pytest.raises(ValueError):
        fp8.grouped_linear_fp8(aq, wq, out=torch.zeros(128 * 65, dtype=BF16, device="cuda").view(128, 65)[:, :64])
    with pytest.raises(ValueError):
        fp8.grouped_linear_fp8(aq, wq, out=torch.zeros(128, 66, device="cuda")[:, 1:65], out_dtype=torch.float32)
    with pytest.raises(ValueError):
        fp8.grouped_linear_fp8(aq, wq, residual=wide[:, 1:65])                                # residual one element off
    with pytest.raises(ValueError):
        fp8.grouped_linear_fp8(aq, wq, residual=torch.zeros(128 * 65, dtype=BF16, device="cuda").view(128, 65)[:, :64])
    with pytest.raises(ValueError):
        fp8.grouped_linear_fp8(aq, wq, bias=torch.zeros(65, device="cuda")[1:])               # bias off float2


# ------------------------------------------------------------------ MXFP8 grouped GEMM
def dequant64(t, rows_mask):
    """float64 dequantised operand: payload times 2^(scale byte - 127) per 32-element block, zero outside rows_mask"""
    fp8 = fp8_mod()
    n, K_ = t.q.shape
    e = fp8.unpack_sf(t).double()
    q = t.q.view(torch.float8_e4m3fn).float().double()
    out = (q.view(n, K_ // 32, 32) * torch.exp2(e - 127)[..., None]).view(n, K_)
    return torch.where(rows_mask[:, None], out, torch.zeros_like(out))


FP8_CASES = {
    "n64_k128_bias_f32_ctas1": dict(rows_per_group=[100, 0, 37], N=64, K_=128, bias=True, out_f32=True, max_ctas=1),
    "n192_k512_gelu_bias_res": dict(rows_per_group=[300, 5], N=192, K_=512, bias=True, residual=True, act=2),
    "n512_k2048_relu_res_f32_mvalid": dict(rows_per_group=[256, 0, 130], N=512, K_=2048, residual=True, out_f32=True,
                                           act=1, m_valid_cut=70),
    "n2048_k512_gelu_bias_f32": dict(rows_per_group=[200, 77], N=2048, K_=512, bias=True, out_f32=True, act=2),
    "n2048_k2048_relu_bias_res": dict(rows_per_group=[1000, 24], N=2048, K_=2048, bias=True, residual=True, act=1),
    "n192_k128_gelu_res_f32_ctas1": dict(rows_per_group=[40, 0, 260], N=192, K_=128, residual=True, out_f32=True, act=2,
                                         max_ctas=1),
    "n64_k2048_mvalid": dict(rows_per_group=[20, 300], N=64, K_=2048, bias=True, m_valid_cut=100),
}


@pytest.mark.gpu
@pytest.mark.parametrize("case", list(FP8_CASES))
def test_grouped_linear_fp8_elementwise(case, record_property):
    """ragged groups padded to 256 rows with an unused tile before group 1 (and at the end unless m_valid cuts the last
    group); rows and weight rows of very different magnitude, so neighbouring rows have different block scales"""
    fp8 = fp8_mod()
    c = dict(FP8_CASES[case])
    rows_per_group, N, K_, cut = c["rows_per_group"], c["N"], c["K_"], c.get("m_valid_cut", 0)
    gen = torch.Generator().manual_seed(list(FP8_CASES).index(case) + 90)
    tiles = tiles_of(rows_per_group, 256, unused_tail=not cut)
    rows, G = len(tiles) * 128, len(rows_per_group)
    m_valid = rows - cut
    assert not cut or tiles[(m_valid - 1) // 128] >= 0 and tiles[-1] >= 0
    a = (torch.randn(rows, K_, generator=gen) * 2.0 ** torch.randint(-6, 7, (rows, 1), generator=gen)).to(BF16).cuda()
    w = (torch.randn(G * N, K_, generator=gen) * K_ ** -0.5 * 2.0 ** torch.randint(-3, 4, (G * N, 1), generator=gen)) \
        .to(BF16).cuda()
    tg = torch.tensor(tiles, dtype=torch.int32, device="cuda")
    aq = fp8.quantize(a, tile_group=tg)
    wq = fp8.quantize(w, tile_rows=fp8.WEIGHT_TILE, groups=G)
    b = cuda_randn(gen, G, N) if c.get("bias") else None
    res = cuda_randn(gen, rows, N, dtype=BF16) if c.get("residual") else None
    out_f32 = c.get("out_f32", False)
    out = sentinel_like((rows, N), torch.float32 if out_f32 else BF16)
    call = lambda: fp8.grouped_linear_fp8(aq, wq, tile_group=tg, bias=b, residual=res, out=out,
                                          out_dtype=out.dtype, m_valid=m_valid if cut else None,
                                          max_ctas=c.get("max_ctas", 0), act=c.get("act", 0))
    call()
    first = out.clone()
    out.view(torch.uint8).fill_(SENTINEL)
    call()
    torch.cuda.synchronize()
    assert same_bytes(first, out), "two identical calls differ"
    grow = tg.long().repeat_interleave(128)
    valid = (grow >= 0) & (torch.arange(rows, device="cuda") < m_valid)
    A = dequant64(aq, grow >= 0)
    W = dequant64(wq, torch.ones(G * N, dtype=torch.bool, device="cuda")).view(G, N, K_)
    nb = K_ // 32
    pre = torch.zeros(rows, N, dtype=torch.float64, device="cuda")
    blocks = torch.zeros_like(pre)       # sum over the K blocks of |partial product of the block|
    mag = torch.zeros_like(pre)          # |A| |W|^T
    for t, g in enumerate(tiles):
        if g < 0:
            continue
        sl = slice(t * 128, (t + 1) * 128)
        parts = torch.einsum("rbk,nbk->rbn", A[sl].view(128, nb, 32), W[g].view(N, nb, 32))
        pre[sl], blocks[sl] = parts.sum(1), parts.abs().sum(1)
        mag[sl] = A[sl].abs() @ W[g].abs().t()
    ref, bound = gemm_epilogue64(pre, blocks, nb + 2, bias=b.double()[grow.clamp(min=0)] if b is not None else None,
                                 act=c.get("act", 0), residual=res, out_f32=out_f32, extra=2.0 ** -FP8_MMA_BITS * mag)
    ratio = within(out[valid], ref[valid], bound[valid], "grouped_linear_fp8", "grouped_linear_fp8")
    assert bool(untouched(out[~valid]).all()), "rows of unused tiles or rows >= m_valid were written"
    record_property("max_err_over_bound", ratio)
