"""
Model widths: the LayerNorm forward / backward and the grouped column sum (csrc/layernorm.cu) at every width that is a
multiple of 128 up to 4096, element by element against float64 oracles, and on top of them transformer experts with
d_model any multiple of 128 in [256, 4096] and FeedforwardBlock(hid) with hid any multiple of 128 up to 1024 training
through ExpertBackend.  Every width the executors' ``supports()`` admits must run natively; the widths just past the
limits must run on the module, never reach a kernel that refuses them.

The kernel oracles and helpers are those of test_expert_kernels.py; the encoder-layer oracle is that of
test_encoder_layer_experts.py.
"""
import copy
import ctypes
from argparse import Namespace

import pytest
import torch
from torch import nn

from test_encoder_layer_experts import GRAD_CHECKED, _backend, _masks, encoder_layer_ref, rel
from test_expert_kernels import (BF16, C_ACC, EPS_BF16, LN_EPS, LN_TILES, U, _lib, cuda_randn, host_abi_only, ln_bwd64,
                                 ln_inputs, run_mgroup, sentinel_like, untouched, within)

import lah_b200
from lah_b200.models.layers import FeedforwardBlock, TransformerEncoderLayer
from lah_b200.ops import kernels as K

REFUSED_WIDTHS = [64, 192, 4224, 8192]            # LayerNorm: not a multiple of 128, or wider than 4096
NEW_LN_WIDTHS = [128, 384, 640, 768, 1152, 1536, 2304, 3072, 3968]


# ------------------------------------------------------------------------------------------------ CPU: refusals
def test_width_table():
    assert K.LN_WIDTHS == tuple(range(128, 4097, 128)) and K.LN_MAX_WIDTH == 4096
    assert all(K.ln_width_ok(c) for c in K.LN_WIDTHS)
    assert not any(K.ln_width_ok(c) for c in REFUSED_WIDTHS + [0, -128])


def test_grouped_colsum_refuses_only_widths_off_128():
    x = torch.zeros(8, 192, dtype=BF16)
    with pytest.raises(ValueError, match="width"):
        K.grouped_colsum(x, None, out=torch.zeros(1, 192))
    with pytest.raises(ValueError, match="width"):
        K.grouped_colsum(x[:, :0], None, out=torch.zeros(1, 0))


@host_abi_only
@pytest.mark.parametrize("C", REFUSED_WIDTHS)
def test_c_abi_refuses_widths(C):
    lib = _lib()
    v = ctypes.c_void_p
    p = [v(0x100000 * (i + 1)) for i in range(12)]
    assert lib.lah_ln_relu_fwd(*p[:7], 8, C, 1, 128, v(0)) == -2
    assert lib.lah_ln_relu_bwd(*p, 8, C, 1, 128, v(0), v(0)) == -2
    assert lib.lah_ln_relu_bwd(*p, 8, C, 1, 16, p[0], v(0)) == -2
    if C % 128:   # the column sum runs any multiple of 128 (the in_proj bias gradient sums 3 d columns)
        assert lib.lah_grouped_colsum(p[0], C, p[1], p[2], C, v(0), 8, 128, v(0)) == -2


@pytest.mark.parametrize("C", REFUSED_WIDTHS)
def test_wrappers_refuse_widths(C):
    """the wrappers raise before anything is launched (CPU tensors: nothing could be)"""
    h = torch.zeros(8, C, dtype=BF16)
    gamma, beta, stat = torch.ones(1, C), torch.zeros(1, C), torch.zeros(8)
    with pytest.raises(ValueError, match="width"):
        K.ln_relu_fwd(h, gamma, beta, None, out=torch.empty_like(h), mean=stat, rstd=stat)
    with pytest.raises(ValueError, match="width"):
        K.ln_relu_bwd(h, h, stat, stat, gamma, beta, None, dh=torch.empty_like(h), dgamma=gamma, dbeta=beta,
                      dbias=beta)
    if C % 128:
        with pytest.raises(ValueError, match="width"):
            K.grouped_colsum(h, None, out=gamma)


# ------------------------------------------------------------------------------------------------ GPU: kernels
def ln_fwd64_depth(h, gamma, beta, relu):
    """float64 LayerNorm(+ReLU) with the error terms of the kernel's one-pass statistics.  A lane sums 8 values per
    256-column chunk; at an odd multiple of 128, lanes 0-15 also sum the last half chunk, so the longest per-lane sum has
    8 ceil(C / 256) terms (C / 32 at a multiple of 256), then a 5-level warp tree; the + 8 below covers the tree."""
    x = h.double()
    C = x.shape[1]
    mu = x.mean(1, keepdim=True)
    var = ((x - mu) ** 2).mean(1, keepdim=True)
    rstd = (var + LN_EPS).rsqrt()
    xhat = (x - mu) * rstd
    y = xhat * gamma.double() + beta.double()
    if relu:
        y = y.clamp(min=0)
    D = 8 * -(-C // 256) + 8
    e_abs, e_sq = x.abs().mean(1, keepdim=True), (x * x).mean(1, keepdim=True)
    d_mean = C_ACC * U * D * e_abs
    d_var = C_ACC * U * D * (e_sq + 2 * mu.abs() * e_abs) + 2 * U * mu * mu
    d_rstd = 0.5 * d_var / (var + LN_EPS) + 4 * U
    g = gamma.double().abs()
    xabs = (x.abs() + mu.abs()) * rstd
    e_y = g * (xhat.abs() * d_rstd + rstd * d_mean + 3 * U * xabs) + 2 * U * (xhat.abs() * g + beta.double().abs())
    return y, mu.squeeze(1), rstd.squeeze(1), dict(e_y=e_y, d_mean=d_mean.squeeze(1), d_rstd=d_rstd.squeeze(1))


def check_forward(h, gamma, beta, tg, grow, tile_rows, relu):
    rows, C = h.shape
    outs = []
    for _ in range(2):
        o = (sentinel_like((rows, C), BF16), sentinel_like((rows,), torch.float32), sentinel_like((rows,), torch.float32))
        K.ln_relu_fwd(h, gamma, beta, tg, out=o[0], mean=o[1], rstd=o[2], relu=relu, tile_rows=tile_rows)
        outs.append(o)
    torch.cuda.synchronize()
    for a, b in zip(*outs):
        assert torch.equal(a.view(torch.uint8), b.view(torch.uint8)), "two identical calls differ"
    out, mean, rstd = outs[0]
    valid = grow >= 0
    gi = grow.clamp(min=0)
    y, mu, rs, b = ln_fwd64_depth(h[valid], gamma[gi[valid]], beta[gi[valid]], relu)
    r1 = within(out[valid], y, EPS_BF16 * y.abs() + (1 + EPS_BF16) * b["e_y"], "LayerNorm output", "ln_fwd")
    r2 = within(mean[valid], mu, b["d_mean"], "saved mean", "ln_fwd")
    r3 = within(rstd[valid], rs, b["d_rstd"] * rs, "saved rstd", "ln_fwd")
    assert bool(untouched(out[~valid]).all() and untouched(mean[~valid]).all() and untouched(rstd[~valid]).all())
    return mean, rstd, max(r1, r2, r3)


@pytest.mark.gpu
@pytest.mark.parametrize("relu", [False, True])
@pytest.mark.parametrize("grouped", [False, True], ids=["tile_group_none", "ragged"])
@pytest.mark.parametrize("tile_rows", [8, 16, 128])
@pytest.mark.parametrize("C", NEW_LN_WIDTHS)
def test_ln_forward_new_widths(C, tile_rows, grouped, relu, record_property):
    h, gamma, beta, tg, grow, _ = ln_inputs(C + tile_rows + 1, C, tile_rows, grouped)
    record_property("max_err_over_bound", check_forward(h, gamma, beta, tg, grow, tile_rows, relu)[2])


@pytest.mark.gpu
@pytest.mark.parametrize("with_dres", [False, True], ids=["no_dres", "dres"])
@pytest.mark.parametrize("relu", [False, True])
@pytest.mark.parametrize("grouped", [False, True], ids=["tile_group_none", "ragged"])
@pytest.mark.parametrize("tile_rows", [8, 16, 128])
@pytest.mark.parametrize("C", NEW_LN_WIDTHS)
def test_ln_backward_new_widths(C, tile_rows, grouped, relu, with_dres, record_property):
    """the bounds of test_expert_kernels.test_ln_backward_elementwise.  Its row means over D_row = 32 sequential fp32
    sums still hold: a thread sums 8 columns, a warp tree adds 5 levels and the CTA adds one partial per warp, at most 16;
    at an odd multiple of 128 the CTA is rounded up to whole warps and the idle threads add exact zeros."""
    h, gamma, beta, tg, grow, gen = ln_inputs(7 * C + tile_rows + 1, C, tile_rows, grouped)
    rows = h.shape[0]
    mean, rstd, _ = check_forward(h, gamma, beta, tg, grow, tile_rows, relu)
    valid = grow >= 0
    gi = grow.clamp(min=0)
    gam, bet = gamma[gi], beta[gi]
    da = cuda_randn(gen, rows, C, dtype=BF16)
    _, _, _, y = ln_bwd64(da, h, mean, rstd, gam, bet, relu)
    xabs = (h.double().abs() + mean.double().abs()[:, None]) * rstd.double()[:, None]
    kink = relu & valid[:, None] & (y.abs() <= C_ACC * U * (xabs * gam.double().abs() + bet.double().abs()))
    assert int(kink.sum()) <= max(2, kink.numel() // 10000), int(kink.sum())
    da = da.masked_fill(kink, 0)
    dres = cuda_randn(gen, rows, C, dtype=BF16) if with_dres else None
    d0 = [cuda_randn(gen, 3, C) for _ in range(3)]
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
    D_row = 32
    r = rstd.double()[:, None]
    gg = (g * gam.double()).abs()
    m1, m2 = gg.mean(1, keepdim=True), (gg * xabs).mean(1, keepdim=True)
    e_dh = C_ACC * U * r * (gg + D_row * m1 + xabs * D_row * m2 + 3 * xabs * gg)
    if with_dres:
        e_dh = e_dh + U * ref_dh.abs()
    ratio = within(dh[valid], ref_dh[valid], EPS_BF16 * ref_dh[valid].abs() + (1 + EPS_BF16) * e_dh[valid], "dh", "ln_bwd")
    assert bool(untouched(dh[~valid]).all()), "rows of unused tiles were written"
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
@pytest.mark.parametrize("C", [128, 384, 1152, 2688, 4224])
def test_grouped_colsum_new_widths(C, tile_rows, record_property):
    gen = torch.Generator().manual_seed(C + tile_rows)
    rows = 5 * tile_rows + 3
    tiles = LN_TILES[:-(-rows // tile_rows)]
    grow = torch.tensor(tiles, device="cuda").repeat_interleave(tile_rows)[:rows]
    x_full = cuda_randn(gen, rows, C + 128, dtype=BF16)
    x = x_full[:, 64:64 + C]                                                 # strided: ldx = C + 128 > C
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


@pytest.mark.gpu
@pytest.mark.parametrize("N", [384, 640])
@pytest.mark.parametrize("site,p,act,residual", [(1, 0.1, 0, True), (2, 0.5, 2, False), (3, 0.1, 0, True)])
def test_grouped_linear_dropout_epilogue_odd_n(N, site, p, act, residual, record_property):
    """256-wide tiles with N % 256 = 128: the last n tile is half used; the mask is a function of the absolute column"""
    _, ratio = run_mgroup(N + site, [300, 0, 77, 128], N, 200, block_n=256, bias=True, residual=residual, act=act,
                          dropout=(p, 4321 + site, site))
    record_property("max_err_over_bound", ratio)


# ------------------------------------------------------------------------------------------------ GPU: ExpertBackend
TORCH_CASES = [   # (d, nhead, ff, norm_first, activation, batch_first, S)
    (384, 6, 1536, False, "relu", True, 300),
    (640, 10, 2560, True, "gelu", False, 512),
    (768, 12, 3072, False, "gelu", True, 512),
    (768, 24, 3072, True, "relu", False, 300),      # head dim 32
    (1280, 20, 5120, True, "gelu", True, 300),
    (1536, 12, 6144, False, "relu", False, 512),    # head dim 128
]


@pytest.mark.gpu
@pytest.mark.parametrize("d,nhead,ff,norm_first,activation,batch_first,S", TORCH_CASES)
def test_expert_backend_trains_torch_encoder_layer_widths(d, nhead, ff, norm_first, activation, batch_first, S):
    """nn.TransformerEncoderLayer(d, nhead, ff, dropout 0.1) through ExpertBackend: forward, dx, weight gradients and three
    AMSGrad steps against the fp32 functional oracle with the same masks; eval mode against the module itself"""
    from lah_b200.ops import native
    from lah_b200.runtime.native_executor import NativeTransformerExecutor, draw_dropout_seed, encoder_layer_spec
    torch.manual_seed(4)
    layer = nn.TransformerEncoderLayer(d, nhead, ff, dropout=0.1, activation=activation, batch_first=batch_first,
                                       norm_first=norm_first).cuda()
    spec = encoder_layer_spec(layer)
    ref = copy.deepcopy(layer)
    ref_opt = torch.optim.Adam(ref.parameters(), lr=1e-4, amsgrad=True)
    shape = (2, S, d) if batch_first else (S, 2, d)
    be = _backend(layer, shape)
    x = torch.randn(*shape, device="cuda")
    g = torch.randn(*shape, device="cuda") * 0.1
    native.reset_launches()
    torch.manual_seed(10)
    seed = draw_dropout_seed()
    torch.manual_seed(10)
    (y,) = be.forward(x)
    assert type(be._executor) is NativeTransformerExecutor and native.launches() > 0
    with torch.no_grad():
        assert rel(y, encoder_layer_ref(ref, x, _masks(seed, spec, 2, S))) < 3e-2
    for it in range(3):
        torch.manual_seed(20 + it)
        seed = draw_dropout_seed()
        torch.manual_seed(20 + it)
        launches = native.launches()
        (gx,) = be.backward(x, g)
        assert native.launches() > launches and gx.shape == x.shape
        xr = x.clone().requires_grad_(True)
        encoder_layer_ref(ref, xr, _masks(seed, spec, 2, S)).backward(g)
        if it == 0:
            assert rel(gx, xr.grad) < 5e-2
            st = be.opt.state_dict()["state"]
            for i, (n, p) in enumerate(ref.named_parameters()):
                if n in GRAD_CHECKED:
                    assert rel(st[i]["exp_avg"] / 0.1, p.grad) < 6e-2, n
        ref_opt.step(), ref_opt.zero_grad()
    sd, rsd = be.state_dict(), ref.state_dict()
    assert max((sd["expert." + k] - v).abs().mean().item() for k, v in rsd.items()) < 1.5e-4
    layer.eval()
    with torch.no_grad():
        assert rel(be.forward(x)[0], layer(x)) < 3e-2


@pytest.mark.gpu
def test_masked_encoder_layer_d768():
    """a key padding mask at d = 768: output, dx and one step against the fp64 module (dropout 0)"""
    from test_key_padding_mask import _backend as masked_backend, _layer_input
    from lah_b200.runtime.native_executor import NativeTransformerExecutor
    torch.manual_seed(768)
    S, d = 200, 768
    layer = nn.TransformerEncoderLayer(d, 12, 3072, dropout=0.0, batch_first=True).cuda()
    ref = copy.deepcopy(layer).double()
    be = masked_backend(layer, S, d)
    x, gy, pad = _layer_input(True, 4, S, d, seed=d)
    (y,) = be.forward(x, pad)
    assert type(be._executor) is NativeTransformerExecutor
    xr = x.double().requires_grad_(True)
    yr = ref(xr, src_key_padding_mask=pad)
    yr.backward(gy.double())
    assert bool(torch.isfinite(y).all()) and rel(y, yr.detach()) < 3e-2
    dx, _ = be.backward(x, pad, gy)
    assert bool(torch.isfinite(dx).all()) and rel(dx, xr.grad) < 5e-2
    torch.optim.Adam(ref.parameters(), lr=1e-4, amsgrad=True).step()
    sd, rsd = be.state_dict(), ref.state_dict()
    assert max((sd["expert." + k] - v).abs().mean().item() for k, v in rsd.items()) < 1.5e-4


def _steps_against_eager(module, shape, make_opt, ref_forward, steps=3):
    """forward and ``steps`` backward calls through ExpertBackend against an eager copy with the same optimizer and the
    same dropout masks: (native forward, eager forward, first dx, eager first dx, max mean |parameter difference|)"""
    from lah_b200.ops import native
    from lah_b200.runtime.native_executor import NativeFFNExecutor, NativeTransformerExecutor, draw_dropout_seed
    ref = copy.deepcopy(module)
    ref_opt = make_opt(ref)
    be = lah_b200.ExpertBackend(name="t", expert=module, opt=make_opt(module),
                                args_schema=(lah_b200.BatchTensorProto(*shape[1:]),),
                                outputs_schema=lah_b200.BatchTensorProto(*shape[1:]), max_batch_size=8)
    gen = torch.Generator().manual_seed(7)
    x = torch.randn(*shape, generator=gen).cuda()
    g = (torch.randn(*shape, generator=gen) * 0.1).cuda()
    native.reset_launches()
    torch.manual_seed(10)
    seed = draw_dropout_seed()
    torch.manual_seed(10)
    (y,) = be.forward(x)
    assert type(be._executor) in (NativeFFNExecutor, NativeTransformerExecutor) and native.launches() > 0
    with torch.no_grad():
        y_ref = ref_forward(ref, x, seed)
    dxs = []
    for it in range(steps):
        torch.manual_seed(20 + it)
        seed = draw_dropout_seed()
        torch.manual_seed(20 + it)
        (gx,) = be.backward(x, g)
        xr = x.clone().requires_grad_(True)
        ref_forward(ref, xr, seed).backward(g)
        if it == 0:
            dxs = [gx, xr.grad]
        ref_opt.step()
        ref_opt.zero_grad()
    sd, rsd = be.state_dict(), ref.state_dict()
    return y, y_ref, dxs[0], dxs[1], max((sd["expert." + k] - v).abs().mean().item() for k, v in rsd.items())


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["torch layer, two-group AdamW", "own layer"])
def test_expert_backend_trains_d768(kind):
    from test_weight_decay import _aw, _ref_forward
    torch.manual_seed(3)
    if kind == "own layer":
        module, shape = TransformerEncoderLayer(768, 12).cuda(), (2, 300, 768)
        make_opt = lambda m: torch.optim.Adam(m.parameters(), lr=1e-4, amsgrad=True)  # noqa: E731
    else:
        module, shape = nn.TransformerEncoderLayer(768, 12, dropout=0.1).cuda(), (300, 2, 768)
        make_opt = _aw
    y, y_ref, dx, dx_ref, dp = _steps_against_eager(module, shape, make_opt, _ref_forward)
    assert rel(y, y_ref) < 3e-2 and rel(dx, dx_ref) < 5e-2 and dp < 1.5e-4


@pytest.mark.gpu
@pytest.mark.parametrize("hid", [384, 640, 768, 896])
def test_expert_backend_trains_ffn_widths(hid):
    torch.manual_seed(hid)
    make_opt = lambda m: torch.optim.Adam(m.parameters(), lr=1e-4, amsgrad=True)  # noqa: E731
    y, y_ref, dx, dx_ref, dp = _steps_against_eager(FeedforwardBlock(hid).cuda(), (200, hid), make_opt,
                                                    lambda m, x, seed: m(x))
    assert rel(y, y_ref) < 3e-2 and rel(dx, dx_ref) < 5e-2 and dp < 1.5e-4


def _sweep_cases():
    cases = []
    for d in list(range(256, 2049, 128)) + [4096]:
        cases += [("torch", d, d // hd) for hd in K.HEAD_DIMS if d % hd == 0]
    cases += [("ffn", hid, 0) for hid in range(128, 1025, 128)]
    return cases


def _one_call_each(module, shape):
    """one forward and one backward through a fresh ExpertBackend; the module's own forward and input gradient (taken
    before the step) for comparison"""
    from lah_b200.ops import native
    gen = torch.Generator().manual_seed(1)
    x = torch.randn(*shape, generator=gen).cuda()
    g = (torch.randn(*shape, generator=gen) * 0.1).cuda()
    xr = x.clone().requires_grad_(True)
    y_ref = module(xr)
    y_ref.backward(g)
    module.zero_grad()
    be = _backend(module, shape)
    native.reset_launches()
    (y,) = be.forward(x)
    (dx,) = be.backward(x, g)
    return be, native.launches(), y, y_ref.detach(), dx, xr.grad


@pytest.mark.gpu
@pytest.mark.parametrize("kind,width,heads", _sweep_cases())
def test_supports_never_lies(kind, width, heads):
    """every width ``supports()`` admits runs natively and agrees with the module (dropout 0, tiny batch, S = 8)"""
    torch.manual_seed(width + heads)
    if kind == "ffn":
        module, shape = FeedforwardBlock(width).cuda(), (16, width)
    else:
        module, shape = nn.TransformerEncoderLayer(width, heads, width + 128, dropout=0.0, batch_first=True).cuda(), (2, 8, width)
    be, launches, y, y_ref, dx, dx_ref = _one_call_each(module, shape)
    assert be._executor is not None and launches > 0
    assert bool(torch.isfinite(y).all() and torch.isfinite(dx).all())
    assert rel(y, y_ref) < 3e-2 and rel(dx, dx_ref) < 5e-2


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["d 4224", "d 320 (10 heads of 32)", "FeedforwardBlock(1152)"])
def test_widths_past_the_limits_run_on_the_module(name):
    torch.manual_seed(6)
    if name == "FeedforwardBlock(1152)":
        module, shape = FeedforwardBlock(1152).cuda().eval(), (16, 1152)
    else:
        d, heads = (4224, 33) if name == "d 4224" else (320, 10)
        module, shape = nn.TransformerEncoderLayer(d, heads, 2 * d, dropout=0.0, batch_first=True).cuda().eval(), (2, 8, d)
    be = _backend(module, shape)
    x = torch.randn(*shape, device="cuda")
    (y,) = be.forward(x)
    assert be._executor is None
    with torch.no_grad():
        assert torch.equal(y, module(x))
    (dx,) = be.backward(x, torch.ones_like(x) * 0.1)
    assert be._executor is None and bool(torch.isfinite(dx).all())


@pytest.mark.gpu
def test_throughput_server_ffn_768_round_trip():
    """``--block-type ffn --hid-dim 768``: one forward and one backward through RemoteExpert on the native executor"""
    from lah_b200.experiments.throughput.throughput_server import build_experts
    from lah_b200.ops import native
    from lah_b200.runtime.native_executor import NativeFFNExecutor
    torch.manual_seed(1)
    args = Namespace(hid_dim=768, block_type="ffn", layers_per_gpu=1, max_batch_size=256)
    experts = build_experts(args)
    srv = lah_b200.TesseractServer(None, experts, port=0, conn_handler_processes=1, device="cuda")
    srv.run_in_background()
    try:
        native.reset_launches()
        remote = lah_b200.RemoteExpert("expert0", "127.0.0.1", srv.port, timeout=120)
        x = torch.randn(64, 768, requires_grad=True)
        y = remote(x)
        assert y.shape == x.shape and bool(torch.isfinite(y).all())
        y.sum().backward()
        assert x.grad is not None and bool(torch.isfinite(x.grad).all())
        be = experts["expert0"]
        assert be.update_count == 1 and type(be._executor) is NativeFFNExecutor and native.launches() > 0
    finally:
        srv.shutdown()


@pytest.mark.gpu
def test_forward_only_layers_d768():
    from lah_b200.models.ffn_native import NativeFFNLayer
    from lah_b200.models.transformer_native import NativeTransformerLayer
    torch.manual_seed(1)
    layer = TransformerEncoderLayer(768, 12).cuda().eval()
    x = torch.randn(3, 300, 768, device="cuda")
    with torch.no_grad():
        ref = layer(x)
    out = NativeTransformerLayer(layer)(x)
    assert out.shape == x.shape and rel(out, ref) < 3e-2
    block = FeedforwardBlock(768).cuda().eval()
    x = torch.randn(512, 768, device="cuda")
    with torch.no_grad():
        ref = block(x)
    out = NativeFFNLayer(block)(x.to(BF16))
    assert out.shape == x.shape and rel(out, ref) < 3e-2
