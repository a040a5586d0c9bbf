"""Gated (SwiGLU) feed-forward experts: GatedFeedforwardBlock against its formula and its scripted form on the CPU; on the
GPU the RMSNorm and SwiGLU kernels against float64 oracles, and the block trained and served through ExpertBackend,
a server and every width ``supports()`` admits, with the refused variants left on the module."""
import copy
from argparse import Namespace

import pytest
import torch
import torch.nn.functional as F

import lah_b200
from lah_b200.models.layers import GatedFeedforwardBlock, gated_inner_dim, name_to_block, name_to_input
from lah_b200.ops import kernels as K
from lah_b200.runtime.native_executor import GatedFFNSpec, encoder_layer_spec, ffn_spec, gated_ffn_spec

BF16 = torch.bfloat16
EPS_BF16 = 2.0 ** -8   # one bf16 rounding, relative


def rel(a, b):
    return ((a.double() - b.double()).norm() / (b.double().norm() + 1e-12)).item()


def _backend(module, hid, opt=None, name="gated"):
    opt = opt if opt is not None else torch.optim.Adam(module.parameters(), lr=1e-4, amsgrad=True)
    return lah_b200.ExpertBackend(name=name, expert=module, opt=opt, args_schema=(lah_b200.BatchTensorProto(hid),),
                                  outputs_schema=lah_b200.BatchTensorProto(hid), max_batch_size=4096)


# ------------------------------------------------------------------------------------------------ CPU
def test_block_is_the_gated_formula_fp64():
    torch.manual_seed(0)
    block = GatedFeedforwardBlock(128, 256, eps=1e-5).double()
    with torch.no_grad():
        block.norm.weight.uniform_(0.5, 1.5)
    x = torch.randn(7, 3, 128, dtype=torch.float64)
    h = F.rms_norm(x, (128,), block.norm.weight, 1e-5)
    ref = x + F.silu(h @ block.w1.weight.t()) * (h @ block.w3.weight.t()) @ block.w2.weight.t()
    assert (block(x) - ref).abs().max().item() < 1e-12


def test_default_inner_dim_names_and_count():
    assert [gated_inner_dim(h) for h in (128, 1024, 4096)] == [384, 2816, 11008]
    assert GatedFeedforwardBlock(1024).w1.out_features == 2816
    block = GatedFeedforwardBlock(128)
    assert [n for n, _ in block.named_parameters()] == ["norm.weight", "w1.weight", "w2.weight", "w3.weight"]
    assert sum(p.numel() for p in block.parameters()) == 128 + 3 * 128 * 384
    assert block.norm.eps == 1e-6 and all(lin.bias is None for lin in (block.w1, block.w2, block.w3))


@pytest.mark.parametrize("train", [False, True])
def test_scripted_block_equals_plain(train):
    torch.manual_seed(1)
    block = GatedFeedforwardBlock(256, 384).train(train)
    scripted = torch.jit.script(copy.deepcopy(block))
    x = torch.randn(9, 256)
    assert torch.equal(block(x), scripted(x))


def test_gated_ffn_spec_and_refusals():
    class Sub(GatedFeedforwardBlock):
        pass
    block = GatedFeedforwardBlock(256, 512, eps=1e-5)
    for m in (block, torch.jit.script(copy.deepcopy(block)), Sub(256, 512, eps=1e-5)):
        assert gated_ffn_spec(m) == GatedFFNSpec(256, 512, 1e-5)
    assert ffn_spec(block) is None and encoder_layer_spec(block) is None
    bias = GatedFeedforwardBlock(128)
    bias.w3 = torch.nn.Linear(128, 384, bias=True)
    no_weight = GatedFeedforwardBlock(128)
    no_weight.norm = torch.nn.RMSNorm(128, elementwise_affine=False)
    eps_none = GatedFeedforwardBlock(128)
    eps_none.norm = torch.nn.RMSNorm(128, eps=None)
    for m in (bias, no_weight, eps_none):
        assert gated_ffn_spec(m) is None and gated_ffn_spec(torch.jit.script(m)) is None
    assert gated_ffn_spec(GatedFeedforwardBlock(128, eps=0.0)) is None
    assert gated_ffn_spec(torch.nn.Linear(4, 4)) is None


def test_name_to_block_and_server_schemas():
    assert isinstance(name_to_block["swiglu"](256), GatedFeedforwardBlock)
    assert name_to_input["swiglu"](5, 256).shape == (5, 256)
    from lah_b200.experiments.throughput.throughput_server import build_experts
    experts = build_experts(Namespace(hid_dim=128, block_type="swiglu", layers_per_gpu=2, max_batch_size=64))
    assert len(experts) == 2
    for be in experts.values():
        assert isinstance(be.expert, GatedFeedforwardBlock)
        assert be.args_schema == (lah_b200.BatchTensorProto(128),) and be.outputs_schema == lah_b200.BatchTensorProto(128)


def test_cpu_backend_runs_the_module_and_infers_its_schema():
    torch.manual_seed(2)
    block = GatedFeedforwardBlock(128, 256)
    ref = copy.deepcopy(block)
    be = lah_b200.ExpertBackend(name="cpu", expert=block, opt=torch.optim.Adam(block.parameters(), lr=1e-3),
                                args_schema=(lah_b200.BatchTensorProto(128),), max_batch_size=8)
    assert be.outputs_schema == lah_b200.BatchTensorProto(128, dtype=torch.float32)
    x = torch.randn(4, 128)
    (y,) = be.forward(x)
    assert be._executor is None and torch.equal(y, ref(x))
    (dx,) = be.backward(x, torch.ones_like(x))
    assert dx.shape == x.shape and be.update_count == 1


def _no_launch(monkeypatch):
    def no_launch():
        raise RuntimeError("a kernel was about to be launched")
    monkeypatch.setattr(K, "_lib", no_launch)


@pytest.mark.parametrize("C", [64, 192, 4224])
def test_rms_norm_wrappers_refuse_widths_before_any_launch(monkeypatch, C):
    _no_launch(monkeypatch)
    x = torch.zeros(16, C, dtype=BF16)
    gamma, rstd = torch.ones(C), torch.zeros(16)
    with pytest.raises(ValueError, match="width"):
        K.rms_norm_fwd(x, gamma, 1e-6, out=torch.empty_like(x), rstd=rstd)
    with pytest.raises(ValueError, match="width"):
        K.rms_norm_bwd(x, x, rstd, gamma, dx=torch.empty_like(x), dgamma=torch.zeros(C))


def test_rms_norm_wrappers_refuse_dtypes_and_shapes_before_any_launch(monkeypatch):
    _no_launch(monkeypatch)
    x = torch.zeros(16, 256, dtype=BF16)
    gamma, rstd = torch.ones(256), torch.zeros(16)
    bad_fwd = [dict(x=x.float()), dict(out=torch.empty(16, 256)), dict(gamma=gamma.to(BF16)), dict(rstd=torch.zeros(8)),
               dict(x=x.t().contiguous().t()), dict(eps=0.0), dict(x=x[None])]
    for bad in bad_fwd:
        kw = dict(x=x, gamma=gamma, eps=1e-6, out=torch.empty_like(x), rstd=rstd)
        kw.update(bad)
        with pytest.raises(ValueError):
            K.rms_norm_fwd(kw["x"], kw["gamma"], kw["eps"], out=kw["out"], rstd=kw["rstd"])
    bad_bwd = [dict(dn=x.float()), dict(dres=torch.zeros(16, 128, dtype=BF16)), dict(dgamma=torch.zeros(128)),
               dict(tile_rows=12), dict(dx=torch.empty(8, 256, dtype=BF16))]
    for bad in bad_bwd:
        kw = dict(dn=x, dx=torch.empty_like(x), dgamma=torch.zeros(256), dres=None, tile_rows=16)
        kw.update(bad)
        with pytest.raises(ValueError):
            K.rms_norm_bwd(kw["dn"], x, rstd, gamma, dx=kw["dx"], dgamma=kw["dgamma"], dres=kw["dres"],
                           tile_rows=kw["tile_rows"])


def test_swiglu_wrappers_refuse_before_any_launch(monkeypatch):
    _no_launch(monkeypatch)
    for h in (torch.zeros(8, 400, dtype=BF16), torch.zeros(8, 256), torch.zeros(8, 2, 128, dtype=BF16),
              torch.zeros(8, 512, dtype=BF16)[:, :256]):
        with pytest.raises(ValueError):
            K.swiglu_fwd(h)
    h = torch.zeros(8, 512, dtype=BF16)
    with pytest.raises(ValueError):
        K.swiglu_fwd(h, out=torch.empty(8, 512, dtype=BF16))
    with pytest.raises(ValueError):
        K.swiglu_bwd(torch.zeros(8, 512, dtype=BF16), h)
    with pytest.raises(ValueError):
        K.swiglu_bwd(torch.zeros(8, 256), h)


def test_oracles_match_autograd_fp64():
    gen = torch.Generator().manual_seed(3)
    x = torch.randn(5, 256, generator=gen, dtype=torch.float64, requires_grad=True)
    gamma = torch.randn(256, generator=gen, dtype=torch.float64, requires_grad=True)
    dn, dres = torch.randn(5, 256, generator=gen, dtype=torch.float64), torch.randn(5, 256, generator=gen, dtype=torch.float64)
    n = F.rms_norm(x, (256,), gamma, 1e-5)
    n.backward(dn)
    n_ref, rstd = K.rms_norm_fwd_ref(x.detach(), gamma.detach(), 1e-5)
    dx, dgamma = K.rms_norm_bwd_ref(dn, x.detach(), gamma.detach(), 1e-5, dres=dres)
    assert (n_ref - n.detach()).abs().max() < 1e-12 and (dx - dres - x.grad).abs().max() < 1e-12
    assert (dgamma - gamma.grad).abs().max() < 1e-12
    h = torch.randn(5, 512, generator=gen, dtype=torch.float64, requires_grad=True)
    da = torch.randn(5, 256, generator=gen, dtype=torch.float64)
    g, u = h.chunk(2, dim=-1)
    a = F.silu(g) * u
    a.backward(da)
    assert (K.swiglu_ref(h.detach()) - a.detach()).abs().max() < 1e-12
    assert (K.swiglu_bwd_ref(da, h.detach()) - h.grad).abs().max() < 1e-12


# ------------------------------------------------------------------------------------------------ GPU: kernels
def _bf16(gen, *shape, scale=1.0):
    return (torch.randn(*shape, generator=gen) * scale).to(BF16).cuda()


@pytest.mark.gpu
@pytest.mark.parametrize("C", K.LN_WIDTHS)
def test_rms_norm_kernels_match_fp64(C):
    """forward and backward at rows 1, 16 and 300 (a tail tile), with and without dres, eps 1e-6 and 1e-5: each output
    within one bf16 rounding of the float64 oracle plus fp32 terms far below it; a second backward is bit-identical"""
    for rows in (1, 16, 300):
        gen = torch.Generator().manual_seed(C + rows)
        x, dn, dres = _bf16(gen, rows, C), _bf16(gen, rows, C, scale=0.5), _bf16(gen, rows, C, scale=0.5)
        gamma = (1 + 0.2 * torch.randn(C, generator=gen)).cuda()
        start = torch.randn(C, generator=gen).cuda()
        for eps in (1e-6, 1e-5):
            n, rstd = torch.empty(rows, C, dtype=BF16, device="cuda"), torch.empty(rows, device="cuda")
            K.rms_norm_fwd(x, gamma, eps, out=n, rstd=rstd)
            n_ref, rstd_ref = K.rms_norm_fwd_ref(x.double(), gamma.double(), eps)
            tol = EPS_BF16 * n_ref.abs() + 1e-5 * (x.double().abs() * rstd_ref[:, None] * gamma.double().abs())
            assert bool(((n.double() - n_ref).abs() <= tol).all()), (C, rows, eps, "n")
            assert ((rstd.double() - rstd_ref).abs() / rstd_ref).max().item() < 5e-5, (C, rows, eps, "rstd")
            for with_dres in (False, True):
                r = dres if with_dres else None
                outs = []
                for _ in range(2):
                    dx, dg = torch.empty(rows, C, dtype=BF16, device="cuda"), start.clone()
                    K.rms_norm_bwd(dn, x, rstd, gamma, dx=dx, dgamma=dg, dres=r)
                    outs.append((dx, dg))
                torch.cuda.synchronize()
                assert torch.equal(outs[0][0], outs[1][0]) and torch.equal(outs[0][1], outs[1][1]), "two calls differ"
                dx, dg = outs[0]
                dx_ref, dg_ref = K.rms_norm_bwd_ref(dn.double(), x.double(), gamma.double(), eps,
                                                    dres=r.double() if r is not None else None)
                rs, xd, gd = rstd_ref[:, None], x.double(), dn.double() * gamma.double()
                mags = rs * gd.abs() + rs ** 3 * xd.abs() * (gd * xd).abs().mean(1, keepdim=True)
                if r is not None:
                    mags = mags + r.double().abs()
                tol = EPS_BF16 * dx_ref.abs() + 1e-4 * mags
                assert bool(((dx.double() - dx_ref).abs() <= tol).all()), (C, rows, eps, with_dres, "dx")
                terms = (dn.double() * xd * rs).abs().sum(0)
                err = (dg.double() - start.double() - dg_ref).abs()
                bound = 1e-4 * terms + 1e-6 * (start.double().abs() + dg.double().abs()) + 1e-30
                assert bool((err <= bound).all()), (C, rows, eps, "dgamma")


@pytest.mark.gpu
@pytest.mark.parametrize("inner", [128, 2816, 11008])
def test_swiglu_kernels_match_fp64(inner):
    rows = 37
    gen = torch.Generator().manual_seed(inner)
    h = torch.randn(rows, 2 * inner, generator=gen) * 3
    special = torch.tensor([0.0, 1e-3, 30.0, 1e4])
    special = torch.cat([special, -special])
    h[:, :len(special)] = special             # g takes every special value in every row
    h[:len(special), :inner:97] = special[:, None]
    h, da = h.to(BF16).cuda(), _bf16(gen, rows, inner)
    a = K.swiglu_fwd(h)
    dh = K.swiglu_bwd(da, h)
    assert torch.equal(a, K.swiglu_fwd(h)) and torch.equal(dh, K.swiglu_bwd(da, h)), "two calls differ"
    assert bool(torch.isfinite(a).all() and torch.isfinite(dh).all())
    hd, dd = h.double(), da.double()
    a_ref, dh_ref = K.swiglu_ref(hd), K.swiglu_bwd_ref(dd, hd)
    assert bool(((a.double() - a_ref).abs() <= (EPS_BF16 + 1e-5) * a_ref.abs() + 1e-30).all())
    g, u = hd.chunk(2, dim=-1)
    s = torch.sigmoid(g)
    tol_g = EPS_BF16 * dh_ref[:, :inner].abs() + 1e-5 * (dd * u).abs() * s * (1 + g.abs() * (1 - s)) + 1e-30
    tol_u = (EPS_BF16 + 1e-5) * dh_ref[:, inner:].abs() + 1e-30
    assert bool(((dh[:, :inner].double() - dh_ref[:, :inner]).abs() <= tol_g).all())
    assert bool(((dh[:, inner:].double() - dh_ref[:, inner:]).abs() <= tol_u).all())


# ------------------------------------------------------------------------------------------------ GPU: ExpertBackend
@pytest.mark.gpu
@pytest.mark.parametrize("rows", [1, 16, 300])
@pytest.mark.parametrize("hid", [128, 1024, 4096])
def test_expert_backend_trains_gated_block(hid, rows):
    """forward and dx against the float64 module, then three AMSGrad steps against eager torch Adam"""
    from lah_b200.ops import native
    from lah_b200.runtime.native_executor import NativeGatedFFNExecutor
    torch.manual_seed(hid + rows)
    block = GatedFeedforwardBlock(hid).cuda()
    with torch.no_grad():
        block.norm.weight.uniform_(0.5, 1.5)
    ref64, ref = copy.deepcopy(block).double(), copy.deepcopy(block)
    ref_opt = torch.optim.Adam(ref.parameters(), lr=1e-4, amsgrad=True)
    be = _backend(block, hid)
    gen = torch.Generator().manual_seed(rows)
    x = torch.randn(rows, hid, generator=gen).cuda()
    g = (torch.randn(rows, hid, generator=gen) * 0.1).cuda()
    native.reset_launches()
    (y,) = be.forward(x)
    assert type(be._executor) is NativeGatedFFNExecutor and native.launches() > 0
    xr = x.double().requires_grad_(True)
    y64 = ref64(xr)
    y64.backward(g.double())
    assert rel(y, y64.detach()) < 3e-2
    del ref64
    for it in range(3):
        launches = native.launches()
        (dx,) = be.backward(x, g)
        assert native.launches() > launches
        if it == 0:
            assert rel(dx, xr.grad) < 5e-2
        ref(x).backward(g)
        ref_opt.step()
        ref_opt.zero_grad()
    sd, rsd = be.state_dict(), ref.state_dict()
    assert max((sd["expert." + k] - v).abs().mean().item() for k, v in rsd.items()) < 1.5e-4


def _split_w1_w3(m, **kw):
    """w1 and w3 in different param groups (with different settings): the [W1; W3] update takes two launches"""
    opt = torch.optim.AdamW([dict(params=[m.norm.weight, m.w1.weight]), dict(params=[m.w3.weight, m.w2.weight])], **kw)
    opt.param_groups[1].update(lr=2e-4, amsgrad=False, weight_decay=0.1)
    return opt


def _no_decay_norm(m, **kw):
    """the usual recipe: decay on the weight matrices, none on the norm (which also gets its own lr)"""
    opt = torch.optim.AdamW([dict(params=[m.w1.weight, m.w2.weight, m.w3.weight]),
                             dict(params=[m.norm.weight], weight_decay=0.0)], **kw)
    opt.param_groups[1].update(lr=2e-4, amsgrad=False)
    return opt


@pytest.mark.gpu
@pytest.mark.parametrize("make_opt", [_no_decay_norm, _split_w1_w3], ids=["norm_no_decay", "w1_w3_split"])
def test_expert_backend_adamw_groups(make_opt):
    """a zero-gradient step is torch AdamW's result bit for bit; three random steps agree with eager AdamW; the
    checkpoint loads into an eager module and optimizer and one more step agrees"""
    from lah_b200.runtime.native_executor import NativeGatedFFNExecutor
    hid, inner, rows = 512, 1024, 40
    kw = dict(lr=1e-4, weight_decay=0.05, amsgrad=True)
    torch.manual_seed(5)
    block = GatedFeedforwardBlock(hid, inner).cuda()
    ref = copy.deepcopy(block)
    be, ref_opt = _backend(block, hid, opt=make_opt(block, **kw)), make_opt(ref, **kw)
    gen = torch.Generator().manual_seed(6)
    x = torch.randn(rows, hid, generator=gen).cuda()
    before = {n: p.detach().clone() for n, p in ref.named_parameters()}
    be.backward(x, torch.zeros_like(x))
    assert type(be._executor) is NativeGatedFFNExecutor
    for p in ref.parameters():
        p.grad = torch.zeros_like(p)
    ref_opt.step()
    ref_opt.zero_grad()
    no_decay = {id(p) for grp in ref_opt.param_groups if grp["weight_decay"] == 0 for p in grp["params"]}
    for (n, p), r in zip(block.named_parameters(), ref.parameters()):
        assert torch.equal(p.detach().view(torch.int32), r.detach().view(torch.int32)), f"{n}: not AdamW's result"
        assert torch.equal(p.detach(), before[n]) == (id(r) in no_decay), n
    g = (torch.randn(rows, hid, generator=gen) * 0.1).cuda()
    for _ in range(3):
        be.backward(x, g)
        ref(x).backward(g)
        ref_opt.step()
        ref_opt.zero_grad()
    sd, rsd = be.state_dict(), ref.state_dict()
    assert max((sd["expert." + k] - v).abs().mean().item() for k, v in rsd.items()) < 1.5e-4
    ck = copy.deepcopy(be.checkpoint())
    fresh = copy.deepcopy(ref)
    fresh.load_state_dict({k[len("expert."):]: v for k, v in ck["model"].items()})
    fresh_opt = make_opt(fresh, **kw)
    fresh_opt.load_state_dict(ck["optimizer"])
    be.backward(x, g)
    fresh(x).backward(g)
    fresh_opt.step()
    sd, fsd = be.state_dict(), fresh.state_dict()
    assert max((sd["expert." + k] - v).abs().mean().item() for k, v in fsd.items()) < 5e-5
    for p, q in zip(be.opt.param_groups[0]["params"], fresh_opt.param_groups[0]["params"]):
        assert float(be.opt.state[p]["step"]) == float(fresh_opt.state[q]["step"]) == 5.0


@pytest.mark.gpu
def test_scripted_block_through_backend_is_bit_identical():
    torch.manual_seed(7)
    block = GatedFeedforwardBlock(1024).cuda()
    scripted = torch.jit.script(copy.deepcopy(block))
    bes = [_backend(m, 1024, name=f"b{i}") for i, m in enumerate((block, scripted))]
    gen = torch.Generator().manual_seed(8)
    x = torch.randn(100, 1024, generator=gen).cuda()
    g = (torch.randn(100, 1024, generator=gen) * 0.1).cuda()
    outs = []
    for be in bes:
        (y,) = be.forward(x)
        (dx,) = be.backward(x, g)
        (y2,) = be.forward(x)
        assert be._executor is not None
        outs.append((y, dx, y2, be.state_dict()))
    (y, dx, y2, sd), (ys, dxs, y2s, sds) = outs
    assert torch.equal(y, ys) and torch.equal(dx, dxs) and torch.equal(y2, y2s)
    assert all(torch.equal(sd[k], sds[k]) for k in sd)


@pytest.mark.gpu
def test_throughput_server_swiglu_round_trip():
    """``--block-type swiglu --hid-dim 1024``: one forward and one backward through RemoteExpert on the native executor"""
    from lah_b200.experiments.throughput.throughput_server import build_experts
    from lah_b200.ops import native
    from lah_b200.runtime.native_executor import NativeGatedFFNExecutor
    torch.manual_seed(1)
    experts = build_experts(Namespace(hid_dim=1024, block_type="swiglu", layers_per_gpu=1, max_batch_size=256))
    srv = lah_b200.TesseractServer(None, experts, port=0, conn_handler_processes=1, device="cuda")
    srv.run_in_background()
    try:
        native.reset_launches()
        remote = lah_b200.RemoteExpert("expert0", "127.0.0.1", srv.port, timeout=120)
        x = torch.randn(64, 1024, requires_grad=True)
        y = remote(x)
        assert y.shape == x.shape and bool(torch.isfinite(y).all())
        y.sum().backward()
        assert x.grad is not None and bool(torch.isfinite(x.grad).all())
        be = experts["expert0"]
        assert be.update_count == 1 and type(be._executor) is NativeGatedFFNExecutor and native.launches() > 0
    finally:
        srv.shutdown()


@pytest.mark.gpu
@pytest.mark.parametrize("hid", list(range(128, 4097, 128)))
def test_supports_never_lies(hid):
    """every width ``supports()`` admits runs natively and agrees with the module (16 rows, inner 256)"""
    from lah_b200.ops import native
    torch.manual_seed(hid)
    module = GatedFeedforwardBlock(hid, 256).cuda()
    gen = torch.Generator().manual_seed(1)
    x = torch.randn(16, hid, generator=gen).cuda()
    g = (torch.randn(16, hid, generator=gen) * 0.1).cuda()
    xr = x.clone().requires_grad_(True)
    y_ref = module(xr)
    y_ref.backward(g)
    module.zero_grad()
    be = _backend(module, hid)
    native.reset_launches()
    (y,) = be.forward(x)
    (dx,) = be.backward(x, g)
    assert be._executor is not None and native.launches() > 0
    assert bool(torch.isfinite(y).all() and torch.isfinite(dx).all())
    assert rel(y, y_ref.detach()) < 3e-2 and rel(dx, xr.grad) < 5e-2


@pytest.mark.gpu
@pytest.mark.parametrize("variant", ["hid 4224", "inner 200", "Linear with a bias", "SGD"])
def test_refused_variants_run_on_the_module(variant):
    torch.manual_seed(9)
    hid = 4224 if variant == "hid 4224" else 256
    module = GatedFeedforwardBlock(hid, 200 if variant == "inner 200" else 256).cuda()
    if variant == "Linear with a bias":
        module.w2 = torch.nn.Linear(256, 256).cuda()
    opt = torch.optim.SGD(module.parameters(), lr=1e-3) if variant == "SGD" else None
    ref = copy.deepcopy(module)
    be = _backend(module, hid, opt=opt)
    x = torch.randn(16, hid, device="cuda")
    (y,) = be.forward(x)
    assert be._executor is None
    with torch.no_grad():
        assert torch.equal(y, ref(x))
    (dx,) = be.backward(x, torch.ones_like(x) * 0.1)
    assert be._executor is None and bool(torch.isfinite(dx).all()) and be.update_count == 1
