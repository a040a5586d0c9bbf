"""
Weight decay in the optimizer kernels and everything that drives them: torch's L2 form (Adam(weight_decay=wd): the gradient
gets wd * p) and its decoupled form (AdamW, Adam(decoupled_weight_decay=True): p *= 1 - lr wd before the moments).

The kernels are checked element by element against the float64 oracle of test_expert_kernels.py, extended here by the
decoupled form: the kernel rounds p * decay to fp32 on its own (decay = 1 - lr wd, rounded to fp32 once on the host), so
the oracle decays p in float64 and adds one fp32 rounding of the decayed value to the bound of p.  Through ExpertBackend,
a two-group AdamW (decay on the weight matrices, none on biases and LayerNorm parameters) runs on the sm_90a executors and
is compared with eager torch: bit for bit on a step whose gradient is zero, within the tolerance of the existing
training tests on random gradients.  The in-box engine's CPU path is compared with one torch optimizer per expert, and the
GPU trainer with that CPU path.
"""
import copy

import pytest
import torch
from torch import nn

from test_expert_kernels import (BF16, SENTINEL, U, adam_ref64, adam_state, f32, poison, sentinel_like,  # noqa: F401
                                 untouched, within)
from test_fused_adam_fp8_kernels import WA_ADAM_ROWS, WA_ADAM_STEPS, same_bytes, wa_adam_setup

import lah_b200
from lah_b200.models.layers import FeedforwardBlock, TransformerEncoderLayer
from lah_b200.ops import kernels as K
from lah_b200.runtime import native_executor as NE


# ---------------------------------------------------------------------------------------------------------------- oracle
def adamw_ref64(p, g, m, v, vmax, seg_sizes, G, *, lr=1e-3, weight_decay=0.0, decoupled=False, decay=None, **kw):
    """``adam_ref64`` with torch's two weight-decay forms.  Decoupled: p is multiplied by ``decay`` (default 1 - lr wd in
    double; pass the fp32 rounding the kernel receives) before the Adam step; the bound of p gains the fp32 rounding of that
    product.  Elements that are not updated keep their p."""
    if not (decoupled and weight_decay):
        return adam_ref64(p, g, m, v, vmax, seg_sizes, G, lr=lr, weight_decay=weight_decay, **kw)
    decay = 1.0 - lr * weight_decay if decay is None else decay
    P = p.double()
    pd = P * decay
    new, upd, bounds = adam_ref64(pd, g, m, v, vmax, seg_sizes, G, lr=lr, **kw)
    new["p"] = torch.where(upd, new["p"], P)
    bounds["p"] = bounds["p"] + U * pd.abs()
    return new, upd, bounds


def kernel_decay(lr, weight_decay):
    """the decoupled factor as the kernels receive it: 1 - lr wd in double, rounded to fp32"""
    return f32(1.0 - lr * weight_decay)


# ---------------------------------------------------------------------------------------------------------------- CPU
@pytest.mark.parametrize("amsgrad", [True, False])
@pytest.mark.parametrize("kind", ["AdamW", "Adam_decoupled"])
def test_decoupled_oracle_matches_torch_step_for_step(kind, amsgrad):
    gen = torch.Generator().manual_seed(5)
    n, lr, betas, eps, wd = 64, 3e-3, (0.8, 0.99), 1e-6, 0.3
    w = torch.nn.Parameter(torch.randn(n, generator=gen, dtype=torch.float64))
    kw = dict(lr=lr, betas=betas, eps=eps, weight_decay=wd, amsgrad=amsgrad)
    opt = torch.optim.AdamW([w], **kw) if kind == "AdamW" else torch.optim.Adam([w], decoupled_weight_decay=True, **kw)
    p, m, v, vmax = (w.detach().clone(),) + tuple(torch.zeros(n, dtype=torch.float64) for _ in range(3))
    for step in range(1, 7):
        grad = torch.randn(n, generator=gen, dtype=torch.float64) * (0.1 if step % 2 else 2.0)
        w.grad = grad.clone()
        opt.step()
        new, upd, _ = adamw_ref64(p, grad, m, v, vmax, [n], 1, step=step, decoupled=True, **kw)
        assert bool(upd.all())
        p, m, v, vmax = new["p"], new["m"], new["v"], new["vmax"]
        st = opt.state[w]
        torch.testing.assert_close(p, w.detach(), rtol=1e-13, atol=1e-15)
        torch.testing.assert_close(m, st["exp_avg"], rtol=1e-13, atol=1e-15)
        torch.testing.assert_close(v, st["exp_avg_sq"], rtol=1e-13, atol=1e-18)
        if amsgrad:
            torch.testing.assert_close(vmax, st["max_exp_avg_sq"], rtol=1e-13, atol=1e-18)


@pytest.mark.parametrize("decoupled", [False, True])
def test_adam_step_ref_weight_decay_matches_torch(decoupled):
    """the fp32 CPU optimizer of the engine's oracle path, per group, against one torch optimizer per group; group 1 is
    inactive (no rows) in the second step and keeps its parameters"""
    gen = torch.Generator().manual_seed(6)
    G, segs, lr, wd = 2, [8, 4], 1e-2, 0.5
    n = G * sum(segs)
    p = torch.randn(n, generator=gen)
    m, v, vmax = torch.zeros(n), torch.zeros(n), torch.zeros(n)
    refs = [[p[g * 8: g * 8 + 8].clone().requires_grad_(), p[16 + g * 4: 20 + g * 4].clone().requires_grad_()] for g in range(G)]
    opts = [torch.optim.Adam(r, lr=lr, amsgrad=True, weight_decay=wd, decoupled_weight_decay=decoupled) for r in refs]
    step = torch.zeros(G, dtype=torch.int32)
    for rows in ([1, 1], [3, 0], [2, 5]):
        grad = torch.randn(n, generator=gen)
        rows = torch.tensor(rows)
        step += (rows > 0).int()
        K.adam_step_ref(p, grad.clone(), m, v, vmax, segs, G, step=step, group_rows=rows, lr=lr, weight_decay=wd,
                        decoupled=decoupled)
        for g in range(G):
            if rows[g] > 0:
                refs[g][0].grad, refs[g][1].grad = grad[g * 8: g * 8 + 8].clone(), grad[16 + g * 4: 20 + g * 4].clone()
                opts[g].step()
    for g in range(G):
        torch.testing.assert_close(p[g * 8: g * 8 + 8], refs[g][0].detach(), rtol=1e-6, atol=1e-7)
        torch.testing.assert_close(p[16 + g * 4: 20 + g * 4], refs[g][1].detach(), rtol=1e-6, atol=1e-7)


def _two_groups(module, opt_cls=torch.optim.AdamW, **kw):
    """the usual transformer recipe: decay on the weight matrices, none on biases and LayerNorm parameters"""
    decay = [p for p in module.parameters() if p.dim() >= 2]
    no_decay = [p for p in module.parameters() if p.dim() < 2]
    return opt_cls([dict(params=decay), dict(params=no_decay, weight_decay=0.0)], **kw)


def _cpu_experts():
    torch.manual_seed(0)
    return [(FeedforwardBlock(128), NE.NativeFFNExecutor._segment_params),
            (TransformerEncoderLayer(256, 4), NE.NativeTransformerExecutor._segment_params),
            (nn.TransformerEncoderLayer(256, 4), NE.NativeTransformerExecutor._segment_params)]


def test_optimizer_groups_accepts_and_refuses():
    for module, seg_params in _cpu_experts():
        params = seg_params(module)
        matrices = sum(1 << s for s, p in enumerate(params) if p.dim() >= 2)
        everything = (1 << len(params)) - 1
        groups = lambda opt: NE.optimizer_groups(opt, params)
        # accepted
        assert groups(_two_groups(module, weight_decay=0.01)) == [matrices, everything & ~matrices]
        assert groups(torch.optim.Adam(module.parameters())) == [everything]
        assert groups(torch.optim.Adam(module.parameters(), weight_decay=0.1, amsgrad=True, foreach=True)) == [everything]
        assert groups(torch.optim.Adam(module.parameters(), weight_decay=0.1, decoupled_weight_decay=True)) == [everything]
        per_lr = _two_groups(module, torch.optim.Adam, lr=1e-3)
        per_lr.param_groups[1].update(lr=5e-4, betas=(0.8, 0.9), eps=1e-6, amsgrad=True)
        assert groups(per_lr) == [matrices, everything & ~matrices]
        one_by_one = torch.optim.AdamW([dict(params=[p], lr=1e-4 * (s + 1)) for s, p in enumerate(params)])
        assert groups(one_by_one) == [1 << s for s in range(len(params))]
        # refused
        assert groups(torch.optim.Adam(module.parameters(), maximize=True)) is None
        assert groups(torch.optim.AdamW(module.parameters(), differentiable=True)) is None
        capt = torch.optim.Adam(module.parameters())
        capt.param_groups[0]["capturable"] = True
        assert groups(capt) is None
        assert groups(torch.optim.Adam(module.parameters(), lr=torch.tensor(1e-3), foreach=False)) is None
        assert groups(torch.optim.Adam(module.parameters(), betas=(torch.tensor(0.9), torch.tensor(0.99)),
                                       foreach=False)) is None
        assert groups(torch.optim.AdamW(params[1:])) is None                          # a parameter missing
        dup = _two_groups(module)
        dup.param_groups[1]["params"].append(params[0])                              # a parameter present twice
        assert groups(dup) is None
        neg = torch.optim.AdamW(module.parameters())
        neg.param_groups[0]["weight_decay"] = -0.1
        assert groups(neg) is None
        assert groups(torch.optim.SGD(module.parameters(), lr=0.1)) is None
        assert groups(type("MyAdam", (torch.optim.Adam,), {})(module.parameters())) is None


@pytest.mark.parametrize("decoupled", [False, True])
def test_engine_cpu_path_weight_decay_matches_torch_per_expert(decoupled):
    """the fused layer's CPU path against one torch optimizer per expert (BaselineDMoE) over three steps, with experts that
    receive no rows in some steps (they are neither stepped nor decayed)"""
    from lah_b200.parallel import baseline, engine as E
    torch.manual_seed(0)
    cfg = E.DMoEConfig(hidden=32, grid_size=(2, 4), k=2, num_layers=1, tokens_per_rank=16, lr=1e-2, weight_decay=0.5,
                       decoupled_weight_decay=decoupled)
    fused = E.FusedDMoE(cfg).train()
    base = baseline.BaselineDMoE(cfg)
    base.load_from_shard(fused.shard)
    base.proj.load_state_dict(fused.proj.state_dict())
    start = [fused.shard.expert_state_dict(e) for e in range(cfg.num_experts)]
    idle = set()
    for it in range(3):
        x = torch.randn(3, 32)
        t = torch.randn(3, 32)
        (fused(x) * t).sum().backward()
        (base(x.clone()) * t).sum().backward()
        idle |= {e for e in range(cfg.num_experts) if int(base._rows[e]) == 0}
        fused.apply_expert_gradients_ref()
        base.apply_expert_gradients()
    assert idle, "every expert received rows in every step: the case of an idle expert was not exercised"
    moved = 0
    for e, expert in enumerate(base.experts):
        sd = fused.shard.expert_state_dict(e, prefix="")
        for k, v in expert.state_dict().items():
            torch.testing.assert_close(sd[k], v, rtol=1e-4, atol=2e-5)   # Adam amplifies last-bit gradient differences
            moved += not torch.equal(sd[k], start[e]["expert." + k])
    assert moved
    group = fused.shard.expert_optimizer_state(0)["param_groups"][0]
    assert group["weight_decay"] == 0.5 and group["decoupled_weight_decay"] == decoupled


# ---------------------------------------------------------------------------------------------------------------- GPU
SEGS12 = [4, 8, 12, 36, 4, 100, 8, 64, 20, 4, 16, 260]
ADAM_WD_CASES = {
    "l2_all_segments_shadow_slots": dict(weight_decay=0.1, decoupled=False, seg_mask=0, G_active=3, amsgrad=True),
    "decoupled_all_segments": dict(weight_decay=0.1, decoupled=True, seg_mask=0, G_active=0, amsgrad=True),
    "decoupled_six_ranges_no_amsgrad": dict(weight_decay=0.3, decoupled=True, seg_mask=0b010101010101, G_active=5,
                                            amsgrad=False),
    "decoupled_merged_ranges_shadow_slots": dict(weight_decay=2.0, decoupled=True, seg_mask=0b110101101011, G_active=4,
                                                 amsgrad=True),
    "l2_two_ranges": dict(weight_decay=0.05, decoupled=False, seg_mask=0b000011100011, G_active=0, amsgrad=False),
}


@pytest.mark.gpu
@pytest.mark.parametrize("case", list(ADAM_WD_CASES))
def test_adam_step_weight_decay_elementwise(case, poison, record_property):
    """two consecutive launches against the oracle; everything outside the update (other segments, inactive and shadow
    groups, the mirror there, vmax without amsgrad) byte for byte untouched"""
    c = dict(ADAM_WD_CASES[case])
    G, lr = 5, 2e-3
    st = adam_state(len(case) + 100, SEGS12, G)
    rows = torch.tensor([3, 0, 1, 7, 2], dtype=torch.int32, device="cuda")
    step = torch.tensor([1, 4, 2, 9, 3], dtype=torch.int32, device="cuda")
    wd, dec, amsgrad = c.pop("weight_decay"), c.pop("decoupled"), c["amsgrad"]
    worst = 0.0
    for _ in range(2):
        t = {k: x.clone() for k, x in st.items()}
        K.adam_step(t["p"], t["g"], t["m"], t["v"], t["vmax"], t["p_bf16"], SEGS12, G, step=step, group_rows=rows, lr=lr,
                    weight_decay=wd, decoupled=dec, zero_mask=0xFFF, **c)
        torch.cuda.synchronize()
        new, upd, bounds = adamw_ref64(st["p"], st["g"], st["m"], st["v"], st["vmax"], SEGS12, G, step=step,
                                       group_rows=rows, lr=f32(lr), betas=(f32(0.9), f32(0.999)), eps=f32(1e-8),
                                       weight_decay=f32(wd), decoupled=dec, decay=kernel_decay(lr, wd), zero_mask=0xFFF, **c)
        assert upd.any() and not upd.all()
        for name in ("p", "m", "v") + (("vmax",) if amsgrad else ()):
            worst = max(worst, within(t[name][upd], new[name][upd], bounds[name][upd], name, "adam_step wd"))
        for name in ("p", "g", "m", "v", "vmax"):
            assert same_bytes(t[name][~upd], st[name][~upd]), f"{name} changed outside the stepped elements"
        if not amsgrad:
            assert same_bytes(t["vmax"], st["vmax"]), "vmax written without amsgrad"
        assert torch.equal(t["g"][upd], torch.zeros_like(t["g"][upd])), "the gradient of the stepped elements is not zeroed"
        assert same_bytes(t["p_bf16"][upd], t["p"][upd].to(BF16)), "p_bf16 is not the bf16 rounding of p"
        assert bool(untouched(t["p_bf16"][~upd]).all())
        st, step = t, step + 1
    record_property("max_err_over_bound", worst)


@pytest.mark.gpu
def test_adam_step_decoupled_zero_gradient_is_torch_mul():
    """a first step with a zero gradient moves p exactly to torch's p.mul_(1 - lr wd) (fp32), on every element"""
    G, segs, lr, wd = 2, [64, 1024], 1e-3, 0.01
    n = G * sum(segs)
    gen = torch.Generator().manual_seed(9)
    p = torch.randn(n, generator=gen).cuda()
    z = lambda: torch.zeros(n, device="cuda")
    t = p.clone()
    K.adam_step(t, z(), z(), z(), z(), torch.empty(n, dtype=BF16, device="cuda"), segs, G, step_scalar=1, lr=lr,
                weight_decay=wd, decoupled=True)
    torch.cuda.synchronize()
    assert same_bytes(t, p.clone().mul_(1 - lr * wd))
    assert not torch.equal(t, p)


WA_WD_CASES = {
    "l2_amsgrad": dict(weight_decay=0.05, decoupled=False, amsgrad=True),
    "l2_adam": dict(weight_decay=0.5, decoupled=False, amsgrad=False),
    "decoupled_amsgrad": dict(weight_decay=0.1, decoupled=True, amsgrad=True),
    "decoupled_adam_n2048_k512": dict(weight_decay=3.0, decoupled=True, amsgrad=False, N=2048, K_=512, max_ctas=80),
}


@pytest.mark.gpu
@pytest.mark.parametrize("case", list(WA_WD_CASES))
def test_wgrad_adam_weight_decay_elementwise(case, poison, record_property):
    """the fused wgrad + AMSGrad kernel with each decay form on the exact-gradient operands of
    test_fused_adam_fp8_kernels.py: two consecutive launches against the oracle, unstepped groups byte for byte untouched"""
    c = dict(WA_WD_CASES[case])
    N, K_, lr, betas, eps = c.get("N", 256), c.get("K_", 384), 2e-3, (0.9, 0.999), 1e-8
    wd, dec, amsgrad = c["weight_decay"], c["decoupled"], c["amsgrad"]
    dy, x, go, gr, skip, rows_eff, stepped, st, grad = wa_adam_setup(list(WA_WD_CASES).index(case) + 120, N, K_)
    G = len(WA_ADAM_ROWS)
    step = torch.tensor(WA_ADAM_STEPS, dtype=torch.int32, device="cuda")
    worst = 0.0
    for _ in range(2):
        t = {k: (x_.clone() if x_ is not None else None) for k, x_ in st.items()}
        K.wgrad_adam(dy, x, go, gr, p=t["p"], m=t["m"], v=t["v"], vmax=t["vmax"], p_bf16=t["p_bf16"], step=step, skip=skip,
                     lr=lr, betas=betas, eps=eps, amsgrad=amsgrad, weight_decay=wd, decoupled=dec,
                     max_ctas=c.get("max_ctas", 0))
        torch.cuda.synchronize()
        new, upd, bounds = adamw_ref64(st["p"].view(-1), grad.view(-1), st["m"].view(-1), st["v"].view(-1),
                                       st["vmax"].view(-1), [N * K_], G, step=step, group_rows=rows_eff, lr=f32(lr),
                                       betas=tuple(map(f32, betas)), eps=f32(eps), amsgrad=amsgrad, grad=grad.view(-1),
                                       weight_decay=f32(wd), decoupled=dec, decay=kernel_decay(lr, wd))
        for name in ("p", "m", "v") + (("vmax",) if amsgrad else ()):
            got = t[name].view(-1)
            worst = max(worst, within(got[upd], new[name][upd], bounds[name][upd], name, "wgrad_adam wd"))
        for g in range(G):
            if not stepped[g]:
                for name, a in t.items():
                    assert same_bytes(a[g], st[name][g]), f"{name} of unstepped group {g} was written"
            else:
                assert same_bytes(t["p_bf16"][g], t["p"][g].to(BF16))
        if not amsgrad:
            assert same_bytes(t["vmax"], st["vmax"]), "vmax written without amsgrad"
        st, step = t, step + torch.tensor(stepped, dtype=torch.int32, device="cuda")
    record_property("max_err_over_bound", worst)


# ------------------------------------------------------------------ ExpertBackend
def _expert(kind):
    torch.manual_seed(3)
    if kind == "ffn":
        return FeedforwardBlock(1024).cuda(), (200, 1024)
    if kind == "own transformer":
        return TransformerEncoderLayer(1024, 16).cuda(), (2, 300, 1024)
    return nn.TransformerEncoderLayer(1024, 16, dropout=0.1).cuda(), (300, 2, 1024)


def _ref_forward(module, x, seed):
    """the eager fp32 forward with the dropout masks the executor draws from ``seed`` (the FFN has no dropout)"""
    from test_encoder_layer_experts import _masks, encoder_layer_ref
    if isinstance(module, FeedforwardBlock):
        return module(x)
    spec = NE.encoder_layer_spec(module)
    batch, S = (x.shape[0], x.shape[1]) if spec.batch_first else (x.shape[1], x.shape[0])
    return encoder_layer_ref(module, x, _masks(seed, spec, batch, S))


AW = dict(lr=1e-4, weight_decay=0.05, amsgrad=True)


def _aw(module):
    """two-group AdamW: the no-decay group also has its own lr and no amsgrad"""
    opt = _two_groups(module, **AW)
    opt.param_groups[1].update(lr=2e-4, amsgrad=False)
    return opt


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["ffn", "own transformer", "torch transformer"])
def test_expert_backend_trains_with_two_group_adamw(kind):
    from lah_b200.ops import native
    from lah_b200.runtime.native_executor import draw_dropout_seed
    module, shape = _expert(kind)
    ref = copy.deepcopy(module)
    ref_opt = _aw(ref)
    be = lah_b200.ExpertBackend(name="t", expert=module, opt=_aw(module), args_schema=(lah_b200.BatchTensorProto(*shape[1:]),),
                                outputs_schema=lah_b200.BatchTensorProto(*shape[1:]), max_batch_size=8)
    gen = torch.Generator().manual_seed(7)
    x = torch.randn(*shape, generator=gen).cuda()
    before = [p.detach().clone() for p in ref.parameters()]
    # a step with a zero output gradient: every gradient is zero, so Adam moves nothing and only the decay acts
    native.reset_launches()
    be.backward(x, torch.zeros_like(x))
    assert type(be._executor) in (NE.NativeFFNExecutor, NE.NativeTransformerExecutor) and native.launches() > 0
    for p in ref.parameters():
        p.grad = torch.zeros_like(p)
    ref_opt.step()
    ref_opt.zero_grad()
    for (n, p), r, b in zip(module.named_parameters(), ref.parameters(), before):
        assert same_bytes(p.detach(), r.detach()), f"{n}: not torch AdamW's result bit for bit"
        assert torch.equal(p.detach(), b) == (p.dim() < 2), f"{n}: decayed {'although' if p.dim() < 2 else 'not'} in a group with decay"
    # random gradients: three steps against the eager fp32 copy with the same dropout masks
    g = (torch.randn(*shape, generator=gen) * 0.1).cuda()
    for it in range(3):
        torch.manual_seed(20 + it)
        seed = draw_dropout_seed()
        torch.manual_seed(20 + it)
        launches = native.launches()
        be.backward(x, g)
        assert native.launches() > launches
        _ref_forward(ref, x, seed).backward(g)
        ref_opt.step()
        ref_opt.zero_grad()
    sd, rsd = be.state_dict(), ref.state_dict()
    assert max((sd["expert." + k] - v).abs().mean().item() for k, v in rsd.items()) < 1.5e-4
    # the checkpoint loads into a fresh eager AdamW and the next step agrees
    ck = copy.deepcopy(be.checkpoint())
    fresh = copy.deepcopy(ref)
    fresh.load_state_dict({k[len("expert."):]: v for k, v in ck["model"].items()})
    fresh_opt = _aw(fresh)
    fresh_opt.load_state_dict(ck["optimizer"])
    assert fresh_opt.param_groups[0]["decoupled_weight_decay"] and fresh_opt.param_groups[0]["weight_decay"] == 0.05
    torch.manual_seed(30)
    seed = draw_dropout_seed()
    torch.manual_seed(30)
    be.backward(x, g)
    _ref_forward(fresh, x, seed).backward(g)
    fresh_opt.step()
    sd, fsd = be.state_dict(), fresh.state_dict()
    assert max((sd["expert." + k] - v).abs().mean().item() for k, v in fsd.items()) < 5e-5   # one step from one state
    for p, q in zip(be.opt.param_groups[0]["params"], fresh_opt.param_groups[0]["params"]):
        st, fst = be.opt.state[p], fresh_opt.state[q]
        assert float(st["step"]) == float(fst["step"]) == 5.0


@pytest.mark.gpu
@pytest.mark.parametrize("refusal", ["maximize", "tensor lr", "missing parameter"])
def test_refused_optimizers_train_on_the_module(refusal):
    """an optimizer the executors refuse leaves the expert on the module, which trains as eager torch does"""
    module, shape = _expert("ffn")
    ref = copy.deepcopy(module)

    def make(m):
        if refusal == "maximize":
            return _two_groups(m, lr=1e-3, weight_decay=0.1, maximize=True)
        if refusal == "tensor lr":
            return torch.optim.AdamW(m.parameters(), lr=torch.tensor(1e-3), weight_decay=0.1, foreach=False)
        return torch.optim.AdamW(list(m.parameters())[2:], lr=1e-3, weight_decay=0.1)
    be = lah_b200.ExpertBackend(name="t", expert=module, opt=make(module), args_schema=(lah_b200.BatchTensorProto(*shape[1:]),),
                                outputs_schema=lah_b200.BatchTensorProto(*shape[1:]), max_batch_size=8)
    ref_opt = make(ref)
    gen = torch.Generator().manual_seed(8)
    x = torch.randn(*shape, generator=gen).cuda()
    before = [p.detach().clone() for p in module.parameters()]
    for it in range(3):
        g = (torch.randn(*shape, generator=gen) * 0.1).cuda()
        be.backward(x, g)
        assert be._executor is None
        ref(x.clone().requires_grad_(True)).backward(g)
        ref_opt.step()
        ref_opt.zero_grad()
    for p, r, b in zip(module.parameters(), ref.parameters(), before):
        torch.testing.assert_close(p, r, rtol=1e-5, atol=1e-6)
    assert any(not torch.equal(p, b) for p, b in zip(module.parameters(), before))


# ------------------------------------------------------------------ DMoETrainer
def _trainer_params(tr):
    return torch.cat([tr.model.blocks[0].shard.expert_state_dict(e)[k].reshape(-1)
                      for e in range(tr.cfg.num_experts) for k in sorted(tr.model.blocks[0].shard.expert_state_dict(e))])


@pytest.mark.gpu
@pytest.mark.parametrize("path", ["small", "big"])
@pytest.mark.parametrize("decoupled", [False, True])
def test_trainer_weight_decay_matches_cpu_path(path, decoupled):
    """DMoETrainer on one GPU against its CPU path from the same weights over three steps: the expert parameters of the
    two are much closer to each other than to a CPU run without weight decay (which they would match if the decay were
    lost), and the losses agree as in the fused-vs-baseline parity check"""
    from lah_b200.parallel import engine as E
    from lah_b200.parallel.trainer import DMoETrainer
    wd = 30.0 if decoupled else 1.0   # per step: p *= 0.97, or an L2 term that dominates the expert gradients
    cfgs = {w: E.DMoEConfig(hidden=512, grid_size=(16,), k=4, num_layers=1, tokens_per_rank=256, lr=1e-3, weight_decay=w,
                            decoupled_weight_decay=decoupled, expert_path=path) for w in (wd, 0.0)}
    gpu = DMoETrainer(cfgs[wd])
    assert gpu.ctx.small == (path == "small")
    cpus = {w: DMoETrainer(cfg, device="cpu") for w, cfg in cfgs.items()}
    for cpu in cpus.values():   # the same starting point: trainer parameters (gate included) and every expert
        with torch.no_grad():
            cpu.flat_p.copy_(gpu.flat_p.cpu())
        for e in range(cfgs[wd].num_experts):
            cpu.model.blocks[0].shard.load_expert_state_dict(e, gpu.model.blocks[0].shard.expert_state_dict(e))
    gen = torch.Generator().manual_seed(0)
    protos = torch.randn(10, cfgs[wd].in_features, generator=gen)
    y = torch.randint(0, 10, (256,), generator=gen)
    x = protos[y] + 3.0 * torch.randn(256, cfgs[wd].in_features, generator=gen)
    start = _trainer_params(gpu)
    losses = {"gpu": [float(gpu.train_step_device(x.cuda(), y.cuda())) for _ in range(3)]}
    gpu.ctx.check_status()
    for w, cpu in cpus.items():
        losses[w] = [float(cpu.train_step_device(x, y)) for _ in range(3)]
    pg = _trainer_params(gpu)
    gpu.close()
    err = (pg - _trainer_params(cpus[wd])).abs().mean().item()
    control = (pg - _trainer_params(cpus[0.0])).abs().mean().item()
    moved = (pg - start).abs().mean().item()
    print(f"path {path} decoupled {decoupled}: |gpu - cpu| {err:.3g}, |gpu - cpu without decay| {control:.3g}, moved {moved:.3g}")
    assert err < 0.2 * control, (err, control)
    assert abs(losses["gpu"][0] - losses[wd][0]) < 2e-2 and abs(losses["gpu"][-1] - losses[wd][-1]) < 0.15, losses
