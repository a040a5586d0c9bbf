"""Router losses of the product-key gate: a load-balancing loss (Switch / GShard) and a router z-loss (ST-MoE), trained
through DMoEConfig(router_aux_loss_coef=..., router_z_loss_coef=...).

CPU: the configuration and its refusals, the float64 oracle K.router_loss_ref against a direct formula and autograd, the
CPU layer's gradients, the micro-batch scaling, and the balance a small trainer reaches with and without the loss.
GPU: the router-loss kernels against the float64 oracle, one layer on both expert paths and both expert kinds against
the bf16 oracle, the trainer under its CUDA graph, and the launch budget."""
import math

import pytest
import torch

import lah_b200  # noqa
from lah_b200.ops import kernels as K
from lah_b200.parallel import baseline, engine as E
from lah_b200.parallel.trainer import DMoETrainer
from routing_support import collapse, cpu_cfg, load, rel
from routing_support import one_thread  # noqa: F401 (fixture)

GRIDS = [(64,), (8, 8), (4, 4, 4), (2, 2, 2, 2)]
COEF = dict(router_aux_loss_coef=0.01, router_z_loss_coef=0.001)


# ======================================================================================================== CPU
def test_defaults_are_zero_and_launch_nothing():
    cfg = E.DMoEConfig()
    assert cfg.router_aux_loss_coef == 0.0 and cfg.router_z_loss_coef == 0.0 and not cfg.router_losses
    layer = E.FusedDMoE(E.DMoEConfig(hidden=64, grid_size=(4,), k=2, num_layers=1))
    assert layer.router_loss is None
    assert E.DMoEConfig(router_z_loss_coef=1e-3).router_losses


@pytest.mark.parametrize("kw", [dict(router_aux_loss_coef=-0.01), dict(router_z_loss_coef=-1e-3),
                                dict(router_aux_loss_coef=float("nan")), dict(router_z_loss_coef=float("inf")),
                                dict(router_aux_loss_coef=0.01, gate_mode="emulator", grid_size=(64,)),
                                dict(router_z_loss_coef=0.001, gate_mode="emulator", grid_size=(64,))])
def test_config_refusals(kw):
    with pytest.raises(ValueError):
        E.DMoEConfig(**kw)


def test_emulator_gate_accepts_zero_coefficients():
    E.DMoEConfig(gate_mode="emulator", grid_size=(64,), router_aux_loss_coef=0.0, router_z_loss_coef=0.0)


@pytest.mark.parametrize("arm", ["BaselineDMoE", "BaselineTrainer", "FastBaselineDMoE", "FastBaselineTrainer"])
def test_baseline_arms_refuse_router_losses(arm):
    from lah_b200.parallel import baseline_fast
    cfg = E.DMoEConfig(hidden=64, grid_size=(4,), k=2, num_layers=1, tokens_per_rank=8, **COEF)
    make = dict(BaselineDMoE=lambda: baseline.BaselineDMoE(cfg), BaselineTrainer=lambda: baseline.BaselineTrainer(cfg),
                FastBaselineDMoE=lambda: baseline_fast.FastBaselineDMoE(cfg, 0, 16),
                FastBaselineTrainer=lambda: baseline_fast.FastBaselineTrainer(cfg))[arm]
    with pytest.raises(ValueError, match="router"):
        make()


def _direct(logits, grid, counts, alive):
    """L_aux and L_z straight from the definitions, with product_key_scores and torch.softmax"""
    s = K.product_key_scores(logits, grid)
    live = alive.bool()
    N = int(live.sum())
    p = torch.softmax(s[:, live], dim=-1)
    z = torch.logsumexp(s[:, live], dim=-1)
    c = counts.to(s.dtype)
    f = c / c.sum()
    B = s.shape[0]
    return N * (f[live] * p.sum(0) / B).sum(), (z ** 2).mean()


def _case(grid, dead, B=24, seed=0, scale=3.0):
    gen = torch.Generator().manual_seed(seed)
    E_ = math.prod(grid)
    logits = (torch.rand(B, sum(grid), generator=gen, dtype=torch.float64) * 2 - 1) * scale
    alive = torch.ones(E_, dtype=torch.uint8)
    if dead:
        alive[torch.randperm(E_, generator=gen)[: E_ // 4]] = 0
    counts = torch.randint(0, 9, (E_,), generator=gen) * alive.long()
    return logits, alive, counts


@pytest.mark.parametrize("dead", [False, True])
@pytest.mark.parametrize("grid", GRIDS)
def test_oracle_equals_the_direct_formula(grid, dead):
    logits, alive, counts = _case(grid, dead)
    aux, z = K.router_loss_ref(logits, grid, counts, alive=alive)
    da, dz = _direct(logits, grid, counts, alive)
    assert aux.dtype == torch.float64
    torch.testing.assert_close(aux, da, rtol=1e-12, atol=0)
    torch.testing.assert_close(z, dz, rtol=1e-12, atol=0)
    # a [R, E] count table is summed over its rows
    table = torch.stack([counts // 2, counts - counts // 2])
    torch.testing.assert_close(K.router_loss_ref(logits, grid, table, alive=alive)[0], aux, rtol=1e-12, atol=0)


@pytest.mark.parametrize("dead", [False, True])
@pytest.mark.parametrize("grid", GRIDS)
def test_uniform_router_with_uniform_counts_gives_one(grid, dead):
    _, alive, _ = _case(grid, dead)
    logits = torch.zeros(5, sum(grid), dtype=torch.float64)
    counts = alive.long() * 7
    aux, z = K.router_loss_ref(logits, grid, counts, alive=alive)
    assert float(aux) == pytest.approx(1.0, abs=1e-14)
    assert float(z) == pytest.approx(math.log(int(alive.sum())) ** 2, rel=1e-14)


@pytest.mark.parametrize("grid", GRIDS)
def test_no_live_expert_or_no_finite_logit_gives_zeros(grid):
    logits, _, counts = _case(grid, False)
    logits.requires_grad_(True)
    aux, z = K.router_loss_ref(logits, grid, counts, alive=torch.zeros(math.prod(grid), dtype=torch.uint8))
    assert float(aux.detach()) == 0.0 and float(z.detach()) == 0.0
    (aux + z).backward()
    assert logits.grad is not None and torch.equal(logits.grad, torch.zeros_like(logits))
    # one token whose logits are all -inf: it adds nothing and gets no gradient, the others are unchanged
    lg = logits.detach().clone()
    lg[3] = float("-inf")
    lg.requires_grad_(True)
    aux, z = K.router_loss_ref(lg, grid, counts)
    (aux + z).backward()
    assert torch.isfinite(aux) and torch.isfinite(z) and torch.isfinite(lg.grad).all()
    assert torch.equal(lg.grad[3], torch.zeros_like(lg.grad[3]))
    keep = torch.cat([logits.detach()[:3], logits.detach()[4:]])
    a2, z2 = K.router_loss_ref(keep, grid, counts)
    B = logits.shape[0]
    torch.testing.assert_close(aux * B, a2 * (B - 1), rtol=1e-12, atol=0)
    torch.testing.assert_close(z * B, z2 * (B - 1), rtol=1e-12, atol=0)


@pytest.mark.parametrize("dead", [False, True])
@pytest.mark.parametrize("grid", GRIDS)
def test_closed_form_gradient_equals_autograd(grid, dead, one_thread):
    """dL/ds_{b,e} = p_{b,e} (alpha N (f_e - F_b) + 2 beta z_b) / B, summed onto each grid dimension's logits"""
    logits, alive, counts = _case(grid, dead, B=6)
    alpha, beta = 0.7, 0.3
    torch.autograd.gradcheck(lambda l: alpha * K.router_loss_ref(l, grid, counts, alive=alive)[0]
                             + beta * K.router_loss_ref(l, grid, counts, alive=alive)[1],
                             (logits.clone().requires_grad_(True),))
    lg = logits.clone().requires_grad_(True)
    aux, z = K.router_loss_ref(lg, grid, counts, alive=alive)
    (auto,) = torch.autograd.grad(alpha * aux + beta * z, lg)
    s = K.product_key_scores(lg, grid)
    live = alive.bool()
    N, B = int(live.sum()), s.shape[0]
    sm = s.masked_fill(~live, float("-inf"))
    zb = torch.logsumexp(sm, -1, keepdim=True)
    p = torch.exp(sm - zb)
    f = counts.double() / counts.sum()
    Fb = (p * f).sum(-1, keepdim=True)
    ds = p * (alpha * N * (f - Fb) + 2 * beta * zb) / B
    (closed,) = torch.autograd.grad(s, lg, ds.detach())   # the transpose of the sum over grid dimensions
    torch.testing.assert_close(closed, auto, rtol=1e-10, atol=1e-13)


@pytest.mark.parametrize("expert", ["ffn", "swiglu"])
def test_cpu_layer_adds_the_router_gradient(expert):
    torch.manual_seed(0)
    plain = E.FusedDMoE(cpu_cfg(expert=expert)).train()
    torch.manual_seed(0)
    cfg = cpu_cfg(expert=expert, router_aux_loss_coef=0.05, router_z_loss_coef=0.01)
    routed = E.FusedDMoE(cfg).train()
    x = torch.randn(32, 64)
    gy = torch.randn(32, 64)
    for layer in (plain, routed):
        layer(x).backward(gy)
    logits = F_linear(x, routed.proj)
    idx, _ = K.gate_topk_ref(logits.detach(), cfg.grid_size, cfg.k)
    counts = torch.bincount(idx[idx >= 0].flatten(), minlength=cfg.num_experts)
    aux, z = K.router_loss_ref(logits, cfg.grid_size, counts)
    (extra,) = torch.autograd.grad(0.05 * aux + 0.01 * z, routed.proj.weight)
    torch.testing.assert_close(routed.proj.weight.grad, plain.proj.weight.grad + extra, rtol=1e-5, atol=1e-7)
    torch.testing.assert_close(routed.router_loss, torch.stack([aux, z]).detach(), rtol=1e-6, atol=0)
    assert float(routed.router_loss[0]) > 0.5


def F_linear(x, proj):
    return torch.nn.functional.linear(x.float(), proj.weight, proj.bias)


def test_cpu_router_loss_is_a_buffer_that_is_not_saved():
    layer = E.FusedDMoE(cpu_cfg(**COEF))
    assert dict(layer.named_buffers())["router_loss"] is layer.router_loss
    assert "router_loss" not in layer.state_dict()
    assert layer.double().router_loss.dtype == torch.float64   # follows the layer's .to()
    assert "router_loss" not in dict(E.FusedDMoE(cpu_cfg()).named_buffers())


def test_cpu_layer_eval_mode_computes_nothing():
    layer = E.FusedDMoE(cpu_cfg(**COEF)).eval()
    layer(torch.randn(8, 64))
    assert torch.equal(layer.router_loss, torch.zeros(2))


def test_zero_coefficients_change_nothing():
    grads = []
    for cfg in (cpu_cfg(), cpu_cfg(router_aux_loss_coef=0.0, router_z_loss_coef=0.0)):
        torch.manual_seed(0)
        layer = E.FusedDMoE(cfg).train()
        torch.manual_seed(1)
        x = torch.randn(32, 64, requires_grad=True)
        layer(x).backward(torch.randn(32, 64))
        leaves = {(e, n): t.grad.clone() for e, d in layer._ref_leaves.items() for n, t in d.items() if t.grad is not None}
        grads.append((x.grad.clone(), layer.proj.weight.grad.clone(), layer.proj.bias.grad.clone(), leaves))
    a, b = grads
    assert all(torch.equal(u, v) for u, v in zip(a[:3], b[:3]))
    assert a[3].keys() == b[3].keys() and all(torch.equal(a[3][k], b[3][k]) for k in a[3])


def _first_trainer_grad(cfg, x, y):
    """the trainer-side gradient (flat_g) of one step; lr = 0 keeps the experts fixed between micro-batches"""
    t = DMoETrainer(cfg)
    got = []
    t._trainer_optimizer_step = lambda: got.append(t.flat_g.clone())
    t.train_step(x, y)
    return got[0]


def test_microbatch_router_gradient_is_the_mean_of_the_micro_batches(one_thread):
    torch.manual_seed(2)
    x, y = torch.randn(64, 16), torch.randint(0, 10, (64,))
    kw = dict(num_layers=2, lr=0.0)
    assert all(b.router_grad_scale == 0.5 for b in DMoETrainer(cpu_cfg(trainer_microbatches=2, **COEF, **kw)).model.blocks)

    def router_part(m, xs, ys):   # the part of the gradient the router losses add (same routing: same parameters)
        return (_first_trainer_grad(cpu_cfg(trainer_microbatches=m, **COEF, **kw), xs, ys)
                - _first_trainer_grad(cpu_cfg(trainer_microbatches=m, **kw), xs, ys))

    two = router_part(2, x, y)
    halves = [router_part(1, x[:32], y[:32]), router_part(1, x[32:], y[32:])]
    assert float(two.abs().max()) > 1e-5
    torch.testing.assert_close(two, 0.5 * (halves[0] + halves[1]), rtol=1e-4, atol=1e-7)


def test_load_balancing_loss_spreads_a_collapsed_router(one_thread):
    """a gate initialised to favour experts 0 and 1: the task loss alone keeps the collapse, the balancing loss undoes
    it; the task loss falls in both runs"""
    gen = torch.Generator().manual_seed(0)
    protos = torch.randn(10, 16, generator=gen) * 2
    y = torch.randint(0, 10, (128,), generator=gen)
    x = protos[y] + 0.5 * torch.randn(128, 16, generator=gen)
    results = {}
    for alpha in (0.0, 0.1):
        cfg = cpu_cfg(grid_size=(8,), k=2, num_layers=1, tokens_per_rank=128, lr=3e-3, router_aux_loss_coef=alpha)
        t = DMoETrainer(cfg)
        collapse(t.model.blocks[0], "product_key")
        before = load(t, x)
        losses = [t.train_step(x, y) for _ in range(120)]
        results[alpha] = (before, load(t, x), losses)
    (b0, a0, l0), (b1, a1, l1) = results[0.0], results[0.1]
    assert b0 == b1 and b0[0] > 3.0            # same start: two of eight experts take (nearly) every row
    assert a1[0] < a0[0] and a1[0] < 2.0, (a0, a1)
    assert l0[-1] < 0.5 * l0[0] and l1[-1] < 0.5 * l1[0], (l0[::20], l1[::20])


# ======================================================================================================== GPU
def _gate_counts(logits, grid, k, alive, failure_rate):
    """routed pairs per expert from the gate kernel itself (failure injection drops pairs before they are counted)"""
    B = logits.shape[0]
    dev = logits.device
    idx = torch.empty(B * k, dtype=torch.int32, device=dev)
    w, pos = torch.empty(B * k, device=dev), torch.empty(B * k, dtype=torch.int32, device=dev)
    counts = torch.zeros(math.prod(grid), dtype=torch.int32, device=dev)
    K.gate_topk(logits, grid, k, alive=alive, failure_rate=failure_rate, seed=11, token_offset=0, idx=idx, w=w, pos=pos,
                counts=counts)
    return counts


def _run_kernels(logits, grid, counts, alive, alpha, beta):
    B, E_ = logits.shape[0], math.prod(grid)
    dev = logits.device
    f = torch.empty(E_ + 1, device=dev)
    z, Fb, loss = torch.empty(B, device=dev), torch.empty(B, device=dev), torch.empty(2, device=dev)
    K.router_loss_fwd(logits, grid, counts.view(1, -1), alive=alive, f=f, z=z, Fb=Fb, loss=loss)
    dl = torch.zeros_like(logits)
    K.router_loss_bwd(logits, grid, alive=alive, f=f, z=z, Fb=Fb, aux_coef=alpha, z_coef=beta, dlogits=dl)
    torch.cuda.synchronize()
    return loss.clone(), dl, f.clone(), z.clone(), Fb.clone()


@pytest.mark.gpu
@pytest.mark.parametrize("B", [1, 7, 256, 65536])
@pytest.mark.parametrize("grid", [(64,), (8, 8), (32, 32), (64, 64), (4, 4, 4, 4)])
def test_kernels_against_the_float64_oracle(grid, B):
    dev = torch.device("cuda")
    E_ = math.prod(grid)
    gen = torch.Generator().manual_seed(B + E_)
    alive = (torch.rand(E_, generator=gen) > 0.2).to(torch.uint8).to(dev)
    for k, mag in ((1, 5.0), (4, 80.0), (8, 20.0)):
        logits = ((torch.rand(B, sum(grid), generator=gen) * 2 - 1) * mag).to(dev)
        counts = _gate_counts(logits, grid, k, alive, failure_rate=0.1)
        alpha, beta = 0.5, 0.02
        loss, dl, f, z, Fb = _run_kernels(logits, grid, counts, alive, alpha, beta)
        lg = logits.double().requires_grad_(True)
        aux, zl = K.router_loss_ref(lg, grid, counts, alive=alive)
        (ref,) = torch.autograd.grad(alpha * aux + beta * zl, lg)
        ref_loss = torch.stack([aux, zl]).detach()
        assert torch.isfinite(loss).all() and torch.isfinite(dl).all()
        err = ((loss.double() - ref_loss).abs() / ref_loss.abs().clamp_min(1e-30)).max().item()
        assert err < 1e-4, (k, loss.tolist(), ref_loss.tolist())
        gerr = ((dl.double() - ref).abs().max() / ref.abs().max().clamp_min(1e-30)).item()
        assert gerr < 1e-4, (k, gerr)
        again = _run_kernels(logits, grid, counts, alive, alpha, beta)
        assert all(torch.equal(a, b) for a, b in zip((loss, dl, f, z, Fb), again))
        del lg, aux, zl, ref


@pytest.mark.gpu
def test_kernels_without_live_experts_or_finite_logits_give_zeros():
    dev = torch.device("cuda")
    grid = (8, 8)
    logits = torch.randn(37, 16, device=dev)
    logits[5] = float("-inf")
    counts = torch.randint(0, 5, (64,), dtype=torch.int32, device=dev)
    dead = torch.zeros(64, dtype=torch.uint8, device=dev)
    loss, dl, *_ = _run_kernels(logits, grid, counts, dead, 1.0, 1.0)
    assert torch.equal(loss, torch.zeros(2, device=dev)) and torch.equal(dl, torch.zeros_like(dl))
    loss, dl, *_ = _run_kernels(logits, grid, counts, None, 1.0, 1.0)
    assert torch.isfinite(loss).all() and torch.equal(dl[5], torch.zeros_like(dl[5])) and torch.isfinite(dl).all()
    aux, zl = K.router_loss_ref(logits.double(), grid, counts)
    torch.testing.assert_close(loss.double(), torch.stack([aux, zl]), rtol=1e-4, atol=0)


@pytest.mark.gpu
def test_wrappers_refuse_bad_arguments_before_launching():
    from lah_b200.ops import native
    dev = torch.device("cuda")
    lg = torch.randn(4, 16, device=dev)
    f, z, Fb, loss = torch.empty(65, device=dev), torch.empty(4, device=dev), torch.empty(4, device=dev), torch.empty(2, device=dev)
    counts = torch.zeros(1, 64, dtype=torch.int32, device=dev)
    ok = dict(alive=None, f=f, z=z, Fb=Fb, loss=loss)
    before = native.launches()
    bad = [((lg.double(), (8, 8), counts), ok), ((lg, (8, 9), counts), ok), ((lg, (8, 8), counts.long()), ok),
           ((lg, (8, 8), torch.zeros(9, 64, dtype=torch.int32, device=dev)), ok),
           ((lg, (8, 8), counts), dict(ok, f=torch.empty(64, device=dev))),
           ((lg, (8, 8), counts), dict(ok, alive=torch.ones(63, dtype=torch.uint8, device=dev))),
           ((torch.randn(4, 5000, device=dev), (5000,), torch.zeros(1, 5000, dtype=torch.int32, device=dev)), ok),
           ((torch.randn(4, 10, device=dev), (2, 2, 2, 2, 2), torch.zeros(1, 32, dtype=torch.int32, device=dev)), ok)]
    for args, kw in bad:
        with pytest.raises(ValueError):
            K.router_loss_fwd(*args, **kw)
    for dl in (torch.zeros(4, 16, dtype=torch.float64, device=dev), torch.zeros(4, 15, device=dev)):
        with pytest.raises(ValueError):
            K.router_loss_bwd(lg, (8, 8), f=f, z=z, Fb=Fb, aux_coef=1.0, z_coef=1.0, dlogits=dl)
    assert native.launches() == before


@pytest.mark.gpu
@pytest.mark.parametrize("expert", ["ffn", "swiglu"])
@pytest.mark.parametrize("path", ["small", "big"])
def test_layer_against_the_bf16_oracle(path, expert):
    from lah_b200.ops import native
    torch.manual_seed(3)
    cfg = E.DMoEConfig(hidden=512, grid_size=(4, 4), k=4, num_layers=1, tokens_per_rank=512, expert=expert,
                       expert_path=path, **COEF)
    ctx = E.EngineContext(cfg)
    try:
        layer = E.FusedDMoE(cfg, ctx).cuda().train()
        assert ctx.small == (path == "small")
        oracle = E.FusedDMoE(cfg, device=torch.device("cuda")).cuda().train()
        oracle.ref_emulate_bf16 = True
        oracle.proj.load_state_dict(layer.proj.state_dict())
        with torch.no_grad():
            oracle.shard.p.copy_(layer.shard.p[:oracle.shard.p.numel()])
        B = 512
        x = torch.randn(B, 512, device="cuda").to(torch.bfloat16)
        gy = torch.randn(B, 512, device="cuda").to(torch.bfloat16)
        logits = layer.gate_logits(x, layer.proj)
        lg = logits.detach().clone().requires_grad_(True)
        n0 = native.launches()
        y = E._FusedDMoEFunction.apply(x, lg, layer)
        y.backward(gy)
        torch.cuda.synchronize()
        ctx.check_status()
        launches = native.launches() - n0
        proj_grad = torch.autograd.grad(logits, layer.proj.weight, lg.grad)[0]
        lr_ = lg.detach().clone().requires_grad_(True)
        yr = oracle._forward_ref(x.float(), lr_, emulate_bf16=True)
        yr.backward(gy.float())
        oracle_proj = torch.autograd.grad(F_linear(x, oracle.proj), oracle.proj.weight, lr_.grad)[0]
        assert rel(layer.router_loss, oracle.router_loss) < 1e-4, (layer.router_loss, oracle.router_loss)
        assert rel(y, yr) < 2e-2 and rel(lg.grad, lr_.grad) < 5e-2 and rel(proj_grad, oracle_proj) < 5e-2
        # the router part alone, against autograd of the oracle's losses on the same routing
        counts = ctx.cnt_all[:1].view(-1)
        aux, zl = K.router_loss_ref(lg.detach().double().requires_grad_(True), cfg.grid_size, counts)
        torch.testing.assert_close(layer.router_loss.double(), torch.stack([aux, zl]).detach(), rtol=1e-4, atol=0)
        # the router gradient alone: with gy = 0, gate_bwd writes exactly 0, so dlogits is the injected gradient.  Against
        # autograd of alpha * L_aux + beta * L_z (float64 oracle, this step's count table) at 1e-4 of max |ref|
        alpha, beta = COEF["router_aux_loss_coef"], COEF["router_z_loss_coef"]

        def router_ref(lgt, scale):
            l64 = lgt.detach().double().requires_grad_(True)
            a, zz = K.router_loss_ref(l64, cfg.grid_size, ctx.cnt_all[:1].view(-1).clone(), alive=ctx.alive)
            (g,) = torch.autograd.grad(scale * (alpha * a + beta * zz), l64)
            assert float(g.abs().max()) > 0
            return g

        lz = logits.detach().clone().requires_grad_(True)
        E._FusedDMoEFunction.apply(x, lz, layer).backward(torch.zeros_like(gy))
        torch.cuda.synchronize()
        ref = router_ref(lz, 1.0)
        assert float((lz.grad.double() - ref).abs().max()) <= 1e-4 * float(ref.abs().max())
        # ... and through the public forward into proj.weight.grad, with the micro-batch scale of a trainer (1 / 2)
        layer.router_grad_scale = 0.5
        layer.proj.weight.grad = None
        layer(x).backward(torch.zeros_like(gy))
        torch.cuda.synchronize()
        ctx.check_status()
        ref_proj = router_ref(logits, 0.5).t() @ x.double()
        got_proj = layer.proj.weight.grad.double()
        assert float((got_proj - ref_proj).abs().max()) <= 1e-4 * float(ref_proj.abs().max())
        # the same forward and backward without router losses: 2 + 1 launches fewer
        plain_cfg = E.DMoEConfig(**{**cfg.__dict__, "router_aux_loss_coef": 0.0, "router_z_loss_coef": 0.0})
        plain = E.FusedDMoE(plain_cfg, ctx).cuda().train()
        n0 = native.launches()
        lp = logits.detach().clone().requires_grad_(True)
        E._FusedDMoEFunction.apply(x, lp, plain).backward(gy)
        torch.cuda.synchronize()
        assert launches == native.launches() - n0 + 3
    finally:
        ctx.close()


@pytest.mark.gpu
def test_layer_with_router_losses_refuses_a_context_without_them():
    plain = E.DMoEConfig(hidden=512, grid_size=(4, 4), k=4, num_layers=1, tokens_per_rank=64)
    ctx = E.EngineContext(plain)
    try:
        with pytest.raises(ValueError, match="EngineContext"):
            E.FusedDMoE(E.DMoEConfig(**{**plain.__dict__, **COEF}), ctx)
        assert E.FusedDMoE(plain, ctx).router_loss is None
    finally:
        ctx.close()


def _trainer_cfg(path, **kw):
    base = dict(hidden=512, grid_size=(16,), k=4, num_layers=2, tokens_per_rank=256, failure_rate=0.1, lr=1e-4,
                expert_path=path, **COEF)
    base.update(kw)
    return E.DMoEConfig(**base)


@pytest.mark.gpu
@pytest.mark.parametrize("expert", ["ffn", "swiglu"])
@pytest.mark.parametrize("path", ["small", "big"])
def test_trainer_graph_equals_eager_and_runs_are_reproducible(path, expert):
    cfg = _trainer_cfg(path, expert=expert)
    torch.manual_seed(0)
    xs = [torch.randn(256, cfg.in_features, device="cuda") for _ in range(5)]
    ys = [torch.randint(0, 10, (256,), device="cuda") for _ in range(5)]
    runs = {}
    for run, graph in (("eager", False), ("graph", True), ("graph2", True)):
        t = DMoETrainer(cfg, use_graph=graph)
        losses, rl = [], []
        for x, y in zip(xs, ys):
            losses.append(t.train_step_device(x, y).clone())
            rl.append(torch.stack([b.router_loss for b in t.model.blocks]).clone())
        assert (t._graph is not None) == graph
        t.ctx.check_status()
        rec = t.log_step()
        assert all("router_aux_loss" in layer and "router_z_loss" in layer for layer in rec["layers"])
        runs[run] = (torch.stack(losses).cpu(), torch.stack(rl).cpu(),
                     torch.cat([b.shard.p for b in t.model.blocks] + [t.flat_p]).cpu())
        t.close()
    assert float(runs["eager"][1][:, :, 0].min()) > 0.5    # L_aux near 1 for a router that is not collapsed
    for a, b in zip(runs["eager"], runs["graph"]):
        assert torch.equal(a, b)
    for a, b in zip(runs["graph"], runs["graph2"]):
        assert torch.equal(a, b)


@pytest.mark.gpu
def test_zero_coefficients_keep_the_launch_count():
    counts = {}
    for name, kw in (("plain", {}), ("zero", dict(router_aux_loss_coef=0.0, router_z_loss_coef=0.0)), ("router", COEF)):
        cfg = _trainer_cfg("small", **{**dict(router_aux_loss_coef=0.0, router_z_loss_coef=0.0), **kw})
        t = DMoETrainer(cfg, use_graph=True)
        x, y = torch.randn(256, cfg.in_features, device="cuda"), torch.randint(0, 10, (256,), device="cuda")
        for _ in range(3):
            t.train_step_device(x, y)
        counts[name] = t._graph_launches
        t.close()
    assert counts["plain"] == counts["zero"]
    assert counts["router"] == counts["plain"] + 3 * 2
