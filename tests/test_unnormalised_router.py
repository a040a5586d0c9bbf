"""Unnormalised top-k weights (DMoEConfig(norm_topk_prob=False), DESIGN.md §6e): the softmax router weights each selected
expert by scale * p_j, with p the softmax over every live expert (Switch, GShard, DeepSeek-V2, Qwen-MoE), and the sigmoid
router by scale * sigma_j.

CPU: the configuration and its refusals, the oracle K.gate_topk_ref(norm=False) against a brute-force float64
implementation, the identities, the gate gradient against float64 autograd, a Switch-shaped CPU trainer whose top-1 gate
trains only without renormalisation, and checkpoints across the setting.
GPU: the gate kernel against the normalised kernel and the oracle, gate_bwd against the float64 formula, the wrappers'
refusals, the layer against the CPU oracle, and the trainer under its CUDA graph."""
import math

import pytest
import torch

import lah_b200  # noqa
from lah_b200.ops import kernels as K
from lah_b200.parallel import baseline, engine as E
from lah_b200.parallel.trainer import DMoETrainer
from routing_support import cpu_cfg, layer_against_the_oracle, run_gate
from routing_support import one_thread, rt, step_counters, world1  # noqa: F401 (fixtures)

UN = dict(norm_topk_prob=False)


# ======================================================================================================== CPU: config
def test_defaults_and_state_dict_keys():
    assert E.DMoEConfig().norm_topk_prob is True
    plain, un = E.FusedDMoE(cpu_cfg()), E.FusedDMoE(cpu_cfg(routed_scaling_factor=2.5, **UN))
    assert plain.norm_topk_prob and not plain.dense_gate
    assert not un.norm_topk_prob and un.dense_gate and un.routed_scale == 2.5
    assert not E.FusedDMoE(cpu_cfg(router_score="sigmoid", **UN)).dense_gate
    assert list(plain.state_dict()) == list(un.state_dict())


@pytest.mark.parametrize("kw,match", [
    (dict(norm_topk_prob=0), "norm_topk_prob"), (dict(norm_topk_prob="False"), "norm_topk_prob"),
    (dict(norm_topk_prob=None), "norm_topk_prob"),
    (dict(routed_scaling_factor=2.5), "routed_scaling_factor"),
    (dict(routed_scaling_factor=0.0, **UN), "routed_scaling_factor"),
    (dict(routed_scaling_factor=float("nan"), **UN), "routed_scaling_factor"),
])
def test_config_refusals(kw, match):
    with pytest.raises(ValueError, match=match):
        E.DMoEConfig(**kw)


@pytest.mark.parametrize("score", ["softmax", "sigmoid"])
@pytest.mark.parametrize("expert", ["ffn", "swiglu"])
@pytest.mark.parametrize("gate", ["product_key", "emulator"])
def test_every_setting_accepts_unnormalised_weights(gate, expert, score):
    extra = dict(router_aux_loss_coef=0.01) if gate == "product_key" else {}
    if gate == "product_key" and score == "softmax":
        extra["router_z_loss_coef"] = 1e-3
    if expert == "swiglu":
        extra["shared_inner_dim"] = 128
    cfg = cpu_cfg(grid_size=(16,), gate_mode=gate, expert=expert, expert_bias_update_rate=1e-3, failure_rate=0.1,
                  trainer_microbatches=2, routed_scaling_factor=2.5, router_score=score, n_group=4, topk_group=2,
                  **UN, **extra)
    for path in ("small", "big"):
        E.DMoEConfig(**{**cfg.__dict__, "expert_path": path})
    E.DMoEConfig(**{**cfg.__dict__, "update_every_steps": 2})
    assert not E.FusedDMoE(cfg).norm_topk_prob


@pytest.mark.parametrize("arm", ["BaselineDMoE", "BaselineTrainer", "FastBaselineDMoE", "FastBaselineTrainer"])
def test_baseline_arms_refuse_unnormalised_weights(arm):
    from lah_b200.parallel import baseline_fast
    cfg = E.DMoEConfig(hidden=64, grid_size=(4,), k=2, num_layers=1, tokens_per_rank=8, **UN)
    make = dict(BaselineDMoE=lambda: baseline.BaselineDMoE(cfg), BaselineTrainer=lambda: baseline.BaselineTrainer(cfg),
                FastBaselineDMoE=lambda: baseline_fast.FastBaselineDMoE(cfg, 0, 16),
                FastBaselineTrainer=lambda: baseline_fast.FastBaselineTrainer(cfg))[arm]
    with pytest.raises(ValueError, match="norm_topk_prob"):
        make()


# ======================================================================================================== CPU: oracles
def _brute_weights(logits, grid, idx, alive, score, c):
    """the written rules in float64, token by token: softmax c * exp(s_j - z_b) with z_b the log-sum-exp over the live
    experts (0 without one); sigmoid c * sigma(s_j); 0 for a missing pair"""
    scores = K.product_key_scores(logits.double(), grid)
    B, E_ = scores.shape
    w = torch.zeros(idx.shape, dtype=torch.float64)
    z = torch.zeros(B, dtype=torch.float64)
    for b in range(B):
        live = [e for e in range(E_) if (alive is None or alive[e]) and math.isfinite(scores[b, e])]
        if live:
            z[b] = max(scores[b, e] for e in live)
            z[b] = z[b] + math.log(sum(math.exp(scores[b, e] - z[b]) for e in live))
        for j, e in enumerate(idx[b].tolist()):
            if e >= 0:
                s = float(scores[b, e])
                w[b, j] = c * (math.exp(s - z[b]) if score == "softmax" else 1.0 / (1.0 + math.exp(-s)))
    return w, z


def _case(grid, B, gen):
    E_ = math.prod(grid)
    logits = torch.randint(-12, 13, (B, sum(grid)), generator=gen).float() / 4   # exact sums in any order
    alive = (torch.rand(E_, generator=gen) > 0.3).to(torch.uint8)
    alive[0] = 1
    fail = torch.rand(B, E_, generator=gen) < 0.2
    bias = torch.randint(-8, 9, (E_,), generator=gen).float() / 16
    return logits, alive, fail, bias


@pytest.mark.parametrize("score", ["softmax", "sigmoid"])
@pytest.mark.parametrize("grid", [(16,), (4, 6), (2, 3, 4)])
def test_oracle_against_brute_force(grid, score):
    gen = torch.Generator().manual_seed(len(grid) * 7 + len(score))
    B, E_ = 24, math.prod(grid)
    logits, alive, fail, bias = _case(grid, B, gen)
    logits[1] = float("-inf")   # no finite score: z = 0, no pairs
    for k in range(1, 9):
        for b in (None, bias):
            c = 2.5 if k % 2 else 1.0
            for n_group in [g for g in range(1, E_ + 1) if E_ % g == 0 and k <= E_]:
                for m in sorted({1, n_group // 2 or 1, n_group}):
                    if k > m * (E_ // n_group):
                        continue
                    kw = dict(alive=alive, fail_mask=fail, bias=b, score=score, n_group=n_group, topk_group=m)
                    idx, w = K.gate_topk_ref(logits, grid, k, scale=c, norm=False, **kw)
                    nidx, _ = K.gate_topk_ref(logits, grid, k, scale=c if score == "sigmoid" else 1.0, **kw)
                    assert torch.equal(idx, nidx)   # the selection does not depend on the setting
                    rw, rz = _brute_weights(logits, grid, idx, alive, score, c)
                    assert torch.allclose(w.double(), rw, rtol=1e-5, atol=1e-12), (k, n_group, m)
                    if score == "softmax":
                        z = K.softmax_lse_ref(K.product_key_scores(logits, grid), alive)
                        assert torch.allclose(z.double(), rz, rtol=1e-6, atol=1e-6)
                    assert bool((w[1] == 0).all()) and bool((idx[1] == -1).all())


@pytest.mark.parametrize("grid", [(8,), (2, 4), (2, 2, 2)])
def test_all_live_experts_selected_gives_the_normalised_weights(grid):
    gen = torch.Generator().manual_seed(1)
    logits = torch.randn(64, sum(grid), generator=gen) * 2
    E_ = math.prod(grid)
    idx, w = K.gate_topk_ref(logits, grid, E_, norm=False, scale=2.5)
    nidx, nw = K.gate_topk_ref(logits, grid, E_)
    assert torch.equal(idx, nidx)
    torch.testing.assert_close(w, 2.5 * nw, rtol=1e-6, atol=1e-7)
    torch.testing.assert_close(w.sum(1), torch.full((64,), 2.5), rtol=1e-6, atol=0)
    # fewer than all: the top k carry less than the scale
    idx, w = K.gate_topk_ref(logits, grid, 1, norm=False)
    assert bool((w.sum(1) < 1).all())


def _dense_formula(scores, idx, w, dw, alive):
    """ds_e = w_e dw_e [e selected] - p_e sum_j w_j dw_j for every live expert (float64)"""
    z = K.softmax_lse_ref(scores, alive)
    live = torch.ones(scores.shape[1], dtype=torch.bool) if alive is None else alive.bool()
    p = torch.exp(scores - z.unsqueeze(-1)) * live
    ds = -p * (w * dw).sum(1, keepdim=True)
    return ds.scatter_add(1, idx.clamp(min=0), torch.where(idx >= 0, w * dw, torch.zeros_like(w)))


def _to_logits(ds_e, grid):
    """dlogits[d][i] = sum of ds_e over the experts whose d-th coordinate is i"""
    t = ds_e.view(ds_e.shape[0], *grid)
    return torch.cat([t.sum(dim=[a + 1 for a in range(len(grid)) if a != d]) if len(grid) > 1 else t
                      for d in range(len(grid))], dim=1)


@pytest.mark.parametrize("grid", [(16,), (4, 4), (2, 3, 4)])
def test_gate_backward_formula_equals_float64_autograd(grid):
    gen = torch.Generator().manual_seed(len(grid))
    B, E_, k, c = 32, math.prod(grid), 3, 2.5
    logits = (torch.randn(B, sum(grid), generator=gen, dtype=torch.float64) * 2).requires_grad_(True)
    alive = (torch.rand(E_, generator=gen) > 0.25).to(torch.uint8)
    idx, _ = K.gate_topk_ref(logits.detach().float(), grid, k, alive=alive, norm=False, scale=c)
    dw = torch.randn(B, k, generator=gen, dtype=torch.float64)
    dw[torch.rand(B, k, generator=gen) < 0.2] = 0.0   # dropped pairs
    scores = K.product_key_scores(logits, grid)
    w = K.softmax_weights_ref(scores, idx, alive, c)
    (ref,) = torch.autograd.grad((w * dw).sum(), logits)
    got = _to_logits(_dense_formula(scores.detach(), idx, w.detach(), dw, alive), grid)
    torch.testing.assert_close(got, ref, rtol=1e-10, atol=1e-12)


def test_cpu_layer_gate_gradient_against_the_formula():
    torch.manual_seed(0)
    grid = (4, 4)
    layer = E.FusedDMoE(cpu_cfg(grid_size=grid, k=2, routed_scaling_factor=2.0, **UN)).train()
    layer.alive_ref = (torch.arange(16) % 5 != 3).to(torch.uint8)
    x = torch.randn(32, 64)
    logits = layer.gate_logits(x, layer.proj).detach().requires_grad_(True)
    out = layer._forward_ref(x, logits)
    gy = torch.randn_like(out)
    (out * gy).sum().backward()
    idx, _ = K.gate_topk_ref(logits.detach(), grid, 2, alive=layer.alive_ref, norm=False, scale=2.0)
    scores = K.product_key_scores(logits.detach().double(), grid)
    w = K.softmax_weights_ref(scores, idx, layer.alive_ref, 2.0)
    with torch.no_grad():
        dw = torch.zeros(32, 2, dtype=torch.float64)
        for b in range(32):
            for j, e in enumerate(idx[b].tolist()):
                y = layer._expert_ref(layer._expert_params(e), x[b:b + 1], lambda t: t)
                dw[b, j] = float((y * gy[b:b + 1]).sum())
    ref = _to_logits(_dense_formula(scores, idx, w, dw, layer.alive_ref), grid)
    err = float((logits.grad.double() - ref).abs().max() / ref.abs().max())
    assert err < 1e-4, err


# ======================================================================================================== CPU: trainer
def _switch_run(norm, steps=5):
    torch.manual_seed(0)
    cfg = cpu_cfg(grid_size=(8,), k=1, gate_mode="product_key", tokens_per_rank=64, weight_decay=0.0,
                  norm_topk_prob=norm)
    t = DMoETrainer(cfg)
    gen = torch.Generator().manual_seed(1)
    gate0 = [p.detach().clone() for p in t.model.blocks[0].proj.parameters()]
    for _ in range(steps):
        t.train_step(torch.randn(64, 16, generator=gen), torch.randint(0, 10, (64,), generator=gen))
    return gate0, [p.detach().clone() for p in t.model.blocks[0].proj.parameters()]


def test_top1_gate_trains_only_without_renormalisation(one_thread):
    """Switch routing at k = 1: every renormalised weight is 1, so the gate gets no gradient from the task and its
    parameters stay bit for bit; the unnormalised weight p_j carries the task's gradient into the gate"""
    before, after = _switch_run(True)
    assert all(torch.equal(a, b) for a, b in zip(before, after))
    before, after = _switch_run(False)
    assert all(not torch.equal(a, b) for a, b in zip(before, after))


def test_checkpoints_load_across_the_setting(one_thread):
    gen = torch.Generator().manual_seed(4)
    xs = [torch.randn(64, 16, generator=gen) for _ in range(4)]
    ys = [torch.randint(0, 10, (64,), generator=gen) for _ in range(4)]
    a = DMoETrainer(cpu_cfg(num_layers=2, **UN))
    for x, y in zip(xs[:2], ys[:2]):
        a.train_step(x, y)
    state = a.state_dict()
    plain = DMoETrainer(cpu_cfg(num_layers=2))
    assert set(state["trainer"]) == set(plain.state_dict()["trainer"])
    plain.load_state_dict(state)
    for ba, bb in zip(a.model.blocks, plain.model.blocks):
        assert torch.equal(ba.proj.weight, bb.proj.weight) and torch.equal(ba.shard.p, bb.shard.p)
    back = DMoETrainer(cpu_cfg(num_layers=2, **UN))
    back.load_state_dict(plain.state_dict())
    la = [a.train_step(x, y) for x, y in zip(xs[2:], ys[2:])]
    lb = [back.train_step(x, y) for x, y in zip(xs[2:], ys[2:])]
    assert la == lb


# ======================================================================================================== GPU
def _grouping(E_):
    g = next(d for d in (8, 5, 4, 3, 2) if E_ % d == 0)
    return g, max(1, g // 2)


@pytest.mark.gpu
@pytest.mark.parametrize("B", [0, 1, 257, 4096])
@pytest.mark.parametrize("grid", [(64,), (256,), (8, 8), (64, 64), (4096,), (3, 5, 7)])
def test_gate_against_the_normalised_kernel_and_the_oracle(step_counters, grid, B):
    E_ = math.prod(grid)
    gen = torch.Generator(device="cuda").manual_seed(B * 3 + E_)
    if len(grid) <= 2:
        logits = torch.randn(B, sum(grid), generator=gen, device="cuda") * 2
    else:   # dyadic logits: the 3-d sums are exact in any order
        logits = torch.randint(-12, 13, (B, sum(grid)), generator=gen, device="cuda").float() / 4
    bias = torch.randint(-8, 9, (E_,), generator=gen, device="cuda").float() / 16
    alive = (torch.rand(E_, generator=gen, device="cuda") > 0.2).to(torch.uint8)
    G, M = _grouping(E_)
    for k in (1, 2, 4, 8):
        c = 2.5 if k % 2 else 1.0
        for score in ("softmax", "sigmoid"):
            for b, (ng, tg) in ((None, (1, 1)), (bias, (1, 1)), (None, (G, M)), (bias, (G, M))):
                kw = dict(alive=alive, rate=0.1, bias=b, score=score, n_group=ng, topk_group=tg)
                idx, w, pos, counts, sig, lse = run_gate(logits, grid, k, scale=c, norm=False, **kw)
                nidx, _, npos, ncounts, nsig, _ = run_gate(logits, grid, k, scale=c if score == "sigmoid" else 1.0,
                                                           **kw)
                assert torch.equal(idx, nidx) and torch.equal(pos, npos) and torch.equal(counts, ncounts), (k, score)
                if sig is not None:
                    assert torch.equal(sig, nsig)
                if B == 0:
                    continue
                scores = K.product_key_scores(logits.double(), grid)
                sel = torch.gather(scores, 1, idx.long().clamp(min=0))
                if score == "softmax":
                    rz = K.softmax_lse_ref(scores, alive)
                    assert float(((lse.double() - rz).abs() / rz.abs().clamp_min(1.0)).max()) < 1e-5, k
                    rw = c * torch.exp(sel - rz.unsqueeze(-1))
                else:
                    rw = c * torch.sigmoid(sel)
                rw = torch.where(idx >= 0, rw, torch.zeros_like(rw))
                err = float(((w.double() - rw).abs() / rw.abs().clamp_min(1e-30)).max())
                assert err < 1e-5, (k, score, ng, err)


@pytest.mark.gpu
def test_wrappers_refuse_bad_arguments_before_launching(step_counters):
    from lah_b200.ops import native
    lg = torch.zeros(4, 16, device="cuda")
    i = torch.zeros(16, dtype=torch.int32, device="cuda")
    ok = dict(idx=i, w=i.float(), pos=i, counts=torch.zeros(16, dtype=torch.int32, device="cuda"))
    lse, sig = torch.zeros(4, device="cuda"), torch.zeros(16, device="cuda")
    before = native.launches()
    for kw in (dict(norm=False), dict(norm=False, lse=torch.zeros(3, device="cuda")),
               dict(norm=False, lse=torch.zeros(4)), dict(norm=False, lse=lse.double()),
               dict(norm=False, lse=lse, scale=0.0), dict(norm=False, lse=lse, scale=float("inf")),
               dict(norm=0, lse=lse), dict(lse=lse), dict(scale=2.0),
               dict(norm=False, score="sigmoid", sig=sig, lse=lse)):
        with pytest.raises(ValueError):
            K.gate_topk(lg, (16,), 4, **ok, **kw)
    g = torch.zeros(4, 256, dtype=torch.bfloat16, device="cuda")
    dl = torch.zeros_like(lg)
    args = (0, g, i, i, i.float(), dl, 4, 16, (16,))
    for kw in (dict(norm=False, logits=lg), dict(norm=False, lse=lse), dict(norm=False, lse=lse, logits=lg[:3]),
               dict(norm=False, lse=lse, logits=lg, alive=torch.ones(15, dtype=torch.uint8, device="cuda")),
               dict(lse=lse), dict(logits=lg), dict(alive=torch.ones(16, dtype=torch.uint8, device="cuda")),
               dict(norm=False, score="sigmoid", sig=sig, scale=1.0, lse=lse)):
        with pytest.raises(ValueError):
            K.gate_bwd(*args, **kw)
    assert native.launches() == before


@pytest.mark.gpu
@pytest.mark.parametrize("score", ["softmax", "sigmoid"])
@pytest.mark.parametrize("k", [1, 4, 8])
@pytest.mark.parametrize("grid,H", [((64,), 256), ((4, 4), 512), ((2, 32), 1024), ((3, 5, 7), 512), ((256,), 1024),
                                    ((64, 64), 512)])
def test_gate_bwd_against_the_float64_formula(rt, grid, H, k, score):
    gen = torch.Generator().manual_seed(k * H + len(grid))
    B, E_, c = 257, math.prod(grid), 2.5
    logits = torch.randn(B, sum(grid), generator=gen) * 2
    alive = (torch.rand(E_, generator=gen) > 0.2).to(torch.uint8)
    alive[0] = 1
    idx, w = K.gate_topk_ref(logits, grid, k, alive=alive, score=score, scale=c, norm=False)
    idx[torch.rand(B, k, generator=gen) < 0.15] = -1
    valid = idx >= 0
    scores = K.product_key_scores(logits.double(), grid)
    sel = torch.gather(scores, 1, idx.clamp(min=0))
    sg = torch.sigmoid(sel) * valid
    w = (K.softmax_weights_ref(scores, idx, alive, c) if score == "softmax" else c * sg).float()
    R = B * k + 50
    pair_row = torch.randperm(R, generator=gen)[: B * k].view(B, k)
    pair_row[torch.rand(B, k, generator=gen) < 0.05] = -1   # pairs that scatter_rows dropped
    pair_row = torch.where(valid, pair_row, torch.full_like(pair_row, -1))
    yo = rt.region[: R * H * 2].view(torch.bfloat16).view(R, H)
    yo.copy_(torch.randn(R, H, generator=gen).to(torch.bfloat16))
    g = torch.randn(B, H, generator=gen).to(torch.bfloat16)
    g[5] = 0                                                  # sum w dw = 0: no gradient at all
    y = yo.cpu().double()[pair_row.clamp(min=0)] * (pair_row >= 0).double().unsqueeze(-1)
    dw = (g.double().unsqueeze(1) * y).sum(-1) * valid
    if score == "softmax":
        ds = _dense_formula(scores, idx, w.double(), dw, alive)
        terms = (w.double() * dw).abs().max()
    else:
        ds = torch.zeros(B, E_, dtype=torch.float64).scatter_add(
            1, idx.clamp(min=0), torch.where(valid, c * sg * (1 - sg) * dw, torch.zeros_like(dw)))
        terms = (c * sg * (1 - sg) * dw).abs().max()
    ref = _to_logits(ds, grid)
    dl = torch.full((B, sum(grid)), 5.0, device="cuda")
    kw = dict(lse=K.softmax_lse_ref(scores, alive).float().cuda(), alive=alive.cuda(), logits=logits.cuda()) \
        if score == "softmax" else dict(score="sigmoid", sig=sg.float().flatten().cuda())
    K.gate_bwd(rt.region_off, g.cuda(), idx.flatten().to(torch.int32).cuda(),
               pair_row.flatten().to(torch.int32).cuda(), w.flatten().cuda(), dl, k, E_, grid, scale=c, norm=False,
               **kw)
    torch.cuda.synchronize()
    dl = dl.cpu().double()
    assert bool((dl[5] == 0).all())
    err = float((dl - ref).abs().max() / terms.clamp_min(1e-30))
    assert err < 1e-4, err
    dl2 = torch.full((B, sum(grid)), 5.0, device="cuda")   # deterministic: the same bits again
    K.gate_bwd(rt.region_off, g.cuda(), idx.flatten().to(torch.int32).cuda(),
               pair_row.flatten().to(torch.int32).cuda(), w.flatten().cuda(), dl2, k, E_, grid, scale=c, norm=False,
               **kw)
    torch.cuda.synchronize()
    assert torch.equal(dl2.cpu().double(), dl)


def _check(r):
    """the unnormalised weights of the tokens routed alike, the dense gate's log-partition, and the router losses"""
    cfg, B = r.layer.cfg, r.idx.shape[0]
    assert float(((r.w - r.rw).abs() / r.rw.abs().clamp_min(1e-30))[r.same].max()) < 1e-5
    if r.layer.dense_gate:
        rz = K.softmax_lse_ref(K.product_key_scores(r.logits.double(), cfg.grid_size), r.ctx.alive)
        assert float((r.layer.ws.lse[:B].double() - rz).abs().max()) < 1e-5 * float(rz.abs().max())
    if r.layer.router_loss is not None:
        torch.testing.assert_close(r.layer.router_loss, r.oracle.router_loss, rtol=1e-3, atol=1e-6)


@pytest.mark.gpu
@pytest.mark.parametrize("score", ["softmax", "sigmoid"])
@pytest.mark.parametrize("gate", ["emulator", "product_key"])
@pytest.mark.parametrize("expert", ["ffn", "swiglu"])
@pytest.mark.parametrize("path", ["small", "big"])
def test_layer_against_the_cpu_oracle(path, expert, gate, score):
    torch.manual_seed(3)
    grid = (16,) if gate == "emulator" else (4, 4)
    cfg = E.DMoEConfig(hidden=512, grid_size=grid, k=4, num_layers=1, tokens_per_rank=512, expert=expert,
                       expert_path=path, gate_mode=gate, routed_scaling_factor=2.5, router_score=score, **UN)
    layer_against_the_oracle(cfg, max_mismatch=2, check=_check)


@pytest.mark.gpu
@pytest.mark.parametrize("path", ["small", "big"])
def test_switch_shaped_layer_against_the_cpu_oracle(path):
    """top-1 of 64 experts on the product-key gate with the load-balancing loss (Switch Transformer)"""
    torch.manual_seed(5)
    cfg = E.DMoEConfig(hidden=512, grid_size=(8, 8), k=1, num_layers=1, tokens_per_rank=512, expert_path=path,
                       router_aux_loss_coef=1e-2, **UN)
    layer_against_the_oracle(cfg, max_mismatch=2, check=_check)


@pytest.mark.gpu
@pytest.mark.parametrize("path", ["small", "big"])
def test_deepseek_v2_shaped_layer_against_the_cpu_oracle(path):
    """SwiGLU experts, a shared expert, 8 groups of which a token may use 3, top-6, c = 16, the load-balancing loss"""
    torch.manual_seed(4)
    cfg = E.DMoEConfig(hidden=512, grid_size=(8, 8), k=6, num_layers=1, tokens_per_rank=512, expert="swiglu",
                       inner_dim=256, shared_inner_dim=512, expert_path=path, n_group=8, topk_group=3,
                       routed_scaling_factor=16.0, router_aux_loss_coef=1e-2, **UN)
    layer_against_the_oracle(cfg, max_mismatch=2, check=_check)


@pytest.mark.gpu
def test_layer_refuses_a_context_of_the_other_setting():
    cfg = E.DMoEConfig(hidden=512, grid_size=(16,), k=4, num_layers=1, tokens_per_rank=256)
    ctx = E.EngineContext(cfg)
    try:
        assert E.FusedDMoE(cfg, ctx).ws.lse is None
        with pytest.raises(ValueError, match="norm_topk_prob"):
            E.FusedDMoE(E.DMoEConfig(**{**cfg.__dict__, **UN}), ctx)
    finally:
        ctx.close()


def _trainer_cfg(path, gate, **kw):
    base = dict(hidden=512, grid_size=(16,), k=4, num_layers=2, tokens_per_rank=256, failure_rate=0.1, lr=1e-4,
                expert_path=path, gate_mode=gate, expert_bias_update_rate=1e-3)
    base.update(kw)
    return E.DMoEConfig(**base)


@pytest.mark.gpu
@pytest.mark.parametrize("score", ["softmax", "sigmoid"])
@pytest.mark.parametrize("gate", ["emulator", "product_key"])
@pytest.mark.parametrize("path", ["small", "big"])
def test_trainer_graph_equals_eager_and_runs_are_reproducible(path, gate, score):
    kw = dict(router_aux_loss_coef=1e-2) if gate == "product_key" else {}
    cfg = _trainer_cfg(path, gate, router_score=score, routed_scaling_factor=2.5, **UN, **kw)
    torch.manual_seed(0)
    xs = [torch.randn(256, cfg.in_features, device="cuda") for _ in range(5)]
    ys = [torch.randint(0, 10, (256,), device="cuda") for _ in range(5)]
    runs = {}
    for run, graph in (("eager", False), ("graph", True), ("graph2", True)):
        t = DMoETrainer(cfg, use_graph=graph)
        losses = [t.train_step_device(x, y).clone() for x, y in zip(xs, ys)]
        assert (t._graph is not None) == graph
        t.ctx.check_status()
        rec = t.log_step()
        assert all(0 < layer["routed_weight_mean"] for layer in rec["layers"])
        runs[run] = (torch.stack(losses).cpu(), torch.cat([b.shard.p for b in t.model.blocks] + [t.flat_p]).cpu())
        t.close()
    for a, b in zip(runs["eager"], runs["graph"]):
        assert torch.equal(a, b)
    for a, b in zip(runs["graph"], runs["graph2"]):
        assert torch.equal(a, b)


@pytest.mark.gpu
@pytest.mark.parametrize("m", [1, 2])
def test_trainer_launches_as_many_kernels_as_the_normalised_one(m):
    counts = {}
    base = dict(hidden=512, grid_size=(16,), k=4, num_layers=2, tokens_per_rank=256, expert_path="small",
                gate_mode="product_key", trainer_microbatches=m, router_aux_loss_coef=1e-2)
    for name, kw in (("norm", {}), ("unnorm", UN)):
        t = DMoETrainer(E.DMoEConfig(**base, **kw), use_graph=True)
        x, y = torch.randn(256, t.cfg.in_features, device="cuda"), torch.randint(0, 10, (256,), device="cuda")
        for _ in range(3):
            t.train_step_device(x, y)
        counts[name] = t._graph_launches
        t.close()
    assert counts["unnorm"] == counts["norm"]
