"""The sigmoid router of DeepSeek-V3 (DMoEConfig(router_score="sigmoid", routed_scaling_factor=c)): affinities sigma(s), top-k
over s (or over sigma(s) + b_e with expert biases), weights c * sigma_j / sum of the selected sigma, and the sigmoid form of
the load-balancing loss.

CPU: the configuration and its refusals, the oracles K.gate_topk_ref(score=...) and K.router_loss_ref(score=...) against
their written formulas in float64, a CPU trainer that balances a collapsed gate with sigmoid keys, and checkpoints.
GPU: the gate, gate_bwd and router-loss kernels against the oracles, one layer on both paths, both expert kinds and both
gates against the CPU oracle (and one DeepSeek-V3-shaped layer), and the trainer under its CUDA graph."""
import math

import pytest
import torch

import lah_b200  # noqa
from lah_b200.ops import kernels as K
from lah_b200.parallel import baseline, engine as E
from lah_b200.parallel.trainer import DMoETrainer
from routing_support import collapse, cpu_cfg, layer_against_the_oracle, load, run_gate, slots
from routing_support import one_thread, rt, step_counters, world1  # noqa: F401 (fixtures)

SIG = dict(router_score="sigmoid")


# ======================================================================================================== CPU: config
def test_defaults_and_state_dict_keys():
    cfg = E.DMoEConfig()
    assert cfg.router_score == "softmax" and cfg.routed_scaling_factor == 1.0
    plain = E.FusedDMoE(cpu_cfg())
    assert plain.router_score == "softmax" and plain.routed_scale == 1.0
    sig = E.FusedDMoE(cpu_cfg(routed_scaling_factor=2.5, **SIG))
    assert sig.router_score == "sigmoid" and sig.routed_scale == 2.5
    # the weight function adds no state: every layer keeps the keys of a default layer
    assert list(plain.state_dict()) == list(E.FusedDMoE(cpu_cfg(router_score="softmax")).state_dict())
    assert list(plain.state_dict()) == list(sig.state_dict())


@pytest.mark.parametrize("kw,match", [
    (dict(router_score="Sigmoid"), "router_score"), (dict(router_score="softmax2"), "router_score"),
    (dict(router_score=None), "router_score"),
    (dict(routed_scaling_factor=0.0, **SIG), "routed_scaling_factor"),
    (dict(routed_scaling_factor=-1.0, **SIG), "routed_scaling_factor"),
    (dict(routed_scaling_factor=float("nan"), **SIG), "routed_scaling_factor"),
    (dict(routed_scaling_factor=float("inf"), **SIG), "routed_scaling_factor"),
    (dict(routed_scaling_factor=2.5), "routed_scaling_factor"),
    (dict(routed_scaling_factor=0.5, router_score="softmax"), "routed_scaling_factor"),
    (dict(router_z_loss_coef=1e-3, **SIG), "router_z_loss_coef"),
])
def test_config_refusals(kw, match):
    with pytest.raises(ValueError, match=match):
        E.DMoEConfig(**kw)


@pytest.mark.parametrize("expert", ["ffn", "swiglu"])
@pytest.mark.parametrize("gate", ["product_key", "emulator"])
def test_every_gate_and_expert_kind_accepts_the_sigmoid_router(gate, expert):
    extra = dict(router_aux_loss_coef=0.01) if gate == "product_key" else {}
    if expert == "swiglu":
        extra["shared_inner_dim"] = 128
    cfg = cpu_cfg(grid_size=(16,), gate_mode=gate, expert=expert, expert_bias_update_rate=1e-3, failure_rate=0.1,
                  trainer_microbatches=2, routed_scaling_factor=2.5, **SIG, **extra)
    for path in ("small", "big"):
        E.DMoEConfig(**{**cfg.__dict__, "expert_path": path})
    E.DMoEConfig(**{**cfg.__dict__, "update_every_steps": 2})
    assert E.FusedDMoE(cfg).router_score == "sigmoid"


@pytest.mark.parametrize("arm", ["BaselineDMoE", "BaselineTrainer", "FastBaselineDMoE", "FastBaselineTrainer"])
def test_baseline_arms_refuse_the_sigmoid_router(arm):
    from lah_b200.parallel import baseline_fast
    cfg = E.DMoEConfig(hidden=64, grid_size=(4,), k=2, num_layers=1, tokens_per_rank=8, **SIG)
    make = dict(BaselineDMoE=lambda: baseline.BaselineDMoE(cfg), BaselineTrainer=lambda: baseline.BaselineTrainer(cfg),
                FastBaselineDMoE=lambda: baseline_fast.FastBaselineDMoE(cfg, 0, 16),
                FastBaselineTrainer=lambda: baseline_fast.FastBaselineTrainer(cfg))[arm]
    with pytest.raises(ValueError, match="router_score"):
        make()


# ======================================================================================================== CPU: oracles
def _case(grid, B, gen, dead=True):
    E_ = math.prod(grid)
    logits = torch.randn(B, sum(grid), generator=gen) * 2
    alive = (torch.rand(E_, generator=gen) > 0.3).to(torch.uint8) if dead else None
    fail = torch.rand(B, E_, generator=gen) < 0.2
    return logits, alive, fail


@pytest.mark.parametrize("grid", [(16,), (4, 4), (2, 3, 4), (2, 2, 2, 2)])
def test_unbiased_sigmoid_selects_like_softmax_and_weights_sum_to_the_scale(grid):
    gen = torch.Generator().manual_seed(1)
    logits, alive, fail = _case(grid, 80, gen)
    scores = K.product_key_scores(logits, grid)
    for k in (1, 3, 8):
        ref_idx, _ = K.gate_topk_ref(logits, grid, k, alive=alive, fail_mask=fail)
        for c in (1.0, 2.5):
            idx, w = K.gate_topk_ref(logits, grid, k, alive=alive, fail_mask=fail, score="sigmoid", scale=c)
            assert torch.equal(idx, ref_idx)
            valid = idx >= 0
            assert bool((w[~valid] == 0).all())
            has = valid.any(1)
            torch.testing.assert_close(w.sum(1)[has], torch.full((int(has.sum()),), c), rtol=0, atol=2e-6 * c)
            sg = torch.sigmoid(torch.gather(scores, 1, idx.clamp(min=0))) * valid
            torch.testing.assert_close(w, c * sg / sg.sum(1, keepdim=True).clamp_min(1e-30), rtol=1e-6, atol=0)


def test_biased_sigmoid_selection_ranks_sigma_plus_bias():
    grid = (16,)
    gen = torch.Generator().manual_seed(2)
    logits, alive, fail = _case(grid, 64, gen)
    bias = torch.randn(16, generator=gen) * 0.3
    idx, w = K.gate_topk_ref(logits, grid, 3, alive=alive, fail_mask=fail, bias=bias, score="sigmoid", scale=2.5)
    scores = K.product_key_scores(logits, grid)
    keys = torch.sigmoid(scores) + bias
    dead = ~alive.bool().view(1, -1) | fail
    for b in range(64):
        live = [e for e in range(16) if not dead[b, e]]
        order = sorted(live, key=lambda e: (-float(keys[b, e]), e))[:3]
        assert idx[b].tolist() == order + [-1] * (3 - len(order))
    sg = torch.sigmoid(torch.gather(scores, 1, idx.clamp(min=0))) * (idx >= 0)
    torch.testing.assert_close(w, 2.5 * sg / sg.sum(1, keepdim=True).clamp_min(1e-30), rtol=1e-6, atol=0)
    # a saturated affinity still loses to a larger bias: the bias is on the [0, 1] scale of sigma
    lg = torch.tensor([[30.0, 0.0, -30.0, 5.0]])
    i2, _ = K.gate_topk_ref(lg, (4,), 1, bias=torch.tensor([0.0, 0.6, 1.5, 0.0]), score="sigmoid")
    assert i2.tolist() == [[2]]


def _gate_bwd_formula(sig, w, dw, valid, c):
    """dL/ds_j = sigma_j (1 - sigma_j) (c dw_j - sum_i w_i dw_i) / S, S over the valid pairs (0 when S = 0)"""
    S = (sig * valid).sum(1, keepdim=True)
    dot = (w * dw).sum(1, keepdim=True)
    ds = sig * (1 - sig) * (c * dw - dot) / torch.where(S > 0, S, torch.ones_like(S))
    return torch.where(valid & (S > 0), ds, torch.zeros_like(ds))


def _scatter_to_logits(ds, idx, grid):
    """the gradient of the grid logits from per-pair score gradients: every grid logit of expert j gets ds_j"""
    B = ds.shape[0]
    dl = torch.zeros(B, sum(grid), dtype=ds.dtype)
    offs = [sum(grid[:d]) for d in range(len(grid))]
    for b in range(B):
        for j in range(idx.shape[1]):
            e = int(idx[b, j])
            if e < 0:
                continue
            rem = e
            for d in reversed(range(len(grid))):
                dl[b, offs[d] + rem % grid[d]] += ds[b, j]
                rem //= grid[d]
    return dl


@pytest.mark.parametrize("grid", [(16,), (4, 4), (2, 3, 4)])
@pytest.mark.parametrize("c", [1.0, 2.5])
def test_gate_backward_formula_equals_float64_autograd(grid, c):
    gen = torch.Generator().manual_seed(3)
    B, k = 40, 4
    logits, alive, fail = _case(grid, B, gen)
    logits = logits.double()
    logits[0] = -1000.0                              # every sigma of token 0 underflows: S = 0, zero weights
    idx, w_ref = K.gate_topk_ref(logits, grid, k, alive=alive, fail_mask=fail, score="sigmoid", scale=c)
    valid = idx >= 0
    assert bool((w_ref[0] == 0).all()) and bool(valid[0].any())
    dw = torch.randn(B, k, generator=gen, dtype=torch.float64) * valid
    dw[1, 0] = 0.0                                   # a pair that scatter_rows dropped: y_j = 0, so dw_j = 0
    lg = logits.clone().requires_grad_(True)
    sel = torch.gather(K.product_key_scores(lg, grid), 1, idx.clamp(min=0))
    w = K.sigmoid_weights_ref(sel, valid, c)
    torch.testing.assert_close(w.detach().float(), w_ref, rtol=1e-6, atol=1e-7)
    (w * dw).sum().backward()
    sig = torch.sigmoid(sel.detach()) * valid
    ds = _gate_bwd_formula(sig, w.detach(), dw, valid, c)
    torch.testing.assert_close(_scatter_to_logits(ds, idx, grid), lg.grad, rtol=1e-12, atol=1e-12)
    assert bool((lg.grad[0] == 0).all()) and torch.isfinite(lg.grad).all()
    assert float(ds[1, 0].abs()) > 0                 # the dropped pair keeps its share of S and gets a gradient


@pytest.mark.parametrize("dead", [False, True])
@pytest.mark.parametrize("grid", [(16,), (4, 4), (2, 3, 4), (2, 2, 2, 2)])
def test_sigmoid_router_loss_ref_equals_the_written_formula(grid, dead):
    gen = torch.Generator().manual_seed(4)
    B, E_ = 24, math.prod(grid)
    logits = torch.randn(B, sum(grid), generator=gen, dtype=torch.float64) * 3
    alive = (torch.rand(E_, generator=gen) > 0.3).to(torch.uint8) if dead else None
    counts = torch.randint(0, 9, (E_,), generator=gen)
    lg = logits.clone().requires_grad_(True)
    aux, zl = K.router_loss_ref(lg, grid, counts, alive=alive, score="sigmoid")
    assert float(zl) == 0.0
    scores = K.product_key_scores(logits, grid)
    live = [e for e in range(E_) if alive is None or alive[e]]
    N, T = len(live), int(counts.sum())
    f = [int(counts[e]) / T for e in range(E_)]
    sig = torch.sigmoid(scores)
    want, grad_s = 0.0, torch.zeros(B, E_, dtype=torch.float64)
    for b in range(B):
        S = sum(float(sig[b, e]) for e in live)
        Fb = sum(f[e] * float(sig[b, e]) for e in live) / S
        want += N * Fb / B
        for e in live:   # dL_aux/ds_{b,e} = (N/B) sigma_e (1 - sigma_e) (f_e - F_b) / S'_b
            grad_s[b, e] = N / B * float(sig[b, e] * (1 - sig[b, e])) * (f[e] - Fb) / S
    assert abs(aux.item() - want) < 1e-12
    (g,) = torch.autograd.grad(aux, lg)
    # the score gradient reaches the grid logits through the product-key sum
    lg2 = logits.clone().requires_grad_(True)
    (want_g,) = torch.autograd.grad((K.product_key_scores(lg2, grid) * grad_s).sum(), lg2)
    torch.testing.assert_close(g, want_g, rtol=1e-10, atol=1e-13)


def test_sigmoid_router_loss_of_underflowed_tokens_is_zero():
    logits = torch.full((3, 8), -1000.0, dtype=torch.float64, requires_grad=True)
    aux, zl = K.router_loss_ref(logits, (8,), torch.ones(8, dtype=torch.int64), score="sigmoid")
    assert aux.item() == 0.0 and zl.item() == 0.0
    aux.backward()
    assert bool((logits.grad == 0).all())


# ======================================================================================================== CPU: trainer
def test_cpu_layer_differentiates_through_the_sigmoid_weights():
    torch.manual_seed(0)
    layer = E.FusedDMoE(cpu_cfg(routed_scaling_factor=2.5, router_aux_loss_coef=0.01, **SIG)).train()
    x = torch.randn(32, 64)
    logits = layer.gate_logits(x, layer.proj).detach().requires_grad_(True)
    out = layer._forward_ref(x, logits)
    gy = torch.randn_like(out)
    (out * gy).sum().backward()
    assert torch.isfinite(logits.grad).all() and float(logits.grad.abs().max()) > 0
    aux, zl = layer.router_loss.tolist()
    assert aux > 0 and zl == 0.0


@pytest.mark.parametrize("gate", ["product_key", "emulator"])
def test_sigmoid_keys_with_expert_biases_spread_a_collapsed_router(one_thread, gate):
    """the §6b setting with the sigmoid router: two of eight experts take most rows; with biases on the affinity scale the
    load spreads to a max/mean below 0.6 of the run without them (and below 1.5), and the task loss falls in both runs"""
    gen = torch.Generator().manual_seed(0)
    protos = torch.randn(10, 16, generator=gen) * 2
    y = torch.randint(0, 10, (128,), generator=gen)
    x = protos[y] + 0.5 * torch.randn(128, 16, generator=gen)
    results = {}
    for rate in (0.0, 0.01):
        cfg = cpu_cfg(grid_size=(8,), k=2, num_layers=1, tokens_per_rank=128, lr=3e-3, gate_mode=gate,
                      expert_bias_update_rate=rate, routed_scaling_factor=2.0, **SIG)
        t = DMoETrainer(cfg)
        collapse(t.model.blocks[0], gate)
        before = load(t, x)
        losses = [t.train_step(x, y) for _ in range(120)]
        results[rate] = (before, load(t, x), losses)
    (b0, a0, l0), (b1, a1, l1) = results[0.0], results[0.01]
    assert b0 == b1 and b0[0] > 3.0
    assert a1[0] < 0.6 * a0[0] and a1[0] < 1.5, (a0, a1)
    assert l0[-1] < 0.5 * l0[0] and l1[-1] < 0.5 * l1[0], (l0[::20], l1[::20])


def test_sigmoid_checkpoint_round_trip(one_thread):
    cfg = cpu_cfg(num_layers=2, expert_bias_update_rate=1e-3, routed_scaling_factor=2.5, router_aux_loss_coef=0.01,
                  **SIG)
    gen = torch.Generator().manual_seed(4)
    xs = [torch.randn(64, 16, generator=gen) for _ in range(6)]
    ys = [torch.randint(0, 10, (64,), generator=gen) for _ in range(6)]
    a = DMoETrainer(cfg)
    for x, y in zip(xs[:3], ys[:3]):
        a.train_step(x, y)
    state = a.state_dict()
    assert state["trainer"]["router_score"] == "sigmoid"
    la = [a.train_step(x, y) for x, y in zip(xs[3:], ys[3:])]
    b = DMoETrainer(cfg)
    b.load_state_dict(state)
    lb = [b.train_step(x, y) for x, y in zip(xs[3:], ys[3:])]
    assert la == lb
    for ba, bb in zip(a.model.blocks, b.model.blocks):
        assert torch.equal(ba.expert_bias, bb.expert_bias) and torch.equal(ba.shard.p, bb.shard.p)
    assert torch.equal(a.flat_p, b.flat_p)


def test_checkpoints_of_the_other_router_score_are_refused(one_thread):
    x, y = torch.randn(64, 16), torch.randint(0, 10, (64,))
    soft, sig = DMoETrainer(cpu_cfg()), DMoETrainer(cpu_cfg(**SIG))
    soft.train_step(x, y)
    sig.train_step(x, y)
    plain = soft.state_dict()
    assert "router_score" not in plain["trainer"]     # default checkpoints keep their keys
    with pytest.raises(ValueError, match="router_score"):
        sig.load_state_dict(plain)
    with pytest.raises(ValueError, match="router_score"):
        soft.load_state_dict(sig.state_dict())
    # the same score loads, with or without the key
    DMoETrainer(cpu_cfg()).load_state_dict(plain)
    DMoETrainer(cpu_cfg(**SIG)).load_state_dict(sig.state_dict())


# ======================================================================================================== GPU
def _clear_tokens(scores, bias, dead, k):
    """tokens whose oracle keys sigma(s) + b among the k + 1 best are pairwise separated by more than 1e-6, or exactly
    tied with equal score and bias (then both sides order them by expert id)"""
    keys = (torch.sigmoid(scores) + bias).masked_fill(dead, float("-inf"))
    kk = min(k + 1, keys.shape[1])
    top_v, top_i = torch.sort(keys, dim=-1, descending=True, stable=True)
    top_v, top_i = top_v[:, :kk], top_i[:, :kk]
    s_sel, b_sel = torch.gather(scores, 1, top_i), bias[top_i]
    gap = (top_v[:, :-1] - top_v[:, 1:]).nan_to_num(float("inf"))   # -inf - -inf: two missing pairs
    same = (s_sel[:, :-1] == s_sel[:, 1:]) & (b_sel[:, :-1] == b_sel[:, 1:])
    return ((gap > 1e-6) | same | torch.isinf(top_v[:, 1:])).all(1)


@pytest.mark.gpu
@pytest.mark.parametrize("B", [1, 7, 256, 65536])
@pytest.mark.parametrize("grid", [(64,), (8, 8), (64, 64), (256,), (4096,), (4, 4, 4, 4)])
def test_sigmoid_gate_topk_against_the_oracle(step_counters, grid, B):
    E_ = math.prod(grid)
    gen = torch.Generator(device="cuda").manual_seed(B * 5 + E_)
    if len(grid) <= 2:   # continuous scores: s = l0 (+ l1) is the same float in any order
        logits = torch.randn(B, sum(grid), generator=gen, device="cuda") * 2
    else:                # dyadic logits: the 4-d sums are exact in any order
        logits = torch.randint(-12, 13, (B, sum(grid)), generator=gen, device="cuda").float() / 4
    dyadic = torch.randint(-12, 13, (B, sum(grid)), generator=gen, device="cuda").float() / 4
    bias = torch.randint(-8, 9, (E_,), generator=gen, device="cuda").float() / 16
    alive = (torch.rand(E_, generator=gen, device="cuda") > 0.2).to(torch.uint8)
    rate = 0.1
    fail = K.gate_fail_mask_ref(B, E_, rate, 99, 0).cuda()
    dead = ~alive.bool().view(1, -1) | fail
    unclear = total = 0
    for k in range(1, 9):
        c = 2.5 if k % 2 else 1.0
        # unbiased: the softmax router's selection, exactly
        idx, w, pos, counts, sig, _ = run_gate(logits, grid, k, alive=alive, rate=rate, bias=None, score="sigmoid",
                                               scale=c)
        ridx, rw = K.gate_topk_ref(logits, grid, k, alive=alive, fail_mask=fail, score="sigmoid", scale=c)
        assert torch.equal(idx.long(), ridx), (k, int((idx.long() != ridx).any(1).sum()))
        assert torch.equal(pos.long(), slots(ridx))
        assert torch.equal(counts.long(), torch.bincount(ridx[ridx >= 0], minlength=E_))
        assert float((w.double() - rw.double()).abs().max()) < 2e-6 * c, k
        rsig = torch.sigmoid(torch.gather(K.product_key_scores(logits, grid), 1, ridx.clamp(min=0))) * (ridx >= 0)
        assert float((sig - rsig).abs().max()) < 1e-6
        assert torch.equal(idx, run_gate(logits, grid, k, alive=alive, rate=rate, bias=None)[0])
        # biased: sigma(s) + b; ids equal wherever the oracle's keys are not near-tied
        idx, w, pos, counts, sig, _ = run_gate(dyadic, grid, k, alive=alive, rate=rate, bias=bias, score="sigmoid",
                                               scale=c)
        ridx, rw = K.gate_topk_ref(dyadic, grid, k, alive=alive, fail_mask=fail, bias=bias, score="sigmoid", scale=c)
        clear = _clear_tokens(K.product_key_scores(dyadic, grid), bias, dead, k)
        unclear += int((~clear).sum())
        total += B
        assert torch.equal(idx.long()[clear], ridx[clear]), (k, int((idx.long() != ridx)[clear].any(1).sum()))
        assert torch.equal(counts.long(), torch.bincount(idx.long()[idx >= 0], minlength=E_))
        assert torch.equal(pos.long(), slots(idx.long()))
        same = (idx.long() == ridx).all(1, keepdim=True)
        assert float(torch.where(same, w.double() - rw.double(), 0.0).abs().max()) < 2e-6 * c, k
    assert unclear <= 1e-3 * total, (unclear, total)


@pytest.mark.gpu
def test_sigmoid_wrappers_refuse_bad_arguments_before_launching():
    from lah_b200.ops import native
    lg = torch.zeros(4, 16, device="cuda")
    i = torch.zeros(16, dtype=torch.int32, device="cuda")
    ok = dict(idx=i, w=i.float(), pos=i, counts=torch.zeros(16, dtype=torch.int32, device="cuda"))
    sig = torch.zeros(16, device="cuda")
    before = native.launches()
    for kw in (dict(score="sigmoid"), dict(score="sigmoid", sig=torch.zeros(15, device="cuda")),
               dict(score="sigmoid", sig=torch.zeros(16)), dict(score="sigmoid", sig=sig.double()),
               dict(score="sigmoid", sig=torch.zeros(32, device="cuda")[::2]),
               dict(score="sigmoid", sig=sig, scale=0.0), dict(score="sigmoid", sig=sig, scale=float("nan")),
               dict(score="softmax", scale=2.0), dict(score="softmax", sig=sig), dict(score="tanh")):
        with pytest.raises(ValueError):
            K.gate_topk(lg, (16,), 4, **ok, **kw)
    f, z = torch.zeros(17, device="cuda"), torch.zeros(4, device="cuda")
    with pytest.raises(ValueError, match="z-loss"):
        K.router_loss_bwd(lg, (16,), f=f, z=z, Fb=z, aux_coef=0.1, z_coef=0.1, dlogits=torch.zeros_like(lg),
                          score="sigmoid")
    with pytest.raises(ValueError):
        K.router_loss_fwd(lg, (16,), i.view(1, -1), f=f, z=z, Fb=z, loss=torch.zeros(2, device="cuda"), score="tanh")
    assert native.launches() == before


@pytest.mark.gpu
@pytest.mark.parametrize("c", [1.0, 2.5])
@pytest.mark.parametrize("k", [1, 4, 8])
@pytest.mark.parametrize("grid,H", [((64,), 256), ((4, 4), 512), ((2, 32), 1024), ((3, 5, 7), 512), ((256,), 1024)])
def test_sigmoid_gate_bwd_against_the_float64_formula(rt, grid, H, k, c):
    gen = torch.Generator().manual_seed(k * H + len(grid))
    B = 257
    logits = torch.randn(B, sum(grid), generator=gen, dtype=torch.float64) * 2
    logits[3] = -1000.0                                    # every sigma underflows: no gradient
    idx, w = K.gate_topk_ref(logits.float(), grid, k, score="sigmoid", scale=c)
    idx[torch.rand(B, k, generator=gen) < 0.15] = -1
    valid = idx >= 0
    scores = K.product_key_scores(logits, grid)
    sig = torch.sigmoid(torch.gather(scores, 1, idx.clamp(min=0))).float() * valid
    w = K.sigmoid_weights_ref(torch.gather(scores, 1, idx.clamp(min=0)), valid, c).float()
    R = B * k + 50
    pair_row = torch.randperm(R, generator=gen)[: B * k].view(B, k)
    pair_row[torch.rand(B, k, generator=gen) < 0.05] = -1   # pairs that scatter_rows dropped
    pair_row = torch.where(valid, pair_row, torch.full_like(pair_row, -1))
    yo = rt.region[: R * H * 2].view(torch.bfloat16).view(R, H)
    yo.copy_(torch.randn(R, H, generator=gen).to(torch.bfloat16))
    g = torch.randn(B, H, generator=gen).to(torch.bfloat16)
    y = yo.cpu().double()[pair_row.clamp(min=0)] * (pair_row >= 0).double().unsqueeze(-1)
    dw = (g.double().unsqueeze(1) * y).sum(-1) * valid
    ds = _gate_bwd_formula(sig.double(), w.double(), dw, valid, c)
    ref = _scatter_to_logits(ds, idx, grid)
    dl = torch.full((B, sum(grid)), 5.0, device="cuda")
    K.gate_bwd(rt.region_off, g.cuda(), idx.flatten().to(torch.int32).cuda(),
               pair_row.flatten().to(torch.int32).cuda(), w.flatten().cuda(), dl, k, math.prod(grid), grid,
               score="sigmoid", scale=c, sig=sig.flatten().cuda())
    torch.cuda.synchronize()
    dl = dl.cpu().double()
    assert bool((dl[3] == 0).all())
    # relative to the largest single term sigma (1 - sigma) c |dw| / S: with k = 1 the exact gradient is 0 and the kernel's
    # is the rounding of c dw - w dw
    S = sig.double().sum(1, keepdim=True)
    terms = sig.double() * (1 - sig.double()) * c * dw.abs() / torch.where(S > 0, S, torch.ones_like(S))
    err = float((dl - ref).abs().max() / terms.max().clamp_min(1e-30))
    assert err < 1e-4, err


def _router_kernels(logits, grid, counts, alive, alpha):
    B, E_ = logits.shape[0], math.prod(grid)
    dev = logits.device
    f = torch.empty(E_ + 1, device=dev)
    z, Fb, loss = torch.empty(B, device=dev), torch.empty(B, device=dev), torch.empty(2, device=dev)
    K.router_loss_fwd(logits, grid, counts.view(1, -1), alive=alive, f=f, z=z, Fb=Fb, loss=loss, score="sigmoid")
    dl = torch.zeros_like(logits)
    K.router_loss_bwd(logits, grid, alive=alive, f=f, z=z, Fb=Fb, aux_coef=alpha, z_coef=0.0, dlogits=dl,
                      score="sigmoid")
    torch.cuda.synchronize()
    return loss.clone(), dl, f.clone(), z.clone(), Fb.clone()


@pytest.mark.gpu
@pytest.mark.parametrize("B", [1, 7, 256, 65536])
@pytest.mark.parametrize("grid", [(64,), (8, 8), (32, 32), (64, 64), (4, 4, 4, 4)])
def test_sigmoid_router_loss_kernels_against_float64_autograd(step_counters, grid, B):
    dev = torch.device("cuda")
    E_ = math.prod(grid)
    gen = torch.Generator().manual_seed(B + E_)
    alive = (torch.rand(E_, generator=gen) > 0.2).to(torch.uint8).to(dev)
    for k, mag in ((1, 2.0), (4, 20.0), (8, 5.0)):
        logits = ((torch.rand(B, sum(grid), generator=gen) * 2 - 1) * mag).to(dev)
        counts = torch.zeros(E_, dtype=torch.int32, device=dev)
        idx = torch.empty(B * k, dtype=torch.int32, device=dev)
        K.gate_topk(logits, grid, k, alive=alive, failure_rate=0.1, seed=11, token_offset=0, idx=idx,
                    w=torch.empty(B * k, device=dev), pos=torch.empty_like(idx), counts=counts, score="sigmoid",
                    scale=1.0, sig=torch.empty(B * k, device=dev))
        alpha = 0.5
        loss, dl, f, z, Fb = _router_kernels(logits, grid, counts, alive, alpha)
        lg = logits.double().requires_grad_(True)
        aux, zl = K.router_loss_ref(lg, grid, counts, alive=alive, score="sigmoid")
        (ref,) = torch.autograd.grad(alpha * aux, lg)
        assert float(loss[1]) == 0.0 and torch.isfinite(dl).all()
        assert abs(float(loss[0]) - aux.item()) <= 1e-4 * abs(aux.item()), (k, loss.tolist(), aux.item())
        gerr = ((dl.double() - ref).abs().max() / ref.abs().max().clamp_min(1e-30)).item()
        assert gerr < 1e-4, (k, gerr)
        again = _router_kernels(logits, grid, counts, alive, alpha)
        assert all(torch.equal(a, b) for a, b in zip((loss, dl, f, z, Fb), again))
        del lg, aux, zl, ref


def _check(r):
    """the weights of the tokens routed alike, the bias update of the routed counts, and the sigmoid router's losses"""
    cfg, E_ = r.layer.cfg, r.layer.cfg.num_experts
    assert float((r.w - r.rw)[r.same].abs().max()) < 2e-6 * cfg.routed_scaling_factor
    assert torch.equal(r.layer.expert_bias, K.expert_bias_update_ref(r.ctx.cnt_all[:1, :E_], r.bias0,
                                                                     cfg.expert_bias_update_rate))
    if bool(r.same.all()):
        assert torch.equal(r.layer.expert_bias, r.oracle.expert_bias)
    if r.layer.router_loss is not None:
        torch.testing.assert_close(r.layer.router_loss, r.oracle.router_loss, rtol=1e-3, atol=1e-6)
        assert float(r.layer.router_loss[1]) == 0.0


@pytest.mark.gpu
@pytest.mark.parametrize("gate", ["emulator", "product_key"])
@pytest.mark.parametrize("expert", ["ffn", "swiglu"])
@pytest.mark.parametrize("path", ["small", "big"])
def test_layer_against_the_cpu_oracle(path, expert, gate):
    torch.manual_seed(3)
    grid = (16,) if gate == "emulator" else (4, 4)
    cfg = E.DMoEConfig(hidden=512, grid_size=grid, k=4, num_layers=1, tokens_per_rank=512, expert=expert,
                       expert_path=path, gate_mode=gate, expert_bias_update_rate=0.01, routed_scaling_factor=2.5, **SIG)
    layer_against_the_oracle(cfg, max_mismatch=2, check=_check)   # near-ties of sigma(s) + b may go either way


@pytest.mark.gpu
@pytest.mark.parametrize("path", ["small", "big"])
def test_deepseek_v3_shaped_layer_against_the_cpu_oracle(path):
    """product-key gate (the emulator gate refuses router losses): SwiGLU experts, a shared expert, expert biases, the
    sigmoid load-balancing loss and c = 2.5"""
    torch.manual_seed(4)
    grid = (8, 8)
    cfg = E.DMoEConfig(hidden=512, grid_size=grid, k=8, num_layers=1, tokens_per_rank=512, expert="swiglu",
                       inner_dim=256, shared_inner_dim=512, expert_path=path, expert_bias_update_rate=1e-3,
                       router_aux_loss_coef=1e-2, routed_scaling_factor=2.5, **SIG)
    layer_against_the_oracle(cfg, max_mismatch=2, check=_check)


@pytest.mark.gpu
def test_layer_refuses_a_context_of_the_other_router_score():
    cfg = E.DMoEConfig(hidden=512, grid_size=(16,), k=4, num_layers=1, tokens_per_rank=256)
    ctx = E.EngineContext(cfg)
    try:
        assert E.FusedDMoE(cfg, ctx).ws.sig is None
        with pytest.raises(ValueError, match="router_score"):
            E.FusedDMoE(E.DMoEConfig(**{**cfg.__dict__, **SIG}), ctx)
    finally:
        ctx.close()


def _trainer_cfg(path, gate, **kw):
    base = dict(hidden=512, grid_size=(16,), k=4, num_layers=2, tokens_per_rank=256, failure_rate=0.1, lr=1e-4,
                expert_path=path, gate_mode=gate, expert_bias_update_rate=1e-3, routed_scaling_factor=2.5, **SIG)
    base.update(kw)
    return E.DMoEConfig(**base)


@pytest.mark.gpu
@pytest.mark.parametrize("gate", ["emulator", "product_key"])
@pytest.mark.parametrize("path", ["small", "big"])
def test_trainer_graph_equals_eager_and_runs_are_reproducible(path, gate):
    kw = dict(router_aux_loss_coef=1e-2) if gate == "product_key" else {}
    cfg = _trainer_cfg(path, gate, **kw)
    torch.manual_seed(0)
    xs = [torch.randn(256, cfg.in_features, device="cuda") for _ in range(5)]
    ys = [torch.randint(0, 10, (256,), device="cuda") for _ in range(5)]
    runs = {}
    for run, graph in (("eager", False), ("graph", True), ("graph2", True)):
        t = DMoETrainer(cfg, use_graph=graph)
        losses, biases = [], []
        for x, y in zip(xs, ys):
            losses.append(t.train_step_device(x, y).clone())
            biases.append(torch.stack([b.expert_bias for b in t.model.blocks]).clone())
        assert (t._graph is not None) == graph
        t.ctx.check_status()
        runs[run] = (torch.stack(losses).cpu(), torch.stack(biases).cpu(),
                     torch.cat([b.shard.p for b in t.model.blocks] + [t.flat_p]).cpu())
        t.close()
    for a, b in zip(runs["eager"], runs["graph"]):
        assert torch.equal(a, b)
    for a, b in zip(runs["graph"], runs["graph2"]):
        assert torch.equal(a, b)


@pytest.mark.gpu
@pytest.mark.parametrize("m", [1, 2])
def test_sigmoid_trainer_launches_as_many_kernels_as_softmax(m):
    counts = {}
    base = dict(hidden=512, grid_size=(16,), k=4, num_layers=2, tokens_per_rank=256, expert_path="small",
                gate_mode="product_key", trainer_microbatches=m, expert_bias_update_rate=1e-3,
                router_aux_loss_coef=1e-2)
    for name, kw in (("softmax", {}), ("sigmoid", dict(routed_scaling_factor=2.5, **SIG))):
        cfg = E.DMoEConfig(**base, **kw)
        t = DMoETrainer(cfg, use_graph=True)
        x, y = torch.randn(256, cfg.in_features, device="cuda"), torch.randint(0, 10, (256,), device="cuda")
        for _ in range(3):
            t.train_step_device(x, y)
        counts[name] = t._graph_launches
        t.close()
    assert counts["sigmoid"] == counts["softmax"]
