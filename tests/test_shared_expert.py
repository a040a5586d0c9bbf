"""Shared-expert isolation (DeepSeek-MoE / Qwen-MoE) in the fused DMoE layer: DMoEConfig(shared_inner_dim=...) adds one
always-active GatedFeedforwardBlock whose ``module(x) - x`` every token receives beside its k routed experts.

CPU: the configuration and its refusals, the flat trainer layout, the engine's oracle against BaselineDMoE with a real
GatedFeedforwardBlock, the export into that module, bit-exact resume (micro-batches, stale trainer gradients) and the
checkpoint rules.
GPU: combine_rows with an addend against an exact oracle, one layer on both expert paths and both sides of the 512-row
GEMM switch against the CPU oracle, the trainer at the bench point under its CUDA graph, close to the CPU trainer and
within its launch budget, and a zeroed W2 that leaves the routed part of a step bit for bit as it was."""
import math

import pytest
import torch

import lah_b200  # noqa
from lah_b200.models import GatedFeedforwardBlock
from lah_b200.models.layers import gated_inner_dim
from lah_b200.ops import kernels as K
from lah_b200.parallel import baseline, engine as E
from lah_b200.parallel.trainer import DMoETrainer
from routing_support import rel
from routing_support import one_thread, rt, world1  # noqa: F401 (fixtures)

BF16 = torch.bfloat16
#: the bench operating point: 64 experts, top-4, 256 samples per step, 4 layers, emulator gate
BENCH = dict(grid_size=(64,), k=4, num_layers=4, tokens_per_rank=256, gate_mode="emulator")
#: kernels the shared expert adds per layer and micro-batch: forward 2 casts + RMSNorm + GEMM + SwiGLU + GEMM; backward
#: GEMM + SwiGLU + GEMM + RMSNorm (2 launches) + 2 wgrads.  The combines take the addend in their existing launch
SHARED_LAUNCHES = 6 + 7


def _cfg(**kw):
    base = dict(hidden=32, grid_size=(2, 4), k=3, num_layers=1, tokens_per_rank=16, expert="swiglu", inner_dim=48,
                shared_inner_dim=40)
    base.update(kw)
    return E.DMoEConfig(**base)


def _shared_params(model):
    return {n: p for n, p in model.named_parameters() if n.rsplit(".", 1)[-1].startswith("shared_")}


# ======================================================================================================== CPU: config
def test_default_is_off_and_adds_nothing():
    assert E.DMoEConfig().shared_inner_dim == 0
    plain = E.FusedDMoE(_cfg(shared_inner_dim=0))
    assert plain.shared_inner == 0 and plain.shared_expert_parameters() == []
    assert not _shared_params(plain)
    with pytest.raises(ValueError, match="no shared expert"):
        plain.shared_expert_state_dict()
    layer = E.FusedDMoE(_cfg())
    assert {n: tuple(p.shape) for n, p in _shared_params(layer).items()} == \
        {"shared_g": (32,), "shared_w13": (80, 32), "shared_w2": (32, 40)}
    assert set(layer.state_dict()) == set(plain.state_dict()) | {"shared_g", "shared_w13", "shared_w2"}


@pytest.mark.parametrize("kw", [dict(expert="ffn", inner_dim=0), dict(shared_inner_dim=-128),
                                dict(shared_inner_dim=-1)])
def test_config_refusals(kw):
    with pytest.raises(ValueError, match="shared_inner_dim"):
        _cfg(**kw)


@pytest.mark.parametrize("width", [40, 200, 64])
def test_gpu_sizes_refused_and_cpu_oracle_takes_any_size(width):
    cfg = _cfg(hidden=128, inner_dim=128, shared_inner_dim=width)
    with pytest.raises(ValueError, match="shared_inner_dim a multiple of 128"):
        cfg.check_native_sizes()
    _cfg(hidden=128, inner_dim=128, shared_inner_dim=256).check_native_sizes()
    assert E.FusedDMoE(cfg)(torch.randn(3, 128)).shape == (3, 128)


@pytest.mark.parametrize("arm", ["FastBaselineDMoE", "FastBaselineTrainer"])
def test_fast_baseline_arms_refuse_a_shared_expert(arm):
    from lah_b200.parallel import baseline_fast
    cfg = E.DMoEConfig(hidden=64, grid_size=(4,), k=2, num_layers=1, tokens_per_rank=8, expert="swiglu",
                       shared_inner_dim=128)
    make = dict(FastBaselineDMoE=lambda: baseline_fast.FastBaselineDMoE(cfg, 0, 16),
                FastBaselineTrainer=lambda: baseline_fast.FastBaselineTrainer(cfg))[arm]
    with pytest.raises(ValueError, match="shared_inner_dim"):
        make()


def test_off_keeps_the_flat_trainer_layout():
    kw = dict(hidden=32, grid_size=(2, 2), k=2, num_layers=2, in_features=12, tokens_per_rank=32, expert="swiglu",
              inner_dim=64)
    plain = DMoETrainer(E.DMoEConfig(**kw))
    zero = DMoETrainer(E.DMoEConfig(**kw, shared_inner_dim=0))
    assert plain.num_trainer_params == zero.num_trainer_params and plain._n_pad == zero._n_pad
    assert torch.equal(plain.flat_p, zero.flat_p)
    offsets = lambda t: [(n, (p.data_ptr() - t.flat_p.data_ptr()) // 4) for n, p in t.model.named_parameters()]
    assert offsets(plain) == offsets(zero)
    # on: the shared tensors are added, each starting at an aligned offset, and the others keep their order
    on = DMoETrainer(E.DMoEConfig(**kw, shared_inner_dim=48))
    assert on.num_trainer_params == plain.num_trainer_params + 2 * (32 + 2 * 48 * 32 + 32 * 48)
    off = dict(offsets(on))
    assert all(off[n] % on.SHARED_ALIGN == 0 for n in _shared_params(on.model))
    assert [n for n, _ in offsets(plain)] == [n for n in off if n not in _shared_params(on.model)]


# ======================================================================================================== CPU: oracle
def test_cpu_oracle_matches_baseline_with_a_real_gated_block_and_one_trainer_step():
    torch.manual_seed(0)
    cfg = _cfg(lr=1e-2)
    fused = E.FusedDMoE(cfg).train()
    base = baseline.BaselineDMoE(cfg)
    assert isinstance(base.shared_expert, GatedFeedforwardBlock)
    base.load_from_shard(fused.shard)
    base.proj.load_state_dict(fused.proj.state_dict())
    base.shared_expert.load_state_dict(fused.shared_expert_state_dict())
    x = torch.randn(12, 32, requires_grad=True)
    x2 = x.detach().clone().requires_grad_(True)
    gy = torch.randn(12, 32)
    y1, y2 = fused(x), base(x2)
    torch.testing.assert_close(y1, y2, atol=1e-5, rtol=1e-5)
    (y1 * gy).sum().backward()
    (y2 * gy).sum().backward()
    torch.testing.assert_close(x.grad, x2.grad, atol=1e-5, rtol=1e-5)
    torch.testing.assert_close(fused.proj.weight.grad, base.proj.weight.grad, atol=1e-5, rtol=1e-5)
    grads = E.GATED_LAYOUT.module_state({n: p.grad for n, p in zip(E.GATED_LAYOUT.names,
                                                                    fused.shared_expert_parameters())})
    for k, p in base.shared_expert.named_parameters():
        torch.testing.assert_close(grads[k], p.grad, atol=1e-5, rtol=1e-5)

    # one trainer step: the engine's CPU trainer against BaselineTrainer (both draw the trainer side from the same seed)
    tcfg = _cfg(num_layers=2, in_features=12, tokens_per_rank=24, lr=1e-2)
    ours, theirs = DMoETrainer(tcfg), baseline.BaselineTrainer(tcfg, device=torch.device("cpu"))
    for a, b in zip(ours.model.blocks, theirs.model.blocks):
        b.load_from_shard(a.shard)
        assert all(torch.equal(v, b.shared_expert.state_dict()[k]) for k, v in a.shared_expert_state_dict().items())
    xs, ys = torch.randn(24, 12), torch.randint(0, 10, (24,))
    assert abs(ours.train_step(xs, ys) - theirs.train_step(xs, ys)) < 1e-5
    for a, b in zip(ours.model.blocks, theirs.model.blocks):
        for k, v in a.shared_expert_state_dict().items():
            torch.testing.assert_close(v, b.shared_expert.state_dict()[k], atol=1e-6, rtol=1e-5)
        torch.testing.assert_close(a.proj.weight, b.proj.weight, atol=1e-6, rtol=1e-5)


def test_exported_gated_block_is_the_shared_term():
    torch.manual_seed(1)
    layer = E.FusedDMoE(_cfg()).eval()
    with torch.no_grad():
        layer.shared_g.uniform_(0.5, 1.5)
    module = GatedFeedforwardBlock(32, 40, eps=E.GATED_EPS)
    module.load_state_dict(layer.shared_expert_state_dict())
    x = torch.randn(20, 32)
    with torch.no_grad():
        y = layer(x)
        layer.shared_w2.zero_()
        routed = layer(x)
        torch.testing.assert_close(y - routed, module(x) - x, atol=1e-5, rtol=1e-5)
    # and back: loading the module's state restores the term
    layer.load_shared_expert_state_dict(module.state_dict())
    with torch.no_grad():
        torch.testing.assert_close(layer(x), y, atol=0, rtol=0)
    with pytest.raises(ValueError, match="shape"):
        layer.load_shared_expert_state_dict(GatedFeedforwardBlock(32, 48).state_dict())


@pytest.mark.parametrize("m,stale", [(1, 0), (2, 0), (1, 1), (2, 1)])
def test_resumed_run_equals_the_continued_run(one_thread, m, stale):
    cfg = E.DMoEConfig(hidden=32, grid_size=(2, 2), k=2, num_layers=2, in_features=12, tokens_per_rank=32, lr=3e-3,
                       expert="swiglu", inner_dim=64, shared_inner_dim=48, trainer_microbatches=m,
                       trainer_staleness=stale)
    gen = torch.Generator().manual_seed(4)
    xs = [torch.randn(32, 12, generator=gen) for _ in range(6)]
    ys = [torch.randint(0, 10, (32,), generator=gen) for _ in range(6)]
    a = DMoETrainer(cfg)
    before = {n: p.detach().clone() for n, p in _shared_params(a.model).items()}
    for x, y in zip(xs[:3], ys[:3]):
        a.train_step(x, y)
    assert all(not torch.equal(before[n], p) for n, p in _shared_params(a.model).items())   # the shared expert trains
    state = a.state_dict()
    assert "blocks.1.shared_w13" in state["trainer"]["model"]
    la = [a.train_step(x, y) for x, y in zip(xs[3:], ys[3:])]
    b = DMoETrainer(cfg)
    b.load_state_dict(state)
    lb = [b.train_step(x, y) for x, y in zip(xs[3:], ys[3:])]
    assert la == lb
    assert torch.equal(a.flat_p, b.flat_p) and torch.equal(a.flat_m, b.flat_m)
    for ba, bb in zip(a.model.blocks, b.model.blocks):
        assert torch.equal(ba.shard.p, bb.shard.p)


def test_checkpoint_mismatches_raise(one_thread):
    kw = dict(hidden=32, grid_size=(2, 2), k=2, num_layers=1, in_features=12, tokens_per_rank=32, expert="swiglu",
              inner_dim=64)
    x, y = torch.randn(32, 12), torch.randint(0, 10, (32,))
    plain, on, wide = (DMoETrainer(E.DMoEConfig(**kw, shared_inner_dim=s)) for s in (0, 48, 64))
    for t in (plain, on, wide):
        t.train_step(x, y)
    with pytest.raises(ValueError, match="shared expert"):
        plain.load_state_dict(on.state_dict())
    with pytest.raises(ValueError, match="shared expert"):
        on.load_state_dict(plain.state_dict())
    with pytest.raises(ValueError, match="widths"):
        on.load_state_dict(wide.state_dict())
    on.load_state_dict(on.state_dict())   # and the matching case loads


# ======================================================================================================== GPU
def _combine_case(B, k, H, R, gen, dyadic):
    idx = torch.randint(0, 16, (B, k), generator=gen)
    idx[torch.rand(B, k, generator=gen) < 0.1] = -1
    pair_row = torch.randperm(R, generator=gen)[:B * k].view(B, k)
    pair_row[torch.rand(B, k, generator=gen) < 0.05] = -1
    idx[0] = -1
    pair_row = torch.where(idx >= 0, pair_row, torch.full_like(pair_row, -1))
    if dyadic:   # eighths in [-4, 4] and weights in sixteenths: every fp32 partial sum is exact
        src = torch.randint(-32, 33, (R, H), generator=gen).float() / 8
        add = torch.randint(-32, 33, (B, H), generator=gen).float() / 8
        w = torch.randint(0, 17, (B, k), generator=gen).float() / 16
    else:
        src, add, w = torch.randn(R, H, generator=gen), torch.randn(B, H, generator=gen), torch.rand(B, k, generator=gen)
    return idx, pair_row, src.to(BF16), add.to(BF16), w


@pytest.mark.gpu
@pytest.mark.parametrize("B", [256, 4000])
@pytest.mark.parametrize("H", [256, 512, 1024])
def test_combine_rows_with_an_addend_against_the_exact_oracle(rt, H, B):
    region, off = rt.region, rt.region_off
    k = 4
    R = B * k + 64
    gen = torch.Generator().manual_seed(H + B)
    src_view = region[:R * H * 2].view(BF16).view(R, H)
    for dyadic in (True, False):
        idx, pair_row, src, add, w = _combine_case(B, k, H, R, gen, dyadic)
        src_view.copy_(src.cuda())
        i32 = lambda t: t.flatten().to(torch.int32).cuda()
        out = {}
        for name, a, wt in (("add", add, w), ("none", None, w), ("zero", torch.zeros_like(add), w), ("sum", add, None)):
            o = torch.full((B, H), 3.0, dtype=BF16, device="cuda")
            K.combine_rows(off, i32(idx), i32(pair_row), None if wt is None else wt.flatten().cuda(), o, k, 16,
                           addend=None if a is None else a.cuda())
            out[name] = o.cpu()
        torch.cuda.synchronize()
        ref = K.combine_rows_ref(src, idx, pair_row, w, add)
        if dyadic:
            assert torch.equal(out["add"], ref)
            assert torch.equal(out["sum"], K.combine_rows_ref(src, idx, pair_row, None, add))
            assert torch.equal(out["none"], K.combine_rows_ref(src, idx, pair_row, w))
        else:   # fp32 accumulation: within one bf16 ulp of the float64 sum, plus the bound of fp32 accumulation (which
            # only matters where the terms cancel)
            exact = K.combine_rows_ref(src, idx, pair_row, w, add).double()
            terms = src.double()[pair_row.clamp(min=0)] * ((pair_row >= 0).double() * w.double()).unsqueeze(-1)
            total = terms.sum(1) + add.double()
            _, e = torch.frexp(total.abs().clamp(min=2.0 ** -126))
            tol = torch.pow(2.0, (e - 8).double()) + (k + 1) * 2.0 ** -23 * (terms.abs().sum(1) + add.double().abs())
            assert bool(((out["add"].double() - total).abs() <= tol).all())
            assert float((out["add"].double() != exact).double().mean()) < 0.01
        # a zero addend is the plain kernel, bit for bit; token 0 has no pair and gets the addend alone
        assert torch.equal(out["zero"], out["none"])
        assert torch.equal(out["add"][0], add[0])


@pytest.mark.gpu
def test_combine_rows_refuses_a_bad_addend(rt):
    from lah_b200.ops import native
    off = rt.region_off
    i = torch.zeros(8, dtype=torch.int32, device="cuda")
    out = torch.zeros(2, 256, dtype=BF16, device="cuda")
    before = native.launches()
    for bad in (torch.zeros(2, 256, device="cuda"), torch.zeros(3, 256, dtype=BF16, device="cuda"),
                torch.zeros(2, 512, dtype=BF16, device="cuda")[:, ::2],
                torch.zeros(2 * 256 + 1, dtype=BF16, device="cuda")[1:].view(2, 256)):
        with pytest.raises(ValueError):
            K.combine_rows(off, i, i, None, out, 4, 16, addend=bad)
    assert native.launches() == before


@pytest.mark.gpu
@pytest.mark.parametrize("failure_rate", [0.0, 0.1])
@pytest.mark.parametrize("B", [200, 600])
@pytest.mark.parametrize("path", ["small", "big"])
def test_layer_against_the_bf16_oracle(path, B, failure_rate):
    """one layer, 16 experts, k = 4, a shared expert of 1024: y, dx, the proj gradient and the three shared gradients
    against the CPU oracle path on the GPU (rounded to bf16 where the GPU path stores bf16), with the tolerances of
    test_dmoe_swiglu.py.  B = 200 runs the swap-AB GEMMs, B = 600 the 128-row tiles; a call at 1000 rows before it
    leaves stale rows in the padding, which must not reach the gradients"""
    torch.manual_seed(3)
    cfg = E.DMoEConfig(hidden=512, grid_size=(4, 4), k=4, num_layers=1, tokens_per_rank=1024, lr=1e-3,
                       expert="swiglu", expert_path=path, shared_inner_dim=1024, failure_rate=failure_rate)
    ctx = E.EngineContext(cfg)
    try:
        layer = E.FusedDMoE(cfg, ctx).cuda().train()
        assert ctx.small == (path == "small")
        big = torch.randn(1000, 512, device="cuda").to(BF16).requires_grad_(True)
        layer(big).backward(torch.randn(1000, 512, device="cuda").to(BF16))
        torch.cuda.synchronize()
        shared = layer.shared_expert_parameters()
        assert all(float(p.grad.abs().max()) > 0 for p in shared)
        for p in shared:
            p.grad.zero_()
        layer.proj.weight.grad = layer.proj.bias.grad = None
        oracle = E.FusedDMoE(cfg, device=torch.device("cuda")).cuda().train()
        oracle.ref_emulate_bf16 = True
        with torch.no_grad():
            oracle.load_state_dict(layer.state_dict())
            oracle.shard.p.copy_(layer.shard.p[:oracle.shard.p.numel()])
        # the failure draws of the layer's second call: its tokens follow the first call's 1000 in the stream
        oracle.ref_fail_mask = (K.gate_fail_mask_ref(B, 16, failure_rate, cfg.seed * 7919, 1000).cuda()
                                if failure_rate else None)
        x = torch.randn(B, 512, device="cuda").to(BF16).requires_grad_(True)
        gy = torch.randn(B, 512, device="cuda").to(BF16)
        y = layer(x)
        y.backward(gy)
        torch.cuda.synchronize()
        ctx.check_status()
        xr = x.detach().float().requires_grad_(True)
        yr = oracle(xr)
        yr.backward(gy.float())
        ridx, _ = K.gate_topk_ref(oracle.gate_logits(xr, oracle.proj).detach(), cfg.grid_size, cfg.k,
                                  fail_mask=oracle.ref_fail_mask)
        assert torch.equal(layer.ws.idx[:B * cfg.k].view(B, cfg.k).long(), ridx)
        if failure_rate:   # the failures changed the routing
            assert not torch.equal(ridx, K.gate_topk_ref(oracle.gate_logits(xr, oracle.proj).detach(), cfg.grid_size,
                                                         cfg.k)[0])
        errs = dict(y=rel(y, yr), dx=rel(x.grad, xr.grad), dproj=rel(layer.proj.weight.grad, oracle.proj.weight.grad))
        werr = {n: rel(a.grad, b.grad) for n, a, b in zip(E.GATED_LAYOUT.names, shared,
                                                          oracle.shared_expert_parameters())}
        assert errs["y"] < 2e-2 and errs["dx"] < 3e-2 and errs["dproj"] < 5e-2, errs
        assert max(werr.values()) < 8e-2, werr
    finally:
        ctx.close()


def _bench_cfg(**kw):
    return E.DMoEConfig(**{**BENCH, "hidden": 512, "expert": "swiglu", "shared_inner_dim": gated_inner_dim(512),
                           "lr": 1e-4, **kw})


def _snapshot(t):
    return torch.cat([b.shard.p for b in t.model.blocks] + [t.flat_p]).cpu()


@pytest.mark.gpu
def test_trainer_graph_equals_eager_and_runs_are_reproducible():
    cfg = _bench_cfg(failure_rate=0.1)
    torch.manual_seed(0)
    xs = [torch.randn(256, cfg.in_features, device="cuda") for _ in range(5)]
    ys = [torch.randint(0, 10, (256,), device="cuda") for _ in range(5)]
    runs = {}
    for run, graph in (("eager", False), ("graph", True), ("graph2", True)):
        t = DMoETrainer(cfg, use_graph=graph)
        assert t.ctx.small
        losses = torch.stack([t.train_step_device(x, y).clone() for x, y in zip(xs, ys)]).cpu()
        assert (t._graph is not None) == graph
        t.ctx.check_status()
        runs[run] = (losses, _snapshot(t))
        t.close()
    for a, b in zip(runs["eager"], runs["graph"]):
        assert torch.equal(a, b)
    for a, b in zip(runs["graph"], runs["graph2"]):
        assert torch.equal(a, b)


@pytest.mark.gpu
@pytest.mark.parametrize("m", [1, 2])
def test_trainer_close_to_the_cpu_trainer(m):
    """3 steps of the GPU trainer against the engine's fp32 CPU trainer started from the same state"""
    cfg = _bench_cfg(trainer_microbatches=m, lr=1e-3)
    torch.manual_seed(1)
    xs = [torch.randn(256, cfg.in_features) for _ in range(3)]
    ys = [torch.randint(0, 10, (256,)) for _ in range(3)]
    gpu = DMoETrainer(cfg)
    cpu = DMoETrainer(cfg, device=torch.device("cpu"))
    cpu.load_state_dict(gpu.state_dict())
    start = {n: p.detach().cpu().clone() for n, p in _shared_params(cpu.model).items()}
    lg = [float(gpu.train_step_device(x.cuda(), y.cuda())) for x, y in zip(xs, ys)]
    lc = [cpu.train_step(x, y) for x, y in zip(xs, ys)]
    gpu.ctx.check_status()
    for a, b in zip(lg, lc):
        assert abs(a - b) < 2e-2 * max(1.0, abs(b)), (lg, lc)
    got = {n: p.detach().cpu() for n, p in _shared_params(gpu.model).items()}
    for n, p in _shared_params(cpu.model).items():
        move = float((p.detach() - start[n]).abs().mean())
        diff = float((got[n] - p.detach()).abs().mean())
        assert move > 0 and diff < 0.25 * move, (n, diff, move)
    gpu.close()


@pytest.mark.gpu
@pytest.mark.parametrize("m", [1, 2])
def test_launch_budget(m):
    counts = {}
    base = dict(hidden=512, grid_size=(16,), k=4, num_layers=2, tokens_per_rank=256, expert_path="small",
                gate_mode="emulator", expert="swiglu", trainer_microbatches=m)
    for name, kw in (("plain", {}), ("zero", dict(shared_inner_dim=0)), ("shared", dict(shared_inner_dim=512))):
        cfg = E.DMoEConfig(**base, **kw)
        t = DMoETrainer(cfg, use_graph=True)
        x, y = torch.randn(256, cfg.in_features, device="cuda"), torch.randint(0, 10, (256,), device="cuda")
        for _ in range(3):
            t.train_step_device(x, y)
        assert t._graph is not None
        counts[name] = t._graph_launches
        t.close()
    assert counts["plain"] == counts["zero"]
    assert counts["shared"] == counts["plain"] + SHARED_LAUNCHES * base["num_layers"] * m


def _record(model):
    """forward hooks: every block's output y and the gradient of its input (its dx)"""
    ys, dxs, handles = [], [], []

    def hook(module, inputs, output):
        ys.append(output.detach().clone())
        inputs[0].register_hook(lambda g: dxs.append(g.detach().clone()))

    for block in model.blocks:
        handles.append(block.register_forward_hook(hook))
    return ys, dxs, handles


@pytest.mark.gpu
@pytest.mark.parametrize("path", ["small", "big"])
def test_zero_w2_leaves_the_routed_step_bit_for_bit(path):
    """with W2 of the shared expert zeroed its term is exactly 0: one eager step equals the same step without a shared
    expert in the loss, every layer's y and dx, the routed experts and the other trainer parameters"""
    torch.manual_seed(2)
    x, y = torch.randn(256, 784, device="cuda"), torch.randint(0, 10, (256,), device="cuda")
    out, start = {}, None
    # one trainer at a time: the device step counters (and with them the failure draws) are process-wide
    for name, width in (("plain", 0), ("shared", gated_inner_dim(512))):
        t = DMoETrainer(_bench_cfg(shared_inner_dim=width, expert_path=path, failure_rate=0.1), use_graph=False)
        if start is None:
            start = {n: p.detach().clone() for n, p in t.model.named_parameters()}
        else:
            own = dict(t.model.named_parameters())
            with torch.no_grad():
                for n, p in start.items():
                    own[n].copy_(p)
                for block in t.model.blocks:
                    block.shared_w2.zero_()
        ys_, dxs, handles = _record(t.model)
        loss = t.train_step_device(x, y).clone()
        torch.cuda.synchronize()
        t.ctx.check_status()
        for h in handles:
            h.remove()
        params = {n: p.detach().cpu().clone() for n, p in t.model.named_parameters() if n not in _shared_params(t.model)}
        out[name] = (loss.cpu(), [v.cpu() for v in ys_], [v.cpu() for v in dxs],
                     torch.cat([b.shard.p for b in t.model.blocks]).cpu(), params)
        if name == "shared":   # the shared W2 itself got a gradient and was stepped
            assert all(float(b.shared_w2.abs().max()) > 0 for b in t.model.blocks)
        t.close()
    (l0, y0, d0, e0, p0), (l1, y1, d1, e1, p1) = out["plain"], out["shared"]
    assert torch.equal(l0, l1)
    assert len(y0) == len(y1) == 4 and all(torch.equal(a, b) for a, b in zip(y0, y1))
    assert len(d0) == len(d1) == 4 and all(torch.equal(a, b) for a, b in zip(d0, d1))
    assert torch.equal(e0, e1)
    assert p0.keys() == p1.keys() and all(torch.equal(p0[n], p1[n]) for n in p0)
