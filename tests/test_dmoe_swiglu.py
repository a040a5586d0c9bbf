"""SwiGLU experts (GatedFeedforwardBlock) in the fused DMoE engine: DMoEConfig(expert="swiglu").

CPU: the configuration, the engine's fp32 oracle against real GatedFeedforwardBlock modules (parallel/baseline.py),
checkpoints interchangeable with the module + torch Adam, a CPU trainer that learns and resumes.
GPU: the grouped RMSNorm kernels against a float64 oracle, one layer on both expert paths against the oracle, the trainer
under its CUDA graph, a trained expert served by ExpertBackend, and (with two GPUs) the sharded step."""
import os
import subprocess
import sys

import pytest
import torch

import lah_b200 as lib
from lah_b200.models import GatedFeedforwardBlock
from lah_b200.models.layers import GATED_LAYOUT, gated_inner_dim
from lah_b200.ops import kernels as K
from lah_b200.parallel import baseline, engine as E
from lah_b200.parallel.trainer import DMoETrainer

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BF16 = torch.bfloat16
# the bench operating point: 64 experts, top-4, 256 samples per step, 4 layers, emulator gate
BENCH = dict(grid_size=(64,), k=4, num_layers=4, tokens_per_rank=256, gate_mode="emulator")


# ======================================================================================================== CPU
def test_inner_width_defaults_and_override():
    assert E.DMoEConfig(hidden=512).inner == 2048
    assert E.DMoEConfig(hidden=512, expert="swiglu").inner == gated_inner_dim(512) == 1408
    assert E.DMoEConfig(hidden=1024, expert="swiglu").inner == 2816
    assert E.DMoEConfig(hidden=1024, expert="swiglu", inner_dim=512).inner == 512
    assert E.DMoEConfig(hidden=64, expert="swiglu").seg_shapes() == {"g": (64,), "w13": (2 * 256, 64), "w2": (64, 256)}


@pytest.mark.parametrize("kw", [dict(expert="ffn", inner_dim=1024), dict(expert="swiglu", expert_dtype="fp8"),
                                dict(expert="moe"), dict(expert="swiglu", inner_dim=-128)])
def test_config_refusals(kw):
    with pytest.raises(ValueError):
        E.DMoEConfig(hidden=512, **kw)


@pytest.mark.parametrize("hidden,inner", [(96, 0), (4224, 128), (512, 200), (64, 128)])
def test_gpu_sizes_refused_and_cpu_oracle_takes_any_size(hidden, inner):
    cfg = E.DMoEConfig(hidden=hidden, expert="swiglu", inner_dim=inner, grid_size=(2,), k=1, num_layers=1,
                       tokens_per_rank=4)
    with pytest.raises(ValueError, match="multiple of 128"):
        cfg.check_native_sizes()
    if hidden <= 512:   # the oracle runs it
        assert E.FusedDMoE(cfg)(torch.randn(3, hidden)).shape == (3, hidden)


def test_resolved_path():
    assert E.DMoEConfig(hidden=1024, expert="swiglu", **BENCH).resolved_path() == "small"
    assert E.DMoEConfig(hidden=512, expert="swiglu", **BENCH).resolved_path() == "small"
    big = dict(BENCH, tokens_per_rank=65536)
    assert E.DMoEConfig(hidden=1024, expert="swiglu", **big).resolved_path() == "big"
    # a width that is not a multiple of 128 cannot stream through the swap-AB kernels
    assert E.DMoEConfig(hidden=1024, expert="swiglu", inner_dim=200, **BENCH).resolved_path() == "big"


def test_layout_splits_and_joins_w13_by_rows():
    H, I = 8, 16
    seg = {"g": torch.randn(H), "w13": torch.randn(2 * I, H), "w2": torch.randn(H, I)}
    state = GATED_LAYOUT.module_state(seg)
    assert list(state) == ["norm.weight", "w1.weight", "w2.weight", "w3.weight"]
    assert list(state) == list(dict(GatedFeedforwardBlock(H, I).named_parameters()))
    assert torch.equal(state["w1.weight"], seg["w13"][:I]) and torch.equal(state["w3.weight"], seg["w13"][I:])
    back = GATED_LAYOUT.segment_state(state)
    assert all(torch.equal(back[n], seg[n]) for n in seg)
    assert GATED_LAYOUT.small_mask == 0b001


def _cfg(**kw):
    base = dict(hidden=32, grid_size=(2, 4), k=3, num_layers=1, tokens_per_rank=16, expert="swiglu", inner_dim=48)
    base.update(kw)
    return E.DMoEConfig(**base)


def test_cpu_oracle_matches_gated_modules_forward_backward_and_one_step():
    torch.manual_seed(0)
    cfg = _cfg(lr=1e-2)
    fused = E.FusedDMoE(cfg).train()
    base = baseline.BaselineDMoE(cfg)
    assert isinstance(base.experts[0], GatedFeedforwardBlock)
    base.load_from_shard(fused.shard)
    base.proj.load_state_dict(fused.proj.state_dict())
    x = torch.randn(12, 32, requires_grad=True)
    x2 = x.detach().clone().requires_grad_(True)
    gy = torch.randn(12, 32)
    y1, y2 = fused(x), base(x2)
    torch.testing.assert_close(y1, y2, atol=1e-5, rtol=1e-5)
    (y1 * gy).sum().backward()
    (y2 * gy).sum().backward()
    torch.testing.assert_close(x.grad, x2.grad, atol=1e-5, rtol=1e-5)
    torch.testing.assert_close(fused.proj.weight.grad, base.proj.weight.grad, atol=1e-5, rtol=1e-5)
    fused.apply_expert_gradients_ref()
    base.apply_expert_gradients()
    for le, expert in enumerate(base.experts):
        got = fused.shard.expert_state_dict(le, prefix="")
        for k, v in expert.state_dict().items():
            torch.testing.assert_close(got[k], v, atol=1e-6, rtol=1e-5)
    assert int((fused.shard.step > 0).sum()) == int((base._rows > 0).sum()) > 0


def _expert_loss(cfg, layer, module, x, gy, e):
    """the part of <layer(x), gy> that flows through expert e, computed with `module` as that expert"""
    logits = layer.gate_logits(x, layer.proj)
    idx, _ = K.gate_topk_ref(logits, cfg.grid_size, cfg.k)
    w = torch.softmax(torch.gather(K.product_key_scores(logits, cfg.grid_size), 1, idx), -1)
    tok, slot = torch.nonzero(idx == e, as_tuple=True)
    return (module(x[tok]) * gy[tok]).sum(-1).mul(w[tok, slot].detach()).sum(), len(tok)


def test_checkpoint_loads_into_module_and_adam_and_back():
    torch.manual_seed(1)
    cfg = _cfg(grid_size=(4,), k=2, num_layers=1, in_features=12, tokens_per_rank=32, lr=1e-2)
    tr = DMoETrainer(cfg)
    x, y = torch.randn(32, 12), torch.randint(0, 10, (32,))
    for _ in range(3):
        tr.train_step(x, y)
    state = tr.state_dict()
    layer = tr.model.blocks[0]
    e = int(torch.argmax(layer.shard.step))
    entry = state["experts"]["layer0." + E.expert_uid(cfg, e)]
    module = GatedFeedforwardBlock(cfg.hidden, cfg.inner)
    module.load_state_dict({k[len("expert."):]: v for k, v in entry["model"].items()}, strict=True)
    opt = torch.optim.Adam(module.parameters(), lr=cfg.lr, betas=cfg.betas, eps=cfg.eps, amsgrad=True)
    opt.load_state_dict(entry["optimizer"])
    assert float(opt.state_dict()["state"][3]["step"]) == int(layer.shard.step[e])
    # one more step on the same rows: the module + torch Adam, and the engine's CPU path
    h = tr.model.stem(x).detach()
    gy = torch.randn(32, cfg.hidden)
    loss, rows = _expert_loss(cfg, layer, module, h, gy, e)
    assert rows > 0
    opt.zero_grad()
    loss.backward()
    opt.step()
    out = layer(h)
    (out * gy).sum().backward()
    layer.apply_expert_gradients_ref()
    got = layer.shard.expert_state_dict(e, prefix="")
    for k, v in module.state_dict().items():
        torch.testing.assert_close(got[k], v, atol=2e-6, rtol=1e-5)
    # and back: the module and its optimizer load into another engine
    other = DMoETrainer(cfg)
    other.model.blocks[0].shard.load_expert_state_dict(e, {"expert." + k: v for k, v in module.state_dict().items()})
    other.model.blocks[0].shard.load_expert_optimizer_state(e, opt.state_dict())
    back = other.model.blocks[0].shard
    for k, v in module.state_dict().items():
        assert torch.equal(back.expert_state_dict(e, prefix="")[k], v)
    ost = back.expert_optimizer_state(e)["state"]
    for i, p in enumerate(module.parameters()):
        for name in ("exp_avg", "exp_avg_sq", "max_exp_avg_sq"):
            assert torch.equal(ost[i][name], opt.state[p][name])


@pytest.mark.parametrize("update_every_steps", [0, 2])
def test_cpu_trainer_learns_and_resumes(update_every_steps):
    torch.manual_seed(0)
    cfg = E.DMoEConfig(hidden=32, grid_size=(2, 2), k=2, num_layers=2, in_features=12, tokens_per_rank=32, lr=3e-3,
                       expert="swiglu", inner_dim=64, update_every_steps=update_every_steps)
    trainer = DMoETrainer(cfg)
    x, y = torch.randn(32, 12), torch.randint(0, 10, (32,))
    losses = [trainer.train_step(x, y) for _ in range(25)]
    assert losses[-1] < 0.5 * losses[0]
    state = trainer.state_dict()
    assert "expert.norm.weight" in state["experts"]["layer0.expert.0.1"]["model"]
    clone = DMoETrainer(cfg)
    clone.load_state_dict(state)
    for _ in range(3):
        assert abs(trainer.train_step(x, y) - clone.train_step(x, y)) < 1e-5
    for b1, b2 in zip(trainer.model.blocks, clone.model.blocks):
        torch.testing.assert_close(b1.shard.p, b2.shard.p, atol=1e-6, rtol=0)


# ======================================================================================================== GPU
def _tile_table(counts, tile_rows, tiles, empty_tail=2):
    """tile_group of groups with `counts` rows padded to tile_rows (empty groups take no tile), then -1 tiles"""
    table = []
    for g, n in enumerate(counts):
        table += [g] * (-(-n // tile_rows))
    table += [-1] * (tiles - len(table))
    return torch.tensor(table, dtype=torch.int32)


@pytest.mark.gpu
@pytest.mark.parametrize("tile_rows", [16, 128])
@pytest.mark.parametrize("C", [128, 384, 512, 1024, 1408, 4096])
def test_grouped_rms_norm_kernels_against_float64(C, tile_rows):
    torch.manual_seed(C + tile_rows)
    counts = [3 * tile_rows, 0, tile_rows, 2 * tile_rows, 0]   # empty groups; -1 tiles at the end and in the middle
    G = len(counts)
    tiles = sum(-(-n // tile_rows) for n in counts) + 3
    tg = _tile_table(counts, tile_rows, tiles)
    tg = torch.cat([tg[:2], torch.tensor([-1], dtype=torch.int32), tg[2:-1]])   # a -1 tile between two used ones
    rows = tiles * tile_rows
    tgc = tg.cuda()
    x = torch.randn(rows, C, device="cuda").to(BF16)
    gamma = (1 + 0.3 * torch.randn(G, C, device="cuda")).contiguous()
    n = torch.full((rows, C), 7.0, device="cuda", dtype=BF16)
    rstd = torch.zeros(rows, device="cuda")
    K.rms_norm_fwd(x, gamma, 1e-6, out=n, rstd=rstd, tile_group=tgc, tile_rows=tile_rows)
    n_ref, rstd_ref = K.rms_norm_grouped_fwd_ref(x.double(), gamma.double(), 1e-6, tg, tile_rows)
    live = K._tile_rows_of(tg, tile_rows, rows).cuda() >= 0
    assert (n.double()[live] - n_ref[live]).abs().max() <= 2 ** -7 * n_ref[live].abs().max()
    assert torch.allclose(rstd.double()[live], rstd_ref[live], rtol=1e-5)
    assert bool((n[~live] == 7.0).all())   # rows of -1 tiles are not written
    dn = torch.randn(rows, C, device="cuda").to(BF16)
    dres = torch.randn(rows, C, device="cuda").to(BF16)
    dx = torch.full((rows, C), 7.0, device="cuda", dtype=BF16)
    dgs = []
    for _ in range(2):
        dg = torch.zeros(G, C, device="cuda")
        K.rms_norm_bwd(dn, x, rstd, gamma, dx=dx, dgamma=dg, dres=dres, tile_rows=tile_rows, tile_group=tgc)
        dgs.append(dg)
    assert torch.equal(dgs[0], dgs[1])   # fixed summation order
    dx_ref, dg_ref = K.rms_norm_grouped_bwd_ref(dn.double(), x.double(), gamma.double(), 1e-6, tg, tile_rows,
                                                dres=dres.double())
    scale = dx_ref[live].abs().max()
    assert (dx.double()[live] - dx_ref[live]).abs().max() <= 2 ** -6 * scale
    assert bool((dx[~live] == 7.0).all())
    assert (dgs[0].double() - dg_ref).abs().max() <= 1e-4 * dg_ref.abs().max()
    empty = [g for g, c in enumerate(counts) if c == 0]
    assert bool((dgs[0][empty] == 0).all())


@pytest.mark.gpu
def test_rms_norm_without_tile_group_is_unchanged():
    torch.manual_seed(0)
    x = torch.randn(80, 1024, device="cuda").to(BF16)
    gamma = torch.randn(1024, device="cuda")
    outs = []
    for kw in ({}, dict(tile_group=None)):
        n, rstd = torch.empty_like(x), torch.empty(80, device="cuda")
        K.rms_norm_fwd(x, gamma, 1e-6, out=n, rstd=rstd, **kw)
        dx, dg = torch.empty_like(x), torch.zeros(1024, device="cuda")
        K.rms_norm_bwd(x, x, rstd, gamma, dx=dx, dgamma=dg, dres=x, **kw)
        outs.append((n, rstd, dx, dg))
    assert all(torch.equal(a, b) for a, b in zip(*outs))


def _rel(a, b):
    a, b = a.detach().float(), b.detach().float()
    return float((a - b).norm() / b.norm().clamp_min(1e-12))


@pytest.mark.gpu
@pytest.mark.parametrize("path", ["small", "big"])
@pytest.mark.parametrize("hidden", [512, 1024])
def test_layer_against_the_bf16_oracle(hidden, path):
    """one layer, 16 experts, k = 4: forward, backward and the AMSGrad step against the CPU oracle path on the GPU
    (fp32 maths rounded to bf16 where the GPU path stores bf16), with the tolerances of tools/gpu_layer_check.py"""
    torch.manual_seed(3)
    cfg = E.DMoEConfig(hidden=hidden, grid_size=(4, 4), k=4, num_layers=1, tokens_per_rank=512, lr=1e-3,
                       expert="swiglu", expert_path=path)
    ctx = E.EngineContext(cfg)
    try:
        layer = E.FusedDMoE(cfg, ctx).cuda()
        assert ctx.small == (path == "small")
        oracle = E.FusedDMoE(cfg, device=torch.device("cuda")).cuda().train()
        oracle.ref_emulate_bf16 = True
        oracle.proj.load_state_dict(layer.proj.state_dict())
        before = {n: layer.shard.views[n][:16].detach().clone() for n in GATED_LAYOUT.names}
        with torch.no_grad():
            oracle.shard.p.copy_(layer.shard.p[:oracle.shard.p.numel()])
        B = 512
        x = torch.randn(B, hidden, device="cuda").to(BF16).requires_grad_(True)
        gy = torch.randn(B, hidden, device="cuda").to(BF16)
        y = layer(x)
        y.backward(gy)
        torch.cuda.synchronize()
        ctx.check_status()
        xr = x.detach().float().requires_grad_(True)
        yr = oracle(xr)
        yr.backward(gy.float())
        grads = {n: torch.stack([oracle._ref_leaves[e][n].grad if e in oracle._ref_leaves and
                                 oracle._ref_leaves[e][n].grad is not None else torch.zeros_like(before[n][e])
                                 for e in range(16)]) for n in GATED_LAYOUT.names}
        oracle.apply_expert_gradients_ref()
        errs = dict(y=_rel(y, yr), dx=_rel(x.grad, xr.grad), dproj=_rel(layer.proj.weight.grad, oracle.proj.weight.grad))
        perr = {n: float((layer.shard.views[n][:16] - oracle.shard.views[n][:16]).abs().mean()) for n in before}
        werr = {n: _rel(layer.shard.m_views[n][:16] / (1 - cfg.betas[0]), grads[n]) for n in before}
        moved = {n: float((layer.shard.views[n][:16] - before[n]).abs().mean()) for n in before}
        assert errs["y"] < 2e-2 and errs["dx"] < 3e-2 and errs["dproj"] < 5e-2, errs
        assert max(perr.values()) < 1e-4, perr
        assert max(werr.values()) < 8e-2, werr
        assert min(moved.values()) > 1e-4, moved   # every segment was stepped
        assert int(layer.shard.step.sum()) == int(oracle.shard.step.sum()) > 0
    finally:
        ctx.close()


def _trainer_cfg(path, **kw):
    base = dict(hidden=512, grid_size=(16,), k=4, num_layers=2, tokens_per_rank=256, gate_mode="emulator",
                failure_rate=0.1, lr=1e-4, expert_path=path, expert="swiglu")
    base.update(kw)
    return E.DMoEConfig(**base)


@pytest.mark.gpu
@pytest.mark.parametrize("path", ["small", "big"])
def test_graph_step_equals_eager_step_and_runs_are_reproducible(path):
    from lah_b200.ops import native
    cfg = _trainer_cfg(path)
    torch.manual_seed(0)
    xs = [torch.randn(256, cfg.in_features, device="cuda") for _ in range(6)]
    ys = [torch.randint(0, 10, (256,), device="cuda") for _ in range(6)]
    losses, params = {}, {}
    for run, graph in (("eager", False), ("graph", True), ("graph2", True)):
        t = DMoETrainer(cfg, use_graph=graph)
        assert t.ctx.small == (path == "small")
        losses[run] = [float(t.train_step_device(x, y)) for x, y in zip(xs, ys)]
        if graph:
            assert t._graph is not None and native.launches() > 0
        t.ctx.check_status()
        params[run] = torch.cat([b.shard.p for b in t.model.blocks]).cpu()
        assert int(t.model.blocks[0].shard.step.max()) == 6
        t.close()
    for a, b in zip(losses["eager"], losses["graph"]):
        assert abs(a - b) < 5e-3 * max(1.0, abs(a)), losses
    assert torch.equal(params["graph"], params["graph2"])   # same seed, same bytes


@pytest.mark.gpu
def test_set_lr_under_the_graph_equals_eager_steps():
    cfg = _trainer_cfg("small", failure_rate=0.0, lr=1e-3)
    torch.manual_seed(1)
    xs = [torch.randn(256, cfg.in_features, device="cuda") for _ in range(6)]
    ys = [torch.randint(0, 10, (256,), device="cuda") for _ in range(6)]
    rates = [1e-3, 1e-3, 1e-3, 5e-4, 2e-4, 1e-4]
    losses = {}
    for graph in (False, True):
        t = DMoETrainer(cfg, use_graph=graph)
        out = []
        for lr, x, y in zip(rates, xs, ys):
            t.set_lr(lr)
            out.append(float(t.train_step_device(x, y)))
        losses[graph] = out
        t.ctx.check_status()
        t.close()
    for a, b in zip(losses[False], losses[True]):
        assert abs(a - b) < 5e-3 * max(1.0, abs(a)), losses


@pytest.mark.gpu
def test_update_every_steps_fires_on_the_schedule():
    cfg = E.DMoEConfig(hidden=512, grid_size=(4, 4), k=4, num_layers=1, tokens_per_rank=256, update_every_inputs=10 ** 6,
                       update_every_steps=3, expert="swiglu")
    t = DMoETrainer(cfg)
    x, y = torch.randn(256, cfg.in_features, device="cuda"), torch.randint(0, 10, (256,), device="cuda")
    steps, g_before = [], []
    for _ in range(7):
        t.train_step_device(x, y)
        steps.append(int(t.model.blocks[0].shard.step.max()))
        g_before.append(float(t.model.blocks[0].shard.grads["g"].abs().sum()))
    t.ctx.check_status()
    assert steps == [0, 0, 1, 1, 1, 2, 2], steps
    # the norm gradient piles up until the expert fires and is zeroed then
    assert 0 < g_before[0] < g_before[1] and g_before[2] == 0
    t.close()


@pytest.mark.gpu
def test_trained_expert_served_by_expert_backend():
    """a GPU-trained expert's checkpoint in ExpertBackend(GatedFeedforwardBlock), which runs NativeGatedFFNExecutor,
    returns what the engine's expert returns on the same rows"""
    from lah_b200.runtime.native_executor import NativeGatedFFNExecutor
    cfg = _trainer_cfg("small", failure_rate=0.0, lr=1e-3, hidden=1024, num_layers=1)
    t = DMoETrainer(cfg)
    torch.manual_seed(2)
    for _ in range(3):
        t.train_step_device(torch.randn(256, cfg.in_features, device="cuda"), torch.randint(0, 10, (256,), device="cuda"))
    state = t.state_dict()
    layer = t.model.blocks[0]
    e = 5
    entry = state["experts"]["layer0." + E.expert_uid(cfg, e)]
    block = GatedFeedforwardBlock(cfg.hidden, cfg.inner).cuda()
    opt = torch.optim.Adam(block.parameters(), lr=cfg.lr, amsgrad=True)
    backend = lib.ExpertBackend(name="e", expert=block, opt=opt, args_schema=(lib.BatchTensorProto(cfg.hidden),),
                                outputs_schema=lib.BatchTensorProto(cfg.hidden), max_batch_size=64)
    backend.load_state_dict(entry["model"])
    opt.load_state_dict(entry["optimizer"])
    assert NativeGatedFFNExecutor.supports(block, opt)
    rows = torch.randn(40, cfg.hidden, device="cuda").to(BF16).float()
    served = backend.forward(rows)[0]
    p = {n: v.cuda() for n, v in GATED_LAYOUT.segment_state(entry["model"], prefix="expert.").items()}
    ref = layer._expert_ref(p, rows, lambda v: v.to(BF16).float())
    assert _rel(served, ref) < 2e-2
    t.close()


@pytest.mark.gpu
def test_two_gpus_sharded_step_with_shadow_slots_matches_one_gpu():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    out = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2",
                          "--master-addr", "127.0.0.1", "--master-port", "29547",
                          os.path.join(ROOT, "tools", "multi_gpu_check.py"), "--swiglu", "--force-shadow"],
                         capture_output=True, text=True, timeout=600)
    assert out.returncode == 0 and "MULTI_GPU_OK" in out.stdout, out.stdout[-3000:] + out.stderr[-3000:]
