"""
Learning-rate schedules on DMoETrainer: ``set_lr`` / ``cfg.lr`` take effect from the next step on the CPU path, in eager GPU
steps and in the replayed CUDA graph, because every optimizer kernel reads the rate from a device block
(``EngineContext.lr_dev``) that the host refreshes between steps.

The kernels are compared with their by-value launches bit for bit (``lr_dev`` holding x == ``lr=x``).  The trainer is
compared with itself: graph == eager under a rate that changes every step, a rate change == a restart from a checkpoint
at the new rate, lr = 0 freezes every parameter while the moments move, and a resumed run == the continued one.
"""
import math

import pytest
import torch

from test_expert_kernels import adam_state, poison  # noqa: F401
from test_fused_adam_fp8_kernels import WA_ADAM_ROWS, WA_ADAM_STEPS, wa_adam_setup

import lah_b200  # noqa: F401
from lah_b200.ops import kernels as K
from lah_b200.parallel import engine as E
from lah_b200.parallel.trainer import DMoETrainer


def snapshot(tr):
    """every optimizer-owned tensor of a trainer, on the CPU: trainer p / m / v / vmax, per layer the expert p, the bf16
    mirror, m, v, vmax and the step counters"""
    out = {f"trainer.{n}": t.detach().cpu().clone() for n, t in
           (("p", tr.flat_p), ("m", tr.flat_m), ("v", tr.flat_v), ("vmax", tr.flat_vmax))}
    for i, block in enumerate(tr.model.blocks):
        for n in ("p", "p_bf16", "m", "v", "vmax", "step"):
            t = getattr(block.shard, n)
            if t is not None:
                out[f"layer{i}.{n}"] = t.detach().cpu().clone()
    return out


def assert_same(a, b, what):
    assert a.keys() == b.keys()
    bad = [k for k in a if not torch.equal(a[k], b[k])]
    assert not bad, f"{what}: not bit-identical: {bad}"


def schedule(step, base=2e-3, warmup=4, total=10):
    """linear warm-up over `warmup` steps, then cosine decay: a different rate at every step"""
    if step < warmup:
        return base * (step + 1) / warmup
    return base * 0.5 * (1.0 + math.cos(math.pi * (step - warmup) / (total - warmup)))


def without_lr(state):
    """a checkpoint as written before the trainer stored its learning rate"""
    state = dict(state)
    state["trainer"] = {k: v for k, v in state["trainer"].items() if k != "lr"}
    return state


# ---------------------------------------------------------------------------------------------------------------- CPU
def cpu_cfg(**kw):
    return E.DMoEConfig(hidden=32, grid_size=(2, 2), k=2, num_layers=2, in_features=12, tokens_per_rank=32, lr=3e-3, **kw)


def cpu_data(steps):
    gen = torch.Generator().manual_seed(11)
    return [(torch.randn(32, 12, generator=gen), torch.randint(0, 10, (32,), generator=gen)) for _ in range(steps)]


def test_set_lr_to_the_current_rate_changes_nothing():
    data = cpu_data(4)
    runs = []
    for call in (False, True):
        torch.manual_seed(0)
        tr = DMoETrainer(cpu_cfg())
        losses = []
        for x, y in data:
            if call:
                tr.set_lr(tr.cfg.lr)
            losses.append(tr.train_step(x, y))
        runs.append((losses, snapshot(tr)))
    assert runs[0][0] == runs[1][0]
    assert_same(runs[0][1], runs[1][1], "set_lr(cfg.lr) before every step")


@pytest.mark.parametrize("decoupled", [False, True])
def test_rate_change_equals_restart_at_the_new_rate(decoupled):
    """k steps at a, set_lr(b), k steps == k steps at a, checkpoint, a trainer built with lr=b loads it, k steps"""
    a, b, k = 3e-3, 7e-4, 3
    data = cpu_data(2 * k)
    kw = dict(weight_decay=0.1, decoupled_weight_decay=True) if decoupled else {}
    torch.manual_seed(0)
    run_a = DMoETrainer(cpu_cfg(**kw))
    for x, y in data[:k]:
        run_a.train_step(x, y)
    state = run_a.state_dict()
    run_a.set_lr(b)
    losses_a = [run_a.train_step(x, y) for x, y in data[k:]]
    cfg_b = cpu_cfg(**kw)
    cfg_b.lr = b
    torch.manual_seed(0)
    run_b = DMoETrainer(cfg_b)
    run_b.load_state_dict(without_lr(state))
    assert run_b.lr == b
    losses_b = [run_b.train_step(x, y) for x, y in data[k:]]
    assert losses_a == losses_b
    assert_same(snapshot(run_a), snapshot(run_b), "rate change vs restart")


@pytest.mark.parametrize("decoupled", [False, True])
def test_zero_rate_freezes_parameters_while_the_moments_move(decoupled):
    kw = dict(weight_decay=0.5, decoupled_weight_decay=True) if decoupled else {}
    data = cpu_data(5)
    tr = DMoETrainer(cpu_cfg(**kw))
    for x, y in data[:2]:
        tr.train_step(x, y)
    tr.set_lr(0.0)
    before = snapshot(tr)
    for x, y in data[2:]:
        tr.train_step(x, y)
    after = snapshot(tr)
    for n in ("trainer.p", "layer0.p", "layer0.p_bf16", "layer1.p", "layer1.p_bf16"):
        assert torch.equal(before[n], after[n]), f"{n} moved at lr = 0"
    for n in ("trainer.m", "layer0.m", "layer1.m"):
        assert not torch.equal(before[n], after[n]), f"{n} did not move"


@pytest.mark.parametrize("bad", [-1e-3, float("nan"), float("inf")])
def test_set_lr_refuses_negative_and_non_finite_rates(bad):
    tr = DMoETrainer(cpu_cfg())
    with pytest.raises(ValueError):
        tr.set_lr(bad)
    assert tr.lr == 3e-3


def test_checkpoint_carries_the_rate():
    tr = DMoETrainer(cpu_cfg())
    x, y = cpu_data(1)[0]
    tr.train_step(x, y)
    tr.set_lr(1.25e-4)
    state = tr.state_dict()
    assert set(state) == {"trainer", "experts", "rng", "token_base"}
    assert state["trainer"]["lr"] == 1.25e-4
    # the exported expert optimizer states report the current rate, so they load into a torch Adam at that rate
    groups = [e["optimizer"]["param_groups"][0]["lr"] for e in state["experts"].values()]
    assert groups and all(g == 1.25e-4 for g in groups)
    fresh = DMoETrainer(cpu_cfg())
    fresh.load_state_dict(state)
    assert fresh.lr == fresh.cfg.lr == 1.25e-4
    old = DMoETrainer(cpu_cfg())
    old.load_state_dict(without_lr(state))
    assert old.lr == 3e-3
    fresh.train_step(x, y), old.train_step(x, y)
    assert not torch.equal(snapshot(fresh)["layer0.p"], snapshot(old)["layer0.p"])


# ---------------------------------------------------------------------------------------------------------------- GPU
WD_MODES = {"none": dict(weight_decay=0.0, decoupled=False), "l2": dict(weight_decay=0.1, decoupled=False),
            "decoupled": dict(weight_decay=0.3, decoupled=True)}
SEGS = [4, 8, 12, 36, 4, 100, 8, 64, 20, 4]


def lr_block(lr, weight_decay, decoupled):
    return torch.tensor(K.lr_block_values(lr, weight_decay, decoupled), dtype=torch.float32, device="cuda")


@pytest.mark.gpu
@pytest.mark.parametrize("lr", [3.7e-3, 0.0])
@pytest.mark.parametrize("seg_mask", [0, E.SMALL_SEG_MASK])
@pytest.mark.parametrize("amsgrad", [True, False])
@pytest.mark.parametrize("mode", list(WD_MODES))
def test_adam_step_device_rate_equals_by_value(mode, amsgrad, seg_mask, lr, poison):
    """the device-rate launch gets a wrong by-value lr on purpose: the rate must come from the block"""
    G = 5
    rows = torch.tensor([3, 0, 1, 0, 2], dtype=torch.int32, device="cuda")   # groups 1 and 3 receive no rows
    step = torch.tensor([1, 4, 2, 9, 3], dtype=torch.int32, device="cuda")
    st = adam_state(7, SEGS, G)
    wd = WD_MODES[mode]
    out = []
    for dev in (False, True):
        t = {k: x.clone() for k, x in st.items()}
        kw = dict(lr_dev=lr_block(lr, **wd), lr=0.5) if dev else dict(lr=lr)
        K.adam_step(t["p"], t["g"], t["m"], t["v"], t["vmax"], t["p_bf16"], SEGS, G, step=step, group_rows=rows,
                    amsgrad=amsgrad, zero_mask=0xFF, seg_mask=seg_mask, **wd, **kw)
        out.append(t)
    torch.cuda.synchronize()
    for n in ("p", "g", "m", "v", "vmax", "p_bf16"):
        assert torch.equal(out[0][n], out[1][n]), n
    assert not torch.equal(out[1]["m"], st["m"])


@pytest.mark.gpu
@pytest.mark.parametrize("max_ctas", [80, 0])
@pytest.mark.parametrize("amsgrad", [True, False])
@pytest.mark.parametrize("mode", list(WD_MODES))
def test_wgrad_adam_device_rate_equals_by_value(mode, amsgrad, max_ctas, poison):
    """groups of 0 rows (and a skipped group) included: WA_ADAM_ROWS; lr = 0 as well (AdamW's factor is then exactly 1)"""
    assert 0 in WA_ADAM_ROWS
    N, K_ = 256, 384
    dy, x, go, gr, skip, _, _, st, _ = wa_adam_setup(31, N, K_)
    step = torch.tensor(WA_ADAM_STEPS, dtype=torch.int32, device="cuda")
    wd = WD_MODES[mode]
    for lr in (2.3e-3, 0.0):
        out = []
        for dev in (False, True):
            t = {k: (v.clone() if v is not None else None) for k, v in st.items()}
            kw = dict(lr_dev=lr_block(lr, **wd), lr=0.5) if dev else dict(lr=lr)
            K.wgrad_adam(dy, x, go, gr, p=t["p"], m=t["m"], v=t["v"], vmax=t["vmax"], p_bf16=t["p_bf16"], step=step,
                         skip=skip, amsgrad=amsgrad, max_ctas=max_ctas, **wd, **kw)
            out.append(t)
        torch.cuda.synchronize()
        for n in ("p", "m", "v", "vmax", "p_bf16"):
            assert torch.equal(out[0][n], out[1][n]), (lr, n)
        assert not torch.equal(out[1]["m"], st["m"]), lr


def gpu_cfg(path, **kw):
    tokens = 256 if path == "small" else 1024
    return E.DMoEConfig(hidden=512, grid_size=(16,), k=4, num_layers=2, tokens_per_rank=tokens, expert_path=path,
                        lr=schedule(0), **kw)


def gpu_data(cfg, steps, seed=0):
    gen = torch.Generator().manual_seed(seed)
    protos = torch.randn(10, cfg.in_features, generator=gen)
    out = []
    for _ in range(steps):
        y = torch.randint(0, 10, (cfg.tokens_per_rank,), generator=gen)
        out.append(((protos[y] + 2.0 * torch.randn(cfg.tokens_per_rank, cfg.in_features, generator=gen)).cuda(), y.cuda()))
    return out


def run(tr, data, rates=None, first=0):
    """train on `data`, setting rates[first + i] before step i; returns the losses"""
    losses = []
    for i, (x, y) in enumerate(data):
        if rates is not None:
            tr.set_lr(rates[first + i])
        losses.append(float(tr.train_step_device(x, y)))
    return losses


GPU_VARIANTS = {"plain": {}, "microbatches_2": dict(trainer_microbatches=2),
                "decoupled": dict(weight_decay=0.05, decoupled_weight_decay=True)}
RATES = [schedule(i) for i in range(10)]


@pytest.mark.gpu
@pytest.mark.parametrize("variant", list(GPU_VARIANTS))
@pytest.mark.parametrize("path", ["small", "big"])
def test_graph_replay_follows_the_schedule_like_eager_steps(path, variant):
    cfg_kw = GPU_VARIANTS[variant]
    data = gpu_data(gpu_cfg(path, **cfg_kw), 10)
    res = {}
    for graph in (False, True):
        torch.manual_seed(0)
        tr = DMoETrainer(gpu_cfg(path, **cfg_kw), use_graph=graph)
        assert tr.ctx.small == (path == "small")
        losses = run(tr, data, RATES)
        assert (tr._graph is not None) == graph
        tr.ctx.check_status()
        res[graph] = (losses, snapshot(tr))
        tr.close()
    assert res[False][0] == res[True][0], res
    assert_same(res[False][1], res[True][1], f"{path} {variant}: graph vs eager under a schedule")


@pytest.mark.gpu
@pytest.mark.parametrize("path", ["small", "big"])
def test_rate_change_under_the_graph_equals_restart_at_the_new_rate(path):
    a, b, k = 2e-3, 4e-4, 4
    data = gpu_data(gpu_cfg(path), 2 * k)
    torch.manual_seed(0)
    cfg = gpu_cfg(path)
    cfg.lr = a
    tr = DMoETrainer(cfg)
    run(tr, data[:k])
    assert tr._graph is not None   # the rate changes after the graph was captured
    state = tr.state_dict()
    tr.set_lr(b)
    losses_a = run(tr, data[k:])
    final_a = snapshot(tr)
    tr.close()
    torch.manual_seed(0)
    cfg = gpu_cfg(path)
    cfg.lr = b
    tr = DMoETrainer(cfg)
    tr.load_state_dict(without_lr(state))
    losses_b = run(tr, data[k:])
    final_b = snapshot(tr)
    tr.close()
    assert losses_a == losses_b
    assert_same(final_a, final_b, f"{path}: rate change under the graph vs restart")


@pytest.mark.gpu
@pytest.mark.parametrize("decoupled", [False, True])
@pytest.mark.parametrize("path", ["small", "big"])
def test_zero_rate_under_the_graph_freezes_parameters(path, decoupled):
    kw = dict(weight_decay=0.5, decoupled_weight_decay=True) if decoupled else {}
    data = gpu_data(gpu_cfg(path, **kw), 6)
    tr = DMoETrainer(gpu_cfg(path, **kw))
    run(tr, data[:3])
    assert tr._graph is not None
    tr.set_lr(0.0)
    before = snapshot(tr)
    run(tr, data[3:])
    after = snapshot(tr)
    tr.ctx.check_status()
    tr.close()
    for n in ("trainer.p", "layer0.p", "layer0.p_bf16", "layer1.p", "layer1.p_bf16"):
        assert torch.equal(before[n], after[n]), f"{n} moved at lr = 0 (the replay kept the captured rate)"
    for n in ("trainer.m", "layer0.m", "layer1.m"):
        assert not torch.equal(before[n], after[n]), f"{n} did not move"


@pytest.mark.gpu
@pytest.mark.parametrize("path", ["small", "big"])
def test_resume_under_a_schedule_equals_the_continued_run(path):
    data = gpu_data(gpu_cfg(path), 10)
    torch.manual_seed(0)
    tr = DMoETrainer(gpu_cfg(path))
    run(tr, data[:5], RATES)
    state = tr.state_dict()
    losses_a = run(tr, data[5:], RATES, first=5)
    final_a = snapshot(tr)
    tr.close()
    torch.manual_seed(0)
    tr = DMoETrainer(gpu_cfg(path))
    tr.load_state_dict(state)
    assert tr.lr == RATES[4]
    losses_b = run(tr, data[5:], RATES, first=5)
    final_b = snapshot(tr)
    tr.close()
    assert losses_a == losses_b
    assert_same(final_a, final_b, f"{path}: resumed vs continued under a schedule")


@pytest.mark.gpu
def test_set_lr_and_a_graph_step_do_not_synchronise():
    cfg = gpu_cfg("small")
    data = gpu_data(cfg, 4)
    tr = DMoETrainer(cfg)
    run(tr, data[:3], RATES)
    assert tr._graph is not None
    x, y = data[3]
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        tr.set_lr(RATES[3])
        loss = tr.train_step_device(x, y)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert math.isfinite(float(loss))
    assert float(tr.ctx.lr_dev[0]) == torch.tensor(RATES[3], dtype=torch.float32).item()
    tr.close()


@pytest.mark.gpu
def test_layer_driven_directly_follows_cfg_lr():
    """FusedDMoE without DMoETrainer (the in-box GatingFunction path): a step begins at forward()"""
    cfg = E.DMoEConfig(hidden=512, grid_size=(16,), k=4, num_layers=1, tokens_per_rank=256, lr=1e-3)
    ctx = E.EngineContext(cfg)
    layer = E.FusedDMoE(cfg, ctx).cuda()
    assert ctx.small
    gen = torch.Generator().manual_seed(3)
    x = torch.randn(256, 512, generator=gen).cuda()
    g = torch.randn(256, 512, generator=gen).cuda()
    layer(x).backward(g)
    cfg.lr = 0.0
    p, m = layer.shard.p.clone(), layer.shard.m.clone()
    layer(x).backward(g)
    torch.cuda.synchronize()
    assert torch.equal(layer.shard.p, p) and not torch.equal(layer.shard.m, m)
    cfg.lr = 1e-3
    layer(x).backward(g)
    torch.cuda.synchronize()
    assert not torch.equal(layer.shard.p, p)
    ctx.close()
