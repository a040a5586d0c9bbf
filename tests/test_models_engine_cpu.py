"""Emulators, oracle engine, checkpoint layout, baseline path, trainer (CPU)"""
import os
import sys
from functools import partial

import pytest
import torch
import torch.nn.functional as F

import lah_b200 as lib
from lah_b200.models import EmulatedDMoE, EmulatedFaultyDMoE, FeedforwardBlock, get_non_expert_params, name_to_block, name_to_input
from lah_b200.ops import kernels as K
from lah_b200.parallel import baseline, engine as E
from lah_b200.parallel.trainer import DMoETrainer

Optimizer = partial(torch.optim.Adam, lr=1e-3, amsgrad=True)


def test_block_shapes_and_param_counts():
    assert sum(p.numel() for p in FeedforwardBlock(512).parameters()) == 6_304_256      # SURVEY appendix C
    assert sum(p.numel() for p in name_to_block["transformer"](1024).parameters()) == 8_399_872
    assert name_to_input["ffn"](7, 32).shape == (7, 32) and name_to_input["transformer"](2, 32).shape == (2, 512, 32)
    assert list(FeedforwardBlock(8).state_dict()) == [f"layers.{i}.{p}" for i in (0, 1, 3, 4, 6) for p in ("weight", "bias")]


def test_emulated_dmoe_state_layout_and_update_rule():
    torch.manual_seed(0)
    layer = EmulatedDMoE(16, num_experts=8, num_active=2, update_every_inputs=4, update_every_steps=3,
                         Expert=FeedforwardBlock, Optimizer=Optimizer)
    keys = set(layer.state_dict())
    assert {"expert_keys", "expert_inputs_since_update", "expert_steps_since_first_input",
            "gating_pre_normalize.weight", "gating_pre_normalize.bias", "experts.0.layers.0.weight",
            "experts.7.layers.6.bias"} <= keys and len(keys) == 5 + 8 * 10
    x = torch.randn(6, 16)
    out = layer(x)
    # parity with the reference's per-sample formulation
    logits = layer.gating_pre_normalize(x) @ F.normalize(layer.expert_keys, dim=-1)
    ids = torch.argsort(logits, dim=-1, descending=True)[:, :2]
    ref = torch.stack([torch.stack([layer.experts[int(e)](x[i]) for e in ids[i]], -1) @ F.softmax(logits[i][ids[i]], -1)
                       for i in range(6)])
    assert torch.allclose(out, ref, atol=1e-5)
    assert int(layer.expert_inputs_since_update.sum()) == 12
    out.sum().backward()
    before = [e.layers[0].weight.clone() for e in layer.experts]
    due = (layer.expert_inputs_since_update >= 4) | (layer.expert_steps_since_first_input >= 3)
    layer(x)  # triggers maybe_update_experts for the experts that are due
    for i, e in enumerate(layer.experts):
        assert (not torch.equal(before[i], e.layers[0].weight)) == bool(due[i])
    # the emulator's gate is excluded from the trainer's parameters (as in the reference)
    model = torch.nn.Sequential(torch.nn.Linear(4, 16), layer, torch.nn.Linear(16, 2))
    assert len(get_non_expert_params(model)) == 4
    layer.eval()
    counts = layer.expert_inputs_since_update.clone()
    layer(x)
    assert torch.equal(counts, layer.expert_inputs_since_update)


def test_faulty_emulator_masks_and_renormalises():
    torch.manual_seed(0)
    layer = EmulatedFaultyDMoE(16, 8, 4, 4, 10, failure_rate=0.5, Expert=FeedforwardBlock, Optimizer=Optimizer)
    x = torch.randn(64, 16)
    torch.manual_seed(5)
    logits = layer.gating_logits(x)
    frac = torch.isinf(logits).float().mean().item()
    assert 0.35 < frac < 0.65
    out = layer(x)
    assert torch.isfinite(out).all()
    assert len(get_non_expert_params(torch.nn.Sequential(layer), (EmulatedFaultyDMoE,))) == 0


def test_gate_oracle_and_adam_ref():
    logits = torch.randn(9, 7)
    idx, w = K.gate_topk_ref(logits, (3, 4), 3)
    scores = (logits[:, :3, None] + logits[:, None, 3:]).flatten(1)
    assert torch.equal(idx, scores.topk(3, -1).indices) and torch.allclose(w.sum(-1), torch.ones(9))
    alive = torch.zeros(12, dtype=torch.uint8)
    alive[[2, 5]] = 1
    idx, w = K.gate_topk_ref(logits, (3, 4), 3, alive=alive)
    assert set(idx.unique().tolist()) == {-1, 2, 5} and torch.allclose(w.sum(-1), torch.ones(9)) and (w[idx < 0] == 0).all()
    # adam_step_ref == torch.optim.Adam(amsgrad) per group, inactive groups untouched
    G, segs = 3, [8, 4]
    n = sum(segs) * G
    p = torch.randn(n); p0 = p.clone()
    m, v, vmax = torch.zeros(n), torch.zeros(n), torch.zeros(n)
    step = torch.zeros(G, dtype=torch.int32)
    refs = [[p0[0 + g * 8: 8 + g * 8].clone().requires_grad_(), p0[24 + g * 4: 28 + g * 4].clone().requires_grad_()] for g in range(G)]
    opts = [torch.optim.Adam(r, lr=1e-2, amsgrad=True) for r in refs]
    for it in range(3):
        grad = torch.randn(n)
        rows = torch.tensor([1, it % 2, 2])
        step += (rows > 0).int()
        K.adam_step_ref(p, grad.clone(), m, v, vmax, segs, G, step=step, group_rows=rows, lr=1e-2)
        for g in range(G):
            if rows[g] > 0:
                refs[g][0].grad, refs[g][1].grad = grad[g * 8: g * 8 + 8].clone(), grad[24 + g * 4: 28 + g * 4].clone()
                opts[g].step()
    for g in range(G):
        assert torch.allclose(p[g * 8: g * 8 + 8], refs[g][0].detach(), atol=1e-6)
        assert torch.allclose(p[24 + g * 4: 28 + g * 4], refs[g][1].detach(), atol=1e-6)


def test_fused_layer_oracle_matches_baseline_and_checkpoints_are_interchangeable(tmp_path):
    torch.manual_seed(0)
    cfg = E.DMoEConfig(hidden=32, grid_size=(2, 4), k=3, num_layers=1, tokens_per_rank=16)
    fused = E.FusedDMoE(cfg).eval()
    base = baseline.BaselineDMoE(cfg)
    base.load_from_shard(fused.shard)
    base.proj.load_state_dict(fused.proj.state_dict())
    x = torch.randn(10, 32, requires_grad=True)
    x2 = x.detach().clone().requires_grad_(True)
    y1, y2 = fused(x), base(x2)
    assert torch.allclose(y1, y2, atol=1e-5)
    y1.sum().backward(), y2.sum().backward()
    assert torch.allclose(x.grad, x2.grad, atol=1e-5) and torch.allclose(fused.proj.weight.grad, base.proj.weight.grad, atol=1e-5)
    # expert checkpoint: ExpertBackend.state_dict() key names, loadable into a reference-style module + torch Adam
    sd = fused.shard.expert_state_dict(3)
    assert list(sd)[0] == "expert.layers.0.weight"
    block = FeedforwardBlock(32)
    be = lib.ExpertBackend(name="x", expert=block, opt=torch.optim.Adam(block.parameters(), amsgrad=True),
                           args_schema=(lib.BatchTensorProto(32),), outputs_schema=lib.BatchTensorProto(32), max_batch_size=4)
    be.load_state_dict(sd)
    assert torch.equal(block.layers[3].weight, fused.shard.views["w2"][3])
    fused.shard.m.normal_(), fused.shard.v.uniform_(), fused.shard.vmax.uniform_()
    fused.shard.step[3] = 7
    opt_state = fused.shard.expert_optimizer_state(3)
    be.opt.load_state_dict(opt_state)  # torch accepts it
    assert float(be.opt.state_dict()["state"][0]["step"]) == 7.0
    other = E.FusedDMoE(cfg)
    other.shard.load_expert_state_dict(3, sd)
    other.shard.load_expert_optimizer_state(3, opt_state)
    assert torch.equal(other.shard.views["w3"][3], fused.shard.views["w3"][3]) and int(other.shard.step[3]) == 7
    off = other.shard.m_views["w2"][3].storage_offset()   # where expert 3's exp_avg of w2 begins in the flat buffer
    assert off == other.shard.slots * sum(other.shard.seg_sizes[:4]) + 3 * other.shard.seg_sizes[4]
    assert torch.equal(other.shard.m[off: off + 10], fused.shard.m[off: off + 10])
    assert E.expert_uid(cfg, 6) == "expert.1.2"


def test_cpu_trainer_learns_and_checkpoint_roundtrip():
    torch.manual_seed(0)
    cfg = E.DMoEConfig(hidden=32, grid_size=(2, 2), k=2, num_layers=2, in_features=12, tokens_per_rank=32, lr=3e-3)
    trainer = DMoETrainer(cfg)
    x, y = torch.randn(32, 12), torch.randint(0, 10, (32,))
    losses = [trainer.train_step(x, y) for _ in range(25)]
    assert losses[-1] < 0.5 * losses[0]
    assert int(trainer.model.blocks[0].shard.step.max()) == 25
    state = trainer.state_dict()
    assert set(state) == {"trainer", "experts", "rng", "token_base"} and "layer1.expert.1.0" in state["experts"]
    assert float(state["trainer"]["exp_avg"].abs().sum()) > 0   # CPU checkpoints carry the trainer optimizer state
    assert "expert.layers.4.bias" in state["experts"]["layer0.expert.0.1"]["model"]
    clone = DMoETrainer(cfg)
    clone.load_state_dict(state)
    ev1, ev2 = trainer.evaluate(x, y), clone.evaluate(x, y)
    assert abs(ev1["loss"] - ev2["loss"]) < 1e-6 and clone.step_count == 25
    assert abs(trainer.train_step(x, y) - clone.train_step(x, y)) < 1e-5
    # resumed run == continued run for several more steps (optimizer state restored, not just the weights)
    for _ in range(3):
        assert abs(trainer.train_step(x, y) - clone.train_step(x, y)) < 1e-5
    # the returned state is a copy, not an alias of live buffers
    before = state["trainer"]["exp_avg"].clone()
    trainer.train_step(x, y)
    assert torch.equal(before, state["trainer"]["exp_avg"])


def test_failure_injection_on_oracle_path():
    torch.manual_seed(0)
    cfg = E.DMoEConfig(hidden=16, grid_size=(4, 4), k=4, num_layers=1, tokens_per_rank=64, failure_rate=0.5)
    layer = E.FusedDMoE(cfg).train()
    x = torch.randn(64, 16)
    layer.eval()
    clean = layer(x)
    layer.train()
    faulty = layer(x)
    assert torch.isfinite(faulty).all() and not torch.allclose(clean, faulty)


def _gloo_worker(rank, world, port, queue):
    import torch.distributed as dist
    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    cfg = E.DMoEConfig(hidden=16, grid_size=(2, 4), k=2, num_layers=2, in_features=6, tokens_per_rank=8)
    trainer = baseline.BaselineTrainer(cfg)
    gen = torch.Generator().manual_seed(7)  # same data on both ranks -> result must equal a single-process run
    x, y = torch.randn(8, 6, generator=gen), torch.randint(0, 10, (8,), generator=gen)
    losses = [trainer.train_step(x, y) for _ in range(3)]
    queue.put((rank, losses))
    dist.barrier()
    dist.destroy_process_group()


def test_baseline_all_to_all_two_processes_matches_single_process():
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    queue = ctx.Queue()
    procs = [ctx.Process(target=_gloo_worker, args=(r, 2, 29631, queue)) for r in range(2)]
    [p.start() for p in procs]
    results = dict(queue.get(timeout=120) for _ in range(2))
    [p.join(30) for p in procs]
    cfg = E.DMoEConfig(hidden=16, grid_size=(2, 4), k=2, num_layers=2, in_features=6, tokens_per_rank=8)
    single = baseline.BaselineTrainer(cfg)
    gen = torch.Generator().manual_seed(7)
    x, y = torch.randn(8, 6, generator=gen), torch.randint(0, 10, (8,), generator=gen)
    ref = [single.train_step(x, y) for _ in range(3)]
    assert results[0] == pytest.approx(results[1], abs=1e-6)
    # first step is identical; later steps differ only because the sharded experts see rows from both ranks
    assert results[0][0] == pytest.approx(ref[0], abs=1e-5)


def test_mxfp8_reference_quantiser_roundtrip():
    """MXFP8 oracle (ops/fp8.py): power-of-two block scales never saturate E4M3 and the relative error is bounded"""
    from lah_b200.ops import fp8
    torch.manual_seed(0)
    x = torch.randn(64, 256) * torch.logspace(-3, 3, 64).unsqueeze(1)
    x[3] = 0
    q, e = fp8.quantize_ref(x)
    assert q.dtype == torch.float8_e4m3fn and e.shape == (64, 8)
    assert float(q.float().abs().max()) <= 448.0
    back = fp8.dequantize_ref(q, e)
    blk_amax = x.view(64, 8, 32).abs().amax(-1, keepdim=True).expand(64, 8, 32).reshape(64, 256)
    assert bool(((back - x).abs() <= blk_amax * 2 ** -3 + 1e-30).all())   # <= 1/2 ulp of a 3-bit mantissa, block-relative
    assert bool((back[3] == 0).all())
    assert fp8.sf_bytes(2048, 3, 512, fp8.WEIGHT_TILE) == 11 * 4 * 2 * 3 * 512
    assert fp8.sf_bytes(384, 1, 512, fp8.ACT_TILE) == 3 * 4 * 512


def test_metrics_log_and_stage_timer(tmp_path):
    """structured JSONL step metrics (SURVEY 5.5) and the (disabled-by-default) stage timer"""
    import json
    from lah_b200.parallel.profiler import MetricsLog, StageTimer
    from lah_b200.parallel.engine import DMoEConfig
    from lah_b200.parallel.trainer import DMoETrainer
    t = StageTimer(enabled=False)
    t.start(), t.mark("a")
    assert t.report() == {}
    path = tmp_path / "m" / "steps.jsonl"
    cfg = DMoEConfig(hidden=32, grid_size=(2, 2), k=2, num_layers=1, in_features=8, tokens_per_rank=16)
    trainer = DMoETrainer(cfg, device="cpu", metrics_path=str(path))
    x, y = torch.randn(16, 8), torch.randint(0, 10, (16,))
    loss = trainer.train_step(x, y)
    handle = trainer.train_step_async(x, y, prefetch=(x, y))   # same API as on the GPU (there it returns before the step ran)
    assert isinstance(handle.result(), float) and handle.result() == handle.result()
    loss = handle.result()
    rec = trainer.log_step(loss=loss, samples=16, step_ms=2.0, note="cpu")
    assert rec["samples_per_s"] == 8000.0 and rec["step"] == 2
    trainer.metrics.close()
    lines = [json.loads(l) for l in open(path)]
    assert len(lines) == 1 and lines[0]["note"] == "cpu" and abs(lines[0]["loss"] - loss) < 1e-6


def test_shadow_plan_balances_skewed_routing():
    """host model of the kernel's hot-expert selection: never makes the worst rank worse, stops when balanced"""
    from lah_b200.parallel.balance import rank_loads, shadow_plan
    gen = torch.Generator().manual_seed(0)
    world, E, E_loc = 8, 64, 8
    # heavy skew: 4 experts take ~85 % of the rows, tokens are i.i.d. across ranks
    probs = torch.full((E,), 0.15 / (E - 4))
    probs[torch.tensor([3, 17, 18, 60])] = 0.85 / 4
    counts = [torch.multinomial(probs, 20000, replacement=True, generator=gen).bincount(minlength=E).tolist() for _ in range(world)]
    before = rank_loads(counts, E_loc)
    shadowed, after = shadow_plan(counts, E_loc, max_shadow=8, tol=1.1, min_rows=64)
    mean = sum(before) / world
    assert sum(after) == sum(before)
    assert max(before) / mean > 2.5 and max(after) / mean <= 1.1
    assert set(shadowed[:4]) == {3, 17, 18, 60} or set(shadowed) >= {3, 17, 18, 60}
    # balanced routing: nothing is shadowed
    uniform = [[100] * E for _ in range(world)]
    assert shadow_plan(uniform, E_loc, 8)[0] == []
    # single rank: never shadows
    assert shadow_plan([counts[0]], E, 8)[0] == []


def test_dead_experts_are_never_routed_to():
    """liveness table (the in-box DHT): experts of a 'dead rank' disappear from the routing, training continues"""
    from lah_b200.parallel.engine import DMoEConfig
    from lah_b200.parallel.trainer import DMoETrainer
    cfg = DMoEConfig(hidden=32, grid_size=(4, 4), k=4, num_layers=2, in_features=8, tokens_per_rank=64)
    trainer = DMoETrainer(cfg, device="cpu")
    x, y = torch.randn(64, 8), torch.randint(0, 10, (64,))
    trainer.train_step(x, y)
    steps_before = [b.shard.step.clone() for b in trainer.model.blocks]
    trainer.mark_rank_dead(1, world=4)          # experts 4..7 vanish
    for _ in range(3):
        loss = trainer.train_step(x, y)
    assert loss == loss
    for before, block in zip(steps_before, trainer.model.blocks):
        delta = block.shard.step - before
        assert int(delta[4:8].sum()) == 0 and int(delta.sum()) > 0   # dead experts received no rows, hence no optimizer steps


def test_fast_nccl_baseline_formulation_learns_on_cpu():
    """parallel/baseline_fast.py (what `bench.py --impl baseline` measures): fixed-capacity dispatch without host syncs"""
    from lah_b200.parallel.baseline_fast import FastBaselineTrainer
    torch.manual_seed(0)
    for gate in ("emulator", "product_key"):
        cfg = E.DMoEConfig(hidden=32, grid_size=(4,) if gate == "emulator" else (2, 2), k=2, num_layers=2, in_features=12,
                           tokens_per_rank=32, lr=3e-3, gate_mode=gate)
        tr = FastBaselineTrainer(cfg, device=torch.device("cpu"))
        x, y = torch.randn(32, 12), torch.randint(0, 10, (32,))
        losses = [float(tr.train_step_device(x, y)) for _ in range(25)]
        assert losses[-1] < 0.6 * losses[0], losses


def test_stale_trainer_gradients_on_cpu():
    """asynchrony knobs of the engine (reference: notebooks' delay_steps, dmoe_emulator.py:70-77)"""
    torch.manual_seed(0)
    cfg = E.DMoEConfig(hidden=32, grid_size=(2, 2), k=2, num_layers=1, in_features=12, tokens_per_rank=32, lr=3e-3,
                       trainer_staleness=2)
    tr = DMoETrainer(cfg)
    x, y = torch.randn(32, 12), torch.randint(0, 10, (32,))
    w0 = tr.model.head.weight.detach().clone()
    tr.train_step(x, y)
    tr.train_step(x, y)
    assert torch.equal(tr.model.head.weight, w0)          # the first two gradients are still in the delay line
    assert int(tr.model.blocks[0].shard.step.max()) == 2  # experts do not wait for anybody
    tr.train_step(x, y)
    assert not torch.equal(tr.model.head.weight, w0)      # ... the gradient of step 0 arrives with step 2
    losses = [tr.train_step(x, y) for _ in range(40)]
    assert losses[-1] < 0.7 * losses[0]


def test_update_every_on_cpu_matches_the_emulator_schedule_and_resumes():
    """DMoEConfig.update_every_inputs / update_every_steps on the CPU oracle path: experts accumulate gradients and step only
    when due (dmoe_emulator.py:70-77; same schedule as the GPU test); the pending counters and the partially accumulated
    gradient are part of the checkpoint"""
    torch.manual_seed(0)
    cfg = E.DMoEConfig(hidden=16, grid_size=(2, 2), k=4, num_layers=1, in_features=8, tokens_per_rank=16,
                       update_every_inputs=10 ** 6, update_every_steps=3)
    tr = DMoETrainer(cfg)
    x, y = torch.randn(16, 8), torch.randint(0, 10, (16,))
    steps, clone = [], None
    for i in range(7):
        tr.train_step(x, y)
        steps.append(int(tr.model.blocks[0].shard.step.max()))
        if i == 3:   # mid-accumulation: one pending step, a non-zero gradient buffer
            state = tr.state_dict()
            assert int(state["pending"][0]["steps"].max()) == 1 and float(state["pending"][0]["grad"].abs().sum()) > 0
            clone = DMoETrainer(cfg)
            clone.load_state_dict(state)
    assert steps == [0, 0, 1, 1, 1, 2, 2], steps
    for _ in range(3):
        clone.train_step(x, y)
    assert torch.allclose(clone.model.blocks[0].shard.p, tr.model.blocks[0].shard.p, atol=1e-6)
    # update_every_inputs: 16 samples x top-4 of 4 experts = 16 rows per expert and step -> due every second step at 32
    cfg2 = E.DMoEConfig(hidden=16, grid_size=(2, 2), k=4, num_layers=1, in_features=8, tokens_per_rank=16, update_every_inputs=32)
    tr2 = DMoETrainer(cfg2)
    seen = []
    for _ in range(4):
        tr2.train_step(x, y)
        seen.append(int(tr2.model.blocks[0].shard.step.max()))
    assert seen == [0, 1, 1, 2], seen


def test_expert_path_selection():
    """"small" (swap-AB weight streaming, fused wgrad+AMSGrad) below 512 rows per expert and step, "big" (128 x 256 tiles) above;
    gradient accumulation and FP8 forward GEMMs live on the big path"""
    named = E.DMoEConfig(hidden=512, grid_size=(64,), k=4, tokens_per_rank=256)
    assert named.resolved_path(1) == "small" and named.resolved_path(8) == "small"      # 16 .. 128 rows per expert
    assert E.DMoEConfig(hidden=512, grid_size=(64,), k=4, tokens_per_rank=65536).resolved_path(1) == "big"
    assert E.DMoEConfig(hidden=512, grid_size=(64,), k=4, tokens_per_rank=256, update_every_steps=3).resolved_path(1) == "big"
    assert E.DMoEConfig(hidden=512, grid_size=(64,), k=4, tokens_per_rank=256, expert_dtype="fp8").resolved_path(1) == "big"
    assert E.DMoEConfig(hidden=512, grid_size=(64,), k=4, tokens_per_rank=256, expert_path="big").resolved_path(1) == "big"
    many = E.DMoEConfig(hidden=512, grid_size=(4096,), k=4, tokens_per_rank=512)     # swap-AB handles <= 1023 groups per rank
    assert many.resolved_path(2) == "big" and many.resolved_path(8) == "small"


def test_trainer_microbatches_step_experts_per_microbatch():
    torch.manual_seed(0)
    cfg = E.DMoEConfig(hidden=32, grid_size=(2, 2), k=2, num_layers=1, in_features=12, tokens_per_rank=32, lr=3e-3,
                       trainer_microbatches=4)
    tr = DMoETrainer(cfg)
    x, y = torch.randn(32, 12), torch.randint(0, 10, (32,))
    l0 = tr.train_step(x, y)
    assert int(tr.model.blocks[0].shard.step.max()) == 4 and tr.step_count == 1     # experts: 4 updates, trainer: 1
    losses = [tr.train_step(x, y) for _ in range(20)]
    assert losses[-1] < 0.6 * l0
