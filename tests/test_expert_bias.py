"""Auxiliary-loss-free expert balancing: a per-expert routing bias added to the gate scores for the top-k selection only,
moved toward balance after the count exchange of every training forward (DMoEConfig(expert_bias_update_rate=...)).

CPU: the configuration and its refusals, the oracles K.gate_topk_ref(bias=...) and K.expert_bias_update_ref, the update
schedule of the CPU layer and trainer, checkpoints, and the balance a small trainer reaches with either gate.
GPU: the biased gate_topk and expert_bias_update kernels against the oracles, one layer on both expert paths, both expert
kinds and both gates against the CPU oracle, and the trainer under its CUDA graph with its launch budget."""
import math

import pytest
import torch

import lah_b200  # noqa
from lah_b200.ops import kernels as K
from lah_b200.parallel import baseline, engine as E
from lah_b200.parallel.trainer import DMoETrainer
from routing_support import collapse, cpu_cfg, layer_against_the_oracle, load, run_gate, slots
from routing_support import one_thread, step_counters  # noqa: F401 (fixtures)

RATE = dict(expert_bias_update_rate=0.01)


# ======================================================================================================== CPU: config
def test_default_rate_is_zero_and_allocates_nothing():
    assert E.DMoEConfig().expert_bias_update_rate == 0.0
    plain = E.FusedDMoE(cpu_cfg())
    zero = E.FusedDMoE(cpu_cfg(expert_bias_update_rate=0.0))
    assert plain.expert_bias is None and zero.expert_bias is None
    assert "expert_bias" not in dict(zero.named_buffers())
    assert list(plain.state_dict()) == list(zero.state_dict())
    biased = E.FusedDMoE(cpu_cfg(**RATE))
    assert set(biased.state_dict()) == set(plain.state_dict()) | {"expert_bias"}
    assert biased.expert_bias.dtype == torch.float32 and torch.equal(biased.expert_bias, torch.zeros(16))


@pytest.mark.parametrize("rate", [-1e-3, float("nan"), float("inf"), float("-inf")])
def test_config_refuses_bad_rates(rate):
    with pytest.raises(ValueError, match="expert_bias_update_rate"):
        E.DMoEConfig(expert_bias_update_rate=rate)


@pytest.mark.parametrize("expert", ["ffn", "swiglu"])
@pytest.mark.parametrize("gate", ["product_key", "emulator"])
def test_every_gate_and_expert_kind_accepts_a_rate(gate, expert):
    cfg = cpu_cfg(grid_size=(16,), gate_mode=gate, expert=expert, **RATE)
    for path in ("small", "big"):
        E.DMoEConfig(**{**cfg.__dict__, "expert_path": path})
    assert E.FusedDMoE(cfg).expert_bias.shape == (16,)


@pytest.mark.parametrize("arm", ["BaselineDMoE", "BaselineTrainer", "FastBaselineDMoE", "FastBaselineTrainer"])
def test_baseline_arms_refuse_the_bias(arm):
    from lah_b200.parallel import baseline_fast
    cfg = E.DMoEConfig(hidden=64, grid_size=(4,), k=2, num_layers=1, tokens_per_rank=8, **RATE)
    make = dict(BaselineDMoE=lambda: baseline.BaselineDMoE(cfg), BaselineTrainer=lambda: baseline.BaselineTrainer(cfg),
                FastBaselineDMoE=lambda: baseline_fast.FastBaselineDMoE(cfg, 0, 16),
                FastBaselineTrainer=lambda: baseline_fast.FastBaselineTrainer(cfg))[arm]
    with pytest.raises(ValueError, match="expert_bias_update_rate"):
        make()


# ======================================================================================================== CPU: oracles
def _dyadic_case(grid, B, gen, dead=False):
    """quarter-integer logits and eighth-integer biases: scores and keys are exact in any summation order, and tie often"""
    E_ = math.prod(grid)
    logits = torch.randint(-12, 13, (B, sum(grid)), generator=gen).float() / 4
    bias = torch.randint(-8, 9, (E_,), generator=gen).float() / 8
    alive = (torch.rand(E_, generator=gen) > 0.3).to(torch.uint8) if dead else None
    return logits, bias, alive


@pytest.mark.parametrize("grid", [(16,), (4, 4), (2, 3, 4), (2, 2, 2, 2)])
def test_zero_bias_selects_like_no_bias(grid):
    gen = torch.Generator().manual_seed(1)
    logits, _, alive = _dyadic_case(grid, 50, gen, dead=True)
    fail = torch.rand(50, math.prod(grid), generator=gen) < 0.2
    for k in (1, 3, 8):
        ref = K.gate_topk_ref(logits, grid, k, alive=alive, fail_mask=fail)
        got = K.gate_topk_ref(logits, grid, k, alive=alive, fail_mask=fail, bias=torch.zeros(math.prod(grid)))
        assert torch.equal(ref[0], got[0]) and torch.equal(ref[1], got[1])


@pytest.mark.parametrize("grid", [(16,), (4, 4), (2, 2, 2, 2)])
def test_bias_changes_the_selection_but_not_the_weights(grid):
    gen = torch.Generator().manual_seed(2)
    logits, bias, _ = _dyadic_case(grid, 64, gen)
    k = 3
    idx, w = K.gate_topk_ref(logits, grid, k, bias=bias)
    assert not torch.equal(idx, K.gate_topk_ref(logits, grid, k)[0])
    scores = K.product_key_scores(logits, grid)
    keys = scores + bias
    # the selected experts hold the k largest keys, equal keys taking the smaller id, in descending key order
    for b in range(64):
        order = sorted(range(scores.shape[1]), key=lambda e: (-float(keys[b, e]), e))[:k]
        assert idx[b].tolist() == order
    # the weights: softmax over the UNBIASED scores of the selected experts
    torch.testing.assert_close(w, torch.softmax(torch.gather(scores, 1, idx), -1), rtol=0, atol=0)


def test_biased_selection_respects_dead_experts_and_failures():
    grid = (8,)
    logits = torch.zeros(3, 8)
    bias = torch.tensor([9.0, 8.0, 7.0, 6.0, 5.0, 4.0, 3.0, 2.0])
    alive = torch.tensor([0, 1, 1, 1, 1, 1, 1, 1], dtype=torch.uint8)
    fail = torch.zeros(3, 8, dtype=torch.bool)
    fail[1, 1] = True
    fail[2, 1:] = True
    idx, w = K.gate_topk_ref(logits, grid, 2, alive=alive, fail_mask=fail, bias=bias)
    assert idx.tolist() == [[1, 2], [2, 3], [-1, -1]]
    assert w.tolist() == [[0.5, 0.5], [0.5, 0.5], [0.0, 0.0]]


def test_update_ref_follows_the_integer_rule():
    g = 0.25
    b0 = torch.tensor([1.0, -2.0, 0.5, 3.0])
    # T = 8, N = 4: N c = [12, 4, 8, 8] against 8 -> down, up, equal, equal
    out = K.expert_bias_update_ref(torch.tensor([3, 1, 2, 2]), b0, g)
    assert out.dtype == torch.float32 and out.tolist() == [0.75, -1.75, 0.5, 3.0]
    # T = 0 changes nothing
    assert torch.equal(K.expert_bias_update_ref(torch.zeros(4, dtype=torch.int32), b0, g), b0)
    # dead experts are left alone and do not count in N: N = 3, T = 6, N c = [9, 3, 6] against 6
    alive = torch.tensor([1, 1, 1, 0], dtype=torch.uint8)
    out = K.expert_bias_update_ref(torch.tensor([3, 1, 2, 0]), b0, g, alive=alive)
    assert out.tolist() == [0.75, -1.75, 0.5, 3.0]
    # an [R, E] table is summed over its R rank rows
    table = torch.tensor([[3, 0, 2, 1], [0, 1, 0, 1]])
    assert torch.equal(K.expert_bias_update_ref(table, b0, g), K.expert_bias_update_ref(torch.tensor([3, 1, 2, 2]), b0, g))
    # one float32 add of the float32 rate
    out = K.expert_bias_update_ref(torch.tensor([0, 1]), torch.tensor([0.1, 0.1]), 1e-3)
    r = torch.tensor(1e-3, dtype=torch.float32)
    assert out.tolist() == [float(torch.tensor(0.1) + r), float(torch.tensor(0.1) - r)]


def test_update_ref_against_a_python_loop():
    gen = torch.Generator().manual_seed(3)
    for R in (1, 3, 8):
        E_ = 37
        counts = torch.randint(0, 6, (R, E_), generator=gen)
        alive = (torch.rand(E_, generator=gen) > 0.25).to(torch.uint8)
        counts *= alive.long()
        b = torch.randn(E_, generator=gen)
        out = K.expert_bias_update_ref(counts, b, 0.01, alive=alive)
        c = counts.sum(0).tolist()
        T, N = sum(c), int(alive.sum())
        r = torch.tensor(0.01, dtype=torch.float32)
        for e in range(E_):
            want = b[e]
            if alive[e] and N * c[e] < T:
                want = b[e] + r
            elif alive[e] and N * c[e] > T:
                want = b[e] - r
            assert float(out[e]) == float(want), e


# ======================================================================================================== CPU: layer, trainer
def _count_updates(monkeypatch):
    calls = []
    real = K.expert_bias_update_ref

    def counted(*a, **kw):
        calls.append(1)
        return real(*a, **kw)

    monkeypatch.setattr(K, "expert_bias_update_ref", counted)
    return calls


@pytest.mark.parametrize("m", [1, 2])
def test_one_update_per_training_forward_and_micro_batch(monkeypatch, one_thread, m):
    calls = _count_updates(monkeypatch)
    t = DMoETrainer(cpu_cfg(num_layers=2, trainer_microbatches=m, **RATE))
    x, y = torch.randn(64, 16), torch.randint(0, 10, (64,))
    t.train_step(x, y)
    assert len(calls) == 2 * m
    t.train_step(x, y)
    assert len(calls) == 4 * m
    assert all(float(b.expert_bias.abs().max()) > 0 for b in t.model.blocks)
    before = [b.expert_bias.clone() for b in t.model.blocks]
    t.evaluate(x, y)
    assert len(calls) == 4 * m
    assert all(torch.equal(a, b.expert_bias) for a, b in zip(before, t.model.blocks))


def test_layer_update_uses_the_routed_pairs_of_the_forward():
    layer = E.FusedDMoE(cpu_cfg(**RATE)).train()
    with torch.no_grad():
        layer.expert_bias.copy_(torch.arange(16).float() / 8 - 1)
    before = layer.expert_bias.clone()
    x = torch.randn(32, 64)
    logits = layer.gate_logits(x, layer.proj)
    idx, _ = K.gate_topk_ref(logits.detach(), layer.grid_size, 4, bias=before)
    layer(x)
    counts = torch.bincount(idx[idx >= 0].flatten(), minlength=16)
    assert torch.equal(layer.expert_bias, K.expert_bias_update_ref(counts, before, 0.01))
    # eval applies the bias and leaves it
    layer.eval()
    layer(x)
    assert not torch.equal(layer.expert_bias, before)
    assert torch.equal(layer.expert_bias, K.expert_bias_update_ref(counts, before, 0.01))


def test_resumed_run_equals_the_continued_run(one_thread):
    cfg = cpu_cfg(num_layers=2, **RATE)
    gen = torch.Generator().manual_seed(4)
    xs = [torch.randn(64, 16, generator=gen) for _ in range(6)]
    ys = [torch.randint(0, 10, (64,), generator=gen) for _ in range(6)]
    a = DMoETrainer(cfg)
    for x, y in zip(xs[:3], ys[:3]):
        a.train_step(x, y)
    state = a.state_dict()
    assert all(f"blocks.{i}.expert_bias" in state["trainer"]["model"] for i in range(2))
    la = [a.train_step(x, y) for x, y in zip(xs[3:], ys[3:])]
    b = DMoETrainer(cfg)
    addr = [blk.expert_bias.data_ptr() for blk in b.model.blocks]
    b.load_state_dict(state)
    assert addr == [blk.expert_bias.data_ptr() for blk in b.model.blocks]   # loaded in place
    lb = [b.train_step(x, y) for x, y in zip(xs[3:], ys[3:])]
    assert la == lb
    for ba, bb in zip(a.model.blocks, b.model.blocks):
        assert torch.equal(ba.expert_bias, bb.expert_bias) and torch.equal(ba.shard.p, bb.shard.p)
    assert torch.equal(a.flat_p, b.flat_p)


def test_checkpoint_rules(one_thread):
    x, y = torch.randn(64, 16), torch.randint(0, 10, (64,))
    biased = DMoETrainer(cpu_cfg(**RATE))
    biased.train_step(x, y)
    with pytest.raises(ValueError, match="expert_bias_update_rate"):
        DMoETrainer(cpu_cfg()).load_state_dict(biased.state_dict())
    # a checkpoint without biases loads into a biased trainer with zero biases
    plain = DMoETrainer(cpu_cfg())
    plain.train_step(x, y)
    assert float(biased.model.blocks[0].expert_bias.abs().max()) > 0
    biased.load_state_dict(plain.state_dict())
    assert torch.equal(biased.model.blocks[0].expert_bias, torch.zeros(16))
    assert torch.equal(biased.flat_p, plain.flat_p)


@pytest.mark.parametrize("gate", ["product_key", "emulator"])
def test_expert_bias_spreads_a_collapsed_router(one_thread, gate):
    """a gate that starts with two of eight experts taking most rows: without the bias the collapse stays, with it the
    load spreads; the task loss falls in both runs.  The emulator gate is frozen, so nothing else could balance it"""
    gen = torch.Generator().manual_seed(0)
    protos = torch.randn(10, 16, generator=gen) * 2
    y = torch.randint(0, 10, (128,), generator=gen)
    x = protos[y] + 0.5 * torch.randn(128, 16, generator=gen)
    results = {}
    for rate in (0.0, 0.05):
        cfg = cpu_cfg(grid_size=(8,), k=2, num_layers=1, tokens_per_rank=128, lr=3e-3, gate_mode=gate,
                      expert_bias_update_rate=rate)
        t = DMoETrainer(cfg)
        collapse(t.model.blocks[0], gate)
        before = load(t, x)
        losses = [t.train_step(x, y) for _ in range(120)]
        results[rate] = (before, load(t, x), losses)
    (b0, a0, l0), (b1, a1, l1) = results[0.0], results[0.05]
    assert b0 == b1 and b0[0] > 3.0
    assert a1[0] < 0.6 * a0[0] and a1[0] < 1.5, (a0, a1)
    assert l0[-1] < 0.5 * l0[0] and l1[-1] < 0.5 * l1[0], (l0[::20], l1[::20])


# ======================================================================================================== GPU
@pytest.mark.gpu
@pytest.mark.parametrize("B", [1, 7, 256, 65536])
@pytest.mark.parametrize("grid", [(64,), (8, 8), (32, 32), (64, 64), (4096,), (4, 4, 4, 4)])
def test_biased_gate_topk_against_the_oracle(step_counters, grid, B):
    """dyadic logits and biases: the keys are exact in any summation order, so idx, pos and counts must be equal"""
    E_ = math.prod(grid)
    gen = torch.Generator(device="cuda").manual_seed(B * 7 + E_)
    logits = torch.randint(-12, 13, (B, sum(grid)), generator=gen, device="cuda").float() / 4
    bias = torch.randint(-8, 9, (E_,), generator=gen, device="cuda").float() / 8
    alive = (torch.rand(E_, generator=gen, device="cuda") > 0.2).to(torch.uint8)
    rate = 0.1
    fail = K.gate_fail_mask_ref(B, E_, rate, 99, 0).cuda()
    for k in range(1, 9):
        idx, w, pos, counts, _, _ = run_gate(logits, grid, k, alive=alive, rate=rate, bias=bias)
        ridx, rw = K.gate_topk_ref(logits, grid, k, alive=alive, fail_mask=fail, bias=bias)
        assert torch.equal(idx.long(), ridx), (k, int((idx.long() != ridx).any(1).sum()))
        assert torch.equal(pos.long(), slots(ridx))
        assert torch.equal(counts.long(), torch.bincount(ridx[ridx >= 0], minlength=E_))
        assert float((w.double() - rw.double()).abs().max()) < 1e-6
        # bias=None is the zero bias, bit for bit
        plain = run_gate(logits, grid, k, alive=alive, rate=rate, bias=None)
        zero = run_gate(logits, grid, k, alive=alive, rate=rate, bias=torch.zeros_like(bias))
        assert all(torch.equal(a, b) for a, b in zip(plain[:4], zero[:4]))


@pytest.mark.gpu
def test_gate_topk_refuses_a_bad_bias():
    from lah_b200.ops import native
    lg = torch.zeros(4, 16, device="cuda")
    i = torch.zeros(16, dtype=torch.int32, device="cuda")
    ok = dict(idx=i, w=i.float(), pos=i, counts=torch.zeros(16, dtype=torch.int32, device="cuda"))
    before = native.launches()
    for bad in (torch.zeros(15, device="cuda"), torch.zeros(16, dtype=torch.float64, device="cuda"), torch.zeros(16),
                torch.zeros(32, device="cuda")[::2]):
        with pytest.raises(ValueError):
            K.gate_topk(lg, (16,), 4, bias=bad, **ok)
    bias = torch.zeros(16, device="cuda")
    for args, kw in (((i.view(1, -1).long(),), {}), ((torch.zeros(9, 16, dtype=torch.int32, device="cuda"),), {}),
                     ((i.view(1, -1),), dict(rate=-1.0)), ((i.view(1, -1),), dict(rate=float("nan"))),
                     ((i.view(1, -1),), dict(bias=torch.zeros(8, device="cuda"))),
                     ((i.view(1, -1),), dict(alive=torch.ones(8, dtype=torch.uint8, device="cuda")))):
        with pytest.raises(ValueError):
            K.expert_bias_update(*args, **{**dict(bias=bias, rate=0.1), **kw})
    assert native.launches() == before


@pytest.mark.gpu
@pytest.mark.parametrize("E_", [1, 64, 1000, 4096])
def test_expert_bias_update_is_bit_equal_to_the_oracle(E_):
    gen = torch.Generator().manual_seed(E_)
    for R in range(1, 9):
        alive = (torch.rand(E_, generator=gen) > 0.2).to(torch.uint8)
        counts = torch.randint(0, 40, (R, E_), generator=gen, dtype=torch.int32) * alive.int()
        if R == 2:
            counts[:, alive.bool()] = 3            # every live expert at the mean: nothing moves
        if R == 3:
            counts.zero_()                         # T = 0
        bias = torch.randn(E_, generator=gen)
        for rate, al in ((1e-3, alive), (0.37, None)):
            got = bias.cuda()
            K.expert_bias_update(counts.cuda(), alive=None if al is None else al.cuda(), bias=got, rate=rate)
            torch.cuda.synchronize()
            want = K.expert_bias_update_ref(counts, bias, rate, alive=al)
            assert torch.equal(got.cpu(), want), (R, rate)
            if R in (2, 3) and al is not None:
                assert torch.equal(got.cpu(), bias)


@pytest.mark.gpu
@pytest.mark.parametrize("gate", ["emulator", "product_key"])
@pytest.mark.parametrize("expert", ["ffn", "swiglu"])
@pytest.mark.parametrize("path", ["small", "big"])
def test_layer_against_the_cpu_oracle(path, expert, gate):
    torch.manual_seed(3)
    grid = (16,) if gate == "emulator" else (4, 4)
    cfg = E.DMoEConfig(hidden=512, grid_size=grid, k=4, num_layers=1, tokens_per_rank=512, expert=expert,
                       expert_path=path, gate_mode=gate, expert_bias_update_rate=0.01)

    def check(r):
        assert r.ctx.small == (path == "small")
        unbiased = K.gate_topk_ref(r.logits, grid, cfg.k, alive=r.ctx.alive)[0]
        assert not torch.equal(r.ridx, unbiased)   # the bias mattered
        assert torch.equal(r.layer.expert_bias, r.oracle.expert_bias)
        assert torch.equal(r.layer.expert_bias, K.expert_bias_update_ref(r.ctx.cnt_all[:1, :16], r.bias0, 0.01))
        assert not torch.equal(r.layer.expert_bias, r.bias0)

    layer_against_the_oracle(cfg, bias_step=1 / 8, check=check)


def _trainer_cfg(path, gate, **kw):
    base = dict(hidden=512, grid_size=(16,), k=4, num_layers=2, tokens_per_rank=256, failure_rate=0.1, lr=1e-4,
                expert_path=path, gate_mode=gate, expert_bias_update_rate=0.01)
    base.update(kw)
    return E.DMoEConfig(**base)


@pytest.mark.gpu
@pytest.mark.parametrize("gate", ["emulator", "product_key"])
@pytest.mark.parametrize("path", ["small", "big"])
def test_trainer_graph_equals_eager_and_runs_are_reproducible(path, gate):
    cfg = _trainer_cfg(path, gate)
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
        rec = t.log_step()
        assert all(layer["expert_bias_absmax"] > 0 for layer in rec["layers"])
        runs[run] = (torch.stack(losses).cpu(), torch.stack(biases).cpu(),
                     torch.cat([b.shard.p for b in t.model.blocks] + [t.flat_p]).cpu())
        t.close()
    for a, b in zip(runs["eager"], runs["graph"]):
        assert torch.equal(a, b)
    for a, b in zip(runs["graph"], runs["graph2"]):
        assert torch.equal(a, b)


@pytest.mark.gpu
@pytest.mark.parametrize("m", [1, 2])
def test_launch_budget(m):
    counts = {}
    base = dict(hidden=512, grid_size=(16,), k=4, num_layers=2, tokens_per_rank=256, expert_path="small",
                gate_mode="emulator", trainer_microbatches=m)
    for name, kw in (("plain", {}), ("zero", dict(expert_bias_update_rate=0.0)), ("bias", dict(expert_bias_update_rate=0.01))):
        cfg = E.DMoEConfig(**base, **kw)
        t = DMoETrainer(cfg, use_graph=True)
        x, y = torch.randn(256, cfg.in_features, device="cuda"), torch.randint(0, 10, (256,), device="cuda")
        for _ in range(3):
            t.train_step_device(x, y)
        counts[name] = t._graph_launches
        t.close()
    assert counts["plain"] == counts["zero"]
    assert counts["bias"] == counts["plain"] + 2 * m


@pytest.mark.gpu
@pytest.mark.parametrize("gate", ["emulator", "product_key"])
def test_zero_biases_make_the_first_step_of_the_plain_run(gate):
    torch.manual_seed(1)
    x, y = torch.randn(256, 784, device="cuda"), torch.randint(0, 10, (256,), device="cuda")
    out = {}
    for rate in (0.0, 0.01):
        t = DMoETrainer(_trainer_cfg("small", gate, expert_bias_update_rate=rate), use_graph=False)
        loss = t.train_step_device(x, y).clone()
        torch.cuda.synchronize()
        out[rate] = (loss.cpu(), torch.cat([b.shard.p for b in t.model.blocks] + [t.flat_p]).cpu())
        t.close()
    assert torch.equal(out[0.0][0], out[0.01][0]) and torch.equal(out[0.0][1], out[0.01][1])
