"""Group-limited routing of DeepSeek-V2/V3 (DMoEConfig(n_group=G, topk_group=M)): the experts form G groups of consecutive
flat ids, each token scores every group (softmax: its best key; sigmoid: the sum of its two best) and picks its k experts
from its M best groups only (DESIGN.md §6d).

CPU: the configuration and its refusals, K.gate_topk_ref(n_group=, topk_group=) against a brute-force implementation of the
written rules, the identities G = 1 and M = G, the at-most-M-groups property, the layer's gate gradient, a CPU trainer that
spreads a collapsed gate without leaving M groups, and checkpoints across groupings.
GPU: the grouped gate kernels against the oracle, the identities bit for bit, argument refusals before any launch, one
layer on both paths, both expert kinds and both gates (and one DeepSeek-V3-shaped layer) against the CPU oracle, and the
trainer under its CUDA graph."""
import math

import pytest
import torch

import lah_b200  # noqa
from lah_b200.ops import kernels as K
from lah_b200.parallel import baseline, baseline_fast, engine as E
from lah_b200.parallel.trainer import DMoETrainer
from routing_support import collapse, cpu_cfg, layer_against_the_oracle, run_gate, slots
from routing_support import one_thread, step_counters  # noqa: F401 (fixtures)

SIG = dict(router_score="sigmoid")
CPU = torch.device("cpu")   # the CPU trainer tests run on the CPU path on a GPU machine too


# ======================================================================================================== CPU: config
def test_defaults_and_state_dict_keys():
    cfg = E.DMoEConfig()
    assert cfg.n_group == 1 and cfg.topk_group == 1
    plain = E.FusedDMoE(cpu_cfg())
    grouped = E.FusedDMoE(cpu_cfg(n_group=4, topk_group=2))
    assert (plain.n_group, plain.topk_group) == (1, 1) and (grouped.n_group, grouped.topk_group) == (4, 2)
    assert list(plain.state_dict()) == list(grouped.state_dict())


@pytest.mark.parametrize("kw,match", [
    (dict(n_group=True), "n_group must be an int"), (dict(n_group=2.0), "n_group must be an int"),
    (dict(topk_group=False), "topk_group must be an int"), (dict(n_group=4, topk_group=1.0), "topk_group must be an int"),
    (dict(n_group=0), "n_group must be in"), (dict(n_group=-4), "n_group must be in"),
    (dict(grid_size=(128,), n_group=128, topk_group=8), "n_group must be in"),
    (dict(n_group=3), "divide"), (dict(grid_size=(2, 3, 4), n_group=5), "divide"),
    (dict(n_group=4, topk_group=0), "topk_group must be in"), (dict(n_group=4, topk_group=5), "topk_group must be in"),
    (dict(n_group=8, topk_group=1, k=3), "cannot come from"), (dict(n_group=16, topk_group=3, k=4), "cannot come from"),
])
def test_config_refusals(kw, match):
    with pytest.raises(ValueError, match=match):
        cpu_cfg(**kw)


def test_config_accepts_the_feasible_corners():
    cpu_cfg(n_group=16, topk_group=4, k=4)         # G = E, k = M
    cpu_cfg(n_group=8, topk_group=2, k=4)          # k = M * E / G
    cpu_cfg(grid_size=(64, 64), n_group=64, topk_group=8, k=8)
    with pytest.raises(ValueError, match="at most 4096"):
        K.check_expert_groups("x", 8192, 2, 1)


@pytest.mark.parametrize("arm", [baseline.BaselineDMoE, baseline.BaselineTrainer,
                                 lambda cfg: baseline_fast.FastBaselineDMoE(cfg, 0, 64),
                                 baseline_fast.FastBaselineTrainer])
def test_baseline_arms_refuse_group_limited_routing(arm):
    with pytest.raises(ValueError, match="n_group=1"):
        arm(cpu_cfg(n_group=4, topk_group=2))


# ======================================================================================================== CPU: oracle
def _brute(scores, sig32, alive, bias, G, M, k, score):
    """the written rules of DESIGN.md §6d, token by token in plain Python over the float32 keys"""
    B, E_ = scores.shape
    gsz = E_ // G
    f32 = lambda v: float(torch.tensor(v, dtype=torch.float32))   # noqa: E731
    out = []
    for b in range(B):
        cand = [e for e in range(E_) if alive[e]]
        key, gkey = {}, {}
        for e in cand:
            s = float(scores[b, e])
            if bias is None:
                key[e] = s
                gkey[e] = float(sig32[b, e]) if score == "sigmoid" else s
            else:
                key[e] = gkey[e] = f32(f32(float(sig32[b, e]) if score == "sigmoid" else s) + float(bias[e]))
        gscore = {}
        for g in range(G):
            vals = sorted((gkey[e] for e in cand if e // gsz == g), reverse=True)
            if vals:
                gscore[g] = vals[0] if (score == "softmax" or len(vals) == 1) else f32(vals[0] + vals[1])
        groups = sorted(gscore, key=lambda g: (-gscore[g], g))[:M]
        pool = sorted((e for e in cand if e // gsz in groups), key=lambda e: (-key[e], e))[:k]
        out.append(pool + [-1] * (k - len(pool)))
    return torch.tensor(out, dtype=torch.int64).view(B, k)


def _divisors(n):
    return [d for d in range(1, min(n, 64) + 1) if n % d == 0]


@pytest.mark.parametrize("alive_kind", ["all", "dead", "dead_group"])
@pytest.mark.parametrize("grid", [(16,), (4, 4), (2, 3, 4), (2, 2, 2, 2), (64,)])
def test_gate_topk_ref_equals_the_written_rules(grid, alive_kind):
    gen = torch.Generator().manual_seed(sum(grid) * 7 + len(alive_kind))
    E_ = math.prod(grid)
    B = 3
    # dyadic logits and biases: sums are exact, and equal keys (ties of experts and of groups) are common
    logits = torch.randint(-6, 7, (B, sum(grid)), generator=gen).float() / 4
    bias = torch.randint(-4, 5, (E_,), generator=gen).float() / 8
    alive = torch.ones(E_, dtype=torch.uint8)
    if alive_kind != "all":
        alive[torch.rand(E_, generator=gen) < 0.3] = 0
    scores = K.product_key_scores(logits, grid)
    sig32 = torch.sigmoid(scores)
    for G in _divisors(E_):
        gsz = E_ // G
        al = alive.clone()
        if alive_kind == "dead_group" and G > 1:
            al[:gsz] = 0                     # a wholly dead group
            al[(G - 1) * gsz + 1:] = 0       # a group with one live expert
        for M in range(1, G + 1):
            for k in range(1, min(8, M * gsz) + 1):
                for score in ("softmax", "sigmoid"):
                    for b in (None, bias):
                        idx, w = K.gate_topk_ref(logits, grid, k, alive=al, bias=b, score=score, n_group=G,
                                                 topk_group=M)
                        want = _brute(scores, sig32, al, b, G, M, k, score)
                        assert torch.equal(idx, want), (G, M, k, score, b is None)
                        valid = idx >= 0
                        assert torch.allclose(w.sum(1)[valid.any(1)], torch.ones(1), atol=1e-5)
                        assert bool((w[~valid] == 0).all())


def test_gate_topk_ref_group_corner_cases():
    # 4 experts in 2 groups; group scores tie -> the smaller group
    lg = torch.tensor([[1.0, 0.0, 0.0, 1.0]])
    assert K.gate_topk_ref(lg, (4,), 2, n_group=2, topk_group=1)[0].tolist() == [[0, 1]]
    # sigmoid: the sum of the best two decides, not the best one
    lg = torch.tensor([[3.0, -3.0, 1.0, 1.0]])
    assert K.gate_topk_ref(lg, (4,), 1, score="sigmoid", n_group=2, topk_group=1)[0].tolist() == [[2]]
    assert K.gate_topk_ref(lg, (4,), 1, n_group=2, topk_group=1)[0].tolist() == [[0]]
    # a sigmoid group with one live expert scores that one key
    alive = torch.tensor([1, 0, 1, 1], dtype=torch.uint8)
    lg = torch.tensor([[4.0, 9.0, 0.0, 0.0]])
    assert K.gate_topk_ref(lg, (4,), 2, alive=alive, score="sigmoid", n_group=2, topk_group=1)[0].tolist() == [[2, 3]]
    # fewer live groups than topk_group: the live ones, then missing pairs
    alive = torch.tensor([0, 0, 1, 0], dtype=torch.uint8)
    idx, w = K.gate_topk_ref(torch.zeros(1, 4), (4,), 2, alive=alive, n_group=2, topk_group=2)
    assert idx.tolist() == [[2, -1]] and w.tolist() == [[1.0, 0.0]]
    # a wholly dead group is never selected, even when it would score best
    alive = torch.tensor([0, 0, 1, 1], dtype=torch.uint8)
    assert K.gate_topk_ref(torch.tensor([[9.0, 9.0, 0.0, 1.0]]), (4,), 2, alive=alive, n_group=2,
                           topk_group=1)[0].tolist() == [[3, 2]]


@pytest.mark.parametrize("grid", [(16,), (4, 4), (2, 3, 4), (64,)])
def test_identities_give_the_ungrouped_oracle(grid):
    gen = torch.Generator().manual_seed(len(grid))
    E_ = math.prod(grid)
    logits = torch.randn(40, sum(grid), generator=gen)
    bias = torch.randn(E_, generator=gen) * 0.1
    alive = (torch.rand(E_, generator=gen) > 0.2).to(torch.uint8)
    fail = torch.rand(40, E_, generator=gen) < 0.1
    for score, scale in (("softmax", 1.0), ("sigmoid", 2.5)):
        for b in (None, bias):
            for k in (1, 4, 8):
                ref = K.gate_topk_ref(logits, grid, k, alive=alive, fail_mask=fail, bias=b, score=score, scale=scale)
                for G in _divisors(E_):
                    for M in {1, G} if G == 1 else {G}:
                        got = K.gate_topk_ref(logits, grid, k, alive=alive, fail_mask=fail, bias=b, score=score,
                                              scale=scale, n_group=G, topk_group=M)
                        assert torch.equal(got[0], ref[0]) and torch.equal(got[1], ref[1])


@pytest.mark.parametrize("world", [2, 4, 8])
def test_selected_experts_lie_in_at_most_topk_group_groups(world):
    gen = torch.Generator().manual_seed(world)
    grid = (8, 8)
    E_ = 64
    logits = torch.randn(500, 16, generator=gen) * 3
    bias = torch.randn(E_, generator=gen)
    for G in (world, 2 * world):
        for M in range(1, min(G, 4) + 1):
            k = min(8, M * E_ // G)
            for score, b in (("softmax", None), ("sigmoid", bias)):
                idx, _ = K.gate_topk_ref(logits, grid, k, bias=b, score=score, n_group=G, topk_group=M)
                assert E.max_groups_per_token(idx, k, E_, G) <= M
                # with G = world and E_loc = E / world a group is one rank: its owners are the groups' ranks
                owners = torch.where(idx >= 0, idx // (E_ // world), -1)
                ranks = max(len(set(r) - {-1}) for r in owners.tolist())
                assert ranks <= (M if G == world else min(world, M))


def test_layer_gate_gradient_equals_float64_autograd_with_the_groups_fixed():
    torch.manual_seed(0)
    for score in ("softmax", "sigmoid"):
        kw = dict(routed_scaling_factor=2.5, **SIG) if score == "sigmoid" else {}
        layer = E.FusedDMoE(cpu_cfg(grid_size=(16,), n_group=4, topk_group=2, **kw)).train()
        x = torch.randn(32, 64)
        logits = layer.gate_logits(x, layer.proj).detach().requires_grad_(True)
        out = layer._forward_ref(x, logits)
        gy = torch.randn_like(out)
        (out * gy).sum().backward()
        # float64: the same expert choice (the group limit fixed), the weights differentiated in float64
        idx, _ = K.gate_topk_ref(logits.detach(), (16,), 4, score=score, n_group=4, topk_group=2)
        assert E.max_groups_per_token(idx, 4, 16, 4) <= 2
        lg = logits.detach().double().requires_grad_(True)
        sel = torch.gather(lg, 1, idx.clamp(min=0))
        w = (K.sigmoid_weights_ref(sel, idx >= 0, 2.5) if score == "sigmoid"
             else torch.softmax(sel.masked_fill(idx < 0, float("-inf")), -1))
        y_e = _expert_outputs(layer, x).double()                     # [B, k, H] outputs of the selected experts
        sel_y = torch.gather(y_e, 1, idx.clamp(min=0).unsqueeze(-1).expand(-1, -1, y_e.shape[-1]))
        ((w.unsqueeze(-1) * sel_y).sum(1) * gy.double()).sum().backward()
        torch.testing.assert_close(logits.grad.double(), lg.grad, rtol=1e-4, atol=1e-5)


def _expert_outputs(layer, x):
    """[B, E, H]: every expert's output on every token, from a copy of the layer routed to one expert at a time"""
    E_ = layer.cfg.num_experts
    probe_cfg = {**layer.cfg.__dict__, "k": 1, "n_group": 1, "topk_group": 1, "router_score": "softmax",
                 "routed_scaling_factor": 1.0}
    probe = E.FusedDMoE(E.DMoEConfig(**probe_cfg)).eval()
    probe.load_state_dict(layer.state_dict())
    with torch.no_grad():
        probe.shard.p.copy_(layer.shard.p)
        outs = []
        for e in range(E_):
            lg = torch.full((x.shape[0], E_), -100.0)
            lg[:, e] = 100.0
            outs.append(probe._forward_ref(x, lg))
    return torch.stack(outs, 1)


def _load(trainer, x):
    """max / mean rows per expert and the most groups per token of every layer on batch x (eval-mode routing)"""
    out, h = [], trainer.model.stem(x)
    with torch.no_grad():
        for block in trainer.model.blocks:
            idx, _ = K.gate_topk_ref(block.gate_logits(h, block.proj), block.grid_size, block.cfg.k,
                                     bias=block.expert_bias, score=block.router_score, n_group=block.n_group,
                                     topk_group=block.topk_group)
            rows = torch.bincount(idx[idx >= 0].flatten(), minlength=block.cfg.num_experts).float()
            out.append((float(rows.max() / rows.mean()),
                        E.max_groups_per_token(idx, block.cfg.k, block.cfg.num_experts, block.n_group)))
            h = block(h)
    return out


def test_v3_shaped_cpu_trainer_spreads_a_collapsed_gate_within_its_groups(one_thread):
    """the §6b / §6c setting with the V3 router (sigmoid, expert biases) and 4 groups of 4, 2 of them per token: two of
    16 experts take most rows; the biases spread the load, and no token ever leaves its 2 groups"""
    gen = torch.Generator().manual_seed(0)
    protos = torch.randn(10, 16, generator=gen) * 2
    y = torch.randint(0, 10, (128,), generator=gen)
    x = protos[y] + 0.5 * torch.randn(128, 16, generator=gen)
    results = {}
    for rate in (0.0, 0.01):
        cfg = cpu_cfg(grid_size=(16,), k=2, tokens_per_rank=128, lr=3e-3, expert_bias_update_rate=rate,
                      routed_scaling_factor=2.0, n_group=4, topk_group=2, **SIG)
        t = DMoETrainer(cfg, device=CPU)
        collapse(t.model.blocks[0], "product_key")
        before = _load(t, x)
        losses = []
        for _ in range(120):
            losses.append(t.train_step(x, y))
            assert _load(t, x)[0][1] <= 2
        results[rate] = (before, _load(t, x), losses)
    (b0, a0, l0), (b1, a1, l1) = results[0.0], results[0.01]
    assert b0 == b1 and b0[0][0] > 3.0
    assert a1[0][0] < 0.6 * a0[0][0] and a1[0][0] < 2.0, (a0, a1)
    assert l0[-1] < 0.5 * l0[0] and l1[-1] < 0.5 * l1[0], (l0[::20], l1[::20])


def test_checkpoints_load_across_groupings(one_thread):
    gen = torch.Generator().manual_seed(4)
    xs = [torch.randn(64, 16, generator=gen) for _ in range(6)]
    ys = [torch.randint(0, 10, (64,), generator=gen) for _ in range(6)]
    base = dict(num_layers=2, expert_bias_update_rate=1e-3, routed_scaling_factor=2.5, **SIG)
    grouped, plain = cpu_cfg(n_group=4, topk_group=2, **base), cpu_cfg(**base)
    for src_cfg, dst_cfg in ((grouped, plain), (plain, grouped)):
        a = DMoETrainer(src_cfg, device=CPU)
        for x, y in zip(xs[:3], ys[:3]):
            a.train_step(x, y)
        state = a.state_dict()
        assert "n_group" not in state["trainer"] and "topk_group" not in state["trainer"]
        la = [a.train_step(x, y) for x, y in zip(xs[3:], ys[3:])]
        b = DMoETrainer(src_cfg, device=CPU)    # the same grouping resumes bit for bit
        b.load_state_dict(state)
        assert [b.train_step(x, y) for x, y in zip(xs[3:], ys[3:])] == la
        c = DMoETrainer(dst_cfg, device=CPU)    # the other grouping loads every parameter and trains on
        c.load_state_dict(state)
        for bc, ba in zip(c.model.blocks, a.model.blocks):
            assert bc.expert_bias.shape == ba.expert_bias.shape
        lc = [c.train_step(x, y) for x, y in zip(xs[3:], ys[3:])]
        assert all(math.isfinite(v) for v in lc)


# ======================================================================================================== GPU
def _gaps_clear(v, n, tol):
    """rows of v (sorted descending, -inf = missing) whose n leading entries are pairwise separated by more than tol"""
    v = v[:, :n]
    gap = (v[:, :-1] - v[:, 1:]).nan_to_num(float("inf"))
    return ((gap > tol) | torch.isinf(v[:, 1:])).all(1)


def _clear_tokens(scores, dead, bias, G, M, k, score):
    """sigmoid arms (sigma is __expf-based in the kernel): tokens whose oracle group scores among the M + 1 best and
    whose keys among the k + 1 best of the selected groups are separated by more than 1e-5"""
    masked = scores.masked_fill(dead, float("-inf"))
    gscore, has = K.expert_group_scores_ref(masked, bias, G, score)
    ok = _gaps_clear(torch.sort(gscore.masked_fill(~has, float("-inf")), -1, descending=True)[0], M + 1, 1e-5)
    narrowed = masked.masked_fill(~K.expert_group_mask_ref(masked, bias, G, M, score), float("-inf"))
    keys = narrowed if bias is None else (torch.sigmoid(narrowed) + bias).masked_fill(~torch.isfinite(narrowed),
                                                                                     float("-inf"))
    return ok & _gaps_clear(torch.sort(keys, -1, descending=True)[0], k + 1, 1e-5)


GROUPINGS = {   # (n_group, topk_group) per grid: G = E, group sizes that are not powers of two, multiples of 32, ...
    (64,): [(8, 2), (8, 4), (64, 8), (16, 3)],
    (8, 8): [(8, 2), (4, 1), (2, 1)],
    (256,): [(8, 4), (64, 2), (32, 5)],
    (64, 64): [(64, 8), (8, 4), (16, 3)],
    (4096,): [(8, 4), (64, 2)],
    (2, 3, 4): [(2, 1), (4, 2), (8, 3), (24, 5)],
    (4, 4, 4, 4): [(16, 4), (64, 8), (2, 1)],
}


@pytest.mark.gpu
@pytest.mark.parametrize("B", [1, 7, 256, 65536])
@pytest.mark.parametrize("grid", list(GROUPINGS))
def test_grouped_gate_topk_against_the_oracle(step_counters, grid, B):
    E_ = math.prod(grid)
    gen = torch.Generator(device="cuda").manual_seed(B * 3 + E_)
    # softmax arms: dyadic logits and biases, every key and group score is exact in any order
    dyadic = torch.randint(-12, 13, (B, sum(grid)), generator=gen, device="cuda").float() / 4
    dbias = torch.randint(-8, 9, (E_,), generator=gen, device="cuda").float() / 16
    # sigmoid arms: continuous values, compared on the clearly separated tokens; scores of standard deviation <= 1, where
    # sigma is not saturated and its differences stay far above the kernel's rounding
    logits = torch.randn(B, sum(grid), generator=gen, device="cuda") / len(grid)
    cbias = torch.randn(E_, generator=gen, device="cuda") * 0.05
    rate = 0.1
    fail = K.gate_fail_mask_ref(B, E_, rate, 99, 0).cuda()
    unclear = total = 0
    for G, M in GROUPINGS[grid]:
        gsz = E_ // G
        alive = (torch.rand(E_, generator=gen, device="cuda") > 0.1).to(torch.uint8)
        alive[gsz:2 * gsz] = 0                       # a wholly dead group
        dead = ~alive.bool().view(1, -1) | fail
        for k in range(1, min(8, M * gsz) + 1):
            for b in (None, dbias):
                idx, w, pos, counts, _, _ = run_gate(dyadic, grid, k, alive=alive, rate=rate, bias=b, n_group=G,
                                                     topk_group=M)
                ridx, rw = K.gate_topk_ref(dyadic, grid, k, alive=alive, fail_mask=fail, bias=b, n_group=G,
                                           topk_group=M)
                assert torch.equal(idx.long(), ridx), (G, M, k, b is None, int((idx.long() != ridx).any(1).sum()))
                assert torch.equal(pos.long(), slots(ridx))
                assert torch.equal(counts.long(), torch.bincount(ridx[ridx >= 0], minlength=E_))
                assert float((w - rw).abs().max()) < 2e-6, (G, M, k)
            c = 2.5 if k % 2 else 1.0
            for b in (None, cbias):
                idx, w, pos, counts, _, _ = run_gate(logits, grid, k, alive=alive, rate=rate, bias=b, score="sigmoid",
                                                     scale=c, n_group=G, topk_group=M)
                ridx, rw = K.gate_topk_ref(logits, grid, k, alive=alive, fail_mask=fail, bias=b, score="sigmoid",
                                           scale=c, n_group=G, topk_group=M)
                clear = _clear_tokens(K.product_key_scores(logits, grid), dead, b, G, M, k, "sigmoid")
                unclear += int((~clear).sum())
                total += B
                assert torch.equal(idx.long()[clear], ridx[clear]), (G, M, k, b is None)
                assert torch.equal(pos.long(), slots(idx.long()))
                assert torch.equal(counts.long(), torch.bincount(idx.long()[idx >= 0], minlength=E_))
                same = (idx.long() == ridx).all(1, keepdim=True)
                assert float(torch.where(same, w.double() - rw.double(), 0.0).abs().max()) < 2e-6 * c, (G, M, k)
                assert E.max_groups_per_token(idx, k, E_, G) <= M
    assert unclear <= max(1e-2 * total, 16), (unclear, total)   # a few near-ties of a small batch are not a share


@pytest.mark.gpu
@pytest.mark.parametrize("grid", [(64,), (8, 8), (2, 3, 4), (64, 64)])
def test_identities_give_the_bits_of_the_ungrouped_gate(step_counters, grid):
    E_ = math.prod(grid)
    gen = torch.Generator(device="cuda").manual_seed(E_)
    logits = torch.randn(999, sum(grid), generator=gen, device="cuda")
    bias = torch.randn(E_, generator=gen, device="cuda") * 0.05
    alive = (torch.rand(E_, generator=gen, device="cuda") > 0.2).to(torch.uint8)
    for score, scale in (("softmax", 1.0), ("sigmoid", 2.5)):
        for b in (None, bias):
            for k in (1, 5, 8):
                ref = run_gate(logits, grid, k, alive=alive, rate=0.1, bias=b, score=score, scale=scale)
                for G, M in ((1, 1), (2, 2), (E_ // 4 if E_ // 4 <= 64 else 64, None)):
                    M = G if M is None else M
                    got = run_gate(logits, grid, k, alive=alive, rate=0.1, bias=b, score=score, scale=scale,
                                   n_group=G, topk_group=M)
                    assert all(torch.equal(x, y) for x, y in zip(got, ref) if x is not None), (score, G, M, k)


@pytest.mark.gpu
def test_wrappers_refuse_bad_groupings_before_launching(step_counters):
    from lah_b200.ops import native
    lg = torch.zeros(4, 16, device="cuda")
    i = torch.zeros(64, dtype=torch.int32, device="cuda")
    ok = dict(idx=i, w=i.float(), pos=i, counts=torch.zeros(16, dtype=torch.int32, device="cuda"))
    before = native.launches()
    for kw in (dict(n_group=0), dict(n_group=3), dict(n_group=32), dict(n_group=True), dict(n_group=4.0),
               dict(n_group=4, topk_group=0), dict(n_group=4, topk_group=5), dict(n_group=4, topk_group=True),
               dict(n_group=65, topk_group=1)):
        with pytest.raises(ValueError):
            K.gate_topk(lg, (16,), 4, **ok, **kw)
    big = torch.zeros(4, 64 + 128, device="cuda")
    with pytest.raises(ValueError, match="at most"):
        K.gate_topk(big, (64, 128), 4, idx=i, w=i.float(), pos=i,
                    counts=torch.zeros(64 * 128, dtype=torch.int32, device="cuda"), n_group=2, topk_group=1)
    assert native.launches() == before


def _check(r):
    """no token beyond its topk_group groups, the weights of the tokens routed alike and, when every token is, the
    oracle's bias update"""
    cfg = r.layer.cfg
    assert E.max_groups_per_token(r.idx, cfg.k, cfg.num_experts, cfg.n_group) <= cfg.topk_group
    assert float((r.w - r.rw)[r.same].abs().max()) < 2e-6 * cfg.routed_scaling_factor
    if bool(r.same.all()):
        assert torch.equal(r.layer.expert_bias, r.oracle.expert_bias)


@pytest.mark.gpu
@pytest.mark.parametrize("gate", ["emulator", "product_key"])
@pytest.mark.parametrize("expert", ["ffn", "swiglu"])
@pytest.mark.parametrize("path", ["small", "big"])
def test_layer_against_the_cpu_oracle(path, expert, gate):
    """softmax gate with expert biases: the keys s + b are the same float32 sums on both sides, so routing is exact"""
    torch.manual_seed(3)
    grid = (16,) if gate == "emulator" else (4, 4)
    cfg = E.DMoEConfig(hidden=512, grid_size=grid, k=4, num_layers=1, tokens_per_rank=512, expert=expert,
                       expert_path=path, gate_mode=gate, expert_bias_update_rate=0.01, n_group=4, topk_group=2)
    layer_against_the_oracle(cfg, max_mismatch=0, check=_check)


@pytest.mark.gpu
@pytest.mark.parametrize("path", ["small", "big"])
def test_deepseek_v3_shaped_layer_against_the_cpu_oracle(path):
    """64 SwiGLU experts in 8 groups, 4 groups per token, k = 8, sigmoid router with biases and c = 2.5, a shared expert"""
    torch.manual_seed(4)
    cfg = E.DMoEConfig(hidden=512, grid_size=(8, 8), k=8, num_layers=1, tokens_per_rank=512, expert="swiglu",
                       inner_dim=256, shared_inner_dim=512, expert_path=path, expert_bias_update_rate=1e-3,
                       router_aux_loss_coef=1e-2, routed_scaling_factor=2.5, n_group=8, topk_group=4, **SIG)
    layer_against_the_oracle(cfg, max_mismatch=2, check=_check)


def _trainer_cfg(path, **kw):
    base = dict(hidden=512, grid_size=(16,), k=4, num_layers=2, tokens_per_rank=256, failure_rate=0.1, lr=1e-4,
                expert_path=path, gate_mode="product_key", expert_bias_update_rate=1e-3, routed_scaling_factor=2.5,
                router_aux_loss_coef=1e-2, **SIG)
    base.update(kw)
    return E.DMoEConfig(**base)


@pytest.mark.gpu
@pytest.mark.parametrize("path", ["small", "big"])
def test_trainer_graph_equals_eager_and_launches_as_many_kernels(path):
    cfg = _trainer_cfg(path, n_group=4, topk_group=2)
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
        assert all(1 <= layer["max_groups_per_token"] <= 2 for layer in rec["layers"]), rec["layers"]
        runs[run] = (torch.stack(losses).cpu(), torch.stack(biases).cpu(),
                     torch.cat([b.shard.p for b in t.model.blocks] + [t.flat_p]).cpu())
        if graph:
            runs[run + "_launches"] = t._graph_launches
        t.close()
    for a, b in zip(runs["eager"], runs["graph"]):
        assert torch.equal(a, b)
    for a, b in zip(runs["graph"], runs["graph2"]):
        assert torch.equal(a, b)
    plain = DMoETrainer(_trainer_cfg(path), use_graph=True)
    for x, y in zip(xs[:3], ys[:3]):
        plain.train_step_device(x, y)
    assert plain._graph_launches == runs["graph_launches"]
    assert all("max_groups_per_token" not in layer for layer in plain.log_step()["layers"])
    plain.close()
