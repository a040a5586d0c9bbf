"""
Expert capacity (DESIGN.md §6f, Switch / GShard capacity factor): DMoEConfig(expert_capacity_factor=f).  Each forward,
expert e keeps at most C = max(1, ceil(f * P / E)) of the P box-wide routed pairs, in rank-major then token order; a
dropped pair sees its expert as the identity.

CPU: the config, the capacity formula, the CPU layer's drops, gradients, router losses, optimizer gating and trainer.
GPU: layout_exchange, scatter_rows, combine_rows and gate_bwd against their oracles, the layer against the CPU oracle
under collapsed routing, bit-identity with f = 0 when nothing drops, graph replay, launch counts, and (two GPUs) the
sharded layer against the whole-batch oracle.
"""
import math
import os
import subprocess
import sys
import zlib

import pytest
import torch

import lah_b200  # noqa: F401
from lah_b200.ops import kernels as K
from lah_b200.parallel import baseline, engine as E
from lah_b200.parallel.trainer import DMoETrainer
from routing_support import F64, cpu_cfg, layer_against_the_oracle, rel
from routing_support import one_thread, rt, world1  # noqa: F401 (fixtures)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BF16 = torch.bfloat16


# ======================================================================================================== CPU: config
def test_default_is_dropless_and_bad_factors_are_refused():
    assert E.DMoEConfig().expert_capacity_factor == 0.0
    for f in (-1.0, -1e-9, float("inf"), float("-inf"), float("nan")):
        with pytest.raises(ValueError, match="expert_capacity_factor"):
            E.DMoEConfig(expert_capacity_factor=f)
    E.DMoEConfig(expert_capacity_factor=1e-6)


@pytest.mark.parametrize("arm", ["BaselineDMoE", "BaselineTrainer", "FastBaselineDMoE", "FastBaselineTrainer"])
def test_baseline_arms_refuse_a_capacity(arm):
    from lah_b200.parallel import baseline_fast
    cfg = E.DMoEConfig(hidden=64, grid_size=(4,), k=2, num_layers=1, tokens_per_rank=8, expert_capacity_factor=1.0)
    make = dict(BaselineDMoE=lambda: baseline.BaselineDMoE(cfg), BaselineTrainer=lambda: baseline.BaselineTrainer(cfg),
                FastBaselineDMoE=lambda: baseline_fast.FastBaselineDMoE(cfg, 0, 16),
                FastBaselineTrainer=lambda: baseline_fast.FastBaselineTrainer(cfg))[arm]
    with pytest.raises(ValueError, match="expert_capacity_factor"):
        make()


@pytest.mark.parametrize("f,P,E_,C", [
    (1.0, 1024, 64, 16), (1.25, 1000, 64, 20), (1.0, 1001, 64, 16), (2.0, 1, 64, 1), (1.0, 0, 64, 1),
    (1e-9, 4096, 64, 1), (0.5, 7, 4, 1), (1.5, 7, 4, 3), (64.0, 1024, 64, 1024), (1.0, 8 * 65536 * 8, 4096, 1024),
    (0.1, 3, 1, 1), (3.0, 10, 3, 10), (1e30, 5, 2, K.CAPACITY_MAX),
])
def test_capacity_formula(f, P, E_, C):
    """C = max(1, ceil((f * P) / E)) in float64, with the floor of one row"""
    assert K.expert_capacity(f, P, E_) == C
    assert C == min(K.CAPACITY_MAX, max(1, math.ceil((f * P) / E_)))


def test_capacity_ref_priority_is_rank_major():
    cnt = torch.tensor([[3, 0, 5, 2], [4, 1, 0, 2], [1, 1, 1, 9]])
    r = K.expert_capacity_ref(cnt, 1.0)   # P = 29, C = ceil(29 / 4) = 8
    assert r["capacity"] == 8
    assert r["kept"].tolist() == [[3, 0, 5, 2], [4, 1, 0, 2], [1, 1, 1, 4]]
    assert r["dropped"] == 5
    kept, C, dropped = K.capacity_keep_ref(torch.tensor([[0, 1], [0, 2], [0, 1], [-1, 0]]), 0.5, 4)
    assert C == 1 and dropped == 4   # P = 7, C = ceil(3.5 / 4) = 1
    assert kept.tolist() == [[True, True], [False, True], [False, False], [False, False]]


# ======================================================================================================== CPU: layer
def _run_ref(layer, x, logits, gy):
    x = x.clone().requires_grad_(True)
    lg = logits.clone().requires_grad_(True)
    out = layer._forward_ref(x, lg)
    (out * gy).sum().backward()
    grads = {(le, n): leaf.grad.clone() for le, leaves in layer._ref_leaves.items() for n, leaf in leaves.items()
             if leaf.grad is not None}
    layer.apply_expert_gradients_ref()
    return out.detach(), x.grad, lg.grad, grads, layer.shard.p.clone()


@pytest.mark.parametrize("expert", ["ffn", "swiglu"])
def test_a_factor_that_drops_nothing_is_identical_to_dropless(expert):
    torch.manual_seed(0)
    cfgs = [cpu_cfg(expert=expert, expert_capacity_factor=f) for f in (0.0, 64.0)]
    layers = [E.FusedDMoE(c).train() for c in cfgs]
    layers[1].load_state_dict(layers[0].state_dict())
    layers[1].shard.p.copy_(layers[0].shard.p)
    x, gy = torch.randn(48, 64), torch.randn(48, 64)
    logits = layers[0].gate_logits(x, layers[0].proj).detach()
    a, b = (_run_ref(l, x, logits, gy) for l in layers)
    assert layers[1]._ref_capacity[1] == 0
    for ta, tb in zip(a[:3] + (a[4],), b[:3] + (b[4],)):
        assert torch.equal(ta, tb)
    assert a[3].keys() == b[3].keys() and all(torch.equal(a[3][n], b[3][n]) for n in a[3])


def test_top1_capacity_one_returns_later_tokens_unchanged():
    """k = 1, C = 1, softmax router: the first token of each expert goes through it, every later one returns exactly x"""
    torch.manual_seed(1)
    layer = E.FusedDMoE(cpu_cfg(grid_size=(8,), k=1, expert_capacity_factor=1e-9)).eval()
    x = torch.randn(40, 64)
    with torch.no_grad():
        y = layer(x)
        idx, _ = K.gate_topk_ref(layer.gate_logits(x, layer.proj), (8,), 1)
    first, seen = torch.zeros(40, dtype=torch.bool), set()
    for b, e in enumerate(idx[:, 0].tolist()):
        first[b] = e not in seen
        seen.add(e)
    assert layer._ref_capacity == (1, 40 - len(seen))
    assert torch.equal(y[~first], x[~first])
    assert bool(((y[first] - x[first]).abs().amax(1) > 0).all())


def _identity_formula(layer, x, logits, kept, idx, score, norm, scale):
    """float64 layer output with an explicit identity for the dropped pairs: sum_j w_j (kept ? expert_j(x) : x)"""
    scores = K.product_key_scores(logits, layer.grid_size)
    valid = idx >= 0
    sel = torch.gather(scores, 1, idx.clamp(min=0))
    if score == "softmax" and norm:
        w = torch.softmax(sel.masked_fill(~valid, float("-inf")), -1)
    elif score == "softmax":
        w = K.softmax_weights_ref(scores, idx, None, scale)
    elif norm:
        w = K.sigmoid_weights_ref(sel, valid, scale)
    else:
        w = scale * torch.sigmoid(sel)
    w = torch.where(valid, w, torch.zeros_like(w))
    out = torch.zeros_like(x)
    for j in range(idx.shape[1]):
        for b in range(x.shape[0]):
            e = int(idx[b, j])
            if e < 0:
                continue
            if kept[b, j]:
                p = {n: v.double() for n, v in layer._expert_params(e, torch.float64).items()}
                yb = layer._expert_ref(p, x[b:b + 1], lambda t: t)[0]
            else:
                yb = x[b]
            out = out.index_add(0, torch.tensor([b]), (w[b, j] * yb).unsqueeze(0))
    return out


@pytest.mark.parametrize("norm", [True, False])
@pytest.mark.parametrize("score", ["softmax", "sigmoid"])
def test_cpu_layer_gradients_with_drops_equal_the_identity_formula(score, norm):
    torch.manual_seed(2)
    scale = 1.0 if score == "softmax" and norm else 2.5
    cfg = cpu_cfg(k=2, tokens_per_rank=32, router_score=score, norm_topk_prob=norm, routed_scaling_factor=scale,
                  expert_capacity_factor=0.75)
    layer = E.FusedDMoE(cfg).eval()   # eval: the leaves of the expert parameters are not created
    x = torch.randn(24, 64)
    with torch.no_grad():
        layer.proj.bias[:4] += torch.tensor([2.0, 0.0, 0.0, 0.0])   # a hot row of the grid: drops
    proj_w = layer.proj.weight.detach().clone().requires_grad_(True)
    xr = x.clone().requires_grad_(True)
    out = layer._forward_ref(xr, torch.nn.functional.linear(xr, proj_w, layer.proj.bias.detach()))
    gy = torch.randn_like(out)
    (out * gy).sum().backward()
    C, dropped = layer._ref_capacity
    assert dropped > 0
    xd = x.double().requires_grad_(True)
    pw = proj_w.detach().double().requires_grad_(True)
    lg = torch.nn.functional.linear(xd, pw, layer.proj.bias.detach().double())
    idx, _ = K.gate_topk_ref(lg.detach().float(), cfg.grid_size, cfg.k, score=score, scale=scale, norm=norm)
    kept, C2, dropped2 = K.capacity_keep_ref(idx, cfg.expert_capacity_factor, cfg.num_experts)
    assert (C2, dropped2) == (C, dropped)
    ref = _identity_formula(layer, xd, lg, kept, idx, score, norm, scale)
    (ref * gy.double()).sum().backward()
    assert rel(out, ref, *F64) < 1e-5
    errs = rel(xr.grad, xd.grad, *F64), rel(proj_w.grad, pw.grad, *F64)
    assert errs[0] < 1e-5 and errs[1] < 1e-5, errs


def test_router_losses_see_the_routed_counts():
    torch.manual_seed(3)
    losses = []
    for f in (0.0, 0.25):
        torch.manual_seed(3)
        layer = E.FusedDMoE(cpu_cfg(router_aux_loss_coef=0.01, router_z_loss_coef=1e-3, expert_capacity_factor=f)).train()
        with torch.no_grad():
            layer.proj.bias[:4] += torch.tensor([3.0, 0.0, 0.0, 0.0])
        layer(torch.randn(64, 64, generator=torch.Generator().manual_seed(0)))
        losses.append(layer.router_loss.clone())
        if f:
            assert layer._ref_capacity[1] > 0
    assert torch.equal(losses[0], losses[1])


def test_experts_step_on_kept_rows_only():
    """C = 1 on a gate that sends everything to one grid row: only the experts with a kept row are stepped, once"""
    torch.manual_seed(4)
    layer = E.FusedDMoE(cpu_cfg(k=1, expert_capacity_factor=1e-9)).train()
    x = torch.randn(32, 64)
    (layer(x) * torch.randn(32, 64)).sum().backward()
    idx, _ = K.gate_topk_ref(layer.gate_logits(x, layer.proj).detach(), layer.grid_size, 1)
    rows = layer._ref_rows.clone()
    assert torch.equal(rows, (torch.bincount(idx.flatten(), minlength=16) > 0).long())
    before = layer.shard.p.clone()
    layer.apply_expert_gradients_ref()
    assert torch.equal(layer.shard.step, rows.to(layer.shard.step.dtype))
    moved = (layer.shard.p - before).view(-1) != 0
    assert bool(moved.any())


def test_cpu_trainer_learns_and_resumes(one_thread):
    gen = torch.Generator().manual_seed(6)
    xs = [torch.randn(64, 16, generator=gen) for _ in range(12)]
    ys = [(x[:, 0] > 0).long() for x in xs]
    cfg = cpu_cfg(num_layers=2, expert_capacity_factor=1.0, lr=3e-3)
    torch.manual_seed(0)
    a = DMoETrainer(cfg)
    losses = [a.train_step(x, y) for x, y in zip(xs[:8], ys[:8])]
    assert losses[-1] < losses[0], losses
    state = a.state_dict()
    plain = DMoETrainer(cpu_cfg(num_layers=2))   # checkpoints load across the setting
    plain.load_state_dict(state)
    b = DMoETrainer(cfg)
    b.load_state_dict(plain.state_dict())
    la = [a.train_step(x, y) for x, y in zip(xs[8:], ys[8:])]
    lb = [b.train_step(x, y) for x, y in zip(xs[8:], ys[8:])]
    assert la == lb


# ======================================================================================================== GPU: kernels
def _counts(kind, gen):
    if kind == "sparse":
        return (torch.randint(0, 40, (64,), generator=gen) * (torch.rand(64, generator=gen) > 0.5)).to(torch.int32)
    if kind == "hot":
        c = torch.zeros(16, dtype=torch.int32)
        c[5], c[0], c[15] = 1000, 3, 17
        return c
    if kind == "e4096":
        return torch.randint(0, 3, (K.LAYOUT_MAX_E,), generator=gen).to(torch.int32)
    return torch.zeros(32, dtype=torch.int32)


CANARY = -777


def _canaried(n, fill=4242):
    t = torch.full((n + 8,), CANARY, dtype=torch.int32, device="cuda")
    t[:n] = fill
    return t


@pytest.mark.gpu
@pytest.mark.parametrize("f", [0.5, 1.0, 1.25, 64.0])
@pytest.mark.parametrize("kind", ["sparse", "hot", "e4096", "empty"])
@pytest.mark.parametrize("align,tile_rows", [(16, 16), (128, 128), (256, 128)])
def test_layout_exchange_with_capacity_matches_the_oracle(rt, align, tile_rows, kind, f):
    """every table follows the kept counts; keep, C and the dropped pairs exact; canaries intact; no overflow with the
    buffer sized for the kept rows"""
    gen = torch.Generator().manual_seed(zlib.crc32(repr((align, kind, f)).encode()))
    counts = _counts(kind, gen)
    E_ = counts.numel()
    cap = K.expert_capacity_ref(counts.view(1, -1), f)
    kept = cap["kept"][0]
    padded = (kept + align - 1) // align * align
    off = torch.cumsum(padded, 0) - padded
    total = int(padded.sum())
    max_rows = total + 2 * align
    max_tiles = max_rows // tile_rows
    tile_group = torch.full((max_tiles,), -1, dtype=torch.long)
    tiles = torch.repeat_interleave(torch.arange(E_), padded // tile_rows)
    tile_group[: len(tiles)] = tiles
    ref = dict(dst_row=off, group_off=torch.cat([off, torch.tensor([total])]), group_rows=kept, tile_group=tile_group,
               total_rows=torch.tensor([total]), step_rows=kept, route_owner=torch.zeros(E_, dtype=torch.long),
               keep=kept, capacity_stats=torch.tensor([cap["capacity"], cap["dropped"]]))
    out = dict(dst_row=_canaried(E_), group_off=_canaried(E_ + 1), group_rows=_canaried(E_), tile_group=_canaried(max_tiles),
               total_rows=_canaried(1), step_rows=_canaried(E_), route_owner=_canaried(E_),
               owned_shadow=_canaried(2 * E_), keep=_canaried(E_), capacity_stats=_canaried(2))
    cnt = counts.cuda()
    rt.step_ctr[0] = 1 << 20
    K.layout_exchange(rt.cnt_all_off, rt.flags_off, K.SLOT_COUNTS, 3, E_, E_, max_rows, align=align,
                      tile_rows=tile_rows, counts=cnt, status=rt.status, shadow_slots=0, capacity_factor=f, **out)
    torch.cuda.synchronize()
    for name, t in out.items():
        n = t.numel() - 8
        assert bool((t[n:] == CANARY).all()), f"{name}: canary overwritten"
        if name != "owned_shadow":
            assert torch.equal(t[:n].long().cpu(), ref[name]), name
    assert torch.equal(rt.cnt_all[0, :E_].cpu(), counts), "the routed counts stay in the table"
    assert bool((cnt == 0).all())
    assert int(rt.status[0]) == 0


@pytest.mark.gpu
def test_layout_exchange_refuses_inconsistent_capacity_arguments(rt):
    i = torch.zeros(16, dtype=torch.int32, device="cuda")
    kw = dict(counts=i, dst_row=i, group_off=i, group_rows=i, tile_group=i, total_rows=i, status=rt.status)
    for extra in (dict(capacity_factor=1.0), dict(capacity_factor=0.0, keep=i, capacity_stats=i),
                  dict(capacity_factor=-1.0, keep=i, capacity_stats=i),
                  dict(capacity_factor=float("nan"), keep=i, capacity_stats=i)):
        with pytest.raises(ValueError):
            K.layout_exchange(rt.cnt_all_off, rt.flags_off, K.SLOT_COUNTS, 1, 4, 4, 64, **kw, **extra)


@pytest.mark.gpu
@pytest.mark.parametrize("H,align", [(256, 16), (512, 128), (1024, 256)])
def test_scatter_rows_drops_exactly_the_pairs_past_keep(rt, H, align):
    gen = torch.Generator().manual_seed(H)
    B, k, E_ = 301, 4, 16
    idx = torch.argsort(torch.rand(B, E_, generator=gen), dim=1)[:, :k]
    idx[torch.rand(B, k, generator=gen) < 0.1] = -1
    idx[:200, 0] = 3   # a hot expert
    kept_mask, C, _ = K.capacity_keep_ref(idx, 0.6, E_)
    flat = idx.flatten()
    key = torch.where(flat >= 0, flat, torch.full_like(flat, E_))
    order = torch.sort(key, stable=True).indices
    pos = torch.empty_like(flat)
    pos[order] = torch.arange(flat.numel()) - torch.searchsorted(key[order], key[order])
    pos[flat < 0] = 0
    keep = torch.bincount(flat[kept_mask.flatten()], minlength=E_)
    padded = (keep + align - 1) // align * align
    off = torch.cumsum(padded, 0) - padded
    max_rows = int(padded.sum()) + align
    row = torch.where(kept_mask.flatten(), off[flat.clamp(min=0)] + pos, torch.full_like(pos, -1))
    buf = rt.region[: (max_rows + 64) * H * 2].view(BF16).view(max_rows + 64, H)
    buf.copy_(torch.randn(max_rows + 64, H, generator=gen).to(BF16))
    before = buf.cpu().clone()
    src = torch.randn(B, H, generator=gen).to(BF16).cuda()
    d = lambda t: t.to(torch.int32).cuda()   # noqa: E731
    pair_row = torch.full((B * k,), 999999, dtype=torch.int32, device="cuda")
    rt.step_ctr[0] = 5000
    K.scatter_rows(src, None, d(flat), d(pos), d(off), pair_row, rt.region_off, rt.flags_off, K.SLOT_DISPATCH, 7, k, E_,
                   max_rows, d(torch.cat([off, padded.sum().view(1)])), d(keep), rt.done_counter, rt.status, align=align,
                   route_owner=torch.zeros(E_, dtype=torch.int32, device="cuda"), num_groups=E_, keep=d(keep))
    torch.cuda.synchronize()
    assert torch.equal(pair_row.long().cpu(), row)
    exp = before.clone()
    p = torch.nonzero(row >= 0).squeeze(1)
    exp[row[p]] = src.cpu()[p // k]
    for e in range(E_):
        exp[int(off[e] + keep[e]):int(off[e] + padded[e])] = 0
    assert torch.equal(buf.cpu().view(torch.int16), exp.view(torch.int16))
    assert int(rt.status[0]) == 0 and int(rt.flags[K.SLOT_DISPATCH, 0]) == 5007


def _bf16_ulp(x):
    _, e = torch.frexp(x.abs().clamp(min=2.0 ** -126))
    return torch.pow(2.0, (e - 8).to(x.dtype))


@pytest.mark.gpu
@pytest.mark.parametrize("addend", [False, True])
@pytest.mark.parametrize("weighted", [True, False])
@pytest.mark.parametrize("H", [256, 512, 1024])
@pytest.mark.parametrize("k", [1, 4, 8])
def test_pass_through_combine_matches_the_oracle(rt, k, H, weighted, addend):
    gen = torch.Generator().manual_seed(k * H + 2 * weighted + addend)
    B, E_ = 333, 16
    R = B * k + 100
    idx = torch.argsort(torch.rand(B, E_, generator=gen), dim=1)[:, :k]
    idx[torch.rand(B, k, generator=gen) < 0.15] = -1
    pair_row = torch.randperm(R, generator=gen)[: B * k].view(B, k)
    pair_row[torch.rand(B, k, generator=gen) < 0.3] = -1   # dropped pairs
    pair_row = torch.where(idx >= 0, pair_row, torch.full_like(pair_row, -1))
    src = rt.region[: R * H * 2].view(BF16).view(R, H)
    src.copy_(torch.randn(R, H, generator=gen).to(BF16))
    w = torch.rand(B, k, generator=gen)
    selfr = torch.randn(B, H, generator=gen).to(BF16)
    add = torch.randn(B, H, generator=gen).to(BF16) if addend else None
    out = torch.full((B, H), 3.0, dtype=BF16, device="cuda")
    K.combine_rows(rt.region_off, idx.flatten().to(torch.int32).cuda(), pair_row.flatten().to(torch.int32).cuda(),
                   w.flatten().cuda() if weighted else None, out, k, E_, addend=add.cuda() if addend else None,
                   pass_self=selfr.cuda(), pass_w=w.flatten().cuda())
    torch.cuda.synchronize()
    ref = K.combine_rows_ref(src.cpu(), idx, pair_row, w if weighted else None, add, selfr, w).double()
    exact = (K.combine_rows_ref(src.cpu().double(), idx, pair_row, w if weighted else None,
                                add.double() if addend else None, selfr.double(), w))
    present = ((idx >= 0) & (pair_row >= 0)).double() * (w.double() if weighted else 1.0)
    mag = (src.cpu().double()[pair_row.clamp(min=0)].abs() * present.unsqueeze(-1)).sum(1) + \
        ((idx >= 0) & (pair_row < 0)).double().mul(w.double()).sum(1, keepdim=True) * selfr.double().abs()
    tol = _bf16_ulp(exact.double()) + (k + 1) * 2.0 ** -23 * mag
    err = (out.cpu().double() - ref).abs()
    assert bool((err <= tol).all()), float((err / _bf16_ulp(exact.double())).max())
    assert torch.equal(ref, exact.double())


def _to_logits(ds, grid):
    """gradient of the grid logits from per-expert score gradients (score = sum of one logit per dim)"""
    B = ds.shape[0]
    out, rem, off = [], torch.arange(math.prod(grid)), 0
    coords = []
    for size in reversed(grid):
        coords.append(rem % size)
        rem = rem // size
    coords = coords[::-1]
    for d, size in enumerate(grid):
        out.append(torch.zeros(B, size, dtype=ds.dtype).index_add(1, coords[d], ds))
    return torch.cat(out, 1)


@pytest.mark.gpu
@pytest.mark.parametrize("norm", [True, False])
@pytest.mark.parametrize("score", ["softmax", "sigmoid"])
@pytest.mark.parametrize("k", [1, 4])
@pytest.mark.parametrize("grid,H", [((64,), 256), ((4, 4), 512), ((2, 32), 1024)])
def test_pass_through_gate_bwd_matches_float64(rt, grid, H, k, score, norm):
    """dlogits of sum_j w_j <g, y_j> with y_j = x_b for a dropped pair, against float64 autograd, every weight mode"""
    gen = torch.Generator().manual_seed(zlib.crc32(repr((grid, H, k, score, norm)).encode()))
    B, E_ = 257, math.prod(grid)
    c = 1.0 if score == "softmax" and norm else 2.5
    logits = torch.randn(B, sum(grid), generator=gen, dtype=torch.float64)
    idx, _ = K.gate_topk_ref(logits.float(), grid, k, score=score, scale=c, norm=norm)
    idx[torch.rand(B, k, generator=gen) < 0.1] = -1
    valid = idx >= 0
    R = B * k + 50
    pair_row = torch.randperm(R, generator=gen)[: B * k].view(B, k)
    pair_row[torch.rand(B, k, generator=gen) < 0.3] = -1
    pair_row = torch.where(valid, pair_row, torch.full_like(pair_row, -1))
    yo = rt.region[: R * H * 2].view(BF16).view(R, H)
    yo.copy_(torch.randn(R, H, generator=gen).to(BF16))
    g = torch.randn(B, H, generator=gen).to(BF16)
    x = torch.randn(B, H, generator=gen).to(BF16)
    lg = logits.clone().requires_grad_(True)
    scores = K.product_key_scores(lg, grid)
    sel = torch.gather(scores, 1, idx.clamp(min=0))
    if score == "softmax" and norm:
        wts = torch.softmax(sel.masked_fill(~valid, float("-inf")), -1)
    elif score == "softmax":
        wts = K.softmax_weights_ref(scores, idx, None, c)
    elif norm:
        wts = K.sigmoid_weights_ref(sel, valid, c)
    else:
        wts = c * torch.sigmoid(sel)
    wts = torch.where(valid, wts, torch.zeros_like(wts)).nan_to_num(0.0)
    y = torch.where((pair_row >= 0).unsqueeze(-1), yo.cpu().double()[pair_row.clamp(min=0)],
                    x.double().unsqueeze(1).expand(B, k, H))
    (wts * (g.double().unsqueeze(1) * y).sum(-1)).sum().backward()
    kw = {}
    if score == "sigmoid":
        kw = dict(score="sigmoid", scale=c, sig=(torch.sigmoid(sel.detach()) * valid).float().flatten().cuda())
    if not norm:
        kw.update(norm=False, scale=c)
        if score == "softmax":
            kw.update(lse=K.softmax_lse_ref(scores.detach()).float().cuda(), logits=logits.float().cuda())
    dl = torch.full((B, sum(grid)), 5.0, device="cuda")
    K.gate_bwd(rt.region_off, g.cuda(), idx.flatten().to(torch.int32).cuda(), pair_row.flatten().to(torch.int32).cuda(),
               wts.detach().float().flatten().cuda(), dl, k, E_, grid, pass_x=x.cuda(), **kw)
    torch.cuda.synchronize()
    # relative to the largest term w_j dw_j: at k = 1 a normalised weight is constant and the gradient is zero up to
    # rounding
    terms = (wts.detach() * (g.double().unsqueeze(1) * y).sum(-1)).abs().max()
    err = float((dl.cpu().double() - lg.grad).abs().max() / terms)
    assert err < 1e-5, err


# ======================================================================================================== GPU: layer
def _collapse(layer):
    """bias the gate so that most tokens pick experts of the first grid row (the first rank's at world > 1)"""
    cfg = layer.cfg
    if cfg.gate_mode == "emulator":
        layer.expert_keys[:, : cfg.num_experts // 4] += 0.5 * layer.expert_keys.abs().mean()
    else:
        layer.proj.bias[0] += 3.0


def _check(r):
    """the capacity and the dropped pairs of the oracle, pass-through rows for the dropped pairs, and the experts the
    oracle's update steps and moves"""
    cfg, B = r.layer.cfg, r.idx.shape[0]
    r.oracle.apply_expert_gradients_ref()
    C, dropped = r.layer.ws.capacity_stats.tolist()
    assert (C, dropped) == r.oracle._ref_capacity and dropped > 0, ((C, dropped), r.oracle._ref_capacity)
    kept, _, _ = K.capacity_keep_ref(r.idx, cfg.expert_capacity_factor, cfg.num_experts)
    pr = r.layer.ws.pair_row[:B * cfg.k].view(B, cfg.k).cpu()
    assert torch.equal(pr[~kept.cpu() & (r.idx.cpu() >= 0)], torch.full_like(pr[~kept.cpu() & (r.idx.cpu() >= 0)], -1))
    assert bool((pr[kept.cpu()] >= 0).all())
    assert torch.equal(r.layer.shard.step.cpu(), r.oracle.shard.step.cpu())
    params_mean_abs = float((r.layer.shard.p[:r.oracle.shard.p.numel()] - r.oracle.shard.p).abs().mean())
    assert params_mean_abs < 1e-4, params_mean_abs


@pytest.mark.gpu
@pytest.mark.parametrize("score", ["softmax", "sigmoid"])
@pytest.mark.parametrize("expert", ["ffn", "swiglu"])
@pytest.mark.parametrize("path", ["small", "big"])
def test_collapsed_layer_matches_the_cpu_oracle(path, expert, score):
    torch.manual_seed(3)
    extra = dict(routed_scaling_factor=2.5) if score == "sigmoid" else {}
    cfg = E.DMoEConfig(hidden=512, grid_size=(4, 4), k=4, num_layers=1, tokens_per_rank=512, expert=expert,
                       expert_path=path, router_score=score, expert_capacity_factor=1.0, **extra)
    layer_against_the_oracle(cfg, prepare=_collapse, dx=True, precision=F64, check=_check)


@pytest.mark.gpu
@pytest.mark.parametrize("path", ["small", "big"])
def test_collapsed_layer_with_a_shared_expert_matches_the_cpu_oracle(path):
    torch.manual_seed(4)
    cfg = E.DMoEConfig(hidden=512, grid_size=(4, 4), k=4, num_layers=1, tokens_per_rank=512, expert="swiglu",
                       shared_inner_dim=256, expert_path=path, expert_capacity_factor=1.25, norm_topk_prob=False)
    layer_against_the_oracle(cfg, prepare=_collapse, dx=True, precision=F64, check=_check)


def _trainer_cfg(path, **kw):
    base = dict(hidden=512, grid_size=(16,), k=4, num_layers=2, tokens_per_rank=256, lr=1e-4, expert_path=path,
                gate_mode="emulator")
    base.update(kw)
    return E.DMoEConfig(**base)


def _trainer_run(cfg, graph, steps=4):
    torch.manual_seed(0)
    gen = torch.Generator().manual_seed(1)
    xs = [torch.randn(256, cfg.in_features, generator=gen).cuda() for _ in range(steps)]
    ys = [torch.randint(0, 10, (256,), generator=gen).cuda() for _ in range(steps)]
    t = DMoETrainer(cfg, use_graph=graph)
    losses = torch.stack([t.train_step_device(x, y).clone() for x, y in zip(xs, ys)]).cpu()
    t.ctx.check_status()
    rec = t.log_step()
    params = torch.cat([b.shard.p for b in t.model.blocks] + [t.flat_p]).cpu()
    launches = t._graph_launches if graph else None
    t.close()
    return losses, params, rec, launches


@pytest.mark.gpu
@pytest.mark.parametrize("path", ["small", "big"])
def test_a_factor_that_drops_nothing_trains_bit_identically(path):
    a = _trainer_run(_trainer_cfg(path), graph=False)
    b = _trainer_run(_trainer_cfg(path, expert_capacity_factor=64.0), graph=False)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])
    C = K.expert_capacity(64.0, 256 * 4, 16)
    assert all(layer["dropped_pairs"] == 0 and layer["expert_capacity"] == C for layer in b[2]["layers"])


@pytest.mark.gpu
@pytest.mark.parametrize("m", [1, 2])
@pytest.mark.parametrize("path", ["small", "big"])
def test_graph_equals_eager_reproducibly_with_the_launches_of_dropless(path, m):
    cfg = _trainer_cfg(path, expert_capacity_factor=1.0, trainer_microbatches=m, failure_rate=0.1,
                       expert_bias_update_rate=1e-3)
    eager = _trainer_run(cfg, graph=False)
    g1, g2 = _trainer_run(cfg, graph=True), _trainer_run(cfg, graph=True)
    for a, b in zip(eager[:2], g1[:2]):
        assert torch.equal(a, b)
    for a, b in zip(g1[:2], g2[:2]):
        assert torch.equal(a, b)
    assert all(layer["expert_capacity"] >= 1 for layer in g1[2]["layers"])
    plain = _trainer_run(_trainer_cfg(path, trainer_microbatches=m, failure_rate=0.1, expert_bias_update_rate=1e-3),
                         graph=True)
    assert g1[3] == plain[3]


@pytest.mark.gpu
def test_layer_refuses_a_context_of_the_other_setting():
    cfg = E.DMoEConfig(hidden=512, grid_size=(16,), k=4, num_layers=1, tokens_per_rank=256)
    ctx = E.EngineContext(cfg)
    try:
        assert E.FusedDMoE(cfg, ctx).ws.keep is None
        with pytest.raises(ValueError, match="expert_capacity_factor"):
            E.FusedDMoE(E.DMoEConfig(**{**cfg.__dict__, "expert_capacity_factor": 1.0}), ctx)
    finally:
        ctx.close()


# ======================================================================================================== two GPUs
@pytest.mark.gpu
@pytest.mark.parametrize("mode", [["--small"], [], ["--force-shadow"]], ids=["small", "big", "big_shadow"])
def test_two_gpus_collapsed_routing_matches_the_whole_batch_oracle(mode):
    """every token routed to the first rank's experts at f = 1: no overflow, and y, dx, the gate gradient and the stepped
    experts equal the world-1 oracle on the concatenated batch under rank-major priority"""
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    out = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2",
                          "--master-addr", "127.0.0.1", "--master-port", "29561",
                          os.path.join(ROOT, "tools", "multi_gpu_check.py"), "--expert-capacity", *mode],
                         capture_output=True, text=True, timeout=600)
    assert out.returncode == 0 and "MULTI_GPU_OK" in out.stdout, out.stdout[-3000:] + out.stderr[-3000:]
