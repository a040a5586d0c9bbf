"""torchrun -n W: the fused P2P engine on W GPUs must reproduce the single-GPU engine on the concatenated batch.

Every rank feeds a different slice of one global batch; rank r hosts experts [r*E/W, (r+1)*E/W).  We compare, for one
DMoE layer: outputs y, input gradients dx, gate gradients, and the expert parameters after the optimizer step, against a
single-process run of the SAME layer code over the whole batch (world=1 path, all experts local)."""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import torch.distributed as dist
import torch.nn.functional as F

import lah_b200  # noqa
from lah_b200.ops import kernels as K
from lah_b200.parallel import engine as E


def rel(a, b):
    return ((a.float() - b.float()).norm() / (b.float().norm() + 1e-12)).item()


def main():
    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    torch.cuda.set_device(int(os.environ["LOCAL_RANK"]))
    dist.init_process_group("nccl", device_id=torch.device("cuda", int(os.environ["LOCAL_RANK"])))
    B = 256
    force_shadow = "--force-shadow" in sys.argv  # shadow as many experts as there are slots (exercises the replica path)
    small = "--small" in sys.argv   # weight-streaming expert path (swap-AB GEMMs + fused wgrad/AMSGrad; no shadowing)
    swiglu = "--swiglu" in sys.argv   # GatedFeedforwardBlock experts (compares [W1; W3] and the RMSNorm weight)
    # router losses of the product-key gate: f from the box-wide count table, P from each rank's own tokens
    router = dict(router_aux_loss_coef=0.01, router_z_loss_coef=0.001) if "--router-loss" in sys.argv else {}
    # auxiliary-loss-free balancing: every rank moves its copy of the expert biases from the same box-wide count table
    bias = dict(expert_bias_update_rate=0.01) if "--expert-bias" in sys.argv else {}
    # a shared expert (trainer-side, replicated): its gradients summed over ranks against the whole-batch oracle, then
    # N trainer steps after which its parameters must hold the same bits on every rank
    shared = dict(shared_inner_dim=512) if "--shared-expert" in sys.argv else {}
    # group-limited routing with one group per rank (DESIGN.md §6d): every token's pairs must reach exactly one rank, and
    # the whole-batch oracle routes with the same limit
    group = dict(n_group=world, topk_group=1) if "--group-limited" in sys.argv else {}
    # expert capacity (DESIGN.md §6f) under collapsed routing: the gate sends every token to the first rank's experts, C =
    # P / E drops most pairs, and the whole-batch oracle drops the same ones under rank-major priority
    capacity = dict(expert_capacity_factor=1.0) if "--expert-capacity" in sys.argv else {}
    # SwiGLU experts with their forward GEMMs on MXFP8 operands: the receive-side wait before the quantising RMSNorm, and
    # (with --force-shadow) the re-quantisation of pulled replicas.  The oracle is fp32, so the bounds are those of
    # tools/gpu_layer_check.py for fp8 (3x)
    fp8 = dict(expert_dtype="fp8", inner_dim=1024) if "--fp8" in sys.argv else {}
    tol = 3.0 if fp8 else 1.0
    swiglu = swiglu or bool(shared) or bool(fp8)
    mat, vec = ("w13", "g") if swiglu else ("w1", "b2")
    cfg = E.DMoEConfig(hidden=512, grid_size=(4, 4), k=4, num_layers=1, tokens_per_rank=B, capacity_factor=float(max(4, world)),
                       shadow_experts=4, shadow_tol=0.0 if force_shadow else 1.1, shadow_min_rows=1 if force_shadow else 64,
                       expert_path="small" if small else "big", expert="swiglu" if swiglu else "ffn", **router, **bias, **shared,
                       **group, **capacity, **fp8)
    ctx = E.EngineContext(cfg)
    torch.manual_seed(0)  # identical gate on every rank (DMoETrainer does the same)
    layer = E.FusedDMoE(cfg, ctx).cuda()
    if capacity:   # the first grid coordinate picks the rank: coordinate 0 gets every token
        with torch.no_grad():
            layer.proj.bias[0] += 50.0
    gen = torch.Generator().manual_seed(0)
    x_all = torch.randn(world * B, 512, generator=gen).to(torch.bfloat16)
    g_all = torch.randn(world * B, 512, generator=gen).to(torch.bfloat16)
    x = x_all[rank * B: (rank + 1) * B].cuda().requires_grad_(True)
    y = layer(x)
    y.backward(g_all[rank * B: (rank + 1) * B].cuda())
    torch.cuda.synchronize()
    ctx.check_status()
    # E_loc = E / world consecutive experts per rank, so with n_group = world a group is a rank
    ranks_per_token = E.max_groups_per_token(layer.ws.idx[:B * cfg.k], cfg.k, cfg.num_experts, world)
    shadowed = int((layer.ws.shadow_info.view(-1, 4)[:, 0] >= 0).sum())
    # the kernel's hot-expert selection must equal the host model (parallel/balance.py) on the exchanged count table
    from lah_b200.parallel.balance import shadow_plan
    counts = ctx.cnt_all[:world].cpu().tolist()
    plan, _ = shadow_plan(counts, ctx.E_loc, ctx.S, tol=cfg.shadow_tol, min_rows=cfg.shadow_min_rows)
    got = [int(e) for e in layer.ws.shadow_info.view(-1, 4)[:, 0].cpu().tolist() if e >= 0]
    plan_ok = plan == got or small or bool(capacity)   # the host model plans from the routed counts, not the kept ones
    # gather what the distributed run produced
    ys = [torch.empty_like(y) for _ in range(world)]
    dxs = [torch.empty_like(x.grad) for _ in range(world)]
    dist.all_gather(ys, y.detach().contiguous())
    dist.all_gather(dxs, x.grad.contiguous())
    gw = layer.proj.weight.grad.clone()
    dist.all_reduce(gw)
    shared_grads = [p.grad.clone() for p in layer.shared_expert_parameters()]
    for g in shared_grads:
        dist.all_reduce(g)
    if router:   # the mean over ranks of the per-rank losses is the box-wide value
        rl = layer.router_loss.clone()
        dist.all_reduce(rl)
        rl /= world
    w1 = layer.shard.views[mat][:layer.E_loc].clone()
    w1s = [torch.empty_like(w1) for _ in range(world)]
    dist.all_gather(w1s, w1)
    b2 = layer.shard.views[vec][:layer.E_loc].clone()
    b2s = [torch.empty_like(b2) for _ in range(world)]
    dist.all_gather(b2s, b2)
    steps = [torch.empty_like(layer.shard.step) for _ in range(world)]
    dist.all_gather(steps, layer.shard.step)
    if router:
        # the router gradient alone: a second step with a zero output gradient, where gate_bwd adds exactly 0 to the gate
        # logits.  Summed over ranks, it is the gradient of the whole-batch losses times the world size
        layer.proj.weight.grad = None
        layer(x.detach()).backward(torch.zeros(B, 512, dtype=torch.bfloat16, device="cuda"))
        torch.cuda.synchronize()
        ctx.check_status()
        g_router = layer.proj.weight.grad.clone()
        dist.all_reduce(g_router)
        counts_box = ctx.cnt_all[:world].clone()   # the box-wide count table of that step, the same on every rank
    bias_ok = True
    if bias:
        # after several more steps on per-rank batches, each step's update must equal the oracle over that step's gathered
        # count table, and every rank must hold the same bits
        gen_r = torch.Generator().manual_seed(100 + rank)
        for _ in range(4):
            before = layer.expert_bias.clone()
            xs = torch.randn(B, 512, generator=gen_r).to(torch.bfloat16).cuda()
            layer(xs).backward(torch.randn(B, 512, generator=gen_r).to(torch.bfloat16).cuda())
            torch.cuda.synchronize()
            ctx.check_status()
            want = K.expert_bias_update_ref(ctx.cnt_all[:world], before, cfg.expert_bias_update_rate)
            bias_ok = bias_ok and torch.equal(layer.expert_bias, want) and not torch.equal(layer.expert_bias, before)
        biases = [torch.empty_like(layer.expert_bias) for _ in range(world)]
        dist.all_gather(biases, layer.expert_bias)
        bias_ok = bias_ok and all(torch.equal(b, biases[0]) for b in biases)
    shared_ok = True
    if shared:
        from lah_b200.parallel.trainer import DMoETrainer
        tcfg = E.DMoEConfig(hidden=512, grid_size=(16,), k=4, num_layers=2, tokens_per_rank=B, gate_mode="emulator",
                            expert="swiglu", expert_path="small" if small else "big", **shared)
        ctx.close()
        trainer = DMoETrainer(tcfg)
        gen_t = torch.Generator().manual_seed(200 + rank)
        for _ in range(5):
            trainer.train_step(torch.randn(B, tcfg.in_features, generator=gen_t).pin_memory(),
                               torch.randint(0, 10, (B,), generator=gen_t).pin_memory())
        trainer.ctx.check_status()
        flat = trainer.flat_p.clone()
        flats = [torch.empty_like(flat) for _ in range(world)]
        dist.all_gather(flats, flat)
        shared_ok = all(torch.equal(f, flats[0]) for f in flats)
        trainer.close()
    rpt = torch.tensor([ranks_per_token], device="cuda")
    dist.all_reduce(rpt, op=dist.ReduceOp.MAX)
    group_ok = not group or int(rpt) == 1
    capacity_ok = True
    if capacity:   # the same (C, dropped pairs) on every rank, some pairs dropped, and the status word clean
        stats = layer.ws.capacity_stats.clone()
        every = [torch.empty_like(stats) for _ in range(world)]
        dist.all_gather(every, stats)
        capacity_ok = all(torch.equal(s, stats) for s in every) and int(stats[1]) > 0 and int(ctx.status[0]) == 0
    ok = True
    if rank == 0:
        # single-GPU reference in the same process: a fresh world-1 context is impossible inside an initialised group,
        # so use the PyTorch oracle of the layer (all experts local) on the whole batch
        # the gate gradients are SUMMED over ranks here (a trainer averages them): the router part of that sum is the
        # gradient of the whole-batch losses times the world size
        ref_cfg = E.DMoEConfig(**{**cfg.__dict__, **{k: v * world for k, v in router.items()}}) if router else cfg
        ref = E.FusedDMoE(ref_cfg, None, device=torch.device("cuda")).cuda()
        ref.proj.load_state_dict(layer.proj.state_dict())
        if shared:
            ref.load_shared_expert_state_dict(layer.shared_expert_state_dict())
        ref.train()
        xr = x_all.cuda().float().requires_grad_(True)
        yr = ref(xr)
        yr.backward(g_all.cuda().float())
        ref.apply_expert_gradients_ref()
        errs = dict(y=rel(torch.cat(ys), yr), dx=rel(torch.cat(dxs), xr.grad), dproj=rel(gw, ref.proj.weight.grad),
                    w1_mean_abs=(torch.cat(w1s) - ref.shard.views[mat]).abs().mean().item(),
                    b2_max_abs=(torch.cat(b2s) - ref.shard.views[vec]).abs().max().item(),
                    steps=bool((torch.cat(steps).cpu() == ref.shard.step.cpu()).all()))
        if shared:
            errs["shared_grad"] = max(rel(a, b.grad) for a, b in zip(shared_grads, ref.shared_expert_parameters()))
            errs["shared_params_bit_identical_after_5_steps"] = shared_ok
        if router:
            errs["router_loss"] = rel(rl, ref.router_loss)
            xa = x_all.cuda()
            l64 = F.linear(xa.float(), layer.proj.weight, layer.proj.bias).detach().double().requires_grad_(True)
            aux, zl = K.router_loss_ref(l64, cfg.grid_size, counts_box)
            (g,) = torch.autograd.grad(world * (cfg.router_aux_loss_coef * aux + cfg.router_z_loss_coef * zl), l64)
            ref_router = g.t() @ xa.double()
            errs["router_grad_max_err"] = ((g_router.double() - ref_router).abs().max() / ref_router.abs().max()).item()
        ok = errs["y"] < 2e-2 * tol and errs["dx"] < 3e-2 * tol and errs["dproj"] < 5e-2 * tol and \
            errs["w1_mean_abs"] < 1e-4 * tol and errs["b2_max_abs"] < 2.5e-3 * tol and errs["steps"]
        ok = ok and (shadowed > 0 or not force_shadow) and plan_ok and errs.get("router_loss", 0.0) < 1e-4
        ok = ok and errs.get("router_grad_max_err", 0.0) < 1e-4 and bias_ok
        ok = ok and errs.get("shared_grad", 0.0) < 8e-2 and shared_ok and group_ok and capacity_ok
        if capacity:
            errs["capacity"] = dict(kernel=layer.ws.capacity_stats.tolist(), oracle=list(ref._ref_capacity),
                                    same_on_every_rank_and_clean=capacity_ok)
            ok = ok and layer.ws.capacity_stats.tolist() == list(ref._ref_capacity)
        if group:
            errs["max_ranks_per_token"] = int(rpt)
        if bias:
            errs["expert_bias_bit_identical_and_equal_to_oracle"] = bias_ok
        print("multi_gpu_check", dict(path="small" if small else "big", expert=cfg.expert, expert_dtype=cfg.expert_dtype, router_loss=bool(router), force_shadow=force_shadow, shadowed_experts=shadowed, plan_matches_host_model=plan_ok,
                                      plan=plan, kernel=got), errs, flush=True)
        print("MULTI_GPU_OK" if ok else "MULTI_GPU_FAILED", flush=True)
    dist.barrier()
    dist.destroy_process_group()
    sys.exit(0 if ok else 1)


if __name__ == "__main__":
    main()
