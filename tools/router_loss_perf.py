"""Cost and effect of the router losses of the product-key gate (writes check_out/router_loss_perf.json).

1. Step time at the bench operating point with the product-key gate (64 experts, top-4, 256 samples per step, 4 layers,
   hidden 512, CUDA graph): (router_aux_loss_coef, router_z_loss_coef) = (0.01, 0.001) against (0, 0), once with lr = 0
   (same parameters, routing and expert work in every step: the cost of the router kernels alone) and once at the default
   lr (training on one fixed batch: the losses also change which experts receive rows; the sums of active experts over
   the layers at the end of each round are reported).  The two arms
   alternate: each round builds the trainer of one arm, warms it up, times WINDOWS windows of ITERS steps with CUDA events
   and closes it (the engine's device counters are process-wide, so two trainers do not live side by side).  Reported:
   the median over all windows of each arm and the median of the per-round ratios.
2. The router-loss kernels alone (forward: 2 launches, backward: 1) at 65,536 tokens and 64, 4096 (64 x 64) and 4096
   (one dimension) experts: CUDA events around ITERS_K forward + backward pairs, median of 5 windows, as us per pass and
   ns per token.
3. The balance effect: STEPS steps of synthetic learnable data (10 Gaussian class prototypes + noise, a fresh batch every
   step) at the bench operating point with router_aux_loss_coef 0 and 0.01; max_rows / mean_rows and the active experts
   of every layer from log_step, averaged over the last 20 steps, and the final loss.
The card's name, power limit and maximum SM clock are read in the same run.
"""
import json
import math
import os
import statistics
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

import lah_b200  # noqa
from lah_b200.ops import kernels as K
from lah_b200.parallel import engine as E
from lah_b200.parallel.trainer import DMoETrainer
from tools import output_path

BENCH = dict(hidden=512, grid_size=(64,), k=4, num_layers=4, tokens_per_rank=256, gate_mode="product_key")
ON = dict(router_aux_loss_coef=0.01, router_z_loss_coef=0.001)
ROUNDS, WINDOWS, ITERS, WARMUP = 6, 3, 20, 10
ITERS_K = 50
STEPS = 300


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else torch.cuda.get_device_name()


def windows(fn, n, iters, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    out = []
    for _ in range(n):
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        for _ in range(iters):
            fn()
        e.record()
        torch.cuda.synchronize()
        out.append(s.elapsed_time(e) / iters)
    return out


def step_time(**kw):
    g = torch.Generator().manual_seed(0)
    x = torch.randn(256, 784, generator=g).cuda()
    y = torch.randint(0, 10, (256,), generator=g).cuda()
    ms = {"off": [], "on": []}
    active = {"off": [], "on": []}
    ratios = []
    for r in range(ROUNDS):
        med = {}
        for arm in (("off", "on") if r % 2 == 0 else ("on", "off")):
            t = DMoETrainer(E.DMoEConfig(**BENCH, **kw, **(ON if arm == "on" else {})))
            w = windows(lambda: t.train_step_device(x, y), WINDOWS, ITERS, WARMUP)
            t.ctx.check_status()
            active[arm].append(sum(layer["active_experts"] for layer in t.log_step()["layers"]))
            assert t._graph is not None
            t.close()
            ms[arm] += w
            med[arm] = statistics.median(w)
        ratios.append(med["on"] / med["off"])
    return dict(**kw, ms_per_step_off=statistics.median(ms["off"]), active_expert_layers_off=active["off"],
                active_expert_layers_on=active["on"], ms_per_step_on=statistics.median(ms["on"]),
                windows_off=ms["off"], windows_on=ms["on"], ratio_per_round=ratios,
                slowdown_pct=(statistics.median(ratios) - 1) * 100)


def kernels_alone(grid, B=65536):
    dev = torch.device("cuda")
    E_ = math.prod(grid)
    g = torch.Generator(device=dev).manual_seed(1)
    logits = torch.randn(B, sum(grid), device=dev, generator=g) * 3
    counts = torch.randint(0, 64, (1, E_), device=dev, dtype=torch.int32, generator=g)
    f = torch.empty(E_ + 1, device=dev)
    z, Fb, loss = torch.empty(B, device=dev), torch.empty(B, device=dev), torch.empty(2, device=dev)
    partials = torch.empty(2 * -(-B // K.ROUTER_WARPS), device=dev)
    ticket = torch.zeros(1, dtype=torch.int32, device=dev)
    dl = torch.zeros_like(logits)

    def fwd():
        K.router_loss_fwd(logits, grid, counts, f=f, z=z, Fb=Fb, loss=loss, partials=partials, ticket=ticket)

    def bwd():
        K.router_loss_bwd(logits, grid, f=f, z=z, Fb=Fb, aux_coef=0.01, z_coef=0.001, dlogits=dl)

    def both():
        fwd()
        bwd()

    out = {}
    for name, fn in (("fwd", fwd), ("bwd", bwd), ("fwd+bwd", both)):
        us = statistics.median(windows(fn, 5, ITERS_K, 5)) * 1e3
        out[name] = dict(us=us, ns_per_token=us * 1e3 / B)
    return dict(grid=list(grid), experts=E_, tokens=B, **out)


def balance(alpha):
    cfg = E.DMoEConfig(**BENCH, router_aux_loss_coef=alpha)
    t = DMoETrainer(cfg)
    g = torch.Generator(device="cuda").manual_seed(0)
    protos = torch.randn(10, cfg.in_features, device="cuda", generator=g) * 2
    recs, losses = [], []
    for s in range(STEPS):
        y = torch.randint(0, 10, (256,), device="cuda", generator=g)
        x = protos[y] + torch.randn(256, cfg.in_features, device="cuda", generator=g)
        losses.append(float(t.train_step_device(x, y)))
        if s >= STEPS - 20:
            recs.append(t.log_step())
    t.ctx.check_status()
    t.close()
    layers = []
    for li in range(cfg.num_layers):
        rows = [r["layers"][li] for r in recs]
        layer = dict(max_over_mean=statistics.mean(r["max_rows"] / r["mean_rows"] for r in rows),
                     active_experts=statistics.mean(r["active_experts"] for r in rows))
        if "router_aux_loss" in rows[0]:
            layer.update(router_aux_loss=statistics.mean(r["router_aux_loss"] for r in rows),
                         router_z_loss=statistics.mean(r["router_z_loss"] for r in rows))
        layers.append(layer)
    return dict(router_aux_loss_coef=alpha, steps=STEPS, first_loss=losses[0],
                final_loss=statistics.mean(losses[-20:]), layers=layers)


def main():
    results = dict(card=card(), device=torch.cuda.get_device_name())
    # lr = 0: the parameters, and with them the routing and the expert work, are the same in every step of both arms, so
    # the difference is the cost of the router kernels; at the default lr the loss also changes which experts get rows
    results["step"] = [step_time(lr=0.0), step_time()]
    for r in results["step"]:
        print(json.dumps({k: v for k, v in r.items() if not k.startswith("windows")}), flush=True)
    results["kernels"] = [kernels_alone(grid) for grid in ((64,), (64, 64), (4096,))]
    for r in results["kernels"]:
        print(json.dumps(r), flush=True)
    results["balance"] = [balance(a) for a in (0.0, 0.01)]
    for r in results["balance"]:
        print(json.dumps(r), flush=True)
    results["card_end"] = card()
    with open(output_path("router_loss_perf.json"), "w") as f:
        json.dump(results, f, indent=1)
    print(json.dumps(dict(card=results["card"], card_end=results["card_end"])), flush=True)


if __name__ == "__main__":
    main()
