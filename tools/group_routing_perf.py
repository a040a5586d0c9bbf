"""Cost and effect of group-limited routing (DMoEConfig(n_group=G, topk_group=M)); writes
check_out/group_routing_perf.json.

1. The gate at 65,536 tokens, grouped against ungrouped of the same score and bias-ness: top-4 of 64 experts with
   (G, M) = (8, 2) and (8, 4) (softmax, no bias); top-8 of 256 with (8, 4), sigmoid with a bias (V3's shape); top-4 of
   4096 as 64 x 64 with (64, 8) and top-8 of 4096 on one dimension with (8, 4) (softmax, no bias).  CUDA events around
   ITERS_K calls (gate_topk_kernel + rank_slots_kernel), median of 10 windows with the arms alternating per window; then
   one torch.profiler pass per arm for gate_topk_kernel alone.
2. Step time at the bench operating point with the README's V3 recipe (64 experts, top-8, SwiGLU inner 256, a shared
   expert of inner 1024, sigmoid, expert biases at 1e-3, c = 2.5), grouped (8, 4) against ungrouped, in alternated
   rounds.  The two arms route differently, so they do not do the same expert work: the per-layer max / mean step_rows
   of each round are reported beside the times.
3. Balance: STEPS steps of the synthetic learnable data of tools/router_score_perf.py for the same two arms: per layer
   max_rows / mean_rows and active experts from log_step averaged over the last 20 steps (and, grouped, the largest
   max_groups_per_token seen); the final loss; ms per step.
The card's name, power limit and maximum SM clock are read in the same run.
"""
import json
import math
import os
import statistics
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

import lah_b200  # noqa
from lah_b200.ops import kernels as K
from lah_b200.parallel import engine as E
from lah_b200.parallel.trainer import DMoETrainer
from tools import output_path
from tools.router_score_perf import BENCH, ITERS, TOKENS, WARMUP, WINDOWS, alternate, card, window

V3 = dict(BENCH, k=8, expert="swiglu", inner_dim=256, shared_inner_dim=1024, router_score="sigmoid",
          expert_bias_update_rate=1e-3, routed_scaling_factor=2.5)
ROUNDS = 6
STEPS = 300
GATES = [((64,), 4, 8, 2, "softmax", False), ((64,), 4, 8, 4, "softmax", False), ((256,), 8, 8, 4, "sigmoid", True),
         ((64, 64), 4, 64, 8, "softmax", False), ((4096,), 8, 8, 4, "softmax", False)]


def gate_alone(grid, k, G, M, score, biased):
    dev = torch.device("cuda")
    E_ = math.prod(grid)
    g = torch.Generator(device=dev).manual_seed(1)
    logits = torch.randn(TOKENS, sum(grid), device=dev, generator=g) * 3
    bias = torch.randn(E_, device=dev, generator=g) * 0.01 if biased else None
    P = TOKENS * k
    idx = torch.empty(P, dtype=torch.int32, device=dev)
    w, pos, sig = torch.empty(P, device=dev), torch.empty(P, dtype=torch.int32, device=dev), torch.empty(P, device=dev)
    counts = torch.zeros(E_, dtype=torch.int32, device=dev)
    kw = dict(score="sigmoid", scale=2.5, sig=sig) if score == "sigmoid" else {}
    calls = {"ungrouped": lambda: K.gate_topk(logits, grid, k, idx=idx, w=w, pos=pos, counts=counts, bias=bias, **kw),
             "grouped": lambda: K.gate_topk(logits, grid, k, idx=idx, w=w, pos=pos, counts=counts, bias=bias,
                                            n_group=G, topk_group=M, **kw)}
    r = alternate(calls, kernel="gate_topk_kernel")
    return dict(grid=list(grid), experts=E_, tokens=TOKENS, k=k, n_group=G, topk_group=M, score=score, bias=biased,
                **r, call_ratio=r["call_us_grouped"] / r["call_us_ungrouped"],
                kernel_ratio=(r["kernel_us_grouped"] / r["kernel_us_ungrouped"]
                              if r["kernel_us_grouped"] and r["kernel_us_ungrouped"] else None))


def _rows(t):
    return [float(b.ws.step_rows.float().max() / b.ws.step_rows.float().mean()) for b in t.model.blocks]


def step_time():
    g = torch.Generator().manual_seed(0)
    x = torch.randn(256, 784, generator=g).cuda()
    y = torch.randint(0, 10, (256,), generator=g).cuda()
    arms = {"ungrouped": {}, "grouped": dict(n_group=8, topk_group=4)}
    ms = {a: [] for a in arms}
    ratios, rows = [], {a: [] for a in arms}
    for r in range(ROUNDS):
        med = {}
        for arm in (list(arms) if r % 2 == 0 else list(arms)[::-1]):
            t = DMoETrainer(E.DMoEConfig(**V3, **arms[arm]))
            for _ in range(WARMUP):
                t.train_step_device(x, y)
            w = [window(lambda: t.train_step_device(x, y), ITERS) for _ in range(WINDOWS)]
            t.ctx.check_status()
            assert t._graph is not None
            rows[arm].append(_rows(t))
            t.close()
            ms[arm] += w
            med[arm] = statistics.median(w)
        ratios.append(med["grouped"] / med["ungrouped"])
    return dict(ms_per_step_ungrouped=statistics.median(ms["ungrouped"]),
                ms_per_step_grouped=statistics.median(ms["grouped"]), ratio_per_round=ratios,
                change_pct=(statistics.median(ratios) - 1) * 100,
                step_rows_max_over_mean_ungrouped=rows["ungrouped"], step_rows_max_over_mean_grouped=rows["grouped"])


def balance(name, **kw):
    cfg = E.DMoEConfig(**{**V3, **kw})
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
    ms = statistics.median([window(lambda: t.train_step_device(x, y), ITERS) for _ in range(WINDOWS)])
    t.ctx.check_status()
    t.close()
    layers = []
    for li in range(cfg.num_layers):
        rows = [r["layers"][li] for r in recs]
        layer = dict(max_over_mean=statistics.mean(r["max_rows"] / r["mean_rows"] for r in rows),
                     active_experts=statistics.mean(r["active_experts"] for r in rows))
        if cfg.n_group > 1:
            layer["max_groups_per_token"] = max(r["max_groups_per_token"] for r in rows)
        layers.append(layer)
    return dict(arm=name, **kw, steps=STEPS, first_loss=losses[0], final_loss=statistics.mean(losses[-20:]),
                ms_per_step=ms, layers=layers)


def main():
    results = dict(card=card(), device=torch.cuda.get_device_name())
    results["gate"] = [gate_alone(*a) for a in GATES]
    for r in results["gate"]:
        print(json.dumps(r), flush=True)
    results["step"] = step_time()
    print(json.dumps(results["step"]), flush=True)
    results["balance"] = [balance("ungrouped"), balance("grouped (8, 4)", n_group=8, topk_group=4)]
    for r in results["balance"]:
        print(json.dumps(r), flush=True)
    results["card_end"] = card()
    with open(output_path("group_routing_perf.json"), "w") as f:
        json.dump(results, f, indent=1)
    print(json.dumps(dict(card=results["card"], card_end=results["card_end"])), flush=True)


if __name__ == "__main__":
    main()
