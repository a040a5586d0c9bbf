"""Cost and effect of unnormalised top-k weights (DMoEConfig(norm_topk_prob=False)); writes check_out/router_norm_perf.json.

1. The gate at 65,536 tokens: top-4 of 64, top-8 of 256 with expert biases, top-4 of 64 x 64 and top-8 of 4096, with the
   softmax and the sigmoid score.  norm=False against norm=True of the same score, bias and grouping.  CUDA events around
   ITERS_K calls (gate_topk_kernel + rank_slots_kernel), median of 10 windows with the arms alternating per window; then
   one torch.profiler pass per arm for gate_topk_kernel alone.
2. gate_bwd at 65,536 tokens, top-4, hidden 512 and 1024, on 64 experts and on 64 x 64 and 4096 experts, timed the same
   way; beside it the router-loss backward (router_loss_bwd_kernel) on the same grid.
3. Step time at the bench operating point (emulator gate, 64 experts, top-4, 256 samples per step, 4 layers, hidden 512,
   CUDA graph) at lr = 0, norm=False against norm=True.  With nothing trained the first layer routes identically in both
   arms (its step_rows are compared after every round); the later layers see different inputs, because the first
   layer's weights differ, so their routing may differ.  ROUNDS rounds, the order of the arms alternating.
4. Balance: STEPS steps of the synthetic learnable data of tools/router_loss_perf.py.  Switch top-1 (product-key gate
   over 8 x 8, aux-loss alpha = 0.01) with norm_topk_prob True and False, and a DeepSeek-V2-shaped SwiGLU recipe (top-6,
   8 groups of which 3, c = 16, a shared expert, alpha = 0.01).  Per layer: max_rows / mean_rows, active experts and
   routed_weight_mean from log_step averaged over the last 20 steps; the final loss; ms per step.
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
from tools.router_score_perf import alternate, card, window

BENCH = dict(hidden=512, grid_size=(64,), k=4, num_layers=4, tokens_per_rank=256, gate_mode="emulator")
ROUNDS, WINDOWS, ITERS, WARMUP = 6, 3, 20, 10
STEPS = 300
TOKENS = 65536


def ratio(a, b):
    """a / b, None when the profiler pass found no kernel for an arm"""
    return None if a is None or b is None else a / b


def gate_alone(grid, k, biased):
    dev = torch.device("cuda")
    E_ = math.prod(grid)
    g = torch.Generator(device=dev).manual_seed(1)
    logits = torch.randn(TOKENS, sum(grid), device=dev, generator=g) * 3
    bias = torch.randn(E_, device=dev, generator=g) * 0.01 if biased else None
    P = TOKENS * k
    idx = torch.empty(P, dtype=torch.int32, device=dev)
    w, pos, sig = torch.empty(P, device=dev), torch.empty(P, dtype=torch.int32, device=dev), torch.empty(P, device=dev)
    lse = torch.empty(TOKENS, device=dev)
    counts = torch.zeros(E_, dtype=torch.int32, device=dev)
    out = dict(grid=list(grid), experts=E_, tokens=TOKENS, k=k, bias=biased)
    for score in ("softmax", "sigmoid"):
        base = dict(score="sigmoid", scale=2.5, sig=sig) if score == "sigmoid" else {}
        arms = {"norm": base, "unnorm": dict(base, norm=False, scale=2.5, **({} if score == "sigmoid" else
                                                                              dict(lse=lse)))}
        calls = {a: (lambda kw=kw: K.gate_topk(logits, grid, k, idx=idx, w=w, pos=pos, counts=counts, bias=bias, **kw))
                 for a, kw in arms.items()}
        r = alternate(calls, kernel="gate_topk_kernel")
        out[score] = dict(r, call_ratio=ratio(r["call_us_unnorm"], r["call_us_norm"]),
                          kernel_ratio=ratio(r["kernel_us_unnorm"], r["kernel_us_norm"]))
    return out


def gate_bwd_alone(grid, H, k=4):
    from lah_b200.parallel.symmetric import SymmetricHeap
    dev = torch.device("cuda")
    E_ = math.prod(grid)
    P = TOKENS * k
    heap = SymmetricHeap(P * H * 2 + (16 << 20))
    try:
        yo, yo_off = heap.alloc((P, H), torch.bfloat16)
        K.set_peers(heap.peer_bases, 0)
        g = torch.Generator(device=dev).manual_seed(2)
        yo.copy_(torch.randn(P, H, device=dev, generator=g))
        logits = torch.randn(TOKENS, sum(grid), device=dev, generator=g) * 3
        alive = torch.ones(E_, dtype=torch.uint8, device=dev)
        idx = torch.empty(P, dtype=torch.int32, device=dev)
        w, w_un, pos = torch.empty(P, device=dev), torch.empty(P, device=dev), torch.empty(P, dtype=torch.int32, device=dev)
        lse = torch.empty(TOKENS, device=dev)
        counts = torch.zeros(E_, dtype=torch.int32, device=dev)
        K.gate_topk(logits, grid, k, idx=idx, w=w, pos=pos, counts=counts)
        K.gate_topk(logits, grid, k, idx=idx, w=w_un, pos=pos, counts=counts, norm=False, lse=lse)
        pair_row = torch.randperm(P, device=dev, generator=g).to(torch.int32)
        gy = torch.randn(TOKENS, H, device=dev, generator=g).to(torch.bfloat16)
        dl = torch.zeros(TOKENS, sum(grid), device=dev)
        f = torch.rand(E_ + 1, device=dev, generator=g)
        z, Fb = torch.randn(TOKENS, device=dev, generator=g), torch.rand(TOKENS, device=dev, generator=g)
        calls = {"norm": lambda: K.gate_bwd(yo_off, gy, idx, pair_row, w, dl, k, E_, grid),
                 "unnorm": lambda: K.gate_bwd(yo_off, gy, idx, pair_row, w_un, dl, k, E_, grid, norm=False, lse=lse,
                                              alive=alive, logits=logits)}
        r = alternate(calls, kernel="gate_bwd_kernel")
        rl = alternate({"router_loss_bwd": lambda: K.router_loss_bwd(logits, grid, alive=alive, f=f, z=z, Fb=Fb,
                                                                     aux_coef=0.01, z_coef=1e-3, dlogits=dl)},
                       kernel="router_loss_bwd_kernel")
        torch.cuda.synchronize()
    finally:
        heap.close()
    return dict(grid=list(grid), tokens=TOKENS, k=k, hidden=H, **r, **rl,
                kernel_ratio=ratio(r["kernel_us_unnorm"], r["kernel_us_norm"]),
                unnorm_over_router_loss_bwd=ratio(r["kernel_us_unnorm"], rl["kernel_us_router_loss_bwd"]))


def step_time():
    g = torch.Generator().manual_seed(0)
    x = torch.randn(256, 784, generator=g).cuda()
    y = torch.randint(0, 10, (256,), generator=g).cuda()
    ms = {"norm": [], "unnorm": []}
    ratios, same_rows = [], []
    for r in range(ROUNDS):
        med, rows = {}, {}
        for arm in (("norm", "unnorm") if r % 2 == 0 else ("unnorm", "norm")):
            t = DMoETrainer(E.DMoEConfig(**BENCH, lr=0.0, norm_topk_prob=arm == "norm"))
            for _ in range(WARMUP):
                t.train_step_device(x, y)
            w = [window(lambda: t.train_step_device(x, y), ITERS) for _ in range(WINDOWS)]
            t.ctx.check_status()
            assert t._graph is not None
            rows[arm] = t.model.blocks[0].ws.step_rows.clone().cpu()
            t.close()
            ms[arm] += w
            med[arm] = statistics.median(w)
        ratios.append(med["unnorm"] / med["norm"])
        same_rows.append(bool(torch.equal(rows["unnorm"], rows["norm"])))
    return dict(ms_per_step_norm=statistics.median(ms["norm"]), ms_per_step_unnorm=statistics.median(ms["unnorm"]),
                ratio_per_round=ratios, slowdown_pct=(statistics.median(ratios) - 1) * 100,
                same_layer0_step_rows_per_round=same_rows)


def balance(name, **kw):
    cfg = E.DMoEConfig(**{**BENCH, **kw})
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
        if "routed_weight_mean" in rows[0]:
            layer["routed_weight_mean"] = statistics.mean(r["routed_weight_mean"] for r in rows)
        layers.append(layer)
    return dict(arm=name, **kw, steps=STEPS, first_loss=losses[0], final_loss=statistics.mean(losses[-20:]),
                ms_per_step=ms, layers=layers)


def main():
    results = dict(card=card(), device=torch.cuda.get_device_name())
    results["gate"] = [gate_alone(grid, k, b) for grid, k, b in
                       (((64,), 4, False), ((256,), 8, True), ((64, 64), 4, False), ((4096,), 8, False))]
    for r in results["gate"]:
        print(json.dumps(r), flush=True)
    results["gate_bwd"] = [gate_bwd_alone(grid, H) for grid in ((64,), (64, 64), (4096,)) for H in (512, 1024)]
    for r in results["gate_bwd"]:
        print(json.dumps(r), flush=True)
    results["step"] = step_time()
    print(json.dumps(results["step"]), flush=True)
    switch = dict(gate_mode="product_key", grid_size=(8, 8), k=1, router_aux_loss_coef=0.01)
    results["balance"] = [
        balance("switch top-1, norm_topk_prob=True", **switch),
        balance("switch top-1, norm_topk_prob=False", **switch, norm_topk_prob=False),
        balance("v2-shaped", gate_mode="product_key", grid_size=(8, 8), k=6, n_group=8, topk_group=3,
                routed_scaling_factor=16.0, router_aux_loss_coef=0.01, expert="swiglu", inner_dim=256,
                shared_inner_dim=1024, norm_topk_prob=False)]
    for r in results["balance"]:
        print(json.dumps(r), flush=True)
    results["card_end"] = card()
    with open(output_path("router_norm_perf.json"), "w") as f:
        json.dump(results, f, indent=1)
    print(json.dumps(dict(card=results["card"], card_end=results["card_end"])), flush=True)


if __name__ == "__main__":
    main()
