"""Cost and effect of auxiliary-loss-free expert balancing (writes check_out/expert_bias_perf.json).

1. The gate alone at 65,536 tokens and 64, 4096 (64 x 64) and 4096 (one dimension) experts: K.gate_topk with a bias
   against without one (the call is gate_topk_kernel + rank_slots_kernel), CUDA events around ITERS_K calls, median of
   5 windows, the arms alternating per window; then one torch.profiler pass per arm for gate_topk_kernel alone.
2. Step time at the bench operating point (emulator gate, 64 experts, top-4, 256 samples per step, 4 layers, hidden 512,
   CUDA graph): expert_bias_update_rate 0 against 1e-30.  A bias of a few thousand times 1e-30 stays far below one ulp
   of any score, so both arms route alike and do the same expert work; the per-layer step_rows of the two arms are
   compared at the end of every round to confirm it.  The difference is the cost of the biased gate and the update
   kernel.  Each round builds the trainer of one arm, warms it up, times WINDOWS windows of ITERS steps with CUDA events
   and closes it; the order of the arms alternates.  Reported: median over the windows of each arm and the median of the
   per-round ratios.
3. The balance effect: STEPS steps of the synthetic learnable data of tools/router_loss_perf.py (10 Gaussian class
   prototypes + noise, a fresh batch every step) at the bench operating point, for the emulator gate with rates 0, 1e-3,
   1e-2 and the product-key gate with nothing, router_aux_loss_coef 0.01 and rate 1e-3.  Per layer: max_rows / mean_rows
   and active experts from log_step averaged over the last 20 steps, the final bias max |b|; the final loss; and ms per
   step of the trained arm on one fixed batch (3 windows of ITERS steps under the graph).
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

BENCH = dict(hidden=512, grid_size=(64,), k=4, num_layers=4, tokens_per_rank=256, gate_mode="emulator")
ROUNDS, WINDOWS, ITERS, WARMUP = 6, 3, 20, 10
ITERS_K = 50
STEPS = 300


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else torch.cuda.get_device_name()


def window(fn, iters):
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(iters):
        fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / iters


def gate_alone(grid, B=65536, k=4):
    dev = torch.device("cuda")
    E_ = math.prod(grid)
    g = torch.Generator(device=dev).manual_seed(1)
    logits = torch.randn(B, sum(grid), device=dev, generator=g) * 3
    bias = torch.randn(E_, device=dev, generator=g) * 0.1
    idx = torch.empty(B * k, dtype=torch.int32, device=dev)
    w, pos = torch.empty(B * k, device=dev), torch.empty(B * k, dtype=torch.int32, device=dev)
    counts = torch.zeros(E_, dtype=torch.int32, device=dev)
    arms = {"plain": None, "bias": bias}

    def call(arm):
        return lambda: K.gate_topk(logits, grid, k, idx=idx, w=w, pos=pos, counts=counts, bias=arms[arm])

    for arm in arms:
        for _ in range(5):
            call(arm)()
    torch.cuda.synchronize()
    us = {"plain": [], "bias": []}
    for i in range(10):
        for arm in (("plain", "bias") if i % 2 == 0 else ("bias", "plain")):
            us[arm].append(window(call(arm), ITERS_K) * 1e3)
    # the gate kernel alone (without rank_slots_kernel), from a profiler pass per arm
    kernel_us = {}
    for arm in arms:
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            for _ in range(ITERS_K):
                call(arm)()
            torch.cuda.synchronize()
        times = [ev.device_time for ev in prof.events() if "gate_topk_kernel" in ev.name]
        kernel_us[arm] = statistics.median(times) if times else None
    out = dict(grid=list(grid), experts=E_, tokens=B, k=k,
               call_us_plain=statistics.median(us["plain"]), call_us_bias=statistics.median(us["bias"]),
               kernel_us_plain=kernel_us["plain"], kernel_us_bias=kernel_us["bias"])
    out["call_slowdown_pct"] = (out["call_us_bias"] / out["call_us_plain"] - 1) * 100
    if kernel_us["plain"] and kernel_us["bias"]:
        out["kernel_slowdown_pct"] = (kernel_us["bias"] / kernel_us["plain"] - 1) * 100
    return out


def step_time():
    g = torch.Generator().manual_seed(0)
    x = torch.randn(256, 784, generator=g).cuda()
    y = torch.randint(0, 10, (256,), generator=g).cuda()
    ms = {"off": [], "on": []}
    ratios, same_rows = [], []
    for r in range(ROUNDS):
        med, rows = {}, {}
        for arm in (("off", "on") if r % 2 == 0 else ("on", "off")):
            t = DMoETrainer(E.DMoEConfig(**BENCH, expert_bias_update_rate=1e-30 if arm == "on" else 0.0))
            for _ in range(WARMUP):
                t.train_step_device(x, y)
            w = [window(lambda: t.train_step_device(x, y), ITERS) for _ in range(WINDOWS)]
            t.ctx.check_status()
            assert t._graph is not None
            rows[arm] = torch.stack([b.ws.step_rows.clone() for b in t.model.blocks]).cpu()
            t.close()
            ms[arm] += w
            med[arm] = statistics.median(w)
        ratios.append(med["on"] / med["off"])
        same_rows.append(bool(torch.equal(rows["on"], rows["off"])))
    return dict(ms_per_step_off=statistics.median(ms["off"]), ms_per_step_on=statistics.median(ms["on"]),
                windows_off=ms["off"], windows_on=ms["on"], ratio_per_round=ratios,
                slowdown_pct=(statistics.median(ratios) - 1) * 100, same_step_rows_per_round=same_rows)


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
        if "expert_bias_absmax" in rows[-1]:
            layer["expert_bias_absmax"] = rows[-1]["expert_bias_absmax"]
        layers.append(layer)
    return dict(arm=name, **kw, steps=STEPS, first_loss=losses[0], final_loss=statistics.mean(losses[-20:]),
                ms_per_step=ms, layers=layers)


def main():
    results = dict(card=card(), device=torch.cuda.get_device_name())
    results["gate"] = [gate_alone(grid) for grid in ((64,), (64, 64), (4096,))]
    for r in results["gate"]:
        print(json.dumps(r), flush=True)
    results["step"] = step_time()
    print(json.dumps({k: v for k, v in results["step"].items() if not k.startswith("windows")}), flush=True)
    pk = dict(gate_mode="product_key")
    results["balance"] = [balance("emulator", expert_bias_update_rate=0.0),
                          balance("emulator", expert_bias_update_rate=1e-3),
                          balance("emulator", expert_bias_update_rate=1e-2),
                          balance("product_key", **pk),
                          balance("product_key", **pk, router_aux_loss_coef=0.01),
                          balance("product_key", **pk, expert_bias_update_rate=1e-3)]
    for r in results["balance"]:
        print(json.dumps(r), flush=True)
    results["card_end"] = card()
    with open(output_path("expert_bias_perf.json"), "w") as f:
        json.dump(results, f, indent=1)
    print(json.dumps(dict(card=results["card"], card_end=results["card_end"])), flush=True)


if __name__ == "__main__":
    main()
