"""Cost and effect of the sigmoid router (DMoEConfig(router_score="sigmoid")); writes check_out/router_score_perf.json.

1. The gate at 65,536 tokens: top-4 of 64, 4096 (64 x 64) and 4096 (one dimension) experts, and top-8 of 256.  The
   sigmoid gate against the softmax gate of the same bias-ness (without a bias, then with one).  CUDA events around
   ITERS_K calls (gate_topk_kernel + rank_slots_kernel), median of 10 windows with the arms alternating per window; then
   one torch.profiler pass per arm for gate_topk_kernel alone.
2. gate_bwd at 65,536 tokens, hidden 512, top-4 of 64 experts, sigmoid against softmax, timed the same way.
3. The router-loss forward + backward (router_f + router_loss_fwd + router_loss_bwd) at 65,536 tokens on 64, 64 x 64 and
   4096 experts, sigmoid against softmax.
4. Step time at the bench operating point (emulator gate, 64 experts, top-4, 256 samples per step, 4 layers, hidden 512,
   CUDA graph), sigmoid against softmax, both at expert_bias_update_rate 0.  Both arms select the same experts (an
   unbiased sigmoid gate ranks the raw scores), so they do the same expert work; the per-layer step_rows are compared
   after every round to confirm it.  Each round builds the trainer of one arm, warms it up, times WINDOWS windows of
   ITERS steps and closes it; the order of the arms alternates.
5. Balance: STEPS steps of the synthetic learnable data of tools/router_loss_perf.py at the bench operating point for
   softmax with rate 1e-3, sigmoid with rate 1e-3, sigmoid with rate 1e-3 and c = 2.5, and a DeepSeek-V3-shaped config
   (SwiGLU experts of inner width 256, a shared expert of inner width 1024, sigmoid, rate 1e-3, c = 2.5).  Per layer:
   max_rows / mean_rows and active experts from log_step averaged over the last 20 steps; the final loss; ms per step.
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
TOKENS = 65536


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


def alternate(calls, kernel=None):
    """median us per call of every arm over 10 alternating windows; with ``kernel``, also the median device time of the
    kernels whose name contains it, from one torch.profiler pass per arm"""
    for fn in calls.values():
        for _ in range(5):
            fn()
    torch.cuda.synchronize()
    names = list(calls)
    us = {n: [] for n in names}
    for i in range(10):
        for n in (names if i % 2 == 0 else names[::-1]):
            us[n].append(window(calls[n], ITERS_K) * 1e3)
    out = {f"call_us_{n}": statistics.median(us[n]) for n in names}
    if kernel:
        for n in names:
            with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
                for _ in range(ITERS_K):
                    calls[n]()
                torch.cuda.synchronize()
            times = [ev.device_time for ev in prof.events() if kernel in ev.name]
            out[f"kernel_us_{n}"] = statistics.median(times) if times else None
    return out


def pct(a, b):
    return None if not a or not b else (a / b - 1) * 100


def gate_alone(grid, k):
    dev = torch.device("cuda")
    E_ = math.prod(grid)
    g = torch.Generator(device=dev).manual_seed(1)
    logits = torch.randn(TOKENS, sum(grid), device=dev, generator=g) * 3
    bias = torch.randn(E_, device=dev, generator=g) * 0.01
    P = TOKENS * k
    idx = torch.empty(P, dtype=torch.int32, device=dev)
    w, pos, sig = torch.empty(P, device=dev), torch.empty(P, dtype=torch.int32, device=dev), torch.empty(P, device=dev)
    counts = torch.zeros(E_, dtype=torch.int32, device=dev)
    out = dict(grid=list(grid), experts=E_, tokens=TOKENS, k=k)
    for b, bname in ((None, "plain"), (bias, "bias")):
        score = {"softmax": dict(), "sigmoid": dict(score="sigmoid", scale=2.5, sig=sig)}
        calls = {s: (lambda kw=kw: K.gate_topk(logits, grid, k, idx=idx, w=w, pos=pos, counts=counts, bias=b, **kw))
                 for s, kw in score.items()}
        r = alternate(calls, kernel="gate_topk_kernel")
        out[bname] = dict(r, call_slowdown_pct=pct(r["call_us_sigmoid"], r["call_us_softmax"]),
                          kernel_slowdown_pct=pct(r["kernel_us_sigmoid"], r["kernel_us_softmax"]))
    return out


def gate_bwd_alone(grid=(64,), k=4, H=512):
    from lah_b200.parallel.symmetric import SymmetricHeap
    dev = torch.device("cuda")
    P = TOKENS * k
    heap = SymmetricHeap(P * H * 2 + (16 << 20))
    try:
        yo, yo_off = heap.alloc((P, H), torch.bfloat16)
        K.set_peers(heap.peer_bases, 0)
        g = torch.Generator(device=dev).manual_seed(2)
        yo.copy_(torch.randn(P, H, device=dev, generator=g))
        logits = torch.randn(TOKENS, sum(grid), device=dev, generator=g) * 3
        idx = torch.empty(P, dtype=torch.int32, device=dev)
        w, pos, sig = torch.empty(P, device=dev), torch.empty(P, dtype=torch.int32, device=dev), torch.empty(P, device=dev)
        K.gate_topk(logits, grid, k, idx=idx, w=w, pos=pos, counts=torch.zeros(64, dtype=torch.int32, device=dev),
                    score="sigmoid", scale=2.5, sig=sig)
        pair_row = torch.randperm(P, device=dev, generator=g).to(torch.int32)
        gy = torch.randn(TOKENS, H, device=dev, generator=g).to(torch.bfloat16)
        dl = torch.empty(TOKENS, sum(grid), device=dev)
        calls = {"softmax": lambda: K.gate_bwd(yo_off, gy, idx, pair_row, w, dl, k, 64, grid),
                 "sigmoid": lambda: K.gate_bwd(yo_off, gy, idx, pair_row, w, dl, k, 64, grid, score="sigmoid",
                                               scale=2.5, sig=sig)}
        r = alternate(calls, kernel="gate_bwd_kernel")
        torch.cuda.synchronize()
    finally:
        heap.close()
    return dict(grid=list(grid), tokens=TOKENS, k=k, hidden=H, **r,
                kernel_slowdown_pct=pct(r["kernel_us_sigmoid"], r["kernel_us_softmax"]))


def router_loss_alone(grid, k=4):
    dev = torch.device("cuda")
    E_ = math.prod(grid)
    g = torch.Generator(device=dev).manual_seed(3)
    logits = torch.randn(TOKENS, sum(grid), device=dev, generator=g) * 3
    counts = torch.randint(0, 100, (1, E_), dtype=torch.int32, device=dev, generator=g)
    f = torch.empty(E_ + 1, device=dev)
    z, Fb, loss = torch.empty(TOKENS, device=dev), torch.empty(TOKENS, device=dev), torch.empty(2, device=dev)
    partials = torch.empty(2 * (TOKENS // K.ROUTER_WARPS + 1), device=dev)
    ticket = torch.zeros(1, dtype=torch.int32, device=dev)
    dl = torch.zeros_like(logits)

    def call(score, zc):
        def run():
            K.router_loss_fwd(logits, grid, counts, f=f, z=z, Fb=Fb, loss=loss, partials=partials, ticket=ticket,
                              score=score)
            K.router_loss_bwd(logits, grid, f=f, z=z, Fb=Fb, aux_coef=0.01, z_coef=zc, dlogits=dl, score=score)
        return run

    r = alternate({"softmax": call("softmax", 1e-3), "sigmoid": call("sigmoid", 0.0)})
    return dict(grid=list(grid), experts=E_, tokens=TOKENS, **r,
                call_slowdown_pct=pct(r["call_us_sigmoid"], r["call_us_softmax"]))


def step_time():
    g = torch.Generator().manual_seed(0)
    x = torch.randn(256, 784, generator=g).cuda()
    y = torch.randint(0, 10, (256,), generator=g).cuda()
    ms = {"softmax": [], "sigmoid": []}
    ratios, same_rows = [], []
    for r in range(ROUNDS):
        med, rows = {}, {}
        for arm in (("softmax", "sigmoid") if r % 2 == 0 else ("sigmoid", "softmax")):
            t = DMoETrainer(E.DMoEConfig(**BENCH, router_score=arm))
            for _ in range(WARMUP):
                t.train_step_device(x, y)
            w = [window(lambda: t.train_step_device(x, y), ITERS) for _ in range(WINDOWS)]
            t.ctx.check_status()
            assert t._graph is not None
            rows[arm] = torch.stack([b.ws.step_rows.clone() for b in t.model.blocks]).cpu()
            t.close()
            ms[arm] += w
            med[arm] = statistics.median(w)
        ratios.append(med["sigmoid"] / med["softmax"])
        same_rows.append(bool(torch.equal(rows["sigmoid"], rows["softmax"])))
    return dict(ms_per_step_softmax=statistics.median(ms["softmax"]), ms_per_step_sigmoid=statistics.median(ms["sigmoid"]),
                windows_softmax=ms["softmax"], windows_sigmoid=ms["sigmoid"], ratio_per_round=ratios,
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
        layers.append(dict(max_over_mean=statistics.mean(r["max_rows"] / r["mean_rows"] for r in rows),
                           active_experts=statistics.mean(r["active_experts"] for r in rows)))
    return dict(arm=name, **kw, steps=STEPS, first_loss=losses[0], final_loss=statistics.mean(losses[-20:]),
                ms_per_step=ms, layers=layers)


def main():
    results = dict(card=card(), device=torch.cuda.get_device_name())
    results["gate"] = [gate_alone(grid, k) for grid, k in (((64,), 4), ((64, 64), 4), ((4096,), 4), ((256,), 8))]
    for r in results["gate"]:
        print(json.dumps(r), flush=True)
    results["gate_bwd"] = gate_bwd_alone()
    print(json.dumps(results["gate_bwd"]), flush=True)
    results["router_loss"] = [router_loss_alone(grid) for grid in ((64,), (64, 64), (4096,))]
    for r in results["router_loss"]:
        print(json.dumps(r), flush=True)
    results["step"] = step_time()
    print(json.dumps({k: v for k, v in results["step"].items() if not k.startswith("windows")}), flush=True)
    rate = dict(expert_bias_update_rate=1e-3)
    results["balance"] = [
        balance("softmax", **rate),
        balance("sigmoid", router_score="sigmoid", **rate),
        balance("sigmoid c=2.5", router_score="sigmoid", routed_scaling_factor=2.5, **rate),
        balance("v3", router_score="sigmoid", routed_scaling_factor=2.5, expert="swiglu", inner_dim=256,
                shared_inner_dim=1024, **rate)]
    for r in results["balance"]:
        print(json.dumps(r), flush=True)
    results["card_end"] = card()
    with open(output_path("router_score_perf.json"), "w") as f:
        json.dump(results, f, indent=1)
    print(json.dumps(dict(card=results["card"], card_end=results["card_end"])), flush=True)


if __name__ == "__main__":
    main()
