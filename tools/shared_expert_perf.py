"""Cost of the shared expert of DMoEConfig(shared_inner_dim=...) (writes check_out/shared_expert_perf.json).

1. Step time at the bench operating point (expert="swiglu", emulator gate, 64 experts, top-4, 256 samples per step,
   4 layers, CUDA graph), hidden 512 and 1024, shared_inner_dim 0, the routed inner width I and 4 I (Qwen-MoE's ratio).
   Each round builds the trainer of one arm, warms it up, times WINDOWS windows of ITERS steps with CUDA events and closes
   it; the order of the arms rotates per round.  Reported: the median over all windows of each arm and the added ms
   against the bytes the shared expert moves per step, computed from its shapes: per parameter 6 B (cast: fp32 read + bf16
   write) + 2 + 2 (bf16 weight reads of the forward and the dgrad) + 8 (fp32 wgrad accumulate: read + write) + 40 (the
   trainer's AMSGrad over p, g, m, v, vmax: 5 reads + 5 writes of fp32), at 3.35 TB/s.  Aim: added ms <= 1.5 x that time.
2. The saturated regime (65,536 tokens, hidden 1024, big path, shared_inner_dim = I): after one training step of a layer,
   the shared expert's forward, dgrad and wgrad GEMMs and the routed experts' grouped GEMMs of the same kind are launched
   again on the layer's own buffers, CUDA events around ITERS_G launches, median of 5 windows.  TFLOP/s from shapes: the
   shared GEMMs on the batch padded to 128 rows, the routed ones on the rows the layout exchange padded (total_rows).
3. combine_rows with and without the addend at 256 and 65,536 tokens, on the routing of that layer's last forward
   (arms alternated, median of 9 windows of ITERS_C launches).
4. A torch.profiler kernel table of one bench-point step (hidden 512, shared = 4 I) in a run of its own.
The card's name, power limit and maximum SM clock are read in the same run.
"""
import gc
import json
import os
import statistics
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

import lah_b200  # noqa
from lah_b200.models.layers import gated_inner_dim
from lah_b200.ops import gemm, kernels as K
from lah_b200.parallel import engine as E
from lah_b200.parallel.trainer import DMoETrainer
from tools import output_path

BENCH = dict(grid_size=(64,), k=4, num_layers=4, tokens_per_rank=256, gate_mode="emulator", expert="swiglu")
ROUNDS, WINDOWS, ITERS, WARMUP = 3, 3, 20, 10
ITERS_G, ITERS_C = 20, 200
HBM = 3.35e12
BYTES_PER_PARAM = 6 + 2 + 2 + 8 + 40


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


def free():
    """return a closed trainer's memory before the next is built (hidden 1024 holds ~48 GB of expert state)"""
    gc.collect()
    torch.cuda.empty_cache()


def shared_params(H, Is, layers):
    return layers * (H + 3 * H * Is)


def step_time(H):
    I = gated_inner_dim(H)
    arms = {"0": 0, "I": I, "4I": 4 * I}
    g = torch.Generator().manual_seed(0)
    x = torch.randn(256, 784, generator=g).cuda()
    y = torch.randint(0, 10, (256,), generator=g).cuda()
    ms = {a: [] for a in arms}
    order = list(arms)
    for r in range(ROUNDS):
        for arm in order[r % 3:] + order[:r % 3]:
            t = DMoETrainer(E.DMoEConfig(**BENCH, hidden=H, shared_inner_dim=arms[arm]))
            for _ in range(WARMUP):
                t.train_step_device(x, y)
            ms[arm] += [window(lambda: t.train_step_device(x, y), ITERS) for _ in range(WINDOWS)]
            t.ctx.check_status()
            assert t._graph is not None
            t.close()
            del t
            free()
    base = statistics.median(ms["0"])
    out = dict(hidden=H, routed_inner=I, ms_per_step={a: statistics.median(v) for a, v in ms.items()}, windows=ms)
    for arm in ("I", "4I"):
        Is = arms[arm]
        nbytes = shared_params(H, Is, BENCH["num_layers"]) * BYTES_PER_PARAM
        added = out["ms_per_step"][arm] - base
        bound = nbytes / HBM * 1e3
        out[arm] = dict(shared_inner_dim=Is, params=shared_params(H, Is, BENCH["num_layers"]), bytes=nbytes,
                        added_ms=added, hbm_ms=bound, added_over_hbm=added / bound, aim_met=added <= 1.5 * bound)
    return out


def gemm_rates():
    H, B = 1024, 65536
    I = gated_inner_dim(H)
    cfg = E.DMoEConfig(hidden=H, grid_size=(64,), k=4, num_layers=1, tokens_per_rank=B, gate_mode="emulator",
                       expert="swiglu", expert_path="big", shared_inner_dim=I)
    ctx = E.EngineContext(cfg)
    layer = E.FusedDMoE(cfg, ctx).cuda().train()
    x = torch.randn(B, H, device="cuda").to(torch.bfloat16).requires_grad_(True)
    layer(x).backward(torch.randn(B, H, device="cuda").to(torch.bfloat16))
    torch.cuda.synchronize()
    ctx.check_status()
    ws, sh = layer.ws, layer.shard
    Bp, plan = layer._shared_plan(B)
    go, tg = plan.group_off, plan.tile_group
    rows = int(ws.total_rows.item())
    G = ctx.G_tot
    w13g, w2g = torch.zeros(1, 2 * I, H, device="cuda"), torch.zeros(1, H, I, device="cuda")
    rw13, rw2 = torch.zeros(G, 2 * I, H, device="cuda"), torch.zeros(G, H, I, device="cuda")
    da, dh, dn = ctx.shared_da[:Bp], ctx.shared_dh[:Bp], ctx.shared_dn[:Bp]
    gys = ws.shared_gy[:Bp]
    calls = {
        "shared_fwd": (lambda: (gemm.grouped_linear(ws.shared_n[:Bp], ws.shared_w13, tile_group=tg, out=ws.shared_h[:Bp]),
                                gemm.grouped_linear(ws.shared_a[:Bp], ws.shared_w2, tile_group=tg, out=ws.shared_y[:Bp])),
                       Bp),
        "shared_dgrad": (lambda: (gemm.grouped_linear(gys, ws.shared_w2, tile_group=tg, w_is_kn=True, out=da),
                                  gemm.grouped_linear(dh, ws.shared_w13, tile_group=tg, w_is_kn=True, out=dn)), Bp),
        "shared_wgrad": (lambda: (gemm.grouped_wgrad(dh, ws.shared_n[:Bp], go, 1, out=w13g, accumulate=True),
                                  gemm.grouped_wgrad(gys, ws.shared_a[:Bp], go, 1, out=w2g, accumulate=True)), Bp),
        "routed_fwd": (lambda: (gemm.grouped_linear(ws.n[:rows], sh.bf16["w13"], tile_group=ws.tile_group, out=ws.h[:rows]),
                                gemm.grouped_linear(ws.a[:rows], sh.bf16["w2"], tile_group=ws.tile_group,
                                                    out=ws.yo[:rows])), rows),
        "routed_dgrad": (lambda: (gemm.grouped_linear(ctx.gyd[:rows], sh.bf16["w2"], tile_group=ws.tile_group,
                                                      w_is_kn=True, out=ctx.da[:rows]),
                                  gemm.grouped_linear(ctx.dh[:rows], sh.bf16["w13"], tile_group=ws.tile_group,
                                                      w_is_kn=True, out=ctx.dn[:rows])), rows),
        "routed_wgrad": (lambda: (gemm.grouped_wgrad(ctx.dh[:rows], ws.n[:rows], ws.group_off, G, out=rw13),
                                  gemm.grouped_wgrad(ctx.gyd[:rows], ws.a[:rows], ws.group_off, G, out=rw2)), rows),
    }
    for fn, _ in calls.values():
        fn()
    torch.cuda.synchronize()
    ms = {n: [] for n in calls}
    for i in range(5):
        for n in (list(calls) if i % 2 == 0 else list(calls)[::-1]):
            ms[n].append(window(calls[n][0], ITERS_G))
    out = dict(tokens=B, hidden=H, inner=I, shared_rows=Bp, routed_rows=rows)
    for n, (_, r) in calls.items():
        flops = 2 * r * H * 3 * I   # [W1; W3] (2 I x H) and W2 (H x I): 3 H I multiply-adds per row
        t = statistics.median(ms[n])
        out[n] = dict(ms=t, tflops=flops / (t * 1e-3) / 1e12)
    for kind in ("fwd", "dgrad", "wgrad"):
        out[f"{kind}_shared_over_routed"] = out[f"shared_{kind}"]["tflops"] / out[f"routed_{kind}"]["tflops"]
    out["combine"] = combine_times(layer, ctx)
    ctx.close()
    del layer, calls, x
    free()
    return out


def combine_times(layer, ctx):
    ws, k = layer.ws, layer.cfg.k
    res = {}
    for B in (256, 65536):
        P = B * k
        idx, pair_row, w = ws.idx[:P], ws.pair_row[:P], ws.w[:P]
        y = torch.empty(B, layer.cfg.hidden, dtype=torch.bfloat16, device="cuda")
        add = ws.shared_y[:B]
        arms = {"plain": None, "addend": add}
        fn = {a: (lambda a=a: K.combine_rows(ws.yo_off, idx, pair_row, w, y, k, ctx.E_loc, route_owner=ws.route_owner,
                                             addend=arms[a])) for a in arms}
        for f in fn.values():
            f()
        us = {a: [] for a in arms}
        for i in range(9):
            for a in (("plain", "addend") if i % 2 == 0 else ("addend", "plain")):
                us[a].append(window(fn[a], ITERS_C) * 1e3)
        m = {a: statistics.median(v) for a, v in us.items()}
        read = B * k * layer.cfg.hidden * 2
        res[str(B)] = dict(us_plain=m["plain"], us_addend=m["addend"], slowdown_pct=(m["addend"] / m["plain"] - 1) * 100,
                           gbps_plain=(read + B * layer.cfg.hidden * 2) / (m["plain"] * 1e-6) / 1e9,
                           gbps_addend=(read + 2 * B * layer.cfg.hidden * 2) / (m["addend"] * 1e-6) / 1e9)
    return res


def profile_step():
    t = DMoETrainer(E.DMoEConfig(**BENCH, hidden=512, shared_inner_dim=4 * gated_inner_dim(512)), use_graph=False)
    g = torch.Generator().manual_seed(0)
    x = torch.randn(256, 784, generator=g).cuda()
    y = torch.randint(0, 10, (256,), generator=g).cuda()
    for _ in range(3):
        t.train_step_device(x, y)
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(5):
            t.train_step_device(x, y)
        torch.cuda.synchronize()
    t.close()
    del t
    free()
    table = {}
    for ev in prof.key_averages():
        if ev.device_time_total > 0:
            table[ev.key] = dict(us_total_per_step=ev.device_time_total / 5, calls_per_step=ev.count / 5)
    return dict(sorted(table.items(), key=lambda kv: -kv[1]["us_total_per_step"])[:30])


def main():
    results = dict(card=card(), device=torch.cuda.get_device_name())
    results["step"] = []
    for H in (512, 1024):
        results["step"].append(step_time(H))
        print(json.dumps({k: v for k, v in results["step"][-1].items() if k != "windows"}), flush=True)
    results["saturated"] = gemm_rates()
    print(json.dumps(results["saturated"]), flush=True)
    results["profile_bench_h512_4I"] = profile_step()
    print(json.dumps(results["profile_bench_h512_4I"]), flush=True)
    results["card_end"] = card()
    with open(output_path("shared_expert_perf.json"), "w") as f:
        json.dump(results, f, indent=1)
    print(json.dumps(dict(card=results["card"], card_end=results["card_end"])), flush=True)


if __name__ == "__main__":
    main()
