"""Training step of the fused DMoE engine with SwiGLU experts (writes check_out/dmoe_swiglu_perf.json).

The bench operating point (64 experts, top-4, 256 samples per step, 4 layers, emulator gate; bench.py has no expert flag):
1. DMoETrainer(expert="swiglu") at hidden 512 and 1024 on the small path (auto) and with expert_path="big";
2. FastBaselineTrainer (torch.topk + all_to_all_single + cuBLAS bmm + fused torch Adam) with the same configuration;
3. the FeedforwardBlock step at hidden 512, for context.
Each arm: train_step_device on one fixed synthetic batch (under the trainer's CUDA graph where it uses one), warm-up, then
the median of 5 windows of 10 steps timed with CUDA events.  The HBM bound of an engine step follows the README's rule:
38 B per parameter of the experts that received rows in the step (counted per layer from the routing of the timed batch) at
3.35 TB/s.  A torch.profiler run of the hidden-1024 small-path step, apart from the timed runs, gives its kernel time by
kernel.  The card's name, power limit and maximum SM clock are read in the same run.
"""
import gc
import json
import os
import statistics
import subprocess
import sys
from collections import defaultdict

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

import lah_b200  # noqa
from lah_b200.parallel import engine as E
from lah_b200.parallel.baseline_fast import FastBaselineTrainer
from lah_b200.parallel.trainer import DMoETrainer
from tools import output_path

BENCH = dict(grid_size=(64,), k=4, num_layers=4, tokens_per_rank=256, gate_mode="emulator")
BYTES_PER_PARAM = 38
HBM_TBPS = 3.35
WINDOWS, ITERS, WARMUP = 5, 10, 5


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else torch.cuda.get_device_name()


def batch(cfg):
    g = torch.Generator().manual_seed(0)
    x = torch.randn(cfg.tokens_per_rank, cfg.in_features, generator=g).cuda()
    y = torch.randint(0, cfg.num_classes, (cfg.tokens_per_rank,), generator=g).cuda()
    return x, y


def time_steps(step):
    for _ in range(WARMUP):
        step()
    torch.cuda.synchronize()
    out = []
    for _ in range(WINDOWS):
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        for _ in range(ITERS):
            step()
        e.record()
        torch.cuda.synchronize()
        out.append(s.elapsed_time(e) / ITERS)
    return statistics.median(out), min(out), max(out)


def release():
    gc.collect()
    torch.cuda.empty_cache()


def engine_arm(profile=False, **kw):
    cfg = E.DMoEConfig(**BENCH, **kw)
    t = DMoETrainer(cfg)
    x, y = batch(cfg)
    ms = time_steps(lambda: t.train_step_device(x, y))
    t.ctx.check_status()
    per_expert = sum(int(torch.tensor(s).prod()) for s in cfg.seg_shapes().values())
    active = sum(int((b.ws.step_rows > 0).sum()) for b in t.model.blocks)
    bound_ms = BYTES_PER_PARAM * per_expert * active / (HBM_TBPS * 1e12) * 1e3
    out = dict(expert=cfg.expert, hidden=cfg.hidden, inner=cfg.inner, path="small" if t.ctx.small else "big",
               graph=t.use_graph, ms_per_step=ms[0], ms_min_max=ms[1:], samples_per_s=cfg.tokens_per_rank / ms[0] * 1e3,
               active_experts=active, params_per_expert=per_expert, hbm_bound_ms=bound_ms,
               fraction_of_hbm_bound=bound_ms / ms[0])
    if profile:
        out["profile"] = kernel_profile(lambda: t.train_step_device(x, y))
    t.close()
    del t
    release()
    return out


def kernel_profile(step, steps=5):
    """kernel time per kernel name (summed over `steps` steps), largest first, as ms per step and share"""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(steps):
            step()
        torch.cuda.synchronize()
    per = defaultdict(float)
    for ev in prof.events():
        if ev.device_type == torch.autograd.DeviceType.CUDA:
            per[ev.name[:90]] += ev.device_time_total / 1e3 / steps
    total = sum(per.values())
    top = sorted(per.items(), key=lambda kv: -kv[1])[:14]
    return dict(kernel_ms_per_step=total, top=[dict(kernel=k, ms=v, share=v / total) for k, v in top])


def baseline_arm(**kw):
    cfg = E.DMoEConfig(**BENCH, **kw)
    t = FastBaselineTrainer(cfg)
    x, y = batch(cfg)
    ms = time_steps(lambda: t.train_step_device(x, y))
    out = dict(arm="baseline_fast", expert=cfg.expert, hidden=cfg.hidden, inner=cfg.inner, ms_per_step=ms[0],
               ms_min_max=ms[1:], samples_per_s=cfg.tokens_per_rank / ms[0] * 1e3)
    del t
    release()
    return out


def main():
    results = dict(card=card(), device=torch.cuda.get_device_name(), arms=[])
    arms = results["arms"]
    for hidden in (512, 1024):
        arms.append(engine_arm(hidden=hidden, expert="swiglu", profile=hidden == 1024))
        print(json.dumps(arms[-1]), flush=True)
        arms.append(engine_arm(hidden=hidden, expert="swiglu", expert_path="big"))
        print(json.dumps(arms[-1]), flush=True)
        arms.append(baseline_arm(hidden=hidden, expert="swiglu"))
        print(json.dumps(arms[-1]), flush=True)
    arms.append(engine_arm(hidden=512, expert="ffn"))
    print(json.dumps(arms[-1]), flush=True)
    for hidden in (512, 1024):
        small = next(a for a in arms if a.get("path") == "small" and a["hidden"] == hidden and a["expert"] == "swiglu")
        base = next(a for a in arms if a.get("arm") == "baseline_fast" and a["hidden"] == hidden)
        results[f"swiglu_{hidden}_small_speedup_over_baseline_fast"] = base["ms_per_step"] / small["ms_per_step"]
    results["card"] = card()   # read again at the end of the run
    with open(output_path("dmoe_swiglu_perf.json"), "w") as f:
        json.dump(results, f, indent=1)
    print(json.dumps({k: v for k, v in results.items() if k != "arms"}), flush=True)


if __name__ == "__main__":
    main()
