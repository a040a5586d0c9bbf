"""Cost and effect of an expert capacity (DMoEConfig(expert_capacity_factor=f), DESIGN.md §6f); writes
check_out/expert_capacity_perf.json.

1. Cost when nothing is dropped: f = 0 against f = 64 (C >= every expert's rows here), ROUNDS rounds with the arms'
   order alternating, CUDA-graph steps timed with CUDA events.  At the bench point (emulator gate, 64 experts, top-4,
   256 tokens per GPU, 4 layers, small path) and on the saturated big path (65,536 tokens, BIG_LAYERS layers).
2. Collapsed routing: the emulator gate's keys are biased so that most tokens pick the first world-th of the experts
   (one rank's at world > 1).  Small and big path, f in {dropless, 2, 1.25, 1}: ms per step, the most rows one rank
   processes (box-wide step_rows of its experts, the largest over ranks) and the dropped share of the routed pairs.
   Under torchrun every rank runs the same program (world = its size); alone it runs at world 1.
The card's name, power limit and maximum SM clock are read in the same run.
"""
import json
import os
import statistics
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import torch.distributed as dist

import lah_b200  # noqa
from lah_b200.parallel import engine as E
from lah_b200.parallel.trainer import DMoETrainer
from tools import output_path
from tools.router_score_perf import card

BENCH = dict(hidden=512, grid_size=(64,), k=4, num_layers=4, tokens_per_rank=256, gate_mode="emulator")
BIG = dict(hidden=512, grid_size=(64,), k=4, num_layers=2, tokens_per_rank=65536, gate_mode="emulator",
           expert_path="big")
ROUNDS, WARMUP, ITERS = 6, 10, 30
FACTORS = (0.0, 2.0, 1.25, 1.0)


def step_ms(t, x, y, iters):
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(iters):
        t.train_step_device(x, y)
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / iters


def batch(cfg, seed):
    g = torch.Generator().manual_seed(seed)
    T = cfg["tokens_per_rank"]
    return torch.randn(T, 784, generator=g).cuda(), torch.randint(0, 10, (T,), generator=g).cuda()


def collapse(t, world):
    """most tokens' top-k inside the first E / max(world, 8) experts"""
    n = t.cfg.num_experts // max(world, 8)
    with torch.no_grad():
        for b in t.model.blocks:
            b.expert_keys[:, :n] += 3.0 * b.expert_keys.abs().mean()


def no_drop_cost(base, iters):
    x, y = batch(base, 0)
    ms = {"f0": [], "f64": []}
    for r in range(ROUNDS):
        for arm in (("f0", "f64") if r % 2 == 0 else ("f64", "f0")):
            t = DMoETrainer(E.DMoEConfig(**base, expert_capacity_factor=0.0 if arm == "f0" else 64.0), use_graph=True)
            for _ in range(WARMUP):
                t.train_step_device(x, y)
            ms[arm].append(step_ms(t, x, y, iters))
            if arm == "f64":
                assert all(layer["dropped_pairs"] == 0 for layer in t.log_step()["layers"])
            t.close()
    med = {a: statistics.median(v) for a, v in ms.items()}
    return dict(ms=ms, median_ms=med, ratio=med["f64"] / med["f0"])


def collapsed(base, world, rank, iters):
    x, y = batch(base, 1 + rank)
    out = {}
    for f in FACTORS:
        t = DMoETrainer(E.DMoEConfig(**base, expert_capacity_factor=f), use_graph=True)
        collapse(t, world)
        for _ in range(WARMUP):
            t.train_step_device(x, y)
        ms = statistics.median(step_ms(t, x, y, iters) for _ in range(3))
        rec = t.log_step()
        rows = torch.tensor([sum(int(b.ws.step_rows.sum()) for b in t.model.blocks)], device="cuda")
        if world > 1:
            dist.all_reduce(rows, op=dist.ReduceOp.MAX)
        routed = base["tokens_per_rank"] * base["k"] * world * base["num_layers"]
        dropped = sum(layer.get("dropped_pairs", 0) for layer in rec["layers"])
        out["dropless" if f == 0.0 else f"f{f}"] = dict(
            step_ms=ms, max_rows_per_rank_all_layers=int(rows), dropped_share=dropped / routed,
            expert_capacity=[layer.get("expert_capacity") for layer in rec["layers"]])
        t.close()
    return out


def main():
    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    if world > 1:
        torch.cuda.set_device(int(os.environ["LOCAL_RANK"]))
        dist.init_process_group("nccl", device_id=torch.device("cuda", int(os.environ["LOCAL_RANK"])))
    res = dict(card=card(), world=world)
    if world == 1:
        res["no_drop_bench_point"] = no_drop_cost(dict(BENCH, expert_path="small"), ITERS)
        res["no_drop_big_65536"] = no_drop_cost(BIG, 5)
    res["collapsed_small"] = collapsed(dict(BENCH, expert_path="small"), world, rank, ITERS)
    res["collapsed_big"] = collapsed(dict(BENCH, expert_path="big"), world, rank, ITERS)
    if rank == 0:
        with open(output_path("expert_capacity_perf.json"), "w") as fh:
            json.dump(res, fh, indent=1)
        print(json.dumps(res, indent=1))
    if world > 1:
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
