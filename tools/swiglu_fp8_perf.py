"""Cost and gain of the FP8 SwiGLU expert forward, DMoEConfig(expert="swiglu", expert_dtype="fp8")
(writes check_out/swiglu_fp8_perf.json).

1. The two MXFP8 emitters at 65,536 rows, hidden 1024 / inner 2816: RMSNorm + quant against the plain RMSNorm, SwiGLU +
   quant against the plain SwiGLU (both writing the bf16 copy, as training does; the RMSNorm also without it, as serving
   does).  TB/s of the bytes each moves, computed from the shapes: bf16 in, bf16 out, fp32 rstd, E4M3 payload and one
   scale byte per 32 values.  Arms alternate inside every round; medians over ROUNDS x WINDOWS windows of ITERS launches.
   Aim: >= 0.9x the plain kernel's rate.
2. The expert forward at 65,536 tokens, top-4, 64 experts, hidden 1024 (inner 2816) and 2048 (inner 5632), on balanced
   routing (4096 rows per expert) in buffers of its own: each GEMM and the whole chain (grouped RMSNorm .. W2 GEMM with
   the residual), bf16 and fp8 alternating.  TFLOP/s from shapes.  The re-quantisation of the weights that the first
   forward after an optimizer step adds is timed on its own.  Aim: the fp8 chain <= 0.8x the bf16 time.
3. The saturated training step: DMoETrainer, hidden 1024, 64 experts, top-4, 65,536 tokens per step, 2 layers, big path,
   CUDA graph, on a learnable task (labels of a fixed random linear teacher).  300 steps per dtype, timed in windows of
   50 steps with CUDA events, then a second round in the other order (5 windows of 20 steps); reported: the median
   ms / step over all windows and the mean loss of the last 10 of the 300 steps.
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
from lah_b200.ops import fp8, gemm, kernels as K
from lah_b200.ops.expert_blocks import RowPlan, swiglu_mlp_forward, swiglu_mlp_forward_fp8
from lah_b200.parallel import engine as E
from lah_b200.parallel.trainer import DMoETrainer
from tools import output_path

ROUNDS, WINDOWS, ITERS = 3, 3, 20
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


def alternate(arms):
    """median ms per launch of every arm, the arms alternating inside each round (order rotated per round)"""
    for fn in arms.values():   # warm-up
        window(fn, 3)
    ms = {a: [] for a in arms}
    order = list(arms)
    for r in range(ROUNDS):
        for a in order[r % len(order):] + order[:r % len(order)]:
            ms[a] += [window(arms[a], ITERS) for _ in range(WINDOWS)]
    return {a: statistics.median(v) for a, v in ms.items()}


def free():
    gc.collect()
    torch.cuda.empty_cache()


def emitters():
    R, H, I = TOKENS, 1024, 2816
    g = torch.Generator().manual_seed(0)
    x = torch.randn(R, H, generator=g).to(torch.bfloat16).cuda()
    gamma = torch.ones(H, device="cuda")
    n, rstd = torch.empty_like(x), torch.empty(R, device="cuda")
    h = torch.randn(R, 2 * I, generator=g).to(torch.bfloat16).cuda()
    a = torch.empty(R, I, dtype=torch.bfloat16, device="cuda")
    nq = fp8.MXFP8Tensor(R, 1, H, fp8.ACT_TILE, "cuda")
    aq = fp8.MXFP8Tensor(R, 1, I, fp8.ACT_TILE, "cuda")
    ms = alternate({
        "rms": lambda: K.rms_norm_fwd(x, gamma, 1e-6, out=n, rstd=rstd),
        "rms_quant": lambda: K.rms_norm_fwd(x, gamma, 1e-6, out=n, rstd=rstd, quant=nq),
        "rms_quant_no_bf16": lambda: K.rms_norm_fwd(x, gamma, 1e-6, out=None, rstd=rstd, quant=nq),
        "swiglu": lambda: K.swiglu_fwd(h, out=a),
        "swiglu_quant": lambda: K.swiglu_fwd(h, out=a, quant=aq),
    })
    q = lambda C: R * C + R * C // 32            # payload + scales
    moved = {"rms": R * H * 4 + R * 4, "rms_quant": R * H * 4 + R * 4 + q(H), "rms_quant_no_bf16": R * H * 2 + R * 4 + q(H),
             "swiglu": R * I * 6, "swiglu_quant": R * I * 6 + q(I)}
    out = {k: dict(ms=ms[k], bytes=moved[k], tb_s=moved[k] / ms[k] / 1e9) for k in ms}
    out["rms_quant_rate_vs_plain"] = out["rms_quant"]["tb_s"] / out["rms"]["tb_s"]
    out["swiglu_quant_rate_vs_plain"] = out["swiglu_quant"]["tb_s"] / out["swiglu"]["tb_s"]
    return out


def expert_forward(H, I):
    """the chain on balanced routing: 65,536 tokens x top-4 over 64 experts = 4096 rows per expert (whole 256-row
    groups), on its own buffers (the layer's dispatch kernels take hidden 256, 512 and 1024 only)"""
    G, R = 64, TOKENS * 4
    gen = torch.Generator(device="cuda").manual_seed(H)
    bf = dict(dtype=torch.bfloat16, device="cuda")
    tg = torch.arange(G, dtype=torch.int32, device="cuda").repeat_interleave(R // G // 128)
    plan = RowPlan(tile_group=tg)
    xd = torch.randn(R, H, device="cuda", generator=gen).to(torch.bfloat16)
    g = 1 + 0.1 * torch.randn(G, H, device="cuda", generator=gen)
    w13 = (torch.randn(G, 2 * I, H, device="cuda", generator=gen) * H ** -0.5).to(torch.bfloat16)
    w2 = (torch.randn(G, H, I, device="cuda", generator=gen) * I ** -0.5).to(torch.bfloat16)
    w13q = fp8.quantize(w13.view(-1, H), tile_rows=fp8.WEIGHT_TILE, groups=G)
    w2q = fp8.quantize(w2.view(-1, I), tile_rows=fp8.WEIGHT_TILE, groups=G)
    n, yo, h, a = torch.empty(R, H, **bf), torch.empty(R, H, **bf), torch.empty(R, 2 * I, **bf), torch.empty(R, I, **bf)
    rstd = torch.empty(R, device="cuda")
    xq, aq = fp8.MXFP8Tensor(R, 1, H, fp8.ACT_TILE, "cuda"), fp8.MXFP8Tensor(R, 1, I, fp8.ACT_TILE, "cuda")

    def norm(quant):
        K.rms_norm_fwd(xd, g, E.GATED_EPS, out=n, rstd=rstd, tile_group=tg, tile_rows=128, quant=quant)

    def chain_bf16():
        norm(None)
        swiglu_mlp_forward(plan, w13, w2, n, h, a, yo, residual=xd)

    def chain_fp8():
        norm(xq)
        swiglu_mlp_forward_fp8(plan, w13q, w2q, xq, h, a, aq, yo, residual=xd)

    def requant():   # what the first forward after an optimizer step adds
        fp8.quantize(w13.view(-1, H), tile_rows=fp8.WEIGHT_TILE, groups=G, out=w13q)
        fp8.quantize(w2.view(-1, I), tile_rows=fp8.WEIGHT_TILE, groups=G, out=w2q)

    chain_fp8()   # fills xq and aq for the GEMM arms
    ms = alternate({
        "w13_bf16": lambda: gemm.grouped_linear(n, w13, tile_group=tg, out=h),
        "w13_fp8": lambda: fp8.grouped_linear_fp8(xq, w13q, tile_group=tg, out=h),
        "w2_bf16": lambda: gemm.grouped_linear(a, w2, tile_group=tg, out=yo, residual=xd),
        "w2_fp8": lambda: fp8.grouped_linear_fp8(aq, w2q, tile_group=tg, out=yo, residual=xd),
        "chain_bf16": chain_bf16,
        "chain_fp8": chain_fp8,
        "weight_requant": requant,
    })
    flops = {"w13": 2.0 * R * 2 * I * H, "w2": 2.0 * R * H * I}
    out = dict(hidden=H, inner=I, rows=R, ms=ms)
    for k in ("w13", "w2"):
        out[k + "_tflops"] = {d: flops[k] / ms[f"{k}_{d}"] / 1e9 for d in ("bf16", "fp8")}
    out["chain_tflops"] = {d: (flops["w13"] + flops["w2"]) / ms[f"chain_{d}"] / 1e9 for d in ("bf16", "fp8")}
    out["chain_fp8_over_bf16"] = ms["chain_fp8"] / ms["chain_bf16"]
    return out


def training_step():
    g = torch.Generator().manual_seed(1)
    teacher = torch.randn(784, 10, generator=g)
    batches = []
    for _ in range(4):
        xb = torch.randn(TOKENS, 784, generator=g)
        batches.append((xb.cuda(), (xb @ teacher).argmax(-1).cuda()))
    res = {d: dict(windows=[]) for d in ("bf16", "fp8")}

    def run(dtype, windows, steps, record_loss):
        torch.manual_seed(0)
        t = DMoETrainer(E.DMoEConfig(hidden=1024, grid_size=(64,), k=4, num_layers=2, tokens_per_rank=TOKENS,
                                     gate_mode="emulator", expert="swiglu", expert_dtype=dtype, expert_path="big",
                                     lr=1e-3), use_graph=True)
        losses, i = [], 0
        for _ in range(3):   # eager, capture, first replay
            losses.append(t.train_step_device(*batches[i % 4]))
            i += 1
        for _ in range(windows):
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            for _ in range(steps):
                losses.append(t.train_step_device(*batches[i % 4]))
                i += 1
            e.record()
            torch.cuda.synchronize()
            res[dtype]["windows"].append(s.elapsed_time(e) / steps)
        t.ctx.check_status()
        if record_loss:
            last = [float(v) for v in losses[-10:]]
            res[dtype]["steps"] = len(losses)
            res[dtype]["loss_first"] = float(losses[0])
            res[dtype]["loss_last10_mean"] = sum(last) / len(last)
        t.close()
        free()

    for dtype in ("bf16", "fp8"):
        run(dtype, 6, 50, True)
    for dtype in ("fp8", "bf16"):
        run(dtype, 5, 20, False)
    for d in res:
        res[d]["ms_per_step_median"] = statistics.median(res[d]["windows"])
    res["fp8_over_bf16"] = res["fp8"]["ms_per_step_median"] / res["bf16"]["ms_per_step_median"]
    return res


def main():
    torch.cuda.set_device(0)
    out = dict(card=card())
    print(out, flush=True)
    parts = [a for a in sys.argv[1:] if not a.startswith("-")] or ["emitters", "forward", "step"]
    if "emitters" in parts:
        out["emitters"] = emitters()
        print(json.dumps(out["emitters"]), flush=True)
        free()
    if "forward" in parts:
        out["expert_forward"] = []
        for H, I in ((1024, 2816), (2048, 5632)):
            out["expert_forward"].append(expert_forward(H, I))
            free()
        print(json.dumps(out["expert_forward"]), flush=True)
    if "step" in parts:
        out["training_step"] = training_step()
        print(json.dumps(out["training_step"]), flush=True)
    with open(output_path("swiglu_fp8_perf.json"), "w") as f:
        json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
