"""GPU cost of the gated (SwiGLU) expert (writes check_out/gated_ffn_perf.json).

1. ExpertBackend.backward (forward recompute + backward + optimizer step) and forward of GatedFeedforwardBlock(1024)
   (inner 2816) and GatedFeedforwardBlock(4096) (inner 11008) at 16, 256 and 4096 rows, native against native=False (the
   fp32 module and torch Adam, amsgrad).  Medians of 5 windows, CUDA events, after warm-up.
2. At 16 rows: the backward's effective optimizer-state bandwidth, 34 B per parameter (p, m, v, vmax read and written,
   the bf16 mirror written) over the 3 hid inner weight parameters, divided by the backward's time.
3. At 4096 rows: the share of the native backward's kernel time taken by the RMSNorm and SwiGLU kernels (and the column
   sum that finishes the RMSNorm backward), from a torch.profiler run kept apart from the timed runs.
4. RMSNorm forward and backward (as the executor runs it: dres, 16-row tiles) at 32,768 rows for hid 1024, 2048 and 4096,
   beside the LayerNorm kernels at the same widths in the same run.  Bytes from the shapes: forward reads x and writes n
   (2 + 2 B per element) and 4 B of rstd per row; backward reads dn, x and dres and writes dx (4 x 2 B per element), reads
   4 B of rstd per row and writes and re-reads one fp32 column sum per tile.  LayerNorm bytes as tools/model_width_perf.py.
The card's name and power limit are read in the same run.
"""
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

import lah_b200  # noqa
from lah_b200.models.layers import GatedFeedforwardBlock
from lah_b200.ops import kernels as K
from tools import output_path
from tools.attention_head_dim_perf import card, time_ms
from tools.model_width_perf import ln_bytes

HIDS = (1024, 4096)
ROWS = (16, 256, 4096)
NORM_ROWS = 32768
NORM_WIDTHS = (1024, 2048, 4096)
STATE_BYTES_PER_PARAM = 34
FUSED_KERNEL_TBPS = 2.85   # the fused wgrad + AMSGrad kernel's state stream in the README


def _backend(hid, rows, native):
    torch.manual_seed(0)
    module = GatedFeedforwardBlock(hid).cuda()
    be = lah_b200.ExpertBackend(name="g", expert=module, opt=torch.optim.Adam(module.parameters(), lr=1e-4, amsgrad=True),
                                args_schema=(lah_b200.BatchTensorProto(hid),), outputs_schema=lah_b200.BatchTensorProto(hid),
                                max_batch_size=rows, native=native)
    x = torch.randn(rows, hid, device="cuda")
    g = torch.randn(rows, hid, device="cuda") * 0.1
    return module, be, x, g


def backend_times(hid, rows, native):
    module, be, x, g = _backend(hid, rows, native)
    iters, warmup = (10, 3) if native else (3, 2)
    bwd = time_ms(lambda: be.backward(x, g), iters=iters, warmup=warmup)
    fwd = time_ms(lambda: be.forward(x), iters=iters, warmup=warmup)
    assert (be._executor is not None) == native, type(be._executor)
    out = dict(backward_ms=bwd[0], backward_ms_min_max=bwd[1:], forward_ms=fwd[0], forward_ms_min_max=fwd[1:])
    if rows == 16 and native:
        weights = 3 * hid * module.w1.out_features
        out["optimizer_state_TBps"] = STATE_BYTES_PER_PARAM * weights / (bwd[0] * 1e-3) / 1e12
        out["of_fused_kernel_figure"] = out["optimizer_state_TBps"] / FUSED_KERNEL_TBPS
    return out


def kernel_shares(hid, rows=4096):
    """share of the native backward's device kernel time per kernel family, from one profiled run of 5 calls"""
    from torch.profiler import ProfilerActivity, profile
    _, be, x, g = _backend(hid, rows, True)
    for _ in range(3):
        be.backward(x, g)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(5):
            be.backward(x, g)
        torch.cuda.synchronize()
    total, fam = 0.0, {"rms_norm": 0.0, "swiglu": 0.0, "group_tile_sum": 0.0}
    for ev in prof.key_averages():
        if ev.device_type != torch.autograd.DeviceType.CUDA:
            continue
        t = ev.device_time_total
        if "memcpy" in ev.key.lower() or "memset" in ev.key.lower():
            continue
        total += t
        for k in fam:
            if k in ev.key:
                fam[k] += t
    return dict(kernel_us_per_call=total / 5, **{f"{k}_share": v / total for k, v in fam.items()},
                norm_and_gate_share=sum(fam.values()) / total)


def norms():
    out = {}
    for C in NORM_WIDTHS:
        gen = torch.Generator().manual_seed(C)
        x = torch.randn(NORM_ROWS, C, generator=gen).to(torch.bfloat16).cuda()
        d = (torch.randn(NORM_ROWS, C, generator=gen) * 0.1).to(torch.bfloat16).cuda()
        res = (torch.randn(NORM_ROWS, C, generator=gen) * 0.1).to(torch.bfloat16).cuda()
        gamma, beta = (1 + 0.1 * torch.randn(C, generator=gen)).cuda(), torch.zeros(1, C, device="cuda")
        n, dx = torch.empty_like(x), torch.empty_like(x)
        rstd, mean = torch.empty(NORM_ROWS, device="cuda"), torch.empty(NORM_ROWS, device="cuda")
        dg = torch.zeros(C, device="cuda")
        grads = [torch.zeros(1, C, device="cuda") for _ in range(3)]
        tiles = NORM_ROWS // 16
        rms_bytes = dict(fwd=4 * NORM_ROWS * C + 4 * NORM_ROWS, bwd=8 * NORM_ROWS * C + 4 * NORM_ROWS + 2 * 4 * C * tiles)
        runs = {
            "rms_fwd": (lambda: K.rms_norm_fwd(x, gamma, 1e-6, out=n, rstd=rstd), rms_bytes["fwd"]),
            "rms_bwd": (lambda: K.rms_norm_bwd(d, x, rstd, gamma, dx=dx, dgamma=dg, dres=res, tile_rows=16), rms_bytes["bwd"]),
            "ln_fwd": (lambda: K.ln_relu_fwd(x, gamma[None], beta, None, out=n, mean=mean, rstd=rstd, relu=False),
                       ln_bytes(C, NORM_ROWS)["fwd"]),
            "ln_bwd": (lambda: K.ln_relu_bwd(d, x, mean, rstd, gamma[None], beta, None, dh=dx, dgamma=grads[0],
                                             dbeta=grads[1], dbias=grads[2], relu=False), ln_bytes(C, NORM_ROWS)["bwd"]),
        }
        for name, (fn, nbytes) in runs.items():
            if name == "rms_bwd":   # the backward reads the rstd of the RMSNorm forward
                K.rms_norm_fwd(x, gamma, 1e-6, out=n, rstd=rstd)
            if name == "ln_bwd":
                K.ln_relu_fwd(x, gamma[None], beta, None, out=n, mean=mean, rstd=rstd, relu=False)
            ms = time_ms(fn)
            out[f"{name} C={C}"] = dict(ms=ms[0], ms_min_max=ms[1:], TBps=nbytes / (ms[0] * 1e-3) / 1e12)
    return out


if __name__ == "__main__":
    assert torch.cuda.is_available(), "this measurement needs a GPU"
    results = dict(card=card(), expert_backend={}, kernel_shares={}, norms={})
    print(results["card"], flush=True)
    for hid in HIDS:
        for rows in ROWS:
            for native in (True, False):
                key = f"GatedFeedforwardBlock({hid}) rows={rows} / {'native' if native else 'eager'}"
                results["expert_backend"][key] = r = backend_times(hid, rows, native)
                print(key, json.dumps(r), flush=True)
                torch.cuda.empty_cache()
    for hid in HIDS:
        results["kernel_shares"][f"GatedFeedforwardBlock({hid}) rows=4096"] = r = kernel_shares(hid)
        print("kernel shares", hid, json.dumps(r), flush=True)
        torch.cuda.empty_cache()
    results["norms"] = norms()
    for k, v in results["norms"].items():
        print("norm", k, json.dumps(v), flush=True)
    with open(output_path("gated_ffn_perf.json"), "w") as f:
        json.dump(results, f, indent=1)
