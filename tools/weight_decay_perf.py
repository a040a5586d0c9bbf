"""GPU cost of weight decay in the optimizer kernels (writes check_out/weight_decay_perf.json).

1. The fused wgrad + AMSGrad kernel at the README's operating point: 64 experts x 16 rows, one 2048 x 2048 weight matrix
   each (34 B of optimizer state and mirror per parameter), on the optimizer stream's 80 CTAs and on all SMs.  No decay,
   L2 and decoupled (AdamW) launches alternate in one process: each round times one window of 20 launches of every mode,
   and each number is the median over 7 rounds.
2. ExpertBackend.backward (forward recompute + backward + optimizer step) with a two-group AdamW (weight_decay 0.01 on the
   weight matrices, none on biases and LayerNorm parameters) for nn.TransformerEncoderLayer(1024, 16) (dropout 0.1,
   32 x 512 tokens) and FeedforwardBlock(1024) (4096 rows): native, native with a single-group Adam (the README's
   configuration), and native=False (the module itself, fp32 eager).  Medians of 5 windows, CUDA events.
The card's name and power limit are read in the same run.
"""
import json
import os
import statistics
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from torch import nn

import lah_b200  # noqa
from lah_b200.models.layers import FeedforwardBlock
from lah_b200.ops import kernels as K
from tools import output_path
from tools.attention_head_dim_perf import card, time_ms

MODES = {"none": dict(), "l2": dict(weight_decay=0.01), "adamw": dict(weight_decay=0.01, decoupled=True)}


def wgrad_adam_modes(max_ctas, rounds=7, iters=20):
    G, N, Kd, rows = 64, 2048, 2048, 16
    off = torch.arange(G, dtype=torch.int32, device="cuda") * rows
    grows = torch.full((G,), rows, dtype=torch.int32, device="cuda")
    dy = (torch.randn(G * rows, N, device="cuda") * 0.1).to(torch.bfloat16)
    x = torch.randn(G * rows, Kd, device="cuda").to(torch.bfloat16)
    p = torch.randn(G, N, Kd, device="cuda") * 0.02
    m, v, vmax = torch.zeros_like(p), torch.zeros_like(p), torch.zeros_like(p)
    pb = torch.empty(G, N, Kd, device="cuda", dtype=torch.bfloat16)
    step = torch.ones(G, dtype=torch.int32, device="cuda")

    def launch(mode):
        K.wgrad_adam(dy, x, off, grows, p=p, m=m, v=v, vmax=vmax, p_bf16=pb, step=step, lr=1e-4, max_ctas=max_ctas,
                     **MODES[mode])
    for mode in MODES:
        for _ in range(3):
            launch(mode)
    torch.cuda.synchronize()
    times = {mode: [] for mode in MODES}
    for _ in range(rounds):
        for mode in MODES:
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            for _ in range(iters):
                launch(mode)
            e.record()
            torch.cuda.synchronize()
            times[mode].append(s.elapsed_time(e) / iters)
    state_bytes = G * N * Kd * 34
    out = {}
    for mode, ts in times.items():
        ms = statistics.median(ts)
        out[mode] = dict(ms=ms, ms_min_max=(min(ts), max(ts)), state_TBps=state_bytes / ms / 1e9)
    return out


def two_group_adamw(module):
    decay = [q for q in module.parameters() if q.dim() >= 2]
    no_decay = [q for q in module.parameters() if q.dim() < 2]
    return torch.optim.AdamW([dict(params=decay), dict(params=no_decay, weight_decay=0.0)], lr=1e-4, weight_decay=0.01,
                             amsgrad=True)


EXPERTS = {
    "nn.TransformerEncoderLayer(1024, 16)": (lambda: nn.TransformerEncoderLayer(1024, 16, batch_first=True), (32, 512, 1024)),
    "FeedforwardBlock(1024)": (lambda: FeedforwardBlock(1024), (4096, 1024)),
}
ARMS = {"native two-group AdamW": (True, two_group_adamw),
        "native single-group Adam": (True, lambda m: torch.optim.Adam(m.parameters(), lr=1e-4, amsgrad=True)),
        "eager two-group AdamW": (False, two_group_adamw)}


def backend_backward(make, shape, native, make_opt):
    torch.manual_seed(0)
    module = make().cuda()
    be = lah_b200.ExpertBackend(name="t", expert=module, opt=make_opt(module), args_schema=(lah_b200.BatchTensorProto(*shape[1:]),),
                                outputs_schema=lah_b200.BatchTensorProto(*shape[1:]), max_batch_size=shape[0], native=native)
    x = torch.randn(*shape, device="cuda")
    g = torch.randn(*shape, device="cuda") * 0.1
    iters, warmup = (20, 3) if native else (5, 2)
    ms = time_ms(lambda: be.backward(x, g), iters=iters, warmup=warmup)
    assert (be._executor is not None) == native, type(be._executor)
    return dict(backward_ms=ms[0], backward_ms_min_max=ms[1:])


if __name__ == "__main__":
    assert torch.cuda.is_available(), "this measurement needs a GPU"
    results = dict(card=card(), wgrad_adam={}, expert_backend={})
    print(results["card"], flush=True)
    for ctas, label in ((80, "80 CTAs"), (0, "all SMs")):
        results["wgrad_adam"][label] = r = wgrad_adam_modes(ctas)
        print("wgrad_adam", label, json.dumps(r), flush=True)
        torch.cuda.empty_cache()
    for name, (make, shape) in EXPERTS.items():
        for arm, (native, make_opt) in ARMS.items():
            results["expert_backend"][f"{name} / {arm}"] = r = backend_backward(make, shape, native, make_opt)
            print(name, arm, r, flush=True)
            torch.cuda.empty_cache()
    with open(output_path("weight_decay_perf.json"), "w") as f:
        json.dump(results, f, indent=1)
