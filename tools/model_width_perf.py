"""GPU cost of the model widths that are odd multiples of 128 or not powers of two (writes check_out/model_width_perf.json).

1. LayerNorm forward and backward (csrc/layernorm.cu) at C = 384, 768, 1536, 3072 beside their power-of-two neighbours
   256 / 512, 512 / 1024, 1024 / 2048, 2048 / 4096, over 32,768 rows (one group, 128-row tiles).  The widths alternate in
   one process: each round times one window of 20 launches of every width, and each number is the median over 7 rounds.
   Bytes are computed from the shapes: forward reads h and writes the output (2 + 2 B per element) plus 8 B of saved
   statistics per row; backward reads da and h, writes dh (2 + 2 + 2 B per element), reads 8 B of statistics per row and
   writes and re-reads 3 fp32 column sums per 128-row tile.  The target is >= 0.9 x the rate of the slower neighbour.
2. ExpertBackend.backward (forward recompute + backward + AMSGrad step) and forward, native against native=False (the
   module itself, fp32 eager), for nn.TransformerEncoderLayer(768, 12, 3072, dropout=0.1, batch_first=True) on 32 x 512
   tokens and FeedforwardBlock(768) on 4096 rows.  Medians of 5 windows, CUDA events.
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

ROWS = 32768
NEIGHBOURS = {384: (256, 512), 768: (512, 1024), 1536: (1024, 2048), 3072: (2048, 4096)}


def ln_bytes(C, rows=ROWS):
    tiles = -(-rows // 128)
    return dict(fwd=4 * rows * C + 8 * rows, bwd=6 * rows * C + 8 * rows + 2 * 3 * 4 * C * tiles)


def ln_widths(rounds=7, iters=20):
    widths = sorted({c for c in NEIGHBOURS} | {n for ns in NEIGHBOURS.values() for n in ns})
    bufs = {}
    for C in widths:
        g = torch.Generator().manual_seed(C)
        h = torch.randn(ROWS, C, generator=g).to(torch.bfloat16).cuda()
        da = (torch.randn(ROWS, C, generator=g) * 0.1).to(torch.bfloat16).cuda()
        gamma, beta = (1 + 0.1 * torch.randn(1, C, generator=g)).cuda(), (0.1 * torch.randn(1, C, generator=g)).cuda()
        bufs[C] = dict(h=h, da=da, a=torch.empty_like(h), dh=torch.empty_like(h), gamma=gamma, beta=beta,
                       mean=torch.empty(ROWS, device="cuda"), rstd=torch.empty(ROWS, device="cuda"),
                       grads=[torch.zeros(1, C, device="cuda") for _ in range(3)])

    def fwd(C):
        b = bufs[C]
        K.ln_relu_fwd(b["h"], b["gamma"], b["beta"], None, out=b["a"], mean=b["mean"], rstd=b["rstd"])

    def bwd(C):
        b = bufs[C]
        dg, db, dbias = b["grads"]
        K.ln_relu_bwd(b["da"], b["h"], b["mean"], b["rstd"], b["gamma"], b["beta"], None, dh=b["dh"], dgamma=dg,
                      dbeta=db, dbias=dbias)

    for C in widths:
        for _ in range(3):
            fwd(C), bwd(C)
    torch.cuda.synchronize()
    times = {(C, k): [] for C in widths for k in ("fwd", "bwd")}
    for _ in range(rounds):
        for C in widths:
            for k, fn in (("fwd", fwd), ("bwd", bwd)):
                s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                s.record()
                for _ in range(iters):
                    fn(C)
                e.record()
                torch.cuda.synchronize()
                times[(C, k)].append(s.elapsed_time(e) / iters)
    rate = {}
    out = {}
    for (C, k), ts in times.items():
        ms = statistics.median(ts)
        rate[(C, k)] = ln_bytes(C)[k] / ms / 1e9
        out[f"{k} C={C}"] = dict(ms=ms, ms_min_max=(min(ts), max(ts)), TBps=rate[(C, k)])
    verdict = {}
    for C, (lo, hi) in NEIGHBOURS.items():
        for k in ("fwd", "bwd"):
            slower = min(rate[(lo, k)], rate[(hi, k)])
            ratio = rate[(C, k)] / slower
            verdict[f"{k} C={C}"] = dict(TBps=rate[(C, k)], slower_neighbour_TBps=slower, ratio=ratio,
                                         target_met=ratio >= 0.9)
    return out, verdict


EXPERTS = {
    "nn.TransformerEncoderLayer(768, 12, 3072)": (
        lambda: nn.TransformerEncoderLayer(768, 12, 3072, dropout=0.1, batch_first=True), (32, 512, 768)),
    "FeedforwardBlock(768)": (lambda: FeedforwardBlock(768), (4096, 768)),
}


def backend_times(make, shape, native):
    torch.manual_seed(0)
    module = make().cuda()
    be = lah_b200.ExpertBackend(name="t", expert=module, opt=torch.optim.Adam(module.parameters(), lr=1e-4, amsgrad=True),
                                args_schema=(lah_b200.BatchTensorProto(*shape[1:]),),
                                outputs_schema=lah_b200.BatchTensorProto(*shape[1:]), max_batch_size=shape[0], native=native)
    x = torch.randn(*shape, device="cuda")
    g = torch.randn(*shape, device="cuda") * 0.1
    iters, warmup = (20, 3) if native else (5, 2)
    bwd = time_ms(lambda: be.backward(x, g), iters=iters, warmup=warmup)
    fwd = time_ms(lambda: be.forward(x), iters=iters, warmup=warmup)
    assert (be._executor is not None) == native, type(be._executor)
    return dict(backward_ms=bwd[0], backward_ms_min_max=bwd[1:], forward_ms=fwd[0], forward_ms_min_max=fwd[1:])


if __name__ == "__main__":
    assert torch.cuda.is_available(), "this measurement needs a GPU"
    results = dict(card=card(), layernorm={}, expert_backend={})
    print(results["card"], flush=True)
    results["layernorm"], results["layernorm_target"] = ln_widths()
    for k, v in results["layernorm"].items():
        print("layernorm", k, json.dumps(v), flush=True)
    for k, v in results["layernorm_target"].items():
        print("target", k, json.dumps(v), flush=True)
    torch.cuda.empty_cache()
    for name, (make, shape) in EXPERTS.items():
        for native in (True, False):
            results["expert_backend"][f"{name} / {'native' if native else 'eager'}"] = r = backend_times(make, shape, native)
            print(name, "native" if native else "eager", json.dumps(r), flush=True)
            torch.cuda.empty_cache()
    with open(output_path("model_width_perf.json"), "w") as f:
        json.dump(results, f, indent=1)
