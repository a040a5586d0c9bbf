"""Tiny driver for ncu captures (run under `ncu -k regex:...`): launches each hot kernel twice at bench-like shapes."""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

import lah_b200  # noqa
from lah_b200.ops import fp8, gemm, kernels as K

torch.manual_seed(0)
G, R = 64, 2048
rows = G * R
tg = torch.arange(G, device="cuda", dtype=torch.int32).repeat_interleave(R // 128)
which = set(sys.argv[1:]) or {"fp8", "bf16", "attn", "ln"}   # + "small"
if "fp8" in which or "bf16" in which:
    N = Kd = 2048
    a = torch.randn(rows, Kd, device="cuda").to(torch.bfloat16)
    w = torch.randn(G * N, Kd, device="cuda").mul_(Kd ** -0.5)
    b = torch.randn(G, N, device="cuda")
    out = torch.empty(rows, N, device="cuda", dtype=torch.bfloat16)
    if "fp8" in which:
        aq, wq = fp8.quantize(a), fp8.quantize(w, tile_rows=fp8.WEIGHT_TILE, groups=G)
        for _ in range(2):
            fp8.grouped_linear_fp8(aq, wq, tile_group=tg, bias=b, out=out)
    if "bf16" in which:
        wb = w.view(G, N, Kd).to(torch.bfloat16)
        for _ in range(2):
            gemm.grouped_linear(a, wb, tile_group=tg, bias=b, out=out)
if "attn" in which:
    qkv = torch.randn(32 * 512, 3 * 1024, device="cuda").to(torch.bfloat16)
    o = torch.empty(32 * 512, 1024, device="cuda", dtype=torch.bfloat16)
    for _ in range(2):
        K.attention_fwd(qkv, 16, out=o)
if "ln" in which:
    h = torch.randn(rows, 2048, device="cuda").to(torch.bfloat16)
    a2 = torch.empty_like(h)
    gamma, beta = torch.rand(G, 2048, device="cuda") + 0.5, torch.randn(G, 2048, device="cuda")
    mean, rstd = torch.empty(rows, device="cuda"), torch.empty(rows, device="cuda")
    aq2 = fp8.MXFP8Tensor(rows, 1, 2048, fp8.ACT_TILE, "cuda")
    for _ in range(2):
        K.ln_relu_fwd(h, gamma, beta, tg, out=a2, mean=mean, rstd=rstd)
    K.ln_relu_fwd(h, gamma, beta, tg, out=a2, mean=mean, rstd=rstd, quant=aq2)
if "small" in which:
    # the small-M kernels at (a) the named config: 64 experts x 16 rows, (b) one rank's share at 8 GPUs with a hot expert
    H, I = 512, 2048
    for rows_list in ([16] * 64, [1500, 200, 100, 60, 40, 30, 20, 16]):
        Gs = len(rows_list)
        padded = [(r + 15) // 16 * 16 for r in rows_list]
        off = torch.tensor([sum(padded[:i]) for i in range(Gs)], dtype=torch.int32, device="cuda")
        rws = torch.tensor(rows_list, dtype=torch.int32, device="cuda")
        total = sum(padded)
        act = torch.randn(total, I, device="cuda").to(torch.bfloat16)
        w2 = torch.randn(Gs, I, I, device="cuda").to(torch.bfloat16)
        hbuf = torch.empty(total, I, device="cuda", dtype=torch.bfloat16)
        K.swapab_linear(act, w2, off, rws, out=hbuf)
        K.swapab_linear(act, w2, off, rws, out=hbuf, w_is_kn=True)
        p = torch.randn(Gs, I, I, device="cuda")
        m, v, vmax = torch.zeros_like(p), torch.zeros_like(p), torch.zeros_like(p)
        pb = torch.zeros(Gs, I, I, device="cuda", dtype=torch.bfloat16)
        step = torch.ones(Gs, dtype=torch.int32, device="cuda")
        dy = (torch.randn(total, I, device="cuda") * 0.1).to(torch.bfloat16)
        K.wgrad_adam(dy, act, off, rws, p=p, m=m, v=v, vmax=vmax, p_bf16=pb, step=step)
        del p, m, v, vmax, pb, w2
torch.cuda.synchronize()
print("prof_driver done")
