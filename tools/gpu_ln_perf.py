"""GPU perf probe for the LayerNorm+ReLU kernels at the bench shapes (run on the GPU; LAH_LN_ROWS=1 = one row per warp)."""
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

import lah_b200  # noqa
from lah_b200.ops import fp8, kernels as K


def timeit(fn, iters=20, warmup=3):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(iters):
        fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / iters


def main():
    G, R, C = 64, 4224, 2048
    rows = G * R
    tg = torch.arange(G, device="cuda", dtype=torch.int32).repeat_interleave(R // 128)
    h = torch.randn(rows, C, device="cuda").to(torch.bfloat16)
    a = torch.empty_like(h)
    gamma, beta = torch.rand(G, C, device="cuda") + 0.5, torch.randn(G, C, device="cuda")
    mean, rstd = torch.empty(rows, device="cuda"), torch.empty(rows, device="cuda")
    aq = fp8.MXFP8Tensor(rows, 1, C, fp8.ACT_TILE, "cuda")
    out = dict(rows_per_warp=os.environ.get("LAH_LN_ROWS", "default"))
    ms = timeit(lambda: K.ln_relu_fwd(h, gamma, beta, tg, out=a, mean=mean, rstd=rstd))
    out["fwd_ms"], out["fwd_tbs"] = ms, rows * C * 4 / ms / 1e9
    ms = timeit(lambda: K.ln_relu_fwd(h, gamma, beta, tg, out=a, mean=mean, rstd=rstd, quant=aq))
    out["fwd_q_ms"], out["fwd_q_tbs"] = ms, rows * C * 5 / ms / 1e9
    ms = timeit(lambda: K.ln_relu_fwd(h, gamma, beta, tg, out=None, mean=mean, rstd=rstd, quant=aq))
    out["fwd_q_only_ms"], out["fwd_q_only_tbs"] = ms, rows * C * 3 / ms / 1e9
    da, dh = torch.randn_like(h), torch.empty_like(h)
    dg, db, dbias = torch.zeros(G, C, device="cuda"), torch.zeros(G, C, device="cuda"), torch.zeros(G, C, device="cuda")
    ms = timeit(lambda: K.ln_relu_bwd(da, h, mean, rstd, gamma, beta, tg, dh=dh, dgamma=dg, dbeta=db, dbias=dbias))
    out["bwd_ms"], out["bwd_tbs"] = ms, rows * C * 6 / ms / 1e9
    ref = K.ln_relu_ref(h[:512], gamma[0], beta[0])
    out["fwd_err"] = ((a[:512].float() - ref).norm() / ref.norm()).item()
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
