"""
Precision of the LayerNorm forward's saved rstd against a common row offset (writes check_out/ln_offset_precision.json).

ln_relu_fwd_kernel computes the variance in one fp32 pass, E[x^2] - mean^2, so its relative error grows with the square of
|mean| / std.  For every C and ratio, 4096 bf16 rows randn + ratio * (+-1) go through the kernel, and the saved rstd is
compared with the float64 1 / sqrt(var + 1e-5) of the same bf16 rows.  Prints the worst and the median relative error.
"""
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

import lah_b200  # noqa
from tools import output_path
from lah_b200.ops import kernels as K


def main():
    assert torch.cuda.is_available(), "needs a GPU"
    print("device:", torch.cuda.get_device_name(0), flush=True)
    gen = torch.Generator().manual_seed(0)
    rows, results = 4096, []
    for C in (512, 1024, 4096):
        for ratio in (0, 16, 32, 64, 128, 256):
            sign = torch.where(torch.rand(rows, 1, generator=gen) < 0.5, -1.0, 1.0)
            h = (torch.randn(rows, C, generator=gen) + ratio * sign).to(torch.bfloat16).cuda()
            gamma, beta = torch.ones(1, C, device="cuda"), torch.zeros(1, C, device="cuda")
            out = torch.empty_like(h)
            mean, rstd = torch.empty(rows, device="cuda"), torch.empty(rows, device="cuda")
            K.ln_relu_fwd(h, gamma, beta, None, out=out, mean=mean, rstd=rstd, relu=False, tile_rows=128)
            ref = 1 / (h.double().var(1, unbiased=False) + 1e-5).sqrt()
            rel = (rstd.double() - ref).abs() / ref
            r = dict(C=C, mean_over_std=ratio, rstd_rel_err_max=rel.max().item(), rstd_rel_err_median=rel.median().item())
            results.append(r)
            print(r, flush=True)
    with open(output_path("ln_offset_precision.json"), "w") as f:
        json.dump(dict(device=torch.cuda.get_device_name(0), rows=rows, results=results), f, indent=1)


if __name__ == "__main__":
    main()
