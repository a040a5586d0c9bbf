"""
Accumulation precision of Hopper's e4m3 wgmma inside one 32-element K block (writes check_out/fp8_mma_precision.json).

The MXFP8 GEMM (csrc/grouped_gemm_fp8.cu) issues one wgmma.m64n128k32.e4m3 per 32-element K block into a zeroed scratch
accumulator.  The 32 products of e4m3 values are exact, but the tensor core does not add them in fp32: it keeps a limited
number of bits below the largest product.  This probe measures how many.

One launch of the GEMM per pattern, K = 128 with only the first 32-element block non-zero, every scale byte 127 (2^0) and
fp32 output: the output element IS the tensor core's sum of one block.  Row r of A and row n of W hold

    big    one product  2^8 * 2^8 = 2^16
    small  31 products  (c 2^(8 - ka)) * (2^(8 - kb)) = c 2^(16 - k),  k = ka + kb,  ka = r % 18, kb = n % 18

with c = 1, 1.5 or 1.875 (rows whose c 2^(8 - ka) is not an e4m3 value are left out), so k runs from 0 to 34 (e4m3
reaches down to 2^-9).  c = 1 puts a small product on a power of two; c = 1.875 puts it just below the next one (7.5 below a
unit of 8), the worst case for a sum that drops the bits below its last retained unit; c = 1.5 puts it halfway between two
units (12 on a grid of 8), which tells truncation (8) from round-to-nearest (16).  Every exact sum has at most 24
significant bits for k <= 19, so an fp32 accumulation would return it exactly.  Patterns: the small products positive,
negative, alternating in sign, the big one first or last, a negative big one, a single small product.  For every pattern
and k the probe prints the kernel's sum, the exact one, and the error relative to sum |a_i b_i|;
F = floor(-log2(worst relative error)) is the number of bits the element-wise bound 2^-F * sum |a_i b_i| in
tests/test_fused_adam_fp8_kernels.py needs.
"""
import json
import math
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

import lah_b200  # noqa
from tools import output_path
from lah_b200.ops import fp8

KMAX = 18                  # exponents 8 .. -9 of e4m3
PATTERNS = {   # name -> (index of the big product, sign of the big product, signs of the 31 small ones, c)
    "big_first_small_pos": (0, 1.0, [1.0] * 31, 1.0),
    "big_first_small_neg": (0, 1.0, [-1.0] * 31, 1.0),
    "big_last_small_pos": (31, 1.0, [1.0] * 31, 1.0),
    "big_neg_small_pos": (0, -1.0, [1.0] * 31, 1.0),
    "big_first_small_alternating": (0, 1.0, [(-1.0) ** i for i in range(31)], 1.0),
    "big_first_one_small": (0, 1.0, [1.0] + [0.0] * 30, 1.0),
    "big_first_small_pos_x1.875": (0, 1.0, [1.0] * 31, 1.875),
    "big_first_small_neg_x1.875": (0, 1.0, [-1.0] * 31, 1.875),
    "big_last_small_pos_x1.875": (31, 1.0, [1.0] * 31, 1.875),
    "big_neg_small_pos_x1.875": (0, -1.0, [1.0] * 31, 1.875),
    "big_first_one_small_x1.875": (0, 1.0, [1.0] + [0.0] * 30, 1.875),
    "big_first_small_pos_x1.5": (0, 1.0, [1.0] * 31, 1.5),
    "big_first_one_small_x1.5": (0, 1.0, [1.0] + [0.0] * 30, 1.5),
}


def is_e4m3(x):
    return abs(x) <= 448.0 and float(torch.tensor(x).float().to(torch.float8_e4m3fn).double()) == x


def run_pattern(big_at, big_sign, signs, c):
    """(A [18, 32] float64, W [18, 32] float64, kernel output [18, 18] float64, usable values of ka) for one pattern"""
    small_pos = [i for i in range(32) if i != big_at]
    a = torch.zeros(KMAX, 32, dtype=torch.float64)
    w = torch.zeros(KMAX, 32, dtype=torch.float64)
    kas = [k for k in range(KMAX) if is_e4m3(c * 2.0 ** (8 - k))]
    for k in range(KMAX):
        w[k, big_at] = 256.0
        for i in small_pos:
            w[k, i] = 2.0 ** (8 - k)
    for k in kas:
        a[k, big_at] = big_sign * 256.0
        for s, i in zip(signs, small_pos):
            a[k, i] = s * c * 2.0 ** (8 - k)
    aq = fp8.MXFP8Tensor(128, 1, 128, fp8.ACT_TILE, "cuda")
    wq = fp8.MXFP8Tensor(64, 1, 128, fp8.WEIGHT_TILE, "cuda")
    for t, src in ((aq, a), (wq, w)):
        full = torch.zeros(t.q.shape, dtype=torch.float64)
        full[:KMAX, :32] = src
        e4m3 = full.float().to(torch.float8_e4m3fn)
        assert torch.equal(e4m3.double(), full), "a probe value is not exact in e4m3"
        t.q.copy_(e4m3.view(torch.uint8).cuda())
        t.sf.fill_(127)    # 2^0
    out = torch.zeros(128, 64, dtype=torch.float32, device="cuda")
    fp8.grouped_linear_fp8(aq, wq, out=out, out_dtype=torch.float32)
    torch.cuda.synchronize()
    return a, w, out[:KMAX, :KMAX].double().cpu(), kas


def main():
    assert torch.cuda.is_available(), "needs a GPU"
    dev = torch.cuda.get_device_name(0)
    print("device:", dev, flush=True)
    results, worst = {}, 0.0
    for name, (big_at, big_sign, signs, c) in PATTERNS.items():
        a, w, got, kas = run_pattern(big_at, big_sign, signs, c)
        exact = a @ w.t()
        mag = a.abs() @ w.abs().t()
        rows = []
        for k in range(2 * KMAX - 1):
            pairs = [(ka, k - ka) for ka in kas if 0 <= k - ka < KMAX]
            if not pairs:
                continue
            err = max(abs(got[i, j].item() - exact[i, j].item()) for i, j in pairs)
            rel = max(abs(got[i, j].item() - exact[i, j].item()) / mag[i, j].item() for i, j in pairs)
            worst = max(worst, rel)
            ka, kb = pairs[0]
            rows.append(dict(k=k, got=got[ka, kb].item(), exact=exact[ka, kb].item(), max_abs_err=err, max_rel_err=rel))
        exact_upto = max([r["k"] for r in rows if r["max_abs_err"] == 0] + [-1])
        first_wrong = min([r["k"] for r in rows if r["max_abs_err"] > 0] + [99])
        results[name] = dict(exact_for_all_k_below=first_wrong, largest_exact_k=exact_upto, by_k=rows)
        print(f"{name}: sums exact for k < {first_wrong}", flush=True)
        for r in rows:
            print(f"  k={r['k']:2d}  got {r['got']!r:>24}  exact {r['exact']!r:>24}  "
                  f"rel err {r['max_rel_err']:.3g}", flush=True)
    F = math.floor(-math.log2(worst)) if worst > 0 else 24
    print(f"worst |error| / sum|a b| = {worst:.4g} (2^{math.log2(worst) if worst > 0 else float('-inf'):.2f}) -> F = {F}")
    with open(output_path("fp8_mma_precision.json"), "w") as f:
        json.dump(dict(device=dev, worst_rel_err=worst, F=F, patterns=results), f, indent=1)


if __name__ == "__main__":
    main()
