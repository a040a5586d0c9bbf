"""GPU check + timing of the small-M (weight-streaming) kernels of csrc/small_m.cu against fp32 PyTorch oracles.

  swapab_linear   forward (K-major weights) and dgrad (MN-major weights) over ragged groups of 0..300 rows
  wgrad_adam      fused weight gradient + AMSGrad vs (dy^T x in fp32) + torch.optim.Adam(amsgrad=True) semantics

Run on the GPU: python tools/gpu_small_check.py [--perf]; writes check_out/small_check.json"""
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

import lah_b200  # noqa
from tools import output_path
from lah_b200.ops import kernels as K

results = {}
PEAKS = {}
try:
    PEAKS = json.load(open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "MEASURED_PEAKS.json")))
except Exception:
    pass
HBM = float(PEAKS.get("hbm_gbs", 3350.0))   # H100 SXM data sheet (HBM3)


def rel(got, ref):
    return ((got.float() - ref.float()).norm() / (ref.float().norm() + 1e-12)).item()


def record(name, **kw):
    results[name] = kw
    print(name, kw, flush=True)


def make_groups(rows_list, align=16):
    off, cur = [], 0
    for r in rows_list:
        off.append(cur)
        cur += (r + align - 1) // align * align
    return (torch.tensor(off, dtype=torch.int32, device="cuda"), torch.tensor(rows_list, dtype=torch.int32, device="cuda"),
            max(cur, align))


def timeit(fn, iters=20, flush=None):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(iters):
        if flush is not None:
            flush.zero_()   # > L2: the next call streams from HBM
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    ts.sort()
    return ts[len(ts) // 2]


def check_swapab():
    torch.manual_seed(0)
    rows_list = [0, 1, 16, 17, 63, 128, 130, 300, 5, 0, 64, 33, 1100, 257]
    G = len(rows_list)
    off, rows, total = make_groups(rows_list)
    for (K_in, M_out) in [(512, 2048), (2048, 2048), (2048, 512)]:
        for kn in (False, True):
            x = torch.zeros(total, K_in, device="cuda", dtype=torch.bfloat16)
            for o, r in zip(off.tolist(), rows_list):
                x[o:o + r] = (torch.randn(r, K_in, device="cuda") * 0.5).to(torch.bfloat16)
            w = (torch.randn(G, M_out, K_in, device="cuda") * K_in ** -0.5).to(torch.bfloat16)
            if kn:
                w = w.transpose(1, 2).contiguous()   # [G, K_in, M_out]
            bias = torch.randn(G, M_out, device="cuda") if not kn else None
            res = torch.randn(total, M_out, device="cuda").to(torch.bfloat16)
            out = torch.full((total, M_out), 7.0, device="cuda", dtype=torch.bfloat16)
            K.swapab_linear(x, w, off, rows, out=out, bias=bias, residual=res, w_is_kn=kn)
            torch.cuda.synchronize()
            ref = K.swapab_linear_ref(x, w, off, rows, bias=bias, residual=res, w_is_kn=kn)
            mask = torch.zeros(total, dtype=torch.bool, device="cuda")
            padded = torch.zeros(total, dtype=torch.bool, device="cuda")
            for o, r in zip(off.tolist(), rows_list):
                mask[o:o + r] = True
                padded[o:o + (r + 15) // 16 * 16] = True   # the kernel also writes the group's padding rows (bias / zeros)
            err = rel(out[mask], ref[mask])
            untouched = bool((out[~padded] == 7.0).all()) and bool(torch.isfinite(out.float()).all())
            record(f"swapab_K{K_in}_M{M_out}_{'dgrad' if kn else 'fwd'}", ok=err < 5e-3 and untouched, rel_err=err,
                   padding_untouched=untouched)


def check_wgrad_adam():
    torch.manual_seed(1)
    rows_list = [0, 1, 16, 17, 70, 200, 5, 33, 600]
    G = len(rows_list)
    off, rows, total = make_groups(rows_list)
    for (N, Kd) in [(256, 128), (2048, 512), (512, 2048)]:
        dy = torch.zeros(total, N, device="cuda", dtype=torch.bfloat16)
        x = torch.zeros(total, Kd, device="cuda", dtype=torch.bfloat16)
        for o, r in zip(off.tolist(), rows_list):
            dy[o:o + r] = (torch.randn(r, N, device="cuda") * 0.3).to(torch.bfloat16)
            x[o:o + r] = torch.randn(r, Kd, device="cuda").to(torch.bfloat16)
        # rows of the NEXT group follow the padded rows: the kernel must not reduce over them (k-step masking)
        p = torch.randn(G, N, Kd, device="cuda")
        p0 = p.clone()
        m, v, vmax = torch.zeros_like(p), torch.zeros_like(p), torch.zeros_like(p)
        pb = torch.zeros(G, N, Kd, device="cuda", dtype=torch.bfloat16)
        step = torch.zeros(G, dtype=torch.int32, device="cuda")
        params = [p0[g].clone().requires_grad_(True) for g in range(G)]
        opts = [torch.optim.Adam([q], lr=1e-2, amsgrad=True) for q in params]
        gerr = 0.0
        for it in range(3):
            K.bump_steps(step, rows)
            K.wgrad_adam(dy, x, off, rows, p=p, m=m, v=v, vmax=vmax, p_bf16=pb, step=step, lr=1e-2)
            torch.cuda.synchronize()
            for g, (o, r) in enumerate(zip(off.tolist(), rows_list)):
                if r > 0:
                    params[g].grad = dy[o:o + r].float().t() @ x[o:o + r].float()
                    opts[g].step()
                    if it == 0:   # first step: m = (1 - beta1) * grad  -> recover the gradient VALUE
                        gerr = max(gerr, rel(m[g] / 0.1, params[g].grad))
        # AMSGrad normalises every element by its own |grad| history: an element whose gradient is ~0 (cancellation) may move
        # by up to lr in a different direction when the tensor-core accumulation order differs from torch's — compare
        # the bulk (mean, 99.99th percentile) and bound the outliers by 2 * lr * steps
        diff = torch.cat([(p[g] - params[g].detach()).abs().flatten() for g in range(G)])
        perr, pmean = diff.max().item(), diff.mean().item()
        p9999 = diff.float().kthvalue(int(diff.numel() * 0.9999)).values.item()
        untouched = bool(torch.equal(p[0], p0[0])) and int(step[0]) == 0
        record(f"wgrad_adam_N{N}_K{Kd}", ok=pmean < 2e-6 and p9999 < 5e-5 and perr < 6e-2 and gerr < 2e-3 and untouched
               and rel(pb[1:], p[1:]) < 5e-3, max_abs_param_err=perr, mean_abs_param_err=pmean, p9999_abs_param_err=p9999,
               wgrad_rel_err=gerr, inactive_untouched=untouched)


def perf():
    """the named config: 64 experts, 16 rows each, hid 512 — weight / state streaming rooflines"""
    torch.manual_seed(2)
    G, H, I = 64, 512, 2048
    rows_list = [16] * G
    off, rows, total = make_groups(rows_list)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    x = torch.randn(total, H, device="cuda").to(torch.bfloat16)
    a = torch.randn(total, I, device="cuda").to(torch.bfloat16)
    w1 = torch.randn(G, I, H, device="cuda").to(torch.bfloat16)
    w2 = torch.randn(G, I, I, device="cuda").to(torch.bfloat16)
    w3 = torch.randn(G, H, I, device="cuda").to(torch.bfloat16)
    h = torch.empty(total, I, device="cuda", dtype=torch.bfloat16)
    y = torch.empty(total, H, device="cuda", dtype=torch.bfloat16)
    for name, fn, nbytes in [
        ("swapab_fwd1_512->2048", lambda: K.swapab_linear(x, w1, off, rows, out=h), w1.numel() * 2),
        ("swapab_fwd2_2048->2048", lambda: K.swapab_linear(a, w2, off, rows, out=h), w2.numel() * 2),
        ("swapab_fwd3_2048->512", lambda: K.swapab_linear(a, w3, off, rows, out=y), w3.numel() * 2),
        ("swapab_dgrad2_2048->2048", lambda: K.swapab_linear(a, w2, off, rows, out=h, w_is_kn=True), w2.numel() * 2),
        ("swapab_dgrad1_2048->512", lambda: K.swapab_linear(a, w1, off, rows, out=y, w_is_kn=True), w1.numel() * 2),
    ]:
        ms = timeit(fn, flush=flush)
        record("perf_" + name, ok=True, ms=ms, weight_GB=nbytes / 1e9, TBps=nbytes / ms / 1e9,
               frac_of_measured_copy=nbytes / ms / 1e6 / HBM)
    p = torch.randn(G, I, I, device="cuda")
    m, v, vmax = torch.zeros_like(p), torch.zeros_like(p), torch.zeros_like(p)
    pb = torch.zeros(G, I, I, device="cuda", dtype=torch.bfloat16)
    step = torch.ones(G, dtype=torch.int32, device="cuda")
    dy = (torch.randn(total, I, device="cuda") * 0.1).to(torch.bfloat16)
    # device-to-device copy of a buffer far larger than L2: the bandwidth this card actually reaches (read + write)
    src = torch.empty(1 << 30, dtype=torch.uint8, device="cuda")
    dst = torch.empty_like(src)
    ms_copy = timeit(lambda: dst.copy_(src))
    copy_gbs = 2 * src.numel() / ms_copy / 1e6
    del src, dst
    record("perf_copy_1GiB", ok=True, ms=ms_copy, GBps=copy_gbs, frac_of_hbm=copy_gbs / HBM)
    nbytes = p.numel() * 34
    # all SMs, and the optimizer stream's share of a 132-SM H100 in the training step (EngineContext, one GPU)
    for tag, ctas in [("", 0), ("_opt_share", 132 * 17 // 28)]:
        ms = timeit(lambda: K.wgrad_adam(dy, a, off, rows, p=p, m=m, v=v, vmax=vmax, p_bf16=pb, step=step, max_ctas=ctas),
                    flush=flush)
        record("perf_wgrad_adam_w2" + tag, ok=True, ms=ms, ctas=ctas or "all", state_GB=nbytes / 1e9,
               TBps=nbytes / ms / 1e9, frac_of_hbm=nbytes / ms / 1e6 / HBM, frac_of_copy=nbytes / ms / 1e6 / copy_gbs)
    # the same step on a split master weight (the small path's format): pb and its low half, 32 B / param
    lo = torch.empty(G, I, I, device="cuda", dtype=torch.int16)
    K.split_encode(p.view(-1), pb.view(-1), lo.view(-1), v.view(-1))
    nbytes = p.numel() * 32
    for tag, ctas in [("", 0), ("_opt_share", 132 * 17 // 28)]:
        ms = timeit(lambda: K.wgrad_adam(dy, a, off, rows, p=None, p_lo=lo, m=m, v=v, vmax=vmax, p_bf16=pb, step=step,
                                         max_ctas=ctas), flush=flush)
        record("perf_wgrad_adam_split_w2" + tag, ok=True, ms=ms, ctas=ctas or "all", state_GB=nbytes / 1e9,
               TBps=nbytes / ms / 1e9, frac_of_hbm=nbytes / ms / 1e6 / HBM, frac_of_copy=nbytes / ms / 1e6 / copy_gbs)
    v.abs_()   # the tie bits out again: p is stale from here on, the unfused pair below only needs the shapes
    # the unfused pair it replaces: fp32 gradient written by a wgrad GEMM + the stand-alone AMSGrad kernel (38 B / param)
    g = torch.randn_like(p)
    rows_all = torch.full((G,), 16, dtype=torch.int32, device="cuda")
    ms2 = timeit(lambda: K.adam_step(p.view(-1), g.view(-1), m.view(-1), v.view(-1), vmax.view(-1), pb.view(-1), [I * I], G,
                                     step=step, group_rows=rows_all), flush=flush)
    record("perf_adam_unfused_w2", ok=True, ms=ms2, TBps=p.numel() * 38 / ms2 / 1e9,
           frac_of_measured_copy=p.numel() * 38 / ms2 / 1e6 / HBM)


def perf_skew():
    """one rank of the 8-GPU named config: 8 experts, 1024 routed rows, one HOT expert (collapsed routing).  The tile of a
    hot expert must not serialise the launch: chunk-parallel swap-AB tiles, pipelined k-blocks in the fused wgrad"""
    torch.manual_seed(3)
    G, H, I = 8, 512, 2048
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    for tag, rows_list in [("uniform128", [128] * 8), ("hot1500", [1500, 200, 100, 60, 40, 30, 20, 16]),
                           ("hot2048", [2048, 0, 0, 0, 0, 0, 0, 0])]:
        off, rows, total = make_groups(rows_list)
        a = torch.randn(total, I, device="cuda").to(torch.bfloat16)
        x = torch.randn(total, H, device="cuda").to(torch.bfloat16)
        w1 = torch.randn(G, I, H, device="cuda").to(torch.bfloat16)
        w2 = torch.randn(G, I, I, device="cuda").to(torch.bfloat16)
        h = torch.empty(total, I, device="cuda", dtype=torch.bfloat16)
        y = torch.empty(total, H, device="cuda", dtype=torch.bfloat16)
        out = {}
        out["fwd1_ms"] = timeit(lambda: K.swapab_linear(x, w1, off, rows, out=h), flush=flush)
        out["fwd2_ms"] = timeit(lambda: K.swapab_linear(a, w2, off, rows, out=h), flush=flush)
        out["dgrad2_ms"] = timeit(lambda: K.swapab_linear(a, w2, off, rows, out=h, w_is_kn=True), flush=flush)
        out["dgrad1_ms"] = timeit(lambda: K.swapab_linear(a, w1, off, rows, out=y, w_is_kn=True), flush=flush)
        out["fwd2_52_ctas_ms"] =timeit(lambda: K.swapab_linear(a, w2, off, rows, out=h, max_ctas=52), flush=flush)
        p = torch.randn(G, I, I, device="cuda")
        m, v, vmax = torch.zeros_like(p), torch.zeros_like(p), torch.zeros_like(p)
        pb = torch.zeros(G, I, I, device="cuda", dtype=torch.bfloat16)
        step = torch.ones(G, dtype=torch.int32, device="cuda")
        dy = (torch.randn(total, I, device="cuda") * 0.1).to(torch.bfloat16)
        out["wgrad_adam_w2_ms"] = timeit(lambda: K.wgrad_adam(dy, a, off, rows, p=p, m=m, v=v, vmax=vmax, p_bf16=pb, step=step),
                                         flush=flush)
        active = sum(1 for r in rows_list if r > 0)
        out["wgrad_adam_TBps"] = active * I * I * 34 / out["wgrad_adam_w2_ms"] / 1e9
        record("perf_skew_" + tag, ok=True, **out)


def main():
    print("device:", torch.cuda.get_device_name(0), flush=True)
    fns = [perf, perf_skew] if "--perf-only" in sys.argv else \
        [check_swapab, check_wgrad_adam] + ([perf, perf_skew] if "--perf" in sys.argv else [])
    for fn in fns:
        try:
            fn()
        except Exception as e:  # noqa
            import traceback
            traceback.print_exc()
            record(fn.__name__ + "_exception", ok=False, error=repr(e))
    with open(output_path("small_check.json"), "w") as f:
        json.dump(results, f, indent=1, default=str)
    print("ALL_OK" if all(v.get("ok") for v in results.values()) else "SOME_FAILED")


if __name__ == "__main__":
    main()
