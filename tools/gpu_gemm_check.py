"""GPU sanity + perf check for the wgmma grouped GEMM (writes check_out/gemm_check.json). Prints one line per case."""
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

import lah_b200  # noqa
from tools import output_path
from lah_b200.ops import gemm


def rel_err(got, ref):
    return ((got.float() - ref.float()).norm() / (ref.float().norm() + 1e-12)).item()


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


def case_mgroup(rows_per_group, N, K, w_is_kn, block_n, bias=True, residual=False, out_f32=False, seed=0, align=128):
    """expert groups padded to `align` rows (128, or 256 as on the big expert path)"""
    torch.manual_seed(seed)
    G = len(rows_per_group)
    tiles = []
    for g, r in enumerate(rows_per_group):
        tiles += [g] * (((r + align - 1) // align) * (align // 128))
    tiles += [-1] * (align // 128)  # unused tile(s) at the end
    rows = len(tiles) * 128
    a = torch.zeros(rows, K, device="cuda", dtype=torch.bfloat16)
    t = 0
    for g, r in enumerate(rows_per_group):
        a[t * 128: t * 128 + r] = torch.randn(r, K, device="cuda").to(torch.bfloat16)
        t += ((r + align - 1) // align) * (align // 128)
    w = (torch.randn(G, K, N, device="cuda") if w_is_kn else torch.randn(G, N, K, device="cuda")).mul_(K ** -0.5).to(torch.bfloat16)
    b = torch.randn(G, N, device="cuda") if bias else None
    res = torch.randn(rows, N, device="cuda").to(torch.bfloat16) if residual else None
    tg = torch.tensor(tiles, device="cuda", dtype=torch.int32)
    out = torch.full((rows, N), 7.0, device="cuda", dtype=torch.float32 if out_f32 else torch.bfloat16)
    gemm.grouped_linear(a, w, tile_group=tg, bias=b, residual=res, w_is_kn=w_is_kn, out=out, block_n=block_n)
    torch.cuda.synchronize()
    ref = gemm.grouped_linear_ref(a, w, tile_group=tg, bias=b, residual=res, w_is_kn=w_is_kn)
    valid = (tg >= 0).repeat_interleave(128)
    err = rel_err(out[valid], ref[valid])
    untouched = bool((out[~valid].float() == 7.0).all())
    return err, untouched


def case_kgroup(rows_per_group, M, N, block_n, seed=0, align=128):
    """expert groups padded to `align` rows (128, or 256 as on the big expert path)"""
    torch.manual_seed(seed)
    G = len(rows_per_group)
    off = [0]
    for r in rows_per_group:
        off.append(off[-1] + ((r + align - 1) // align) * align)
    rows = off[-1] + 128
    dy = torch.zeros(rows, M, device="cuda", dtype=torch.bfloat16)
    x = torch.zeros(rows, N, device="cuda", dtype=torch.bfloat16)
    for g, r in enumerate(rows_per_group):
        dy[off[g]: off[g] + r] = torch.randn(r, M, device="cuda").to(torch.bfloat16)
        x[off[g]: off[g] + r] = torch.randn(r, N, device="cuda").to(torch.bfloat16)
    go = torch.tensor(off, device="cuda", dtype=torch.int32)
    out = gemm.grouped_wgrad(dy, x, go, G, block_n=block_n)
    torch.cuda.synchronize()
    ref = gemm.grouped_wgrad_ref(dy, x, go, G)
    return rel_err(out, ref)


def main():
    results = {}
    print("device:", torch.cuda.get_device_name(0), flush=True)
    # ---------------- correctness
    for (name, args) in [
        ("mg_kmajor_bn256", dict(rows_per_group=[128, 300, 0, 77], N=512, K=512, w_is_kn=False, block_n=256)),
        ("mg_kmajor_bn128", dict(rows_per_group=[128, 300, 0, 77], N=384, K=192, w_is_kn=False, block_n=128)),
        ("mg_kmajor_bn64", dict(rows_per_group=[256, 1], N=64, K=64, w_is_kn=False, block_n=64)),
        ("mg_kmajor_res_f32", dict(rows_per_group=[200, 130], N=512, K=2048, w_is_kn=False, block_n=256, residual=True, out_f32=True)),
        ("mg_kn_bn256", dict(rows_per_group=[128, 300, 0, 77], N=512, K=2048, w_is_kn=True, block_n=256, bias=False)),
        ("mg_kn_bn128", dict(rows_per_group=[130, 5], N=256, K=512, w_is_kn=True, block_n=128, bias=False, residual=True)),
        ("mg_kn_bn64", dict(rows_per_group=[512], N=64, K=512, w_is_kn=True, block_n=64, bias=False)),
    ]:
        try:
            err, untouched = case_mgroup(**args)
            results[name] = dict(rel_err=err, untouched=untouched, ok=bool(err < 2e-2 and untouched))
        except Exception as e:  # noqa
            results[name] = dict(error=repr(e), ok=False)
        print(name, results[name], flush=True)
    for (name, args) in [
        ("mg_align256_kmajor", dict(rows_per_group=[128, 300, 0, 77, 1000], N=512, K=512, w_is_kn=False, block_n=256, align=256)),
        ("mg_align256_kmajor_res_f32", dict(rows_per_group=[200, 530], N=512, K=2048, w_is_kn=False, block_n=256, residual=True, out_f32=True, align=256)),
        ("mg_align256_kn", dict(rows_per_group=[128, 300, 0, 77], N=2048, K=512, w_is_kn=True, block_n=256, bias=False, align=256)),
        ("mg_align256_kn_res", dict(rows_per_group=[640, 5], N=512, K=2048, w_is_kn=True, block_n=256, bias=False, residual=True, align=256)),
    ]:
        try:
            err, untouched = case_mgroup(**args)
            results[name] = dict(rel_err=err, untouched=untouched, ok=bool(err < 2e-2 and untouched))
        except Exception as e:  # noqa
            results[name] = dict(error=repr(e), ok=False)
        print(name, results[name], flush=True)
    for (name, args) in [
        ("kg_align256_a", dict(rows_per_group=[128, 300, 0, 77], M=256, N=512, block_n=256, align=256)),
        ("kg_align256_b", dict(rows_per_group=[2048, 640], M=2048, N=2048, block_n=256, align=256)),
        ("kg_bn256", dict(rows_per_group=[128, 300, 0, 77], M=256, N=512, block_n=256)),
        ("kg_bn128", dict(rows_per_group=[1000, 64], M=128, N=384, block_n=128)),
        ("kg_bn64", dict(rows_per_group=[512, 512], M=512, N=64, block_n=64)),
    ]:
        try:
            err = case_kgroup(**args)
            results[name] = dict(rel_err=err, ok=bool(err < 2e-2))
        except Exception as e:  # noqa
            results[name] = dict(error=repr(e), ok=False)
        print(name, results[name], flush=True)

    # ---------------- perf (expert-FFN shapes, hid 512, 64 experts x 2048 rows)
    try:
        G, R = 64, 2048
        rows = G * R
        tg = torch.arange(G, device="cuda", dtype=torch.int32).repeat_interleave(R // 128)
        go = (torch.arange(G + 1, device="cuda", dtype=torch.int32) * R).contiguous()
        for (nm, K, N) in [("fwd1_512x2048", 512, 2048), ("fwd2_2048x2048", 2048, 2048), ("fwd3_2048x512", 2048, 512)]:
            a = torch.randn(rows, K, device="cuda").to(torch.bfloat16)
            w = torch.randn(G, N, K, device="cuda").to(torch.bfloat16)
            wkn = torch.randn(G, K, N, device="cuda").to(torch.bfloat16)
            out = torch.empty(rows, N, device="cuda", dtype=torch.bfloat16)
            fl = 2.0 * rows * K * N
            for bn in (256, 128):
                ms = timeit(lambda: gemm.grouped_linear(a, w, tile_group=tg, out=out, block_n=bn))
                results[f"perf_{nm}_kmajor_bn{bn}"] = dict(ms=ms, tflops=fl / ms / 1e9)
                print(f"perf_{nm}_kmajor_bn{bn}", results[f"perf_{nm}_kmajor_bn{bn}"], flush=True)
            ms = timeit(lambda: gemm.grouped_linear(a, wkn, tile_group=tg, out=out, w_is_kn=True, block_n=256))
            results[f"perf_{nm}_kn_bn256"] = dict(ms=ms, tflops=fl / ms / 1e9)
            print(f"perf_{nm}_kn_bn256", results[f"perf_{nm}_kn_bn256"], flush=True)
            # cuBLAS reference: bmm over groups
            a3 = a.view(G, R, K)
            ms = timeit(lambda: torch.bmm(a3, w.transpose(1, 2)))
            results[f"perf_{nm}_cublas_bmm"] = dict(ms=ms, tflops=fl / ms / 1e9)
            print(f"perf_{nm}_cublas_bmm", results[f"perf_{nm}_cublas_bmm"], flush=True)
        for (nm, M, N) in [("wg1_2048x512", 2048, 512), ("wg2_2048x2048", 2048, 2048), ("wg3_512x2048", 512, 2048)]:
            dy = torch.randn(rows, M, device="cuda").to(torch.bfloat16)
            x = torch.randn(rows, N, device="cuda").to(torch.bfloat16)
            out = torch.empty(G, M, N, device="cuda", dtype=torch.float32)
            fl = 2.0 * rows * M * N
            ms = timeit(lambda: gemm.grouped_wgrad(dy, x, go, G, out=out, block_n=256))
            results[f"perf_{nm}"] = dict(ms=ms, tflops=fl / ms / 1e9)
            print(f"perf_{nm}", results[f"perf_{nm}"], flush=True)
            ms = timeit(lambda: torch.bmm(dy.view(G, R, M).transpose(1, 2), x.view(G, R, N)))
            results[f"perf_{nm}_cublas_bmm"] = dict(ms=ms, tflops=fl / ms / 1e9)
            print(f"perf_{nm}_cublas_bmm", results[f"perf_{nm}_cublas_bmm"], flush=True)
    except Exception as e:  # noqa
        results["perf_error"] = repr(e)
        print("perf_error", repr(e), flush=True)

    with open(output_path("gemm_check.json"), "w") as f:
        json.dump(results, f, indent=1)
    print("ALL_OK" if all(v.get("ok", True) for v in results.values() if isinstance(v, dict)) else "SOME_FAILED")


if __name__ == "__main__":
    main()
