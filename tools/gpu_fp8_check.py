"""GPU check: MXFP8 quantisation kernel + block-scaled wgmma grouped GEMM vs PyTorch oracles (writes check_out/fp8_check.json)."""
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

import lah_b200  # noqa
from tools import output_path
from lah_b200.ops import fp8, gemm

results = {}


def rel(a, b):
    return ((a.float() - b.float()).norm() / (b.float().norm() + 1e-12)).item()


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


def check_quant():
    torch.manual_seed(0)
    for name, rows, groups, K, tile, dtype in [("act", 384, 1, 512, fp8.ACT_TILE, torch.bfloat16),
                                                ("weight", 2048, 3, 512, fp8.WEIGHT_TILE, torch.float32),
                                                ("weight_small", 512, 2, 2048, fp8.WEIGHT_TILE, torch.bfloat16)]:
        x = (torch.randn(rows * groups, K, device="cuda") * torch.rand(rows * groups, 1, device="cuda") * 3).to(dtype)
        x[5] = 0
        t = fp8.quantize(x, tile_rows=tile, groups=groups)
        torch.cuda.synchronize()
        q_ref, e_ref = fp8.quantize_ref(x)
        e_got = fp8.unpack_sf(t)
        q_got = t.q.view(torch.float8_e4m3fn)
        ok_e = bool((e_got == e_ref).all())
        ok_q = bool((q_got.float() == q_ref.float()).all())
        deq = rel(fp8.dequantize_ref(q_got, e_got), x)
        results[f"quant_{name}"] = dict(ok=ok_e and ok_q and deq < 0.05, scales_equal=ok_e, payload_equal=ok_q, dequant_err=deq)
        print(f"quant_{name}", results[f"quant_{name}"], flush=True)


def case_gemm(rows_per_group, N, K, bias=True, residual=False, out_f32=False, act=0, seed=0):
    torch.manual_seed(seed)
    G = len(rows_per_group)
    tiles = []
    for g, r in enumerate(rows_per_group):
        tiles += [g] * (((r + 255) // 256) * 2)
    tiles += [-1, -1]
    rows = len(tiles) * 128
    a = torch.zeros(rows, K, device="cuda", dtype=torch.bfloat16)
    t = 0
    for g, r in enumerate(rows_per_group):
        a[t * 128: t * 128 + r] = torch.randn(r, K, device="cuda").to(torch.bfloat16)
        t += ((r + 255) // 256) * 2
    w = torch.randn(G * N, K, device="cuda").mul_(K ** -0.5)
    b = torch.randn(G, N, device="cuda") if bias else None
    res = torch.randn(rows, N, device="cuda").to(torch.bfloat16) if residual else None
    tg = torch.tensor(tiles, device="cuda", dtype=torch.int32)
    aq = fp8.quantize(a, tile_group=tg)
    wq = fp8.quantize(w, tile_rows=fp8.WEIGHT_TILE, groups=G)
    out = torch.full((rows, N), 7.0, device="cuda", dtype=torch.float32 if out_f32 else torch.bfloat16)
    fp8.grouped_linear_fp8(aq, wq, tile_group=tg, bias=b, residual=res, out=out, act=act)
    torch.cuda.synchronize()
    valid = (tg >= 0).repeat_interleave(128)
    # exact oracle: dequantised operands, fp32 matmul
    a_dq = torch.zeros(rows, K, device="cuda")
    a_dq[valid] = fp8.dequantize_ref(aq.q.view(torch.float8_e4m3fn)[valid], fp8.unpack_sf(aq)[valid])
    w_dq = fp8.dequantize_ref(wq.q.view(torch.float8_e4m3fn), fp8.unpack_sf(wq)).view(G, N, K)
    ref = gemm.grouped_linear_ref(a_dq, w_dq, tile_group=tg, bias=b)
    if act == 1:
        ref = torch.relu(ref)
    if res is not None:
        ref = ref + res.float()
    ref_bf16 = gemm.grouped_linear_ref(a, w.view(G, N, K), tile_group=tg, bias=b)
    if act == 1:
        ref_bf16 = torch.relu(ref_bf16)
    if res is not None:
        ref_bf16 = ref_bf16 + res.float()
    err = rel(out[valid], ref[valid])
    err_unq = rel(out[valid], ref_bf16[valid])
    untouched = bool((out[~valid].float() == 7.0).all())
    return err, err_unq, untouched


def check_gemm():
    cases = {
        "one_tile_k128": dict(rows_per_group=[256], N=192, K=128, bias=False),
        "one_tile_k512": dict(rows_per_group=[256], N=192, K=512),
        "n2048_k512": dict(rows_per_group=[300, 0, 77, 512], N=2048, K=512),
        "n512_k2048_res": dict(rows_per_group=[200, 130], N=512, K=2048, residual=True),
        "n2048_k2048_relu_f32": dict(rows_per_group=[1000, 24], N=2048, K=2048, act=1, out_f32=True),
        "n64_k128": dict(rows_per_group=[100], N=64, K=128),
    }
    for name, kw in cases.items():
        err, err_unq, untouched = case_gemm(**kw)
        results[f"gemm_{name}"] = dict(ok=err < 1e-2 and untouched, err_vs_dequant=err, err_vs_unquantized=err_unq,
                                       untouched=untouched)
        print(f"gemm_{name}", results[f"gemm_{name}"], flush=True)


def check_perf():
    """expert-FFN shapes at a bench-like load: 64 experts x 4096 rows"""
    torch.manual_seed(0)
    G, R = 64, 4096
    rows = G * R
    tg = torch.arange(G, device="cuda", dtype=torch.int32).repeat_interleave(R // 128)
    for name, N, K in [("fwd1", 2048, 512), ("fwd2", 2048, 2048), ("fwd3", 512, 2048)]:
        a = torch.randn(rows, K, device="cuda").to(torch.bfloat16)
        w = torch.randn(G * N, K, device="cuda").mul_(K ** -0.5)
        wb = w.view(G, N, K).to(torch.bfloat16)
        b = torch.randn(G, N, device="cuda")
        aq = fp8.quantize(a)
        wq = fp8.quantize(w, tile_rows=fp8.WEIGHT_TILE, groups=G)
        out = torch.empty(rows, N, device="cuda", dtype=torch.bfloat16)
        ms8 = timeit(lambda: fp8.grouped_linear_fp8(aq, wq, tile_group=tg, bias=b, out=out))
        ms16 = timeit(lambda: gemm.grouped_linear(a, wb, tile_group=tg, bias=b, out=out))
        msq = timeit(lambda: fp8.quantize(a, out=aq))
        flops = 2.0 * rows * N * K
        results[f"perf_{name}"] = dict(ok=True, fp8_ms=ms8, fp8_tflops=flops / ms8 / 1e9, bf16_ms=ms16,
                                       bf16_tflops=flops / ms16 / 1e9, quant_act_ms=msq,
                                       quant_gbs=(rows * K * 3 / msq / 1e6))
        print(f"perf_{name}", results[f"perf_{name}"], flush=True)


if __name__ == "__main__":
    for fn in (check_quant, check_gemm, check_perf):
        try:
            fn()
        except Exception as e:  # noqa
            import traceback
            traceback.print_exc()
            results[fn.__name__] = dict(ok=False, error=repr(e))
    json.dump(results, open(output_path("fp8_check.json"), "w"), indent=1)
    print("ALL_OK" if all(v.get("ok") for v in results.values()) else "SOME_FAILED")
