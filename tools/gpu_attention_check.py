"""GPU check: wgmma attention kernel and the native transformer layer vs PyTorch oracles (writes check_out/native_layers_check.json)."""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

import lah_b200  # noqa
from tools import output_path
from lah_b200.models.layers import TransformerEncoderLayer
from lah_b200.models.transformer_native import NativeTransformerLayer
from lah_b200.ops import kernels as K

results = {}


def rel(a, b):
    return ((a.float() - b.float()).norm() / (b.float().norm() + 1e-12)).item()


def timeit(fn, iters=10, warmup=2):
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


def check_attention():
    torch.manual_seed(0)
    for batch, heads in [(1, 2), (3, 16)]:
        d = heads * 64
        qkv = (torch.randn(batch * 512, 3 * d, device="cuda") * 1.5).to(torch.bfloat16)
        out = K.attention_fwd(qkv, heads)
        torch.cuda.synchronize()
        ref = K.attention_ref(qkv, heads)
        err = rel(out, ref)
        results[f"attention_b{batch}_h{heads}"] = dict(ok=err < 2e-2, err=err)
        print(f"attention_b{batch}_h{heads}", results[f"attention_b{batch}_h{heads}"], flush=True)
    batch, heads, d = 32, 16, 1024
    qkv = torch.randn(batch * 512, 3 * d, device="cuda").to(torch.bfloat16)
    out = torch.empty(batch * 512, d, device="cuda", dtype=torch.bfloat16)
    ms = timeit(lambda: K.attention_fwd(qkv, heads, out=out))
    flops = 4.0 * batch * heads * 512 * 512 * 64
    q4 = qkv.view(batch, 512, 3, heads, 64)
    q, k, v = (q4[:, :, i].transpose(1, 2) for i in range(3))
    ms_sdpa = timeit(lambda: torch.nn.functional.scaled_dot_product_attention(q, k, v))
    results["attention_perf"] = dict(ok=True, ms=ms, tflops=flops / ms / 1e9, sdpa_ms=ms_sdpa, sdpa_tflops=flops / ms_sdpa / 1e9)
    print("attention_perf", results["attention_perf"], flush=True)


def check_attention_bwd():
    """wgmma attention backward (csrc/attention_bwd.cu) vs autograd through the fp32 reference attention"""
    torch.manual_seed(3)
    for batch, heads in [(1, 2), (2, 16)]:
        d = heads * 64
        qkv = (torch.randn(batch * 512, 3 * d, device="cuda") * 1.2).to(torch.bfloat16)
        dout = torch.randn(batch * 512, d, device="cuda").to(torch.bfloat16)
        lse = torch.empty(batch * 512, heads, device="cuda")
        out = K.attention_fwd(qkv, heads, lse=lse)
        dqkv = K.attention_bwd(qkv, out, dout, lse, heads)
        torch.cuda.synchronize()
        ref_in = qkv.float().requires_grad_(True)
        K.attention_ref(ref_in, heads).backward(dout.float())
        g = ref_in.grad
        errs = dict(dq=rel(dqkv[:, :d], g[:, :d]), dk=rel(dqkv[:, d:2 * d], g[:, d:2 * d]), dv=rel(dqkv[:, 2 * d:], g[:, 2 * d:]))
        # log-sum-exp emitted by the forward (base 2)
        q, k, _ = qkv.float().view(batch, 512, 3, heads, 64).unbind(2)
        s2 = torch.einsum("bqhd,bkhd->bhqk", q, k) * (0.125 * 1.4426950408889634)
        lse_ref = torch.logsumexp(s2 * 0.6931471805599453, dim=-1) / 0.6931471805599453     # log2 sum 2^s
        errs["lse"] = (lse.view(batch, 512, heads).transpose(1, 2) - lse_ref).abs().max().item()
        results[f"attention_bwd_b{batch}_h{heads}"] = dict(ok=all(v < 3e-2 for v in errs.values()), **errs)
        print(f"attention_bwd_b{batch}_h{heads}", results[f"attention_bwd_b{batch}_h{heads}"], flush=True)
    batch, heads, d = 32, 16, 1024
    qkv = torch.randn(batch * 512, 3 * d, device="cuda").to(torch.bfloat16)
    dout = torch.randn(batch * 512, d, device="cuda").to(torch.bfloat16)
    lse = torch.empty(batch * 512, heads, device="cuda")
    out = K.attention_fwd(qkv, heads, lse=lse)
    ms = timeit(lambda: K.attention_bwd(qkv, out, dout, lse, heads))
    flops = 10.0 * batch * heads * 512 * 512 * 64
    q4 = qkv.view(batch, 512, 3, heads, 64)
    q, k, v = (q4[:, :, i].transpose(1, 2).detach().requires_grad_(True) for i in range(3))
    o = torch.nn.functional.scaled_dot_product_attention(q, k, v)
    go = dout.view(batch, 512, heads, 64).transpose(1, 2)
    ms_sdpa = timeit(lambda: torch.autograd.grad(o, (q, k, v), go, retain_graph=True))
    results["attention_bwd_perf"] = dict(ok=True, ms=ms, tflops=flops / ms / 1e9, sdpa_bwd_ms=ms_sdpa)
    print("attention_bwd_perf", results["attention_bwd_perf"], flush=True)


def check_transformer_train():
    """the TRAINABLE sm_90a transformer expert (ExpertBackend + NativeTransformerExecutor): forward, input gradients and three
    AMSGrad steps against the fp32 nn.Module + torch.optim.Adam"""
    import copy
    import lah_b200 as lib
    torch.manual_seed(4)
    layer = TransformerEncoderLayer(1024, 16, dropout=0.0).cuda()
    ref = copy.deepcopy(layer)
    ref_opt = torch.optim.Adam(ref.parameters(), lr=1e-4, amsgrad=True)
    be = lib.ExpertBackend(name="t", expert=layer, opt=torch.optim.Adam(layer.parameters(), lr=1e-4, amsgrad=True),
                           args_schema=(lib.BatchTensorProto(512, 1024),), outputs_schema=lib.BatchTensorProto(512, 1024),
                           max_batch_size=8)
    x = torch.randn(2, 512, 1024, device="cuda")
    g = torch.randn(2, 512, 1024, device="cuda") * 0.1
    (y,) = be.forward(x)
    native_used = type(be._executor).__name__ == "NativeTransformerExecutor"
    errs = dict(fwd=rel(y, ref(x)))
    for it in range(3):
        (gx,) = be.backward(x, g)
        xr = x.clone().requires_grad_(True)
        ref(xr).backward(g)
        if it == 0:
            errs["dx"] = rel(gx, xr.grad)
            # VALUE of the weight gradients: first Adam step -> exp_avg = 0.1 * grad
            st = be.opt.state_dict()["state"]
            names = [n for n, _ in ref.named_parameters()]
            for i, (n, p) in enumerate(ref.named_parameters()):
                if n in ("self_attn.in_proj_weight", "linear1.weight", "linear2.weight", "self_attn.out_proj.weight",
                         "self_attn.in_proj_bias", "norm1.weight"):
                    errs["g_" + n] = rel(st[i]["exp_avg"] / 0.1, p.grad)
        ref_opt.step(), ref_opt.zero_grad()
    sd, rsd = be.state_dict(), ref.state_dict()
    errs["param_mean_abs_diff"] = max((sd["expert." + k] - v).abs().mean().item() for k, v in rsd.items())
    ok = native_used and errs["fwd"] < 3e-2 and errs["dx"] < 5e-2 and errs["param_mean_abs_diff"] < 1.5e-4 and \
        all(v < 6e-2 for k, v in errs.items() if k.startswith("g_"))
    results["transformer_train"] = dict(ok=bool(ok), native=native_used, **errs)
    print("transformer_train", results["transformer_train"], flush=True)
    xb = torch.randn(8, 512, 1024, device="cuda")
    gb = torch.randn(8, 512, 1024, device="cuda") * 0.1
    ms = timeit(lambda: be.backward(xb, gb), iters=5)
    ref_bf = copy.deepcopy(ref)

    def torch_step():
        xr = xb.clone().requires_grad_(True)
        with torch.autocast("cuda", dtype=torch.bfloat16):
            out = ref_bf(xr)
        out.backward(gb)
        ref_opt_bf.step(), ref_opt_bf.zero_grad()

    ref_opt_bf = torch.optim.Adam(ref_bf.parameters(), lr=1e-4, amsgrad=True, fused=True)
    ms_t = timeit(torch_step, iters=5)
    results["transformer_train_perf"] = dict(ok=True, ms_fwd_bwd_adam_8seq=ms, torch_bf16_autocast_ms=ms_t, seqs_per_s=8 / ms * 1e3)
    print("transformer_train_perf", results["transformer_train_perf"], flush=True)


def check_layer():
    torch.manual_seed(1)
    layer = TransformerEncoderLayer(1024, 16).cuda().eval()
    native = NativeTransformerLayer(layer)
    x = torch.randn(4, 512, 1024, device="cuda")
    with torch.no_grad():
        ref = layer(x)
    out = native(x)
    torch.cuda.synchronize()
    err = rel(out, ref)
    results["transformer_layer"] = dict(ok=err < 3e-2, err=err)
    print("transformer_layer", results["transformer_layer"], flush=True)
    xb = torch.randn(32, 512, 1024, device="cuda").to(torch.bfloat16)
    ms = timeit(lambda: native(xb))
    layer_bf16 = layer.to(torch.bfloat16)
    with torch.no_grad():
        ms_torch = timeit(lambda: layer_bf16(xb))
    tokens = 32 * 512
    flops = tokens * (2.0 * 8_399_872 - 2 * 4 * 1024) + 4.0 * 32 * 16 * 512 * 512 * 64
    results["transformer_perf"] = dict(ok=True, ms=ms, tflops=flops / ms / 1e9, torch_bf16_ms=ms_torch,
                                       seqs_per_s=32 / ms * 1e3, torch_seqs_per_s=32 / ms_torch * 1e3)
    print("transformer_perf", results["transformer_perf"], flush=True)


def check_ffn_native():
    """sm_90a forward of the FFN expert (bf16 and MXFP8) vs the fp32 nn.Module; throughput of the fwd-only chain layer"""
    from lah_b200.models.layers import FeedforwardBlock
    from lah_b200.models.ffn_native import NativeFFNLayer
    torch.manual_seed(2)
    block = FeedforwardBlock(1024).cuda().eval()
    x = torch.randn(2048, 1024, device="cuda")
    with torch.no_grad():
        ref = block(x)
    xb = x.to(torch.bfloat16)
    for dtype, tol in (("bf16", 2e-2), ("fp8", 6e-2)):
        layer = NativeFFNLayer(block, dtype=dtype)
        out = layer(xb)
        torch.cuda.synchronize()
        err = rel(out, ref)
        big = torch.randn(32768, 1024, device="cuda").to(torch.bfloat16)
        o2 = torch.empty_like(big)
        ms = timeit(lambda: layer(big, out=o2))
        flops = 2.0 * 32768 * 25_165_824
        results[f"ffn_native_{dtype}"] = dict(ok=err < tol, err=err, ms_32768rows=ms, tflops=flops / ms / 1e9,
                                              rows_per_s=32768 / ms * 1e3)
        print(f"ffn_native_{dtype}", results[f"ffn_native_{dtype}"], flush=True)
    block_bf16 = block.to(torch.bfloat16)
    with torch.no_grad():
        ms_t = timeit(lambda: block_bf16(big))
    results["ffn_torch_bf16"] = dict(ok=True, ms_32768rows=ms_t, rows_per_s=32768 / ms_t * 1e3)
    print("ffn_torch_bf16", results["ffn_torch_bf16"], flush=True)


def check_chain():
    """in-box throughput experiment, 1 GPU, short chain (plumbing check; the full config runs via the module CLI)"""
    from lah_b200.experiments.throughput import inbox_chain
    for bt, dt in (("ffn", "bf16"), ("ffn", "fp8"), ("transformer", "bf16")):
        args = inbox_chain.make_parser().parse_args(["--block-type", bt, "--layers-per-gpu", "4", "--jobs", "8",
                                                     "--passes", "2", "--dtype", dt])
        out = inbox_chain.run(args)
        results[f"chain_{bt}_{dt}"] = dict(ok=bool(out["ok"]), samples_per_s=out["value"], layer_ms=out["layer_ms"])
        print(f"chain_{bt}_{dt}", results[f"chain_{bt}_{dt}"], flush=True)


if __name__ == "__main__":
    for fn in (check_attention, check_attention_bwd, check_layer, check_transformer_train, check_ffn_native, check_chain):
        try:
            fn()
        except Exception as e:  # noqa
            import traceback
            traceback.print_exc()
            results[fn.__name__] = dict(ok=False, error=repr(e))
    import json
    json.dump(results, open(output_path("native_layers_check.json"), "w"), indent=1)
    print("ALL_OK" if all(v.get("ok") for v in results.values()) else "SOME_FAILED")
