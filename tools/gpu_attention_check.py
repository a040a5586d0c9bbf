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


# ------------------------------------------------------------------------------------------------ dropout (csrc/dropout.cuh)
def check_dropout_mask():
    """K.dropout_mask (the device mask definition) == K.dropout_mask_ref (CPU Philox) bit for bit; the elementwise dropout
    kernels apply that mask"""
    cases = [((1, 2, 512, 512), 0.1, 1234, 0), ((2, 3, 512, 512), 0.5, 2 ** 63 + 17, 0), ((512, 1024), 0.1, 99, 1),
             ((1024, 2048), 0.1, 2 ** 40 + 5, 2), ((256, 256), 0.3, 7, 3), ((4096, 1024), 0.1, 2 ** 64 - 1, 3)]
    for shape, p, seed, site in cases:
        got = K.dropout_mask(shape, p, seed, site).cpu()
        ref = K.dropout_mask_ref(shape, p, seed, site)
        name = f"dropout_mask_site{site}_{'x'.join(map(str, shape))}"
        results[name] = dict(ok=bool(torch.equal(got, ref)), mismatches=int((got != ref).sum()), keep=float(got.float().mean()))
        print(name, results[name], flush=True)
    torch.manual_seed(5)
    f = torch.randn(512, 2048, device="cuda").to(torch.bfloat16)
    dg = torch.randn(512, 2048, device="cuda").to(torch.bfloat16)
    m = K.dropout_mask((512, 2048), 0.1, 77, 2).float()
    errs = dict(apply=rel(K.dropout_apply(dg, 0.1, 77, 2), dg.float() * m / 0.9),
                gelu=rel(K.gelu_dropout(f, 0.1, 77, 2), torch.nn.functional.gelu(f.float()) * m / 0.9))
    fr = f.float().requires_grad_(True)
    (torch.nn.functional.gelu(fr) * m / 0.9).backward(dg.float())
    errs["gelu_bwd"] = rel(K.gelu_dropout_bwd(dg, f, 0.1, 77, 2), fr.grad)
    results["dropout_elementwise"] = dict(ok=all(v < 1e-2 for v in errs.values()), **errs)
    print("dropout_elementwise", results["dropout_elementwise"], flush=True)


def attention_dropout_ref(qkv, num_heads, mask, p, seq_len=512):
    """fp32 oracle: (M o softmax(q k^T / sqrt(d))) v / (1 - p) per head, mask [B, H, S, S]"""
    tokens, three_d = qkv.shape
    d = three_d // 3
    q, k, v = qkv.float().view(tokens // seq_len, seq_len, 3, num_heads, d // num_heads).unbind(2)
    q, k, v = (t.transpose(1, 2) for t in (q, k, v))
    att = torch.softmax(q @ k.transpose(-1, -2) / (d // num_heads) ** 0.5, dim=-1) * mask / (1 - p)
    return (att @ v).transpose(1, 2).reshape(tokens, d)


def check_attention_dropout():
    """attention forward / backward with p = 0.1 vs the fp32 oracle with the materialised mask; p = 0 is byte-identical
    to no dropout"""
    torch.manual_seed(6)
    p = 0.1
    for batch, heads in [(1, 2), (2, 16)]:
        d, seed = heads * 64, 1000 + batch
        qkv = (torch.randn(batch * 512, 3 * d, device="cuda") * 1.2).to(torch.bfloat16)
        dout = torch.randn(batch * 512, d, device="cuda").to(torch.bfloat16)
        lse = torch.empty(batch * 512, heads, device="cuda")
        out = K.attention_fwd(qkv, heads, lse=lse, dropout=(p, seed))
        dqkv = K.attention_bwd(qkv, out, dout, lse, heads, dropout=(p, seed))
        mask = K.dropout_mask((batch, heads, 512, 512), p, seed, K.SITE_ATTN).float()
        ref_in = qkv.float().requires_grad_(True)
        ref = attention_dropout_ref(ref_in, heads, mask, p)
        ref.backward(dout.float())
        g = ref_in.grad
        errs = dict(dq=rel(dqkv[:, :d], g[:, :d]), dk=rel(dqkv[:, d:2 * d], g[:, d:2 * d]), dv=rel(dqkv[:, 2 * d:], g[:, 2 * d:]))
        q, k, _ = qkv.float().view(batch, 512, 3, heads, 64).unbind(2)
        s2 = torch.einsum("bqhd,bkhd->bhqk", q, k) * (0.125 * 1.4426950408889634)
        lse_ref = torch.logsumexp(s2 * 0.6931471805599453, dim=-1) / 0.6931471805599453   # undropped softmax
        errs["lse"] = (lse.view(batch, 512, heads).transpose(1, 2) - lse_ref).abs().max().item()
        fwd = rel(out, ref.detach())
        # p = 0: the same launch as without dropout, byte for byte
        lse0, lse0d = torch.empty_like(lse), torch.empty_like(lse)
        o0 = K.attention_fwd(qkv, heads, lse=lse0)
        o0d = K.attention_fwd(qkv, heads, lse=lse0d, dropout=(0.0, seed))
        g0 = K.attention_bwd(qkv, o0, dout, lse0, heads)
        g0d = K.attention_bwd(qkv, o0d, dout, lse0d, heads, dropout=(0.0, seed))
        same = bool(torch.equal(o0, o0d) and torch.equal(lse0, lse0d) and torch.equal(g0, g0d))
        name = f"attention_dropout_b{batch}_h{heads}"
        results[name] = dict(ok=fwd < 2e-2 and all(v < 3e-2 for v in errs.values()) and same, fwd=fwd, p0_byte_equal=same, **errs)
        print(name, results[name], flush=True)
    batch, heads, d = 32, 16, 1024
    qkv = torch.randn(batch * 512, 3 * d, device="cuda").to(torch.bfloat16)
    dout = torch.randn(batch * 512, d, device="cuda").to(torch.bfloat16)
    lse = torch.empty(batch * 512, heads, device="cuda")
    out = torch.empty(batch * 512, d, device="cuda", dtype=torch.bfloat16)
    perf = {}
    for pp in (0.0, 0.1):
        dr = (pp, 7) if pp else None
        perf[f"fwd_ms_p{pp}"] = timeit(lambda: K.attention_fwd(qkv, heads, out=out, lse=lse, dropout=dr), iters=20)
        perf[f"bwd_ms_p{pp}"] = timeit(lambda: K.attention_bwd(qkv, out, dout, lse, heads, dropout=dr), iters=20)
    results["attention_dropout_perf_32seq"] = dict(ok=True, **perf)
    print("attention_dropout_perf_32seq", results["attention_dropout_perf_32seq"], flush=True)


def transformer_layer_ref(layer, x, masks=None, ps=None):
    """fp32 functional forward of models.layers.TransformerEncoderLayer with given keep masks (site order of
    kernels.dropout_mask: attention [B, H, S, S], dropout1 [T, d], dropout [T, ff], dropout2 [T, d]); None = no dropout"""
    B, S, d = x.shape
    T, a = B * S, layer.self_attn
    H = a.num_heads
    F = torch.nn.functional

    def drop(t, i):
        return t if masks is None else t * masks[i] / (1 - ps[i])

    qkv = F.linear(x.reshape(T, d), a.in_proj_weight, a.in_proj_bias)
    q, k, v = (t.transpose(1, 2) for t in qkv.view(B, S, 3, H, d // H).unbind(2))
    att = drop(torch.softmax(q @ k.transpose(-1, -2) / (d // H) ** 0.5, dim=-1), 0)
    o = (att @ v).transpose(1, 2).reshape(T, d)
    x1 = F.layer_norm(x.reshape(T, d) + drop(F.linear(o, a.out_proj.weight, a.out_proj.bias), 1), (d,), layer.norm1.weight,
                      layer.norm1.bias, layer.norm1.eps)
    g = drop(F.gelu(F.linear(x1, layer.linear1.weight, layer.linear1.bias)), 2)
    y = x1 + drop(F.linear(g, layer.linear2.weight, layer.linear2.bias), 3)
    return F.layer_norm(y, (d,), layer.norm2.weight, layer.norm2.bias, layer.norm2.eps).view(B, S, d)


def dropout_masks(seed, ps, batch, heads, d, ff):
    T = batch * 512
    shapes = ((batch, heads, 512, 512), (T, d), (T, ff), (T, d))
    return [K.dropout_mask(shape, p, seed, site).float() for site, (shape, p) in enumerate(zip(shapes, ps))]


def check_transformer_train_dropout():
    """the reference's default transformer expert (dropout 0.1 at all four sites) trained by ExpertBackend on the sm_90a
    kernels: forward, dx, weight gradients and three AMSGrad steps vs an fp32 functional oracle with the same masks; eval
    mode == p = 0 bit for bit; re-seeding reproduces training-mode forwards; the throughput server's experts run natively"""
    import copy
    import lah_b200 as lib
    from lah_b200.models.layers import name_to_block
    from lah_b200.ops import native
    from lah_b200.runtime.native_executor import NativeTransformerExecutor, draw_dropout_seed
    torch.manual_seed(4)
    layer = name_to_block["transformer"](1024).cuda()
    ref = copy.deepcopy(layer)
    ref_opt = torch.optim.Adam(ref.parameters(), lr=1e-4, amsgrad=True)
    be = lib.ExpertBackend(name="t", expert=layer, opt=torch.optim.Adam(layer.parameters(), lr=1e-4, amsgrad=True),
                           args_schema=(lib.BatchTensorProto(512, 1024),), outputs_schema=lib.BatchTensorProto(512, 1024),
                           max_batch_size=8)
    ps = NativeTransformerExecutor._dropout_ps(layer)
    x = torch.randn(2, 512, 1024, device="cuda")
    g = torch.randn(2, 512, 1024, device="cuda") * 0.1
    torch.manual_seed(10)
    seed = draw_dropout_seed()
    torch.manual_seed(10)
    (y,) = be.forward(x)
    native_used = type(be._executor).__name__ == "NativeTransformerExecutor"
    with torch.no_grad():
        errs = dict(fwd=rel(y, transformer_layer_ref(ref, x, dropout_masks(seed, ps, 2, 16, 1024, 2048), ps)))
    for it in range(3):
        torch.manual_seed(20 + it)
        seed = draw_dropout_seed()
        torch.manual_seed(20 + it)
        (gx,) = be.backward(x, g)
        xr = x.clone().requires_grad_(True)
        transformer_layer_ref(ref, xr, dropout_masks(seed, ps, 2, 16, 1024, 2048), ps).backward(g)
        if it == 0:
            errs["dx"] = rel(gx, xr.grad)
            st = be.opt.state_dict()["state"]
            for i, (n, p) in enumerate(ref.named_parameters()):
                if n in ("self_attn.in_proj_weight", "linear1.weight", "linear2.weight", "self_attn.out_proj.weight",
                         "self_attn.in_proj_bias", "self_attn.out_proj.bias", "linear2.bias", "linear1.bias", "norm1.weight"):
                    errs["g_" + n] = rel(st[i]["exp_avg"] / 0.1, p.grad)
        ref_opt.step(), ref_opt.zero_grad()
    sd, rsd = be.state_dict(), ref.state_dict()
    errs["param_mean_abs_diff"] = max((sd["expert." + k] - v).abs().mean().item() for k, v in rsd.items())
    ok = native_used and ps == (0.1,) * 4 and errs["fwd"] < 3e-2 and errs["dx"] < 5e-2 and \
        errs["param_mean_abs_diff"] < 1.5e-4 and all(v < 6e-2 for k, v in errs.items() if k.startswith("g_"))
    results["transformer_train_dropout"] = dict(ok=bool(ok), native=native_used, **errs)
    print("transformer_train_dropout", results["transformer_train_dropout"], flush=True)

    # training-mode forwards: fresh mask per call, reproducible under torch.manual_seed
    torch.manual_seed(5)
    y1, y2 = be.forward(x)[0], be.forward(x)[0]
    torch.manual_seed(5)
    y1b, y2b = be.forward(x)[0], be.forward(x)[0]
    reseed = dict(differ=not torch.equal(y1, y2), reproduced=bool(torch.equal(y1, y1b) and torch.equal(y2, y2b)))
    # eval mode: the p = 0 kernels, bit for bit
    layer0 = copy.deepcopy(layer)
    layer0.dropout.p = layer0.dropout1.p = layer0.dropout2.p = 0.0
    layer0.self_attn.dropout = 0.0
    be0 = lib.ExpertBackend(name="t0", expert=layer0, opt=torch.optim.Adam(layer0.parameters(), lr=1e-4, amsgrad=True),
                            args_schema=(lib.BatchTensorProto(512, 1024),), outputs_schema=lib.BatchTensorProto(512, 1024),
                            max_batch_size=8)
    layer.eval()
    reseed["eval_equals_p0"] = bool(torch.equal(be.forward(x)[0], be0.forward(x)[0]))
    reseed["eval_native"] = type(be0._executor).__name__ == "NativeTransformerExecutor"
    layer.train()
    # the throughput server's transformer experts (reference definition, default Adam) are served natively
    from lah_b200.experiments.throughput import throughput_server
    args = throughput_server.make_parser().parse_args(["-p", "0", "--gpu", "0", "--block-type", "transformer",
                                                          "--layers-per-gpu", "1"])
    sbe = throughput_server.build_experts(args)["expert0"]
    sbe.expert.cuda()
    native.reset_launches()
    sbe.forward(torch.randn(2, 512, 1024, device="cuda"))
    torch.cuda.synchronize()
    reseed["server_launches"] = native.launches()
    reseed["server_native"] = type(sbe._executor).__name__ == "NativeTransformerExecutor"
    results["transformer_dropout_semantics"] = dict(ok=all(bool(v) for v in reseed.values()), **reseed)
    print("transformer_dropout_semantics", results["transformer_dropout_semantics"], flush=True)

    xb = torch.randn(8, 512, 1024, device="cuda")
    gb = torch.randn(8, 512, 1024, device="cuda") * 0.1
    ms = timeit(lambda: be.backward(xb, gb), iters=5)
    ref_bf = copy.deepcopy(ref).train()
    ref_opt_bf = torch.optim.Adam(ref_bf.parameters(), lr=1e-4, amsgrad=True, fused=True)

    def torch_step():
        xr = xb.clone().requires_grad_(True)
        with torch.autocast("cuda", dtype=torch.bfloat16):
            out = ref_bf(xr)
        out.backward(gb)
        ref_opt_bf.step(), ref_opt_bf.zero_grad()

    ms_t = timeit(torch_step, iters=5)
    results["transformer_train_dropout_perf"] = dict(ok=True, ms_fwd_bwd_adam_8seq=ms, torch_bf16_autocast_ms=ms_t,
                                                     seqs_per_s=8 / ms * 1e3)
    print("transformer_train_dropout_perf", results["transformer_train_dropout_perf"], flush=True)


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
    for fn in (check_attention, check_attention_bwd, check_layer, check_transformer_train, check_dropout_mask,
               check_attention_dropout, check_transformer_train_dropout, check_ffn_native, check_chain):
        try:
            fn()
        except Exception as e:  # noqa
            import traceback
            traceback.print_exc()
            results[fn.__name__] = dict(ok=False, error=repr(e))
    import json
    json.dump(results, open(output_path("native_layers_check.json"), "w"), indent=1)
    print("ALL_OK" if all(v.get("ok") for v in results.values()) else "SOME_FAILED")
