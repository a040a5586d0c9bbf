"""GPU check of the non-GEMM kernels and of one full FusedDMoE layer against PyTorch oracles (writes check_out/layer_check.json)."""
import json
import os
import sys
from functools import partial

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import torch.nn.functional as F

import lah_b200  # noqa
from tools import output_path
from lah_b200.ops import kernels as K
from lah_b200.models.layers import FeedforwardBlock
from lah_b200.parallel import engine as E

results = {}


def rel(got, ref):
    return ((got.float() - ref.float()).norm() / (ref.float().norm() + 1e-12)).item()


def record(name, **kw):
    results[name] = kw
    print(name, kw, flush=True)


def check_gate():
    torch.manual_seed(0)
    for grid, k, B in [((8, 8), 4, 1000), ((32, 32), 4, 300), ((4, 4, 4), 3, 500), ((16,), 8, 64)]:
        En = 1
        for g in grid:
            En *= g
        logits = torch.randn(B, sum(grid), device="cuda")
        alive = (torch.rand(En, device="cuda") > 0.3).to(torch.uint8)
        idx = torch.empty(B * k, dtype=torch.int32, device="cuda")
        pos = torch.empty_like(idx)
        w = torch.empty(B * k, device="cuda")
        counts = torch.zeros(En, dtype=torch.int32, device="cuda")
        K.gate_topk(logits, grid, k, alive=alive, idx=idx, w=w, pos=pos, counts=counts)
        torch.cuda.synchronize()
        ridx, rw = K.gate_topk_ref(logits, grid, k, alive=alive)
        ok_idx = bool((idx.view(B, k).long() == ridx).all())
        werr = (w.view(B, k) - rw).abs().max().item()
        cnt_ref = torch.bincount(ridx[ridx >= 0].flatten(), minlength=En)
        ok_cnt = bool((counts.long() == cnt_ref).all())
        # positions must be a permutation of 0..count-1 per expert
        ok_pos = True
        iv, pv = idx.long(), pos.long()
        for e in range(min(En, 64)):
            ps = pv[iv == e].sort().values
            ok_pos &= bool((ps == torch.arange(len(ps), device="cuda")).all())
        record(f"gate_{'x'.join(map(str, grid))}_k{k}", ok=ok_idx and ok_cnt and ok_pos and werr < 1e-5, idx=ok_idx,
               cnt=ok_cnt, pos=ok_pos, werr=werr)
    # failure injection: statistical check
    grid, k, B = (8, 8), 4, 4096
    logits = torch.randn(B, 16, device="cuda")
    idx = torch.empty(B * k, dtype=torch.int32, device="cuda")
    pos, w = torch.empty_like(idx), torch.empty(B * k, device="cuda")
    counts = torch.zeros(64, dtype=torch.int32, device="cuda")
    K.gate_topk(logits, grid, k, failure_rate=0.5, seed=123, idx=idx, w=w, pos=pos, counts=counts)
    ridx, _ = K.gate_topk_ref(logits, grid, k)
    changed = (idx.view(B, k).long() != ridx).any(dim=1).float().mean().item()
    wsum = w.view(B, k).sum(1)
    record("gate_failure_injection", ok=bool(changed > 0.8 and (wsum - 1).abs().max().item() < 1e-4), changed=changed)


def check_ln():
    torch.manual_seed(1)
    for C in (2048, 512, 4096):
        G, R = 3, 640
        tg = torch.tensor([0, 2, -1, 1, 1], dtype=torch.int32, device="cuda")
        h = (torch.randn(R, C, device="cuda") * 2 + 0.5).to(torch.bfloat16)
        gamma = torch.rand(G, C, device="cuda") + 0.5
        beta = torch.randn(G, C, device="cuda") * 0.1
        a = torch.zeros(R, C, dtype=torch.bfloat16, device="cuda")
        mean, rstd = torch.zeros(R, device="cuda"), torch.zeros(R, device="cuda")
        K.ln_relu_fwd(h, gamma, beta, tg, out=a, mean=mean, rstd=rstd)
        rows_g = tg.repeat_interleave(128)
        valid = rows_g >= 0
        hf = h.float().requires_grad_(True)
        gsel, bsel = gamma[rows_g.clamp(min=0).long()], beta[rows_g.clamp(min=0).long()]
        gsel.requires_grad_(True); bsel.requires_grad_(True)
        mu = hf.mean(-1, keepdim=True)
        var = hf.var(-1, unbiased=False, keepdim=True)
        y = F.relu((hf - mu) * torch.rsqrt(var + 1e-5) * gsel + bsel)
        fwd_err = rel(a[valid], y[valid])
        da = torch.randn(R, C, device="cuda").to(torch.bfloat16)
        (y * da.float() * valid.unsqueeze(-1)).sum().backward()
        dh = torch.zeros(R, C, dtype=torch.bfloat16, device="cuda")
        dg, db, dbias = torch.zeros(G, C, device="cuda"), torch.zeros(G, C, device="cuda"), torch.zeros(G, C, device="cuda")
        K.ln_relu_bwd(da, h, mean, rstd, gamma, beta, tg, dh=dh, dgamma=dg, dbeta=db, dbias=dbias)
        torch.cuda.synchronize()
        dh_err = rel(dh[valid], hf.grad[valid])
        dg_ref = torch.zeros(G, C, device="cuda").index_add_(0, rows_g.clamp(min=0).long()[valid], gsel.grad[valid])
        db_ref = torch.zeros(G, C, device="cuda").index_add_(0, rows_g.clamp(min=0).long()[valid], bsel.grad[valid])
        dbias_ref = torch.zeros(G, C, device="cuda").index_add_(0, rows_g.clamp(min=0).long()[valid], hf.grad[valid])
        errs = dict(fwd=fwd_err, dh=dh_err, dgamma=rel(dg, dg_ref), dbeta=rel(db, db_ref), dbias=rel(dbias, dbias_ref))
        record(f"ln_C{C}", ok=all(v < 2e-2 for v in errs.values()), **errs)
        if C == 512:
            cs = torch.zeros(G, C, device="cuda")
            K.grouped_colsum(da, tg, out=cs)
            cs_ref = torch.zeros(G, C, device="cuda").index_add_(0, rows_g.clamp(min=0).long()[valid], da.float()[valid])
            record("colsum", ok=rel(cs, cs_ref) < 1e-3, err=rel(cs, cs_ref))


def check_adam():
    torch.manual_seed(2)
    G, segs = 3, [64, 8, 32]
    n = sum(segs) * G
    p = torch.randn(n, device="cuda")
    p0 = p.clone()
    g = torch.zeros(n, device="cuda")
    m, v, vmax = torch.zeros(n, device="cuda"), torch.zeros(n, device="cuda"), torch.zeros(n, device="cuda")
    pb = torch.zeros(n, dtype=torch.bfloat16, device="cuda")
    step = torch.zeros(G, dtype=torch.int32, device="cuda")
    # torch reference: one Adam per group over its three tensors
    views, off = [], 0
    for s in segs:
        views.append((off, s))
        off += s * G
    ref_params = [[p0[o + gi * s: o + (gi + 1) * s].clone().requires_grad_(True) for (o, s) in views] for gi in range(G)]
    opts = [torch.optim.Adam(ps, lr=1e-2, amsgrad=True) for ps in ref_params]
    for it in range(4):
        rows = torch.tensor([5, 0 if it % 2 else 3, 7], dtype=torch.int32, device="cuda")
        g.copy_(torch.randn(n, device="cuda"))
        for gi in range(G):
            if rows[gi] > 0:
                for t, (o, s) in zip(ref_params[gi], views):
                    t.grad = g[o + gi * s: o + (gi + 1) * s].clone()
                opts[gi].step()
        K.bump_steps(step, rows)
        K.adam_step(p, g, m, v, vmax, pb, segs, G, step=step, group_rows=rows, lr=1e-2, amsgrad=True, zero_mask=0b010)
    torch.cuda.synchronize()
    err = 0.0
    for gi in range(G):
        for t, (o, s) in zip(ref_params[gi], views):
            err = max(err, (p[o + gi * s: o + (gi + 1) * s] - t.detach()).abs().max().item())
    zero_ok = bool((g[views[1][0]: views[1][0] + 8 * G].view(G, 8)[[0, 2]] == 0).all()) and bool((g[:64] != 0).any())
    record("adam_amsgrad", ok=err < 2e-5 and zero_ok and rel(pb, p) < 5e-3, max_abs_err=err, zero_ok=zero_ok)


def check_layer_fp8():
    """same layer with the forward GEMMs on block-scaled FP8 tensor cores (looser tolerances: E4M3 has 3 mantissa bits)"""
    check_layer(expert_dtype="fp8")


def check_layer_small():
    """same layer through the weight-streaming kernels (swap-AB GEMMs, fused wgrad + AMSGrad; csrc/small_m.cu)"""
    check_layer(expert_path="small")


def check_layer(expert_dtype="bf16", expert_path="big"):
    torch.manual_seed(3)
    cfg = E.DMoEConfig(hidden=512, grid_size=(4, 4), k=4, num_layers=1, tokens_per_rank=512, lr=1e-3,
                       expert_dtype=expert_dtype, expert_path=expert_path)
    ctx = E.EngineContext(cfg)
    layer = E.FusedDMoE(cfg, ctx).cuda()
    B = 512
    x = torch.randn(B, 512, device="cuda").to(torch.bfloat16).requires_grad_(True)
    # reference experts as real nn.Modules + one torch Adam each
    experts, opts = [], []
    for le in range(16):
        blk = FeedforwardBlock(512).cuda()
        blk.load_state_dict({k[len("expert."):]: v for k, v in layer.shard.expert_state_dict(le).items()})
        experts.append(blk)
        opts.append(torch.optim.Adam(blk.parameters(), lr=1e-3, amsgrad=True))
    y = layer(x)
    gy = torch.randn(B, 512, device="cuda").to(torch.bfloat16)
    y.backward(gy)
    torch.cuda.synchronize()
    ctx.check_status()
    # oracle
    xr = x.detach().float().requires_grad_(True)
    logits = F.linear(xr, layer.proj.weight.detach(), layer.proj.bias.detach())
    logits.retain_grad()
    idx, _ = K.gate_topk_ref(logits.detach(), cfg.grid_size, cfg.k)
    scores = K.product_key_scores(logits, cfg.grid_size)
    wts = torch.softmax(torch.gather(scores, 1, idx), dim=-1)
    out = torch.zeros(B, 512, device="cuda")
    for e in range(16):
        tok, slot = torch.nonzero(idx == e, as_tuple=True)
        if len(tok):
            out = out.index_put((tok,), experts[e](xr[tok]) * wts[tok, slot].unsqueeze(-1), accumulate=True)
    out.backward(gy.float())
    for e in range(16):
        if (idx == e).any():
            opts[e].step()
    errs = dict(y=rel(y, out), dx=rel(x.grad, xr.grad))
    # gradient w.r.t. proj (through dlogits) — compare proj.weight.grad of the fused layer with the oracle's
    dW_ref = logits.grad.t() @ xr.detach()
    errs["dproj"] = rel(layer.proj.weight.grad, dW_ref)
    perr = {}
    for n in E.SEG_NAMES:
        ref = torch.stack([experts[e].state_dict()[E.REF_KEYS[n]] for e in range(16)])
        before = torch.stack([layer.shard.expert_state_dict(e)["expert." + E.REF_KEYS[n]] for e in range(16)]).cuda()
        perr[n] = (before - ref).abs().mean().item()
    errs["param_mean_abs_diff_after_step"] = max(perr.values())
    # VALUE of the weight gradients: after the first AMSGrad step exp_avg = (1 - beta1) * grad.  The oracle here is a pure fp32
    # nn.Module: ~0.4 % of the ReLU gates of a bf16 forward differ from an fp32 forward, which bounds the agreement of dW1 / dW2
    # at ~5 % rel-L2 (dW3, upstream of no ReLU, agrees to 0.4 %); bench.py's parity pass uses the bf16-rounding oracle (< 2 %)
    werr = {}
    for n, li in (("w1", 0), ("w2", 3), ("w3", 6)):
        ref = torch.stack([experts[e].layers[li].weight.grad if experts[e].layers[li].weight.grad is not None
                           else torch.zeros_like(experts[e].layers[li].weight) for e in range(16)])
        werr[n] = rel(layer.shard.m_views[n][:16] / (1 - cfg.betas[0]), ref)
    errs["wgrad_rel_err"] = max(werr.values())
    # first Adam step moves every parameter by ~lr*sign(grad): a mean |diff| << lr means the gradients agree in sign
    tol = 1.0 if expert_dtype == "bf16" else 3.0
    ok = errs["y"] < 2e-2 * tol and errs["dx"] < 3e-2 * tol and errs["dproj"] < 5e-2 * tol and \
        errs["param_mean_abs_diff_after_step"] < 1e-4 * tol and errs["wgrad_rel_err"] < 8e-2 * (tol if tol == 1.0 else 4.0)
    record("layer_16experts" + ("" if expert_dtype == "bf16" else "_" + expert_dtype) + ("" if expert_path == "big" else "_" + expert_path),
           ok=bool(ok), **errs, per_param=perr, wgrad=werr, steps=layer.shard.step.tolist())
    ctx.close()


def main():
    print("device:", torch.cuda.get_device_name(0), flush=True)
    selected = [a for a in sys.argv[1:] if not a.startswith("-")]
    fns = (check_gate, check_ln, check_adam, check_layer, check_layer_small, check_layer_fp8)
    if selected:   # e.g. under compute-sanitizer: python tools/gpu_layer_check.py check_layer check_layer_small
        fns = [globals()[name] for name in selected]
    for fn in fns:
        try:
            fn()
        except Exception as e:  # noqa
            import traceback
            traceback.print_exc()
            record(fn.__name__ + "_exception", ok=False, error=repr(e))
    with open(output_path("layer_check.json"), "w") as f:
        json.dump(results, f, indent=1, default=str)
    print("ALL_OK" if all(v.get("ok") for v in results.values()) else "SOME_FAILED")


if __name__ == "__main__":
    main()
