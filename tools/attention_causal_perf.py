"""GPU timing of causal against bidirectional attention (writes check_out/attention_causal_perf.json).

Attention forward and backward with 16 heads at head dim 64 and 128 (d_model 1024, 2048), S = 512, 2048 and 4096, 16,384
tokens (batch = 16384 // S): the bidirectional kernels, the causal kernels, and torch's scaled_dot_product_attention on the
flash backend with is_causal=True on the same q, k, v (forward, and forward + backward under autograd).  TFLOP/s of the causal
runs count the (query, key) pairs with key <= query, S (S + 1) / 2 per head: half the bidirectional count plus the
diagonal; forward 4, backward 10, forward + backward 14 flops per pair and head-dim column, as tools/attention_head_dim_perf.py.
Then one ExpertBackend.backward (forward recompute + backward + AMSGrad) of TransformerEncoderLayer(1024, 16) (dropout 0.1,
training mode) on 32 x 512 tokens, causal against bidirectional.  Each number is the median of 5 windows (20 calls) after a
warm-up, CUDA events; the two variants of each shape are timed back to back in the same process.  The card's name and power
limit are read in the same run.
"""
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import torch.nn.functional as F

import lah_b200  # noqa
from tools import output_path
from tools.attention_head_dim_perf import card, time_ms
from lah_b200.models.layers import TransformerEncoderLayer
from lah_b200.ops import kernels as K

TOKENS, HEADS = 16384, 16
HDS, SEQS = (64, 128), (512, 2048, 4096)


def attention(hd, S):
    from torch.nn.attention import SDPBackend, sdpa_kernel
    d, batch = HEADS * hd, TOKENS // S
    T = batch * S
    g = torch.Generator().manual_seed(hd + S)
    qkv = torch.randn(T, 3 * d, generator=g).to(torch.bfloat16).cuda()
    dout = torch.randn(T, d, generator=g).to(torch.bfloat16).cuda()
    out = torch.empty(T, d, dtype=torch.bfloat16, device="cuda")
    lse = torch.empty(T, HEADS, device="cuda")
    pairs = {False: batch * HEADS * S * S * hd, True: batch * HEADS * (S * (S + 1) // 2) * hd}
    res = {}
    for causal in (False, True):
        fwd = time_ms(lambda: K.attention_fwd(qkv, HEADS, out=out, lse=lse, seq_len=S, causal=causal))
        bwd = time_ms(lambda: K.attention_bwd(qkv, out, dout, lse, HEADS, seq_len=S, causal=causal))
        f = pairs[causal]
        res["causal" if causal else "bidirectional"] = dict(
            fwd_ms=fwd[0], fwd_ms_min_max=fwd[1:], fwd_tflops=4.0 * f / fwd[0] / 1e9, bwd_ms=bwd[0], bwd_ms_min_max=bwd[1:],
            bwd_tflops=10.0 * f / bwd[0] / 1e9, fwd_plus_bwd_ms=fwd[0] + bwd[0])
    q, k, v = (t.transpose(1, 2) for t in qkv.view(batch, S, 3, HEADS, hd).unbind(2))   # [B, H, S, hd] views
    go = dout.view(batch, S, HEADS, hd).transpose(1, 2)
    qg, kg, vg = (t.detach().requires_grad_(True) for t in (q, k, v))

    def sdpa_fwd_bwd():
        o = F.scaled_dot_product_attention(qg, kg, vg, is_causal=True)
        torch.autograd.grad(o, (qg, kg, vg), go)

    with sdpa_kernel(SDPBackend.FLASH_ATTENTION):
        sf = time_ms(lambda: F.scaled_dot_product_attention(q, k, v, is_causal=True))
        sfb = time_ms(sdpa_fwd_bwd)
    f = pairs[True]
    res["sdpa_flash_causal"] = dict(fwd_ms=sf[0], fwd_ms_min_max=sf[1:], fwd_tflops=4.0 * f / sf[0] / 1e9,
                                    fwd_bwd_ms=sfb[0], fwd_bwd_ms_min_max=sfb[1:], fwd_bwd_tflops=14.0 * f / sfb[0] / 1e9)
    c, b = res["causal"], res["bidirectional"]
    res["causal_vs_bidirectional"] = dict(fwd=c["fwd_ms"] / b["fwd_ms"], bwd=c["bwd_ms"] / b["bwd_ms"])
    res["causal_vs_sdpa"] = dict(fwd=c["fwd_ms"] / sf[0], fwd_bwd=c["fwd_plus_bwd_ms"] / sfb[0])
    return dict(d_model=d, batch=batch, tokens=T, cases=res)


def expert(causal, batch=32, S=512, d=1024):
    torch.manual_seed(0)
    layer = TransformerEncoderLayer(d, HEADS, causal=causal).cuda()
    be = lah_b200.ExpertBackend(name="t", expert=layer, opt=torch.optim.Adam(layer.parameters(), lr=1e-4, amsgrad=True),
                                args_schema=(lah_b200.BatchTensorProto(S, d),), outputs_schema=lah_b200.BatchTensorProto(S, d),
                                max_batch_size=batch)
    x = torch.randn(batch, S, d, device="cuda")
    g = torch.randn(batch, S, d, device="cuda") * 0.1
    ms = time_ms(lambda: be.backward(x, g))
    assert type(be._executor).__name__ == "NativeTransformerExecutor" and be._executor.causal == causal
    return dict(backward_ms=ms[0], backward_ms_min_max=ms[1:])


if __name__ == "__main__":
    assert torch.cuda.is_available(), "this measurement needs a GPU"
    results = dict(card=card(), heads=HEADS, tokens=TOKENS, attention={}, expert={})
    print(results["card"], flush=True)
    for hd in HDS:
        for S in SEQS:
            results["attention"][f"hd{hd}_S{S}"] = r = attention(hd, S)
            for kind, c in r["cases"].items():
                print(f"attention hd={hd} S={S} {kind}", {k: round(v, 4) for k, v in c.items() if not k.endswith("min_max")},
                      flush=True)
            torch.cuda.empty_cache()
    for causal in (False, True):
        results["expert"]["causal" if causal else "bidirectional"] = r = expert(causal)
        print("expert backward", "causal" if causal else "bidirectional", r, flush=True)
    results["expert"]["causal_vs_bidirectional"] = \
        results["expert"]["causal"]["backward_ms"] / results["expert"]["bidirectional"]["backward_ms"]
    print("expert backward causal / bidirectional", results["expert"]["causal_vs_bidirectional"], flush=True)
    with open(output_path("attention_causal_perf.json"), "w") as f:
        json.dump(results, f, indent=1)
