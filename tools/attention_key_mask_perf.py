"""GPU timing of key padding masks in the attention kernels and the transformer expert (writes
check_out/attention_key_mask_perf.json).

Attention forward and backward at d_model 1024 and 2048 with 16 heads (head dim 64, 128), S = 512 and 2048, 16,384 tokens
(batch = 16384 // S), for these masks:
  * none          the unmasked kernels
  * all_false     the masked kernels with a mask that masks nothing
  * right_50      every sequence padded on the right to S / 2 (half the key blocks are skipped)
  * uniform       lengths uniform in [S / 4, S], right padding
  * holes_30      30 % of the keys masked at random (no key block can be skipped)
  * sdpa_uniform  torch's scaled_dot_product_attention (bf16) with the uniform mask, for reference: forward, and
                  forward + backward under autograd as "bwd"
Then one ExpertBackend.backward (forward recompute + backward + AMSGrad) and one forward of
nn.TransformerEncoderLayer(1024, 16, batch_first=True) (dropout 0.1, training mode) on 32 x 512 tokens with the uniform
mask, through the sm_90a executor and with native=False.  Each number is the median of 5 windows (20 calls for kernels and
the native expert, 5 for eager) after a warm-up, CUDA events.  The card's name and power limit are read in the same run.
"""
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import torch.nn.functional as F
from torch import nn

import lah_b200  # noqa
from tools import output_path
from tools.attention_head_dim_perf import card, time_ms
from lah_b200.ops import kernels as K

TOKENS, HEADS = 16384, 16
SHAPES = ((1024, 512), (1024, 2048), (2048, 512), (2048, 2048))   # (d_model, S)


def pad_mask(kind, batch, S, seed=0):
    """bool [batch, S], True = padding key"""
    g = torch.Generator().manual_seed(seed)
    pos = torch.arange(S)
    if kind == "all_false":
        return torch.zeros(batch, S, dtype=torch.bool)
    if kind == "right_50":
        return (pos >= S // 2).expand(batch, S).contiguous()
    if kind == "uniform":
        lengths = torch.randint(S // 4, S + 1, (batch, 1), generator=g)
        return pos >= lengths
    if kind == "holes_30":
        return torch.rand(batch, S, generator=g) < 0.3
    raise ValueError(kind)


def attention(d, S):
    batch = TOKENS // S
    T = batch * S
    g = torch.Generator().manual_seed(S + d)
    qkv = torch.randn(T, 3 * d, generator=g).to(torch.bfloat16).cuda()
    dout = torch.randn(T, d, generator=g).to(torch.bfloat16).cuda()
    out = torch.empty(T, d, dtype=torch.bfloat16, device="cuda")
    lse = torch.empty(T, HEADS, device="cuda")
    res = {}
    for kind in ("none", "all_false", "right_50", "uniform", "holes_30"):
        km = None if kind == "none" else K.pack_key_mask(pad_mask(kind, batch, S).cuda())
        fwd = time_ms(lambda: K.attention_fwd(qkv, HEADS, out=out, lse=lse, seq_len=S, key_mask=km))
        bwd = time_ms(lambda: K.attention_bwd(qkv, out, dout, lse, HEADS, seq_len=S, key_mask=km))
        res[kind] = dict(fwd_ms=fwd[0], fwd_ms_min_max=fwd[1:], bwd_ms=bwd[0], bwd_ms_min_max=bwd[1:])
    for kind in ("all_false", "right_50", "uniform", "holes_30"):
        res[kind]["fwd_vs_none"] = res[kind]["fwd_ms"] / res["none"]["fwd_ms"]
        res[kind]["bwd_vs_none"] = res[kind]["bwd_ms"] / res["none"]["bwd_ms"]
    q, k, v = (t.transpose(1, 2).contiguous().requires_grad_(True)
               for t in qkv.view(batch, S, 3, HEADS, d // HEADS).unbind(2))
    allowed = ~pad_mask("uniform", batch, S).cuda().view(batch, 1, 1, S)   # SDPA: True = takes part
    do = dout.view(batch, S, HEADS, d // HEADS).transpose(1, 2)

    def sdpa_fwd():
        with torch.no_grad():
            F.scaled_dot_product_attention(q, k, v, attn_mask=allowed)

    def sdpa_fwd_bwd():
        torch.autograd.grad(F.scaled_dot_product_attention(q, k, v, attn_mask=allowed), (q, k, v), do)

    fwd, both = time_ms(sdpa_fwd), time_ms(sdpa_fwd_bwd)
    res["sdpa_uniform"] = dict(fwd_ms=fwd[0], fwd_ms_min_max=fwd[1:], fwd_bwd_ms=both[0], fwd_bwd_ms_min_max=both[1:])
    return dict(batch=batch, tokens=T, cases=res)


def expert(native, batch=32, S=512, d=1024):
    torch.manual_seed(0)
    layer = nn.TransformerEncoderLayer(d, HEADS, batch_first=True).cuda()
    be = lah_b200.ExpertBackend(name="t", expert=layer, opt=torch.optim.Adam(layer.parameters(), lr=1e-4, amsgrad=True),
                                args_schema=(lah_b200.BatchTensorProto(S, d),),
                                kwargs_schema={"src_key_padding_mask": lah_b200.BatchTensorProto(S, dtype=torch.bool)},
                                outputs_schema=lah_b200.BatchTensorProto(S, d), max_batch_size=batch, native=native)
    x = torch.randn(batch, S, d, device="cuda")
    g = torch.randn(batch, S, d, device="cuda") * 0.1
    m = pad_mask("uniform", batch, S, seed=1).cuda()
    iters, warmup = (20, 3) if native else (5, 2)
    bwd = time_ms(lambda: be.backward(x, m, g), iters=iters, warmup=warmup)
    fwd = time_ms(lambda: be.forward(x, m), iters=iters, warmup=warmup)
    executor = type(be._executor).__name__ if be._executor is not None else None
    assert executor == ("NativeTransformerExecutor" if native else None), executor
    return dict(backward_ms=bwd[0], backward_ms_min_max=bwd[1:], forward_ms=fwd[0], forward_ms_min_max=fwd[1:])


if __name__ == "__main__":
    assert torch.cuda.is_available(), "this measurement needs a GPU"
    results = dict(card=card(), heads=HEADS, tokens=TOKENS, attention={}, expert={})
    print(results["card"], flush=True)
    for d, S in SHAPES:
        results["attention"][f"d{d}_S{S}"] = r = attention(d, S)
        for kind, c in r["cases"].items():
            print(f"attention d={d} S={S} {kind}", {k: v for k, v in c.items() if not k.endswith("min_max")}, flush=True)
        torch.cuda.empty_cache()
    for native in (True, False):
        results["expert"]["native" if native else "eager"] = r = expert(native)
        print("expert", "native" if native else "eager", r, flush=True)
        torch.cuda.empty_cache()
    with open(output_path("attention_key_mask_perf.json"), "w") as f:
        json.dump(results, f, indent=1)
