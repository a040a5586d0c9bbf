"""GPU timing of the transformer expert over head dims (writes check_out/attention_head_dim_perf.json).

For hd in {32, 64, 128}: d_model = 16 hd (16 heads, the reference's nhead), 16,384 tokens, S in {512, 2048}:
  * our attention forward and backward without dropout, TFLOP/s from 4 B H S^2 hd forward and 10 B H S^2 hd backward;
  * torch.nn.functional.scaled_dot_product_attention on the same bf16 q, k, v ([B, H, S, hd] views of the same qkv) with
    the flash backend only: forward, and forward + backward.
And one ExpertBackend.backward (forward recompute + backward + AMSGrad) of name_to_block["transformer"](d) (dropout 0.1)
at d = 512 and 2048, 32 sequences of 512 tokens: natively, and on the eager module path (native=False) that those widths
took before the kernels ran head dims 32 and 128.
Each number is the median of 5 windows of 20 calls (5 for the eager step) after a warm-up, CUDA events.  The card's name and
power limit are read in the same run.
"""
import json
import os
import statistics
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

import lah_b200  # noqa
from tools import output_path
from lah_b200.ops import kernels as K

HEADS, TOKENS = 16, 16384
SEQS = (512, 2048)
STEP_WIDTHS, STEP_BATCH, STEP_SEQ = (512, 2048), 32, 512


def time_ms(fn, iters=20, windows=5, warmup=3):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    out = []
    for _ in range(windows):
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        for _ in range(iters):
            fn()
        e.record()
        torch.cuda.synchronize()
        out.append(s.elapsed_time(e) / iters)
    return statistics.median(out), min(out), max(out)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else torch.cuda.get_device_name()


def attention(hd, S):
    from torch.nn.attention import SDPBackend, sdpa_kernel
    d, batch = HEADS * hd, TOKENS // S
    T = batch * S
    g = torch.Generator().manual_seed(hd + S)
    qkv = torch.randn(T, 3 * d, generator=g).to(torch.bfloat16).cuda()
    dout = torch.randn(T, d, generator=g).to(torch.bfloat16).cuda()
    out = torch.empty(T, d, dtype=torch.bfloat16, device="cuda")
    lse = torch.empty(T, HEADS, device="cuda")
    fwd = time_ms(lambda: K.attention_fwd(qkv, HEADS, out=out, lse=lse, seq_len=S))
    bwd = time_ms(lambda: K.attention_bwd(qkv, out, dout, lse, HEADS, seq_len=S))
    q, k, v = (t.transpose(1, 2) for t in qkv.view(batch, S, 3, HEADS, hd).unbind(2))   # [B, H, S, hd] views
    go = dout.view(batch, S, HEADS, hd).transpose(1, 2)
    qg, kg, vg = (t.detach().requires_grad_(True) for t in (q, k, v))

    def sdpa_fwd_bwd():
        o = torch.nn.functional.scaled_dot_product_attention(qg, kg, vg)
        torch.autograd.grad(o, (qg, kg, vg), go)

    with sdpa_kernel(SDPBackend.FLASH_ATTENTION):
        sdpa_fwd = time_ms(lambda: torch.nn.functional.scaled_dot_product_attention(q, k, v))
        sdpa_fb = time_ms(sdpa_fwd_bwd)
    flops = batch * HEADS * S * S * hd
    return dict(d_model=d, batch=batch, tokens=T, fwd_ms=fwd[0], fwd_ms_min_max=fwd[1:], fwd_tflops=4.0 * flops / fwd[0] / 1e9,
                bwd_ms=bwd[0], bwd_ms_min_max=bwd[1:], bwd_tflops=10.0 * flops / bwd[0] / 1e9,
                fwd_plus_bwd_ms=fwd[0] + bwd[0], sdpa_flash_fwd_ms=sdpa_fwd[0], sdpa_flash_fwd_tflops=4.0 * flops / sdpa_fwd[0] / 1e9,
                sdpa_flash_fwd_bwd_ms=sdpa_fb[0], sdpa_flash_fwd_bwd_tflops=14.0 * flops / sdpa_fb[0] / 1e9)


def train_step(d, native):
    from lah_b200.models.layers import name_to_block
    torch.manual_seed(0)
    layer = name_to_block["transformer"](d).cuda()
    be = lah_b200.ExpertBackend(name="t", expert=layer, opt=torch.optim.Adam(layer.parameters(), lr=1e-4, amsgrad=True),
                                args_schema=(lah_b200.BatchTensorProto(STEP_SEQ, d),),
                                outputs_schema=lah_b200.BatchTensorProto(STEP_SEQ, d), max_batch_size=STEP_BATCH, native=native)
    x = torch.randn(STEP_BATCH, STEP_SEQ, d, device="cuda")
    g = torch.randn(STEP_BATCH, STEP_SEQ, d, device="cuda") * 0.1
    ms = time_ms(lambda: be.backward(x, g), iters=20 if native else 5, warmup=3 if native else 2)
    executor = type(be._executor).__name__ if be._executor is not None else None
    assert executor == ("NativeTransformerExecutor" if native else None), executor
    return dict(step_ms=ms[0], step_ms_min_max=ms[1:], seqs_per_s=STEP_BATCH / ms[0] * 1e3)


if __name__ == "__main__":
    assert torch.cuda.is_available(), "this measurement needs a GPU"
    results = dict(card=card(), heads=HEADS, tokens=TOKENS, attention={}, train_step={})
    print(results["card"], flush=True)
    for hd in K.HEAD_DIMS:
        for S in SEQS:
            results["attention"][f"hd{hd}_S{S}"] = r = attention(hd, S)
            print("attention", hd, S, r, flush=True)
            torch.cuda.empty_cache()
    for d in STEP_WIDTHS:
        for native in (True, False):
            results["train_step"][f"d{d}_{'native' if native else 'eager'}"] = r = train_step(d, native)
            print("train_step", d, "native" if native else "eager", r, flush=True)
            torch.cuda.empty_cache()
    with open(output_path("attention_head_dim_perf.json"), "w") as f:
        json.dump(results, f, indent=1)
