"""GPU timing of the transformer expert over sequence lengths (writes check_out/attention_seq_len_perf.json).

For S in {128, 256, 512, 1000, 1024, 2048, 4096} at a fixed ~16,384 tokens (batch = 16384 // S sequences), d_model 1024 and
16 heads:
  * attention forward and backward without dropout, CUDA events, TFLOP/s from the flop counts of gpu_attention_check.py
    (forward 4 B H S^2 64, backward 10 B H S^2 64; a partial last block is not counted);
  * the default expert (dropout 0.1) trained through ExpertBackend: one backward task = forward recompute, backward and
    AMSGrad step, in sequences/s.
Each number is the median of 5 windows of 20 calls (10 for the training step) after a warm-up.  The card's name and power
limit are read in the same run.
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

SEQS = (128, 256, 512, 1000, 1024, 2048, 4096)
TOKENS, D, HEADS = 16384, 1024, 16


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


def attention(S):
    batch = TOKENS // S
    T = batch * S
    g = torch.Generator().manual_seed(S)
    qkv = torch.randn(T, 3 * D, generator=g).to(torch.bfloat16).cuda()
    dout = torch.randn(T, D, generator=g).to(torch.bfloat16).cuda()
    out = torch.empty(T, D, dtype=torch.bfloat16, device="cuda")
    lse = torch.empty(T, HEADS, device="cuda")
    fwd = time_ms(lambda: K.attention_fwd(qkv, HEADS, out=out, lse=lse, seq_len=S))
    bwd = time_ms(lambda: K.attention_bwd(qkv, out, dout, lse, HEADS, seq_len=S))
    flops = batch * HEADS * S * S * 64
    return dict(batch=batch, tokens=T, fwd_ms=fwd[0], fwd_ms_min_max=fwd[1:], fwd_tflops=4.0 * flops / fwd[0] / 1e9,
                bwd_ms=bwd[0], bwd_ms_min_max=bwd[1:], bwd_tflops=10.0 * flops / bwd[0] / 1e9)


def train_step(S):
    from lah_b200.models.layers import name_to_block
    batch = TOKENS // S
    torch.manual_seed(0)
    layer = name_to_block["transformer"](D).cuda()
    be = lah_b200.ExpertBackend(name="t", expert=layer, opt=torch.optim.Adam(layer.parameters(), lr=1e-4, amsgrad=True),
                                args_schema=(lah_b200.BatchTensorProto(S, D),), outputs_schema=lah_b200.BatchTensorProto(S, D),
                                max_batch_size=batch)
    x = torch.randn(batch, S, D, device="cuda")
    g = torch.randn(batch, S, D, device="cuda") * 0.1
    ms = time_ms(lambda: be.backward(x, g), iters=10)
    assert type(be._executor).__name__ == "NativeTransformerExecutor"
    return dict(batch=batch, step_ms=ms[0], step_ms_min_max=ms[1:], seqs_per_s=batch / ms[0] * 1e3)


if __name__ == "__main__":
    assert torch.cuda.is_available(), "this measurement needs a GPU"
    results = dict(card=card(), d_model=D, heads=HEADS, tokens=TOKENS, attention={}, train_step={})
    print(results["card"], flush=True)
    for S in SEQS:
        results["attention"][S] = attention(S)
        print("attention", S, results["attention"][S], flush=True)
    for S in SEQS:
        results["train_step"][S] = train_step(S)
        print("train_step", S, results["train_step"][S], flush=True)
        torch.cuda.empty_cache()
    with open(output_path("attention_seq_len_perf.json"), "w") as f:
        json.dump(results, f, indent=1)
