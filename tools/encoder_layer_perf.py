"""GPU timing of torch.nn.TransformerEncoderLayer and TorchScript experts behind ExpertBackend, native against eager
(writes check_out/encoder_layer_perf.json).

d_model 1024, 16 heads, dim_feedforward 2048, dropout 0.1, 32 sequences of 512 tokens; experts:
  * nn.TransformerEncoderLayer(1024, 16, batch_first=True)                    (ReLU, post-LN: torch's defaults)
  * the same with norm_first=True                                            (pre-LN)
  * the same with activation="gelu"
  * torch.jit.script(name_to_block["transformer"](1024))                     (how the reference builds its experts)
For each, one ExpertBackend.backward (forward recompute + backward + AMSGrad) and one ExpertBackend.forward in training
mode, with the sm_90a executor and with native=False (the module itself, fp32 eager).  Each number is the median of 5
windows of 20 calls (5 for eager) after a warm-up, CUDA events.  The card's name and power limit are read in the same run.
"""
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from torch import nn

import lah_b200  # noqa
from tools import output_path
from tools.attention_head_dim_perf import card, time_ms

D, HEADS, BATCH, SEQ = 1024, 16, 32, 512
EXPERTS = {
    "torch relu post-LN": lambda: nn.TransformerEncoderLayer(D, HEADS, batch_first=True),
    "torch relu pre-LN": lambda: nn.TransformerEncoderLayer(D, HEADS, batch_first=True, norm_first=True),
    "torch gelu post-LN": lambda: nn.TransformerEncoderLayer(D, HEADS, batch_first=True, activation="gelu"),
    "scripted name_to_block": lambda: torch.jit.script(_own_block()),
}


def _own_block():
    from lah_b200.models.layers import name_to_block
    return name_to_block["transformer"](D)


def measure(make, native):
    torch.manual_seed(0)
    module = make().cuda()
    be = lah_b200.ExpertBackend(name="t", expert=module, opt=torch.optim.Adam(module.parameters(), lr=1e-4, amsgrad=True),
                                args_schema=(lah_b200.BatchTensorProto(SEQ, D),), outputs_schema=lah_b200.BatchTensorProto(SEQ, D),
                                max_batch_size=BATCH, native=native)
    x = torch.randn(BATCH, SEQ, D, device="cuda")
    g = torch.randn(BATCH, SEQ, D, device="cuda") * 0.1
    iters, warmup = (20, 3) if native else (5, 2)
    bwd = time_ms(lambda: be.backward(x, g), iters=iters, warmup=warmup)
    fwd = time_ms(lambda: be.forward(x), iters=iters, warmup=warmup)
    executor = type(be._executor).__name__ if be._executor is not None else None
    assert executor == ("NativeTransformerExecutor" if native else None), executor
    return dict(backward_ms=bwd[0], backward_ms_min_max=bwd[1:], forward_ms=fwd[0], forward_ms_min_max=fwd[1:])


if __name__ == "__main__":
    assert torch.cuda.is_available(), "this measurement needs a GPU"
    results = dict(card=card(), d_model=D, heads=HEADS, batch=BATCH, seq=SEQ, dropout=0.1, experts={})
    print(results["card"], flush=True)
    for name, make in EXPERTS.items():
        for native in (True, False):
            results["experts"][f"{name} / {'native' if native else 'eager'}"] = r = measure(make, native)
            print(name, "native" if native else "eager", r, flush=True)
            torch.cuda.empty_cache()
    with open(output_path("encoder_layer_perf.json"), "w") as f:
        json.dump(results, f, indent=1)
