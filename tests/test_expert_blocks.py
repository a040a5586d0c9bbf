"""The expert programs of ops/expert_blocks.py: on the CPU, with the kernels replaced by recorders, every weight gradient is
taken after the dgrad that reads the same weights (the caller may update them in place), and the plan alone picks the
GEMM; on the GPU, the FFN and SwiGLU experts of the DMoE trainer, the ExpertBackend executors and NativeFFNLayer compute
the bits of tests/golden/expert_block_digests.json (tools/expert_block_digests.py)."""
import json
import os

import pytest
import torch

import lah_b200  # noqa
from lah_b200.ops import expert_blocks as XB

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "expert_block_digests.json")


class Recorder:
    """stands in for a kernel module: every call is appended to ``log`` as (function name, args, kwargs)"""

    def __init__(self, log):
        self.log = log

    def __getattr__(self, name):
        return lambda *args, **kw: self.log.append((name, args, kw))


PLANS = {
    "swapab": XB.RowPlan(torch.zeros(2, dtype=torch.int32), torch.ones(1, dtype=torch.int32), None, 16, rows=16,
                         max_ctas=100),
    "tiles": XB.RowPlan(torch.zeros(2, dtype=torch.int32), None, torch.zeros(1, dtype=torch.int32)),
}


def _run(monkeypatch, plan, program):
    log = []
    monkeypatch.setattr(XB, "K", Recorder(log))
    monkeypatch.setattr(XB, "gemm", Recorder(log))
    weights = {n: f"weight {n}" for n in ("w1", "w2", "w3", "w13")}
    t = torch.zeros(32, 8)
    if program == "ffn":
        p = {n: None for n in ("b1", "b2", "b3", "g1", "be1", "g2", "be2")}
        XB.ffn_backward(plan, weights, p, dict(p), t, (t,) * 4, (t,) * 4, t, t, t, t, t,
                        lambda name, dy, x: log.append(("wgrad", (name,), {})))
        names = ("w3", "w2", "w1")
    else:
        XB.swiglu_mlp_backward(plan, weights["w13"], weights["w2"], t, t, t, t, t, t, t,
                               lambda name, dy, x: log.append(("wgrad", (name,), {})))
        names = ("w2", "w13")
    return log, weights, names


@pytest.mark.parametrize("plan", sorted(PLANS))
@pytest.mark.parametrize("program", ["ffn", "swiglu"])
def test_each_wgrad_follows_the_dgrad_of_its_weights(monkeypatch, plan, program):
    log, weights, names = _run(monkeypatch, PLANS[plan], program)
    gemm = "swapab_linear" if plan == "swapab" else "grouped_linear"
    dgrads = {args[1]: i for i, (fn, args, kw) in enumerate(log) if kw.get("w_is_kn")}
    wgrads = [(i, args[0]) for i, (fn, args, _) in enumerate(log) if fn == "wgrad"]
    assert [name for _, name in wgrads] == list(names)
    assert len(dgrads) == len(names)
    for i, name in wgrads:
        assert dgrads[weights[name]] < i, (name, log)
    for fn, args, kw in log:
        if kw.get("w_is_kn"):
            assert fn == gemm and kw["max_ctas"] == PLANS[plan].max_ctas


@pytest.mark.gpu
def test_expert_programs_match_the_golden_digests():
    from tools import expert_block_digests
    with open(GOLDEN) as f:
        golden = json.load(f)
    assert expert_block_digests.compute() == golden
