"""SHA-256 digests of what the FFN and SwiGLU expert programs compute, through public APIs only:

- 3-step ``DMoETrainer`` runs (the third step replays the captured graph) on the small and big expert paths, FFN (bf16
  and MXFP8) and SwiGLU experts, the shared expert on both sides of its 512-row GEMM switch, failure injection and two
  micro-batches: every step's loss, every layer's expert parameters and AMSGrad state, the trainer parameters and their
  state, and the kernel launches of one replay;
- ``ExpertBackend`` on the FFN and gated-FFN executors at row counts that need padding: 3 backward calls each, with Adam
  and with a two-group AdamW that puts w1 and w3 in different groups;
- the forward of ``NativeFFNLayer`` in bf16 and MXFP8.

tests/golden/expert_block_digests.json holds the digests; tests/test_expert_blocks.py recomputes them, so a change of a
single bit in these programs fails there.  A change that means to alter these bits regenerates the file:

    python tools/expert_block_digests.py OUT.json      # needs a GPU; computes everything twice and checks it is repeatable
"""
import hashlib
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

import lah_b200  # noqa

BENCH = dict(hidden=512, grid_size=(16,), k=4, num_layers=2, tokens_per_rank=256, gate_mode="emulator", lr=1e-3)
TRAINER_RUNS = {
    "ffn_small": dict(expert_path="small"),
    "ffn_big": dict(expert_path="big"),
    "ffn_big_fp8": dict(expert_path="big", expert_dtype="fp8"),
    "swiglu_small": dict(expert="swiglu", expert_path="small"),
    "swiglu_big": dict(expert="swiglu", expert_path="big"),
    "swiglu_shared_256": dict(expert="swiglu", expert_path="small", shared_inner_dim=1408),
    "swiglu_shared_640": dict(expert="swiglu", expert_path="big", shared_inner_dim=1408, tokens_per_rank=640),
    "ffn_small_failures": dict(expert_path="small", failure_rate=0.1),
    "swiglu_shared_microbatches": dict(expert="swiglu", expert_path="small", shared_inner_dim=1408,
                                       trainer_microbatches=2),
}
BACKEND_ROWS = (37, 300)


def sha(*tensors):
    h = hashlib.sha256()
    for t in tensors:
        t = t.detach().contiguous().cpu()
        h.update(f"{t.dtype}{tuple(t.shape)}".encode())
        h.update(t.reshape(-1).view(torch.uint8).numpy().tobytes())
    return h.hexdigest()


def trainer_run(index, name, kw):
    from lah_b200.parallel.engine import DMoEConfig
    from lah_b200.parallel.trainer import DMoETrainer
    cfg = DMoEConfig(**{**BENCH, **kw})
    B = cfg.tokens_per_rank
    gen = torch.Generator().manual_seed(100 + index)
    xs = [torch.randn(B, cfg.in_features, generator=gen).cuda() for _ in range(3)]
    ys = [torch.randint(0, cfg.num_classes, (B,), generator=gen).cuda() for _ in range(3)]
    t = DMoETrainer(cfg, use_graph=True)
    losses = torch.stack([t.train_step_device(x, y).clone() for x, y in zip(xs, ys)])
    assert t._graph is not None
    t.ctx.check_status()
    out = {f"{name}_loss": sha(losses), f"{name}_launches": int(t._graph_launches),
           f"{name}_trainer": sha(t.flat_p, t.flat_m, t.flat_v, t.flat_vmax)}
    for i, b in enumerate(t.model.blocks):
        sh = b.shard
        out[f"{name}_layer{i}_expert"] = sha(sh.p, sh.m, sh.v, sh.vmax)
    t.close()
    return out


def _ffn_opt(m):
    return torch.optim.Adam(m.parameters(), lr=1e-3, amsgrad=True)


def _gated_opt(m):
    """two AdamW groups; w1 and w3 in different ones, so [W1; W3] takes two fused wgrad + AMSGrad launches"""
    opt = torch.optim.AdamW([dict(params=[m.norm.weight, m.w1.weight]), dict(params=[m.w3.weight, m.w2.weight])],
                            lr=1e-3, amsgrad=True, weight_decay=0.01)
    opt.param_groups[1].update(lr=2e-4, amsgrad=False, weight_decay=0.1)
    return opt


def backend_run(name, make, make_opt, executor, rows):
    torch.manual_seed(11)
    module = make().cuda()
    hid = 512
    opt = make_opt(module)
    be = lah_b200.ExpertBackend(name=name, expert=module, opt=opt, args_schema=(lah_b200.BatchTensorProto(hid),),
                                outputs_schema=lah_b200.BatchTensorProto(hid), max_batch_size=4096)
    gen = torch.Generator().manual_seed(rows)
    ys, dxs = [], []
    for _ in range(3):
        x = torch.randn(rows, hid, generator=gen).cuda()
        g = (torch.randn(rows, hid, generator=gen) * 0.1).cuda()
        (y,) = be.forward(x)
        (dx,) = be.backward(x, g)
        ys.append(y)
        dxs.append(dx)
    assert type(be._executor).__name__ == executor, be._executor
    state = [t for st in opt.state_dict()["state"].values() for _, t in sorted(st.items())]
    return {f"{name}_{rows}_y": sha(*ys), f"{name}_{rows}_dx": sha(*dxs),
            f"{name}_{rows}_params": sha(*[v for _, v in sorted(module.state_dict().items())]),
            f"{name}_{rows}_opt_state": sha(*state)}


def ffn_layer_run(dtype):
    from lah_b200.models.ffn_native import NativeFFNLayer
    from lah_b200.models.layers import FeedforwardBlock
    torch.manual_seed(5)
    block = FeedforwardBlock(512).cuda().eval()
    x = torch.randn(512, 512, generator=torch.Generator().manual_seed(5)).to(torch.bfloat16).cuda()
    return {f"ffn_native_{dtype}": sha(NativeFFNLayer(block, dtype=dtype)(x))}


def compute():
    from lah_b200.models.layers import FeedforwardBlock, GatedFeedforwardBlock
    out = {}
    for index, (name, kw) in enumerate(TRAINER_RUNS.items()):
        out.update(trainer_run(index, name, kw))
    for rows in BACKEND_ROWS:
        out.update(backend_run("ffn", lambda: FeedforwardBlock(512), _ffn_opt, "NativeFFNExecutor", rows))
        out.update(backend_run("gated", lambda: GatedFeedforwardBlock(512, 1408), _gated_opt, "NativeGatedFFNExecutor",
                               rows))
    for dtype in ("bf16", "fp8"):
        out.update(ffn_layer_run(dtype))
    torch.cuda.synchronize()
    return out


if __name__ == "__main__":
    first, second = compute(), compute()
    assert first == second, "the digests are not repeatable"
    with open(sys.argv[1], "w") as f:
        json.dump(first, f, indent=1, sort_keys=True)
        f.write("\n")
    print(json.dumps(first, indent=1, sort_keys=True))
