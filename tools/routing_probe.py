"""GPU probe: how does expert routing evolve while the flagship model trains on synthetic data?  (run on the GPU)

Prints, per step and DMoE layer: active experts, share of the hottest expert, and the per-rank load imbalance
(max / mean padded rows) that an 8-way expert-parallel placement would see.  `--labels teacher` draws labels from a fixed
random linear teacher (learnable, MNIST-like: the label is a function of the input); `random` = i.i.d. labels."""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

import lah_b200  # noqa
from lah_b200.parallel.engine import DMoEConfig
from lah_b200.parallel.trainer import DMoETrainer


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=16384)
    ap.add_argument("--steps", type=int, default=40)
    ap.add_argument("--labels", default="teacher")
    ap.add_argument("--gate", default="emulator")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    cfg = DMoEConfig(hidden=512, grid_size=(64,) if args.gate == "emulator" else (8, 8), k=4, num_layers=4,
                     tokens_per_rank=args.batch, gate_mode=args.gate)
    tr = DMoETrainer(cfg)
    gen = torch.Generator().manual_seed(0)
    teacher = torch.randn(784, 10, generator=gen)
    rows = []
    for step in range(args.steps):
        x = torch.randn(args.batch, 784, generator=gen)
        y = (x @ teacher).argmax(-1) if args.labels == "teacher" else torch.randint(0, 10, (args.batch,), generator=gen)
        loss = float(tr.train_step_device(x.cuda(), y.cuda()))
        rec = dict(step=step, loss=round(loss, 4), layers=[])
        for block in tr.model.blocks:
            r = block.ws.step_rows.float().cpu()
            per_rank = r.view(8, -1).sum(1)
            rec["layers"].append(dict(active=int((r > 0).sum()), top_share=round(float(r.max() / r.sum()), 3),
                                      imb8=round(float(per_rank.max() / per_rank.mean()), 2)))
        rows.append(rec)
        if step % 4 == 0 or step == args.steps - 1:
            print(json.dumps(rec), flush=True)
    if args.out:
        json.dump(rows, open(args.out, "w"))


if __name__ == "__main__":
    main()
