"""
Convergence experiment runner — script form of the three reference notebooks
(/root/reference/experiments/convergence/*.ipynb, cells 1-4): `num_trainers` asynchronous trainers share one model;
each computes gradients of the NON-expert parameters, sleeps `delay_ms * Weibull(1)` (emulated network latency) and then
applies its — by now stale — gradients; experts update themselves inside the emulated DMoE layer.  Metrics
(`train_history` = {loss, delay_steps}, `val_history` = {loss, acc, num_updates}) are pickled to
`logs/delay{ms}ms_dmoe{k}outof{E}experts_seed{seed}.pkl` exactly like the notebooks.

Setups (README.md:51-65 grid):  --setup dmoe | faulty | largeffn

Data: MNIST is not available offline, so a synthetic MNIST-shaped task is used (784-d inputs, 10 classes, class
prototypes + noise; deterministic per seed).  Works on CPU (BASELINE config #1: 16 experts x 4 layers, 2 trainers) and
on a GPU (`--device cuda`).  `--backend engine` trains the same model on the sm_90a engine (synchronous trainers).
"""
import os
import pickle
import random
import threading
import time
from argparse import ArgumentParser
from functools import partial

import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F

from ...models import EmulatedDMoE, EmulatedFaultyDMoE, FeedforwardBlock, get_non_expert_params


class SyntheticMNIST:
    """10 Gaussian class prototypes in 784-d (+ structured noise); train/test splits are different noise draws"""

    def __init__(self, seed=0, in_features=784, num_classes=10, noise=3.0, device="cpu"):
        gen = torch.Generator().manual_seed(seed)
        self.prototypes = torch.randn(num_classes, in_features, generator=gen)
        self.noise, self.num_classes, self.in_features, self.device = noise, num_classes, in_features, device

    def batch(self, batch_size, generator):
        y = torch.randint(0, self.num_classes, (batch_size,), generator=generator)
        x = self.prototypes[y] + self.noise * torch.randn(batch_size, self.in_features, generator=generator)
        return x.to(self.device), y.to(self.device)


def build_model(args, device):
    Optimizer = partial(torch.optim.Adam, lr=args.lr, amsgrad=True)
    if args.setup == "largeffn":
        blocks = [FeedforwardBlock(args.layer_dim) for _ in range(args.num_blocks)]
        dmoe_types = ()
    else:
        def make():
            common = dict(num_experts=args.num_experts, num_active=args.num_active, update_every_inputs=args.batch_size,
                          update_every_steps=args.update_every_steps, Expert=FeedforwardBlock, Optimizer=Optimizer)
            if args.setup == "faulty":
                return EmulatedFaultyDMoE(args.layer_dim, failure_rate=args.failure_rate, **common)
            return EmulatedDMoE(args.layer_dim, **common)
        blocks = [make() for _ in range(args.num_blocks)]
        dmoe_types = (EmulatedDMoE,)
    model = nn.Sequential(nn.Linear(args.in_features, args.layer_dim), *blocks, nn.LayerNorm(args.layer_dim),
                          nn.Linear(args.layer_dim, args.num_classes)).to(device)
    params = get_non_expert_params(model, dmoe_types) if dmoe_types else list(model.parameters())
    return model, params, Optimizer(params)


def evaluate(model, data, args, lock):
    gen = torch.Generator().manual_seed(args.seed + 10_000)
    with lock, torch.no_grad():
        model.train(False)
        loss_sum = acc_sum = count = 0.0
        for _ in range(args.eval_batches):
            xb, yb = data.batch(args.eval_batch_size, gen)
            logits = model(xb)
            loss_sum += F.cross_entropy(logits, yb).item() * len(yb)
            acc_sum += (logits.argmax(-1) == yb).float().sum().item()
            count += len(yb)
    return dict(loss=loss_sum / count, acc=acc_sum / count)


def run(args, printer=print):
    torch.manual_seed(args.seed), np.random.seed(args.seed), random.seed(args.seed)
    device = torch.device(args.device)
    data = SyntheticMNIST(args.seed, args.in_features, args.num_classes, device=device)
    if args.backend == "engine":
        return run_engine(args, data, printer)
    model, params, opt = build_model(args, device)
    # create initial gradients (notebook cell 2) so that stale gradients can always be written back in place
    model(torch.zeros(1, args.in_features, device=device)).sum().backward()
    opt.zero_grad(set_to_none=False)
    lock, need_eval, done = threading.Lock(), threading.Event(), threading.Event()
    train_history, val_history = [], []

    def trainer(index):
        gen = torch.Generator().manual_seed(args.seed * 1000 + index)
        while not done.is_set():
            xb, yb = data.batch(args.batch_size, gen)
            with lock:
                model.train(True)
                start_step = len(train_history)
                loss = F.cross_entropy(model(xb), yb)
                opt.zero_grad(set_to_none=False)
                loss.backward()
                grads = [p.grad.clone() if p.grad is not None else None for p in params]
            if args.delay_ms:
                time.sleep(args.delay_ms / 1000.0 * np.random.weibull(1))  # emulated network latency
            with lock:
                if done.is_set():
                    return
                model.train(True)
                opt.zero_grad(set_to_none=False)
                for p, g in zip(params, grads):
                    if g is not None:
                        p.grad[...] = g  # stale gradient
                opt.step()
                train_history.append(dict(loss=loss.item(), delay_steps=len(train_history) - start_step))
                n = len(train_history)
                if n % args.eval_interval == 0 or n >= args.total_steps:
                    need_eval.set()
                if n >= args.total_steps:
                    done.set()

    threads = [threading.Thread(target=trainer, args=(i,), daemon=True) for i in range(args.num_trainers)]
    t0 = time.time()
    [t.start() for t in threads]
    while not done.is_set() or need_eval.is_set():
        if not need_eval.wait(timeout=0.5):
            continue
        need_eval.clear()
        metrics = evaluate(model, data, args, lock)
        metrics["num_updates"] = len(train_history)
        val_history.append(metrics)
        last = train_history[-1]
        printer(f"#{metrics['num_updates']}\tloss={last['loss']:.4f}\tdelay={last['delay_steps']}\t"
                f"val_loss={metrics['loss']:.4f}\tval_acc={metrics['acc']:.4f}")
    [t.join(timeout=5) for t in threads]
    elapsed = time.time() - t0
    result = dict(train_history=train_history, val_history=val_history, updates_per_sec=len(train_history) / elapsed,
                  samples_per_sec=len(train_history) * args.batch_size / elapsed)
    save_history(args, result)
    printer(f"{len(train_history)} updates in {elapsed:.1f}s = {result['updates_per_sec']:.2f} updates/s "
            f"= {result['samples_per_sec']:.1f} samples/s")
    return result


def run_engine(args, data, printer):
    """same model on the in-box engine (synchronous: one fused step per batch of num_trainers * batch_size samples)"""
    from ...parallel.engine import DMoEConfig
    from ...parallel.trainer import DMoETrainer
    side = int(round(args.num_experts ** 0.5))
    assert side * side == args.num_experts, "--backend engine needs a square number of experts (product-key grid)"
    batch = args.num_trainers * args.batch_size
    cfg = DMoEConfig(hidden=args.layer_dim, grid_size=(side, side), k=args.num_active, num_layers=args.num_blocks,
                     in_features=args.in_features, num_classes=args.num_classes, tokens_per_rank=max(batch, args.eval_batch_size),
                     failure_rate=args.failure_rate if args.setup == "faulty" else 0.0, lr=args.lr, seed=args.seed)
    trainer = DMoETrainer(cfg)
    gen = torch.Generator().manual_seed(args.seed)
    train_history, val_history, t0 = [], [], time.time()
    steps = args.total_steps // max(1, args.num_trainers)
    for step in range(1, steps + 1):
        xb, yb = data.batch(batch, gen)
        loss = trainer.train_step(xb.cpu(), yb.cpu())
        train_history.append(dict(loss=loss, delay_steps=0))
        if step % max(1, args.eval_interval // args.num_trainers) == 0 or step == steps:
            egen = torch.Generator().manual_seed(args.seed + 10_000)
            xe, ye = data.batch(args.eval_batch_size, egen)
            metrics = trainer.evaluate(xe, ye)
            metrics["num_updates"] = step * args.num_trainers
            val_history.append(metrics)
            printer(f"#{metrics['num_updates']}\tloss={loss:.4f}\tval_loss={metrics['loss']:.4f}\tval_acc={metrics['acc']:.4f}")
    elapsed = time.time() - t0
    result = dict(train_history=train_history, val_history=val_history, updates_per_sec=steps / elapsed,
                  samples_per_sec=steps * batch / elapsed)
    printer(f"{steps} fused steps ({steps * args.num_trainers} trainer updates) in {elapsed:.1f}s = "
            f"{result['samples_per_sec']:.1f} samples/s")
    save_history(args, result)
    return result


def save_history(args, result):
    if not args.logdir:
        return
    os.makedirs(args.logdir, exist_ok=True)
    if args.setup == "largeffn":
        name = f"delay{args.delay_ms}ms_largeffn_seed{args.seed}.pkl"
    else:
        name = f"delay{args.delay_ms}ms_dmoe{args.num_active}outof{args.num_experts}experts_seed{args.seed}.pkl"
    with open(os.path.join(args.logdir, name), "wb") as f:
        pickle.dump(dict(train_history=result["train_history"], val_history=result["val_history"]), f)


def make_parser():
    p = ArgumentParser()
    p.add_argument("--setup", choices=["dmoe", "faulty", "largeffn"], default="dmoe")
    p.add_argument("--backend", choices=["emulator", "engine"], default="emulator")
    p.add_argument("--seed", type=int, default=1337)
    p.add_argument("--device", default="cuda" if torch.cuda.is_available() else "cpu")
    p.add_argument("--layer-dim", type=int, default=512)
    p.add_argument("--num-blocks", type=int, default=4)
    p.add_argument("--num-experts", type=int, default=64)
    p.add_argument("--num-active", type=int, default=4)
    p.add_argument("--batch-size", type=int, default=4)
    p.add_argument("--num-trainers", type=int, default=64)
    p.add_argument("--delay-ms", type=int, default=1000)
    p.add_argument("--failure-rate", type=float, default=0.1)
    p.add_argument("--eval-interval", type=int, default=1024)
    p.add_argument("--total-steps", type=int, default=1024 * 20)
    p.add_argument("--update-every-steps", type=int, default=10)
    p.add_argument("--lr", type=float, default=1e-3)
    p.add_argument("--in-features", type=int, default=28 ** 2)
    p.add_argument("--num-classes", type=int, default=10)
    p.add_argument("--eval-batches", type=int, default=8)
    p.add_argument("--eval-batch-size", type=int, default=256)
    p.add_argument("--logdir", default="logs")
    return p


if __name__ == "__main__":
    run(make_parser().parse_args())
