"""Generates the three convergence notebooks (experiments/convergence/*.ipynb) — same names, configurations and metric
files as the reference notebooks (/root/reference/experiments/convergence/*.ipynb, cells 1-4), written against this package:
config cell -> data / model -> asynchronous trainer threads with stale gradients -> evaluation curve + metrics pickle ->
the same experiment on the sm_90a engine.  `LAH_NB_SMOKE=1` shrinks every size so that tests can execute the cells on CPU.

    python tools/make_notebooks.py
"""
import json
import os

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT = os.path.join(ROOT, "learning-at-home_b200", "experiments", "convergence")

SETUPS = {
    "convergence_mnist_64workers_1000ms_seed1337_dmoe64x4.ipynb": dict(
        title="DMoE, 64 experts x 4 layers, top-4, 64 trainers x batch 4, 1000 ms delay, seed 1337",
        ref_lines="config: raw lines 35-53; trainer loop: 146-191; evaluation: 194-215; metrics pickle: 250-263",
        setup="dmoe", seed=1337, layer_dim=512, num_blocks=4, num_experts=64, num_active=4, batch_size=4, num_trainers=64,
        delay_ms=1000, failure_rate=0.0, device="'cuda' if torch.cuda.is_available() else 'cpu'"),
    "convergence_mnist_64workers_1000ms_seed1337_largeffn.ipynb": dict(
        title="Large FFN baseline (hid 1024, 4 blocks), 64 trainers x batch 4, 1000 ms delay, seed 1337",
        ref_lines="config: raw lines 35-51; trainer loop: 134-179",
        setup="largeffn", seed=1337, layer_dim=1024, num_blocks=4, num_experts=0, num_active=0, batch_size=4, num_trainers=64,
        delay_ms=1000, failure_rate=0.0, device="'cuda' if torch.cuda.is_available() else 'cpu'"),
    "convergence_mnist_fail01_64workers_1000ms_seed1338_dmoe1024x4_cpu.ipynb": dict(
        title="Faulty DMoE, 1024 experts x 4 layers (4096 experts), 10 % expert failures, top-4, 64 trainers x batch 8, 1000 ms "
              "delay, seed 1338 (the reference ran this one on 48 CPU threads)",
        ref_lines="environment: raw lines 12-20; config: 48-67; trainer loop: 161-206",
        setup="faulty", seed=1338, layer_dim=512, num_blocks=4, num_experts=1024, num_active=4, batch_size=8, num_trainers=64,
        delay_ms=1000, failure_rate=0.1, device="'cpu'"),
}


def md(text):
    return dict(cell_type="markdown", metadata={}, source=text.splitlines(keepends=True))


def code(text):
    return dict(cell_type="code", metadata={}, execution_count=None, outputs=[], source=text.strip("\n").splitlines(keepends=True))


def build(name, s):
    cells = [md(f"""# {s['title']}

Counterpart of `/root/reference/experiments/convergence/{name}` ({s['ref_lines']}).

`num_trainers` asynchronous trainers share one model: each one computes the gradients of the NON-expert parameters under a
lock, sleeps `delay_ms * Weibull(1)` (emulated network latency) and then applies its — by now stale — gradients; experts
update themselves inside the emulated DMoE layer once they have seen `update_every_inputs` inputs or `update_every_steps`
steps.  MNIST is not available offline: the data is a synthetic MNIST-shaped task (784-d inputs, 10 classes, class
prototypes + noise).  The last section trains the same model on the sm_90a engine (`DMoETrainer`, stale trainer gradients
through `DMoEConfig.trainer_staleness`).  `LAH_NB_SMOKE=1` runs a tiny version of every cell.""")]
    cells.append(code(f"""
import os, sys, time, pickle, random, threading
sys.path.insert(0, os.path.abspath(os.path.join(os.getcwd(), '..', '..', '..')) if '__file__' not in globals() else os.getcwd())
import numpy as np
import torch, torch.nn as nn, torch.nn.functional as F
import lah_b200
from lah_b200.experiments.convergence.run import SyntheticMNIST, build_model, make_parser, save_history

SMOKE = bool(os.environ.get('LAH_NB_SMOKE'))
# ---- experiment constants (reference notebook configuration cell)
seed = {s['seed']}
setup = '{s['setup']}'
layer_dim, num_blocks = {s['layer_dim']}, {s['num_blocks']}
num_experts, num_active = {s['num_experts']}, {s['num_active']}
batch_size, num_trainers = {s['batch_size']}, {s['num_trainers']}
delay_ms, failure_rate = {s['delay_ms']}, {s['failure_rate']}
update_every_steps = 10
eval_interval, total_steps = 1024, 1024 * 20
device = torch.device({s['device']})
if SMOKE:
    layer_dim, num_blocks, num_experts, num_trainers = 16, 2, (4 if num_experts else 0), 2
    num_active = 2 if num_experts else 0
    delay_ms, eval_interval, total_steps, device = 1, 3, 6, torch.device('cpu')
args = make_parser().parse_args(['--setup', setup, '--seed', str(seed), '--layer-dim', str(layer_dim), '--num-blocks', str(num_blocks),
                                 '--num-experts', str(max(num_experts, 1)), '--num-active', str(max(num_active, 1)),
                                 '--batch-size', str(batch_size), '--num-trainers', str(num_trainers), '--delay-ms', str(delay_ms),
                                 '--failure-rate', str(failure_rate), '--update-every-steps', str(update_every_steps),
                                 '--device', str(device), '--logdir', os.environ.get('LAH_NB_LOGDIR', 'logs')])
torch.manual_seed(seed); np.random.seed(seed); random.seed(seed)
"""))
    cells.append(code("""
# ---- data and model: Linear(784, layer_dim) -> num_blocks x (EmulatedDMoE | EmulatedFaultyDMoE | FeedforwardBlock) -> LayerNorm -> Linear(10)
data = SyntheticMNIST(seed, 28 ** 2, 10, device=device)
model, trainer_params, opt = build_model(args, device)     # Adam(lr=1e-3, amsgrad=True) for the trainer AND for every expert
print(sum(p.numel() for p in model.parameters()) / 1e6, 'M parameters;', len(trainer_params), 'trainer-side tensors')
model(torch.zeros(1, 28 ** 2, device=device)).sum().backward()   # materialise .grad so stale gradients can be written in place
opt.zero_grad(set_to_none=False)
"""))
    cells.append(code("""
# ---- asynchronous trainers with stale gradients (reference cell 3)
lock, need_eval, done = threading.Lock(), threading.Event(), threading.Event()
train_history, val_history = [], []

def evaluate(num_batches=2 if SMOKE else 8, eval_batch=16 if SMOKE else 256):
    gen = torch.Generator().manual_seed(seed + 10_000)
    with lock, torch.no_grad():
        model.train(False)
        loss = acc = count = 0.0
        for _ in range(num_batches):
            xb, yb = data.batch(eval_batch, gen)
            logits = model(xb)
            loss += F.cross_entropy(logits, yb).item() * len(yb); acc += (logits.argmax(-1) == yb).float().sum().item(); count += len(yb)
    return dict(loss=loss / count, acc=acc / count)

def trainer_thread(index):
    gen = torch.Generator().manual_seed(seed * 1000 + index)
    while not done.is_set():
        xb, yb = data.batch(batch_size, gen)
        with lock:                                   # forward + backward under the lock, keep a copy of the trainer gradients
            model.train(True)
            started_at = len(train_history)
            loss = F.cross_entropy(model(xb), yb)
            opt.zero_grad(set_to_none=False)
            loss.backward()
            grads = [p.grad.clone() if p.grad is not None else None for p in trainer_params]
        time.sleep(delay_ms / 1000.0 * np.random.weibull(1))       # emulated network latency
        with lock:                                   # ... and apply them, stale by however many updates happened meanwhile
            if done.is_set():
                return
            opt.zero_grad(set_to_none=False)
            for p, g in zip(trainer_params, grads):
                if g is not None:
                    p.grad[...] = g
            opt.step()
            train_history.append(dict(loss=loss.item(), delay_steps=len(train_history) - started_at))
            n = len(train_history)
            if n % eval_interval == 0 or n >= total_steps: need_eval.set()
            if n >= total_steps: done.set()

threads = [threading.Thread(target=trainer_thread, args=(i,), daemon=True) for i in range(num_trainers)]
t0 = time.time(); [t.start() for t in threads]
while not done.is_set() or need_eval.is_set():
    if not need_eval.wait(timeout=0.5): continue
    need_eval.clear()
    metrics = dict(evaluate(), num_updates=len(train_history)); val_history.append(metrics)
    print(f"#{metrics['num_updates']}\\tloss={train_history[-1]['loss']:.4f}\\tdelay={train_history[-1]['delay_steps']}\\tval_acc={metrics['acc']:.4f}")
[t.join(timeout=5) for t in threads]
elapsed = time.time() - t0
print(f"{len(train_history)} updates in {elapsed:.1f}s = {len(train_history) / elapsed:.2f} updates/s = {len(train_history) * batch_size / elapsed:.1f} samples/s")
"""))
    cells.append(code("""
# ---- metrics file (same name and layout as the reference: dict(train_history, val_history)) and the accuracy curve
result = dict(train_history=train_history, val_history=val_history)
save_history(args, result)
try:
    import matplotlib.pyplot as plt
    fig, ax = plt.subplots(1, 2, figsize=(12, 4))
    ax[0].plot([v['num_updates'] for v in val_history], [v['acc'] for v in val_history]); ax[0].set_xlabel('updates'); ax[0].set_ylabel('validation accuracy'); ax[0].grid()
    ax[1].plot([h['delay_steps'] for h in train_history]); ax[1].set_xlabel('update'); ax[1].set_ylabel('gradient staleness (updates)'); ax[1].grid()
except ImportError:                                   # no matplotlib on this image: print the curve
    for v in val_history: print(v['num_updates'], round(v['acc'], 4), round(v['loss'], 4))
mean_delay = float(np.mean([h['delay_steps'] for h in train_history]))
print('final val acc', val_history[-1]['acc'], '| mean staleness', round(mean_delay, 1), 'updates')
"""))
    if s["setup"] != "largeffn":
        cells.append(md("""## The same experiment on the sm_90a engine

One `DMoETrainer` per GPU: the 64 trainers x batch become ONE fused step of `num_trainers * batch_size` samples, experts step
themselves after every backward (fused wgrad + AMSGrad kernel), the trainer-side optimizer applies gradients that are
`trainer_staleness` steps old (the measured mean staleness above divided by the number of trainers folded into a step)."""))
        cells.append(code("""
if torch.cuda.is_available() and not SMOKE:
    from lah_b200.parallel.engine import DMoEConfig
    from lah_b200.parallel.trainer import DMoETrainer
    B = num_trainers * batch_size
    cfg = DMoEConfig(hidden=layer_dim, grid_size=(num_experts,), gate_mode='emulator', k=num_active, num_layers=num_blocks,
                     tokens_per_rank=max(B, 256), failure_rate=failure_rate, seed=seed,
                     trainer_staleness=max(0, int(round(mean_delay / num_trainers))))
    engine = DMoETrainer(cfg)
    gen, engine_val, t0 = torch.Generator().manual_seed(seed), [], time.time()
    steps = total_steps // num_trainers
    for step in range(1, steps + 1):
        xb, yb = data.batch(B, gen)
        loss = engine.train_step_device(xb.to(engine.device), yb.to(engine.device))
        if step % max(1, eval_interval // num_trainers) == 0 or step == steps:
            xe, ye = data.batch(256, torch.Generator().manual_seed(seed + 10_000))
            engine_val.append(dict(engine.evaluate(xe, ye), num_updates=step * num_trainers))
            print(engine_val[-1])
    torch.cuda.synchronize(); dt = time.time() - t0
    print(f"engine: {steps} fused steps = {steps * num_trainers} trainer updates in {dt:.1f}s = {steps * B / dt:.0f} samples/s "
          f"(emulator above: {len(train_history) * batch_size / elapsed:.1f} samples/s)")
    engine.close()
else:
    print('no GPU (or smoke mode): engine section skipped')
"""))
    return dict(cells=cells, metadata=dict(kernelspec=dict(display_name="Python 3", language="python", name="python3"),
                                           language_info=dict(name="python")), nbformat=4, nbformat_minor=5)


def main():
    for name, s in SETUPS.items():
        with open(os.path.join(OUT, name), "w") as f:
            json.dump(build(name, s), f, indent=1)
        print("wrote", name)


if __name__ == "__main__":
    main()
