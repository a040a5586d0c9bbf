#!/usr/bin/env python
"""
Headline benchmark: DMoE training samples/sec (whole job, device-timed, max over ranks).

Config = BASELINE.json "DMoE 256 experts (64x4) FFN block, top-4 gating, bf16": the convergence-notebook model
(Linear(784,512) -> 4 x DMoE[64 experts, top-4, FeedforwardBlock(512)] -> LayerNorm -> Linear(512,10)), full training
step = forward + backward + per-expert AMSGrad + trainer AMSGrad, synthetic MNIST-shaped data, random-init weights.

    python bench.py [--gpus N] [--steps K] [--warmup W] [--batch-per-gpu B]          # our engine
    python bench.py --impl reference ...                                             # unmodified reference (baseline/_ref)
    python -m torch.distributed.run --nnodes=1 --nproc-per-node N ... bench.py --gpus N ...   (N > 1)

Prints ONE JSON line on rank 0.
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import threading
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

import torch


def parse_args():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--impl", choices=["ours", "reference", "baseline"], default="ours",
                    help="baseline = the same step written with torch.topk + NCCL all_to_all_single + cuBLAS + torch Adam "
                         "(lah_b200/parallel/baseline.py): 'the baseline, not the product'")
    ap.add_argument("--batch-per-gpu", type=int, default=256,
                    help="samples per GPU per step (weak scaling); 256 = the reference's operating point: 64 trainers x batch 4 "
                         "(convergence notebooks, SURVEY App. D)")
    ap.add_argument("--ref-batch", type=int, default=0, help="samples per step for the reference arm (0 = --batch-per-gpu)")
    ap.add_argument("--saturated-batch", type=int, default=65536,
                    help="secondary measurement reported under 'saturated': samples per GPU per step in the compute-bound regime")
    ap.add_argument("--no-saturated", action="store_true")
    ap.add_argument("--no-parity", action="store_true")
    ap.add_argument("--extras-timeout", type=float, default=420.0,
                    help="seconds the secondary measurements may take before the headline line is printed without them")
    ap.add_argument("--no-nccl-baseline", action="store_true",
                    help="skip the in-run NCCL(all_to_all_single)+cuBLAS(bmm)+fused-Adam measurement of the same step")
    ap.add_argument("--no-extra-configs", action="store_true", help="skip BASELINE config 5 (failure 0.1) reported as an extra field")
    ap.add_argument("--config4", action="store_true", help="also measure BASELINE config 4 (4096 experts = 1024 x 4, fp8 forward GEMMs; >= 4 GPUs)")
    ap.add_argument("--expert-path", choices=["auto", "small", "big"], default="auto")
    ap.add_argument("--no-graph", action="store_true", help="eager launches instead of the captured CUDA graph (profiling)")
    ap.add_argument("--hidden", type=int, default=512)
    ap.add_argument("--grid", type=int, nargs="+", default=[64])
    ap.add_argument("--gate", choices=["emulator", "product_key"], default="emulator",
                    help="emulator = EmulatedDMoE gate of the reference arm (LayerNorm + normalized keys, not trained)")
    ap.add_argument("--layers", type=int, default=4)
    ap.add_argument("--k", type=int, default=4)
    ap.add_argument("--failure-rate", type=float, default=0.0)
    ap.add_argument("--capacity-factor", type=float, default=0.0,
                    help="receive-buffer rows / local (token, expert) pairs; 0 = auto (retry with a larger one on overflow)")
    ap.add_argument("--shadow-experts", type=int, default=16,
                    help="max hot experts per layer and step that are processed data-parallel on every rank (0 = static placement)")
    ap.add_argument("--shadow-tol", type=float, default=1.04,
                    help="shadow selection stops once the most loaded rank is within this factor of the mean load")
    ap.add_argument("--expert-dtype", choices=["bf16", "fp8"], default="bf16",
                    help="fp8 = forward expert GEMMs on block-scaled FP8 tensor cores (MXFP8)")
    ap.add_argument("--no-e2e", action="store_true")
    ap.add_argument("--dump-outputs", metavar="DIR", default=None,
                    help="after the timed steps, write what the last timed step computed (its loss, the loss of every timed "
                         "step, a fixed sample of the updated parameters) as DIR/<name>.npy, float32")
    return ap.parse_args()


# ------------------------------------------------------------------------------------------------ helpers
class ClockSampler:
    """samples nvidia-smi clocks / throttle reasons of this rank's GPU while the timed region runs"""
    QUERY = ("index,clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.active,clocks_event_reasons.hw_slowdown,"
             "clocks_event_reasons.hw_thermal_slowdown,clocks_event_reasons.sw_thermal_slowdown,"
             "clocks_event_reasons.sw_power_cap")

    def __init__(self, gpu_index):
        self.gpu, self.proc, self.path = gpu_index, None, None
        self.thread, self.stop_flag, self.samples = None, threading.Event(), []

    # NVML in-process (a sample costs ~50 us, one every 4 ms): the timed region of the named config is only tens of ms long at
    # 8 GPUs, shorter than nvidia-smi's start-up, so a subprocess sampler would return nothing.  nvidia-smi is the fallback.
    def _nvml_handle(self):
        import pynvml
        pynvml.nvmlInit()
        try:
            uuid = str(torch.cuda.get_device_properties(self.gpu).uuid)
            return pynvml, pynvml.nvmlDeviceGetHandleByUUID(("GPU-" + uuid) if not uuid.startswith("GPU-") else uuid)
        except Exception:
            visible = os.environ.get("CUDA_VISIBLE_DEVICES")
            index = int(visible.split(",")[self.gpu]) if visible and visible.split(",")[self.gpu].isdigit() else self.gpu
            return pynvml, pynvml.nvmlDeviceGetHandleByIndex(index)

    def _nvml_loop(self, nv, handle):
        names = {"hw_slowdown": nv.nvmlClocksEventReasonHwSlowdown, "hw_thermal_slowdown": nv.nvmlClocksEventReasonHwThermalSlowdown,
                 "sw_thermal_slowdown": nv.nvmlClocksEventReasonSwThermalSlowdown, "sw_power_cap": nv.nvmlClocksEventReasonSwPowerCap,
                 "hw_power_brake_slowdown": nv.nvmlClocksEventReasonHwPowerBrakeSlowdown}
        mx = nv.nvmlDeviceGetMaxClockInfo(handle, nv.NVML_CLOCK_SM)
        while not self.stop_flag.is_set():
            try:
                mask = nv.nvmlDeviceGetCurrentClocksEventReasons(handle)
                self.samples.append((float(nv.nvmlDeviceGetClockInfo(handle, nv.NVML_CLOCK_SM)), float(mx),
                                     nv.nvmlDeviceGetPowerUsage(handle) / 1e3, [k for k, bit in names.items() if mask & bit]))
            except Exception:
                pass
            self.stop_flag.wait(0.004)

    def start(self):
        try:
            nv, handle = self._nvml_handle()
            self.thread = threading.Thread(target=self._nvml_loop, args=(nv, handle), daemon=True)
            self.thread.start()
            return
        except Exception:
            self.thread = None
        try:
            fd, self.path = tempfile.mkstemp(suffix=".csv")
            os.close(fd)
            self.proc = subprocess.Popen(["nvidia-smi", f"--query-gpu={self.QUERY}", "--format=csv,noheader,nounits",
                                          "-lms", "100", "-i", str(self.gpu)], stdout=open(self.path, "w"),
                                         stderr=subprocess.DEVNULL)
        except Exception:
            self.proc = None

    def stop(self):
        out = dict(sm_mhz=None, sm_max_mhz=None, reasons=[])
        if self.thread is not None:
            self.stop_flag.set()
            self.thread.join(timeout=2)
            if self.samples:
                sm = sorted(s[0] for s in self.samples)
                out = dict(sm_mhz=sm[len(sm) // 2], sm_min_mhz=sm[0], sm_max_mhz=max(s[1] for s in self.samples),
                           power_w_max=max(s[2] for s in self.samples), samples=len(sm), sampler="nvml, every 4 ms",
                           reasons=sorted({r for s in self.samples for r in s[3]}))
            return out
        if self.proc is None:
            return out
        time.sleep(0.15)
        self.proc.terminate()
        try:
            self.proc.wait(timeout=5)
        except Exception:
            self.proc.kill()
        sm, mx, reasons, power = [], [], set(), []
        try:
            for line in open(self.path):
                f = [t.strip() for t in line.split(",")]
                if len(f) < 9:
                    continue
                try:
                    sm.append(float(f[1])); mx.append(float(f[2])); power.append(float(f[3]))
                except ValueError:
                    continue
                for name, val in zip(("hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"), f[5:9]):
                    if val.lower().startswith("active"):
                        reasons.add(name)
            os.unlink(self.path)
        except Exception:
            pass
        if sm:
            loaded = sorted(sm)[len(sm) // 2]
            out = dict(sm_mhz=loaded, sm_max_mhz=max(mx), power_w_max=max(power) if power else None,
                       samples=len(sm), sampler="nvidia-smi -lms 100", reasons=sorted(reasons))
        return out


def dist_setup(n_gpus):
    import torch.distributed as dist
    rank = int(os.environ.get("RANK", "0"))
    world = int(os.environ.get("WORLD_SIZE", "1"))
    local_rank = int(os.environ.get("LOCAL_RANK", "0"))
    if torch.cuda.is_available():
        torch.cuda.set_device(local_rank)
        try:  # run next to the GPU: the pinned staging buffers of the end-to-end path are placed by first touch
            import lah_b200  # noqa
            from lah_b200.utils.affinity import bind_to_gpu_numa_node
            bind_to_gpu_numa_node(local_rank)
        except Exception:
            pass
    if world > 1:
        os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
        dist.init_process_group("nccl" if torch.cuda.is_available() else "gloo",
                                device_id=torch.device("cuda", local_rank) if torch.cuda.is_available() else None)
    return rank, world, local_rank


def max_over_ranks(value, world):
    if world == 1:
        return value
    import torch.distributed as dist
    t = torch.tensor([value], dtype=torch.float64, device="cuda")
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    return float(t.item())


def gather_ranks(value, world):
    if world == 1:
        return [round(value, 4)]
    import torch.distributed as dist
    out = [torch.zeros(1, dtype=torch.float64, device="cuda") for _ in range(world)]
    dist.all_gather(out, torch.tensor([value], dtype=torch.float64, device="cuda"))
    return [round(float(t.item()), 4) for t in out]


def barrier_sync(world):
    torch.cuda.synchronize()
    if world > 1:
        import torch.distributed as dist
        dist.barrier()
        torch.cuda.synchronize()


def timed(fn_step, steps, world):
    """EXACTLY `steps` calls bracketed by barrier + synchronize; CUDA events on the launching stream; max over ranks"""
    barrier_sync(world)
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for i in range(steps):
        fn_step(i)
    end.record()
    torch.cuda.synchronize()
    ms = start.elapsed_time(end)
    barrier_sync(world)
    return max_over_ranks(ms, world)


# ------------------------------------------------------------------------------------------------ data
MODEL_STR = "Linear(784,{h}) -> {L} x DMoE[{E} experts FeedforwardBlock({h}), top-{k}] -> LayerNorm -> Linear({h},10)"


def synthetic_mnist(batch, n_batches, seed, in_features=784, num_classes=10, noise=3.0):
    """MNIST-shaped LEARNABLE task (MNIST itself is not on disk): 10 Gaussian class prototypes + noise; the same generator
    feeds both arms (baseline/ref_bench.py has its own copy so that the reference arm imports nothing of ours)."""
    gen = torch.Generator().manual_seed(4242)
    protos = torch.randn(num_classes, in_features, generator=gen)
    gen = torch.Generator().manual_seed(seed)
    xs, ys = [], []
    for _ in range(n_batches):
        y = torch.randint(0, num_classes, (batch,), generator=gen)
        xs.append((protos[y] + noise * torch.randn(batch, in_features, generator=gen)).pin_memory())
        ys.append(y.pin_memory())
    return xs, ys


# ------------------------------------------------------------------------------------------------ our engine
def run_ours(args):
    rank, world, local_rank = dist_setup(args.gpus)
    if not torch.cuda.is_available():
        print(json.dumps({"impl": "ours", "unavailable": "no CUDA device visible"}))
        return
    out = _measure_ours(args, rank, world, local_rank, args.batch_per_gpu, path=args.expert_path, tag="named")
    extras = {}
    # the headline line must never be lost to a secondary measurement: if the extras (NCCL baseline, parity pass, saturated
    # regime, config 5) do not finish in time, every rank prints / exits with what it has
    printed = threading.Event()

    def emergency():
        if rank == 0 and not printed.is_set():
            printed.set()
            line = dict(out)
            line.update(extras)
            line["extras_timed_out_after_s"] = args.extras_timeout
            print(json.dumps(line), flush=True)
        os._exit(0)

    watchdog = threading.Timer(args.extras_timeout, emergency)
    watchdog.daemon = True
    watchdog.start()
    if not args.no_nccl_baseline:
        try:
            nb = measure_nccl_baseline(args, rank, world, local_rank, args.batch_per_gpu, steps=max(10, args.steps))
            extras["nccl_baseline"] = nb
            extras["vs_nccl_baseline"] = (out["value"] / nb["value"]) if out else None
        except Exception as e:
            extras["nccl_baseline"] = {"error": f"{type(e).__name__}: {e}"[:300]}
    if not args.no_parity:
        try:
            extras["parity"] = parity_check(rank, world)
        except Exception as e:  # a failed verification is reported, never hidden
            extras["parity"] = {"ok": False, "error": f"{type(e).__name__}: {e}"[:300]}
    if args.saturated_batch > 0 and not args.no_saturated:
        try:
            sat = _measure_ours(args, rank, world, local_rank, args.saturated_batch, path="big", tag="saturated",
                                steps=max(3, min(args.steps, 10)), warmup=3)
            if sat:
                extras["saturated"] = {k: sat[k] for k in ("value", "unit", "ms_per_step", "e2e", "clocks", "gpu_launches",
                                                           "exposed_comm_wait_ms_per_step", "stage_ms_rank0", "config",
                                                           "steps", "warmup", "loss_first_last")}
        except Exception as e:
            extras["saturated"] = {"error": f"{type(e).__name__}: {e}"[:300]}
        if world > 1 and args.saturated_batch % world == 0:
            # STRONG scaling of the saturated regime: the same GLOBAL batch (the 1-GPU "saturated" field) split over N ranks
            try:
                ss = _measure_ours(args, rank, world, local_rank, args.saturated_batch // world, path="big", tag="strong",
                                   steps=max(3, min(args.steps, 10)), warmup=3)
                if ss:
                    extras["strong_scaling_saturated"] = {
                        "global_batch": args.saturated_batch, "scaling": "strong",
                        **{k: ss[k] for k in ("value", "unit", "ms_per_step", "exposed_comm_wait_ms_per_step", "steps", "warmup")},
                        "e2e_ms_per_step": ss["e2e"]["ms_per_step"] if ss.get("e2e") else None}
            except Exception as e:
                extras["strong_scaling_saturated"] = {"error": f"{type(e).__name__}: {e}"[:300]}
    if not args.no_extra_configs:
        # BASELINE.json configs 5 (10 % expert failures, every N) and 4 (4096 experts = 1024 x 4, FP8 forward GEMMs, 64 trainers x
        # batch 8; needs the 8-GPU box: 25.8 B expert parameters + AMSGrad state = 71 GB per rank)
        extra = [("config5_failure01", dict(failure_rate=0.1))]
        if args.config4 and world >= 4:   # opt-in: 71 GB of expert state per rank at 8 GPUs; never risk the headline line for it
            extra.append(("config4_4096experts_fp8", dict(grid=[1024], batch=8 * 64, expert_dtype="fp8", path="big")))
        for name, kw in extra:
            try:
                a2 = argparse.Namespace(**vars(args))
                a2.grid = kw.get("grid", args.grid)
                a2.failure_rate = kw.get("failure_rate", args.failure_rate)
                a2.expert_dtype = kw.get("expert_dtype", args.expert_dtype)
                r = _measure_ours(a2, rank, world, local_rank, kw.get("batch", args.batch_per_gpu), path=kw.get("path", args.expert_path),
                                  tag=name, steps=max(3, min(args.steps, 5)), warmup=3)
                if r:
                    extras[name] = {k: r[k] for k in ("value", "unit", "ms_per_step", "e2e", "config", "clocks", "steps", "warmup",
                                                      "loss_first_last")}
            except Exception as e:
                extras[name] = {"error": f"{type(e).__name__}: {e}"[:300]}
    watchdog.cancel()
    if rank == 0 and not printed.is_set():
        printed.set()
        out.update(extras)
        print(json.dumps(out), flush=True)
    if world > 1:
        import torch.distributed as dist
        dist.barrier()
        dist.destroy_process_group()


def _measure_ours(args, rank, world, local_rank, B, path="auto", tag="named", steps=None, warmup=None):
    import gc
    import lah_b200  # noqa
    from lah_b200.ops import native
    from lah_b200.parallel.engine import DMoEConfig
    from lah_b200.parallel.trainer import DMoETrainer
    steps = steps or args.steps
    warmup = max(3, warmup if warmup is not None else args.warmup)
    # identical configuration at every N: worst-case receive buffers in the small-batch regime (nothing can overflow: at
    # most world x pairs rows reach one rank); shadowing + 2x buffers in the saturated regime
    small_cfg = DMoEConfig(hidden=args.hidden, grid_size=tuple(args.grid), k=args.k, num_layers=args.layers, tokens_per_rank=B,
                           expert_path=path, expert_dtype=args.expert_dtype)
    is_small = small_cfg.resolved_path(world) == "small"
    capacity = args.capacity_factor if args.capacity_factor > 0 else (float(world) if is_small else 2.0)
    cfg = DMoEConfig(hidden=args.hidden, grid_size=tuple(args.grid), k=args.k, num_layers=args.layers,
                     tokens_per_rank=B, capacity_factor=capacity, failure_rate=args.failure_rate,
                     gate_mode=args.gate, shadow_experts=args.shadow_experts, shadow_tol=args.shadow_tol,
                     expert_dtype=args.expert_dtype, expert_path=path)
    torch.manual_seed(4321 + rank)   # same weights on every run: outputs of two builds can be compared one to one
    trainer = DMoETrainer(cfg, use_graph=False if args.no_graph else None)
    n_batches = 4
    xs_host, ys_host = synthetic_mnist(B, n_batches, seed=1234 + rank, in_features=cfg.in_features)
    xs_dev = [x.cuda(non_blocking=True) for x in xs_host]
    ys_dev = [y.cuda(non_blocking=True) for y in ys_host]
    dev_losses = []

    def step_device(i):
        dev_losses.append(trainer.train_step_device(xs_dev[i % n_batches], ys_dev[i % n_batches]).reshape(1).clone())

    losses, pending = [], []

    def step_e2e(i):
        # end to end through the public API: pinned host inputs -> H2D (the next step's inputs cross PCIe on a copy stream
        # while this step computes) -> step -> D2H loss.  The loss of step i is read (blocking) right after step i+1 has
        # been enqueued, so every step's result reaches the host inside the timed region but the host stays one step ahead
        nxt = (i + 1) % n_batches
        pending.append(trainer.train_step_async(xs_host[i % n_batches], ys_host[i % n_batches],
                                                prefetch=(xs_host[nxt], ys_host[nxt])))
        if len(pending) > 1:
            losses.append(pending.pop(0).result())

    def drain_e2e():
        while pending:
            losses.append(pending.pop(0).result())

    def check_all_ranks():
        code = int(trainer.ctx.status.item())
        if world > 1:
            import torch.distributed as dist
            t = torch.tensor([code & 1, code & 2], device="cuda")  # NCCL has no bitwise-or: MAX per status bit
            dist.all_reduce(t, op=dist.ReduceOp.MAX)
            code = int(t[0].item()) | int(t[1].item())
        if code:
            trainer.ctx.status.fill_(code)
            try:
                trainer.ctx.check_status()
            finally:
                trainer.ctx.heap.close()

    barrier_sync(world)   # ranks finish building their host batches at different times: start the first step together
    for i in range(warmup):
        step_device(i)
    check_all_ranks()
    sampler = ClockSampler(local_rank)
    sampler.start()
    native.reset_launches()
    trainer.ctx.exposed_wait_ms(reset=True)
    profiling = bool(os.environ.get("LAH_CUDA_PROFILE"))  # ncu --profile-from-start off
    if profiling:
        torch.cuda.profiler.start()
    ms = timed(step_device, steps, world)
    if profiling:
        torch.cuda.profiler.stop()
    launches = native.launches()
    exposed_local = trainer.ctx.exposed_wait_ms(reset=True) / steps
    exposed_ms = max_over_ranks(exposed_local, world)
    exposed_ranks = gather_ranks(exposed_local, world)   # the rank with the SMALLEST wait is the step's straggler
    clocks = sampler.stop()
    check_all_ranks()
    if args.dump_outputs and tag == "named":
        dump_outputs(args.dump_outputs, trainer, dev_losses[-steps:], rank)
    global_batch = B * world
    value = global_batch * steps / (ms / 1e3)
    loss_curve = [float(t) for t in torch.cat(dev_losses).cpu()]

    e2e = None
    if not args.no_e2e:
        for i in range(2):
            step_e2e(i)
        drain_e2e()

        def e2e_steps(i):   # the last timed step also waits for its own loss: all K results are on the host at the end
            step_e2e(i)
            if i == steps - 1:
                drain_e2e()

        ms_e2e = timed(e2e_steps, steps, world)
        check_all_ranks()
        e2e = {"value": global_batch * steps / (ms_e2e / 1e3), "unit": "samples/s",
               "ms_per_step": ms_e2e / steps,
               "h2d_bytes_per_step": int(xs_host[0].numel() * 4 + ys_host[0].numel() * 8),
               "d2h_bytes_per_step": 4, "last_loss": losses[-1] if losses else None}

    # per-stage breakdown of ONE extra (untimed, eager) step: CUDA events between the stages, synchronised afterwards
    trainer.ctx.timer.enabled = True
    trainer.train_step_device(xs_dev[0], ys_dev[0])
    stage_ms = {k: round(v, 3) for k, v in trainer.last_stage_ms.items()}
    trainer.ctx.timer.enabled = False
    routing = []
    active_total = 0
    for block in trainer.model.blocks:  # tokens-per-expert histogram of the last step (observability, SURVEY 5.5)
        rows = block.ws.step_rows.float()
        active_total += int((rows > 0).sum())
        routing.append({"active_experts": int((rows > 0).sum()), "max_rows": int(rows.max()), "mean_rows": float(rows.mean()),
                        "padded_rows": int(block.ws.total_rows.item()),
                        "shadowed_experts": int((block.ws.shadow_info.view(-1, 4)[:, 0] >= 0).sum())})
    hottest = [int(max_over_ranks(float(r["max_rows"]), world)) for r in routing]   # over ALL ranks (load skew)
    # step roofline in the weight-streaming regime: every ACTIVE expert streams its bf16 weights twice (forward, dgrad) and
    # its fp32 optimizer state once (34 B / parameter with the fused wgrad+AMSGrad kernel); rank 0's share
    per_expert = sum(int(torch.tensor(s).prod()) for s in cfg.seg_shapes().values())
    hbm = float(_peaks().get("hbm_gbs", 3350.0))   # H100 SXM data sheet
    ideal_ms = active_total * per_expert * (2 + 2 + 34) / (hbm * 1e9) * 1e3
    out = None
    result = {
        "metric": "DMoE training samples/sec (whole job, device-timed, max over ranks)",
        "impl": "ours", "value": value, "unit": "samples/s", "n_gpus": world, "steps": steps,
        "warmup": warmup, "ms_per_step": ms / steps, "higher_is_better": True, "scaling": "weak",
        "vs_baseline": value / 16.8, "dtype": "bf16", "data": DATA_STR,
        "config": {"model": MODEL_STR.format(h=cfg.hidden, L=cfg.num_layers, E=cfg.num_experts, k=cfg.k),
                   "step": "fwd+bwd+per-expert AMSGrad (stepped after every backward)+trainer AMSGrad",
                   "global_batch": global_batch, "batch_per_gpu": B, "trainers_x_batch": "64 x 4 per GPU" if B == 256 else None,
                   "seq_len": 1, "parallelism": f"ep{world}+dp{world}",
                   "expert_path": "small (swap-AB weight streaming, fused wgrad+AMSGrad, CUDA graph)" if trainer.ctx.small
                   else "big (128x256 wgmma tiles)",
                   "cuda_graph": bool(trainer.use_graph),
                   "capacity_factor": capacity, "shadow_experts": trainer.ctx.S, "shadow_tol": cfg.shadow_tol,
                   "expert_gemm_dtype": cfg.expert_dtype + (" forward, bf16 dgrad/wgrad" if cfg.expert_dtype == "fp8" else ""),
                   "experts_total": cfg.num_experts * cfg.num_layers, "failure_rate": cfg.failure_rate,
                   "gate": cfg.gate_mode + (" (LayerNorm(x) @ normalize(keys); gate params not trained, exactly like the reference's EmulatedDMoE)" if cfg.gate_mode == "emulator" else " (trainable product-key proj, lib.GatingFunction)"),
                   "l2_policy": "working set per step (optimizer state + weights of the active experts, >10 GB) exceeds the 50 MB L2; no explicit flush"},
        "clocks": clocks, "gpu_launches": launches, "e2e": e2e, "routing_rank0": routing,
        "exposed_comm_wait_ms_per_step": exposed_ms, "exposed_comm_wait_ms_per_rank": exposed_ranks,
        "hottest_expert_rows_per_layer": hottest, "stage_ms_rank0": stage_ms,
        "loss_first_last": [loss_curve[0], loss_curve[-1]] if loss_curve else None,
        "roofline": {"active_experts_rank0": active_total, "ideal_ms_hbm_bound_rank0": round(ideal_ms, 3),
                     "frac_of_measured_copy": round(ideal_ms / (ms / steps), 3) if trainer.ctx.small else None,
                     "note": "38 B per parameter of every active expert at hbm_gbs of MEASURED_PEAKS.json if present, else the 3.35 TB/s data sheet"},
        "baseline_note": "vs_baseline = value / 16.8 samples/s (reference notebook dmoe64x4, BASELINE.md)",
    }
    trainer.close()
    del trainer, xs_dev, ys_dev
    gc.collect()
    torch.cuda.empty_cache()
    return result


def dump_outputs(out_dir, trainer, step_losses, rank):
    """What the timed path handed back and left behind in its last step, as float32 .npy files (a few MB in all):
    loss (the last step's loss), losses (every timed step), and a fixed, seeded sample of 65536 entries of every updated
    parameter group (each expert layer's fp32 master weights, the trainer's dense parameters)."""
    import numpy as np
    os.makedirs(out_dir, exist_ok=True)
    suffix = f"_rank{rank}" if rank else ""
    losses = torch.cat(step_losses).float().cpu().numpy()
    arrays = {"loss": losses[-1:], "losses": losses}
    gen = torch.Generator().manual_seed(99)
    for i, block in enumerate(trainer.model.blocks):
        p = block.shard.p.detach().float().flatten()
        idx = torch.randint(0, p.numel(), (min(65536, p.numel()),), generator=gen).to(p.device)
        arrays[f"layer{i}_expert_params_sample"] = p[idx].cpu().numpy()
    for name in ("stem", "norm", "head"):
        mod = getattr(trainer.model, name, None)
        if mod is not None:
            for pname, t in mod.named_parameters():
                arrays[f"{name}_{pname}"] = t.detach().float().cpu().numpy()
    for name, a in arrays.items():
        np.save(os.path.join(out_dir, name + suffix + ".npy"), a.astype(np.float32))


DATA_STR = "synthetic (MNIST-shaped 784-d fp32 rows: 10 Gaussian class prototypes + noise, learnable; random-init weights)"


def _peaks():
    try:
        return json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))
    except Exception:
        return {}


def parity_check(rank, world):
    """Correctness INSIDE the benchmark process, outside the timed region: ONE DMoE layer (16 experts over all ranks),
    forward + backward + expert AMSGrad through the fused P2P engine on `world` GPUs against the dense fp32 PyTorch oracle
    (FusedDMoE(ctx=None)._forward_ref) of the SAME layer on the concatenated batch.  Two passes: the small-batch path and
    the saturated path with every shadow slot forced (replica pull + fused gradient reduce)."""
    import torch.distributed as dist
    import lah_b200  # noqa
    from lah_b200.parallel import engine as E
    out = {}

    def rel(a, b):
        return ((a.float() - b.float()).norm() / (b.float().norm() + 1e-12)).item()

    for name, kw in (("small", dict(expert_path="small")),
                     ("big_forced_shadow", dict(expert_path="big", shadow_experts=4, shadow_tol=0.0, shadow_min_rows=1))):
        B = 256
        cfg = E.DMoEConfig(hidden=512, grid_size=(4, 4), k=4, num_layers=1, tokens_per_rank=B, capacity_factor=float(max(world, 2)),
                           lr=1e-3, **kw)
        ctx = E.EngineContext(cfg)
        torch.manual_seed(0)
        layer = E.FusedDMoE(cfg, ctx).cuda()
        torch.manual_seed(0)
        oracle = E.FusedDMoE(cfg, None, device=torch.device("cuda")).cuda()   # all experts local, plain PyTorch fp32
        # fp32 maths, but activations / GEMM operands rounded to bf16 exactly where the engine stores bf16: without it ~0.4 % of
        # the ReLU gates differ between an fp32 and a bf16 forward, which alone is ~5 % rel-L2 on the weight gradients
        oracle.ref_emulate_bf16 = True
        gen = torch.Generator().manual_seed(7)
        x_all = torch.randn(world * B, 512, generator=gen).to(torch.bfloat16)
        g_all = torch.randn(world * B, 512, generator=gen).to(torch.bfloat16)
        sl = slice(rank * B, (rank + 1) * B)
        x = x_all[sl].cuda().requires_grad_(True)
        layer.train()
        y = layer(x)
        y.backward(g_all[sl].cuda())
        xo = x_all.cuda().float().requires_grad_(True)
        oracle.train()
        yo = oracle(xo)
        yo.backward(g_all.cuda().float())
        oracle.apply_expert_gradients_ref()
        torch.cuda.synchronize()
        ctx.check_status()
        gw = layer.proj.weight.grad.clone()
        if world > 1:
            dist.all_reduce(gw)
        lo, hi = layer.first_expert, layer.first_expert + layer.E_loc
        errs = dict(y=rel(y, yo[sl]), dx=rel(x.grad, xo.grad[sl]), dproj=rel(gw, oracle.proj.weight.grad),
                    w1=(layer.shard.views["w1"][:layer.E_loc] - oracle.shard.views["w1"][lo:hi]).abs().mean().item(),
                    wgrad_w2=rel(layer.shard.m_views["w2"][:layer.E_loc], oracle.shard.m_views["w2"][lo:hi]),
                    steps_equal=float(torch.equal(layer.shard.step.cpu(), oracle.shard.step[lo:hi].cpu().to(layer.shard.step.dtype))))
        shadowed = int((layer.ws.shadow_info.view(-1, 4)[:, 0] >= 0).sum())
        t = torch.tensor([errs[k] for k in ("y", "dx", "dproj", "w1", "wgrad_w2")], device="cuda", dtype=torch.float64)
        mn = torch.tensor([errs["steps_equal"]], device="cuda", dtype=torch.float64)
        if world > 1:
            dist.all_reduce(t, op=dist.ReduceOp.MAX)
            dist.all_reduce(mn, op=dist.ReduceOp.MIN)
        e = dict(zip(("y", "dx", "dproj", "w1", "wgrad_w2"), [float(v) for v in t]))
        e["steps_equal"] = bool(mn.item() == 1.0)
        e["shadowed_experts"] = shadowed
        e["ok"] = bool(e["y"] < 1e-2 and e["dx"] < 2e-2 and e["dproj"] < 3e-2 and e["w1"] < 1e-4 and e["wgrad_w2"] < 2e-2
                       and e["steps_equal"] and (name == "small" or world == 1 or shadowed > 0))
        out[name] = e
        torch.cuda.synchronize()
        if world > 1:
            dist.barrier()
        ctx.close()
        del layer, oracle, ctx
        torch.cuda.empty_cache()
    out["ok"] = all(v["ok"] for v in out.values())
    out["what"] = "1 DMoE layer fwd+bwd+AMSGrad on all ranks vs dense PyTorch oracle (fp32 maths, bf16-rounded activations); rel-L2 errors (w1: mean |diff| after the step), max over ranks"
    return out


# ------------------------------------------------------------------------------------------------ NCCL + cuBLAS baseline
def measure_nccl_baseline(args, rank, world, local_rank, B, steps=None, warmup=3):
    """the same step through parallel/baseline_fast.py: same gate, fixed-capacity buffers, all_to_all_single (NCCL, equal
    splits), cuBLAS bmm under bf16 autocast, fused torch Adam(amsgrad) — no host synchronisation inside a step"""
    import gc
    import lah_b200  # noqa
    from lah_b200.parallel.engine import DMoEConfig
    from lah_b200.parallel.baseline_fast import FastBaselineTrainer
    steps = max(10, steps or args.steps)
    cfg = DMoEConfig(hidden=args.hidden, grid_size=tuple(args.grid), k=args.k, num_layers=args.layers, tokens_per_rank=B,
                     gate_mode=args.gate)
    trainer = FastBaselineTrainer(cfg)
    xs_host, ys_host = synthetic_mnist(B, 4, seed=1234 + rank, in_features=cfg.in_features)
    xs = [x.cuda() for x in xs_host]
    ys = [y.cuda() for y in ys_host]
    losses = []

    def step(i):
        losses.append(trainer.train_step_device(xs[i % 4], ys[i % 4]).reshape(1))

    barrier_sync(world)
    for i in range(max(3, warmup)):
        step(i)
    sampler = ClockSampler(local_rank)
    sampler.start()
    ms = timed(step, steps, world)
    clocks = sampler.stop()
    curve = [float(t) for t in torch.cat(losses).cpu()]
    value = B * world * steps / (ms / 1e3)
    out = {"impl": "baseline (torch.topk + NCCL all_to_all_single + cuBLAS bmm + fused torch Adam; parallel/baseline_fast.py)",
           "value": value, "unit": "samples/s", "ms_per_step": ms / steps, "steps": steps, "warmup": max(3, warmup),
           "capacity_rows_per_expert_and_rank": trainer.capacity, "clocks": clocks,
           "loss_first_last": [curve[0], curve[-1]], "global_batch": B * world}
    del trainer, xs, ys
    gc.collect()
    torch.cuda.empty_cache()
    return out


def run_baseline(args):
    rank, world, local_rank = dist_setup(args.gpus)
    if not torch.cuda.is_available():
        print(json.dumps({"impl": "baseline", "unavailable": "no CUDA device visible"}))
        return
    r = measure_nccl_baseline(args, rank, world, local_rank, args.batch_per_gpu)
    if rank == 0:
        E = int(torch.tensor(args.grid).prod())
        print(json.dumps({
            "metric": "DMoE training samples/sec (whole job, device-timed, max over ranks)", "impl": "baseline",
            "value": r["value"], "unit": "samples/s", "n_gpus": world, "steps": r["steps"], "warmup": r["warmup"],
            "ms_per_step": r["ms_per_step"], "higher_is_better": True, "scaling": "weak", "vs_baseline": r["value"] / 16.8,
            "dtype": "bf16 autocast", "data": DATA_STR,
            "config": {"model": MODEL_STR.format(h=args.hidden, L=args.layers, E=E, k=args.k), "implementation": r["impl"],
                       "global_batch": r["global_batch"], "batch_per_gpu": args.batch_per_gpu, "seq_len": 1,
                       "parallelism": f"ep{world}+dp{world} (NCCL all_to_all_single)",
                       "capacity_rows_per_expert_and_rank": r["capacity_rows_per_expert_and_rank"]},
            "clocks": r["clocks"], "gpu_launches": 0, "loss_first_last": r["loss_first_last"]}))
    if world > 1:
        import torch.distributed as dist
        dist.barrier()
        dist.destroy_process_group()


# ------------------------------------------------------------------------------------------------ reference arm
def run_reference(args):
    ref_root = os.path.join(ROOT, "baseline", "_ref")
    if not os.path.isdir(os.path.join(ref_root, "experiments", "convergence")):
        print(json.dumps({"impl": "reference", "unavailable": "baseline/_ref missing (run baseline/install_reference.sh)"}))
        return
    rank, world, local_rank = dist_setup(args.gpus)
    if not torch.cuda.is_available():
        print(json.dumps({"impl": "reference", "unavailable": "no CUDA device visible"}))
        return
    sys.path.insert(0, ref_root)
    from baseline.ref_bench import build_reference_trainer
    B = args.ref_batch or args.batch_per_gpu
    step, info = build_reference_trainer(hidden=args.hidden, num_experts=1 if not args.grid else int(torch.tensor(args.grid).prod()),
                                         num_active=args.k, num_layers=args.layers, batch_size=B,
                                         failure_rate=args.failure_rate, seed=1337 + rank)
    for i in range(args.warmup):
        step(i, e2e=False)
    sampler = ClockSampler(local_rank)
    sampler.start()
    ms = timed(lambda i: step(i, e2e=False), args.steps, world)
    clocks = sampler.stop()
    value = B * world * args.steps / (ms / 1e3)
    e2e = None
    if not args.no_e2e:
        ms_e2e = timed(lambda i: step(i, e2e=True), args.steps, world)
        e2e = {"value": B * world * args.steps / (ms_e2e / 1e3), "unit": "samples/s", "ms_per_step": ms_e2e / args.steps,
               "h2d_bytes_per_step": B * 784 * 4 + B * 8, "d2h_bytes_per_step": 4}
    if rank == 0:
        print(json.dumps({
            "metric": "DMoE training samples/sec (whole job, device-timed, max over ranks)", "impl": "reference",
            "value": value, "unit": "samples/s", "n_gpus": world, "steps": args.steps, "warmup": args.warmup,
            "ms_per_step": ms / args.steps, "higher_is_better": True, "scaling": "weak", "vs_baseline": value / 16.8,
            "dtype": "fp32", "data": DATA_STR,
            "config": {"model": MODEL_STR.format(h=args.hidden, L=args.layers, E=int(torch.tensor(args.grid).prod()), k=args.k),
                       "step": "fwd+bwd+per-expert AMSGrad (update_every_inputs=batch)+trainer AMSGrad",
                       "global_batch": B * world, "batch_per_gpu": B, "trainers_x_batch": "64 x 4 per GPU" if B == 256 else None,
                       "seq_len": 1, "implementation": info,
                       "parallelism": f"dp{world}: 1 independent replica per GPU (the reference emulator is single-process and has "
                                      "no collective; the reference's multi-GPU stack is TCP RPC, see profiles/)"},
            "clocks": clocks, "gpu_launches": 0, "e2e": e2e}))
    if world > 1:
        import torch.distributed as dist
        dist.barrier()
        dist.destroy_process_group()


if __name__ == "__main__":
    a = parse_args()
    if a.impl == "baseline":
        run_baseline(a)
    elif a.impl == "reference":
        try:
            run_reference(a)
        except Exception as e:  # the reference arm must never fail the driver
            print(json.dumps({"impl": "reference", "unavailable": f"{type(e).__name__}: {e}"[:300]}))
    else:
        run_ours(a)
