"""
``DMoETrainer`` — the public training API of the in-box engine (what ``bench.py`` and the experiments call).

One trainer per rank.  It owns the flagship model of the convergence experiments (Linear -> N x DMoE -> LayerNorm ->
Linear, reference notebook cell 2), the symmetric-heap context, and the trainer-side optimizer:

* expert parameters are updated inside ``backward`` by the experts' own fused Adam (``FusedDMoE.apply_expert_gradients``)
* the small replicated trainer parameters (stem, gates, head) live in one flat fp32 buffer whose gradient buffer sits in
  the symmetric heap; ``lah_adam_step`` reads every rank's gradient over NVLink, averages and applies AMSGrad in ONE
  kernel (the reference keeps per-trainer copies and never synchronises them; the emulator notebooks share them under a
  lock — averaging is the synchronous equivalent).

``train_step(x_host, y_host)`` is the end-to-end call: pinned host tensors in, python float (loss) out.
"""
import math
from typing import Optional

import torch
import torch.nn as nn
import torch.nn.functional as F

from ..ops import kernels as K, native
from .engine import DMoEConfig, EngineContext, DMoEClassifier, max_groups_per_token


class PendingLoss:
    """handle of an enqueued training step (``DMoETrainer.train_step_async``)"""

    def __init__(self, event=None, host=None, value=None):
        self._event, self._host, self._value = event, host, value

    def result(self) -> float:
        if self._value is None:
            self._event.synchronize()
            self._value = float(self._host[0])
        return self._value


class DMoETrainer:
    def __init__(self, cfg: DMoEConfig, group=None, device: Optional[torch.device] = None, profile_stages: bool = False,
                 metrics_path: Optional[str] = None, use_graph: Optional[bool] = None):
        """
        :param profile_stages: time every stage of a step with CUDA events (+ NVTX ranges); see ``last_stage_ms``
        :param metrics_path: append one JSON record per ``log_step()`` call to this file (structured step metrics)
        :param use_graph: capture the WHOLE training step (forward, loss, backward, expert and trainer optimizers, the peer
            flag protocol) in one CUDA graph after two eager steps and replay it afterwards.  Everything that changes from
            step to step (flag epochs, failure-injection stream, Adam step counters, the learning rate) lives in device
            memory, so the replayed graph is exact.  None = automatic: on for the small-batch (weight-streaming) regime
            where a step is ~130 short kernels, off for the saturated regime where launch latency is hidden anyway.
        """
        from .profiler import MetricsLog
        self.cfg = cfg
        self.metrics = MetricsLog(metrics_path)
        self.last_stage_ms = {}
        self.cuda = torch.cuda.is_available() and (device is None or torch.device(device).type == "cuda")
        if self.cuda:
            native.have_cuda_kernels()  # loads liblah_cuda.so or raises: no silent fallback on a GPU box
            self.ctx = EngineContext(cfg, group=group, device=device)
            self.device = self.ctx.device
            self.world, self.rank = self.ctx.world, self.ctx.rank
            self.ctx.timer.enabled = profile_stages
            self.ctx.timer.nvtx = profile_stages
        else:
            self.ctx, self.device, self.world, self.rank = None, torch.device("cpu"), 1, 0
        torch.manual_seed(cfg.seed)  # identical trainer parameters on every rank
        self.model = DMoEClassifier(cfg, self.ctx, device=self.device).to(self.device)
        for block in self.model.blocks:   # every micro-batch's router gradient is scaled like its cross-entropy
            block.router_grad_scale = 1.0 / max(1, int(cfg.trainer_microbatches))
        self._flatten_trainer_params()
        self.step_count = 0
        # automatic: whenever a step is short enough to be launch-bound (always on the small path; on the big path up to a few
        # thousand rows per rank)
        auto = self.cuda and (self.ctx.small or cfg.tokens_per_rank <= 4096)
        self.use_graph = bool(self.cuda and (auto if use_graph is None else use_graph))
        self._graph, self._graph_B, self._eager_steps = None, -1, 0
        B = cfg.tokens_per_rank
        if self.cuda:
            self.step_dev = torch.zeros(1, dtype=torch.int32, device=self.device)   # trainer AMSGrad step count (device side)
            self._one = torch.ones(1, dtype=torch.int32, device=self.device)
            # double-buffered staging: the NEXT step's inputs can cross PCIe on a copy stream while this step computes
            self._x_dev = [torch.empty(B, cfg.in_features, device=self.device) for _ in range(2)]
            self._y_dev = [torch.empty(B, dtype=torch.int64, device=self.device) for _ in range(2)]
            self._copy_stream = torch.cuda.Stream(device=self.device)
            self._copy_done = [torch.cuda.Event(), torch.cuda.Event()]
            self._compute_done = [torch.cuda.Event(), torch.cuda.Event()]
            self._staged = [None, None]   # (id(x_host), id(y_host), rows) currently resident in each staging buffer
            self._slot = 0
            self._loss_host = [torch.empty(1, dtype=torch.float32).pin_memory() for _ in range(2)]

    def close(self):
        """flush the metrics log and release the peer-mapped symmetric heap (GPU runs); idempotent"""
        self.metrics.close()
        self.stop_heartbeats()
        if self.cuda and self.ctx is not None:
            torch.cuda.synchronize(self.device)
            self.ctx.close()

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()
        return False

    # ------------------------------------------------------------------ learning rate
    @property
    def lr(self) -> float:
        """the learning rate of every expert and trainer optimizer (``cfg.lr``)"""
        return self.cfg.lr

    def set_lr(self, lr: float) -> None:
        """Set the learning rate of every expert and trainer optimizer from the next step on: eager, CPU and CUDA-graph
        replay alike, without re-capturing (the kernels read it from device memory).  Assigning ``cfg.lr`` does the same.
        Collective on multi-GPU runs: every rank must set the same value before the same step, or the replicated trainer
        parameters diverge."""
        lr = float(lr)
        if not math.isfinite(lr) or lr < 0.0:
            raise ValueError(f"Invalid learning rate: {lr}")
        self.cfg.lr = lr

    # ------------------------------------------------------------------ trainer-side flat parameters
    #: the shared experts' tensors start at a multiple of this many floats of the flat buffers: their GEMM operands are
    #: cast and their gradients accumulated by vector accesses
    SHARED_ALIGN = 64

    def _flatten_trainer_params(self):
        params = [p for p in self.model.parameters() if p.requires_grad]  # a frozen (emulator-style) gate stays out
        aligned = {id(p) for block in self.model.blocks for p in block.shared_expert_parameters()}
        offsets, off = [], 0
        for p in params:   # without a shared expert no tensor is aligned: the layout of earlier checkpoints
            if id(p) in aligned:
                off = -(-off // self.SHARED_ALIGN) * self.SHARED_ALIGN
            offsets.append(off)
            off += p.numel()
        n = sum(p.numel() for p in params)
        n_pad = (off + 3) // 4 * 4
        dev = self.device
        self.flat_p = torch.zeros(n_pad, device=dev)
        if self.cuda:
            self.flat_g, self.flat_g_off = self.ctx.heap.alloc((n_pad,), torch.float32)
            self.flat_g.zero_()
        else:
            self.flat_g, self.flat_g_off = torch.zeros(n_pad), -1
        self.flat_m, self.flat_v = torch.zeros(n_pad, device=dev), torch.zeros(n_pad, device=dev)
        self.flat_vmax = torch.zeros(n_pad, device=dev)
        for p, off in zip(params, offsets):
            sl = slice(off, off + p.numel())
            self.flat_p[sl].copy_(p.detach().reshape(-1))
            p.data = self.flat_p[sl].view_as(p)
            p.grad = self.flat_g[sl].view_as(p)
        self.num_trainer_params = n
        self._n_pad = n_pad
        d = int(self.cfg.trainer_staleness)
        self._stale_ring = torch.zeros(d, n_pad, device=dev) if d > 0 else None
        if self.cuda:
            self.ctx.heap.barrier()

    def _trainer_optimizer_step(self):
        cfg = self.cfg
        self.step_count += 1
        if not self.cuda:
            # CPU path: the same flat AMSGrad maths as csrc/adam.cu on the SAME state buffers (flat_m / flat_v / flat_vmax),
            # so checkpoints taken on CPU carry the optimizer state
            with torch.no_grad():
                K.adam_step_ref(self.flat_p, self.flat_g, self.flat_m, self.flat_v, self.flat_vmax, [self._n_pad], 1,
                                step=torch.tensor([self.step_count]), **cfg.adam_kwargs(), zero_mask=1)
            return
        c = self.ctx
        K.bump_steps(self.step_dev, self._one)
        if c.world > 1 and c.dead_mask:
            # degraded mode: some ranks are excluded -> P2P gradient reduce over the survivors only (the switch reduction would
            # include the stale buffers of the excluded ranks)
            alive = c.world - bin(c.dead_mask).count("1")
            epoch = c.next_epoch()
            K.signal_wait(c.flags_off, K.SLOT_TRAINER, epoch, c.status, signal=True, wait=True)
            K.adam_step(self.flat_p, self.flat_g, self.flat_m, self.flat_v, self.flat_vmax, None, [self._n_pad], 1,
                        step=self.step_dev, **c.adam_kwargs(),
                        world=c.world, peer_grad_off=self.flat_g_off, peer_bases=c.heap.peer_bases,
                        grad_scale=1.0 / alive, dead_mask=c.dead_mask)
            K.signal_wait(c.flags_off, K.SLOT_BARRIER, epoch, c.status, signal=True, wait=True)
            self.flat_g.zero_()
        elif c.world > 1 and c.heap.mc_base:
            # NVLS: gradients complete everywhere -> in-switch all-reduce (multimem.ld_reduce + multimem.st, every rank gets the
            # bit-identical mean) -> all slices written -> plain local AMSGrad that also zeroes the gradient buffer
            epoch = c.next_epoch()
            K.signal_wait(c.flags_off, K.SLOT_TRAINER, epoch, c.status, signal=True, wait=True)
            K.nvls_allreduce(self.flat_g_off, self._n_pad, 1.0 / c.world)
            K.signal_wait(c.flags_off, K.SLOT_BARRIER, epoch, c.status, signal=True, wait=True)
            K.adam_step(self.flat_p, self.flat_g, self.flat_m, self.flat_v, self.flat_vmax, None, [self._n_pad], 1,
                        step=self.step_dev, **c.adam_kwargs(), zero_mask=1)
        elif c.world > 1:
            epoch = c.next_epoch()
            K.signal_wait(c.flags_off, K.SLOT_TRAINER, epoch, c.status, signal=True, wait=True)
            K.adam_step(self.flat_p, self.flat_g, self.flat_m, self.flat_v, self.flat_vmax, None, [self._n_pad], 1,
                        step=self.step_dev, **c.adam_kwargs(),
                        world=c.world, peer_grad_off=self.flat_g_off, peer_bases=c.heap.peer_bases,
                        grad_scale=1.0 / c.world)
            # nobody may overwrite its gradient buffer before every peer has consumed it
            K.signal_wait(c.flags_off, K.SLOT_BARRIER, epoch, c.status, signal=True, wait=True)
            self.flat_g.zero_()
        else:
            K.adam_step(self.flat_p, self.flat_g, self.flat_m, self.flat_v, self.flat_vmax, None, [self._n_pad], 1,
                        step=self.step_dev, **c.adam_kwargs(), zero_mask=1)

    # ------------------------------------------------------------------ steps
    def train_step_device(self, x: torch.Tensor, y: torch.Tensor) -> torch.Tensor:
        """one optimisation step on device tensors; returns the (device) loss tensor, no host synchronisation.  With
        ``use_graph`` the third and later calls replay ONE captured CUDA graph of the whole step."""
        if not (self.use_graph and not self.ctx.timer.enabled):
            return self._step_eager(x, y)
        B = x.shape[0]
        if self._graph is None or self._graph_B != B:
            if self._eager_steps < 2:   # lazy initialisation (function attributes, cuBLAS workspaces, autograd threads)
                self._eager_steps += 1
                return self._step_eager(x, y)
            self._capture(B)
        self._gx.copy_(x, non_blocking=True)
        self._gy.copy_(y, non_blocking=True)
        self.ctx.refresh_lr()
        self._graph.replay()
        self.step_count += 1
        native.count_launch(self._graph_launches)
        return self._gloss

    def _capture(self, B: int):
        """capture one whole training step (fixed batch B) into a CUDA graph; nothing is executed here"""
        cfg = self.cfg
        self._gx = torch.zeros(B, cfg.in_features, device=self.device)
        self._gy = torch.zeros(B, dtype=torch.int64, device=self.device)
        torch.cuda.synchronize(self.device)
        before, count_before = native.launches(), self.step_count
        self._graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(self._graph):
            self._gloss = self._step_eager(self._gx, self._gy)
        self._graph_launches = native.launches() - before   # our kernels per replay (bench: gpu_launches)
        native.count_launch(-self._graph_launches)           # capture launched nothing
        self.step_count = count_before
        self._graph_B = B

    def _step_eager(self, x: torch.Tensor, y: torch.Tensor) -> torch.Tensor:
        self.model.train()
        timer = self.ctx.timer if self.cuda else None
        if self.cuda:
            self.ctx.refresh_lr()   # skipped while this step is being captured
            self.ctx.begin_step()
            self.ctx.defer_join = True   # this step joins the optimizer stream itself (below), not at the end of backward()
        if timer is not None:
            timer.start()
        m = max(1, int(self.cfg.trainer_microbatches))
        if m == 1:
            logits = self.model(x)
            loss = F.cross_entropy(logits.float(), y)
            if timer is not None:
                timer.mark("head+loss")
            loss.backward()  # expert updates happen inside (server-side semantics), trainer grads land in flat_g
            if not self.cuda:
                for block in self.model.blocks:
                    block.apply_expert_gradients_ref()
        else:
            # several trainers per rank (reference: num_trainers threads, each with its own small batch): the batch is processed
            # as m micro-batches ONE AFTER THE OTHER; every micro-batch's backward steps the experts it used (so later trainers
            # of the same step already see the updated experts, like concurrent trainers of the reference do), while the
            # trainer-side gradients are averaged over the micro-batches and applied once (optionally stale)
            assert x.shape[0] % m == 0, "trainer_microbatches must divide the batch"
            total = None
            for xm, ym in zip(x.chunk(m), y.chunk(m)):
                loss_m = F.cross_entropy(self.model(xm).float(), ym) / m
                loss_m.backward()
                if not self.cuda:
                    for block in self.model.blocks:
                        block.apply_expert_gradients_ref()
                else:
                    self.ctx.join_optimizer_stream()
                total = loss_m.detach() if total is None else total + loss_m.detach()
            loss = total
        if timer is not None:
            timer.mark("trainer_bwd(stem+gates)")
        if self._stale_ring is not None:
            # delay line of trainer gradients: apply the gradient of `trainer_staleness` steps ago (static buffers: graph-safe)
            with torch.no_grad():
                oldest = self._stale_ring[0].clone()
                if self._stale_ring.shape[0] > 1:
                    self._stale_ring[:-1] = self._stale_ring[1:].clone()
                self._stale_ring[-1].copy_(self.flat_g)
                self.flat_g.copy_(oldest)
        self._trainer_optimizer_step()
        if self.cuda:
            # the expert optimizers of this step (second stream) complete inside the step; joined AFTER the trainer-side
            # all-reduce + AMSGrad so that the last layer's expert updates overlap with them
            self.ctx.join_optimizer_stream()
            self.ctx.defer_join = False
        if timer is not None:
            timer.mark("trainer_adam")
            if timer.enabled:
                self.last_stage_ms = timer.report()
        return loss.detach()

    def log_step(self, loss=None, samples=None, step_ms=None, **extra):
        """structured step record (SURVEY.md 5.5): routing statistics of every DMoE layer, exposed communication wait,
        per-stage ms (when profile_stages), throughput; written to ``metrics_path`` and returned"""
        rec = dict(step=self.step_count, rank=self.rank, world=self.world)
        if loss is not None:
            rec["loss"] = float(loss)
        if samples is not None and step_ms:
            rec["samples_per_s"] = samples / step_ms * 1e3
            rec["step_ms"] = step_ms
        if self.cuda:
            rec["exposed_comm_wait_ms"] = self.ctx.exposed_wait_ms(reset=True)
            layers = []
            for block in self.model.blocks:
                rows = block.ws.step_rows.float()
                layer = dict(active_experts=int((rows > 0).sum()), max_rows=int(rows.max()),
                             mean_rows=float(rows.mean()), padded_rows=int(block.ws.total_rows.item()),
                             shadowed_experts=int((block.ws.shadow_info.view(-1, 4)[:, 0] >= 0).sum()))
                if block.router_loss is not None:   # this rank's unweighted router losses of the layer's last forward
                    aux, z = block.router_loss.tolist()
                    layer.update(router_aux_loss=aux, router_z_loss=z)
                if block.expert_bias is not None:
                    layer["expert_bias_absmax"] = float(block.expert_bias.abs().max())
                if block.n_group > 1:   # the user's check of the limit (at n_group = world: the most ranks a token reached)
                    layer["max_groups_per_token"] = max_groups_per_token(
                        block.ws.idx[:block._last_pairs], self.cfg.k, self.cfg.num_experts, block.n_group)
                if not block.norm_topk_prob and block._last_pairs:   # the router mass the top k carries (DESIGN.md §6e)
                    layer["routed_weight_mean"] = float(
                        block.ws.w[:block._last_pairs].view(-1, self.cfg.k).sum(1).mean())
                if block.ws.capacity_stats is not None:   # the layer's last forward, box-wide (DESIGN.md §6f)
                    cap, dropped = block.ws.capacity_stats.tolist()
                    layer.update(expert_capacity=cap, dropped_pairs=dropped)
                layers.append(layer)
            rec["layers"] = layers
            if self.last_stage_ms:
                rec["stage_ms"] = dict(self.last_stage_ms)
        rec.update(extra)
        return self.metrics.write(**rec)

    def _stage(self, slot, x_host, y_host):
        """enqueue the H2D copies of one batch into staging buffer `slot` on the copy stream"""
        B = x_host.shape[0]
        with torch.cuda.stream(self._copy_stream):
            self._copy_stream.wait_event(self._compute_done[slot])   # the previous user of this buffer has finished
            self._x_dev[slot][:B].copy_(x_host, non_blocking=True)
            self._y_dev[slot][:B].copy_(y_host, non_blocking=True)
            self._copy_done[slot].record(self._copy_stream)
        self._staged[slot] = (id(x_host), id(y_host), B)

    def train_step(self, x_host: torch.Tensor, y_host: torch.Tensor, prefetch=None) -> float:
        """END-TO-END step: host (pinned) inputs -> H2D -> fwd/bwd/optimizers -> D2H loss -> python float.

        :param prefetch: optional ``(x_next, y_next)`` pinned host tensors of the NEXT call: their H2D copy is started
            now on a copy stream and overlaps this step's compute (the next call then finds its inputs on the device)."""
        return self.train_step_async(x_host, y_host, prefetch=prefetch).result()

    def train_step_async(self, x_host: torch.Tensor, y_host: torch.Tensor, prefetch=None) -> "PendingLoss":
        """Same step, but returns immediately with a handle; ``handle.result()`` waits for THIS step's loss (D2H read).
        Calling ``result()`` of step i after step i+1 has been enqueued keeps the host one step ahead of the device, so
        launch latency and the host-side skew between ranks never reach the GPUs (at 8 GPUs the synchronous call costs
        ~10 % — every rank's first kernels wait for its own Python)."""
        if not self.cuda:
            return PendingLoss(value=float(self.train_step_device(x_host, y_host)))
        B = x_host.shape[0]
        slot = self._slot
        if self._staged[slot] != (id(x_host), id(y_host), B):
            self._stage(slot, x_host, y_host)
        stream = torch.cuda.current_stream(self.device)
        stream.wait_event(self._copy_done[slot])
        if prefetch is not None:
            self._stage(slot ^ 1, *prefetch)
        loss = self.train_step_device(self._x_dev[slot][:B], self._y_dev[slot][:B])
        self._compute_done[slot].record(stream)
        self._staged[slot] = None
        self._slot = slot ^ 1
        host = self._loss_host[slot]
        host.copy_(loss.reshape(1), non_blocking=True)
        done = torch.cuda.Event()
        done.record(stream)
        return PendingLoss(event=done, host=host)

    # ------------------------------------------------------------------ failure detection / recovery on the fused path
    def start_heartbeats(self, period: float = 1.0):
        """background thread: every ``period`` s declare this rank's experts alive in the device-resident table of every rank
        (the in-box NetworkHandlerThread, /root/reference/lib/server/network_handler.py:17-20)"""
        import threading
        if getattr(self, "_hb_thread", None) is not None:
            return
        self._hb_stop = threading.Event()

        def loop():
            torch.cuda.set_device(self.device)
            while not self._hb_stop.wait(period):
                self.ctx.heartbeat()

        self.ctx.heartbeat()
        self._hb_thread = threading.Thread(target=loop, daemon=True, name="lah-heartbeat")
        self._hb_thread.start()

    def stop_heartbeats(self):
        if getattr(self, "_hb_thread", None) is not None:
            self._hb_stop.set()
            self._hb_thread.join(timeout=5)
            self._hb_thread = None

    def step_failed(self) -> bool:
        return bool(self.cuda and self.ctx.step_failed())

    def recover(self, max_age: float = 5.0):
        """after a failed step: exclude the ranks whose heartbeats stopped (all survivors read the same table and reach the
        same verdict) and resume training over the surviving ranks / experts.  Returns the excluded ranks."""
        dead = self.ctx.detect_dead_ranks(max_age)
        self.ctx.exclude_ranks(dead)     # also clears the failure flag
        self._graph, self._eager_steps = None, 2   # kernel arguments changed (reduce set): re-capture at the next step
        for block in self.model.blocks:
            block.release_workspace()
        return dead

    # ------------------------------------------------------------------ liveness (failure detection / emulation, SURVEY 5.3)
    @torch.no_grad()
    def set_alive(self, alive) -> None:
        """Install the expert liveness table the gate reads: ``alive`` is a bool / 0-1 tensor of ``num_experts`` entries
        (shared by all DMoE layers, like one DHT) — e.g. ``InBoxNetwork.alive_mask(grid, prefix)`` after heartbeats expired.
        Dead experts are never selected; the softmax renormalises over the survivors (gating_function.py:55-57)."""
        alive = torch.as_tensor(alive).to(torch.uint8).reshape(-1)
        assert alive.numel() == self.cfg.num_experts
        if self.cuda:
            self.ctx.alive.copy_(alive.to(self.device))
        else:
            for block in self.model.blocks:
                block.alive_ref = alive.clone()

    def mark_rank_dead(self, rank: int, world: Optional[int] = None) -> None:
        """emulate the loss of one GPU: every expert it hosts disappears from the routing tables of all trainers"""
        world = world or self.world
        e_loc = self.cfg.num_experts // world
        alive = torch.ones(self.cfg.num_experts, dtype=torch.uint8)
        alive[rank * e_loc: (rank + 1) * e_loc] = 0
        self.set_alive(alive)

    @torch.no_grad()
    def evaluate(self, x: torch.Tensor, y: torch.Tensor):
        """loss / accuracy of one batch.  COLLECTIVE on multi-GPU runs: the experts are sharded over the ranks, so every
        rank must call it at the same point (with its own batch of at most ``tokens_per_rank`` rows)."""
        self.model.eval()
        if self.cuda:
            self.ctx.begin_step()
        logits = self.model(x.to(self.device))
        y = y.to(self.device)
        return dict(loss=float(F.cross_entropy(logits.float(), y)), acc=float((logits.argmax(-1) == y).float().mean()))

    # ------------------------------------------------------------------ checkpoints (SURVEY.md §5.4)
    def state_dict(self):
        """{'trainer': non-expert params + optimizer, 'experts': {uid: {'model': ExpertBackend-style keys,
        'optimizer': torch Adam state_dict}}} for the experts hosted on THIS rank (shardable per rank)."""
        from .engine import expert_uid
        experts = {}
        for li, block in enumerate(self.model.blocks):
            for le in range(block.E_loc):
                uid = f"layer{li}." + expert_uid(self.cfg, block.first_expert + le)
                experts[uid] = dict(model=block.shard.expert_state_dict(le),
                                    optimizer=block.shard.expert_optimizer_state(le))
        if self.cuda:
            torch.cuda.synchronize(self.device)
        trainer = dict(model={k: v.detach().clone().cpu() for k, v in self.model.state_dict().items()},
                       exp_avg=self.flat_m.detach().clone().cpu(), exp_avg_sq=self.flat_v.detach().clone().cpu(),
                       max_exp_avg_sq=self.flat_vmax.detach().clone().cpu(), step=self.step_count, lr=self.lr)
        # the failure-injection stream position: device-side token base on GPU runs (csrc/moe.cu Peers::step_ctr)
        token_base = int(self.ctx.step_ctr[2:4].view(torch.int64).item()) if self.cuda else 0
        state = dict(trainer=trainer, experts=experts, rng=torch.get_rng_state(), token_base=token_base)
        # what is IN FLIGHT in the asynchronous modes: the delay line of stale trainer gradients and, with update_every_*,
        # every expert's pending row / step counters and its partially accumulated gradient (per rank, like `experts`)
        if self._stale_ring is not None:
            trainer["stale_ring"] = self._stale_ring.detach().clone().cpu()
        if self.cfg.router_score != "softmax":   # only then: default checkpoints keep their keys
            trainer["router_score"] = self.cfg.router_score
        if self.cfg.accumulate:
            state["pending"] = [dict(rows=b.shard.pending_rows.clone().cpu(), steps=b.shard.pending_steps.clone().cpu(),
                                     grad=b.shard.g.detach().clone().cpu()) for b in self.model.blocks]
        return state

    def load_state_dict(self, state):
        from .engine import expert_uid
        own = self.model.state_dict()
        saved = state["trainer"]["model"]
        shared = lambda sd: {k: tuple(v.shape) for k, v in sd.items() if k.rsplit(".", 1)[-1].startswith("shared_")}
        own_shared, saved_shared = shared(own), shared(saved)
        if bool(own_shared) != bool(saved_shared):
            raise ValueError(f"checkpoint {'has' if saved_shared else 'has no'} shared expert, this trainer "
                             f"{'has' if own_shared else 'has none'} (DMoEConfig.shared_inner_dim = "
                             f"{self.cfg.shared_inner_dim}); build the trainer with the checkpoint's shared_inner_dim")
        if own_shared != saved_shared:
            raise ValueError(f"checkpoint's shared expert has other widths than this trainer's (shared_inner_dim = "
                             f"{self.cfg.shared_inner_dim}): {saved_shared} against {own_shared}")
        saved_score = state["trainer"].get("router_score", "softmax")
        if saved_score != self.cfg.router_score:
            # the gate (and any expert biases) were trained against the other weight function
            raise ValueError(f"checkpoint was trained with router_score={saved_score!r}, this trainer has "
                             f"router_score={self.cfg.router_score!r}; build it with the checkpoint's router_score")
        biases = [k for k in own if k.endswith(".expert_bias")]
        if any(k.endswith(".expert_bias") and k not in own for k in saved):
            # dropping the saved biases would silently change which experts the gates select
            raise ValueError("checkpoint holds expert routing biases, but this trainer has expert_bias_update_rate=0; "
                             "build it with expert_bias_update_rate > 0 to resume them")
        with torch.no_grad():
            for k in biases:   # a checkpoint without biases starts them at zero (in place: a captured graph reads them)
                if k not in saved:
                    own[k].zero_()
            for k, v in saved.items():
                own[k].copy_(v)
            self.flat_m.copy_(state["trainer"]["exp_avg"])
            self.flat_v.copy_(state["trainer"]["exp_avg_sq"])
            self.flat_vmax.copy_(state["trainer"]["max_exp_avg_sq"])
            if self._stale_ring is not None and "stale_ring" in state["trainer"]:
                self._stale_ring.copy_(state["trainer"]["stale_ring"])
            for block, pend in zip(self.model.blocks, state.get("pending", [])):
                block.shard.pending_rows.copy_(pend["rows"])
                block.shard.pending_steps.copy_(pend["steps"])
                block.shard.g.copy_(pend["grad"])
        self.step_count = int(state["trainer"]["step"])
        if "lr" in state["trainer"]:   # checkpoints without it keep cfg.lr
            self.set_lr(state["trainer"]["lr"])
        if self.cuda:
            self.step_dev.fill_(self.step_count)
            self.ctx.step_ctr[2:4].view(torch.int64).fill_(int(state.get("token_base", 0)))
        for li, block in enumerate(self.model.blocks):
            for le in range(block.E_loc):
                uid = f"layer{li}." + expert_uid(self.cfg, block.first_expert + le)
                if uid in state["experts"]:
                    block.shard.load_expert_state_dict(le, state["experts"][uid]["model"])
                    block.shard.load_expert_optimizer_state(le, state["experts"][uid]["optimizer"])
        if "rng" in state:
            torch.set_rng_state(state["rng"])
        self._graph, self._eager_steps = None, 0   # cached derived tensors (bf16 gate keys, ...) are rebuilt eagerly first
