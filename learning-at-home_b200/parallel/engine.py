"""
The in-box DMoE engine: every rank (one process per H100) is BOTH a trainer and the host of a shard of experts.

Mapping to the reference (SURVEY.md §7.0):
  * ``GatingFunction.forward``  (/root/reference/lib/client/gating_function.py:25-66)   -> ``FusedDMoE.forward``
  * ``RemoteExpert`` fwd/bwd RPCs (/root/reference/lib/client/remote_expert.py:53-76)   -> P2P scatter / combine kernels
  * ``TaskPool`` batching (/root/reference/lib/runtime/task_pool.py:105-172)            -> expert-grouped row layout
  * ``ExpertBackend.forward/backward/apply_gradients`` (lib/runtime/expert_backend.py:64-97)
                                                            -> grouped wgmma GEMMs, fused LN/ReLU, fused Adam(AMSGrad)
  * DHT liveness (/root/reference/lib/network/__init__.py:88-129)                       -> ``alive`` table read by the gate

Activations of the experts stay resident on the expert's GPU between forward and backward (the reference recomputes
the forward and re-sends the inputs); the optimizer step of an expert happens inside the backward pass, once per step,
for experts that received at least one row — per-expert Adam state and step counters, exactly like one
``torch.optim.Adam(amsgrad=True)`` per ``ExpertBackend``.

On a machine without a GPU the same modules run a plain PyTorch implementation of identical maths (``_forward_ref``),
which is also the numerical oracle of the GPU tests.
"""
import math
from dataclasses import dataclass, field
from typing import Dict, List, Optional, Sequence, Tuple

import torch
import torch.nn as nn
import torch.nn.functional as F

from ..ops import fp8, gemm, kernels as K, native

SEG_NAMES = ("w1", "b1", "g1", "be1", "w2", "b2", "g2", "be2", "w3", "b3")
#: name of each segment inside a reference FeedforwardBlock state_dict (layers.py:8-16)
REF_KEYS = {"w1": "layers.0.weight", "b1": "layers.0.bias", "g1": "layers.1.weight", "be1": "layers.1.bias",
            "w2": "layers.3.weight", "b2": "layers.3.bias", "g2": "layers.4.weight", "be2": "layers.4.bias",
            "w3": "layers.6.weight", "b3": "layers.6.bias"}
SMALL_SEG_MASK = sum(1 << i for i, n in enumerate(SEG_NAMES) if not n.startswith("w"))


@dataclass
class DMoEConfig:
    hidden: int = 512
    grid_size: Tuple[int, ...] = (8, 8)
    k: int = 4
    num_layers: int = 4
    in_features: int = 784
    num_classes: int = 10
    tokens_per_rank: int = 1024          # maximum batch (rows) a rank feeds per step
    capacity_factor: float = 2.0         # receive-buffer rows = capacity_factor * tokens_per_rank * k (+ padding)
    failure_rate: float = 0.0            # Bernoulli per (token, expert) failure injection (faulty_dmoe_emulator.py:49-51)
    lr: float = 1e-3
    betas: Tuple[float, float] = (0.9, 0.999)
    eps: float = 1e-8
    amsgrad: bool = True
    seed: int = 1337
    uid_prefix: str = "expert"
    two_cta: bool = True                 # wide 128x256 GEMM tiles with fused activation; expert groups padded to 256 rows
    # gate of the fused layer:
    #   "product_key": lib.GatingFunction semantics — trainable proj = Linear(hidden, sum(grid)), score = sum of per-dim logits
    #   "emulator":    EmulatedDMoE semantics (dmoe_emulator.py:47) — logits = LayerNorm(x) @ F.normalize(expert_keys, -1);
    #                  like in the reference emulator these gate parameters are NOT trained (get_non_expert_params excludes
    #                  them and no expert optimizer owns them); requires a 1-d grid (grid_size=(num_experts,))
    gate_mode: str = "product_key"
    # hot-expert shadowing (multi-GPU load balancing, csrc/moe.cu layout_exchange_kernel): up to `shadow_experts` experts
    # per layer and step are processed data-parallel (every rank keeps its own rows and a replica of the weights, the
    # owner's optimizer sums the partial gradients); selection stops once max rank load <= shadow_tol * mean
    shadow_experts: int = 8
    shadow_tol: float = 1.1
    shadow_min_rows: int = 1024
    # "bf16" or "fp8": with "fp8" the three forward GEMMs of every expert run on block-scaled FP8 tensor cores (MXFP8:
    # E4M3 + UE8M0 scale per 1x32 block, csrc/grouped_gemm_fp8.cu); dgrad / wgrad / optimizer are unchanged (bf16 / fp32)
    expert_dtype: str = "bf16"
    # which expert kernels run (csrc/):
    #   "big":   rows grouped per expert and padded to 256 rows, 128x256 wgmma tiles (grouped_gemm.cu) — compute-bound regime
    #   "small": the reference's operating point (64 trainers x batch 4 => O(16) rows per expert): swap-AB wgmma tiles
    #            that stream every weight once (small_m.cu), groups padded to 16 rows, weight gradient + AMSGrad fused in
    #            one kernel (the gradient never reaches HBM)
    #   "auto":  "small" when a step brings fewer than 512 rows per expert on average (up to there streaming the weights
    #            through 128-token swap-AB tiles, with the fused optimizer and the step in one CUDA graph, beats padding every
    #            expert to 256 rows; beyond, the wide tiles of the big path win)
    expert_path: str = "auto"
    # small path: run the fused weight-gradient + AMSGrad kernels (bandwidth-bound, ~75 % of the step) on a SECOND stream,
    # concurrently with the latency-bound chain of the backward pass (dgrads, LayerNorm backward, combine, the next layer's
    # dispatch).  `optimizer_ctas` SMs stream optimizer state, the chain keeps the remaining ones (persistent kernels of both
    # sides are launched with matching CTA limits so that neither starves the other).  0 disables the overlap, -1 = automatic:
    # 11/14 of the SMs on one GPU, 9/14 when the experts are sharded (the sharded chain waits on peers and needs more SMs)
    optimizer_ctas: int = -1
    # asynchronous expert updates (reference: EmulatedDMoE.update_every_inputs / update_every_steps,
    # experiments/convergence/dmoe_emulator.py:70-77): an expert accumulates weight gradients and steps once it has seen
    # >= update_every_inputs rows or >= update_every_steps steps since its first pending row (either suffices; a 0 leaves that
    # clause unset).  (0, 0) = step after every backward batch (lib/runtime/expert_backend.py:95-97), the default.
    update_every_inputs: int = 0
    update_every_steps: int = 0
    # stale trainer gradients (reference notebooks, cell 3: a trainer computes the gradients of the non-expert parameters,
    # sleeps delay_ms and applies them `delay_steps` updates later): the trainer-side optimizer applies the gradient computed
    # `trainer_staleness` steps ago; experts keep updating themselves immediately, exactly like the reference
    trainer_staleness: int = 0
    # trainers per rank and step: the batch is split into this many micro-batches processed one after the other; the experts
    # step after EVERY micro-batch's backward (per-backward-batch updates of lib/runtime/expert_backend.py:90-97), the trainer
    # parameters once per step
    trainer_microbatches: int = 1
    # peer-flag wait timeout in ms (0 = ~10 s).  On expiry the waiting rank marks the step degraded (status bit) and goes on
    # with whatever arrived — the fused-path analogue of run_and_await_k's timeout_after_k_min (lib/utils/threading.py:76-125)
    peer_timeout_ms: int = 0

    def resolved_path(self, world: int = 1) -> str:
        if self.accumulate:
            return "big"      # gradient accumulation across steps needs the weight gradient in HBM (unfused wgrad + AMSGrad)
        if self.expert_path != "auto":
            return self.expert_path
        rows_per_expert = self.tokens_per_rank * world * self.k / max(1, self.num_experts)
        experts_per_rank = -(-self.num_experts // max(1, world))
        return "small" if (rows_per_expert < 512 and self.expert_dtype == "bf16" and self.inner % 128 == 0
                           and self.hidden % 128 == 0
                           and experts_per_rank <= 1023) else "big"   # swap-AB keeps a per-group prefix table in smem (MAX_G)

    @property
    def accumulate(self) -> bool:
        return self.update_every_inputs > 1 or self.update_every_steps > 1

    def update_thresholds(self) -> Tuple[int, int]:
        """(rows, steps) an expert must have pending to be stepped — either one suffices, like the reference's
        ``inputs >= update_every_inputs or steps >= update_every_steps``; 0 leaves that clause unset (never fires on its own)"""
        never = 2 ** 31 - 1
        return (self.update_every_inputs if self.update_every_inputs > 0 else never,
                self.update_every_steps if self.update_every_steps > 0 else never)

    @property
    def num_experts(self) -> int:
        return int(math.prod(self.grid_size))

    @property
    def inner(self) -> int:
        return 4 * self.hidden

    def seg_shapes(self) -> Dict[str, Tuple[int, ...]]:
        H, I = self.hidden, self.inner
        return {"w1": (I, H), "b1": (I,), "g1": (I,), "be1": (I,), "w2": (I, I), "b2": (I,), "g2": (I,), "be2": (I,),
                "w3": (H, I), "b3": (H,)}


def expert_uid(cfg: DMoEConfig, e: int) -> str:
    """global expert index -> 'prefix.i0.i1...' (row-major over the grid; reference uid schema README.md:106)"""
    parts = []
    for size in reversed(cfg.grid_size):
        parts.append(str(e % size))
        e //= size
    return ".".join([cfg.uid_prefix] + parts[::-1])


# =========================================================================================================
# process-wide context: symmetric heap, flags, epochs
# =========================================================================================================
class EngineContext:
    """Per-process state shared by all DMoE layers: symmetric heap, signal flags, scratch counters, epoch counter."""

    def __init__(self, cfg: DMoEConfig, group=None, device=None, heap_bytes: Optional[int] = None):
        from .symmetric import SymmetricHeap
        import torch.distributed as dist
        self.cfg = cfg
        self.device = device or torch.device("cuda", torch.cuda.current_device())
        distributed = dist.is_available() and dist.is_initialized()
        self.world = dist.get_world_size(group) if distributed else 1
        self.rank = dist.get_rank(group) if distributed else 0
        assert cfg.num_experts % self.world == 0, "experts must divide evenly over ranks"
        self.E = cfg.num_experts
        self.E_loc = self.E // self.world
        pairs = cfg.tokens_per_rank * cfg.k
        cap = pairs if self.world == 1 else int(math.ceil(pairs * cfg.capacity_factor))
        import os
        self.small = cfg.resolved_path(self.world) == "small"
        if self.small:
            # weight-streaming regime: hot-expert replicas would move 12.6 MB of weights to save a few rows -> static placement
            self.two_cta = False
            self.align = self.tile_rows = 16
            self.S = 0
        else:
            self.two_cta = cfg.two_cta and os.environ.get("LAH_TWO_CTA", "1") != "0" and cfg.inner % 256 == 0 \
                and cfg.hidden % 256 == 0
            self.align = 256 if self.two_cta else 128   # expert groups are padded to this many rows
            self.tile_rows = 128
            self.S = min(int(cfg.shadow_experts), 2 * K.MAX_WORLD) if self.world > 1 else 0   # shadow slots per rank / layer
        self.G_tot = self.E_loc + self.S
        self.max_rows = ((cap + self.align - 1) // self.align + self.G_tot) * self.align
        self.max_rows = (self.max_rows + 127) // 128 * 128
        self.max_tiles = self.max_rows // self.tile_rows
        H = cfg.hidden
        sym_rows_bytes = self.max_rows * H * 2
        need = (3 * cfg.num_layers + 2) * (sym_rows_bytes + 4096) + K.MAX_WORLD * self.E * 4 + (32 << 20)
        if self.S:  # parameters, bf16 mirror and gradients of the shards are peer-visible (replica pull / gradient reduce)
            rec = sum(int(math.prod(shape)) for shape in cfg.seg_shapes().values())
            need += cfg.num_layers * (self.G_tot * rec * 10 + (1 << 20))
        self.heap = SymmetricHeap(heap_bytes or need, group=group, device=self.device)
        self.flags, self.flags_off = self.heap.alloc((K.NUM_SLOTS, K.MAX_WORLD), torch.int32)
        self.cnt_all, self.cnt_all_off = self.heap.alloc((K.MAX_WORLD, self.E), torch.int32)
        i32 = dict(dtype=torch.int32, device=self.device)
        self.counts = torch.zeros(self.E, **i32)
        self.done_counter = torch.zeros(1, **i32)
        # [0] status bits; [2:4] = 64-bit counter of ns spent blocked on peer flags ("exposed" communication), written by
        # the wait loops of csrc/moe.cu (through lah_set_wait_counter) and by the receive-side wait fused into the GEMMs
        self._status_buf = torch.zeros(4, **i32)
        self.status = self._status_buf[:1]
        self.wait_ns = self._status_buf[2:4].view(torch.int64)
        K.set_wait_counter(self.wait_ns)
        # device-resident step counters: epochs / token offsets passed to the kernels are RELATIVE to them, so a captured
        # CUDA graph of a whole step stays valid from one replay to the next (see csrc/moe.cu Peers::step_ctr)
        self.step_ctr = torch.zeros(4, **i32)
        K.set_step_counters(self.step_ctr)
        K.set_spin_timeout_ms(cfg.peer_timeout_ms)
        self.step_ctr[1] = int(cfg.peer_timeout_ms)   # the GEMM producers read the timeout from the same device words
        self.dead_mask = 0                            # ranks excluded from every flag wait / reduce (host-decided)
        import os as _os
        octas = int(_os.environ.get("LAH_OPTIMIZER_CTAS", cfg.optimizer_ctas))
        sms = torch.cuda.get_device_properties(self.device).multi_processor_count
        if octas < 0:
            octas = sms * (11 if self.world == 1 else 9) // 14
        self.opt_ctas = octas if (self.small and 0 < octas < sms - 8) else 0     # CTAs of the optimizer stream (0: no overlap)
        self.chain_ctas = sms - self.opt_ctas if self.opt_ctas else 0            # CTA limit of the persistent chain kernels
        self.opt_stream = torch.cuda.Stream(self.device) if self.opt_ctas else None
        self._opt_pending = False
        self.defer_join = False   # DMoETrainer joins the optimizer stream itself, at the very end of its step
        K.set_poison_word(self.status)   # a step in which a peer timed out applies no optimizer update (the batch fails)
        assert 2 * cfg.num_layers + 4 < self.EPOCH_STRIDE
        self.alive = torch.ones(self.E, dtype=torch.uint8, device=self.device)
        # device-resident expert index shared by ALL ranks ("DHT collapse", SURVEY 5.8): hb[e] = last heartbeat (ms) of expert
        # e, stamped into every rank's copy by its owner (multimem.st through NVSwitch / P2P stores); refresh_alive() turns
        # it into the liveness mask the gate kernel reads.  All ones until heartbeats are used.
        self.hb, self.hb_off = self.heap.alloc((self.E,), torch.int64)
        self.hb.zero_()
        self._hb_stream = None
        self.epoch = 0
        self.token_counter = 0
        from .profiler import StageTimer
        self.timer = StageTimer(enabled=False)   # DMoETrainer(profile_stages=True) switches it on
        # transient backward buffers shared by all layers
        self.gyd, self.gyd_off = self.heap.alloc((self.max_rows, H), torch.bfloat16)
        self.dxd, self.dxd_off = self.heap.alloc((self.max_rows, H), torch.bfloat16)
        bf = dict(dtype=torch.bfloat16, device=self.device)
        self.da = torch.empty(self.max_rows, cfg.inner, **bf)
        self.dh = torch.empty(self.max_rows, cfg.inner, **bf)
        self.heap.barrier()

    EPOCH_STRIDE = 64   # epochs a step may consume; the device-side base advances by this much per begin_step()

    def close(self):
        """release the symmetric heap (peer mappings + the arena); idempotent.  All tensors carved out of the heap become
        invalid, so call it only when the trainer / layers of this context are no longer used."""
        K.set_wait_counter(None)
        K.set_step_counters(None)
        K.set_poison_word(None)
        self.heap.close()

    # ------------------------------------------------------------------ liveness (heartbeat -> device table -> gate kernel)
    def heartbeat(self, experts=None, now: Optional[float] = None):
        """declare my experts alive on EVERY rank (reference: NetworkHandlerThread -> declare_experts,
        /root/reference/lib/server/network_handler.py:17-20).  ``experts``: (first, count) range of GLOBAL expert ids hosted
        here, default all of mine.  Runs on a side stream so that a heartbeat thread never interleaves with a step."""
        import time
        first, count = experts if experts is not None else (self.rank * self.E_loc, self.E_loc)
        now_ms = int((time.time() if now is None else now) * 1000)
        if self._hb_stream is None:
            self._hb_stream = torch.cuda.Stream(self.device)
        with torch.cuda.stream(self._hb_stream):
            K.heartbeat(self.hb_off, first, count, now_ms)

    def refresh_alive(self, heartbeat_expiration: float = 120.0, now: Optional[float] = None):
        """alive[e] = heartbeat of e is younger than ``heartbeat_expiration`` seconds (on the device, no host copy)"""
        import time
        now_ms = int((time.time() if now is None else now) * 1000)
        if self._hb_stream is None:
            self._hb_stream = torch.cuda.Stream(self.device)
        with torch.cuda.stream(self._hb_stream):
            K.alive_from_heartbeats(self.hb, self.alive, now_ms, int(heartbeat_expiration * 1000))
            self._apply_dead_mask()

    # ------------------------------------------------------------------ failures (SURVEY 5.3): bounded waits, excluded ranks
    def step_failed(self) -> bool:
        """did a peer-flag wait time out since the last clear_failure()?  (synchronises).  A failed step applied NO optimizer
        update (the kernels check the status word) — the batch is lost, like a GatingFunction call with fewer than k_min
        responders (/root/reference/lib/utils/threading.py:120-125), the job is not."""
        return bool(int(self.status.item()) & K.STATUS_TIMEOUT)

    def clear_failure(self):
        self._status_buf[0] = 0

    def detect_dead_ranks(self, max_age: float, now: Optional[float] = None):
        """ranks none of whose experts sent a heartbeat during the last ``max_age`` seconds (every rank reads the SAME
        device-resident table, so the survivors agree without talking to each other)"""
        ages = self.heartbeat_ages(now).view(self.world, self.E_loc)
        return [r for r in range(self.world) if r != self.rank and float(ages[r].min()) > max_age]

    def exclude_ranks(self, ranks):
        """stop waiting for / reducing over ``ranks``: their flags are skipped by every wait, their dispatch counts read as
        zero, their experts disappear from the gate (softmax renormalises over the survivors), trainer gradients are
        averaged over the remaining ranks.  All survivors must exclude the same set (see detect_dead_ranks)."""
        for r in ranks:
            self.dead_mask |= 1 << int(r)
        self._status_buf[1] = self.dead_mask
        self._apply_dead_mask()
        self.clear_failure()

    def readmit_ranks(self, ranks):
        for r in ranks:
            self.dead_mask &= ~(1 << int(r))
        self._status_buf[1] = self.dead_mask

    def _apply_dead_mask(self):
        if self.dead_mask:
            view = self.alive.view(self.world, self.E_loc)
            for r in range(self.world):
                if (self.dead_mask >> r) & 1:
                    view[r] = 0

    def heartbeat_ages(self, now: Optional[float] = None) -> torch.Tensor:
        """seconds since the last heartbeat of every expert (inf = never declared); synchronises"""
        import time
        if self._hb_stream is not None:
            self._hb_stream.synchronize()
        hb = self.hb.cpu().double()
        now_ms = (time.time() if now is None else now) * 1000
        return torch.where(hb > 0, (now_ms - hb) / 1000.0, torch.full_like(hb, float("inf")))

    def join_optimizer_stream(self):
        """the launching stream waits for the fused wgrad+AMSGrad kernels of this step (they run on `opt_stream`); called once
        per step before anything may read the updated weights.  Inside a CUDA-graph capture this is a graph edge."""
        if self.opt_stream is not None and self._opt_pending:
            torch.cuda.current_stream(self.device).wait_stream(self.opt_stream)
            self._opt_pending = False

    def begin_step(self):
        """advance the device-side epoch / token bases (one tiny kernel) and restart the step-relative counters; called at
        the top of every training / evaluation step by ALL ranks (collective by construction: every rank runs the same
        program).  Inside a captured CUDA graph the bump is part of the graph."""
        K.step_begin(self.EPOCH_STRIDE, self.cfg.num_layers * self.cfg.tokens_per_rank)
        self.epoch = 0
        self.token_counter = 0

    def next_epoch(self) -> int:
        if self.epoch + 1 >= self.EPOCH_STRIDE:   # a caller that never begins steps (layer-level tests) wraps here
            self.begin_step()
        self.epoch += 1
        return self.epoch

    def exposed_wait_ms(self, reset: bool = True) -> float:
        """ms this rank's stream was blocked on peer flags since the last reset (synchronises)"""
        ms = float(self.wait_ns.item()) * 1e-6
        if reset:
            self.wait_ns.zero_()
        return ms

    def check_status(self):
        """host-side check of the device status word (synchronises); raises on timeouts / capacity overflow"""
        code = int(self.status.item())
        if code & K.STATUS_TIMEOUT:
            raise RuntimeError("DMoE engine: timed out waiting for a peer GPU (dead rank?)")
        if code & K.STATUS_OVERFLOW:
            raise RuntimeError("DMoE engine: expert receive buffer overflow; raise DMoEConfig.capacity_factor")


# =========================================================================================================
# expert parameters of one DMoE layer hosted on this rank
# =========================================================================================================
class ExpertShard:
    """Stacked parameters / gradients / Adam state of the E_loc local experts of one layer (flat fp32 buffers, segments
    [E_loc, size] per tensor kind) plus the bf16 mirror consumed by the GEMMs."""

    def __init__(self, cfg: DMoEConfig, E_loc: int, first_expert: int, device, layer_index: int = 0, ctx=None):
        self.cfg, self.E_loc, self.first_expert = cfg, E_loc, first_expert
        # slots = owned experts + shadow slots (replicas of other ranks' hot experts, only on multi-GPU runs)
        self.slots = slots = E_loc + (ctx.S if ctx is not None else 0)
        shapes = cfg.seg_shapes()
        self.seg_sizes = [int(math.prod(shapes[n])) for n in SEG_NAMES]
        total = sum(self.seg_sizes) * slots
        f32 = dict(dtype=torch.float32, device=device)
        self.p_off = self.g_off = self.pbf16_off = -1
        if ctx is not None and ctx.S > 0:   # peer-visible: replicas are pulled from p / p_bf16, partial grads read from g
            self.p, self.p_off = ctx.heap.alloc((total,), torch.float32)
            self.g, self.g_off = ctx.heap.alloc((total,), torch.float32)
            self.p_bf16, self.pbf16_off = ctx.heap.alloc((total,), torch.bfloat16)
            self.p.zero_(), self.g.zero_(), self.p_bf16.zero_()
        else:
            self.p = torch.zeros(total, **f32)
            self.g = torch.zeros(total, **f32)
            self.p_bf16 = torch.zeros(total, dtype=torch.bfloat16, device=device)
        self.m = torch.zeros(total, **f32)
        self.v = torch.zeros(total, **f32)
        self.vmax = torch.zeros(total, **f32) if cfg.amsgrad else None
        self.step = torch.zeros(E_loc, dtype=torch.int32, device=device)
        self.views: Dict[str, torch.Tensor] = {}
        self.grads: Dict[str, torch.Tensor] = {}
        self.bf16: Dict[str, torch.Tensor] = {}
        self.m_views: Dict[str, torch.Tensor] = {}
        self.v_views: Dict[str, torch.Tensor] = {}
        self.vmax_views: Dict[str, torch.Tensor] = {}
        off = 0
        for name, size in zip(SEG_NAMES, self.seg_sizes):
            sl = slice(off, off + size * slots)
            self.views[name] = self.p[sl].view(slots, *shapes[name])
            self.grads[name] = self.g[sl].view(slots, *shapes[name])
            self.bf16[name] = self.p_bf16[sl].view(slots, *shapes[name])
            self.m_views[name] = self.m[sl].view(slots, *shapes[name])
            self.v_views[name] = self.v[sl].view(slots, *shapes[name])
            if self.vmax is not None:
                self.vmax_views[name] = self.vmax[sl].view(slots, *shapes[name])
            off += size * slots
        # asynchronous-update bookkeeping (DMoEConfig.update_every_*): rows / steps pending since the last optimizer step
        self.pending_rows = torch.zeros(E_loc, dtype=torch.int32, device=device)
        self.pending_steps = torch.zeros(E_loc, dtype=torch.int32, device=device)
        self.fire = torch.zeros(E_loc, dtype=torch.int32, device=device)
        self.w8 = None        # MXFP8 copies of w1/w2/w3 (expert_dtype == "fp8"), refreshed lazily from the bf16 mirror
        self.w8_dirty = True
        if cfg.expert_dtype == "fp8" and ctx is not None:
            self.w8 = {n: fp8.MXFP8Tensor(shapes[n][0], slots, shapes[n][1], fp8.WEIGHT_TILE, device)
                       for n in ("w1", "w2", "w3")}
        self.reset_parameters(layer_index)

    @torch.no_grad()
    def reset_parameters(self, layer_index: int = 0):
        """nn.Linear / nn.LayerNorm default initialisation, seeded per (layer, global expert) so that the same expert
        gets the same weights regardless of the number of ranks"""
        cfg = self.cfg
        dev = self.p.device
        for le in range(self.E_loc):
            gen = torch.Generator(device=dev)
            gen.manual_seed(cfg.seed * 1000003 + layer_index * 10007 + self.first_expert + le)
            for w, b in (("w1", "b1"), ("w2", "b2"), ("w3", "b3")):
                fan_in = self.views[w].shape[-1]
                bound = 1.0 / math.sqrt(fan_in)
                self.views[w][le].uniform_(-bound, bound, generator=gen)
                self.views[b][le].uniform_(-bound, bound, generator=gen)
            for gname, bname in (("g1", "be1"), ("g2", "be2")):
                self.views[gname][le].fill_(1.0)
                self.views[bname][le].zero_()
        self.sync_bf16()

    def fp8_weights(self):
        """MXFP8 weights of all slots, re-quantised from the bf16 mirror when it changed (optimizer step / replica pull)"""
        if self.w8_dirty:
            for n, t in self.w8.items():
                fp8.quantize(self.bf16[n].view(-1, t.K), tile_rows=fp8.WEIGHT_TILE, groups=self.slots, out=t)
            self.w8_dirty = False
        return self.w8

    def sync_bf16(self):
        self.w8_dirty = True
        if self.p.is_cuda:
            K.cast_bf16(self.p, self.p_bf16)
        else:
            self.p_bf16.copy_(self.p)

    # ------------------------------------------------------------------ checkpoint layout (SURVEY.md §5.4)
    def expert_state_dict(self, le: int, prefix: str = "expert.") -> Dict[str, torch.Tensor]:
        """state of local expert `le` with the key names of ``ExpertBackend.state_dict()`` of the reference"""
        return {prefix + REF_KEYS[n]: self.views[n][le].detach().clone().cpu() for n in SEG_NAMES}

    def expert_optimizer_state(self, le: int) -> Dict:
        """torch.optim.Adam-compatible state_dict of local expert `le` (parameter order = module.parameters())"""
        state = {}
        for i, n in enumerate(SEG_NAMES):
            off = self._seg_offset(n) + le * self.seg_sizes[i]
            sl = slice(off, off + self.seg_sizes[i])
            shape = self.views[n].shape[1:]
            entry = dict(step=torch.tensor(float(self.step[le].item())), exp_avg=self.m[sl].view(shape).clone().cpu(),
                         exp_avg_sq=self.v[sl].view(shape).clone().cpu())
            if self.vmax is not None:
                entry["max_exp_avg_sq"] = self.vmax[sl].view(shape).clone().cpu()
            state[i] = entry
        cfg = self.cfg
        group = dict(lr=cfg.lr, betas=cfg.betas, eps=cfg.eps, weight_decay=0, amsgrad=cfg.amsgrad,
                     params=list(range(len(SEG_NAMES))))
        return dict(state=state, param_groups=[group])

    def load_expert_state_dict(self, le: int, state: Dict[str, torch.Tensor], prefix: str = "expert."):
        with torch.no_grad():
            for n in SEG_NAMES:
                self.views[n][le].copy_(state[prefix + REF_KEYS[n]])
        self.sync_bf16()

    def load_expert_optimizer_state(self, le: int, opt_state: Dict):
        with torch.no_grad():
            for i, n in enumerate(SEG_NAMES):
                entry = opt_state["state"].get(i)
                if entry is None:
                    continue
                off = self._seg_offset(n) + le * self.seg_sizes[i]
                sl = slice(off, off + self.seg_sizes[i])
                self.m[sl].copy_(entry["exp_avg"].reshape(-1))
                self.v[sl].copy_(entry["exp_avg_sq"].reshape(-1))
                if self.vmax is not None and "max_exp_avg_sq" in entry:
                    self.vmax[sl].copy_(entry["max_exp_avg_sq"].reshape(-1))
                self.step[le] = int(entry["step"])

    def _seg_offset(self, name: str) -> int:
        off = 0
        for n, size in zip(SEG_NAMES, self.seg_sizes):
            if n == name:
                return off
            off += size * self.slots
        raise KeyError(name)


# =========================================================================================================
# per-layer workspace (activations that stay resident between forward and backward)
# =========================================================================================================
class LayerWorkspace:
    def __init__(self, ctx: EngineContext):
        cfg, dev, R = ctx.cfg, ctx.device, ctx.max_rows
        H, I = cfg.hidden, cfg.inner
        bf = dict(dtype=torch.bfloat16, device=dev)
        i32 = dict(dtype=torch.int32, device=dev)
        f32 = dict(dtype=torch.float32, device=dev)
        self.xd, self.xd_off = ctx.heap.alloc((R, H), torch.bfloat16)   # dispatched inputs (peers push)
        self.yo, self.yo_off = ctx.heap.alloc((R, H), torch.bfloat16)   # expert outputs (peers pull)
        self.h1, self.a1 = torch.empty(R, I, **bf), torch.empty(R, I, **bf)
        self.h2, self.a2 = torch.empty(R, I, **bf), torch.empty(R, I, **bf)
        self.xq = self.aq = None
        if cfg.expert_dtype == "fp8":   # MXFP8 operands of the forward GEMMs (aq is shared by a1 and a2)
            self.xq = fp8.MXFP8Tensor(R, 1, H, fp8.ACT_TILE, dev)
            self.aq = fp8.MXFP8Tensor(R, 1, I, fp8.ACT_TILE, dev)
        self.mean1, self.rstd1 = torch.empty(R, **f32), torch.empty(R, **f32)
        self.mean2, self.rstd2 = torch.empty(R, **f32), torch.empty(R, **f32)
        P = cfg.tokens_per_rank * cfg.k
        self.idx, self.pos, self.pair_row = torch.empty(P, **i32), torch.empty(P, **i32), torch.empty(P, **i32)
        self.w = torch.empty(P, **f32)
        self.dst_row = torch.empty(ctx.E, **i32)
        self.route_owner = torch.zeros(ctx.E, **i32)            # rank whose buffer holds MY rows of expert e
        self.group_off = torch.zeros(ctx.G_tot + 1, **i32)      # owned experts, then shadow slots
        self.group_rows = torch.zeros(ctx.G_tot, **i32)         # rows in MY buffer per group
        self.step_rows = torch.zeros(ctx.E_loc, **i32)          # global rows per owned expert (optimizer gating, stats)
        self.shadow_info = torch.full((max(ctx.S, 1) * 4,), -1, **i32)
        self.owned_shadow = torch.full((ctx.E_loc * 2,), -1, **i32)
        self.tile_group = torch.full((ctx.max_tiles,), -1, **i32)
        self.total_rows = torch.zeros(1, **i32)
        self.outstanding = False   # a training-mode forward whose backward has not run yet owns this workspace
        # small path with optimizer overlap: the fused wgrad+AMSGrad kernels of layer L read dY buffers while the main stream is
        # already in the backward of layer L-1, so they must be per layer (a few MB each at this batch size)
        if ctx.small and ctx.opt_stream is not None:
            self.gyd, self.gyd_off = ctx.heap.alloc((R, H), torch.bfloat16)
            self.dh2, self.dh1 = torch.zeros(R, I, **bf), torch.zeros(R, I, **bf)
        else:
            self.gyd, self.gyd_off, self.dh2, self.dh1 = ctx.gyd, ctx.gyd_off, ctx.dh, ctx.dh


# =========================================================================================================
# the DMoE layer
# =========================================================================================================
class _FusedDMoEFunction(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, logits, layer):
        ctx.layer = layer
        ctx.B = x.shape[0]
        ws = layer.ws
        if ws.outstanding:
            raise RuntimeError("FusedDMoE: forward() called again before the backward of the previous training-mode forward "
                               "(activations of a layer are single-buffered; run evaluate() / the next micro-batch after "
                               "backward, or call layer.release_workspace() to drop the pending forward)")
        ctx.tracked = bool(x.requires_grad or logits.requires_grad)
        ws.outstanding = ctx.tracked
        return layer._forward_cuda(x, logits)

    @staticmethod
    def backward(ctx, grad_out):
        if not ctx.layer.ws.outstanding:
            raise RuntimeError("FusedDMoE: backward() without a pending forward (the workspace was released or reused)")
        dx, dlogits = ctx.layer._backward_cuda(grad_out.contiguous(), ctx.B)
        ctx.layer.ws.outstanding = False
        ec = ctx.layer.ctx
        if ec._opt_pending and not ec.defer_join:
            # layer-level callers (no DMoETrainer): when the whole backward pass is over, the launching stream waits for the
            # expert optimizers on the second stream, so reading the parameters right after backward() is safe
            torch.autograd.Variable._execution_engine.queue_callback(ec.join_optimizer_stream)
        return dx, dlogits, None


class FusedDMoE(nn.Module):
    """
    Decentralized-MoE layer over the experts of the whole box.  Trainer-side parameters: ``proj`` (product-key gating,
    identical to ``GatingFunction.proj``: Linear(in_features, sum(grid_size))).  Expert parameters live in
    ``self.shard`` and are updated by the layer itself during backward (they are NOT nn.Parameters, mirroring
    ``get_non_expert_params`` of the reference emulator).
    """

    def __init__(self, cfg: DMoEConfig, ctx: Optional[EngineContext] = None, layer_index: int = 0, device=None):
        super().__init__()
        self.cfg, self.ctx, self.layer_index = cfg, ctx, layer_index
        self.grid_size = tuple(cfg.grid_size)
        if cfg.gate_mode == "emulator":
            assert len(self.grid_size) == 1, "gate_mode='emulator' scores experts densely: use grid_size=(num_experts,)"
            self.gating_pre_normalize = nn.LayerNorm(cfg.hidden)
            self.expert_keys = nn.Parameter(torch.randn(cfg.hidden, cfg.num_experts), requires_grad=False)
            self.gating_pre_normalize.requires_grad_(False)
            self.proj = None
        else:
            self.proj = nn.Linear(cfg.hidden, sum(cfg.grid_size))
        if ctx is not None:
            self.E_loc, self.first_expert, dev = ctx.E_loc, ctx.rank * ctx.E_loc, ctx.device
            self.ws = LayerWorkspace(ctx)
        else:  # CPU / oracle mode: all experts local
            self.E_loc, self.first_expert, dev = cfg.num_experts, 0, device or torch.device("cpu")
            self.ws = None
        self.shard = ExpertShard(cfg, self.E_loc, self.first_expert, dev, layer_index, ctx=ctx)
        self.ref_fail_mask = None  # tests can inject an explicit failure mask into the oracle path
        self.ref_emulate_bf16 = False   # oracle path: round activations / weights to bf16 where the GPU path stores bf16
        self._ref_rows = None
        self._ref_leaves = {}   # CPU mode: local expert -> {segment: leaf view} of the experts used since the last update

    # ------------------------------------------------------------------ public forward
    def forward(self, x):
        return self.forward_with_gate(x, self.proj)

    def gate_logits(self, x, proj=None):
        if self.cfg.gate_mode == "emulator" and proj is None:
            if x.is_cuda and x.dtype == torch.bfloat16:
                # trainer-side gate on the activation dtype: one bf16 LayerNorm + one small tensor-core GEMM instead of
                # fp32 casts of the whole [B, H] activation (4 % of the step); accumulation stays fp32 inside the ops.
                # The gate parameters are frozen (like the reference emulator's): their bf16 / normalised forms are cached
                # (keyed on the tensors' version counters), which removes four small kernels per layer and step
                ln = self.gating_pre_normalize
                key = (self.expert_keys._version, ln.weight._version, ln.bias._version, self.expert_keys.data_ptr())
                if getattr(self, "_gate_cache_key", None) != key:
                    with torch.no_grad():
                        self._gate_cache = (ln.weight.to(x.dtype), ln.bias.to(x.dtype),
                                            F.normalize(self.expert_keys, dim=-1).to(x.dtype).contiguous())
                    self._gate_cache_key = key
                w_ln, b_ln, keys = self._gate_cache
                xn = F.layer_norm(x, (x.shape[-1],), w_ln, b_ln, ln.eps)
                return (xn @ keys).float()
            return self.gating_pre_normalize(x.float()) @ F.normalize(self.expert_keys, dim=-1)
        return F.linear(x.float(), proj.weight, proj.bias)

    def forward_with_gate(self, x, proj: Optional[nn.Linear]):
        """run the layer with an externally owned gate (``lib.GatingFunction.proj`` on the fused in-box path)"""
        assert x.dim() == 2 and x.shape[1] == self.cfg.hidden
        logits = self.gate_logits(x, proj)
        if self.ctx is None:
            return self._forward_ref(x, logits, emulate_bf16=self.ref_emulate_bf16)
        assert x.shape[0] <= self.cfg.tokens_per_rank, "batch exceeds DMoEConfig.tokens_per_rank"
        return _FusedDMoEFunction.apply(x.to(torch.bfloat16).contiguous(), logits.contiguous(), self)

    def release_workspace(self):
        """forget a training-mode forward whose backward will never run (e.g. an exception between forward and backward)"""
        if self.ws is not None:
            self.ws.outstanding = False

    # ------------------------------------------------------------------ sm_90a path
    def _forward_cuda(self, x, logits):
        c, ws, sh, cfg = self.ctx, self.ws, self.shard, self.cfg
        B, k = x.shape[0], cfg.k
        P = B * k
        c.join_optimizer_stream()   # no-op inside DMoETrainer steps (joined there); protects layer-level callers
        epoch = c.next_epoch()
        idx, w, pos, pair_row = ws.idx[:P], ws.w[:P], ws.pos[:P], ws.pair_row[:P]
        K.gate_topk(logits, self.grid_size, k, alive=c.alive, failure_rate=cfg.failure_rate if self.training else 0.0,
                    seed=cfg.seed * 7919 + self.layer_index, token_offset=c.token_counter, idx=idx, w=w, pos=pos,
                    counts=c.counts)
        c.token_counter += B
        c.timer.mark("gate_topk")
        K.layout_exchange(c.cnt_all_off, c.flags_off, K.SLOT_COUNTS, epoch, c.E, c.E_loc, c.max_rows, align=c.align,
                          tile_rows=c.tile_rows, counts=c.counts,
                          dst_row=ws.dst_row, group_off=ws.group_off, group_rows=ws.group_rows,
                          tile_group=ws.tile_group, total_rows=ws.total_rows, status=c.status, shadow_slots=c.S,
                          shadow_tol=cfg.shadow_tol, min_shadow_rows=cfg.shadow_min_rows, route_owner=ws.route_owner,
                          step_rows=ws.step_rows, shadow_info=ws.shadow_info, owned_shadow=ws.owned_shadow)
        if c.S:  # replicas of this step's hot experts: weights from the owners' bf16 mirror, small params from fp32
            K.pull_shadow(ws.shadow_info, c.S, c.E_loc, sh.p_off, sh.pbf16_off, sh.seg_sizes, SMALL_SEG_MASK)
            sh.w8_dirty = True
        K.scatter_rows(x, None, idx, pos, ws.dst_row, pair_row, ws.xd_off, c.flags_off, K.SLOT_DISPATCH, epoch, k,
                       c.E_loc, c.max_rows, ws.group_off, ws.group_rows, c.done_counter, c.status, align=c.align,
                       route_owner=ws.route_owner, num_groups=c.G_tot)
        c.timer.mark("dispatch(layout+pull+scatter)")
        # ---- expert FFN on the rows this rank received (grouped by expert).  Receive-side fusion: the first GEMM's TMA
        # producer polls the peers' dispatch flags itself (no separate wait kernel)
        tg = ws.tile_group
        wait = (c.flags[K.SLOT_DISPATCH, :c.world], epoch, c.status) if c.world > 1 else None
        if c.small:
            # weight-streaming regime: swap-AB tiles (weights on MMA-M, the group's 16..128 tokens on MMA-N), groups of 16 rows
            go, gr_, T = ws.group_off, ws.group_rows, c.tile_rows
            K.swapab_linear(ws.xd, sh.bf16["w1"], go, gr_, out=ws.h1, bias=sh.views["b1"], wait=wait)
            K.ln_relu_fwd(ws.h1, sh.views["g1"], sh.views["be1"], tg, out=ws.a1, mean=ws.mean1, rstd=ws.rstd1, tile_rows=T)
            K.swapab_linear(ws.a1, sh.bf16["w2"], go, gr_, out=ws.h2, bias=sh.views["b2"])
            K.ln_relu_fwd(ws.h2, sh.views["g2"], sh.views["be2"], tg, out=ws.a2, mean=ws.mean2, rstd=ws.rstd2, tile_rows=T)
            K.swapab_linear(ws.a2, sh.bf16["w3"], go, gr_, out=ws.yo, bias=sh.views["b3"], residual=ws.xd)
        elif cfg.expert_dtype == "fp8":
            self._expert_ffn_fp8(wait, epoch)
        else:
            gemm.grouped_linear(ws.xd, sh.bf16["w1"], tile_group=tg, bias=sh.views["b1"], out=ws.h1, two_cta=c.two_cta,
                                wait=wait)
            K.ln_relu_fwd(ws.h1, sh.views["g1"], sh.views["be1"], tg, out=ws.a1, mean=ws.mean1, rstd=ws.rstd1)
            gemm.grouped_linear(ws.a1, sh.bf16["w2"], tile_group=tg, bias=sh.views["b2"], out=ws.h2, two_cta=c.two_cta)
            K.ln_relu_fwd(ws.h2, sh.views["g2"], sh.views["be2"], tg, out=ws.a2, mean=ws.mean2, rstd=ws.rstd2)
            gemm.grouped_linear(ws.a2, sh.bf16["w3"], tile_group=tg, bias=sh.views["b3"], residual=ws.xd, out=ws.yo,
                                two_cta=c.two_cta)
        c.timer.mark("expert_ffn_fwd")
        y = torch.empty(B, cfg.hidden, dtype=torch.bfloat16, device=x.device)
        K.combine_rows(ws.yo_off, idx, pair_row, w, y, k, c.E_loc, flags_off=c.flags_off, slot=K.SLOT_OUTPUT, epoch=epoch,
                       signal=c.world > 1, wait=c.world > 1, status=c.status, route_owner=ws.route_owner)
        c.timer.mark("combine")
        return y

    def _expert_ffn_fp8(self, wait, epoch):
        """forward GEMMs on block-scaled FP8 tensor cores; LayerNorm emits the next GEMM's MXFP8 operand directly (and the
        bf16 copy the bf16 wgrad needs)"""
        c, ws, sh = self.ctx, self.ws, self.shard
        assert c.two_cta, "the FP8 path needs the 256-row expert groups of the wide-tile layout (hidden and 4*hidden multiples of 256)"
        tg = ws.tile_group
        if wait is not None:  # the quantiser is the first consumer of the rows pushed by the peers
            K.signal_wait(c.flags_off, K.SLOT_DISPATCH, epoch, c.status, signal=False, wait=True)
        w8 = sh.fp8_weights()
        fp8.quantize(ws.xd, tile_group=tg, out=ws.xq)
        fp8.grouped_linear_fp8(ws.xq, w8["w1"], tile_group=tg, bias=sh.views["b1"], out=ws.h1)
        K.ln_relu_fwd(ws.h1, sh.views["g1"], sh.views["be1"], tg, out=ws.a1, mean=ws.mean1, rstd=ws.rstd1, quant=ws.aq)
        fp8.grouped_linear_fp8(ws.aq, w8["w2"], tile_group=tg, bias=sh.views["b2"], out=ws.h2)
        K.ln_relu_fwd(ws.h2, sh.views["g2"], sh.views["be2"], tg, out=ws.a2, mean=ws.mean2, rstd=ws.rstd2, quant=ws.aq)
        fp8.grouped_linear_fp8(ws.aq, w8["w3"], tile_group=tg, bias=sh.views["b3"], residual=ws.xd, out=ws.yo)

    def _backward_cuda(self, gy, B):
        c, ws, sh, cfg = self.ctx, self.ws, self.shard, self.cfg
        k = cfg.k
        P = B * k
        epoch = c.next_epoch()
        idx, w, pos, pair_row = ws.idx[:P], ws.w[:P], ws.pos[:P], ws.pair_row[:P]
        gy = gy.to(torch.bfloat16)
        dlogits = torch.empty(B, sum(self.grid_size), dtype=torch.float32, device=gy.device)
        K.gate_bwd(ws.yo_off, gy, idx, pair_row, w, dlogits, k, c.E_loc, self.grid_size, route_owner=ws.route_owner)
        K.scatter_rows(gy, w, idx, pos, None, pair_row, ws.gyd_off, c.flags_off, K.SLOT_GRAD, epoch, k, c.E_loc,
                       c.max_rows, ws.group_off, ws.group_rows, c.done_counter, c.status, align=c.align,
                       route_owner=ws.route_owner, num_groups=c.G_tot)
        if c.S:  # atomically accumulated (bias / LayerNorm) partial gradients of my shadow slots start from zero
            K.zero_slots(sh.g, sh.seg_sizes, c.G_tot, c.E_loc, c.S, SMALL_SEG_MASK)
        if c.world > 1:  # the first consumers of the pushed gradients are the colsum / wgrad kernels
            K.signal_wait(c.flags_off, K.SLOT_GRAD, epoch, c.status, signal=False, wait=True)
        c.timer.mark("bwd_gate+dispatch_grad")
        tg, go, G = ws.tile_group, ws.group_off, c.G_tot
        gr = sh.grads
        if c.small:
            self._backward_small(epoch)
            c.timer.mark("expert_ffn_bwd(dgrad+ln+fused wgrad/AMSGrad)")
            dx = torch.empty(B, cfg.hidden, dtype=torch.bfloat16, device=gy.device)
            K.combine_rows(c.dxd_off, idx, pair_row, None, dx, k, c.E_loc, flags_off=c.flags_off, slot=K.SLOT_DINPUT,
                           epoch=epoch, signal=c.world > 1, wait=c.world > 1, status=c.status, route_owner=ws.route_owner)
            c.timer.mark("bwd_combine")
            return dx, dlogits
        K.grouped_colsum(c.gyd, tg, out=gr["b3"])
        gemm.grouped_wgrad(c.gyd, ws.a2, go, G, out=gr["w3"], two_cta=c.two_cta, accumulate=cfg.accumulate)
        gemm.grouped_linear(c.gyd, sh.bf16["w3"], tile_group=tg, w_is_kn=True, out=c.da, two_cta=c.two_cta)
        K.ln_relu_bwd(c.da, ws.h2, ws.mean2, ws.rstd2, sh.views["g2"], sh.views["be2"], tg, dh=c.dh, dgamma=gr["g2"],
                      dbeta=gr["be2"], dbias=gr["b2"])
        gemm.grouped_wgrad(c.dh, ws.a1, go, G, out=gr["w2"], two_cta=c.two_cta, accumulate=cfg.accumulate)
        gemm.grouped_linear(c.dh, sh.bf16["w2"], tile_group=tg, w_is_kn=True, out=c.da, two_cta=c.two_cta)
        K.ln_relu_bwd(c.da, ws.h1, ws.mean1, ws.rstd1, sh.views["g1"], sh.views["be1"], tg, dh=c.dh, dgamma=gr["g1"],
                      dbeta=gr["be1"], dbias=gr["b1"])
        gemm.grouped_wgrad(c.dh, ws.xd, go, G, out=gr["w1"], two_cta=c.two_cta, accumulate=cfg.accumulate)
        gemm.grouped_linear(c.dh, sh.bf16["w1"], tile_group=tg, w_is_kn=True, residual=c.gyd, out=c.dxd,
                            two_cta=c.two_cta)
        c.timer.mark("expert_ffn_bwd(wgrad+dgrad+ln)")
        # ---- expert-side optimizer step (reference: ExpertBackend.apply_gradients right after backward)
        if c.S:  # the owners read every rank's partial gradients of the shadowed experts: all ranks must be done
            K.signal_wait(c.flags_off, K.SLOT_SHADOW, epoch, c.status, signal=True, wait=True)
        self.apply_expert_gradients()
        c.timer.mark("expert_adam")
        dx = torch.empty(B, cfg.hidden, dtype=torch.bfloat16, device=gy.device)
        K.combine_rows(c.dxd_off, idx, pair_row, None, dx, k, c.E_loc, flags_off=c.flags_off, slot=K.SLOT_DINPUT,
                       epoch=epoch, signal=c.world > 1, wait=c.world > 1, status=c.status, route_owner=ws.route_owner)
        c.timer.mark("bwd_combine")
        return dx, dlogits

    def _backward_small(self, epoch):
        """expert backward of the weight-streaming regime.  Order matters: the dgrad of a Linear reads the OLD weights, so
        it runs before the fused wgrad+AMSGrad kernel of the same matrix updates them in place (reference: the optimizer
        step follows the whole backward, lib/runtime/expert_backend.py:85-90)."""
        c, ws, sh, cfg = self.ctx, self.ws, self.shard, self.cfg
        tg, go, rows, T = ws.tile_group, ws.group_off, ws.group_rows, c.tile_rows
        gr = sh.grads
        opt = dict(lr=cfg.lr, betas=cfg.betas, eps=cfg.eps, amsgrad=cfg.amsgrad)
        main = torch.cuda.current_stream(c.device)
        side, chain_ctas = c.opt_stream, c.chain_ctas

        def wgrad(name, dy, x):
            """dW never reaches HBM: register accumulator -> AMSGrad epilogue -> p / m / v / vmax updated in place.  With the overlap
            enabled the kernel goes to the optimizer stream, ordered after everything the main stream has launched so far (in
            particular the dgrad that still reads the OLD weights); its inputs live in per-layer buffers."""
            kw = dict(p=sh.views[name][:self.E_loc], m=sh.m_views[name][:self.E_loc], v=sh.v_views[name][:self.E_loc],
                      vmax=sh.vmax_views[name][:self.E_loc] if cfg.amsgrad else None, p_bf16=sh.bf16[name], step=sh.step, **opt)
            if side is None:
                K.wgrad_adam(dy, x, go, rows, **kw)
                return
            side.wait_stream(main)
            with torch.cuda.stream(side):
                K.wgrad_adam(dy, x, go, rows, max_ctas=c.opt_ctas, **kw)
            c._opt_pending = True

        gyd, dh2, dh1 = ws.gyd, ws.dh2, ws.dh1
        K.bump_steps(sh.step, ws.step_rows)
        K.grouped_colsum(gyd, tg, out=gr["b3"], tile_rows=T)
        K.swapab_linear(gyd, sh.bf16["w3"], go, rows, out=c.da, w_is_kn=True, max_ctas=chain_ctas)
        wgrad("w3", gyd, ws.a2)
        K.ln_relu_bwd(c.da, ws.h2, ws.mean2, ws.rstd2, sh.views["g2"], sh.views["be2"], tg, dh=dh2, dgamma=gr["g2"],
                      dbeta=gr["be2"], dbias=gr["b2"], tile_rows=T)
        K.swapab_linear(dh2, sh.bf16["w2"], go, rows, out=c.da, w_is_kn=True, max_ctas=chain_ctas)
        wgrad("w2", dh2, ws.a1)
        K.ln_relu_bwd(c.da, ws.h1, ws.mean1, ws.rstd1, sh.views["g1"], sh.views["be1"], tg, dh=dh1, dgamma=gr["g1"],
                      dbeta=gr["be1"], dbias=gr["b1"], tile_rows=T)
        K.swapab_linear(dh1, sh.bf16["w1"], go, rows, out=c.dxd, w_is_kn=True, residual=gyd, max_ctas=chain_ctas)
        wgrad("w1", dh1, ws.xd)
        # biases / LayerNorm affine: the ordinary fused AMSGrad restricted to the small segments
        K.adam_step(sh.p, sh.g, sh.m, sh.v, sh.vmax, sh.p_bf16, sh.seg_sizes, sh.slots, step=sh.step,
                    group_rows=ws.step_rows, zero_mask=SMALL_SEG_MASK, G_active=self.E_loc, seg_mask=SMALL_SEG_MASK, **opt)
        sh.w8_dirty = True

    def apply_expert_gradients(self):
        sh, cfg, ws, c = self.shard, self.cfg, self.ws, self.ctx
        rows, zero_mask = ws.step_rows, SMALL_SEG_MASK
        if cfg.accumulate:
            # asynchronous expert updates (dmoe_emulator.py:70-77): gradients accumulate in sh.g (wgrad accumulate=True) until
            # the expert has seen >= update_every_inputs rows or >= update_every_steps steps since its first pending row
            sh.pending_rows += ws.step_rows
            sh.pending_steps += (sh.pending_rows > 0).to(torch.int32)
            thr_rows, thr_steps = cfg.update_thresholds()
            due = (sh.pending_rows > 0) & ((sh.pending_rows >= thr_rows) | (sh.pending_steps >= thr_steps))
            sh.fire.copy_(due.to(torch.int32))
            sh.pending_rows.mul_(1 - sh.fire)
            sh.pending_steps.mul_(1 - sh.fire)
            rows, zero_mask = sh.fire, (1 << len(SEG_NAMES)) - 1
        K.bump_steps(sh.step, rows)
        K.adam_step(sh.p, sh.g, sh.m, sh.v, sh.vmax, sh.p_bf16, sh.seg_sizes, sh.slots, step=sh.step,
                    group_rows=rows, lr=cfg.lr, betas=cfg.betas, eps=cfg.eps, amsgrad=cfg.amsgrad,
                    zero_mask=zero_mask, G_active=self.E_loc, world=c.world,
                    peer_bases=c.heap.peer_bases if c.S else None, shadow_of=ws.owned_shadow if c.S else None,
                    shadow_g_off=sh.g_off, me=c.rank)
        sh.w8_dirty = True

    def failure_rate_ref(self) -> float:
        return self.cfg.failure_rate if (self.training and self.ctx is None) else 0.0

    # ------------------------------------------------------------------ PyTorch oracle (CPU path, tests)
    def _expert_params(self, e_local: int, dtype=torch.float32):
        if self.ctx is None and torch.is_grad_enabled() and self.training:
            # CPU mode: every parameter of the expert is a LEAF VIEW into the flat buffer (detached, same storage), so
            # autograd produces one small gradient per tensor; apply_expert_gradients_ref copies them into shard.g.
            # (Slicing one big leaf instead makes autograd materialise a full-size zero tensor per slice.)
            leaves = self._ref_leaves.get(e_local)
            if leaves is None:
                leaves = {n: self.shard.views[n][e_local].detach().requires_grad_(True) for n in SEG_NAMES}
                self._ref_leaves[e_local] = leaves
            return leaves
        return {n: self.shard.views[n][e_local].to(dtype) for n in SEG_NAMES}

    def apply_expert_gradients_ref(self):
        """CPU-mode counterpart of apply_expert_gradients (same per-expert AMSGrad rule, PyTorch ops)"""
        sh, cfg = self.shard, self.cfg
        if self._ref_rows is None:
            return
        rows, zero_mask = self._ref_rows, 0
        with torch.no_grad():
            for le, leaves in self._ref_leaves.items():   # gather the per-tensor gradients into the flat gradient buffer
                for n, leaf in leaves.items():
                    if cfg.accumulate:                    # update_every_*: gradients pile up until the expert is due
                        if leaf.grad is not None:
                            sh.grads[n][le].add_(leaf.grad)
                    elif leaf.grad is not None:
                        sh.grads[n][le].copy_(leaf.grad)
                    else:
                        sh.grads[n][le].zero_()
                    leaf.grad = None
            if cfg.accumulate:   # same bookkeeping as apply_expert_gradients (dmoe_emulator.py:70-77)
                sh.pending_rows += rows.to(sh.pending_rows.dtype)
                sh.pending_steps += (sh.pending_rows > 0).to(sh.pending_steps.dtype)
                thr_rows, thr_steps = cfg.update_thresholds()
                due = (sh.pending_rows > 0) & ((sh.pending_rows >= thr_rows) | (sh.pending_steps >= thr_steps))
                keep = (~due).to(sh.pending_rows.dtype)
                sh.pending_rows.mul_(keep)
                sh.pending_steps.mul_(keep)
                rows, zero_mask = due.to(rows.dtype), (1 << len(SEG_NAMES)) - 1
            sh.step += (rows > 0).to(sh.step.dtype)
            K.adam_step_ref(sh.p, sh.g, sh.m, sh.v, sh.vmax, sh.seg_sizes, self.E_loc, step=sh.step,
                            group_rows=rows, lr=cfg.lr, betas=cfg.betas, eps=cfg.eps, amsgrad=cfg.amsgrad,
                            zero_mask=zero_mask)
        sh.sync_bf16()
        self._ref_rows = None
        self._ref_leaves = {}

    def _forward_ref(self, x, logits, emulate_bf16: bool = False):
        """Dense reference of the layer: same routing, fp32 expert maths, differentiable w.r.t. x and logits only
        (expert parameters are buffers).  ``emulate_bf16`` rounds activations like the GPU path does."""
        cfg = self.cfg
        fail_mask = self.ref_fail_mask
        if fail_mask is None and self.failure_rate_ref() > 0:
            fail_mask = torch.rand(x.shape[0], cfg.num_experts, device=x.device) < cfg.failure_rate
        idx, w_sel = K.gate_topk_ref(logits.detach(), self.grid_size, cfg.k,
                                     alive=self.ctx.alive if self.ctx is not None else getattr(self, "alive_ref", None),
                                     fail_mask=fail_mask)
        # differentiable weights: softmax over the selected logits
        scores = K.product_key_scores(logits, self.grid_size)
        safe_idx = idx.clamp(min=0)
        sel = torch.gather(scores, 1, safe_idx).masked_fill(idx < 0, float("-inf"))
        weights = torch.softmax(sel, dim=-1)
        weights = torch.where(idx >= 0, weights, torch.zeros_like(weights))
        xf = x.float()
        out = torch.zeros(x.shape[0], cfg.hidden, dtype=torch.float32, device=x.device)
        rnd = (lambda t: t.to(torch.bfloat16).float()) if emulate_bf16 else (lambda t: t)
        if self.training:
            rows = torch.bincount(idx[idx >= 0].flatten() - self.first_expert, minlength=self.E_loc)
            self._ref_rows = rows if self._ref_rows is None else self._ref_rows + rows
        for e in idx[idx >= 0].unique().tolist():
            le = e - self.first_expert
            p = self._expert_params(le)
            if emulate_bf16:
                p = {n: (rnd(v) if n.startswith("w") else v) for n, v in p.items()}
            tok, slot = torch.nonzero(idx == e, as_tuple=True)
            xe = rnd(xf[tok])
            h1 = rnd(F.linear(xe, p["w1"], p["b1"]))
            a1 = rnd(F.relu(F.layer_norm(h1, (cfg.inner,), p["g1"], p["be1"])))
            h2 = rnd(F.linear(a1, p["w2"], p["b2"]))
            a2 = rnd(F.relu(F.layer_norm(h2, (cfg.inner,), p["g2"], p["be2"])))
            ye = rnd(F.linear(a2, p["w3"], p["b3"]) + xe)
            out = out.index_put((tok,), ye * weights[tok, slot].unsqueeze(-1), accumulate=True)
        return out.to(x.dtype)


# =========================================================================================================
# flagship model + trainer  (convergence notebook model, cell 2: Linear -> 4 x DMoE -> LayerNorm -> Linear)
# =========================================================================================================
class DMoEClassifier(nn.Module):
    def __init__(self, cfg: DMoEConfig, ctx: Optional[EngineContext] = None, device=None):
        super().__init__()
        self.cfg = cfg
        self.stem = nn.Linear(cfg.in_features, cfg.hidden)
        self.blocks = nn.ModuleList([FusedDMoE(cfg, ctx, layer_index=i, device=device) for i in range(cfg.num_layers)])
        self.norm = nn.LayerNorm(cfg.hidden)
        self.head = nn.Linear(cfg.hidden, cfg.num_classes)

    def forward(self, x):
        on_gpu = self.blocks[0].ctx is not None
        if on_gpu:
            h = F.linear(x.to(torch.bfloat16), self.stem.weight.to(torch.bfloat16), self.stem.bias.to(torch.bfloat16))
        else:
            h = self.stem(x)
        for block in self.blocks:
            h = block(h)
        h = self.norm(h.float())
        return self.head(h)

    def non_expert_parameters(self):
        return list(self.parameters())  # expert parameters are not nn.Parameters by construction
