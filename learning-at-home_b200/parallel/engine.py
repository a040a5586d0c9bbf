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

from ..models.layers import FFN_SEG_KEYS as REF_KEYS, FFN_SEG_NAMES as SEG_NAMES, FFN_SMALL_SEG_MASK as SMALL_SEG_MASK
from ..models.layers import EXPERT_LAYOUTS, GATED_LAYOUT, GatedFeedforwardBlock, gated_inner_dim
from ..ops import fp8, gemm, kernels as K, native
from ..ops.expert_blocks import (RowPlan, ffn_backward, ffn_forward, ffn_forward_fp8, swiglu_mlp_backward,
                                 swiglu_mlp_forward, swiglu_mlp_forward_fp8)

#: eps of the gated expert's RMSNorm (GatedFeedforwardBlock's default)
GATED_EPS = 1e-6
#: the shared expert's GEMMs stream its weights through swap-AB tiles below this many rows per call, and run on 128-row
#: wgmma tiles from there on (the routed experts' "auto" switch)
SHARED_SWAPAB_ROWS = 512
#: rows of the shared expert's buffers are padded to this (the 128-row tiles; swap-AB and wgrad read whole pads)
SHARED_PAD = 128


@dataclass
class DMoEConfig:
    hidden: int = 512
    grid_size: Tuple[int, ...] = (8, 8)
    k: int = 4
    num_layers: int = 4
    in_features: int = 784
    num_classes: int = 10
    tokens_per_rank: int = 1024          # maximum batch (rows) a rank feeds per step
    # receive-buffer rows = capacity_factor * tokens_per_rank * k (+ padding) in dropless mode (expert_capacity_factor = 0);
    # not used when expert_capacity_factor > 0, which bounds the buffer itself
    capacity_factor: float = 2.0
    failure_rate: float = 0.0            # Bernoulli per (token, expert) failure injection (faulty_dmoe_emulator.py:49-51)
    lr: float = 1e-3
    betas: Tuple[float, float] = (0.9, 0.999)
    eps: float = 1e-8
    amsgrad: bool = True
    # weight decay of every expert and trainer parameter, with torch's two forms: L2 (Adam(weight_decay=...): wd * p is added
    # to the gradient) or decoupled (AdamW: p *= 1 - lr * wd before the update).  An expert that receives no rows in a step
    # is not stepped and so not decayed, as with one torch optimizer per expert
    weight_decay: float = 0.0
    decoupled_weight_decay: bool = False
    seed: int = 1337
    uid_prefix: str = "expert"
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
    # "bf16" or "fp8": with "fp8" the forward GEMMs of every expert (FeedforwardBlock: three; GatedFeedforwardBlock:
    # [W1; W3] and W2) run on block-scaled FP8 tensor cores on the big expert path (MXFP8: E4M3 + UE8M0 scale per 1x32
    # block, csrc/grouped_gemm_fp8.cu); dgrad / wgrad / optimizer are unchanged (bf16 / fp32)
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
    # 17/28 of the SMs on one GPU (80 of an H100's 132: the state stream already runs near copy bandwidth there, and the
    # chain gains from the rest), 9/14 when the experts are sharded (the sharded chain waits on peers and needs more SMs)
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
    # the expert architecture, a ``name_to_block`` key: "ffn" = FeedforwardBlock (the reference's expert), "swiglu" =
    # GatedFeedforwardBlock (RMSNorm -> [W1; W3] -> silu(g) * u -> W2, + x: the expert of Mixtral / DeepSeek-MoE / Qwen-MoE)
    expert: str = "ffn"
    # inner width of a "swiglu" expert; 0 = gated_inner_dim(hidden).  "ffn" is fixed at 4 * hidden (must stay 0)
    inner_dim: int = 0
    # router losses of the product-key gate (DESIGN.md §6a): every training forward adds the gradient of
    # router_aux_loss_coef * L_aux + router_z_loss_coef * L_z to the gate's logits in its backward, so the objective is the
    # task loss plus the sum over layers of those terms.  L_aux = N * sum_e f_e * mean_b p_{b,e} is the load-balancing loss
    # of Switch / GShard (f_e: share of the box-wide routed pairs that went to expert e, p: softmax over the N live experts),
    # L_z = mean_b logsumexp_e(s_{b,e})^2 the router z-loss of ST-MoE.  A layer reads them at construction: they are fixed
    # for the life of a layer or trainer.  0 and 0 (the default) launch nothing
    router_aux_loss_coef: float = 0.0
    router_z_loss_coef: float = 0.0
    # auxiliary-loss-free balancing (DESIGN.md §6b, DeepSeek-V3): each layer keeps a bias per expert that is added to the
    # scores for the top-k selection only (the weights stay the softmax over the unbiased scores).  After the count
    # exchange of every training forward, each live expert's bias moves by this rate toward balance: + when it received
    # fewer than the mean box-wide routed pairs, - when more.  No loss and no gradient, so it also balances the frozen
    # emulator gate.  Read at construction; 0 (the default) allocates and launches nothing
    expert_bias_update_rate: float = 0.0
    # the gate's weight function (DESIGN.md §6c): "softmax" over the selected scores, or "sigmoid" (DeepSeek-V3): affinities
    # sigma(s), the selected ones normalised to sum to routed_scaling_factor.  With "sigmoid" an expert bias is added to
    # sigma(s) for the selection, and the load-balancing loss uses p = sigma / sum of sigma; there is no z-loss.  Both are
    # read at construction; a factor other than 1 needs "sigmoid"
    router_score: str = "softmax"
    routed_scaling_factor: float = 1.0
    # group-limited routing (DESIGN.md §6d, DeepSeek-V2/V3 n_group / topk_group): the experts form n_group groups of
    # consecutive flat ids, each group is scored per token (softmax: its best key; sigmoid: the sum of its two best), and a
    # token picks its k experts from its topk_group best groups only.  With n_group = world (or a multiple), every group
    # lives on one rank, so a token's pairs reach at most topk_group ranks.  Read at construction; 1 / 1 changes nothing
    n_group: int = 1
    topk_group: int = 1
    # renormalise the selected weights (DESIGN.md §6e, HF norm_topk_prob).  False weights each selected expert by its
    # unnormalised router probability, times routed_scaling_factor: "softmax" uses p = the softmax over every live expert
    # (Switch, GShard, DeepSeek-V2, Qwen-MoE; at k = 1 the router then trains through the task loss), "sigmoid" uses
    # sigma(s) (DeepSeek-V3 with norm_topk_prob=False).  Read at construction; True changes nothing
    norm_topk_prob: bool = True
    # shared-expert isolation (DESIGN.md §9c, DeepSeek-MoE / Qwen-MoE): every token also passes through one always-active
    # GatedFeedforwardBlock of this inner width, added to the combine of the routed experts with weight 1 and without a
    # second residual.  Its parameters are trainer-side (replicated on every rank, averaged over ranks, stepped once per
    # step, like proj).  expert="swiglu" only; 0 (the default) allocates and launches nothing
    shared_inner_dim: int = 0
    # expert capacity (DESIGN.md §6f, Switch / GShard): each forward, expert e takes at most C = max(1, ceil(f * P / E))
    # of the P box-wide routed pairs, rank 0's first, then rank 1's, ..., each rank's in token order.  A dropped pair sees
    # its expert as the identity (adds w_j * x_b; the weights are not renormalised), so a token whose pairs all drop rides
    # the residual.  The router losses and the bias update see the routed counts, the layout and the optimizer the kept
    # ones.  Bounds the receive buffer (no overflow) and the rows of a hot expert's owner.  Read at construction; 0 (the
    # default) is dropless and changes nothing
    expert_capacity_factor: float = 0.0

    def __post_init__(self):
        if self.expert not in EXPERT_LAYOUTS:
            raise ValueError(f"DMoEConfig.expert must be one of {sorted(EXPERT_LAYOUTS)}, got {self.expert!r}")
        if self.expert == "ffn" and self.inner_dim:
            raise ValueError("DMoEConfig.inner_dim: FeedforwardBlock experts are 4 * hidden wide; inner_dim is for "
                             "expert='swiglu' only")
        if self.inner_dim < 0:
            raise ValueError(f"DMoEConfig.inner_dim must be >= 0, got {self.inner_dim}")
        if self.expert == "swiglu" and self.expert_dtype == "fp8" and (self.hidden % 256 or self.inner % 256):
            # the FP8 forward runs on expert groups padded to 256 rows, which needs every GEMM width a multiple of 256
            raise ValueError("expert='swiglu' with expert_dtype='fp8' needs hidden and the inner width to be multiples of "
                             f"256; got hidden={self.hidden}, inner={self.inner}")
        for name in ("router_aux_loss_coef", "router_z_loss_coef"):
            v = float(getattr(self, name))
            if not math.isfinite(v) or v < 0.0:
                raise ValueError(f"DMoEConfig.{name} must be a finite value >= 0, got {v}")
            if v > 0.0 and self.gate_mode == "emulator":
                raise ValueError(f"DMoEConfig.{name}: the emulator gate is frozen (not trained), so a router loss would "
                                 "train nothing; use gate_mode='product_key'")
        v = float(self.expert_bias_update_rate)
        if not math.isfinite(v) or v < 0.0:
            raise ValueError(f"DMoEConfig.expert_bias_update_rate must be a finite value >= 0, got {v}")
        if self.router_score not in K.ROUTER_SCORES:
            raise ValueError(f"DMoEConfig.router_score must be one of {K.ROUTER_SCORES}, got {self.router_score!r}")
        v = float(self.routed_scaling_factor)
        if not math.isfinite(v) or v <= 0.0:
            raise ValueError(f"DMoEConfig.routed_scaling_factor must be a finite value > 0, got {v}")
        if not isinstance(self.norm_topk_prob, bool):
            raise ValueError(f"DMoEConfig.norm_topk_prob must be a bool, got {self.norm_topk_prob!r}")
        if v != 1.0 and self.router_score != "sigmoid" and self.norm_topk_prob:
            raise ValueError("DMoEConfig.routed_scaling_factor scales the normalised sigmoid weights; with "
                             f"router_score={self.router_score!r} it must be 1, got {v} (or set norm_topk_prob=False)")
        if self.router_score == "sigmoid" and self.router_z_loss_coef > 0.0:
            raise ValueError("DMoEConfig.router_z_loss_coef: the z-loss penalises the softmax log-partition, which "
                             "router_score='sigmoid' does not have; set it to 0")
        if self.shared_inner_dim < 0:
            raise ValueError(f"DMoEConfig.shared_inner_dim must be >= 0, got {self.shared_inner_dim}")
        K.check_expert_groups("DMoEConfig", self.num_experts, self.n_group, self.topk_group, self.k)
        K.check_capacity_factor("DMoEConfig.expert_capacity_factor", self.expert_capacity_factor)
        if self.shared_inner_dim and self.expert != "swiglu":
            raise ValueError("DMoEConfig.shared_inner_dim: the shared expert is a GatedFeedforwardBlock and needs "
                             f"expert='swiglu', got expert={self.expert!r}")

    @property
    def router_losses(self) -> bool:
        """a router loss is trained (a coefficient is nonzero)"""
        return self.router_aux_loss_coef > 0.0 or self.router_z_loss_coef > 0.0

    def check_native_sizes(self):
        """the widths the sm_90a kernels run for this expert (the CPU oracle path takes any size)"""
        if self.expert == "swiglu" and (self.hidden % 128 or not 128 <= self.hidden <= K.LN_MAX_WIDTH or self.inner % 128):
            raise ValueError(f"expert='swiglu' on the GPU needs hidden a multiple of 128 in [128, {K.LN_MAX_WIDTH}] and "
                             f"an inner width that is a multiple of 128; got hidden={self.hidden}, inner={self.inner}")
        if self.shared_inner_dim % 128:
            raise ValueError("the shared expert on the GPU needs shared_inner_dim a multiple of 128; got "
                             f"{self.shared_inner_dim}")

    @property
    def layout(self):
        """the segment layout of the expert kind (models/layers.py)"""
        return EXPERT_LAYOUTS[self.expert]

    def gemm_widths(self) -> Tuple[int, ...]:
        """N of the expert's GEMMs (forward and dgrad): every one must be a multiple of 256 for 256-row groups"""
        H, I = self.hidden, self.inner
        return (2 * I, H, I) if self.expert == "swiglu" else (I, H)

    def resolved_path(self, world: int = 1) -> str:
        if self.accumulate:
            return "big"      # gradient accumulation across steps needs the weight gradient in HBM (unfused wgrad + AMSGrad)
        if self.expert_path != "auto":
            return self.expert_path
        rows_per_expert = self.tokens_per_rank * world * self.k / max(1, self.num_experts)
        experts_per_rank = -(-self.num_experts // max(1, world))
        return "small" if (rows_per_expert < 512 and self.expert_dtype == "bf16"
                           and all(n % 128 == 0 for n in self.gemm_widths())
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
        """the expert's inner width: 4 * hidden for "ffn", inner_dim or gated_inner_dim(hidden) for "swiglu\""""
        if self.expert == "swiglu":
            return self.inner_dim or gated_inner_dim(self.hidden)
        return 4 * self.hidden

    def adam_kwargs(self) -> Dict:
        """the optimizer settings as keywords of ``K.adam_step`` / ``K.wgrad_adam`` / ``K.adam_step_ref``"""
        return dict(lr=self.lr, betas=self.betas, eps=self.eps, amsgrad=self.amsgrad, weight_decay=self.weight_decay,
                    decoupled=self.decoupled_weight_decay)

    def seg_shapes(self) -> Dict[str, Tuple[int, ...]]:
        return self.layout.shapes(self.hidden, self.inner)


def refuse_router_losses(cfg: DMoEConfig, arm: str):
    """the baseline arms train no router loss: refuse nonzero coefficients instead of silently dropping them"""
    if cfg.router_losses:
        raise ValueError(f"{arm} does not train router losses; set router_aux_loss_coef and router_z_loss_coef to 0 "
                         "(FusedDMoE / DMoETrainer train them)")


def refuse_expert_bias(cfg: DMoEConfig, arm: str):
    """the baseline arms route without expert biases: refuse a nonzero update rate instead of silently dropping it"""
    if cfg.expert_bias_update_rate > 0.0:
        raise ValueError(f"{arm} does not balance with expert biases; set expert_bias_update_rate to 0 "
                         "(FusedDMoE / DMoETrainer apply them)")


def refuse_router_score(cfg: DMoEConfig, arm: str):
    """the baseline arms weight the selected experts with a softmax: refuse the sigmoid router instead of silently
    routing with a softmax"""
    if cfg.router_score != "softmax":
        raise ValueError(f"{arm} weights the selected experts with a softmax; set router_score='softmax' "
                         "(FusedDMoE / DMoETrainer route with sigmoid affinities)")
    if not cfg.norm_topk_prob:
        raise ValueError(f"{arm} renormalises the weights over the selected experts; set norm_topk_prob=True "
                         "(FusedDMoE / DMoETrainer weight them by their unnormalised router probabilities)")


def dense_gate_backward(cfg: DMoEConfig) -> bool:
    """the unnormalised softmax router (DESIGN.md §6e): every live expert's probability depends on every score, so the
    gate backward reads the logits and the log-partition of the forward"""
    return cfg.router_score == "softmax" and not cfg.norm_topk_prob


def refuse_group_limited_routing(cfg: DMoEConfig, arm: str):
    """the baseline arms route each token over all experts: refuse n_group > 1 instead of silently ignoring the limit"""
    if cfg.n_group > 1:
        raise ValueError(f"{arm} routes each token over all experts; set n_group=1 (FusedDMoE / DMoETrainer limit the "
                         "routing to the topk_group best expert groups)")


def max_groups_per_token(idx, k: int, num_experts: int, n_group: int) -> int:
    """the most expert groups (of num_experts / n_group consecutive ids) any token's routed pairs reach; ``idx``: the
    [B * k] or [B, k] expert ids of a gate, -1 for a missing pair.  0 for an empty batch"""
    idx = idx.reshape(-1, k).long()
    if idx.numel() == 0:
        return 0
    g = torch.where(idx >= 0, idx // (num_experts // n_group), torch.full_like(idx, n_group))
    hit = torch.zeros(idx.shape[0], n_group + 1, dtype=torch.bool, device=idx.device).scatter_(1, g, True)
    return int(hit[:, :n_group].sum(1).max())


def refuse_shared_expert(cfg: DMoEConfig, arm: str):
    """an arm without a shared expert: refuse shared_inner_dim > 0 instead of silently dropping it"""
    if cfg.shared_inner_dim > 0:
        raise ValueError(f"{arm} has no shared expert; set shared_inner_dim to 0 (FusedDMoE / DMoETrainer / "
                         "BaselineDMoE train it)")


def refuse_expert_capacity(cfg: DMoEConfig, arm: str):
    """the baseline arms process every routed pair: refuse an expert capacity instead of silently ignoring it"""
    if cfg.expert_capacity_factor > 0.0:
        raise ValueError(f"{arm} processes every routed pair; set expert_capacity_factor to 0 (FusedDMoE / DMoETrainer "
                         "cap the rows of each expert)")


def capacity_buffer_rows(cfg: DMoEConfig, world: int, E_loc: int, shadow_slots: int, align: int) -> int:
    """receive-buffer rows that no routing can exceed with an expert capacity (DESIGN.md §6f): the largest C that
    tokens_per_rank, world and k allow, for each owned group and shadow slot, never more than one row per token and
    expert, each group padded to align"""
    T = cfg.tokens_per_rank
    C = K.expert_capacity(cfg.expert_capacity_factor, world * T * cfg.k, cfg.num_experts)
    pad = lambda r: -(-r // align) * align   # noqa: E731
    owned = min(E_loc * pad(min(C, world * T)), pad(min(E_loc * min(C, world * T), world * T * cfg.k)) + E_loc * align)
    return owned + shadow_slots * pad(min(C, T))


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
        cfg.check_native_sizes()
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
        self.small = cfg.resolved_path(self.world) == "small"
        if self.small:
            # weight-streaming regime: hot-expert replicas would move 12.6 MB of weights to save a few rows -> static placement
            self.align = self.tile_rows = 16
            self.S = 0
        else:
            # expert groups are padded to this many rows: 256 when every GEMM of the expert runs on 128 x 256 tiles
            self.align = 256 if all(n % 256 == 0 for n in cfg.gemm_widths()) else 128
            self.tile_rows = 128
            self.S = min(int(cfg.shadow_experts), 2 * K.MAX_WORLD) if self.world > 1 else 0   # shadow slots per rank / layer
        self.G_tot = self.E_loc + self.S
        if cfg.expert_capacity_factor > 0.0:
            self.max_rows = capacity_buffer_rows(cfg, self.world, self.E_loc, self.S, self.align)
        else:
            self.max_rows = ((cap + self.align - 1) // self.align + self.G_tot) * self.align
        self.max_rows = (self.max_rows + 127) // 128 * 128
        self.max_tiles = self.max_rows // self.tile_rows
        H = cfg.hidden
        sym_rows_bytes = self.max_rows * H * 2
        need = (3 * cfg.num_layers + 2) * (sym_rows_bytes + 4096) + K.MAX_WORLD * self.E * 4 + (32 << 20)
        if self.S:  # parameters, bf16 mirror and gradients of the shards are peer-visible (replica pull / gradient reduce)
            rec = sum(int(math.prod(shape)) for shape in cfg.seg_shapes().values())
            need += cfg.num_layers * (self.G_tot * rec * 10 + (1 << 20))
        if cfg.shared_inner_dim:   # DMoETrainer's flat gradient in the heap also holds the shared experts' gradients
            need += cfg.num_layers * (H + 3 * H * cfg.shared_inner_dim + 256) * 4
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
            octas = sms * (17 if self.world == 1 else 18) // 28
        self.opt_ctas = octas if (self.small and 0 < octas < sms - 8) else 0     # CTAs of the optimizer stream (0: no overlap)
        self.chain_ctas = sms - self.opt_ctas if self.opt_ctas else 0            # CTA limit of the persistent chain kernels
        self.opt_stream = torch.cuda.Stream(self.device) if self.opt_ctas else None
        self._opt_pending = False
        self.defer_join = False   # DMoETrainer joins the optimizer stream itself, at the very end of its step
        K.set_poison_word(self.status)   # a step in which a peer timed out applies no optimizer update (the batch fails)
        # learning rate of every expert and trainer optimizer launch, read by the kernels from device memory (K.lr_block_values:
        # [lr, 1 - lr * wd]) so that a captured graph of the step follows cfg.lr.  Allocated once: the graph holds its address
        self._lr_written = K.lr_block_values(cfg.lr, cfg.weight_decay, cfg.decoupled_weight_decay)
        self.lr_dev = torch.tensor(self._lr_written, dtype=torch.float32, device=self.device)
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
        if cfg.router_losses:   # scratch of the router-loss forward, shared by all layers: per-CTA sums and a CTA ticket
            blocks = -(-cfg.tokens_per_rank // K.ROUTER_WARPS)
            self.router_partials = torch.zeros(2 * blocks, dtype=torch.float32, device=self.device)
            self.router_ticket = torch.zeros(1, dtype=torch.int32, device=self.device)
        bf = dict(dtype=torch.bfloat16, device=self.device)
        # the expert's backward temporaries (FeedforwardBlock: da, dh; GatedFeedforwardBlock: da, dh = [dg | du], dn)
        for name, width in cfg.layout.buffers(H, cfg.inner)["scratch"].items():
            setattr(self, name, torch.empty(self.max_rows, width, **bf))
        if cfg.shared_inner_dim:
            # the shared expert's backward temporaries (shared by all layers; zero, so that padding rows start at zero) and
            # its one-group tables: row t of shared_go is the group_off [0, 128 (t + 1)] of a batch padded to 128 (t + 1)
            # rows, its column 1 the group_rows; shared_tg is the tile_group of the 128-row GEMMs (every tile in group 0)
            Is, R = cfg.shared_inner_dim, -(-cfg.tokens_per_rank // SHARED_PAD) * SHARED_PAD
            self.shared_da = torch.zeros(R, Is, **bf)
            self.shared_dh = torch.zeros(R, 2 * Is, **bf)
            self.shared_dn = torch.zeros(R, H, **bf)
            self.shared_dx = torch.zeros(R, H, **bf)
            tiles = torch.arange(1, R // SHARED_PAD + 1, dtype=torch.int32) * SHARED_PAD
            self.shared_go = torch.stack([torch.zeros_like(tiles), tiles], 1).to(self.device)
            self.shared_tg = torch.zeros(R // SHARED_PAD, dtype=torch.int32, device=self.device)
        self.heap.barrier()

    EPOCH_STRIDE = 64   # epochs a step may consume; the device-side base advances by this much per begin_step()

    def adam_kwargs(self) -> Dict:
        """``cfg.adam_kwargs()`` plus the device block ``lr_dev``: the keywords of every optimizer launch on the GPU"""
        return dict(self.cfg.adam_kwargs(), lr_dev=self.lr_dev)

    def refresh_lr(self):
        """Write cfg.lr (and the decoupled factor it implies) into ``lr_dev`` when it differs from the last value written.
        Call at a step boundary: the optimizer stream of the previous step has been joined, and the next step's optimizer
        launches wait on the current stream.  Two in-place fills on the current stream, so the host does not wait.  Never
        while a graph is being captured: a captured write would put the capture-time rate back at every replay."""
        cfg = self.cfg
        vals = K.lr_block_values(cfg.lr, cfg.weight_decay, cfg.decoupled_weight_decay)
        if vals == self._lr_written or torch.cuda.is_current_stream_capturing():
            return
        self.lr_dev[0].fill_(vals[0])
        self.lr_dev[1].fill_(vals[1])
        self._lr_written = vals

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
    [E_loc, size] per tensor kind) plus the bf16 mirror consumed by the GEMMs.

    On the small expert path (``split``) the weight matrices are kept split: the mirror plus their low 16 bits in ``lo``,
    with the tie bit of the rounding in the sign of exp_avg_sq (``K.split_encode``).  The fused wgrad + AMSGrad kernel
    then streams 32 B per parameter instead of 34, and computes the same bits.  ``p``, ``views``, ``v`` and ``v_views``
    hide the format: they return the fp32 values, decoded on access; after writing ``p`` / ``views``, ``sync_bf16()``
    encodes them.  The kernels work on ``p_raw``, ``raw_views``, ``v_raw`` and ``v_raw_views``, whose matrix segments
    hold stale weights and tie bits in a split shard."""

    def __init__(self, cfg: DMoEConfig, E_loc: int, first_expert: int, device, layer_index: int = 0, ctx=None):
        self.cfg, self.E_loc, self.first_expert = cfg, E_loc, first_expert
        # slots = owned experts + shadow slots (replicas of other ranks' hot experts, only on multi-GPU runs)
        self.slots = slots = E_loc + (ctx.S if ctx is not None else 0)
        self.layout = cfg.layout
        shapes = cfg.seg_shapes()
        shapes = {n: shapes[n] for n in self.layout.names}   # in segment order
        self.seg_sizes = [int(math.prod(shape)) for shape in shapes.values()]
        total = sum(self.seg_sizes) * slots
        f32 = dict(dtype=torch.float32, device=device)
        self.p_off = self.g_off = self.pbf16_off = -1
        if ctx is not None and ctx.S > 0:   # peer-visible: replicas are pulled from p / p_bf16, partial grads read from g
            self.p_raw, self.p_off = ctx.heap.alloc((total,), torch.float32)
            self.g, self.g_off = ctx.heap.alloc((total,), torch.float32)
            self.p_bf16, self.pbf16_off = ctx.heap.alloc((total,), torch.bfloat16)
            self.p_raw.zero_(), self.g.zero_(), self.p_bf16.zero_()
        else:
            self.p_raw = torch.zeros(total, **f32)
            self.g = torch.zeros(total, **f32)
            self.p_bf16 = torch.zeros(total, dtype=torch.bfloat16, device=device)
        self.m = torch.zeros(total, **f32)
        self.v_raw = torch.zeros(total, **f32)
        self.vmax = torch.zeros(total, **f32) if cfg.amsgrad else None
        self.step = torch.zeros(E_loc, dtype=torch.int32, device=device)
        self._shapes = shapes
        self.raw_views, self.grads, self.bf16, self.m_views, self.v_raw_views = (
            K.segment_views(flat, shapes, slots) for flat in (self.p_raw, self.g, self.p_bf16, self.m, self.v_raw))
        self.vmax_views = K.segment_views(self.vmax, shapes, slots) if self.vmax is not None else {}
        # the small path updates the weight matrices only in the fused wgrad + AMSGrad kernel, which takes them split
        self.split = ctx is not None and ctx.small
        self.matrices = [n for s, n in enumerate(self.layout.names) if not (self.layout.small_mask >> s) & 1]
        self.lo_views = {}
        if self.split:
            self.lo_views = {n: torch.zeros(self.raw_views[n].shape, dtype=torch.int16, device=device)
                             for n in self.matrices}
        # asynchronous-update bookkeeping (DMoEConfig.update_every_*): rows / steps pending since the last optimizer step
        self.pending_rows = torch.zeros(E_loc, dtype=torch.int32, device=device)
        self.pending_steps = torch.zeros(E_loc, dtype=torch.int32, device=device)
        self.fire = torch.zeros(E_loc, dtype=torch.int32, device=device)
        self.w8 = None        # MXFP8 copies of the matrices (expert_dtype == "fp8"), refreshed lazily from the bf16 mirror
        self.w8_dirty = True
        if cfg.expert_dtype == "fp8" and ctx is not None:
            self.w8 = {n: fp8.MXFP8Tensor(shapes[n][0], slots, shapes[n][1], fp8.WEIGHT_TILE, device)
                       for n in self.matrices}
        self.reset_parameters(layer_index)

    @torch.no_grad()
    def reset_parameters(self, layer_index: int = 0):
        """nn.Linear / nn.LayerNorm / nn.RMSNorm default initialisation (weights and biases uniform in +-1/sqrt(fan_in),
        norm weights 1, norm biases 0), seeded per (layer, global expert) so that the same expert gets the same weights
        regardless of the number of ranks"""
        cfg = self.cfg
        dev = self.p_raw.device
        views = self.raw_views   # every weight of the owned experts is written, then encoded by sync_bf16()
        for le in range(self.E_loc):
            gen = torch.Generator(device=dev)
            gen.manual_seed(cfg.seed * 1000003 + layer_index * 10007 + self.first_expert + le)
            for n in self.layout.names:   # segment order: a matrix is followed by its bias (FeedforwardBlock)
                t = views[n][le]
                if n.startswith("be"):       # LayerNorm bias
                    t.zero_()
                elif n.startswith("g"):      # LayerNorm / RMSNorm weight
                    t.fill_(1.0)
                else:                        # Linear weight wX or its bias bX (fan_in from wX)
                    fan_in = views["w" + n[1:]].shape[-1]
                    bound = 1.0 / math.sqrt(fan_in)
                    t.uniform_(-bound, bound, generator=gen)
        self.sync_bf16()

    def fp8_weights(self):
        """MXFP8 weights of all slots, re-quantised from the bf16 mirror when it changed (optimizer step / replica pull)"""
        if self.w8_dirty:
            for n, t in self.w8.items():
                fp8.quantize(self.bf16[n].view(-1, t.K), tile_rows=fp8.WEIGHT_TILE, groups=self.slots, out=t)
            self.w8_dirty = False
        return self.w8

    def sync_bf16(self):
        """the mirror (and in a split shard lo and the tie bits) from the fp32 weights in ``p_raw``"""
        self.w8_dirty = True
        if self.p_raw.is_cuda:
            K.cast_bf16(self.p_raw, self.p_bf16)
        else:
            self.p_bf16.copy_(self.p_raw)
        for n in (self.matrices if self.split else ()):
            K.split_encode(self.raw_views[n], self.bf16[n], self.lo_views[n], self.v_raw_views[n])

    @property
    def p(self) -> torch.Tensor:
        """the flat fp32 weights; a split shard decodes its matrices into ``p_raw`` first"""
        for n in (self.matrices if self.split else ()):
            K.split_decode(self.bf16[n], self.lo_views[n], self.v_raw_views[n], out=self.raw_views[n])
        return self.p_raw

    @property
    def views(self) -> Dict[str, torch.Tensor]:
        self.p
        return self.raw_views

    @property
    def v(self) -> torch.Tensor:
        """the flat exp_avg_sq; in a split shard a copy without the tie bits"""
        return self.v_raw.abs() if self.split else self.v_raw

    @property
    def v_views(self) -> Dict[str, torch.Tensor]:
        return K.segment_views(self.v, self._shapes, self.slots) if self.split else self.v_raw_views

    # ------------------------------------------------------------------ checkpoint layout (SURVEY.md §5.4)
    def _expert_tensors(self, views, le: int) -> Dict[str, torch.Tensor]:
        """one expert's rows of a per-segment view, as the module's tensors (parameters() order)"""
        return self.layout.module_state({n: views[n][le] for n in self.layout.names})

    def expert_state_dict(self, le: int, prefix: str = "expert.") -> Dict[str, torch.Tensor]:
        """state of local expert `le` with the key names of ``ExpertBackend.state_dict()`` of the reference (the module of
        ``cfg.expert``: FeedforwardBlock or GatedFeedforwardBlock)"""
        return {prefix + k: t.detach().clone().cpu() for k, t in self._expert_tensors(self.views, le).items()}

    def expert_optimizer_state(self, le: int) -> Dict:
        """torch.optim.Adam-compatible state_dict of local expert `le` (parameter order = module.parameters())"""
        step = torch.tensor(float(self.step[le].item()))
        moments = [("exp_avg", self.m_views), ("exp_avg_sq", self.v_views)]
        if self.vmax is not None:
            moments.append(("max_exp_avg_sq", self.vmax_views))
        per_key = {name: self._expert_tensors(views, le) for name, views in moments}
        state = {i: dict(step=step.clone(), **{name: per_key[name][k].clone().cpu() for name, _ in moments})
                 for i, k in enumerate(self.layout.params)}
        cfg = self.cfg
        group = dict(lr=cfg.lr, betas=cfg.betas, eps=cfg.eps, weight_decay=cfg.weight_decay, amsgrad=cfg.amsgrad,
                     decoupled_weight_decay=cfg.decoupled_weight_decay, params=list(range(len(self.layout.params))))
        return dict(state=state, param_groups=[group])

    def load_expert_state_dict(self, le: int, state: Dict[str, torch.Tensor], prefix: str = "expert."):
        with torch.no_grad():
            views = self.views   # decoded once: a split shard's next decode would overwrite what is written here
            for n, t in self.layout.segment_state(state, prefix).items():
                views[n][le].copy_(t)
        self.sync_bf16()

    def load_expert_optimizer_state(self, le: int, opt_state: Dict):
        with torch.no_grad():
            self.p   # a split shard decodes its weights while v still holds their tie bits, and encodes them again below
            for i, k in enumerate(self.layout.params):
                entry = opt_state["state"].get(i)
                if entry is None:
                    continue
                n, block, parts = self.layout.slices[k]
                for name, views in (("exp_avg", self.m_views), ("exp_avg_sq", self.v_raw_views),
                                    ("max_exp_avg_sq", self.vmax_views if self.vmax is not None else None)):
                    if views is None or name not in entry:
                        continue
                    dst = views[n][le]
                    dst = dst.chunk(parts, 0)[block] if parts > 1 else dst
                    dst.copy_(entry[name].reshape(dst.shape))
                self.step[le] = int(entry["step"])
            if self.split:
                self.sync_bf16()


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
        # the expert's activations (FeedforwardBlock: h1, a1, h2, a2 and the LayerNorm statistics; GatedFeedforwardBlock:
        # n = RMSNorm(xd), h = [hg | hu], a = silu(hg) * hu and rstd)
        buffers = cfg.layout.buffers(H, I)
        for name, width in buffers["rows"].items():
            setattr(self, name, torch.empty(R, width, **bf))
        for name in buffers["stats"]:
            setattr(self, name, torch.empty(R, **f32))
        self.xq = self.aq = None
        # MXFP8 operands of the forward GEMMs: FeedforwardBlock: xq = x, aq = a1 then a2; GatedFeedforwardBlock: xq = n,
        # aq = a
        if cfg.expert_dtype == "fp8":
            self.xq = fp8.MXFP8Tensor(R, 1, H, fp8.ACT_TILE, dev)
            self.aq = fp8.MXFP8Tensor(R, 1, I, fp8.ACT_TILE, dev)
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
        # expert capacity (DESIGN.md §6f): this rank's kept pairs per expert and (C, box-wide dropped pairs), written by
        # layout_exchange
        self.keep = self.capacity_stats = None
        if cfg.expert_capacity_factor > 0.0:
            self.keep = torch.zeros(ctx.E, **i32)
            self.capacity_stats = torch.zeros(2, **i32)
        # the sigmoid router (DESIGN.md §6c): sigma of every selected pair, written by gate_topk and read by gate_bwd
        self.sig = torch.zeros(P, **f32) if cfg.router_score == "sigmoid" else None
        # the unnormalised softmax router (DESIGN.md §6e): each token's log-partition z_b, written by gate_topk and read by
        # gate_bwd
        self.lse = torch.zeros(cfg.tokens_per_rank, **f32) if dense_gate_backward(cfg) else None
        self.router_loss = None
        if cfg.router_losses:
            # router losses: f (box-wide routing shares, snapshotted from the count table the next layer overwrites, then
            # N), z_b and F_b of every token for the backward, and the layer's unweighted (L_aux, L_z)
            self.router_f = torch.zeros(ctx.E + 1, **f32)
            self.router_z = torch.zeros(cfg.tokens_per_rank, **f32)
            self.router_F = torch.zeros(cfg.tokens_per_rank, **f32)
            self.router_loss = torch.zeros(2, **f32)
        if cfg.shared_inner_dim:
            # the shared expert's activations on this rank's rows, padded to SHARED_PAD rows (zero, so that the padding rows
            # start at zero), its output ys (the forward combine's addend), the padded copy of the output gradient and the
            # bf16 GEMM operands cast from the fp32 parameters at every forward
            Is, Rs = cfg.shared_inner_dim, -(-cfg.tokens_per_rank // SHARED_PAD) * SHARED_PAD
            self.shared_n, self.shared_h = torch.zeros(Rs, H, **bf), torch.zeros(Rs, 2 * Is, **bf)
            self.shared_a, self.shared_y = torch.zeros(Rs, Is, **bf), torch.zeros(Rs, H, **bf)
            self.shared_gy = torch.zeros(Rs, H, **bf)
            self.shared_rstd = torch.zeros(Rs, **f32)
            self.shared_w13 = torch.zeros(1, 2 * Is, H, **bf)
            self.shared_w2 = torch.zeros(1, H, Is, **bf)
        self.outstanding = False   # a training-mode forward whose backward has not run yet owns this workspace
        # small path with optimizer overlap: the fused wgrad+AMSGrad kernels of layer L read dY buffers while the main stream is
        # already in the backward of layer L-1, so they must be per layer (a few MB each at this batch size)
        # (FeedforwardBlock: dh2 and dh1; GatedFeedforwardBlock: dh13 = [dg | du]; its other inputs, a and n, are activations)
        if ctx.small and ctx.opt_stream is not None:
            self.gyd, self.gyd_off = ctx.heap.alloc((R, H), torch.bfloat16)
            for name, shared in buffers["per_layer"].items():
                setattr(self, name, torch.zeros_like(getattr(ctx, shared)))
        else:
            self.gyd, self.gyd_off = ctx.gyd, ctx.gyd_off
            for name, shared in buffers["per_layer"].items():
                setattr(self, name, getattr(ctx, shared))


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
        ctx.router = layer.training and layer.router_on
        ctx.dense = layer.dense_gate   # the gate backward of the unnormalised softmax reads the logits too
        # the shared expert's norm backward and the dropped pairs of an expert capacity (gate_bwd) read the layer input
        ctx.shared = layer.shared_inner > 0 or layer.capacity_factor > 0.0
        if ctx.router or ctx.dense or ctx.shared:
            ctx.save_for_backward(*([logits] if ctx.router or ctx.dense else []), *([x] if ctx.shared else []))
        return layer._forward_cuda(x, logits)

    @staticmethod
    def backward(ctx, grad_out):
        if not ctx.layer.ws.outstanding:
            raise RuntimeError("FusedDMoE: backward() without a pending forward (the workspace was released or reused)")
        saved = ctx.saved_tensors
        logits = saved[0] if ctx.router or ctx.dense else None
        x = saved[-1] if ctx.shared else None
        dx, dlogits = ctx.layer._backward_cuda(grad_out.contiguous(), ctx.B, logits, x, router=ctx.router)
        ctx.layer.ws.outstanding = False
        ec = ctx.layer.ctx
        if ec._opt_pending and not ec.defer_join:
            # layer-level callers (no DMoETrainer): when the whole backward pass is over, the launching stream waits for the
            # expert optimizers on the second stream, so reading the parameters right after backward() is safe
            torch.autograd.Variable._execution_engine.queue_callback(ec.join_optimizer_stream)
        return dx, dlogits, None


class _AddRouterLoss(torch.autograd.Function):
    """identity on the layer output whose backward also sends gradient 1 into the router-loss term: the term joins the
    objective without the caller adding it to the loss (the CPU counterpart of the router-loss kernels)"""

    @staticmethod
    def forward(ctx, out, aux):
        ctx.aux_dtype = aux.dtype
        return out.view_as(out)

    @staticmethod
    def backward(ctx, grad_out):
        return grad_out, torch.ones((), dtype=ctx.aux_dtype, device=grad_out.device)


class FusedDMoE(nn.Module):
    """
    Decentralized-MoE layer over the experts of the whole box.  Trainer-side parameters: ``proj`` (product-key gating,
    identical to ``GatingFunction.proj``: Linear(in_features, sum(grid_size))).  Expert parameters live in
    ``self.shard`` and are updated by the layer itself during backward (they are NOT nn.Parameters, mirroring
    ``get_non_expert_params`` of the reference emulator).  With ``cfg.shared_inner_dim`` the layer also owns a shared
    expert (DESIGN.md §9c): the trainer-side parameters ``shared_g`` [H], ``shared_w13`` [2 I_s, H] and ``shared_w2``
    [H, I_s] of one GatedFeedforwardBlock, whose ``module(x) - x`` is added to every token's combined output.
    """

    def __init__(self, cfg: DMoEConfig, ctx: Optional[EngineContext] = None, layer_index: int = 0, device=None):
        super().__init__()
        if ctx is not None and cfg.router_losses and not ctx.cfg.router_losses:
            # the router-loss buffers (per layer and the shared scratch) are allocated from the context's configuration
            raise ValueError("FusedDMoE: router losses need an EngineContext built from a DMoEConfig with a nonzero "
                             "router_aux_loss_coef or router_z_loss_coef (the context allocates their buffers)")
        if ctx is not None and cfg.router_score != ctx.cfg.router_score:
            # the workspace (the sigma array of the sigmoid gate) is allocated from the context's configuration
            raise ValueError(f"FusedDMoE: router_score={cfg.router_score!r} needs an EngineContext built with the same "
                             f"router_score, got {ctx.cfg.router_score!r}")
        if ctx is not None and (cfg.expert_capacity_factor > 0.0) != (ctx.cfg.expert_capacity_factor > 0.0):
            # the receive buffer and the workspace's keep table follow the context's configuration
            raise ValueError(f"FusedDMoE: expert_capacity_factor={cfg.expert_capacity_factor} needs an EngineContext "
                             f"built with an expert capacity as well, got {ctx.cfg.expert_capacity_factor}")
        if ctx is not None and cfg.norm_topk_prob != ctx.cfg.norm_topk_prob:
            # the workspace (the log-partition array of the unnormalised softmax gate) follows the context's configuration
            raise ValueError(f"FusedDMoE: norm_topk_prob={cfg.norm_topk_prob!r} needs an EngineContext built with the "
                             f"same norm_topk_prob, got {ctx.cfg.norm_topk_prob!r}")
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
        # router losses (cfg.router_*_coef, read here once): the unweighted (L_aux, L_z) of the last training forward, this
        # rank's term, on the layer's device (kernels write it on the GPU path, so it stays valid after graph replay)
        self.router_aux_coef = float(cfg.router_aux_loss_coef)
        self.router_z_coef = float(cfg.router_z_loss_coef)
        self.router_on = self.router_aux_coef > 0.0 or self.router_z_coef > 0.0
        self.router_grad_scale = 1.0   # DMoETrainer: 1 / trainer_microbatches, like each micro-batch's cross-entropy
        if self.ws is not None:   # written by the kernels at a fixed address (a captured graph holds it)
            self.router_loss = self.ws.router_loss if self.router_on else None
        else:                     # a buffer, so that .to() / .cuda() move it with the layer (not saved in state_dict)
            self.register_buffer("router_loss", torch.zeros(2, device=dev) if self.router_on else None, persistent=False)
        # auxiliary-loss-free balancing (cfg.expert_bias_update_rate, read here once): router state like proj, the same on
        # every rank; a persistent buffer, so it is saved with the trainer-side parameters, and kept at one device address
        # (a captured graph reads it)
        self.expert_bias_rate = float(cfg.expert_bias_update_rate)
        self.register_buffer("expert_bias", torch.zeros(cfg.num_experts, dtype=torch.float32, device=dev)
                             if self.expert_bias_rate > 0.0 else None)
        # the gate's weight function (cfg.router_score / routed_scaling_factor, read here once; DESIGN.md §6c)
        self.router_score = cfg.router_score
        self.routed_scale = float(cfg.routed_scaling_factor)
        # unnormalised weights (cfg.norm_topk_prob, read here once; DESIGN.md §6e)
        self.norm_topk_prob = bool(cfg.norm_topk_prob)
        self.dense_gate = dense_gate_backward(cfg)
        # group-limited routing (cfg.n_group / topk_group, read here once; DESIGN.md §6d)
        self.n_group, self.topk_group = int(cfg.n_group), int(cfg.topk_group)
        # expert capacity (cfg.expert_capacity_factor, read here once; DESIGN.md §6f)
        self.capacity_factor = float(cfg.expert_capacity_factor)
        self._ref_capacity = None   # CPU path: (C, dropped pairs) of the last forward
        self._last_pairs = 0   # GPU path: routed pairs (B * k) of the last forward, whose ws.idx log_step reads
        # shared expert (cfg.shared_inner_dim, read here once): initialised like GatedFeedforwardBlock(hidden, I_s), drawn
        # from the global RNG like proj (DMoETrainer seeds it, so every rank starts identical), kept as the segments of
        # GATED_LAYOUT so that [W1; W3] is one GEMM operand and one contiguous gradient
        self.shared_inner = int(cfg.shared_inner_dim)
        if self.shared_inner:
            block = GatedFeedforwardBlock(cfg.hidden, self.shared_inner, eps=GATED_EPS)
            seg = GATED_LAYOUT.segment_state({k: v.detach() for k, v in block.state_dict().items()})
            self.shared_g = nn.Parameter(seg["g"].clone())
            self.shared_w13 = nn.Parameter(seg["w13"].clone())
            self.shared_w2 = nn.Parameter(seg["w2"].clone())

    # ------------------------------------------------------------------ shared expert (DESIGN.md §9c)
    def shared_expert_parameters(self) -> List[nn.Parameter]:
        """the shared expert's parameters in segment order (g, w13, w2); [] without a shared expert"""
        return [self.shared_g, self.shared_w13, self.shared_w2] if self.shared_inner else []

    def _shared_segments(self) -> Dict[str, torch.Tensor]:
        if not self.shared_inner:
            raise ValueError("this FusedDMoE has no shared expert (DMoEConfig.shared_inner_dim = 0)")
        return dict(zip(GATED_LAYOUT.names, self.shared_expert_parameters()))

    def shared_expert_state_dict(self, prefix: str = "") -> Dict[str, torch.Tensor]:
        """the shared expert as a ``GatedFeedforwardBlock(hidden, shared_inner_dim)`` state_dict (``norm.weight``,
        ``w1.weight``, ``w2.weight``, ``w3.weight``): that module's ``module(x) - x`` is the layer's shared term"""
        return {prefix + k: t.detach().clone().cpu() for k, t in GATED_LAYOUT.module_state(self._shared_segments()).items()}

    def load_shared_expert_state_dict(self, state: Dict[str, torch.Tensor], prefix: str = ""):
        """load a ``GatedFeedforwardBlock`` state_dict into the shared expert (in place: a captured graph reads it)"""
        segs = self._shared_segments()
        with torch.no_grad():
            for n, t in GATED_LAYOUT.segment_state(state, prefix).items():
                if tuple(t.shape) != tuple(segs[n].shape):
                    raise ValueError(f"shared expert: {n} has shape {tuple(t.shape)}, this layer {tuple(segs[n].shape)}")
                segs[n].copy_(t)

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
        c.refresh_lr()              # layer-level callers: a step begins here (DMoETrainer refreshed before the step)
        epoch = c.next_epoch()
        idx, w, pos, pair_row = ws.idx[:P], ws.w[:P], ws.pos[:P], ws.pair_row[:P]
        K.gate_topk(logits, self.grid_size, k, alive=c.alive, failure_rate=cfg.failure_rate if self.training else 0.0,
                    seed=cfg.seed * 7919 + self.layer_index, token_offset=c.token_counter, idx=idx, w=w, pos=pos,
                    counts=c.counts, bias=self.expert_bias, n_group=self.n_group, topk_group=self.topk_group,
                    **self._score_args(P, B))
        self._last_pairs = P
        c.token_counter += B
        c.timer.mark("gate_topk")
        K.layout_exchange(c.cnt_all_off, c.flags_off, K.SLOT_COUNTS, epoch, c.E, c.E_loc, c.max_rows, align=c.align,
                          tile_rows=c.tile_rows, counts=c.counts,
                          dst_row=ws.dst_row, group_off=ws.group_off, group_rows=ws.group_rows,
                          tile_group=ws.tile_group, total_rows=ws.total_rows, status=c.status, shadow_slots=c.S,
                          shadow_tol=cfg.shadow_tol, min_shadow_rows=cfg.shadow_min_rows, route_owner=ws.route_owner,
                          step_rows=ws.step_rows, shadow_info=ws.shadow_info, owned_shadow=ws.owned_shadow,
                          capacity_factor=self.capacity_factor, keep=ws.keep, capacity_stats=ws.capacity_stats)
        if self.training and self.router_on:
            # before combine_rows: no peer can reach the next layer's count exchange (which rewrites cnt_all) until this
            # rank's combine has signalled
            K.router_loss_fwd(logits, self.grid_size, c.cnt_all[:c.world], alive=c.alive, f=ws.router_f, z=ws.router_z,
                              Fb=ws.router_F, loss=ws.router_loss, partials=c.router_partials, ticket=c.router_ticket,
                              score=self.router_score)
        if self.training and self.expert_bias is not None:   # same cnt_all lifetime as the router losses above
            K.expert_bias_update(c.cnt_all[:c.world], alive=c.alive, bias=self.expert_bias, rate=self.expert_bias_rate)
        if c.S:  # replicas of this step's hot experts: weights from the owners' bf16 mirror, small params from fp32
            K.pull_shadow(ws.shadow_info, c.S, c.E_loc, sh.p_off, sh.pbf16_off, sh.seg_sizes, sh.layout.small_mask)
            sh.w8_dirty = True
        K.scatter_rows(x, None, idx, pos, ws.dst_row, pair_row, ws.xd_off, c.flags_off, K.SLOT_DISPATCH, epoch, k,
                       c.E_loc, c.max_rows, ws.group_off, ws.group_rows, c.done_counter, c.status, align=c.align,
                       route_owner=ws.route_owner, num_groups=c.G_tot, keep=ws.keep)
        c.timer.mark("dispatch(layout+pull+scatter)")
        # the shared expert needs only this rank's rows: at world > 1 it runs while the peers' rows are in flight
        ys = self._shared_expert_fwd(x) if self.shared_inner else None
        if ys is not None:
            c.timer.mark("shared_expert_fwd")
        # ---- expert FFN on the rows this rank received (grouped by expert).  Receive-side fusion: the first GEMM's TMA
        # producer polls the peers' dispatch flags itself (no separate wait kernel)
        wait = (c.flags[K.SLOT_DISPATCH, :c.world], epoch, c.status) if c.world > 1 else None
        plan = self._expert_plan()
        if cfg.expert == "swiglu":
            # the rows of unused tiles (group -1) of n, h and a hold stale values that no result reads: the big path's
            # GEMMs skip -1 tiles; the small path's power-of-two TMA boxes may reach past a group's padded rows, but those
            # GEMM columns are not stored, the wgrads read only the groups' rows and SwiGLU maps rows elementwise
            if wait is not None:  # the norm, not a GEMM, is the first consumer of the rows pushed by the peers
                K.signal_wait(c.flags_off, K.SLOT_DISPATCH, epoch, c.status, signal=False, wait=True)
            fp8_fwd = not c.small and cfg.expert_dtype == "fp8"
            # FP8: the norm and the SwiGLU also write the next GEMM's MXFP8 operand (xq holds n, aq holds a); the bf16 n
            # and a stay, for the weight gradients
            K.rms_norm_fwd(ws.xd, sh.raw_views["g"], GATED_EPS, out=ws.n, rstd=ws.rstd, tile_group=plan.tile_group,
                           tile_rows=plan.tile_rows, quant=ws.xq if fp8_fwd else None)
            if fp8_fwd:
                assert c.align == 256, "the FP8 path needs 256-row expert groups (hidden and inner multiples of 256)"
                w8 = sh.fp8_weights()
                swiglu_mlp_forward_fp8(plan, w8["w13"], w8["w2"], ws.xq, ws.h, ws.a, ws.aq, ws.yo, residual=ws.xd)
            else:
                swiglu_mlp_forward(plan, sh.bf16["w13"], sh.bf16["w2"], ws.n, ws.h, ws.a, ws.yo, residual=ws.xd)
        elif c.small or cfg.expert_dtype != "fp8":
            ffn_forward(plan, sh.bf16, sh.raw_views, ws.xd, (ws.h1, ws.a1, ws.h2, ws.a2),
                        (ws.mean1, ws.rstd1, ws.mean2, ws.rstd2), ws.yo, wait=wait)
        else:
            # forward GEMMs on block-scaled FP8 tensor cores; LayerNorm emits the next GEMM's MXFP8 operand directly (and
            # the bf16 copy the bf16 wgrad needs)
            assert c.align == 256, "the FP8 path needs 256-row expert groups (hidden and 4*hidden multiples of 256)"
            if wait is not None:  # the quantiser is the first consumer of the rows pushed by the peers
                K.signal_wait(c.flags_off, K.SLOT_DISPATCH, epoch, c.status, signal=False, wait=True)
            ffn_forward_fp8(plan, sh.fp8_weights(), sh.raw_views, ws.xd, ws.xq, ws.aq, (ws.h1, ws.a1, ws.h2, ws.a2),
                            (ws.mean1, ws.rstd1, ws.mean2, ws.rstd2), ws.yo)
        c.timer.mark("expert_ffn_fwd")
        y = torch.empty(B, cfg.hidden, dtype=torch.bfloat16, device=x.device)
        # expert capacity: a dropped pair adds w_j * x_b (its expert as the identity)
        passing = dict(pass_self=x, pass_w=w) if self.capacity_factor > 0.0 else {}
        K.combine_rows(ws.yo_off, idx, pair_row, w, y, k, c.E_loc, flags_off=c.flags_off, slot=K.SLOT_OUTPUT, epoch=epoch,
                       signal=c.world > 1, wait=c.world > 1, status=c.status, route_owner=ws.route_owner, addend=ys,
                       **passing)
        c.timer.mark("combine")
        return y

    def _score_args(self, P, B):
        """the weight-function keywords of K.gate_topk / K.gate_bwd for P routed pairs of B tokens (none for the default
        softmax gate)"""
        args = {} if self.router_score == "softmax" else dict(score=self.router_score, scale=self.routed_scale,
                                                               sig=self.ws.sig[:P])
        if not self.norm_topk_prob:
            args.update(norm=False, scale=self.routed_scale)
            if self.dense_gate:
                args["lse"] = self.ws.lse[:B]
        return args

    def _expert_plan(self):
        """swap-AB groups of 16 rows on the small path (backward GEMMs on ``chain_ctas``), 128-row tiles on the big one"""
        c, ws = self.ctx, self.ws
        if c.small:
            return RowPlan(ws.group_off, ws.group_rows, ws.tile_group, c.tile_rows, max_ctas=c.chain_ctas)
        return RowPlan(ws.group_off, None, ws.tile_group, c.tile_rows)

    def _shared_plan(self, B):
        """(B padded to SHARED_PAD, the shared expert's RowPlan): swap-AB below SHARED_SWAPAB_ROWS, 128-row tiles from
        there; the backward GEMMs keep to ``chain_ctas`` (the last fused wgrad + AMSGrad may still run beside them)"""
        c = self.ctx
        Bp = -(-B // SHARED_PAD) * SHARED_PAD
        go = c.shared_go[Bp // SHARED_PAD - 1]
        return Bp, RowPlan(go, go[1:] if B < SHARED_SWAPAB_ROWS else None, c.shared_tg, max_ctas=c.chain_ctas)

    def _shared_expert_fwd(self, x):
        """the shared expert on this rank's B rows: n = RMSNorm(x), h = n [W1; W3]^T, a = silu(hg) * hu, ys = a W2^T (no
        residual), into rows padded to SHARED_PAD.  The padding rows of n are zeroed here (an earlier, larger batch may have
        written them), so those of h, a and ys are zero as well and add nothing to the weight gradients.  The bf16
        operands are cast from the fp32 parameters at every forward, so any optimizer that steps them is seen.  Returns
        ys[:B], the combine's addend."""
        ws = self.ws
        B = x.shape[0]
        Bp, plan = self._shared_plan(B)
        K.cast_bf16(self.shared_w13.detach(), ws.shared_w13)
        K.cast_bf16(self.shared_w2.detach(), ws.shared_w2)
        n, h, a, ys = ws.shared_n[:Bp], ws.shared_h[:Bp], ws.shared_a[:Bp], ws.shared_y[:Bp]
        K.rms_norm_fwd(x, self.shared_g.detach(), GATED_EPS, out=n[:B], rstd=ws.shared_rstd[:B])
        if Bp > B:
            n[B:].zero_()
        swiglu_mlp_forward(plan, ws.shared_w13, ws.shared_w2, n, h, a, ys)
        return ys[:B]

    def _shared_expert_bwd(self, gy, x):
        """backward of ``_shared_expert_fwd`` on the main stream: the dgrads, SwiGLU and RMSNorm backward give dxs (the
        backward combine's addend), dgamma is added into ``shared_g.grad`` and the weight gradients into
        ``shared_w13.grad`` / ``shared_w2.grad`` (the flat trainer gradient under DMoETrainer, so micro-batches add up).
        The copy of gy is zero-padded, so the padding rows add nothing.  Returns dxs [B, H]."""
        c, ws = self.ctx, self.ws
        B = gy.shape[0]
        Bp, plan = self._shared_plan(B)
        for p in self.shared_expert_parameters():   # layer-level callers: zero gradients on first use
            if p.grad is None:
                p.grad = torch.zeros_like(p)
        gys = ws.shared_gy[:Bp]
        gys[:B].copy_(gy)
        if Bp > B:
            gys[B:].zero_()
        da, dh, dn, dxs = c.shared_da[:Bp], c.shared_dh[:Bp], c.shared_dn[:Bp], c.shared_dx[:B]
        h, n, a = ws.shared_h[:Bp], ws.shared_n[:Bp], ws.shared_a[:Bp]
        Is, H = self.shared_inner, self.cfg.hidden
        grads = {"w13": self.shared_w13.grad.view(1, 2 * Is, H), "w2": self.shared_w2.grad.view(1, H, Is)}

        def wgrad(name, dy, xin):
            gemm.grouped_wgrad(dy, xin, plan.group_off, 1, out=grads[name], accumulate=True, max_ctas=plan.max_ctas)

        swiglu_mlp_backward(plan, ws.shared_w13, ws.shared_w2, n, h, a, gys, da, dh, dn, wgrad)
        K.rms_norm_bwd(dn[:B], x, ws.shared_rstd[:B], self.shared_g.detach(), dx=dxs, dgamma=self.shared_g.grad)
        return dxs

    def _backward_cuda(self, gy, B, logits=None, x=None, router=False):
        """:param logits: the gate logits of the forward when it computed router losses or the layer has the dense gate
        backward of the unnormalised softmax router
        :param x: the layer input of the forward, when the layer has a shared expert or an expert capacity
        :param router: the forward computed router losses (their gradient is added here)"""
        c, ws, sh, cfg = self.ctx, self.ws, self.shard, self.cfg
        k = cfg.k
        P = B * k
        epoch = c.next_epoch()
        idx, w, pos, pair_row = ws.idx[:P], ws.w[:P], ws.pos[:P], ws.pair_row[:P]
        gy = gy.to(torch.bfloat16)
        dlogits = torch.empty(B, sum(self.grid_size), dtype=torch.float32, device=gy.device)
        dense = dict(alive=c.alive, logits=logits) if self.dense_gate else {}
        capped = self.capacity_factor > 0.0   # a dropped pair: dw_j = <g_b, x_b>, and w_j * g_b joins dx
        K.gate_bwd(ws.yo_off, gy, idx, pair_row, w, dlogits, k, c.E_loc, self.grid_size, route_owner=ws.route_owner,
                   pass_x=x if capped else None, **self._score_args(P, B), **dense)
        if router:
            K.router_loss_bwd(logits, self.grid_size, alive=c.alive, f=ws.router_f, z=ws.router_z, Fb=ws.router_F,
                              aux_coef=self.router_aux_coef * self.router_grad_scale,
                              z_coef=self.router_z_coef * self.router_grad_scale, dlogits=dlogits,
                              score=self.router_score)
        K.scatter_rows(gy, w, idx, pos, None, pair_row, ws.gyd_off, c.flags_off, K.SLOT_GRAD, epoch, k, c.E_loc,
                       c.max_rows, ws.group_off, ws.group_rows, c.done_counter, c.status, align=c.align,
                       route_owner=ws.route_owner, num_groups=c.G_tot)
        if c.S:  # atomically accumulated (bias / norm) partial gradients of my shadow slots start from zero
            K.zero_slots(sh.g, sh.seg_sizes, c.G_tot, c.E_loc, c.S, sh.layout.small_mask)
        # the shared expert's backward needs only this rank's gradient: at world > 1 it runs while the peers' are in flight
        dxs = self._shared_expert_bwd(gy, x) if self.shared_inner else None
        if c.world > 1:  # the first consumers of the pushed gradients are the colsum / wgrad kernels
            K.signal_wait(c.flags_off, K.SLOT_GRAD, epoch, c.status, signal=False, wait=True)
        c.timer.mark("bwd_gate+dispatch_grad")
        plan, go, gr = self._expert_plan(), ws.group_off, sh.grads
        if c.small:
            # dW never reaches HBM: register accumulator -> AMSGrad epilogue -> p / m / v / vmax updated in place.  With
            # the overlap enabled the kernel goes to the optimizer stream, ordered after everything the main stream has
            # launched so far (in particular the dgrad that still reads the OLD weights); its inputs live in per-layer
            # buffers.  The optimizer step follows the whole backward in the reference (lib/runtime/expert_backend.py:85-90)
            opt, E = c.adam_kwargs(), self.E_loc
            main, side = torch.cuda.current_stream(c.device), c.opt_stream

            def wgrad(name, dy, xin):
                kw = dict(p=None, p_lo=sh.lo_views[name][:E], p_bf16=sh.bf16[name][:E]) if sh.split else \
                    dict(p=sh.raw_views[name][:E], p_bf16=sh.bf16[name])
                kw.update(m=sh.m_views[name][:E], v=sh.v_raw_views[name][:E],
                          vmax=sh.vmax_views[name][:E] if cfg.amsgrad else None, step=sh.step, **opt)
                if side is None:
                    K.wgrad_adam(dy, xin, go, ws.group_rows, **kw)
                    return
                side.wait_stream(main)
                with torch.cuda.stream(side):
                    K.wgrad_adam(dy, xin, go, ws.group_rows, max_ctas=c.opt_ctas, **kw)
                c._opt_pending = True

            K.bump_steps(sh.step, ws.step_rows)
        else:
            def wgrad(name, dy, xin):
                gemm.grouped_wgrad(dy, xin, go, c.G_tot, out=gr[name], accumulate=cfg.accumulate)

        if cfg.expert == "swiglu":
            # padding rows: scatter_rows zeroed them in xd and gyd, so da, dh and dn are zero there, and the RMSNorm
            # backward of a row with dn = 0 adds nothing to dgamma.  dgamma is added (+=) to the gradient buffer, which
            # the expert's optimizer step zeroes (with update_every_* it accumulates until then)
            swiglu_mlp_backward(plan, sh.bf16["w13"], sh.bf16["w2"], ws.n, ws.h, ws.a, ws.gyd, c.da, ws.dh13, c.dn, wgrad)
            K.rms_norm_bwd(c.dn, ws.xd, ws.rstd, sh.raw_views["g"], dx=c.dxd, dgamma=gr["g"], dres=ws.gyd,
                           tile_rows=plan.tile_rows, tile_group=plan.tile_group)
        else:
            ffn_backward(plan, sh.bf16, sh.raw_views, gr, ws.xd, (ws.h1, ws.a1, ws.h2, ws.a2),
                         (ws.mean1, ws.rstd1, ws.mean2, ws.rstd2), ws.gyd, c.da, ws.dh2, ws.dh1, c.dxd, wgrad)
        if c.small:
            # biases / norm weights: the ordinary fused AMSGrad restricted to the small segments
            small = sh.layout.small_mask
            K.adam_step(sh.p_raw, sh.g, sh.m, sh.v_raw, sh.vmax, sh.p_bf16, sh.seg_sizes, sh.slots, step=sh.step,
                        group_rows=ws.step_rows, zero_mask=small, G_active=self.E_loc, seg_mask=small, **opt)
            sh.w8_dirty = True
            c.timer.mark("expert_ffn_bwd(dgrad+ln+fused wgrad/AMSGrad)")
        else:
            c.timer.mark("expert_ffn_bwd(wgrad+dgrad+ln)")
            # ---- expert-side optimizer step (reference: ExpertBackend.apply_gradients right after backward)
            if c.S:  # the owners read every rank's partial gradients of the shadowed experts: all ranks must be done
                K.signal_wait(c.flags_off, K.SLOT_SHADOW, epoch, c.status, signal=True, wait=True)
            self.apply_expert_gradients()
            c.timer.mark("expert_adam")
        dx = torch.empty(B, cfg.hidden, dtype=torch.bfloat16, device=gy.device)
        K.combine_rows(c.dxd_off, idx, pair_row, None, dx, k, c.E_loc, flags_off=c.flags_off, slot=K.SLOT_DINPUT,
                       epoch=epoch, signal=c.world > 1, wait=c.world > 1, status=c.status, route_owner=ws.route_owner,
                       addend=dxs, **(dict(pass_self=gy, pass_w=w) if capped else {}))
        c.timer.mark("bwd_combine")
        return dx, dlogits

    def apply_expert_gradients(self):
        sh, cfg, ws, c = self.shard, self.cfg, self.ws, self.ctx
        rows, zero_mask = ws.step_rows, sh.layout.small_mask
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
            rows, zero_mask = sh.fire, (1 << len(sh.layout.names)) - 1
        K.bump_steps(sh.step, rows)
        K.adam_step(sh.p_raw, sh.g, sh.m, sh.v_raw, sh.vmax, sh.p_bf16, sh.seg_sizes, sh.slots, step=sh.step,
                    group_rows=rows, **c.adam_kwargs(), zero_mask=zero_mask, G_active=self.E_loc, world=c.world,
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
                leaves = {n: self.shard.views[n][e_local].detach().requires_grad_(True) for n in self.shard.layout.names}
                self._ref_leaves[e_local] = leaves
            return leaves
        return {n: self.shard.views[n][e_local].to(dtype) for n in self.shard.layout.names}

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
                rows, zero_mask = due.to(rows.dtype), (1 << len(sh.layout.names)) - 1
            sh.step += (rows > 0).to(sh.step.dtype)
            K.adam_step_ref(sh.p_raw, sh.g, sh.m, sh.v_raw, sh.vmax, sh.seg_sizes, self.E_loc, step=sh.step,
                            group_rows=rows, **cfg.adam_kwargs(), zero_mask=zero_mask)
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
        alive = self.ctx.alive if self.ctx is not None else getattr(self, "alive_ref", None)
        idx, w_sel = K.gate_topk_ref(logits.detach(), self.grid_size, cfg.k, alive=alive, fail_mask=fail_mask,
                                     bias=self.expert_bias, score=self.router_score, scale=self.routed_scale,
                                     n_group=self.n_group, topk_group=self.topk_group)
        if self.training and self.expert_bias is not None:
            with torch.no_grad():
                counts = torch.bincount(idx[idx >= 0].flatten(), minlength=cfg.num_experts)
                self.expert_bias.copy_(K.expert_bias_update_ref(counts, self.expert_bias, self.expert_bias_rate, alive))
        # differentiable weights: softmax over the selected logits, or their normalised sigmoid affinities; without
        # renormalisation the softmax over every live expert, or the sigmoid affinities, times the scale (DESIGN.md §6e)
        scores = K.product_key_scores(logits, self.grid_size)
        safe_idx = idx.clamp(min=0)
        if not self.norm_topk_prob and self.router_score == "softmax":
            weights = K.softmax_weights_ref(scores, idx, alive, self.routed_scale)
        elif not self.norm_topk_prob:
            sg = torch.sigmoid(torch.gather(scores, 1, safe_idx))
            weights = torch.where(idx >= 0, self.routed_scale * sg, torch.zeros_like(sg))
        elif self.router_score == "sigmoid":
            weights = K.sigmoid_weights_ref(torch.gather(scores, 1, safe_idx), idx >= 0, self.routed_scale)
        else:
            sel = torch.gather(scores, 1, safe_idx).masked_fill(idx < 0, float("-inf"))
            weights = torch.softmax(sel, dim=-1)
            weights = torch.where(idx >= 0, weights, torch.zeros_like(weights))
        xf = x.float()
        out = torch.zeros(x.shape[0], cfg.hidden, dtype=torch.float32, device=x.device)
        rnd = (lambda t: t.to(torch.bfloat16).float()) if emulate_bf16 else (lambda t: t)
        routed = idx   # the router losses see every routed pair
        if self.capacity_factor > 0.0:
            # expert capacity (DESIGN.md §6f): the pairs past C of their expert, in token order, see the expert as the
            # identity; the experts and their optimizer steps see the kept pairs only
            kept, C, dropped = K.capacity_keep_ref(idx, self.capacity_factor, cfg.num_experts)
            self._ref_capacity = (C, dropped)
            drop_w = torch.where(kept | (idx < 0), torch.zeros_like(weights), weights)
            out = out + drop_w.sum(1, keepdim=True) * rnd(xf)
            idx = torch.where(kept, idx, torch.full_like(idx, -1))
        if self.training:
            rows = torch.bincount(idx[idx >= 0].flatten() - self.first_expert, minlength=self.E_loc)
            self._ref_rows = rows if self._ref_rows is None else self._ref_rows + rows
        for e in idx[idx >= 0].unique().tolist():
            le = e - self.first_expert
            p = self._expert_params(le)
            if emulate_bf16:
                p = {n: (rnd(v) if n.startswith("w") else v) for n, v in p.items()}
            tok, slot = torch.nonzero(idx == e, as_tuple=True)
            ye = self._expert_ref(p, rnd(xf[tok]), rnd)
            out = out.index_put((tok,), ye * weights[tok, slot].unsqueeze(-1), accumulate=True)
        if self.shared_inner:   # the shared expert: weight 1, no residual; autograd reaches its parameters
            p = self._shared_segments()
            if emulate_bf16:
                p = {n: (rnd(v) if n.startswith("w") else v) for n, v in p.items()}
            out = out + rnd(self._gated_branch(p, rnd(xf), rnd))
        if self.training and self.router_on:
            counts = torch.bincount(routed[routed >= 0].flatten(), minlength=cfg.num_experts)
            l_aux, l_z = K.router_loss_ref(logits, self.grid_size, counts, alive=alive, score=self.router_score)
            with torch.no_grad():
                self.router_loss.copy_(torch.stack([l_aux, l_z]).detach())
            if torch.is_grad_enabled() and logits.requires_grad:
                aux = self.router_grad_scale * (self.router_aux_coef * l_aux + self.router_z_coef * l_z)
                out = _AddRouterLoss.apply(out, aux)
        return out.to(x.dtype)

    def _gated_branch(self, p, xe, rnd):
        """w2(silu(w1 n) * w3 n), n = RMSNorm(x), of GatedFeedforwardBlock segments ``p`` in fp32, without the residual
        and without rounding the result"""
        n = rnd(F.rms_norm(xe, (self.cfg.hidden,), p["g"], GATED_EPS))
        hg, hu = rnd(F.linear(n, p["w13"])).chunk(2, dim=-1)
        a = rnd(F.silu(hg) * hu)
        return F.linear(a, p["w2"])

    def _expert_ref(self, p, xe, rnd):
        """one expert on its rows in fp32; ``rnd`` rounds where the GPU path stores bf16"""
        cfg = self.cfg
        if cfg.expert == "swiglu":   # GatedFeedforwardBlock: x + w2(silu(w1 n) * w3 n), n = RMSNorm(x)
            return rnd(self._gated_branch(p, xe, rnd) + xe)
        h1 = rnd(F.linear(xe, p["w1"], p["b1"]))
        a1 = rnd(F.relu(F.layer_norm(h1, (cfg.inner,), p["g1"], p["be1"])))
        h2 = rnd(F.linear(a1, p["w2"], p["b2"]))
        a2 = rnd(F.relu(F.layer_norm(h2, (cfg.inner,), p["g2"], p["be2"])))
        return rnd(F.linear(a2, p["w3"], p["b3"]) + xe)


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
