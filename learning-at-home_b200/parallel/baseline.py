"""
The BASELINE formulation of the same DMoE step: torch.topk + index_select permute + ``all_to_all_single`` (NCCL on GPUs,
gloo on CPU) + cuBLAS ``F.linear`` + ``torch.optim.Adam`` per expert.  "A path that only calls NCCL all-to-all is the
baseline, not the product" (BASELINE.json) — this module exists to be measured against (``bench.py --impl baseline``)
and as a second, independently written oracle for the fused engine (same routing, same maths, autograd everywhere).

Experts are real ``FeedforwardBlock`` modules (reference architecture, /root/reference/experiments/throughput/layers.py),
or ``GatedFeedforwardBlock`` modules with ``DMoEConfig(expert="swiglu")``; ``DMoEConfig(shared_inner_dim=...)`` adds a real
``GatedFeedforwardBlock`` shared expert whose ``module(x) - x`` every token receives.
"""
import math
from typing import List, Optional

import torch
import torch.distributed as dist
import torch.nn as nn
import torch.nn.functional as F

from ..models.layers import FeedforwardBlock, GatedFeedforwardBlock
from ..ops.kernels import product_key_scores
from .engine import (GATED_EPS, DMoEConfig, refuse_expert_bias, refuse_expert_capacity, refuse_group_limited_routing,
                     refuse_router_losses, refuse_router_score)


class _AllToAll(torch.autograd.Function):
    """differentiable all_to_all_single with explicit split sizes (backward = the transposed exchange)"""

    @staticmethod
    def forward(ctx, x, send_counts: List[int], recv_counts: List[int], group):
        ctx.send_counts, ctx.recv_counts, ctx.group = send_counts, recv_counts, group
        out = x.new_empty((sum(recv_counts), *x.shape[1:]))
        if dist.is_initialized() and dist.get_world_size(group) > 1:
            dist.all_to_all_single(out, x.contiguous(), recv_counts, send_counts, group=group)
        else:
            out.copy_(x)
        return out

    @staticmethod
    def backward(ctx, grad):
        out = grad.new_empty((sum(ctx.send_counts), *grad.shape[1:]))
        if dist.is_initialized() and dist.get_world_size(ctx.group) > 1:
            dist.all_to_all_single(out, grad.contiguous(), ctx.send_counts, ctx.recv_counts, group=ctx.group)
        else:
            out.copy_(grad)
        return out, None, None, None


class BaselineDMoE(nn.Module):
    def __init__(self, cfg: DMoEConfig, layer_index: int = 0, group=None, device=None, dtype=torch.float32):
        super().__init__()
        refuse_router_losses(cfg, "BaselineDMoE")
        refuse_expert_bias(cfg, "BaselineDMoE")
        refuse_router_score(cfg, "BaselineDMoE")
        refuse_group_limited_routing(cfg, "BaselineDMoE")
        refuse_expert_capacity(cfg, "BaselineDMoE")
        self.cfg, self.group, self.dtype = cfg, group, dtype
        distributed = dist.is_available() and dist.is_initialized()
        self.world = dist.get_world_size(group) if distributed else 1
        self.rank = dist.get_rank(group) if distributed else 0
        assert cfg.num_experts % self.world == 0
        self.E_loc = cfg.num_experts // self.world
        self.first_expert = self.rank * self.E_loc
        self.proj = nn.Linear(cfg.hidden, sum(cfg.grid_size))
        experts = []
        for le in range(self.E_loc):  # per-(layer, global expert) seed: identical weights for any number of ranks
            with torch.random.fork_rng(devices=[]):
                torch.manual_seed(cfg.seed * 1000003 + layer_index * 10007 + self.first_expert + le)
                experts.append(GatedFeedforwardBlock(cfg.hidden, cfg.inner, eps=GATED_EPS) if cfg.expert == "swiglu"
                               else FeedforwardBlock(cfg.hidden))
        self.experts = nn.ModuleList(experts)
        # the shared expert: a trainer-side module (replicated, averaged over ranks by BaselineTrainer), like proj
        self.shared_expert = (GatedFeedforwardBlock(cfg.hidden, cfg.shared_inner_dim, eps=GATED_EPS)
                              if cfg.shared_inner_dim else None)
        if device is not None:
            self.to(device)
        self.expert_optimizers = [torch.optim.Adam(e.parameters(), lr=cfg.lr, betas=cfg.betas, eps=cfg.eps,
                                                   amsgrad=cfg.amsgrad, weight_decay=cfg.weight_decay,
                                                   decoupled_weight_decay=cfg.decoupled_weight_decay)
                                  for e in self.experts]
        self.fail_mask = None

    def load_from_shard(self, shard):
        """copy the parameters of a fused-engine ExpertShard (same rank / same experts)"""
        with torch.no_grad():
            for le, expert in enumerate(self.experts):
                expert.load_state_dict(shard.layout.module_state({n: shard.views[n][le] for n in shard.layout.names}))

    def non_expert_parameters(self):
        shared = list(self.shared_expert.parameters()) if self.shared_expert is not None else []
        return list(self.proj.parameters()) + shared

    def forward(self, x):
        cfg, k = self.cfg, self.cfg.k
        B = x.shape[0]
        logits = self.proj(x.float())
        scores = product_key_scores(logits, cfg.grid_size)
        masked = scores if self.fail_mask is None else scores.masked_fill(self.fail_mask, float("-inf"))
        top_v, top_i = torch.topk(masked, k, dim=-1)
        valid = torch.isfinite(top_v)
        weights = torch.softmax(top_v.masked_fill(~valid, float("-inf")), dim=-1)
        weights = torch.where(valid, weights, torch.zeros_like(weights))

        flat_e = top_i.reshape(-1)
        flat_valid = valid.reshape(-1)
        pair_ids = torch.nonzero(flat_valid).flatten()
        order = pair_ids[torch.argsort(flat_e[pair_ids], stable=True)]  # pairs sorted by global expert id
        sorted_e = flat_e[order]
        send_per_expert = torch.bincount(sorted_e, minlength=cfg.num_experts)
        if self.world > 1:
            recv_per_expert = torch.empty_like(send_per_expert)
            dist.all_to_all_single(recv_per_expert, send_per_expert, group=self.group)  # [src rank, local expert]
        else:
            recv_per_expert = send_per_expert.clone()
        send_counts = send_per_expert.view(self.world, self.E_loc).sum(1).tolist()
        recv_matrix = recv_per_expert.view(self.world, self.E_loc)
        recv_counts = recv_matrix.sum(1).tolist()

        tokens = torch.div(order, k, rounding_mode="floor")
        sent = x.to(self.dtype)[tokens]
        received = _AllToAll.apply(sent, send_counts, recv_counts, self.group)
        # received rows are ordered (src rank, local expert); regroup per expert
        le_of_row = torch.repeat_interleave(
            torch.arange(self.E_loc, device=x.device).repeat(self.world), recv_matrix.reshape(-1))
        perm = torch.argsort(le_of_row, stable=True)
        grouped = received[perm]
        sizes = torch.bincount(le_of_row, minlength=self.E_loc).tolist()
        outs, start = [], 0
        for le, n in enumerate(sizes):
            if n:
                outs.append(self.experts[le](grouped[start: start + n]))
            start += n
        processed = torch.cat(outs, 0) if outs else grouped
        back = torch.empty_like(processed)
        back = back.index_copy(0, perm, processed) if len(perm) else processed
        returned = _AllToAll.apply(back, recv_counts, send_counts, self.group)
        w_pairs = weights.reshape(-1)[order].to(returned.dtype)
        out = torch.zeros(B, cfg.hidden, dtype=returned.dtype, device=x.device)
        out = out.index_add(0, tokens, returned * w_pairs.unsqueeze(-1))
        if self.shared_expert is not None:
            xs = x.to(self.dtype)
            out = out + (self.shared_expert(xs) - xs)
        self._rows = torch.tensor(sizes)
        return out.to(x.dtype)

    def apply_expert_gradients(self):
        """step the optimizer of every expert that received rows (server-side update semantics)"""
        for le, opt in enumerate(self.expert_optimizers):
            if int(self._rows[le]) > 0:
                opt.step()
            opt.zero_grad()


class BaselineClassifier(nn.Module):
    def __init__(self, cfg: DMoEConfig, group=None, device=None, dtype=torch.float32):
        super().__init__()
        self.cfg = cfg
        self.stem = nn.Linear(cfg.in_features, cfg.hidden)
        self.blocks = nn.ModuleList([BaselineDMoE(cfg, i, group, device, dtype) for i in range(cfg.num_layers)])
        self.norm = nn.LayerNorm(cfg.hidden)
        self.head = nn.Linear(cfg.hidden, cfg.num_classes)
        if device is not None:
            self.to(device)

    def forward(self, x):
        h = self.stem(x)
        for block in self.blocks:
            h = block(h)
        return self.head(self.norm(h.float()))

    def non_expert_parameters(self):
        params = list(self.stem.parameters()) + list(self.norm.parameters()) + list(self.head.parameters())
        for block in self.blocks:
            params += block.non_expert_parameters()
        return params


class BaselineTrainer:
    """NCCL(+cuBLAS) baseline trainer with the same interface as DMoETrainer"""

    def __init__(self, cfg: DMoEConfig, group=None, device=None, dtype=torch.float32):
        refuse_router_losses(cfg, "BaselineTrainer")
        refuse_expert_bias(cfg, "BaselineTrainer")
        refuse_router_score(cfg, "BaselineTrainer")
        refuse_group_limited_routing(cfg, "BaselineTrainer")
        refuse_expert_capacity(cfg, "BaselineTrainer")
        self.cfg, self.group = cfg, group
        self.device = device or (torch.device("cuda", torch.cuda.current_device()) if torch.cuda.is_available()
                                 else torch.device("cpu"))
        distributed = dist.is_available() and dist.is_initialized()
        self.world = dist.get_world_size(group) if distributed else 1
        torch.manual_seed(cfg.seed)
        self.model = BaselineClassifier(cfg, group, self.device, dtype)
        self.params = self.model.non_expert_parameters()
        self.opt = torch.optim.Adam(self.params, lr=cfg.lr, betas=cfg.betas, eps=cfg.eps, amsgrad=cfg.amsgrad,
                                    weight_decay=cfg.weight_decay, decoupled_weight_decay=cfg.decoupled_weight_decay)
        self.autocast = dtype == torch.bfloat16

    def train_step_device(self, x, y):
        self.model.train()
        with torch.autocast(self.device.type, dtype=torch.bfloat16, enabled=self.autocast):
            logits = self.model(x)
        loss = F.cross_entropy(logits.float(), y)
        self.opt.zero_grad()
        loss.backward()
        for block in self.model.blocks:
            block.apply_expert_gradients()
        if self.world > 1:
            flat = torch.cat([p.grad.reshape(-1) for p in self.params])
            dist.all_reduce(flat, group=self.group)
            flat /= self.world
            off = 0
            for p in self.params:
                p.grad.copy_(flat[off: off + p.numel()].view_as(p))
                off += p.numel()
        self.opt.step()
        return loss.detach()

    def train_step(self, x_host, y_host) -> float:
        x = x_host.to(self.device, non_blocking=True)
        y = y_host.to(self.device, non_blocking=True)
        return float(self.train_step_device(x, y))
