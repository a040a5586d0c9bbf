"""
The GPU-BOUND NCCL + cuBLAS formulation of the same DMoE training step — "the baseline, not the product" (BASELINE.json),
written the way a competent PyTorch user would write it, with NO host synchronisation inside a step:

  gate            same gate as the engine (emulator: LayerNorm(x) @ normalize(keys); or product-key proj), torch.topk
  dispatch        fixed-capacity buffers [experts, capacity, hidden] filled by one index_put (sort + rank inside the expert)
  all-to-all      ``dist.all_to_all_single`` with EQUAL splits (NCCL) — shapes never depend on the routing, so there is no
                  .tolist() / .item() anywhere
  experts         stacked parameters [E_loc, ...]; three ``torch.bmm`` (cuBLAS batched GEMM, bf16 autocast of fp32 masters),
                  ``F.layer_norm`` + per-expert affine, autograd backward; SwiGLU experts (``expert="swiglu"``):
                  ``F.rms_norm`` * per-expert weight, one bmm over [W1 | W3], silu(g) * u, one bmm over W2
  optimizers      ONE fused ``torch.optim.Adam(amsgrad=True, fused=True)`` over the stacked expert parameters, one over the
                  trainer parameters (gradients all-reduced with NCCL)

Differences from the engine's semantics, all in the baseline's favour or neutral: rows beyond an expert's capacity are
DROPPED (the engine never drops); every expert is stepped every step (the engine and the reference skip experts that
received no rows).  ``parallel/baseline.py`` (per-expert modules, exact semantics, host-synchronising) stays as the second
numerical oracle of the tests; this module is what ``bench.py --impl baseline`` measures.
"""
import math
from typing import Optional

import torch
import torch.distributed as dist
import torch.nn as nn
import torch.nn.functional as F

from ..ops.kernels import product_key_scores
from .engine import (GATED_EPS, DMoEConfig, refuse_expert_bias, refuse_expert_capacity, refuse_group_limited_routing,
                     refuse_router_losses, refuse_router_score, refuse_shared_expert)


class _EqualAllToAll(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, group):
        ctx.group = group
        if not (dist.is_initialized() and dist.get_world_size(group) > 1):
            return x
        out = torch.empty_like(x)
        dist.all_to_all_single(out, x.contiguous(), group=group)
        return out

    @staticmethod
    def backward(ctx, grad):
        if not (dist.is_initialized() and dist.get_world_size(ctx.group) > 1):
            return grad, None
        out = torch.empty_like(grad)
        dist.all_to_all_single(out, grad.contiguous(), group=ctx.group)
        return out, None


class FastBaselineDMoE(nn.Module):
    def __init__(self, cfg: DMoEConfig, layer_index: int, capacity: int, group=None, device=None):
        super().__init__()
        refuse_router_losses(cfg, "FastBaselineDMoE")
        refuse_expert_bias(cfg, "FastBaselineDMoE")
        refuse_router_score(cfg, "FastBaselineDMoE")
        refuse_group_limited_routing(cfg, "FastBaselineDMoE")
        refuse_expert_capacity(cfg, "FastBaselineDMoE")
        refuse_shared_expert(cfg, "FastBaselineDMoE")
        self.cfg, self.group, self.capacity = cfg, group, capacity
        distributed = dist.is_available() and dist.is_initialized()
        self.world = dist.get_world_size(group) if distributed else 1
        self.rank = dist.get_rank(group) if distributed else 0
        E, H, I = cfg.num_experts, cfg.hidden, cfg.inner
        self.E_loc = E // self.world
        if cfg.gate_mode == "emulator":
            self.gating_pre_normalize = nn.LayerNorm(H).requires_grad_(False)
            self.expert_keys = nn.Parameter(torch.randn(H, E), requires_grad=False)
            self.proj = None
        else:
            self.proj = nn.Linear(H, sum(cfg.grid_size))

        def lin(o, i):
            bound = 1.0 / math.sqrt(i)
            return (nn.Parameter(torch.empty(self.E_loc, i, o, device=device).uniform_(-bound, bound)),
                    nn.Parameter(torch.empty(self.E_loc, 1, o, device=device).uniform_(-bound, bound)))

        if cfg.expert == "swiglu":
            # GatedFeedforwardBlock: RMSNorm weight, [W1 | W3] as one [H, 2I] bmm operand (w1 columns first), W2
            self.w13 = nn.Parameter(torch.empty(self.E_loc, H, 2 * I, device=device).uniform_(-1 / math.sqrt(H), 1 / math.sqrt(H)))
            self.w2 = nn.Parameter(torch.empty(self.E_loc, I, H, device=device).uniform_(-1 / math.sqrt(I), 1 / math.sqrt(I)))
            self.g = nn.Parameter(torch.ones(self.E_loc, 1, H, device=device))
            return
        self.w1, self.b1 = lin(I, H)
        self.w2, self.b2 = lin(I, I)
        self.w3, self.b3 = lin(H, I)
        self.g1, self.be1 = nn.Parameter(torch.ones(self.E_loc, 1, I, device=device)), nn.Parameter(torch.zeros(self.E_loc, 1, I, device=device))
        self.g2, self.be2 = nn.Parameter(torch.ones(self.E_loc, 1, I, device=device)), nn.Parameter(torch.zeros(self.E_loc, 1, I, device=device))

    def expert_parameters(self):
        if self.cfg.expert == "swiglu":
            return [self.g, self.w13, self.w2]
        return [self.w1, self.b1, self.g1, self.be1, self.w2, self.b2, self.g2, self.be2, self.w3, self.b3]

    def gate_parameters(self):
        return list(self.proj.parameters()) if self.proj is not None else []

    def forward(self, x):
        cfg, k, C = self.cfg, self.cfg.k, self.capacity
        B, H = x.shape
        E = cfg.num_experts
        if self.proj is None:
            scores = self.gating_pre_normalize(x.float()) @ F.normalize(self.expert_keys, dim=-1)
        else:
            scores = product_key_scores(self.proj(x.float()), cfg.grid_size)
        top_v, top_i = torch.topk(scores, k, dim=-1)
        weights = torch.softmax(top_v, dim=-1)
        flat_e = top_i.reshape(-1)                                            # [B*k]
        order = torch.argsort(flat_e, stable=True)
        sorted_e = flat_e[order]
        first = torch.searchsorted(sorted_e, torch.arange(E, device=x.device))
        pos = torch.arange(B * k, device=x.device) - first[sorted_e]          # rank of the pair inside its expert
        keep = pos < C
        slot = torch.where(keep, sorted_e * C + pos, torch.full_like(pos, E * C))   # dropped pairs -> scratch row
        tokens = torch.div(order, k, rounding_mode="floor")
        buf = torch.zeros(E * C + 1, H, dtype=torch.bfloat16, device=x.device)
        buf = buf.index_copy(0, slot, x.to(torch.bfloat16)[tokens])
        send = buf[:E * C].view(self.world, self.E_loc * C, H)                # destination rank major
        recv = _EqualAllToAll.apply(send, self.group)                        # [src rank, E_loc * C, H]
        rows = recv.view(self.world, self.E_loc, C, H).transpose(0, 1).reshape(self.E_loc, self.world * C, H)
        if not x.is_cuda:
            rows = rows.float()   # CPU smoke path of this arm: fp32 maths
        with torch.autocast("cuda", dtype=torch.bfloat16, enabled=x.is_cuda):
            if cfg.expert == "swiglu":
                y = self._gated_experts(rows)
            else:
                y = self._ffn_experts(rows)
        y = y.to(torch.bfloat16).view(self.E_loc, self.world, C, H).transpose(0, 1).reshape(self.world, self.E_loc * C, H)
        back = _EqualAllToAll.apply(y.contiguous(), self.group).reshape(E * C, H)
        back = torch.cat([back, back.new_zeros(1, H)], 0)
        pair_out = back[slot] * (weights.reshape(-1)[order] * keep).to(back.dtype).unsqueeze(-1)
        out = torch.zeros(B, H, dtype=pair_out.dtype, device=x.device).index_add(0, tokens, pair_out)
        return out.to(x.dtype)

    def _ffn_experts(self, rows):
        cfg = self.cfg
        h = torch.baddbmm(self.b1, rows, self.w1)
        a = F.relu(F.layer_norm(h, (cfg.inner,)) * self.g1 + self.be1)
        h = torch.baddbmm(self.b2, a, self.w2)
        a = F.relu(F.layer_norm(h, (cfg.inner,)) * self.g2 + self.be2)
        return torch.baddbmm(self.b3, a, self.w3) + rows

    def _gated_experts(self, rows):
        """rms_norm -> bmm over [W1 | W3] -> silu(g) * u -> bmm(W2) + rows"""
        n = F.rms_norm(rows, (self.cfg.hidden,), eps=GATED_EPS) * self.g
        hg, hu = torch.bmm(n, self.w13).chunk(2, dim=-1)
        return torch.bmm(F.silu(hg) * hu, self.w2) + rows


class FastBaselineTrainer:
    def __init__(self, cfg: DMoEConfig, group=None, device=None, capacity_factor: float = 0.0):
        refuse_router_losses(cfg, "FastBaselineTrainer")
        refuse_expert_bias(cfg, "FastBaselineTrainer")
        refuse_router_score(cfg, "FastBaselineTrainer")
        refuse_group_limited_routing(cfg, "FastBaselineTrainer")
        refuse_expert_capacity(cfg, "FastBaselineTrainer")
        refuse_shared_expert(cfg, "FastBaselineTrainer")
        self.cfg, self.group = cfg, group
        self.device = device or torch.device("cuda", torch.cuda.current_device())
        distributed = dist.is_available() and dist.is_initialized()
        self.world = dist.get_world_size(group) if distributed else 1
        B, k, E = cfg.tokens_per_rank, cfg.k, cfg.num_experts
        mean_rows = B * k / E
        # rows one rank may send to one expert: never more than its batch; small batches get the exact bound (no drops)
        self.capacity = int(min(B, max(16, math.ceil(mean_rows * (capacity_factor or (B if mean_rows < 64 else 2.0))))))
        self.capacity = (self.capacity + 15) // 16 * 16
        torch.manual_seed(cfg.seed)
        dev = self.device
        self.stem = nn.Linear(cfg.in_features, cfg.hidden).to(dev)
        self.blocks = [FastBaselineDMoE(cfg, i, self.capacity, group, dev).to(dev) for i in range(cfg.num_layers)]
        self.norm = nn.LayerNorm(cfg.hidden).to(dev)
        self.head = nn.Linear(cfg.hidden, cfg.num_classes).to(dev)
        self.trainer_params = list(self.stem.parameters()) + list(self.norm.parameters()) + list(self.head.parameters())
        for b in self.blocks:
            self.trainer_params += b.gate_parameters()
        kw = dict(lr=cfg.lr, betas=cfg.betas, eps=cfg.eps, amsgrad=cfg.amsgrad, weight_decay=cfg.weight_decay,
                  decoupled_weight_decay=cfg.decoupled_weight_decay)
        fused = dict(fused=True) if dev.type == "cuda" else {}
        self.opt = torch.optim.Adam(self.trainer_params, **kw, **fused)
        self.expert_opt = torch.optim.Adam([p for b in self.blocks for p in b.expert_parameters()], **kw, **fused)

    def train_step_device(self, x, y):
        h = self.stem(x.float()).to(torch.bfloat16) if x.is_cuda else self.stem(x)
        for block in self.blocks:
            h = block(h)
        logits = self.head(self.norm(h.float()))
        loss = F.cross_entropy(logits, y)
        self.opt.zero_grad(set_to_none=True)
        self.expert_opt.zero_grad(set_to_none=True)
        loss.backward()
        self.expert_opt.step()
        if self.world > 1:
            flat = torch.cat([p.grad.reshape(-1) for p in self.trainer_params])
            dist.all_reduce(flat, group=self.group)
            flat /= self.world
            off = 0
            for p in self.trainer_params:
                p.grad = flat[off: off + p.numel()].view_as(p)
                off += p.numel()
        self.opt.step()
        return loss.detach()
