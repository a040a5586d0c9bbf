"""Fixtures and helpers shared by the routing test modules: CPU configs and relative errors, the step counters and a
world-1 symmetric heap, the gate runner and its pos oracle, the load probes of the CPU trainer tests, and one fused
layer against its bf16-emulating CPU oracle.  A test module imports the fixtures it uses by name."""
import ctypes
import math
from types import SimpleNamespace

import pytest
import torch

import lah_b200  # noqa: F401
from lah_b200.ops import kernels as K
from lah_b200.parallel import engine as E

#: ``rel`` arguments of the comparisons taken in float64
F64 = (torch.float64, 1e-30)


@pytest.fixture
def one_thread():
    """the CPU trainer tests run many tiny ops: one intra-op thread is faster, and does not compete with the threads
    other tests of the session may have left behind"""
    n = torch.get_num_threads()
    torch.set_num_threads(1)
    yield
    torch.set_num_threads(n)


def cpu_cfg(**kw):
    base = dict(hidden=64, grid_size=(4, 4), k=4, num_layers=1, in_features=16, tokens_per_rank=64, seed=5)
    base.update(kw)
    return E.DMoEConfig(**base)


def rel(a, b, dtype=torch.float32, floor=1e-12):
    """relative L2 error of a against b, in ``dtype``"""
    a, b = a.detach().to(dtype), b.detach().to(dtype)
    return float((a - b).norm() / b.norm().clamp_min(floor))


def _installed():
    """the step counters and the poison word installed now (device pointers, None when none is)"""
    lib = K._lib()
    lib.lah_get_epoch_base.restype = ctypes.c_void_p
    lib.lah_get_poison_word.restype = ctypes.c_void_p
    return lib.lah_get_epoch_base(), lib.lah_get_poison_word()


@pytest.fixture
def step_counters():
    """the gate adds the device token base (step counters [2:4]) to its failure-injection stream: zeroed counters,
    installed for the test's direct kernel calls; whatever was installed before is put back"""
    prev, _ = _installed()
    ctr = torch.zeros(4, dtype=torch.int32, device="cuda")
    K.set_step_counters(ctr)
    yield ctr
    torch.cuda.synchronize()
    K._lib().lah_set_step_counters(ctypes.c_void_p(prev))


@pytest.fixture(scope="module")
def world1():
    """a world-1 symmetric heap made directly (no EngineContext), whose rank is its only peer: flag words, the
    count-exchange table and one 96 MB receive region, with its own step counters, status / poison word and done
    counter.  The step counters and the poison word installed before are put back"""
    from lah_b200.ops import native
    from lah_b200.parallel.symmetric import SymmetricHeap
    prev_ctr, prev_poison = _installed()
    heap = SymmetricHeap(128 << 20)
    flags, flags_off = heap.alloc((K.NUM_SLOTS, K.MAX_WORLD), torch.int32)
    cnt_all, cnt_all_off = heap.alloc((K.MAX_WORLD, K.LAYOUT_MAX_E), torch.int32)
    region, region_off = heap.alloc((96 << 20,), torch.uint8)
    i32 = dict(dtype=torch.int32, device="cuda")
    w = SimpleNamespace(heap=heap, native=native, flags=flags, flags_off=flags_off, cnt_all=cnt_all,
                        cnt_all_off=cnt_all_off, region=region, region_off=region_off, step_ctr=torch.zeros(4, **i32),
                        status=torch.zeros(4, **i32), done_counter=torch.zeros(1, **i32))
    yield w
    torch.cuda.synchronize()
    lib = K._lib()
    lib.lah_set_step_counters(ctypes.c_void_p(prev_ctr))
    lib.lah_set_poison_word(ctypes.c_void_p(prev_poison))
    heap.close()


@pytest.fixture
def rt(world1):
    """world1 with its peer table and process-global counters (re)installed and zeroed: an EngineContext made by another
    test installs its own and clears them on close"""
    w = world1
    K.set_peers(w.heap.peer_bases, 0)
    K.set_multicast(0)
    K.set_step_counters(w.step_ctr)
    K.set_poison_word(w.status)
    w.status.zero_()
    w.step_ctr.zero_()
    w.done_counter.zero_()
    return w


def run_gate(logits, grid, k, *, alive, rate, bias, score="softmax", scale=1.0, norm=True, n_group=1, topk_group=1):
    """gate_topk (seed 99, token offset 0) into outputs prefilled with garbage: idx, w, pos [B, k], counts [E], and sig
    [B, k] (sigmoid router) and lse [B] (unnormalised softmax router), None where the setting writes none"""
    B = logits.shape[0]
    idx = torch.full((B * k,), 12345, dtype=torch.int32, device="cuda")
    pos, w = torch.full_like(idx, 12345), torch.full((B * k,), 7.0, device="cuda")
    sig = torch.full((B * k,), 7.0, device="cuda") if score == "sigmoid" else None
    lse = torch.full((B,), 7.0, device="cuda") if score == "softmax" and not norm else None
    counts = torch.zeros(math.prod(grid), dtype=torch.int32, device="cuda")
    K.gate_topk(logits, grid, k, alive=alive, failure_rate=rate, seed=99, token_offset=0, idx=idx, w=w, pos=pos,
                counts=counts, bias=bias, score=score, scale=scale, sig=sig, norm=norm, lse=lse, n_group=n_group,
                topk_group=topk_group)
    torch.cuda.synchronize()
    return idx.view(B, k), w.view(B, k), pos.view(B, k), counts, None if sig is None else sig.view(B, k), lse


def slots(idx):
    """pos oracle: the number of earlier pairs (token-major) routed to the same expert; 0 for missing pairs"""
    flat = idx.reshape(-1).long()
    order = torch.argsort(flat, stable=True)
    srt = flat[order]
    first = torch.searchsorted(srt, srt, side="left")
    pos = torch.empty_like(flat)
    pos[order] = torch.arange(flat.numel(), device=flat.device) - first
    return torch.where(flat >= 0, pos, torch.zeros_like(pos)).view_as(idx)


def load(trainer, x):
    """max / mean rows per expert of every layer on batch x (eval-mode routing, with the layers' biases)"""
    out, h = [], trainer.model.stem(x)
    with torch.no_grad():
        for block in trainer.model.blocks:
            idx, _ = K.gate_topk_ref(block.gate_logits(h, block.proj), block.grid_size, block.cfg.k,
                                     bias=block.expert_bias, score=block.router_score)
            rows = torch.bincount(idx[idx >= 0].flatten(), minlength=block.cfg.num_experts).float()
            out.append(float(rows.max() / rows.mean()))
            h = block(h)
    return out


def collapse(block, gate):
    with torch.no_grad():
        if gate == "product_key":   # the gate's bias favours experts 0 and 1
            block.proj.bias[:2] += 2.0
        else:                       # frozen keys whose first two columns win most rows
            block.gating_pre_normalize.bias.fill_(0.5)
            block.expert_keys[:, :2] += 0.5


def layer_against_the_oracle(cfg, *, check, prepare=None, bias_step=1 / 16, max_mismatch=0, dx=False,
                             precision=(torch.float32, 1e-12)):
    """one training forward and backward of the fused layer on 512 random bf16 rows against the bf16-emulating CPU
    oracle (run on the GPU) with the same weights.  A layer with expert biases starts from multiples of ``bias_step`` in
    [-8, 8] * bias_step, exact in any float32 sum; then ``prepare(layer)`` runs, without autograd, before the oracle
    copies the layer's state.

    Checked here: the status word; at most ``max_mismatch`` tokens routed unlike the oracle's top-k; the count table
    against the routed pairs; then ``check(r)``, the module's own assertions, with ``r`` holding ctx, layer, oracle,
    logits, the starting biases bias0, the kernel's idx and w [B, k], the oracle's ridx and rw, and ``same``, the
    tokens routed alike; last, the relative L2 errors ``rel(..., *precision)`` of y (< 2e-2), dlogits (< 5e-2) and,
    with ``dx``, dx (< 3e-2)."""
    ctx = E.EngineContext(cfg)
    try:
        layer = E.FusedDMoE(cfg, ctx).cuda().train()
        oracle = E.FusedDMoE(cfg, device=torch.device("cuda")).cuda().train()
        oracle.ref_emulate_bf16 = True
        with torch.no_grad():
            if layer.expert_bias is not None:
                layer.expert_bias.copy_((torch.randint(-8, 9, (cfg.num_experts,)).float() * bias_step).cuda())
            if prepare is not None:
                prepare(layer)
            oracle.load_state_dict(layer.state_dict())
            oracle.shard.p.copy_(layer.shard.p[:oracle.shard.p.numel()])
        bias0 = None if layer.expert_bias is None else layer.expert_bias.clone()
        B = 512
        x = torch.randn(B, cfg.hidden, device="cuda").to(torch.bfloat16)
        gy = torch.randn(B, cfg.hidden, device="cuda").to(torch.bfloat16)
        logits = layer.gate_logits(x, layer.proj).detach()
        xf, lg = x.clone().requires_grad_(dx), logits.clone().requires_grad_(True)
        y = E._FusedDMoEFunction.apply(xf, lg, layer)
        idx = layer.ws.idx[:B * cfg.k].view(B, cfg.k).long().clone()
        y.backward(gy)
        torch.cuda.synchronize()
        ctx.check_status()
        xr, lr_ = x.float().requires_grad_(dx), logits.clone().requires_grad_(True)
        yr = oracle._forward_ref(xr, lr_, emulate_bf16=True)
        yr.backward(gy.float())
        ridx, rw = K.gate_topk_ref(logits, cfg.grid_size, cfg.k, alive=ctx.alive, bias=bias0, score=cfg.router_score,
                                   scale=cfg.routed_scaling_factor, n_group=cfg.n_group, topk_group=cfg.topk_group,
                                   norm=cfg.norm_topk_prob)
        same = (idx == ridx).all(1)
        assert int((~same).sum()) <= max_mismatch, int((~same).sum())
        E_ = cfg.num_experts
        assert torch.equal(ctx.cnt_all[0, :E_].long(), torch.bincount(idx[idx >= 0], minlength=E_))
        check(SimpleNamespace(ctx=ctx, layer=layer, oracle=oracle, logits=logits, bias0=bias0, idx=idx,
                              w=layer.ws.w[:B * cfg.k].view(B, cfg.k), ridx=ridx, rw=rw, same=same))
        errs = dict(y=rel(y, yr, *precision), dlogits=rel(lg.grad, lr_.grad, *precision))
        if dx:
            errs["dx"] = rel(xf.grad, xr.grad, *precision)
        assert errs["y"] < 2e-2 and errs["dlogits"] < 5e-2 and errs.get("dx", 0.0) < 3e-2, errs
    finally:
        ctx.close()
