"""SwiGLU experts with their forward GEMMs on block-scaled FP8 tensor cores: DMoEConfig(expert="swiglu",
expert_dtype="fp8").

CPU: the configuration matrix, the CPU trainer (the fp32 oracle) learning and resuming, checkpoints across bf16 and fp8,
and the host checks of the two new C entry points (lah_rms_norm_fwd_q, lah_swiglu_fwd_q), which refuse before any launch.

GPU: the two MXFP8 emitters element by element against float64 oracles.  A scale byte must equal ``fp8.quantize_ref``'s
exponent of the float64 value, except in a block whose amax / 448 lies within 2^-20 relative of a power of two (the fp32
value the kernel sees may fall on either side); a payload byte must equal the round-to-nearest-even E4M3 of the float64
value times 2^-e, except for a value within 2^-18 relative of a rounding midpoint.  Such exceptions are counted and
recorded.  Then the layer's forward against a float64 oracle on the kernels' own quantised operands (the bound of the FP8
GEMM, test_fused_adam_fp8_kernels.py), its backward and optimizer step against an oracle on the bf16 activations the FP8
forward saved, the layer against fp32 GatedFeedforwardBlock modules (the loosened bounds tools/gpu_layer_check.py uses
for the FFN in fp8), the trainer under its CUDA graph, and serving (NativeGatedFFNLayer, ExpertBackend).
"""
import ctypes
import os
import subprocess
import sys

import pytest
import torch

import lah_b200  # noqa: F401
import lib
from lah_b200.models.layers import GATED_LAYOUT, GatedFeedforwardBlock, gated_inner_dim
from lah_b200.ops import fp8, kernels as K
from lah_b200.parallel import engine as E
from lah_b200.parallel.trainer import DMoETrainer

from test_expert_kernels import BF16, SENTINEL, _lib, gemm_epilogue64, report_worst_ratios, within  # noqa: F401
from test_fused_adam_fp8_kernels import FP8_MMA_BITS, dequant64, e4m3_bytes, sf_index

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SCALE_TIE = 2.0 ** -20     # a block's amax / 448 this close (relative) to a power of two may take either scale
MIDPOINT = 2.0 ** -18      # a value this close (relative) to an E4M3 rounding midpoint may round either way


# ================================================================================================================= CPU
@pytest.mark.parametrize("hidden,inner", [(1024, 0), (512, 1024), (2048, 5632), (256, 0)])
def test_config_accepts_widths_that_are_multiples_of_256(hidden, inner):
    cfg = E.DMoEConfig(hidden=hidden, inner_dim=inner, expert="swiglu", expert_dtype="fp8")
    assert cfg.inner % 256 == 0 and cfg.hidden % 256 == 0
    assert cfg.resolved_path() == "big"
    assert E.DMoEConfig(hidden=hidden, inner_dim=inner, expert="swiglu", expert_dtype="fp8", tokens_per_rank=16,
                        grid_size=(64,)).resolved_path() == "big"   # "auto" sends fp8 to big at any batch
    assert E.DMoEConfig(hidden=hidden, inner_dim=inner, expert="swiglu", expert_dtype="fp8",
                        expert_path="small").resolved_path() == "small"


@pytest.mark.parametrize("hidden,inner", [(512, 0), (640, 0), (640, 1024), (640, 1280), (1024, 1408), (2048, 0)])
def test_config_refuses_other_widths(hidden, inner):
    """512 and 2048 default to 1408 and 5504 (gated_inner_dim), which are odd multiples of 128"""
    with pytest.raises(ValueError, match=f"hidden={hidden}, inner={inner or gated_inner_dim(hidden)}"):
        E.DMoEConfig(hidden=hidden, inner_dim=inner, expert="swiglu", expert_dtype="fp8")
    E.DMoEConfig(hidden=hidden, inner_dim=inner, expert="swiglu")   # the same widths in bf16 are fine


def test_ffn_fp8_config_is_unchanged():
    cfg = E.DMoEConfig(hidden=512, expert_dtype="fp8")
    assert cfg.expert == "ffn" and cfg.resolved_path() == "big"
    assert E.DMoEConfig(hidden=640, expert_dtype="fp8").inner == 2560   # the FFN has no 256 condition in the config
    with pytest.raises(ValueError):
        E.DMoEConfig(hidden=512, expert_dtype="fp8", inner_dim=1024)


def _cpu_cfg(dtype, **kw):
    base = dict(hidden=256, grid_size=(2, 2), k=2, num_layers=2, in_features=12, tokens_per_rank=32, lr=3e-3,
                expert="swiglu", inner_dim=256, expert_dtype=dtype)
    base.update(kw)
    return E.DMoEConfig(**base)


def test_cpu_trainer_runs_the_fp32_oracle_learns_and_resumes():
    """the CPU path is the fp32 oracle whatever the dtype: fp8 and bf16 trainers give the same losses"""
    x, y = torch.randn(32, 12, generator=torch.Generator().manual_seed(0)), torch.randint(0, 10, (32,))
    losses = {}
    for dtype in ("bf16", "fp8"):
        torch.manual_seed(0)
        trainer = DMoETrainer(_cpu_cfg(dtype))
        losses[dtype] = [trainer.train_step(x, y) for _ in range(20)]
    assert losses["fp8"] == losses["bf16"]
    assert losses["fp8"][-1] < 0.5 * losses["fp8"][0]
    clone = DMoETrainer(_cpu_cfg("fp8"))
    clone.load_state_dict(trainer.state_dict())
    for _ in range(3):
        assert abs(trainer.train_step(x, y) - clone.train_step(x, y)) < 1e-5
    for b1, b2 in zip(trainer.model.blocks, clone.model.blocks):
        torch.testing.assert_close(b1.shard.p, b2.shard.p, atol=1e-6, rtol=0)


@pytest.mark.parametrize("src,dst", [("bf16", "fp8"), ("fp8", "bf16")])
def test_checkpoint_round_trips_between_bf16_and_fp8(src, dst):
    x, y = torch.randn(32, 12, generator=torch.Generator().manual_seed(1)), torch.randint(0, 10, (32,))
    torch.manual_seed(1)
    a = DMoETrainer(_cpu_cfg(src))
    for _ in range(3):
        a.train_step(x, y)
    state = a.state_dict()
    b = DMoETrainer(_cpu_cfg(dst))
    b.load_state_dict(state)
    back = DMoETrainer(_cpu_cfg(src))
    back.load_state_dict(b.state_dict())
    for b1, b2 in zip(a.model.blocks, back.model.blocks):
        assert torch.equal(b1.shard.p, b2.shard.p) and torch.equal(b1.shard.step, b2.shard.step)
    assert abs(a.train_step(x, y) - b.train_step(x, y)) < 1e-5


def test_c_entry_points_refuse_bad_widths_and_misaligned_operands():
    """rows = 0 passes every host check and launches nothing: the controls return 0 on any machine"""
    lib_ = _lib()
    K._lib()
    v = ctypes.c_void_p

    def rms(C=1024, x=0x200000, n=0x300000, nq=0x400000, sf=0x500000, eps=1e-6, tg=0, tile_rows=128):
        return lib_.lah_rms_norm_fwd_q(v(x), v(n), v(0x600000), v(0x700000), 0, C, eps, v(tg), tile_rows, v(nq), v(sf),
                                       v(0))
    assert rms() == 0 and rms(n=0) == 0 and rms(tg=0x800000) == 0 and rms(C=256) == 0 and rms(C=4096) == 0
    for kw in (dict(C=128), dict(C=384), dict(C=1408), dict(C=4352), dict(C=0),   # not a multiple of 256 in [256, 4096]
               dict(x=0x200008), dict(n=0x300008), dict(nq=0x400004),          # x, n off 16 bytes; nq off 8
               dict(nq=0), dict(sf=0), dict(eps=0.0), dict(tg=0x800000, tile_rows=100)):
        assert rms(**kw) == -2, kw

    def sw(inner=2816, h=0x200000, a=0x300000, aq=0x400000, sf=0x500000, rows=0):
        return lib_.lah_swiglu_fwd_q(v(h), v(a), v(aq), v(sf), rows, inner, v(0), v(0), v(0))
    assert sw() == 0 and sw(a=0) == 0 and sw(inner=128) == 0 and sw(inner=11008) == 0
    for kw in (dict(inner=64), dict(inner=200), dict(inner=0), dict(rows=-1),   # inner not a multiple of 128
               dict(h=0x200008), dict(a=0x300008), dict(aq=0x400004), dict(aq=0), dict(sf=0)):
        assert sw(**kw) == -2, kw


# ================================================================================================================= GPU
def _e4m3_rne64(v):
    """round-to-nearest-even E4M3 bytes of float64 values (saturating, as the kernels' SATFINITE conversion)"""
    return e4m3_bytes(v.clamp(-448.0, 448.0).to(torch.float8_e4m3fn).view(torch.uint8))


def check_mxfp8_operand(t: fp8.MXFP8Tensor, val64, live, record_property, what):
    """the payload and scale bytes of t against the float64 values val64 [rows, K] for the rows in ``live``; every byte
    of the other rows (and of tile padding) must still hold SENTINEL.  Returns (scale exceptions, payload exceptions)"""
    rows, K_ = val64.shape
    got_q, got_e = t.q[:rows], fp8.unpack_sf(t)[:rows]
    v = val64[live]
    _, e_ref = fp8.quantize_ref(v)
    e_got = got_e[live]
    blocks = v.view(-1, K_ // 32, 32)
    amax = blocks.abs().amax(-1)
    r = amax / 448.0
    near_pow2 = (r > 0) & ((r / torch.exp2(torch.round(torch.log2(r.clamp_min(1e-300))))) - 1).abs().le(SCALE_TIE)
    bad_e = e_got != e_ref
    assert bool((~bad_e | near_pow2).all()), f"{what}: {int((bad_e & ~near_pow2).sum())} scale bytes differ"
    scaled = blocks * torch.exp2(127.0 - e_got.double())[..., None]
    want = _e4m3_rne64(scaled)
    tie = (_e4m3_rne64(scaled * (1 + MIDPOINT)) != want) | (_e4m3_rne64(scaled * (1 - MIDPOINT)) != want)
    got = e4m3_bytes(got_q[live]).view(-1, K_ // 32, 32)
    bad_q = got != want
    assert bool((~bad_q | tie).all()), f"{what}: {int((bad_q & ~tie).sum())} payload bytes differ"
    assert bool((got_q[~live] == SENTINEL).all()), f"{what}: payload rows the kernel must skip were written"
    written = torch.zeros(t.sf.numel(), dtype=torch.bool, device=t.sf.device)
    written[sf_index(t)[:rows][live].reshape(-1)] = True
    assert bool((t.sf[~written] == SENTINEL).all()), f"{what}: scale bytes of skipped rows or tile padding were written"
    record_property(f"{what}_scale_exceptions", int(bad_e.sum()))
    record_property(f"{what}_payload_exceptions", int(bad_q.sum()))
    return int(bad_e.sum()), int(bad_q.sum())


def _operand(rows, K_):
    t = fp8.MXFP8Tensor(rows, 1, K_, fp8.ACT_TILE, "cuda")
    t.q.fill_(SENTINEL)
    t.sf.fill_(SENTINEL)
    return t


RMS_WIDTHS = list(range(256, 4097, 256))


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["grouped", "grouped_no_bf16", "one_gamma"])
@pytest.mark.parametrize("C", RMS_WIDTHS)
def test_rms_norm_emitter_elementwise(C, mode, record_property):
    gen = torch.Generator().manual_seed(C)
    tiles = [0, -1, 2, 2, -1, 1] if mode != "one_gamma" else [0] * 3
    rows, G = 128 * len(tiles), 3
    # rows of very different magnitude, so neighbouring rows get different scales
    x = (torch.randn(rows, C, generator=gen) * 2.0 ** torch.randint(-8, 9, (rows, 1), generator=gen)).to(BF16).cuda()
    gamma = (1 + 0.5 * torch.randn(G if mode != "one_gamma" else 1, C, generator=gen)).cuda()
    grouped = mode != "one_gamma"
    tg = torch.tensor(tiles, dtype=torch.int32, device="cuda") if grouped else None
    gam = gamma if grouped else gamma[0]
    n_plain, rstd_plain = torch.full((rows, C), 7.0, dtype=BF16, device="cuda"), torch.zeros(rows, device="cuda")
    K.rms_norm_fwd(x, gam, 1e-6, out=n_plain, rstd=rstd_plain, tile_group=tg, tile_rows=128)
    q = _operand(rows, C)
    n = None if mode == "grouped_no_bf16" else torch.full((rows, C), 7.0, dtype=BF16, device="cuda")
    rstd = torch.zeros(rows, device="cuda")
    K.rms_norm_fwd(x, gam, 1e-6, out=n, rstd=rstd, tile_group=tg, tile_rows=128, quant=q)
    torch.cuda.synchronize()
    if n is not None:
        assert torch.equal(n.view(torch.int16), n_plain.view(torch.int16)), "the bf16 n differs from rms_norm_fwd's"
    assert torch.equal(rstd, rstd_plain)
    if grouped:
        ref, _ = K.rms_norm_grouped_fwd_ref(x.double(), gamma.double(), 1e-6, tg.cpu(), 128)
    else:
        ref, _ = K.rms_norm_fwd_ref(x.double(), gamma[0].double(), 1e-6)
    live = (torch.tensor(tiles).repeat_interleave(128) >= 0).cuda()
    check_mxfp8_operand(q, ref, live, record_property, "rms_norm")


@pytest.mark.gpu
@pytest.mark.parametrize("with_bf16", [True, False], ids=["bf16_a", "no_bf16_a"])
@pytest.mark.parametrize("inner", [256, 2816, 5632, 11008])
def test_swiglu_emitter_elementwise(inner, with_bf16, record_property):
    gen = torch.Generator().manual_seed(inner + with_bf16)
    tiles = [0, -1, 1, 3, -1]
    total = 128 * 3 + 77          # read on the device: rows from here on are skipped, inside a live tile
    rows = 128 * len(tiles)
    h = (torch.randn(rows, 2 * inner, generator=gen) * 2.0 ** torch.randint(-4, 5, (rows, 1), generator=gen)) \
        .to(BF16).cuda()
    plain = K.swiglu_fwd(h)
    q = _operand(rows, inner)
    a = torch.full((rows, inner), 7.0, dtype=BF16, device="cuda") if with_bf16 else None
    tg = torch.tensor(tiles, dtype=torch.int32, device="cuda")
    total_dev = torch.tensor([total], dtype=torch.int32, device="cuda")
    K.swiglu_fwd(h, out=a, quant=q, tile_group=tg, total_rows=total_dev)
    torch.cuda.synchronize()
    r = torch.arange(rows, device="cuda")
    live = (tg.long()[r // 128] >= 0) & (r < total)
    if a is not None:
        assert torch.equal(a[live].view(torch.int16), plain[live].view(torch.int16)), "bf16 a differs from swiglu_fwd's"
        assert bool((a[~live] == 7.0).all()), "bf16 rows the kernel must skip were written"
    check_mxfp8_operand(q, K.swiglu_ref(h.double()), live, record_property, "swiglu")


@pytest.mark.gpu
def test_swiglu_fwd_without_quant_refuses_row_limits():
    h = torch.zeros(128, 512, dtype=BF16, device="cuda")
    with pytest.raises(ValueError):
        K.swiglu_fwd(h, tile_group=torch.zeros(1, dtype=torch.int32, device="cuda"))
    with pytest.raises(ValueError):
        K.rms_norm_fwd(torch.zeros(128, 384, dtype=BF16, device="cuda"), torch.ones(384, device="cuda"), 1e-6, out=None,
                       rstd=torch.zeros(128, device="cuda"), quant=_operand(128, 384))


# ------------------------------------------------------------------------------------------------ the layer
def _layer_cfg(**kw):
    base = dict(hidden=512, inner_dim=1024, grid_size=(4, 4), k=4, num_layers=1, tokens_per_rank=512, lr=1e-3,
                expert="swiglu", expert_dtype="fp8")
    base.update(kw)
    return E.DMoEConfig(**base)


def _rel(a, b):
    a, b = a.detach().double(), b.detach().double()
    return float((a - b).norm() / b.norm().clamp_min(1e-300))


def _fp8_gemm64(a: fp8.MXFP8Tensor, w: fp8.MXFP8Tensor, tiles, N, residual=None):
    """float64 reference and element bound of grouped_linear_fp8 (bf16 out) on its own quantised operands"""
    rows, K_ = 128 * len(tiles), a.K
    grow = torch.tensor(tiles, device="cuda").long().repeat_interleave(128)
    mask = torch.zeros(a.q.shape[0], dtype=torch.bool, device="cuda")
    mask[:rows] = grow >= 0
    A = dequant64(a, mask)[:rows]
    W = dequant64(w, torch.ones(w.q.shape[0], dtype=torch.bool, device="cuda")).view(w.groups, N, K_)
    nb = K_ // 32
    pre = torch.zeros(rows, N, dtype=torch.float64, device="cuda")
    blocks, mag = torch.zeros_like(pre), torch.zeros_like(pre)
    for t, g in enumerate(tiles):
        if g < 0:
            continue
        sl = slice(t * 128, (t + 1) * 128)
        parts = torch.einsum("rbk,nbk->rbn", A[sl].view(128, nb, 32), W[g].view(N, nb, 32))
        pre[sl], blocks[sl] = parts.sum(1), parts.abs().sum(1)
        mag[sl] = A[sl].abs() @ W[g].abs().t()
    return gemm_epilogue64(pre, blocks, nb + 2, residual=residual, extra=2.0 ** -FP8_MMA_BITS * mag), grow >= 0


@pytest.mark.gpu
def test_layer_forward_against_float64_on_the_quantised_operands(record_property):
    torch.manual_seed(3)
    cfg = _layer_cfg()
    ctx = E.EngineContext(cfg)
    try:
        layer = E.FusedDMoE(cfg, ctx).cuda()
        with torch.no_grad():   # distinct norm weights per expert, so the grouped gamma is exercised
            layer.shard.raw_views["g"].copy_(1 + 0.3 * torch.randn_like(layer.shard.raw_views["g"]))
            layer.shard.sync_bf16()
        x = torch.randn(512, 512, device="cuda").to(BF16)
        ws, sh = layer.ws, layer.shard
        ws.xq.q.fill_(SENTINEL), ws.xq.sf.fill_(SENTINEL), ws.aq.q.fill_(SENTINEL), ws.aq.sf.fill_(SENTINEL)
        layer.eval()
        with torch.no_grad():
            layer(x)
        torch.cuda.synchronize()
        ctx.check_status()
        tiles = ws.tile_group.tolist()
        rows = 128 * (max(t for t, g in enumerate(tiles) if g >= 0) + 1)
        tiles = tiles[:rows // 128]
        live = torch.tensor(tiles, device="cuda").repeat_interleave(128) >= 0
        H, I = cfg.hidden, cfg.inner
        # the emitters: n from the dispatched rows, a from the bf16 h the first GEMM wrote
        n_ref, _ = K.rms_norm_grouped_fwd_ref(ws.xd[:rows].double(), sh.raw_views["g"].double(), E.GATED_EPS,
                                             ws.tile_group[:rows // 128].cpu(), 128)
        check_mxfp8_operand(ws.xq, n_ref, live, record_property, "layer_n")
        check_mxfp8_operand(ws.aq, K.swiglu_ref(ws.h[:rows].double()), live, record_property, "layer_a")
        w8 = sh.w8
        for name in ("w13", "w2"):   # the weight copies are the quantiser's output of the bf16 mirror
            want = fp8.quantize(sh.bf16[name].view(-1, w8[name].K), tile_rows=fp8.WEIGHT_TILE, groups=sh.slots)
            assert torch.equal(want.q, w8[name].q) and torch.equal(want.sf, w8[name].sf), name
        (h_ref, h_bound), _ = _fp8_gemm64(ws.xq, w8["w13"], tiles, 2 * I)
        r1 = within(ws.h[:rows][live], h_ref[live], h_bound[live], "h = n [W1; W3]^T", "layer_fp8_h")
        (y_ref, y_bound), _ = _fp8_gemm64(ws.aq, w8["w2"], tiles, H, residual=ws.xd[:rows])
        r2 = within(ws.yo[:rows][live], y_ref[live], y_bound[live], "y = a W2^T + x", "layer_fp8_y")
        record_property("max_err_over_bound", dict(h=r1, y=r2))
    finally:
        ctx.close()


def _gated_bwd_oracle(ws, tiles, rows, w13, w2, g, eps):
    """float64 backward of the experts on the bf16 activations the forward saved: (dx rows, dW13, dW2, dg) per group"""
    G = w13.shape[0]
    xd, n, h, a, gy = (t[:rows].double() for t in (ws.xd, ws.n, ws.h, ws.a, ws.gyd))
    grow = torch.tensor(tiles, device="cuda").long().repeat_interleave(128)
    dx = torch.zeros_like(xd)
    dw13, dw2, dg = torch.zeros_like(w13, dtype=torch.float64), torch.zeros_like(w2, dtype=torch.float64), \
        torch.zeros(G, xd.shape[1], dtype=torch.float64, device="cuda")
    for e in range(G):
        m = grow == e
        if not bool(m.any()):
            continue
        da = gy[m] @ w2[e].double()
        dw2[e] = gy[m].t() @ a[m]
        dh = K.swiglu_bwd_ref(da, h[m])
        dw13[e] = dh.t() @ n[m]
        dn = dh @ w13[e].double()
        d, gg = K.rms_norm_bwd_ref(dn, xd[m], g[e].double(), eps, dres=gy[m])
        dx[m], dg[e] = d, gg
    return dx, dw13, dw2, dg


@pytest.mark.gpu
def test_layer_backward_and_step_against_the_saved_activations(record_property):
    """the backward reads the bf16 n, h and a that the fp8 forward wrote: an oracle on them gives dx and the weight
    gradients with the tolerances of the big-path layer test in test_dmoe_swiglu.py"""
    torch.manual_seed(4)
    cfg = _layer_cfg()
    ctx = E.EngineContext(cfg)
    try:
        layer = E.FusedDMoE(cfg, ctx).cuda()
        sh, ws = layer.shard, layer.ws
        before = {n: sh.views[n][:16].detach().clone() for n in GATED_LAYOUT.names}
        wb = {n: sh.bf16[n][:16].clone() for n in ("w13", "w2")}
        x = torch.randn(512, 512, device="cuda").to(BF16).requires_grad_(True)
        gy = torch.randn(512, 512, device="cuda").to(BF16)
        layer(x).backward(gy)
        torch.cuda.synchronize()
        ctx.check_status()
        tiles = ws.tile_group.tolist()
        rows = 128 * (max(t for t, g in enumerate(tiles) if g >= 0) + 1)
        tiles = tiles[:rows // 128]
        dx, dw13, dw2, dg = _gated_bwd_oracle(ws, tiles, rows, wb["w13"], wb["w2"], before["g"], E.GATED_EPS)
        live = torch.tensor(tiles, device="cuda").repeat_interleave(128) >= 0
        errs = dict(dx_rows=_rel(ctx.dxd[:rows][live], dx[live]))
        grads = dict(w13=dw13, w2=dw2, g=dg)
        werr = {n: _rel(sh.m_views[n][:16] / (1 - cfg.betas[0]), grads[n]) for n in grads}
        stepped = sh.step > 0
        # the first AMSGrad step moves every parameter by ~lr sign(grad)
        perr = {n: float((sh.views[n][:16][stepped] - (before[n] - cfg.lr * grads[n].sign())[stepped]).abs().mean())
                for n in grads}
        record_property("errors", dict(errs, wgrad=werr, param=perr))
        assert errs["dx_rows"] < 3e-2, errs
        assert max(werr.values()) < 8e-2, werr
        assert max(perr.values()) < 1e-4, perr
        assert int(stepped.sum()) == sum(1 for e in range(16) if e in tiles)
        # the MXFP8 weights follow the step: the next forward re-quantises the new mirror
        assert sh.w8_dirty
    finally:
        ctx.close()


@pytest.mark.gpu
def test_layer_against_fp32_gated_modules(record_property):
    """forward, backward and one AMSGrad step against 16 fp32 GatedFeedforwardBlock modules with torch Adam, within the
    fp8 bounds of tools/gpu_layer_check.py (3x the bf16 ones, 4x for the weight gradients)"""
    torch.manual_seed(3)
    cfg = _layer_cfg()
    ctx = E.EngineContext(cfg)
    try:
        layer = E.FusedDMoE(cfg, ctx).cuda()
        oracle = E.FusedDMoE(cfg, device=torch.device("cuda")).cuda().train()   # the fp32 CPU-path layer on the GPU
        oracle.proj.load_state_dict(layer.proj.state_dict())
        with torch.no_grad():
            oracle.shard.p.copy_(layer.shard.p[:oracle.shard.p.numel()])
        experts = []
        for le in range(16):
            blk = GatedFeedforwardBlock(cfg.hidden, cfg.inner).cuda()
            blk.load_state_dict({k[len("expert."):]: v for k, v in layer.shard.expert_state_dict(le).items()})
            experts.append(blk)
        x = torch.randn(512, 512, device="cuda").to(BF16).requires_grad_(True)
        gy = torch.randn(512, 512, device="cuda").to(BF16)
        y = layer(x)
        y.backward(gy)
        torch.cuda.synchronize()
        ctx.check_status()
        xr = x.detach().float().requires_grad_(True)
        yr = oracle(xr)
        yr.backward(gy.float())
        grads = {n: torch.stack([oracle._ref_leaves[e][n].grad if e in oracle._ref_leaves and
                                 oracle._ref_leaves[e][n].grad is not None else torch.zeros_like(layer.shard.views[n][e])
                                 for e in range(16)]) for n in GATED_LAYOUT.names}
        oracle.apply_expert_gradients_ref()
        # the oracle's experts are the modules: same forward as GatedFeedforwardBlock on the same weights
        e0 = int(layer.shard.step.argmax())
        xe = torch.randn(8, 512, device="cuda")
        p0 = {n: v[e0] for n, v in oracle.shard.views.items()}
        with torch.no_grad():
            blk = GatedFeedforwardBlock(cfg.hidden, cfg.inner).cuda()
            blk.load_state_dict({k[len("expert."):]: v for k, v in oracle.shard.expert_state_dict(e0).items()})
            torch.testing.assert_close(oracle._expert_ref(p0, xe, lambda v: v), blk(xe), rtol=1e-5, atol=1e-5)
        errs = dict(y=_rel(y, yr), dx=_rel(x.grad, xr.grad), dproj=_rel(layer.proj.weight.grad, oracle.proj.weight.grad))
        perr = {n: float((layer.shard.views[n][:16] - oracle.shard.views[n][:16]).abs().mean()) for n in grads}
        werr = {n: _rel(layer.shard.m_views[n][:16] / (1 - cfg.betas[0]), grads[n]) for n in grads}
        record_property("errors", dict(errs, param_mean_abs_diff=perr, wgrad=werr))
        assert errs["y"] < 6e-2 and errs["dx"] < 9e-2 and errs["dproj"] < 1.5e-1, errs
        assert max(perr.values()) < 3e-4, perr
        assert max(werr.values()) < 8e-2 * 4, werr
    finally:
        ctx.close()


# ------------------------------------------------------------------------------------------------ the trainer
def _trainer_cfg(**kw):
    base = dict(hidden=512, inner_dim=1024, grid_size=(16,), k=4, num_layers=2, tokens_per_rank=256,
                gate_mode="emulator", lr=1e-4, expert="swiglu", expert_dtype="fp8")
    base.update(kw)
    return E.DMoEConfig(**base)


def _snapshot(t):
    return torch.cat([b.shard.p for b in t.model.blocks] + [t.flat_p]).cpu()


@pytest.mark.gpu
@pytest.mark.parametrize("kw", [dict(), dict(failure_rate=0.1), dict(update_every_steps=2),
                                dict(shared_inner_dim=512, failure_rate=0.1)],
                         ids=["plain", "failures", "update_every_2", "shared_expert"])
def test_trainer_graph_equals_eager_and_runs_are_reproducible(kw):
    """the MXFP8 weights are refreshed from host state (w8_dirty): a graph that kept stale ones would differ from eager
    steps after the first optimizer step"""
    cfg = _trainer_cfg(**kw)
    torch.manual_seed(0)
    xs = [torch.randn(256, cfg.in_features, device="cuda") for _ in range(6)]
    ys = [torch.randint(0, 10, (256,), device="cuda") for _ in range(6)]
    runs = {}
    for run, graph in (("eager", False), ("graph", True), ("graph2", True)):
        t = DMoETrainer(cfg, use_graph=graph)
        assert not t.ctx.small and t.model.blocks[0].shard.w8 is not None
        losses = torch.stack([t.train_step_device(x, y).clone() for x, y in zip(xs, ys)]).cpu()
        assert (t._graph is not None) == graph
        t.ctx.check_status()
        runs[run] = (losses, _snapshot(t))
        assert int(t.model.blocks[0].shard.step.max()) == (3 if kw.get("update_every_steps") else 6)
        t.close()
    for a, b in zip(runs["eager"], runs["graph"]):
        assert torch.equal(a, b)
    for a, b in zip(runs["graph"], runs["graph2"]):
        assert torch.equal(a, b)


@pytest.mark.gpu
def test_trainer_learns_synthetic_data_like_bf16(record_property):
    """200 steps on a learnable task (labels of a fixed random linear teacher): the fp8 loss falls as the bf16 one does"""
    gen = torch.Generator().manual_seed(5)
    teacher = torch.randn(64, 10, generator=gen)
    xs = torch.randn(8, 256, 64, generator=gen)
    ys = (xs @ teacher).argmax(-1)
    out = {}
    for dtype in ("bf16", "fp8"):
        torch.manual_seed(0)
        t = DMoETrainer(_trainer_cfg(expert_dtype=dtype, expert_path="big", in_features=64, lr=1e-3))
        losses = [float(t.train_step_device(xs[i % 8].cuda(), ys[i % 8].cuda())) for i in range(200)]
        t.ctx.check_status()
        t.close()
        out[dtype] = (sum(losses[:10]) / 10, sum(losses[-10:]) / 10)
    record_property("loss_first10_last10", out)
    assert out["fp8"][1] < 0.5 * out["fp8"][0], out
    assert out["fp8"][1] < out["bf16"][1] + 0.1, out


# ------------------------------------------------------------------------------------------------ serving
@pytest.mark.gpu
@pytest.mark.parametrize("dtype", ["bf16", "fp8"])
def test_native_gated_ffn_layer(dtype, record_property):
    from lah_b200.models.ffn_native import NativeGatedFFNLayer
    torch.manual_seed(6)
    H, I, rows = 1024, 2816, 512
    block = GatedFeedforwardBlock(H).cuda()
    with torch.no_grad():
        block.norm.weight.copy_(1 + 0.3 * torch.randn(H))
    layer = NativeGatedFFNLayer(block, dtype=dtype)
    x = torch.randn(rows, H, device="cuda").to(BF16)
    y = layer(x)
    torch.cuda.synchronize()
    with torch.no_grad():
        ref = block(x.float())
    rel = _rel(y, ref)
    record_property("rel_err_vs_fp32_module", rel)
    ws = layer._ws[rows]
    if dtype == "bf16":
        assert rel < 2e-2
        assert set(ws) == {"h", "rstd", "n", "a"}
        return
    assert rel < 6e-2
    assert set(ws) == {"h", "rstd", "nq", "aq"}   # no bf16 n or a
    live = torch.ones(rows, dtype=torch.bool, device="cuda")
    n_ref, _ = K.rms_norm_fwd_ref(x.double(), block.norm.weight.detach().double(), block.norm.eps)
    check_mxfp8_operand(ws["nq"], n_ref, live, record_property, "serve_n")
    check_mxfp8_operand(ws["aq"], K.swiglu_ref(ws["h"].double()), live, record_property, "serve_a")
    tiles = [0] * (rows // 128)
    (h_ref, h_bound), _ = _fp8_gemm64(ws["nq"], layer.w13, tiles, 2 * I)
    within(ws["h"][live], h_ref[live], h_bound[live], "serve h", "serve_fp8_h")
    (y_ref, y_bound), _ = _fp8_gemm64(ws["aq"], layer.w2, tiles, H, residual=x)
    within(y, y_ref, y_bound, "serve y", "serve_fp8_y")
    w13 = torch.cat([block.w1.weight, block.w3.weight]).detach().float().contiguous()
    want = fp8.quantize(w13, tile_rows=fp8.WEIGHT_TILE)
    assert torch.equal(want.q, layer.w13.q) and torch.equal(want.sf, layer.w13.sf)


@pytest.mark.gpu
def test_trained_fp8_expert_served_by_expert_backend():
    """a checkpoint of an fp8-trained expert in ExpertBackend(GatedFeedforwardBlock) (NativeGatedFFNExecutor, bf16)
    returns what the engine's expert oracle returns on the same rows"""
    from lah_b200.runtime.native_executor import NativeGatedFFNExecutor
    cfg = _trainer_cfg(hidden=1024, inner_dim=0, num_layers=1, lr=1e-3)
    t = DMoETrainer(cfg)
    torch.manual_seed(2)
    for _ in range(3):
        t.train_step_device(torch.randn(256, cfg.in_features, device="cuda"), torch.randint(0, 10, (256,), device="cuda"))
    state = t.state_dict()
    layer = t.model.blocks[0]
    e = int(layer.shard.step.argmax())
    assert int(layer.shard.step[e]) > 0
    entry = state["experts"]["layer0." + E.expert_uid(cfg, e)]
    block = GatedFeedforwardBlock(cfg.hidden, cfg.inner).cuda()
    opt = torch.optim.Adam(block.parameters(), lr=cfg.lr, amsgrad=True)
    backend = lib.ExpertBackend(name="e", expert=block, opt=opt, args_schema=(lib.BatchTensorProto(cfg.hidden),),
                                outputs_schema=lib.BatchTensorProto(cfg.hidden), max_batch_size=64)
    backend.load_state_dict(entry["model"])
    opt.load_state_dict(entry["optimizer"])
    assert NativeGatedFFNExecutor.supports(block, opt)
    rows = torch.randn(40, cfg.hidden, device="cuda").to(BF16).float()
    served = backend.forward(rows)[0]
    p = {n: v.cuda() for n, v in GATED_LAYOUT.segment_state(entry["model"], prefix="expert.").items()}
    ref = layer._expert_ref(p, rows, lambda v: v.to(BF16).float())
    assert _rel(served, ref) < 2e-2
    t.close()


@pytest.mark.gpu
@pytest.mark.parametrize("shadow", [False, True], ids=["static", "force_shadow"])
def test_two_gpus_fp8_matches_the_whole_batch_oracle(shadow):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    args = ["--swiglu", "--fp8"] + (["--force-shadow"] if shadow else [])
    out = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2",
                          "--master-addr", "127.0.0.1", "--master-port", str(29561 + shadow),
                          os.path.join(ROOT, "tools", "multi_gpu_check.py"), *args],
                         capture_output=True, text=True, timeout=600)
    assert out.returncode == 0 and "MULTI_GPU_OK" in out.stdout, out.stdout[-3000:] + out.stderr[-3000:]
