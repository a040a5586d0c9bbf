"""
Split master weights: an fp32 weight kept as its bf16 GEMM operand (hi, round to nearest even) plus its low 16 bits (lo),
with the one bit 32 bits cannot spare, whether a tie (lo == 0x8000) was rounded up, in the sign of the weight's
exp_avg_sq.  The small expert path keeps its weight matrices this way, so the fused wgrad + AMSGrad kernel streams 32 B per
parameter instead of 34.  Checked here: the encoding over every fp32 bit pattern, the encode / decode kernels, the SPLIT
instantiation of the fused kernel against the fp32 one (same bits of p, m, v, vmax and the mirror, ties forced), and a
small-path layer whose shard.p / views / v match those of an fp32 shard bit for bit.
"""
import numpy as np
import pytest
import torch

from test_fused_adam_fp8_kernels import wa_inputs

import lah_b200.parallel.engine as E
from lah_b200.ops import kernels as K

TIE = 0x8000


def encode_ref(b):
    """(hi, lo, tie_up) of fp32 bit patterns b (uint32)"""
    t, lo = b >> 16, b & 0xFFFF
    tie = (lo == TIE) & ((t & 1) == 1)
    hi = (t + ((lo > TIE) | tie)) & 0xFFFF
    return hi, lo, tie


def decode_ref(hi, lo, tie):
    up = ((lo > TIE) | ((lo == TIE) & tie)).astype(np.uint32)
    return (((hi - up) & 0xFFFF) << 16) | lo


def test_encoding_is_exact_for_every_finite_fp32():
    chunk = 1 << 24
    offsets = np.arange(chunk, dtype=np.uint32)
    for start in range(0, 1 << 32, chunk):
        b = offsets + np.uint32(start)
        hi, lo, tie = encode_ref(b)
        assert np.array_equal(decode_ref(hi, lo, tie), b), hex(start)
        # hi is torch's bf16 cast (round to nearest even), the mirror the GEMMs read, for every finite pattern: the chunk's
        # second half is inf and NaN when its top byte is 0x7f or 0xff
        n = chunk // 2 if (start >> 24) & 0x7F == 0x7F else chunk
        rne = torch.from_numpy(b[:n].view(np.float32)).to(torch.bfloat16).view(torch.int16).numpy().view(np.uint16)
        assert np.array_equal(hi[:n].astype(np.uint16), rne), hex(start)


def random_bits_with_ties(gen, n):
    """finite fp32 bit patterns, a quarter of them ties (low half 0x8000) with odd and even upper halves"""
    b = np.random.default_rng(gen).integers(0, 1 << 32, n, dtype=np.uint64).astype(np.uint32)
    b &= ~np.uint32(0x40000000)   # exponent below 0x80: finite, |p| < 2
    tie = np.random.default_rng(gen + 1).random(n) < 0.25
    b[tie] = (b[tie] & np.uint32(0xFFFF0000)) | TIE
    return b


def as_f32(b):
    return torch.from_numpy(b.view(np.float32).copy()).cuda()


def bits(t):
    return t.contiguous().view(torch.int32)


@pytest.mark.gpu
def test_encode_and_decode_kernels():
    n = 1 << 20
    b = random_bits_with_ties(7, n)
    hi_r, lo_r, tie_r = encode_ref(b)
    p = as_f32(b)
    v0 = torch.rand(n, device="cuda")
    v0[:1000] = 0.0
    v = v0.clone()
    hi = torch.empty(n, dtype=torch.bfloat16, device="cuda")
    lo = torch.empty(n, dtype=torch.int16, device="cuda")
    K.split_encode(p, hi, lo, v)
    assert np.array_equal(hi.view(torch.int16).cpu().numpy().view(np.uint16), hi_r.astype(np.uint16))
    assert np.array_equal(lo.cpu().numpy().view(np.uint16), lo_r.astype(np.uint16))
    assert np.array_equal(torch.signbit(v).cpu().numpy(), tie_r) and tie_r.any() and not tie_r.all()
    assert torch.equal(v.abs(), v0)
    out = torch.empty_like(p)
    K.split_decode(hi, lo, v, out)
    assert torch.equal(bits(out), bits(p))


MODES = {
    "amsgrad": dict(amsgrad=True),
    "adam": dict(amsgrad=False),
    "l2_amsgrad": dict(amsgrad=True, weight_decay=0.05),
    "decoupled_amsgrad": dict(amsgrad=True, weight_decay=0.1, decoupled=True),
}


@pytest.mark.gpu
@pytest.mark.parametrize("lr", [0.0, 1e-3])   # lr 0 keeps the forced ties through the update, so they are encoded too
@pytest.mark.parametrize("mode", list(MODES))
def test_split_wgrad_adam_matches_fp32(mode, lr):
    G, N, Kd = 3, 256, 384
    gen = torch.Generator().manual_seed(11)
    dy, x, offs = wa_inputs(gen, [17, 0, 300], N, Kd)
    go = torch.tensor(offs, dtype=torch.int32, device="cuda")
    rows = torch.tensor([17, 0, 300], dtype=torch.int32, device="cuda")
    step = torch.tensor([1, 4, 9], dtype=torch.int32, device="cuda")
    p = as_f32(random_bits_with_ties(3, G * N * Kd)).view(G, N, Kd)
    m = torch.randn(G, N, Kd, device="cuda") * 1e-2
    v = torch.rand(G, N, Kd, device="cuda") * 1e-3
    vmax = v * 1.5
    kw = dict(step=step, lr=lr, **MODES[mode])
    amsgrad = MODES[mode]["amsgrad"]

    f32 = dict(p=p.clone(), m=m.clone(), v=v.clone(), vmax=vmax.clone() if amsgrad else None,
               p_bf16=torch.zeros(G, N, Kd, dtype=torch.bfloat16, device="cuda"))
    K.wgrad_adam(dy, x, go, rows, **f32, **kw)

    hi = torch.empty(G, N, Kd, dtype=torch.bfloat16, device="cuda")
    lo = torch.empty(G, N, Kd, dtype=torch.int16, device="cuda")
    sv = v.clone()
    K.split_encode(p.view(-1), hi.view(-1), lo.view(-1), sv.view(-1))
    split = dict(p=None, p_lo=lo, p_bf16=hi, m=m.clone(), v=sv, vmax=vmax.clone() if amsgrad else None)
    K.wgrad_adam(dy, x, go, rows, **split, **kw)
    out = torch.empty_like(p)
    K.split_decode(hi.view(-1), lo.view(-1), sv.view(-1), out.view(-1))
    torch.cuda.synchronize()

    assert torch.equal(bits(out), bits(f32["p"]))
    assert torch.equal(bits(split["m"]), bits(f32["m"]))
    assert torch.equal(bits(sv.abs()), bits(f32["v"]))
    if amsgrad:
        assert torch.equal(bits(split["vmax"]), bits(f32["vmax"]))
    # the mirror of the stepped groups; the skipped group keeps the planes it had, the fp32 run never wrote its mirror
    assert torch.equal(hi[[0, 2]].view(torch.int16), f32["p_bf16"][[0, 2]].view(torch.int16))
    assert not torch.equal(bits(out[[0, 2]]), bits(p[[0, 2]])) or lr == 0.0
    if lr == 0.0:   # ties went in and came out again
        assert bool(torch.signbit(sv[[0, 2]]).any())


@pytest.mark.gpu
def test_small_path_layer_matches_fp32_shard():
    """the split shard of a small-path layer against the same layer with its shard turned back into fp32 + mirror"""
    cfg = E.DMoEConfig(hidden=512, grid_size=(16,), k=4, num_layers=1, tokens_per_rank=256, lr=1e-3)
    gen = torch.Generator().manual_seed(5)
    data = [(torch.randn(256, 512, generator=gen), torch.randn(256, 512, generator=gen)) for _ in range(3)]
    result = {}
    for split in (True, False):
        torch.manual_seed(0)   # the gate's parameters
        ctx = E.EngineContext(cfg)
        layer = E.FusedDMoE(cfg, ctx).cuda()
        sh = layer.shard
        assert ctx.small and sh.split
        if not split:   # fp32 master weights + mirror, the format of the big path
            sh.p
            sh.v_raw.abs_()
            sh.split = False
        for x, g in data:
            layer(x.cuda()).backward(g.cuda())
        torch.cuda.synchronize()
        result[split] = dict(p=sh.p.clone(), v=sh.v.clone(), m=sh.m.clone(), vmax=sh.vmax.clone(),
                             bf16=sh.p_bf16.clone(), w2=sh.views["w2"].clone(), step=sh.step.clone())
        ctx.close()
    for k, t in result[True].items():
        assert torch.equal(t.view(torch.int16) if t.dtype == torch.bfloat16 else t.view(torch.int32),
                           result[False][k].view(torch.int16) if t.dtype == torch.bfloat16 else
                           result[False][k].view(torch.int32)), k
    assert not torch.equal(result[True]["step"], torch.zeros_like(result[True]["step"]))
