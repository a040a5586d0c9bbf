"""The transformer expert at any sequence length 1 <= S <= MAX_SEQ: the site-0 dropout counter beyond 512 tokens (CPU), and on
the GPU the attention kernels, their dropout, the trained expert behind ExpertBackend and a server, and the in-box layer
against fp32 oracles; S = 512 stays bit-identical to the 512-token kernels (tests/golden/seq512_digests.json)."""
import copy
import json
import math
import os

import pytest
import torch

import lah_b200  # noqa
from lah_b200.ops import kernels as K

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "seq512_digests.json")
SEQS = [1, 2, 17, 100, 127, 128, 129, 384, 512, 640, 1000, 2048, 4096]
SHAPES = [(1024, 16), (256, 4)]   # (d_model, heads)
GRAD_CHECKED = ("self_attn.in_proj_weight", "linear1.weight", "linear2.weight", "self_attn.out_proj.weight",
                "self_attn.in_proj_bias", "self_attn.out_proj.bias", "linear2.bias", "linear1.bias", "norm1.weight")


def rel(a, b):
    return ((a.float() - b.float()).norm() / (b.float().norm() + 1e-12)).item()


def grad_errs(dqkv, ref, d):
    """relative L2 errors of dQ, dK, dV.  At S = 1 the softmax is constant, so the exact dQ and dK are 0 and the kernel's
    are rounding noise; a slice whose reference is exactly 0 is measured against the norm of the whole gradient."""
    errs = {}
    for i, name in enumerate(("dq", "dk", "dv")):
        a, b = dqkv[:, i * d:(i + 1) * d].float(), ref[:, i * d:(i + 1) * d].float()
        scale = b.norm() if b.norm() > 0 else ref.float().norm()
        errs[name] = ((a - b).norm() / scale).item()
    return errs


def keep_512_layout(p, seed, b, h, q, k):
    """the site-0 keep decision of the 512-token kernels, written out: counter (gq * 128 + gk | (q & 1) << 14, h, b, 0)"""
    gq, gk = (q >> 4) * 4 + ((q >> 1) & 3), (k >> 4) * 4 + ((k >> 1) & 3)
    q, k, gq, gk = torch.broadcast_tensors(q, k, gq, gk)
    ctr = ((gq * 128 + gk) | ((q & 1) << 14), torch.full_like(q, h), torch.full_like(q, b), torch.zeros_like(q))
    lane = ((q >> 3) & 1) * 4 + ((k & 1) | (((k >> 3) & 1) << 1))
    words = torch.stack(K.philox4x32_10_ref(ctr, (seed & 0xFFFFFFFF, seed >> 32)), dim=-1)
    w = words.gather(-1, (lane >> 1).unsqueeze(-1)).squeeze(-1)
    return torch.where((lane & 1) == 1, w >> 16, w & 0xFFFF) >= K.dropout_threshold(p)


# ------------------------------------------------------------------------------------------------ CPU: the dropout counter
@pytest.mark.parametrize("seed", [0, 12345, 2 ** 64 - 3])
@pytest.mark.parametrize("b,h", [(0, 0), (5, 13)])
def test_site0_mask_unchanged_below_512(seed, b, h):
    q, k = torch.arange(512).view(-1, 1), torch.arange(512).view(1, -1)
    assert torch.equal(K.dropout_keep_ref(0.1, seed, K.SITE_ATTN, b, h, q, k), keep_512_layout(0.1, seed, b, h, q, k))


def test_site0_counter_is_injective_at_2048():
    q, k = torch.arange(2048).view(-1, 1), torch.arange(2048).view(1, -1)
    (x, y, z, w), lane = K.dropout_counter_ref(K.SITE_ATTN, 1, 2, q, k)
    assert int(y.unique().numel()) == 1 and int(z.unique().numel()) == 1
    assert int(x.max()) < 2 ** 15 and int(w.max()) < 2 ** 32 and int(lane.max()) < 8
    code = (w * 2 ** 15 + x) * 8 + lane
    assert code.unique().numel() == 2048 * 2048


def test_site0_counters_differ_from_sites_1_to_3():
    """site 0 keeps the low byte of the last counter word at 0; sites 1-3 put their site number there"""
    q, k = torch.arange(0, 4096, 7).view(-1, 1), torch.arange(0, 4096, 5).view(1, -1)
    w0 = K.dropout_counter_ref(K.SITE_ATTN, 3, 1, q, k)[0][3]
    assert int((w0 & 0xFF).max()) == 0 and int(w0.max()) > 0
    r, n = torch.arange(0, 65536, 97).view(-1, 1), torch.arange(0, 4096, 3).view(1, -1)
    for site in (1, 2, 3):
        assert int((K.dropout_counter_ref(site, r, n)[0][3] != site).sum()) == 0


def test_keep_fraction_at_2048_within_5_sigma():
    keep = K.dropout_mask_ref((1, 1, 2048, 2048), 0.1, 987654321, K.SITE_ATTN)
    n = keep.numel()
    assert abs(keep.float().mean().item() - 0.9) < 5 * math.sqrt(0.1 * 0.9 / n)


# ------------------------------------------------------------------------------------------------ GPU: attention kernels
def _qkv(batch, S, d, scale, seed):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(batch * S, 3 * d, generator=g) * scale).to(torch.bfloat16).cuda()


def _lse_ref(qkv, batch, S, heads):
    q, k, _ = qkv.float().view(batch, S, 3, heads, 64).unbind(2)
    s2 = torch.einsum("bqhd,bkhd->bhqk", q, k) * (0.125 * 1.4426950408889634)
    return torch.logsumexp(s2 * 0.6931471805599453, dim=-1) / 0.6931471805599453   # [B, H, S], log2 sum 2^s


@pytest.mark.gpu
@pytest.mark.parametrize("d,heads", SHAPES)
@pytest.mark.parametrize("batch", [1, 3])
@pytest.mark.parametrize("S", SEQS)
def test_attention_fwd_any_seq_len(S, batch, d, heads):
    T = batch * S
    qkv = _qkv(batch, S, d, 1.5, S * 10 + batch)
    out_buf = torch.full((T + 16, d), 7.0, dtype=torch.bfloat16, device="cuda")
    lse_buf = torch.full((T + 16, heads), -123.0, device="cuda")
    out = K.attention_fwd(qkv, heads, out=out_buf[:T], lse=lse_buf[:T], seq_len=S)
    torch.cuda.synchronize()
    assert out.data_ptr() == out_buf.data_ptr()
    assert rel(out, K.attention_ref(qkv, heads, seq_len=S)) < 2e-2
    lse_err = (lse_buf[:T].view(batch, S, heads).transpose(1, 2) - _lse_ref(qkv, batch, S, heads)).abs().max().item()
    assert lse_err < 3e-2
    assert bool((out_buf[T:] == 7.0).all()) and bool((lse_buf[T:] == -123.0).all())


@pytest.mark.gpu
@pytest.mark.parametrize("d,heads", SHAPES)
@pytest.mark.parametrize("batch", [1, 3])
@pytest.mark.parametrize("S", SEQS)
def test_attention_bwd_any_seq_len(S, batch, d, heads):
    T = batch * S
    qkv = _qkv(batch, S, d, 1.2, S * 10 + batch + 1)
    g = torch.Generator().manual_seed(S)
    dout = torch.randn(T, d, generator=g).to(torch.bfloat16).cuda()
    lse = torch.empty(T, heads, device="cuda")
    out = K.attention_fwd(qkv, heads, lse=lse, seq_len=S)
    dqkv_buf = torch.full((T + 16, 3 * d), 5.0, dtype=torch.bfloat16, device="cuda")
    dqkv = K.attention_bwd(qkv, out, dout, lse, heads, seq_len=S, dqkv=dqkv_buf[:T])
    torch.cuda.synchronize()
    assert bool(torch.isfinite(dqkv).all())
    assert bool((dqkv_buf[T:] == 5.0).all())
    ref_in = qkv.float().requires_grad_(True)
    K.attention_ref(ref_in, heads, seq_len=S).backward(dout.float())
    errs = grad_errs(dqkv, ref_in.grad, d)
    assert all(v < 3e-2 for v in errs.values()), errs


@pytest.mark.gpu
def test_attention_rejects_bad_seq_len_masked_or_not():
    qkv = torch.zeros(300, 3 * 256, dtype=torch.bfloat16, device="cuda")
    for S in (0, 7, K.MAX_SEQ + 1):
        with pytest.raises(Exception):
            K.attention_fwd(qkv, 4, seq_len=S)
    from lah_b200.ops.native import c_void_p, stream_ptr
    lib = K._lib()
    mask = torch.full((1, 1), -1, dtype=torch.int32, device="cuda")   # never read: the host checks refuse first
    for key_mask in (c_void_p(0), c_void_p(mask.data_ptr())):
        for tokens, S in ((300, 7), (K.MAX_SEQ + 1, K.MAX_SEQ + 1), (300, 0)):
            assert lib.lah_attention_fwd(c_void_p(qkv.data_ptr()), c_void_p(0), c_void_p(0), tokens, S, 4, 256, 0, -1, 1.0,
                                         stream_ptr(), key_mask) == -2
            assert lib.lah_attention_bwd(c_void_p(qkv.data_ptr()), c_void_p(0), c_void_p(0), c_void_p(0), c_void_p(0),
                                         c_void_p(0), c_void_p(0), tokens, S, 4, 256, 0, -1, 1.0, stream_ptr(), key_mask) == -2


@pytest.mark.gpu
@pytest.mark.parametrize("S", [100, 640, 2048])
def test_dropout_mask_beyond_512_matches_cpu(S):
    shape = (1 if S > 1000 else 2, 2, S, S)
    seed = 2 ** 63 + S
    assert torch.equal(K.dropout_mask(shape, 0.1, seed, K.SITE_ATTN).cpu(), K.dropout_mask_ref(shape, 0.1, seed, K.SITE_ATTN))


@pytest.mark.gpu
@pytest.mark.parametrize("S", [100, 1000, 2048])
def test_attention_dropout_any_seq_len(S):
    from tools.gpu_attention_check import attention_dropout_ref
    batch, heads, d, p, seed = 2, 16, 1024, 0.1, 4242 + S
    T = batch * S
    qkv = _qkv(batch, S, d, 1.2, S + 7)
    g = torch.Generator().manual_seed(S + 8)
    dout = torch.randn(T, d, generator=g).to(torch.bfloat16).cuda()
    lse = torch.empty(T, heads, device="cuda")
    out = K.attention_fwd(qkv, heads, lse=lse, dropout=(p, seed), seq_len=S)
    dqkv = K.attention_bwd(qkv, out, dout, lse, heads, dropout=(p, seed), seq_len=S)
    mask = K.dropout_mask((batch, heads, S, S), p, seed, K.SITE_ATTN).float()
    ref_in = qkv.float().requires_grad_(True)
    ref = attention_dropout_ref(ref_in, heads, mask, p, seq_len=S)
    ref.backward(dout.float())
    assert rel(out, ref.detach()) < 2e-2
    assert bool(torch.isfinite(dqkv).all())
    errs = grad_errs(dqkv, ref_in.grad, d)
    assert all(v < 3e-2 for v in errs.values()), errs
    lse_err = (lse.view(batch, S, heads).transpose(1, 2) - _lse_ref(qkv, batch, S, heads)).abs().max().item()
    assert lse_err < 3e-2   # the LSE of the undropped softmax


@pytest.mark.gpu
def test_seq512_bit_identical_to_512_token_kernels():
    from tools import seq512_digests
    with open(GOLDEN) as f:
        golden = json.load(f)
    assert seq512_digests.compute() == golden


# ------------------------------------------------------------------------------------------------ GPU: public interface
def _dropout_masks(seed, ps, batch, heads, S, d, ff):
    T = batch * S
    shapes = ((batch, heads, S, S), (T, d), (T, ff), (T, d))
    return [K.dropout_mask(shape, p, seed, site).float() for site, (shape, p) in enumerate(zip(shapes, ps))]


def _backend(layer, S, name="t"):
    return lah_b200.ExpertBackend(name=name, expert=layer, opt=torch.optim.Adam(layer.parameters(), lr=1e-4, amsgrad=True),
                                  args_schema=(lah_b200.BatchTensorProto(S, 1024),),
                                  outputs_schema=lah_b200.BatchTensorProto(S, 1024), max_batch_size=8)


@pytest.mark.gpu
@pytest.mark.parametrize("S", [128, 300, 1024])
def test_expert_backend_trains_default_expert_at_seq_len(S):
    """the reference's default expert (dropout 0.1) through ExpertBackend at S != 512: forward, dx, weight gradients and
    three AMSGrad steps against the fp32 functional oracle with the same masks; eval mode against the oracle without
    dropout (tolerances of tools/gpu_attention_check.py::check_transformer_train_dropout)"""
    from lah_b200.models.layers import name_to_block
    from lah_b200.ops import native
    from lah_b200.runtime.native_executor import NativeTransformerExecutor, draw_dropout_seed
    from tools.gpu_attention_check import transformer_layer_ref
    torch.manual_seed(4)
    layer = name_to_block["transformer"](1024).cuda()
    ref = copy.deepcopy(layer)
    ref_opt = torch.optim.Adam(ref.parameters(), lr=1e-4, amsgrad=True)
    be = _backend(layer, S)
    ps = NativeTransformerExecutor._dropout_ps(layer)
    assert ps == (0.1,) * 4
    x = torch.randn(2, S, 1024, device="cuda")
    g = torch.randn(2, S, 1024, device="cuda") * 0.1
    native.reset_launches()
    torch.manual_seed(10)
    seed = draw_dropout_seed()
    torch.manual_seed(10)
    (y,) = be.forward(x)
    assert type(be._executor) is NativeTransformerExecutor and native.launches() > 0
    with torch.no_grad():
        assert rel(y, transformer_layer_ref(ref, x, _dropout_masks(seed, ps, 2, 16, S, 1024, 2048), ps)) < 3e-2
    for it in range(3):
        torch.manual_seed(20 + it)
        seed = draw_dropout_seed()
        torch.manual_seed(20 + it)
        launches = native.launches()
        (gx,) = be.backward(x, g)
        assert native.launches() > launches
        xr = x.clone().requires_grad_(True)
        transformer_layer_ref(ref, xr, _dropout_masks(seed, ps, 2, 16, S, 1024, 2048), ps).backward(g)
        if it == 0:
            assert rel(gx, xr.grad) < 5e-2
            st = be.opt.state_dict()["state"]
            for i, (n, p) in enumerate(ref.named_parameters()):
                if n in GRAD_CHECKED:
                    assert rel(st[i]["exp_avg"] / 0.1, p.grad) < 6e-2, n
        ref_opt.step(), ref_opt.zero_grad()
    sd, rsd = be.state_dict(), ref.state_dict()
    assert max((sd["expert." + k] - v).abs().mean().item() for k, v in rsd.items()) < 1.5e-4
    layer.eval()
    ref.eval()
    with torch.no_grad():
        assert rel(be.forward(x)[0], transformer_layer_ref(ref, x)) < 3e-2


@pytest.mark.gpu
def test_server_round_trip_at_seq_256():
    from lah_b200.models.layers import name_to_block
    from lah_b200.runtime.native_executor import NativeTransformerExecutor
    torch.manual_seed(1)
    layer = name_to_block["transformer"](1024).cuda()
    be = _backend(layer, 256, name="t256")
    srv = lah_b200.TesseractServer(None, {"t256": be}, port=0, conn_handler_processes=1, device="cuda")
    srv.run_in_background()
    try:
        remote = lah_b200.RemoteExpert("t256", "127.0.0.1", srv.port, timeout=120)
        x = torch.randn(2, 256, 1024, requires_grad=True)
        y = remote(x)   # an err_ reply raises RemoteExpertError
        assert y.shape == x.shape and bool(torch.isfinite(y).all())
        y.sum().backward()
        assert x.grad is not None and x.grad.shape == x.shape and bool(torch.isfinite(x.grad).all())
        assert be.update_count == 1 and type(be._executor) is NativeTransformerExecutor
    finally:
        srv.shutdown()


@pytest.mark.gpu
def test_executors_accept_only_what_they_run():
    from lah_b200.models.layers import FeedforwardBlock, name_to_block
    from lah_b200.runtime.native_executor import make_executor
    layer = name_to_block["transformer"](1024).cuda()
    ex = make_executor(layer, torch.optim.Adam(layer.parameters(), lr=1e-4, amsgrad=True))
    meta = dict(device="meta")
    assert ex.accepts(torch.empty(2, 1, 1024, **meta)) and ex.accepts(torch.empty(1, K.MAX_SEQ, 1024, **meta))
    assert not ex.accepts(torch.empty(1, K.MAX_SEQ + 1, 1024, **meta))
    assert not ex.accepts(torch.empty(2, 300, 512, **meta))
    assert not ex.accepts(torch.empty(2, 0, 1024, **meta)) and not ex.accepts(torch.empty(300, 1024, **meta))
    block = FeedforwardBlock(128).cuda()
    fex = make_executor(block, torch.optim.Adam(block.parameters(), amsgrad=True))
    assert fex.accepts(torch.empty(5, 128, **meta))
    assert not fex.accepts(torch.empty(5, 64, **meta)) and not fex.accepts(torch.empty(2, 5, 128, **meta))


@pytest.mark.gpu
@pytest.mark.parametrize("S", [200, 1024])
def test_inbox_layer_any_seq_len(S):
    from lah_b200.models.layers import TransformerEncoderLayer
    from lah_b200.models.transformer_native import NativeTransformerLayer
    torch.manual_seed(1)
    layer = TransformerEncoderLayer(1024, 16).cuda().eval()
    native = NativeTransformerLayer(layer)
    x = torch.randn(3, S, 1024, device="cuda")
    with torch.no_grad():
        ref = layer(x)
    out = native(x)
    assert out.shape == x.shape and rel(out, ref) < 3e-2
