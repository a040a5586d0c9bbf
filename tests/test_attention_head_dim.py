"""The transformer expert at head dims 32 and 128 (d_model / heads; the reference's nhead = 16 gives them at hid_dim 512 and
2048): the attention kernels with and without dropout against fp32 oracles, determinism of the backward, refusal of every
other head dim, and on top of them the trained expert behind ExpertBackend, a server and the in-box layer.  Head dim 64 is
covered by tests/test_transformer_seq_len.py."""
import copy

import pytest
import torch

import lah_b200  # noqa
from lah_b200.ops import kernels as K

SEQS = [1, 17, 127, 128, 129, 300, 512, 1000, 2048]
SHAPES = [(512, 16), (256, 8), (2048, 16), (1024, 8)]   # (d_model, heads): head dims 32, 32, 128, 128
REFUSED = [(1024, 64), (768, 16), (768, 8), (2048, 8)]   # head dims 16, 48, 96, 256
GRAD_CHECKED = ("self_attn.in_proj_weight", "linear1.weight", "linear2.weight", "self_attn.out_proj.weight",
                "self_attn.in_proj_bias", "self_attn.out_proj.bias", "linear2.bias", "linear1.bias", "norm1.weight")


def test_head_dims():
    assert K.HEAD_DIMS == (32, 64, 128)


def rel(a, b):
    return ((a.float() - b.float()).norm() / (b.float().norm() + 1e-12)).item()


def grad_errs(dqkv, ref, d):
    """relative L2 errors of dQ, dK, dV; a slice whose reference is exactly 0 (S = 1) is measured against the whole gradient"""
    errs = {}
    for i, name in enumerate(("dq", "dk", "dv")):
        a, b = dqkv[:, i * d:(i + 1) * d].float(), ref[:, i * d:(i + 1) * d].float()
        scale = b.norm() if b.norm() > 0 else ref.float().norm()
        errs[name] = ((a - b).norm() / scale).item()
    return errs


def _qkv(batch, S, d, scale, seed):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(batch * S, 3 * d, generator=g) * scale).to(torch.bfloat16).cuda()


def _lse_ref(qkv, batch, S, heads):
    """base-2 row log-sum-exp of the scaled scores, [B, H, S]"""
    hd = qkv.shape[1] // 3 // heads
    q, k, _ = qkv.float().view(batch, S, 3, heads, hd).unbind(2)
    s = torch.einsum("bqhd,bkhd->bhqk", q, k) / hd ** 0.5
    return torch.logsumexp(s, dim=-1) / 0.6931471805599453


# ------------------------------------------------------------------------------------------------ GPU: attention kernels
@pytest.mark.gpu
@pytest.mark.parametrize("d,heads", SHAPES)
@pytest.mark.parametrize("batch", [1, 3])
@pytest.mark.parametrize("S", SEQS)
def test_attention_fwd_head_dim(S, batch, d, heads):
    T = batch * S
    qkv = _qkv(batch, S, d, 1.5, S * 10 + batch + d)
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
def test_attention_bwd_head_dim(S, batch, d, heads):
    T = batch * S
    qkv = _qkv(batch, S, d, 1.2, S * 10 + batch + d + 1)
    g = torch.Generator().manual_seed(S + d)
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


# ------------------------------------------------------------------------------------------------ GPU: dropout, determinism
@pytest.mark.gpu
@pytest.mark.parametrize("d", [512, 2048])
@pytest.mark.parametrize("S", [100, 512, 1000])
def test_attention_dropout_head_dim(S, d):
    from tools.gpu_attention_check import attention_dropout_ref
    batch, heads, p, seed = 2, 16, 0.1, 777 + S + d
    T = batch * S
    qkv = _qkv(batch, S, d, 1.2, S + d + 7)
    g = torch.Generator().manual_seed(S + d + 8)
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
@pytest.mark.parametrize("d,heads", [(512, 16), (2048, 16)])
def test_attention_p0_is_no_dropout(d, heads):
    S, batch = 300, 2
    T = batch * S
    qkv = _qkv(batch, S, d, 1.2, d + 3)
    dout = torch.randn(T, d, generator=torch.Generator().manual_seed(d)).to(torch.bfloat16).cuda()
    res = []
    for dropout in (None, (0.0, 1234)):
        lse = torch.empty(T, heads, device="cuda")
        out = K.attention_fwd(qkv, heads, lse=lse, dropout=dropout, seq_len=S)
        dqkv = K.attention_bwd(qkv, out, dout, lse, heads, dropout=dropout, seq_len=S)
        res.append((out, lse, dqkv))
    torch.cuda.synchronize()
    for a, b in zip(*res):
        assert torch.equal(a.view(torch.uint8) if a.dtype == torch.bfloat16 else a.view(torch.int32),
                           b.view(torch.uint8) if b.dtype == torch.bfloat16 else b.view(torch.int32))


@pytest.mark.gpu
@pytest.mark.parametrize("dropout", [None, (0.1, 99)])
def test_attention_bwd_hd128_is_deterministic(dropout):
    S, batch, d, heads = 1000, 2, 2048, 16
    T = batch * S
    qkv = _qkv(batch, S, d, 1.2, 5)
    dout = torch.randn(T, d, generator=torch.Generator().manual_seed(6)).to(torch.bfloat16).cuda()
    lse = torch.empty(T, heads, device="cuda")
    out = K.attention_fwd(qkv, heads, lse=lse, dropout=dropout, seq_len=S)
    a = K.attention_bwd(qkv, out, dout, lse, heads, dropout=dropout, seq_len=S).clone()
    b = K.attention_bwd(qkv, out, dout, lse, heads, dropout=dropout, seq_len=S)
    torch.cuda.synchronize()
    assert torch.equal(a.view(torch.uint8), b.view(torch.uint8))


# ------------------------------------------------------------------------------------------------ GPU: refused head dims
@pytest.mark.gpu
@pytest.mark.parametrize("d,heads", REFUSED + [(1000, 16)])
def test_attention_refuses_other_head_dims_masked_or_not(d, heads):
    from lah_b200.ops.native import c_void_p, stream_ptr
    S = 128
    qkv = torch.zeros(S, 3 * d, dtype=torch.bfloat16, device="cuda")
    out = torch.zeros(S, d, dtype=torch.bfloat16, device="cuda")
    lse = torch.zeros(S, heads, device="cuda")
    mask = torch.full((1, S // 32), -1, dtype=torch.int32, device="cuda")   # every key valid
    lib = K._lib()
    P = c_void_p
    for key_mask in (P(0), P(mask.data_ptr())):
        assert lib.lah_attention_fwd(P(qkv.data_ptr()), P(out.data_ptr()), P(lse.data_ptr()), S, S, heads, d, 0, -1, 1.0,
                                     stream_ptr(), key_mask) == -2
        assert lib.lah_attention_bwd(P(qkv.data_ptr()), P(out.data_ptr()), P(out.data_ptr()), P(lse.data_ptr()), P(0), P(0),
                                     P(0), S, S, heads, d, 0, -1, 1.0, stream_ptr(), key_mask) == -2
    with pytest.raises(Exception):
        K.attention_fwd(qkv, heads, seq_len=S)
    with pytest.raises(Exception):
        K.attention_bwd(qkv, out, out, lse, heads, seq_len=S)


@pytest.mark.gpu
@pytest.mark.parametrize("d,heads", REFUSED)
def test_backend_falls_back_for_other_head_dims(d, heads):
    from lah_b200.models.layers import TransformerEncoderLayer
    from lah_b200.runtime.native_executor import NativeTransformerExecutor, make_executor
    torch.manual_seed(0)
    layer = TransformerEncoderLayer(d, heads).cuda()
    opt = torch.optim.Adam(layer.parameters(), lr=1e-4, amsgrad=True)
    assert not NativeTransformerExecutor.supports(layer, opt)
    assert not isinstance(make_executor(layer, opt), NativeTransformerExecutor)
    be = lah_b200.ExpertBackend(name="r", expert=layer, opt=opt, args_schema=(lah_b200.BatchTensorProto(64, d),),
                                outputs_schema=lah_b200.BatchTensorProto(64, d), max_batch_size=4)
    layer.eval()
    x = torch.randn(2, 64, d, device="cuda")
    (y,) = be.forward(x)
    assert be._executor is None
    with torch.no_grad():
        assert torch.allclose(y, layer(x))


# ------------------------------------------------------------------------------------------------ GPU: public interface
def _dropout_masks(seed, ps, batch, heads, S, d, ff):
    T = batch * S
    shapes = ((batch, heads, S, S), (T, d), (T, ff), (T, d))
    return [K.dropout_mask(shape, p, seed, site).float() for site, (shape, p) in enumerate(zip(shapes, ps))]


def _backend(layer, S, d, name="t"):
    return lah_b200.ExpertBackend(name=name, expert=layer, opt=torch.optim.Adam(layer.parameters(), lr=1e-4, amsgrad=True),
                                  args_schema=(lah_b200.BatchTensorProto(S, d),),
                                  outputs_schema=lah_b200.BatchTensorProto(S, d), max_batch_size=8)


@pytest.mark.gpu
@pytest.mark.parametrize("d", [512, 2048])
@pytest.mark.parametrize("S", [512, 300])
def test_expert_backend_trains_default_expert_at_head_dim(S, d):
    """name_to_block["transformer"](d) (16 heads, dropout 0.1) through ExpertBackend: forward, dx, weight gradients and
    three AMSGrad steps against the fp32 functional oracle with the same masks; eval mode against the oracle without
    dropout (the tolerances of tests/test_transformer_seq_len.py)"""
    from lah_b200.models.layers import name_to_block
    from lah_b200.ops import native
    from lah_b200.runtime.native_executor import NativeTransformerExecutor, draw_dropout_seed
    from tools.gpu_attention_check import transformer_layer_ref
    torch.manual_seed(4)
    layer = name_to_block["transformer"](d).cuda()
    ff = layer.linear1.out_features
    ref = copy.deepcopy(layer)
    ref_opt = torch.optim.Adam(ref.parameters(), lr=1e-4, amsgrad=True)
    be = _backend(layer, S, d)
    ps = NativeTransformerExecutor._dropout_ps(layer)
    assert ps == (0.1,) * 4
    x = torch.randn(2, S, d, device="cuda")
    g = torch.randn(2, S, d, device="cuda") * 0.1
    native.reset_launches()
    torch.manual_seed(10)
    seed = draw_dropout_seed()
    torch.manual_seed(10)
    (y,) = be.forward(x)
    assert type(be._executor) is NativeTransformerExecutor and native.launches() > 0
    with torch.no_grad():
        assert rel(y, transformer_layer_ref(ref, x, _dropout_masks(seed, ps, 2, 16, S, d, ff), ps)) < 3e-2
    for it in range(3):
        torch.manual_seed(20 + it)
        seed = draw_dropout_seed()
        torch.manual_seed(20 + it)
        launches = native.launches()
        (gx,) = be.backward(x, g)
        assert native.launches() > launches
        xr = x.clone().requires_grad_(True)
        transformer_layer_ref(ref, xr, _dropout_masks(seed, ps, 2, 16, S, d, ff), ps).backward(g)
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
def test_server_round_trip_at_d2048():
    from lah_b200.models.layers import name_to_block
    from lah_b200.runtime.native_executor import NativeTransformerExecutor
    torch.manual_seed(1)
    layer = name_to_block["transformer"](2048).cuda()
    be = _backend(layer, 256, 2048, name="t2048")
    srv = lah_b200.TesseractServer(None, {"t2048": be}, port=0, conn_handler_processes=1, device="cuda")
    srv.run_in_background()
    try:
        remote = lah_b200.RemoteExpert("t2048", "127.0.0.1", srv.port, timeout=120)
        x = torch.randn(2, 256, 2048, requires_grad=True)
        y = remote(x)   # an err_ reply raises RemoteExpertError
        assert y.shape == x.shape and bool(torch.isfinite(y).all())
        y.sum().backward()
        assert x.grad is not None and x.grad.shape == x.shape and bool(torch.isfinite(x.grad).all())
        assert be.update_count == 1 and type(be._executor) is NativeTransformerExecutor
    finally:
        srv.shutdown()


@pytest.mark.gpu
@pytest.mark.parametrize("d", [512, 2048])
def test_inbox_layer_head_dim(d):
    from lah_b200.models.layers import TransformerEncoderLayer
    from lah_b200.models.transformer_native import NativeTransformerLayer
    torch.manual_seed(1)
    layer = TransformerEncoderLayer(d, 16).cuda().eval()
    native = NativeTransformerLayer(layer)
    x = torch.randn(3, 300, d, device="cuda")
    with torch.no_grad():
        ref = layer(x)
    out = native(x)
    assert out.shape == x.shape and rel(out, ref) < 3e-2


@pytest.mark.gpu
def test_inbox_layer_refuses_other_head_dims():
    from lah_b200.models.layers import TransformerEncoderLayer
    from lah_b200.models.transformer_native import NativeTransformerLayer
    with pytest.raises(AssertionError):
        NativeTransformerLayer(TransformerEncoderLayer(2048, 8).cuda().eval())
