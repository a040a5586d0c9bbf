"""Causal self-attention (position t attends to positions <= t): this package's TransformerEncoderLayer(causal=True) against
torch's layer with is_causal=True on the CPU; on the GPU the causal attention kernels against a float64 oracle, their exact
properties (no leak from later tokens, the dropout mask of the bidirectional kernel on key <= query), and the causal layer
behind ExpertBackend, a server and NativeTransformerLayer."""
import copy

import pytest
import torch
import torch.nn.functional as F

import lah_b200
from lah_b200.models.layers import TransformerEncoderLayer, name_to_block
from lah_b200.ops import kernels as K
from lah_b200.runtime.native_executor import EncoderLayerSpec, encoder_layer_spec

SEQS = [1, 100, 128, 300, 512, 1000, 2048]
GRAD_CHECKED = ("self_attn.in_proj_weight", "linear1.weight", "linear2.weight", "self_attn.out_proj.weight",
                "self_attn.in_proj_bias", "self_attn.out_proj.bias", "linear2.bias", "linear1.bias", "norm1.weight")


def rel(a, b):
    return ((a.double() - b.double()).norm() / (b.double().norm() + 1e-12)).item()


def _parent_forward(layer, src):
    """the forward of TransformerEncoderLayer before it had ``causal``, op for op"""
    x = src.transpose(0, 1)
    attn = layer.self_attn(x, x, x, need_weights=False)[0]
    x = layer.norm1(x + layer.dropout1(attn))
    ff = layer.linear2(layer.dropout(layer.activation(layer.linear1(x))))
    x = layer.norm2(x + layer.dropout2(ff))
    return x.transpose(0, 1)


def _torch_twin(layer):
    """nn.TransformerEncoderLayer with the weights of ``layer`` (batch-first, post-LN, erf GELU)"""
    a = layer.self_attn
    twin = torch.nn.TransformerEncoderLayer(a.embed_dim, a.num_heads, layer.linear1.out_features, dropout=layer.dropout.p,
                                            activation="gelu", batch_first=True, dtype=a.in_proj_weight.dtype)
    twin.load_state_dict(layer.state_dict())
    return twin


# ------------------------------------------------------------------------------------------------ CPU
@pytest.mark.parametrize("train", [False, True])
def test_non_causal_layer_is_unchanged(train):
    """causal=False (the default) has the parameters of the layer before the flag and computes the same result, bit for
    bit, dropout included"""
    torch.manual_seed(0)
    layer = TransformerEncoderLayer(64, 4, 128)
    assert layer.causal is False and not TransformerEncoderLayer(64, 4, 128, causal=False).causal
    torch.manual_seed(0)
    again = TransformerEncoderLayer(64, 4, 128, causal=True)
    assert [n for n, _ in layer.named_parameters()] == [n for n, _ in again.named_parameters()]
    assert all(torch.equal(p, q) for p, q in zip(layer.parameters(), again.parameters()))
    layer.train(train)
    x = torch.randn(3, 37, 64)
    torch.manual_seed(5)
    y = layer(x)
    torch.manual_seed(5)
    assert torch.equal(y, _parent_forward(layer, x))
    assert not name_to_block["transformer"](256).causal


@pytest.mark.parametrize("S", [1, 17, 64])
def test_causal_layer_matches_torch_is_causal_fp64(S):
    torch.manual_seed(S)
    layer = TransformerEncoderLayer(32, 4, 64, causal=True).double().eval()
    twin = _torch_twin(layer).eval()
    x = torch.randn(3, S, 32, dtype=torch.float64)
    mask = torch.nn.Transformer.generate_square_subsequent_mask(S, dtype=torch.float64)
    y = layer(x)
    assert (y - twin(x, src_mask=mask, is_causal=True)).abs().max().item() < 1e-12
    # and the causal oracle of the kernels, inside in_proj / out_proj, in training mode with dropout 0 (gradients too)
    layer.train()
    for m in (layer.dropout, layer.dropout1, layer.dropout2):
        m.p = 0.0
    layer.self_attn.dropout = 0.0
    xr = x.clone().requires_grad_(True)
    ref = layer(xr)
    g = torch.randn_like(ref)
    dx_ref, = torch.autograd.grad(ref, xr, g)
    a = layer.self_attn
    x2 = x.clone().requires_grad_(True)
    att = K.attention_ref(F.linear(x2.reshape(3 * S, 32), a.in_proj_weight, a.in_proj_bias), 4, seq_len=S, causal=True)
    h = layer.norm1(x2 + F.linear(att, a.out_proj.weight, a.out_proj.bias).view(3, S, 32))
    out = layer.norm2(h + layer.linear2(F.gelu(layer.linear1(h))))
    dx, = torch.autograd.grad(out, x2, g)
    assert (out - ref).abs().max().item() < 1e-12 and (dx - dx_ref).abs().max().item() < 1e-12


def test_later_tokens_do_not_change_earlier_outputs_cpu():
    torch.manual_seed(1)
    layer = TransformerEncoderLayer(32, 4, 64, causal=True).double().eval()
    x = torch.randn(2, 20, 32, dtype=torch.float64)
    x2 = x.clone()
    x2[:, 9:] = torch.randn(2, 11, 32, dtype=torch.float64)
    assert (layer(x)[:, :9] - layer(x2)[:, :9]).abs().max().item() < 1e-12


@pytest.mark.parametrize("train", [False, True])
def test_scripted_causal_layer_equals_plain(train):
    torch.manual_seed(2)
    layer = TransformerEncoderLayer(64, 4, 128, causal=True).train(train)
    scripted = torch.jit.script(copy.deepcopy(layer))
    x = torch.randn(2, 33, 64)
    torch.manual_seed(9)
    y = layer(x)
    torch.manual_seed(9)
    assert torch.equal(y, scripted(x))


def test_encoder_layer_spec_reports_causal():
    spec = encoder_layer_spec(TransformerEncoderLayer(512, 16, causal=True))
    assert spec == EncoderLayerSpec(512, 16, 2048, False, "gelu", True, (0.1,) * 4, True) and spec.causal
    assert encoder_layer_spec(torch.jit.script(TransformerEncoderLayer(512, 16, causal=True))).causal
    assert not encoder_layer_spec(TransformerEncoderLayer(512, 16)).causal
    assert not encoder_layer_spec(torch.nn.TransformerEncoderLayer(512, 16)).causal


@pytest.mark.parametrize("tokens,S", [(300, 7), (300, 0), (0, K.MAX_SEQ + 1)])
def test_causal_wrappers_refuse_bad_sequence_lengths_before_any_launch(monkeypatch, tokens, S):
    def no_launch():
        raise RuntimeError("a kernel was about to be launched")

    monkeypatch.setattr(K, "_lib", no_launch)
    qkv = torch.zeros(tokens, 3 * 256, dtype=torch.bfloat16)
    out = torch.zeros(tokens, 256, dtype=torch.bfloat16)
    lse = torch.zeros(tokens, 4)
    with pytest.raises(AssertionError):
        K.attention_fwd(qkv, 4, seq_len=S, causal=True)
    with pytest.raises(AssertionError):
        K.attention_bwd(qkv, out, out, lse, 4, seq_len=S, causal=True)


# ------------------------------------------------------------------------------------------------ GPU: kernels
def _qkv(batch, S, d, seed, scale=1.2):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(batch * S, 3 * d, generator=g) * scale).to(torch.bfloat16).cuda()


def _causal_ref(qkv, heads, S, drop_mask=None, p=0.0):
    """float64 oracle: causal masked softmax, with an optional site-0 keep mask [B, H, S, S]"""
    T, d = qkv.shape[0], qkv.shape[1] // 3
    q, k, v = (t.transpose(1, 2) for t in qkv.view(T // S, S, 3, heads, d // heads).unbind(2))
    s = (q @ k.transpose(-1, -2) / (d // heads) ** 0.5).masked_fill(
        torch.ones(S, S, dtype=torch.bool, device=qkv.device).triu(1), float("-inf"))
    att = torch.softmax(s, dim=-1)
    if drop_mask is not None:
        att = att * drop_mask / (1 - p)
    return (att @ v).transpose(1, 2).reshape(T, d)


def _run(qkv, heads, S, dout, dropout=None):
    T = qkv.shape[0]
    lse = torch.empty(T, heads, device="cuda")
    out = K.attention_fwd(qkv, heads, lse=lse, seq_len=S, dropout=dropout, causal=True)
    dqkv = K.attention_bwd(qkv, out, dout, lse, heads, seq_len=S, dropout=dropout, causal=True)
    return out, lse, dqkv


@pytest.mark.gpu
@pytest.mark.parametrize("drop", [False, True])
@pytest.mark.parametrize("hd", K.HEAD_DIMS)
@pytest.mark.parametrize("S", SEQS)
def test_causal_attention_matches_fp64_oracle(S, hd, drop):
    B, heads = 3, 2
    d, T = heads * hd, 3 * S
    qkv = _qkv(B, S, d, S * 7 + hd)
    dout = (torch.randn(T, d, generator=torch.Generator().manual_seed(S + 1)) * 0.5).to(torch.bfloat16).cuda()
    p, seed = 0.1, 99 + S
    dropout = (p, seed) if drop else None
    out, lse, dqkv = _run(qkv, heads, S, dout, dropout)
    torch.cuda.synchronize()
    drop_mask = K.dropout_mask((B, heads, S, S), p, seed, K.SITE_ATTN).double() if drop else None
    ref_in = qkv.double().requires_grad_(True)
    ref = _causal_ref(ref_in, heads, S, drop_mask, p)
    ref.backward(dout.double())
    assert rel(out, ref.detach()) < 2e-2
    assert bool(torch.isfinite(dqkv).all())
    g = ref_in.grad
    for i, name in enumerate(("dq", "dk", "dv")):
        a, r = dqkv[:, i * d:(i + 1) * d].double(), g[:, i * d:(i + 1) * d]
        # a part that vanishes (dQ at S = 1: one key, P = 1, dS = 0) is measured against the whole gradient
        scale = r.norm() if r.norm() > 1e-6 * g.norm() else g.norm()
        err = ((a - r).norm() / scale).item()
        assert err < 3e-2, (name, err)
    # the base-2 LSE of the undropped causal softmax
    q, k, _ = qkv.double().view(B, S, 3, heads, hd).unbind(2)
    s = torch.einsum("bqhd,bkhd->bhqk", q, k) / hd ** 0.5
    s = s.masked_fill(torch.ones(S, S, dtype=torch.bool, device="cuda").triu(1), float("-inf"))
    lse_ref = torch.logsumexp(s, dim=-1) * 1.4426950408889634
    assert (lse.view(B, S, heads).transpose(1, 2).double() - lse_ref).abs().max().item() < 3e-2
    # a second backward is bit-identical
    dqkv2 = K.attention_bwd(qkv, out, dout, lse, heads, seq_len=S, dropout=dropout, causal=True)
    assert torch.equal(dqkv, dqkv2)


@pytest.mark.gpu
@pytest.mark.parametrize("drop", [False, True])
@pytest.mark.parametrize("hd", K.HEAD_DIMS)
@pytest.mark.parametrize("S,t", [(300, 0), (300, 127), (300, 200), (1000, 511), (1000, 700)])
def test_later_tokens_do_not_leak(S, t, hd, drop):
    """other q / k / v in the rows after position t leave the forward rows <= t bit-identical; with a zero output gradient
    after t, the backward rows <= t (dQ, and the dK / dV that queries <= t contribute) are bit-identical too"""
    B, heads = 2, 2
    d = heads * hd
    qkv = _qkv(B, S, d, S + t + hd)
    later = (torch.arange(B * S, device="cuda") % S) > t
    other = qkv.clone()
    other[later] = (torch.randn(int(later.sum()), 3 * d, device="cuda") * 3).to(torch.bfloat16)
    dout = torch.randn(B * S, d, generator=torch.Generator().manual_seed(t)).to(torch.bfloat16).cuda()
    dout[later] = 0
    dropout = (0.1, 4321) if drop else None
    a, b = _run(qkv, heads, S, dout, dropout), _run(other, heads, S, dout, dropout)
    for x, y in zip(a, b):
        assert torch.equal(x[~later], y[~later])


@pytest.mark.gpu
@pytest.mark.parametrize("drop", [False, True])
def test_causal_dropout_mask_is_the_bidirectional_mask_on_keys_up_to_the_query(drop):
    """exact: with q = k = 0 every kept probability is 1 / (q + 1) and V (dO) one-hot in the keys (queries) of one block, so
    out (dV) is nonzero exactly where key <= query and the bidirectional site-0 mask keeps the pair"""
    B, heads, hd, S = 2, 2, 128, 256
    d, T = heads * hd, B * S
    p, seed = 0.1, 2024
    dropout = (p, seed) if drop else None
    keep = K.dropout_mask((B, heads, S, S), p, seed, K.SITE_ATTN) if drop else torch.ones(B, heads, S, S, dtype=torch.bool, device="cuda")
    allowed = keep & torch.ones(S, S, dtype=torch.bool, device="cuda").tril()
    pos = torch.arange(T, device="cuda") % S
    eye = torch.eye(128, device="cuda").to(torch.bfloat16)
    for blk in range(S // 128):
        mine = (pos // 128) == blk
        qkv = torch.zeros(T, 3 * d, dtype=torch.bfloat16, device="cuda")
        dout = torch.zeros(T, d, dtype=torch.bfloat16, device="cuda")
        for h in range(heads):
            qkv[mine, 2 * d + h * hd:2 * d + (h + 1) * hd] = eye.repeat(B, 1)   # V[key] = e_(key % 128)
            dout[mine, h * hd:(h + 1) * hd] = eye.repeat(B, 1)                   # dO[query] = e_(query % 128)
        out, _, dqkv = _run(qkv, heads, S, dout, dropout)
        o = out.view(B, S, heads, hd).permute(0, 2, 1, 3)                      # [B, H, query, key % 128]
        assert torch.equal(o != 0, allowed[..., blk * 128:(blk + 1) * 128])
        dv = dqkv[:, 2 * d:].view(B, S, heads, hd).permute(0, 2, 1, 3)         # [B, H, key, query % 128]
        assert torch.equal(dv != 0, allowed[:, :, blk * 128:(blk + 1) * 128, :].transpose(-1, -2))


@pytest.mark.gpu
def test_causal_entry_points_refuse_invalid_shapes():
    from lah_b200.ops.native import c_void_p, stream_ptr
    qkv = torch.zeros(300, 3 * 256, dtype=torch.bfloat16, device="cuda")
    lib = K._lib()
    P = c_void_p
    for tokens, S, heads, d in ((300, 7, 4, 256), (K.MAX_SEQ + 1, K.MAX_SEQ + 1, 4, 256), (300, 0, 4, 256),
                                (300, 300, 16, 256), (300, 300, 3, 256)):
        assert lib.lah_attention_fwd_causal(P(qkv.data_ptr()), P(0), P(0), tokens, S, heads, d, 0, -1, 1.0, stream_ptr()) == -2
        assert lib.lah_attention_bwd_causal(P(qkv.data_ptr()), P(0), P(0), P(0), P(0), P(0), P(0), tokens, S, heads, d, 0, -1,
                                            1.0, stream_ptr()) == -2
    with pytest.raises(AssertionError):
        K.attention_fwd(qkv, 4, seq_len=300, causal=True, key_mask=torch.zeros(1, 10, dtype=torch.int32, device="cuda"))


# ------------------------------------------------------------------------------------------------ GPU: public interface
def _backend(layer, S, d, name="causal", lr=1e-4):
    return lah_b200.ExpertBackend(name=name, expert=layer, opt=torch.optim.Adam(layer.parameters(), lr=lr, amsgrad=True),
                                  args_schema=(lah_b200.BatchTensorProto(S, d),), outputs_schema=lah_b200.BatchTensorProto(S, d),
                                  max_batch_size=4096)


def _functional_ref(layer, x, masks=None, ps=None):
    """fp32 functional forward of the causal layer with given keep masks (sites of K.dropout_mask: attention [B, H, S, S],
    dropout1 [T, d], dropout [T, ff], dropout2 [T, d]); None = no dropout"""
    B, S, d = x.shape
    T, a = B * S, layer.self_attn

    def drop(t, i):
        return t if masks is None else t * masks[i] / (1 - ps[i])

    qkv = F.linear(x.reshape(T, d), a.in_proj_weight, a.in_proj_bias)
    H = a.num_heads
    q, k, v = (t.transpose(1, 2) for t in qkv.view(B, S, 3, H, d // H).unbind(2))
    s = (q @ k.transpose(-1, -2) / (d // H) ** 0.5).masked_fill(
        torch.ones(S, S, dtype=torch.bool, device=x.device).triu(1), float("-inf"))
    o = (drop(torch.softmax(s, dim=-1), 0) @ v).transpose(1, 2).reshape(T, d)
    x1 = F.layer_norm(x.reshape(T, d) + drop(F.linear(o, a.out_proj.weight, a.out_proj.bias), 1), (d,), layer.norm1.weight,
                      layer.norm1.bias, layer.norm1.eps)
    g = drop(F.gelu(F.linear(x1, layer.linear1.weight, layer.linear1.bias)), 2)
    y = x1 + drop(F.linear(g, layer.linear2.weight, layer.linear2.bias), 3)
    return F.layer_norm(y, (d,), layer.norm2.weight, layer.norm2.bias, layer.norm2.eps).view(B, S, d)


def _masks(seed, ps, B, S, heads, d, ff):
    T = B * S
    shapes = ((B, heads, S, S), (T, d), (T, ff), (T, d))
    return [K.dropout_mask(shape, p, seed, site).float() for site, (shape, p) in enumerate(zip(shapes, ps))]


@pytest.mark.gpu
@pytest.mark.parametrize("S", [300, 512])
@pytest.mark.parametrize("d", [512, 1024, 2048])
def test_expert_backend_causal_layer(d, S):
    """dropout 0: forward, dx and the gradients against the fp64 module; three AMSGrad steps against an eager fp32 copy; the
    checkpoint loads into an eager module and optimizer whose next step agrees"""
    from lah_b200.ops import native
    from lah_b200.runtime.native_executor import NativeTransformerExecutor
    torch.manual_seed(d + S)
    layer = TransformerEncoderLayer(d, 16, dropout=0.0, causal=True).cuda()
    ref64 = copy.deepcopy(layer).double()
    ref = copy.deepcopy(layer)
    ref_opt = torch.optim.Adam(ref.parameters(), lr=1e-4, amsgrad=True)
    be = _backend(layer, S, d)
    g = torch.Generator().manual_seed(d)
    x = torch.randn(2, S, d, generator=g).cuda()
    gy = (torch.randn(2, S, d, generator=g) * 0.1).cuda()
    native.reset_launches()
    (y,) = be.forward(x)
    assert type(be._executor) is NativeTransformerExecutor and be._executor.causal and native.launches() > 0
    xr = x.double().requires_grad_(True)
    yr = ref64(xr)
    yr.backward(gy.double())
    assert rel(y, yr.detach()) < 3e-2
    launches = native.launches()
    (dx,) = be.backward(x, gy)
    assert native.launches() > launches
    assert bool(torch.isfinite(dx).all()) and rel(dx, xr.grad) < 5e-2
    st = be.opt.state_dict()["state"]
    for i, (n, p) in enumerate(ref64.named_parameters()):
        if n in GRAD_CHECKED:
            assert rel(st[i]["exp_avg"] / 0.1, p.grad) < 6e-2, n
    ref(x).backward(gy)
    ref_opt.step()
    ref_opt.zero_grad()
    for _ in range(2):
        be.backward(x, gy)
        ref(x).backward(gy)
        ref_opt.step()
        ref_opt.zero_grad()
    assert be.update_count == 3
    sd, rsd = be.state_dict(), ref.state_dict()
    assert max((sd["expert." + k] - v).abs().mean().item() for k, v in rsd.items()) < 1.5e-4
    ck = copy.deepcopy(be.checkpoint())
    fresh = TransformerEncoderLayer(d, 16, dropout=0.0, causal=True).cuda()
    fresh.load_state_dict({k[len("expert."):]: v for k, v in ck["model"].items()})
    fresh_opt = torch.optim.Adam(fresh.parameters(), lr=1e-4, amsgrad=True)
    fresh_opt.load_state_dict(ck["optimizer"])
    be.backward(x, gy)
    fresh(x).backward(gy)
    fresh_opt.step()
    sd, fsd = be.state_dict(), fresh.state_dict()
    assert max((sd["expert." + k] - v).abs().mean().item() for k, v in fsd.items()) < 5e-5
    assert float(fresh_opt.state[fresh.linear1.weight]["step"]) == 4.0


@pytest.mark.gpu
@pytest.mark.parametrize("d", [512, 1024, 2048])
def test_expert_backend_causal_layer_dropout(d):
    """dropout 0.1 at all four sites: forward, dx and the optimizer state against the fp32 functional oracle with the
    kernels' masks"""
    from lah_b200.runtime.native_executor import NativeTransformerExecutor, draw_dropout_seed
    torch.manual_seed(d)
    S, B = 512, 2
    layer = TransformerEncoderLayer(d, 16, causal=True).cuda()
    ref = copy.deepcopy(layer)
    ps = NativeTransformerExecutor._dropout_ps(layer)
    assert ps == (0.1,) * 4
    be = _backend(layer, S, d)
    g = torch.Generator().manual_seed(d + 1)
    x = torch.randn(B, S, d, generator=g).cuda()
    gy = (torch.randn(B, S, d, generator=g) * 0.1).cuda()
    torch.manual_seed(10)
    seed = draw_dropout_seed()
    torch.manual_seed(10)
    (y,) = be.forward(x)
    assert type(be._executor) is NativeTransformerExecutor
    with torch.no_grad():
        assert rel(y, _functional_ref(ref, x, _masks(seed, ps, B, S, 16, d, 2048), ps)) < 3e-2
    torch.manual_seed(20)
    seed = draw_dropout_seed()
    torch.manual_seed(20)
    (dx,) = be.backward(x, gy)
    xr = x.clone().requires_grad_(True)
    _functional_ref(ref, xr, _masks(seed, ps, B, S, 16, d, 2048), ps).backward(gy)
    assert rel(dx, xr.grad) < 5e-2
    st = be.opt.state_dict()["state"]
    for i, (n, p) in enumerate(ref.named_parameters()):
        if n in GRAD_CHECKED:
            assert rel(st[i]["exp_avg"] / 0.1, p.grad) < 6e-2, n


@pytest.mark.gpu
def test_scripted_causal_layer_bit_identical_through_expert_backend():
    torch.manual_seed(2)
    S, d = 300, 1024
    layer = TransformerEncoderLayer(d, 16, causal=True).cuda()
    twin = copy.deepcopy(layer)
    plain, scripted = _backend(layer, S, d, name="p"), _backend(torch.jit.script(twin), S, d, name="s")
    x = torch.randn(4, S, d, device="cuda")
    gy = torch.randn(4, S, d, device="cuda") * 0.1
    outs = []
    for be in (plain, scripted):
        torch.manual_seed(11)
        (y,) = be.forward(x)
        torch.manual_seed(12)
        (dx,) = be.backward(x, gy)
        outs.append((y, dx, be.state_dict()))
        assert be._executor is not None and be._executor.causal
    (y0, dx0, sd0), (y1, dx1, sd1) = outs
    assert torch.equal(y0, y1) and torch.equal(dx0, dx1)
    assert all(torch.equal(sd0[k], sd1[k]) for k in sd0)


@pytest.mark.gpu
def test_server_round_trip_causal_layer():
    from lah_b200.runtime.native_executor import NativeTransformerExecutor
    torch.manual_seed(1)
    S, d = 300, 1024
    layer = TransformerEncoderLayer(d, 16, causal=True).cuda()
    be = _backend(layer, S, d, name="causal300")
    srv = lah_b200.TesseractServer(None, {"causal300": be}, port=0, conn_handler_processes=1, device="cuda")
    srv.run_in_background()
    try:
        remote = lah_b200.RemoteExpert("causal300", "127.0.0.1", srv.port, timeout=120)
        x = torch.randn(2, S, d, requires_grad=True)
        y = remote(x)
        assert y.shape == x.shape and bool(torch.isfinite(y).all())
        y[:, :100].sum().backward()
        assert x.grad is not None and bool(torch.isfinite(x.grad).all())
        assert int(torch.count_nonzero(x.grad[:, 100:])) == 0   # later positions do not reach earlier outputs
        assert be.update_count == 1 and type(be._executor) is NativeTransformerExecutor
    finally:
        srv.shutdown()


@pytest.mark.gpu
@pytest.mark.parametrize("d", [512, 1024, 2048])
def test_native_transformer_layer_causal(d):
    from lah_b200.models.transformer_native import NativeTransformerLayer
    torch.manual_seed(d)
    layer = TransformerEncoderLayer(d, 16, causal=True).cuda().eval()
    x = torch.randn(3, 300, d, device="cuda")
    with torch.no_grad():
        ref = layer.double()(x.double())
        native = NativeTransformerLayer(layer)
        out = native(x)
        bidirectional = TransformerEncoderLayer(d, 16).cuda().eval().double()
        bidirectional.load_state_dict(layer.state_dict())
        assert native.causal and rel(out, ref) < 3e-2 and rel(out, bidirectional(x.double())) > 5e-2
