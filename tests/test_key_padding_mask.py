"""Key padding masks (torch's src_key_padding_mask) in the sm_90a attention kernels and the transformer expert: the masked
oracle against torch in fp64 and the mask packing (CPU); on the GPU the masked kernels against the oracle, their exact
properties, and torch.nn.TransformerEncoderLayer with a mask behind ExpertBackend and a server."""
import copy

import pytest
import torch
import torch.nn.functional as F

import lah_b200  # noqa
from lah_b200.ops import kernels as K

SEQS = [1, 17, 127, 128, 129, 300, 512, 1000, 2048]
GRAD_CHECKED = ("self_attn.in_proj_weight", "linear1.weight", "linear2.weight", "self_attn.out_proj.weight",
                "self_attn.in_proj_bias", "self_attn.out_proj.bias", "linear2.bias", "linear1.bias", "norm1.weight")


def rel(a, b):
    return ((a.float() - b.float()).norm() / (b.float().norm() + 1e-12)).item()


def mask_families(S, seed=0):
    """bool [8, S], True = padding: right padding to lengths 0, 1, S - 1 and S; left padding; 30 % random holes; keys
    128-255 masked (the middle block from S = 384 on, else the second half); keys 0-127 masked"""
    g = torch.Generator().manual_seed(seed)
    pos = torch.arange(S)
    rows = [pos >= length for length in (0, 1, max(S - 1, 0), S)]
    rows.append(pos < S // 3)
    rows.append(torch.rand(S, generator=g) < 0.3)
    rows.append((pos >= 128) & (pos < 256) if S >= 384 else pos >= S // 2)
    rows.append(pos < 128)
    return torch.stack(rows)


# ------------------------------------------------------------------------------------------------ CPU
@pytest.mark.parametrize("S", [5, 37])
def test_masked_attention_ref_matches_torch_mha_fp64(S):
    """attention_ref with a mask, inside in_proj / out_proj, equals nn.MultiheadAttention (training mode) in fp64: output,
    the input gradient and the in_proj weight gradient; a fully masked sequence gives out_proj.bias and zero gradient"""
    torch.manual_seed(S)
    d, heads = 16, 2
    mha = torch.nn.MultiheadAttention(d, heads, batch_first=True, dtype=torch.float64)
    pad = mask_families(S, seed=S)
    B = pad.shape[0]
    x = torch.randn(B, S, d, dtype=torch.float64, requires_grad=True)
    ref, _ = mha(x, x, x, key_padding_mask=pad, need_weights=False)
    g = torch.randn_like(ref)
    dx_ref, dw_ref = torch.autograd.grad(ref, (x, mha.in_proj_weight), g)
    x2 = x.detach().clone().requires_grad_(True)
    qkv = F.linear(x2.reshape(B * S, d), mha.in_proj_weight, mha.in_proj_bias)
    out = F.linear(K.attention_ref(qkv, heads, seq_len=S, key_mask=pad), mha.out_proj.weight, mha.out_proj.bias).view(B, S, d)
    dx, dw = torch.autograd.grad(out, (x2, mha.in_proj_weight), g)
    assert bool(torch.isfinite(out).all()) and bool(torch.isfinite(dx).all())
    for a, b in ((out, ref), (dx, dx_ref), (dw, dw_ref)):
        assert (a - b).abs().max().item() < 1e-12
    assert torch.equal(out[0], mha.out_proj.bias.detach().expand(S, d))   # length 0: attention output 0
    assert int(torch.count_nonzero(dx[0])) == 0


def test_masked_attention_ref_matches_torch_encoder_layer_fp64():
    """the whole encoder layer (training mode, dropout 0) from attention_ref, against torch's layer with the mask"""
    torch.manual_seed(3)
    d, heads, S = 32, 4, 45
    layer = torch.nn.TransformerEncoderLayer(d, heads, 64, dropout=0.0, batch_first=True, dtype=torch.float64)
    pad = mask_families(S, seed=1)
    B = pad.shape[0]
    x = torch.randn(B, S, d, dtype=torch.float64)
    ref = layer(x, src_key_padding_mask=pad)
    a = layer.self_attn
    att = K.attention_ref(F.linear(x.reshape(B * S, d), a.in_proj_weight, a.in_proj_bias), heads, seq_len=S, key_mask=pad)
    h = layer.norm1(x + F.linear(att, a.out_proj.weight, a.out_proj.bias).view(B, S, d))
    y = layer.norm2(h + layer.linear2(F.relu(layer.linear1(h))))
    assert (y - ref).abs().max().item() < 1e-12


@pytest.mark.parametrize("S", [1, 17, 31, 32, 33, 100, 128, 300])
def test_pack_key_mask_ref(S):
    pad = mask_families(S, seed=S)
    words = K.pack_key_mask_ref(pad).long() & 0xFFFFFFFF
    assert words.shape == (pad.shape[0], (S + 31) // 32)
    for b in range(pad.shape[0]):
        for k in range(words.shape[1] * 32):
            bit = (int(words[b, k // 32]) >> (k % 32)) & 1
            assert bit == (k < S and not bool(pad[b, k])), (b, k)


# ------------------------------------------------------------------------------------------------ GPU: kernels
def _qkv(batch, S, d, seed, scale=1.2):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(batch * S, 3 * d, generator=g) * scale).to(torch.bfloat16).cuda()


def _masked_ref(qkv, heads, S, pad, drop_mask=None, p=0.0):
    """fp32 oracle with an optional site-0 keep mask [B, H, S, S]"""
    if drop_mask is None:
        return K.attention_ref(qkv, heads, seq_len=S, key_mask=pad)
    T, d = qkv.shape[0], qkv.shape[1] // 3
    q, k, v = (t.transpose(1, 2) for t in qkv.float().view(T // S, S, 3, heads, d // heads).unbind(2))
    s = (q @ k.transpose(-1, -2) / (d // heads) ** 0.5).masked_fill(pad.cuda().view(T // S, 1, 1, S), float("-inf"))
    att = torch.softmax(s, dim=-1).nan_to_num(0.0) * drop_mask / (1 - p)
    return (att @ v).transpose(1, 2).reshape(T, d)


def _grad_errs(dqkv, ref, d):
    errs = {}
    for i, name in enumerate(("dq", "dk", "dv")):
        a, b = dqkv[:, i * d:(i + 1) * d].float(), ref[:, i * d:(i + 1) * d].float()
        scale = b.norm() if b.norm() > 0 else ref.float().norm()
        errs[name] = ((a - b).norm() / scale).item()
    return errs


def _run(qkv, heads, S, dout, key_mask=None, dropout=None):
    T = qkv.shape[0]
    lse = torch.empty(T, heads, device="cuda")
    out = K.attention_fwd(qkv, heads, lse=lse, seq_len=S, dropout=dropout, key_mask=key_mask)
    dqkv = K.attention_bwd(qkv, out, dout, lse, heads, seq_len=S, dropout=dropout, key_mask=key_mask)
    return out, lse, dqkv


@pytest.mark.gpu
@pytest.mark.parametrize("S", [1, 17, 31, 32, 33, 100, 128, 300, 2048])
def test_pack_key_mask_matches_ref(S):
    pad = mask_families(S, seed=S + 1)
    assert torch.equal(K.pack_key_mask(pad.cuda()).cpu(), K.pack_key_mask_ref(pad))


@pytest.mark.gpu
@pytest.mark.parametrize("drop", [False, True])
@pytest.mark.parametrize("hd", K.HEAD_DIMS)
@pytest.mark.parametrize("S", SEQS)
def test_masked_attention_matches_oracle(S, hd, drop):
    heads = 2
    d = heads * hd
    pad = mask_families(S, seed=S + hd)
    B, T = pad.shape[0], pad.shape[0] * S
    qkv = _qkv(B, S, d, S * 7 + hd)
    dout = (torch.randn(T, d, generator=torch.Generator().manual_seed(S + 1)) * 0.5).to(torch.bfloat16).cuda()
    p, seed = 0.1, 99 + S
    dropout = (p, seed) if drop else None
    out, lse, dqkv = _run(qkv, heads, S, dout, K.pack_key_mask(pad.cuda()), dropout)
    torch.cuda.synchronize()
    drop_mask = K.dropout_mask((B, heads, S, S), p, seed, K.SITE_ATTN).float() if drop else None
    ref_in = qkv.float().requires_grad_(True)
    ref = _masked_ref(ref_in, heads, S, pad, drop_mask, p)
    ref.backward(dout.float())
    assert rel(out, ref.detach()) < 2e-2
    assert bool(torch.isfinite(dqkv).all())
    errs = _grad_errs(dqkv, ref_in.grad, d)
    assert all(v < 3e-2 for v in errs.values()), errs
    # the LSE of the undropped masked softmax; +inf for a sequence without a valid key
    q, k, _ = qkv.float().view(B, S, 3, heads, hd).unbind(2)
    s2 = torch.einsum("bqhd,bkhd->bhqk", q, k) / hd ** 0.5 * 1.4426950408889634
    s2 = s2.masked_fill(pad.cuda().view(B, 1, 1, S), float("-inf"))
    lse_ref = torch.logsumexp(s2 * 0.6931471805599453, dim=-1) / 0.6931471805599453
    lse_k = lse.view(B, S, heads).transpose(1, 2)
    full = pad.all(dim=1).cuda()
    assert bool((lse_k[full] == float("inf")).all())
    assert (lse_k[~full] - lse_ref[~full]).abs().max().item() < 3e-2
    # exact zeros: every output and gradient of a fully masked sequence, the dK / dV rows of every masked key
    rows = full.repeat_interleave(S)
    assert int(torch.count_nonzero(out[rows])) == 0 and int(torch.count_nonzero(dqkv[rows])) == 0
    masked = pad.cuda().reshape(T)
    assert int(torch.count_nonzero(dqkv[masked, d:])) == 0


@pytest.mark.gpu
@pytest.mark.parametrize("drop", [False, True])
@pytest.mark.parametrize("hd", K.HEAD_DIMS)
@pytest.mark.parametrize("S", [129, 512, 1000])
def test_all_false_mask_bit_identical_to_unmasked(S, hd, drop):
    heads, B = 4, 3
    d = heads * hd
    qkv = _qkv(B, S, d, S + hd)
    dout = torch.randn(B * S, d, generator=torch.Generator().manual_seed(5)).to(torch.bfloat16).cuda()
    dropout = (0.1, 1234) if drop else None
    a = _run(qkv, heads, S, dout, None, dropout)
    b = _run(qkv, heads, S, dout, K.pack_key_mask(torch.zeros(B, S, dtype=torch.bool, device="cuda")), dropout)
    for x, y in zip(a, b):
        assert torch.equal(x, y)


@pytest.mark.gpu
@pytest.mark.parametrize("hd", K.HEAD_DIMS)
@pytest.mark.parametrize("S", [100, 300, 1000])
def test_masked_key_values_do_not_matter(S, hd):
    """other finite K / V values in masked key rows leave out, lse and dqkv bit-identical (Q of a padded position is a real
    query and is not replaced)"""
    heads = 2
    d = heads * hd
    pad = mask_families(S, seed=7)
    B, T = pad.shape[0], pad.shape[0] * S
    qkv = _qkv(B, S, d, S)
    dout = torch.randn(T, d, generator=torch.Generator().manual_seed(6)).to(torch.bfloat16).cuda()
    km = K.pack_key_mask(pad.cuda())
    a = _run(qkv, heads, S, dout, km, (0.1, 77))
    other = qkv.clone()
    masked = pad.cuda().reshape(T)
    other[masked, d:] = (torch.randn(int(masked.sum()), 2 * d, device="cuda") * 30).to(torch.bfloat16)
    b = _run(other, heads, S, dout, km, (0.1, 77))
    for x, y in zip(a, b):
        assert torch.equal(x, y)


# ------------------------------------------------------------------------------------------------ GPU: public interface
def _backend(layer, S, d, name="kpm", kwargs_proto=None, **kw):
    kw.setdefault("outputs_schema", lah_b200.BatchTensorProto(S, d))   # no dummy run of a CUDA module on CPU tensors
    return lah_b200.ExpertBackend(
        name=name, expert=layer, opt=torch.optim.Adam(layer.parameters(), lr=1e-4, amsgrad=True),
        args_schema=(lah_b200.BatchTensorProto(S, d),),
        kwargs_schema={"src_key_padding_mask": kwargs_proto or lah_b200.BatchTensorProto(S, dtype=torch.bool)},
        max_batch_size=4096, **kw)


def _layer_input(batch_first, B, S, d, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, S, d, generator=g)
    gy = torch.randn(B, S, d, generator=g) * 0.1
    if not batch_first:
        x, gy = x.transpose(0, 1).contiguous(), gy.transpose(0, 1).contiguous()
    pad = mask_families(S, seed=seed)[[0, 2, 4, 5]]   # fully masked, one padded key, left padding, holes
    return x.cuda(), gy.cuda(), pad.cuda()


@pytest.mark.gpu
@pytest.mark.parametrize("batch_first,norm_first,act,d", [(True, False, "relu", 1024), (False, True, "gelu", 512),
                                                          (True, True, "gelu", 2048), (False, False, "relu", 1024),
                                                          (True, False, "gelu", 512)])
def test_expert_backend_masked_encoder_layer(batch_first, norm_first, act, d):
    """output, dx and the optimizer step of torch's layer with a key padding mask through ExpertBackend against the fp64
    module in training mode (dropout 0); eval mode gives the same output"""
    from lah_b200.ops import native
    from lah_b200.runtime.native_executor import NativeTransformerExecutor
    torch.manual_seed(d)
    S = 200
    layer = torch.nn.TransformerEncoderLayer(d, 16, 2 * d, dropout=0.0, activation=act, batch_first=batch_first,
                                             norm_first=norm_first).cuda()
    ref = copy.deepcopy(layer).double()
    be = _backend(layer, S, d)
    x, gy, pad = _layer_input(batch_first, 4, S, d, seed=d)
    native.reset_launches()
    (y,) = be.forward(x, pad)
    assert type(be._executor) is NativeTransformerExecutor and native.launches() > 0
    xr = x.double().requires_grad_(True)
    yr = ref(xr, src_key_padding_mask=pad)
    yr.backward(gy.double())
    assert bool(torch.isfinite(y).all()) and rel(y, yr.detach()) < 3e-2
    launches = native.launches()
    dx, dmask = be.backward(x, pad, gy)
    assert native.launches() > launches and be.update_count == 1
    assert dmask.dtype == torch.bool and dmask.shape == pad.shape and not bool(dmask.any())
    assert bool(torch.isfinite(dx).all()) and rel(dx, xr.grad) < 5e-2
    st = be.opt.state_dict()["state"]
    for i, (n, p) in enumerate(ref.named_parameters()):
        if n in GRAD_CHECKED:
            assert rel(st[i]["exp_avg"] / 0.1, p.grad) < 6e-2, n
    ref_opt = torch.optim.Adam(ref.parameters(), lr=1e-4, amsgrad=True)
    ref_opt.step()
    sd, rsd = be.state_dict(), ref.state_dict()
    assert all(bool(torch.isfinite(v).all()) for v in sd.values())
    assert max((sd["expert." + k] - v).abs().mean().item() for k, v in rsd.items()) < 1.5e-4
    layer.eval()   # torch's eval fast path would give NaN for the fully masked sequence; the executor does not
    (y_eval,) = be.forward(x, pad)
    assert bool(torch.isfinite(y_eval).all()) and rel(y_eval, ref(x.double(), src_key_padding_mask=pad)) < 3e-2


@pytest.mark.gpu
def test_scripted_masked_layer_bit_identical():
    torch.manual_seed(2)
    S, d = 300, 1024
    layer = torch.nn.TransformerEncoderLayer(d, 16, 2048, dropout=0.1, batch_first=True).cuda()
    twin = copy.deepcopy(layer)
    plain, scripted = _backend(layer, S, d, name="p"), _backend(torch.jit.script(twin), S, d, name="s")
    x, gy, pad = _layer_input(True, 4, S, d, seed=3)
    outs = []
    for be in (plain, scripted):
        torch.manual_seed(11)
        (y,) = be.forward(x, pad)
        torch.manual_seed(12)
        dx, _ = be.backward(x, pad, gy)
        outs.append((y, dx, be.state_dict()))
        assert be._executor is not None
    (y0, dx0, sd0), (y1, dx1, sd1) = outs
    assert torch.equal(y0, y1) and torch.equal(dx0, dx1)
    assert all(torch.equal(sd0[k], sd1[k]) for k in sd0)


@pytest.mark.gpu
def test_server_round_trip_with_key_padding_mask():
    from lah_b200.runtime.native_executor import NativeTransformerExecutor
    torch.manual_seed(1)
    S, d = 200, 1024
    layer = torch.nn.TransformerEncoderLayer(d, 16, batch_first=True).cuda()
    be = _backend(layer, S, d, name="kpm200")
    srv = lah_b200.TesseractServer(None, {"kpm200": be}, port=0, conn_handler_processes=1, device="cuda")
    srv.run_in_background()
    try:
        remote = lah_b200.RemoteExpert("kpm200", "127.0.0.1", srv.port, timeout=120)
        x = torch.randn(2, S, d, requires_grad=True)
        pad = torch.zeros(2, S, dtype=torch.bool)
        pad[0, 150:] = True
        y = remote(x, src_key_padding_mask=pad)
        assert y.shape == x.shape and bool(torch.isfinite(y).all())
        y.sum().backward()
        assert x.grad is not None and x.grad.shape == x.shape and bool(torch.isfinite(x.grad).all())
        assert be.update_count == 1 and type(be._executor) is NativeTransformerExecutor
    finally:
        srv.shutdown()


@pytest.mark.gpu
def test_other_masks_and_layers_stay_on_the_module():
    """a float mask, a src_mask keyword, this package's layer and a mask of the wrong shape run on the module"""
    from lah_b200.models.layers import TransformerEncoderLayer
    from lah_b200.ops import native
    S, d = 64, 512
    x = torch.randn(2, S, d, device="cuda")
    layer = torch.nn.TransformerEncoderLayer(d, 16, 1024, dropout=0.0, batch_first=True).cuda()
    fbe = _backend(layer, S, d, kwargs_proto=lah_b200.BatchTensorProto(S, dtype=torch.float32))
    native.reset_launches()
    fbe.forward(x, torch.zeros(2, S, device="cuda"))
    assert native.launches() == 0 and fbe.native_executor((x,)) is None
    sbe = lah_b200.ExpertBackend(name="sm", expert=layer, opt=torch.optim.Adam(layer.parameters()),
                                 args_schema=(lah_b200.BatchTensorProto(S, d),),
                                 kwargs_schema={"src_mask": lah_b200.BatchTensorProto(S, dtype=torch.bool)},
                                 outputs_schema=lah_b200.BatchTensorProto(S, d), max_batch_size=8)
    assert sbe.native_executor((x,)) is None
    own = TransformerEncoderLayer(d, 16).cuda()
    obe = _backend(own, S, d, name="own", outputs_schema=lah_b200.BatchTensorProto(S, d))
    assert obe.native_executor((x,)) is None
    ex = _backend(layer, S, d, name="shape").native_executor((x,))
    assert ex is not None and ex.accepts(x, torch.zeros(2, S, dtype=torch.bool, device="cuda"))
    assert not ex.accepts(x, torch.zeros(2, S + 1, dtype=torch.bool, device="cuda"))
    assert not ex.accepts(x, torch.zeros(3, S, dtype=torch.bool, device="cuda"))
    assert not ex.accepts(x, torch.zeros(2, S, device="cuda"))
    assert not ex.accepts(x, torch.zeros(2, S, dtype=torch.bool))
