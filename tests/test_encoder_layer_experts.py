"""torch.nn.TransformerEncoderLayer (ReLU or erf GELU, post- or pre-LN, batch- or sequence-first) and torch.jit.script-ed
experts on the sm_90a executors: which modules ``encoder_layer_spec`` / ``ffn_spec`` accept, the two kernels the new graphs
need (LayerNorm backward with a residual gradient, ReLU + dropout) and their fp32 oracles, and on top of them training
through ExpertBackend, scripted == unscripted bit for bit, a server round trip, checkpoints and the refused variants."""
import copy

import pytest
import torch
import torch.nn.functional as F
from torch import nn

import lah_b200  # noqa
from lah_b200.models.layers import FeedforwardBlock, TransformerEncoderLayer
from lah_b200.ops import kernels as K
from lah_b200.runtime.native_executor import EncoderLayerSpec, FFNSpec, encoder_layer_spec, ffn_spec

GRAD_CHECKED = ("self_attn.in_proj_weight", "linear1.weight", "linear2.weight", "self_attn.out_proj.weight",
                "self_attn.in_proj_bias", "self_attn.out_proj.bias", "linear2.bias", "linear1.bias", "norm1.weight")
ACTIVATIONS = {"relu": "relu", "gelu": "gelu", "F.relu": F.relu, "nn.ReLU": nn.ReLU(), "nn.GELU": nn.GELU()}


class LookalikeEncoderLayer(nn.Module):
    """the submodules and attributes of torch's encoder layer under another class: its forward is not torch's, so it must
    stay on the module"""

    def __init__(self, d, nhead):
        super().__init__()
        self.self_attn = nn.MultiheadAttention(d, nhead, batch_first=True)
        self.linear1, self.linear2 = nn.Linear(d, 2 * d), nn.Linear(2 * d, d)
        self.norm1, self.norm2 = nn.LayerNorm(d), nn.LayerNorm(d)
        self.dropout, self.dropout1, self.dropout2 = nn.Dropout(0.1), nn.Dropout(0.1), nn.Dropout(0.1)
        self.activation = nn.ReLU()
        self.norm_first = False
        self.activation_relu_or_gelu = 1

    def forward(self, x):
        return self.norm2(x + self.linear2(self.activation(self.linear1(self.norm1(x)))))


def rel(a, b):
    return ((a.float() - b.float()).norm() / (b.float().norm() + 1e-12)).item()


# ------------------------------------------------------------------------------------------------ CPU: module specs
@pytest.mark.parametrize("scripted", [False, True])
@pytest.mark.parametrize("act", list(ACTIVATIONS))
@pytest.mark.parametrize("batch_first", [True, False])
@pytest.mark.parametrize("norm_first", [False, True])
def test_torch_encoder_layer_spec(norm_first, batch_first, act, scripted):
    layer = nn.TransformerEncoderLayer(64, 4, dim_feedforward=128, dropout=0.1, activation=ACTIVATIONS[act],
                                       batch_first=batch_first, norm_first=norm_first)
    layer.self_attn.dropout = 0.25
    layer.dropout2.p = 0.5
    module = torch.jit.script(layer) if scripted else layer
    assert encoder_layer_spec(module) == EncoderLayerSpec(64, 4, 128, norm_first, "relu" if "relu" in act.lower() else "gelu",
                                                          batch_first, (0.25, 0.1, 0.1, 0.5))
    assert ffn_spec(module) is None


@pytest.mark.parametrize("scripted", [False, True])
def test_own_layer_specs(scripted):
    layer, ffn = TransformerEncoderLayer(256, 16, dim_feedforward=512, dropout=0.2), FeedforwardBlock(64)
    if scripted:
        layer, ffn = torch.jit.script(layer), torch.jit.script(ffn)
    assert encoder_layer_spec(layer) == EncoderLayerSpec(256, 16, 512, False, "gelu", True, (0.2,) * 4)
    assert ffn_spec(ffn) == FFNSpec(64, 256)
    assert encoder_layer_spec(ffn) is None and ffn_spec(layer) is None


def _refused():
    def torch_layer(**kw):
        kw = dict(dict(dim_feedforward=128), **kw)
        return nn.TransformerEncoderLayer(64, kw.pop("nhead", 4), **kw)

    kdim = torch_layer()
    kdim.self_attn = nn.MultiheadAttention(64, 4, kdim=32, vdim=32)
    bias_kv = torch_layer()
    bias_kv.self_attn = nn.MultiheadAttention(64, 4, add_bias_kv=True)
    zero_attn = torch_layer()
    zero_attn.self_attn = nn.MultiheadAttention(64, 4, add_zero_attn=True)
    no_affine = torch_layer()
    no_affine.norm2 = nn.LayerNorm(64, elementwise_affine=False)
    return {"tanh GELU": torch_layer(activation=nn.GELU(approximate="tanh")), "SiLU": torch_layer(activation=nn.SiLU()),
            "eps 1e-6": torch_layer(layer_norm_eps=1e-6), "bias=False": torch_layer(bias=False), "kdim": kdim,
            "add_bias_kv": bias_kv, "add_zero_attn": zero_attn, "no LayerNorm affine": no_affine,
            "lookalike": LookalikeEncoderLayer(64, 4)}


NOT_SCRIPTABLE = ("kdim", "bias=False", "no LayerNorm affine")   # torch's forward reads a bias or weight that is None


@pytest.mark.parametrize("scripted", [False, True])
@pytest.mark.parametrize("name", list(_refused()))
def test_refused_module_specs(name, scripted):
    module = _refused()[name]
    if scripted:
        if name in NOT_SCRIPTABLE:
            pytest.skip("torch.jit.script refuses this module")
        module = torch.jit.script(module)
    assert encoder_layer_spec(module) is None and ffn_spec(module) is None


def test_head_dim_48_is_refused_by_supports_not_by_spec():
    """the spec describes the layer; head dims are the executor's limit (supports)"""
    spec = encoder_layer_spec(nn.TransformerEncoderLayer(768, 16))
    assert spec is not None and spec.d // spec.heads == 48 and 48 not in K.HEAD_DIMS


def test_traced_module_is_refused():
    layer = nn.TransformerEncoderLayer(64, 4, dim_feedforward=128, batch_first=True).eval()
    with torch.no_grad():
        traced = torch.jit.trace(layer, torch.randn(2, 8, 64), check_trace=False)
    assert encoder_layer_spec(traced) is None


# ------------------------------------------------------------------------------------------------ CPU: fp32 oracles
@pytest.mark.parametrize("relu", [False, True])
@pytest.mark.parametrize("with_res", [False, True])
def test_ln_relu_bwd_ref_matches_autograd(relu, with_res):
    g = torch.Generator().manual_seed(3)
    rows, C = 37, 48
    h, da, dres = (torch.randn(rows, C, generator=g, dtype=torch.float64) for _ in range(3))
    gamma, beta = 1 + 0.1 * torch.randn(C, generator=g, dtype=torch.float64), 0.1 * torch.randn(C, generator=g, dtype=torch.float64)
    hh, gg, bb = (t.clone().requires_grad_(True) for t in (h, gamma, beta))
    y = F.layer_norm(hh, (C,), gg, bb, 1e-5)
    (F.relu(y) if relu else y).backward(da)
    dh, dgamma, dbeta, dbias = K.ln_relu_bwd_ref(da, h, gamma, beta, relu=relu, dres=dres if with_res else None)
    want = hh.grad + (dres if with_res else 0)
    for a, b in ((dh, want), (dgamma, gg.grad), (dbeta, bb.grad), (dbias, want.sum(0))):
        assert torch.allclose(a.double(), b, rtol=1e-5, atol=1e-5)


def test_relu_dropout_refs_match_autograd():
    g = torch.Generator().manual_seed(4)
    f, dg = torch.randn(32, 48, generator=g, dtype=torch.float64), torch.randn(32, 48, generator=g, dtype=torch.float64)
    mask, p = torch.rand(32, 48, generator=g) > 0.3, 0.3
    ff = f.clone().requires_grad_(True)
    (mask * F.relu(ff) / (1 - p)).backward(dg)
    assert torch.allclose(K.relu_dropout_ref(f, mask, p).double(), (mask * F.relu(f) / (1 - p)), rtol=1e-6, atol=1e-6)
    assert torch.allclose(K.relu_dropout_bwd_ref(dg, f, mask, p).double(), ff.grad, rtol=1e-6, atol=1e-6)


# ------------------------------------------------------------------------------------------------ GPU: kernels
@pytest.mark.gpu
@pytest.mark.parametrize("tile_rows", [16, 128])
@pytest.mark.parametrize("C", [512, 1024, 2048, 4096])
def test_ln_bwd_with_residual_gradient(C, tile_rows):
    g = torch.Generator().manual_seed(C + tile_rows)
    rows = 300
    h = (torch.randn(rows, C, generator=g) * 2 + 0.5).to(torch.bfloat16).cuda()
    da, dres = (torch.randn(rows, C, generator=g).to(torch.bfloat16).cuda() for _ in range(2))
    gamma = (1 + 0.2 * torch.randn(C, generator=g)).cuda()
    beta = (0.2 * torch.randn(C, generator=g)).cuda()
    mean, rstd = torch.empty(rows, device="cuda"), torch.empty(rows, device="cuda")
    K.ln_relu_fwd(h, gamma, beta, None, out=torch.empty_like(h), mean=mean, rstd=rstd, relu=False, tile_rows=tile_rows)
    runs = []
    for _ in range(2):
        dh = torch.empty_like(h)
        sums = [torch.zeros(C, device="cuda") for _ in range(3)]
        K.ln_relu_bwd(da, h, mean, rstd, gamma, beta, None, dh=dh, dgamma=sums[0], dbeta=sums[1], dbias=sums[2], relu=False,
                      tile_rows=tile_rows, dres=dres)
        runs.append([dh] + sums)
    torch.cuda.synchronize()
    ref = K.ln_relu_bwd_ref(da, h, gamma, beta, relu=False, dres=dres)
    for name, a, b in zip(("dh", "dgamma", "dbeta", "dbias"), runs[0], ref):
        assert rel(a, b) < 1e-2, name
    for a, b in zip(*runs):
        assert torch.equal(a.view(torch.uint8) if a.dtype == torch.bfloat16 else a.view(torch.int32),
                           b.view(torch.uint8) if b.dtype == torch.bfloat16 else b.view(torch.int32))


@pytest.mark.gpu
@pytest.mark.parametrize("p", [0.1, 0.5])
def test_relu_dropout_kernels(p):
    rows, cols, seed = 384, 1024, 1234
    g = torch.Generator().manual_seed(5)
    f, dg = (torch.randn(rows, cols, generator=g).to(torch.bfloat16).cuda() for _ in range(2))
    mask = K.dropout_mask((rows, cols), p, seed, K.SITE_FF)
    out = K.relu_dropout(f, p, seed, K.SITE_FF)
    dgrad = K.relu_dropout_bwd(dg, f, p, seed, K.SITE_FF)
    torch.cuda.synchronize()
    for a, b in ((out, K.relu_dropout_ref(f, mask, p)), (dgrad, K.relu_dropout_bwd_ref(dg, f, mask, p))):
        assert ((a.float() - b).abs() <= b.abs() * 2 ** -8 + 1e-30).all()
        assert torch.equal(a == 0, b == 0)


@pytest.mark.gpu
def test_relu_dropout_p0_is_relu():
    g = torch.Generator().manual_seed(6)
    f, dg = (torch.randn(256, 512, generator=g).to(torch.bfloat16).cuda() for _ in range(2))
    out = K.relu_dropout(f, 0.0, 77, K.SITE_FF)
    dgrad = K.relu_dropout_bwd(dg, f, 0.0, 77, K.SITE_FF)
    torch.cuda.synchronize()
    assert torch.equal(out.view(torch.uint8), torch.relu(f).view(torch.uint8))
    assert torch.equal(dgrad.view(torch.uint8), torch.ops.aten.threshold_backward(dg, f, 0).view(torch.uint8))


# ------------------------------------------------------------------------------------------------ GPU: ExpertBackend
def encoder_layer_ref(layer, x, masks=None):
    """fp32 functional forward of an encoder layer ``encoder_layer_spec`` accepts, with given keep masks (site order of
    kernels.dropout_mask, batch-major token rows: attention [B, H, S, S], dropout1 [T, d], dropout [T, ff],
    dropout2 [T, d]); None = no dropout"""
    spec = encoder_layer_spec(layer)
    xb = x if spec.batch_first else x.transpose(0, 1)
    B, S, d = xb.shape
    T, H, a, ps = B * S, spec.heads, layer.self_attn, spec.ps
    act = F.relu if spec.activation == "relu" else F.gelu

    def drop(t, i):
        return t if masks is None else t * masks[i] / (1 - ps[i])

    def ln(t, norm):
        return F.layer_norm(t, (d,), norm.weight, norm.bias, 1e-5)

    def attn_block(t):
        qkv = F.linear(t, a.in_proj_weight, a.in_proj_bias)
        q, k, v = (u.transpose(1, 2) for u in qkv.view(B, S, 3, H, d // H).unbind(2))
        att = drop(torch.softmax(q @ k.transpose(-1, -2) / (d // H) ** 0.5, dim=-1), 0)
        return drop(F.linear((att @ v).transpose(1, 2).reshape(T, d), a.out_proj.weight, a.out_proj.bias), 1)

    def ff_block(t):
        return drop(F.linear(drop(act(F.linear(t, layer.linear1.weight, layer.linear1.bias)), 2), layer.linear2.weight,
                             layer.linear2.bias), 3)

    x0 = xb.reshape(T, d)
    if spec.norm_first:
        h = x0 + attn_block(ln(x0, layer.norm1))
        y = h + ff_block(ln(h, layer.norm2))
    else:
        h = ln(x0 + attn_block(x0), layer.norm1)
        y = ln(h + ff_block(h), layer.norm2)
    y = y.view(B, S, d)
    return y if spec.batch_first else y.transpose(0, 1)


def _masks(seed, spec, batch, S):
    T = batch * S
    shapes = ((batch, spec.heads, S, S), (T, spec.d), (T, spec.ff), (T, spec.d))
    return [K.dropout_mask(shape, p, seed, site).float() for site, (shape, p) in enumerate(zip(shapes, spec.ps))]


def _backend(module, shape, name="t", **kw):
    opt = torch.optim.Adam(module.parameters(), lr=1e-4, amsgrad=True)
    return lah_b200.ExpertBackend(name=name, expert=module, opt=opt, args_schema=(lah_b200.BatchTensorProto(*shape[1:]),),
                                  outputs_schema=lah_b200.BatchTensorProto(*shape[1:]), max_batch_size=8, **kw)


CASES = [   # (d, norm_first, activation, batch_first, S): every value of every axis appears
    (512, False, "relu", False, 300),
    (512, True, "relu", True, 512),
    (1024, True, "gelu", False, 300),
    (1024, True, "relu", False, 512),
    (2048, False, "gelu", True, 512),
    (2048, True, "relu", False, 300),
]


@pytest.mark.gpu
@pytest.mark.parametrize("d,norm_first,activation,batch_first,S", CASES)
def test_expert_backend_trains_torch_encoder_layer(d, norm_first, activation, batch_first, S):
    """nn.TransformerEncoderLayer(d, 16, dropout 0.1) through ExpertBackend: forward, dx, weight gradients and three AMSGrad
    steps against the fp32 functional oracle with the same masks; eval mode against the module itself"""
    from lah_b200.ops import native
    from lah_b200.runtime.native_executor import NativeTransformerExecutor, draw_dropout_seed
    torch.manual_seed(4)
    layer = nn.TransformerEncoderLayer(d, 16, dropout=0.1, activation=activation, batch_first=batch_first,
                                       norm_first=norm_first).cuda()
    spec = encoder_layer_spec(layer)
    ref = copy.deepcopy(layer)
    ref_opt = torch.optim.Adam(ref.parameters(), lr=1e-4, amsgrad=True)
    shape = (2, S, d) if batch_first else (S, 2, d)
    be = _backend(layer, shape)
    x = torch.randn(*shape, device="cuda")
    g = torch.randn(*shape, device="cuda") * 0.1
    native.reset_launches()
    torch.manual_seed(10)
    seed = draw_dropout_seed()
    torch.manual_seed(10)
    (y,) = be.forward(x)
    assert type(be._executor) is NativeTransformerExecutor and native.launches() > 0
    assert y.shape == x.shape and y.is_contiguous()
    with torch.no_grad():
        assert rel(y, encoder_layer_ref(ref, x, _masks(seed, spec, 2, S))) < 3e-2
    for it in range(3):
        torch.manual_seed(20 + it)
        seed = draw_dropout_seed()
        torch.manual_seed(20 + it)
        launches = native.launches()
        (gx,) = be.backward(x, g)
        assert native.launches() > launches and gx.shape == x.shape
        xr = x.clone().requires_grad_(True)
        encoder_layer_ref(ref, xr, _masks(seed, spec, 2, S)).backward(g)
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
    with torch.no_grad():
        assert rel(be.forward(x)[0], layer(x)) < 3e-2


def _run_steps(module, shape, steps=3):
    """forward, then ``steps`` backward calls through ExpertBackend with fixed seeds; outputs, input gradients and the
    parameters afterwards"""
    from lah_b200.runtime.native_executor import NativeFFNExecutor, NativeTransformerExecutor
    be = _backend(module, shape)
    gen = torch.Generator().manual_seed(7)
    x = torch.randn(*shape, generator=gen).cuda()
    g = (torch.randn(*shape, generator=gen) * 0.1).cuda()
    torch.manual_seed(30)
    res = [be.forward(x)[0]]
    for it in range(steps):
        torch.manual_seed(40 + it)
        res.append(be.backward(x, g)[0])
    assert type(be._executor) in (NativeFFNExecutor, NativeTransformerExecutor)
    torch.cuda.synchronize()
    return res + [v.clone() for v in be.state_dict().values()]


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["own transformer", "ffn", "torch transformer"])
def test_scripted_expert_is_bit_identical_to_unscripted(kind):
    torch.manual_seed(2)
    if kind == "own transformer":
        module, shape = TransformerEncoderLayer(1024, 16), (2, 300, 1024)
    elif kind == "ffn":
        module, shape = FeedforwardBlock(1024), (200, 1024)
    else:
        module, shape = nn.TransformerEncoderLayer(1024, 16, norm_first=True), (300, 2, 1024)
    module = module.cuda()
    scripted = torch.jit.script(copy.deepcopy(module))
    for a, b in zip(_run_steps(module, shape), _run_steps(scripted, shape)):
        assert torch.equal(a, b)


@pytest.mark.gpu
def test_server_round_trip_with_scripted_torch_layer():
    from lah_b200.ops import native
    from lah_b200.runtime.native_executor import NativeTransformerExecutor
    torch.manual_seed(1)
    layer = torch.jit.script(nn.TransformerEncoderLayer(1024, 16, batch_first=True).cuda())
    be = _backend(layer, (2, 256, 1024), name="tjit")
    srv = lah_b200.TesseractServer(None, {"tjit": be}, port=0, conn_handler_processes=1, device="cuda")
    srv.run_in_background()
    try:
        native.reset_launches()
        remote = lah_b200.RemoteExpert("tjit", "127.0.0.1", srv.port, timeout=120)
        x = torch.randn(2, 256, 1024, requires_grad=True)
        y = remote(x)
        assert y.shape == x.shape and bool(torch.isfinite(y).all())
        y.sum().backward()
        assert x.grad is not None and bool(torch.isfinite(x.grad).all())
        assert be.update_count == 1 and type(be._executor) is NativeTransformerExecutor and native.launches() > 0
    finally:
        srv.shutdown()


@pytest.mark.gpu
def test_checkpoint_rebinds_executor_of_scripted_layer():
    torch.manual_seed(3)
    layer = torch.jit.script(nn.TransformerEncoderLayer(1024, 16, batch_first=True).cuda())
    be = _backend(layer, (2, 128, 1024))
    x, g = torch.randn(2, 128, 1024, device="cuda"), torch.randn(2, 128, 1024, device="cuda") * 0.1
    be.backward(x, g)
    ckpt = be.checkpoint()
    be.backward(x, g)
    be.load_checkpoint(ckpt)
    ex = be._executor
    for name, p in layer.named_parameters():
        assert torch.equal(p.detach().cpu(), ckpt["model"]["expert." + name]), name
        assert ex.p.data_ptr() <= p.data_ptr() < ex.p.data_ptr() + ex.p.numel() * 4, name   # a view of the flat buffer again
    for st in be.opt.state.values():
        assert ex.m.data_ptr() <= st["exp_avg"].data_ptr() < ex.m.data_ptr() + ex.m.numel() * 4
    before = {k: v.clone() for k, v in be.state_dict().items()}
    be.backward(x, g)
    assert be._executor is ex and be.update_count == 2   # the checkpoint restored update_count 1
    assert all(not torch.equal(before[k], v) for k, v in be.state_dict().items())


@pytest.mark.gpu
@pytest.mark.parametrize("scripted", [False, True])
@pytest.mark.parametrize("name", ["tanh GELU", "SiLU", "eps 1e-6", "bias=False", "head dim 48", "lookalike"])
def test_refused_variants_run_on_the_module(name, scripted):
    torch.manual_seed(5)
    d = 768 if name == "head dim 48" else 512
    kw = dict(batch_first=True, dim_feedforward=1024)
    module = {"tanh GELU": lambda: nn.TransformerEncoderLayer(d, 16, activation=nn.GELU(approximate="tanh"), **kw),
              "SiLU": lambda: nn.TransformerEncoderLayer(d, 16, activation=nn.SiLU(), **kw),
              "eps 1e-6": lambda: nn.TransformerEncoderLayer(d, 16, layer_norm_eps=1e-6, **kw),
              "bias=False": lambda: nn.TransformerEncoderLayer(d, 16, bias=False, **kw),
              "head dim 48": lambda: nn.TransformerEncoderLayer(d, 16, **kw),
              "lookalike": lambda: LookalikeEncoderLayer(d, 16)}[name]().cuda().eval()
    if scripted:
        if name in NOT_SCRIPTABLE:
            pytest.skip("torch.jit.script refuses this module")
        module = torch.jit.script(module)
    be = _backend(module, (2, 128, d))
    x = torch.randn(2, 128, d, device="cuda")
    (y,) = be.forward(x)
    assert be._executor is None
    with torch.no_grad():
        assert torch.equal(y, module(x))
