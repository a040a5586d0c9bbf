"""
The optimizer-state stream of the fused weight gradient + AMSGrad kernel (csrc/small_m.cu, ``wgrad_adam``) at the shapes of
the benchmark step: FeedforwardBlock(512) experts, w1 [2048, 512], w2 [2048, 2048] and w3 [512, 2048], over groups of 0, 1,
15, 16, 17 and 300 rows.  Every state element a launch updates is compared with the float64 oracle (the exact-gradient
operands and bounds of test_fused_adam_fp8_kernels.py and test_weight_decay.py), in each weight-decay form, with AMSGrad on
and off.  p, m, v, vmax and the bf16 mirror are views into larger buffers whose guard regions before and after are
canaries, so a chunk that lands in the wrong rows or columns, or outside the tensors, shows up byte for byte; a second
launch from the same state must give the same bytes.
"""
import pytest
import torch

from test_expert_kernels import BF16, U, f32, poison, sentinel_like, within  # noqa: F401
from test_fused_adam_fp8_kernels import OPT_CTAS, same_bytes, wa_inputs, wgrad64
from test_weight_decay import adamw_ref64, kernel_decay

from lah_b200.ops import kernels as K

STREAM_ROWS = [0, 1, 15, 16, 17, 300]
STREAM_STEPS = [3, 1, 2, 10, 1000, 7]
GUARD = 8192   # canary elements before and after every array: more than one 128-column row run of the widest tile

SHAPES = {"w1_n2048_k512": (2048, 512), "w2_n2048_k2048": (2048, 2048), "w3_n512_k2048": (512, 2048)}
MODES = {
    "amsgrad": dict(amsgrad=True),
    "adam": dict(amsgrad=False),
    "l2_amsgrad": dict(amsgrad=True, weight_decay=0.05),
    "decoupled_adam": dict(amsgrad=False, weight_decay=0.1, decoupled=True),
}


def guarded(shape, dtype, fill):
    """a [G, N, K] view into a flat buffer with GUARD canary elements on both sides; fill(view) sets the inside"""
    n = shape[0] * shape[1] * shape[2]
    buf = sentinel_like((n + 2 * GUARD,), dtype)
    view = buf[GUARD:GUARD + n].view(shape)
    fill(view)
    return buf, view


def stream_state(seed, G, N, K_, stepped):
    """random state in the stepped groups (vmax on both sides of v), canaries in the other groups and the whole mirror"""
    cg = torch.Generator(device="cuda").manual_seed(seed)
    shape = (G, N, K_)
    v = torch.rand(shape, generator=cg, device="cuda") * 1e-3
    vals = dict(p=torch.randn(shape, generator=cg, device="cuda"),
                m=torch.randn(shape, generator=cg, device="cuda") * 1e-2,
                v=v, vmax=v * (0.5 + torch.rand(shape, generator=cg, device="cuda")))
    mask = torch.tensor(stepped, device="cuda")
    bufs = {}
    for name, val in vals.items():
        def fill(t, val=val):
            t[mask] = val[mask]
        bufs[name] = guarded(shape, torch.float32, fill)[0]
    bufs["p_bf16"] = guarded(shape, BF16, lambda t: None)[0]
    return bufs


def views(bufs, shape):
    n = shape[0] * shape[1] * shape[2]
    return {k: b[GUARD:GUARD + n].view(shape) for k, b in bufs.items()}


def launch(bufs, shape, dy, x, go, gr, step, *, lr, mode, max_ctas):
    out = {k: b.clone() for k, b in bufs.items()}
    t = views(out, shape)
    K.wgrad_adam(dy, x, go, gr, p=t["p"], m=t["m"], v=t["v"], vmax=t["vmax"], p_bf16=t["p_bf16"], step=step, lr=lr,
                 amsgrad=mode["amsgrad"], weight_decay=mode.get("weight_decay", 0.0),
                 decoupled=mode.get("decoupled", False), max_ctas=max_ctas)
    torch.cuda.synchronize()
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("mode", list(MODES))
@pytest.mark.parametrize("shape", list(SHAPES))
def test_wgrad_adam_stream_benchmark_shapes(shape, mode, poison, record_property):
    N, K_ = SHAPES[shape]
    md = MODES[mode]
    seed = 200 + 10 * list(SHAPES).index(shape) + list(MODES).index(mode)
    gen = torch.Generator().manual_seed(seed)
    G, lr = len(STREAM_ROWS), 2e-3
    dy, x, offs = wa_inputs(gen, STREAM_ROWS, N, K_, exact=True)
    stepped = [r > 0 for r in STREAM_ROWS]
    grad = torch.zeros(G, N, K_, dtype=torch.float64, device="cuda")
    for g, ref in enumerate(wgrad64(dy, x, offs, STREAM_ROWS)):
        if ref is not None:
            grad[g] = ref[0]
    go = torch.tensor(offs, dtype=torch.int32, device="cuda")
    gr = torch.tensor(STREAM_ROWS, dtype=torch.int32, device="cuda")
    step = torch.tensor(STREAM_STEPS, dtype=torch.int32, device="cuda")
    bufs = stream_state(seed, G, N, K_, stepped)
    max_ctas = OPT_CTAS if list(MODES).index(mode) % 2 == 0 else 0
    out = launch(bufs, (G, N, K_), dy, x, go, gr, step, lr=lr, mode=md, max_ctas=max_ctas)
    again = launch(bufs, (G, N, K_), dy, x, go, gr, step, lr=lr, mode=md, max_ctas=max_ctas)
    for name in out:
        assert same_bytes(out[name], again[name]), f"two identical launches differ in {name}"
        assert same_bytes(out[name][:GUARD], bufs[name][:GUARD]), f"written before {name}"
        assert same_bytes(out[name][-GUARD:], bufs[name][-GUARD:]), f"written after {name}"

    st, t = views(bufs, (G, N, K_)), views(out, (G, N, K_))
    wd = md.get("weight_decay", 0.0)
    new, upd, bounds = adamw_ref64(st["p"].view(-1), grad.view(-1), st["m"].view(-1), st["v"].view(-1),
                                   st["vmax"].view(-1), [N * K_], G, step=step, group_rows=gr.cpu(), lr=f32(lr),
                                   betas=(f32(0.9), f32(0.999)), eps=f32(1e-8), amsgrad=md["amsgrad"], grad=grad.view(-1),
                                   weight_decay=f32(wd), decoupled=md.get("decoupled", False),
                                   decay=kernel_decay(lr, wd))
    assert upd.view(G, -1).all(1).tolist() == stepped
    worst = 0.0
    for name in ("p", "m", "v") + (("vmax",) if md["amsgrad"] else ()):
        got = t[name].view(-1)
        worst = max(worst, within(got[upd], new[name][upd], bounds[name][upd], name, "wgrad_adam stream"))
    if not md["amsgrad"]:
        assert same_bytes(t["vmax"], st["vmax"]), "vmax written without amsgrad"
    for g in range(G):
        if stepped[g]:
            assert same_bytes(t["p_bf16"][g], t["p"][g].to(BF16)), f"p_bf16 of group {g} is not the rounding of p"
        else:
            for name in t:
                assert same_bytes(t[name][g], st[name][g]), f"{name} of empty group {g} was written"
    record_property("max_err_over_bound", worst)
