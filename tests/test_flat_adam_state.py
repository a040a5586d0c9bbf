"""
FlatAdamState (runtime/native_executor.py) on CPU tensors: the flat-buffer layout and the binding of a module and its torch
optimizer to it, the host code the sm_90a executors share.  Nothing here launches a kernel: on a CPU buffer ``bind()``
refreshes the bf16 mirror with a plain copy.
"""
import copy

import torch

import lah_b200  # noqa: F401
from lah_b200.models.layers import FFN_SEG_KEYS, FFN_SEG_NAMES, FeedforwardBlock
from lah_b200.ops import kernels as K
from lah_b200.parallel import engine as E
from lah_b200.runtime.native_executor import FlatAdamState, NativeFFNExecutor

STATE_KEYS = ("exp_avg", "exp_avg_sq", "max_exp_avg_sq")


def inside(t, flat):
    """``t`` is a view inside the flat buffer ``flat``"""
    lo = flat.data_ptr()
    return lo <= t.data_ptr() and t.data_ptr() + t.numel() * t.element_size() <= lo + flat.numel() * flat.element_size()


def two_groups(params, **kw):
    """weight matrices in group 0, vectors in group 1 with amsgrad"""
    return torch.optim.AdamW([dict(params=[p for p in params if p.dim() >= 2]),
                              dict(params=[p for p in params if p.dim() < 2], weight_decay=0.0, amsgrad=True)], **kw)


def eager_steps(block, opt, n):
    for _ in range(n):
        block(torch.randn(5, 8)).square().sum().backward()
        opt.step(), opt.zero_grad()


def state_copy(opt, params):
    return [{k: v.clone() for k, v in opt.state[p].items()} for p in params]


def assert_bound(st, opt, params, amsgrad_of):
    """parameters and optimizer state are views of the flat buffers, ``max_exp_avg_sq`` exactly where amsgrad is on"""
    for s, p in enumerate(params):
        assert inside(p.data, st.p) and p.grad is None
        state = opt.state[p]
        assert inside(state["exp_avg"], st.m) and inside(state["exp_avg_sq"], st.v)
        assert ("max_exp_avg_sq" in state) == amsgrad_of(p)
        if amsgrad_of(p):
            assert inside(state["max_exp_avg_sq"], st.vmax)
        assert state["exp_avg"].data_ptr() == st.mv[st.names[s]].data_ptr()   # segment s is params[s]


def test_construction_binds_parameters_and_fresh_state():
    torch.manual_seed(0)
    block = FeedforwardBlock(8)
    params = NativeFFNExecutor._segment_params(block)
    assert [id(p) for p in params] == [id(block.get_parameter(FFN_SEG_KEYS[n])) for n in FFN_SEG_NAMES]
    before = [p.detach().clone() for p in params]
    sd_before = {k: v.clone() for k, v in block.state_dict().items()}
    opt = torch.optim.Adam(block.parameters(), amsgrad=True)
    st = FlatAdamState(opt, params, FFN_SEG_NAMES, torch.device("cpu"))
    assert st.groups == [st.all_segs] and st.steps_host == 0 and int(st.step) == 0
    assert st.sizes == [p.numel() for p in params] and st.p.numel() == sum(st.sizes)
    assert_bound(st, opt, params, lambda p: True)
    for p, b in zip(params, before):
        assert torch.equal(p.detach(), b)
    assert all(torch.equal(v, sd_before[k]) for k, v in block.state_dict().items())   # keys, shapes and values unchanged
    assert all(not opt.state[p]["exp_avg"].any() and float(opt.state[p]["step"]) == 0.0 for p in params)
    assert torch.equal(st.p_bf16, st.p.to(torch.bfloat16))
    st.pv["b2"][0].fill_(3.0)   # live: the module sees a write to the buffer
    assert bool((block.layers[3].bias == 3.0).all())


def test_amsgrad_state_exists_for_exactly_the_groups_that_have_it():
    torch.manual_seed(1)
    params = [torch.nn.Parameter(torch.randn(*shape)) for shape in ((4, 3), (4,), (2, 4), (2,))]
    opt = two_groups(params, lr=1e-2, weight_decay=0.1)
    st = FlatAdamState(opt, params, ("wa", "ba", "wb", "bb"), torch.device("cpu"))
    assert st.groups == [0b0101, 0b1010]
    assert_bound(st, opt, params, lambda p: p.dim() < 2)
    hypers = st.hypers()
    assert [mask for _, mask in hypers] == st.groups
    assert [h["amsgrad"] for h, _ in hypers] == [False, True] and [h["weight_decay"] for h, _ in hypers] == [0.1, 0.0]
    opt.param_groups[0]["lr"] = 5e-3   # a schedule: read at the next call
    assert st.hypers()[0][0]["lr"] == 5e-3 and st.hypers()[1][0]["lr"] == 1e-2


def test_state_of_eager_steps_survives_bind():
    torch.manual_seed(2)
    block = FeedforwardBlock(8)
    params = NativeFFNExecutor._segment_params(block)
    opt = two_groups(params, lr=1e-2)
    eager_steps(block, opt, 3)
    want_p, want = [p.detach().clone() for p in params], state_copy(opt, params)
    st = FlatAdamState(opt, params, FFN_SEG_NAMES, torch.device("cpu"))
    assert st.steps_host == 3 and int(st.step) == 3
    assert_bound(st, opt, params, lambda p: p.dim() < 2)
    for p, wp, w in zip(params, want_p, want):
        assert torch.equal(p.detach(), wp)
        assert all(torch.equal(opt.state[p][k], w[k]) for k in STATE_KEYS if k in w)
        assert float(opt.state[p]["step"]) == 3.0
    assert len({id(opt.state[p]["step"]) for p in params}) == len(params)   # one step tensor per parameter
    st.end_step()
    assert st.steps_host == 4 and all(float(opt.state[p]["step"]) == 4.0 for p in params)
    assert len({id(opt.state[p]["step"]) for p in params}) == len(params)
    eager_steps(block, opt, 1)   # torch's optimizer keeps working on the bound state, in place
    assert_bound(st, opt, params, lambda p: p.dim() < 2)
    assert all(float(opt.state[p]["step"]) == 5.0 for p in params)


def test_bind_after_load_state_dict_restores_the_checkpoint():
    torch.manual_seed(3)
    block = FeedforwardBlock(8)
    params = NativeFFNExecutor._segment_params(block)
    opt = two_groups(params, lr=1e-2)
    st = FlatAdamState(opt, params, FFN_SEG_NAMES, torch.device("cpu"))
    eager_steps(block, opt, 2)
    saved_model, saved_opt = copy.deepcopy(block.state_dict()), copy.deepcopy(opt.state_dict())
    want = state_copy(opt, params)
    eager_steps(block, opt, 2)
    block.load_state_dict(saved_model)
    opt.load_state_dict(saved_opt)   # the optimizer now owns fresh state tensors
    assert not any(inside(opt.state[p]["exp_avg"], st.m) for p in params)
    st.bind()
    assert st.steps_host == 2 and int(st.step) == 2
    assert_bound(st, opt, params, lambda p: p.dim() < 2)
    for n, p, w in zip(FFN_SEG_NAMES, params, want):
        assert torch.equal(p.detach(), saved_model[FFN_SEG_KEYS[n]])
        assert all(torch.equal(opt.state[p][k], w[k]) for k in STATE_KEYS if k in w)
        assert float(opt.state[p]["step"]) == 2.0
    assert torch.equal(st.p_bf16, st.p.to(torch.bfloat16)) and bool(st.p_bf16.any())
    assert list(opt.state_dict()["state"]) == list(saved_opt["state"])


def test_segment_views_is_the_layout_of_the_expert_shard():
    cfg = E.DMoEConfig(hidden=8, grid_size=(3,), k=1, num_layers=1, tokens_per_rank=4)
    shard = E.ExpertShard(cfg, 3, 0, torch.device("cpu"))
    shapes = {n: cfg.seg_shapes()[n] for n in E.SEG_NAMES}
    flat = torch.arange(shard.p.numel(), dtype=torch.float32)
    views = K.segment_views(flat, shapes, slots=3)
    assert list(views) == list(E.SEG_NAMES)
    off = 0
    for n, size in zip(E.SEG_NAMES, shard.seg_sizes):
        assert views[n].shape == (3, *shapes[n]) and views[n].storage_offset() == off and views[n].is_contiguous()
        for table in (shard.views, shard.grads, shard.bf16, shard.m_views, shard.v_views, shard.vmax_views):
            assert table[n].shape == views[n].shape and table[n].storage_offset() == off
        assert views[n][2].reshape(-1)[0] == off + 2 * size   # slot 2 of segment n begins two tensors into the segment
        off += 3 * size
    assert off == flat.numel()
    assert shard.views["w2"].data_ptr() == shard.p.data_ptr() + 4 * shard.views["w2"].storage_offset()
