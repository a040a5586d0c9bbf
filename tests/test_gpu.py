"""GPU tests (run on an H100: `pytest -m gpu`).  Every sm_90a kernel is compared against a plain PyTorch fp32 oracle."""
import json
import os
import subprocess
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def gemm_check():
    from tools import gpu_gemm_check
    return gpu_gemm_check


@pytest.mark.parametrize("args", [
    dict(rows_per_group=[128, 300, 0, 77], N=512, K=512, w_is_kn=False, block_n=256),
    dict(rows_per_group=[128, 300, 0, 77], N=384, K=192, w_is_kn=False, block_n=128),
    dict(rows_per_group=[256, 1], N=64, K=64, w_is_kn=False, block_n=64),
    dict(rows_per_group=[200, 130], N=512, K=2048, w_is_kn=False, block_n=256, residual=True, out_f32=True),
    dict(rows_per_group=[128, 300, 0, 77], N=512, K=2048, w_is_kn=True, block_n=256, bias=False),
    dict(rows_per_group=[130, 5], N=256, K=512, w_is_kn=True, block_n=128, bias=False, residual=True),
    dict(rows_per_group=[512], N=64, K=512, w_is_kn=True, block_n=64, bias=False),
    dict(rows_per_group=[1000, 24, 2048], N=2048, K=512, w_is_kn=False, block_n=256),
])
def test_grouped_gemm_forward_and_dgrad(gemm_check, args):
    err, untouched = gemm_check.case_mgroup(**args)
    assert err < 1e-2 and untouched


@pytest.mark.parametrize("args", [
    dict(rows_per_group=[128, 300, 0, 77], M=256, N=512, block_n=256),
    dict(rows_per_group=[1000, 64], M=128, N=384, block_n=128),
    dict(rows_per_group=[512, 512], M=512, N=64, block_n=64),
    dict(rows_per_group=[2048, 0, 640], M=2048, N=2048, block_n=256),
])
def test_grouped_gemm_wgrad(gemm_check, args):
    assert gemm_check.case_kgroup(**args) < 1e-3


@pytest.mark.parametrize("args", [
    dict(rows_per_group=[256, 300, 0, 77], N=512, K=512, w_is_kn=False, block_n=256),
    dict(rows_per_group=[200, 130], N=512, K=2048, w_is_kn=False, block_n=256, residual=True, out_f32=True),
    dict(rows_per_group=[128, 300, 0, 77], N=512, K=2048, w_is_kn=True, block_n=256, bias=False),
    dict(rows_per_group=[130, 5], N=256, K=512, w_is_kn=True, block_n=256, bias=False, residual=True),
    dict(rows_per_group=[1000, 24, 2048], N=2048, K=512, w_is_kn=False, block_n=256),
    dict(rows_per_group=[700, 1, 513], N=2048, K=2048, w_is_kn=True, block_n=256, bias=False),
])
def test_cta_pair_gemm_forward_and_dgrad(gemm_check, args):
    """the PRODUCTION entry point of the big path (lah_gemm_mgroup2: 128x256 tiles, 256-row expert groups)"""
    err, untouched = gemm_check.case_mgroup(two_cta=True, **args)
    assert err < 1e-2 and untouched


@pytest.mark.parametrize("args", [
    dict(rows_per_group=[256, 300, 0, 77], M=256, N=512, block_n=256),
    dict(rows_per_group=[512, 512], M=512, N=2048, block_n=256),
    dict(rows_per_group=[2048, 0, 640], M=2048, N=2048, block_n=256),
    dict(rows_per_group=[1000, 64], M=2048, N=512, block_n=256),
])
def test_cta_pair_gemm_wgrad_values(gemm_check, args):
    """wgrad of the production kernel compared by VALUE (rel. L2 error vs the fp32 matmul of the same bf16 operands)"""
    assert gemm_check.case_kgroup(two_cta=True, **args) < 1e-3


@pytest.mark.parametrize("check", ["check_swapab", "check_wgrad_adam"])
def test_small_m_kernels(check):
    """swap-AB weight-streaming GEMM (forward + dgrad) and the fused wgrad+AMSGrad kernel (csrc/small_m.cu)"""
    from tools import gpu_small_check as S
    S.results.clear()
    getattr(S, check)()
    bad = {k: v for k, v in S.results.items() if not v.get("ok")}
    assert S.results and not bad, bad


@pytest.mark.parametrize("path", ["small", "big"])
def test_cuda_graph_step_equals_eager_step(path):
    """the whole training step captured in ONE CUDA graph (device-side epochs / step counters) == the eager step"""
    import lah_b200  # noqa
    from lah_b200.ops import native
    from lah_b200.parallel import engine as E
    from lah_b200.parallel.trainer import DMoETrainer
    cfg = E.DMoEConfig(hidden=512, grid_size=(16,), k=4, num_layers=2, tokens_per_rank=256, gate_mode="emulator", failure_rate=0.1,
                       lr=1e-4, expert_path=path)   # small lr: atomics-order noise must not be amplified by the optimisation
    torch.manual_seed(0)
    xs = [torch.randn(256, cfg.in_features, device="cuda") for _ in range(6)]
    ys = [torch.randint(0, 10, (256,), device="cuda") for _ in range(6)]
    losses = {}
    for graph in (False, True):
        t = DMoETrainer(cfg, use_graph=graph)
        assert t.ctx.small == (path == "small")
        losses[graph] = [float(t.train_step_device(x, y)) for x, y in zip(xs, ys)]
        if graph:
            assert t._graph is not None and t._graph_launches > 20 and native.launches() > 0
        t.ctx.check_status()
        t.close()
    for a, b in zip(losses[False], losses[True]):
        assert abs(a - b) < 5e-3 * max(1.0, abs(a)), losses
    assert losses[True][-1] == losses[True][-1]


def test_update_every_inputs_accumulates_like_the_emulator():
    """DMoEConfig.update_every_inputs / update_every_steps (dmoe_emulator.py:70-77): experts step only when due"""
    import lah_b200  # noqa
    from lah_b200.parallel import engine as E
    from lah_b200.parallel.trainer import DMoETrainer
    cfg = E.DMoEConfig(hidden=512, grid_size=(4, 4), k=4, num_layers=1, tokens_per_rank=256, update_every_inputs=10 ** 6,
                       update_every_steps=3)
    t = DMoETrainer(cfg)
    x, y = torch.randn(256, cfg.in_features, device="cuda"), torch.randint(0, 10, (256,), device="cuda")
    steps = []
    for _ in range(7):
        t.train_step_device(x, y)
        steps.append(int(t.model.blocks[0].shard.step.max()))
    t.ctx.check_status()
    assert steps == [0, 0, 1, 1, 1, 2, 2], steps
    t.close()


def test_trainer_microbatches_on_gpu():
    """several trainers per rank: experts step after every micro-batch's backward, the trainer once per step (graph-captured)"""
    import lah_b200  # noqa
    from lah_b200.parallel import engine as E
    from lah_b200.parallel.trainer import DMoETrainer
    cfg = E.DMoEConfig(hidden=512, grid_size=(4, 4), k=4, num_layers=2, tokens_per_rank=256, trainer_microbatches=2, trainer_staleness=1)
    t = DMoETrainer(cfg)
    x, y = torch.randn(256, cfg.in_features, device="cuda"), torch.randint(0, 10, (256,), device="cuda")
    losses = [float(t.train_step_device(x, y)) for _ in range(6)]
    t.ctx.check_status()
    assert int(t.model.blocks[0].shard.step.max()) == 12 and t._graph is not None
    assert losses[-1] < losses[0]
    t.close()


def test_public_api_runs_the_engine():
    """README-style code (lib.GatingFunction over a network) on CUDA tensors runs the sm_90a layer:
    InBoxNetwork.bind_engine -> GatingFunction.forward -> FusedDMoE.forward_with_gate; heartbeats reach the gate kernel
    through the device-resident table; result == the generic RemoteExpert/TCP path on the same experts"""
    import lah_b200 as lib
    from lah_b200.models import FeedforwardBlock
    from lah_b200.ops import native
    from lah_b200.parallel import engine as E
    cfg = E.DMoEConfig(hidden=256, grid_size=(2, 4), k=2, num_layers=1, tokens_per_rank=64, uid_prefix="expert")
    ctx = E.EngineContext(cfg)
    layer = E.FusedDMoE(cfg, ctx).cuda()
    uids = [E.expert_uid(cfg, e) for e in range(cfg.num_experts)]
    # the same experts behind a TCP server (eager CPU modules with identical weights)
    backends = {}
    for e, uid in enumerate(uids):
        block = FeedforwardBlock(256)
        block.load_state_dict({k[len("expert."):]: v for k, v in layer.shard.expert_state_dict(e).items()})
        backends[uid] = lib.ExpertBackend(name=uid, expert=block, opt=torch.optim.SGD(block.parameters(), lr=0.0),
                                          args_schema=(lib.BatchTensorProto(256),), outputs_schema=lib.BatchTensorProto(256),
                                          max_batch_size=64)
    net = lib.InBoxNetwork()
    server = lib.TesseractServer(net, backends, port=0, conn_handler_processes=4, update_period=1000)
    server.run_in_background()
    try:
        net.declare_experts(uids, "127.0.0.1", server.port)
        gating = lib.GatingFunction(in_features=256, grid_size=(2, 4), network=net, k_best=2, uid_prefix="expert")
        x = torch.randn(16, 256)
        y_tcp = gating(x)                                  # generic path: beam search + RemoteExpert RPCs
        net.bind_engine(layer)
        net.declare_experts(uids, "127.0.0.1", server.port)   # heartbeats -> device table (this rank hosts all of them)
        net.sync_alive()
        torch.cuda.synchronize()
        assert int(ctx.alive.sum()) == cfg.num_experts
        gating.cuda()
        before = native.launches()
        xc = x.cuda().requires_grad_(True)
        y_fused = gating(xc)
        assert native.launches() > before, "the fused path must launch sm_90a kernels"
        assert (y_fused.float().cpu() - y_tcp).norm() / y_tcp.norm() < 3e-2
        y_fused.sum().backward()
        assert gating.proj.weight.grad is not None and xc.grad is not None
        # an expert whose heartbeat expired disappears from the gate kernel's table
        ctx.hb[3] = 1
        net.sync_alive(heartbeat_expiration=120)
        torch.cuda.synchronize()
        assert int(ctx.alive[3]) == 0 and int(ctx.alive.sum()) == cfg.num_experts - 1
        assert net.get_experts([uids[0]])[0] is not None
    finally:
        server.shutdown()
        ctx.check_status()
        ctx.close()


def test_expert_backend_runs_native_kernels():
    """ExpertBackend (the TesseractServer's unit of work) executes a FeedforwardBlock on the sm_90a kernels: forward and
    backward (recompute + dgrad + fused wgrad/AMSGrad) agree with eager PyTorch + torch.optim.Adam(amsgrad=True)"""
    import copy
    import lah_b200 as lib
    from lah_b200.models import FeedforwardBlock
    from lah_b200.ops import native
    torch.manual_seed(0)
    block = FeedforwardBlock(256).cuda()
    ref = copy.deepcopy(block)
    ref_opt = torch.optim.Adam(ref.parameters(), lr=1e-3, amsgrad=True)
    be = lib.ExpertBackend(name="e", expert=block, opt=torch.optim.Adam(block.parameters(), lr=1e-3, amsgrad=True),
                           args_schema=(lib.BatchTensorProto(256),), outputs_schema=lib.BatchTensorProto(256), max_batch_size=64)
    x = torch.randn(37, 256, device="cuda")
    g = torch.randn(37, 256, device="cuda")
    before = native.launches()
    (y,) = be.forward(x)
    assert native.launches() > before and be._executor is not None
    assert (y - ref(x)).norm() / ref(x).norm() < 2e-2
    for it in range(3):
        (gx,) = be.backward(x, g)
        xr = x.clone().requires_grad_(True)
        ref(xr).backward(g)
        ref_opt.step(), ref_opt.zero_grad()
        if it == 0:   # same weights on both sides: only bf16 activation rounding (incl. ~0.4 % flipped ReLU gates) differs
            assert (gx - xr.grad).norm() / xr.grad.norm() < 5e-2
    assert (gx - xr.grad).norm() / xr.grad.norm() < 1e-1
    assert be.update_count == 3
    sd, rsd = be.state_dict(), ref.state_dict()
    for k, v in rsd.items():   # three AMSGrad steps of lr 1e-3: parameters track the eager run
        assert (sd["expert." + k] - v).abs().mean() < 2e-4, k
    ost = be.opt.state_dict()["state"]
    assert float(ost[0]["step"]) == 3.0 and ost[0]["exp_avg"].abs().sum() > 0 and "max_exp_avg_sq" in ost[0]
    ck = be.checkpoint()
    be.load_checkpoint(ck)
    (y2,) = be.forward(x)
    assert torch.isfinite(y2).all()


@pytest.fixture(scope="module")
def layer_check():
    from tools import gpu_layer_check
    return gpu_layer_check


@pytest.mark.parametrize("check", ["check_gate", "check_ln", "check_adam", "check_layer", "check_layer_small", "check_layer_fp8"])
def test_kernels_and_fused_layer_against_oracles(layer_check, check):
    layer_check.results.clear()
    getattr(layer_check, check)()
    assert layer_check.results, "no results recorded"
    bad = {k: v for k, v in layer_check.results.items() if not v.get("ok")}
    assert not bad, bad


def test_smoke_entry_point():
    import __graft_entry__
    __graft_entry__.smoke()


def test_native_library_is_what_runs():
    """the hot path must be the in-tree sm_90a library, not a PyTorch fallback"""
    from lah_b200.ops import native
    assert native.have_cuda_kernels()
    maps = open("/proc/self/maps").read()
    assert "liblah_cuda.so" in maps


def test_fused_trainer_matches_baseline_trainer_one_step():
    """fused engine vs the NCCL/cuBLAS-style baseline (fp32 autograd) on the same weights: same loss, same routing"""
    import lah_b200  # noqa
    from lah_b200.parallel import baseline, engine as E
    from lah_b200.parallel.trainer import DMoETrainer
    cfg = E.DMoEConfig(hidden=512, grid_size=(4, 4), k=4, num_layers=2, tokens_per_rank=512)
    fused = DMoETrainer(cfg)
    base = baseline.BaselineTrainer(cfg)
    with torch.no_grad():
        for name in ("stem", "norm", "head"):
            getattr(base.model, name).load_state_dict(getattr(fused.model, name).state_dict())
        for fb, bb in zip(fused.model.blocks, base.model.blocks):
            bb.load_from_shard(fb.shard)
            bb.proj.load_state_dict(fb.proj.state_dict())
    # a learnable task (10 class prototypes + noise) drawn on the CPU: the loss must fall, and the sample must not depend on
    # the GPU (the CUDA generator's output depends on the device's SM count)
    gen = torch.Generator().manual_seed(0)
    protos = torch.randn(10, cfg.in_features, generator=gen)
    y = torch.randint(0, 10, (512,), generator=gen)
    x = (protos[y] + 3.0 * torch.randn(512, cfg.in_features, generator=gen)).cuda()
    y = y.cuda()
    l_fused = [float(fused.train_step_device(x, y)) for _ in range(4)]
    l_base = [float(base.train_step_device(x, y)) for _ in range(4)]
    fused.ctx.check_status()
    fused.close()   # unregisters the context's status word from the optimizer kernels before it is freed
    assert abs(l_fused[0] - l_base[0]) < 2e-2, (l_fused, l_base)
    assert l_fused[-1] < l_fused[0] and abs(l_fused[-1] - l_base[-1]) < 0.15, (l_fused, l_base)


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
@pytest.mark.parametrize("extra", [[], ["--force-shadow"], ["--small"]])
def test_two_gpu_p2p_dispatch_matches_single_gpu(extra):
    """fused P2P engine on 2 GPUs == single-process oracle; with --force-shadow the hot-expert replica path (weights pulled
    over NVLink, partial weight gradients reduced inside the owner's Adam kernel) is exercised for 4 experts"""
    out = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2",
                          "--master-addr", "127.0.0.1", "--master-port", "29541",
                          os.path.join(ROOT, "tools", "multi_gpu_check.py"), *extra], capture_output=True, text=True, timeout=600)
    assert out.returncode == 0, out.stdout[-3000:] + out.stderr[-3000:]
    assert "MULTI_GPU_OK" in out.stdout, out.stdout[-3000:]


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_rank_failure_is_detected_and_survivors_continue():
    """bounded peer-flag waits + device-resident heartbeat table: one rank stops mid-run, the other excludes it and trains on"""
    out = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2",
                          "--master-addr", "127.0.0.1", "--master-port", "29547",
                          os.path.join(ROOT, "tools", "fault_check.py")], capture_output=True, text=True, timeout=600)
    assert out.returncode == 0 and "FAULT_OK" in out.stdout, out.stdout[-3000:] + out.stderr[-3000:]


@pytest.mark.parametrize("check", ["check_attention", "check_attention_bwd", "check_layer", "check_transformer_train",
                                   "check_ffn_native", "check_chain"])
def test_attention_kernel_and_native_transformer_expert(check):
    """wgmma attention (csrc/attention.cu) and the sm_90a transformer expert vs fp32 PyTorch oracles"""
    from tools import gpu_attention_check as A
    A.results.clear()
    getattr(A, check)()
    bad = {k: v for k, v in A.results.items() if not v.get("ok")}
    assert A.results and not bad, bad


@pytest.mark.parametrize("check", ["check_quant", "check_gemm"])
def test_mxfp8_quantiser_and_block_scaled_gemm(check):
    """MXFP8 quantisation kernel == PyTorch oracle bit for bit; block-scaled FP8 (E4M3 wgmma) grouped GEMM == fp32
    matmul of the dequantised operands"""
    from tools import gpu_fp8_check as Q
    Q.results.clear()
    getattr(Q, check)()
    bad = {k: v for k, v in Q.results.items() if not v.get("ok")}
    assert Q.results and not bad, bad
