"""
In-box version of the throughput experiment (BASELINE.json config "throughput_client transformer-block 56 layers/GPU,
64 trainers, experts sharded over 8xH100"; reference: experiments/throughput/throughput_client.py:40-68
+ throughput_server.py:13-33).

The reference chains 56 x H remote layers, interleaved across the H servers, and keeps them busy with 64 concurrent
trainer processes, each forward pass being one 8 MiB TCP RPC per layer.  Here every rank (one process per H100) hosts
``layers_per_gpu`` experts executed by the sm_90a kernels (NativeTransformerLayer / NativeFFNLayer); layer i of the
chain lives on rank i % W exactly like the reference's interleaving; the 64 trainers' batches travel in W waves, one per
rank per pipeline tick, and the LAST kernel of every layer writes its output straight into the NEXT rank's input buffer
over NVLink (plain stores to peer memory from the LayerNorm / GEMM epilogue — no copy kernel, no NCCL), followed by a
release/acquire flag handshake.  Forward only, like the reference experiment.

    python -m lah_b200.experiments.throughput.inbox_chain --block-type transformer            (1 GPU)
    python -m torch.distributed.run --nproc-per-node 8 -m lah_b200.experiments.throughput.inbox_chain --block-type ffn

Prints one JSON line: samples/s = jobs * batch_size * passes / device time (max over ranks), the reference's definition
(throughput_client.py:64) with CUDA-event timing.
"""
import json
import os
from argparse import ArgumentParser

import torch

from ...models.layers import name_to_block, SEQ_LEN
from ...ops import kernels as K, native


def chain_schedule(tick: int, rank: int, world: int, num_layers: int):
    """which wave this rank works on at pipeline tick ``tick`` and where that wave is in the chain.

    Layer i of the chain lives on rank i % world (the reference client interleaves the servers the same way,
    throughput_client.py:48); wave w enters layer 0 at tick w, so at tick t rank r holds wave (t - r) % world, which is at
    chain position (t - wave) % num_layers — a layer hosted by r by construction.  Returns (wave, global layer, local layer).
    """
    wave = (tick - rank) % world
    layer_global = (tick - wave) % num_layers
    return wave, layer_global, layer_global // world


def make_parser():
    p = ArgumentParser()
    p.add_argument("--block-type", choices=["ffn", "swiglu", "transformer"], default="transformer")
    p.add_argument("--hid-dim", type=int, default=1024)
    p.add_argument("--layers-per-gpu", type=int, default=56)
    p.add_argument("-j", "--jobs", type=int, default=64, help="concurrent trainers")
    p.add_argument("--batch-size", type=int, default=None, help="samples per trainer batch (default: 4 sequences / 2048 rows)")
    p.add_argument("--passes", type=int, default=3, help="timed passes of all trainers' batches through the whole chain")
    p.add_argument("--warmup", type=int, default=1)
    p.add_argument("--dtype", choices=["bf16", "fp8"], default="bf16", help="fp8: MXFP8 GEMMs (ffn and swiglu blocks)")
    return p


def run(args):
    import torch.distributed as dist
    from ...parallel.symmetric import SymmetricHeap, _CudaBuffer
    rank, world = int(os.environ.get("RANK", 0)), int(os.environ.get("WORLD_SIZE", 1))
    torch.cuda.set_device(int(os.environ.get("LOCAL_RANK", 0)))
    dev = torch.device("cuda", torch.cuda.current_device())
    if world > 1 and not dist.is_initialized():
        os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
        dist.init_process_group("nccl", device_id=dev)
    native.have_cuda_kernels()
    transformer = args.block_type == "transformer"
    batch = args.batch_size or (4 if transformer else 2048)
    assert args.jobs % world == 0, "trainers must divide evenly into one wave per rank"
    wave_samples = args.jobs // world * batch
    rows = wave_samples * (SEQ_LEN if transformer else 1)
    d = args.hid_dim
    # ---- experts hosted here (random init; identical seed scheme on every rank: layer l of the chain -> seed l)
    if transformer:
        from ...models.transformer_native import NativeTransformerLayer as Native
        kw = {}
    elif args.block_type == "swiglu":
        from ...models.ffn_native import NativeGatedFFNLayer as Native
        kw = dict(dtype=args.dtype)
    else:
        from ...models.ffn_native import NativeFFNLayer as Native
        kw = dict(dtype=args.dtype)
    layers = []
    for li in range(args.layers_per_gpu):
        torch.manual_seed(1000 + li * world + rank)
        layers.append(Native(name_to_block[args.block_type](d), device=dev, **kw))
    L = args.layers_per_gpu * world
    # ---- symmetric double-buffered activation slots: rank r reads buf[t % 2], writes buf[(t + 1) % 2] of rank r + 1
    heap = SymmetricHeap(2 * rows * d * 2 + (1 << 20))
    flags, flags_off = heap.alloc((K.NUM_SLOTS, K.MAX_WORLD), torch.int32)
    flags.zero_()
    bufs, offs = zip(*(heap.alloc((rows, d), torch.bfloat16) for _ in range(2)))
    status = torch.zeros(4, dtype=torch.int32, device=dev)
    nxt = (rank + 1) % world
    peer_bufs = [torch.as_tensor(_CudaBuffer(heap.peer_bases[nxt] + off, rows * d * 2), device=dev).view(torch.bfloat16)
                 .view(rows, d) for off in offs]
    for b in bufs:
        b.copy_(torch.randn(rows, d, device=dev).to(torch.bfloat16))
    heap.barrier()

    def shape(t):
        return t.view(wave_samples, SEQ_LEN, d) if transformer else t

    tick = [0]

    def one_tick():
        t = tick[0]
        _, _, local_layer = chain_schedule(t, rank, world, L)
        layers[local_layer](shape(bufs[t % 2]), out=shape(peer_bufs[(t + 1) % 2]))
        if world > 1:
            K.signal_wait(flags_off, K.SLOT_DISPATCH, t + 1, status, signal=True, wait=True)
        tick[0] = t + 1

    for _ in range(args.warmup * L):
        one_tick()
    torch.cuda.synchronize()
    if world > 1:
        dist.barrier()
    native.reset_launches()
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(args.passes * L):
        one_tick()
    end.record()
    torch.cuda.synchronize()
    ms = torch.tensor([start.elapsed_time(end)], device=dev, dtype=torch.float64)
    if world > 1:
        dist.all_reduce(ms, op=dist.ReduceOp.MAX)
    ms = float(ms)
    ok = int(status[0].item()) == 0 and bool(torch.isfinite(bufs[0].float()).all())
    samples = args.jobs * batch * args.passes
    out = dict(metric="throughput experiment samples/s (forward, device-timed, max over ranks)", value=samples / ms * 1e3,
               unit="samples/s (sequences of 512 tokens)" if transformer else "samples/s (rows)", n_gpus=world,
               ms_per_pass=ms / args.passes, layers_total=L, layers_per_gpu=args.layers_per_gpu, jobs=args.jobs,
               batch_size=batch, block_type=args.block_type, hid_dim=d, dtype=args.dtype, ok=ok,
               gpu_launches=native.launches(),
               layer_ms=ms / (args.passes * L), tokens_per_layer_call=rows)
    heap.barrier()
    if world > 1 and dist.is_initialized():
        dist.barrier()
        dist.destroy_process_group()
    if rank == 0:
        print(json.dumps(out), flush=True)
    return out


if __name__ == "__main__":
    run(make_parser().parse_args())
