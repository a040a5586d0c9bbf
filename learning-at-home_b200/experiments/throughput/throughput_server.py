"""
Expert server for the throughput experiment: one server per GPU hosting `--layers-per-gpu` experts `expert{i}`
(CLI parity: /root/reference/experiments/throughput/throughput_server.py:13-47; same flags).

    python -m lah_b200.experiments.throughput.throughput_server -a 16 -p 8080 --block-type ffn --gpu 0
"""
import sys
from argparse import ArgumentParser

import torch

from ... import ExpertBackend, TesseractServer, BatchTensorProto
from ...models.layers import name_to_block, SEQ_LEN


def build_experts(args, device=None):
    inp_shape = (args.hid_dim,) if args.block_type in ("ffn", "swiglu") else (SEQ_LEN, args.hid_dim)
    experts = {}
    for i in range(args.layers_per_gpu):
        expert = name_to_block[args.block_type](args.hid_dim)
        experts[f"expert{i}"] = ExpertBackend(
            name=f"expert{i}", expert=expert, opt=torch.optim.Adam(expert.parameters()),
            args_schema=(BatchTensorProto(*inp_shape),), outputs_schema=BatchTensorProto(*inp_shape),
            max_batch_size=args.max_batch_size, pool_size=8)
    return experts


def main(args):
    device = torch.device("cuda", args.gpu) if torch.cuda.is_available() and args.gpu >= 0 else torch.device("cpu")
    experts = build_experts(args)
    server = TesseractServer(None, experts, port=args.port, conn_handler_processes=args.handler_processes,
                             sender_threads=4, device=device)
    try:
        server.start()
    except KeyboardInterrupt:
        print("Finishing")
        server.shutdown()


def make_parser():
    parser = ArgumentParser()
    parser.add_argument("-a", "--handler-processes", type=int, default=256)
    parser.add_argument("-p", "--port", type=int, required=True)
    parser.add_argument("--hid-dim", type=int, default=1024)
    parser.add_argument("--max-batch-size", type=int, default=2048)
    parser.add_argument("--gpu", type=int, required=True)
    parser.add_argument("--layers-per-gpu", type=int, default=56)
    parser.add_argument("--block-type", "--block_type", choices=name_to_block.keys(), required=True)
    return parser


if __name__ == "__main__":
    main(make_parser().parse_args())
