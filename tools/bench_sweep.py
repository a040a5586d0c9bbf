"""
Sweep of the named-config step over expert paths / optimizer-stream CTA partitions inside ONE torchrun job (one rendezvous,
one import, a fresh engine per point): `torchrun --nproc-per-node N tools/bench_sweep.py --gpus N --points small:0 small:64 big`
Prints one JSON line per point (rank 0) and writes check_out/sweep_n{N}.jsonl.
"""
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bench  # noqa: E402
from tools import output_path  # noqa: E402


def main():
    points = ["small:0", "small:64", "small:96", "big"]
    argv = sys.argv[1:]
    if "--points" in argv:
        i = argv.index("--points")
        points = argv[i + 1:]
        argv = argv[:i]
    sys.argv = [sys.argv[0]] + argv
    args = bench.parse_args()
    args.no_e2e = True
    rank, world, local_rank = bench.dist_setup(args.gpus)
    lines = []
    for pt in points:
        path, _, ctas = pt.partition(":")
        if ctas:
            os.environ["LAH_OPTIMIZER_CTAS"] = ctas
        else:
            os.environ.pop("LAH_OPTIMIZER_CTAS", None)
        try:
            r = bench._measure_ours(args, rank, world, local_rank, args.batch_per_gpu, path=path, tag=pt)
            line = {"point": pt, "n_gpus": world, "ms_per_step": round(r["ms_per_step"], 4), "samples_per_s": round(r["value"]),
                    "exposed_wait_ms_per_rank": r["exposed_comm_wait_ms_per_rank"],
                    "hottest_expert_rows_per_layer": r["hottest_expert_rows_per_layer"], "stage_ms_rank0": r["stage_ms_rank0"],
                    "graph": r["config"]["cuda_graph"], "gpu_launches": r["gpu_launches"], "clocks": r["clocks"]}
        except Exception as e:  # noqa
            line = {"point": pt, "error": f"{type(e).__name__}: {e}"[:300]}
        lines.append(line)
        if rank == 0:
            print(json.dumps(line), flush=True)
    if rank == 0:
        with open(output_path(f"sweep_n{world}.jsonl"), "w") as f:
            for line in lines:
                f.write(json.dumps(line) + "\n")
    if world > 1:
        import torch.distributed as dist
        dist.barrier()
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
