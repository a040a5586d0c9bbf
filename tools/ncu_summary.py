"""Summarise an .ncu-rep (read on the CPU box with `ncu -i`) into a small JSON.
    python tools/ncu_summary.py prof.ncu-rep ncu_<name>.json"""
import csv
import io
import json
import subprocess
import sys

METRICS = {
    "gpu__time_duration.sum": "duration_us",
    "dram__bytes_read.sum": "dram_read",
    "dram__bytes_write.sum": "dram_write",
    "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed": "dram_pct",
    "sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active": "tensor_pipe_pct",
    "lts__throughput.avg.pct_of_peak_sustained_elapsed": "l2_pct",
    "l1tex__throughput.avg.pct_of_peak_sustained_elapsed": "l1tex_pct",
    "sm__throughput.avg.pct_of_peak_sustained_elapsed": "sm_pct",
    "sm__inst_executed_pipe_xu.avg.pct_of_peak_sustained_active": "xu_pipe_pct",
    "sm__warps_active.avg.pct_of_peak_sustained_active": "warps_active_pct",
    "launch__registers_per_thread": "regs",
    "launch__grid_size": "grid",
    "launch__block_size": "block",
    "launch__shared_mem_per_block_dynamic": "dyn_smem",
}


def main(rep, out):
    raw = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], capture_output=True, text=True, check=True).stdout
    rows = list(csv.reader(io.StringIO(raw)))
    hdr, units = rows[0], rows[1]
    idx = {h: i for i, h in enumerate(hdr)}
    kernels = []
    for r in rows[2:]:
        rec = {"kernel": r[idx["Kernel Name"]][:120]}
        for metric, name in METRICS.items():
            if metric in idx:
                rec[name] = f"{r[idx[metric]]} {units[idx[metric]]}".strip()
        kernels.append(rec)
    json.dump({"source": rep, "how": "ncu --set full --clock-control none --import-source on (cold caches, serialised "
               "launches: compare shares, not absolute times)", "kernels": kernels}, open(out, "w"), indent=1)
    print(f"{len(kernels)} kernels -> {out}")


if __name__ == "__main__":
    main(sys.argv[1], sys.argv[2])
