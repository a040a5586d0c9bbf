"""Streaming probe of the fused wgrad + AMSGrad kernel's optimizer state (tools/opt_stream_probe.cu).

The state stream alone — no MMA, no AMSGrad math — at the shapes of the benchmark step: four fp32 [G*N, K] arrays (p, m, v,
vmax) read and written back, 58 experts of FeedforwardBlock(512): w1 [2048, 512], w2 [2048, 2048], w3 [512, 2048].  One
"step" is the three launches.  Every chunk geometry of the probe kernel runs at 80 CTAs (the optimizer stream's share of a
132-SM H100 in the training step) and on all SMs, TMA only and with the bf16 mirror written by the consumer warps, next to a
device-to-device copy of the same byte count.  "split_planes" streams the master weight as its bf16 GEMM operand plus a
16-bit low half (hi, lo, m, v, vmax: 32 B per parameter, all by TMA) instead of fp32 p + the mirror (34 B); every
configuration's rate counts the bytes it really moves, and the step times compare directly.  Configurations alternate
inside every timing window; the report is the median over windows.

Run on the GPU: python tools/opt_stream_probe.py [--windows N] [--steps N]; writes check_out/opt_stream_probe.json"""
import argparse
import ctypes
import json
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch

from tools import output_path

GEOS = {"cols_128x32": 0, "rows_32x128": 1, "bands_3d_swz": 2, "bands_3d_flat": 3, "split_planes": 4}
SPLIT = GEOS["split_planes"]
SHAPES = [(2048, 512), (2048, 2048), (512, 2048)]
STATE_BYTES_PER_PARAM = 4 * 4 * 2 + 2   # p, m, v, vmax read and written + the bf16 mirror
SPLIT_BYTES_PER_PARAM = (2 + 2 + 4 * 3) * 2   # hi, lo, m, v, vmax read and written


def build(tmp):
    from lah_b200.build_native import NVCC_FLAGS, _nvcc, CSRC
    so = os.path.join(tmp, "opt_stream_probe.so")
    src = os.path.join(ROOT, "tools", "opt_stream_probe.cu")
    subprocess.run([_nvcc(), *NVCC_FLAGS, "-shared", "-I", str(CSRC), src, "-o", so], check=True)
    lib = ctypes.CDLL(so)
    lib.probe_stream.argtypes = [ctypes.c_int] * 4 + [ctypes.c_void_p] * 6 + [ctypes.c_int, ctypes.c_void_p]
    lib.probe_stream.restype = ctypes.c_int
    return lib


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:  # noqa
        q = f"unknown ({e!r})"
    return name, q


def make_state(G, N, K):
    arrs = [torch.empty(G * N, K, device="cuda").uniform_(0.5, 1.5) for _ in range(4)]
    mir = torch.zeros(G * N, K, device="cuda", dtype=torch.bfloat16)
    return arrs, mir, torch.randint(-2 ** 15, 2 ** 15, (G * N, K), device="cuda", dtype=torch.int16)


def launch(lib, geo, mirror_on, st, ctas):
    (p, m, v, vm), mir, lo = st
    r = lib.probe_stream(geo, mirror_on, p.shape[0], p.shape[1], p.data_ptr(), m.data_ptr(), v.data_ptr(), vm.data_ptr(),
                         mir.data_ptr(), lo.data_ptr(), ctas, torch.cuda.current_stream().cuda_stream)
    if r:
        raise RuntimeError(f"probe_stream returned {r}")


def check_geometries(lib):
    """every geometry moves each element back where it came from and writes the mirror of every element"""
    out = {}
    for name, geo in GEOS.items():
        st = make_state(3, 256, 384)
        if geo == SPLIT:   # no mirror: every plane and array comes back as it was
            st[1].copy_(st[0][0])
            ref = [a.clone() for a in (*st[0][1:], st[1], st[2])]
            launch(lib, geo, 0, st, 0)
            torch.cuda.synchronize()
            out[name] = {"state_unchanged": all(torch.equal(a, b) for a, b in zip((*st[0][1:], st[1], st[2]), ref))}
            continue
        ref = [a.clone() for a in st[0]]
        launch(lib, geo, 1, st, 0)
        torch.cuda.synchronize()
        same = all(torch.equal(a, b) for a, b in zip(st[0], ref))
        mir = torch.equal(st[1], ref[0].to(torch.bfloat16))
        out[name] = {"state_unchanged": same, "mirror_complete": mir}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--experts", type=int, default=58)
    ap.add_argument("--windows", type=int, default=7)
    ap.add_argument("--steps", type=int, default=5)
    args = ap.parse_args()
    torch.cuda.init()
    name, limits = card()
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    print(f"device: {name}; power.limit, clocks.max.sm: {limits}; SMs: {sms}", flush=True)
    with tempfile.TemporaryDirectory() as tmp:
        lib = build(tmp)
        checks = check_geometries(lib)
        print("geometry checks:", checks, flush=True)
        G = args.experts
        states = [make_state(G, N, K) for N, K in SHAPES]
        params = sum(G * N * K for N, K in SHAPES)
        nbytes = params * STATE_BYTES_PER_PARAM
        src = torch.empty(nbytes // 2, dtype=torch.uint8, device="cuda")
        dst = torch.empty_like(src)
        configs = {"copy": lambda: dst.copy_(src)}
        moved = {"copy": nbytes}
        for gname, geo in GEOS.items():
            for mirror_on in ((0,) if geo == SPLIT else (0, 1)):
                for ctas in (80, sms):
                    def step(geo=geo, mirror_on=mirror_on, ctas=ctas):
                        for st in states:
                            launch(lib, geo, mirror_on, st, ctas)
                    key = f"{gname}{'_mirror' if mirror_on else ''}_{ctas}ctas"
                    configs[key] = step
                    per_param = SPLIT_BYTES_PER_PARAM if geo == SPLIT else 4 * 4 * 2 + 2 * mirror_on
                    moved[key] = params * per_param
        for fn in configs.values():
            fn()
        torch.cuda.synchronize()
        times = {k: [] for k in configs}
        for _ in range(args.windows):
            for k, fn in configs.items():
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                for _ in range(args.steps):
                    fn()
                b.record()
                torch.cuda.synchronize()
                times[k].append(a.elapsed_time(b) / args.steps)
        report = {"device": name, "power_limit_and_max_sm_clock": limits, "experts": G, "bytes_per_step": nbytes,
                  "geometry_checks": checks, "results": {}}
        for k, ts in times.items():
            ts.sort()
            ms = ts[len(ts) // 2]
            report["results"][k] = {"ms": ms, "bytes": moved[k], "TBps": moved[k] / ms / 1e9, "spread_ms": [ts[0], ts[-1]]}
            print(f"{k:32s} {ms:8.3f} ms  {moved[k] / ms / 1e9:6.3f} TB/s  (windows {ts[0]:.3f} .. {ts[-1]:.3f})", flush=True)
    with open(output_path("opt_stream_probe.json"), "w") as f:
        json.dump(report, f, indent=1)
    ok = all(all(v.values()) for v in checks.values())
    print("ALL_OK" if ok else "SOME_FAILED")
    return 0 if ok else 1


if __name__ == "__main__":
    sys.exit(main())
