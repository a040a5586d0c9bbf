"""
Builds the native parts of the framework IN-TREE (so the shared objects travel with a repo snapshot):

  _C/liblah_cuda.so   every .cu under csrc/  -> nvcc -gencode arch=compute_90a,code=sm_90a (sm_90a ONLY)
  _C/liblah_host.so   every .cpp under csrc/ -> g++ (C++ host runtime: batching queue, framing, DHT routing table)

Both expose a plain C ABI and are loaded with ctypes (see ops/native.py); there is deliberately no dependency on
torch headers, so a full rebuild takes seconds and works on a box without a GPU (nvcc cross-compiles).
"""
import hashlib
import os
import shutil
import subprocess
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent
CSRC = ROOT / "csrc"
OUT = ROOT / "_C"

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
    "--use_fast_math", "-Xcompiler", "-fPIC", "-Xcompiler", "-fvisibility=default",
]
GXX_FLAGS = ["-O3", "-std=c++17", "-fPIC", "-shared", "-pthread", "-Wall"]


def _nvcc() -> str:
    for cand in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found")


def _digest(paths, extra=""):
    h = hashlib.sha256(extra.encode())
    for p in sorted(paths):
        h.update(p.name.encode())
        h.update(p.read_bytes())
    return h.hexdigest()


def _needs_build(target: Path, digest: str) -> bool:
    stamp = target.with_suffix(target.suffix + ".stamp")
    return not (target.exists() and stamp.exists() and stamp.read_text() == digest)


def _run(cmd, verbose):
    if verbose:
        print("+", " ".join(map(str, cmd)), flush=True)
    res = subprocess.run(list(map(str, cmd)), capture_output=True, text=True)
    if res.returncode != 0:
        sys.stderr.write(res.stdout + res.stderr)
        raise RuntimeError(f"native build failed: {' '.join(map(str, cmd[:3]))} ...")
    if verbose and (res.stdout or res.stderr):
        print(res.stdout + res.stderr)


def build_cuda(force=False, verbose=False, ptxas_verbose=False) -> Path:
    OUT.mkdir(exist_ok=True)
    target = OUT / "liblah_cuda.so"
    cus = sorted(CSRC.glob("*.cu"))
    hdrs = sorted(CSRC.glob("*.cuh")) + sorted(CSRC.glob("*.h"))
    digest = _digest(cus + hdrs, " ".join(NVCC_FLAGS))
    if not force and not _needs_build(target, digest):
        return target
    objs = []
    procs = []
    objdir = OUT / "obj"
    objdir.mkdir(exist_ok=True)
    for cu in cus:
        obj = objdir / (cu.stem + ".o")
        cmd = [_nvcc(), *NVCC_FLAGS, *( ["-Xptxas", "-v"] if ptxas_verbose else []), "-I", CSRC, "-c", cu, "-o", obj]
        if verbose:
            print("+", " ".join(map(str, cmd)), flush=True)
        procs.append((cu, subprocess.Popen(list(map(str, cmd)), stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
        objs.append(obj)
    for cu, proc in procs:
        out, _ = proc.communicate()
        if proc.returncode != 0:
            sys.stderr.write(out)
            raise RuntimeError(f"nvcc failed on {cu.name}")
        if (verbose or ptxas_verbose) and out:
            print(out)
    _run([_nvcc(), "-shared", "-o", target, *objs], verbose)
    target.with_suffix(".so.stamp").write_text(digest)
    return target


def build_host(force=False, verbose=False) -> Path:
    OUT.mkdir(exist_ok=True)
    target = OUT / "liblah_host.so"
    cpps = sorted(CSRC.glob("*.cpp"))
    hdrs = sorted(CSRC.glob("*.hpp"))
    if not cpps:
        return target
    digest = _digest(cpps + hdrs, " ".join(GXX_FLAGS))
    if not force and not _needs_build(target, digest):
        return target
    _run(["g++", *GXX_FLAGS, "-I", CSRC, "-o", target, *cpps], verbose)
    target.with_suffix(".so.stamp").write_text(digest)
    return target


def build_all(force=False, verbose=False):
    return build_cuda(force, verbose), build_host(force, verbose)


if __name__ == "__main__":
    force = "--force" in sys.argv
    c, h = build_cuda(force, verbose=True, ptxas_verbose="--ptxas" in sys.argv), build_host(force, verbose=True)
    print("built:", c, h)
