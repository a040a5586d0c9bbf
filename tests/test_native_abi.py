"""The ctypes bindings of ops/ agree with the C entry points of csrc/: a wrong argument list only shows on the GPU, as a
corrupted launch or a device fault, so the parameter counts are checked here on the CPU."""
import glob
import os
import re

import pytest

import lah_b200  # noqa
from lah_b200 import build_native

CSRC = os.path.join(os.path.dirname(os.path.abspath(build_native.__file__)), "csrc")


def _c_entry_points():
    """name -> parameter count of every lah_* function defined in csrc/*.cu"""
    defs = {}
    for path in glob.glob(os.path.join(CSRC, "*.cu")):
        with open(path) as f:
            src = f.read()
        for name, params in re.findall(r"\b(lah_\w+)\(([^()]*)\)\s*\{", src):
            assert name not in defs, f"{name} defined twice"
            defs[name] = 0 if params.strip() in ("", "void") else params.count(",") + 1
    return defs


def test_ctypes_bindings_match_c_entry_points():
    try:
        build_native._nvcc()
    except RuntimeError:
        pytest.skip("nvcc not found")
    from lah_b200.ops import fp8, gemm, kernels, native
    build_native.build_cuda()
    for module in (gemm, kernels, fp8):
        module._lib()
    bound = {n: f.argtypes for n, f in vars(native.cuda_lib()).items() if n.startswith("lah_") and f.argtypes is not None}
    defs = _c_entry_points()
    assert len(bound) > 40
    bad = {n: (len(a), defs.get(n)) for n, a in bound.items() if defs.get(n) != len(a)}
    assert not bad, f"binding: (ctypes argtypes, C parameters): {bad}"
