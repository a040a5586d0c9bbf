"""
ctypes bindings for the in-tree native libraries (built by ``build_native.py``):

* ``liblah_cuda.so`` — hand-written sm_90a kernels (wgmma grouped GEMM, LayerNorm/ReLU, gate/top-k, P2P dispatch /
  combine, fused Adam, symmetric-heap helpers).  Loading it REQUIRES a CUDA device at call time; on a GPU box a missing
  library is a hard error (``cuda_lib()`` raises) — there is no silent PyTorch fallback on the GPU hot path.
* ``liblah_host.so`` — C++ host runtime (batch former, wire framing, DHT routing table); usable on CPU-only machines.
"""
import ctypes
import os
import threading
from pathlib import Path

import torch

_PKG = Path(__file__).resolve().parent.parent
_LOCK = threading.Lock()
_CUDA = None
_HOST = None

c_void_p, c_int, c_ll, c_float = ctypes.c_void_p, ctypes.c_int, ctypes.c_longlong, ctypes.c_float


class NativeError(RuntimeError):
    pass


def _load(name, builder):
    path = _PKG / "_C" / name
    if not path.exists() or os.environ.get("LAH_REBUILD"):
        from .. import build_native
        getattr(build_native, builder)()
    if not path.exists():
        raise NativeError(f"{path} is missing and could not be built")
    return ctypes.CDLL(str(path))


def cuda_lib():
    global _CUDA
    if _CUDA is None:
        with _LOCK:
            if _CUDA is None:
                _CUDA = _load("liblah_cuda.so", "build_cuda")
    return _CUDA


def host_lib():
    global _HOST
    if _HOST is None:
        with _LOCK:
            if _HOST is None:
                _HOST = _load("liblah_host.so", "build_host")
    return _HOST


def have_cuda_kernels() -> bool:
    """True when the sm_90a kernels can actually run here (GPU present).  On a GPU box this also loads the library,
    so a broken build fails loudly instead of silently taking a PyTorch path."""
    if not torch.cuda.is_available():
        return False
    cuda_lib()
    return True


def ptr(t):
    """device/host pointer of a tensor (None -> NULL)"""
    if t is None:
        return c_void_p(0)
    return c_void_p(t.data_ptr())


def stream_ptr(stream=None):
    s = stream if stream is not None else torch.cuda.current_stream()
    return c_void_p(s.cuda_stream)


def check(code: int, what: str):
    if code != 0:
        raise NativeError(f"{what} failed with code {code}")


# kernel launch counter (bench.py reports it as gpu_launches)
_launches = 0


def count_launch(n=1):
    global _launches
    _launches += n


def launches() -> int:
    return _launches


def reset_launches():
    global _launches
    _launches = 0
