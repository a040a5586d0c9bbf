"""
``lib`` — drop-in name of the reference package (``import lib`` in README snippets and experiment scripts of
mryab/learning-at-home).  Everything is implemented in ``lah_b200`` (directory ``learning-at-home_b200/``); this module
only re-exports the public surface: lib.RemoteExpert, lib.GatingFunction, lib.TesseractServer, lib.TesseractNetwork,
lib.ExpertBackend, lib.TesseractRuntime, lib.TaskPool, lib.BatchTensorProto, the lib.utils helpers and the expert
blocks of lib.models (FeedforwardBlock, GatedFeedforwardBlock, TransformerEncoderLayer).
"""
import sys as _sys

import lah_b200 as _pkg
from lah_b200.utils import *  # noqa: F401,F403
from lah_b200 import utils  # noqa: F401

_sys.modules.setdefault("lib.utils", utils)
for _name in ("client", "runtime", "server", "network", "models"):
    try:
        _mod = __import__(f"lah_b200.{_name}", fromlist=["*"])
    except ImportError:  # pragma: no cover - partially built tree
        continue
    _sys.modules.setdefault(f"lib.{_name}", _mod)
    globals()[_name] = _mod
    for _attr in getattr(_mod, "__all__", ()):
        globals()[_attr] = getattr(_mod, _attr)
