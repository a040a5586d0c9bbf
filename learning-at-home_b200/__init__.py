"""
lah_b200 — a Hopper-native Decentralized Mixture-of-Experts engine with the public API of mryab/learning-at-home.

    import lah_b200 as lib                      # or `import lib` (compat alias at the repository root)
    lib.RemoteExpert, lib.GatingFunction        # trainer side           (client/)
    lib.TesseractServer, lib.ExpertBackend      # expert server          (server/, runtime/)
    lib.TesseractNetwork, lib.InBoxNetwork      # discovery              (network/)
    lib.DMoETrainer, lib.DMoEConfig, lib.FusedDMoE   # sm_90a in-box engine (parallel/)

See README.md and DESIGN.md.
"""
__version__ = "0.1.0"

from .utils import *  # noqa: F401,F403
from . import utils, client, runtime, server, network, models, ops, parallel  # noqa: F401
from .client import RemoteExpert, GatingFunction
from .runtime import ExpertBackend, TesseractRuntime, TaskPool, TaskPoolBase
from .server import TesseractServer
from .network import TesseractNetwork, InBoxNetwork
from .parallel.engine import DMoEConfig, FusedDMoE, DMoEClassifier, ExpertShard
from .parallel.trainer import DMoETrainer
