"""
InBoxNetwork — the in-box replacement of the Kademlia DHT (SURVEY.md §5.8 "DHT collapse").

Inside one NVSwitch box every expert is a known (owner rank, local slot); discovery is an O(1) lookup in a native hash
index (csrc/host_runtime.cpp ``lah_index_*``) and liveness is a heartbeat timestamp per expert and per uid prefix.
The class implements the SAME methods as ``TesseractNetwork`` (``declare_experts`` / ``get_experts`` /
``first_k_active``), so ``GatingFunction`` and ``TesseractServer`` run unchanged on top of it; additionally
``alive_mask(grid, prefix)`` exports the liveness table that the fused gate kernel reads (``EngineContext.alive``).
"""
import ctypes
import threading
import time
from typing import Dict, List, Optional, Sequence, Tuple

from ..ops import host

UID_DELIMETER = "."
HEARTBEAT_EXPIRATION = 120


class InBoxNetwork:
    UID_DELIMETER = UID_DELIMETER
    HEARTBEAT_EXPIRATION = HEARTBEAT_EXPIRATION
    make_key = "{}::{}".format

    def __init__(self, *initial_peers, port=None, start=True):
        self._lib = host.lib()
        self._index = self._lib.lah_index_create(1024) if self._lib is not None else None
        self._py: Dict[int, Tuple[int, int, float]] = {}
        self._endpoints: Dict[str, Tuple[str, int]] = {}
        self._lock = threading.Lock()
        self._alive = bool(start)
        self.fused_layer = None      # set by bind_engine(): GatingFunction then runs the sm_90a layer for CUDA inputs
        self._engine = None          # (ctx, cfg) of the bound in-box engine
        self._last_sync = 0.0
        self._ages_cache = (0.0, None)

    # ------------------------------------------------------------------ in-box engine binding
    def bind_engine(self, layer, sync_period: float = 1.0):
        """Attach a ``lah_b200.parallel.engine.FusedDMoE`` layer (or a ``DMoETrainer`` -> its first DMoE layer).

        * ``lib.GatingFunction(network=this, ...)`` called on a CUDA tensor then runs the fused layer (product-key gate with
          the GatingFunction's own ``proj``, P2P dispatch, wgmma expert FFN, combine; backward + expert AMSGrad);
        * ``declare_experts`` of uids that belong to the engine's grid and live on THIS rank stamps their heartbeat into the
          device-resident table of EVERY rank (multimem.st over NVSwitch), and the gate kernel's liveness mask is refreshed
          from that table at most every ``sync_period`` seconds — heartbeats reach the kernel without a host-side table;
        * ``get_experts`` / ``first_k_active`` answer for the experts of ALL ranks from the same table."""
        layer = getattr(layer, "model", layer)
        layer = layer.blocks[0] if hasattr(layer, "blocks") else layer
        assert getattr(layer, "ctx", None) is not None, "bind_engine needs a GPU FusedDMoE layer (EngineContext)"
        self.fused_layer, self._engine, self._sync_period = layer, (layer.ctx, layer.cfg), sync_period
        return self

    def _engine_index(self, uid: str) -> Optional[int]:
        """global expert id of ``uid`` in the bound engine's grid, or None"""
        if self._engine is None:
            return None
        _, cfg = self._engine
        parts = uid.split(self.UID_DELIMETER)
        nd = len(cfg.grid_size)
        if len(parts) != nd + 1 or self.UID_DELIMETER.join(parts[:-nd]) != cfg.uid_prefix:
            return None
        try:
            coords = [int(p) for p in parts[-nd:]]
        except ValueError:
            return None
        e = 0
        for c, size in zip(coords, cfg.grid_size):
            if not 0 <= c < size:
                return None
            e = e * size + c
        return e

    def sync_alive(self, heartbeat_expiration=HEARTBEAT_EXPIRATION, force: bool = True):
        """refresh the gate kernel's liveness mask from the device-resident heartbeat table (rate limited unless forced)"""
        if self._engine is None:
            return
        now = time.time()
        if force or now - self._last_sync >= self._sync_period:
            self._engine[0].refresh_alive(heartbeat_expiration, now)
            self._last_sync = now

    def _engine_age(self, e: int) -> float:
        now = time.time()
        if self._ages_cache[1] is None or now - self._ages_cache[0] > 0.2:
            self._ages_cache = (now, self._engine[0].heartbeat_ages(now))
        return float(self._ages_cache[1][e]) + (now - self._ages_cache[0])

    # process-like API of TesseractNetwork
    def start(self):
        self._alive = True

    def is_alive(self) -> bool:
        return self._alive

    def shutdown(self):
        self._alive = False

    def join(self, timeout=None):
        pass

    # ------------------------------------------------------------------ index primitives
    def _hash(self, kind: str, name: str) -> int:
        key = self.make_key(kind, name).encode()
        if self._lib is not None:
            return int(self._lib.lah_hash_bytes(key, len(key)))
        return hash(key) & (2 ** 63 - 1) or 1

    def _put(self, kind, name, owner=0, slot=0, now=None):
        now = time.time() if now is None else now
        h = self._hash(kind, name)
        if self._index is not None:
            self._lib.lah_index_put(self._index, h, owner, slot, now)
        else:
            with self._lock:
                self._py[h] = (owner, slot, now)

    def _fresh(self, kind, name, max_age) -> Optional[Tuple[int, int]]:
        h = self._hash(kind, name)
        if self._index is not None:
            owner, slot, hb = ctypes.c_int(), ctypes.c_int(), ctypes.c_double()
            ok = self._lib.lah_index_get(self._index, h, time.time(), float(max_age), ctypes.byref(owner),
                                         ctypes.byref(slot), ctypes.byref(hb))
            return (owner.value, slot.value) if ok else None
        with self._lock:
            entry = self._py.get(h)
        if entry is None or time.time() - entry[2] > max_age:
            return None
        return entry[0], entry[1]

    # ------------------------------------------------------------------ TesseractNetwork API
    def declare_experts(self, uids: Sequence[str], addr, port, wait_timeout=0, owner: int = 0, slots=None):
        now = time.time()
        if self._engine is not None:   # heartbeats of engine experts hosted here go to the device table of every rank
            ctx = self._engine[0]
            mine = sorted(e for e in (self._engine_index(uid) for uid in uids)
                          if e is not None and e // ctx.E_loc == ctx.rank)
            start = 0
            while start < len(mine):   # contiguous runs -> one launch each
                end = start
                while end + 1 < len(mine) and mine[end + 1] == mine[end] + 1:
                    end += 1
                ctx.heartbeat((mine[start], end - start + 1), now)
                start = end + 1
            self._ages_cache = (0.0, None)
        for i, uid in enumerate(uids):
            self._put("expert", uid, owner, slots[i] if slots is not None else i, now)
            with self._lock:
                self._endpoints[uid] = (addr, port)
            parts = uid.split(self.UID_DELIMETER)
            for j in range(len(parts)):
                self._put("prefix", self.UID_DELIMETER.join(parts[:j + 1]), owner, 0, now)

    def get_experts(self, uids: List[str], heartbeat_expiration=HEARTBEAT_EXPIRATION):
        from ..client.remote_expert import RemoteExpert
        out = []
        for uid in uids:
            hit = self._fresh("expert", uid, heartbeat_expiration)
            if hit is None and self._engine is not None:   # an expert of another rank: device-resident table
                e = self._engine_index(uid)
                if e is not None and self._engine_age(e) <= heartbeat_expiration:
                    hit = (e // self._engine[0].E_loc, e % self._engine[0].E_loc)
            if hit is None:
                out.append(None)
            else:
                host_, port = self._endpoints.get(uid, ("127.0.0.1", 0))
                out.append(RemoteExpert(uid=uid, host=host_, port=port))
        return out

    def first_k_active(self, prefixes: List[str], k: int, heartbeat_expiration=HEARTBEAT_EXPIRATION, max_prefetch=None):
        active = []
        for prefix in prefixes:
            if self._fresh("prefix", prefix, heartbeat_expiration) is not None:
                active.append(prefix)
                if len(active) >= k:
                    break
        return active

    # ------------------------------------------------------------------ export for the gate kernel
    def alive_mask(self, grid_size: Sequence[int], uid_prefix: str, heartbeat_expiration=HEARTBEAT_EXPIRATION):
        """uint8 tensor [prod(grid)] (row-major expert index): 1 where the expert's heartbeat is fresh"""
        import itertools
        import torch
        flags = []
        for coords in itertools.product(*(range(g) for g in grid_size)):
            uid = self.UID_DELIMETER.join([uid_prefix] + [str(c) for c in coords])
            flags.append(1 if self._fresh("expert", uid, heartbeat_expiration) is not None else 0)
        return torch.tensor(flags, dtype=torch.uint8)

    def __del__(self):
        if getattr(self, "_index", None) is not None and self._lib is not None:
            self._lib.lah_index_destroy(self._index)
            self._index = None
