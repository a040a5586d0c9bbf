"""
GatingFunction — the trainer-side DMoE layer: product-key gating, beam search over alive experts, fan-out to the chosen
experts, softmax-weighted combine over the experts that responded
(API parity: /root/reference/lib/client/gating_function.py:14-153).

Two execution paths behind one module:

* **fused in-box path** — when ``network`` is bound to an in-box engine layer (``network.fused_layer``, see
  ``lah_b200.parallel.engine.FusedDMoE``) and the input lives on that GPU, the whole layer (top-k, dispatch, expert FFN,
  combine; and their backward + expert optimizer) runs in the sm_90a kernels; ``self.proj`` is the gate in both paths.
* **generic path** — any ``TesseractNetwork``-like object + ``RemoteExpert`` RPCs.  Same results as the reference, but
  rows are grouped PER EXPERT: one forward RPC per chosen expert carrying all of its rows (the reference issues one RPC
  per (sample, expert) with a single row and relies on the server to re-batch).  Fault tolerance is unchanged: experts
  that fail or miss the deadline are dropped and the softmax renormalises over the responders; a sample with fewer than
  ``k_min`` responders fails the batch.

Fixed quirks (SURVEY.md §7.4): ``expert_padding=None`` no longer crashes when fewer than k_best prefixes are alive;
the return annotation matches what is returned.
"""
import threading
import time
from functools import partial
from multiprocessing.pool import ThreadPool
from typing import Any, Dict, List, Optional, Sequence, Tuple

import numpy as np
import torch
import torch.nn as nn

from .remote_expert import RemoteExpert
from ..utils import check_numpy, nested_flatten, nested_map, nested_pack, run_and_await_k


class GatingFunction(nn.Module):
    def __init__(self, *, in_features, grid_size: Sequence[int], network, num_workers=None, k_best, k_min=1,
                 timeout_after_k_min=1.0, uid_prefix="", expert_padding=None):
        super().__init__()
        self.network, self.grid_size = network, tuple(grid_size)
        self.uid_prefix, self.expert_padding = uid_prefix, expert_padding
        self.k_best, self.k_min, self.timeout_after_k_min = k_best, k_min, timeout_after_k_min
        self.thread_pool = ThreadPool(num_workers or k_best * 2)
        self.proj = nn.Linear(in_features, sum(self.grid_size))  # jointly predicts the logits of all grid dimensions

    def close(self):
        pool, self.thread_pool = getattr(self, "thread_pool", None), None
        if pool is not None:
            try:
                pool.terminate()
            except Exception:  # noqa: interpreter shutdown
                pass

    def __del__(self):
        self.close()

    # ------------------------------------------------------------------ forward
    def forward(self, input: torch.Tensor, *args, **kwargs) -> torch.Tensor:
        """
        Choose the k best alive experts per sample, call them, and mix their outputs with softmax weights computed over
        the experts that DID respond.
        :param input: [batch, in_features]; extra *args / **kwargs are batch-first tensors forwarded to the experts
        """
        assert input.dim() == 2
        fused = getattr(self.network, "fused_layer", None)
        if fused is not None and input.is_cuda and not args and not kwargs:
            # in-box fast path (InBoxNetwork.bind_engine): liveness comes from the device-resident heartbeat table, the whole
            # layer runs in the sm_90a kernels; k_min / timeout_after_k_min map to DMoEConfig.peer_timeout_ms
            self.network.sync_alive(force=False)
            return fused.forward_with_gate(input, self.proj)

        grid_scores = self.proj(input).split_with_sizes(self.grid_size, dim=-1)
        batch_experts = self.beam_search(grid_scores, self.k_best)  # List[batch] of List[RemoteExpert]
        expert_logits = self._score_experts(grid_scores, batch_experts)  # List[batch] of {expert: logit}
        outputs_by_sample = self._call_experts_grouped(batch_experts, input, args, kwargs)

        mixed = []
        for sample_outputs, logits in zip(outputs_by_sample, expert_logits):
            experts = list(sample_outputs.keys())
            weights = torch.softmax(torch.stack([logits[e] for e in experts]), dim=-1)
            mixed.append(nested_map(lambda *tensors: sum(t * w for t, w in zip(tensors, weights)),
                                    *[sample_outputs[e] for e in experts]))
        return nested_map(lambda *tensors: torch.cat(tensors, dim=0), *mixed)

    # ------------------------------------------------------------------ expert calls (grouped per expert)
    def _call_experts_grouped(self, batch_experts: List[List[RemoteExpert]], input, args, kwargs):
        """returns List[batch] of {expert: nested output with a leading dim of 1} for the experts that responded"""
        batch_size = len(batch_experts)
        rows_of: Dict[RemoteExpert, List[int]] = {}
        for i, chosen in enumerate(batch_experts):
            for expert in chosen:
                rows_of.setdefault(expert, []).append(i)
        for i, chosen in enumerate(batch_experts):
            if len(chosen) < self.k_min:
                raise ValueError(f"Could not get enough results: sample {i} has only {len(chosen)} alive experts.")
        experts = list(rows_of.keys())
        results: Dict[RemoteExpert, Any] = {}
        successes = np.zeros(batch_size, dtype=np.int64)
        outstanding = np.array([len(chosen) for chosen in batch_experts], dtype=np.int64)
        cv = threading.Condition()

        def job(expert):
            rows = torch.as_tensor(rows_of[expert], device=input.device)
            try:
                out = expert(input[rows], *(t[rows] for t in args), **{k: t[rows] for k, t in kwargs.items()})
                ok = True
            except Exception as e:  # noqa: failed experts are simply dropped
                out, ok = e, False
            with cv:
                if ok:
                    results[expert] = out
                    successes[rows_of[expert]] += 1
                outstanding[rows_of[expert]] -= 1
                cv.notify_all()

        for expert in experts:
            threading.Thread(target=job, args=(expert,), daemon=True).start()

        def satisfied():
            return bool(np.all(successes >= self.k_min))

        def hopeless():
            return bool(np.any(successes + outstanding < self.k_min))

        with cv:
            while not satisfied() and not hopeless():
                cv.wait()
            if satisfied() and outstanding.any():
                deadline = time.monotonic() + self.timeout_after_k_min
                while outstanding.any():
                    remaining = deadline - time.monotonic()
                    if remaining <= 0:
                        break
                    cv.wait(remaining)
            if not satisfied():
                raise ValueError("Could not get enough results: too many jobs failed.")
            done = dict(results)

        per_sample: List[Dict[RemoteExpert, Any]] = [dict() for _ in range(batch_size)]
        for expert, out in done.items():
            for j, i in enumerate(rows_of[expert]):
                per_sample[i][expert] = nested_map(lambda t: t[j: j + 1], out)
        return per_sample

    def _run_experts(self, experts: List[RemoteExpert], *args, **kwargs) -> Dict[RemoteExpert, torch.Tensor]:
        """call several experts on the same inputs; {expert: output} for those that succeeded in time"""
        outputs = run_and_await_k([partial(expert, *args, **kwargs) for expert in experts], k=self.k_min,
                                  timeout_after_k=self.timeout_after_k_min)
        return {expert: out for expert, out in zip(experts, outputs) if not isinstance(out, BaseException)}

    # ------------------------------------------------------------------ beam search over the product grid
    def beam_search(self, grid_scores: Sequence[torch.Tensor], k_best: int, **kwargs) -> List[List[RemoteExpert]]:
        """
        Beam search (width k_best) over the grid with liveness filtering at every dimension, like the reference's.  With
        additive scores it returns the exact top-k whenever liveness prunes nothing; with holes in the grid it is a heuristic
        (a live prefix may win a level and have only poor descendants) — the fused in-box gate scores all alive experts.
        :param grid_scores: per grid dimension, a [batch, grid_size[d]] tensor of scores
        :returns: per sample, up to k_best alive RemoteExperts ordered by decreasing total score
        """
        assert len(grid_scores) == len(self.grid_size)
        batch_size = len(grid_scores[0])
        delimeter = self.network.UID_DELIMETER
        beams: List[List[Tuple[str, float]]] = [[(self.uid_prefix, 0.0)] for _ in range(batch_size)]
        for dim, dim_scores in enumerate(grid_scores):
            dim_scores = check_numpy(dim_scores).astype(np.float64)
            assert dim_scores.shape == (batch_size, self.grid_size[dim])
            lookups, tables = [], []
            for b in range(batch_size):
                prefixes = [p for p, _ in beams[b]]
                scores = np.array([s for _, s in beams[b]])[:, None] + dim_scores[b][None, :]
                order = np.argsort(-scores, axis=None, kind="stable")
                cands = [prefixes[i // self.grid_size[dim]] + delimeter + str(i % self.grid_size[dim]) for i in order]
                tables.append(dict(zip(cands, scores.reshape(-1)[order])))
                lookups.append(self.thread_pool.apply_async(self.network.first_k_active, args=(cands, k_best), kwds=kwargs))
            beams = [[(prefix, float(table[prefix])) for prefix in lookup.get()]
                     for lookup, table in zip(lookups, tables)]
        uids = sorted({uid for beam in beams for uid, _ in beam})
        found = self.network.get_experts(uids) if uids else []
        by_uid = {uid: expert for uid, expert in zip(uids, found) if expert is not None}
        return [[by_uid[uid] for uid, _ in beam if uid in by_uid] for beam in beams]

    # ------------------------------------------------------------------ differentiable scores of the chosen experts
    def _score_experts(self, grid_scores: Sequence[torch.Tensor],
                       experts: List[List[RemoteExpert]]) -> List[Dict[RemoteExpert, torch.Tensor]]:
        flat_experts = [expert for row in experts for expert in row]
        device = grid_scores[0].device
        batch_idx = torch.tensor([i for i, row in enumerate(experts) for _ in row], dtype=torch.long, device=device)
        skip = len(self.uid_prefix) + len(self.network.UID_DELIMETER)
        grid_idx = np.zeros((len(flat_experts), len(grid_scores)), dtype=np.int64)
        for i, expert in enumerate(flat_experts):
            grid_idx[i] = [int(part) for part in expert.uid[skip:].split(self.network.UID_DELIMETER)]
        if len(flat_experts):
            flat_scores = sum(dim_scores[batch_idx, torch.as_tensor(grid_idx[:, d], device=device)]
                              for d, dim_scores in enumerate(grid_scores))
        else:
            flat_scores = torch.zeros(0, device=device)
        out: List[Dict[RemoteExpert, torch.Tensor]] = [dict() for _ in experts]
        for i, expert, score in zip(batch_idx.tolist(), flat_experts, flat_scores):
            out[i][expert] = score
        return out
