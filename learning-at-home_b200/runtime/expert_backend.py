"""
ExpertBackend — how one expert processes forward / backward tasks on the server
(API parity: /root/reference/lib/runtime/expert_backend.py:10-104).

Semantics kept from the reference:
  * ``forward(*flat_inputs)`` runs the expert under ``no_grad`` and returns a flat tuple of outputs;
  * ``backward(*flat_inputs, *flat_grad_outputs)`` re-runs the forward with grad enabled on detached inputs,
    back-propagates, applies the optimizer IMMEDIATELY (one asynchronous step per backward batch) and returns the
    gradients w.r.t. every input (zeros where an input received no gradient);
  * ``state_dict()`` keys are ``expert.<param>``; the optimizer is a plain attribute;
  * ``get_info()`` -> dict(forward_schema, outputs_schema, keyword_names).

Differences: inputs are never mutated (the reference's transformer block transposes its input in place, which makes
``backward`` raise — SURVEY.md §0.3); the inferred ``outputs_schema`` does not capture ``requires_grad``/device of the
dummy run; ``checkpoint()`` / ``load_checkpoint()`` give the uid-addressed layout of SURVEY.md §5.4.
"""
from typing import Any, Dict, Sequence, Tuple, Union

import torch
from torch import nn

from .task_pool import TaskPool
from ..utils import BatchTensorProto, DUMMY_BATCH_SIZE, nested_compare, nested_flatten, nested_map, nested_pack


class ExpertBackend(nn.Module):
    def __init__(self, name: str, expert: nn.Module, opt: torch.optim.Optimizer, *,
                 args_schema: Tuple[BatchTensorProto, ...] = None, kwargs_schema: Dict[str, BatchTensorProto] = None,
                 outputs_schema: Union[BatchTensorProto, Tuple[BatchTensorProto, ...]] = None, native: bool = True,
                 **kwargs):
        """:param native: run experts that live on a CUDA device in fp32 through the sm_90a kernels
        (runtime/native_executor.py) instead of eager PyTorch, with ``torch.optim.Adam`` or ``torch.optim.AdamW`` whose
        param groups hold every parameter of the expert once (per group any lr, betas, eps, weight_decay, amsgrad and
        decoupled_weight_decay; ``maximize``, ``capturable``, ``differentiable``, tensor lr / betas and other optimizers
        run on the module).  These modules run natively, plain or ``torch.jit.script``-ed:
          * ``FeedforwardBlock(hid)`` with hid a multiple of 128 up to 1024 (swap-AB wgmma GEMMs, fused LayerNorm, fused
            weight-gradient + AMSGrad);
          * this package's ``TransformerEncoderLayer`` and ``torch.nn.TransformerEncoderLayer`` with ReLU or erf GELU,
            ``norm_first`` True or False, ``batch_first`` True or False, LayerNorm eps 1e-5 and all biases, head dim
            d_model / nhead in (32, 64, 128), d_model a multiple of 128 with 256 <= d_model <= 4096, dim_feedforward a
            multiple of 128, dropout p < 1 at every site, sequence length 1 <= S <= 65536 (wgmma attention and GEMMs,
            in-kernel dropout, fused AMSGrad).  This package's layer with ``causal=True`` (position t attends to
            positions <= t) runs natively under the same conditions, on the causal attention kernels;
          * ``GatedFeedforwardBlock(hid, inner)`` (the SwiGLU expert MLP with its RMSNorm pre-norm and residual) with hid
            a multiple of 128 in [128, 4096], inner any multiple of 128 (so up to hid 4096, inner 11008), no biases, an
            RMSNorm with a weight, ``normalized_shape`` (hid,) and any eps > 0 (RMSNorm and SwiGLU kernels, one swap-AB GEMM
            and one fused weight-gradient + AMSGrad launch over the adjacent [W1; W3]).
        ``torch.nn.TransformerEncoderLayer`` also runs natively with a key padding mask: one positional input and
        ``kwargs_schema={"src_key_padding_mask": BatchTensorProto(S, dtype=torch.bool)}`` (True = padding key, [batch, S]
        for sequence-first layers too).  The flat inputs are then (src, mask) for forward and (src, mask, grad_out) for
        backward, which returns (dx, zeros_like(mask)), as on the module.  A sequence whose keys are all masked gets the
        result of torch's layer in training mode (zero attention output) in eval mode too; torch's eval fast path returns
        NaN for it.
        Anything else (another class, tanh GELU, kdim / vdim, bias=False in the encoder layers, biases in the gated block,
        other widths or inputs, float masks, other keyword inputs, CPU tensors) runs on the module itself"""
        super().__init__()
        self.expert, self.opt, self.name = expert, opt, name
        self.native, self._executor, self._executor_key = native, None, None
        self.args_schema = args_schema = tuple(args_schema or ())
        self.kwargs_schema = kwargs_schema = dict(kwargs_schema or {})
        assert args_schema or kwargs_schema, ("expert must receive at least one positional or keyword input. "
                                              "Did you forget to provide args_schema/kwargs_schema?")
        if outputs_schema is None:
            # one throw-away run to learn what the expert returns
            with torch.no_grad():
                dummy_args = tuple(proto.make_empty(DUMMY_BATCH_SIZE).zero_() for proto in args_schema)
                dummy_kwargs = {k: proto.make_empty(DUMMY_BATCH_SIZE).zero_() for k, proto in kwargs_schema.items()}
                dummy_out = self.expert(*dummy_args, **dummy_kwargs)
            outputs_schema = nested_map(lambda t: BatchTensorProto(*t.shape[1:], dtype=t.dtype), dummy_out)
        self.forward_schema = (self.args_schema, self.kwargs_schema)
        self.outputs_schema = outputs_schema
        self.backward_schema = (self.forward_schema, self.outputs_schema)  # original inputs + grads w.r.t. outputs
        self.forward_pool = TaskPool(self.forward, inputs_schema=tuple(nested_flatten(self.forward_schema)),
                                     outputs_schema=tuple(nested_flatten(self.outputs_schema)),
                                     uid=f"{self.name}_forward", **kwargs)
        self.backward_pool = TaskPool(self.backward, inputs_schema=tuple(nested_flatten(self.backward_schema)),
                                      outputs_schema=tuple(nested_flatten(self.forward_schema)),
                                      uid=f"{self.name}_backward", **kwargs)
        self.update_count = 0

    # ------------------------------------------------------------------ tasks
    def _key_padding_schema(self) -> bool:
        """True when the keyword inputs are exactly a bool key padding mask [batch, S]"""
        proto = self.kwargs_schema.get("src_key_padding_mask")
        return (len(self.kwargs_schema) == 1 and proto is not None and len(proto.size) == 2
                and proto == BatchTensorProto(proto.size[1], dtype=torch.bool))

    def native_executor(self, inputs):
        """the sm_90a executor of this expert, or None (CPU tensors, unsupported expert / optimizer / keyword inputs, no
        GPU).  Inputs the executor does not accept (``executor.accepts``: rank, feature size, sequence length, mask shape)
        run on the module itself."""
        if not self.native or len(inputs) < 1 or not inputs[0].is_cuda or len(self.args_schema) != 1:
            return None
        if self.kwargs_schema and not self._key_padding_schema():
            return None
        first = next(self.expert.parameters(), None)
        key = (id(first), first.device if first is not None else None)
        if self._executor_key != key:   # (re)build after .to(device) / load_checkpoint
            from .native_executor import make_executor
            self._executor, self._executor_key = make_executor(self.expert, self.opt), key
            if self._executor is not None:
                self._executor_key = (id(next(self.expert.parameters())), first.device)
        if self.kwargs_schema and not getattr(self._executor, "takes_key_padding_mask", False):
            return None
        return self._executor

    def forward(self, *inputs: torch.Tensor) -> Tuple[torch.Tensor, ...]:
        executor = self.native_executor(inputs)
        mask = inputs[1:2] if self.kwargs_schema else ()   # (src_key_padding_mask,) when the schema has it
        if executor is not None and len(inputs) == 1 + len(mask) and executor.accepts(inputs[0], *mask):
            return (executor.forward(inputs[0], *mask),)
        args, kwargs = nested_pack(inputs, structure=self.forward_schema)
        with torch.no_grad():
            outputs = self.expert(*args, **kwargs)
        return tuple(nested_flatten(outputs))

    def backward(self, *inputs: torch.Tensor) -> Tuple[torch.Tensor, ...]:
        executor = self.native_executor(inputs)
        mask = inputs[1:2] if self.kwargs_schema else ()
        n = 1 + len(mask)
        if executor is not None and len(inputs) == n + 1 and executor.accepts(inputs[0], *mask):
            # dgrad + fused wgrad/AMSGrad: one update
            grad_x = executor.backward(inputs[0], inputs[n].to(inputs[0].device), *mask)
            self.update_count += 1
            return (grad_x, *(torch.zeros_like(m) for m in mask))
        (args, kwargs), grad_outputs = nested_pack(inputs, structure=self.backward_schema)
        with torch.enable_grad():
            args = [t.detach().clone().requires_grad_(t.is_floating_point()) for t in args]
            kwargs = {k: t.detach().clone().requires_grad_(t.is_floating_point()) for k, t in kwargs.items()}
            outputs = self.expert(*args, **kwargs)
            assert nested_compare(outputs, grad_outputs), "outputs and grad_outputs must have the same structure"
            flat_out = tuple(nested_flatten(outputs))
            flat_grads = tuple(g.to(device=o.device, dtype=o.dtype, non_blocking=True)
                               for g, o in zip(nested_flatten(grad_outputs), flat_out))
            torch.autograd.backward(flat_out, grad_tensors=flat_grads, create_graph=False, retain_graph=False)
            self.apply_gradients()
        return tuple(x.grad if isinstance(x.grad, torch.Tensor) else torch.zeros_like(x)
                     for x in nested_flatten((args, kwargs)))

    def apply_gradients(self) -> None:
        """one optimizer step per backward batch (asynchronous per-expert SGD, as in the reference)"""
        self.opt.step()
        self.opt.zero_grad()
        self.update_count += 1

    # ------------------------------------------------------------------ introspection
    def get_pools(self) -> Sequence[TaskPool]:
        return self.forward_pool, self.backward_pool

    def get_info(self) -> Dict[str, Any]:
        # tensor_wire: this server also understands raw-tensor frames (utils/tensor_wire.py); reference clients ignore it
        return dict(forward_schema=self.forward_schema, outputs_schema=self.outputs_schema,
                    keyword_names=tuple(self.kwargs_schema.keys()), tensor_wire=1)

    # ------------------------------------------------------------------ checkpoints (absent in the reference)
    def checkpoint(self) -> Dict[str, Any]:
        return dict(uid=self.name, model={k: v.detach().cpu() for k, v in self.state_dict().items()},
                    optimizer=self.opt.state_dict(), update_count=self.update_count)

    def load_checkpoint(self, ckpt: Dict[str, Any]) -> None:
        self.load_state_dict(ckpt["model"])
        self.opt.load_state_dict(ckpt["optimizer"])
        self.update_count = int(ckpt.get("update_count", 0))
        if self._executor is not None:   # the optimizer now owns fresh state tensors: re-bind them to the flat buffers
            self._executor.bind()
