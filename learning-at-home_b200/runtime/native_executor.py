"""
NativeFFNExecutor — runs ``ExpertBackend.forward`` / ``ExpertBackend.backward`` of a ``FeedforwardBlock`` expert on the
hand-written sm_90a kernels instead of eager PyTorch, so that a ``TesseractServer``'s runtime loop
(the reference's lib/runtime/__init__.py:42-47 -> lib/runtime/expert_backend.py:64-97) executes wgmma code:

  forward   swap-AB grouped linear (weights streamed once per 128 rows, csrc/small_m.cu) x 3 + fused LayerNorm+ReLU x 2
  backward  the reference semantics — recompute the forward from the inputs the client re-sent, back-propagate, step the
            expert's optimizer immediately, return the gradients w.r.t. the inputs — with swap-AB dgrads, the LayerNorm
            backward kernel and the FUSED weight-gradient + AMSGrad kernel (the gradient of a weight matrix never reaches HBM)

NativeGatedFFNExecutor does the same for a ``GatedFeedforwardBlock`` (RMSNorm, one GEMM over [W1; W3], SwiGLU, W2) and
NativeTransformerExecutor for encoder layers.
The module's parameters and the torch optimizer's state tensors are re-bound as VIEWS of the executor's flat fp32 buffers:
``expert.state_dict()``, ``opt.state_dict()`` and ``ExpertBackend.checkpoint()`` stay live and keep the reference layout.
"""
import re
from typing import List, NamedTuple, Optional, Tuple

import torch
import torch.nn.functional as F

from ..models.layers import (FFN_SEG_KEYS, FFN_SEG_NAMES, FFN_SMALL_SEG_MASK, FeedforwardBlock, GatedFeedforwardBlock,
                              TransformerEncoderLayer)
from ..ops import kernels as K, native
from ..ops.expert_blocks import RowPlan, ffn_backward, ffn_forward, swiglu_mlp_backward, swiglu_mlp_forward

TORCH_ENCODER_LAYER = "torch.nn.modules.transformer.TransformerEncoderLayer"
OWN_ENCODER_LAYER = "lah_b200.models.layers.TransformerEncoderLayer"
OWN_FFN = "lah_b200.models.layers.FeedforwardBlock"
OWN_GATED_FFN = "lah_b200.models.layers.GatedFeedforwardBlock"
LN_EPS = 1e-5   # the LayerNorm epsilon compiled into csrc/layernorm.cu


def class_name(module) -> str:
    """qualified name of the class a module was built from: for a ``torch.jit.script`` module that of its original class
    (TorchScript's ``__torch__.`` prefix and ``___torch_mangle_N.`` parts removed).  Subclasses of this package's layers
    report the layer they extend, as ``isinstance`` would; any other class reports itself, so a subclass of a torch layer
    that overrides ``forward`` is not mistaken for it."""
    if type(module) is torch.jit.RecursiveScriptModule:
        name = module._c._type().qualified_name()
        return re.sub(r"___torch_mangle_\d+\.", "", name[len("__torch__."):] if name.startswith("__torch__.") else name)
    for own in (TransformerEncoderLayer, FeedforwardBlock, GatedFeedforwardBlock):
        if isinstance(module, own):
            return f"{own.__module__}.{own.__qualname__}"
    return f"{type(module).__module__}.{type(module).__qualname__}"


class FFNSpec(NamedTuple):
    hid: int
    inner: int


class EncoderLayerSpec(NamedTuple):
    d: int
    heads: int
    ff: int
    norm_first: bool         # pre-LN: h = x + attn(LN1(x)), y = h + ffn(LN2(h)); post-LN: LN2(x1 + ffn(x1)), x1 = LN1(x + attn(x))
    activation: str          # "relu" or "gelu" (erf)
    batch_first: bool        # interface layout: [B, S, d] or [S, B, d]
    ps: Tuple[float, float, float, float]   # drop probabilities of sites 0-3: attention, dropout1, dropout, dropout2
    causal: bool = False     # position t attends to positions <= t (this package's layer with causal=True)


def ffn_spec(module) -> Optional[FFNSpec]:
    """what NativeFFNExecutor needs of a FeedforwardBlock (plain or scripted), or None for any other module"""
    if class_name(module) != OWN_FFN:
        return None
    return FFNSpec(module.layers[0].in_features, module.layers[0].out_features)


class GatedFFNSpec(NamedTuple):
    hid: int
    inner: int
    eps: float


def gated_ffn_spec(module) -> Optional[GatedFFNSpec]:
    """what NativeGatedFFNExecutor needs of a GatedFeedforwardBlock (plain or scripted), or None when it cannot run it:
    refused are a Linear with a bias, an RMSNorm without a weight, an eps that is None or <= 0, a ``normalized_shape``
    other than (hid,), and every other class"""
    if class_name(module) != OWN_GATED_FFN:
        return None
    norm, w1, w2, w3 = module.norm, module.w1, module.w2, module.w3
    if any(lin.bias is not None for lin in (w1, w2, w3)) or norm.weight is None:
        return None
    if norm.eps is None or not float(norm.eps) > 0:
        return None
    hid, inner = int(w1.in_features), int(w1.out_features)
    if tuple(norm.normalized_shape) != (hid,):
        return None
    return GatedFFNSpec(hid, inner, float(norm.eps))


def _activation(layer) -> Optional[str]:
    """"relu" / "gelu" for the activations the executor implements, None for any other (tanh GELU included)"""
    act = getattr(layer, "activation", None)
    if act is None:   # a scripted layer does not keep a function activation as an attribute: F.relu -> 1, F.gelu -> 2
        return {1: "relu", 2: "gelu"}.get(int(layer.activation_relu_or_gelu))
    if act is F.relu or class_name(act) == "torch.nn.modules.activation.ReLU":
        return "relu"
    if act is F.gelu or (class_name(act) == "torch.nn.modules.activation.GELU" and act.approximate == "none"):
        return "gelu"
    return None


def encoder_layer_spec(module) -> Optional[EncoderLayerSpec]:
    """
    What NativeTransformerExecutor needs of an encoder layer, or None when it cannot run it.  Accepted, plain or
    ``torch.jit.script``-ed: this package's TransformerEncoderLayer (batch-first, post-LN, GELU, ``causal`` read from the
    module) and
    torch.nn.TransformerEncoderLayer with either ``norm_first`` and ``batch_first``, ReLU or erf GELU.  Refused: any other
    activation (tanh GELU too), a LayerNorm eps other than 1e-5, missing biases or LayerNorm affine parameters, ``kdim`` /
    ``vdim`` other than d_model, ``add_bias_kv``, ``add_zero_attn``, and every other class.
    """
    name = class_name(module)
    if name == OWN_ENCODER_LAYER:
        norm_first, activation, batch_first, causal = False, "gelu", True, bool(module.causal)
    elif name == TORCH_ENCODER_LAYER:   # is_causal is an argument of its forward, not of the layer: never causal here
        norm_first, activation, batch_first = bool(module.norm_first), _activation(module), bool(module.self_attn.batch_first)
        causal = False
        if activation is None:
            return None
    else:
        return None
    attn = module.self_attn
    if not attn._qkv_same_embed_dim or attn.bias_k is not None or attn.add_zero_attn:
        return None
    linears = (attn.out_proj, module.linear1, module.linear2)
    norms = (module.norm1, module.norm2)
    if attn.in_proj_bias is None or any(m.bias is None for m in linears + norms) or any(n.weight is None for n in norms):
        return None
    if any(float(n.eps) != LN_EPS for n in norms):
        return None
    ps = (float(attn.dropout), float(module.dropout1.p), float(module.dropout.p), float(module.dropout2.p))
    return EncoderLayerSpec(int(attn.embed_dim), int(attn.num_heads), int(module.linear1.out_features), norm_first,
                            activation, batch_first, ps, causal)

def optimizer_groups(opt, params) -> Optional[List[int]]:
    """
    The executors' view of ``opt``: for each of its param groups the mask of the segments it holds (segment s is
    ``params[s]``), or None when the optimizer must stay on the module.  Accepted: ``torch.optim.Adam`` and
    ``torch.optim.AdamW`` whose groups together hold exactly ``params``, each once; per group any ``lr``, ``betas``,
    ``eps``, ``weight_decay`` >= 0, ``amsgrad`` and ``decoupled_weight_decay`` (``foreach`` and ``fused`` do not change the
    maths).  Refused: ``maximize``, ``capturable``, ``differentiable``, a tensor ``lr`` or ``betas``, a parameter missing
    or present twice, any other optimizer class.
    """
    if type(opt) not in (torch.optim.Adam, torch.optim.AdamW):
        return None
    index = {id(p): s for s, p in enumerate(params)}
    masks, seen = [], 0
    for g in opt.param_groups:
        if g.get("maximize", False) or g.get("capturable", False) or g.get("differentiable", False):
            return None
        if torch.is_tensor(g["lr"]) or any(torch.is_tensor(b) for b in g["betas"]) or not g["weight_decay"] >= 0:
            return None
        mask = 0
        for p in g["params"]:
            s = index.get(id(p))
            if s is None or (seen >> s) & 1:
                return None
            mask |= 1 << s
            seen |= 1 << s
        masks.append(mask)
    return masks if seen == (1 << len(params)) - 1 else None


def group_hyper(group) -> dict:
    """the optimizer keywords of ``K.adam_step`` / ``K.wgrad_adam`` for one param group, read at every call so that
    learning-rate and weight-decay schedules take effect on the next step, as in torch"""
    return dict(lr=float(group["lr"]), betas=(float(group["betas"][0]), float(group["betas"][1])), eps=float(group["eps"]),
                weight_decay=float(group["weight_decay"]), decoupled=bool(group.get("decoupled_weight_decay", False)),
                amsgrad=bool(group.get("amsgrad", False)))


class FlatAdamState:
    """
    The parameters, gradients and Adam state of one expert as flat fp32 buffers in the layout of ``K.adam_step`` (one
    segment per parameter, ``names`` / ``params`` in segment order) with a bf16 mirror of the parameters, and the binding
    of the module and the torch optimizer to them: the parameters and the optimizer's state tensors are views of the
    buffers, so ``state_dict()`` of both stays live and keeps torch's layout.
    """

    def __init__(self, opt, params, names, device):
        self.opt, self.params, self.names = opt, params, names
        self.groups = optimizer_groups(opt, params)
        self.sizes = [p.numel() for p in params]
        self.all_segs = (1 << len(params)) - 1
        total = sum(self.sizes)
        f32 = dict(dtype=torch.float32, device=device)
        self.p, self.g = torch.zeros(total, **f32), torch.zeros(total, **f32)
        self.m, self.v, self.vmax = torch.zeros(total, **f32), torch.zeros(total, **f32), torch.zeros(total, **f32)
        self.p_bf16 = torch.zeros(total, dtype=torch.bfloat16, device=device)
        self.step = torch.zeros(1, dtype=torch.int32, device=device)   # the step count the kernels read
        self.one = torch.ones(1, dtype=torch.int32, device=device)
        shapes = {name: p.shape for name, p in zip(names, params)}
        self.pv, self.gv, self.mv, self.vv, self.vmv, self.bv = (
            K.segment_views(flat, shapes) for flat in (self.p, self.g, self.m, self.v, self.vmax, self.p_bf16))
        self.bind()

    @torch.no_grad()
    def bind(self):
        """(re)load the module's parameters and the optimizer's state into the flat buffers and make them views of it; the
        step count becomes the largest of the parameters'.  ``max_exp_avg_sq`` exists for the groups with amsgrad, as in
        torch."""
        amsgrad = {}
        for g, mask in zip(self.opt.param_groups, self.groups):
            for s in range(len(self.params)):
                if (mask >> s) & 1:
                    amsgrad[s] = bool(g.get("amsgrad", False))
        steps = 0
        for s, (name, param) in enumerate(zip(self.names, self.params)):
            self.pv[name][0].copy_(param.data)
            param.data = self.pv[name][0]
            param.grad = None
            st = self.opt.state.get(param, {})
            if st:
                self.mv[name][0].copy_(st["exp_avg"])
                self.vv[name][0].copy_(st["exp_avg_sq"])
                if amsgrad[s] and "max_exp_avg_sq" in st:
                    self.vmv[name][0].copy_(st["max_exp_avg_sq"])
                steps = max(steps, int(float(st["step"])))
            new = dict(step=torch.tensor(float(steps)), exp_avg=self.mv[name][0], exp_avg_sq=self.vv[name][0])
            if amsgrad[s]:
                new["max_exp_avg_sq"] = self.vmv[name][0]
            self.opt.state[param] = new
        self.steps_host = steps
        self.step.fill_(steps)
        if self.p.is_cuda:
            K.cast_bf16(self.p, self.p_bf16)
        else:
            self.p_bf16.copy_(self.p)

    def hypers(self):
        """[(``group_hyper`` of the group, mask of its segments)] of the optimizer's param groups"""
        return [(group_hyper(g), mask) for g, mask in zip(self.opt.param_groups, self.groups)]

    def begin_step(self):
        """count the step on the device; before the first optimizer kernel of a backward call"""
        K.bump_steps(self.step, self.one)

    def adam_step(self, segs):
        """step the segments of the mask ``segs`` from the gradients in ``g`` and zero those gradients: one launch per
        param group that holds any of them"""
        for hyper, mask in self.hypers():
            m = mask & segs
            if m:
                K.adam_step(self.p, self.g, self.m, self.v, self.vmax, self.p_bf16, self.sizes, 1, step=self.step,
                            zero_mask=segs, seg_mask=0 if m == self.all_segs else m, **hyper)

    def end_step(self):
        """count the step on the host, in the optimizer's state"""
        self.steps_host += 1
        # one step tensor per parameter, as torch keeps them: an eager optimizer that loads a shared one from a checkpoint
        # increments it once per parameter
        for param in self.params:
            self.opt.state[param]["step"] = torch.tensor(float(self.steps_host))


def _runs_natively(params, opt) -> bool:
    """what every executor asks of the segment parameters and the optimizer: fp32 CUDA parameters, an optimizer
    ``optimizer_groups`` accepts, and the compiled kernels"""
    if not params[0].is_cuda or params[0].dtype != torch.float32:
        return False
    if optimizer_groups(opt, params) is None:
        return False
    return native.have_cuda_kernels()


ALIGN = 16


class NativeFFNExecutor:
    """
    Trainable sm_90a ``FeedforwardBlock(hid)`` expert (the module docstring lists the kernels) for hid a multiple of 128
    with 4 * hid <= K.LN_MAX_WIDTH = 4096, i.e. hid in 128, 256, ..., 1024: both LayerNorms run at 4 * hid columns.  Wider
    blocks stay on the module.
    """
    INPUT_DIMS = 2   # [rows, hid]

    def accepts(self, x) -> bool:
        """True when ``x`` is an input this executor runs: [rows, hid]"""
        return x.dim() == self.INPUT_DIMS and x.shape[1] == self.hid

    @staticmethod
    def supports(expert, opt) -> bool:
        spec = ffn_spec(expert)
        if spec is None or not torch.cuda.is_available():
            return False
        hid = spec.hid
        # both LayerNorms run at 4 * hid columns
        if hid % 128 or 4 * hid > K.LN_MAX_WIDTH or not list(expert.parameters()):
            return False
        return _runs_natively(NativeFFNExecutor._segment_params(expert), opt)

    @staticmethod
    def _segment_params(expert):
        """the parameters in the order of FFN_SEG_NAMES (the segments of the flat buffers); the layers are reached by
        index, which a scripted block allows too"""
        keys = (key.split(".") for key in FFN_SEG_KEYS.values())   # "layers.3.weight" -> expert.layers[3].weight
        return [getattr(expert.layers[int(index)], attr) for _, index, attr in keys]

    def __init__(self, expert, opt):
        self.expert, self.opt = expert, opt
        dev = next(expert.parameters()).device
        self.device = dev
        self.hid, self.inner = expert.layers[0].in_features, expert.layers[0].out_features
        self.state = FlatAdamState(opt, self._segment_params(expert), FFN_SEG_NAMES, dev)
        self.p, self.m = self.state.p, self.state.m   # the flat parameter and exp_avg buffers
        self.group_off = torch.zeros(1, dtype=torch.int32, device=dev)
        self.group_rows = torch.zeros(1, dtype=torch.int32, device=dev)
        self._cap = 0

    def bind(self):
        """re-bind after the module or the optimizer was loaded from a checkpoint (``FlatAdamState.bind``)"""
        self.state.bind()

    def _workspace(self, rows: int):
        cap = (rows + ALIGN - 1) // ALIGN * ALIGN
        if cap > self._cap:
            cap = max(cap, 2 * self._cap, 128)
            bf = dict(dtype=torch.bfloat16, device=self.device)
            H, I = self.hid, self.inner
            self.xd, self.yo, self.gyd, self.dxd = (torch.zeros(cap, H, **bf) for _ in range(4))
            self.h1, self.a1, self.h2, self.a2, self.da, self.dh = (torch.zeros(cap, I, **bf) for _ in range(6))
            self.stats = torch.zeros(4, cap, device=self.device)
            self._cap = cap
        self.group_rows.fill_(rows)
        return (rows + ALIGN - 1) // ALIGN * ALIGN

    # ------------------------------------------------------------------ tasks
    def _forward(self, x: torch.Tensor):
        rows = x.shape[0]
        padded = self._workspace(rows)
        self.xd[:rows].copy_(x)
        if padded > rows:
            self.xd[rows:padded].zero_()
        plan = RowPlan(self.group_off, self.group_rows, tile_rows=ALIGN, rows=padded)
        ffn_forward(plan, self.state.bv, self.state.pv, self.xd, (self.h1, self.a1, self.h2, self.a2), self.stats, self.yo)
        return rows, plan

    @torch.no_grad()
    def forward(self, x: torch.Tensor) -> torch.Tensor:
        rows, _ = self._forward(x)
        return self.yo[:rows].to(x.dtype)

    @torch.no_grad()
    def backward(self, x: torch.Tensor, grad_out: torch.Tensor) -> torch.Tensor:
        """recompute forward, back-propagate, ONE optimizer step (reference: expert_backend.py:73-97); returns dL/dx"""
        rows, plan = self._forward(x)
        padded = plan.rows
        self.gyd[:rows].copy_(grad_out)
        if padded > rows:
            self.gyd[rows:padded].zero_()
        st = self.state
        seg_hyper = {name: h for h, mask in st.hypers() for s, name in enumerate(st.names) if (mask >> s) & 1}
        st.begin_step()

        def wgrad(name, dy, xin):   # each weight matrix with the settings of its own group
            hyper = seg_hyper[name]
            K.wgrad_adam(dy, xin, self.group_off, self.group_rows, p=st.pv[name], m=st.mv[name], v=st.vv[name],
                         vmax=st.vmv[name] if hyper["amsgrad"] else None, p_bf16=st.bv[name], step=st.step, **hyper)

        ffn_backward(plan, st.bv, st.pv, st.gv, self.xd, (self.h1, self.a1, self.h2, self.a2), self.stats, self.gyd,
                     self.da, self.dh, self.dh, self.dxd, wgrad)
        st.adam_step(FFN_SMALL_SEG_MASK)   # the small vectors
        st.end_step()
        return self.dxd[:rows].to(x.dtype)


class NativeGatedFFNExecutor:
    """
    Trainable sm_90a ``GatedFeedforwardBlock(hid, inner)`` expert (``gated_ffn_spec``) for hid a multiple of 128 in
    [128, K.LN_MAX_WIDTH = 4096] (the RMSNorm kernels' widest row) and inner any multiple of 128, so up to the Llama-7B
    shape hid 4096, inner 11008.  Rows are padded to a multiple of 16 with zero rows, as in NativeFFNExecutor.

      forward   xd = bf16(x);  n, rstd = RMSNorm(xd);  h = [g | u] = n [W1; W3]^T (one swap-AB GEMM);  a = silu(g) o u;
                y = a W2^T + xd (swap-AB GEMM, residual in its epilogue)
      backward  the reference semantics (recompute the forward, one optimizer step, return dx):
                da = gy W2 (swap-AB dgrad);  W2 <- fused wgrad + AMSGrad(gy, a)
                dh = SwiGLU backward(da, h)
                dn = dh [W1; W3] (one dgrad);  [W1; W3] <- fused wgrad + AMSGrad(dh, n)
                dx = gy + RMSNorm backward(dn) (the residual gradient added before the one rounding), dgamma into the
                gradient buffer;  Adam step of the norm segment

    The flat buffers hold the segments ("g", "w1", "w3", "w2"): w1 and w3 are adjacent in p, m, v, vmax and the bf16
    mirror, so [W1; W3] is one contiguous [2 inner, hid] matrix, which takes one GEMM forward, one dgrad and, when w1 and
    w3 are in the same param group, one fused wgrad + AMSGrad launch (two launches, one per half of dh, when they are not).
    Module parameters and optimizer state are views of the flat buffers (``FlatAdamState``).

    Padding rows contribute exactly zero to every gradient: their gy is zero, so their rows of da, dh and dn are zero (the
    GEMMs write the padding rows of a 16-row block from zero inputs, and SwiGLU backward of da = 0 is 0), and the RMSNorm
    backward of a zero row with a zero dn adds nothing to dgamma.
    """
    NAMES = ("g", "w1", "w3", "w2")
    INPUT_DIMS = 2   # [rows, hid]

    def accepts(self, x) -> bool:
        """True when ``x`` is an input this executor runs: [rows, hid]"""
        return x.dim() == self.INPUT_DIMS and x.shape[1] == self.hid

    @staticmethod
    def supports(expert, opt) -> bool:
        spec = gated_ffn_spec(expert)
        if spec is None or not torch.cuda.is_available():
            return False
        if spec.hid % 128 or not 128 <= spec.hid <= K.LN_MAX_WIDTH or spec.inner <= 0 or spec.inner % 128:
            return False
        return _runs_natively(NativeGatedFFNExecutor._segment_params(expert), opt)

    @staticmethod
    def _segment_params(expert):
        """the parameters in the order of NAMES (the segments of the flat buffers)"""
        return [expert.norm.weight, expert.w1.weight, expert.w3.weight, expert.w2.weight]

    def __init__(self, expert, opt):
        self.expert, self.opt = expert, opt
        spec = gated_ffn_spec(expert)
        self.hid, self.inner, self.eps = spec.hid, spec.inner, spec.eps
        params = self._segment_params(expert)
        self.device = params[0].device
        self.state = st = FlatAdamState(opt, params, self.NAMES, self.device)
        self.p, self.m = st.p, st.m   # the flat parameter and exp_avg buffers
        H, I = self.hid, self.inner
        # [W1; W3] in every flat buffer: the two segments after the norm's
        self.w13 = {name: flat[H: H + 2 * I * H].view(1, 2 * I, H)
                    for name, flat in (("p", st.p), ("m", st.m), ("v", st.v), ("vmax", st.vmax), ("bf16", st.p_bf16))}
        self.group_off = torch.zeros(1, dtype=torch.int32, device=self.device)
        self.group_rows = torch.zeros(1, dtype=torch.int32, device=self.device)
        self._cap = 0

    def bind(self):
        """re-bind after the module or the optimizer was loaded from a checkpoint (``FlatAdamState.bind``)"""
        self.state.bind()

    def _workspace(self, rows: int):
        cap = (rows + ALIGN - 1) // ALIGN * ALIGN
        if cap > self._cap:
            cap = max(cap, 2 * self._cap, 128)
            bf = dict(dtype=torch.bfloat16, device=self.device)
            H, I = self.hid, self.inner
            self.xd, self.n, self.yo, self.gyd, self.dn, self.dxd = (torch.zeros(cap, H, **bf) for _ in range(6))
            self.h, self.dh = torch.zeros(cap, 2 * I, **bf), torch.zeros(cap, 2 * I, **bf)
            self.a, self.da = torch.zeros(cap, I, **bf), torch.zeros(cap, I, **bf)
            self.rstd = torch.zeros(cap, device=self.device)
            self._cap = cap
        self.group_rows.fill_(rows)
        return (rows + ALIGN - 1) // ALIGN * ALIGN

    def _forward(self, x: torch.Tensor):
        rows = x.shape[0]
        padded = self._workspace(rows)
        self.xd[:rows].copy_(x)
        if padded > rows:
            self.xd[rows:padded].zero_()
        K.rms_norm_fwd(self.xd[:padded], self.state.pv["g"][0], self.eps, out=self.n[:padded], rstd=self.rstd[:padded])
        plan = RowPlan(self.group_off, self.group_rows, rows=padded)
        swiglu_mlp_forward(plan, self.w13["bf16"], self.state.bv["w2"], self.n, self.h, self.a, self.yo, residual=self.xd)
        return rows, plan

    @torch.no_grad()
    def forward(self, x: torch.Tensor) -> torch.Tensor:
        rows, _ = self._forward(x)
        return self.yo[:rows].to(x.dtype)

    @torch.no_grad()
    def backward(self, x: torch.Tensor, grad_out: torch.Tensor) -> torch.Tensor:
        """recompute forward, back-propagate, ONE optimizer step (reference: expert_backend.py:73-97); returns dL/dx"""
        rows, plan = self._forward(x)
        padded = plan.rows
        self.gyd[:rows].copy_(grad_out)
        if padded > rows:
            self.gyd[rows:padded].zero_()
        st = self.state
        pv, gv, I = st.pv, st.gv, self.inner
        hypers = st.hypers()
        group_of = {name: k for k, (_, mask) in enumerate(hypers) for s, name in enumerate(st.names) if (mask >> s) & 1}
        st.begin_step()

        def wgrad(name, dy, xin):   # each segment with the settings of its group: [W1; W3] in one launch if they share one
            if name == "w13" and group_of["w1"] != group_of["w3"]:
                wgrad("w1", dy[:, :I], xin)
                wgrad("w3", dy[:, I:], xin)
                return
            w = self.w13 if name == "w13" else dict(p=st.pv[name], m=st.mv[name], v=st.vv[name], vmax=st.vmv[name],
                                                    bf16=st.bv[name])
            hyper = hypers[group_of["w1" if name == "w13" else name]][0]
            K.wgrad_adam(dy, xin, self.group_off, self.group_rows, p=w["p"], m=w["m"], v=w["v"],
                         vmax=w["vmax"] if hyper["amsgrad"] else None, p_bf16=w["bf16"], step=st.step, **hyper)

        swiglu_mlp_backward(plan, self.w13["bf16"], st.bv["w2"], self.n, self.h, self.a, self.gyd, self.da, self.dh,
                            self.dn, wgrad)
        K.rms_norm_bwd(self.dn[:padded], self.xd[:padded], self.rstd[:padded], pv["g"][0], dx=self.dxd[:padded],
                       dgamma=gv["g"][0], dres=self.gyd[:padded], tile_rows=ALIGN)
        st.adam_step(1 << self.NAMES.index("g"))
        st.end_step()
        return self.dxd[:rows].to(x.dtype)


def draw_dropout_seed() -> int:
    """the 64-bit seed of one dropout executor call, drawn from torch's default CPU generator (no device read, no sync;
    ``torch.manual_seed`` makes it reproducible)"""
    lo, hi = torch.randint(0, 2 ** 32, (2,), dtype=torch.int64).tolist()
    return (hi << 32) | lo


class NativeTransformerExecutor:
    """
    Trainable sm_90a transformer expert: an encoder layer ``encoder_layer_spec`` accepts (this package's post-LN GELU layer,
    the layer of the reference's experiments/throughput/layers.py:22-51, which the reference's block cannot train; and
    torch.nn.TransformerEncoderLayer post- or pre-LN, ReLU or erf GELU, batch- or sequence-first; each plain or scripted)
    with any sequence length 1 <= S <= K.MAX_SEQ, head_dim d / nhead in K.HEAD_DIMS = (32, 64, 128), d a multiple of 128
    with 256 <= d <= K.LN_MAX_WIDTH = 4096 (the LayerNorm kernels' widest row), dim_feedforward any multiple of 128 and
    every dropout probability in [0, 1).  That includes d = 384 (6 heads), 768 (12 heads, BERT-base / ViT-B), 1280 and
    1536; any other layer stays on the module.

    Sequences: the token dimension B*S is padded with zero rows to a multiple of 128 for the GEMM, LayerNorm and dropout
    kernels; attention sees only the B*S real rows and is told S.  Padding rows contribute exactly zero to every parameter
    gradient: their output gradient is zero, so every gradient row the backward forms for them is zero, except the rows of
    dqkv, which attention_bwd does not write and which are zeroed before the in_proj bias and weight gradients.  The
    workspace is batch-major whatever the interface layout (a sequence-first input [S, B, d] is transposed on the copy in,
    and the output and the input gradient on the copy out), so dropout sites 1-3 index token row b*S + s, as an unpadded
    batch-first layer would.

      forward   in_proj GEMM -> wgmma flash attention (emits the row log-sum-exp; attention dropout in-kernel) -> out_proj
                GEMM (+bias, dropout1, +residual) -> LayerNorm -> linear1 GEMM -> GELU / ReLU (+dropout: csrc/dropout.cu)
                -> linear2 GEMM (+bias, dropout2, +residual) -> LayerNorm;  pre-LN moves each LayerNorm in front of its
                branch (LN1 before in_proj, LN2 before linear1; the residuals are the un-normalised x and h) and has no
                final LayerNorm
      backward  LayerNorm backward kernels (they also produce the bias gradients of the preceding Linear when its dropout is
                off; pre-LN: they add the residual gradient that bypasses the LayerNorm), 128 x 256-tile wgmma dgrad /
                wgrad GEMMs for the four projections, the wgmma ATTENTION BACKWARD kernel (csrc/attention_bwd.cu), the
                activation's backward (aten elementwise, or the fused activation + dropout backward kernel), one fused
                AMSGrad/Adam step over the flat parameter buffer

    Dropout (the reference's default layer has p = 0.1 at all four sites) applies iff ``expert.training``, like nn.Dropout.
    Every call with dropout draws one seed (``draw_dropout_seed``); a backward call uses it for its forward recompute and
    its backward, so a backward task re-runs the forward with a fresh mask, as the reference's ExpertBackend does.  Masks
    are regenerated from (seed, site, position) inside the kernels (csrc/dropout.cuh) and never stored.  With dropout
    applied to a Linear's output, the branch gradient M o dh / (1 - p) is formed by a masking kernel and its bias gradient
    by the grouped column sum; the residual still receives dh unmasked.

    Like the FFN executor, module parameters and optimizer state are views of flat fp32 buffers (state_dict / checkpoints
    keep the reference key names: self_attn.in_proj_weight, linear1.weight, norm1.weight, ...).

    Key padding mask (torch.nn.TransformerEncoderLayer only, ``takes_key_padding_mask``): ``forward`` / ``backward`` take
    torch's bool ``src_key_padding_mask`` [batch, S] (sequence-first layers too; True = key ignored).  It is packed once per
    call (``K.pack_key_mask``) and given to the attention forward, its backward recompute and the attention backward; every
    other kernel is unchanged.  A sequence whose keys are all masked gets a zero attention output, as torch's layer in
    training mode; torch's eval fast path returns NaN for it.

    Causal layers (this package's layer with ``causal=True``): the attention forward, its backward recompute and the
    attention backward run the causal kernels (``causal=True`` of ``K.attention_fwd`` / ``K.attention_bwd``); every other
    kernel is unchanged.
    """
    NAMES = ("w_in", "b_in", "w_out", "b_out", "w1", "b1", "w2", "b2", "g1", "be1", "g2", "be2")
    INPUT_DIMS = 3   # [batch, seq, d_model], or [seq, batch, d_model] for a sequence-first layer

    def accepts(self, x, key_padding_mask=None) -> bool:
        """True when ``x`` is an input this executor runs: [batch, S, d_model] (sequence-first: [S, batch, d_model]) with
        1 <= S <= K.MAX_SEQ, and ``key_padding_mask`` None or (torch's layer only) a bool [batch, S] tensor on x's device"""
        seq = x.shape[1 if self.batch_first else 0] if x.dim() == self.INPUT_DIMS else 0
        if not (x.dim() == self.INPUT_DIMS and x.shape[2] == self.d and 1 <= seq <= K.MAX_SEQ):
            return False
        m = key_padding_mask
        return m is None or (self.takes_key_padding_mask and m.dtype == torch.bool and m.device == x.device
                             and tuple(m.shape) == self._batch_seq(x))

    @staticmethod
    def supports(expert, opt) -> bool:
        spec = encoder_layer_spec(expert)
        if spec is None or not torch.cuda.is_available():
            return False
        d, heads, ff = spec.d, spec.heads, spec.ff
        # d = 128 stays refused: its GEMMs would run 128-wide tiles, and the dropout epilogue runs 256-wide ones only
        if d % heads or d // heads not in K.HEAD_DIMS or d % 128 or not 256 <= d <= K.LN_MAX_WIDTH or ff % 128:
            return False
        if not all(0.0 <= p < 1.0 for p in spec.ps):
            return False   # p = 1 zeroes a whole branch: eager PyTorch handles that configuration
        return _runs_natively(NativeTransformerExecutor._segment_params(expert), opt)

    @staticmethod
    def _segment_params(expert):
        """the parameters in the order of NAMES (the segments of the flat buffers)"""
        attn = expert.self_attn
        return [attn.in_proj_weight, attn.in_proj_bias, attn.out_proj.weight, attn.out_proj.bias, expert.linear1.weight,
                expert.linear1.bias, expert.linear2.weight, expert.linear2.bias, expert.norm1.weight, expert.norm1.bias,
                expert.norm2.weight, expert.norm2.bias]

    @staticmethod
    def _dropout_ps(expert):
        """drop probabilities of the kernels' sites 0-3: attention, dropout1, dropout (after the activation), dropout2"""
        return encoder_layer_spec(expert).ps

    def _dropout(self):
        """(seed, (p_attn, p_1, p_ff, p_2)) for one call, or None in eval mode / without dropout"""
        ps = self._dropout_ps(self.expert)
        if not self.expert.training or not any(ps):
            return None
        return draw_dropout_seed(), ps

    def __init__(self, expert, opt):
        self.expert, self.opt = expert, opt
        spec = encoder_layer_spec(expert)
        self.d, self.heads, self.ff = spec.d, spec.heads, spec.ff
        self.takes_key_padding_mask = class_name(expert) == TORCH_ENCODER_LAYER   # this package's layer has no mask input
        self.norm_first, self.relu, self.batch_first = spec.norm_first, spec.activation == "relu", spec.batch_first
        self.causal = spec.causal
        params = self._segment_params(expert)
        self.device = params[0].device
        self.state = FlatAdamState(opt, params, self.NAMES, self.device)
        self.p, self.m = self.state.p, self.state.m   # the flat parameter and exp_avg buffers
        self._ws = {}

    def bind(self):
        """re-bind after the module or the optimizer was loaded from a checkpoint (``FlatAdamState.bind``)"""
        self.state.bind()

    def _workspace(self, T):
        """buffers for T padded token rows (T a multiple of 128)"""
        ws = self._ws.get(T)
        if ws is None:
            bf = dict(dtype=torch.bfloat16, device=self.device)
            d, ff = self.d, self.ff
            f32 = dict(dtype=torch.float32, device=self.device)
            ws = dict(x=torch.empty(T, d, **bf), qkv=torch.empty(T, 3 * d, **bf), att=torch.empty(T, d, **bf), h=torch.empty(T, d, **bf),
                      x1=torch.empty(T, d, **bf), f=torch.empty(T, ff, **bf), y=torch.empty(T, d, **bf), out=torch.empty(T, d, **bf),
                      lse=torch.empty(T, self.heads, **f32), stats=torch.empty(4, T, **f32),
                      group_off=torch.tensor([0, T], dtype=torch.int32, device=self.device))
            if self.norm_first:
                ws["xa"] = torch.empty(T, d, **bf)   # LN1(x), the input of in_proj
            self._ws = {T: ws}
        return ws

    def _batch_seq(self, t):
        """(batch, seq) of an interface tensor"""
        return (t.shape[0], t.shape[1]) if self.batch_first else (t.shape[1], t.shape[0])

    def _to_rows(self, dst, t):
        """copy the interface tensor ``t`` into the batch-major token rows ``dst`` [batch * seq, d]"""
        if self.batch_first:
            dst.copy_(t.reshape(dst.shape))
        else:
            dst.view(t.shape[1], t.shape[0], t.shape[2]).copy_(t.transpose(0, 1))

    def _from_rows(self, rows, like):
        """the batch-major token rows [batch * seq, d] as a tensor of the shape, layout and dtype of ``like``"""
        if self.batch_first:
            return rows.view(like.shape).to(like.dtype)
        seq, batch, d = like.shape
        return rows.view(batch, seq, d).transpose(0, 1).to(like.dtype, memory_format=torch.contiguous_format)

    @staticmethod
    def _site(drop, site):
        """kernel dropout argument of one site: (p, seed) for attention, (p, seed, site) for the others; None when off"""
        if drop is None or not drop[1][site]:
            return None
        return (drop[1][site], drop[0]) if site == K.SITE_ATTN else (drop[1][site], drop[0], site)

    @staticmethod
    def _pack(key_padding_mask):
        return None if key_padding_mask is None else K.pack_key_mask(key_padding_mask.contiguous())

    def _forward(self, src, drop=None, key_mask=None):
        """returns the workspace, the real token rows Tr = batch * seq and the padded rows T (a multiple of 128);
        key_mask: packed key padding mask (``_pack``) or None"""
        from ..ops import gemm
        assert self.accepts(src), (tuple(src.shape), self.d)
        batch, seq = self._batch_seq(src)
        Tr = batch * seq
        T = (Tr + 127) // 128 * 128
        ws = self._workspace(T)
        self._to_rows(ws["x"][:Tr], src)
        if T > Tr:
            ws["x"][Tr:].zero_()
            ws["att"][Tr:].zero_()   # attention writes only the real rows
        x, bv, pv, site, stats = ws["x"], self.state.bv, self.state.pv, self._site, ws["stats"]
        if self.norm_first:
            K.ln_relu_fwd(x, pv["g1"], pv["be1"], None, out=ws["xa"], mean=stats[0], rstd=stats[1], relu=False)
        gemm.grouped_linear(ws["xa"] if self.norm_first else x, bv["w_in"], bias=pv["b_in"], out=ws["qkv"])
        K.attention_fwd(ws["qkv"][:Tr], self.heads, out=ws["att"][:Tr], lse=ws["lse"][:Tr], dropout=site(drop, K.SITE_ATTN),
                        seq_len=seq, key_mask=key_mask, causal=self.causal)
        gemm.grouped_linear(ws["att"], bv["w_out"], bias=pv["b_out"], residual=x, out=ws["h"],
                            dropout=site(drop, K.SITE_OUT_PROJ))
        if self.norm_first:   # x1 = LN2(h) feeds the feed-forward branch, h is its residual
            K.ln_relu_fwd(ws["h"], pv["g2"], pv["be2"], None, out=ws["x1"], mean=stats[2], rstd=stats[3], relu=False)
        else:                 # x1 = LN1(h) is both
            K.ln_relu_fwd(ws["h"], pv["g1"], pv["be1"], None, out=ws["x1"], mean=stats[0], rstd=stats[1], relu=False)
        gemm.grouped_linear(ws["x1"], bv["w1"], bias=pv["b1"], out=ws["f"])       # pre-activation kept for backward
        ff = site(drop, K.SITE_FF)
        if self.relu:
            ws["gact"] = K.relu_dropout(ws["f"], *ff) if ff else torch.relu(ws["f"])
        else:
            ws["gact"] = K.gelu_dropout(ws["f"], *ff) if ff else torch.nn.functional.gelu(ws["f"])
        gemm.grouped_linear(ws["gact"], bv["w2"], bias=pv["b2"], residual=ws["h"] if self.norm_first else ws["x1"], out=ws["y"],
                            dropout=site(drop, K.SITE_LINEAR2))
        if not self.norm_first:
            K.ln_relu_fwd(ws["y"], pv["g2"], pv["be2"], None, out=ws["out"], mean=stats[2], rstd=stats[3], relu=False)
        return ws, Tr, T

    @torch.no_grad()
    def forward(self, src: torch.Tensor, key_padding_mask: Optional[torch.Tensor] = None) -> torch.Tensor:
        ws, Tr, T = self._forward(src, self._dropout(), self._pack(key_padding_mask))
        return self._from_rows(ws["y" if self.norm_first else "out"][:Tr], src)

    @torch.no_grad()
    def backward(self, src: torch.Tensor, grad_out: torch.Tensor, key_padding_mask: Optional[torch.Tensor] = None) -> torch.Tensor:
        from ..ops import gemm
        drop = self._dropout()
        key_mask = self._pack(key_padding_mask)
        ws, Tr, T = self._forward(src, drop, key_mask)   # reference semantics: the client re-sends the inputs, the server recomputes the forward
        st = self.state
        d, bv, pv, gv, site, stats = self.d, st.bv, st.pv, st.gv, self._site, ws["stats"]
        go = ws["group_off"]
        bf = dict(dtype=torch.bfloat16, device=self.device)
        seq = self._batch_seq(src)[1]
        if T > Tr or not self.batch_first:   # zero gradient on the padding rows
            dout = torch.zeros(T, d, **bf) if T > Tr else torch.empty(T, d, **bf)
            self._to_rows(dout[:Tr], grad_out)
        else:
            dout = grad_out.reshape(T, d).to(torch.bfloat16).contiguous()

        def branch_grad(dres, drop_site, bias_grad):
            """gradient of a Linear whose output went through dropout `drop_site` into a residual sum: M o dres / (1 - p)
            and its bias gradient (without dropout the LayerNorm backward already produced the bias gradient)"""
            s = site(drop, drop_site)
            if s is None:
                return dres
            dbr = K.dropout_apply(dres, *s)
            K.grouped_colsum(dbr, None, out=bias_grad)
            return dbr

        # with dropout at site 3 / 1 the bias gradient comes from the masked branch gradient, so the LayerNorm backward's
        # column sum goes to a scratch row; pre-LN's LN1 backward has no bias to feed and always uses it
        scratch = torch.empty(1, d, dtype=torch.float32, device=self.device) if drop is not None or self.norm_first else None
        if self.norm_first:   # y = h + branch: no LayerNorm after it, the branch and the residual both receive dout
            dy = dout
            if site(drop, K.SITE_LINEAR2) is None:
                K.grouped_colsum(dy, None, out=gv["b2"])
        else:
            dy = torch.empty(T, d, **bf)
            K.ln_relu_bwd(dout, ws["y"], stats[2], stats[3], pv["g2"], pv["be2"], None, dh=dy, dgamma=gv["g2"],
                          dbeta=gv["be2"], dbias=scratch if site(drop, K.SITE_LINEAR2) else gv["b2"], relu=False)
        dff = branch_grad(dy, K.SITE_LINEAR2, gv["b2"])
        gemm.grouped_wgrad(dff, ws["gact"], go, 1, out=gv["w2"])
        dg = gemm.grouped_linear(dff, bv["w2"], w_is_kn=True)
        ff = site(drop, K.SITE_FF)
        if self.relu:
            df = K.relu_dropout_bwd(dg, ws["f"], *ff) if ff else torch.ops.aten.threshold_backward(dg, ws["f"], 0)
        else:
            df = K.gelu_dropout_bwd(dg, ws["f"], *ff) if ff else torch.ops.aten.gelu_backward(dg, ws["f"])
        K.grouped_colsum(df, None, out=gv["b1"])
        gemm.grouped_wgrad(df, ws["x1"], go, 1, out=gv["w1"])
        if self.norm_first:   # dh = dy + LN2 backward(dx1): the residual gradient is added inside the LayerNorm backward
            dx1 = gemm.grouped_linear(df, bv["w1"], w_is_kn=True)
            dh = torch.empty(T, d, **bf)
            K.ln_relu_bwd(dx1, ws["h"], stats[2], stats[3], pv["g2"], pv["be2"], None, dh=dh, dgamma=gv["g2"],
                          dbeta=gv["be2"], dbias=scratch if site(drop, K.SITE_OUT_PROJ) else gv["b_out"], relu=False, dres=dy)
        else:
            dx1 = gemm.grouped_linear(df, bv["w1"], w_is_kn=True, residual=dy)
            dh = torch.empty(T, d, **bf)
            K.ln_relu_bwd(dx1, ws["h"], stats[0], stats[1], pv["g1"], pv["be1"], None, dh=dh, dgamma=gv["g1"],
                          dbeta=gv["be1"], dbias=scratch if site(drop, K.SITE_OUT_PROJ) else gv["b_out"], relu=False)
        dhb = branch_grad(dh, K.SITE_OUT_PROJ, gv["b_out"])
        gemm.grouped_wgrad(dhb, ws["att"], go, 1, out=gv["w_out"])
        datt = gemm.grouped_linear(dhb, bv["w_out"], w_is_kn=True)
        if T > Tr:   # attention_bwd does not write the padding rows
            dqkv = torch.empty(T, 3 * d, **bf)
            dqkv[Tr:].zero_()
            K.attention_bwd(ws["qkv"][:Tr], ws["att"][:Tr], datt[:Tr], ws["lse"][:Tr], self.heads, dropout=site(drop, K.SITE_ATTN),
                            seq_len=seq, dqkv=dqkv[:Tr], key_mask=key_mask, causal=self.causal)
        else:
            dqkv = K.attention_bwd(ws["qkv"], ws["att"], datt, ws["lse"], self.heads, dropout=site(drop, K.SITE_ATTN), seq_len=seq,
                                   key_mask=key_mask, causal=self.causal)
        K.grouped_colsum(dqkv, None, out=gv["b_in"])
        if self.norm_first:   # dx = dh + LN1 backward(dxa)
            gemm.grouped_wgrad(dqkv, ws["xa"], go, 1, out=gv["w_in"])
            dxa = gemm.grouped_linear(dqkv, bv["w_in"], w_is_kn=True)
            dx = torch.empty(T, d, **bf)
            K.ln_relu_bwd(dxa, ws["x"], stats[0], stats[1], pv["g1"], pv["be1"], None, dh=dx, dgamma=gv["g1"], dbeta=gv["be1"],
                          dbias=scratch, relu=False, dres=dh)
        else:
            gemm.grouped_wgrad(dqkv, ws["x"], go, 1, out=gv["w_in"])
            dx = gemm.grouped_linear(dqkv, bv["w_in"], w_is_kn=True, residual=dh)
        st.begin_step()
        st.adam_step(st.all_segs)
        st.end_step()
        return self._from_rows(dx[:Tr], src)


def make_executor(expert, opt):
    try:
        if NativeTransformerExecutor.supports(expert, opt):
            return NativeTransformerExecutor(expert, opt)
        if NativeFFNExecutor.supports(expert, opt):
            return NativeFFNExecutor(expert, opt)
        if NativeGatedFFNExecutor.supports(expert, opt):
            return NativeGatedFFNExecutor(expert, opt)
    except Exception as e:  # noqa: an executor that cannot be built must not break the server; eager PyTorch still works
        print(f"[lah_b200] native expert executor unavailable ({type(e).__name__}: {e}); using eager PyTorch", flush=True)
    return None
