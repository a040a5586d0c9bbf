"""
NativeFFNExecutor — runs ``ExpertBackend.forward`` / ``ExpertBackend.backward`` of a ``FeedforwardBlock`` expert on the
hand-written sm_90a kernels instead of eager PyTorch, so that a ``TesseractServer``'s runtime loop
(the reference's lib/runtime/__init__.py:42-47 -> lib/runtime/expert_backend.py:64-97) executes wgmma code:

  forward   swap-AB grouped linear (weights streamed once per 128 rows, csrc/small_m.cu) x 3 + fused LayerNorm+ReLU x 2
  backward  the reference semantics — recompute the forward from the inputs the client re-sent, back-propagate, step the
            expert's optimizer immediately, return the gradients w.r.t. the inputs — with swap-AB dgrads, the LayerNorm
            backward kernel and the FUSED weight-gradient + AMSGrad kernel (the gradient of a weight matrix never reaches HBM)

The module's parameters and the torch optimizer's state tensors are re-bound as VIEWS of the executor's flat fp32 buffers:
``expert.state_dict()``, ``opt.state_dict()`` and ``ExpertBackend.checkpoint()`` stay live and keep the reference layout.
"""
from typing import Optional

import torch

from ..models.layers import FeedforwardBlock
from ..ops import kernels as K, native

SEGS = (("w1", 0, "weight"), ("b1", 0, "bias"), ("g1", 1, "weight"), ("be1", 1, "bias"), ("w2", 3, "weight"),
        ("b2", 3, "bias"), ("g2", 4, "weight"), ("be2", 4, "bias"), ("w3", 6, "weight"), ("b3", 6, "bias"))
SMALL_MASK = sum(1 << i for i, (n, _, _) in enumerate(SEGS) if not n.startswith("w"))
ALIGN = 16


class NativeFFNExecutor:
    INPUT_DIMS = 2   # [rows, hid]

    @staticmethod
    def supports(expert, opt) -> bool:
        if not isinstance(expert, FeedforwardBlock) or not torch.cuda.is_available():
            return False
        hid = expert.layers[0].in_features
        params = list(expert.parameters())
        if hid % 128 or not params or not params[0].is_cuda or params[0].dtype != torch.float32:
            return False
        if type(opt) is not torch.optim.Adam or len(opt.param_groups) != 1:
            return False
        g = opt.param_groups[0]
        if g.get("weight_decay", 0) or g.get("maximize", False) or g.get("capturable", False) or g.get("differentiable", False):
            return False
        if {id(p) for p in g["params"]} != {id(p) for p in params}:
            return False
        return native.have_cuda_kernels()

    def __init__(self, expert: FeedforwardBlock, opt: torch.optim.Adam):
        self.expert, self.opt = expert, opt
        dev = next(expert.parameters()).device
        self.device = dev
        self.hid, self.inner = expert.layers[0].in_features, expert.layers[0].out_features
        self.params = [getattr(expert.layers[li], attr) for _, li, attr in SEGS]
        self.sizes = [p.numel() for p in self.params]
        total = sum(self.sizes)
        f32 = dict(dtype=torch.float32, device=dev)
        self.p, self.g = torch.zeros(total, **f32), torch.zeros(total, **f32)
        self.m, self.v, self.vmax = torch.zeros(total, **f32), torch.zeros(total, **f32), torch.zeros(total, **f32)
        self.p_bf16 = torch.zeros(total, dtype=torch.bfloat16, device=dev)
        self.step = torch.zeros(1, dtype=torch.int32, device=dev)
        self.one = torch.ones(1, dtype=torch.int32, device=dev)
        self.group_off = torch.zeros(1, dtype=torch.int32, device=dev)
        self.group_rows = torch.zeros(1, dtype=torch.int32, device=dev)
        self.steps_host = 0
        self._cap = 0
        self.bind()

    # ------------------------------------------------------------------ parameter / optimizer-state binding
    def _views(self, flat):
        out, off = {}, 0
        for (name, _, _), p, n in zip(SEGS, self.params, self.sizes):
            out[name] = flat[off: off + n].view(1, *p.shape)
            off += n
        return out

    @torch.no_grad()
    def bind(self):
        """(re)load the module's parameters and the optimizer's state into the flat buffers and make them views of it"""
        group = self.opt.param_groups[0]
        amsgrad = bool(group.get("amsgrad", False))
        self.pv, self.gv = self._views(self.p), self._views(self.g)
        self.mv, self.vv, self.vmv, self.bv = self._views(self.m), self._views(self.v), self._views(self.vmax), self._views(self.p_bf16)
        steps = 0
        for (name, _, _), param in zip(SEGS, self.params):
            self.pv[name][0].copy_(param.data)
            param.data = self.pv[name][0]
            param.grad = None
            st = self.opt.state.get(param, {})
            if st:
                self.mv[name][0].copy_(st["exp_avg"])
                self.vv[name][0].copy_(st["exp_avg_sq"])
                if amsgrad and "max_exp_avg_sq" in st:
                    self.vmv[name][0].copy_(st["max_exp_avg_sq"])
                steps = max(steps, int(float(st["step"])))
            new = dict(step=torch.tensor(float(steps)), exp_avg=self.mv[name][0], exp_avg_sq=self.vv[name][0])
            if amsgrad:
                new["max_exp_avg_sq"] = self.vmv[name][0]
            self.opt.state[param] = new
        self.steps_host = steps
        self.step.fill_(steps)
        K.cast_bf16(self.p, self.p_bf16)

    def _hyper(self):
        g = self.opt.param_groups[0]
        return dict(lr=float(g["lr"]), betas=tuple(g["betas"]), eps=float(g["eps"]), amsgrad=bool(g.get("amsgrad", False)))

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
        go, gr, pv, bv = self.group_off, self.group_rows, self.pv, self.bv
        K.swapab_linear(self.xd, bv["w1"], go, gr, out=self.h1, bias=pv["b1"])
        K.ln_relu_fwd(self.h1[:padded], pv["g1"], pv["be1"], None, out=self.a1[:padded], mean=self.stats[0], rstd=self.stats[1],
                      tile_rows=ALIGN)
        K.swapab_linear(self.a1, bv["w2"], go, gr, out=self.h2, bias=pv["b2"])
        K.ln_relu_fwd(self.h2[:padded], pv["g2"], pv["be2"], None, out=self.a2[:padded], mean=self.stats[2], rstd=self.stats[3],
                      tile_rows=ALIGN)
        K.swapab_linear(self.a2, bv["w3"], go, gr, out=self.yo, bias=pv["b3"], residual=self.xd)
        return rows, padded

    @torch.no_grad()
    def forward(self, x: torch.Tensor) -> torch.Tensor:
        rows, _ = self._forward(x)
        return self.yo[:rows].to(x.dtype)

    @torch.no_grad()
    def backward(self, x: torch.Tensor, grad_out: torch.Tensor) -> torch.Tensor:
        """recompute forward, back-propagate, ONE optimizer step (reference: expert_backend.py:73-97); returns dL/dx"""
        rows, padded = self._forward(x)
        self.gyd[:rows].copy_(grad_out)
        if padded > rows:
            self.gyd[rows:padded].zero_()
        go, gr, pv, bv, gv = self.group_off, self.group_rows, self.pv, self.bv, self.gv
        hyper = self._hyper()
        K.bump_steps(self.step, self.one)

        def wgrad(name, dy, xin):
            K.wgrad_adam(dy, xin, go, gr, p=pv[name], m=self.mv[name], v=self.vv[name],
                         vmax=self.vmv[name] if hyper["amsgrad"] else None, p_bf16=bv[name], step=self.step, **hyper)

        K.grouped_colsum(self.gyd[:padded], None, out=gv["b3"], tile_rows=ALIGN)
        K.swapab_linear(self.gyd, bv["w3"], go, gr, out=self.da, w_is_kn=True)
        wgrad("w3", self.gyd, self.a2)
        K.ln_relu_bwd(self.da[:padded], self.h2[:padded], self.stats[2], self.stats[3], pv["g2"], pv["be2"], None,
                      dh=self.dh[:padded], dgamma=gv["g2"], dbeta=gv["be2"], dbias=gv["b2"], tile_rows=ALIGN)
        K.swapab_linear(self.dh, bv["w2"], go, gr, out=self.da, w_is_kn=True)
        wgrad("w2", self.dh, self.a1)
        K.ln_relu_bwd(self.da[:padded], self.h1[:padded], self.stats[0], self.stats[1], pv["g1"], pv["be1"], None,
                      dh=self.dh[:padded], dgamma=gv["g1"], dbeta=gv["be1"], dbias=gv["b1"], tile_rows=ALIGN)
        K.swapab_linear(self.dh, bv["w1"], go, gr, out=self.dxd, w_is_kn=True, residual=self.gyd)
        wgrad("w1", self.dh, self.xd)
        K.adam_step(self.p, self.g, self.m, self.v, self.vmax, self.p_bf16, self.sizes, 1, step=self.step, zero_mask=SMALL_MASK,
                    seg_mask=SMALL_MASK, **hyper)
        self.steps_host += 1
        step_t = torch.tensor(float(self.steps_host))
        for param in self.params:
            self.opt.state[param]["step"] = step_t
        return self.dxd[:rows].to(x.dtype)


class NativeTransformerExecutor:
    """
    Trainable sm_90a transformer expert (post-LN encoder layer of the reference's experiments/throughput/layers.py:22-51,
    batch-first [B, 512, d], head_dim 64, dropout must be 0 for training — the reference's block cannot be trained at all).

      forward   in_proj GEMM -> wgmma flash attention (emits the row log-sum-exp) -> out_proj GEMM (+bias +residual) ->
                LayerNorm -> linear1 GEMM -> GELU -> linear2 GEMM (+bias +residual) -> LayerNorm
      backward  LayerNorm backward kernels (they also produce the bias gradients of the preceding Linear), wide-tile wgmma
                dgrad / wgrad GEMMs for the four projections, the wgmma ATTENTION BACKWARD kernel (csrc/attention_bwd.cu),
                GELU backward (aten elementwise), one fused AMSGrad/Adam step over the flat parameter buffer

    Like the FFN executor, module parameters and optimizer state are views of flat fp32 buffers (state_dict / checkpoints
    keep the reference key names: self_attn.in_proj_weight, linear1.weight, norm1.weight, ...).
    """
    NAMES = ("w_in", "b_in", "w_out", "b_out", "w1", "b1", "w2", "b2", "g1", "be1", "g2", "be2")
    INPUT_DIMS = 3   # [batch, 512, d_model]

    @staticmethod
    def supports(expert, opt) -> bool:
        from ..models.layers import TransformerEncoderLayer, SEQ_LEN  # noqa
        if not isinstance(expert, TransformerEncoderLayer) or not torch.cuda.is_available():
            return False
        attn = expert.self_attn
        d, ff = attn.embed_dim, expert.linear1.out_features
        params = list(expert.parameters())
        if d // attn.num_heads != 64 or d % 256 or ff % 256 or not params[0].is_cuda or params[0].dtype != torch.float32:
            return False
        if expert.dropout.p or expert.dropout1.p or expert.dropout2.p or attn.dropout:
            return False   # dropout masks are not implemented in the kernels: eager PyTorch handles that configuration
        if type(opt) is not torch.optim.Adam or len(opt.param_groups) != 1:
            return False
        g = opt.param_groups[0]
        if g.get("weight_decay", 0) or g.get("maximize", False) or g.get("capturable", False) or g.get("differentiable", False):
            return False
        if {id(p) for p in g["params"]} != {id(p) for p in params}:
            return False
        return native.have_cuda_kernels()

    def __init__(self, expert, opt):
        self.expert, self.opt = expert, opt
        attn = expert.self_attn
        self.d, self.heads, self.ff = attn.embed_dim, attn.num_heads, expert.linear1.out_features
        self.params = [attn.in_proj_weight, attn.in_proj_bias, attn.out_proj.weight, attn.out_proj.bias, expert.linear1.weight,
                       expert.linear1.bias, expert.linear2.weight, expert.linear2.bias, expert.norm1.weight, expert.norm1.bias,
                       expert.norm2.weight, expert.norm2.bias]
        dev = self.params[0].device
        self.device = dev
        self.sizes = [p.numel() for p in self.params]
        total = sum(self.sizes)
        f32 = dict(dtype=torch.float32, device=dev)
        self.p, self.g = torch.zeros(total, **f32), torch.zeros(total, **f32)
        self.m, self.v, self.vmax = torch.zeros(total, **f32), torch.zeros(total, **f32), torch.zeros(total, **f32)
        self.p_bf16 = torch.zeros(total, dtype=torch.bfloat16, device=dev)
        self.step = torch.zeros(1, dtype=torch.int32, device=dev)
        self.one = torch.ones(1, dtype=torch.int32, device=dev)
        self.steps_host = 0
        self._ws = {}
        self.bind()

    def _views(self, flat):
        out, off = {}, 0
        for name, p, n in zip(self.NAMES, self.params, self.sizes):
            out[name] = flat[off: off + n].view(1, *p.shape)
            off += n
        return out

    @torch.no_grad()
    def bind(self):
        amsgrad = bool(self.opt.param_groups[0].get("amsgrad", False))
        self.pv, self.gv, self.bv = self._views(self.p), self._views(self.g), self._views(self.p_bf16)
        mv, vv, vmv = self._views(self.m), self._views(self.v), self._views(self.vmax)
        steps = 0
        for name, param in zip(self.NAMES, self.params):
            self.pv[name][0].copy_(param.data)
            param.data = self.pv[name][0]
            param.grad = None
            st = self.opt.state.get(param, {})
            if st:
                mv[name][0].copy_(st["exp_avg"])
                vv[name][0].copy_(st["exp_avg_sq"])
                if amsgrad and "max_exp_avg_sq" in st:
                    vmv[name][0].copy_(st["max_exp_avg_sq"])
                steps = max(steps, int(float(st["step"])))
            new = dict(step=torch.tensor(float(steps)), exp_avg=mv[name][0], exp_avg_sq=vv[name][0])
            if amsgrad:
                new["max_exp_avg_sq"] = vmv[name][0]
            self.opt.state[param] = new
        self.steps_host = steps
        self.step.fill_(steps)
        K.cast_bf16(self.p, self.p_bf16)

    def _workspace(self, T):
        ws = self._ws.get(T)
        if ws is None:
            bf = dict(dtype=torch.bfloat16, device=self.device)
            d, ff = self.d, self.ff
            f32 = dict(dtype=torch.float32, device=self.device)
            ws = dict(x=torch.empty(T, d, **bf), qkv=torch.empty(T, 3 * d, **bf), att=torch.empty(T, d, **bf), h=torch.empty(T, d, **bf),
                      x1=torch.empty(T, d, **bf), f=torch.empty(T, ff, **bf), y=torch.empty(T, d, **bf), out=torch.empty(T, d, **bf),
                      lse=torch.empty(T, self.heads, **f32), stats=torch.empty(4, T, **f32),
                      group_off=torch.tensor([0, T], dtype=torch.int32, device=self.device))
            self._ws = {T: ws}
        return ws

    def _forward(self, src):
        from ..ops import gemm
        batch, seq, d = src.shape
        assert seq == 512 and d == self.d
        T = batch * seq
        ws = self._workspace(T)
        ws["x"].copy_(src.reshape(T, d))
        x, bv, pv = ws["x"], self.bv, self.pv
        gemm.grouped_linear(x, bv["w_in"], bias=pv["b_in"], out=ws["qkv"], two_cta=True)
        K.attention_fwd(ws["qkv"], self.heads, out=ws["att"], lse=ws["lse"])
        gemm.grouped_linear(ws["att"], bv["w_out"], bias=pv["b_out"], residual=x, out=ws["h"], two_cta=True)
        K.ln_relu_fwd(ws["h"], pv["g1"], pv["be1"], None, out=ws["x1"], mean=ws["stats"][0], rstd=ws["stats"][1], relu=False)
        gemm.grouped_linear(ws["x1"], bv["w1"], bias=pv["b1"], out=ws["f"], two_cta=True)       # pre-activation kept for backward
        ws["gact"] = torch.nn.functional.gelu(ws["f"])
        gemm.grouped_linear(ws["gact"], bv["w2"], bias=pv["b2"], residual=ws["x1"], out=ws["y"], two_cta=True)
        K.ln_relu_fwd(ws["y"], pv["g2"], pv["be2"], None, out=ws["out"], mean=ws["stats"][2], rstd=ws["stats"][3], relu=False)
        return ws, T

    @torch.no_grad()
    def forward(self, src: torch.Tensor) -> torch.Tensor:
        ws, T = self._forward(src)
        return ws["out"].view(src.shape).to(src.dtype)

    @torch.no_grad()
    def backward(self, src: torch.Tensor, grad_out: torch.Tensor) -> torch.Tensor:
        from ..ops import gemm
        ws, T = self._forward(src)   # reference semantics: the client re-sends the inputs, the server recomputes the forward
        d, bv, pv, gv = self.d, self.bv, self.pv, self.gv
        go = ws["group_off"]
        bf = dict(dtype=torch.bfloat16, device=self.device)
        dout = grad_out.reshape(T, d).to(torch.bfloat16).contiguous()
        dy = torch.empty(T, d, **bf)
        K.ln_relu_bwd(dout, ws["y"], ws["stats"][2], ws["stats"][3], pv["g2"], pv["be2"], None, dh=dy, dgamma=gv["g2"],
                      dbeta=gv["be2"], dbias=gv["b2"], relu=False)
        gemm.grouped_wgrad(dy, ws["gact"], go, 1, out=gv["w2"], two_cta=True)
        dg = gemm.grouped_linear(dy, bv["w2"], w_is_kn=True, two_cta=True)
        df = torch.ops.aten.gelu_backward(dg, ws["f"])
        K.grouped_colsum(df, None, out=gv["b1"])
        gemm.grouped_wgrad(df, ws["x1"], go, 1, out=gv["w1"], two_cta=True)
        dx1 = gemm.grouped_linear(df, bv["w1"], w_is_kn=True, residual=dy, two_cta=True)
        dh = torch.empty(T, d, **bf)
        K.ln_relu_bwd(dx1, ws["h"], ws["stats"][0], ws["stats"][1], pv["g1"], pv["be1"], None, dh=dh, dgamma=gv["g1"],
                      dbeta=gv["be1"], dbias=gv["b_out"], relu=False)
        gemm.grouped_wgrad(dh, ws["att"], go, 1, out=gv["w_out"], two_cta=True)
        datt = gemm.grouped_linear(dh, bv["w_out"], w_is_kn=True, two_cta=True)
        dqkv = K.attention_bwd(ws["qkv"], ws["att"], datt, ws["lse"], self.heads)
        K.grouped_colsum(dqkv, None, out=gv["b_in"])
        gemm.grouped_wgrad(dqkv, ws["x"], go, 1, out=gv["w_in"], two_cta=True)
        dx = gemm.grouped_linear(dqkv, bv["w_in"], w_is_kn=True, residual=dh, two_cta=True)
        g = self.opt.param_groups[0]
        K.bump_steps(self.step, self.one)
        K.adam_step(self.p, self.g, self.m, self.v, self.vmax, self.p_bf16, self.sizes, 1, step=self.step, lr=float(g["lr"]),
                    betas=tuple(g["betas"]), eps=float(g["eps"]), amsgrad=bool(g.get("amsgrad", False)),
                    zero_mask=(1 << len(self.sizes)) - 1)
        self.steps_host += 1
        step_t = torch.tensor(float(self.steps_host))
        for param in self.params:
            self.opt.state[param]["step"] = step_t
        return dx.view(src.shape).to(src.dtype)


def make_executor(expert, opt):
    try:
        if NativeTransformerExecutor.supports(expert, opt):
            return NativeTransformerExecutor(expert, opt)
        if NativeFFNExecutor.supports(expert, opt):
            return NativeFFNExecutor(expert, opt)
    except Exception as e:  # noqa: an executor that cannot be built must not break the server; eager PyTorch still works
        print(f"[lah_b200] native expert executor unavailable ({type(e).__name__}: {e}); using eager PyTorch", flush=True)
    return None
