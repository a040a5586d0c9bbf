"""
sm_90a forward of the FFN expert (``FeedforwardBlock``, the reference's experiments/throughput/layers.py:5-19) for the
forward-only throughput experiment: three wgmma GEMMs with fused bias (+ residual) epilogues and the fused
LayerNorm+ReLU kernel in between.  ``dtype="fp8"`` runs the GEMMs on block-scaled FP8 tensor cores (MXFP8); LayerNorm
then emits the next GEMM's FP8 operand directly and no bf16 activation is written at all.

``NativeGatedFFNLayer`` is the same for the SwiGLU expert (``GatedFeedforwardBlock``): RMSNorm, one GEMM over [W1; W3],
SwiGLU and the W2 GEMM with the residual.  In fp8 the RMSNorm and the SwiGLU emit the MXFP8 operands n and a, and
neither is written in bf16.
"""
import torch
import torch.nn as nn

from ..ops import fp8, kernels as K
from ..ops.expert_blocks import RowPlan, ffn_forward, ffn_forward_fp8, swiglu_mlp_forward, swiglu_mlp_forward_fp8
from .layers import FeedforwardBlock, GatedFeedforwardBlock


class NativeFFNLayer(nn.Module):
    def __init__(self, block: FeedforwardBlock, device=None, dtype: str = "bf16"):
        super().__init__()
        device = device or torch.device("cuda", torch.cuda.current_device())
        self.dtype = dtype
        lin1, ln1, lin2, ln2, lin3 = (block.layers[i] for i in (0, 1, 3, 4, 6))
        self.hid, self.inner = lin1.in_features, lin1.out_features

        def f(t):
            return t.detach().to(device=device, dtype=torch.float32).unsqueeze(0).contiguous()

        self.p = dict(b1=f(lin1.bias), b2=f(lin2.bias), b3=f(lin3.bias), g1=f(ln1.weight), be1=f(ln1.bias),
                      g2=f(ln2.weight), be2=f(ln2.bias))
        ws = {n: m.weight.detach().to(device=device) for n, m in (("w1", lin1), ("w2", lin2), ("w3", lin3))}
        if dtype == "fp8":
            self.w = {n: fp8.quantize(w.float().contiguous(), tile_rows=fp8.WEIGHT_TILE, groups=1) for n, w in ws.items()}
        else:
            self.w = {n: w.to(torch.bfloat16).unsqueeze(0).contiguous() for n, w in ws.items()}
        self._ws = {}

    def _workspace(self, rows, device):
        ws = self._ws.get(rows)
        if ws is None:
            bf = dict(dtype=torch.bfloat16, device=device)
            ws = dict(h=torch.empty(rows, self.inner, **bf))
            if self.dtype == "fp8":
                ws["xq"] = fp8.MXFP8Tensor(rows, 1, self.hid, fp8.ACT_TILE, device)
                ws["aq"] = fp8.MXFP8Tensor(rows, 1, self.inner, fp8.ACT_TILE, device)
            else:
                ws["a"] = torch.empty(rows, self.inner, **bf)
            self._ws = {rows: ws}
        return ws

    @torch.no_grad()
    def forward(self, x, out=None):
        """x: [rows, hid] bf16 (rows % 256 == 0); returns bf16 [rows, hid] (written into ``out`` — which may live in a
        peer GPU's memory — when given)"""
        rows, hid = x.shape
        assert hid == self.hid and rows % 256 == 0 and x.dtype == torch.bfloat16 and x.is_contiguous()
        ws = self._workspace(rows, x.device)
        if out is None:
            out = torch.empty_like(x)
        plan = RowPlan()   # 128-row tiles of one group
        if self.dtype == "fp8":   # no bf16 activation or LayerNorm statistics: nothing reads them
            ffn_forward_fp8(plan, self.w, self.p, x, ws["xq"], ws["aq"], (ws["h"], None, ws["h"], None), (None,) * 4, out)
        else:
            stat = ws.setdefault("stat", torch.empty(rows, device=x.device))
            ffn_forward(plan, self.w, self.p, x, (ws["h"], ws["a"], ws["h"], ws["a"]), (stat,) * 4, out)
        return out


class NativeGatedFFNLayer(nn.Module):
    """forward of one ``GatedFeedforwardBlock`` (x + w2(silu(w1 n) * w3 n), n = RMSNorm(x)) on the sm_90a kernels;
    ``dtype="fp8"`` quantises the weights once and runs both GEMMs on MXFP8 operands"""

    def __init__(self, block: GatedFeedforwardBlock, device=None, dtype: str = "bf16"):
        super().__init__()
        if dtype not in ("bf16", "fp8"):
            raise ValueError(f"NativeGatedFFNLayer: dtype must be 'bf16' or 'fp8', got {dtype!r}")
        device = device or torch.device("cuda", torch.cuda.current_device())
        self.dtype = dtype
        self.hid, self.inner = block.w1.in_features, block.w1.out_features
        if any(lin.bias is not None for lin in (block.w1, block.w2, block.w3)) or block.norm.weight is None or \
                block.norm.eps is None or not float(block.norm.eps) > 0:
            raise ValueError("NativeGatedFFNLayer: the block must have bias-free Linears and an RMSNorm with a weight and "
                             "an eps > 0")
        if self.hid % 128 or not 128 <= self.hid <= K.LN_MAX_WIDTH or self.inner % 128:
            raise ValueError(f"NativeGatedFFNLayer: hidden must be a multiple of 128 in [128, {K.LN_MAX_WIDTH}] and "
                             f"inner a multiple of 128; got {self.hid}, {self.inner}")
        if dtype == "fp8" and (self.hid % 256 or self.inner % 256):
            raise ValueError(f"NativeGatedFFNLayer: fp8 needs hidden and inner multiples of 256; got {self.hid}, "
                             f"{self.inner}")
        self.eps = float(block.norm.eps)
        self.g = block.norm.weight.detach().to(device=device, dtype=torch.float32).contiguous()
        w13 = torch.cat([block.w1.weight.detach(), block.w3.weight.detach()]).to(device)
        w2 = block.w2.weight.detach().to(device)
        if dtype == "fp8":
            self.w13, self.w2 = (fp8.quantize(w.float().contiguous(), tile_rows=fp8.WEIGHT_TILE, groups=1)
                                 for w in (w13, w2))
        else:
            self.w13, self.w2 = (w.to(torch.bfloat16).unsqueeze(0).contiguous() for w in (w13, w2))
        self._ws = {}

    def _workspace(self, rows, device):
        ws = self._ws.get(rows)
        if ws is None:
            bf = dict(dtype=torch.bfloat16, device=device)
            ws = dict(h=torch.empty(rows, 2 * self.inner, **bf), rstd=torch.empty(rows, device=device))
            if self.dtype == "fp8":
                ws["nq"] = fp8.MXFP8Tensor(rows, 1, self.hid, fp8.ACT_TILE, device)
                ws["aq"] = fp8.MXFP8Tensor(rows, 1, self.inner, fp8.ACT_TILE, device)
            else:
                ws["n"] = torch.empty(rows, self.hid, **bf)
                ws["a"] = torch.empty(rows, self.inner, **bf)
            self._ws = {rows: ws}
        return ws

    @torch.no_grad()
    def forward(self, x, out=None):
        """x: [rows, hid] bf16 (rows % 256 == 0); returns bf16 [rows, hid] (written into ``out`` when given)"""
        rows, hid = x.shape
        assert hid == self.hid and rows % 256 == 0 and x.dtype == torch.bfloat16 and x.is_contiguous()
        ws = self._workspace(rows, x.device)
        if out is None:
            out = torch.empty_like(x)
        plan = RowPlan()   # 128-row tiles of one group
        if self.dtype == "fp8":   # no bf16 n or a: nothing reads them
            K.rms_norm_fwd(x, self.g, self.eps, out=None, rstd=ws["rstd"], quant=ws["nq"])
            swiglu_mlp_forward_fp8(plan, self.w13, self.w2, ws["nq"], ws["h"], None, ws["aq"], out, residual=x)
        else:
            K.rms_norm_fwd(x, self.g, self.eps, out=ws["n"], rstd=ws["rstd"])
            swiglu_mlp_forward(plan, self.w13, self.w2, ws["n"], ws["h"], ws["a"], out, residual=x)
        return out
