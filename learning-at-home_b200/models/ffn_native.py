"""
sm_90a forward of the FFN expert (``FeedforwardBlock``, the reference's experiments/throughput/layers.py:5-19) for the
forward-only throughput experiment: three wgmma GEMMs with fused bias (+ residual) epilogues and the fused
LayerNorm+ReLU kernel in between.  ``dtype="fp8"`` runs the GEMMs on block-scaled FP8 tensor cores (MXFP8); LayerNorm
then emits the next GEMM's FP8 operand directly and no bf16 activation is written at all.
"""
import torch
import torch.nn as nn

from ..ops import fp8, gemm, kernels as K
from .layers import FeedforwardBlock


class NativeFFNLayer(nn.Module):
    def __init__(self, block: FeedforwardBlock, device=None, dtype: str = "bf16"):
        super().__init__()
        device = device or torch.device("cuda", torch.cuda.current_device())
        self.dtype = dtype
        lin1, ln1, lin2, ln2, lin3 = (block.layers[i] for i in (0, 1, 3, 4, 6))
        self.hid, self.inner = lin1.in_features, lin1.out_features

        def f(t):
            return t.detach().to(device=device, dtype=torch.float32).unsqueeze(0).contiguous()

        self.b = [f(m.bias) for m in (lin1, lin2, lin3)]
        self.ln = [(f(m.weight), f(m.bias)) for m in (ln1, ln2)]
        ws = [m.weight.detach().to(device=device) for m in (lin1, lin2, lin3)]
        if dtype == "fp8":
            self.w = [fp8.quantize(w.float().contiguous(), tile_rows=fp8.WEIGHT_TILE, groups=1) for w in ws]
        else:
            self.w = [w.to(torch.bfloat16).unsqueeze(0).contiguous() for w in ws]
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
        (g1, be1), (g2, be2) = self.ln
        if self.dtype == "fp8":
            fp8.quantize(x, out=ws["xq"])
            fp8.grouped_linear_fp8(ws["xq"], self.w[0], bias=self.b[0], out=ws["h"])
            K.ln_relu_fwd(ws["h"], g1, be1, None, out=None, mean=None, rstd=None, quant=ws["aq"])
            fp8.grouped_linear_fp8(ws["aq"], self.w[1], bias=self.b[1], out=ws["h"])
            K.ln_relu_fwd(ws["h"], g2, be2, None, out=None, mean=None, rstd=None, quant=ws["aq"])
            fp8.grouped_linear_fp8(ws["aq"], self.w[2], bias=self.b[2], residual=x, out=out)
        else:
            mean = rstd = ws.setdefault("stat", torch.empty(rows, device=x.device))
            gemm.grouped_linear(x, self.w[0], bias=self.b[0], out=ws["h"], two_cta=True)
            K.ln_relu_fwd(ws["h"], g1, be1, None, out=ws["a"], mean=mean, rstd=rstd)
            gemm.grouped_linear(ws["a"], self.w[1], bias=self.b[1], out=ws["h"], two_cta=True)
            K.ln_relu_fwd(ws["h"], g2, be2, None, out=ws["a"], mean=mean, rstd=rstd)
            gemm.grouped_linear(ws["a"], self.w[2], bias=self.b[2], residual=x, out=out, two_cta=True)
        return out
