"""
sm_90a forward of the FFN expert (``FeedforwardBlock``, the reference's experiments/throughput/layers.py:5-19) for the
forward-only throughput experiment: three wgmma GEMMs with fused bias (+ residual) epilogues and the fused
LayerNorm+ReLU kernel in between.  ``dtype="fp8"`` runs the GEMMs on block-scaled FP8 tensor cores (MXFP8); LayerNorm
then emits the next GEMM's FP8 operand directly and no bf16 activation is written at all.
"""
import torch
import torch.nn as nn

from ..ops import fp8
from ..ops.expert_blocks import RowPlan, ffn_forward, ffn_forward_fp8
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
