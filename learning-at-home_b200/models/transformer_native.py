"""
sm_90a execution of the transformer expert (post-LN encoder layer, GELU; architecture of
the reference's experiments/throughput/layers.py:22-51): QKV / out / MLP projections on the 128 x 256-tile wgmma GEMM with
fused bias / GELU / residual epilogues, attention on csrc/attention.cu (S and P never leave the SM), LayerNorm on
csrc/layernorm.cu.  Forward (inference / throughput experiment) only; training of transformer experts goes through
``ExpertBackend``, whose sm_90a executor (runtime/native_executor.py) trains the same layer.  Dropout is the identity here
(the throughput experiment is forward-only; see DESIGN.md).  Any sequence length 1 <= S <= kernels.MAX_SEQ: the token rows
are padded with zeros to a multiple of 128 for the GEMM and LayerNorm kernels, and attention sees only the real rows.
"""
import torch
import torch.nn as nn

from ..ops import gemm, kernels as K
from .layers import TransformerEncoderLayer


class NativeTransformerLayer(nn.Module):
    def __init__(self, layer: TransformerEncoderLayer, device=None):
        super().__init__()
        device = device or torch.device("cuda", torch.cuda.current_device())
        attn = layer.self_attn
        self.d_model, self.num_heads = attn.embed_dim, attn.num_heads
        self.causal = bool(layer.causal)   # a causal layer runs the causal attention kernel, never the bidirectional one
        assert self.d_model % self.num_heads == 0 and self.d_model // self.num_heads in K.HEAD_DIMS, \
            f"the attention kernels run head_dim {K.HEAD_DIMS}, not {self.d_model} / {self.num_heads}"

        def w(t):  # [1, N, K] bf16: the grouped GEMM with a single group
            return t.detach().to(device=device, dtype=torch.bfloat16).unsqueeze(0).contiguous()

        def f(t):
            return t.detach().to(device=device, dtype=torch.float32).unsqueeze(0).contiguous()

        self.w_in, self.b_in = w(attn.in_proj_weight), f(attn.in_proj_bias)
        self.w_out, self.b_out = w(attn.out_proj.weight), f(attn.out_proj.bias)
        self.w1, self.b1 = w(layer.linear1.weight), f(layer.linear1.bias)
        self.w2, self.b2 = w(layer.linear2.weight), f(layer.linear2.bias)
        self.g1, self.be1 = f(layer.norm1.weight), f(layer.norm1.bias)
        self.g2, self.be2 = f(layer.norm2.weight), f(layer.norm2.bias)
        self._ws = {}

    def _workspace(self, tokens, device):
        ws = self._ws.get(tokens)
        if ws is None:
            bf = dict(dtype=torch.bfloat16, device=device)
            d, ff = self.d_model, self.w1.shape[1]
            ws = dict(x=torch.empty(tokens, d, **bf), qkv=torch.empty(tokens, 3 * d, **bf), att=torch.empty(tokens, d, **bf),
                      h=torch.empty(tokens, d, **bf),
                      x1=torch.empty(tokens, d, **bf), f=torch.empty(tokens, ff, **bf), y=torch.empty(tokens, d, **bf),
                      mean=torch.empty(tokens, device=device), rstd=torch.empty(tokens, device=device))
            self._ws = {tokens: ws}
        return ws

    @torch.no_grad()
    def forward(self, src, out=None):
        """src: [batch, S, d_model] (bf16 preferred), 1 <= S <= kernels.MAX_SEQ; returns a bf16 tensor of the same shape"""
        batch, seq, d = src.shape
        assert 1 <= seq <= K.MAX_SEQ and d == self.d_model, (tuple(src.shape), self.d_model)
        rows = batch * seq
        tokens = (rows + 127) // 128 * 128
        x = src.reshape(rows, d)
        ws = self._workspace(tokens, x.device)
        if tokens > rows:   # zero padding rows; attention writes only the real rows of att
            ws["x"][:rows].copy_(x)
            ws["x"][rows:].zero_()
            ws["att"][rows:].zero_()
            x = ws["x"]
        elif x.dtype != torch.bfloat16 or not x.is_contiguous():
            x = x.to(torch.bfloat16).contiguous()
        gemm.grouped_linear(x, self.w_in, bias=self.b_in, out=ws["qkv"])
        K.attention_fwd(ws["qkv"][:rows], self.num_heads, out=ws["att"][:rows], seq_len=seq, causal=self.causal)
        gemm.grouped_linear(ws["att"], self.w_out, bias=self.b_out, residual=x, out=ws["h"])
        K.ln_relu_fwd(ws["h"], self.g1, self.be1, None, out=ws["x1"], mean=ws["mean"], rstd=ws["rstd"], relu=False)
        gemm.grouped_linear(ws["x1"], self.w1, bias=self.b1, out=ws["f"], act=2)
        gemm.grouped_linear(ws["f"], self.w2, bias=self.b2, residual=ws["x1"], out=ws["y"])
        if tokens > rows:
            res = torch.empty(tokens, d, dtype=torch.bfloat16, device=x.device)
            K.ln_relu_fwd(ws["y"], self.g2, self.be2, None, out=res, mean=ws["mean"], rstd=ws["rstd"], relu=False)
            res = res[:rows]
            out = res if out is None else out.view(rows, d).copy_(res)
            return out.view(batch, seq, d)
        out = torch.empty(rows, d, dtype=torch.bfloat16, device=x.device) if out is None else out.view(rows, d)
        K.ln_relu_fwd(ws["y"], self.g2, self.be2, None, out=out, mean=ws["mean"], rstd=ws["rstd"], relu=False)
        return out.view(batch, seq, d)
