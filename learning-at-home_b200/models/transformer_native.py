"""
sm_90a execution of the transformer expert (post-LN encoder layer, GELU; architecture of
the reference's experiments/throughput/layers.py:22-51): QKV / out / MLP projections on the wide-tile wgmma GEMM with
fused bias / GELU / residual epilogues, attention on csrc/attention.cu (S and P never leave the SM), LayerNorm on
csrc/layernorm.cu.  Forward (inference / throughput experiment) only; training of transformer experts goes through the
PyTorch module (``TransformerEncoderLayer`` + ``ExpertBackend``), which — unlike the reference's — is trainable.
Dropout is the identity here (the throughput experiment is forward-only; see DESIGN.md).
"""
import torch
import torch.nn as nn

from ..ops import gemm, kernels as K
from .layers import TransformerEncoderLayer, SEQ_LEN


class NativeTransformerLayer(nn.Module):
    def __init__(self, layer: TransformerEncoderLayer, device=None):
        super().__init__()
        device = device or torch.device("cuda", torch.cuda.current_device())
        attn = layer.self_attn
        self.d_model, self.num_heads = attn.embed_dim, attn.num_heads
        assert self.d_model // self.num_heads == 64, "the attention kernel is specialised for head_dim = 64"

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
            ws = dict(qkv=torch.empty(tokens, 3 * d, **bf), att=torch.empty(tokens, d, **bf), h=torch.empty(tokens, d, **bf),
                      x1=torch.empty(tokens, d, **bf), f=torch.empty(tokens, ff, **bf), y=torch.empty(tokens, d, **bf),
                      mean=torch.empty(tokens, device=device), rstd=torch.empty(tokens, device=device))
            self._ws = {tokens: ws}
        return ws

    @torch.no_grad()
    def forward(self, src, out=None):
        """src: [batch, 512, d_model] (bf16 preferred); returns a bf16 tensor of the same shape"""
        batch, seq, d = src.shape
        assert seq == SEQ_LEN and d == self.d_model
        x = src.reshape(batch * seq, d)
        if x.dtype != torch.bfloat16 or not x.is_contiguous():
            x = x.to(torch.bfloat16).contiguous()
        ws = self._workspace(batch * seq, x.device)
        gemm.grouped_linear(x, self.w_in, bias=self.b_in, out=ws["qkv"], two_cta=True)
        K.attention_fwd(ws["qkv"], self.num_heads, out=ws["att"])
        gemm.grouped_linear(ws["att"], self.w_out, bias=self.b_out, residual=x, out=ws["h"], two_cta=True)
        K.ln_relu_fwd(ws["h"], self.g1, self.be1, None, out=ws["x1"], mean=ws["mean"], rstd=ws["rstd"], relu=False)
        gemm.grouped_linear(ws["x1"], self.w1, bias=self.b1, out=ws["f"], two_cta=True, act=2)
        gemm.grouped_linear(ws["f"], self.w2, bias=self.b2, residual=ws["x1"], out=ws["y"], two_cta=True)
        out = torch.empty(batch * seq, d, dtype=torch.bfloat16, device=x.device) if out is None else out.view(batch * seq, d)
        K.ln_relu_fwd(ws["y"], self.g2, self.be2, None, out=out, mean=ws["mean"], rstd=ws["rstd"], relu=False)
        return out.view(batch, seq, d)
