"""
The expert programs as sm_90a kernel chains, written once for the routed and shared experts of ``FusedDMoE``, the
``ExpertBackend`` executors, ``NativeFFNLayer`` and ``NativeGatedFFNLayer``: ``FeedforwardBlock`` (``ffn_forward``,
``ffn_forward_fp8``, ``ffn_backward``) and the MLP of ``GatedFeedforwardBlock`` after its RMSNorm, which stays with each
caller (``swiglu_mlp_forward``, ``swiglu_mlp_forward_fp8``, ``swiglu_mlp_backward``).  A ``RowPlan`` says how one call's
kernels see their rows.

Weight gradients go to the caller's ``wgrad(name, dy, x)``.  The backward functions call it for a matrix only after the
dgrad that reads that matrix, so the callback may update the weights in place (fused wgrad + AMSGrad).
"""
from typing import NamedTuple, Optional

import torch

from . import fp8, gemm, kernels as K


class RowPlan(NamedTuple):
    """How the kernels of one call see their rows.

    group_off, group_rows: int32 group tables.  With ``group_rows`` the GEMMs are swap-AB (``K.swapab_linear``), without
        it they run on 128-row tiles (``gemm.grouped_linear``) mapped by ``tile_group``
    tile_group, tile_rows: the group of every ``tile_rows`` rows, for the LayerNorm and column-sum kernels
    rows: the rows the LayerNorm, column-sum and SwiGLU kernels cover (None = whole buffers); GEMMs take whole buffers
    max_ctas: the CTA limit of the backward GEMMs (0 = none)
    """
    group_off: Optional[torch.Tensor] = None
    group_rows: Optional[torch.Tensor] = None
    tile_group: Optional[torch.Tensor] = None
    tile_rows: int = 128
    rows: Optional[int] = None
    max_ctas: int = 0

    def linear(self, x, w, **kw):
        if self.group_rows is not None:
            return K.swapab_linear(x, w, self.group_off, self.group_rows, **kw)
        return gemm.grouped_linear(x, w, tile_group=self.tile_group, **kw)

    def dgrad(self, dy, w, **kw):
        return self.linear(dy, w, w_is_kn=True, max_ctas=self.max_ctas, **kw)

    def span(self, t):
        return t if t is None or self.rows is None else t[:self.rows]

    def ln_relu_fwd(self, h, gamma, beta, out, mean, rstd, quant=None):
        K.ln_relu_fwd(self.span(h), gamma, beta, self.tile_group, out=self.span(out), mean=mean, rstd=rstd, quant=quant,
                      tile_rows=self.tile_rows)

    def ln_relu_bwd(self, da, h, mean, rstd, gamma, beta, dh, dgamma, dbeta, dbias):
        K.ln_relu_bwd(self.span(da), self.span(h), mean, rstd, gamma, beta, self.tile_group, dh=self.span(dh),
                      dgamma=dgamma, dbeta=dbeta, dbias=dbias, tile_rows=self.tile_rows)


# FeedforwardBlock.  w: bf16 weights "w1", "w2", "w3"; p: fp32 "b1", "b2", "b3", "g1", "be1", "g2", "be2"; acts: the
# forward's activations (h1, a1, h2, a2); stats: its LayerNorm statistics (mean1, rstd1, mean2, rstd2)
def ffn_forward(plan: RowPlan, w, p, x, acts, stats, y, wait=None):
    """y = x + Linear3(LN-ReLU(Linear2(LN-ReLU(Linear1(x))))); ``wait``: the first GEMM's receive-side flag wait"""
    h1, a1, h2, a2 = acts
    mean1, rstd1, mean2, rstd2 = stats
    plan.linear(x, w["w1"], out=h1, bias=p["b1"], wait=wait)
    plan.ln_relu_fwd(h1, p["g1"], p["be1"], a1, mean1, rstd1)
    plan.linear(a1, w["w2"], out=h2, bias=p["b2"])
    plan.ln_relu_fwd(h2, p["g2"], p["be2"], a2, mean2, rstd2)
    plan.linear(a2, w["w3"], out=y, bias=p["b3"], residual=x)


def ffn_forward_fp8(plan: RowPlan, w8, p, x, xq, aq, acts, stats, y):
    """``ffn_forward`` on block-scaled FP8 tensor cores: x is quantised into ``xq``, each LayerNorm writes the next GEMM's
    MXFP8 operand ``aq`` (and the bf16 activation unless it is None)"""
    h1, a1, h2, a2 = acts
    mean1, rstd1, mean2, rstd2 = stats
    fp8.quantize(x, tile_group=plan.tile_group, out=xq)
    fp8.grouped_linear_fp8(xq, w8["w1"], tile_group=plan.tile_group, bias=p["b1"], out=h1)
    plan.ln_relu_fwd(h1, p["g1"], p["be1"], a1, mean1, rstd1, quant=aq)
    fp8.grouped_linear_fp8(aq, w8["w2"], tile_group=plan.tile_group, bias=p["b2"], out=h2)
    plan.ln_relu_fwd(h2, p["g2"], p["be2"], a2, mean2, rstd2, quant=aq)
    fp8.grouped_linear_fp8(aq, w8["w3"], tile_group=plan.tile_group, bias=p["b3"], residual=x, out=y)


def ffn_backward(plan: RowPlan, w, p, g, x, acts, stats, gy, da, dh2, dh1, dx, wgrad):
    """dx = gy + the chain's input gradient; bias and LayerNorm gradients are added into ``g`` (the keys of ``p``).
    dh2 and dh1 may be one buffer when ``wgrad`` has read dh2 before later launches on the stream write dh1."""
    h1, a1, h2, a2 = acts
    mean1, rstd1, mean2, rstd2 = stats
    K.grouped_colsum(plan.span(gy), plan.tile_group, out=g["b3"], tile_rows=plan.tile_rows)
    plan.dgrad(gy, w["w3"], out=da)
    wgrad("w3", gy, a2)
    plan.ln_relu_bwd(da, h2, mean2, rstd2, p["g2"], p["be2"], dh2, g["g2"], g["be2"], g["b2"])
    plan.dgrad(dh2, w["w2"], out=da)
    wgrad("w2", dh2, a1)
    plan.ln_relu_bwd(da, h1, mean1, rstd1, p["g1"], p["be1"], dh1, g["g1"], g["be1"], g["b1"])
    plan.dgrad(dh1, w["w1"], out=dx, residual=gy)
    wgrad("w1", dh1, x)


# GatedFeedforwardBlock after its RMSNorm
def swiglu_mlp_forward(plan: RowPlan, w13, w2, n, h, a, y, residual=None):
    """h = [hg | hu] = n [W1; W3]^T (one GEMM), a = silu(hg) * hu, y = a W2^T (+ residual)"""
    plan.linear(n, w13, out=h)
    K.swiglu_fwd(plan.span(h), out=plan.span(a))
    plan.linear(a, w2, out=y, residual=residual)


def swiglu_mlp_forward_fp8(plan: RowPlan, w13q, w2q, nq, h, a, aq, y, residual=None):
    """``swiglu_mlp_forward`` on block-scaled FP8 tensor cores, from the MXFP8 copy ``nq`` of n (the caller's RMSNorm
    writes it): h = nq [W1; W3]^T in bf16, then the SwiGLU writes the W2 operand ``aq`` (and the bf16 a unless it is
    None), y = aq W2^T (+ residual).  Rows of -1 tiles of ``plan.tile_group`` are skipped throughout"""
    fp8.grouped_linear_fp8(nq, w13q, tile_group=plan.tile_group, out=h)
    K.swiglu_fwd(plan.span(h), out=plan.span(a), quant=aq, tile_group=plan.tile_group)
    fp8.grouped_linear_fp8(aq, w2q, tile_group=plan.tile_group, residual=residual, out=y)


def swiglu_mlp_backward(plan: RowPlan, w13, w2, n, h, a, gy, da, dh, dn, wgrad):
    """dn, the gradient of n (the residual's gradient is the caller's), and the ``wgrad`` calls of w2 and w13"""
    plan.dgrad(gy, w2, out=da)
    wgrad("w2", gy, a)
    K.swiglu_bwd(plan.span(da), plan.span(h), out=plan.span(dh))
    plan.dgrad(dh, w13, out=dn)
    wgrad("w13", dh, n)
