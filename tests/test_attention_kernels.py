"""
The attention kernels (csrc/attention.cu forward, csrc/attention_bwd.cu backward with its Delta prologue and dQ reduction)
and the element-wise dropout kernels of the transformer expert (csrc/dropout.cu), element by element against float64
oracles, in the style of test_expert_kernels.py.

Every oracle runs in float64 on the same bf16 operands the kernels read, one (batch, head) at a time, in chunks of query
rows for long sequences.  With c = log2(e) / sqrt(HD), x = c q k^T, the valid keys of a query (k < S, not masked, k <= q
when causal), lse2 = log2 sum_valid 2^x, p = 2^(x - lse2), the site-0 keep mask M and r = the fp32 1 / (1 - p_drop):

    out = r (M o p) V                        (a query without a valid key: out = 0, lse2 = +inf)
    backward from the kernel's own lse and out (as ln_bwd64 starts from the kernel's statistics):
    P = 2^(x - lse_kernel), Delta = rowsum(dO o out_kernel), dS = P o (r M o dO V^T - Delta) / sqrt(HD),
    dV = r (M o P)^T dO, dK = dS^T Q, dQ = dS K

Each element has its own bound.  U = 2^-24 (an fp32 rounding), EPS_BF16 = 2^-8 (a bf16 rounding), C_ACC = 4 (the constant
of every fp32 summation of depth n: C_ACC n U (sum of the absolute terms)); |A||B| is the float64 product of absolute values.

Forward.  The kernel forms P~ = bf16(ex2(fma(s, c~, -fl(m c~)))) per 128-key block against the running row maximum m,
rescales the accumulators by alpha = ex2((m_old - m_new) c~) and returns out = bf16(o r / l), lse2 = m c~ + lg2(l).
  - argument of ex2 (log2 units) for key k processed in the block with running maximum cm_k (final cm_f):
        D_k = C_ACC c HD U (|Q||K|^T)                      scores: fp32 wgmma of HD products
            + 4 U |x|                                      FMA rounding; c~ = fp32(log2e) / sqrtf(HD) is within 3 U of c
            + 10 U |cm_k| + 5 U |cm_f|                     the rounded m c~, and the alphas of the later blocks
                                                           (m_old - m_new, its product with c~, c~ itself: 5 U per step)
  - relative error of the effective weight of key k:  eps_k = (1 + EPS_BF16)(1 + 4U)^(nkb + 1) 2^D_k - 1
        (the bf16 rounding of P~, ex2.approx (2 ulp) of P~ and of every later alpha); a flushed subnormal adds TINY
  - the kernel divides by l = the sum of the SAME rounded weights, so with A = r (M o p eps)|V|, B = sum_k p_k eps_k:
        |out - ref| <= EPS_BF16 |out| + (1 + EPS_BF16) ((A + B |out|) / (1 - B) + C_ACC U (S (r (M o p)|V|) + D_l |out|)
                                                          + 4 U |out|)
        S: the depth of the fp32 P V accumulation; D_l = 36 + 2 nkb: the per-thread sum of 32 weights per block, the
        chain over blocks with its alpha products and the quad reduction; 4 U: the approximate division
  - |lse2 - ref| <= -log2(1 - B) + C_ACC D_l U / ln 2 + 2^-21 (lg2.approx) + 2 U |lse2|
Backward.  The kernel recomputes P_b = ex2(fma(s, c_b, -lse)) in fp32 (c_b = fp32(1 / sqrtf(HD)) fp32(log2e)).
  - argument:  D_b = C_ACC c HD U (|Q||K|^T) + U |lse| + 5 U |x|;  eps_b = (1 + 4U) 2^D_b - 1;  P~ = bf16(M o P_b) for dV:
    eps_pp = (1 + eps_b)(1 + EPS_BF16) - 1
  - dP = dO V^T: C_ACC HD U (|dO||V|^T); Delta: C_ACC HD U sum |dO o out|; the subtraction and the dropout product 2 U
    (r M |dP| + |Delta|): together e_t
  - dS (stored once as bf16, used by dK and dQ):
        e_dS = EPS_BF16 |dS| + (1 + EPS_BF16) (|dS| (eps_b + 4 U) + P (1 + eps_b) e_t / sqrt(HD))    (4 U: fp32 1/sqrt(HD)
        and two products)
  - dV: EPS_BF16 |dV| + (1 + EPS_BF16) (r (M o P eps_pp)^T |dO| + C_ACC S U r (M o P)^T |dO| + U |dV|)
  - dK: EPS_BF16 |dK| + (1 + EPS_BF16) (e_dS^T |Q| + C_ACC S U (|dS| + e_dS)^T |Q|)
  - dQ: the bf16 partial of every 128-key block j (dq_part), summed in fp32 over nkb blocks:
        e_part = e_dS |K| + C_ACC 128 U (|dS| + e_dS)|K|
        EPS_BF16 |dQ| + (1 + EPS_BF16) ((1 + EPS_BF16) e_part + (EPS_BF16 + C_ACC nkb U) (sum_j |part_j| + e_part))
        with part_j = dS[:, block j] K[block j] formed in float64

Exact where the kernels are exact: a sequence without a valid key has out = 0, dqkv = 0 and lse = +inf; the dK / dV rows of
masked keys are 0; p = 0 is byte-equal to no dropout; every row past the T tokens of a larger out / lse / dqkv buffer keeps
its canary bytes; zero tokens touch nothing; two identical calls are byte-equal, forward and backward.

Inputs target the online softmax and the masking: gauss (randn * 0.5 / 1.5); sharp (scores over about +-60 log2 units:
near one-hot rows, most P~ underflow); rising (+24 log2 units per 128-key block: the row maximum arrives in the last block
and every alpha is large); falling (the maximum in block 0, later blocks round to 0); negative (every valid score below
-30 log2 units; masked keys score +34 and the zero-filled keys past S exactly 0; in causal mode key q + d of the diagonal
block scores above every valid key, >= 0 from d = 8: a leaked key dominates); ties (q = 0, or all keys equal: exactly
uniform P).  dO is either randn or aligned with out (dP - Delta cancels).

Dropout element-wise ops (sites 1-3, exact site masks from dropout_mask): apply and ReLU are one fp32 product and a bf16
rounding: EPS_BF16 |ref| + (1 + EPS_BF16) U |ref|.  GELU adds erff (2 ulp: C_ACC U |erf|), its rounded argument
(2/sqrt(pi) e^-z^2 2 U |z|), the 1 + erf sum and the products; gelu' adds __expf (C_ACC U (x^2 / 2 + 2) relative).

The CPU tests check the float64 oracles against torch.autograd of explicit softmax attention and of the element-wise ops.
"""
import math

import pytest
import torch
import torch.nn.functional as F

import lah_b200  # noqa: F401
from lah_b200.ops import kernels as K
from test_expert_kernels import (BF16, C_ACC, EPS_BF16, SENTINEL, U, f32, gelu64, report_worst_ratios,  # noqa: F401
                                 sentinel_like, untouched, within)
from test_key_padding_mask import mask_families

LN2 = math.log(2.0)
LOG2E = 1.0 / LN2
KB = 128                  # keys per block of both kernels; dq_part holds one partial per block
TINY = 2.0 ** -120        # a weight flushed to zero (ex2.approx.ftz) or a subnormal accumulator: far below any bound term
ROWS_PER_CHUNK = 2 ** 26  # query rows x keys of one float64 oracle chunk


# ---------------------------------------------------------------------------------------------------------------- oracles
def _absfin(t):
    return torch.where(torch.isfinite(t), t.abs(), torch.zeros_like(t))


def attn_fwd64(q, k, v, valid, keep=None, r=1.0):
    """
    float64 forward of one (batch, head): query rows q [R, HD] against the keys / values k, v [S, HD] of the sequence
    (key 0 starts block 0); valid, keep: bool [R, S].  Returns (out, lse2, bound of out, bound of lse2); a row without a
    valid key gets out = 0, lse2 = +inf.
    """
    R, HD = q.shape
    S = k.shape[0]
    nkb = -(-S // KB)
    c = LOG2E / math.sqrt(HD)
    qd, kd, vd = q.double(), k.double(), v.double()
    x = c * (qd @ kd.t())
    xm = x.masked_fill(~valid, -math.inf)
    live = valid.any(1)
    lse2 = torch.where(live, torch.logsumexp(xm * LN2, 1) / LN2, torch.full_like(xm[:, 0], math.inf))
    p = torch.exp2(xm - lse2[:, None])                       # 0 for invalid keys and rows without a valid key
    wk = keep.double() * r if keep is not None else torch.ones_like(p)
    o = (p * wk) @ vd
    # running row maximum (log2 units) after each block, as the kernel meets the blocks in order
    blk = F.pad(xm, (0, nkb * KB - S), value=-math.inf).view(R, nkb, KB).amax(-1).cummax(1).values
    cm = blk.repeat_interleave(KB, 1)[:, :S]
    D = C_ACC * c * HD * U * (qd.abs() @ kd.abs().t()) + 4 * U * x.abs() + 10 * U * _absfin(cm) + 5 * U * _absfin(blk[:, -1:])
    eps = (1 + EPS_BF16) * (1 + 4 * U) ** (nkb + 1) * torch.exp2(D) - 1
    pe = torch.where(valid, p * eps + TINY, torch.zeros_like(p))
    A = (pe * wk) @ vd.abs()
    B = pe.sum(1, keepdim=True)
    A0 = (p * wk) @ vd.abs()
    D_l = 36 + 2 * nkb
    oa = o.abs()
    b_o = EPS_BF16 * oa + (1 + EPS_BF16) * ((A + B * oa) / (1 - B) + C_ACC * U * (S * A0 + D_l * oa) + 4 * U * oa)
    b_lse = -torch.log2(1 - B[:, 0]) + C_ACC * D_l * U / LN2 + 2.0 ** -21 + 2 * U * _absfin(lse2)
    return o, lse2, b_o, b_lse


def attn_bwd64(q, k, v, dout, out, lse2, valid, keep=None, r=1.0):
    """
    float64 backward of one (batch, head) from the kernel's lse2 [R] and out [R, HD] of the query rows q [R, HD]: returns
    dict(dq [R, HD] with its bound e_dq, and the contributions of these rows to dk, dv [S, HD] and to the terms s_dk, s_dv
    of their bounds (kv_bounds)).
    """
    R, HD = q.shape
    S = k.shape[0]
    nkb = -(-S // KB)
    c = LOG2E / math.sqrt(HD)
    sq = math.sqrt(HD)
    qd, kd, vd, dod, od = q.double(), k.double(), v.double(), dout.double(), out.double()
    l2 = lse2.double()
    x = c * (qd @ kd.t())
    ok = valid & torch.isfinite(l2)[:, None]
    l2f = torch.where(torch.isfinite(l2), l2, torch.zeros_like(l2))
    P = torch.where(ok, torch.exp2(x - l2f[:, None]), torch.zeros_like(x))
    delta = (dod * od).sum(1, keepdim=True)
    dP = dod @ vd.t()
    Mr = keep.double() * r if keep is not None else torch.ones_like(P)
    t = Mr * dP - delta
    dS = P * t / sq
    res = dict(dv=(Mr * P).t() @ dod, dk=dS.t() @ qd, dq=dS @ kd)
    # bounds
    Db = C_ACC * c * HD * U * (qd.abs() @ kd.abs().t()) + U * l2f.abs()[:, None] + 5 * U * x.abs()
    eps_b = torch.where(ok, (1 + 4 * U) * torch.exp2(Db) - 1, torch.zeros_like(P))
    eps_pp = (1 + eps_b) * (1 + EPS_BF16) - 1
    tiny = ok.double() * TINY
    e_t = Mr * C_ACC * HD * U * (dod.abs() @ vd.abs().t()) + C_ACC * HD * U * (dod.abs() * od.abs()).sum(1, keepdim=True) \
        + 2 * U * (Mr * dP.abs() + delta.abs())
    aS = dS.abs()
    e_dd = EPS_BF16 * aS + (1 + EPS_BF16) * (aS * (eps_b + 4 * U) + (P * (1 + eps_b) + tiny) * e_t / sq + tiny * t.abs() / sq)
    # the query sums of dK and dV: their terms add over chunks of query rows; kv_bounds finishes them
    res["s_dv"] = (Mr * (P * eps_pp + tiny)).t() @ dod.abs() + C_ACC * S * U * (Mr * P * (1 + eps_pp)).t() @ dod.abs()
    res["s_dk"] = e_dd.t() @ qd.abs() + C_ACC * S * U * ((aS + e_dd).t() @ qd.abs())
    kpad = F.pad(kd, (0, 0, 0, nkb * KB - S)).view(nkb, KB, HD)
    parts = torch.einsum("rjk,jkd->jrd", F.pad(dS, (0, nkb * KB - S)).view(R, nkb, KB), kpad)
    e_part = e_dd @ kd.abs() + C_ACC * KB * U * ((aS + e_dd) @ kd.abs())
    res["e_dq"] = EPS_BF16 * res["dq"].abs() + (1 + EPS_BF16) * (
        (1 + EPS_BF16) * e_part + (EPS_BF16 + C_ACC * nkb * U) * (parts.abs().sum(0) + e_part))
    return res


def kv_bounds(dk, dv, s_dk, s_dv):
    """bounds of dK and dV from the summed terms of attn_bwd64 over all query rows: the fp32 rescale of dV and the bf16
    stores"""
    return (EPS_BF16 * dk.abs() + (1 + EPS_BF16) * s_dk,
            EPS_BF16 * dv.abs() + (1 + EPS_BF16) * (s_dv + U * dv.abs()))


# element-wise dropout ops: (ref, bound) from the keep mask and the fp32 r the kernel multiplies by
def _erf_terms(x):
    """float64 erf(x / sqrt 2) and the bound of the kernel's 1 + erff(fl(x * fp32(1 / sqrt 2)))"""
    z = x / math.sqrt(2.0)
    e = torch.special.erf(z)
    err = C_ACC * U * e.abs() + 2 / math.sqrt(math.pi) * torch.exp(-z * z) * 2 * U * z.abs() + U * (1 + e)
    return e, err


def dropout_ew64(op, x, f, keep, r):
    """float64 ref and bound of lah_dropout_ew op (csrc/dropout.cu) at keep mask `keep` and scale r"""
    xd = x.double()
    s = keep.double() * r
    if op == "apply":
        ref, e = xd * s, torch.zeros_like(xd)
    elif op == "relu":
        ref, e = xd.clamp(min=0) * s, torch.zeros_like(xd)
    elif op == "relu_bwd":
        ref, e = (f.double() > 0) * xd * s, torch.zeros_like(xd)
    elif op == "gelu":
        erf, e_erf = _erf_terms(xd)
        g = 0.5 * xd * (1 + erf)
        ref = g * s
        e = s * (0.5 * xd.abs() * e_erf + U * g.abs())
    else:                                                   # gelu_bwd: gelu'(f) o M o dg r
        fd = f.double()
        erf, e_erf = _erf_terms(fd)
        t1 = 0.5 * (1 + erf)
        t2 = fd / math.sqrt(2 * math.pi) * torch.exp(-0.5 * fd * fd)
        gp = t1 + t2
        ref = gp * xd * s
        e_gp = 0.5 * e_erf + U * t1 + t2.abs() * C_ACC * U * (0.5 * fd * fd + 2) + U * gp.abs()
        e = (xd * s).abs() * e_gp + U * ref.abs()
    return ref, EPS_BF16 * ref.abs() + (1 + EPS_BF16) * (e + U * ref.abs())


# ---------------------------------------------------------------------------------------------------------------- CPU
def _explicit_attention(q, k, v, valid, keep, r):
    """autograd-able float64 softmax attention of one head; rows without a valid key give 0"""
    s = (q @ k.t()) / math.sqrt(q.shape[1])
    s = s.masked_fill(~valid, -math.inf)
    a = torch.softmax(s, dim=-1).nan_to_num(0.0)
    if keep is not None:
        a = a * keep.double() * r
    lse2 = torch.logsumexp(s, dim=-1) / LN2
    return a @ v, lse2


def _cpu_case(S, HD, masked, causal, p, seed):
    g = torch.Generator().manual_seed(seed)
    q, k, v, do = (torch.randn(S, HD, generator=g, dtype=torch.float64) * 1.3 for _ in range(4))
    valid = torch.ones(S, S, dtype=torch.bool)
    if masked:
        valid &= (torch.rand(S, generator=g) > 0.3)[None, :]
        valid[:, 5] = True
    if causal:
        valid &= torch.ones(S, S, dtype=torch.bool).tril()
    keep = torch.rand(S, S, generator=g) >= p if p else None
    return q, k, v, do, valid, keep, (1.0 / (1.0 - p) if p else 1.0)


CPU_CASES = [(300, 32, False, False, 0.0), (300, 64, True, False, 0.3), (200, 16, False, True, 0.5), (129, 128, True, False, 0.0)]


@pytest.mark.parametrize("S,HD,masked,causal,p", CPU_CASES)
def test_fwd_oracle_matches_explicit_softmax_attention(S, HD, masked, causal, p):
    q, k, v, _, valid, keep, r = _cpu_case(S, HD, masked, causal, p, S + HD)
    ref, lse_ref = _explicit_attention(q, k, v, valid, keep, r)
    o, lse2, b_o, b_lse = attn_fwd64(q, k, v, valid, keep, r)
    torch.testing.assert_close(o, ref, rtol=1e-12, atol=1e-12)
    # two float64 logsumexps of differently rounded scores: torch's vectorised CPU kernels have been seen to differ by
    # about 1e-10 between runs on the same host, so 1e-9 here (the bound of lse2 is above 2^-21)
    torch.testing.assert_close(lse2, lse_ref, rtol=1e-9, atol=1e-9)
    assert bool((b_o >= 0).all() and (b_lse > 0).all())
    # a row without a valid key: out = 0, lse2 = +inf
    dead = valid.clone()
    dead[3] = False
    o, lse2, _, _ = attn_fwd64(q, k, v, dead, keep, r)
    assert bool((o[3] == 0).all()) and lse2[3].item() == math.inf


@pytest.mark.parametrize("S,HD,masked,causal,p", CPU_CASES)
def test_bwd_oracle_matches_autograd(S, HD, masked, causal, p):
    q, k, v, do, valid, keep, r = _cpu_case(S, HD, masked, causal, p, 7 * S + HD)
    qa, ka, va = (t.clone().requires_grad_(True) for t in (q, k, v))
    out, lse2 = _explicit_attention(qa, ka, va, valid, keep, r)
    out.backward(do)
    res = attn_bwd64(q, k, v, do, out.detach(), lse2.detach(), valid, keep, r)
    e_dk, e_dv = kv_bounds(res["dk"], res["dv"], res["s_dk"], res["s_dv"])
    for name, grad, e in (("dq", qa.grad, res["e_dq"]), ("dk", ka.grad, e_dk), ("dv", va.grad, e_dv)):
        torch.testing.assert_close(res[name], grad, rtol=1e-10, atol=1e-12)
        assert bool((e >= 0).all())


def test_bwd_oracle_chunks_add_up():
    """dK and dV of a query-chunked oracle are the sums of the chunks' contributions; dQ of a chunk is its rows"""
    q, k, v, do, valid, keep, r = _cpu_case(260, 32, True, False, 0.2, 5)
    out, lse2 = _explicit_attention(q, k, v, valid, keep, r)
    whole = attn_bwd64(q, k, v, do, out, lse2, valid, keep, r)
    parts = [attn_bwd64(q[a:a + 100], k, v, do[a:a + 100], out[a:a + 100], lse2[a:a + 100], valid[a:a + 100],
                        keep[a:a + 100], r) for a in (0, 100, 200)]
    for name in ("dk", "dv", "s_dk", "s_dv"):
        torch.testing.assert_close(sum(x[name] for x in parts), whole[name], rtol=1e-12, atol=1e-14)
    torch.testing.assert_close(torch.cat([x["dq"] for x in parts]), whole["dq"], rtol=0, atol=0)


@pytest.mark.parametrize("op", ["apply", "relu", "relu_bwd", "gelu", "gelu_bwd"])
def test_dropout_refs_match_autograd(op):
    g = torch.Generator().manual_seed(3)
    x = torch.cat([torch.linspace(-10, 10, 401, dtype=torch.float64), torch.tensor([0.0, 1.4, -1.4, 1e-30, -1e-30])])
    keep = torch.rand(x.shape, generator=g) >= 0.3
    dg = torch.randn(x.shape, generator=g, dtype=torch.float64)
    r = 1 / 0.7
    xa = x.clone().requires_grad_(True)
    act = {"apply": lambda t: t, "relu": F.relu, "relu_bwd": F.relu, "gelu": gelu64, "gelu_bwd": gelu64}[op]
    y = act(xa) * keep * r
    if op.endswith("bwd"):
        y.backward(dg)
        ref, b = dropout_ew64(op, dg, x, keep, r)
        torch.testing.assert_close(ref, xa.grad, rtol=1e-12, atol=1e-15)
    else:
        ref, b = dropout_ew64(op, x, None, keep, r)
        torch.testing.assert_close(ref, y.detach(), rtol=1e-12, atol=1e-15)
    if op == "gelu":
        torch.testing.assert_close(ref, F.gelu(x) * keep * r, rtol=1e-12, atol=1e-15)
    assert bool((b >= 0).all())


# ---------------------------------------------------------------------------------------------------------------- inputs
def family_qkv(family, B, S, H, HD, seed, pad=None, causal=False):
    """qkv [B S, 3 H HD] bf16 of one input family (module docstring); pad: bool [B, S], True = masked key"""
    g = torch.Generator().manual_seed(seed)
    c = LOG2E / math.sqrt(HD)
    shape = (B, S, H, HD)
    rn = lambda s=1.0: torch.randn(*shape, generator=g) * s  # noqa: E731
    pos = torch.arange(S, dtype=torch.float32).view(1, S, 1)
    if family.startswith("gauss"):
        sc = float(family[5:])
        q, k, v = rn(sc), rn(sc), rn(sc)
    elif family == "sharp":                    # c s = log2(e) 3.7^2 N(0, 1): about +-60 at 3 sd
        q, k, v = rn(3.7), rn(3.7), rn()
    elif family in ("rising", "falling"):      # c s grows (falls) by 24 per 128-key block
        q, k, v = rn(0.5), rn(0.5), rn()
        q[..., 0] = 2.0
        k[..., 0] = (24 / (KB * c * 2)) * pos * (1 if family == "rising" else -1)
    elif family == "negative" and causal:
        # s = [same 128-key block] beta (key - query) - T, beta = T / 8, exactly (every product and sum is exact in bf16 /
        # fp32; the block test is a one-hot of the block index mod 8, so S <= 1024), plus a small noise: the own key and every
        # earlier one score <= -T (c T >= 32), key q + d of the block -T + d T / 8, above every valid key and >= 0 from d = 8
        assert S <= 8 * KB, S
        q, k, v = rn(0.3), rn(0.3), rn()
        T = 256.0 if HD <= 64 else 512.0
        beta = T / 8
        il, I = pos % KB - 64, torch.div(pos, KB, rounding_mode="floor").long()
        hot = F.one_hot(I.view(S) % 8, 8).float().view(1, S, 1, 8)
        q[..., :17] = torch.cat([hot, hot * il[..., None], torch.ones(1, S, 1, 1)], -1)
        k[..., :17] = torch.cat([hot * (beta * il[..., None]), hot * -beta, torch.full((1, S, 1, 1), -T)], -1)
    elif family == "negative":                 # valid keys: c s in [-44, -34]; masked keys c s = +34
        q, k, v = rn(0.3), rn(0.3), rn()
        T = 34 / c
        u = torch.rand(B, S, H, generator=g) * 10 / c
        masked = (pad.view(B, S, 1) if pad is not None else torch.zeros(B, S, 1, dtype=torch.bool)).expand(B, S, H)
        q[..., 0] = 2.0
        k[..., 0] = torch.where(masked, T / 2, -(T + u) / 2)
    elif family == "ties_q0":                  # q = 0: every score 0
        q, k, v = torch.zeros(shape), rn(), rn()
    elif family == "ties_k":                   # every key of a sequence and head equal
        q, k, v = rn(), rn()[:, :1].expand(shape).clone(), rn()
    else:
        raise ValueError(family)
    return torch.cat([t.reshape(B * S, H * HD) for t in (q, k, v)], 1).to(BF16).cuda()


def edge_masks(S):
    """bool [9, S], True = masked: only key 0 valid; only the last key valid; valid keys only in the last (partial)
    block; whole 128-key blocks masked between valid ones; validity switching at the word edges 31 / 32 / 33 (twice);
    every key masked; none masked; keys of one 32-key word masked in every block"""
    pos = torch.arange(S)
    last_block = KB * ((S - 1) // KB)
    rows = [pos != 0, pos != S - 1, pos < last_block if S > KB else pos < S // 2,
            (pos // KB) % 2 == 1 if S > KB else (pos // 32) % 2 == 1,
            (pos >= 31) & (pos < 33), (pos % 32 == 31) | (pos % 32 == 1),
            torch.ones(S, dtype=torch.bool), torch.zeros(S, dtype=torch.bool), (pos % KB >= 32) & (pos % KB < 64)]
    return torch.stack(rows)


def all_masks(S, seed=0):
    return torch.cat([mask_families(S, seed), edge_masks(S)])


# ---------------------------------------------------------------------------------------------------------------- GPU
def run_attention(qkv, H, S, *, pad=None, causal=False, p=0.0, seed=0, dout="randn", bwd=True):
    """forward (and backward) twice each into canary-filled buffers 3 rows longer than T; every output against the float64
    oracle, element by element; returns (out, lse, dqkv)"""
    T, D = qkv.shape[0], qkv.shape[1] // 3
    HD, B = D // H, T // S
    km = K.pack_key_mask(pad.cuda()) if pad is not None else None
    kw = dict(seq_len=S, key_mask=km, causal=causal, dropout=(p, seed) if p else None)
    runs = []
    for _ in range(2):
        of, lf = sentinel_like((T + 3, D), BF16), sentinel_like((T + 3, H), torch.float32)
        K.attention_fwd(qkv, H, out=of[:T], lse=lf[:T], **kw)
        runs.append((of, lf))
    torch.cuda.synchronize()
    for a, b in zip(*runs):
        assert torch.equal(a.view(torch.uint8), b.view(torch.uint8)), "two identical forward calls differ"
        assert bool(untouched(a[T:]).all()), "the forward wrote past the T rows of its output"
    out, lse = runs[0][0][:T], runs[0][1][:T]
    assert bool(torch.isfinite(out).all())
    gen = torch.Generator().manual_seed(seed + 1)
    if dout == "aligned":                      # dO ~ out: dP - Delta cancels
        do = (out.float().cpu() * 4 + 0.01 * torch.randn(T, D, generator=gen)).to(BF16).cuda()
    else:
        do = torch.randn(T, D, generator=gen).to(BF16).cuda()
    dqkv = None
    if bwd:
        druns = []
        for _ in range(2):
            df = sentinel_like((T + 3, 3 * D), BF16)
            K.attention_bwd(qkv, out, do, lse, H, dqkv=df[:T], **kw)
            druns.append(df)
        torch.cuda.synchronize()
        assert torch.equal(druns[0].view(torch.uint8), druns[1].view(torch.uint8)), "two identical backward calls differ"
        assert bool(untouched(druns[0][T:]).all()), "the backward wrote past the T rows of dqkv"
        dqkv = druns[0][:T]
        assert bool(torch.isfinite(dqkv).all())
    r = f32(1.0 / (1.0 - p)) if p else 1.0
    keep_all = K.dropout_mask((B, H, S, S), p, seed, K.SITE_ATTN) if p else None
    kvalid_all = ~pad.cuda() if pad is not None else torch.ones(B, S, dtype=torch.bool, device="cuda")
    chunk = max(1, ROWS_PER_CHUNK // S)
    keys = torch.arange(S, device="cuda")
    for b in range(B):
        rows = slice(b * S, (b + 1) * S)
        for h in range(H):
            cols = slice(h * HD, (h + 1) * HD)
            q, k, v = qkv[rows, cols], qkv[rows, D + h * HD:D + (h + 1) * HD], qkv[rows, 2 * D + h * HD:2 * D + (h + 1) * HD]
            dk = dv = s_dk = s_dv = 0.0
            for r0 in range(0, S, chunk):
                r1 = min(S, r0 + chunk)
                valid = kvalid_all[b][None, :].expand(r1 - r0, S)
                if causal:
                    valid = valid & (keys[None, :] <= torch.arange(r0, r1, device="cuda")[:, None])
                keep = keep_all[b, h, r0:r1] if p else None
                o_k, l_k = out[rows][r0:r1, cols], lse[rows][r0:r1, h]
                o, l2, b_o, b_l = attn_fwd64(q[r0:r1], k, v, valid, keep, r)
                where = f"b {b} h {h} rows {r0}.."
                within(o_k, o, b_o, f"out ({where})", "attn_fwd out")
                live = valid.any(1)
                assert bool((l_k[~live] == math.inf).all()), "lse of a row without a valid key is not +inf"
                within(l_k[live], l2[live], b_l[live], f"lse2 ({where})", "attn_fwd lse2")
                if bwd:
                    res = attn_bwd64(q[r0:r1], k, v, do[rows][r0:r1, cols], o_k, l_k, valid, keep, r)
                    within(dqkv[rows][r0:r1, cols], res["dq"], res["e_dq"], f"dQ ({where})", "attn_bwd dQ")
                    dk, dv = dk + res["dk"], dv + res["dv"]
                    s_dk, s_dv = s_dk + res["s_dk"], s_dv + res["s_dv"]
            if bwd:
                e_dk, e_dv = kv_bounds(dk, dv, s_dk, s_dv)
                within(dqkv[rows, D + h * HD:D + (h + 1) * HD], dk, e_dk, f"dK (b {b} h {h})", "attn_bwd dK")
                within(dqkv[rows, 2 * D + h * HD:2 * D + (h + 1) * HD], dv, e_dv, f"dV (b {b} h {h})", "attn_bwd dV")
    if pad is not None:                        # exact zeros of masked keys and of sequences without a valid key
        dead = pad.cuda().all(1).repeat_interleave(S)
        assert int(torch.count_nonzero(out[dead])) == 0
        assert bool((lse[dead] == math.inf).all())
        if bwd:
            assert int(torch.count_nonzero(dqkv[dead])) == 0
            assert int(torch.count_nonzero(dqkv[pad.cuda().reshape(T), D:])) == 0, "a masked key has dK / dV != 0"
    return out, lse, dqkv


TILE_SEQS = [1, 2, 31, 63, 64, 65, 127, 128, 129, 191, 192, 193, 255, 257, 300, 1000, 2048]
VARIANTS = ["plain", "drop", "mask", "mask_drop", "causal", "causal_drop"]
P_CYCLE = (0.1, 0.5, 0.9)


def _variant(variant, S, i):
    """(pad, causal, p) of a variant; the dropout probability cycles over P_CYCLE with i"""
    pad = all_masks(S, seed=S) if variant.startswith("mask") else None
    return pad, variant.startswith("causal"), P_CYCLE[i % 3] if variant.endswith("drop") else 0.0


@pytest.mark.gpu
@pytest.mark.parametrize("S", TILE_SEQS)
@pytest.mark.parametrize("HD", K.HEAD_DIMS)
@pytest.mark.parametrize("variant", VARIANTS)
def test_attention_gauss_tile_edges(variant, HD, S):
    i = TILE_SEQS.index(S)
    pad, causal, p = _variant(variant, S, i + HD // 32)
    B, H = (pad.shape[0], 1) if pad is not None else (2, 2)
    qkv = family_qkv(("gauss0.5", "gauss1.5")[i % 2], B, S, H, HD, seed=S * 3 + HD, pad=pad)
    run_attention(qkv, H, S, pad=pad, causal=causal, p=p, seed=1000 + S, dout=("randn", "aligned")[(i // 2) % 2])


FAMILIES = ["sharp", "rising", "falling", "negative", "ties_q0", "ties_k"]
FAMILY_SEQS = [65, 129, 193, 300, 1000]


@pytest.mark.gpu
@pytest.mark.parametrize("S", FAMILY_SEQS)
@pytest.mark.parametrize("HD", K.HEAD_DIMS)
@pytest.mark.parametrize("variant", ["plain", "drop", "causal"])
@pytest.mark.parametrize("family", FAMILIES)
def test_attention_input_families(family, variant, HD, S):
    i = FAMILY_SEQS.index(S)
    _, causal, p = _variant(variant, S, i + FAMILIES.index(family))
    qkv = family_qkv(family, 2, S, 2, HD, seed=S + HD + 7 * FAMILIES.index(family), causal=causal)
    run_attention(qkv, 2, S, causal=causal, p=p, seed=77 + S, dout=("randn", "aligned")[i % 2])


@pytest.mark.gpu
@pytest.mark.parametrize("p", [0.0, 0.5])
@pytest.mark.parametrize("S", FAMILY_SEQS)
@pytest.mark.parametrize("HD", K.HEAD_DIMS)
@pytest.mark.parametrize("family", ["negative", "rising"])
def test_attention_key_masks_where_a_leak_dominates(family, HD, S, p):
    """every mask family beside a masked key that would dominate its row (negative: masked keys score +34 log2 units, the
    valid ones below -34) or a maximum that arrives late (rising)"""
    pad = all_masks(S, seed=S + HD)
    qkv = family_qkv(family, pad.shape[0], S, 1, HD, seed=5 * S + HD, pad=pad)
    run_attention(qkv, 1, S, pad=pad, p=p, seed=31 + S)


@pytest.mark.gpu
@pytest.mark.parametrize("B", [1, 3])
@pytest.mark.parametrize("H", [1, 3, 16])
def test_attention_heads_and_batch(H, B):
    HD = K.HEAD_DIMS[(H + B) % 3]
    qkv = family_qkv("gauss1.5", B, 193, H, HD, seed=H * 10 + B)
    run_attention(qkv, H, 193, p=0.1 if H == 3 else 0.0, seed=H + B)


@pytest.mark.gpu
@pytest.mark.parametrize("HD", K.HEAD_DIMS)
@pytest.mark.parametrize("B,H", [(1, 1), (3, 3), (1, 17)])
def test_causal_launch_groups(B, H, HD):
    """causal CTAs run in groups of CAUSAL_GROUP = 8 (batch, head) pairs: 1 pair, 9 (a full group and a partial one of 1)
    and 17 (two full groups and one of 1)"""
    qkv = family_qkv("negative", B, 300, H, HD, seed=B * H + HD, causal=True)
    run_attention(qkv, H, 300, causal=True, p=0.5 if HD == 64 else 0.0, seed=B + H)


LONG = [(4096, 64, "plain"), (4096, 128, "plain"), (8192, 64, "plain"), (8192, 128, "plain"), (32768, 32, "plain"),
        (4096, 64, "drop"), (8192, 128, "causal")]


@pytest.mark.gpu
@pytest.mark.parametrize("S,HD,variant", LONG)
def test_attention_long_sequences(S, HD, variant):
    """one sequence and head: ceil(S / 128) = 32 .. 256 key blocks and bf16 dQ partials"""
    _, causal, p = _variant(variant, S, 0)
    qkv = family_qkv("gauss1.5" if variant == "plain" else "rising", 1, S, 1, HD, seed=S + HD)
    run_attention(qkv, 1, S, causal=causal, p=p, seed=S)


@pytest.mark.gpu
@pytest.mark.parametrize("causal", [False, True])
def test_attention_p0_is_no_dropout(causal):
    S, H, HD = 300, 2, 64
    qkv = family_qkv("gauss1.5", 2, S, H, HD, seed=3)
    do = torch.randn(2 * S, H * HD, generator=torch.Generator().manual_seed(4)).to(BF16).cuda()
    outs = []
    for dropout in (None, (0.0, 1234)):
        lse = torch.empty(2 * S, H, device="cuda")
        out = K.attention_fwd(qkv, H, lse=lse, seq_len=S, dropout=dropout, causal=causal)
        dqkv = K.attention_bwd(qkv, out, do, lse, H, seq_len=S, dropout=dropout, causal=causal)
        outs.append((out, lse, dqkv))
    torch.cuda.synchronize()
    for a, b in zip(*outs):
        assert torch.equal(a.view(torch.uint8), b.view(torch.uint8))


@pytest.mark.gpu
@pytest.mark.parametrize("causal", [False, True])
def test_attention_zero_tokens_touch_nothing(causal):
    S, H, HD = 129, 2, 32
    D = H * HD
    qkv = torch.empty(0, 3 * D, dtype=BF16, device="cuda")
    of, lf, df = sentinel_like((3, D), BF16), sentinel_like((3, H), torch.float32), sentinel_like((3, 3 * D), BF16)
    km = None if causal else torch.empty(0, (S + 31) // 32, dtype=torch.int32, device="cuda")
    kw = dict(seq_len=S, causal=causal, key_mask=km, dropout=(0.1, 5))
    K.attention_fwd(qkv, H, out=of[:0], lse=lf[:0], **kw)
    K.attention_bwd(qkv, of[:0], of[:0], lf[:0], H, dqkv=df[:0], **kw)
    torch.cuda.synchronize()
    assert bool(untouched(of).all() and untouched(lf).all() and untouched(df).all())


# ------------------------------------------------------------------ dropout element-wise kernels
EW_OPS = {"apply": (K.dropout_apply, False), "gelu": (K.gelu_dropout, False), "gelu_bwd": (K.gelu_dropout_bwd, True),
          "relu": (K.relu_dropout, False), "relu_bwd": (K.relu_dropout_bwd, True)}
SEED_HI = 0xA5C3_91E7_0000_0000   # high 32 bits set: they are the second Philox key word


def ew_inputs(rows, cols, seed):
    """values in [-10, 10] with 0, -0, the peak of gelu' (x ~ 1.4), tiny values and their neighbourhoods"""
    g = torch.Generator().manual_seed(seed)
    x = torch.rand(rows * cols, generator=g) * 20 - 10
    special = torch.tensor([0.0, -0.0, 1.4, -1.4, 1.41, 10.0, -10.0, 1e-30, -1e-30, 1e-20, 3e-38, 0.7071, -0.75, 5.0, -5.0])
    x[:special.numel()] = special
    sel = torch.rand(rows * cols, generator=g)
    x = torch.where(sel < 0.1, 1.4 + 0.1 * torch.randn(rows * cols, generator=g), x)
    x = torch.where((sel >= 0.1) & (sel < 0.15), torch.randn(rows * cols, generator=g) * 1e-25, x)
    x = torch.where((sel >= 0.15) & (sel < 0.2), torch.zeros_like(x), x)
    return x.view(rows, cols).to(BF16).cuda()


@pytest.mark.gpu
@pytest.mark.parametrize("site,p,seed", [(1, 0.0, SEED_HI | 7), (2, 0.1, SEED_HI | 99), (3, 0.5, 12345)])
@pytest.mark.parametrize("shape", [(16, 16), (48, 1040), (65552, 32)])
@pytest.mark.parametrize("op", list(EW_OPS))
def test_dropout_elementwise(op, shape, site, p, seed):
    fn, two = EW_OPS[op]
    if two:                                    # x = dg, f = the forward's input
        x = torch.randn(*shape, generator=torch.Generator().manual_seed(site)).to(BF16).cuda()
        f = ew_inputs(*shape, seed=site + shape[1] + 1)
    else:
        x, f = ew_inputs(*shape, seed=site + shape[1]), None
    outs = []
    for _ in range(2):
        out = sentinel_like(shape, BF16)
        fn(x, f, p, seed, site, out=out) if two else fn(x, p, seed, site, out=out)
        outs.append(out)
    torch.cuda.synchronize()
    assert torch.equal(outs[0].view(torch.uint8), outs[1].view(torch.uint8)), "two identical calls differ"
    keep = K.dropout_mask(shape, p, seed, site)
    assert bool(keep.all()) if p == 0 else 0 < int(keep.sum()) < keep.numel()
    ref, bound = dropout_ew64(op, x, f, keep, f32(1.0 / (1.0 - p)))
    within(outs[0], ref, bound, op, "dropout " + op)
    assert bool((outs[0][~keep] == 0).all()), "a dropped element is not 0"


@pytest.mark.gpu
@pytest.mark.parametrize("shape", [(16, 24), (24, 16), (8, 8)])
def test_dropout_elementwise_refuses_shapes_off_16_before_launch(shape):
    from lah_b200.ops.native import NativeError
    x = torch.randn(*shape, device="cuda").to(BF16)
    for op, (fn, two) in EW_OPS.items():
        out = sentinel_like(shape, BF16)
        with pytest.raises(NativeError):
            fn(x, x, 0.1, 3, 2, out=out) if two else fn(x, 0.1, 3, 2, out=out)
        torch.cuda.synchronize()
        assert bool(untouched(out).all()), op
