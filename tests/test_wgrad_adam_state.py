"""GPU test of the fused wgrad + Adam kernel (csrc/small_m.cu) on the paths the AMSGrad check does not take: plain Adam
(amsgrad=False: no vmax traffic at all), shadowed groups (`skip`), and a hot group whose many k-blocks interleave with the
state chunks it streams."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def test_wgrad_adam_plain_adam_skip_and_hot_group():
    import lah_b200  # noqa
    from lah_b200.ops import kernels as K
    from tools.gpu_small_check import make_groups

    torch.manual_seed(4)
    rows_list = [16, 0, 300, 33, 5]
    skipped = {3}
    G, N, Kd = len(rows_list), 256, 384
    off, rows, total = make_groups(rows_list)
    dy = torch.zeros(total, N, device="cuda", dtype=torch.bfloat16)
    x = torch.zeros(total, Kd, device="cuda", dtype=torch.bfloat16)
    for o, r in zip(off.tolist(), rows_list):
        dy[o:o + r] = (torch.randn(r, N, device="cuda") * 0.3).to(torch.bfloat16)
        x[o:o + r] = torch.randn(r, Kd, device="cuda").to(torch.bfloat16)
    p = torch.randn(G, N, Kd, device="cuda")
    m = torch.randn(G, N, Kd, device="cuda") * 0.01
    v = 1e-3 + torch.rand(G, N, Kd, device="cuda") * 0.01   # bounded away from 0: the update stays well conditioned
    vmax = torch.full((G, N, Kd), 7.0, device="cuda")
    pb = torch.zeros(G, N, Kd, device="cuda", dtype=torch.bfloat16)
    p0, m0, v0 = p.clone(), m.clone(), v.clone()
    skip = torch.full((G, 2), -1, dtype=torch.int32, device="cuda")
    for g in skipped:
        skip[g, 0] = 0
    step = torch.full((G,), 3, dtype=torch.int32, device="cuda")
    lr, b1, b2, eps = 1e-2, 0.9, 0.999, 1e-8
    K.wgrad_adam(dy, x, off, rows, p=p, m=m, v=v, vmax=vmax, p_bf16=pb, step=step, skip=skip, lr=lr, betas=(b1, b2),
                 eps=eps, amsgrad=False)
    torch.cuda.synchronize()

    assert torch.equal(vmax, torch.full_like(vmax, 7.0)), "amsgrad=False must not touch vmax"
    for g, (o, r) in enumerate(zip(off.tolist(), rows_list)):
        if r == 0 or g in skipped:
            assert torch.equal(p[g], p0[g]) and torch.equal(m[g], m0[g]) and torch.equal(v[g], v0[g]), g
            assert not pb[g].any(), g
            continue
        grad = dy[o:o + r].float().t() @ x[o:o + r].float()
        m_ref = m0[g] + (1 - b1) * (grad - m0[g])
        v_ref = v0[g] * b2 + (1 - b2) * grad * grad
        p_ref = p0[g] - lr / (1 - b1 ** 3) * m_ref / (v_ref.sqrt() / (1 - b2 ** 3) ** 0.5 + eps)
        assert ((m[g] - m_ref).norm() / m_ref.norm()).item() < 2e-3, g
        assert ((v[g] - v_ref).norm() / v_ref.norm()).item() < 2e-3, g
        assert (p[g] - p_ref).abs().max().item() < 1e-4, g
        assert torch.equal(pb[g], p[g].to(torch.bfloat16)), g
